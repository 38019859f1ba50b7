"""Batch handles (fluid_create_batch) at the member counts they are benchmarked and sized for, B = 256 to 65535, member
by member against the oracle.

One oracle run per member is out of reach at B = 65535, so members share a few inputs in a pattern that exposes any
mix-up between members (plan()):
* member m holds data set m mod 7 (DATA: rand_fields, nasty_fields, exp_tiled over the whole fp32 range, far_field,
  tiny-divergence sites of jacobi_tb_model.cases, rand_fields with a second seed, and exp_tiled over 2^-20 .. 2^20) and per-member values VALUES[(m + k) mod 3] in step k (CURL, PRESSURE,
  both dissipations, SPLAT_RADIUS and dt; one row per dissipation at 1e20, where div_n_by divides by IEEE);
* a few unique members hold data and values of their own: 0, 1, B - 2, B - 1 and the members a case names.
A combo is one (data set, values) pair, or one unique member.  The period 21 is odd, so neighbouring members always
differ and m, m + 2^k never share a data set: a kernel that reads the wrong member, masks a member index to a power
of two or drops the high bits of an offset leaves some member unequal to its combo.

Each combo is one oracle.OracleSim.  Every field of every member is compared on the GPU with its combo's arrays,
uploaded once: equal bits, or NaN on both sides where the combo's arrays hold NaN.  Splats: every member takes its
combo's two records, the first through the host path and the second through the device path, each call in shuffled
member order; a member of each combo is read back, checked inside splat_model's interval and adopted into its
combo's oracle state, and the comparison then holds every member of the combo to its bits.  Draws: one ordinary
handle per combo, launching what its draws launch.  After every step the launch counters equal an ordinary handle's,
and the exact-tail counter has grown where some combo's step surely runs the exact tail.  Only that growth is asserted:
every step holds members of the special-value set, whose non-finite divergence sends streams through the exact tail,
so no step here may leave the counter where it was.

one_chunk: B = 16 * SMs + 1 streams every member as one chunk over its whole 128-row height in every streaming
kernel, whatever the occupancy the library reads.  At W = 128 (sm_90: at most 64 resident warps and 32 CTAs per SM):
* cvd_stream_kernel: CVD2_VALID = 120 output columns per window gives 2 windows per member; with at most 64 resident
  warps per SM, stream_args' chunks = floor(SMs * occ / (2 B)) <= floor(64 SMs / (32 SMs + 2)) = 1.
* gradient_stream_kernel: 128 columns per window gives 1 window and warps_per_sm = 32: floor(32 SMs / B) = 1 once
  B > 32 SMs / 2.
* jacobi_tb_kernel<K>: TB<K>::VALID = 128 - 2 * HX, HX = (K + 2) / 4 * 4, gives 2 windows per member at K > 1 and 1
  at K = 1; one-warp CTAs, at most 32 resident per SM: tb_rows' chunks = max(1, floor(32 SMs / (windows * B))) = 1
  once B > 8 SMs (K > 1) or 16 SMs (K = 1), and its rows (at least 4K, rounded to the unroll) are capped at 128.
"""
import numpy as np
import pytest

import splat_model as SM
from display_model import ALL3, BLOOM, SHADING, SUNRAYS
from jacobi_tb_model import BIG_IN, TINY, cases
from conftest import golden
from sim_harness import exp_tiled, far_field, jacobi_plan, make, nasty_fields, nasty_records, rand_fields
from sim_harness import pkg, torch  # noqa: F401 -- fixtures

F = np.float32
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
MAX_MEMBERS = 65535                      # FLUID_MAX_MEMBERS, the grid-z limit
PERIOD_DATA, PERIOD_VALUES = 7, 3
BIG_DISS = 1e20                          # 1 + diss * dt above 2^60: div_n_by divides by IEEE in every cell
VALUES = [
    dict(CURL=30.0, PRESSURE=0.8, VELOCITY_DISSIPATION=0.2, DENSITY_DISSIPATION=1.0, SPLAT_RADIUS=0.25),
    dict(CURL=0.0, PRESSURE=0.0, VELOCITY_DISSIPATION=BIG_DISS, DENSITY_DISSIPATION=0.0, SPLAT_RADIUS=0.01),
    dict(CURL=1e4, PRESSURE=2.0, VELOCITY_DISSIPATION=4.0, DENSITY_DISSIPATION=BIG_DISS, SPLAT_RADIUS=1.0),
]
DTS = [0.016666, 0.05, 0.1]
DATA = ("rand", "nasty", "exp_tiled", "far_field", "tiny", "rand2", "exp_narrow")
CHUNK_BYTES = 1 << 30                    # a field is read back at most this many bytes at a time


def one_chunk_members(sms):
    return 16 * sms + 1


# name: (sizes, PRESSURE_ITERATIONS, B (None: one_chunk_members of the device), the unique members past 0, 1, B-2, B-1,
# steps)
CASES = {
    "readme": ((128, 128, 1024, 1024), 20, 256, (), 3),
    "sweep50": ((256, 256, 256, 256), 50, 256, (), 2),
    "past_4gib": ((128, 128, 1024, 1024), 20, 300, (255, 256), 2),    # member 256's dye starts 2^32 B into its slot
    "one_chunk": ((128, 128, 128, 128), 20, None, (), 2),
    "grid_z_limit": ((128, 2, 128, 2), 20, MAX_MEMBERS, (), 2),
}
THUMBS = ((128, 128, 256, 256), (256, 256), 256)         # sizes, canvas, B: bench_batch_draw's thumbnail workload
SUBSETS = {"past_4gib": [299, 256, 255, 0], "grid_z_limit": [65534, 0, 32767]}
PLANNED_B = {"readme": 256, "sweep50": 256, "past_4gib": 300, "one_chunk": one_chunk_members(132),
             "grid_z_limit": MAX_MEMBERS, "thumbnails": 256}


# ---- the combo planner (CPU) ---------------------------------------------------------------------------------
def plan(B, extra=()):
    """(combo of each member (int array of B), uniques): combo (m mod 7) * 3 + (m mod 3) for an ordinary member,
    21 + k for uniques[k]."""
    uniques = sorted({0, 1, B - 2, B - 1, *extra} & set(range(B)))
    m = np.arange(B)
    combo = (m % PERIOD_DATA) * PERIOD_VALUES + m % PERIOD_VALUES
    for k, u in enumerate(uniques):
        combo[u] = PERIOD_DATA * PERIOD_VALUES + k
    return combo, uniques


def data_set(combo):
    return combo // PERIOD_VALUES if combo < PERIOD_DATA * PERIOD_VALUES else None


def values_row(combo, k):
    return (combo + k) % PERIOD_VALUES


def unique_values(u, k):
    """The values and dt of the u-th unique member in step k."""
    return (dict(CURL=5.0 + 7 * u + k, PRESSURE=0.3 + 0.1 * u, VELOCITY_DISSIPATION=0.5 + u,
                 DENSITY_DISSIPATION=0.25 * (u + k), SPLAT_RADIUS=0.05 * (u + 1)), 0.01 + 0.003 * u + 0.002 * k)


def combo_values(combo, k):
    n = PERIOD_DATA * PERIOD_VALUES
    if combo >= n:
        return unique_values(combo - n, k)
    r = values_row(combo, k)
    return VALUES[r], DTS[r]


def stream_chunks(sms, B, windows, warps_per_sm):
    """stream_args / tb_rows: warp streams per member and window of one wave of `warps_per_sm` warps per SM."""
    return max(1, sms * warps_per_sm // (windows * B))


def tb_windows(K, W=128):
    hx = (K + 2) // 4 * 4
    return -(-W // (128 - 2 * hx))


@pytest.mark.parametrize("name", list(PLANNED_B))
def test_plan(name):
    B = PLANNED_B[name]
    extra = CASES[name][3] if name in CASES else ()
    combo, uniques = plan(B, extra)
    n = PERIOD_DATA * PERIOD_VALUES
    assert uniques == sorted({0, 1, B - 2, B - 1, *extra})
    assert np.array_equal(np.flatnonzero(combo >= n), uniques)
    assert len(set(combo[uniques].tolist())) == len(uniques)
    assert (combo[1:] != combo[:-1]).all()
    ds = np.array([-1 - c if data_set(c) is None else data_set(c) for c in combo])
    for k in range(17):
        s = 1 << k
        if s < B:
            assert (ds[s:] != ds[:-s]).all(), k
    ordinary = [c for c in combo if c < n]
    assert {data_set(c) for c in ordinary} == set(range(PERIOD_DATA))
    for k in range(3):
        assert {values_row(c, k) for c in ordinary} == set(range(PERIOD_VALUES))
    assert any(v["VELOCITY_DISSIPATION"] >= BIG_DISS for v in VALUES)
    assert any(v["DENSITY_DISSIPATION"] >= BIG_DISS for v in VALUES)


@pytest.mark.parametrize("sms", [114, 132])
def test_one_chunk_bound(sms):
    """The docstring's derivation: at B = 16 SMs + 1 every streaming kernel cuts a 128-row member into one chunk at
    the per-SM maxima of sm_90, and at B = 16 SMs the cvd kernel would not."""
    B = one_chunk_members(sms)
    assert tb_windows(1) == 1 and all(tb_windows(K) == 2 for K in range(2, 14))
    assert stream_chunks(sms, B, 2, 64) == 1                    # cvd: 2 windows of CVD2_VALID = 120
    assert stream_chunks(sms, B, 1, 32) == 1                    # gradient: one 128-column window
    for K in range(1, 14):
        assert stream_chunks(sms, B, tb_windows(K), 32) == 1, K
    assert stream_chunks(sms, B - 1, 2, 64) == 2
    assert B <= MAX_MEMBERS


# ---- data -----------------------------------------------------------------------------------------------------
def member_data(O, W, H, Wd, Hd, combo, seed):
    """velocity, dye, pressure of a combo."""
    d = data_set(combo)
    s = seed + 97 * combo
    if d is None or d in (0, 5) or (d == 4 and not cases(W, H)):
        return rand_fields(W, H, Wd, Hd, s)
    if d == 1:
        return nasty_fields(W, H, Wd, Hd, s)
    if d == 2:
        return exp_tiled((H, W, 2), s), exp_tiled((Hd, Wd, 4), s + 2, tile=(4, 8)), exp_tiled((H, W), s + 1)
    if d == 3:
        v = far_field(O, W, H, 2, s)
        return v, far_field(O, Wd, Hd, 4, s + 1), np.ascontiguousarray(v[..., 0] * F(0.01))
    if d == 4:
        c = cases(W, H)[0]
        return c["v"].copy(), far_field(O, Wd, Hd, 4, s), c["p0"].copy()
    return (exp_tiled((H, W, 2), s, lo=-20, hi=20), exp_tiled((Hd, Wd, 4), s + 2, lo=-10, hi=10),
            exp_tiled((H, W), s + 1, lo=-20, hi=20))


def surely_exact(ref, p_cleared):
    """Whether the blocked solve of a combo's step surely runs the exact tail somewhere: its divergence holds a tiny
    value (0 < |d| < 2^-123), or the cleared pressure or the divergence, level-0 inputs of the first launch, reach
    BIG_IN."""
    d = ref.divergence
    if ((d != 0) & (np.abs(d) < F(TINY))).any():
        return True
    with np.errstate(invalid="ignore", over="ignore"):
        pm = float(np.nanmax(np.abs(p_cleared), initial=0.0))
        dm = float(np.nanmax(np.abs(d), initial=0.0))
    return max(pm, dm) >= BIG_IN


# ---- the GPU side ---------------------------------------------------------------------------------------------
class Expected:
    """Each combo's arrays of every field on the GPU, and the members' combos."""

    def __init__(self, torch, combo):
        self.torch = torch
        self.combo = np.asarray(combo)
        self.idx = torch.from_numpy(self.combo.astype(np.int64)).cuda()
        self.tabs = {}
        self.nan_ok = {}

    def set(self, name, arrays):
        """arrays: one array per combo."""
        t = self.torch
        a = np.stack([np.ascontiguousarray(x, F).reshape(-1) for x in arrays])
        self.tabs[name] = t.from_numpy(a).cuda()
        self.nan_ok[name] = t.from_numpy(np.isnan(a).any(axis=1)).cuda()

    def check(self, b, name, what):
        """Every member of field `name` against its combo's array, on the GPU, in chunks of CHUNK_BYTES."""
        t = self.torch
        tab, nan_ok = self.tabs[name], self.nan_ok[name]
        per = tab.shape[1]
        B = len(self.combo)
        chunk = max(1, min(B, CHUNK_BYTES // (4 * per)))
        buf = t.empty(chunk * per, dtype=t.float32, device="cuda")
        for m0 in range(0, B, chunk):
            n = min(chunk, B - m0)
            out = buf[:n * per]
            if n == B:
                b.readField(name, out=out)
            else:
                b.readField(name, out=out, members=list(range(m0, m0 + n)))
            got = out.view(n, per)
            ci = self.idx[m0:m0 + n]
            want = tab[ci]
            ok = got.view(t.int32) == want.view(t.int32)
            ok |= got.isnan() & want.isnan() & nan_ok[ci][:, None]
            if not bool(ok.all()):
                bad = (~ok).nonzero()[0].tolist()
                m = m0 + bad[0]
                c = int(self.combo[m])
                ds = data_set(c)
                raise AssertionError(f"{what}: member {m}, field {name}, combo {c} (data set "
                                     f"{'unique' if ds is None else DATA[ds]}), flat index {bad[1]}: got {float(got[bad[0], bad[1]])}, "
                                     f"want {float(want[bad[0], bad[1]])}; {int((~ok).sum())} elements differ")
            del got, want, ok
        del buf

    def check_all(self, b, what, fields=FIELDS):
        for name in fields:
            self.check(b, name, what)


def batch(pkg, B, W, H, Wd, Hd, flags=0, **cfg):
    c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}
    c.update(cfg)
    b = pkg.FluidBatch(B, c, canvas_width=W, canvas_height=H, sizes=(W, H, Wd, Hd), flags=flags)
    assert b.members == B
    return b


def write_members(torch, b, combo, arrays, name):
    """Writes field `name` of every member from the combos' arrays, assembled on the GPU: the whole field when it
    fits in CHUNK_BYTES, else members in chunks (fluid_write_members)."""
    tab = torch.from_numpy(np.stack([np.ascontiguousarray(x, F).reshape(-1) for x in arrays])).cuda()
    per = tab.shape[1]
    B = len(combo)
    idx = torch.from_numpy(np.asarray(combo, np.int64)).cuda()
    chunk = max(1, min(B, CHUNK_BYTES // (4 * per)))
    for m0 in range(0, B, chunk):
        n = min(chunk, B - m0)
        src = tab[idx[m0:m0 + n]].reshape(-1).contiguous()
        if n == B:
            b.writeField(name, src)
        else:
            b.writeField(name, src, members=list(range(m0, m0 + n)))
        del src
    del tab


def set_values(b, combo, uniques, k):
    """member_config and the dts of step k; returns the dts."""
    B = len(combo)
    dts = np.empty(B, F)
    rows = (combo + k) % PERIOD_VALUES
    for r in range(PERIOD_VALUES):
        dts[rows == r] = DTS[r]
    cfgs = [dict(VALUES[r]) for r in range(PERIOD_VALUES)]
    b.member_config = [dict(cfgs[r]) for r in rows.tolist()]
    for u in uniques:
        vals, dt = combo_values(int(combo[u]), k)
        b.member_config[u] = dict(vals)
        dts[u] = dt
    return dts


def growth(s, stats, fn):
    n0 = {k: s.stat(k) for k in stats}
    fn()
    return {k: s.stat(k) - n0[k] for k in stats}


STATS = ("cvd_stream_launches", "gradient_stream_launches", "advect4_launches", "jacobi_launches", "launches",
         "jacobi_exact_streams")


def run_case(pkg, O, torch, name, graph=True):
    (W, H, Wd, Hd), iters, B, extra, steps = CASES[name]
    if B is None:
        B = one_chunk_members(torch.cuda.get_device_properties(0).multi_processor_count)
    flags = 0 if graph else pkg.FLAG_NO_GRAPH
    combo, uniques = plan(B, extra)
    ncombo = int(combo.max()) + 1
    reps = [int(np.flatnonzero(combo == c)[0]) for c in range(ncombo)]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    b = batch(pkg, B, W, H, Wd, Hd, flags=flags, PRESSURE_ITERATIONS=iters)
    torch.cuda.synchronize()
    print(f"{name}: B = {B}, device memory taken by the handle {(free0 - torch.cuda.mem_get_info()[0]) / 2**30:.2f} GiB")
    twin = make(pkg, W, H, Wd, Hd, flags=flags, PRESSURE_ITERATIONS=iters)
    E = Expected(torch, combo)

    refs = []
    for c in range(ncombo):
        vals, _ = combo_values(c, 0)
        ref = O.OracleSim(W, H, Wd, Hd, PRESSURE_ITERATIONS=iters, **vals)
        ref.velocity, ref.dye, ref.pressure = member_data(O, W, H, Wd, Hd, c, seed=W + Hd)
        refs.append(ref)
    for k, f in enumerate(("velocity", "dye", "pressure")):
        write_members(torch, b, combo, [getattr(r, f) for r in refs], f)
    for f in FIELDS:
        E.set(f, [getattr(r, f) for r in refs])
    E.check_all(b, f"{name}: written")

    # splats: two records per member, one call through each path, members in shuffled order
    set_values(b, combo, uniques, 0)
    recs = [nasty_records(2, 1000 + c) for c in range(ncombo)]
    rng = np.random.default_rng(B)
    aspect = SM.aspect_of(W, H)
    before = {c: (refs[c].velocity.copy(), refs[c].dye.copy()) for c in range(ncombo)}
    for r in range(2):
        order = rng.permutation(B).astype(np.int32)
        rec = np.stack([recs[c][r] for c in combo[order]])
        if r == 0:
            n0 = b.stat("launches")
            b.splats(order, rec)
            if B > 64 * 1000:
                assert b.stat("launches") - n0 > 1000
        else:
            b.splats(torch.from_numpy(order).cuda(), torch.from_numpy(rec).cuda())
    for c in range(ncombo):
        m = reps[c]
        rad = SM.radius_of(combo_values(c, 0)[0]["SPLAT_RADIUS"], W, H)
        got = {}
        for f, base in zip(("velocity", "dye"), before[c]):
            got[f] = b.readField(f, members=[m])[0]
            with np.errstate(invalid="ignore", over="ignore"):
                lo, hi = SM.splat_interval(base, recs[c], aspect, rad)
            n_bad, first = SM.check_splat(got[f], lo, hi)
            assert n_bad == 0, (name, "splat", m, c, f, first)
        refs[c].velocity, refs[c].dye = got["velocity"].copy(), got["dye"].copy()
    E.set("velocity", [r.velocity for r in refs])
    E.set("dye", [r.dye for r in refs])
    E.check_all(b, f"{name}: splats", ("velocity", "dye"))

    # steps with per-member values and dts that change between steps
    launches = len(jacobi_plan(W, H, False, iters))
    for k in range(steps):
        dts = set_values(b, combo, uniques, k)
        exact = False
        for c, ref in enumerate(refs):
            vals, dt = combo_values(c, k)
            for key, v in vals.items():
                setattr(ref, key, v)
            with np.errstate(all="ignore"):
                p_cleared = O.clear(ref.pressure, ref.PRESSURE)
                ref.step(dt)
            exact |= surely_exact(ref, p_cleared)
        n = growth(b, STATS, lambda: b.step(dts))
        t = growth(twin, ("launches",), lambda: twin.step(DTS[0]))
        assert (n["cvd_stream_launches"], n["gradient_stream_launches"], n["advect4_launches"],
                n["jacobi_launches"]) == (1, 1, 2, launches), (name, k, n)
        assert n["launches"] == t["launches"], (name, k, n, t)
        assert exact and n["jacobi_exact_streams"] > 0, (name, k, n)
        for f in FIELDS:
            E.set(f, [getattr(r, f) for r in refs])
        E.check_all(b, f"{name}: step {k}")
    assert b.stat("graph_launches") == (steps if graph else 0)
    twin.close()
    return b, E, refs, combo


def subset_calls(torch, b, E, refs, combo, members):
    """Member-subset reads and writes, host and device, with 16- and 4-byte-aligned buffers, and reset, on `members`;
    after each, every member of the batch against its combo."""
    n = len(members)
    for f in FIELDS:
        per = E.tabs[f].shape[1]
        want = E.tabs[f][E.idx[members]]
        same = lambda got: bool(((got.view(torch.int32) == want.view(torch.int32)) | (got.isnan() & want.isnan())).all())  # noqa: E731
        host = b.readField(f, members=members)
        assert same(torch.from_numpy(np.ascontiguousarray(host).reshape(n, per)).cuda()), (f, "host read")
        for off in (0, 1):                                 # 16-byte and 4-byte aligned device buffers
            buf = torch.full((n * per + 4,), 7.25, dtype=torch.float32, device="cuda")
            out = buf[off:off + n * per]
            b.readField(f, out=out, members=members)
            assert same(out.view(n, per)), (f, "device read", off)
            assert bool((buf[:off] == 7.25).all()) and bool((buf[off + n * per:] == 7.25).all()), (f, off)

    def expect(state):
        E.combo = state
        E.idx = torch.from_numpy(state.astype(np.int64)).cuda()

    # member members[k] takes the state of members[k + 1] through the host path, its own again from a 4-byte-aligned
    # device buffer, and members[k + 1]'s from a 16-byte-aligned one
    rot = members[1:] + members[:1]
    rotated = combo.copy()
    rotated[members] = combo[rot]
    for f in FIELDS:
        b.writeField(f, b.readField(f, members=rot), members=members)
    expect(rotated)
    E.check_all(b, "host member writes")
    for off, state in ((1, combo), (0, rotated)):
        for f in FIELDS:
            per = E.tabs[f].shape[1]
            buf = torch.empty(n * per + 4, dtype=torch.float32, device="cuda")
            src = buf[off:off + n * per]
            src.copy_(E.tabs[f][torch.from_numpy(state[members].astype(np.int64)).cuda()].reshape(-1))
            b.writeField(f, src, members=members)
        expect(state)
        E.check_all(b, f"device member writes, buffer offset {4 * off} bytes")
    # reset: the listed members back to zero fields and dye alpha 1
    b.reset(members)
    z = len(refs)
    zeroed = rotated.copy()
    zeroed[members] = z
    for f in FIELDS:
        a = np.zeros_like(getattr(refs[0], f))
        if f == "dye":
            a[..., 3] = 1.0
        E.tabs[f] = torch.cat([E.tabs[f], torch.from_numpy(a.reshape(1, -1)).cuda()])
        E.nan_ok[f] = torch.cat([E.nan_ok[f], torch.zeros(1, dtype=torch.bool, device="cuda")])
    expect(zeroed)
    E.check_all(b, "reset")


@pytest.mark.gpu
@pytest.mark.parametrize("name,graph", [("readme", True), ("sweep50", True), ("past_4gib", True), ("one_chunk", True),
                                        ("one_chunk", False), ("grid_z_limit", True)])
def test_steps(pkg, oracle, torch, name, graph):
    """Writes, splats through both paths and steps with per-member values and dts, every member of every field
    against its combo's oracle state after each call; past_4gib and grid_z_limit then member-subset reads, writes and
    reset."""
    b, E, refs, combo = run_case(pkg, oracle, torch, name, graph)
    if name in SUBSETS:
        subset_calls(torch, b, E, refs, combo, SUBSETS[name])
    b.close()
    torch.cuda.empty_cache()


# ---- draws ------------------------------------------------------------------------------------------------------
LOOKS = [dict(BLOOM_INTENSITY=0.8, BLOOM_THRESHOLD=0.6, BLOOM_SOFT_KNEE=0.7, SUNRAYS_WEIGHT=1.0,
              BACK_COLOR={"r": 10, "g": 20, "b": 30}, TRANSPARENT=False),
         dict(BLOOM_INTENSITY=1.3, BLOOM_THRESHOLD=0.05, BLOOM_SOFT_KNEE=0.7, SUNRAYS_WEIGHT=0.6,
              BACK_COLOR={"r": 0, "g": 255, "b": 0}, TRANSPARENT=True),
         dict(BLOOM_INTENSITY=0.1, BLOOM_THRESHOLD=0.0, BLOOM_SOFT_KNEE=0.0, SUNRAYS_WEIGHT=4.0,
              BACK_COLOR={"r": 255, "g": 0, "b": 255}, TRANSPARENT=False)]


def unique_look(u):
    return dict(BLOOM_INTENSITY=0.5 + 0.2 * u, BLOOM_THRESHOLD=0.1 * u, BLOOM_SOFT_KNEE=0.3, SUNRAYS_WEIGHT=0.5 + u,
                BACK_COLOR={"r": 40 * u, "g": 3, "b": 250 - 40 * u}, TRANSPARENT=u % 2 == 1)


def set_keywords(s, kw):
    s.config.update(SHADING=bool(kw & SHADING), BLOOM=bool(kw & BLOOM), SUNRAYS=bool(kw & SUNRAYS))


def combo_look(c):
    n = PERIOD_DATA * PERIOD_VALUES
    return unique_look(c - n) if c >= n else LOOKS[c % PERIOD_VALUES]


@pytest.mark.gpu
def test_thumbnails(pkg, oracle, torch):
    """bench_batch_draw's thumbnail workload: 256 members of 128^2 / 256^2 on a 256^2 canvas, SHADING, BLOOM and
    SUNRAYS with the default post-FX geometry (a 256^2 bloom FBO and its whole pyramid, a 196^2 sunrays target), canvas
    and capture into device tensors, a look per image cycled with period 3: every image equals byte for byte its
    combo's ordinary handle's, and each batch draw launches what one draw of the ordinary handle launches, the first
    (post-FX targets made on first use) as its first and a second as its last."""
    O = oracle
    (W, H, Wd, Hd), canvas, B = THUMBS
    cfg = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd), "CAPTURE_RESOLUTION": 256}
    dither = golden("postfx_64_to_128")["dither"].astype(F)
    combo, _ = plan(B)
    ncombo = int(combo.max()) + 1
    b = pkg.FluidBatch(B, dict(cfg), canvas_width=canvas[0], canvas_height=canvas[1], sizes=(W, H, Wd, Hd))
    b.dithering = dither
    for m in range(B):
        b.member_config[m].update(combo_look(int(combo[m])))
    dyes = [member_data(O, W, H, Wd, Hd, c, seed=7)[1] for c in range(ncombo)]
    write_members(torch, b, combo, dyes, "dye")
    set_keywords(b, ALL3)
    idx = torch.from_numpy(combo.astype(np.int64)).cuda()
    t = pkg.FluidSimulation(dict(cfg), canvas_width=canvas[0], canvas_height=canvas[1], sizes=(W, H, Wd, Hd))
    t.dithering = dither
    base = dict(t.config)
    assert (b.config["BLOOM_RESOLUTION"], b.config["SUNRAYS_RESOLUTION"]) == (256, 196)
    draw = lambda s, call, out=None: s.render_canvas(out=out) if call == "canvas" else s.captureScreenshot(out=out)  # noqa: E731
    for call in ("canvas", "capture"):
        want, t_launches = [], []
        for c in range(ncombo):
            t.writeField("dye", dyes[c])
            t.config.clear()
            t.config.update(base)
            t.config.update(combo_look(c))
            set_keywords(t, ALL3)
            n0 = t.launch_count()
            with np.errstate(all="ignore"):
                want.append(draw(t, call))
            t_launches.append(t.launch_count() - n0)
        want = torch.from_numpy(np.stack(want)).cuda()
        for r, t_n in enumerate((t_launches[0], t_launches[-1])):
            got = torch.full((B,) + tuple(want.shape[1:]), 0xA5, dtype=torch.uint8, device="cuda")
            n0 = b.launch_count()
            with np.errstate(all="ignore"):
                assert draw(b, call, got) is got
            assert b.launch_count() - n0 == t_n, (call, r, b.launch_count() - n0, t_launches)
            ok = (got == want[idx]).reshape(B, -1).all(dim=1)
            if not bool(ok.all()):
                m = int((~ok).nonzero()[0, 0])
                raise AssertionError(f"{call}, draw {r}: image {m} (combo {int(combo[m])}) differs from its ordinary "
                                     f"handle's")
    t.close()
    b.close()
