"""Batch handles (fluid_create_batch): B simulations stepped, splatted, read and written together.  The oracle is
one ordinary handle per member, its twin, given that member's inputs: after every call each field of each member
equals its twin bit for bit.  Twins at small sizes run the tiled passes and the one-sweep Jacobi kernel, which
are checked against the CPU oracle elsewhere; the batch always runs the row-streaming, blocked and 4-cell
kernels with a member axis, so the comparison pins those against the checked ones."""
import ctypes as C

import numpy as np
import pytest

import arena_model as A
import splat_model as SM
from sim_harness import (Arena, _DeviceBytes, address_range, delta, exp_tiled, make, nasty_records, near_max_patch, pkg, rand_fields,  # noqa: F401
                         same_bits, torch)

pytestmark = pytest.mark.gpu

FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
DEFAULT = (128, 128, 1024, 1024)
INVALID = -1


def batch(pkg, B, W, H, Wd, Hd, flags=0, jb=0, **cfg):
    c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}
    c.update(cfg)
    b = pkg.FluidBatch(B, c, canvas_width=W, canvas_height=H, sizes=(W, H, Wd, Hd), flags=flags, jacobi_block=jb)
    assert b.members == B
    return b


def pair(pkg, B, size, flags=0, jb=0, **cfg):
    """A batch of B members and its B twins, all with the same config."""
    return batch(pkg, B, *size, flags=flags, jb=jb, **cfg), [make(pkg, *size, flags=flags, jb=jb, **cfg) for _ in range(B)]


def assert_twins(b, twins, what, fields=FIELDS):
    for name in fields:
        got = b.readField(name)
        for m, t in enumerate(twins):
            assert same_bits(got[m], t.readField(name)), (what, name, m)


def seed(b, twins, size, salt=0):
    """Different written fields in every member."""
    W, H, Wd, Hd = size
    data = [rand_fields(W, H, Wd, Hd, 1000 * salt + m) for m in range(len(twins))]
    for k, name in enumerate(("velocity", "dye", "pressure")):
        b.writeField(name, np.stack([d[k] for d in data]))
        for t, d in zip(twins, data):
            t.writeField(name, d[k])


def member_records(B, seed_):
    """0..3 records per member, from nasty_records: (members, records) in a shuffled call order."""
    rng = np.random.default_rng(seed_)
    counts = rng.integers(0, 4, B)
    members = np.repeat(np.arange(B, dtype=np.int32), counts)
    recs = nasty_records(len(members), seed_)
    order = rng.permutation(len(members))
    return members[order], recs[order]


def splat_both(b, twins, members, recs):
    b.splats(members, recs)
    for m, t in enumerate(twins):
        own = recs[members == m]
        if len(own):
            t.splats(own)


class BatchArena(Arena):
    """The guarded arena of a batch handle.  Its slots hold the B members back to back, which is the layout
    of an ordinary handle whose grids are the members stacked as rows: W x B*H and Wd x B*Hd."""

    def __init__(self, torch, s, members):
        self.members = members
        super().__init__(torch, s)

    def attach(self):
        s, B = self.s, self.members
        (W, H), (Wd, Hd) = s._dims("velocity")[:2], s._dims("dye")[:2]
        self.L = L = A.layout(W, B * H, Wd, B * Hd)
        s.sync()
        self.base, size = address_range(s.device_ptr("velocity"))
        assert size >= L.bytes, (size, L.bytes)
        assert self.base == s.device_ptr("velocity") - L.v[self.parity()["velocity"]]
        self.t = self.torch.as_tensor(_DeviceBytes(self.base, L.bytes), device="cuda")

    def member_range(self, field, side, m, par):
        """[lo, hi) of member m's part of `field`.read / .write."""
        lo, hi = A.extent_range(self.L, f"{field}.{side}", par)
        n = (hi - lo) // self.members
        return lo + m * n, lo + (m + 1) * n


def close(b, twins):
    b.close()
    for t in twins:
        t.close()


# (B, size, PRESSURE_ITERATIONS, JACOBI_BLOCK, graph): the default size, SAME dye, a 4:1 grid, the smallest height,
# depth-13 launches at 50 iterations, depth 1 (twins run the one-sweep kernel), 10 and 13, graph and NO_GRAPH
TWIN_CASES = [
    (1, DEFAULT, 20, 0, True),
    (2, DEFAULT, 20, 0, False),
    (5, (256, 256, 256, 256), 50, 0, True),
    (5, (512, 128, 1024, 256), 20, 10, False),
    (2, (128, 2, 128, 2), 20, 0, True),
    (2, (128, 2, 256, 4), 50, 13, False),
    (5, DEFAULT, 20, 1, True),
    (2, (256, 256, 256, 256), 50, 13, False),
    (64, DEFAULT, 20, 0, True),
]


@pytest.mark.parametrize("B,size,iters,jb,graph", TWIN_CASES)
def test_twins(pkg, B, size, iters, jb, graph):
    flags = 0 if graph else pkg.FLAG_NO_GRAPH
    b, twins = pair(pkg, B, size, flags=flags, jb=jb, PRESSURE_ITERATIONS=iters)
    assert_twins(b, twins, "created")
    seed(b, twins, size, salt=B)
    assert_twins(b, twins, "written")
    members, recs = member_records(B, seed_=B + iters)
    splat_both(b, twins, members, recs)
    assert_twins(b, twins, "splats")
    rng = np.random.default_rng(B)
    for k in range(3 if B < 64 else 2):
        dt = float(np.float32(0.016666 * rng.uniform(0.5, 1.0)))
        b.step(dt)
        for t in twins:
            t.step(dt)
        assert_twins(b, twins, f"step {k}")
        for s in [b] + twins:                              # live config, as the reference reads it
            s.config["CURL"] = 30 + 7 * (k + 1)
            s.config["PRESSURE"] = 0.8 - 0.1 * (k + 1)
            s.config["VELOCITY_DISSIPATION"] = 0.2 + 0.05 * k
    close(b, twins)


def test_isolation(pkg):
    """One member holds NaN, +-inf, subnormal, tiny (0 < |d| < 2^-123) and near-FLT_MAX data, on its first and
    last rows too; its neighbours hold ordinary data.  Every member still equals its twin, and the exact-tail
    counter grows exactly when some twin's does."""
    W = H = Wd = Hd = 256
    size, B = (W, H, Wd, Hd), 4
    b, twins = pair(pkg, B, size, PRESSURE_ITERATIONS=50)
    seed(b, twins, size, salt=7)
    v = b.readField("velocity")
    p = b.readField("pressure")
    v[1] = exp_tiled((H, W, 2), 5, lo=-149, hi=60)          # divergence with tiny and huge values
    p[1] = exp_tiled((H, W), 6, lo=-149, hi=100)
    for r in (0, H - 1):
        p[1, r, ::7] = [np.nan, np.inf, -np.inf, 1e-40, -3e-39, 1e-38][r % 6]
        p[1, r, 3::11] = np.float32(8.5e37 / 0.8)
    d = np.zeros((H, W), np.float32)
    near_max_patch(p[1], d, H - 9, H - 1, 100, 140, 0.8)
    near_max_patch(p[1], d, 1, 8, 10, 30, 0.8)
    for name, a in (("velocity", v), ("pressure", p)):
        b.writeField(name, a)
        for m, t in enumerate(twins):
            t.writeField(name, a[m])
    for k in range(2):
        e_b = b.stat("jacobi_exact_streams")
        e_t = [t.stat("jacobi_exact_streams") for t in twins]
        b.step(0.016)
        for t in twins:
            t.step(0.016)
        assert_twins(b, twins, f"step {k}")
        grew = any(t.stat("jacobi_exact_streams") > e for t, e in zip(twins, e_t))
        assert (b.stat("jacobi_exact_streams") > e_b) == grew, k
    # divergence written with tiny values on member edges rebuilds every member's map region
    dv = b.readField("divergence")
    dv[2, 0, :] = np.float32(1e-40)
    dv[2, H - 1, :] = np.float32(-5e-39)
    b.writeField("divergence", dv)
    assert same_bits(b.readField("divergence"), dv)
    close(b, twins)


@pytest.mark.parametrize("size", [DEFAULT, (256, 256, 256, 256), (512, 128, 1024, 256), (128, 2, 128, 2)])
def test_kernels_and_launches(pkg, size):
    """A batch step runs the streaming cvd and gradient kernels and the 4-cell advections at every accepted
    size, with a twin's launch count, whatever B."""
    counts = {}
    for B in (1, 8):
        b, (t,) = batch(pkg, B, *size, flags=pkg.FLAG_NO_GRAPH), [make(pkg, *size, flags=pkg.FLAG_NO_GRAPH)]
        for stat in ("cvd_stream_launches", "gradient_stream_launches"):
            assert delta(b, stat, lambda: b.step(0.016)) == 1, (B, stat)
        assert delta(b, "advect4_launches", lambda: b.step(0.016)) == 2
        counts[B] = delta(b, "launches", lambda: b.step(0.016))
        assert counts[B] == delta(t, "launches", lambda: t.step(0.016)), (B, size)
        b.close(); t.close()
    assert counts[1] == counts[8]


def test_graph_replays(pkg):
    b = batch(pkg, 8, *DEFAULT)
    rng = np.random.default_rng(3)
    for _ in range(200):
        b.step(float(np.float32(rng.uniform(0.001, 0.016666))))
    b.sync()
    assert b.stat("graph_captures") <= 2 and b.stat("graph_launches") == 200
    b.close()


def test_splats(pkg):
    """Records in shuffled order to 66 of 70 members, 300 of them: more than one launch of 128 records and of
    64 member groups.  Each named member equals a twin that took its own records in order; the others keep
    every byte; the texels stay inside the splat model's interval."""
    size, B = (128, 128, 256, 256), 70
    b, twins = pair(pkg, B, size)
    seed(b, twins, size, salt=11)
    rng = np.random.default_rng(12)
    named = np.setdiff1d(np.arange(B), [3, 17, 40, 69])
    members = rng.choice(named, 300).astype(np.int32)
    members[:len(named)] = named
    rng.shuffle(members)
    recs = nasty_records(300, 13)
    before = {n: b.readField(n) for n in ("velocity", "dye")}
    launches = delta(b, "launches", lambda: splat_both(b, twins, members, recs))
    assert launches >= 3
    assert_twins(b, twins, "splats", ("velocity", "dye"))
    after = {n: b.readField(n) for n in ("velocity", "dye")}
    for m in (3, 17, 40, 69):
        for n in after:
            assert after[n][m].tobytes() == before[n][m].tobytes(), (m, n)
    m = int(members[0])
    aspect, rad = SM.aspect_of(size[0], size[1]), SM.radius_of(0.25, size[0], size[1])
    for n in ("velocity", "dye"):
        lo, hi = SM.splat_interval(before[n][m], recs[members == m], aspect, rad)
        assert SM.check_splat(after[n][m], lo, hi)[0] == 0, n
    # n == 0, and refused records: nothing moves
    L, h = b._L, b._h
    assert L.fluid_splats_batch(h, None, None, 0) == 0
    rec = np.ascontiguousarray(recs[:2])
    fp = rec.ctypes.data_as(C.POINTER(C.c_float))
    for bad in ([0, B], [-1, 0], [5, 2 ** 31 - 1]):
        mm = np.array(bad, np.int32)
        assert L.fluid_splats_batch(h, mm.ctypes.data_as(C.POINTER(C.c_int32)), fp, 2) == INVALID, bad
    mm = np.zeros(2, np.int32)
    assert L.fluid_splats_batch(h, mm.ctypes.data_as(C.POINTER(C.c_int32)), fp, -1) == INVALID
    assert L.fluid_splats_batch(h, None, fp, 2) == INVALID
    assert L.fluid_splats_batch(h, mm.ctypes.data_as(C.POINTER(C.c_int32)), None, 2) == INVALID
    assert_twins(b, twins, "refused splats", ("velocity", "dye"))
    close(b, twins)


def test_device_io(pkg, torch):
    """readField(out=tensor) equals the host read and the twins stacked; writeField(tensor) equals a host write;
    the bytes around the tensor stay as they were."""
    size, B = (128, 128, 256, 256), 3
    b, twins = pair(pkg, B, size)
    seed(b, twins, size, salt=21)
    b.step(0.016)
    for t in twins:
        t.step(0.016)
    G = 4096
    for name in FIELDS:
        host = b.readField(name)
        n = host.size
        buf = torch.full((n + 2 * G,), 7.25, dtype=torch.float32, device="cuda")
        out = buf[G:G + n]
        assert b.readField(name, out=out) is out
        assert same_bits(out.cpu().numpy().reshape(host.shape), host), name
        assert same_bits(host, np.stack([t.readField(name) for t in twins])), name
        assert bool((buf[:G] == 7.25).all()) and bool((buf[G + n:] == 7.25).all()), name
        new = np.random.default_rng(len(name)).standard_normal(host.shape).astype(np.float32)
        buf[G:G + n] = torch.from_numpy(new.reshape(-1)).cuda()
        b.writeField(name, buf[G:G + n])
        assert same_bits(b.readField(name), new), name
        assert bool((buf[:G] == 7.25).all()) and bool((buf[G + n:] == 7.25).all()), name
    close(b, twins)


def test_arena_guard(pkg, torch):
    """With the arena poisoned outside the call's inputs, a step moves only the slots it may write, and a splat
    call only the named members' .read regions."""
    size, B = (128, 128, 256, 256), 3
    W, H, Wd, Hd = size
    b, twins = pair(pkg, B, size)
    seed(b, twins, size, salt=31)
    inputs = {n: b.readField(n) for n in ("velocity", "dye", "pressure")}
    for t in twins:
        t.step(0.016)
    g = BatchArena(torch, b, B)
    for value in (0xFF, 0x3C):
        for n, a in inputs.items():
            b.writeField(n, a)
        g.run("step", lambda: b.step(0.016), tuple(inputs), value)
        assert_twins(b, twins, ("step", value))
    members = np.array([2, 0, 2], np.int32)
    recs = nasty_records(3, 41)
    par = g.parity()
    before = g.image()
    b.splats(members, recs)
    after = g.image()
    moved = np.flatnonzero(before != after)
    allowed = [g.member_range(f, "read", m, par) for f in ("velocity", "dye") for m in (0, 2)]
    out = A.outside(moved, allowed)
    assert len(out) == 0, A.report(g.L, out)
    assert g.parity() == par
    close(b, twins)


def test_refusals(pkg):
    L = pkg.lib()
    cfg = pkg.sim.Config()
    L.fluid_config_default(C.byref(cfg))
    h = C.c_void_p()

    def create(B, **kw):
        c = pkg.sim.Config.from_buffer_copy(cfg)
        for k, v in kw.items():
            setattr(c, k, v)
        rc = L.fluid_create_batch(C.byref(c), B, C.byref(h))
        if rc == 0:
            L.fluid_destroy(h)
        return rc

    assert create(2) == 0 and create(1, flags=pkg.FLAG_NO_GRAPH) == 0
    for B in (0, -1, 65536):
        assert create(B) == INVALID, B
    flags = [pkg.FLAG_UNFUSED, pkg.FLAG_NAIVE_JACOBI, pkg.FLAG_TILED_PASSES, pkg.FLAG_HALF_STORAGE,
             pkg.FLAG_HALF_POSTFX, pkg.FLAG_NEAREST_FILTERING, pkg.FLAG_LINEAR_ADVECTION, 0x100]
    for f in flags:
        assert create(2, flags=f) == INVALID and create(2, flags=f | pkg.FLAG_NO_GRAPH) == INVALID, f
    for kw in ({"sim_w": 96}, {"sim_w": 64}, {"dye_w": 64}, {"sim_h": 1}, {"dye_h": 1}, {"sim_h": 100},
               {"dye_h": 768}, {"sim_w": 0}):
        assert create(2, **kw) == INVALID, kw
    assert create(2, sim_h=2, dye_h=2, dye_w=128) == 0
    assert create(65535, sim_w=1024, sim_h=1024, dye_w=1024, dye_h=1024) == -6      # FLUID_ERR_NOMEM

    size = (128, 128, 256, 256)
    b, (t,) = pair(pkg, 1, size)
    bh = b._h
    assert L.fluid_members(bh) == 1 and L.fluid_members(t._h) == 1
    f = np.zeros(4 * 64 * 64, np.float32)
    u8 = np.zeros(4 * 64 * 64, np.uint8)
    fp, up, vp = f.ctypes.data_as(C.POINTER(C.c_float)), u8.ctypes.data_as(C.c_void_p), f.ctypes.data_as(C.c_void_p)
    fx = pkg.sim.PostFX(8, 256, 0.8, 0.6, 0.7, 196, 1.0)
    i0, i1 = C.c_int(), C.c_int()
    calls = {
        "render": lambda: L.fluid_render(bh, 64, 64, 0, 0, 0, 0, vp, f.size),
        "render_keywords": lambda: L.fluid_render_keywords(bh, 64, 64, 0, None, None, 0, 0, 0, 0, 0, vp, f.size, None, None),
        "render_postfx": lambda: L.fluid_render_postfx(bh, 64, 64, C.byref(fx), vp, 64, 64, 0, 0, 0, vp, f.size, None, None),
        "capture": lambda: L.fluid_capture(bh, 64, 64, 64, 64, 0, 0, None, None, 0, 0, 0, 0, 0, up, u8.size),
        "capture_device": lambda: L.fluid_capture_device(bh, 64, 64, 64, 64, 0, 0, None, None, 0, 0, 0, 0, 0, up, u8.size),
        "render_canvas": lambda: L.fluid_render_canvas(bh, 64, 64, 0, 0, None, None, 0, 0, 0, 0, 0, up, u8.size, 0),
        "render_band": lambda: L.fluid_render_band(bh, 64, C.byref(i0), C.byref(i1)),
        "resize": lambda: L.fluid_resize(bh, 256, 256, 256, 256),
        "pressure_solve_host": lambda: L.fluid_pressure_solve_host(bh, vp, vp, 5),
        "splat": lambda: L.fluid_splat(bh, 0.5, 0.5, 1, 1, 1, 1, 1),
        "splats": lambda: L.fluid_splats(bh, fp, 1),
        "p2p_export": lambda: L.fluid_p2p_export(bh, vp, 256),
        "p2p_connect": lambda: L.fluid_p2p_connect(bh, None, None),
        "p2p_disable": lambda: L.fluid_p2p_disable(bh),
        "splats_batch on an ordinary handle": lambda: L.fluid_splats_batch(t._h, None, fp, 0),
    }
    for n in ("curl", "divergence", "clear_pressure", "pressure_solve", "gradient_subtract"):
        calls["pass_" + n] = lambda n=n: getattr(L, "fluid_pass_" + n)(bh)
    for n in ("vorticity", "advect_velocity", "advect_dye", "curl_vorticity_divergence"):
        calls["pass_" + n] = lambda n=n: getattr(L, "fluid_pass_" + n)(bh, 0.016)
    calls["pass_jacobi"] = lambda: L.fluid_pass_jacobi(bh, 3)
    seed(b, [t], size, salt=51)
    for name, call in calls.items():
        assert call() == INVALID, name
        b.step(0.016)                                      # the handle stays usable
        t.step(0.016)
    assert_twins(b, [t], "after the refusals")
    assert L.fluid_field_elems(bh, 1) == 256 * 256 * 4
    close(b, [t])


def test_large(pkg):
    """B = 16 at 1024^2 / 1024^2 with 50 iterations."""
    size, B = (1024, 1024, 1024, 1024), 16
    b, twins = pair(pkg, B, size, PRESSURE_ITERATIONS=50)
    seed(b, twins, size, salt=61)
    members, recs = member_records(B, 62)
    splat_both(b, twins, members, recs)
    for k in range(2):
        b.step(0.016)
        for t in twins:
            t.step(0.016)
    assert_twins(b, twins, "steps")
    close(b, twins)
