"""Per-member values of batch handles: fluid_set_param_members, fluid_get_param_members and fluid_step_members, and
FluidBatch.member_config / step(array) over them.  The oracle is one ordinary handle per member, its twin, created
with the batch's config and given that member's values through fluid_set_param_f64 and its dt: after every call
each field of each member equals its twin bit for bit."""
import ctypes as C

import numpy as np
import pytest

import arena_model as A
from sim_harness import (Arena, _DeviceBytes, address_range, delta, make, nasty_records, near_max_patch, pkg,  # noqa: F401
                         rand_fields, same_bits, torch, exp_tiled)

pytestmark = pytest.mark.gpu

FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
DEFAULT = (128, 128, 1024, 1024)
INVALID = -1
KEYS = ("DENSITY_DISSIPATION", "VELOCITY_DISSIPATION", "PRESSURE", "CURL", "SPLAT_RADIUS")
# SPLAT_RADIUS 5e-5 puts the radius (5e-7) below the fast division's range: those members' blocks divide by IEEE
VALUES = {"CURL": (0.0, 30.0, 1e4), "PRESSURE": (0.0, 0.8, 1.0, 2.0), "VELOCITY_DISSIPATION": (0.0, 0.2, 1.0, 4.0),
          "DENSITY_DISSIPATION": (0.0, 1.0, 4.0), "SPLAT_RADIUS": (0.01, 0.25, 3.0, 5e-5)}


def batch(pkg, B, W, H, Wd, Hd, flags=0, jb=0, canvas=None, **cfg):
    c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}
    c.update(cfg)
    cw, ch = canvas or (W, H)
    b = pkg.FluidBatch(B, c, canvas_width=cw, canvas_height=ch, sizes=(W, H, Wd, Hd), flags=flags, jacobi_block=jb)
    assert b.members == B
    return b


def twins_of(pkg, B, size, flags=0, jb=0, canvas=None, **cfg):
    ts = [make(pkg, *size, flags=flags, jb=jb, **cfg) for _ in range(B)]
    if canvas:
        for t in ts:
            t.canvas = {"width": canvas[0], "height": canvas[1]}
    return ts


def assert_twins(b, twins, what, fields=FIELDS):
    for name in fields:
        got = b.readField(name)
        for m, t in enumerate(twins):
            assert same_bits(got[m], t.readField(name)), (what, name, m)


def seed(b, twins, size, salt=0):
    W, H, Wd, Hd = size
    data = [rand_fields(W, H, Wd, Hd, 1000 * salt + m) for m in range(len(twins))]
    for k, name in enumerate(("velocity", "dye", "pressure")):
        b.writeField(name, np.stack([d[k] for d in data]))
        for t, d in zip(twins, data):
            t.writeField(name, d[k])


def draw_values(B, rng):
    """One value per member and key from VALUES."""
    return {k: [float(rng.choice(VALUES[k])) for _ in range(B)] for k in KEYS}


def draw_dts(B, rng):
    pool = [0.0, 1.0 / 60, None, 0.1]
    return np.array([np.float32(0.016666 * rng.uniform(0.5, 1.0)) if d is None else d
                     for d in (pool[i] for i in rng.integers(0, 4, B))], np.float32)


def give(b, twins, values):
    """member_config of the batch, config of each twin."""
    for m, t in enumerate(twins):
        for k, v in values.items():
            b.member_config[m][k] = v[m]
            t.config[k] = v[m]


def splat_both(b, twins, seed_):
    rng = np.random.default_rng(seed_)
    B = len(twins)
    members = np.repeat(np.arange(B, dtype=np.int32), rng.integers(0, 3, B))
    recs = nasty_records(len(members), seed_)
    order = rng.permutation(len(members))
    members, recs = members[order], recs[order]
    b.splats(members, recs)
    for m, t in enumerate(twins):
        own = recs[members == m]
        if len(own):
            t.splats(own)


def step_both(b, twins, dts):
    b.step(dts)
    for t, d in zip(twins, dts):
        t.step(float(d))


def close(b, twins):
    b.close()
    for t in twins:
        t.close()


def set_members(L, h, key, values):
    v = np.ascontiguousarray(values, np.float64)
    return L.fluid_set_param_members(h, key, v.ctypes.data_as(C.POINTER(C.c_double)), v.size)


def get_members(L, h, key, n):
    out = np.full(n, -7.0, np.float32)
    return L.fluid_get_param_members(h, key, out.ctypes.data_as(C.POINTER(C.c_float)), n), out


def step_members(L, h, dts):
    d = np.ascontiguousarray(dts, np.float32)
    return L.fluid_step_members(h, d.ctypes.data_as(C.POINTER(C.c_float)), d.size)


# (B, size, PRESSURE_ITERATIONS, JACOBI_BLOCK, graph), from test_gpu_batch's TWIN_CASES: the default size, depth-13
# launches at 256^2 x 50, depth 10 on a 4:1 grid, the smallest height, and B from 1 to 64
CASES = [
    (5, DEFAULT, 20, 0, True),
    (3, (256, 256, 256, 256), 50, 13, False),
    (4, (512, 128, 1024, 256), 20, 10, False),
    (4, (128, 2, 256, 4), 50, 0, True),
    (1, DEFAULT, 20, 0, False),
    (64, DEFAULT, 20, 0, True),
]


@pytest.mark.parametrize("B,size,iters,jb,graph", CASES)
def test_members_equal_twins(pkg, B, size, iters, jb, graph):
    """A session of seeded fields, shuffled splats and three steps, each member with its own values and dt, changed
    between steps."""
    flags = 0 if graph else pkg.FLAG_NO_GRAPH
    b = batch(pkg, B, *size, flags=flags, jb=jb, PRESSURE_ITERATIONS=iters)
    twins = twins_of(pkg, B, size, flags=flags, jb=jb, PRESSURE_ITERATIONS=iters)
    seed(b, twins, size, salt=B + iters)
    rng = np.random.default_rng(B * 7 + iters)
    for k in range(3 if B < 64 else 2):
        give(b, twins, draw_values(B, rng))
        splat_both(b, twins, 100 * B + k)
        assert_twins(b, twins, f"splats {k}", ("velocity", "dye"))
        step_both(b, twins, draw_dts(B, rng))
        assert_twins(b, twins, f"step {k}")
    close(b, twins)


@pytest.mark.parametrize("iters", [0, 1])
def test_clear_and_depth_one(pkg, iters):
    """PRESSURE_ITERATIONS 0 clears in the flat batch launch, 1 in a depth-1 SCALE launch, each member by its own
    PRESSURE."""
    size, B = (128, 128, 256, 256), 4
    b = batch(pkg, B, *size, flags=pkg.FLAG_NO_GRAPH, PRESSURE_ITERATIONS=iters)
    twins = twins_of(pkg, B, size, flags=pkg.FLAG_NO_GRAPH, PRESSURE_ITERATIONS=iters)
    seed(b, twins, size, salt=3 + iters)
    for k, p in enumerate(([0.0, 0.8, 1.0, 2.0], [2.0, -0.5, 0.8, 0.0])):
        give(b, twins, {"PRESSURE": p})
        step_both(b, twins, np.full(B, 0.016, np.float32))
        assert_twins(b, twins, (iters, k))
    close(b, twins)


def test_exact_tail(pkg):
    """Near-FLT_MAX pressure patches and tiny divergence in members with different PRESSURE: the bits match, and the
    exact-tail counter grows exactly when some twin's does."""
    W = H = Wd = Hd = 256
    size, B = (W, H, Wd, Hd), 4
    b = batch(pkg, B, *size, PRESSURE_ITERATIONS=50)
    twins = twins_of(pkg, B, size, PRESSURE_ITERATIONS=50)
    seed(b, twins, size, salt=7)
    give(b, twins, {"PRESSURE": [0.8, 2.0, 1.0, 0.0]})
    v = b.readField("velocity")
    p = b.readField("pressure")
    for m in (1, 2):
        v[m] = exp_tiled((H, W, 2), 5 + m, lo=-149, hi=60)     # divergence with tiny and huge values
        p[m] = exp_tiled((H, W), 6 + m, lo=-149, hi=100)
        d = np.zeros((H, W), np.float32)
        near_max_patch(p[m], d, H - 9, H - 1, 100, 140, 0.8)
        near_max_patch(p[m], d, 1, 8, 10, 30, 0.8)
    for name, a in (("velocity", v), ("pressure", p)):
        b.writeField(name, a)
        for m, t in enumerate(twins):
            t.writeField(name, a[m])
    for k in range(2):
        e_b = b.stat("jacobi_exact_streams")
        e_t = [t.stat("jacobi_exact_streams") for t in twins]
        step_both(b, twins, np.full(B, 0.016, np.float32))
        assert_twins(b, twins, f"step {k}")
        grew = any(t.stat("jacobi_exact_streams") > e for t, e in zip(twins, e_t))
        assert (b.stat("jacobi_exact_streams") > e_b) == grew, k
    close(b, twins)


def test_uniform_values_change_nothing(pkg):
    """Per-member arrays that all equal config, and equal dts, give the bits and launch counts of fluid_set_param
    and fluid_step."""
    size, B = DEFAULT, 3
    a, c = (batch(pkg, B, *size, flags=pkg.FLAG_NO_GRAPH) for _ in range(2))
    data = [rand_fields(*size, 90 + m) for m in range(B)]
    for s in (a, c):
        for k, name in enumerate(("velocity", "dye", "pressure")):
            s.writeField(name, np.stack([d[k] for d in data]))
    L = pkg.lib()
    vals = {"CURL": 12.5, "PRESSURE": 0.6, "VELOCITY_DISSIPATION": 0.3, "DENSITY_DISSIPATION": 0.9, "SPLAT_RADIUS": 0.3}
    for k, v in vals.items():
        assert L.fluid_set_param_f64(a._h, pkg.PARAM[k], v) == 0
        assert set_members(L, c._h, pkg.PARAM[k], [v] * B) == 0
    recs = nasty_records(4, 5)
    members = np.array([0, 2, 2, 1], np.int32)
    for s in (a, c):
        L.fluid_splats_batch(s._h, members.ctypes.data_as(C.POINTER(C.c_int32)), recs.ctypes.data_as(C.POINTER(C.c_float)), 4)
    n_a = delta(a, "launches", lambda: L.fluid_step(a._h, 0.0125))
    n_c = delta(c, "launches", lambda: step_members(L, c._h, [0.0125] * B))
    assert n_a == n_c
    for name in FIELDS:
        assert same_bits(a.readField(name), c.readField(name)), name
    a.close(); c.close()


def test_graphs(pkg):
    """Values and dts changed at every one of 200 steps replay at most two graphs, and give a NO_GRAPH batch's bits."""
    B = 8
    g = batch(pkg, B, *DEFAULT)
    n = batch(pkg, B, *DEFAULT, flags=pkg.FLAG_NO_GRAPH)
    data = [rand_fields(*DEFAULT, 200 + m) for m in range(B)]
    for s in (g, n):
        for k, name in enumerate(("velocity", "dye", "pressure")):
            s.writeField(name, np.stack([d[k] for d in data]))
    L = pkg.lib()
    rng = np.random.default_rng(9)
    for _ in range(200):
        vals = draw_values(B, rng)
        dts = draw_dts(B, rng)
        for s in (g, n):
            for k in ("CURL", "PRESSURE", "VELOCITY_DISSIPATION", "DENSITY_DISSIPATION"):
                assert set_members(L, s._h, pkg.PARAM[k], vals[k]) == 0
            assert step_members(L, s._h, dts) == 0
    g.sync()
    assert g.stat("graph_captures") <= 2 and g.stat("graph_launches") == 200
    for name in FIELDS:
        assert same_bits(g.readField(name), n.readField(name)), name
    g.close(); n.close()


def radius_pair(aspect):
    """Two SPLAT_RADIUS doubles with the same float32 whose correctRadius differs: only double arithmetic tells
    them apart."""
    r0 = 0.25
    for k in range(1, 1000):
        r1 = r0 + k * 1e-10                                  # inside r0's float32 rounding interval (+-1.5e-8)
        if np.float32(r1) != np.float32(r0):
            break
        if np.float32(r1 / 100.0 * aspect) != np.float32(r0 / 100.0 * aspect):
            return r0, float(r1)
    raise AssertionError("no such pair")


def test_precedence(pkg):
    size, B = (128, 128, 256, 256), 3
    canvas = (142, 100)
    b = batch(pkg, B, *size, canvas=canvas)
    L, h = pkg.lib(), b._h
    key = pkg.PARAM["CURL"]
    assert set_members(L, h, key, [0.1, 2.0, 3.0]) == 0
    rc, got = get_members(L, h, key, B)
    assert rc == 0 and got.tolist() == [np.float32(0.1), 2.0, 3.0]
    one = C.c_float()
    assert L.fluid_get_param(h, key, C.byref(one)) == 0 and one.value == np.float32(0.1)
    assert L.fluid_set_param(h, key, 7.0) == 0                         # every member again
    assert get_members(L, h, key, B)[1].tolist() == [7.0] * B
    assert set_members(L, h, key, [1.0, 2.0, 3.0]) == 0
    assert L.fluid_set_param_f64(h, key, 5.0) == 0
    assert get_members(L, h, key, B)[1].tolist() == [5.0] * B
    # SPLAT_RADIUS values that differ only in double arithmetic on a 142x100 canvas
    r0, r1 = radius_pair(canvas[0] / canvas[1])
    twins = twins_of(pkg, B, size, canvas=canvas)
    seed(b, twins, size, salt=17)
    give(b, twins, {"SPLAT_RADIUS": [r0, r1, r0]})
    assert b.member_params("SPLAT_RADIUS").tolist() == [np.float32(r0)] * B
    recs = nasty_records(3, 19)
    members = np.array([0, 1, 2], np.int32)
    b.splats(members, recs)
    for m, t in enumerate(twins):
        t.splats(recs[m:m + 1])
    assert_twins(b, twins, "radius pair", ("velocity", "dye"))
    close(b, twins)


def test_launches(pkg):
    """fluid_step_members launches what fluid_step launches, the same at B = 1 and B = 8."""
    L = pkg.lib()
    counts = {}
    for B in (1, 8):
        b = batch(pkg, B, *DEFAULT, flags=pkg.FLAG_NO_GRAPH)
        one = delta(b, "launches", lambda: L.fluid_step(b._h, 0.016))
        many = delta(b, "launches", lambda: step_members(L, b._h, np.linspace(0, 0.1, B)))
        assert one == many, B
        counts[B] = many
        b.close()
    assert counts[1] == counts[8]


class BatchArena(Arena):
    """The guarded arena of a batch handle: the layout of an ordinary handle whose grids are the B members stacked
    as rows (W x B*H and Wd x B*Hd)."""

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
        lo, hi = A.extent_range(self.L, f"{field}.{side}", par)
        n = (hi - lo) // self.members
        return lo + m * n, lo + (m + 1) * n


def test_arena_guard(pkg, torch):
    """Under both poisons a per-member step moves only the slots a step may write, and a splat call with per-member
    radii only the named members' .read regions."""
    size, B = (128, 128, 256, 256), 3
    b = batch(pkg, B, *size)
    twins = twins_of(pkg, B, size)
    seed(b, twins, size, salt=31)
    give(b, twins, {"CURL": [0.0, 30.0, 1e4], "PRESSURE": [0.8, 2.0, 0.0], "SPLAT_RADIUS": [0.01, 3.0, 5e-5]})
    inputs = {n: b.readField(n) for n in ("velocity", "dye", "pressure")}
    dts = np.array([0.0, 0.1, 0.016], np.float32)
    for t, d in zip(twins, dts):
        t.step(float(d))
    g = BatchArena(torch, b, B)
    for value in (0xFF, 0x3C):
        for n, a in inputs.items():
            b.writeField(n, a)
        g.run("step", lambda: b.step(dts), tuple(inputs), value)           # writes what a step may
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
    close(b, twins)


def test_refusals(pkg):
    size, B = (128, 128, 256, 256), 2
    b = batch(pkg, B, *size)
    (t,) = twins_of(pkg, 1, size)
    twins = twins_of(pkg, B, size)
    seed(b, twins, size, salt=51)
    give(b, twins, {"CURL": [3.0, 4.0], "SPLAT_RADIUS": [0.1, 0.2]})
    b._push_config()
    L, h = pkg.lib(), b._h
    P = pkg.PARAM
    before = {k: b.member_params(k).tolist() for k in KEYS}
    two = np.array([1.0, 2.0])
    dp = two.ctypes.data_as(C.POINTER(C.c_double))
    fl = np.zeros(4, np.float32)
    fp = fl.ctypes.data_as(C.POINTER(C.c_float))
    calls = {
        "set on an ordinary handle": lambda: L.fluid_set_param_members(t._h, P["CURL"], dp, 1),
        "get on an ordinary handle": lambda: L.fluid_get_param_members(t._h, P["CURL"], fp, 1),
        "step on an ordinary handle": lambda: L.fluid_step_members(t._h, fp, 1),
        "set n < B": lambda: L.fluid_set_param_members(h, P["CURL"], dp, 1),
        "set n > B": lambda: L.fluid_set_param_members(h, P["CURL"], dp, 3),
        "get n != B": lambda: L.fluid_get_param_members(h, P["CURL"], fp, 3),
        "step n != B": lambda: L.fluid_step_members(h, fp, 1),
        "step n = 0": lambda: L.fluid_step_members(h, fp, 0),
        "set NULL": lambda: L.fluid_set_param_members(h, P["CURL"], None, B),
        "get NULL": lambda: L.fluid_get_param_members(h, P["CURL"], None, B),
        "step NULL": lambda: L.fluid_step_members(h, None, B),
        "unknown key": lambda: L.fluid_set_param_members(h, 99, dp, B),
        "get unknown key": lambda: L.fluid_get_param_members(h, -1, fp, B),
    }
    for k in ("PRESSURE_ITERATIONS", "JACOBI_BLOCK", "ASPECT", "BACKGROUND"):
        calls["set " + k] = lambda k=k: L.fluid_set_param_members(h, P[k], dp, B)
        calls["get " + k] = lambda k=k: L.fluid_get_param_members(h, P[k], fp, B)
    fields = {n: b.readField(n) for n in FIELDS}
    for name, call in calls.items():
        assert call() == INVALID, name
        assert {k: b.member_params(k).tolist() for k in KEYS} == before, name
    for n, a in fields.items():
        assert same_bits(b.readField(n), a), n
    step_both(b, twins, np.array([0.016, 0.02], np.float32))  # the handle stays usable
    assert_twins(b, twins, "after the refusals")
    close(b, twins + [t])


def test_python_matches_c(pkg):
    """member_config and step(array) give the bits of the C calls; misuse raises ValueError."""
    size, B = (128, 128, 256, 256), 3
    py, c = batch(pkg, B, *size), batch(pkg, B, *size)
    data = [rand_fields(*size, 300 + m) for m in range(B)]
    for s in (py, c):
        for k, name in enumerate(("velocity", "dye", "pressure")):
            s.writeField(name, np.stack([d[k] for d in data]))
    L = pkg.lib()
    vals = {"CURL": [0.0, 30.0, 1e4], "PRESSURE": [0.8, 0.8, 2.0], "SPLAT_RADIUS": [0.25, 3.0, 0.01]}
    for m in range(B):
        for k, v in vals.items():
            py.member_config[m][k] = v[m]
    for k, v in vals.items():
        assert set_members(L, c._h, pkg.PARAM[k], v) == 0
    dts = [0.016, 0.1, 0.0]
    recs = nasty_records(3, 7)
    for s in (py, c):
        s.splats([0, 1, 2], recs)
    py.step(dts)
    assert step_members(L, c._h, dts) == 0
    for name in FIELDS:
        assert same_bits(py.readField(name), c.readField(name)), name
    for k, v in vals.items():
        assert py.member_params(k).tolist() == np.float32(v).tolist(), k
    for bad in ([0.016] * (B + 1), [0.016], [[0.016] * B]):
        with pytest.raises(ValueError):
            py.step(bad)
    py.member_config[1]["ASPECT"] = 2.0
    with pytest.raises(ValueError):
        py.step(0.016)
    del py.member_config[1]["ASPECT"]
    py.member_config.append({})
    with pytest.raises(ValueError):
        py.step(0.016)
    py.member_config.pop()
    for m in range(B):                                         # overrides removed: the shared config again
        py.member_config[m].clear()
    py.step(0.016)
    assert py.member_params("CURL").tolist() == [np.float32(py.config["CURL"])] * B
    py.close(); c.close()
