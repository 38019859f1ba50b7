"""fluid_splats / FluidSimulation.splats(): n splat records applied in one call must give the bits of n
splat() calls, in fp32 and half storage, at every grid shape, across the 128-record launch boundary."""
import ctypes as C

import numpy as np
import pytest

import splat_model as M
from conftest import bits_equal
from test_gpu_parity import SIZES, make

pytestmark = pytest.mark.gpu
DT = 0.016666
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")


@pytest.fixture(scope="module")
def pkg():
    import webgl_fluid_simulation_b200 as p
    return p


def nasty_fields(W, H, Wd, Hd, seed):
    """Seeded fields with -0.0, subnormals, +-inf and NaN sprinkled over ordinary values."""
    rng = np.random.default_rng(seed)

    def sprinkle(a):
        flat = a.reshape(-1)
        specials = np.array([-0.0, 0.0, 1e-40, -3e-39, 1.4e-45, np.inf, -np.inf, np.nan], np.float32)
        k = max(1, flat.size // 7)
        flat[rng.integers(0, flat.size, k)] = rng.choice(specials, k)
        return a
    v = sprinkle((rng.standard_normal((H, W, 2)) * 50).astype(np.float32))
    d = sprinkle(rng.uniform(-1, 2, (Hd, Wd, 4)).astype(np.float32))
    p = rng.standard_normal((H, W)).astype(np.float32)
    return v, d, p


def nasty_records(n, seed):
    """Points inside and outside [0, 1], negative colours, large forces, and far points whose weights
    end in the subnormal range or at zero."""
    rng = np.random.default_rng(seed)
    r = np.empty((n, 7), np.float32)
    r[:, 0:2] = rng.uniform(-0.5, 1.5, (n, 2))
    r[:, 2:4] = rng.uniform(-1, 1, (n, 2)) * 10.0 ** rng.integers(0, 5, (n, 1))
    r[:, 4:7] = rng.uniform(-1.5, 1.5, (n, 3))
    far = rng.random(n) < 0.2
    r[far, 0] = rng.choice([-0.45, 1.45, 3.0, -40.0], far.sum())
    exact = rng.random(n) < 0.1                         # a point on a texel centre: d == 0 there
    r[exact, 0:2] = 0.5
    return r


def pair(pkg, W, H, Wd, Hd, seed, flags=0):
    """Two handles with the same seeded state: [0] gets splats(), [1] one splat() per record."""
    v, d, p = nasty_fields(W, H, Wd, Hd, seed)
    if flags & pkg.FLAG_HALF_STORAGE:
        v, d, p = (x.astype(np.float16).astype(np.float32) for x in (v, d, p))
    sims = [make(pkg, W, H, Wd, Hd, flags=flags) for _ in range(2)]
    for s in sims:
        s.writeField("velocity", v); s.writeField("dye", d); s.writeField("pressure", p)
    return sims


def one_at_a_time(s, recs):
    for x, y, dx, dy, r, g, b in recs.tolist():
        s.splat(x, y, dx, dy, (r, g, b))


def check_same(sims, before):
    for n in ("velocity", "dye"):
        assert bits_equal(sims[0].readField(n), sims[1].readField(n)), n
    for n in ("pressure", "divergence", "curl"):
        for s in sims:
            assert bits_equal(s.readField(n), before[n]), n


@pytest.mark.parametrize("flags", [0, 0x10], ids=["fp32", "half"])
@pytest.mark.parametrize("n", [1, 2, 24, 128, 129, 300])
@pytest.mark.parametrize("W,H,Wd,Hd", SIZES + [(4096, 4096, 4096, 4096)])
def test_batched_equals_one_at_a_time_bitwise(pkg, W, H, Wd, Hd, n, flags):
    if W == 4096 and n not in (1, 129, 300):
        pytest.skip("the 4096^2 case covers one launch, the boundary and three launches")
    sims = pair(pkg, W, H, Wd, Hd, seed=W * 31 + H + n, flags=flags)
    before = {f: sims[0].readField(f) for f in ("pressure", "divergence", "curl")}
    recs = nasty_records(n, seed=n + W)
    sims[0].splats(recs)
    one_at_a_time(sims[1], recs)
    check_same(sims, before)
    assert np.all(sims[0].readField("dye")[..., 3] == 1.0)
    for s in sims:
        s.close()


@pytest.mark.parametrize("flags", [0, 0x10], ids=["fp32", "half"])
@pytest.mark.parametrize("canvas", [(300, 200), (200, 300)], ids=["wide", "tall"])
def test_radius_and_aspect_changes_between_calls(pkg, canvas, flags):
    """correctRadius multiplies by the aspect only when it is above 1 (S:1457-1462); SPLAT_RADIUS and
    the canvas are read anew by every call."""
    W, H, Wd, Hd = 48, 32, 96, 64
    sims = pair(pkg, W, H, Wd, Hd, seed=5, flags=flags)
    before = {f: sims[0].readField(f) for f in ("pressure", "divergence", "curl")}
    for s in sims:
        s.canvas = {"width": canvas[0], "height": canvas[1]}
    for k, rad in enumerate((0.25, 0.07, 1.3)):
        recs = nasty_records(40, seed=k)
        for s in sims:
            s.config["SPLAT_RADIUS"] = rad
        sims[0].splats(recs)
        one_at_a_time(sims[1], recs)
    check_same(sims, before)
    for s in sims:
        s.close()


def test_burst_vs_oracle(pkg, oracle):
    """The independent anchor: a 24-splat burst and 24 oracle splat() calls, both inside the per-texel
    interval of the shader arithmetic."""
    O = oracle
    W, H, Wd, Hd = 64, 48, 128, 96
    rng = np.random.default_rng(11)
    v = (rng.standard_normal((H, W, 2)) * 50).astype(np.float32)
    d = rng.random((Hd, Wd, 4), dtype=np.float32)
    s = make(pkg, W, H, Wd, Hd)
    s.writeField("velocity", v); s.writeField("dye", d)
    recs = nasty_records(24, seed=12)
    recs[:, 0:2] = rng.uniform(0, 1, (24, 2))
    s.splats(recs)
    ref = O.OracleSim(W, H, Wd, Hd)
    ref.velocity, ref.dye = v.copy(), d.copy()
    for rec in recs.tolist():
        ref.splat(*rec)
    # the GPU and the oracle (glibc expf) both inside the per-texel interval of splat_model
    aspect, rad = M.aspect_of(W, H), M.radius_of(0.25, W, H)
    for name, base in (("velocity", v), ("dye", d)):
        lo, hi = M.splat_interval(base, recs, aspect, rad)
        for who, got in (("gpu", s.readField(name)), ("oracle", getattr(ref, name))):
            n, bad = M.check_splat(got, lo, hi)
            assert n == 0, (name, who, n, bad)
    assert np.all(s.readField("dye")[..., 3] == 1.0)
    s.close()


def test_frame_loop_with_graphs_equals_per_record_splats(pkg):
    """splats(k) -> step(dt) for 20 frames on a graph-replaying handle, against per-record splat()
    and pass-by-pass steps (FLAG_NO_GRAPH)."""
    W = H = 128; Wd = Hd = 256
    sims = [make(pkg, W, H, Wd, Hd, flags=f) for f in (0, pkg.FLAG_NO_GRAPH)]
    rng = np.random.default_rng(21)
    for frame in range(20):
        k = int(rng.integers(1, 12))
        recs = np.empty((k, 7), np.float32)
        recs[:, 0:2] = rng.uniform(0, 1, (k, 2))
        recs[:, 2:4] = rng.uniform(-500, 500, (k, 2))
        recs[:, 4:7] = rng.uniform(0, 1.5, (k, 3))
        dt = float(rng.uniform(0.005, 0.016666))
        sims[0].splats(recs); sims[0].step(dt)
        one_at_a_time(sims[1], recs); sims[1].step(dt)
    assert sims[0].stat("graph_captures") <= 2
    for n in FIELDS:
        assert bits_equal(sims[0].readField(n), sims[1].readField(n)), n
    for s in sims:
        s.close()


@pytest.mark.parametrize("flags", [0, 0x10], ids=["fp32", "half"])
def test_launch_counts(pkg, flags):
    s = make(pkg, 64, 64, 128, 128, flags=flags)
    for n in (1, 127, 128, 129, 256, 257, 300):
        l0 = s.launch_count()
        s.splats(np.tile(np.float32([0.5, 0.5, 1, 1, 0.1, 0.2, 0.3]), (n, 1)))
        assert s.launch_count() - l0 == (n + 127) // 128, n
    l0 = s.launch_count()
    s.splat(0.3, 0.3, 1.0, 2.0, (0.1, 0.2, 0.3))
    assert s.launch_count() - l0 == 1
    s.close()


def test_zero_records_launch_nothing_and_touch_nothing(pkg):
    W, H, Wd, Hd = 32, 32, 64, 64
    v, d, p = nasty_fields(W, H, Wd, Hd, 3)
    d[..., 3] = 0.25                                   # a splat would set it to 1
    s = make(pkg, W, H, Wd, Hd)
    s.writeField("velocity", v); s.writeField("dye", d); s.writeField("pressure", p)
    before = {f: s.readField(f) for f in FIELDS}
    l0 = s.launch_count()
    s.splats(np.zeros((0, 7), np.float32))
    assert s._L.fluid_splats(s._h, None, 0) == 0
    assert s.launch_count() == l0
    for f in FIELDS:
        assert bits_equal(s.readField(f), before[f]), f
    s.close()


def test_refusals_leave_the_handle_usable(pkg):
    W, H, Wd, Hd = 32, 32, 64, 64
    sims = pair(pkg, W, H, Wd, Hd, seed=9)
    s = sims[0]
    before = {f: s.readField(f) for f in FIELDS}
    recs = nasty_records(5, seed=9)
    ptr = recs.ctypes.data_as(C.POINTER(C.c_float))
    l0 = s.launch_count()
    assert s._L.fluid_splats(s._h, None, 5) == -1
    assert s._L.fluid_splats(s._h, ptr, -1) == -1
    assert s._L.fluid_splats(s._h, ptr, -(2 ** 31)) == -1
    assert s._L.fluid_last_error(s._h)
    assert s.launch_count() == l0
    for f in FIELDS:
        assert bits_equal(s.readField(f), before[f]), f
    with pytest.raises(ValueError):
        s.splats(np.zeros((5, 6), np.float32))
    s.splats(recs)                                     # the next good call succeeds
    one_at_a_time(sims[1], recs)
    check_same(sims, {f: before[f] for f in ("pressure", "divergence", "curl")})
    for t in sims:
        t.close()
