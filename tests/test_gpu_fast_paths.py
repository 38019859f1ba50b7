"""The size-selected fast paths of step() against the oracle, with data that reaches every branch of
their arithmetic.

* cvd_stream_kernel / gradient_stream_kernel run only on grids big enough to give every SM a warp
  stream (fluid.cu do_cvd / do_gradient); the launch counters prove which kernel ran.
* vort_pre / quot_fast (passes.cuh) take the branch-free scaled sqrt and division only when a whole
  warp agrees (`__all_sync(ok)`); exponent-tiled fields give warps at every scale, so some take the
  scaled fast path at tiny magnitudes and others fall back.
* cvd_stream_kernel flags divergence in (0, 2^-123) for the Jacobi kernel (DESIGN §5.2): whole steps
  from far fields at streaming sizes, and the headline 4096^2 step.
* div_n_by (advection) picks the fast quotient or the IEEE division per thread; tap_pair clamps
  back-traces that land up to ~1700 texels outside the grid.
Bitwise everywhere, NaN-aware (NaN in the same places, every other element bitwise) for the data
set with NaN / inf: CPU and GPU NaN payloads differ."""
import numpy as np
import pytest

from conftest import bits_equal
from sim_harness import STREAM_SHAPES, exp_tiled, far_field, make, nasty_fields, same_bits
from sim_harness import pkg  # noqa: F401 -- a fixture

DT = 0.016666
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
TILED = [(520, 33), (130, 66)]            # too few warps / W % 4 != 0: the tiled kernels
DATA = ["exp_tiled", "far_field", "special"]


def stencil_fields(O, W, H, data, seed):
    """(velocity, pressure) of one data set."""
    if data == "exp_tiled":
        return exp_tiled((H, W, 2), seed), exp_tiled((H, W), seed + 1)
    if data == "far_field":
        v = far_field(O, W, H, 2, seed)
        return v, np.ascontiguousarray(v[..., 0] * np.float32(0.01))
    v, _, p = nasty_fields(W, H, 1, 1, seed)
    return v, p


def vort_ok(c):
    """numpy restatement of vort_pre()'s `ok` (passes.cuh) on a curl field, per cell, with the
    numbers the predicate is built from: s2 and the smaller non-zero numerator."""
    c = np.asarray(c, np.float32)
    H, W = c.shape
    Lf = c[:, np.maximum(np.arange(W) - 1, 0)]; Rf = c[:, np.minimum(np.arange(W) + 1, W - 1)]
    Bf = c[np.maximum(np.arange(H) - 1, 0), :]; Tf = c[np.minimum(np.arange(H) + 1, H - 1), :]
    half = np.float32(0.5)
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        fx = half * (np.abs(Tf) - np.abs(Bf)); fy = half * (np.abs(Rf) - np.abs(Lf))
        s2 = fx * fx + fy * fy
        den = np.sqrt(s2) + np.float32(1e-4)
        thr = np.maximum(den * np.float32(2.0 ** -125), np.float32(2.0 ** -124))
        ax, ay = np.abs(fx), np.abs(fy)
        ok = (s2 <= np.float32(2.0 ** 100)) & ((ax >= thr) | (ax == 0)) & ((ay >= thr) | (ay == 0))
        num = np.minimum(np.where(ax > 0, ax, np.inf), np.where(ay > 0, ay, np.inf))
    return ok, s2, num


def warps(a, cols=120):
    """Group a per-cell (H, W) array by cvd_stream_kernel warp: one row, 120 output columns."""
    H, W = a.shape
    n = -(-W // cols)
    pad = np.full((H, n * cols), np.nan if a.dtype.kind == "f" else True, a.dtype)
    pad[:, :W] = a
    return pad.reshape(H * n, cols)


@pytest.mark.parametrize("W,H", [(1024, 512), (964, 600), (124, 2050)])
def test_exponent_tiled_data_reaches_every_branch_of_vort_pre(oracle, W, H):
    """Premise of the exp_tiled data set (CPU only): its curl holds warps that take the fast path with
    the 2^96 sqrt scaling (s2 < 2^-60), warps that take it with the 2^64 quotient scaling (a numerator
    < 2^-40), and warps that fall back (a subnormal ring, s2 > 2^100 or infinite)."""
    v, _ = stencil_fields(oracle, W, H, "exp_tiled", W + H)
    ok, s2, num = vort_ok(oracle.curl(v))
    ok_w = warps(ok).all(axis=1)
    small_s2 = (warps(s2) < np.float32(2.0 ** -60)).any(axis=1)
    small_num = (warps(num) < np.float32(2.0 ** -40)).any(axis=1)
    assert (ok_w & small_s2).sum() > 10
    assert (ok_w & small_num).sum() > 10
    assert (~ok_w).sum() > 10 and ok_w.sum() > 10


@pytest.mark.gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("W,H", STREAM_SHAPES + TILED)
def test_cvd_and_gradient_fast_arithmetic_vs_oracle(pkg, oracle, W, H, data):
    """curl-vorticity-divergence then gradientSubtract, per pass, against the oracle."""
    O = oracle
    v, p = stencil_fields(O, W, H, data, W * 3 + H)
    cmp = same_bits if data == "special" else bits_equal
    s = make(pkg, W, H, W, H)
    s.writeField("velocity", v); s.writeField("pressure", p)
    c0, g0 = s.stat("cvd_stream_launches"), s.stat("gradient_stream_launches")
    s.pass_("curl_vorticity_divergence", DT)
    c = O.curl(v); v2 = O.vorticity(v, c, 30.0, DT)
    assert cmp(s.readField("curl"), c)
    got_v2 = s.readField("velocity")
    assert bits_equal(got_v2, v2)                     # the vorticity clamp turns NaN into -1000
    assert cmp(s.readField("divergence"), O.divergence(v2))
    s.pass_("gradient_subtract")
    assert cmp(s.readField("velocity"), O.gradient_subtract(p, got_v2))
    streaming = (W, H) in STREAM_SHAPES
    assert s.stat("cvd_stream_launches") - c0 == int(streaming)
    assert s.stat("gradient_stream_launches") - g0 == int(streaming)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("W,H,Wd,Hd,steps", [(1024, 512, 1024, 512, 3), (1024, 1024, 2048, 2048, 2)])
def test_whole_steps_far_field_at_streaming_size(pkg, oracle, W, H, Wd, Hd, steps):
    """Whole steps (graph replay) from written far-field velocity and dye, every field bitwise after
    every step: the tiny-divergence flags cvd_stream_kernel writes for the Jacobi kernel, the scaled
    vorticity arithmetic and div_n_by on subnormal dye, all on the streaming path."""
    O = oracle
    v = far_field(O, W, H, 2, 1); dye = far_field(O, Wd, Hd, 4, 2)
    s = make(pkg, W, H, Wd, Hd)
    ref = O.OracleSim(W, H, Wd, Hd)
    s.writeField("velocity", v); s.writeField("dye", dye)
    ref.velocity, ref.dye = v.copy(), dye.copy()
    c0, g0 = s.stat("cvd_stream_launches"), s.stat("gradient_stream_launches")
    for k in range(steps):
        s.step(DT); ref.step(DT)
        if k == 0:                                    # the premise: divergence the contracted Jacobi tail must not see
            d = np.abs(ref.divergence)
            assert ((d > 0) & (d < np.float32(2.0 ** -123))).any()
        for n in FIELDS:
            assert bits_equal(s.readField(n), getattr(ref, n)), (k, n)
    assert s.stat("cvd_stream_launches") - c0 == steps
    assert s.stat("gradient_stream_launches") - g0 == steps
    s.close()


@pytest.mark.gpu
def test_headline_step_4096_bitwise_vs_oracle(pkg, oracle):
    """The configuration the README quotes: 4096^2 sim + 4096^2 dye, 50 iterations, the default block
    depth, step() as a CUDA graph.  One step from written fields (normal data with a far-field patch),
    all five fields bitwise against the oracle."""
    O = oracle
    O.use_all_cores()
    W = H = 4096
    rng = np.random.default_rng(4096)
    v = (rng.standard_normal((H, W, 2)) * 50).astype(np.float32)
    v[1024:1536, 2048:2560] = far_field(O, 512, 512, 2, 3)
    dye = rng.random((H, W, 4), dtype=np.float32)
    p = rng.standard_normal((H, W)).astype(np.float32)
    s = make(pkg, W, H, W, H, PRESSURE_ITERATIONS=50)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    c0, g0 = s.stat("cvd_stream_launches"), s.stat("gradient_stream_launches")
    s.step(DT)
    assert s.stat("graph_launches") == 1
    assert s.stat("cvd_stream_launches") - c0 == 1 and s.stat("gradient_stream_launches") - g0 == 1
    got = {n: s.readField(n) for n in FIELDS}
    s.close()
    ref = O.OracleSim(W, H, W, H, PRESSURE_ITERATIONS=50)
    ref.velocity, ref.dye, ref.pressure = v, dye, p
    ref.step(DT)
    for n in FIELDS:
        assert bits_equal(got[n], getattr(ref, n)), n


ADVECT_SHAPES = [(256, 256, 256, 256), (128, 128, 256, 256), (64, 64, 128, 128), (64, 64, 64, 64),
                 (36, 20, 54, 30), (1, 9, 3, 27), (9, 1, 27, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("data", ["far", "special"])
@pytest.mark.parametrize("W,H,Wd,Hd", ADVECT_SHAPES)
def test_advection_far_outside_the_grid_vs_oracle(pkg, oracle, W, H, Wd, Hd, data):
    """advect_velocity / advect_dye per pass: every fp32 kernel variant (velocity4, dye4<SAME>,
    dye4<!SAME>, the one-cell POW2 and ragged kernels), back-traces up to ~1700 texels outside the
    grid (tap_pair's integer clamp), dye from 2^100 down to subnormals (both sides of div_n_by's
    range split), dissipation 0, 0.2, 1 and 4."""
    O = oracle
    rng = np.random.default_rng(W * 5 + Wd)
    if data == "far":
        tiles = (-(-H // 4), -(-W // 8))
        mag = np.repeat(np.repeat(10.0 ** rng.uniform(0, 5, tiles), 4, 0), 8, 1)[:H, :W, None]
        v = (rng.uniform(-1, 1, (H, W, 2)) * mag).astype(np.float32)
        dye = exp_tiled((Hd, Wd, 4), W + H, tile=(4, 8))
        cmp = bits_equal
    else:
        v, dye, _ = nasty_fields(W, H, Wd, Hd, W + Hd)
        cmp = same_bits
    s = make(pkg, W, H, Wd, Hd)
    for diss in (0.0, 0.2, 1.0, 4.0):
        s.config["VELOCITY_DISSIPATION"] = diss; s.config["DENSITY_DISSIPATION"] = diss
        s.writeField("velocity", v); s.writeField("dye", dye)
        s.pass_("advect_velocity", DT); v2 = s.readField("velocity")
        assert cmp(v2, O.advect(v, v, DT, diss)), diss
        s.pass_("advect_dye", DT)
        assert cmp(s.readField("dye"), O.advect(v2, dye, DT, diss)), diss
    s.close()
