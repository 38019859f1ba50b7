"""GPU parity: the CUDA library, called through the C ABI, against the CPU oracle and the golden
vectors.  Bitwise for every pass whose arithmetic is IEEE-exact (all but splat's expf)."""
import numpy as np
import pytest

import display_model as DM
import gamma_model as G
import splat_model as M
from conftest import bits_equal, golden, max_rel
from sim_harness import SIZES, STREAM_SHAPES, TILED_SHAPES, make, nasty_fields, rand_fields, same_bits
from sim_harness import pkg  # noqa: F401 -- a fixture
from webgl_fluid_simulation_b200 import slab

pytestmark = pytest.mark.gpu
DT = 0.016666
SPLAT_TOL = 2e-6   # expf: CUDA <= 2 ulp, glibc < 1 ulp; on a term that is added to the base


@pytest.mark.parametrize("W,H,Wd,Hd", SIZES)
def test_every_pass_bitwise_vs_oracle(pkg, oracle, W, H, Wd, Hd):
    O = oracle
    v, dye, p = rand_fields(W, H, Wd, Hd, W * 7 + H)
    s = make(pkg, W, H, Wd, Hd)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    s.pass_("curl"); c = s.readField("curl"); assert bits_equal(c, O.curl(v))
    s.pass_("vorticity", DT); v2 = s.readField("velocity")
    assert bits_equal(v2, O.vorticity(v, c, 30.0, DT))
    s.pass_("divergence"); d = s.readField("divergence"); assert bits_equal(d, O.divergence(v2))
    s.pass_("clear_pressure"); p1 = s.readField("pressure"); assert bits_equal(p1, O.clear(p, 0.8))
    s.pass_("jacobi", 1); p2 = s.readField("pressure"); assert bits_equal(p2, O.jacobi(p1, d, 1))
    s.pass_("jacobi", 13); p3 = s.readField("pressure"); assert bits_equal(p3, O.jacobi(p2, d, 13))
    s.pass_("gradient_subtract"); v3 = s.readField("velocity")
    assert bits_equal(v3, O.gradient_subtract(p3, v2))
    s.pass_("advect_velocity", DT); v4 = s.readField("velocity")
    assert bits_equal(v4, O.advect(v3, v3, DT, 0.2))
    s.pass_("advect_dye", DT); d2 = s.readField("dye")
    assert bits_equal(d2, O.advect(v4, dye, DT, 1.0))
    s.splat(0.3, 0.6, 123.0, -456.0, (0.5, 0.2, 0.9))
    # splat: every texel within the fp32 shader arithmetic with an expf inside EXPF_ULP (splat_model)
    rec = np.array([[0.3, 0.6, 123.0, -456.0, 0.5, 0.2, 0.9]], np.float32)
    aspect, rad = M.aspect_of(W, H), M.radius_of(0.25, W, H)
    for name, base in (("velocity", v4), ("dye", d2)):
        n, bad = M.check_splat(s.readField(name), *M.splat_interval(base, rec, aspect, rad))
        assert n == 0, (name, n, bad)
    assert np.all(s.readField("dye")[..., 3] == 1.0)
    s.close()


@pytest.mark.parametrize("name", ["pass_32x32_64x64", "pass_64x32_128x64", "pass_16x16_16x16"])
def test_passes_vs_golden_reference_shader_outputs(pkg, name):
    """Straight against the vectors cut by executing the reference's GLSL text (power-of-two grids:
    bitwise for everything but splat)."""
    g = golden(name)
    W, H, Wd, Hd = (int(g[k]) for k in ("W", "H", "Wd", "Hd")); dt = float(g["dt"])
    s = make(pkg, W, H, Wd, Hd, flags=pkg.FLAG_UNFUSED)
    s.writeField("velocity", g["in_velocity"]); s.writeField("dye", g["in_dye"])
    s.writeField("pressure", g["in_pressure"])
    s.pass_("curl"); assert bits_equal(s.readField("curl"), g["curl"])
    s.pass_("vorticity", dt); assert bits_equal(s.readField("velocity"), g["vorticity"])
    s.pass_("divergence"); assert bits_equal(s.readField("divergence"), g["divergence"])
    s.pass_("clear_pressure"); assert bits_equal(s.readField("pressure"), g["clear"])
    s.pass_("jacobi", 1); assert bits_equal(s.readField("pressure"), g["jacobi1"])
    s.pass_("jacobi", 12); assert bits_equal(s.readField("pressure"), g["jacobi13"])
    s.pass_("gradient_subtract"); assert bits_equal(s.readField("velocity"), g["gradient"])
    s.pass_("advect_velocity", dt); assert bits_equal(s.readField("velocity"), g["advect_velocity"])
    s.pass_("advect_dye", dt); assert bits_equal(s.readField("dye"), g["advect_dye"])
    sp = g["splat_args"]
    s.splat(*[float(x) for x in sp[:4]], tuple(float(x) for x in sp[4:]))
    assert max_rel(s.readField("velocity"), g["splat_velocity"]) < SPLAT_TOL
    assert max_rel(s.readField("dye"), g["splat_dye"]) < SPLAT_TOL
    s.close()


@pytest.mark.parametrize("W,H", TILED_SHAPES + STREAM_SHAPES)
def test_fused_curl_vorticity_divergence_equals_three_passes(pkg, oracle, W, H):
    """fluid_pass_curl_vorticity_divergence == curl, vorticity, divergence of the oracle, bitwise, and
    == the tiled kernel (FLAG_TILED_PASSES).  STREAM_SHAPES must run cvd_stream_kernel, TILED_SHAPES
    curl_vorticity_divergence_kernel: the launch counter says which one ran."""
    O = oracle
    v, _, _ = rand_fields(W, H, W, H, 11)
    c = O.curl(v); v2 = O.vorticity(v, c, 30.0, DT); d = O.divergence(v2)
    outs = []
    for flags in (0, pkg.FLAG_TILED_PASSES):
        s = make(pkg, W, H, W, H, flags=flags)
        s.writeField("velocity", v)
        n0 = s.stat("cvd_stream_launches")
        s.pass_("curl_vorticity_divergence", DT)
        streamed = s.stat("cvd_stream_launches") - n0
        assert streamed == (1 if flags == 0 and (W, H) in STREAM_SHAPES else 0), streamed
        outs.append([s.readField(n) for n in ("curl", "velocity", "divergence")])
        s.close()
    for got, tiled, want in zip(outs[0], outs[1], (c, v2, d)):
        assert bits_equal(got, want)
        assert bits_equal(got, tiled)


@pytest.mark.parametrize("W,H", TILED_SHAPES + STREAM_SHAPES)
def test_gradient_subtract_streaming_and_tiled_vs_oracle(pkg, oracle, W, H):
    """fluid_pass_gradient_subtract == the oracle bitwise and == the tiled kernel; STREAM_SHAPES run
    gradient_stream_kernel, TILED_SHAPES gradient_subtract_kernel."""
    O = oracle
    v, _, p = rand_fields(W, H, W, H, 12)
    want = O.gradient_subtract(p, v)
    outs = []
    for flags in (0, pkg.FLAG_TILED_PASSES):
        s = make(pkg, W, H, W, H, flags=flags)
        s.writeField("velocity", v); s.writeField("pressure", p)
        n0 = s.stat("gradient_stream_launches")
        s.pass_("gradient_subtract")
        streamed = s.stat("gradient_stream_launches") - n0
        assert streamed == (1 if flags == 0 and (W, H) in STREAM_SHAPES else 0), streamed
        outs.append(s.readField("velocity"))
        s.close()
    assert bits_equal(outs[0], want)
    assert bits_equal(outs[0], outs[1])


@pytest.mark.parametrize("W,H,iters,jb", [(128, 64, 20, 8), (256, 200, 50, 8), (512, 96, 30, 10),
                                          (16, 16, 9, 4), (1024, 1024, 50, 8), (132, 45, 17, 5),
                                          (240, 300, 33, 7), (112, 2, 6, 3), (2048, 512, 40, 10),
                                          (4096, 96, 50, 10), (1000, 64, 24, 12)])
def test_temporally_blocked_jacobi_bitwise_equals_naive_and_oracle(pkg, oracle, W, H, iters, jb):
    """P5: K sweeps per launch == K launches of one sweep == the oracle, bit for bit; the fused
    clear pass included (fluid_pass_pressure_solve == clear + iters x jacobi).  W = 4096 at K = 10 has
    the last window whose mirrored lanes lie outside the staged box."""
    O = oracle
    rng = np.random.default_rng(W + H + iters)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    outs = []
    for flags, block in ((0, jb), (pkg.FLAG_NAIVE_JACOBI, 1)):
        s = make(pkg, W, H, W, H, flags=flags, jb=block, PRESSURE_ITERATIONS=iters)
        s.writeField("pressure", p); s.writeField("divergence", d)
        s.pass_("pressure_solve")
        outs.append(s.readField("pressure"))
        assert s.stat("jacobi_exact_streams") == 0          # ordinary data: every stream contracted
        s.close()
    assert bits_equal(outs[0], outs[1])
    if W * H <= 1 << 20:
        assert bits_equal(outs[0], O.jacobi(O.clear(p, 0.8), d, iters))


@pytest.mark.parametrize("name,tol", [("step_curl30_32", 1e-5), ("step_curl30_48x32", 5e-5),
                                      ("step_curl0_32", 2e-5)])
def test_full_step_vs_golden_scenarios(pkg, name, tol):
    """P2/P3: whole step() through the public API against the executed-reference scenarios."""
    g = golden(name)
    cfg = dict(zip([str(k) for k in g["config_keys"]], [float(x) for x in g["config_vals"]]))
    W, H, Wd, Hd = (int(g[k]) for k in ("W", "H", "Wd", "Hd"))
    s = make(pkg, W, H, Wd, Hd, CURL=cfg["CURL"], PRESSURE_ITERATIONS=int(cfg["PRESSURE_ITERATIONS"]))
    for a in g["splats"]:
        s.splat(*[float(x) for x in a[:4]], tuple(float(x) for x in a[4:]))
    steps = int(g["steps"])
    for k in range(1, steps + 1):
        s.step(float(g["dt"]))
        if k in (1, 2, steps):
            for n in ("velocity", "dye", "pressure", "divergence", "curl"):
                assert max_rel(s.readField(n), g[f"s{k}_{n}"]) < tol, (k, n)
    s.close()


def test_full_step_bitwise_vs_oracle_when_no_splat_arithmetic(pkg, oracle):
    """With identical start fields (written, not splatted) a whole step is bit-identical to the
    oracle: fused kernels, temporal blocking and all."""
    O = oracle
    W = H = 256; Wd = Hd = 512
    v, dye, p = rand_fields(W, H, Wd, Hd, 3)
    s = make(pkg, W, H, Wd, Hd)
    ref = O.OracleSim(W, H, Wd, Hd)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    for _ in range(3):
        s.step(DT); ref.step(DT)
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert bits_equal(s.readField(n), getattr(ref, n)), n
    s.close()


def test_properties_at_full_size_4096(pkg):
    """Size-independent properties at BASELINE config 3 (4096^2, 50 iterations), where the oracle
    is too slow to run in a test: (1) blocked == naive bitwise; (2) linearity of the Jacobi map in
    (p, div) for power-of-two scalings (exact in fp32); (3) constant p, zero div is a fixed point;
    (4) the mirror symmetry of the clamp boundary: a left-right flipped input gives a flipped output."""
    W = H = 4096; iters = 50
    rng = np.random.default_rng(0)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)

    def solve(pp, dd, flags=0, jb=0, pressure=0.8):
        # jb = 0: the library's default block depth, PRESSURE 0.8 with the clear pass fused into the
        # first launch -- exactly the configuration bench.py times
        s = make(pkg, W, H, 64, 64, flags=flags, jb=jb, PRESSURE_ITERATIONS=iters, PRESSURE=pressure)
        s.writeField("pressure", pp); s.writeField("divergence", dd)
        s.pass_("pressure_solve"); out = s.readField("pressure")
        assert s.stat("jacobi_exact_streams") == 0
        s.close()
        return out
    a = solve(p, d)
    assert bits_equal(a, solve(p, d, flags=pkg.FLAG_NAIVE_JACOBI, jb=1))
    assert bits_equal(a, solve(p, d, jb=8))                           # another block depth, same bits
    assert bits_equal(solve(4 * p, 4 * d), 4 * a)
    assert bits_equal(solve(np.full_like(p, 2.5), np.zeros_like(d), pressure=1.0), np.full_like(p, 2.5))
    assert bits_equal(solve(p[:, ::-1].copy(), d[:, ::-1].copy()), a[:, ::-1])
    # a slice of the full-size result against the oracle: the Jacobi stencil's cone of influence is
    # `iters` cells, so rows [0, 192) of the solve depend only on rows [0, 192 + iters) of the input
    # with the true bottom wall -- recompute that strip on the CPU and compare the part that is exact
    from oracle import oracle as O
    strip = 192 + iters
    ref = O.jacobi(O.clear(p[:strip], 0.8), d[:strip], iters)
    assert bits_equal(a[:192], ref[:192])


def test_config0_whole_steps_vs_executed_reference_and_oracle(pkg, oracle):
    """BASELINE configs[0]: 128x128 sim / 256x256 dye, 20 iterations.  (a) two whole steps after
    multipleSplats(5) against the golden cut from the executed reference shaders (tolerances as in
    tests/test_oracle_golden.py: splat expf last place, amplified by vorticity confinement);
    (b) from written (not splatted) fields: 4 whole steps bit-identical to the oracle."""
    g = golden("config0_128_256")
    s = make(pkg, 128, 128, 256, 256, CURL=30, PRESSURE_ITERATIONS=20)
    for a in g["splats"]:
        s.splat(*[float(x) for x in a[:4]], tuple(float(x) for x in a[4:]))
    for k, tol in ((1, 1e-5), (2, 5e-5)):
        s.step(float(g["dt"]))
        for n in ("velocity", "dye", "pressure", "divergence", "curl"):
            assert max_rel(s.readField(n), g[f"s{k}_{n}"]) < tol, (k, n)
    s.close()
    O = oracle
    v, dye, p = rand_fields(128, 128, 256, 256, 17)
    s = make(pkg, 128, 128, 256, 256, PRESSURE_ITERATIONS=20)
    ref = O.OracleSim(128, 128, 256, 256)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    for _ in range(4):
        s.step(DT); ref.step(DT)
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert bits_equal(s.readField(n), getattr(ref, n)), n
    s.close()


def test_config1_whole_steps_bitwise_vs_oracle(pkg, oracle):
    """BASELINE configs[1]: 1024x1024 sim / 2048x2048 dye, 30 iterations, fp32: two whole steps from
    written fields, every field bit-identical to the CPU oracle (graph replay, fused kernels,
    temporally blocked Jacobi at its default depth)."""
    O = oracle
    W = H = 1024; Wd = Hd = 2048
    v, dye, p = rand_fields(W, H, Wd, Hd, 5)
    s = make(pkg, W, H, Wd, Hd, PRESSURE_ITERATIONS=30)
    ref = O.OracleSim(W, H, Wd, Hd, PRESSURE_ITERATIONS=30)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    for _ in range(2):
        s.step(DT); ref.step(DT)
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert bits_equal(s.readField(n), getattr(ref, n)), n
    s.close()


def test_update_loop_with_jittered_dt_replays_two_graphs(pkg):
    """calcDeltaTime() (S:1188-1194) yields a different dt on every frame; dt lives in device
    memory, so 200 update() calls replay the same two instantiated graphs (one per ping-pong
    parity) and stay bit-identical to the pass-by-pass path."""
    W = H = 128; Wd = Hd = 256
    v, dye, p = rand_fields(W, H, Wd, Hd, 33)
    sims = [make(pkg, W, H, Wd, Hd, flags=f) for f in (0, pkg.FLAG_NO_GRAPH)]
    for s in sims:
        s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
        s.lastUpdateTime = 0.0
    rng = np.random.default_rng(8)
    now = 0.0
    for k in range(200):
        now += float(rng.uniform(3.0, 21.0))          # ms between frames: mostly below the 16.666 ms clamp
        for s in sims:
            s.update(now_ms=now)
    assert sims[0].stat("graph_captures") <= 2 and sims[0].stat("graph_launches") == 200
    for n in ("velocity", "dye", "pressure"):
        assert bits_equal(sims[0].readField(n), sims[1].readField(n)), n
    for s in sims:
        s.close()


@pytest.mark.parametrize("case", ["all_subnormal", "tiny_div_patch", "tiny_div_everywhere", "zeros_and_tiny"])
def test_blocked_jacobi_bitwise_with_subnormal_and_tiny_values(pkg, oracle, case):
    """The contracted tail fma(S, 0.25, -0.25 d) is exact only for d == 0 or |d| >= 2^-123
    (tests/test_fma_contraction_cpu.py); cells of divergence below that are flagged in the
    tiny-value map and their warps run the un-contracted form.  Fields full of subnormals, a patch
    of tiny divergence inside ordinary data, and exact zeros must all stay bit-identical to the
    oracle (which runs without flush-to-zero)."""
    O = oracle
    W, H, iters = 512, 200, 30
    rng = np.random.default_rng(5)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    tiny = (rng.integers(1, 2 ** 23, (H, W)) * 2.0 ** -149).astype(np.float32) * rng.choice([-1, 1], (H, W)).astype(np.float32)
    if case == "all_subnormal":
        p = (tiny * 3).astype(np.float32); d = tiny.copy()
    elif case == "tiny_div_patch":
        d[60:90, 100:300] = tiny[60:90, 100:300]; p[55:95, 90:310] *= np.float32(2.0 ** -125)
    elif case == "tiny_div_everywhere":
        d = tiny.copy(); p *= np.float32(2.0 ** -124)
    else:
        d[:] = 0; d[::7, ::5] = tiny[::7, ::5]; p[:, : W // 2] = 0; p[:, W // 2:] *= np.float32(2.0 ** -126)
    for jb in (0, 7):
        s = make(pkg, W, H, 8, 8, jb=jb, PRESSURE_ITERATIONS=iters)
        s.writeField("pressure", p); s.writeField("divergence", d)
        s.pass_("pressure_solve")
        got = s.readField("pressure")
        assert s.stat("jacobi_exact_streams") > 0, (case, jb)     # the tiny map sent streams to the exact tail
        s.close()
        assert bits_equal(got, O.jacobi(O.clear(p, 0.8), d, iters)), (case, jb)


def test_whole_step_bitwise_with_splat_far_field_subnormals(pkg, oracle):
    """A Gaussian splat's far field underflows gradually (exp(-r^2/0.0025) passes through the
    subnormal range), so real velocity / divergence fields DO contain tiny values: the fused
    curl-vorticity-divergence pass must flag them for the Jacobi kernel.  Fields are written (the
    same bits on both sides), then two whole steps must be bit-identical to the oracle."""
    O = oracle
    W = H = 256
    z = np.zeros((H, W, 2), np.float32)
    v = O.splat(z, 1.0, 0.3, 0.4, (400.0, -300.0, 0.0), O.correct_radius(0.25, 1.0))
    v = O.splat(v, 1.0, 0.8, 0.7, (-250.0, 120.0, 0.0), O.correct_radius(0.25, 1.0))
    assert ((np.abs(v) > 0) & (np.abs(v) < 2.0 ** -123)).any()          # the premise
    dye = np.zeros((H, W, 4), np.float32); dye[..., 3] = 1
    s = make(pkg, W, H, W, H)
    ref = O.OracleSim(W, H, W, H)
    s.writeField("velocity", v); s.writeField("dye", dye)
    ref.velocity, ref.dye = v.copy(), dye.copy()
    for _ in range(2):
        s.step(DT); ref.step(DT)
    for n in ("velocity", "pressure", "divergence", "curl"):
        assert bits_equal(s.readField(n), getattr(ref, n)), n
    s.close()


def test_host_pressure_solve_matches_resident_path(pkg):
    W = H = 512
    rng = np.random.default_rng(1)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    s = make(pkg, W, H, 64, 64, PRESSURE_ITERATIONS=30)
    s.writeField("pressure", p); s.writeField("divergence", d)
    s.pass_("pressure_solve"); a = s.readField("pressure")
    ph = p.copy()
    s.pressure_solve_host(d, ph, 30)
    assert bits_equal(a, ph)
    s.close()


# (W, H, iters, JACOBI_BLOCK, bands x launches per band); W = 1000 is not a multiple of a window's payload
@pytest.mark.parametrize("W,H,iters,jb,launches", [(1024, 2048, 50, 0, 8 * 5), (256, 1000, 20, 0, 3 * 2),
                                                   (4096, 4096, 50, 0, 16 * 5), (1000, 2048, 50, 0, 8 * 5),
                                                   (1000, 2048, 50, 13, 8 * 4), (4096, 4096, 50, 13, 16 * 4)])
def test_host_pressure_solve_banded_pipeline(pkg, W, H, iters, jb, launches):
    """fluid_pressure_solve_host cuts the grid into row bands and solves each behind the copies
    (fluid.cu solve_host_banded): same bits as the resident one-piece solve, result also left in the
    device field, tiny divergence values (un-contracted instantiation) included, ragged last band.
    The launches of a band read band-private rows through their own tensor maps, from a local row 0
    that is not the field's; the band schedule (bands x launches) is pinned."""
    rng = np.random.default_rng(5)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    d[H // 3, W // 5] = np.float32(2.0 ** -130)            # defeats the fma contraction: flagged through the scan of the band
    d[H - 7, 3] = np.float32(-2.0 ** -140)
    s = make(pkg, W, H, 64, 64, jb=jb, PRESSURE_ITERATIONS=iters)
    s.writeField("pressure", p); s.writeField("divergence", d)
    s.pass_("pressure_solve"); a = s.readField("pressure")
    ph = p.copy()
    n0 = s.stat("jacobi_launches")
    s.pressure_solve_host(d, ph, iters)
    n_host = s.stat("jacobi_launches") - n0
    assert n_host == launches
    assert n_host == sum(len(b["launches"]) for b in slab.host_bands(H, iters, block=jb))
    assert bits_equal(a, ph)
    assert bits_equal(s.readField("pressure"), ph)
    assert bits_equal(s.readField("divergence"), d)
    ph2 = ph.copy()
    s.pressure_solve_host(d, ph2, iters)                   # a second call (ping-pong parity flipped, private rows reused)
    s.writeField("pressure", ph); s.pass_("pressure_solve")
    assert bits_equal(s.readField("pressure"), ph2)
    s.close()


def test_resize_carries_state_like_resizeDoubleFBO(pkg, oracle):
    O = oracle
    v, dye, p = rand_fields(32, 32, 64, 64, 9)
    s = make(pkg, 32, 32, 64, 64)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    s.config["SIM_RESOLUTION"] = 48; s.config["DYE_RESOLUTION"] = 96
    s.canvas = {"width": 512, "height": 512}; s._sizes = None
    s.initFramebuffers()
    assert bits_equal(s.readField("velocity"), O.resample(v, 48, 48))
    assert bits_equal(s.readField("dye"), O.resample(dye, 96, 96))
    assert not s.readField("pressure").any() and not s.readField("divergence").any()
    s.close()
    # and straight against the executed copyShader: power-of-two sizes bitwise, ragged ones at the tolerance
    # of test_oracle_golden.py (the rasteriser's vUv differs from (i + .5) / W in the last place)
    g = golden("resample_dye_64_to_32")
    s = make(pkg, 16, 16, 64, 64)
    s.writeField("dye", g["src"])
    s._sizes = (16, 16, 32, 32); s.initFramebuffers()
    assert bits_equal(s.readField("dye"), g["linear"])
    s.close()
    for name, plane in (("resample_v_32_to_48", "velocity"), ("resample_dye_40x28_to_64x48", "dye")):
        g = golden(name)
        Hs, Ws = g["src"].shape[:2]
        Wn, Hn = int(g["Wd"]), int(g["Hd"])
        s = make(pkg, *((Ws, Hs, 8, 8) if plane == "velocity" else (8, 8, Ws, Hs)))
        s.writeField(plane, g["src"])
        s._sizes = (Wn, Hn, 8, 8) if plane == "velocity" else (8, 8, Wn, Hn)
        s.initFramebuffers()
        got = s.readField(plane)
        assert bits_equal(got, O.resample(g["src"], Wn, Hn)), name
        assert max_rel(got, g["linear"]) < 2e-6, name
        s.close()


@pytest.mark.parametrize("src,dst", [((36, 20, 54, 30), (23, 41, 97, 31)),          # ragged, down and up
                                     ((23, 41, 97, 31), (36, 20, 54, 30)),
                                     ((1024, 512, 1024, 512), (37, 23, 37, 23)),    # a large down-scale
                                     ((1, 9, 3, 27), (9, 1, 27, 3)),                # 1-column -> 1-row grids
                                     ((9, 1, 27, 3), (1, 9, 3, 27))])
def test_resize_ragged_and_degenerate_sizes_like_resizeDoubleFBO(pkg, oracle, src, dst):
    """initFramebuffers() on an fp32 handle (fluid_resize) at the sizes of its half-storage sibling and
    beyond: velocity and dye resampled with the LINEAR copy, bitwise against the oracle, inf / NaN dye
    NaN-aware; pressure, divergence and curl start over at zero."""
    O = oracle
    v, _, p = rand_fields(*src, 9)
    _, dye, _ = nasty_fields(1, 1, src[2], src[3], 10)             # inf / NaN / subnormal dye
    s = make(pkg, *src)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    s._sizes = dst; s.initFramebuffers()
    W, H, Wd, Hd = dst
    assert s._dims("velocity")[:2] == (W, H) and s._dims("dye")[:2] == (Wd, Hd)
    assert bits_equal(s.readField("velocity"), O.resample(v, W, H))
    assert same_bits(s.readField("dye"), O.resample(dye, Wd, Hd))
    for n in ("pressure", "divergence", "curl"):
        assert not s.readField(n).any(), n
    s.close()


def test_live_config_and_error_paths(pkg):
    s = make(pkg, 64, 64, 64, 64)
    s.config["PRESSURE_ITERATIONS"] = 3
    s.step(DT)
    with pytest.raises(pkg.FluidError):
        s.writeField("velocity", np.zeros(5, np.float32))
    with pytest.raises(pkg.FluidError):
        s.set_param("CURL", 1.0) or s._check(s._L.fluid_set_param(s._h, 99, 0.0))
    assert s.launch_count() > 0
    s.close()


def test_graph_replay_equals_pass_by_pass(pkg):
    """fluid_step as a cached CUDA graph (default) == the same step launched kernel by kernel
    (FLUID_FLAG_NO_GRAPH), bit for bit, across cache misses (new dt, changed config, both
    ping-pong parities) and hits; writes and splats between steps must be seen by the replays."""
    W = H = 128; Wd = Hd = 256
    v, dye, p = rand_fields(W, H, Wd, Hd, 21)
    sims = [make(pkg, W, H, Wd, Hd, flags=f) for f in (0, pkg.FLAG_NO_GRAPH)]
    for s in sims:
        s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    dts = [0.016666, 0.016666, 0.016666, 0.01, 0.016666, 0.01, 0.016666, 0.016666]
    for k, dt in enumerate(dts):
        for s in sims:
            if k == 3:
                s.config["CURL"] = 12.5
            if k == 5:
                s.splat(0.4, 0.7, 200.0, -100.0, (0.3, 0.6, 0.9))
            if k == 6:
                s.config["PRESSURE_ITERATIONS"] = 33
            s.step(dt)
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert bits_equal(sims[0].readField(n), sims[1].readField(n)), n
    assert sims[0].launch_count() == sims[1].launch_count()
    for s in sims:
        s.close()


def test_random_shapes_blocked_jacobi_vs_oracle(pkg, oracle):
    """Randomised sweep (seeded) over grid shapes, iteration counts and block depths: widths that
    are / are not multiples of 4 and of the 104..120-column window payload, 1-row and 2-row grids,
    depths 1..12.  Every case bitwise against the oracle, fused clear included."""
    O = oracle
    rng = np.random.default_rng(2024)
    for case in range(40):
        W = int(rng.choice([rng.integers(1, 40), 4 * rng.integers(4, 160), rng.integers(16, 700)]))
        H = int(rng.choice([1, 2, rng.integers(3, 40), rng.integers(40, 300)]))
        iters = int(rng.integers(1, 45)); jb = int(rng.integers(1, 13))
        p = rng.standard_normal((H, W)).astype(np.float32)
        d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
        s = make(pkg, W, H, 8, 8, jb=jb, PRESSURE_ITERATIONS=iters)
        s.writeField("pressure", p); s.writeField("divergence", d)
        s.pass_("pressure_solve")
        got = s.readField("pressure"); s.close()
        assert bits_equal(got, O.jacobi(O.clear(p, 0.8), d, iters)), (case, W, H, iters, jb)


@pytest.mark.parametrize("Wd,Hd,w,h", [(64, 64, 128, 128), (40, 28, 50, 30), (256, 256, 333, 200)])
def test_render_display_bitwise_vs_oracle(pkg, oracle, Wd, Hd, w, h):
    """The display pass ("next" row): fluid_render == the oracle bit for bit, shaded and flat, and
    equals the executed-reference golden on the power-of-two case."""
    rng = np.random.default_rng(Wd + w)
    dye = (rng.random((Hd, Wd, 4), dtype=np.float32) * 2).astype(np.float32); dye[..., 3] = 1
    s = make(pkg, 16, 16, Wd, Hd)
    s.writeField("dye", dye)
    s.config["BACK_COLOR"] = {"r": 30, "g": 60, "b": 200}
    for shading in (True, False):
        s.config["SHADING"] = shading
        got = s.render(w, h)
        assert bits_equal(got, oracle.display(dye, w, h, shading, (30 / 255, 60 / 255, 200 / 255))), shading
    img = s.textureToCanvas(got)
    assert img.dtype == np.uint8 and img.shape == (h, w, 4)
    # config.TRANSPARENT: checkerboard under the display on the screen, bare display into a capture target
    s.config["TRANSPARENT"] = True; s.canvas = {"width": w, "height": h}
    assert bits_equal(s.render(w, h), oracle.display(dye, w, h, False, background=oracle.BG_CHECKERBOARD))
    assert bits_equal(s.render(w, h, target=True), oracle.display(dye, w, h, False, background=oracle.BG_NONE))
    s.config["TRANSPARENT"] = False
    assert bits_equal(s.render(w, h), got)
    s.close()
    if (Wd, w) == (64, 128):
        g = golden("display_transparent_64x32_to_128x64")        # executed checkerboardShader + displayShader
        s = make(pkg, 16, 16, 64, 32); s.canvas = {"width": 128, "height": 64}
        s.writeField("dye", g["in_dye"]); s.config["TRANSPARENT"] = True
        assert bits_equal(s.render(128, 64), g["checker"]) and bits_equal(s.render(128, 64, target=True), g["bare"])
        s.close()
        g = golden("display_64_to_128")
        s = make(pkg, 16, 16, 64, 64)
        s.writeField("dye", g["in_dye"]); s.config["BACK_COLOR"] = {"r": 30, "g": 60, "b": 200}
        assert bits_equal(s.render(128, 128), g["shaded"])
        s.close()


@pytest.mark.parametrize("name", ["postfx_64_to_128", "postfx_48x32_to_50x75"])
def test_render_postfx_vs_oracle_and_executed_shaders(pkg, oracle, name):
    """render() with SHADING + BLOOM + SUNRAYS: bloom FBO and sunrays texture bit-identical to the
    oracle, every value of the final frame within the per-texel powf interval of display_model.py, and
    within the golden's tolerance of the executed reference shaders."""
    g = golden(name)
    Wd, Hd, w, h = (int(g[k]) for k in ("Wd", "Hd", "w", "h"))
    fxcfg = dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]))
    dither = g["dither"].astype(np.float32)
    s = make(pkg, 16, 16, Wd, Hd)
    s.writeField("dye", g["in_dye"])
    s.config.update(BLOOM=True, SUNRAYS=True, SHADING=True, BACK_COLOR={"r": 10, "g": 20, "b": 30}, **fxcfg)
    s.dithering = dither
    got = s.render(w, h)
    ref = oracle.render_postfx(g["in_dye"], w, h, dither, cfg=fxcfg, back_rgb=(10 / 255, 20 / 255, 30 / 255))
    assert bits_equal(s.last_bloom, ref["bloom"])
    assert bits_equal(s.last_sunrays, ref["sunrays"])
    d = DM.display(g["in_dye"], w, h, DM.ALL3, s.last_bloom, s.last_sunrays, dither, (10 / 255, 20 / 255, 30 / 255),
                   oracle.BG_COLOR, w / h)
    n, bad = G.check_display(got, d["lo"], d["hi"])           # powf: per texel, within POWF_ULP of pow
    assert n == 0, (n, bad)
    assert max_rel(got, g["target"]) < 3e-4
    assert bits_equal(s.readField("dye"), g["in_dye"])        # the mask scribbles on dye.write only (S:1300)
    s.close()


def half_every_pass(pkg, O, W, H, Wd, Hd):
    """Each pass of a half-storage handle against the oracle, rounded to fp16 after every blit."""
    v, dye, p = rand_fields(W, H, Wd, Hd, 77)
    v, dye, p = O.round_half(v), O.round_half(dye), O.round_half(p)
    s = make(pkg, W, H, Wd, Hd, flags=pkg.FLAG_HALF_STORAGE)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    assert bits_equal(s.readField("velocity"), v)                       # narrow + widen is the identity on fp16 values
    R = O.round_half
    s.pass_("curl"); c = s.readField("curl"); assert bits_equal(c, R(O.curl(v)))
    s.pass_("vorticity", DT); v2 = s.readField("velocity"); assert bits_equal(v2, R(O.vorticity(v, c, 30.0, DT)))
    s.pass_("divergence"); d = s.readField("divergence"); assert bits_equal(d, R(O.divergence(v2)))
    s.pass_("clear_pressure"); p1 = s.readField("pressure"); assert bits_equal(p1, R(O.clear(p, 0.8)))
    s.pass_("jacobi", 5); p2 = p1
    for _ in range(5):
        p2 = R(O.jacobi(p2, d, 1))
    assert bits_equal(s.readField("pressure"), p2)
    s.pass_("gradient_subtract"); v3 = s.readField("velocity"); assert bits_equal(v3, R(O.gradient_subtract(p2, v2)))
    s.pass_("advect_velocity", DT); v4 = s.readField("velocity"); assert bits_equal(v4, R(O.advect(v3, v3, DT, 0.2)))
    s.pass_("advect_dye", DT); assert bits_equal(s.readField("dye"), R(O.advect(v4, dye, DT, 1.0)))
    s.close()


def half_whole_steps(pkg, O, W, H, Wd, Hd):
    """Three whole steps (graph replay, 20 iterations) of a half-storage handle against the oracle's
    half mode, every field, then render() of the fp16 dye through the fp32 display shader."""
    R = O.round_half
    v, dye, p = rand_fields(W, H, Wd, Hd, 78)
    v, dye, p = R(v), R(dye), R(p)
    s = make(pkg, W, H, Wd, Hd, flags=pkg.FLAG_HALF_STORAGE)
    ref = O.OracleSim(W, H, Wd, Hd, half_storage=True)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    for _ in range(3):
        s.step(DT); ref.step(DT)
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert bits_equal(s.readField(n), getattr(ref, n)), n
    assert bits_equal(s.render(64, 64), O.display(ref.dye, 64, 64, True, (0.0, 0.0, 0.0)))
    s.close()


def test_half_storage_every_pass_and_whole_steps_bitwise_vs_oracle(pkg, oracle):
    """FLUID_FLAG_HALF_STORAGE: the reference's own storage format (half-float textures, S:138-147,
    S:986-1006): fp32 arithmetic, fp16 round-to-nearest-even on every pass write.  Per pass and for
    whole steps bit-identical to the oracle's half_storage mode (oracle_round_half after every blit)."""
    half_every_pass(pkg, oracle, 64, 48, 128, 96)
    half_whole_steps(pkg, oracle, 128, 128, 256, 256)


# half storage at every parity size and where the kernel choice changes: hs::jacobi8_kernel
# (W % 8 == 0, W >= 64) fetches across warps only when W/8 > 32; 264 has one live lane in the second
# warp, 520 several full warps and a partial one, 1024 four warps per row (the roofline_half_storage
# size); W = 100 (W % 8 = 4) runs the one-cell jacobi_scalar_kernel<hs::StoreHalf>
HALF_SIZES = SIZES + [(264, 40, 528, 80), (520, 33, 780, 50), (100, 60, 150, 90), (1024, 1024, 1024, 1024)]


@pytest.mark.parametrize("W,H,Wd,Hd", HALF_SIZES)
def test_half_storage_passes_and_steps_at_every_jacobi_width(pkg, oracle, W, H, Wd, Hd):
    """The same two checks as above at shapes that select each half-storage Jacobi path and reach
    hs::jacobi8_kernel's cross-warp fetches."""
    half_every_pass(pkg, oracle, W, H, Wd, Hd)
    half_whole_steps(pkg, oracle, W, H, Wd, Hd)


@pytest.mark.parametrize("src,dst", [((64, 48, 128, 96), (100, 75, 150, 113)),
                                     ((36, 20, 54, 30), (23, 41, 97, 31))])
def test_half_storage_resize_carries_state_like_resizeDoubleFBO(pkg, oracle, src, dst):
    """initFramebuffers() on a half-storage handle (fluid_resize): velocity and dye resampled with the
    LINEAR copy, then rounded to fp16 like the reference's half-float target; pressure, divergence
    and curl start over at zero.  Ragged sizes, up and down."""
    O = oracle
    R = O.round_half
    v, dye, p = (R(a) for a in rand_fields(*src, 41))
    s = make(pkg, *src, flags=pkg.FLAG_HALF_STORAGE)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    s._sizes = dst; s.initFramebuffers()
    W, H, Wd, Hd = dst
    assert s._dims("velocity")[:2] == (W, H) and s._dims("dye")[:2] == (Wd, Hd)
    assert bits_equal(s.readField("velocity"), R(O.resample(v, W, H)))
    assert bits_equal(s.readField("dye"), R(O.resample(dye, Wd, Hd)))
    for n in ("pressure", "divergence", "curl"):
        assert not s.readField(n).any(), n
    s.close()


def test_half_storage_vs_executed_reference_with_half_textures(pkg):
    """The closest thing to a real WebGL run this repository can produce: the executed reference
    shaders with LINEAR samplers and half-float textures (tests/golden/p4_linear_half_32.npz).
    The half-storage mode must land within 1e-3 of it after one step (its only differences: expf /
    LINEAR-weight last places ahead of the fp16 rounding) -- the fp32-storage mode is 4e-3 away."""
    g = golden("p4_linear_half_32")
    W, H, Wd, Hd = (int(g[k]) for k in ("W", "H", "Wd", "Hd"))
    s = make(pkg, W, H, Wd, Hd, flags=pkg.FLAG_HALF_STORAGE)
    for a in g["splats"]:
        s.splat(*[float(x) for x in a[:4]], tuple(float(x) for x in a[4:]))
    s.step(float(g["dt"]))
    for n in ("velocity", "dye", "pressure"):
        assert max_rel(s.readField(n), g[f"s1_{n}"]) < 1e-3, n
    s.close()
