"""The CPU oracle against the golden vectors cut by executing the reference's GLSL text
(tests/golden/make_golden.py -> oracle/glsl_exec.py).  Runs without a GPU."""
import numpy as np
import pytest

from conftest import bits_equal, golden, max_rel

PASS_FILES = ["pass_32x32_64x64", "pass_24x16_40x28", "pass_64x32_128x64", "pass_16x16_16x16"]
# exp() is implementation-defined in GLSL: numpy's and glibc's expf differ in the last place
SPLAT_TOL = 5e-7
# for non-power-of-two grids the rasteriser's interpolated vUv and (i+.5)/W differ by an ulp,
# which moves the bilinear taps' weights: value-level agreement only
NONPOW2_ADVECT_TOL = 2e-5


def _pow2(g):
    return all(int(g[k]) & (int(g[k]) - 1) == 0 for k in ("W", "H", "Wd", "Hd"))


@pytest.mark.parametrize("name", PASS_FILES)
def test_passes_match_reference_shaders(oracle, name):
    g = golden(name); O = oracle
    dt = float(g["dt"]); v = g["in_velocity"]; p = g["in_pressure"]; dye = g["in_dye"]
    W, H = int(g["W"]), int(g["H"])
    c = O.curl(v); assert bits_equal(c, g["curl"])
    v2 = O.vorticity(v, c, 30.0, dt); assert bits_equal(v2, g["vorticity"])
    d = O.divergence(v2); assert bits_equal(d, g["divergence"])
    p1 = O.clear(p, 0.8); assert bits_equal(p1, g["clear"])
    p2 = O.jacobi(p1, d, 1); assert bits_equal(p2, g["jacobi1"])
    p3 = O.jacobi(p2, d, 12); assert bits_equal(p3, g["jacobi13"])
    v3 = O.gradient_subtract(p3, v2); assert bits_equal(v3, g["gradient"])
    v4 = O.advect(v3, v3, dt, 0.2)
    d2 = O.advect(g["advect_velocity"], dye, dt, 1.0)
    if _pow2(g):
        assert bits_equal(v4, g["advect_velocity"]) and bits_equal(d2, g["advect_dye"])
    else:
        assert max_rel(v4, g["advect_velocity"]) < NONPOW2_ADVECT_TOL
        assert max_rel(d2, g["advect_dye"]) < NONPOW2_ADVECT_TOL
    sp = g["splat_args"]; rad = O.correct_radius(0.25, W / H)
    sv = O.splat(g["advect_velocity"], W / H, sp[0], sp[1], (sp[2], sp[3], 0.0), rad)
    sd = O.splat(g["advect_dye"], W / H, sp[0], sp[1], tuple(sp[4:]), rad)
    assert max_rel(sv, g["splat_velocity"]) < SPLAT_TOL
    assert max_rel(sd, g["splat_dye"]) < SPLAT_TOL
    assert np.all(sd[..., 3] == 1.0)       # splat forces alpha to 1 (S:742)


def _run_scenario(O, g, sim_cls):
    cfg = dict(zip([str(k) for k in g["config_keys"]], g["config_vals"]))
    s = sim_cls(int(g["W"]), int(g["H"]), int(g["Wd"]), int(g["Hd"]))
    s.CURL = float(cfg["CURL"]); s.PRESSURE_ITERATIONS = int(cfg["PRESSURE_ITERATIONS"])
    for a in g["splats"]:
        s.splat(*[float(x) for x in a])
    return s


@pytest.mark.parametrize("name,tol", [("step_curl30_32", 1e-5), ("step_curl30_48x32", 5e-5),  # 48 is not a power of two: vUv rounding
                                      ("step_curl0_32", 2e-5)])
def test_full_step_matches_reference_orchestration(oracle, name, tol):
    """P2 / P3 of SURVEY §8c: short horizon with CURL=30, 20 steps with CURL=0."""
    g = golden(name); O = oracle
    s = _run_scenario(O, g, O.OracleSim)
    assert max_rel(s.velocity, g["init_velocity"]) < SPLAT_TOL
    assert max_rel(s.dye, g["init_dye"]) < SPLAT_TOL
    steps = int(g["steps"])
    for k in range(1, steps + 1):
        s.step(float(g["dt"]))
        if k in (1, 2, steps):
            for n in ("velocity", "dye", "pressure", "divergence", "curl"):
                assert max_rel(getattr(s, n), g[f"s{k}_{n}"]) < tol, (k, n)


def test_c_step_equals_python_orchestration(oracle):
    """oracle_sim_step (C, used for CPU timing) == the per-pass Python orchestration, bitwise."""
    O = oracle; g = golden("step_curl30_32")
    a = _run_scenario(O, g, O.OracleSim)
    b = O.OracleSimC(32, 32, 64, 64)
    for sp in g["splats"]:
        b.splat(*[float(x) for x in sp])
    for _ in range(3):
        a.step(float(g["dt"])); b.step(float(g["dt"]))
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert bits_equal(getattr(a, n), b.field(n)), n
    b.close()


def test_c_splat_equals_python_splat_when_the_radius_depends_on_the_aspect_narrowing(oracle):
    """oracle_sim_splat == OracleSim.splat, bitwise, on a 142x100 grid: correctRadius multiplies by the
    aspect in double, and float32(142 / 100) widened back to double gives a radius one ulp lower."""
    O = oracle
    a = O.OracleSim(142, 100, 142, 100)
    b = O.OracleSimC(142, 100, 142, 100)
    for rec in ((0.3, 0.6, 123.0, -456.0, 0.5, 0.2, 0.9), (0.71, 0.2, -40.0, 7.0, 1.2, -0.3, 0.05)):
        a.splat(*rec); b.splat(*rec)
    for n in ("velocity", "dye"):
        assert bits_equal(getattr(a, n), b.field(n)), n
    b.close()


def test_p4_report_distance_to_desktop_webgl(oracle, capsys):
    """REPORT ONLY (never gates): distance from the fp32 oracle to the reference as a desktop
    browser runs it (LINEAR samplers, half-float textures).  Bounds are loose sanity rails."""
    O = oracle
    for name, bound in (("p4_linear_fp32_32", 1e-4), ("p4_linear_half_32", 5e-2)):
        g = golden(name)
        s = _run_scenario(O, g, O.OracleSim)
        s.step(float(g["dt"]))
        e = {n: max_rel(getattr(s, n), g[f"s1_{n}"]) for n in ("velocity", "dye", "pressure")}
        with capsys.disabled():
            print(f"\n[P4] {name}: 1-step max-rel vs fp32 oracle: " +
                  ", ".join(f"{k}={v:.2e}" for k, v in e.items()))
        assert max(e.values()) < bound


@pytest.mark.parametrize("name,exact", [("display_64_to_128", True), ("display_40x28_to_50x30", False)])
def test_display_matches_executed_reference_shaders(oracle, name, exact):
    """render() with bloom / sunrays off (SURVEY §8f rank 1, first half) against the executed
    colorShader + displayShaderSource + blend."""
    g = golden(name); O = oracle
    back = tuple(float(x) / 255 for x in g["back"])
    for key, shading in (("shaded", True), ("flat", False)):
        got = O.display(g["in_dye"], int(g["w"]), int(g["h"]), shading, back)
        if exact:
            assert bits_equal(got, g[key]), key
        else:
            assert max_rel(got, g[key]) < 1e-5, key


@pytest.mark.parametrize("name,pow2", [("postfx_64_to_128", True), ("postfx_48x32_to_50x75", False)])
def test_postfx_chain_matches_executed_reference_shaders(oracle, name, pow2):
    """Oracle side of SURVEY 8f rank 1, second half (no CUDA yet): bloom prefilter + 7-level pyramid
    with additive up-sampling + final, sunrays mask / 16-step march / separable blur, and the full
    display shader (SHADING + BLOOM + SUNRAYS, dithering texture, gamma), against the executed
    shaders.  Power-of-two sizes: the bloom chain and the mask are bit-identical; the sunrays FBO is
    48 wide here (196 by default — never a power of two) and pow() is implementation-defined, hence the small tolerances."""
    g = golden(name); O = oracle
    dither = g["dither"].astype(np.float32)
    r = O.render_postfx(g["in_dye"], int(g["w"]), int(g["h"]), dither,
                        cfg=dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"])),
                        back_rgb=tuple(float(x) / 255 for x in g["back"]))
    n = len([k for k in g.files if k.startswith("pyr")])
    assert len(r["pyramid"]) == n
    if pow2:
        assert bits_equal(r["bloom"], g["bloom"]) and bits_equal(r["mask_alpha"], g["mask_alpha"])
        assert all(bits_equal(r["pyramid"][k], g[f"pyr{k}"]) for k in range(n))
        assert max_rel(r["sunrays"], g["sunrays"]) < 2e-6 and max_rel(r["target"], g["target"]) < 2e-6
    else:
        tol = 3e-4                      # vUv rounding on ragged grids, amplified by br * 20 in the mask
        assert max_rel(r["bloom"], g["bloom"]) < tol and max_rel(r["mask_alpha"], g["mask_alpha"]) < tol
        assert max_rel(r["sunrays"], g["sunrays"]) < tol and max_rel(r["target"], g["target"]) < tol


@pytest.mark.parametrize("name,exact", [("resample_dye_64_to_32", True), ("resample_v_32_to_48", False),
                                        ("resample_dye_40x28_to_64x48", False)])
def test_resample_matches_executed_copy_shader(oracle, name, exact):
    """resizeFBO (S:1108-1114): oracle_resample against the executed copyShader drawn through a
    LINEAR sampler.  Power-of-two sizes: bit-identical; otherwise the rasteriser's interpolated vUv
    differs from (i+.5)/W in the last place, which moves the weights (value-level agreement)."""
    g = golden(name)
    got = oracle.resample(g["src"], int(g["Wd"]), int(g["Hd"]))
    if exact:
        assert bits_equal(got, g["linear"])
    else:
        assert max_rel(got, g["linear"]) < 2e-6


def test_config0_matches_reference_orchestration(oracle):
    """BASELINE configs[0] (128x128 sim / 256x256 dye, 20 Jacobi iterations): two whole steps after
    multipleSplats(5), against the executed reference shaders.  Step 1 at the P2 tolerance 1e-5
    (SURVEY §8c); step 2 at 5e-5: the only difference between the two runs is exp()'s last place in
    the splats (1.5e-7 of the field), which vorticity confinement's force/(|force|+1e-4) amplifies
    by ~10x per step on the divergence (measured: 1.7e-6 after one step, 2.5e-5 after two)."""
    g = golden("config0_128_256"); O = oracle
    s = _run_scenario(O, g, O.OracleSim)
    for k, tol in ((1, 1e-5), (2, 5e-5)):
        s.step(float(g["dt"]))
        for n in ("velocity", "dye", "pressure", "divergence", "curl"):
            assert max_rel(getattr(s, n), g[f"s{k}_{n}"]) < tol, (k, n)


def test_transparent_display_matches_executed_shaders(oracle):
    """config.TRANSPARENT (S:1303-1312): checkerboardShader under the display on the screen, the bare
    un-blended display into a capture target -- against the executed reference shaders, bitwise."""
    g = golden("display_transparent_64x32_to_128x64")
    assert bits_equal(oracle.display(g["in_dye"], 128, 64, True, background=oracle.BG_CHECKERBOARD), g["checker"])
    assert bits_equal(oracle.display(g["in_dye"], 128, 64, True, background=oracle.BG_NONE), g["bare"])
