"""FLUID_FLAG_LINEAR_ADVECTION on the CPU: the fp32 model of tests/linear_advection_model.py against the
executed LINEAR advection shaders (tests/golden/make_golden_linear.py -> linear_*.npz), the goldens'
power to tell the two advection shaders apart, and the distance left to the desktop-browser scenarios."""
import os
import re

import numpy as np
import pytest

import linear_advection_model as M
from conftest import ROOT, bits_equal, golden, max_rel
from sim_harness import same_bits

PASS = ["32x32_64x64", "64x32_128x64", "16x16_16x16", "128x128_256x256", "24x16_40x28"]
STEP = ["32x32_64x64", "64x32_128x64"]
TAGS = ["fp32", "half"]
RAGGED = "24x16_40x28"
NONPOW2_ADVECT_TOL = 2e-5       # the MANUAL goldens' bound for the library's (i + .5) / n against the rasteriser's vUv
NONPOW2_ADVECT_TOL_HALF = 1e-3  # the same ulp of vUv, seen through fp16 storage: one fp16 ulp (2^-10) of the field's largest value


def store(half):
    from oracle import oracle as O
    return O.round_half if half else (lambda a: a)


def run_pass(g, pre="", **kw):
    """advect velocity, then dye by the golden's advected velocity (the reference's order, S:1275-1293)."""
    R = store(bool(g["half"])); dt = float(g["dt"])
    v = g[pre + "in_velocity"]
    v2 = R(M.advect(v, v, dt, float(g["velocity_dissipation"]), **kw))
    d2 = R(M.advect(g[pre + "advect_velocity"], g[pre + "in_dye"], dt, float(g["density_dissipation"]), **kw))
    return v2, d2


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("shape", PASS)
def test_model_matches_executed_linear_shader_per_pass(oracle, tag, shape, capsys):
    """Bit for bit on power-of-two shapes, the non-finite cases included.  On the ragged shape the
    library's cell centres (i + .5) / n and the rasteriser's vUv differ by an ulp: bit for bit with the
    rasteriser's vUv, within the MANUAL goldens' tolerance with the library's (worst distance printed)."""
    g = golden(f"linear_pass_{tag}_{shape}")
    v2, d2 = run_pass(g)
    if shape != RAGGED:
        assert bits_equal(v2, g["advect_velocity"]) and bits_equal(d2, g["advect_dye"])
        if "special_in_velocity" in g:
            sv, sd = run_pass(g, "special_")
            assert np.isnan(g["special_advect_velocity"]).any() and np.isinf(g["special_in_velocity"]).any()
            assert same_bits(sv, g["special_advect_velocity"]) and same_bits(sd, g["special_advect_dye"])
        return
    rv, rd = run_pass(g, uv="raster")
    assert bits_equal(rv, g["advect_velocity"]) and bits_equal(rd, g["advect_dye"])
    ev, ed = max_rel(v2, g["advect_velocity"]), max_rel(d2, g["advect_dye"])
    with capsys.disabled():
        print(f"\n[linear advection {tag} {shape}] library cell centres vs executed vUv: velocity {ev:.2e}, dye {ed:.2e}")
    tol = NONPOW2_ADVECT_TOL_HALF if tag == "half" else NONPOW2_ADVECT_TOL
    assert ev < tol and ed < tol


def run_steps(g, sim_cls=M.LinearOracleSim):
    W, H, Wd, Hd = (int(g[k]) for k in ("W", "H", "Wd", "Hd"))
    s = sim_cls(W, H, Wd, Hd, half_storage=bool(g["half"]), CURL=float(g["curl"]),
                PRESSURE_ITERATIONS=int(g["pressure_iterations"]))
    s.velocity = g["init_velocity"].copy(); s.dye = g["init_dye"].copy()
    out = []
    for _ in range(int(g["steps"])):
        s.step(float(g["dt"]))
        out.append({n: getattr(s, n).copy() for n in ("velocity", "dye", "pressure", "divergence", "curl")})
    return out


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("shape", STEP)
def test_linear_oracle_sim_matches_executed_steps(oracle, tag, shape):
    """Two whole steps from written fields (no splats, so no expf): every field bit for bit."""
    g = golden(f"linear_step_{tag}_{shape}")
    for k, f in enumerate(run_steps(g), 1):
        for n, a in f.items():
            assert bits_equal(a, g[f"s{k}_{n}"]), (k, n)


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("shape", PASS)
def test_goldens_tell_the_advection_shaders_apart(oracle, tag, shape):
    """The MANUAL_FILTERING advection (oracle.advect) differs from every LINEAR golden in at least one texel."""
    O = oracle
    g = golden(f"linear_pass_{tag}_{shape}")
    R = store(tag == "half"); dt = float(g["dt"]); v = g["in_velocity"]
    mv = R(O.advect(v, v, dt, 0.2))
    md = R(O.advect(g["advect_velocity"], g["in_dye"], dt, 1.0))
    assert not (bits_equal(mv, g["advect_velocity"]) and bits_equal(md, g["advect_dye"]))


def _rejected(**mutant):
    """Does test 1 or 2 above fail for the model with this mutation?  Per-pass goldens are compared the
    way those tests compare them (ragged: with the rasteriser's vUv, bit for bit)."""
    for tag in TAGS:
        for shape in PASS:
            g = golden(f"linear_pass_{tag}_{shape}")
            kw = dict(mutant, uv="raster") if shape == RAGGED else mutant
            v2, d2 = run_pass(g, **kw)
            if not (bits_equal(v2, g["advect_velocity"]) and bits_equal(d2, g["advect_dye"])):
                return True
            if "special_in_velocity" in g:
                sv, sd = run_pass(g, "special_", **kw)
                if not (same_bits(sv, g["special_advect_velocity"]) and same_bits(sd, g["special_advect_dye"])):
                    return True
    return False


@pytest.mark.parametrize("mutant", [dict(weights="mix"), dict(coord="uvts"), dict(own_texel=True)],
                         ids=["mix_of_mix_weights", "uv_over_ts_coordinate", "own_texel_velocity_sample"])
def test_goldens_reject_each_mutant(oracle, mutant):
    assert _rejected(**mutant)


def test_own_texel_mutant_is_caught_only_by_a_non_finite_neighbour(oracle):
    """On power-of-two grids the cell-centre weights are (1, 0, 0, 0): the own texel gives the same bits
    for finite fields, and NaN where 0 * inf enters (the special_* cases)."""
    g = golden("linear_pass_fp32_32x32_64x64")
    a, _ = run_pass(g, own_texel=True)
    assert bits_equal(a, g["advect_velocity"])
    b, _ = run_pass(g, "special_", own_texel=True)
    assert not same_bits(b, g["special_advect_velocity"])


@pytest.mark.parametrize("name,gate", [("p4_linear_fp32_32", 1e-5), ("p4_linear_half_32", M.P4_HALF_GATE)])
def test_p4_desktop_scenarios_after_one_step(oracle, name, gate, capsys):
    """The desktop-browser scenarios (8 splats, LINEAR samplers, fp32 or fp16 textures) one step on.  With
    LINEAR advection only the splats' expf can differ from the executed shaders (numpy's against glibc's,
    last places).  Measured: fp32 2.2e-6 (dye; velocity 1.3e-6, pressure 1.1e-7), gated at 1e-5, the MANUAL
    executed-reference bound; half 0 in every field (fp16 storage rounds the expf differences away), gated
    at 1e-6.  These scenarios are smooth splats on power-of-two grids, where the MANUAL oracle lands equally
    close: the per-pass and step goldens above are what tell the two shaders apart."""
    g = golden(name)
    s = M.LinearOracleSim(int(g["W"]), int(g["H"]), int(g["Wd"]), int(g["Hd"]), half_storage="half" in name)
    cfg = dict(zip([str(k) for k in g["config_keys"]], g["config_vals"]))
    s.CURL = float(cfg["CURL"]); s.PRESSURE_ITERATIONS = int(cfg["PRESSURE_ITERATIONS"])
    for a in g["splats"]:
        s.splat(*[float(x) for x in a])
    s.step(float(g["dt"]))
    e = {n: max_rel(getattr(s, n), g[f"s1_{n}"]) for n in ("velocity", "dye", "pressure")}
    with capsys.disabled():
        print(f"\n[P4 linear] {name}: 1-step max-rel vs executed shaders: " + ", ".join(f"{k}={v:.2e}" for k, v in e.items()))
    assert max(e.values()) < gate


def test_flag_value_is_the_same_everywhere():
    import webgl_fluid_simulation_b200 as pkg
    h = open(os.path.join(ROOT, "include", "fluid.h")).read()
    js = open(os.path.join(ROOT, "webgl_fluid_simulation_b200", "js", "fluid-sim.js")).read()
    c = int(re.search(r"#define FLUID_FLAG_LINEAR_ADVECTION (0x[0-9a-fA-F]+)u", h).group(1), 16)
    j = int(re.search(r"LINEAR_ADVECTION: (0x[0-9a-fA-F]+)", js).group(1), 16)
    assert c == j == pkg.FLAG_LINEAR_ADVECTION == 0x80
    s = int(re.search(r"FLUID_STAT_ADVECT4_LAUNCHES = (\d+)", h).group(1))
    assert s == pkg._lib.STAT["advect4_launches"] == int(re.search(r"advect4Launches: (\d+)", js).group(1))
