"""FLUID_FLAG_LINEAR_ADVECTION on one H100: the advection passes and whole steps against the fp32 model
of tests/linear_advection_model.py and the executed LINEAR shaders (linear_*.npz), bit for bit.

Which kernel runs is the MANUAL handle's rule (fluid.cu do_advect_velocity / do_advect_dye): the 4-cell
LINEAR kernels on fp32 power-of-two grids at least 128 wide without FLUID_FLAG_TILED_PASSES, the one-cell
LINEAR kernels (fp32 or fp16 storage, POW2 or ragged) everywhere else.  FLUID_STAT_ADVECT4_LAUNCHES
says which ran."""
import ctypes as C

import numpy as np
import pytest

import linear_advection_model as M
from conftest import bits_equal, golden, max_rel
from sim_harness import Arena, check, exp_tiled, jacobi_plan, make, nasty_fields, pressure_swaps, rand_fields, same_bits
from sim_harness import pkg, torch  # noqa: F401 -- fixtures

pytestmark = pytest.mark.gpu

DT = 0.016666
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
ADVECT_SHAPES = [(256, 256, 256, 256, False), (128, 128, 256, 256, False), (64, 64, 128, 128, False),
                 (64, 64, 64, 64, False), (36, 20, 54, 30, False), (1, 9, 3, 27, False), (9, 1, 27, 3, False),
                 (256, 256, 256, 256, True)]


def pow2(n):
    return n & (n - 1) == 0


def advect4_expected(W, H, Wd, Hd, half, tiled):
    """(velocity, dye) pass: 1 when the 4-cell kernel is the one the size rule picks."""
    fast = not half and not tiled and all(pow2(n) for n in (W, H))
    return int(fast and W >= 128), int(fast and pow2(Wd) and pow2(Hd) and Wd >= 128)


def linear_data(O, W, H, Wd, Hd, data):
    rng = np.random.default_rng(W * 5 + Wd + len(data))
    if data == "random":
        v, dye, _ = rand_fields(W, H, Wd, Hd, W * 3 + Hd)
    elif data == "far":                        # back-traces up to ~1700 texels outside the grid
        tiles = (-(-H // 4), -(-W // 8))
        mag = np.repeat(np.repeat(10.0 ** rng.uniform(0, 5, tiles), 4, 0), 8, 1)[:H, :W, None]
        v = (rng.uniform(-1, 1, (H, W, 2)) * mag).astype(np.float32)
        dye = exp_tiled((Hd, Wd, 4), W + H, tile=(4, 8))
    else:                                      # +-0, subnormals, +-inf and NaN in velocity and dye
        v, dye, _ = nasty_fields(W, H, Wd, Hd, W + Hd)
        if W > 2 and H > 1:                    # an inf neighbour right of a finite cell-centre texel
            v[H // 2, W // 2] = (1.5, -2.0)
            v[H // 2, W // 2 + 1] = (np.inf, 3.0)
    return v, dye


@pytest.mark.parametrize("data", ["random", "far", "special"])
@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
@pytest.mark.parametrize("W,H,Wd,Hd,tiled", ADVECT_SHAPES)
def test_advection_passes_vs_model(pkg, oracle, W, H, Wd, Hd, tiled, half, data):
    O = oracle
    R = O.round_half if half else (lambda a: a)
    v, dye = (R(a) for a in linear_data(O, W, H, Wd, Hd, data))
    flags = pkg.FLAG_LINEAR_ADVECTION | (pkg.FLAG_HALF_STORAGE if half else 0) | (pkg.FLAG_TILED_PASSES if tiled else 0)
    s = make(pkg, W, H, Wd, Hd, flags=flags)
    ev, ed = advect4_expected(W, H, Wd, Hd, half, tiled)
    for diss in (0.0, 0.2, 1.0, 4.0):
        s.config["VELOCITY_DISSIPATION"] = diss; s.config["DENSITY_DISSIPATION"] = diss
        s.writeField("velocity", v); s.writeField("dye", dye)
        n0 = s.stat("advect4_launches")
        s.pass_("advect_velocity", DT); v2 = s.readField("velocity")
        n1 = s.stat("advect4_launches")
        assert n1 - n0 == ev, diss
        assert same_bits(v2, R(M.advect(v, v, DT, diss))), diss
        s.pass_("advect_dye", DT)
        assert s.stat("advect4_launches") - n1 == ed, diss
        assert same_bits(s.readField("dye"), R(M.advect(v2, dye, DT, diss))), diss
    s.close()


STEP_SHAPES = [(32, 32, 64, 64), (264, 40, 528, 80), (1024, 1024, 2048, 2048)]
MODES = {"graph": 0, "no_graph": "FLAG_NO_GRAPH", "unfused": "FLAG_NO_GRAPH|FLAG_UNFUSED", "tiled": "FLAG_TILED_PASSES"}


def mode_flags(pkg, mode):
    return 0 if not MODES[mode] else sum(getattr(pkg, f) for f in MODES[mode].split("|"))


def step_once(pkg, W, H, Wd, Hd, flags, fields, iters=20):
    s = make(pkg, W, H, Wd, Hd, flags=flags, PRESSURE_ITERATIONS=iters)
    for n, a in fields.items():
        s.writeField(n, a)
    n0 = s.launch_count()
    s.step(DT)
    out = {n: s.readField(n) for n in FIELDS}
    launches = s.launch_count() - n0
    s.close()
    return out, launches


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
@pytest.mark.parametrize("W,H,Wd,Hd", STEP_SHAPES)
def test_whole_step_every_mode_vs_model(pkg, oracle, W, H, Wd, Hd, half):
    """Graph, NO_GRAPH, UNFUSED and TILED_PASSES give the same bits as each other and as LinearOracleSim,
    and each launches what a MANUAL twin handle launches."""
    O = oracle
    O.use_all_cores()
    R = O.round_half if half else (lambda a: a)
    v, dye, p = (R(a) for a in rand_fields(W, H, Wd, Hd, W + Hd))
    ref = M.LinearOracleSim(W, H, Wd, Hd, half_storage=half)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    ref.step(DT)
    base = pkg.FLAG_HALF_STORAGE if half else 0
    for mode in MODES:
        f = base | mode_flags(pkg, mode)
        got, n_lin = step_once(pkg, W, H, Wd, Hd, f | pkg.FLAG_LINEAR_ADVECTION, {"velocity": v, "dye": dye, "pressure": p})
        _, n_man = step_once(pkg, W, H, Wd, Hd, f, {"velocity": v, "dye": dye, "pressure": p})
        assert n_lin == n_man, (mode, n_lin, n_man)
        for n in FIELDS:
            assert bits_equal(got[n], getattr(ref, n)), (mode, n)


def test_headline_step_4096(pkg, oracle):
    """One 4096^2 / 4096^2 fp32 step with 50 pressure iterations: the 4-cell LINEAR kernels (velocity and
    dye<SAME>), bit for bit."""
    O = oracle
    O.use_all_cores()
    W = 4096
    v, dye, p = rand_fields(W, W, W, W, 4096)
    s = make(pkg, W, W, W, W, flags=pkg.FLAG_LINEAR_ADVECTION, PRESSURE_ITERATIONS=50)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    a0 = s.stat("advect4_launches")
    s.step(DT)
    assert s.stat("advect4_launches") - a0 == 2
    got = {n: s.readField(n) for n in FIELDS}
    s.close()
    ref = M.LinearOracleSim(W, W, W, W, PRESSURE_ITERATIONS=50)
    ref.velocity, ref.dye, ref.pressure = v, dye, p
    ref.step(DT)
    for n in FIELDS:
        assert bits_equal(got[n], getattr(ref, n)), n


PASS = ["32x32_64x64", "64x32_128x64", "16x16_16x16", "128x128_256x256"]


@pytest.mark.parametrize("tag", ["fp32", "half"])
@pytest.mark.parametrize("shape", PASS)
def test_passes_vs_executed_linear_shaders(pkg, tag, shape):
    g = golden(f"linear_pass_{tag}_{shape}")
    W, H, Wd, Hd = (int(g[k]) for k in ("W", "H", "Wd", "Hd"))
    flags = pkg.FLAG_LINEAR_ADVECTION | (pkg.FLAG_HALF_STORAGE if tag == "half" else 0)
    s = make(pkg, W, H, Wd, Hd, flags=flags)
    for pre in ("", "special_"):
        if pre + "in_velocity" not in g:
            continue
        s.writeField("velocity", g[pre + "in_velocity"]); s.writeField("dye", g[pre + "in_dye"])
        s.pass_("advect_velocity", float(g["dt"]))
        assert same_bits(s.readField("velocity"), g[pre + "advect_velocity"]), pre
        s.pass_("advect_dye", float(g["dt"]))
        assert same_bits(s.readField("dye"), g[pre + "advect_dye"]), pre
    s.close()


@pytest.mark.parametrize("tag", ["fp32", "half"])
@pytest.mark.parametrize("shape", ["32x32_64x64", "64x32_128x64"])
def test_steps_vs_executed_linear_shaders(pkg, tag, shape):
    g = golden(f"linear_step_{tag}_{shape}")
    W, H, Wd, Hd = (int(g[k]) for k in ("W", "H", "Wd", "Hd"))
    flags = pkg.FLAG_LINEAR_ADVECTION | (pkg.FLAG_HALF_STORAGE if tag == "half" else 0)
    s = make(pkg, W, H, Wd, Hd, flags=flags, CURL=float(g["curl"]), PRESSURE_ITERATIONS=int(g["pressure_iterations"]))
    s.writeField("velocity", g["init_velocity"]); s.writeField("dye", g["init_dye"])
    s.writeField("pressure", np.zeros((H, W), np.float32))
    for k in range(1, int(g["steps"]) + 1):
        s.step(float(g["dt"]))
        for n in FIELDS:
            assert bits_equal(s.readField(n), g[f"s{k}_{n}"]), (k, n)
    s.close()


def test_desktop_configuration(pkg, capsys):
    """HALF_STORAGE | HALF_POSTFX | LINEAR_ADVECTION, the desktop browser's frame and step: the splats of
    p4_linear_half_32 and one step land within the CPU gate of the same scenario."""
    g = golden("p4_linear_half_32")
    flags = pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX | pkg.FLAG_LINEAR_ADVECTION
    cfg = dict(zip([str(k) for k in g["config_keys"]], g["config_vals"]))
    s = make(pkg, int(g["W"]), int(g["H"]), int(g["Wd"]), int(g["Hd"]), flags=flags,
             CURL=float(cfg["CURL"]), PRESSURE_ITERATIONS=int(cfg["PRESSURE_ITERATIONS"]))
    for a in g["splats"]:
        a = [float(x) for x in a]
        s.splat(a[0], a[1], a[2], a[3], tuple(a[4:7]))
    s.step(float(g["dt"]))
    e = {n: max_rel(s.readField(n), g[f"s1_{n}"]) for n in ("velocity", "dye", "pressure")}
    s.close()
    with capsys.disabled():
        print("\n[desktop configuration] 1-step max-rel vs executed shaders: " + ", ".join(f"{k}={v:.2e}" for k, v in e.items()))
    assert max(e.values()) < M.P4_HALF_GATE


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
def test_arena_guard(pkg, torch, oracle, half):
    """Both LINEAR passes and one whole step write nothing outside their outputs, under both poisons."""
    O = oracle
    W, H, Wd, Hd = (256, 256, 256, 256) if not half else (100, 60, 150, 90)
    R = O.round_half if half else (lambda a: a)
    v, dye, p = (R(a) for a in rand_fields(W, H, Wd, Hd, 77))
    flags = pkg.FLAG_LINEAR_ADVECTION | (pkg.FLAG_HALF_STORAGE if half else 0)
    s = make(pkg, W, H, Wd, Hd, flags=flags)
    g = Arena(torch, s, half)
    v4 = R(M.advect(v, v, DT, 0.2))
    check(g, "advect_velocity", lambda: s.pass_("advect_velocity", DT), {"velocity": v}, {"velocity": v4},
          swaps=("velocity",))
    check(g, "advect_dye", lambda: s.pass_("advect_dye", DT), {"velocity": v4, "dye": dye},
          {"dye": R(M.advect(v4, dye, DT, 1.0))}, swaps=("dye",))
    ref = M.LinearOracleSim(W, H, Wd, Hd, half_storage=half)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    ref.step(DT)
    swaps = ("velocity", "dye") + pressure_swaps(len(jacobi_plan(W, H, half, 20)) + half)
    check(g, "step", lambda: s.step(DT), {"velocity": v, "dye": dye, "pressure": p},
          {n: getattr(ref, n) for n in FIELDS}, swaps=swaps)
    s.close()


def test_resize_then_step(pkg, oracle):
    """fluid_resize on a LINEAR handle (ragged up, then down) and a step after each, bit for bit."""
    O = oracle
    s = make(pkg, 64, 64, 128, 128, flags=pkg.FLAG_LINEAR_ADVECTION)
    v, dye, _ = rand_fields(64, 64, 128, 128, 9)
    s.writeField("velocity", v); s.writeField("dye", dye)
    for sizes in [(72, 40, 150, 90), (20, 30, 40, 28)]:
        v0, d0 = s.readField("velocity"), s.readField("dye")
        s._sizes = sizes; s.initFramebuffers()
        W, H, Wd, Hd = sizes
        v1, d1 = O.resample(v0, W, H), O.resample(d0, Wd, Hd)
        assert bits_equal(s.readField("velocity"), v1) and bits_equal(s.readField("dye"), d1), sizes
        ref = M.LinearOracleSim(W, H, Wd, Hd)
        ref.velocity, ref.dye = v1, d1
        ref.pressure = s.readField("pressure")
        ref.step(DT); s.step(DT)
        for n in FIELDS:
            assert bits_equal(s.readField(n), getattr(ref, n)), (sizes, n)
    s.close()


def _create(pkg, flags, slab=False):
    L = pkg.lib()
    cfg = pkg._lib.Config()
    L.fluid_config_default(C.byref(cfg))
    cfg.sim_w, cfg.sim_h, cfg.dye_w, cfg.dye_h = 64, 64, 64, 64
    cfg.flags = flags
    h = C.c_void_p()
    if slab:
        uid = C.create_string_buffer(128)
        rc = L.fluid_create_slab(C.byref(cfg), 0, 2, uid, 128, C.byref(h))
    else:
        rc = L.fluid_create(C.byref(cfg), C.byref(h))
    msg = L.fluid_last_error(None)
    return rc, h, (msg.decode() if isinstance(msg, bytes) else str(msg))


def test_refusals(pkg):
    rc, h, msg = _create(pkg, pkg.FLAG_LINEAR_ADVECTION | pkg.FLAG_NEAREST_FILTERING)
    assert rc == -1 and not h.value and "NEAREST_FILTERING" in msg, msg
    rc, h, msg = _create(pkg, pkg.FLAG_LINEAR_ADVECTION, slab=True)
    assert rc == -1 and not h.value and "single-GPU" in msg, msg
    rc, h, _ = _create(pkg, pkg.FLAG_LINEAR_ADVECTION)
    assert rc == 0 and h.value
    pkg.lib().fluid_destroy(h)
