"""Every single-GPU entry point writes only its outputs inside the field arena.

All fields of a handle live in one allocation (tests/arena_model.py), so a store past a field's last row
lands in its slot's padding or, where the extent is a multiple of 2 MiB, in the next slot; a kernel that
writes an input or a slot it should only read, or forgets to store a cell of its write slot, leaves
values that the next pass may overwrite before anyone reads them.  Parity tests read fields through
fluid_read, which sees only the extents, and memcheck sees only the allocation.

Each call here runs twice on one handle, once with every arena byte that is not an input extent set to
0xFF (NaN in fp32 and fp16) and once with 0x3C (fp32 0.0115, fp16 1.06: a finite value that fmaxf / fminf
do not drop).  Around each run the whole arena [0, L.bytes) is snapshotted on the device through its
__cuda_array_interface__ alias, and nothing outside arena_model.may_change may move; the slot parity
comes from fluid_device_ptr before and after.  The outputs must equal the oracle (splats: inside the
splat_model interval; frames: the display models) and be bit-identical between the two poisons.  The
size-selected kernels are pinned with fluid_stat where a counter tells them apart."""
import numpy as np
import pytest

import arena_model as A
import display_harness as DH
import display_model as DM
import splat_model as SM
from conftest import bits_equal
from sim_harness import (POISONS, STREAM_SHAPES, Arena, check, delta, jacobi_plan, make, nasty_records, near_max_patch,
                         pressure_swaps, rand_fields, same_bits)
from sim_harness import pkg, torch  # noqa: F401 -- fixtures

pytestmark = pytest.mark.gpu
DT = 0.016666
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
FLUID_ERR_NOMEM = -6


def every_pass(pkg, torch, O, W, H, Wd, Hd, half, jacobi_iters=(1, 13)):
    """Each fluid_pass_* under both poisons against the oracle (fp16-rounded after every blit in half
    storage), then fluid_write / fluid_read of every field."""
    R = O.round_half if half else (lambda a: a)
    s = make(pkg, W, H, Wd, Hd, flags=pkg.FLAG_HALF_STORAGE if half else 0)
    g = Arena(torch, s, half)
    v, dye, p = (R(a) for a in rand_fields(W, H, Wd, Hd, W * 7 + H))
    P = s.pass_
    c = R(O.curl(v))
    check(g, "curl", lambda: P("curl"), {"velocity": v}, {"curl": c}, swaps=())
    v2 = R(O.vorticity(v, c, 30.0, DT))
    check(g, "vorticity", lambda: P("vorticity", DT), {"velocity": v, "curl": c}, {"velocity": v2}, swaps=("velocity",))
    d = R(O.divergence(v2))
    check(g, "divergence", lambda: P("divergence"), {"velocity": v2}, {"divergence": d}, swaps=())
    p1 = R(O.clear(p, 0.8))
    check(g, "clear_pressure", lambda: P("clear_pressure"), {"pressure": p}, {"pressure": p1}, swaps=("pressure",))

    def jac(q, n):
        if not half:
            return O.jacobi(q, d, n)
        for _ in range(n):
            q = R(O.jacobi(q, d, 1))
        return q
    for n in jacobi_iters:
        want = jac(p1, n)
        plan = jacobi_plan(W, H, half, n)
        launches = delta(s, "jacobi_launches", lambda: check(g, "jacobi", lambda: P("jacobi", n),
                                                             {"pressure": p1, "divergence": d}, {"pressure": want},
                                                             swaps=pressure_swaps(len(plan))))
        assert launches == 2 * len(plan), (n, launches)
    p3 = want
    v3 = R(O.gradient_subtract(p3, v2))
    check(g, "gradient_subtract", lambda: P("gradient_subtract"), {"pressure": p3, "velocity": v2}, {"velocity": v3},
          swaps=("velocity",))
    v4 = R(O.advect(v3, v3, DT, 0.2))
    check(g, "advect_velocity", lambda: P("advect_velocity", DT), {"velocity": v3}, {"velocity": v4}, swaps=("velocity",))
    check(g, "advect_dye", lambda: P("advect_dye", DT), {"velocity": v4, "dye": dye}, {"dye": R(O.advect(v4, dye, DT, 1.0))},
          swaps=("dye",))
    if not half:                              # half storage runs the three passes above for it
        check(g, "curl_vorticity_divergence", lambda: P("curl_vorticity_divergence", DT), {"velocity": v},
              {"curl": c, "velocity": v2, "divergence": d}, swaps=("velocity",))
    # half storage clears in a launch of its own; fp32 fuses the clear into the first sweep
    check(g, "pressure_solve", lambda: P("pressure_solve"), {"pressure": p, "divergence": d}, {"pressure": jac(p1, 20)},
          swaps=pressure_swaps(len(jacobi_plan(W, H, half, 20)) + half))
    for f, a in zip(FIELDS, (v, dye, p, d, c)):
        check(g, "write", lambda: s.writeField(f, a), {}, {f: a}, field=f, swaps=())
        check(g, "read", lambda: s.readField(f), {f: a}, {f: a}, swaps=())
    s.close()


# fp32: jacobi_scalar_kernel (7 % 4 != 0); 1000 x 524: pressure 1152 B of padding, less than a row; 1024 x 512:
# no padding in any slot.  Every fp32 advection variant (fluid.cu do_advect_velocity / do_advect_dye):
# velocity4 at 256 / 128; one-cell POW2 velocity at 64 / 32; dye4<SAME> at 256^2 -> 256^2; dye4<!SAME> at
# 128^2 -> 256^2 and 64^2 -> 128^2; one-cell POW2 dye <SAME> at 64^2 -> 64^2 and <!SAME> at 32^2 -> 64^2 (a dye
# grid narrower than 128); the ragged kernels at 36 x 20 / 54 x 30, 1 x 9 / 3 x 27 and 9 x 1 / 27 x 3
FP32_SIZES = [(7, 5, 9, 6), (1000, 524, 1000, 524), (1024, 512, 1024, 512), (256, 256, 256, 256),
              (128, 128, 256, 256), (64, 64, 64, 64), (64, 64, 128, 128), (32, 32, 64, 64), (36, 20, 54, 30),
              (1, 9, 3, 27), (9, 1, 27, 3)]
# half: 1024^2 has 2 MiB pressure slots with no padding; hs::jacobi8_kernel across warps at W = 264, 520, 1024;
# the one-cell half jacobi_scalar_kernel at W = 100
HALF_SIZES = [(1024, 1024, 1024, 1024), (100, 60, 150, 90), (264, 40, 528, 80), (520, 33, 780, 50)]


@pytest.mark.parametrize("W,H,Wd,Hd", FP32_SIZES)
def test_every_pass_fp32(pkg, torch, oracle, W, H, Wd, Hd):
    every_pass(pkg, torch, oracle, W, H, Wd, Hd, False)


@pytest.mark.parametrize("W,H,Wd,Hd", HALF_SIZES)
def test_every_pass_half(pkg, torch, oracle, W, H, Wd, Hd):
    every_pass(pkg, torch, oracle, W, H, Wd, Hd, True, jacobi_iters=(1, 5))


TILED = [(520, 33), (130, 66)]


@pytest.mark.parametrize("W,H", [(1024, 512), (964, 600), (16900, 3), (124, 2050)] + TILED)
def test_curl_vorticity_divergence_and_gradient_streaming_and_tiled(pkg, torch, oracle, W, H):
    """cvd_stream_kernel's 120-of-128-column windows and gradient_stream_kernel's GS_U-rounded row groups at
    streaming sizes, the tiled kernels where too few warps (or W % 4 != 0) select them."""
    O = oracle
    s = make(pkg, W, H, 8, 8)
    g = Arena(torch, s)
    v, _, p = rand_fields(W, H, 8, 8, W + 3 * H)
    c = O.curl(v); v2 = O.vorticity(v, c, 30.0, DT)
    n = delta(s, "cvd_stream_launches", lambda: check(
        g, "curl_vorticity_divergence", lambda: s.pass_("curl_vorticity_divergence", DT), {"velocity": v},
        {"curl": c, "velocity": v2, "divergence": O.divergence(v2)}, swaps=("velocity",)))
    streaming = (W, H) in STREAM_SHAPES
    assert n == 2 * streaming
    n = delta(s, "gradient_stream_launches", lambda: check(
        g, "gradient_subtract", lambda: s.pass_("gradient_subtract"), {"pressure": p, "velocity": v2},
        {"velocity": O.gradient_subtract(p, v2)}, swaps=("velocity",)))
    assert n == 2 * streaming
    s.close()


def solve_case(pkg, torch, O, W, H, cases, p, d, flags=0, cmp=bits_equal):
    """fluid_pass_pressure_solve (clear fused into the first launch) for each (JACOBI_BLOCK, sweeps, launch
    depths) of `cases`: the depths are those of jacobi_plan, and the library launches that many kernels."""
    s = make(pkg, W, H, 8, 8, flags=flags)
    g = Arena(torch, s)
    for jb, iters, depths in cases:
        plan = jacobi_plan(W, H, False, iters, jb, naive=bool(flags & pkg.FLAG_NAIVE_JACOBI))
        assert plan == depths, (jb, iters, plan)
        s.set_param("JACOBI_BLOCK", jb)
        s.config["PRESSURE_ITERATIONS"] = iters
        want = O.jacobi(O.clear(p, 0.8), d, iters)
        n = delta(s, "jacobi_launches", lambda: check(g, "pressure_solve", lambda: s.pass_("pressure_solve"),
                                                      {"pressure": p, "divergence": d}, {"pressure": want}, cmp=cmp,
                                                      swaps=pressure_swaps(len(plan))))
        assert n == 2 * len(plan), (jb, n)
    return s


@pytest.mark.parametrize("W,H", [(1000, 524), (132, 45)])
def test_blocked_jacobi_every_depth(pkg, torch, oracle, W, H):
    """JACOBI_BLOCK K = 2..13 with 3K - 1 sweeps: JacobiPlan splits them into launches of depth K, K, K - 1, so
    every jacobi_tb_kernel instantiation runs (overlapped windows, chunk ends, ragged widths), each followed
    by a shallower one; K = 1 is one jacobi_sweep_kernel per sweep."""
    _, _, p = rand_fields(W, H, 8, 8, W + H)
    d = np.random.default_rng(W).uniform(-1, 1, (H, W)).astype(np.float32)
    cases = [(1, 2, [1, 1])] + [(K, 3 * K - 1, [K, K, K - 1]) for K in range(2, 14)]
    solve_case(pkg, torch, oracle, W, H, cases, p, d).close()


def test_naive_jacobi_flag(pkg, torch, oracle):
    _, _, p = rand_fields(1000, 524, 8, 8, 5)
    d = np.random.default_rng(5).uniform(-1, 1, (524, 1000)).astype(np.float32)
    solve_case(pkg, torch, oracle, 1000, 524, [(0, 5, [1] * 5)], p, d, flags=pkg.FLAG_NAIVE_JACOBI).close()


@pytest.mark.parametrize("W,H,iters,depths", [(1024, 512, 20, [10, 10]), (4096, 4096, 50, [13, 13, 12, 12])])
def test_blocked_jacobi_default_depth(pkg, torch, oracle, W, H, iters, depths):
    """The default depth where no slot has padding: 1024 x 512 (2 MiB pressure), and the headline 4096^2 x 50
    solve in 4 launches of depth 13 / 13 / 12 / 12."""
    if W == 4096:
        oracle.use_all_cores()
    rng = np.random.default_rng(W + iters)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    solve_case(pkg, torch, oracle, W, H, [(0, iters, depths)], p, d).close()


@pytest.mark.parametrize("case", ["tiny_divergence", "near_max"])
def test_blocked_jacobi_exact_streams(pkg, torch, oracle, case):
    """The un-contracted streams and the exact re-run of the blocked kernel under poison: divergence in
    (0, 2^-123) on a patch, or a patch near FLT_MAX whose first sweep overflows."""
    W, H = 1000, 524
    rng = np.random.default_rng(17)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    if case == "tiny_divergence":
        d[200:240, 500:620] = np.float32(2.0 ** -130)
    else:
        near_max_patch(p, d, 300, 340, 400, 440, 0.8)
    with np.errstate(over="ignore", invalid="ignore"):
        s = solve_case(pkg, torch, oracle, W, H, [(0, 20, [10, 10])], p, d, cmp=same_bits)
    assert s.stat("jacobi_exact_streams") > 0                  # counted since the handle was created
    s.close()


@pytest.mark.parametrize("W,H,launches,swaps", [(1000, 300, 2, ()), (256, 2000, 7 * 2, ("pressure",))])
def test_host_pressure_solve(pkg, torch, oracle, W, H, launches, swaps):
    """fluid_pressure_solve_host in one piece (300 rows: fewer than two bands; two launches of 10, two swaps)
    and banded (7 bands of 286 rows at depth 10, the last one 284; one swap): uploads into divergence and
    pressure.read, the result in pressure.write; the band buffers are outside the arena."""
    rng = np.random.default_rng(W * H)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    want = oracle.jacobi(oracle.clear(p, 0.8), d, 20)
    s = make(pkg, W, H, 8, 8)
    g = Arena(torch, s)
    for value in POISONS:
        ph = p.copy()
        n0 = s.stat("jacobi_launches")
        g.run("pressure_solve_host", lambda: s.pressure_solve_host(d, ph, 20), (), value, swaps=swaps)
        assert s.stat("jacobi_launches") - n0 == launches
        assert bits_equal(ph, want) and bits_equal(s.readField("pressure"), want)
        assert bits_equal(s.readField("divergence"), d)
    s.close()


@pytest.mark.parametrize("n", [1, 128, 129, 300])
@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
def test_splats(pkg, torch, oracle, n, half):
    """fluid_splats: the first launch reads .read, later ones continue in place on .write.  512 x 256 fp32 dye
    is exactly 2 MiB: no padding between dye[0] and dye[1]."""
    W, H, Wd, Hd = 256, 256, 512, 256
    R = oracle.round_half if half else (lambda a: a)
    v, dye, _ = (R(a) for a in rand_fields(W, H, Wd, Hd, n))
    recs = nasty_records(n, seed=n)
    aspect, rad = SM.aspect_of(W, H), SM.radius_of(0.25, W, H)
    expect = {}
    for name, base in (("velocity", v), ("dye", dye)):
        lo, hi = SM.splat_interval(base, recs, aspect, rad, half)
        expect[name] = lambda got, lo=lo, hi=hi: SM.check_splat(got, lo, hi)[0] == 0
    s = make(pkg, W, H, Wd, Hd, flags=pkg.FLAG_HALF_STORAGE if half else 0)
    g = Arena(torch, s, half)
    launches = []
    check(g, "splats", lambda: launches.append(delta(s, "launches", lambda: s.splats(recs))), {"velocity": v, "dye": dye},
          expect, swaps=("velocity", "dye"))
    assert launches == [-(-n // 128)] * 2
    s.close()


STEP_CASES = [(128, 128, 256, 256, 0), (128, 128, 256, 256, "no_graph"), (128, 128, 256, 256, "unfused"),
              (1024, 512, 1024, 512, 0), (100, 60, 150, 90, "half"), (128, 128, 256, 256, "half_no_graph"),
              (4096, 4096, 4096, 4096, 0)]


@pytest.mark.parametrize("W,H,Wd,Hd,mode", STEP_CASES)
def test_whole_step(pkg, torch, oracle, W, H, Wd, Hd, mode):
    """step() as a graph and with FLUID_FLAG_NO_GRAPH (and UNFUSED), fp32 and half, every field against the
    oracle.  4096^2 with 50 iterations is the headline step: no padding in any slot."""
    O = oracle
    flags = {0: 0, "no_graph": pkg.FLAG_NO_GRAPH, "unfused": pkg.FLAG_NO_GRAPH | pkg.FLAG_UNFUSED,
             "half": pkg.FLAG_HALF_STORAGE, "half_no_graph": pkg.FLAG_HALF_STORAGE | pkg.FLAG_NO_GRAPH}[mode]
    half = bool(flags & pkg.FLAG_HALF_STORAGE)
    iters = 50 if W == 4096 else 20
    if W == 4096:
        O.use_all_cores()
    R = O.round_half if half else (lambda a: a)
    v, dye, p = (R(a) for a in rand_fields(W, H, Wd, Hd, W + H + len(str(mode))))
    ref = O.OracleSim(W, H, Wd, Hd, half_storage=half, PRESSURE_ITERATIONS=iters)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    ref.step(DT)
    s = make(pkg, W, H, Wd, Hd, flags=flags, PRESSURE_ITERATIONS=iters)
    g = Arena(torch, s, half)
    graphs = s.stat("graph_launches")
    # velocity swaps three times (vorticity or the fused pass, gradientSubtract, advection), dye once, pressure
    # once per Jacobi launch plus half storage's own clear launch
    swaps = ("velocity", "dye") + pressure_swaps(len(jacobi_plan(W, H, half, iters)) + half)
    check(g, "step", lambda: s.step(DT), {"velocity": v, "dye": dye, "pressure": p},
          {n: getattr(ref, n) for n in FIELDS}, swaps=swaps)
    assert s.stat("graph_launches") - graphs == (0 if flags & pkg.FLAG_NO_GRAPH else 2)
    s.close()


FRAME_GEOMETRIES = [(64, 64, 128, 128), (48, 32, 50, 75)]


@pytest.mark.parametrize("handle", ["fp32", "half_half_postfx", "nearest"])
@pytest.mark.parametrize("Wd,Hd,w,h", FRAME_GEOMETRIES)
def test_frames_and_captures(pkg, torch, oracle, handle, Wd, Hd, w, h):
    """render() with all eight keyword sets: the arena is untouched except dye.write with SUNRAYS (the mask),
    and with dye.write poisoned the frame equals the display model.  captureScreenshot() the same way; its
    bytes equal the capture this handle drew before anything was poisoned."""
    kind = "nearest_fp32" if handle == "nearest" else handle
    dither = DH.golden_dither()
    dye = DH.stored(kind, DH.seeded_dye(Wd, Hd, Wd + w))
    s = DH.make(pkg, Wd, Hd, w, h, DH.flags_of(pkg, kind))
    s.config["CAPTURE_RESOLUTION"] = min(w, h)
    s.writeField("dye", dye)
    s.dithering = dither
    clean = []
    for kw in range(8):
        DH.set_keywords(s, kw)
        clean.append(s.captureScreenshot())
    g = Arena(torch, s, handle.startswith("half"))
    with np.errstate(invalid="ignore", over="ignore"):
        for kw in range(8):
            DH.set_keywords(s, kw)
            want = DH.model_frame(kind, dye, w, h, kw, dither, DH.FXCFG, oracle.BG_COLOR)
            call = "render_sunrays" if kw & pkg.DISPLAY_SUNRAYS else "render"
            frames, caps = [], []
            for value in POISONS:
                got = g.run(call, lambda: s.render(w, h), ("dye",), value, swaps=())
                DH.check_frame(s, got, want, kw, (handle, kw, hex(value)))
                frames.append(got)
                caps.append(g.run(call, lambda: s.captureScreenshot(), ("dye",), value, swaps=()))
                assert np.array_equal(caps[-1], clean[kw]), (kw, hex(value))
                assert bits_equal(s.readField("dye"), dye)
            assert bits_equal(frames[0], frames[1]), kw
    s.close()


RESIZES = [("linear", (36, 20, 54, 30), (23, 41, 97, 31)), ("nearest", (64, 48, 128, 96), (100, 75, 150, 113)),
           ("half", (64, 48, 128, 96), (100, 75, 150, 113)), ("same_size_velocity", (36, 20, 54, 30), (36, 20, 97, 31)),
           ("no_padding", (1000, 524, 512, 256), (1024, 512, 1000, 524))]


@pytest.mark.parametrize("mode,src,dst", RESIZES, ids=[r[0] for r in RESIZES])
def test_resize_builds_a_clean_arena(pkg, torch, oracle, mode, src, dst):
    """fluid_resize from a poisoned arena: the new arena is byte for byte make_arena's image (zero padding,
    flag words, pressure, divergence, curl and velocity.write; dye.write (0, 0, 0, 1)) with the carried
    velocity and dye, resampled like the oracle, in the slots of the pairs' unchanged parity."""
    O = oracle
    flags = {"nearest": pkg.FLAG_NEAREST_FILTERING, "half": pkg.FLAG_HALF_STORAGE}.get(mode, 0)
    half = mode == "half"
    R = O.round_half if half else (lambda a: a)
    v, dye, p = (R(a) for a in rand_fields(*src, 41))
    W, H, Wd, Hd = dst
    if mode == "nearest":
        v2, dye2 = DM.resize(v, W, H), DM.resize(dye, Wd, Hd)
    else:
        v2 = v if (W, H) == src[:2] else R(O.resample(v, W, H))
        dye2 = R(O.resample(dye, Wd, Hd))
    for value in POISONS:
        s = make(pkg, *src, flags=flags)
        s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
        s.step(DT)                                    # both pairs swapped at least once, every field written
        s.writeField("velocity", v); s.writeField("dye", dye)
        g = Arena(torch, s, half)
        g.poison(("velocity", "dye"), value)
        torch.cuda.synchronize()
        s._sizes = dst
        s.initFramebuffers()
        g.attach()
        par = g.parity()
        want = A.fresh(g.L)
        A.put(want, g.L.v[par["velocity"]], v2, half)
        A.put(want, g.L.dye[par["dye"]], dye2, half)
        n, rep = A.changes_outside(want, g.image(), [], g.L)
        assert n == 0, (mode, hex(value), n, rep)
        assert bits_equal(s.readField("velocity"), v2) and bits_equal(s.readField("dye"), dye2)
        s.close()


def test_refused_resize_changes_no_byte(pkg, torch):
    """FLUID_ERR_NOMEM (an fp32 81920^2 dye is 100 GiB): the arena, padding and flag words included, is
    byte-identical afterwards."""
    s = make(pkg, 64, 64, 128, 128)
    rng = np.random.default_rng(12)
    s.writeField("velocity", (rng.standard_normal((64, 64, 2)) * 50).astype(np.float32))
    s.writeField("dye", rng.random((128, 128, 4), dtype=np.float32))
    s.step(DT)
    g = Arena(torch, s)
    for value in POISONS:
        rc = g.run("read", lambda: s._L.fluid_resize(s._h, 64, 64, 81920, 81920), FIELDS, value, swaps=())
        assert rc == FLUID_ERR_NOMEM
        assert s._dims("dye")[:2] == (128, 128)
    s.close()
