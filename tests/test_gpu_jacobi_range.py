"""The blocked pressure solve at the top of the fp32 range and on inf / NaN.

Its contracted tail fma(S, 0.25, -0.25 d) differs from the reference's (S - d) * 0.25 where S and d are
finite and S - d rounds to +-inf (tests/test_fma_contraction_cpu.py).  A warp stream whose level-0 inputs
reach 2^122 therefore runs again with the exact tail (csrc/jacobi.cuh).  On the data sets of
tests/jacobi_tb_model.py -- a patch of p near FLT_MAX / 4 over d = -1e37, its mirror image, divergence
in [2^126, FLT_MAX], inf / NaN sprinkled, binary exponents -149..127 -- the blocked solve equals one sweep
per launch and the oracle: mirrored windows and ragged widths, every depth, with and without the fused
clear, the host solve banded and in one piece, and whole steps after such a solve.  The
jacobi_exact_streams counter shows the exact tail ran."""
import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import KINDS, equal, overflow_sweep, special_fields
from sim_harness import make, near_max_patch, same_bits, solve
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu
DT = 0.016666
PRESSURES = (0.8, 1.0, 2.0)
OVERFLOWING = ("near_max", "near_max_neg", "huge_div")
# (W, H, depths): 4096 has the last window's mirrored lanes outside the staged box at K = 10; 1000 and 132
# are not multiples of a window's payload; 112 x 2 puts both y walls in every block.  0 = default depth.
SHAPES = [(4096, 96, (10, 0)), (1000, 64, tuple(range(2, 14)) + (0,)), (132, 45, tuple(range(2, 14)) + (0,)),
          (112, 2, tuple(range(2, 14)) + (0,))]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("W,H,depths", SHAPES)
def test_blocked_equals_naive_and_oracle_at_the_top_of_the_range(pkg, oracle, kind, W, H, depths):
    blocked, naive = make(pkg, W, H, 8, 8), make(pkg, W, H, 8, 8, pkg.FLAG_NAIVE_JACOBI, 1)
    for n, jb in enumerate(depths):
        iters = 2 * jb + 1 if jb else 30
        for pressure in (PRESSURES[n % 3], None):
            p, d = special_fields(kind, W, H, W + H + jb, 1.0 if pressure is None else pressure)
            if kind in OVERFLOWING:       # the premise: the contracted tail alone would differ somewhere
                assert overflow_sweep(oracle, p, d, iters, 1.0 if pressure is None else pressure), (W, H, jb, pressure)
            want = oracle.jacobi(p if pressure is None else oracle.clear(p, pressure), d, iters)
            e0 = blocked.stat("jacobi_exact_streams")
            got = solve(blocked, p, d, iters, pressure, jb)
            ref = solve(naive, p, d, iters, pressure)
            assert equal(kind, got, ref), (kind, W, H, jb, pressure)
            assert equal(kind, got, want), (kind, W, H, jb, pressure)
            # exact streams ran iff some level-0 input reached 2^122 or the tiny map flagged divergence
            # (full_range on a 2-row grid may hold neither)
            q = np.abs(p if pressure is None else oracle.clear(p, pressure))
            big = np.nanmax(q) >= 2.0 ** 122 or np.nanmax(np.abs(d)) >= 2.0 ** 122
            tiny = ((d != 0) & (np.abs(d) < np.float32(2.0 ** -123))).any()
            assert (blocked.stat("jacobi_exact_streams") > e0) == (big or tiny), (kind, W, H, jb, pressure)
            if kind != "full_range":
                assert big, kind
    assert naive.stat("jacobi_exact_streams") == 0
    blocked.close(); naive.close()


@pytest.mark.parametrize("W,H,iters,jb,launches", [(1024, 2048, 50, 0, 8 * 5), (1000, 2048, 50, 13, 8 * 4),
                                                   (1000, 300, 50, 0, 4)])
def test_host_pressure_solve_with_a_near_max_patch(pkg, oracle, W, H, iters, jb, launches):
    """fluid_pressure_solve_host, banded (the patch inside one band, rows 300..340 of 256-row bands) and in one
    piece (300 rows: fewer than two bands), against one sweep per launch on a resident field."""
    rng = np.random.default_rng(W + H)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    r0, r1 = (H - 100, H - 60) if H < 512 else (300, 340)
    near_max_patch(p, d, r0, r1, 400, 440, 0.8)
    crop = (slice(r0 - 8, r1 + 8), slice(392, 448))
    assert overflow_sweep(oracle, p[crop], d[crop], 1, 0.8) == 1
    s = make(pkg, W, H, 8, 8, jb=jb); s.config["PRESSURE_ITERATIONS"] = iters
    n0, e0 = s.stat("jacobi_launches"), s.stat("jacobi_exact_streams")
    ph = p.copy()
    s.pressure_solve_host(d, ph, iters)
    assert s.stat("jacobi_launches") - n0 == launches
    assert s.stat("jacobi_exact_streams") > e0
    s.close()
    s = make(pkg, W, H, 8, 8, pkg.FLAG_NAIVE_JACOBI, 1)
    ref = solve(s, p, d, iters, 0.8)
    s.close()
    assert np.isinf(ref).any()
    assert bits_equal(ph, ref)


@pytest.mark.parametrize("flags", [0, "no_graph"])
def test_steps_after_a_near_max_solve_bitwise_vs_oracle(pkg, oracle, flags):
    """A solve that overflows in the reference, then two whole steps (graph replay or pass by pass): every
    field equals OracleSim's.  A ragged grid, so that advection interpolates like the oracle even where
    the overflowed pressure has made velocity inf / NaN."""
    O = oracle
    W, H, Wd, Hd = 132, 100, 198, 150
    rng = np.random.default_rng(21)
    v = (rng.standard_normal((H, W, 2)) * 50).astype(np.float32)
    dye = rng.random((Hd, Wd, 4), dtype=np.float32)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    near_max_patch(p, d, 40, 52, 50, 70, 0.8)
    f = 0 if flags == 0 else pkg.FLAG_NO_GRAPH
    s = pkg.FluidSimulation({"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}, canvas_width=W,
                            canvas_height=H, flags=f, sizes=(W, H, Wd, Hd))
    ref = O.OracleSim(W, H, Wd, Hd)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p); s.writeField("divergence", d)
    s.pass_("pressure_solve")
    ref.velocity, ref.dye = v.copy(), dye.copy()
    ref.pressure = O.jacobi(O.clear(p, 0.8), d, 20)
    assert np.isinf(ref.pressure).any()
    assert same_bits(s.readField("pressure"), ref.pressure)
    for _ in range(2):
        s.step(DT); ref.step(DT)
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert same_bits(s.readField(n), getattr(ref, n)), n
    assert s.stat("jacobi_exact_streams") > 0
    s.close()
