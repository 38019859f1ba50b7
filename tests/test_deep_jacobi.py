"""Depth 13, the cap of the blocked pressure solve and the single-GPU default (50 sweeps in 4 launches
of 13 / 12 instead of 5 of 10).

CPU: the lane-level model at K = 13 against the oracle.  GPU: the library's blocked solve at depth 13
against one sweep per launch and the oracle, bit for bit, and its launch count."""
import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import jacobi_tb_model
from webgl_fluid_simulation_b200 import slab
from webgl_fluid_simulation_b200.slab import KMAX as K_MAX

TINY = 9.4039548e-38                # 2^-123: below it the contracted tail is not exact (EXACT streams)


# ---- CPU: the lane-level model at depth 13 ----------------------------------------------------------
@pytest.mark.parametrize("W,H,R", [(4 * 43, 47, 27), (96, 40, 52), (256, 31, 13), (388, 70, 30)])
def test_model_k13_equals_oracle_sweeps(oracle, W, H, R):
    """Walls, mirrored x-halos (W not a multiple of the 96-column payload) and chunk seams."""
    rng = np.random.default_rng(W + H + R)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.standard_normal((H, W)).astype(np.float32)
    assert bits_equal(jacobi_tb_model(p, d, K_MAX, R), oracle.jacobi(p, d, K_MAX))


def test_model_k13_fused_clear_and_slab(oracle):
    K = K_MAX
    rng = np.random.default_rng(13)
    H, W = 3 * K + 20, 136
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.standard_normal((H, W)).astype(np.float32)
    assert bits_equal(jacobi_tb_model(p, d, K, 4 * K, scale=0.8), oracle.jacobi(oracle.clear(p, 0.8), d, K))
    full = oracle.jacobi(p, d, K)
    r0, r1 = K + 3, H - K - 2                          # an interior slab: local rows = owned +- K ghosts
    lo, hi = r0 - K, r1 + K
    got = jacobi_tb_model(p[lo:hi], d[lo:hi], K, 9, row_off=lo, out_lo=r0, out_hi=r1, H=H)
    assert bits_equal(got[r0 - lo:r1 - lo], full[r0:r1])


# ---- GPU: the library's blocked solve at depth 13 ---------------------------------------------------
# (W, H, iters, JACOBI_BLOCK, tiny): W = 4096 has the last window with mirrored lanes outside the staged
# box; the other widths are not multiples of the 96-column payload; short grids; iteration counts that
# are not multiples of 13; 0 = the library's default depth; tiny = a patch of divergence values in
# (0, 2^-123), so that the un-contracted (EXACT) streams run too.
DEEP_CASES = [(4096, 96, 50, 0, True), (4096, 64, 26, 13, False), (4096, 80, 50, 13, True),
              (1000, 45, 50, 0, False), (364, 30, 31, 13, True), (532, 7, 15, 0, False),
              (200, 300, 33, 13, True), (92, 3, 16, 0, False), (1028, 130, 39, 0, True)]


@pytest.mark.gpu
def test_depth13_bitwise_vs_naive_and_oracle(oracle):
    """The blocked solve (depth 13 by default) and one sweep per launch both equal the oracle bit for bit."""
    import webgl_fluid_simulation_b200 as pkg
    for W, H, iters, jb, tiny in DEEP_CASES:
        rng = np.random.default_rng(W + 3 * H + iters + jb)
        p = rng.standard_normal((H, W)).astype(np.float32)
        d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
        if tiny:
            r, c = min(4, H - H // 3), min(40, W - W // 2)
            d[H // 3:H // 3 + r, W // 2:W // 2 + c] = rng.uniform(0.5, 1, (r, c)).astype(np.float32) * np.float32(TINY)
            assert np.any((d != 0) & (np.abs(d) < np.float32(TINY)))
        want = oracle.jacobi(oracle.clear(p, 0.8), d, iters)
        for flags, block in ((0, jb), (pkg.FLAG_NAIVE_JACOBI, 1)):
            s = pkg.FluidSimulation({"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": 8, "PRESSURE_ITERATIONS": iters},
                                    canvas_width=W, canvas_height=H, flags=flags, jacobi_block=block, sizes=(W, H, 8, 8))
            s.writeField("pressure", p); s.writeField("divergence", d); s.pass_("pressure_solve")
            got, launches, exact = s.readField("pressure"), s.stat("jacobi_launches"), s.stat("jacobi_exact_streams")
            s.close()
            assert (exact > 0) == (tiny and not flags), (W, H, iters, jb, flags, exact)
            assert bits_equal(got, want), (W, H, iters, jb, flags)
            if not flags:
                assert launches == -(-iters // K_MAX), (W, H, iters, jb)
            assert launches == len(slab.jacobi_launches(iters, slab.SlabPlan(H, 8, 0, 1).block(block))), (W, H, iters, flags)
