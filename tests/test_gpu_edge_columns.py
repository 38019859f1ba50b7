"""The blocked pressure solve with each window's edge lanes fed from the staged box.

Lane 0 and lane 31 of a window have no neighbour lane on one side.  At level 1 they take the level-0 column just
outside the window (x0 - 1, x0 + 128) from the staged p box, so a depth-K launch recomputes roundup(K - 1, 4)
halo columns per side instead of roundup(K, 4): depths 1, 5, 9 and 13 keep 8 more columns per window, and at
those depths the outermost valid output of every window depends on the edge column.  An edge column read from
the wrong place (wrong column, wrong row, wrong stage, not mirrored at a wall, not scaled by PRESSURE) changes
bits, so: blocked == one sweep per launch, bit for bit, at widths around the window payloads 104 / 112 / 120 /
128, with one chunk and with several, on ordinary data, on columns of large distinct values at every float4
boundary, on inf / NaN and on tiny divergence."""
import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import special_fields
from sim_harness import make, same_bits, solve
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu
WIDTHS = (104, 108, 112, 120, 128, 132, 208, 1000, 1040, 4096)
HEIGHTS = (40, 300)                 # one chunk of rows per window; several
# (jacobi_block, sweeps): K and 3K - 1 sweeps at depths 5, 9, 13 and the default; one sweep alone is a depth-1
# launch (a handle asked for jacobi_block = 1 does not run the blocked kernel at all)
PLANS = [(5, 5), (5, 14), (9, 9), (9, 26), (13, 13), (13, 38), (13, 1), (0, 13), (0, 38)]


def fields(kind, W, H, seed):
    rng = np.random.default_rng(seed)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    if kind == "spikes":            # every column that is first or last of a float4: window and lane boundaries
        c = np.arange(W)
        edge = (c % 4 == 0) | (c % 4 == 3)
        p[:, edge] += (1000.0 * (c[edge] + 1))[None, :].astype(np.float32) + np.arange(H, dtype=np.float32)[:, None]
    return p, d


@pytest.mark.parametrize("H", HEIGHTS)
@pytest.mark.parametrize("W", WIDTHS)
def test_blocked_equals_one_sweep_per_launch(pkg, W, H):
    blocked, naive = make(pkg, W, H, 8, 8), make(pkg, W, H, 8, 8, pkg.FLAG_NAIVE_JACOBI, 1)
    for n, (jb, iters) in enumerate(PLANS):
        for kind in ("random", "spikes"):
            p, d = fields(kind, W, H, 7 * W + H + n)
            for pressure in (0.8, None):
                n0 = blocked.stat("jacobi_launches")
                got = solve(blocked, p, d, iters, pressure, jb)
                if jb:
                    assert blocked.stat("jacobi_launches") - n0 == -(-iters // jb), (W, H, jb, iters)
                ref = solve(naive, p, d, iters, pressure)
                assert bits_equal(got, ref), (W, H, jb, iters, kind, pressure)
    assert blocked.stat("jacobi_exact_streams") == 0      # ordinary data runs contracted
    blocked.close(); naive.close()


@pytest.mark.parametrize("W,H", [(104, 40), (132, 300), (1040, 300), (4096, 96)])
def test_nonfinite_inputs(pkg, W, H):
    blocked, naive = make(pkg, W, H, 8, 8), make(pkg, W, H, 8, 8, pkg.FLAG_NAIVE_JACOBI, 1)
    for jb, iters in ((13, 13), (9, 9), (5, 14), (0, 38)):
        p, d = special_fields("nonfinite", W, H, W + H + jb)
        for pressure in (0.8, None):
            assert same_bits(solve(blocked, p, d, iters, pressure, jb), solve(naive, p, d, iters, pressure))
    blocked.close(); naive.close()


@pytest.mark.parametrize("W,H", [(132, 300), (1040, 300), (4096, 96)])
def test_a_huge_edge_column_sends_its_window_through_the_exact_tail(pkg, W, H):
    """Window 0 of a depth-K launch spans columns -HX .. 127 - HX and reads column 128 - HX only as lane 31's
    edge column.  With p = 3.4e38 there and d = -5e36 (below 2^122) beside it, S - d overflows to inf in the
    reference at column 127 - HX while fma(S, 0.25, -0.25 d) stays finite, and that cell reaches window 0's
    last valid column.  No other input of window 0 reaches 2^122: only folding the edge column into the
    stream's largest magnitude sends it through the exact tail."""
    blocked, naive = make(pkg, W, H, 8, 8), make(pkg, W, H, 8, 8, pkg.FLAG_NAIVE_JACOBI, 1)
    for jb, iters, hx in ((13, 13, 12), (9, 9, 8), (5, 5, 4), (0, 38, 12)):
        p, d = fields("random", W, H, W + jb)
        col = 128 - hx
        p[:, col] = np.float32(3.4e38); d[:, col - 1] = np.float32(-5e36)
        e0 = blocked.stat("jacobi_exact_streams")
        got, ref = solve(blocked, p, d, iters, None, jb), solve(naive, p, d, iters, None)
        assert np.isinf(ref[:, col - 1 - hx]).any() or np.isnan(ref[:, col - 1 - hx]).any()
        assert same_bits(got, ref), (W, H, jb)
        assert blocked.stat("jacobi_exact_streams") > e0
    blocked.close(); naive.close()


@pytest.mark.parametrize("W,H", [(208, 300), (1000, 96)])
def test_tiny_divergence_runs_exact_streams(pkg, W, H):
    blocked, naive = make(pkg, W, H, 8, 8), make(pkg, W, H, 8, 8, pkg.FLAG_NAIVE_JACOBI, 1)
    for jb, iters in ((13, 13), (9, 26), (5, 5), (13, 1)):
        p, d = fields("spikes", W, H, W + jb)
        d[H // 2, ::7] = np.float32(2.0 ** -130)
        e0 = blocked.stat("jacobi_exact_streams")
        for pressure in (0.8, None):
            assert bits_equal(solve(blocked, p, d, iters, pressure, jb), solve(naive, p, d, iters, pressure)), (W, jb)
        assert blocked.stat("jacobi_exact_streams") > e0
    blocked.close(); naive.close()


@pytest.mark.parametrize("jb,launches", [(13, 2 * 4), (0, 2 * 5)])
def test_banded_host_solve_equals_the_resident_solve(pkg, jb, launches):
    W, H, iters = 4096, 512, 50
    p, d = fields("spikes", W, H, 99)
    s = make(pkg, W, H, 8, 8, jb=jb); s.config["PRESSURE_ITERATIONS"] = iters
    want = solve(s, p, d, iters, 0.8)
    n0 = s.stat("jacobi_launches")
    ph = p.copy()
    s.pressure_solve_host(d, ph, iters)
    assert s.stat("jacobi_launches") - n0 == launches
    assert s.stat("jacobi_exact_streams") == 0
    s.close()
    assert bits_equal(ph, want)
