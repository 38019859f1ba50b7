"""The temporally-blocked Jacobi kernel's algorithm (lane-level model of the CUDA code) must equal
K plain sweeps of the oracle BITWISE — including walls, mirrored x-halos, chunk seams."""
import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import KINDS, NONFINITE_KINDS, equal, jacobi_tb_model, overflow_sweep, special_fields


@pytest.mark.parametrize("W,H,K,R", [(128, 40, 3, 16), (256, 33, 8, 12), (16, 9, 2, 4),
                                     (132, 50, 5, 50), (240, 31, 1, 7), (112, 2, 4, 2),
                                     (360, 21, 10, 9)])
def test_model_equals_k_oracle_sweeps(oracle, W, H, K, R):
    rng = np.random.default_rng(W * 1000 + H * 10 + K)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.standard_normal((H, W)).astype(np.float32)
    got = jacobi_tb_model(p, d, K, R)
    assert bits_equal(got, oracle.jacobi(p, d, K))


def test_model_with_fused_clear(oracle):
    rng = np.random.default_rng(5)
    p = rng.standard_normal((24, 64)).astype(np.float32)
    d = rng.standard_normal((24, 64)).astype(np.float32)
    got = jacobi_tb_model(p, d, 4, 8, scale=0.8)
    assert bits_equal(got, oracle.jacobi(oracle.clear(p, 0.8), d, 4))


def test_model_on_a_slab_with_ghost_rows(oracle):
    """Interior slab of a taller grid: local buffer = owned rows +- K ghost rows; no wall logic."""
    rng = np.random.default_rng(6)
    H, W, K = 64, 128, 4
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.standard_normal((H, W)).astype(np.float32)
    full = oracle.jacobi(p, d, K)
    for r0, r1 in [(0, 20), (20, 44), (44, 64)]:
        lo, hi = max(r0 - K, 0), min(r1 + K, H)
        got = jacobi_tb_model(p[lo:hi], d[lo:hi], K, 10, row_off=lo, out_lo=r0, out_hi=r1, H=H)
        assert bits_equal(got[r0 - lo:r1 - lo], full[r0:r1])


# ---- the top of the fp32 range, inf and NaN ------------------------------------------------------------
@pytest.mark.parametrize("kind", ["near_max", "near_max_neg", "huge_div"])
def test_model_with_the_tiny_map_rule_alone_differs_from_the_oracle(oracle, kind):
    """The premise, on the CPU: selecting the exact tail by the tiny-divergence map only (the rule before
    BIG_IN) lets the contracted tail run where S - d overflows, and the result differs from the oracle."""
    W, H, K, R = 256, 40, 4, 16
    p, d = special_fields(kind, W, H, 3)
    assert overflow_sweep(oracle, p, d, K, 1.0) == (2 if kind == "huge_div" else 1)
    want = oracle.jacobi(p, d, K)
    st = {}
    assert not bits_equal(jacobi_tb_model(p, d, K, R, scale=1.0, select="tiny", stats=st), want)
    assert st["exact_streams"] == 0
    assert bits_equal(jacobi_tb_model(p, d, K, R, scale=1.0, select="exact"), want)


@pytest.mark.parametrize("pressure", [0.8, 1.0, 2.0])
@pytest.mark.parametrize("kind", KINDS)
def test_model_with_the_kernel_rule_equals_the_oracle(oracle, kind, pressure):
    """The kernel's selection (tiny map, then a rerun of every stream whose level-0 inputs reach 2^122)
    equals clear + K oracle sweeps on every data set, fused clear at PRESSURE 0.8, 1 and 2.  Every data set
    sends some streams through the exact tail (inf counts as large); with a patch, the others stay contracted."""
    for W, H, K, R in ((256, 40, 4, 16), (132, 45, 13, 27)):
        p, d = special_fields(kind, W, H, 4, pressure)
        if kind in ("near_max", "near_max_neg", "huge_div"):
            assert overflow_sweep(oracle, p, d, K, pressure) is not None, (kind, pressure)
        st = {}
        got = jacobi_tb_model(p, d, K, R, scale=pressure, stats=st)
        assert equal(kind, got, oracle.jacobi(oracle.clear(p, pressure), d, K)), (kind, pressure, W, K)
        streams = -(-W // (128 - 2 * ((K + 3) // 4 * 4))) * -(-H // R)
        assert 0 < st["exact_streams"] <= streams, (kind, st)
        if kind not in NONFINITE_KINDS:         # a patch: the streams that do not read it stay contracted
            assert st["exact_streams"] < streams, (kind, st)


def test_model_runs_ordinary_data_contracted(oracle):
    """No exact stream on ordinary data: the guard costs the common case nothing but the tracking."""
    rng = np.random.default_rng(8)
    p = rng.standard_normal((40, 256)).astype(np.float32) * np.float32(1e30)
    d = rng.uniform(-1, 1, (40, 256)).astype(np.float32) * np.float32(1e30)
    st = {}
    assert bits_equal(jacobi_tb_model(p, d, 5, 16, scale=0.8, stats=st), oracle.jacobi(oracle.clear(p, 0.8), d, 5))
    assert st["exact_streams"] == 0
