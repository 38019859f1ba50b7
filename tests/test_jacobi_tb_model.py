"""The temporally-blocked Jacobi kernel's algorithm (lane-level model of the CUDA code) must equal
K plain sweeps of the oracle BITWISE — including walls, mirrored x-halos, chunk seams."""
import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import jacobi_tb_model


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
# Data sets the contracted tail must survive (shared with the GPU tests).  Stored pressure is divided by
# PRESSURE so that the fused clear brings the patch to the magnitude that overflows at once.
KINDS = ["near_max", "near_max_neg", "huge_div", "nonfinite", "full_range"]
NONFINITE_KINDS = {"nonfinite", "full_range"}          # inf / NaN in the inputs
# results that can hold NaN (inf - inf of overflowed neighbours), whose bits differ between x86 and the GPU:
# compared NaN-aware, the others bitwise
NAN_KINDS = NONFINITE_KINDS | {"huge_div"}


def special_fields(kind, W, H, seed, pressure=1.0):
    """(p, d) of one data set: ordinary fields with
    near_max      p = 8.5e37 / PRESSURE over a patch and d = -1e37 under it: four such neighbours sum to
                  3.4e38 and S - d rounds to +inf in the first sweep, while S/4 - d/4 is finite;
    near_max_neg  the same with both signs flipped;
    huge_div      |d| in [2^126, FLT_MAX] over a patch of ordinary p: the first sweep leaves p ~ -d/4 and
                  the second one overflows;
    nonfinite     +-inf and NaN sprinkled into both p and d;
    full_range    binary exponents -149..127 tile by tile for both (subnormals to inf)."""
    from test_gpu_fast_paths import exp_tiled
    rng = np.random.default_rng(seed)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    r0, r1 = H // 4, min(H // 4 + max(3, H // 3), H)
    c0, c1 = W // 3, W // 3 + max(8, W // 4)
    if kind in ("near_max", "near_max_neg"):
        sg = np.float32(1.0 if kind == "near_max" else -1.0)
        p[r0:r1, c0:c1] = sg * np.float32(8.5e37 / pressure)
        d[max(r0 - 1, 0):r1 + 1, c0 - 1:c1 + 1] = -sg * np.float32(1e37)
    elif kind == "huge_div":
        mag = rng.uniform(2.0 ** 126, float(np.finfo(np.float32).max), (r1 - r0, c1 - c0))
        d[r0:r1, c0:c1] = (mag * rng.choice([-1.0, 1.0], mag.shape)).astype(np.float32)
    elif kind == "nonfinite":
        for a in (p, d):
            k = rng.choice(H * W, size=max(6, H * W // 500), replace=False)
            a.flat[k] = rng.choice(np.array([np.inf, -np.inf, np.nan], np.float32), k.size)
    else:
        p = exp_tiled((H, W), seed, lo=-149, hi=127, tile=(4, 16))
        d = exp_tiled((H, W), seed + 1, lo=-149, hi=127, tile=(4, 16))
    return p, d


def overflow_sweep(oracle, p, d, iters, pressure):
    """First sweep (1-based) of the oracle's clear + `iters` sweeps with a cell whose S and d are finite and
    whose rn(S - d) is infinite -- where the contracted tail would differ -- or None."""
    q = oracle.clear(p, pressure)
    for k in range(1, iters + 1):
        e = np.pad(q, 1, mode="edge")
        with np.errstate(invalid="ignore", over="ignore"):
            S = ((e[1:-1, :-2] + e[1:-1, 2:]) + e[:-2, 1:-1]) + e[2:, 1:-1]
            hit = np.isfinite(S) & np.isfinite(d) & np.isinf(S - d)
        if hit.any():
            return k
        q = oracle.jacobi(q, d, 1)
    return None


def equal(kind, a, b):
    from test_gpu_fast_paths import same_or_both_nan
    return same_or_both_nan(a, b) if kind in NAN_KINDS else bits_equal(a, b)


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
