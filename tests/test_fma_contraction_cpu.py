"""The arithmetic identity the temporally blocked Jacobi kernel (csrc/jacobi.cuh, generation 7) relies on:

        fma(S, 0.25, -0.25*d)  ==  (S - d) * 0.25        bit for bit in fp32,

whenever d == 0 or |d| >= 2^-123, and rn(S - d) is finite.  Both conditions are needed:
  * for 0 < |d| < 2^-123 the two sides can differ (double rounding into the subnormal range), which is
    why the producers of `divergence` keep the tiny-value map and flagged warps run the exact form;
  * for finite S and d with |S - d| >= 2^128 - 2^103 the reference rounds S - d to +-inf and the fma
    gives the finite S/4 - d/4.  That needs max(|S|, |d|) >= 2^127 - 2^102; a contracted stream whose
    level-0 inputs reach BIG_IN = 2^122 runs again with the exact form, and below that no sweep of a
    launch of depth <= 13 gets there (test_big_in_keeps_every_level_of_a_launch_finite proves it).
Non-finite operands give the same result on both sides.  Checked here with exact rational arithmetic
and IEEE special-value rules (no GPU, no fma instruction needed)."""
import os
import re
from fractions import Fraction

import numpy as np

from jacobi_tb_model import BIG_IN, _finite, add32, fma, fma32, fma_tail, mul32, ref

F32 = np.float32
TINY = 2.0 ** -123
FLT_MAX = float(np.finfo(np.float32).max)              # 2^128 - 2^104
OVERFLOW = Fraction(2) ** 128 - Fraction(2) ** 103     # rn32(x) is +-inf iff |x| >= this
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(x):
    return np.array([x], F32).view(np.uint32)[0]


def _same(x, y):
    return (np.isnan(x) and np.isnan(y)) or _bits(x) == _bits(y)


def _samples(rng, n):
    """(S, d) pairs stressing cancellation and both ends of the exponent range."""
    out = []
    for _ in range(n):
        kind = rng.integers(0, 7)
        if kind == 0:       # ordinary magnitudes
            S, d = rng.standard_normal() * 10 ** rng.uniform(-3, 3), rng.uniform(-1, 1)
        elif kind == 1:     # heavy cancellation: S within a few ulps of d
            d = rng.standard_normal()
            S = float(F32(d)) * (1 + rng.integers(-8, 9) * 2.0 ** -23)
        elif kind == 2:     # both near the bottom of the normal range
            S, d = rng.uniform(-1, 1) * 2.0 ** rng.integers(-126, -110), rng.uniform(-1, 1) * 2.0 ** rng.integers(-123, -110)
        elif kind == 3:     # subnormal S, d just above the guard
            S, d = rng.uniform(-1, 1) * 2.0 ** -127, (1 + rng.uniform(0, 1)) * 2.0 ** -123 * rng.choice([-1, 1])
        elif kind == 4:     # d == 0 with tiny S
            S, d = rng.uniform(-1, 1) * 2.0 ** rng.integers(-149, -120), 0.0
        elif kind == 5:     # |S - d| lands in the double-rounding band [2^-125, 2^-124) with a safe d
            d = (1 + rng.uniform(0, 1)) * 2.0 ** -123
            S = d + rng.uniform(1, 2) * 2.0 ** -125 * rng.choice([-1, 1])
        else:               # the top of the range: |S - d| on either side of the overflow threshold
            S = rng.uniform(1, 2) * 2.0 ** rng.integers(124, 128) * rng.choice([-1, 1])
            d = rng.uniform(1, 2) * 2.0 ** rng.integers(120, 128) * rng.choice([-1, 1])
        out.append((F32(min(max(S, -FLT_MAX), FLT_MAX)), F32(min(max(d, -FLT_MAX), FLT_MAX))))
    return out


def test_contracted_tail_equals_reference_outside_the_guard():
    """Outside both guards -- d is 0 or |d| >= 2^-123, and rn(S - d) is finite -- the tails agree; at the
    top of the range they agree exactly when rn(S - d) is finite, i.e. |S - d| < 2^128 - 2^103."""
    rng = np.random.default_rng(123)
    checked = overflowed = 0
    for S, d in _samples(rng, 7000):
        if d != 0 and abs(float(d)) < TINY:
            continue
        r, f = ref(S, d), fma(S, d)
        diff = abs(Fraction(float(S)) - Fraction(float(d)))
        assert np.isinf(add32(S, -d)) == (diff >= OVERFLOW), (float(S), float(d))
        if diff >= OVERFLOW:
            assert np.isinf(r) and np.isfinite(f), (float(S), float(d))
            overflowed += 1
        else:
            assert _bits(r) == _bits(f), (float(S), float(d))
            checked += 1
    assert checked > 5000 and overflowed > 40


def test_guard_is_needed_for_tiny_nonzero_divergence():
    """A concrete pair with 0 < |d| < 2^-123 where the contraction is NOT bit-exact."""
    rng = np.random.default_rng(7)
    found = 0
    for _ in range(4000):
        d = F32(rng.integers(1, 2 ** 22) * 2.0 ** -149 * rng.choice([-1, 1]))          # subnormal d
        S = F32(rng.uniform(1, 2) * 2.0 ** -125 * rng.choice([-1, 1]))
        if _bits(ref(S, d)) != _bits(fma(S, d)):
            found += 1
    assert found > 0


def test_contraction_fails_where_s_minus_d_overflows():
    """Finite S and d with rn(S - d) = +-inf: the reference gives +-inf, the fma a finite value.  The three
    pairs of the Jacobi update that reach it (four neighbours of 8.5e37 over d = -1e37, ...) and sampled
    pairs with |S - d| >= 2^128 - 2^103."""
    four = add32(add32(add32(F32(8.5e37), F32(8.5e37)), F32(8.5e37)), F32(8.5e37))
    for S, d, want in ((four, F32(-1e37), np.inf), (F32(2e38), F32(-2e38), np.inf), (F32(-3e38), F32(1e38), -np.inf)):
        r, f = ref(S, d), fma(S, d)
        assert r == want and np.isfinite(f), (float(S), float(d), r, f)
    rng = np.random.default_rng(11)
    found = 0
    for _ in range(3000):
        S = F32(rng.uniform(2.0 ** 126, FLT_MAX))
        d = F32(-rng.uniform(2.0 ** 126, FLT_MAX))
        sg = rng.choice([-1, 1])
        S, d = F32(sg * S), F32(sg * d)
        if abs(Fraction(float(S)) - Fraction(float(d))) < OVERFLOW:
            continue
        r, f = ref(S, d), fma(S, d)
        assert np.isinf(r) and np.sign(r) == sg and np.isfinite(f), (float(S), float(d))
        found += 1
    assert found > 1000


def test_nonfinite_operands_agree():
    """Every combination of +-inf, NaN, +-0 and finite values in S and d gives the same result on both
    tails (NaN on both, or the same bits): the guard has nothing to do for them."""
    vals = [F32(np.inf), F32(-np.inf), F32(np.nan), F32(0.0), F32(-0.0), F32(1.5), F32(-3.25),
            F32(FLT_MAX), F32(-FLT_MAX), F32(2.0 ** -120), F32(-(2.0 ** -149))]
    n = 0
    for S in vals:
        for d in vals:
            if d != 0 and abs(float(d)) < TINY:
                continue                      # tiny divergence: the other guard
            if _finite(S, d) and abs(Fraction(float(S)) - Fraction(float(d))) >= OVERFLOW:
                continue                      # finite overflow: the failure above
            if not (_finite(S, d) and S != 0 and d != 0) or (S == 0 and d == 0):
                n += 1
            assert _same(ref(S, d), fma(S, d)), (S, d, ref(S, d), fma(S, d))
    assert n > 60


def test_signed_zeros_agree():
    for S in (F32(0.0), F32(-0.0)):
        for d in (F32(0.0), F32(-0.0)):
            assert _bits(ref(S, d)) == _bits(fma(S, d))
    assert _bits(ref(F32(-0.0), F32(0.0))) == _bits(F32(-0.0))     # the zero signs are modelled, not lost


def test_contraction_is_exact_below_the_overflow_bound():
    """Neighbours below 2^125 and |d| < 2^126 (the most a launch reaches from level-0 inputs below BIG_IN,
    next test): rn(S - d) is finite and both tails agree, sampled at the edge of that box."""
    below125, below126 = F32(2.0 ** 125 - 2.0 ** 101), F32(2.0 ** 126 - 2.0 ** 102)
    # the largest |S| four such neighbours can sum to, through the monotone roundings of the reference's order
    smax = add32(add32(add32(below125, below125), below125), below125)
    assert Fraction(float(smax)) + Fraction(float(below126)) < OVERFLOW
    rng = np.random.default_rng(3)
    for _ in range(4000):
        nb = [F32(rng.choice([-1, 1]) * float(below125) * (1 - rng.integers(0, 4) * 2.0 ** -23 * rng.integers(0, 2)))
              for _ in range(4)]
        S = add32(add32(add32(nb[0], nb[1]), nb[2]), nb[3])
        d = F32(rng.choice([-1, 1]) * float(below126) * (1 - rng.uniform(0, 2.0 ** -10) * rng.integers(0, 2)))
        r = ref(S, d)
        assert np.isfinite(r) and _bits(r) == _bits(fma(S, d)), (nb, float(d))


def _big_in_and_kmax():
    src = open(os.path.join(ROOT, "webgl_fluid_simulation_b200", "csrc", "jacobi.cuh")).read()
    big = float(re.search(r"constexpr float BIG_IN = ([0-9.e+]+)f;", src).group(1))
    kmax = int(re.search(r"constexpr int KMAX = (\d+);",
                         open(os.path.join(ROOT, "webgl_fluid_simulation_b200", "csrc", "fluid.cu")).read()).group(1))
    return big, kmax


def test_big_in_keeps_every_level_of_a_launch_finite():
    """The threshold the kernel tests, proved.  Round to nearest is monotone and odd, so |rn(a + b)| <=
    rn(A + B) for |a| <= A, |b| <= B, and likewise for the other operations: running the reference's update
    on the magnitude bounds bounds every finite value of the next level.  (A cell with an inf or NaN operand
    is inf or NaN in both tails, previous test; inf among the inputs also reaches BIG_IN.)  Starting from
    level-0 inputs below BIG_IN (scaled pressure and divergence alike), every level that feeds a sweep of a
    launch of depth <= KMAX stays below 2^125 and |d| below 2^126: the box of the previous test."""
    big, kmax = _big_in_and_kmax()
    assert big == 2.0 ** 122 == BIG_IN
    below = F32(np.nextafter(F32(big), F32(0)))
    P, D = below, below
    for t in range(kmax):                     # P bounds level t, the input of sweep t + 1
        assert float(P) < 2.0 ** 125 and float(D) < 2.0 ** 126, t
        S = add32(add32(add32(P, P), P), P)
        P = mul32(add32(S, D), F32(0.25))
    assert float(P) < 2.0 ** 125              # one sweep of slack beyond KMAX
    # and the threshold is not idle: 2^124 would let a depth-KMAX launch reach an overflowing tail
    P = D = F32(2.0 ** 124)
    for t in range(kmax):
        S = add32(add32(add32(P, P), P), P)
        if Fraction(float(S)) + Fraction(float(D)) >= OVERFLOW:
            break
        P = mul32(add32(S, D), F32(0.25))
    else:
        raise AssertionError("2^124 inputs never reach the overflow")


def test_model_fma_emulation_is_exact():
    """jacobi_tb_model emulates the fma as rn32(float64(S * 0.25) + float64(d')): S * 0.25 and the sum
    of two fp32 values are exact or rounded once in float64, and a float64 (53-bit) rounding followed by
    an fp32 (24-bit) one equals the direct rounding for addition since 53 >= 2*24 + 2 (Figueroa).  Checked
    against the exact fma here on every sampled pair, non-finite and signed-zero operands included."""
    rng = np.random.default_rng(99)
    pairs = _samples(rng, 5000)
    specials = [F32(np.inf), F32(-np.inf), F32(np.nan), F32(0.0), F32(-0.0), F32(FLT_MAX), F32(2.0 ** -149)]
    pairs += [(S, d) for S in specials for d in specials]
    S = np.array([p[0] for p in pairs], F32)
    dq = np.array([mul32(p[1], F32(-0.25)) for p in pairs], F32)
    with np.errstate(invalid="ignore", over="ignore"):
        got = fma_tail(S, dq)
    for k, (s, d) in enumerate(pairs):
        assert _same(got[k], fma32(s, F32(0.25), dq[k])), (float(s), float(d))
