"""A per-texel interval for the display shader with BLOOM (displayShaderSource S:549-612, linearToGamma
S:565-568), independent of the library: the powf bounds display_model.display builds it from, and the
comparisons the tests make against it.

Everything before linearToGamma's pow is fp32 arithmetic that numpy reproduces bit for bit in the
kernel's order (no contraction; the library is built with --fmad=false): the LINEAR fetches of dye and
bloom, SHADING's diffuse, the sunrays multiply of both, the REPEAT dithering fetch at
vUv * getTextureScale (JS doubles narrowed once), noise / 255 and fmaxf(bk, 0).  Every max and min has
C semantics (np.fmax / np.fmin drop a NaN argument, as fmaxf / fminf do in CUDA and in the oracle).

p = powf(bk, 0.416666667f) is not exactly reproducible: the device's powf is within POWF_ULP ulp of
pow(bk, y) (the CUDA Math API's documented maximum error), glibc's within 1.  So p is bounded by
[lo, hi]: pow(float64(bk), float64(y)) rounded to fp32 and widened by POWF_ULP steps of nextafter,
clamped at 0.  powf's special cases at the arguments bk can take are exact, and kept exact here:
pow(0, y) = 0, pow(1, y) = 1, pow(inf, y) = inf (bk is never negative or NaN after fmaxf(bk, 0)).

Every later step is monotone in each of its arguments, so [lo, hi] carries through texel by texel:
fmaxf(1.055f * p - 0.055f, 0), c + that; alpha = fmaxf of the three channels; the blend c + bg * (1 - a)
with bg >= 0 (a channel's low end takes alpha's high end and the reverse) and alpha's a + 1 * (1 - a)
(each of a's two occurrences bounded on its own); for captureScreenshot the fp16 background of
capture_model.back16 and the byte map B, which is monotone: a byte lies in [B(lo), B(hi)].

Non-finite values are exact at both ends: an inf or NaN in c is the same in lo and hi, the bloom term
is +0 or finite where bk is finite, and inf only where bk is inf, where powf is exact.  The bloom term
is never -0 (fmaxf(x, +0) with x != -0), so with BLOOM no channel is -0 and fmaxf(-0, +0) -- on which
C libraries and the device need not agree -- is never evaluated by alpha."""
from __future__ import annotations

import numpy as np

from splat_model import check_splat, step_ulps

F32 = np.float32
# CUDA C++ Programming Guide, Mathematical Functions, single precision: powf(x, y) maximum error
# 4 ulp (full range, without -use_fast_math)
POWF_ULP = 4
Y = F32(0.416666667)                     # linearToGamma's exponent


def pow_rn(bk, y=Y) -> np.ndarray:
    """pow(bk, y) correctly rounded to fp32 (float64 pow is far more accurate than half an fp32 ulp)."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        return np.power(np.asarray(bk, np.float64), np.float64(y)).astype(F32)


def powf_bounds(bk, ulp: int = POWF_ULP):
    """[lo, hi] holding powf(bk, y) of any implementation within `ulp` of pow(bk, y), for bk >= 0."""
    p = pow_rn(bk)
    exact = (bk == 0) | (bk == 1) | np.isinf(bk)
    lo = np.where(exact, p, np.fmax(step_ulps(p, -ulp), F32(0.0)))
    hi = np.where(exact, p, step_ulps(p, ulp))
    return lo, hi


def check_display(got, lo, hi, limit: int = 8):
    """The values of `got` outside [lo, hi]: NaN where the interval is NaN and nowhere else, infinities
    exactly, the sign of a zero where both ends are that zero (check_splat's rule).  Returns (number of
    offending values, the first `limit` as (index, got, lo, hi))."""
    assert np.array_equal(np.isnan(lo), np.isnan(hi)), "an interval end is NaN where the other is not"
    return check_splat(got, lo, hi, limit)


def bytes_outside(got, lo, hi) -> int:
    """How many bytes of `got` lie outside [lo, hi] (the byte bracket of display_model.capture)."""
    return int(np.count_nonzero((got < lo) | (got > hi)))


def same_bits(a, b) -> bool:
    """fp32 arrays equal bit for bit with NaN in the same places, NaN payloads ignored (the device's
    canonical NaN is 0x7fffffff, x86's default NaN 0xffc00000)."""
    a = np.ascontiguousarray(a, F32); b = np.ascontiguousarray(b, F32)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    keep = ~np.isnan(a)
    return np.array_equal(a.view(np.uint32)[keep], b.view(np.uint32)[keep])
