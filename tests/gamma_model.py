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

from sim_harness import same_bits  # noqa: F401 -- G.same_bits of the display tests
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


# ---- half-float post-FX targets (FLUID_FLAG_HALF_POSTFX) against the executed shaders, CPU and GPU ----
CAPTURE_SETS = ["none", "shading", "bloom", "shading_bloom", "sunrays", "shading_sunrays", "bloom_sunrays",
                "shading_bloom_sunrays"]        # index = FLUID_DISPLAY_* mask
POW2, RAGGED = "keywords_half_64_to_128", "keywords_half_48x32_to_50x75"
# Frames against the executed shaders, max_rel (field-normalised).  Measured, oracle vs executed: 0 on
# the power-of-two fixture (bit for bit), 2.52e-4 on the ragged one (shading_sunrays 2.40e-4, bloom
# 4.7e-5), all from the ragged chains below.  The GPU adds powf's <= 4 ulp with BLOOM.
FRAME_TOL = 3e-4
# The ragged fixture's chains, measured: at most 1 fp16 ulp, in 2 of 24576 bloom values, 3 of 3456
# sunrays texels and 1 of 1536 mask texels.  Cause: the rasteriser's vUv = aPosition * 0.5 + 0.5 is not
# (i + .5) / W in fp32 for a W that is not a power of two (DESIGN §2, non-power-of-two advection); the
# LINEAR weights move by an fp32 ulp and now and then that flips an fp16 rounding.  The pyramid levels
# are bit for bit.
RAGGED_CHAIN_TEXELS = {"bloom": 2, "sunrays": 3, "mask_alpha": 1}


def cfg_of(g):
    return dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]))


def fp16_ulps(a, b):
    a = np.asarray(a, np.float16).view(np.int16).astype(np.int64)
    b = np.asarray(b, np.float16).view(np.int16).astype(np.int64)
    return int(np.abs(a - b).max())
