"""A per-texel interval for the display shader with BLOOM (displayShaderSource S:549-612, linearToGamma
S:565-568), independent of the library: numpy plus the fetches of display_keywords_model.py.

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

import capture_model as CM
import display_keywords_model as M
from oracle import oracle as O
from splat_model import check_splat, step_ulps

F32 = np.float32
# CUDA C++ Programming Guide, Mathematical Functions, single precision: powf(x, y) maximum error
# 4 ulp (full range, without -use_fast_math)
POWF_ULP = 4
Y = M.GAMMA_EXPONENT


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


def gamma_interval(dye, w, h, keywords, bloom, sun, dither, scale=None):
    """[lo, hi] of the display colour c + linearToGamma(bloom) of a w x h target, (h, w, 3) each, before
    alpha and the background.  `scale`: getTextureScale of the target unless given."""
    assert keywords & M.BLOOM, keywords
    with np.errstate(invalid="ignore", over="ignore"):
        c, bl = M.colour_terms(np.ascontiguousarray(dye, F32), w, h, keywords, bloom, sun)
        bk = M.gamma_argument(bl, np.ascontiguousarray(dither, F32), w, h, scale)
        plo, phi = powf_bounds(bk)
        return c + M.linear_to_gamma(plo), c + M.linear_to_gamma(phi)


def blend_interval(clo, chi, back_rgb, background, aspect):
    """[lo, hi] (h, w, 4) of the frame from the colour interval: alpha and render()'s blend over the
    background (O.BG_COLOR / BG_CHECKERBOARD), or bare (BG_NONE)."""
    alo, ahi = M.alpha_of(clo), M.alpha_of(chi)
    if background == O.BG_NONE:
        return np.concatenate([clo, alo], axis=-1), np.concatenate([chi, ahi], axis=-1)
    h, w = clo.shape[:2]
    bg = M.background_colour(w, h, back_rgb, background, aspect)
    one = F32(1)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = np.concatenate([clo + bg * (one - ahi), alo + one * (one - ahi)], axis=-1)
        hi = np.concatenate([chi + bg * (one - alo), ahi + one * (one - alo)], axis=-1)
    return lo, hi


def display_interval(dye, w, h, keywords, bloom, sun, dither, back_rgb, background, aspect):
    """[lo, hi] of every value of render()'s frame with `keywords` (which include BLOOM)."""
    clo, chi = gamma_interval(dye, w, h, keywords, bloom, sun, dither)
    return blend_interval(clo, chi, back_rgb, background, aspect)


def capture_interval(dye, w, h, canvas_w, canvas_h, dither, keywords, transparent, back_rgb, cfg=None, scale=None):
    """[lo, hi] of every byte of captureScreenshot() with `keywords` (which include BLOOM), top row first:
    the bloom and sunrays chains of the oracle at the canvas size, the display at the target size over
    the fp16 background, then B.  `scale` overrides the target's getTextureScale (a negative control)."""
    r = O.render_postfx(np.ascontiguousarray(dye, F32), canvas_w, canvas_h, np.ascontiguousarray(dither, F32), cfg=cfg)
    clo, chi = gamma_interval(dye, w, h, keywords, r["bloom"], r["sunrays"], dither, scale)
    lo, hi = blend_interval(clo, chi, CM.back16(back_rgb), O.BG_NONE if transparent else O.BG_COLOR, w / h)
    return CM.to_bytes(lo)[::-1], CM.to_bytes(hi)[::-1]


def check_display(got, lo, hi, limit: int = 8):
    """The values of `got` outside [lo, hi]: NaN where the interval is NaN and nowhere else, infinities
    exactly, the sign of a zero where both ends are that zero (check_splat's rule).  Returns (number of
    offending values, the first `limit` as (index, got, lo, hi))."""
    assert np.array_equal(np.isnan(lo), np.isnan(hi)), "an interval end is NaN where the other is not"
    return check_splat(got, lo, hi, limit)


def bytes_outside(got, lo, hi) -> int:
    """How many bytes of `got` lie outside [lo, hi] (capture_interval)."""
    return int(np.count_nonzero((got < lo) | (got > hi)))


def same_bits(a, b) -> bool:
    """fp32 arrays equal bit for bit with NaN in the same places, NaN payloads ignored (the device's
    canonical NaN is 0x7fffffff, x86's default NaN 0xffc00000)."""
    a = np.ascontiguousarray(a, F32); b = np.ascontiguousarray(b, F32)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    keep = ~np.isnan(a)
    return np.array_equal(a.view(np.uint32)[keep], b.view(np.uint32)[keep])
