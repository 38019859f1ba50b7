"""CPU model of captureScreenshot() (S:287-299) up to normalizeTexture (S:309-327).  Test infrastructure.

Built on display_keywords_model.py: the bloom and sunrays chains come from the oracle's render_postfx run
at the CANVAS size (initBloomFramebuffers / initSunraysFramebuffers size them from the drawing buffer,
S:1012-1043), the display shader is the model's numpy restatement at the TARGET size (texelSize and
ditherScale use the target, S:1332-1344) over drawColor(BACK_COLOR) stored in fp16, or bare with
TRANSPARENT.  Then the fp16 store of the RGBA half-float target, normalizeTexture's clamp01 * 255
truncated to uint8, and its flip (top row first).

The byte tolerance rule: B(x) = trunc(clamp01(fp16(x)) * 255) is monotone in x, so a byte is accepted
when it lies in [B(v - d), B(v + d)] with v the model's fp32 pre-store value and d = delta * max(1, |v|),
delta being the fp32 tolerance of the same comparison against the executed shaders.  Against this
build, captures with BLOOM are checked per texel instead (gamma_model.capture_interval).
"""
import numpy as np

import display_keywords_model as M
from oracle import oracle as O

SHADING, BLOOM, SUNRAYS = M.SHADING, M.BLOOM, M.SUNRAYS


def half_round(x):
    """The RGBA16F store: round to nearest even, overflow to +-Inf (numpy's float16 cast)."""
    with np.errstate(over="ignore"):
        return np.asarray(x).astype(np.float16)


def to_bytes(x):
    """B(x): the fp16 store of x, then normalizeTexture's clamp01(v) * 255 into a Uint8Array (ToUint8:
    NaN -> 0, otherwise truncation).  Same row order as x."""
    v = half_round(x).astype(np.float64)
    c = np.minimum(np.maximum(v, 0.0), 1.0) * 255.0
    return np.where(np.isnan(c), 0.0, np.trunc(c)).astype(np.uint8)


def back16(back_rgb):
    """drawColor's store of normalizeColor(BACK_COLOR) (fp32 uniform) into the half-float target."""
    return tuple(float(half_round(np.float32(c))) for c in back_rgb)


def capture(dye, w, h, canvas_w, canvas_h, dither, keywords, transparent, back_rgb, cfg=None, fx_size=None):
    """captureScreenshot with `keywords` into a w x h target on a canvas_w x canvas_h canvas.  Returns
    dict(pre = the fp32 value before the fp16 store (h, w, 4), row 0 = bottom; rgba8 = the uint8 image,
    row 0 = top).  fx_size: the (w, h) the post-FX FBOs are sized from instead of the canvas (a negative
    control: the reference does not do this)."""
    dye = np.ascontiguousarray(dye, np.float32)
    fw, fh = fx_size or (canvas_w, canvas_h)
    dith = np.ascontiguousarray(dither, np.float32) if keywords & BLOOM else M._NO_DITHER
    bloom = sun = None
    if keywords & (BLOOM | SUNRAYS):
        r = O.render_postfx(dye, fw, fh, dith, cfg=cfg)
        bloom, sun = r["bloom"], r["sunrays"]
    pre = M._display(dye, w, h, keywords, bloom, sun, dith, back16(back_rgb), O.BG_NONE if transparent else O.BG_COLOR,
                     w / h)
    return dict(pre=pre, rgba8=to_bytes(pre)[::-1].copy())


def byte_bracket(pre, delta):
    """[B(v - d), B(v + d)] of the rule, flipped to the image's top-first row order."""
    v = np.asarray(pre, np.float64)
    d = delta * np.maximum(1.0, np.abs(v))
    return to_bytes(v - d)[::-1], to_bytes(v + d)[::-1]


def bytes_outside(got, pre, delta):
    """How many bytes of `got` (top row first) fall outside the rule's bracket around `pre`."""
    lo, hi = byte_bracket(pre, delta)
    return int(np.count_nonzero((got < lo) | (got > hi)))
