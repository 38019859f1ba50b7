"""The bytes of captureScreenshot() (S:287-299): the fp16 store of its RGBA half-float target, normalizeTexture's
clamp01 * 255 truncated to uint8 (S:309-327), the fp16 background, and the byte tolerance rule.  Test
infrastructure; display_model.capture draws the values these quantise.

The byte tolerance rule: B(x) = trunc(clamp01(fp16(x)) * 255) is monotone in x, so a byte is accepted
when it lies in [B(v - d), B(v + d)] with v the model's fp32 pre-store value and d = delta * max(1, |v|),
delta being the fp32 tolerance of the same comparison against the executed shaders.  Against this
build, captures with BLOOM are checked per texel instead (the lo / hi bytes of display_model.capture).
"""
import numpy as np


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


def byte_bracket(pre, delta):
    """[B(v - d), B(v + d)] of the rule, flipped to the image's top-first row order."""
    v = np.asarray(pre, np.float64)
    d = delta * np.maximum(1.0, np.abs(v))
    return to_bytes(v - d)[::-1], to_bytes(v + d)[::-1]


def bytes_outside(got, pre, delta):
    """How many bytes of `got` (top row first) fall outside the rule's bracket around `pre`."""
    lo, hi = byte_bracket(pre, delta)
    return int(np.count_nonzero((got < lo) | (got > hi)))
