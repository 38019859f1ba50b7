"""CPU model of render(null) on the canvas's RGBA8 drawing buffer (fluid_render_canvas, include/fluid.h).
Test infrastructure.

The input is the bare display fragment (c, a) of the same handle: render(w, h, target=True) with
TRANSPARENT, i.e. FLUID_BACKGROUND 2, the display kernel with no blend, row 0 = bottom.  Everything below is
numpy float32, where every operation is rounded on its own, like the kernel's __fmul_rn / __fadd_rn /
__fsub_rn / __fdiv_rn:

    clamp(x) = fmin(fmax(x, 0), 1)             NaN -> 0, +inf -> 1
    u8(x)    = rint(clamp(x) * 255)            round to nearest, ties to even
    d8       = u8(BACK_COLOR / 255), or u8(checkerboard) with TRANSPARENT; alpha byte 255
    d        = d8 / 255
    out      = clamp(c) + d * (1 - clamp(a)),  alpha clamp(a) + 1 * (1 - clamp(a))
    byte     = u8(out), rows stored top row first.

`canvas(..., mutant=name)` applies one wrong rule instead, so the tests can show that their inputs tell it
from the right one: "no_clamp" (the fp32 blend of render(), quantised afterwards), "truncate",
"unquantised_dst" (d = the fp32 background), "fused" (d * (1 - a) + c rounded once) and "bottom_first".
"""
import numpy as np

from display_model import checkerboard

F = np.float32
MUTANTS = ("no_clamp", "truncate", "unquantised_dst", "fused", "bottom_first")


def clamp(x):
    return np.fmin(np.fmax(np.asarray(x, F), F(0)), F(1))


def u8(x, truncate=False):
    """The float-to-unorm conversion of the drawing buffer: clamp(x) * 255 rounded to nearest even."""
    s = clamp(x) * F(255)
    return (np.trunc(s) if truncate else np.rint(s)).astype(np.uint8)


def background(w, h, back_rgb, transparent, aspect):
    """The fp32 colour drawn under the display, (h, w, 3), row 0 = bottom: BACK_COLOR / 255 or the checkerboard."""
    if transparent:
        v = checkerboard(w, h, aspect)
        return np.stack([v, v, v], axis=-1)
    return np.broadcast_to(np.asarray(back_rgb, F), (h, w, 3)).astype(F)


def destination_bytes(w, h, back_rgb, transparent, aspect):
    """d8 of the three colour channels, (h, w, 3) uint8, row 0 = bottom (the alpha byte is 255)."""
    return u8(background(w, h, back_rgb, transparent, aspect))


def canvas(frag, back_rgb, transparent, aspect, mutant=None):
    """The canvas bytes (h, w, 4) uint8, TOP row first, for the bare fragment `frag` (h, w, 4) float32
    (row 0 = bottom), over BACK_COLOR (`back_rgb` = BACK_COLOR / 255) or the checkerboard."""
    assert mutant is None or mutant in MUTANTS, mutant
    frag = np.asarray(frag, F)
    h, w = frag.shape[:2]
    c, a = frag[..., :3], frag[..., 3:4]
    if mutant == "unquantised_dst":
        d = background(w, h, back_rgb, transparent, aspect)
    else:
        d = destination_bytes(w, h, back_rgb, transparent, aspect).astype(F) / F(255)
    d = np.concatenate([d, np.ones((h, w, 1), F)], axis=-1)        # u8(1) / 255 = 1: the destination alpha
    src = np.concatenate([c, a], axis=-1)
    if mutant != "no_clamp":
        src, a = clamp(src), clamp(a)
    k = F(1) - a
    with np.errstate(invalid="ignore", over="ignore"):
        if mutant == "fused":
            out = (d.astype(np.float64) * k.astype(np.float64) + src.astype(np.float64)).astype(F)
        else:
            out = src + d * k
    img = u8(out, truncate=mutant == "truncate")
    return img if mutant == "bottom_first" else img[::-1].copy()


def fused_witnesses(d, n, rng, half=True):
    """n texels (r, 0, a) whose red byte over destination value d differs between the rule and the fused
    mutant: a = max channel, so out.r = r + d * (1 - a).  With `half`, r and a are fp16-representable, so
    they survive a half-storage dye unchanged.  Returns an (n, 3) float32 array of (r, 0, a)."""
    d = F(d)
    grid = np.arange(1, 0x3C00, dtype=np.uint16).view(np.float16).astype(F) if half else \
        rng.random(1 << 15, dtype=F)                                  # the positive fp16 values below 1
    found = []
    while len(found) < n:
        a = rng.choice(grid[grid > F(0.05)], 64)[:, None]
        r = grid[None, :]
        k = F(1) - a
        ok = r <= a
        rule = u8(r + d * k)
        fused = u8((d.astype(np.float64) * k.astype(np.float64) + r).astype(F))
        hit = np.argwhere(ok & (rule != fused))
        for i, j in hit[: n - len(found)]:
            found.append((r[0, j], F(0), a[i, 0]))
    return np.asarray(found, F)
