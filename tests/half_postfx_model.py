"""CPU model of render() and captureScreenshot() with FLUID_FLAG_HALF_POSTFX.  Test infrastructure.

The bloom FBO, each pyramid level, sunrays and sunraysTemp are RGBA16F / R16F like the reference's FBOs
(initBloomFramebuffers / initSunraysFramebuffers S:1012-1043, halfFloatTexType S:138-147): every blit's fp32
result is rounded to fp16 when it is stored (nearest even, overflow to +-inf, NaN stays NaN).  The additive
up-pass (blendFunc(ONE, ONE), S:1374-1375) adds the widened destination in fp32 and rounds once.  The
sunrays mask is drawn into dye.write (S:1300), so it has the dye's storage: fp16 on a half-storage handle
(half_mask).

The chains are the oracle's per-blit C functions (those oracle.render_postfx calls) with oracle.round_half
after each call; the display shader, the background, the powf interval and the capture bytes are those of
display_keywords_model.py, capture_model.py and gamma_model.py, fed with these chains.  With
half_targets = half_mask = False every function here returns what its counterpart there returns.
"""
import ctypes as C

import numpy as np

import capture_model as CM
import display_keywords_model as M
import gamma_model as G
from oracle import oracle as O

F = np.float32
SHADING, BLOOM, SUNRAYS = M.SHADING, M.BLOOM, M.SUNRAYS


def _chain_lib():
    """The oracle library with the signatures of its per-blit post-FX functions (as oracle.render_postfx
    declares them)."""
    L = O.lib(); i, f, fp = C.c_int, C.c_float, O._f
    L.oracle_bloom_prefilter.argtypes = [fp, i, i, fp, i, i, f, f, f, f]
    L.oracle_box4.argtypes = [fp, i, i, fp, i, i, f, i]
    L.oracle_sunrays_mask.argtypes = [fp, fp, i, i]
    L.oracle_sunrays.argtypes = [fp, i, i, fp, i, i, f]
    L.oracle_blur3.argtypes = [fp, fp, i, i, f, f]
    for fn in (L.oracle_bloom_prefilter, L.oracle_box4, L.oracle_sunrays_mask, L.oracle_sunrays, L.oracle_blur3):
        fn.restype = None
    return L


def render_postfx(dye, w, h, dither, cfg=None, back_rgb=(0.0, 0.0, 0.0), background=O.BG_COLOR, aspect=None,
                  half_targets=False, half_mask=False):
    """oracle.render_postfx (SHADING + BLOOM + SUNRAYS) with the chains stored as above.  Without either
    keyword it is oracle.render_postfx itself; with them the frame is display_keywords_model's display
    shader over the rounded chains."""
    if not (half_targets or half_mask):
        return O.render_postfx(dye, w, h, dither, cfg=cfg, back_rgb=back_rgb, background=background, aspect=aspect)
    L, p = _chain_lib(), O._p
    rt = O.round_half if half_targets else (lambda a: a)
    rm = O.round_half if half_mask else (lambda a: a)
    c = dict(BLOOM_ITERATIONS=8, BLOOM_RESOLUTION=256, BLOOM_INTENSITY=0.8, BLOOM_THRESHOLD=0.6,
             BLOOM_SOFT_KNEE=0.7, SUNRAYS_RESOLUTION=196, SUNRAYS_WEIGHT=1.0)
    c.update(cfg or {})
    dye = np.ascontiguousarray(dye, F); Hd, Wd, _ = dye.shape
    dither = np.ascontiguousarray(dither, F)
    aspect = w / h if aspect is None else aspect

    def get_resolution(res):                                  # S:1612-1624
        ar = w / h
        if ar < 1: ar = 1.0 / ar
        mn, mx = int(np.floor(res + 0.5)), int(np.floor(res * ar + 0.5))
        return (mx, mn) if w > h else (mn, mx)

    bw, bh = get_resolution(c["BLOOM_RESOLUTION"])
    bloom = np.zeros((bh, bw, 4), F); bloom[..., 3] = 1.0        # createFBO's (0,0,0,1): exact in fp16
    sizes = []
    for k in range(c["BLOOM_ITERATIONS"]):
        pw, ph = bw >> (k + 1), bh >> (k + 1)
        if pw < 2 or ph < 2: break
        sizes.append((pw, ph))
    pyr = []
    if len(sizes) >= 2:
        knee = c["BLOOM_THRESHOLD"] * c["BLOOM_SOFT_KNEE"] + 0.0001
        L.oracle_bloom_prefilter(p(dye), Wd, Hd, p(bloom), bw, bh, c["BLOOM_THRESHOLD"] - knee, knee * 2,
                                 0.25 / knee, c["BLOOM_THRESHOLD"])
        bloom = rt(bloom)
        last, lw, lh = bloom, bw, bh
        for pw, ph in sizes:
            t = np.empty((ph, pw, 4), F)
            L.oracle_box4(p(last), lw, lh, p(t), pw, ph, 1.0, 0)
            t = rt(t); pyr.append(t); last, lw, lh = t, pw, ph
        for k in range(len(pyr) - 2, -1, -1):
            pw, ph = sizes[k]
            L.oracle_box4(p(last), lw, lh, p(pyr[k]), pw, ph, 1.0, 1)     # fragment + widened destination
            pyr[k] = rt(pyr[k]); last, lw, lh = pyr[k], pw, ph
        L.oracle_box4(p(last), lw, lh, p(bloom), bw, bh, c["BLOOM_INTENSITY"], 0)
        bloom = rt(bloom)
    sw, sh = get_resolution(c["SUNRAYS_RESOLUTION"])
    mask = np.empty_like(dye)
    L.oracle_sunrays_mask(p(dye), p(mask), Wd, Hd)
    mask = rm(mask)
    sun = np.empty((sh, sw), F)
    L.oracle_sunrays(p(mask), Wd, Hd, p(sun), sw, sh, c["SUNRAYS_WEIGHT"])
    sun = rt(sun); tmp = np.empty_like(sun)
    L.oracle_blur3(p(sun), p(tmp), sw, sh, 1.0 / sw, 0.0)
    tmp = rt(tmp)
    L.oracle_blur3(p(tmp), p(sun), sw, sh, 0.0, 1.0 / sh)
    sun = rt(sun)
    target = M._display(dye, w, h, SHADING | BLOOM | SUNRAYS, bloom, sun, dither, back_rgb, background, aspect)
    return dict(target=target, bloom=bloom, sunrays=sun, mask_alpha=mask[..., 3].copy(), pyramid=pyr)


def render_keywords(dye, w, h, dither, cfg=None, back_rgb=(0.0, 0.0, 0.0), background=O.BG_COLOR, aspect=None,
                    keywords=SHADING | BLOOM | SUNRAYS, half_targets=False, half_mask=False):
    """display_keywords_model.render_keywords over the chains of render_postfx."""
    dye = np.ascontiguousarray(dye, F)
    aspect = w / h if aspect is None else aspect
    if not keywords & (BLOOM | SUNRAYS) or not (half_targets or half_mask):
        return M.render_keywords(dye, w, h, dither, cfg=cfg, back_rgb=back_rgb, background=background, aspect=aspect,
                                 keywords=keywords)
    dith = np.ascontiguousarray(dither, F) if keywords & BLOOM else M._NO_DITHER
    r = render_postfx(dye, w, h, dith, cfg=cfg, back_rgb=back_rgb, background=background, aspect=aspect,
                      half_targets=half_targets, half_mask=half_mask)
    if keywords != SHADING | BLOOM | SUNRAYS:
        r["target"] = M._display(dye, w, h, keywords, r["bloom"], r["sunrays"], dith, back_rgb, background, aspect)
    if not keywords & BLOOM:
        r.update(bloom=None, pyramid=[])
    if not keywords & SUNRAYS:
        r.update(sunrays=None, mask_alpha=None)
    return r


def capture(dye, w, h, canvas_w, canvas_h, dither, keywords, transparent, back_rgb, cfg=None,
            half_targets=False, half_mask=False):
    """capture_model.capture over the chains of render_postfx at the canvas size."""
    dye = np.ascontiguousarray(dye, F)
    dith = np.ascontiguousarray(dither, F) if keywords & BLOOM else M._NO_DITHER
    bloom = sun = None
    if keywords & (BLOOM | SUNRAYS):
        r = render_postfx(dye, canvas_w, canvas_h, dith, cfg=cfg, half_targets=half_targets, half_mask=half_mask)
        bloom, sun = r["bloom"], r["sunrays"]
    pre = M._display(dye, w, h, keywords, bloom, sun, dith, CM.back16(back_rgb), O.BG_NONE if transparent else O.BG_COLOR,
                     w / h)
    return dict(pre=pre, rgba8=CM.to_bytes(pre)[::-1].copy())


def capture_interval(dye, w, h, canvas_w, canvas_h, dither, keywords, transparent, back_rgb, cfg=None,
                     half_targets=False, half_mask=False):
    """gamma_model.capture_interval over the chains of render_postfx at the canvas size: [B(lo), B(hi)] of
    every byte, top row first (keywords include BLOOM)."""
    r = render_postfx(np.ascontiguousarray(dye, F), canvas_w, canvas_h, np.ascontiguousarray(dither, F), cfg=cfg,
                      half_targets=half_targets, half_mask=half_mask)
    clo, chi = G.gamma_interval(dye, w, h, keywords, r["bloom"], r["sunrays"], dither)
    lo, hi = G.blend_interval(clo, chi, CM.back16(back_rgb), O.BG_NONE if transparent else O.BG_COLOR, w / h)
    return CM.to_bytes(lo)[::-1], CM.to_bytes(hi)[::-1]
