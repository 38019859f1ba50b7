"""CPU model of render(), captureScreenshot() and resizeFBO with FLUID_FLAG_NEAREST_FILTERING: the reference
on a device without float linear filtering (S:127-134), whose dye, velocity (S:990), bloom FBO and pyramid
(S:1017), sunrays and sunraysTemp (S:1039) are NEAREST + CLAMP_TO_EDGE textures.  Test infrastructure.

The six kernels that sample them -- resample (copyShader, resizeFBO S:1108-1114), bloom prefilter, box4
(bloom blur / final), sunrays mask, sunrays and blur3 -- and the display shader are restated in numpy in
the oracle's fp32 operation order, no contraction (the library is built with --fmad=false), with the NEAREST
fetch: texel clamp(floor(uv * n), 0, n - 1), NaN -> 0.  The dithering texture stays LINEAR + REPEAT.  The
background, alpha, linearToGamma, the powf interval and the capture bytes are those of
display_keywords_model.py, gamma_model.py and capture_model.py; half targets and a half mask are rounded
after each blit as half_postfx_model.py does.

vUv: under NEAREST one ulp of a coordinate can move a tap to the next texel, so the convention is an
argument.  LIBRARY is the kernels' (i + .5) / w, taps uv +- texelSize; RASTER is the rasteriser's as
glsl_exec.Program.blit and the vertex shaders compute it: x = (i + .5) / w * 2 - 1, vUv = x * .5 + .5, and
the vertex shader's taps from that vUv.  Both are exact at power-of-two sizes.
"""
import numpy as np

import capture_model as CM
import display_keywords_model as M
import gamma_model as G
from oracle import oracle as O

F = np.float32
SHADING, BLOOM, SUNRAYS = M.SHADING, M.BLOOM, M.SUNRAYS
LIBRARY, RASTER = "library", "raster"
SETS = {"none": 0, "shading": SHADING, "bloom": BLOOM, "shading_bloom": SHADING | BLOOM, "sunrays": SUNRAYS,
        "shading_sunrays": SHADING | SUNRAYS, "bloom_sunrays": BLOOM | SUNRAYS,
        "shading_bloom_sunrays": SHADING | BLOOM | SUNRAYS}
_ID = lambda a: a                                                                  # noqa: E731


def uv_grid(w, h, conv=LIBRARY):
    """vUv of every texel of a w x h target, (h, w) fp32 arrays, in convention `conv`."""
    if conv == LIBRARY:
        return M.uv_grid(w, h)
    with np.errstate(invalid="ignore"):
        x = (np.arange(w, dtype=F) + F(0.5)) / F(w) * F(2.0) - F(1.0)
        y = (np.arange(h, dtype=F) + F(0.5)) / F(h) * F(2.0) - F(1.0)
        ux, uy = x * F(0.5) + F(0.5), y * F(0.5) + F(0.5)
    return ux[None, :].repeat(h, 0), uy[:, None].repeat(w, 1)


def texel(tex, uvx, uvy):
    """The NEAREST + CLAMP_TO_EDGE texel indices (j, i) of a (H, W, ...) texture at (uvx, uvy)."""
    H, W = tex.shape[:2]
    with np.errstate(invalid="ignore", over="ignore"):
        return M._texel(np.floor(uvy * F(H)), H), M._texel(np.floor(uvx * F(W)), W)


def fetch(tex, uvx, uvy):
    """The NEAREST fetch (nearest_fetch of the library)."""
    j, i = texel(tex, uvx, uvy)
    return tex[j, i]


# ---- the chain kernels (postfx.cuh) ---------------------------------------------------------------------
def prefilter(dye, bw, bh, threshold, soft_knee, conv=LIBRARY):
    """bloomPrefilterShader S:614-631 into a bw x bh target."""
    knee = threshold * soft_knee + 0.0001
    c0, c1, c2, th = F(threshold - knee), F(knee * 2), F(0.25 / knee), F(threshold)
    c = fetch(dye, *uv_grid(bw, bh, conv))
    br = np.fmax(c[..., 0], np.fmax(c[..., 1], c[..., 2]))
    rq = np.fmin(np.fmax(br - c0, F(0)), c1)
    rq = (c2 * rq) * rq
    f = (np.fmax(rq, br - th) / np.fmax(br, F(0.0001)))[..., None]
    out = np.concatenate([c[..., :3] * f, np.zeros_like(f)], axis=-1)
    return out.astype(F)


def box4(src, w, h, scale=1.0, dst=None, conv=LIBRARY):
    """bloomBlurShader / bloomFinalShader S:633-674 into a w x h target; dst: the additive up-pass's
    destination (blendFunc(ONE, ONE))."""
    hs, ws = src.shape[:2]
    tsx, tsy = F(1.0 / ws), F(1.0 / hs)
    uvx, uvy = uv_grid(w, h, conv)
    L, R = fetch(src, uvx - tsx, uvy), fetch(src, uvx + tsx, uvy)
    T, B = fetch(src, uvx, uvy + tsy), fetch(src, uvx, uvy - tsy)
    s = ((((F(0) + L) + R) + T) + B) * F(0.25) * F(scale)
    return (s + dst if dst is not None else s).astype(F)


def sunrays_mask(dye, conv=LIBRARY):
    """sunraysMaskShader S:676-691 (drawn into dye.write: the dye's size)."""
    Hd, Wd = dye.shape[:2]
    c = fetch(dye, *uv_grid(Wd, Hd, conv)).copy()
    br = np.fmax(c[..., 0], np.fmax(c[..., 1], c[..., 2]))
    c[..., 3] = F(1) - np.fmin(np.fmax(br * F(20), F(0)), F(0.8))
    return c


def sunrays(mask, w, h, weight, conv=LIBRARY):
    """sunraysShader S:693-724 into a w x h one-channel target."""
    f = F(1.0 / 16.0) * F(0.3)
    uvx, uvy = uv_grid(w, h, conv)
    cx, cy = uvx, uvy
    dx, dy = (uvx - F(0.5)) * f, (uvy - F(0.5)) * f
    illum = F(1)
    color = fetch(mask, uvx, uvy)[..., 3]
    for _ in range(16):
        cx = cx - dx; cy = cy - dy
        color = color + (fetch(mask, cx, cy)[..., 3] * illum) * F(weight)
        illum = illum * F(0.95)
    return (color * F(0.7)).astype(F)


def blur3(src, tsx, tsy, conv=LIBRARY):
    """blurShader + blurVertexShader S:461-494 on a one-channel texture."""
    h, w = src.shape
    t = src[..., None]
    off = F(1.33333333)
    uvx, uvy = uv_grid(w, h, conv)
    tsx, tsy = F(tsx), F(tsy)
    c = fetch(t, uvx, uvy)[..., 0]
    l = fetch(t, uvx - tsx * off, uvy - tsy * off)[..., 0]
    r = fetch(t, uvx + tsx * off, uvy + tsy * off)[..., 0]
    s = c * F(0.29411764)
    s = s + l * F(0.35294117)
    return (s + r * F(0.35294117)).astype(F)


def get_resolution(res, w, h):
    """getResolution (S:1612-1624) on a w x h drawing buffer."""
    ar = w / h
    if ar < 1: ar = 1.0 / ar
    mn, mx = int(np.floor(res + 0.5)), int(np.floor(res * ar + 0.5))
    return (mx, mn) if w > h else (mn, mx)


def chains(dye, w, h, keywords, cfg=None, half_targets=False, half_mask=False, conv=LIBRARY):
    """applyBloom with BLOOM and applySunrays + blur with SUNRAYS (S:1350-1419) on a w x h drawing buffer:
    dict(bloom, pyramid, sunrays, mask_alpha), None / [] for a chain that is off."""
    c = dict(BLOOM_ITERATIONS=8, BLOOM_RESOLUTION=256, BLOOM_INTENSITY=0.8, BLOOM_THRESHOLD=0.6,
             BLOOM_SOFT_KNEE=0.7, SUNRAYS_RESOLUTION=196, SUNRAYS_WEIGHT=1.0)
    c.update(cfg or {})
    rt = CM.half_round if half_targets else _ID
    rt32 = (lambda a: rt(a).astype(F))                                             # noqa: E731
    rm = (lambda a: CM.half_round(a).astype(F)) if half_mask else _ID              # noqa: E731
    dye = np.ascontiguousarray(dye, F)
    r = dict(bloom=None, pyramid=[], sunrays=None, mask_alpha=None)
    if keywords & BLOOM:
        bw, bh = get_resolution(c["BLOOM_RESOLUTION"], w, h)
        bloom = np.zeros((bh, bw, 4), F); bloom[..., 3] = 1
        sizes = []
        for k in range(c["BLOOM_ITERATIONS"]):
            pw, ph = bw >> (k + 1), bh >> (k + 1)
            if pw < 2 or ph < 2: break
            sizes.append((pw, ph))
        pyr = []
        if len(sizes) >= 2:
            with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
                bloom = rt32(prefilter(dye, bw, bh, c["BLOOM_THRESHOLD"], c["BLOOM_SOFT_KNEE"], conv))
                last = bloom
                for pw, ph in sizes:
                    last = rt32(box4(last, pw, ph, conv=conv)); pyr.append(last)
                for k in range(len(pyr) - 2, -1, -1):
                    pyr[k] = rt32(box4(last, *sizes[k], dst=pyr[k], conv=conv)); last = pyr[k]
                bloom = rt32(box4(last, bw, bh, c["BLOOM_INTENSITY"], conv=conv))
        r.update(bloom=bloom, pyramid=pyr)
    if keywords & SUNRAYS:
        sw, sh = get_resolution(c["SUNRAYS_RESOLUTION"], w, h)
        with np.errstate(invalid="ignore", over="ignore"):
            mask = rm(sunrays_mask(dye, conv))
            sun = rt32(sunrays(mask, sw, sh, c["SUNRAYS_WEIGHT"], conv))
            tmp = rt32(blur3(sun, 1.0 / sw, 0.0, conv))
            sun = rt32(blur3(tmp, 0.0, 1.0 / sh, conv))
        r.update(sunrays=sun, mask_alpha=mask[..., 3].copy())
    return r


# ---- the display shader (displayShaderSource S:549-612) ----------------------------------------------------
def colour_terms(dye, w, h, keywords, bloom, sun, conv=LIBRARY):
    """display_keywords_model.colour_terms with NEAREST fetches of dye, bloom and sunrays."""
    tsx, tsy = F(1.0 / w), F(1.0 / h)
    uvx, uvy = uv_grid(w, h, conv)
    with np.errstate(invalid="ignore", over="ignore"):
        c = fetch(dye, uvx, uvy)[..., :3]
        if keywords & SHADING:
            dx = M._len3(fetch(dye, uvx + tsx, uvy)) - M._len3(fetch(dye, uvx - tsx, uvy))
            dy = M._len3(fetch(dye, uvx, uvy + tsy)) - M._len3(fetch(dye, uvx, uvy - tsy))
            nz = np.sqrt(tsx * tsx + tsy * tsy)
            nl = np.sqrt((dx * dx + dy * dy) + nz * nz)
            d = ((dx / nl) * F(0) + (dy / nl) * F(0)) + (nz / nl) * F(1)
            c = c * np.fmin(np.fmax(d + F(0.7), F(0.7)), F(1))[..., None]
        bl = fetch(bloom, uvx, uvy)[..., :3] if keywords & BLOOM else None
        if keywords & SUNRAYS:
            s = fetch(sun[..., None], uvx, uvy)
            c = c * s
            if keywords & BLOOM:
                bl = bl * s
    return c, bl


def _gamma_argument(bl, dither, w, h, conv):
    """display_keywords_model.gamma_argument at the convention's vUv: the dithering stays LINEAR + REPEAT."""
    dsx, dsy = M.dither_scale(w, h, dither)
    uvx, uvy = uv_grid(w, h, conv)
    with np.errstate(invalid="ignore", over="ignore"):
        noise = M._fetch(dither, uvx * dsx, uvy * dsy, repeat=True)[..., :1] * F(2) - F(1)
        return np.fmax(bl + noise / F(255), F(0))


def _background(w, h, back_rgb, background, aspect, conv):
    if background == O.BG_CHECKERBOARD:
        uvx, uvy = uv_grid(w, h, conv)
        x = np.floor((uvx * F(25)) * F(aspect)); y = np.floor((uvy * F(25)) * F(1))
        sxy = x + y
        v = (sxy - F(2) * np.floor(sxy / F(2))) * F(0.1) + F(0.8)
        return np.stack([v, v, v], axis=-1)
    return np.broadcast_to(np.asarray(back_rgb, F), (h, w, 3))


def _over(c, a, back_rgb, background, aspect, conv):
    if background == O.BG_NONE:
        return np.concatenate([c, a], axis=-1).astype(F)
    h, w = c.shape[:2]
    with np.errstate(invalid="ignore", over="ignore"):
        k = F(1) - a
        return np.concatenate([c + _background(w, h, back_rgb, background, aspect, conv) * k, a + F(1) * k], axis=-1).astype(F)


def _interval(c, bl, dither, w, h, back_rgb, background, aspect, conv):
    bk = _gamma_argument(bl, dither, w, h, conv)
    plo, phi = G.powf_bounds(bk)
    with np.errstate(invalid="ignore", over="ignore"):
        clo, chi = c + M.linear_to_gamma(plo), c + M.linear_to_gamma(phi)
    if background == O.BG_CHECKERBOARD and conv != LIBRARY:
        bg = _background(w, h, back_rgb, background, aspect, conv)
        alo, ahi = M.alpha_of(clo), M.alpha_of(chi)
        one = F(1)
        with np.errstate(invalid="ignore", over="ignore"):
            return (np.concatenate([clo + bg * (one - ahi), alo + one * (one - ahi)], axis=-1),
                    np.concatenate([chi + bg * (one - alo), ahi + one * (one - alo)], axis=-1))
    return G.blend_interval(clo, chi, back_rgb, background, aspect)


def display(dye, w, h, keywords, bloom, sun, dither, back_rgb, background, aspect, conv=LIBRARY):
    """The frame of render() over `background` (oracle BG_* modes): dict(target) without BLOOM (exact),
    dict(lo, hi) with BLOOM (the powf interval of gamma_model, texel by texel)."""
    dye = np.ascontiguousarray(dye, F)
    c, bl = colour_terms(dye, w, h, keywords, bloom, sun, conv)
    if keywords & BLOOM:
        lo, hi = _interval(c, bl, np.ascontiguousarray(dither, F), w, h, back_rgb, background, aspect, conv)
        return dict(lo=lo, hi=hi)
    return dict(target=_over(c, M.alpha_of(c), back_rgb, background, aspect, conv))


def render(dye, w, h, dither, keywords, cfg=None, back_rgb=(0.0, 0.0, 0.0), background=O.BG_COLOR, aspect=None,
           half_targets=False, half_mask=False, conv=LIBRARY):
    """render(null) on a w x h canvas: the chains of `keywords`, then display()."""
    aspect = w / h if aspect is None else aspect
    r = chains(dye, w, h, keywords, cfg, half_targets, half_mask, conv)
    r.update(display(dye, w, h, keywords, r["bloom"], r["sunrays"], dither, back_rgb, background, aspect, conv))
    return r


def capture(dye, w, h, canvas_w, canvas_h, dither, keywords, transparent, back_rgb, cfg=None,
            half_targets=False, half_mask=False, conv=LIBRARY):
    """captureScreenshot into a w x h target on a canvas_w x canvas_h canvas, top row first: dict(rgba8) exact
    without BLOOM, dict(lo, hi) byte bracket with BLOOM (gamma_model.capture_interval's rule)."""
    r = chains(dye, canvas_w, canvas_h, keywords, cfg, half_targets, half_mask, conv)
    d = display(dye, w, h, keywords, r["bloom"], r["sunrays"], dither, CM.back16(back_rgb),
                O.BG_NONE if transparent else O.BG_COLOR, w / h, conv)
    if "target" in d:
        return dict(rgba8=CM.to_bytes(d["target"])[::-1].copy())
    return dict(lo=CM.to_bytes(d["lo"])[::-1].copy(), hi=CM.to_bytes(d["hi"])[::-1].copy())


def resize(src, Wn, Hn, half=False, conv=LIBRARY):
    """resizeFBO's copy (S:1108-1114) of an (H, W, C) field through its NEAREST sampler into Wn x Hn, stored
    in fp16 when `half`."""
    out = fetch(np.ascontiguousarray(src, F), *uv_grid(Wn, Hn, conv))
    return CM.half_round(out).astype(F) if half else out.astype(F)
