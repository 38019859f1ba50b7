"""CPU model of render(null), captureScreenshot() and resizeFBO for every display keyword set (updateKeywords,
S:1160-1166), both samplers and both target storages.  Test infrastructure.

Two switches select what the model draws:

* the sampler.  LINEAR runs each post-FX blit through the oracle's per-blit C functions (oracle/fluid_oracle.c,
  the ones oracle.render_postfx calls), which are pinned to the executed shaders.  NEAREST (a device without
  float linear filtering, S:127-134: dye, velocity S:990, bloom S:1017 and sunrays S:1039 textures are NEAREST
  + CLAMP_TO_EDGE) restates those kernels here in numpy, in the library's fp32 operation order without
  contraction (it is built with --fmad=false), with the fetch texel clamp(floor(uv * n), 0, n - 1), NaN -> 0.
* the storage.  half_targets: the bloom FBO, each pyramid level, sunrays and sunraysTemp are RGBA16F / R16F
  (initBloomFramebuffers / initSunraysFramebuffers S:1012-1043): every blit's fp32 result is rounded to fp16
  when stored; the additive up-pass (blendFunc(ONE, ONE), S:1374-1375) adds the widened destination in fp32
  and rounds once.  half_mask: the sunrays mask is drawn into dye.write (S:1300), fp16 on a half-storage handle.

displayShaderSource (S:549-612) is restated in numpy for either sampler -- the dithering texture stays LINEAR +
REPEAT -- with C's fmaxf / fminf (np.fmax / np.fmin drop a NaN argument).  Without BLOOM the frame is exact.
With it, linearToGamma's powf is not reproducible, so the frame also comes as the interval [lo, hi] of
gamma_model.powf_bounds carried through the later, monotone steps (gamma_model.py explains why that holds).

vUv: under NEAREST one ulp of a coordinate can move a tap to the next texel, so the convention is an argument.
LIBRARY is the kernels' (i + .5) / w, taps uv +- texelSize; RASTER is the rasteriser's as glsl_exec.Program.blit
and the vertex shaders compute it: x = (i + .5) / w * 2 - 1, vUv = x * .5 + .5, and the vertex shader's taps from
that vUv.  Both are exact at power-of-two sizes.  The LINEAR C functions use LIBRARY.
"""
import numpy as np

import capture_model as CM
import gamma_model as G
from oracle import oracle as O

F = np.float32
SHADING, BLOOM, SUNRAYS = 1, 2, 4       # FLUID_DISPLAY_* of include/fluid.h
ALL3 = SHADING | BLOOM | SUNRAYS
SETS = {"none": 0, "shading": SHADING, "bloom": BLOOM, "shading_bloom": SHADING | BLOOM, "sunrays": SUNRAYS,
        "shading_sunrays": SHADING | SUNRAYS, "bloom_sunrays": BLOOM | SUNRAYS, "shading_bloom_sunrays": ALL3}
LIBRARY, RASTER = "library", "raster"
# the reference's desktop post-FX config (S:70-84)
FX_DEFAULTS = dict(BLOOM_ITERATIONS=8, BLOOM_RESOLUTION=256, BLOOM_INTENSITY=0.8, BLOOM_THRESHOLD=0.6,
                   BLOOM_SOFT_KNEE=0.7, SUNRAYS_RESOLUTION=196, SUNRAYS_WEIGHT=1.0)


def get_resolution(res, w, h):
    """getResolution (S:1612-1624) on a w x h drawing buffer: (width, height)."""
    ar = w / h
    if ar < 1:
        ar = 1.0 / ar
    mn, mx = int(np.floor(res + 0.5)), int(np.floor(res * ar + 0.5))
    return (mx, mn) if w > h else (mn, mx)


def uv_grid(w, h, conv=LIBRARY):
    """vUv of every texel of a w x h target, (h, w) fp32 arrays, in convention `conv`."""
    with np.errstate(invalid="ignore"):
        x = (np.arange(w, dtype=F) + F(0.5)) / F(w)
        y = (np.arange(h, dtype=F) + F(0.5)) / F(h)
        if conv == RASTER:
            x = (x * F(2.0) - F(1.0)) * F(0.5) + F(0.5)
            y = (y * F(2.0) - F(1.0)) * F(0.5) + F(0.5)
    return x[None, :].repeat(h, 0), y[:, None].repeat(w, 1)


# ---- the samplers --------------------------------------------------------------------------------------------
def _clamp_index(f, n):
    """CLAMP_TO_EDGE index of a floored coordinate (texel_index of the oracle): NaN -> 0."""
    return np.where(~(f > 0), 0, np.where(f >= F(n - 1), n - 1, np.maximum(f, 0))).astype(np.int64)


def linear_fetch(tex, uvx, uvy, repeat=False):
    """GL-spec LINEAR fetch of an (H, W, C) texture at (uvx, uvy) fp32 arrays (linear_fetch / linear_fetch_w of
    the oracle): weights (1-a)(1-b) .. ab, summed left to right; CLAMP_TO_EDGE, or REPEAT."""
    H, W = tex.shape[:2]
    u = uvx * F(W) - F(0.5); v = uvy * F(H) - F(0.5)
    fi = np.floor(u); fj = np.floor(v)
    a = (u - fi)[..., None]; b = (v - fj)[..., None]
    if repeat:
        i0 = np.mod(fi.astype(np.int64), W); j0 = np.mod(fj.astype(np.int64), H)
        i1 = (i0 + 1) % W; j1 = (j0 + 1) % H
    else:
        i0, i1 = _clamp_index(fi, W), _clamp_index(fi + F(1), W)
        j0, j1 = _clamp_index(fj, H), _clamp_index(fj + F(1), H)
    one = F(1)
    w00 = (one - a) * (one - b); w10 = a * (one - b); w01 = (one - a) * b; w11 = a * b
    return ((w00 * tex[j0, i0] + w10 * tex[j0, i1]) + w01 * tex[j1, i0]) + w11 * tex[j1, i1]


def texel(tex, uvx, uvy):
    """The NEAREST + CLAMP_TO_EDGE texel indices (j, i) of a (H, W, ...) texture at (uvx, uvy)."""
    H, W = tex.shape[:2]
    with np.errstate(invalid="ignore", over="ignore"):
        return _clamp_index(np.floor(uvy * F(H)), H), _clamp_index(np.floor(uvx * F(W)), W)


def nearest_fetch(tex, uvx, uvy):
    """The NEAREST fetch (nearest_fetch of the library)."""
    j, i = texel(tex, uvx, uvy)
    return tex[j, i]


def fetch(tex, uvx, uvy, nearest=False):
    return nearest_fetch(tex, uvx, uvy) if nearest else linear_fetch(tex, uvx, uvy)


# ---- the chain kernels (postfx.cuh) ------------------------------------------------------------------------
def curve(threshold, soft_knee, fp32=False):
    """(curve.x, curve.y, curve.z, threshold) as the prefilter receives them: applyBloom derives them in JS
    doubles (S:1358-1363) and gl.uniform narrows each once; `fp32` derives them in fp32 instead."""
    if fp32:
        t, k = F(threshold), F(soft_knee)
        knee = t * k + F(0.0001)
        return t - knee, knee * F(2), F(0.25) / knee, t
    knee = threshold * soft_knee + 0.0001
    return F(threshold - knee), F(knee * 2), F(0.25 / knee), F(threshold)


class Linear:
    """The LINEAR blits: the oracle's per-blit C functions."""

    @staticmethod
    def prefilter(dye, bw, bh, crv):
        out = np.empty((bh, bw, 4), F)
        O.lib().oracle_bloom_prefilter(O._p(dye), dye.shape[1], dye.shape[0], O._p(out), bw, bh, *(float(c) for c in crv))
        return out

    @staticmethod
    def box4(src, w, h, scale=1.0, dst=None):
        out = np.empty((h, w, 4), F) if dst is None else np.array(dst, F)
        O.lib().oracle_box4(O._p(src), src.shape[1], src.shape[0], O._p(out), w, h, scale, int(dst is not None))
        return out

    @staticmethod
    def sunrays_mask(dye):
        out = np.empty_like(dye)
        O.lib().oracle_sunrays_mask(O._p(dye), O._p(out), dye.shape[1], dye.shape[0])
        return out

    @staticmethod
    def sunrays(mask, w, h, weight):
        out = np.empty((h, w), F)
        O.lib().oracle_sunrays(O._p(mask), mask.shape[1], mask.shape[0], O._p(out), w, h, weight)
        return out

    @staticmethod
    def blur3(src, tsx, tsy):
        out = np.empty_like(src)
        O.lib().oracle_blur3(O._p(src), O._p(out), src.shape[1], src.shape[0], tsx, tsy)
        return out


class Nearest:
    """The NEAREST blits in numpy, at the vUv of convention `conv`."""

    def __init__(self, conv=LIBRARY):
        self.conv = conv

    def prefilter(self, dye, bw, bh, crv):
        """bloomPrefilterShader S:614-631 into a bw x bh target."""
        c0, c1, c2, th = (F(c) for c in crv)
        c = nearest_fetch(dye, *uv_grid(bw, bh, self.conv))
        br = np.fmax(c[..., 0], np.fmax(c[..., 1], c[..., 2]))
        rq = np.fmin(np.fmax(br - c0, F(0)), c1)
        rq = (c2 * rq) * rq
        f = (np.fmax(rq, br - th) / np.fmax(br, F(0.0001)))[..., None]
        return np.concatenate([c[..., :3] * f, np.zeros_like(f)], axis=-1).astype(F)

    def box4(self, src, w, h, scale=1.0, dst=None):
        """bloomBlurShader / bloomFinalShader S:633-674 into a w x h target; dst: the additive up-pass's
        destination (blendFunc(ONE, ONE))."""
        tsx, tsy = F(1.0 / src.shape[1]), F(1.0 / src.shape[0])
        uvx, uvy = uv_grid(w, h, self.conv)
        L, R = nearest_fetch(src, uvx - tsx, uvy), nearest_fetch(src, uvx + tsx, uvy)
        T, B = nearest_fetch(src, uvx, uvy + tsy), nearest_fetch(src, uvx, uvy - tsy)
        s = ((((F(0) + L) + R) + T) + B) * F(0.25) * F(scale)
        return (s + dst if dst is not None else s).astype(F)

    def sunrays_mask(self, dye):
        """sunraysMaskShader S:676-691 (drawn into dye.write: the dye's size)."""
        c = nearest_fetch(dye, *uv_grid(dye.shape[1], dye.shape[0], self.conv)).copy()
        br = np.fmax(c[..., 0], np.fmax(c[..., 1], c[..., 2]))
        c[..., 3] = F(1) - np.fmin(np.fmax(br * F(20), F(0)), F(0.8))
        return c

    def sunrays(self, mask, w, h, weight):
        """sunraysShader S:693-724 into a w x h one-channel target."""
        f = F(1.0 / 16.0) * F(0.3)
        cx, cy = uvx, uvy = uv_grid(w, h, self.conv)
        dx, dy = (uvx - F(0.5)) * f, (uvy - F(0.5)) * f
        illum = F(1)
        color = nearest_fetch(mask, uvx, uvy)[..., 3]
        for _ in range(16):
            cx = cx - dx; cy = cy - dy
            color = color + (nearest_fetch(mask, cx, cy)[..., 3] * illum) * F(weight)
            illum = illum * F(0.95)
        return (color * F(0.7)).astype(F)

    def blur3(self, src, tsx, tsy):
        """blurShader + blurVertexShader S:461-494 on a one-channel texture."""
        t = src[..., None]
        off = F(1.33333333)
        uvx, uvy = uv_grid(src.shape[1], src.shape[0], self.conv)
        tsx, tsy = F(tsx), F(tsy)
        c = nearest_fetch(t, uvx, uvy)[..., 0]
        l = nearest_fetch(t, uvx - tsx * off, uvy - tsy * off)[..., 0]
        r = nearest_fetch(t, uvx + tsx * off, uvy + tsy * off)[..., 0]
        s = c * F(0.29411764)
        s = s + l * F(0.35294117)
        return (s + r * F(0.35294117)).astype(F)


def _stored(half):
    return O.round_half if half else (lambda a: a)


def chains(dye, w, h, keywords=BLOOM | SUNRAYS, cfg=None, *, nearest=False, half_targets=False, half_mask=False,
           conv=LIBRARY, fp32_curve=False, intensity_on_up_pass=False):
    """applyBloom with BLOOM and applySunrays + blur with SUNRAYS (S:1350-1419) on a w x h drawing buffer:
    dict(bloom, pyramid, sunrays, mask_alpha), None / [] for a chain that is off.  fp32_curve and
    intensity_on_up_pass are wrong rules, for the tests to show that their inputs tell them from the right ones:
    the prefilter's curve derived in fp32, BLOOM_INTENSITY applied on the up-pass instead of the final blit."""
    c = dict(FX_DEFAULTS, **(cfg or {}))
    k = Nearest(conv) if nearest else Linear
    st, sm = _stored(half_targets), _stored(half_mask)
    dye = np.ascontiguousarray(dye, F)
    r = dict(bloom=None, pyramid=[], sunrays=None, mask_alpha=None)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if keywords & BLOOM:
            bw, bh = get_resolution(c["BLOOM_RESOLUTION"], w, h)
            bloom = np.zeros((bh, bw, 4), F); bloom[..., 3] = 1           # createFBO's (0, 0, 0, 1): exact in fp16
            sizes = [(bw >> (i + 1), bh >> (i + 1)) for i in range(c["BLOOM_ITERATIONS"])]
            sizes = sizes[:next((i for i, (pw, ph) in enumerate(sizes) if pw < 2 or ph < 2), len(sizes))]
            pyr = []
            if len(sizes) >= 2:
                up, final = (c["BLOOM_INTENSITY"], 1.0) if intensity_on_up_pass else (1.0, c["BLOOM_INTENSITY"])
                bloom = last = st(k.prefilter(dye, bw, bh, curve(c["BLOOM_THRESHOLD"], c["BLOOM_SOFT_KNEE"], fp32_curve)))
                for pw, ph in sizes:
                    last = st(k.box4(last, pw, ph)); pyr.append(last)
                for i in range(len(pyr) - 2, -1, -1):
                    pyr[i] = last = st(k.box4(last, *sizes[i], up, dst=pyr[i]))
                bloom = st(k.box4(last, bw, bh, final))
            r.update(bloom=bloom, pyramid=pyr)
        if keywords & SUNRAYS:
            sw, sh = get_resolution(c["SUNRAYS_RESOLUTION"], w, h)
            mask = sm(k.sunrays_mask(dye))
            sun = st(k.sunrays(mask, sw, sh, c["SUNRAYS_WEIGHT"]))
            sun = st(k.blur3(st(k.blur3(sun, 1.0 / sw, 0.0)), 0.0, 1.0 / sh))
            r.update(sunrays=sun, mask_alpha=mask[..., 3].copy())
    return r


# ---- the display shader (displayShaderSource S:549-612) and the background ------------------------------------
def _len3(c):
    return np.sqrt((c[..., 0] * c[..., 0] + c[..., 1] * c[..., 1]) + c[..., 2] * c[..., 2])


def colour_terms(dye, w, h, keywords, bloom, sun, nearest=False, conv=LIBRARY):
    """displayShaderSource up to the dithering: the dye colour c (SHADING's diffuse, the sunrays multiply) and,
    with BLOOM, the bloom colour bl (sunrays multiply), else None."""
    tsx, tsy = F(1.0 / w), F(1.0 / h)
    uvx, uvy = uv_grid(w, h, conv)
    dye = np.ascontiguousarray(dye, F)
    with np.errstate(invalid="ignore", over="ignore"):
        c = fetch(dye, uvx, uvy, nearest)[..., :3]
        if keywords & SHADING:
            dx = _len3(fetch(dye, uvx + tsx, uvy, nearest)) - _len3(fetch(dye, uvx - tsx, uvy, nearest))
            dy = _len3(fetch(dye, uvx, uvy + tsy, nearest)) - _len3(fetch(dye, uvx, uvy - tsy, nearest))
            nz = np.sqrt(tsx * tsx + tsy * tsy)
            nl = np.sqrt((dx * dx + dy * dy) + nz * nz)
            d = ((dx / nl) * F(0) + (dy / nl) * F(0)) + (nz / nl) * F(1)
            c = c * np.fmin(np.fmax(d + F(0.7), F(0.7)), F(1))[..., None]
        bl = fetch(bloom, uvx, uvy, nearest)[..., :3] if keywords & BLOOM else None
        if keywords & SUNRAYS:
            s = fetch(sun[..., None], uvx, uvy, nearest)
            c = c * s
            if keywords & BLOOM:
                bl = bl * s
    return c, bl


def dither_scale(w, h, dither):
    """getTextureScale (S:1626-1631) of the dithering texture on a w x h target: JS doubles, narrowed once."""
    return F(w / dither.shape[1]), F(h / dither.shape[0])


def gamma_argument(bl, dither, w, h, scale=None, conv=LIBRARY, repeat=True):
    """The argument of linearToGamma's pow: fmaxf(bl + noise / 255, 0), noise = the REPEAT LINEAR fetch of the
    dithering texture at vUv * getTextureScale, * 2 - 1.  `scale` defaults to the w x h target's."""
    dsx, dsy = scale if scale is not None else dither_scale(w, h, dither)
    uvx, uvy = uv_grid(w, h, conv)
    with np.errstate(invalid="ignore", over="ignore"):
        noise = linear_fetch(np.ascontiguousarray(dither, F), uvx * dsx, uvy * dsy, repeat)[..., :1] * F(2) - F(1)
        return np.fmax(bl + noise / F(255), F(0))


def linear_to_gamma(p):
    """linearToGamma (S:565-568) after its pow: fmaxf(1.055 * p - 0.055, 0), p = pow(bk, 0.416666667)."""
    return np.fmax(F(1.055) * p - F(0.055), F(0))


def alpha_of(c):
    """The display's alpha: fmaxf(c.r, fmaxf(c.g, c.b))."""
    return np.fmax(c[..., 0], np.fmax(c[..., 1], c[..., 2]))[..., None]


def checkerboard(w, h, aspect, conv=LIBRARY):
    """checkerboardShader (S:531-547) as the display kernel computes it: (h, w) fp32, row 0 = bottom."""
    uvx, uvy = uv_grid(w, h, conv)
    x = np.floor((uvx * F(25)) * F(aspect)); y = np.floor((uvy * F(25)) * F(1))
    sxy = x + y
    return (sxy - F(2) * np.floor(sxy / F(2))) * F(0.1) + F(0.8)


def background_colour(w, h, back_rgb, background, aspect, conv=LIBRARY):
    """What the display is blended over, (h, w, 3): BACK_COLOR, or the checkerboard (oracle BG_* modes)."""
    if background == O.BG_CHECKERBOARD:
        return np.repeat(checkerboard(w, h, aspect, conv)[..., None], 3, axis=-1)
    return np.broadcast_to(np.asarray(back_rgb, F), (h, w, 3))


def over_background(c, a, back_rgb, background, aspect, conv=LIBRARY):
    """render()'s blend ONE / ONE_MINUS_SRC_ALPHA of (c, a) over the background, or (c, a) bare (BG_NONE)."""
    if background == O.BG_NONE:
        return np.concatenate([c, a], axis=-1).astype(F)
    h, w = c.shape[:2]
    with np.errstate(invalid="ignore", over="ignore"):
        k = F(1) - a
        return np.concatenate([c + background_colour(w, h, back_rgb, background, aspect, conv) * k, a + F(1) * k],
                              axis=-1).astype(F)


def blend_interval(clo, chi, back_rgb, background, aspect, conv=LIBRARY):
    """[lo, hi] (h, w, 4) of the frame from the colour interval: alpha and the blend, each end taking the other
    end of alpha (bg >= 0), or bare (BG_NONE)."""
    alo, ahi = alpha_of(clo), alpha_of(chi)
    if background == O.BG_NONE:
        return np.concatenate([clo, alo], axis=-1), np.concatenate([chi, ahi], axis=-1)
    h, w = clo.shape[:2]
    bg = background_colour(w, h, back_rgb, background, aspect, conv)
    one = F(1)
    with np.errstate(invalid="ignore", over="ignore"):
        return (np.concatenate([clo + bg * (one - ahi), alo + one * (one - ahi)], axis=-1),
                np.concatenate([chi + bg * (one - alo), ahi + one * (one - alo)], axis=-1))


def display(dye, w, h, keywords, bloom, sun, dither, back_rgb, background, aspect, *, nearest=False, conv=LIBRARY,
            scale=None):
    """The frame of render() over `background`: dict(target), exact without BLOOM; with BLOOM target takes numpy's
    pow, and lo / hi bound every value for any powf within gamma_model.POWF_ULP.  scale: see gamma_argument."""
    c, bl = colour_terms(dye, w, h, keywords, bloom, sun, nearest, conv)
    if not keywords & BLOOM:
        return dict(target=over_background(c, alpha_of(c), back_rgb, background, aspect, conv))
    bk = gamma_argument(bl, dither, w, h, scale, conv)
    plo, phi = G.powf_bounds(bk)
    with np.errstate(invalid="ignore", over="ignore"):
        out = c + linear_to_gamma(np.power(bk, G.Y))
        lo, hi = blend_interval(c + linear_to_gamma(plo), c + linear_to_gamma(phi), back_rgb, background, aspect, conv)
    return dict(target=over_background(out, alpha_of(out), back_rgb, background, aspect, conv), lo=lo, hi=hi)


def render(dye, w, h, dither, keywords, cfg=None, back_rgb=(0.0, 0.0, 0.0), background=O.BG_COLOR, aspect=None, *,
           nearest=False, half_targets=False, half_mask=False, conv=LIBRARY):
    """render(null) on a w x h canvas: the chains of `keywords`, then display(): dict(bloom, pyramid, sunrays,
    mask_alpha, target[, lo, hi]).  dither is read only with BLOOM."""
    aspect = w / h if aspect is None else aspect
    r = chains(dye, w, h, keywords, cfg, nearest=nearest, half_targets=half_targets, half_mask=half_mask, conv=conv)
    r.update(display(dye, w, h, keywords, r["bloom"], r["sunrays"], dither, back_rgb, background, aspect,
                     nearest=nearest, conv=conv))
    return r


def capture(dye, w, h, canvas_w, canvas_h, dither, keywords, transparent, back_rgb, cfg=None, *, nearest=False,
            half_targets=False, half_mask=False, conv=LIBRARY, fx_size=None, scale=None):
    """captureScreenshot() (S:287-327) into a w x h target on a canvas_w x canvas_h canvas: the chains at the
    canvas size (the post-FX FBOs are sized from the drawing buffer, S:1012-1043), the display at the target
    size over the fp16 store of BACK_COLOR, or bare with TRANSPARENT.  dict(pre = the fp32 value before the fp16
    store, row 0 = bottom; rgba8 = its bytes, top row first) and, with BLOOM, lo / hi: the byte bracket [B(lo),
    B(hi)], top row first.  fx_size (the post-FX FBOs sized from it instead of the canvas) and scale (see
    gamma_argument) are wrong rules, for negative controls."""
    r = chains(dye, *(fx_size or (canvas_w, canvas_h)), keywords, cfg, nearest=nearest, half_targets=half_targets,
               half_mask=half_mask, conv=conv)
    d = display(dye, w, h, keywords, r["bloom"], r["sunrays"], dither, CM.back16(back_rgb),
                O.BG_NONE if transparent else O.BG_COLOR, w / h, nearest=nearest, conv=conv, scale=scale)
    out = dict(pre=d["target"], rgba8=CM.to_bytes(d["target"])[::-1].copy())
    if keywords & BLOOM:
        out.update(lo=CM.to_bytes(d["lo"])[::-1].copy(), hi=CM.to_bytes(d["hi"])[::-1].copy())
    return out


def resize(src, Wn, Hn, half=False, conv=LIBRARY):
    """resizeFBO's copy (S:1108-1114) of an (H, W, C) field through its NEAREST sampler into Wn x Hn, stored in
    fp16 when `half`."""
    return _stored(half)(nearest_fetch(np.ascontiguousarray(src, F), *uv_grid(Wn, Hn, conv)).astype(F))
