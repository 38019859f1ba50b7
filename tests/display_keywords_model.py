"""CPU model of render() for any display keyword set (updateKeywords, S:1160-1166).  Test infrastructure.

The CPU oracle (oracle/oracle.py) pins two ends: `display` (no keyword / SHADING, bloom and sunrays
off) and `render_postfx` (SHADING + BLOOM + SUNRAYS).  This module covers the five sets between them:
the bloom and sunrays chains come from the oracle's `render_postfx` (they do not depend on the
keywords), and displayShaderSource (S:549-612) is restated here in numpy with the oracle's fp32
operation order -- the LINEAR fetch of oracle_display / oracle_display_full, no contraction -- so that
sets without BLOOM are exact and the others differ from C only in pow() (linearToGamma).
"""
import numpy as np

from oracle import oracle as O

SHADING, BLOOM, SUNRAYS = 1, 2, 4       # FLUID_DISPLAY_* of include/fluid.h
F = np.float32
_NO_DITHER = np.zeros((1, 1, 3), F)      # the oracle's chains need a texture; without BLOOM it is never read


def _texel(f, n):
    """CLAMP_TO_EDGE index of a floored coordinate (texel_index of the oracle)."""
    return np.where(~(f > 0), 0, np.where(f >= F(n - 1), n - 1, np.maximum(f, 0))).astype(np.int64)


def _fetch(tex, uvx, uvy, repeat=False):
    """GL-spec LINEAR fetch of an (H, W, C) texture at (uvx, uvy) fp32 arrays (linear_fetch /
    linear_fetch_w of the oracle): weights (1-a)(1-b) .. ab, summed left to right."""
    H, W = tex.shape[:2]
    u = uvx * F(W) - F(0.5); v = uvy * F(H) - F(0.5)
    fi = np.floor(u); fj = np.floor(v)
    a = (u - fi)[..., None]; b = (v - fj)[..., None]
    if repeat:
        i0 = np.mod(fi.astype(np.int64), W); j0 = np.mod(fj.astype(np.int64), H)
        i1 = (i0 + 1) % W; j1 = (j0 + 1) % H
    else:
        i0, i1, j0, j1 = _texel(fi, W), _texel(fi + F(1), W), _texel(fj, H), _texel(fj + F(1), H)
    one = F(1)
    w00 = (one - a) * (one - b); w10 = a * (one - b); w01 = (one - a) * b; w11 = a * b
    return ((w00 * tex[j0, i0] + w10 * tex[j0, i1]) + w01 * tex[j1, i0]) + w11 * tex[j1, i1]


def _len3(c):
    return np.sqrt((c[..., 0] * c[..., 0] + c[..., 1] * c[..., 1]) + c[..., 2] * c[..., 2])


def uv_grid(w, h):
    """vUv of every texel of a w x h target: (h, w) fp32 arrays (i + .5) / w and (j + .5) / h."""
    uvx = ((np.arange(w, dtype=F) + F(0.5)) / F(w))[None, :].repeat(h, 0)
    uvy = ((np.arange(h, dtype=F) + F(0.5)) / F(h))[:, None].repeat(w, 1)
    return uvx, uvy


def colour_terms(dye, w, h, keywords, bloom, sun):
    """displayShaderSource up to the dithering: the dye colour c (LINEAR fetch, SHADING's diffuse, the
    sunrays multiply) and, with BLOOM, the bloom colour bl (LINEAR fetch, sunrays multiply), else None.
    Every max / min is C's fmaxf / fminf (np.fmax / np.fmin: a NaN argument is dropped)."""
    tsx, tsy = F(1.0 / w), F(1.0 / h)
    uvx, uvy = uv_grid(w, h)
    c = _fetch(dye, uvx, uvy)[..., :3]
    if keywords & SHADING:
        dx = _len3(_fetch(dye, uvx + tsx, uvy)) - _len3(_fetch(dye, uvx - tsx, uvy))
        dy = _len3(_fetch(dye, uvx, uvy + tsy)) - _len3(_fetch(dye, uvx, uvy - tsy))
        nz = np.sqrt(tsx * tsx + tsy * tsy)
        nl = np.sqrt((dx * dx + dy * dy) + nz * nz)
        d = ((dx / nl) * F(0) + (dy / nl) * F(0)) + (nz / nl) * F(1)
        diffuse = np.fmin(np.fmax(d + F(0.7), F(0.7)), F(1))
        c = c * diffuse[..., None]
    bl = _fetch(bloom, uvx, uvy)[..., :3] if keywords & BLOOM else None
    if keywords & SUNRAYS:
        s = _fetch(sun[..., None], uvx, uvy)
        c = c * s
        if keywords & BLOOM:
            bl = bl * s
    return c, bl


def dither_scale(w, h, dither):
    """getTextureScale (S:1626-1631) of the dithering texture on a w x h target: JS doubles, narrowed once."""
    return F(w / dither.shape[1]), F(h / dither.shape[0])


def gamma_argument(bl, dither, w, h, scale=None):
    """The argument of linearToGamma's pow: fmaxf(bl + noise / 255, 0), noise = the REPEAT LINEAR fetch of
    the dithering texture at vUv * getTextureScale, * 2 - 1.  `scale` defaults to the w x h target's."""
    dsx, dsy = scale if scale is not None else dither_scale(w, h, dither)
    uvx, uvy = uv_grid(w, h)
    noise = _fetch(dither, uvx * dsx, uvy * dsy, repeat=True)[..., :1] * F(2) - F(1)
    return np.fmax(bl + noise / F(255), F(0))


GAMMA_EXPONENT = F(0.416666667)


def linear_to_gamma(p):
    """linearToGamma (S:565-568) after its pow: fmaxf(1.055 * p - 0.055, 0), p = pow(bk, 0.416666667)."""
    return np.fmax(F(1.055) * p - F(0.055), F(0))


def background_colour(w, h, back_rgb, background, aspect):
    """What the display is blended over, (h, w, 3): BACK_COLOR, or checkerboardShader (S:531-547)."""
    if background == O.BG_CHECKERBOARD:
        uvx, uvy = uv_grid(w, h)
        x = np.floor((uvx * F(25)) * F(aspect)); y = np.floor((uvy * F(25)) * F(1))
        sxy = x + y
        v = (sxy - F(2) * np.floor(sxy / F(2))) * F(0.1) + F(0.8)
        return np.stack([v, v, v], axis=-1)
    return np.broadcast_to(np.asarray(back_rgb, F), (h, w, 3))


def alpha_of(c):
    """The display's alpha: fmaxf(c.r, fmaxf(c.g, c.b))."""
    return np.fmax(c[..., 0], np.fmax(c[..., 1], c[..., 2]))[..., None]


def over_background(c, a, back_rgb, background, aspect):
    """render()'s blend ONE / ONE_MINUS_SRC_ALPHA of (c, a) over the background, or (c, a) bare (BG_NONE)."""
    if background == O.BG_NONE:
        return np.concatenate([c, a], axis=-1).astype(F)
    h, w = c.shape[:2]
    bg = background_colour(w, h, back_rgb, background, aspect)
    k = F(1) - a
    return np.concatenate([c + bg * k, a + F(1) * k], axis=-1).astype(F)


def _display(dye, w, h, keywords, bloom, sun, dither, back_rgb, background, aspect):
    """displayShaderSource with `keywords`, then the background of render() (oracle background modes)."""
    c, bl = colour_terms(dye, w, h, keywords, bloom, sun)
    if keywords & BLOOM:
        bk = gamma_argument(bl, dither, w, h)
        c = c + linear_to_gamma(np.power(bk, GAMMA_EXPONENT))      # linearToGamma S:565-568
    return over_background(c, alpha_of(c), back_rgb, background, aspect)


def render_keywords(dye, w, h, dither, cfg=None, back_rgb=(0.0, 0.0, 0.0), background=O.BG_COLOR, aspect=None,
                    keywords=SHADING | BLOOM | SUNRAYS):
    """render(null) with the display keywords `keywords`: the dict of oracle.render_postfx, with None
    (pyramid: []) for the outputs of a chain that is off.  dither is read only with BLOOM."""
    dye = np.ascontiguousarray(dye, F)
    aspect = w / h if aspect is None else aspect
    if not keywords & (BLOOM | SUNRAYS):
        return dict(target=O.display(dye, w, h, bool(keywords & SHADING), back_rgb, background, aspect),
                    bloom=None, sunrays=None, mask_alpha=None, pyramid=[])
    dith = np.ascontiguousarray(dither, F) if keywords & BLOOM else _NO_DITHER
    r = O.render_postfx(dye, w, h, dith, cfg=cfg, back_rgb=back_rgb, background=background, aspect=aspect)
    if keywords != SHADING | BLOOM | SUNRAYS:
        r["target"] = _display(dye, w, h, keywords, r["bloom"], r["sunrays"], dith, back_rgb, background, aspect)
    if not keywords & BLOOM:
        r.update(bloom=None, pyramid=[])
    if not keywords & SUNRAYS:
        r.update(sunrays=None, mask_alpha=None)
    return r
