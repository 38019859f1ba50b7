"""A plain reference for splat() (splatShader S:726-744) with a per-texel interval, independent of the
oracle and of the library: numpy only.

Everything in the shader but exp() is fp32 arithmetic that numpy reproduces bit for bit (float32
operations are IEEE round-to-nearest and numpy never contracts a*b+c into an fma; the library is
built with --fmad=false):

    uv = (i + .5) / W                   (a multiplication by the exact 1/W on power-of-two grids:
                                         the same value)
    dx = (uvx - x) * aspect;  dy = uvy - y;  d = dx*dx + dy*dy;  q = -d / radius
    v' = base + e * c                   per channel, rounded to the storage format; dye alpha = 1

with aspect = float32(canvas_w / canvas_h) and radius = correctRadius(SPLAT_RADIUS / 100): double
arithmetic, multiplied by the aspect only when it is above 1, narrowed to fp32 once (S:1457-1462).

e = expf(q) is not exactly reproducible: the device's expf is within EXPF_ULP ulp of exp(q) (the CUDA
Math API's documented maximum error), glibc's within 1.  So e is bounded by [lo, hi]: exp(float64(q))
rounded to fp32 and widened by EXPF_ULP steps of nextafter, clamped at 0 (subnormal results step by
the subnormal ulp).  Every later step is monotone in e and in the base -- e*c (non-decreasing for
c >= 0, non-increasing for c < 0), base + t, the fp16 rounding of half storage -- so [lo, hi] carries
through any number of records, texel by texel.  A NaN base stays NaN and an inf base the same inf;
where lo and hi are zeros of one sign the result is that zero (-0 + e*c with e*c == +0 is +0).

The cases the CPU premises (tests/test_splat_model_cpu.py) and the GPU bounds (tests/test_gpu_splat_bounds.py)
share close the file: grids, starting fields, radii, canvases and records.
"""
from __future__ import annotations

import numpy as np

from sim_harness import SIZES, exp_tiled, nasty_fields, nasty_records

F32 = np.float32
# CUDA Math API, expf: maximum error 2 ulp (full range, without -use_fast_math)
EXPF_ULP = 2


def aspect_of(canvas_w, canvas_h) -> np.float32:
    """The aspectRatio uniform: the canvas ratio in double, narrowed once."""
    return F32(canvas_w / canvas_h)


def radius_of(splat_radius, canvas_w, canvas_h) -> np.float32:
    """correctRadius(SPLAT_RADIUS / 100), S:1447 + S:1457-1462: JS doubles, one fp32 narrowing."""
    r = float(splat_radius) / 100.0
    a = canvas_w / canvas_h
    if a > 1:
        r *= a
    return F32(r)


def uv(n: int) -> np.ndarray:
    """Texel centres (i + .5) / n of an n-texel axis, in fp32."""
    return (np.arange(n, dtype=F32) + F32(0.5)) / F32(n)


def quotient(uvx, uvy, x, y, aspect, radius) -> np.ndarray:
    """q = -(dx*dx + dy*dy) / radius on the (len(uvy), len(uvx)) texels, in the shader's fp32 order."""
    dx = (uvx - F32(x)) * F32(aspect)
    dy = uvy - F32(y)
    d = (dx * dx)[None, :] + (dy * dy)[:, None]
    return -d / F32(radius)


def exp_rn(q) -> np.ndarray:
    """exp(q) correctly rounded to fp32 (float64 exp is far more accurate than half an fp32 ulp)."""
    return np.exp(np.asarray(q, np.float64)).astype(F32)


def step_ulps(a, k) -> np.ndarray:
    """a moved k fp32 ulps up (k > 0) or down (k < 0)."""
    a = np.asarray(a, F32)
    to = F32(np.inf) if k > 0 else F32(-np.inf)
    for _ in range(abs(k)):
        a = np.nextafter(a, to)
    return a


def expf_bounds(q):
    """[lo, hi] holding expf(q) of any implementation within EXPF_ULP of exp(q)."""
    e = exp_rn(q)
    return np.maximum(step_ulps(e, -EXPF_ULP), F32(0.0)), step_ulps(e, EXPF_ULP)


def store(v, half: bool) -> np.ndarray:
    """The storage format's rounding: identity for fp32, RN-even to fp16 (overflow to inf) for half."""
    if not half:
        return v
    with np.errstate(over="ignore"):
        return v.astype(np.float16).astype(F32)


def apply(lo, hi, elo, ehi, col, half: bool = False):
    """One record on one plane: [lo, hi] (H, W, C) and e in [elo, ehi] (H, W) -> the new interval.
    col holds one colour per channel that is splatted (2 for velocity, 3 for dye); a 4th channel is
    dye alpha and becomes 1."""
    lo, hi = lo.copy(), hi.copy()
    for k, c in enumerate(np.asarray(col, F32)):
        c = F32(c)
        tlo, thi = (ehi * c, elo * c) if c < 0 else (elo * c, ehi * c)
        lo[..., k] = store(lo[..., k] + tlo, half)
        hi[..., k] = store(hi[..., k] + thi, half)
    if lo.shape[-1] == 4:
        lo[..., 3] = F32(1.0)
        hi[..., 3] = F32(1.0)
    return lo, hi


def plane_colours(recs, channels: int) -> np.ndarray:
    """Per-record colours of a plane: (dx, dy) for velocity, (r, g, b) for dye."""
    recs = np.asarray(recs, F32)
    return recs[:, 2:4] if channels == 2 else recs[:, 4:7]


def splat_interval(base, recs, aspect, radius, half: bool = False, rows=None, H: int | None = None):
    """[lo, hi] of every texel of `base` (rows, W, C) after the records (n, 7) of (x, y, dx, dy, r, g, b)
    in order.  `rows` are the global row indices of base's rows on a grid of H rows (default: all)."""
    base = np.ascontiguousarray(base, F32)
    W, C = base.shape[1], base.shape[2]
    if rows is None:
        rows, H = np.arange(base.shape[0]), base.shape[0]
    uvx = uv(W)
    uvy = ((np.asarray(rows).astype(F32) + F32(0.5)) / F32(H)).astype(F32)
    recs = np.asarray(recs, F32).reshape(-1, 7)
    cols = plane_colours(recs, C)
    lo, hi = base.copy(), base.copy()
    for r, col in zip(recs, cols):
        q = quotient(uvx, uvy, r[0], r[1], aspect, radius)
        elo, ehi = expf_bounds(q)
        lo, hi = apply(lo, hi, elo, ehi, col, half)
    return lo, hi


def check_splat(got, lo, hi, limit: int = 8):
    """The texels of `got` outside [lo, hi] (NaN where the interval is NaN, the sign of a zero where
    both ends are that zero): (number of offending elements, the first `limit` of them as
    (index, got, lo, hi)) -- an empty list means every texel is inside."""
    got = np.asarray(got, F32); lo = np.asarray(lo, F32); hi = np.asarray(hi, F32)
    assert got.shape == lo.shape == hi.shape, (got.shape, lo.shape)
    nan = np.isnan(lo) | np.isnan(hi)
    with np.errstate(invalid="ignore"):
        ok = np.where(nan, np.isnan(got), (got >= lo) & (got <= hi))
    zero = (lo == 0) & (hi == 0) & (np.signbit(lo) == np.signbit(hi))
    ok &= ~zero | (np.signbit(got) == np.signbit(lo))
    bad = np.argwhere(~ok)
    out = [(tuple(int(t) for t in ix), float(got[tuple(ix)]), float(lo[tuple(ix)]), float(hi[tuple(ix)]))
           for ix in bad[:limit]]
    return int(len(bad)), out


# ---- the cases -------------------------------------------------------------------------------------------
# SIZES plus partial 128x16 splat tiles in both directions on both planes
GRIDS = SIZES + [(129, 17, 257, 33)]
BASES = ["zero", "exp_tiled", "nasty"]
RADII = [0.25, 0.01, 1.0, 5e-5]          # 5e-5: radius 5e-7 < 2^-20, every warp takes the IEEE division
# aspect 1, > 1, < 1, and a canvas whose radius depends on narrowing the aspect before the multiply
CANVASES = [(100, 100), (300, 200), (200, 300), (142, 100)]
NARROWING_CANVAS = (142, 100)


def records(n, seed, planes):
    """nasty_records (far points, points outside [0, 1], large forces, (.5, .5)) with every 4th record
    from the second on moved onto a texel centre of one of `planes` ((W, H) pairs): d == 0 there."""
    r = nasty_records(n, seed)
    rng = np.random.default_rng(seed + 1)
    for k in range(1, n, 4):
        W, H = planes[(k // 4) % len(planes)]
        r[k, 0] = uv(W)[rng.integers(0, W)]
        r[k, 1] = uv(H)[rng.integers(0, H)]
    return r


def bases(kind, W, H, Wd, Hd, seed):
    """(velocity, dye) starting fields: zeros, one binary exponent in [-149, 100] per tile with random
    mantissas and signs, or nasty_fields (-0, subnormals, +-inf, NaN over ordinary values)."""
    if kind == "zero":
        return np.zeros((H, W, 2), F32), np.zeros((Hd, Wd, 4), F32)
    if kind == "exp_tiled":
        return exp_tiled((H, W, 2), seed, tile=(4, 8)), exp_tiled((Hd, Wd, 4), seed + 1, tile=(4, 8))
    v, d, _ = nasty_fields(W, H, Wd, Hd, seed)
    return v, d
