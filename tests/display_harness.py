"""What the display tests share: their input data -- among it the inputs of the display interval and the post-FX
slider sets that both the CPU premises and the GPU tests draw -- the `dither` fixture, and the GPU side of render()
and captureScreenshot() -- handles of every storage and sampler kind, and their frames and captures checked
against display_model.
Test infrastructure; the handles need the built package and a GPU, the data does not.

A handle kind names the flags a handle is made with: "fp32" or "half" (FLUID_FLAG_HALF_STORAGE), then
"_half_postfx" (FLUID_FLAG_HALF_POSTFX: fp16 post-FX targets), all behind "nearest_"
(FLUID_FLAG_NEAREST_FILTERING) for the NEAREST samplers.  The model of a kind draws with its sampler and
storage: half_targets with HALF_POSTFX, half_mask (the sunrays mask lives in dye.write) with HALF_STORAGE."""
import numpy as np
import pytest

import display_model as M
import gamma_model as G
from conftest import golden
from oracle import oracle as O

F32 = np.float32
BACK = {"r": 10, "g": 20, "b": 30}
BACK_RGB = (10 / 255, 20 / 255, 30 / 255)
FXCFG = dict(BLOOM_RESOLUTION=64, SUNRAYS_RESOLUTION=48)
BACKGROUNDS = {"back": O.BG_COLOR, "checker": O.BG_CHECKERBOARD, "bare": O.BG_NONE}
MODES = {"back": (False, False), "checker": (True, False), "bare": (True, True)}     # (TRANSPARENT, target)


# ---- input data ----------------------------------------------------------------------------------------------
def seeded_dye(Wd, Hd, seed, scale=3.0):
    rng = np.random.default_rng(seed)
    dye = (rng.random((Hd, Wd, 4), dtype=F32) ** 4 * F32(scale)).astype(F32)
    dye[..., 3] = 1
    return dye


def nonfinite_dye(Wd, Hd, seed):
    """Seeded dye with +-inf, NaN, -2, a subnormal and 1e30 in whole texels and in single channels: at
    the four corners, along the four edges and inside."""
    dye = seeded_dye(Wd, Hd, seed)
    specials = [np.inf, -np.inf, np.nan, -2.0, 1e-40, 1e30]
    rng = np.random.default_rng(seed + 1)
    spots = [(0, 0), (0, Wd - 1), (Hd - 1, 0), (Hd - 1, Wd - 1), (0, Wd // 2), (Hd - 1, Wd // 3),
             (Hd // 2, 0), (Hd // 3, Wd - 1)] + [tuple(rng.integers(1, (Hd - 1, Wd - 1))) for _ in range(16)]
    for k, (j, i) in enumerate(spots):
        v = F32(specials[k % len(specials)])
        if k < 12:
            dye[j, i, :3] = v                    # the whole colour
        else:                                    # one channel of a bright texel
            dye[j, i, :3] = 2.0
            dye[j, i, k % 3] = v
    return dye


def golden_dither():
    return golden("postfx_64_to_128")["dither"].astype(F32)


@pytest.fixture(scope="module")
def dither():
    return golden_dither()


# ---- handles -------------------------------------------------------------------------------------------------
def kind_of(kind):
    """(nearest, half_targets, half_mask) of a handle kind."""
    base = kind[len("nearest_"):] if kind.startswith("nearest_") else kind
    assert base in ("fp32", "half", "fp32_half_postfx", "half_half_postfx"), kind
    return kind.startswith("nearest_"), base.endswith("_half_postfx"), base.startswith("half")


def flags_of(pkg, kind):
    nearest, half_targets, half_mask = kind_of(kind)
    return ((pkg.FLAG_NEAREST_FILTERING if nearest else 0) | (pkg.FLAG_HALF_POSTFX if half_targets else 0)
            | (pkg.FLAG_HALF_STORAGE if half_mask else 0))


def allowed(kind, kw):
    """Half storage without HALF_POSTFX draws only the sets without BLOOM and SUNRAYS."""
    _, half_targets, half_mask = kind_of(kind)
    return half_targets or not half_mask or not kw & (M.BLOOM | M.SUNRAYS)


def make(pkg, Wd, Hd, w, h, flags=0, **cfg):
    """A handle of Wd x Hd dye on a w x h canvas, BACK_COLOR (10, 20, 30), the post-FX sizes of FXCFG unless cfg
    says otherwise."""
    s = pkg.FluidSimulation({"SIM_RESOLUTION": 16, "DYE_RESOLUTION": min(Wd, Hd)}, canvas_width=w, canvas_height=h,
                            flags=flags, sizes=(16, 16, Wd, Hd))
    s.config.update(BACK_COLOR=BACK, **FXCFG)
    s.config.update(cfg)
    return s


def set_keywords(s, kw):
    s.config.update(SHADING=bool(kw & M.SHADING), BLOOM=bool(kw & M.BLOOM), SUNRAYS=bool(kw & M.SUNRAYS))


def stored(kind, dye):
    """The dye as a handle of `kind` holds it after writeField: fp16-rounded with half storage."""
    return O.round_half(dye) if kind_of(kind)[2] else np.ascontiguousarray(dye, F32)


# ---- the model of a kind, and the checks ---------------------------------------------------------------------
def model_frame(kind, dye, w, h, kw, dither, cfg, background):
    """display_model.render with the kind's sampler and storage: chains, target, and lo / hi with BLOOM."""
    nearest, half_targets, half_mask = kind_of(kind)
    return M.render(dye, w, h, dither, kw, cfg, back_rgb=BACK_RGB, background=background, aspect=w / h,
                    nearest=nearest, half_targets=half_targets, half_mask=half_mask)


def model_capture(kind, dye, w, h, cw, ch, kw, dither, cfg, transparent):
    """display_model.capture with the kind's sampler and storage: rgba8, and the byte bracket lo / hi with BLOOM."""
    nearest, half_targets, half_mask = kind_of(kind)
    return M.capture(dye, w, h, cw, ch, dither, kw, transparent, BACK_RGB, cfg=cfg, nearest=nearest,
                     half_targets=half_targets, half_mask=half_mask)


def check_frame(s, got, want, kw, what):
    """The handle's bloom FBO and sunrays texture bit for bit against the model's (NaN in the same places), None
    when their keyword is off; the frame bit for bit without BLOOM, inside the model's powf interval with it."""
    if kw & M.BLOOM:
        assert G.same_bits(s.last_bloom, want["bloom"]), what
        n, bad = G.check_display(got, want["lo"], want["hi"])
        assert n == 0, (what, n, bad)
    else:
        assert s.last_bloom is None and G.same_bits(got, want["target"]), what
    if kw & M.SUNRAYS:
        assert G.same_bits(s.last_sunrays, want["sunrays"]), what
    else:
        assert s.last_sunrays is None, what


def check_capture(got, want, kw, what):
    """The capture's bytes: the model's exactly without BLOOM, inside its byte bracket with it."""
    if kw & M.BLOOM:
        assert G.bytes_outside(got, want["lo"], want["hi"]) == 0, what
    else:
        assert np.array_equal(got, want["rgba8"]), what


def draw_all(pkg, kind, dye_in, w, h, dither, cfg=FXCFG, sets=range(8), modes=MODES):
    """Every allowed keyword set of `sets` x background of `modes` on a fresh handle of `kind`: check_frame against
    the kind's model, and dye.read unchanged afterwards."""
    cfg = dict(FXCFG, **cfg)
    s = make(pkg, dye_in.shape[1], dye_in.shape[0], w, h, flags_of(pkg, kind), **cfg)
    s.writeField("dye", dye_in)
    s.dithering = dither
    dye = stored(kind, dye_in)
    with np.errstate(invalid="ignore", over="ignore"):
        for kw in (k for k in sets if allowed(kind, k)):
            set_keywords(s, kw)
            for bg in modes:
                s.config["TRANSPARENT"] = MODES[bg][0]
                got = s.render(w, h, target=MODES[bg][1])
                check_frame(s, got, model_frame(kind, dye, w, h, kw, dither, cfg, BACKGROUNDS[bg]), kw, (kind, kw, bg))
                assert G.same_bits(s.readField("dye"), dye), (kind, kw, bg)
    s.close()


# ---- the inputs of the display interval (gamma_model), CPU and GPU -----------------------------------------
# dim dye (seeded_dye(scale=1) * 0.25) with bloom this faint puts bk on both sides of linearToGamma's knee
# (fmaxf(1.055 p - 0.055, 0) = 0 below bk = 8.3e-4): about 10 % of values at 0, 10 % between 0 and the knee
DIM_CFG = dict(FXCFG, BLOOM_INTENSITY=0.005, BLOOM_THRESHOLD=0.0)


def wide_dither(seed, shape=(64, 64)):
    """Dithering values 2^-1 .. 2^60 (random exponent and mantissa)."""
    rng = np.random.default_rng(seed)
    e = rng.integers(-1, 60, shape + (3,))
    return (np.ldexp(1.0 + rng.random(shape + (3,)), e) / 2).clip(0.5, 2.0 ** 60).astype(F32)


def overflow_dither(seed, shape=(64, 64)):
    """The golden dithering texture with a third of its texels above FLT_MAX / 2 in magnitude, of either
    sign: noise = d * 2 - 1 is +-inf there, and so is bk."""
    d = golden_dither().copy()
    rng = np.random.default_rng(seed)
    m = rng.random(shape) < 1 / 3
    big = F32(2.0 ** 127) * (1 + rng.random((int(m.sum()), 3)).astype(F32) * F32(0.99))
    d[m] = np.where(rng.random((int(m.sum()), 1)) < 0.5, big, -big).astype(F32)
    return d


def case(dye, w, h, dither, cfg=FXCFG):
    return dict(dye=np.ascontiguousarray(dye, F32), w=w, h=h, dither=np.ascontiguousarray(dither, F32), cfg=dict(cfg))


def golden_case(name):
    g = golden(name)
    return case(g["in_dye"], int(g["w"]), int(g["h"]), g["dither"].astype(F32),
                dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"])))


def make_cases():
    """The inputs, by name: (dye, target w x h, dithering texture, post-FX keys)."""
    s = seeded_dye(64, 64, 192)
    rng = np.random.default_rng(5)
    return {
        "postfx_64_to_128": golden_case("postfx_64_to_128"),
        "postfx_48x32_to_50x75": golden_case("postfx_48x32_to_50x75"),
        "keywords_transparent_64x32_to_128x64": golden_case("keywords_transparent_64x32_to_128x64"),
        "seeded": case(s, 128, 128, golden_dither()),
        "zero": case(np.zeros((64, 64, 4), F32), 128, 128, golden_dither()),
        "dim": case(seeded_dye(64, 64, 192, scale=1.0) * F32(0.25), 128, 128, golden_dither(), DIM_CFG),
        "wide_dither": case(s, 128, 128, wide_dither(3)),
        "overflow_dither": case(s, 128, 128, overflow_dither(4)),
        "dither_37x23": case(s, 128, 128, rng.random((23, 37, 3), dtype=F32)),
        "dither_1x1": case(s, 128, 128, np.full((1, 1, 3), 0.6, F32)),
        "nonfinite": case(nonfinite_dye(64, 64, 8), 128, 128, golden_dither()),
    }


CASES = make_cases()


# ---- the post-FX sliders away from their defaults, CPU and GPU ----------------------------------------------
DEFAULTS = dict(BLOOM_INTENSITY=0.8, BLOOM_THRESHOLD=0.6, BLOOM_SOFT_KNEE=0.7, SUNRAYS_WEIGHT=1.0)   # S:79-84
# (I, T, K, W).  t033_k07 and t039_k1 are slider positions where knee / curve narrowed from fp32 arithmetic
# differ from the JS doubles narrowed once (all three curve components); t005 differs in curve.x and curve.z.
SETS = {
    "t0_k1": (0.8, 0.0, 1.0, 1.0),           # threshold 0: curve = (-1e-4, 2e-4, 2500); the knee is wider than the threshold
    "t0_k0_w4": (0.1, 0.0, 0.0, 4.0),        # sunrays above 1: alpha above 1, the canvas clamps
    "t005": (1.3, 0.05, 0.7, 0.6),
    "t033_k07": (0.55, 0.33, 0.7, 0.45),
    "t039_k1": (1.6, 0.39, 1.0, 0.85),
    "t1_k0_i2_w03": (2.0, 1.0, 0.0, 0.3),    # knee 0: knee = 1e-4, a hard step
    "t1_k1": (0.1, 1.0, 1.0, 1.0),
    "i0_w0": (0.0, 0.6, 0.7, 0.0),
    "overflow": (70000.0, 0.6, 0.7, 1.0),    # the final blit overflows fp16 to +inf on about half the HALF_POSTFX texels
    "above": (0.8, 5.0, 0.2, 0.5),           # curve.x = 4 above every br of the dye: the prefilter draws zeros
}
KEYS = ("BLOOM_INTENSITY", "BLOOM_THRESHOLD", "BLOOM_SOFT_KNEE", "SUNRAYS_WEIGHT")
# (dye w, dye h, canvas w, canvas h, BLOOM_RESOLUTION, SUNRAYS_RESOLUTION, CAPTURE_RESOLUTION): every size a
# power of two (bloom 64 x 32, sunrays 32 x 16, capture 64 x 32), and a ragged dye on a portrait canvas
# (bloom 48 x 64, sunrays 30 x 40, capture 45 x 60)
GEOMETRIES = {"pow2": (64, 64, 128, 64, 32, 16, 32), "portrait": (40, 56, 90, 120, 48, 30, 45)}
DYE_SEED = 2718


def cfg_of(name, geometry="pow2"):
    """The config keys of parameter set `name` on `geometry`."""
    I, T, K, W = SETS[name]
    bres, sres, cres = GEOMETRIES[geometry][4:]
    return dict(BLOOM_INTENSITY=I, BLOOM_THRESHOLD=T, BLOOM_SOFT_KNEE=K, SUNRAYS_WEIGHT=W, BLOOM_RESOLUTION=bres,
                SUNRAYS_RESOLUTION=sres, CAPTURE_RESOLUTION=cres)


def params_dye(Wd, Hd, seed=DYE_SEED):
    """Finite dye whose brightest channel br (the prefilter's) falls in 4 x 4 blocks of one kind each, so that a
    LINEAR fetch at ragged sizes mostly mixes texels of one kind: exact zeros (the other channels in -2e-3 .. -1e-3), fp32
    subnormals, negatives down to -2, +-1e-7 .. 1e-4 around the threshold-0 knee, values inside the knee
    [T - knee, T + knee] of a set of SETS but `above` (a hard step's knee is 2e-4 wide: no uniform draw would land there),
    and bright values 3.2 u^1.5 (u uniform) reaching every knee.  One channel holds br, the other two a
    fraction of it (more negative for a negative br); which channel is the same across a block.  Alpha 1.  No channel is -0, in fp32 or
    rounded to fp16: where the display's alpha is fmaxf(-0, +0), the device and C need not agree."""
    rng = np.random.default_rng(seed)
    bh, bw = (Hd + 3) // 4, (Wd + 3) // 4
    up = lambda a: np.kron(a, np.ones((4, 4), a.dtype))[:Hd, :Wd]             # noqa: E731
    kind = up(rng.choice(6, size=(bh, bw), p=[0.07, 0.06, 0.09, 0.09, 0.19, 0.50]))
    knees = np.array([(t, t * k + 0.0001) for n, (_, t, k, _) in SETS.items() if n != "above"])
    pick = up(rng.integers(0, len(knees), (bh, bw)))
    u = rng.random((Hd, Wd))
    sign = np.where(rng.random((Hd, Wd)) < 0.5, -1.0, 1.0)
    br = np.select([kind == 0, kind == 1, kind == 2, kind == 3, kind == 4],
                   [np.zeros_like(u), 1e-45 + u * 1.1e-38, -np.exp(np.log(1e-6) + u * np.log(2e6)),
                    sign * np.exp(np.log(1e-7) + u * np.log(1e3)), knees[pick, 0] + knees[pick, 1] * (2 * u - 1)],
                   3.2 * u ** 1.5).astype(F32)
    frac = rng.random((Hd, Wd, 3)).astype(F32)
    c = np.where(br[..., None] >= 0, br[..., None] * frac, br[..., None] * (F32(1) + frac))
    c[kind == 0] = -(F32(1) + frac[kind == 0]) * F32(1e-3)
    top = up(rng.integers(0, 3, (bh, bw)))
    np.put_along_axis(c, top[..., None], br[..., None], axis=-1)
    dye = np.concatenate([c, np.ones((Hd, Wd, 1), F32)], axis=-1).astype(F32)
    assert np.isfinite(dye).all() and not ((dye == 0) & np.signbit(dye)).any()
    assert not ((O.round_half(dye) == 0) & np.signbit(O.round_half(dye))).any()
    return dye


FIXTURES = [f"postfx_params_{n}_64_to_128x64" for n in ("t033_k07", "t0_k1", "t1_k0_i2_w03")]


def fixture_cfg(g):
    return dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]),
                BLOOM_INTENSITY=float(g["intensity"]), BLOOM_THRESHOLD=float(g["threshold"]),
                BLOOM_SOFT_KNEE=float(g["soft_knee"]), SUNRAYS_WEIGHT=float(g["weight"]))
