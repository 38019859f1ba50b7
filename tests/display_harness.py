"""What the display tests share: their input data, and the GPU side of render() and captureScreenshot() --
handles of every storage and sampler kind, and their frames and captures checked against display_model.
Test infrastructure; the handles need the built package and a GPU, the data does not.

A handle kind names the flags a handle is made with: "fp32" or "half" (FLUID_FLAG_HALF_STORAGE), then
"_half_postfx" (FLUID_FLAG_HALF_POSTFX: fp16 post-FX targets), all behind "nearest_"
(FLUID_FLAG_NEAREST_FILTERING) for the NEAREST samplers.  The model of a kind draws with its sampler and
storage: half_targets with HALF_POSTFX, half_mask (the sunrays mask lives in dye.write) with HALF_STORAGE."""
import numpy as np

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
