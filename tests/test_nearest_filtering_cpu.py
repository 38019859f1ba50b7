"""FLUID_FLAG_NEAREST_FILTERING without a GPU: display_model.py's NEAREST sampler against the executed NEAREST shaders
(tests/golden/make_golden_nearest.py) and the `nearest` keys of the resize fixtures; the two vUv
conventions; the flag's value in every binding; default_config's override (S:109-114).

No comparison here uses a value tolerance for a NEAREST fetch: frames without BLOOM and every chain
texture are compared bit for bit, frames with BLOOM against gamma_model's per-texel powf interval."""
import os
import re

import numpy as np
import pytest

import capture_model as CM
import display_model as M
import gamma_model as G
from conftest import golden
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
POW2 = ["nearest_64_to_128_plain", "nearest_64_to_128_bloom"]
HALF = ["nearest_half_64_to_128_plain", "nearest_half_64_to_128_bloom"]
RAGGED = "nearest_48x32_to_50x75"
TRANSPARENT = "nearest_transparent_64x32_to_128x64"
BACKGROUNDS = {"target": O.BG_COLOR, "checker": O.BG_CHECKERBOARD, "bare": O.BG_NONE}


def cfg_of(g):
    return dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]))


def model_of(g, tag, conv, key="target"):
    w, h = int(g["w"]), int(g["h"])
    half = bool(g["half"])
    return M.render(g["in_dye"], w, h, g["dither"].astype(F32), M.SETS[tag], cfg_of(g), back_rgb=tuple(g["back"] / 255),
                    background=BACKGROUNDS[key], nearest=True, half_targets=half, half_mask=half, conv=conv)


def check_against(g, conv):
    """Every chain texture bit for bit, every frame bit for bit (without BLOOM) or inside the interval."""
    keys = [k for k in ("target", "checker", "bare") if any(f"{t}_{k}" in g for t in g["sets"])]
    for tag in (str(t) for t in g["sets"]):
        for key in keys:
            r = model_of(g, tag, conv, key)
            for k in ("bloom", "sunrays", "mask_alpha"):
                if r[k] is not None:
                    assert G.same_bits(r[k], g[k]), (tag, k)
            for k, t in enumerate(r["pyramid"]):
                assert G.same_bits(t, g[f"pyr{k}"]), (tag, k)
            want = g[f"{tag}_{key}"]
            if not M.SETS[tag] & M.BLOOM:
                assert G.same_bits(r["target"], want), (tag, key)
            else:
                n, bad = G.check_display(want, r["lo"], r["hi"])
                assert n == 0, (tag, key, bad)


@pytest.mark.parametrize("name", POW2 + [RAGGED] + HALF + [TRANSPARENT])
def test_raster_convention_equals_executed_shaders(name):
    check_against(golden(name), M.RASTER)


@pytest.mark.parametrize("name", POW2 + HALF + [TRANSPARENT])
def test_library_convention_equals_executed_shaders_at_power_of_two(name):
    check_against(golden(name), M.LIBRARY)


@pytest.mark.parametrize("bg", ["back", "transparent"])
@pytest.mark.parametrize("conv", [M.RASTER, M.LIBRARY])
def test_captures_equal_executed_shaders(bg, conv):
    g = golden(f"nearest_capture_64_canvas_128_{bg}")
    dye, w, h, cw, ch = g["in_dye"], int(g["w"]), int(g["h"]), int(g["canvas_w"]), int(g["canvas_h"])
    for tag in (str(t) for t in g["sets"]):
        r = M.capture(dye, w, h, cw, ch, g["dither"].astype(F32), M.SETS[tag], bool(g["transparent"]),
                      tuple(g["back"] / 255), cfg=cfg_of(g), nearest=True, conv=conv)
        want = g[f"{tag}_rgba8"]
        if not M.SETS[tag] & M.BLOOM:
            assert np.array_equal(r["rgba8"], want), tag
        else:
            assert G.bytes_outside(want, r["lo"], r["hi"]) == 0, tag


# ---- the ragged size: what the two conventions disagree on ------------------------------------------------
class Taps:
    """Records the (j, i) texel of every NEAREST fetch a call makes."""

    def __enter__(self):
        self.taps, self._fetch = [], M.nearest_fetch

        def fetch(tex, uvx, uvy):
            self.taps.append(M.texel(tex, uvx, uvy))
            return self._fetch(tex, uvx, uvy)
        M.nearest_fetch = fetch
        return self

    def __exit__(self, *exc):
        M.nearest_fetch = self._fetch


def flips(call):
    """Runs call(conv) in both conventions on the same inputs: (texels where the outputs differ, texels
    where some tap picked another texel)."""
    with Taps() as a:
        out_l = call(M.LIBRARY)
    with Taps() as b:
        out_r = call(M.RASTER)
    assert len(a.taps) == len(b.taps)
    shape = out_l.shape[:2]
    moved = np.zeros(shape, bool)
    for (jl, il), (jr, ir) in zip(a.taps, b.taps):
        moved |= np.broadcast_to((jl != jr) | (il != ir), shape)
    differ = (out_l != out_r) & ~(np.isnan(out_l) & np.isnan(out_r))
    if differ.ndim == 3:
        differ = differ.any(-1)
    return differ, moved


def ragged_passes(g):
    """Every NEAREST pass of the ragged fixture, each fed the executed shaders' own input textures."""
    w, h = int(g["w"]), int(g["h"])
    dye = g["in_dye"]
    c = dict(M.chains(dye, w, h, M.BLOOM | M.SUNRAYS, cfg_of(g), nearest=True, conv=M.RASTER))
    bh, bw = c["bloom"].shape[:2]
    sh, sw = c["sunrays"].shape
    pyr = [g[f"pyr{k}"] for k in range(len(c["pyramid"]))]
    N, crv = M.Nearest(M.RASTER), M.curve(0.6, 0.7)
    mask = N.sunrays_mask(dye)
    tmp = N.blur3(N.sunrays(mask, sw, sh, 1.0), 1.0 / sw, 0.0)
    prefiltered = N.prefilter(dye, bw, bh, crv)
    passes = {"prefilter": lambda cv: M.Nearest(cv).prefilter(dye, bw, bh, crv),
              "down0": lambda cv: M.Nearest(cv).box4(prefiltered, *pyr[0].shape[1::-1]),
              "mask": lambda cv: M.Nearest(cv).sunrays_mask(dye),
              "sunrays": lambda cv: M.Nearest(cv).sunrays(mask, sw, sh, 1.0),
              "blur_y": lambda cv: M.Nearest(cv).blur3(tmp, 0.0, 1.0 / sh)}
    for k in range(1, len(pyr)):
        passes[f"down{k}"] = (lambda src, size: lambda cv: M.Nearest(cv).box4(src, *size))(_down(dye, g, k - 1), pyr[k].shape[1::-1])
    for tag in ("none", "shading", "sunrays", "shading_sunrays"):
        passes[f"display_{tag}"] = (lambda kw: lambda cv: M.display(dye, w, h, kw, None, g["sunrays"], None, tuple(g["back"] / 255),
                                                                      O.BG_COLOR, w / h, nearest=True, conv=cv)["target"])(M.SETS[tag])
    return passes


def _down(dye, g, k):
    """Level k of the bloom pyramid on the way down, before the up-pass adds to it."""
    w, h = int(g["w"]), int(g["h"])
    bw, bh = M.get_resolution(int(g["bloom_res"]), w, h)
    N = M.Nearest(M.RASTER)
    last = N.prefilter(dye, bw, bh, M.curve(0.6, 0.7))
    for i in range(k + 1):
        last = N.box4(last, bw >> (i + 1), bh >> (i + 1))
    return last


RAGGED_FLIPS = {}


def test_ragged_differences_are_texel_flips():
    """At 48x32 -> 50x75 every texel where the library's vUv and the rasteriser's give different results,
    pass by pass on the same inputs, has a tap that landed on another texel.  The counts are recorded."""
    g = golden(RAGGED)
    counts = {}
    for name, call in ragged_passes(g).items():
        differ, moved = flips(call)
        assert not (differ & ~moved).any(), (name, np.argwhere(differ & ~moved)[:5])
        counts[name] = int(differ.sum())
    RAGGED_FLIPS.update(counts)
    print("ragged 48x32 -> 50x75, texels that differ between the conventions:", counts)
    assert sum(counts.values()) > 0          # the conventions do disagree here: the model must take one


def test_index_arithmetic_of_the_conventions():
    """Centre taps agree at 48->50, 32->75, 910->1920 and 1024->300; the SHADING tap uv + texelSize does not
    at dye 512 -> target 1080 and at 40 -> 50."""
    def centre(n_tex, n_tgt, conv):
        u = M.uv_grid(n_tgt, 1, conv)[0][0]
        return M.texel(np.zeros((1, n_tex)), u, np.zeros_like(u))[1]

    def plus_ts(n_tex, n_tgt, conv):
        u = M.uv_grid(n_tgt, 1, conv)[0][0] + F32(1.0 / n_tgt)
        return M.texel(np.zeros((1, n_tex)), u, np.zeros_like(u))[1]
    for n_tex, n_tgt in ((50, 48), (32, 75), (910, 1920), (1024, 300)):
        assert np.array_equal(centre(n_tex, n_tgt, M.LIBRARY), centre(n_tex, n_tgt, M.RASTER)), (n_tex, n_tgt)
    for n_tex, n_tgt in ((512, 1080), (40, 50)):
        assert not np.array_equal(plus_ts(n_tex, n_tgt, M.LIBRARY), plus_ts(n_tex, n_tgt, M.RASTER)), (n_tex, n_tgt)


@pytest.mark.parametrize("name", ["resample_dye_40x28_to_64x48", "resample_dye_64_to_32", "resample_v_32_to_48"])
def test_resample_nearest_keys(name):
    g = golden(name)
    for conv in (M.LIBRARY, M.RASTER):
        assert G.same_bits(M.resize(g["src"], int(g["Wd"]), int(g["Hd"]), conv=conv), g["nearest"]), (name, conv)


@pytest.mark.parametrize("name", POW2 + [RAGGED] + HALF)
def test_fixtures_discriminate_linear_from_nearest(name):
    """The LINEAR model's frame differs from every NEAREST frame of the fixture."""
    g = golden(name)
    w, h = int(g["w"]), int(g["h"])
    dye = g["in_dye"]
    for tag in (str(t) for t in g["sets"]):
        lin = M.render(dye, w, h, g["dither"].astype(F32), M.SETS[tag], cfg_of(g), back_rgb=tuple(g["back"] / 255))
        assert not np.array_equal(lin["target"], g[f"{tag}_target"]), tag


def test_flag_value_in_every_binding():
    import webgl_fluid_simulation_b200 as pkg
    hdr = open(os.path.join(ROOT, "include", "fluid.h")).read()
    js = open(os.path.join(ROOT, "webgl_fluid_simulation_b200", "js", "fluid-sim.js")).read()
    h = int(re.search(r"#define FLUID_FLAG_NEAREST_FILTERING (0x[0-9a-f]+)u", hdr).group(1), 16)
    j = int(re.search(r"NEAREST_FILTERING: (0x[0-9a-f]+)", js).group(1), 16)
    assert h == j == pkg.FLAG_NEAREST_FILTERING == 0x40
    others = [int(v, 16) for v in re.findall(r"#define FLUID_FLAG_\w+ (0x[0-9a-f]+)u", hdr)]
    assert others.count(0x40) == 1


def test_default_config_applies_the_no_linear_override():
    import webgl_fluid_simulation_b200 as pkg
    d, n = pkg.default_config(), pkg.default_config(pkg.FLAG_NEAREST_FILTERING)
    assert (n["DYE_RESOLUTION"], n["SHADING"], n["BLOOM"], n["SUNRAYS"]) == (512, False, False, False)
    assert {k: v for k, v in n.items() if k not in ("DYE_RESOLUTION", "SHADING", "BLOOM", "SUNRAYS")} == \
           {k: v for k, v in d.items() if k not in ("DYE_RESOLUTION", "SHADING", "BLOOM", "SUNRAYS")}
    assert pkg.default_config(pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX) == d


def test_model_nearest_fetch_on_nonfinite_and_out_of_range_coordinates():
    """NaN -> texel 0, -inf / negative -> 0, +inf / >= 1 -> n - 1; a NaN texel reaches only its own texels."""
    tex = np.arange(12, dtype=F32).reshape(3, 4, 1)
    u = np.array([np.nan, -np.inf, -0.3, 0.0, 0.24, 0.26, 0.99, 1.0, np.inf], F32)
    got = M.nearest_fetch(tex, u, np.zeros_like(u))[..., 0]
    assert got.tolist() == [0, 0, 0, 0, 0, 1, 3, 3, 3]
    dye = np.zeros((4, 4, 4), F32); dye[..., 3] = 1; dye[1, 2, 0] = np.nan
    frame = M.display(dye, 8, 8, 0, None, None, None, (0, 0, 0), O.BG_COLOR, 1.0, nearest=True)["target"]
    assert np.argwhere(np.isnan(frame[..., 0])).tolist() == [[2, 4], [2, 5], [3, 4], [3, 5]]
    assert CM.to_bytes(frame).shape == frame.shape
