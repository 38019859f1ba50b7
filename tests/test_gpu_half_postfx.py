"""FLUID_FLAG_HALF_POSTFX on the GPU: fp16 bloom FBO, pyramid, sunrays and sunraysTemp, on an fp32 handle
and on a half-storage handle (FLUID_FLAG_HALF_STORAGE | FLUID_FLAG_HALF_POSTFX: the reference's desktop
frame), against display_model with half_targets and the executed half-float
shaders; overflow and non-finite dye; captures; launches and target reuse; the slab refusal."""
import ctypes as C

import numpy as np
import pytest

import capture_model as CM
import display_model as M
import gamma_model as G
from conftest import golden, max_rel
from display_harness import (FXCFG, check_capture, check_frame, draw_all, flags_of, golden_dither, make, model_capture,
                             model_frame, nonfinite_dye, seeded_dye, set_keywords, stored)
from oracle import oracle as O
from sim_harness import pkg  # noqa: F401 -- a fixture
from gamma_model import CAPTURE_SETS, FRAME_TOL, POW2, RAGGED, RAGGED_CHAIN_TEXELS, cfg_of, fp16_ulps

pytestmark = pytest.mark.gpu
F32 = np.float32
ALL3 = M.ALL3
HANDLES = ["fp32", "half"]


def kind(handle):
    """The display_harness kind of a handle with FLUID_FLAG_HALF_POSTFX."""
    return handle + "_half_postfx"


@pytest.mark.parametrize("handle", HANDLES)
@pytest.mark.parametrize("Wd,Hd,w,h", [(64, 64, 128, 128), (48, 32, 50, 75)])
def test_every_keyword_set_and_background(pkg, oracle, handle, Wd, Hd, w, h):
    """All eight sets x the three backgrounds; dye.read is unchanged afterwards."""
    draw_all(pkg, kind(handle), seeded_dye(Wd, Hd, Wd + w), w, h, golden_dither())


@pytest.mark.parametrize("name", [POW2, RAGGED])
def test_vs_executed_half_float_shaders(pkg, name):
    """The desktop storage against the executed shaders: chains bit for bit on the power-of-two fixture and
    within the measured ragged bound (test_half_postfx_cpu.py) on the other; frames within FRAME_TOL."""
    g = golden(name)
    Wd, Hd, w, h = (int(g[k]) for k in ("Wd", "Hd", "w", "h"))
    s = make(pkg, Wd, Hd, w, h, flags_of(pkg, "half_half_postfx"), **cfg_of(g))
    s.writeField("dye", g["in_dye"])
    s.dithering = g["dither"].astype(F32)
    for tag in (str(t) for t in g["sets"]):
        s.config.update(SHADING="shading" in tag, BLOOM="bloom" in tag, SUNRAYS="sunrays" in tag)
        got = s.render(w, h)
        for key, tex in (("bloom", s.last_bloom), ("sunrays", s.last_sunrays)):
            if tex is None:
                continue
            if name == POW2:
                assert G.same_bits(tex, g[key]), (tag, key)
            else:
                assert np.count_nonzero(tex != g[key]) <= RAGGED_CHAIN_TEXELS[key] and fp16_ulps(tex, g[key]) <= 1, (tag, key)
        assert max_rel(got, g[f"{tag}_target"]) < FRAME_TOL, tag
    s.close()


def test_bloom_overflow_goes_to_inf_where_the_model_does(pkg, oracle):
    """fp32 dye whose prefiltered bloom exceeds 65504: the fp16 bloom FBO holds +inf in exactly the model's
    texels, and the frames stay inside the interval (inf exactly)."""
    dye = seeded_dye(64, 64, 77)
    dye[20:24, 30:34, 0] = 2.0e5
    dye[40, 10, 1] = 1.0e6
    ref = M.chains(dye, 128, 128, M.BLOOM, FXCFG, half_targets=True)
    assert np.isinf(ref["bloom"]).any() and not np.isinf(dye).any()
    draw_all(pkg, "fp32_half_postfx", dye, 128, 128, golden_dither(), sets=[M.BLOOM, ALL3], modes=["back", "bare"])


@pytest.mark.parametrize("handle", HANDLES)
def test_nonfinite_dye_every_set(pkg, oracle, handle):
    """The non-finite dye of test_gamma_model_cpu.py through all eight sets and backgrounds: bit for bit
    without BLOOM (NaN in the same places), inside the interval with it."""
    draw_all(pkg, kind(handle), nonfinite_dye(64, 64, 8), 128, 128, golden_dither())


@pytest.mark.parametrize("bg", ["back", "transparent"])
def test_half_storage_captures(pkg, oracle, bg):
    """The executed-shader capture fixture on a half-storage handle with the flag, all eight sets: with BLOOM
    every byte within [B(lo), B(hi)] of the half_targets interval, without it the model's (= the
    executed) bytes exactly; every byte within the byte rule at FRAME_TOL of the model; and each capture equals the quantised
    render(target=True) frame of a canvas-sized copy where canvas = target."""
    g = golden(f"capture_half_64_canvas_128_{bg}")
    dye, w, h, cw, ch = g["in_dye"], int(g["w"]), int(g["h"]), int(g["canvas_w"]), int(g["canvas_h"])
    cfg, dither, transparent = cfg_of(g), g["dither"].astype(F32), bool(g["transparent"])
    s = make(pkg, dye.shape[1], dye.shape[0], cw, ch, flags_of(pkg, "half_half_postfx"),
             CAPTURE_RESOLUTION=int(g["capture_res"]), TRANSPARENT=transparent, **cfg)
    s.writeField("dye", dye)
    s.dithering = dither
    for kw, tag in enumerate(CAPTURE_SETS):
        set_keywords(s, kw)
        got = s.captureScreenshot()
        model = model_capture("half_half_postfx", dye, w, h, cw, ch, kw, dither, cfg, transparent)
        check_capture(got, model, kw, tag)
        assert CM.bytes_outside(got, model["pre"], FRAME_TOL) == 0, tag
        if not kw & M.BLOOM:                          # the model's bytes are the executed ones (CPU test)
            assert np.array_equal(got, g[f"{tag}_rgba8"]), tag
    s.close()
    # canvas = target: capture == flip(B(render frame))
    s = make(pkg, 64, 64, 64, 64, flags_of(pkg, "half_half_postfx"), CAPTURE_RESOLUTION=64, BLOOM_RESOLUTION=32,
             SUNRAYS_RESOLUTION=24)
    s.config["BACK_COLOR"] = {"r": 0, "g": 0, "b": 0}
    s.writeField("dye", dye)
    s.dithering = dither
    for kw in range(8):
        set_keywords(s, kw)
        s.config["TRANSPARENT"] = transparent
        frame = s.render(64, 64, target=True)
        assert np.array_equal(s.captureScreenshot(), CM.to_bytes(frame)[::-1]), kw
    s.close()


@pytest.mark.parametrize("handle", HANDLES)
@pytest.mark.parametrize("iterations,levels", [(8, 5), (1, 1)])
def test_launches(pkg, handle, iterations, levels):
    """Steady state: 1 display, + 4 with SUNRAYS, + 2L + 1 with BLOOM and L >= 2, and on a half-storage handle
    the one dye widen of the display source; a capture launches what render() does."""
    s = make(pkg, 64, 64, 128, 128, flags_of(pkg, kind(handle)), CAPTURE_RESOLUTION=64, BLOOM_ITERATIONS=iterations)
    s.writeField("dye", seeded_dye(64, 64, 5))
    s.dithering = golden_dither()
    for kw in range(8):
        set_keywords(s, kw)
        want = (1 + (4 if kw & M.SUNRAYS else 0) + (2 * levels + 1 if kw & M.BLOOM and levels >= 2 else 0)
                + (1 if handle == "half" else 0))
        for call in (lambda: s.render(128, 128), s.captureScreenshot):
            call()
            n0 = s.launch_count()
            call()
            assert s.launch_count() - n0 == want, (kw, iterations, handle)
    s.close()


@pytest.mark.parametrize("handle", HANDLES)
def test_targets_reused_and_remade_on_resize(pkg, oracle, handle):
    """w1 x h1, then w2 x h2 with another BLOOM_RESOLUTION and BLOOM_ITERATIONS, then w1 x h1 again, then a
    pyramid too short to run (the fp16 bloom FBO reads as freshly cleared: (0, 0, 0, 1))."""
    dye_in = seeded_dye(64, 48, 9)
    s = make(pkg, 64, 48, 128, 96, flags_of(pkg, kind(handle)))
    s.writeField("dye", dye_in)
    s.dithering = golden_dither()
    dye = stored(kind(handle), dye_in)
    set_keywords(s, ALL3)
    frames = [(128, 96, dict(BLOOM_RESOLUTION=64, BLOOM_ITERATIONS=8, SUNRAYS_RESOLUTION=48)),
              (90, 160, dict(BLOOM_RESOLUTION=40, BLOOM_ITERATIONS=3, SUNRAYS_RESOLUTION=30)),
              (128, 96, dict(BLOOM_RESOLUTION=64, BLOOM_ITERATIONS=8, SUNRAYS_RESOLUTION=48)),
              (128, 96, dict(BLOOM_RESOLUTION=64, BLOOM_ITERATIONS=1, SUNRAYS_RESOLUTION=48))]
    for w, h, fx in frames:
        s.config.update(fx)
        s.canvas = {"width": w, "height": h}
        got = s.render(w, h)
        check_frame(s, got, model_frame(kind(handle), dye, w, h, ALL3, golden_dither(), dict(FXCFG, **fx), O.BG_COLOR),
                    ALL3, (handle, w, h))
    assert np.all(s.last_bloom == np.array([0, 0, 0, 1], F32))
    s.close()


def test_reference_size_frame_within_interval(pkg, oracle):
    """The reference's desktop frame: 1024^2 fp16 dye drawn to 1920 x 1080 with BLOOM_RESOLUTION 256 and
    SUNRAYS_RESOLUTION 196, all three keywords."""
    draw_all(pkg, "half_half_postfx", seeded_dye(1024, 1024, 1920), 1920, 1080, golden_dither(),
             cfg=dict(BLOOM_RESOLUTION=256, SUNRAYS_RESOLUTION=196), sets=[ALL3], modes=["back"])


def test_half_storage_without_the_flag_still_refuses(pkg, oracle):
    s = pkg.FluidSimulation({"SIM_RESOLUTION": 16, "DYE_RESOLUTION": 64}, canvas_width=64, canvas_height=64,
                            flags=pkg.FLAG_HALF_STORAGE, sizes=(16, 16, 64, 64))
    s.config.update(FXCFG, BLOOM=True, SUNRAYS=True)
    s.dithering = golden_dither()
    with pytest.raises(pkg.FluidError) as e:
        s.render(64, 64)
    assert e.value.code == -1 and "HALF_STORAGE" in str(e.value) and "HALF_POSTFX" in str(e.value)
    s.close()


def test_slab_with_the_flag_is_refused(pkg):
    """fluid_create_slab(world = 2) with FLUID_FLAG_HALF_POSTFX: FLUID_ERR_INVALID before any communicator."""
    L = pkg.lib()
    cfg = pkg._lib.Config()
    L.fluid_config_default(C.byref(cfg))
    cfg.sim_w, cfg.sim_h, cfg.dye_w, cfg.dye_h = 64, 64, 64, 64
    cfg.flags = pkg.FLAG_HALF_POSTFX
    h = C.c_void_p()
    uid = C.create_string_buffer(128)
    assert L.fluid_create_slab(C.byref(cfg), 0, 2, uid, 128, C.byref(h)) == -1
    assert not h.value
