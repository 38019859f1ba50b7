"""render() with every display keyword set (updateKeywords, S:1160-1166) on the GPU: fluid_render_keywords
against the CPU model over the oracle (display_model.py) and the executed reference shaders,
the passes it launches, the reuse of its post-FX targets across frames, and what it refuses."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits_equal, golden, max_rel
from display_harness import BACK_RGB, FXCFG, check_frame, make, model_frame, seeded_dye, set_keywords
from display_harness import dither  # noqa: F401 -- a fixture
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("Wd,Hd,w,h", [(64, 64, 128, 128), (48, 32, 50, 75)])
def test_every_keyword_set_and_background_vs_oracle(pkg, oracle, dither, Wd, Hd, w, h):
    """All eight keyword sets x the three backgrounds (BACK_COLOR, TRANSPARENT on the screen, TRANSPARENT
    into a capture target), on a power-of-two and a ragged geometry; dye.read is never modified."""
    dye = seeded_dye(Wd, Hd, Wd + w)
    s = make(pkg, Wd, Hd, w, h)
    s.writeField("dye", dye)
    s.dithering = dither
    for kw in range(8):
        set_keywords(s, kw)
        for bg, transparent, target in ((oracle.BG_COLOR, False, False), (oracle.BG_CHECKERBOARD, True, False),
                                        (oracle.BG_NONE, True, True)):
            s.config["TRANSPARENT"] = transparent
            got = s.render(w, h, target=target)
            check_frame(s, got, model_frame("fp32", dye, w, h, kw, dither, FXCFG, bg), kw, (kw, bg))
            assert bits_equal(s.readField("dye"), dye), (kw, bg)
    s.close()


@pytest.mark.parametrize("name", ["keywords_bloom_64_to_128", "keywords_sunrays_64_to_128", "keywords_bloom_sunrays_64_to_128",
                                  "keywords_shading_bloom_64_to_128", "keywords_shading_sunrays_64_to_128",
                                  "keywords_48x32_to_50x75", "keywords_transparent_64x32_to_128x64"])
def test_keyword_sets_vs_executed_shaders(pkg, name):
    """Straight against the executed reference shaders, within the golden tolerance of
    test_render_postfx_vs_oracle_and_executed_shaders."""
    g = golden(name)
    Wd, Hd, w, h = (int(g[k]) for k in ("Wd", "Hd", "w", "h"))
    s = make(pkg, Wd, Hd, w, h)
    s.config.update(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]))
    s.writeField("dye", g["in_dye"])
    s.dithering = g["dither"].astype(np.float32)
    modes = [("checker", True, False), ("bare", True, True)] if "transparent" in name else [("target", False, False)]
    for tag in (str(t) for t in g["sets"]):
        s.config.update(SHADING="shading" in tag, BLOOM="bloom" in tag, SUNRAYS="sunrays" in tag)
        for key, transparent, target in modes:
            s.config["TRANSPARENT"] = transparent
            got = s.render(w, h, target=target)
            assert max_rel(got, g[f"{tag}_{key}"]) < 3e-4, (tag, key)
    s.close()


@pytest.mark.parametrize("iterations,levels", [(8, 5), (1, 1)])
def test_only_enabled_passes_launch(pkg, dither, iterations, levels):
    """Steady state (second call at the same sizes): one display blit, + 4 with SUNRAYS (mask, march,
    two blur passes), + 2L + 1 with BLOOM and a pyramid of L >= 2 levels (prefilter, L down, L - 1 up,
    final) -- the reference's blit count for the set.  A 64^2 bloom FBO has 5 levels of >= 2 texels."""
    s = make(pkg, 64, 64, 128, 128)
    s.writeField("dye", seeded_dye(64, 64, 5))
    s.dithering = dither
    s.config["BLOOM_ITERATIONS"] = iterations
    for kw in range(8):
        set_keywords(s, kw)
        s.render(128, 128)
        n0 = s.launch_count()
        s.render(128, 128)
        want = 1 + (4 if kw & pkg.DISPLAY_SUNRAYS else 0) + (2 * levels + 1 if kw & pkg.DISPLAY_BLOOM and levels >= 2 else 0)
        assert s.launch_count() - n0 == want, (kw, iterations)
    s.close()


def test_post_fx_targets_are_reused_and_remade_on_resize(pkg, oracle, dither):
    """The handle keeps its bloom / sunrays / dithering targets across frames and makes them again when a
    size changes: w1 x h1, then w2 x h2 with another BLOOM_RESOLUTION and BLOOM_ITERATIONS, then w1 x h1
    again, then w1 x h1 with a pyramid too short to run (the bloom FBO must read as freshly cleared)."""
    dye = seeded_dye(64, 48, 9)
    s = make(pkg, 64, 48, 128, 96)
    s.writeField("dye", dye)
    s.dithering = dither
    kw = pkg.DISPLAY_SHADING | pkg.DISPLAY_BLOOM | pkg.DISPLAY_SUNRAYS
    set_keywords(s, kw)
    frames = [(128, 96, dict(BLOOM_RESOLUTION=64, BLOOM_ITERATIONS=8, SUNRAYS_RESOLUTION=48)),
              (90, 160, dict(BLOOM_RESOLUTION=40, BLOOM_ITERATIONS=3, SUNRAYS_RESOLUTION=30)),
              (128, 96, dict(BLOOM_RESOLUTION=64, BLOOM_ITERATIONS=8, SUNRAYS_RESOLUTION=48)),
              (128, 96, dict(BLOOM_RESOLUTION=64, BLOOM_ITERATIONS=1, SUNRAYS_RESOLUTION=48))]
    for w, h, fx in frames:
        s.config.update(fx)
        s.canvas = {"width": w, "height": h}
        got = s.render(w, h)
        check_frame(s, got, model_frame("fp32", dye, w, h, kw, dither, fx, oracle.BG_COLOR), kw, (w, h))
    assert np.all(s.last_bloom == np.array([0, 0, 0, 1], np.float32))
    s.close()


def test_half_storage_refuses_post_fx_and_draws_shading(pkg, oracle, dither):
    """A half-storage handle refuses BLOOM or SUNRAYS (FLUID_ERR_INVALID), stays usable, and draws the
    SHADING-only set exactly as fluid_render does.  Unknown keyword bits are refused too."""
    s = make(pkg, 64, 64, 64, 64, flags=pkg.FLAG_HALF_STORAGE)
    s.writeField("dye", oracle.round_half(seeded_dye(64, 64, 3)))
    s.dithering = dither
    for bloom, sunrays in ((True, False), (False, True), (True, True)):
        s.config.update(SHADING=True, BLOOM=bloom, SUNRAYS=sunrays)
        with pytest.raises(pkg.FluidError) as e:
            s.render(64, 64)
        assert e.value.code == -1 and "HALF_STORAGE" in str(e.value)
    s.config.update(SHADING=True, BLOOM=False, SUNRAYS=False)
    got = s.render(64, 64)
    want = np.empty((64, 64, 4), np.float32)
    assert s._L.fluid_render(s._h, 64, 64, 1, *BACK_RGB, want.ctypes.data_as(C.c_void_p), want.size) == 0
    assert bits_equal(got, want)
    assert s._L.fluid_render_keywords(s._h, 64, 64, 8, None, None, 0, 0, *BACK_RGB, want.ctypes.data_as(C.c_void_p),
                                      want.size, None, None) == -1
    s.close()


@pytest.mark.parametrize("entry", ["fluid_render", "fluid_render_keywords", "fluid_render_postfx"])
def test_refusals_leave_the_handle_usable(pkg, dither, entry):
    """Every bad argument gets FLUID_ERR_INVALID, and the next good call on the same handle draws the same
    bits as the first one.  fluid_render has no keywords, fluid_render_postfx no keyword mask."""
    s = make(pkg, 64, 64, 128, 128)
    s.writeField("dye", seeded_dye(64, 64, 7))
    s.dithering = dither
    all3 = pkg.DISPLAY_SHADING | pkg.DISPLAY_BLOOM | pkg.DISPLAY_SUNRAYS
    set_keywords(s, all3)
    _, fx, dith = pkg.postfx_inputs(s.config, dither)
    out = np.empty((128, 128, 4), np.float32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)        # noqa: E731
    L = s._L

    def call(w=128, h=128, kw=all3, fx_=C.byref(fx), d=ptr(dith), dw=dith.shape[1], n=out.size, dst=ptr(out)):
        if entry == "fluid_render":
            return L.fluid_render(s._h, w, h, 1, *BACK_RGB, dst, n)
        if entry == "fluid_render_keywords":
            return L.fluid_render_keywords(s._h, w, h, kw, fx_, d, dw, dith.shape[0], *BACK_RGB, dst, n, None, None)
        return L.fluid_render_postfx(s._h, w, h, fx_, d, dw, dith.shape[0], *BACK_RGB, dst, n, None, None)

    assert call() == 0
    good = out.copy()
    bad = [dict(n=out.size - 1), dict(n=out.size + 1), dict(w=0), dict(h=0), dict(dst=None)]
    if entry != "fluid_render":
        bad += [dict(kw=pkg.DISPLAY_BLOOM, d=None), dict(kw=pkg.DISPLAY_BLOOM, dw=0),
                dict(kw=pkg.DISPLAY_BLOOM, fx_=None), dict(kw=pkg.DISPLAY_SUNRAYS, fx_=None)]
    if entry == "fluid_render_keywords":
        bad += [dict(kw=8), dict(kw=all3 | 0x10)]
    for b in bad:
        assert call(**b) == -1, b
        out[...] = np.nan
        assert call() == 0, b
        assert bits_equal(out, good), b
    s.close()
