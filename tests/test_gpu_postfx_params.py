"""The post-FX sliders BLOOM_INTENSITY / BLOOM_THRESHOLD / BLOOM_SOFT_KNEE / SUNRAYS_WEIGHT on the GPU: every
parameter set of display_harness.SETS on every handle kind that draws post-FX (fp32, fp32 + HALF_POSTFX,
HALF_STORAGE | HALF_POSTFX, NEAREST_FILTERING, NEAREST_FILTERING | HALF_STORAGE | HALF_POSTFX) with BLOOM,
SUNRAYS, BLOOM + SUNRAYS and SHADING + BLOOM + SUNRAYS: the bloom FBO and sunrays texture bit for bit against
the matching model (display_model), the frame inside its powf interval (bit for bit without BLOOM), captures and canvases
against their models; sliders changed between frames on one handle; the executed reference shaders."""
import numpy as np
import pytest

import canvas_model as CV
import display_model as M
import gamma_model as G
from conftest import golden, max_rel
from display_harness import (BACK_RGB, DEFAULTS, FIXTURES, GEOMETRIES, KEYS, SETS, cfg_of, check_capture, check_frame,
                             fixture_cfg, flags_of, golden_dither, make, model_capture, model_frame, params_dye,
                             set_keywords, stored)
from sim_harness import pkg, torch  # noqa: F401 -- fixtures

pytestmark = pytest.mark.gpu
F32 = np.float32
HANDLES = ["fp32", "fp32_half_postfx", "half_half_postfx", "nearest_fp32", "nearest_half_half_postfx"]
KEYWORD_SETS = [M.BLOOM, M.SUNRAYS, M.BLOOM | M.SUNRAYS, M.ALL3]


def handle_for(pkg, handle, geometry, cfg):
    """A handle of kind `handle` on `geometry` holding the parameter dye, and the dye as it holds it."""
    Wd, Hd, w, h = GEOMETRIES[geometry][:4]
    s = make(pkg, Wd, Hd, w, h, flags_of(pkg, handle), **cfg)
    dye = params_dye(Wd, Hd)
    s.writeField("dye", dye)
    s.dithering = golden_dither()
    return s, stored(handle, dye)


@pytest.mark.parametrize("name", list(SETS))
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("handle", HANDLES)
def test_set_on_every_handle_kind(pkg, oracle, torch, handle, geometry, name):
    """The four keyword sets: the frame over BACK_COLOR and bare (render(target=True) with TRANSPARENT), the
    capture over BACK_COLOR and bare, and the canvas over BACK_COLOR and the checkerboard, into host and device
    memory, against canvas_model applied to the handle's bare fragment."""
    cfg = cfg_of(name, geometry)
    w, h = GEOMETRIES[geometry][2:4]
    tw, th = M.get_resolution(cfg["CAPTURE_RESOLUTION"], w, h)            # the capture target
    s, dye = handle_for(pkg, handle, geometry, cfg)
    dev = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for kw in KEYWORD_SETS:
            set_keywords(s, kw)
            for transparent in (False, True):
                what = (handle, geometry, name, kw, transparent)
                s.config["TRANSPARENT"] = transparent
                frame = s.render(w, h, target=transparent)
                want = model_frame(handle, dye, w, h, kw, golden_dither(), cfg,
                                   oracle.BG_NONE if transparent else oracle.BG_COLOR)
                check_frame(s, frame, want, kw, what)
                got = s.captureScreenshot()
                check_capture(got, model_capture(handle, dye, tw, th, w, h, kw, golden_dither(), cfg, transparent), kw, what)
                if transparent:
                    bare = frame
            for transparent in (False, True):
                s.config["TRANSPARENT"] = transparent
                want = CV.canvas(bare, BACK_RGB, transparent, w / h)
                assert np.array_equal(s.render_canvas(), want), (handle, geometry, name, kw, transparent)
                s.render_canvas(out=dev)
                assert np.array_equal(dev.cpu().numpy(), want), (handle, geometry, name, kw, transparent, "device")
            assert G.same_bits(s.readField("dye"), dye)
    s.close()


def outputs(s, torch, w, h):
    """Everything one frame of the handle shows with the sliders its config holds now."""
    dev = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    s.config["TRANSPARENT"] = False
    frame = s.render(w, h)
    bloom, sun = s.last_bloom.copy(), s.last_sunrays.copy()
    s.config["TRANSPARENT"] = True
    bare = s.render(w, h, target=True)
    cap = s.captureScreenshot()
    host = s.render_canvas()
    s.render_canvas(out=dev)
    s.config["TRANSPARENT"] = False
    return dict(frame=frame, bare=bare, bloom=bloom, sunrays=sun, capture=cap, canvas=host, device=dev.cpu().numpy())


def same(a, b):
    return all(G.same_bits(a[k], b[k]) if a[k].dtype == F32 else np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize("handle", HANDLES)
def test_sliders_changed_between_frames(pkg, oracle, torch, handle):
    """One handle driven through s.config: sets A, B, A, then the defaults, all three keywords.  Every output of
    each frame equals, bit for bit, a fresh handle's with that set on the same dye; postfx_inputs hands the
    library what the config holds."""
    geometry = "pow2"
    w, h = GEOMETRIES[geometry][2:4]
    base = cfg_of("t1_k0_i2_w03", geometry)
    s, _ = handle_for(pkg, handle, geometry, base)
    set_keywords(s, M.ALL3)
    seen = []
    with np.errstate(invalid="ignore", over="ignore"):
        for name in ("t1_k0_i2_w03", "t039_k1", "t1_k0_i2_w03", None):
            sliders = DEFAULTS if name is None else cfg_of(name, geometry)
            for k in KEYS:
                s.config[k] = sliders[k]
            fx = pkg.postfx_inputs(s.config, golden_dither())[1]
            assert (fx.bloom_intensity, fx.bloom_threshold, fx.bloom_soft_knee, fx.sunrays_weight) == \
                tuple(float(sliders[k]) for k in KEYS)
            got = outputs(s, torch, w, h)
            fresh, _ = handle_for(pkg, handle, geometry, dict(base, **{k: sliders[k] for k in KEYS}))
            set_keywords(fresh, M.ALL3)
            assert same(got, outputs(fresh, torch, w, h)), (handle, name)
            fresh.close()
            seen.append(got)
    s.close()
    assert same(seen[0], seen[2]) and not same(seen[0], seen[1]) and not same(seen[1], seen[3])


@pytest.mark.parametrize("name", FIXTURES)
def test_vs_executed_shaders(pkg, name):
    """The executed reference shaders with the fixture's sliders on an fp32 handle: bloom FBO and sunrays bit
    for bit, the frame within the keyword goldens' 3e-4 (test_gpu_display_keywords.py)."""
    g = golden(name)
    Wd, Hd, w, h = (int(g[k]) for k in ("Wd", "Hd", "w", "h"))
    s = make(pkg, Wd, Hd, w, h, 0, **fixture_cfg(g))
    s.writeField("dye", g["in_dye"])
    s.dithering = g["dither"].astype(F32)
    set_keywords(s, M.ALL3)
    got = s.render(w, h)
    assert G.same_bits(s.last_bloom, g["bloom"]) and G.same_bits(s.last_sunrays, g["sunrays"])
    assert max_rel(got, g["target"]) < 3e-4
    s.close()
