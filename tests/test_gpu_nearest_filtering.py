"""FLUID_FLAG_NEAREST_FILTERING on the GPU: display, post-FX chains, captures and resize through NEAREST
samplers, against display_model.py's NEAREST sampler with the library's vUv (bit for bit; BLOOM frames inside gamma_model's
powf interval after the bloom FBO and sunrays texture matched bit for bit) and against the executed
NEAREST shaders; non-finite dye; a simulation that does not change by one bit or one launch; refusals.
No comparison uses a value tolerance for a NEAREST fetch."""
import ctypes as C

import numpy as np
import pytest

import display_model as M
import gamma_model as G
from conftest import golden
from display_harness import (BACK_RGB, BACKGROUNDS, MODES, allowed, check_capture, draw_all, flags_of, golden_dither,
                             make, model_capture, nonfinite_dye, seeded_dye, set_keywords)
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu
F32 = np.float32
HANDLES = ["fp32", "fp32_half_postfx", "half", "half_half_postfx"]
ALL3 = M.ALL3


def kind(handle):
    """The display_harness kind of a handle with FLUID_FLAG_NEAREST_FILTERING."""
    return "nearest_" + handle


@pytest.mark.parametrize("handle", HANDLES)
@pytest.mark.parametrize("Wd,Hd,w,h", [(64, 64, 128, 128), (48, 32, 50, 75)])
def test_every_keyword_set_and_background(pkg, oracle, handle, Wd, Hd, w, h):
    draw_all(pkg, kind(handle), seeded_dye(Wd, Hd, Wd + w), w, h, golden_dither())


@pytest.mark.parametrize("handle", HANDLES)
def test_minification(pkg, oracle, handle):
    """A 1024^2 dye drawn on a 300 x 200 canvas."""
    draw_all(pkg, kind(handle), seeded_dye(1024, 1024, 300), 300, 200, golden_dither(), modes=["back", "bare"])


@pytest.mark.parametrize("handle", ["fp32", "half_half_postfx"])
def test_the_profiles_own_frame(pkg, oracle, handle):
    """getResolution(512) of 1920 x 1080 (910 x 512) drawn at 1920 x 1080 with all three keywords and the
    reference's BLOOM / SUNRAYS resolutions: HALF_STORAGE | HALF_POSTFX | NEAREST is a WebGL2 device without
    OES_texture_float_linear."""
    import webgl_fluid_simulation_b200 as p
    assert (p.getResolution(512, 1920, 1080)["width"], p.getResolution(512, 1920, 1080)["height"]) == (910, 512)
    draw_all(pkg, kind(handle), seeded_dye(910, 512, 1080), 1920, 1080, golden_dither(),
             cfg=dict(BLOOM_RESOLUTION=256, SUNRAYS_RESOLUTION=196), sets=[ALL3], modes=["back"])


@pytest.mark.parametrize("handle", HANDLES)
def test_nonfinite_dye_every_set(pkg, oracle, handle):
    """+-inf and NaN in dye: bit for bit without BLOOM (NaN in the model's texels only: NEAREST reads one
    texel, so a NaN does not reach its neighbours), inside the interval with it."""
    draw_all(pkg, kind(handle), nonfinite_dye(64, 64, 8), 128, 128, golden_dither())


def test_nan_stays_in_its_own_texels(pkg):
    dye = np.zeros((16, 16, 4), F32); dye[..., 3] = 1; dye[5, 7, :3] = np.nan
    s = make(pkg, 16, 16, 64, 64, pkg.FLAG_NEAREST_FILTERING)
    s.writeField("dye", dye)
    set_keywords(s, 0)
    got = s.render(64, 64)
    assert sorted(map(tuple, np.argwhere(np.isnan(got[..., 0])).tolist())) == [(j, i) for j in range(20, 24) for i in range(28, 32)]
    s.close()


@pytest.mark.parametrize("name", ["nearest_64_to_128_plain", "nearest_64_to_128_bloom", "nearest_half_64_to_128_plain",
                                  "nearest_half_64_to_128_bloom", "nearest_transparent_64x32_to_128x64"])
def test_vs_executed_nearest_shaders(pkg, name):
    """The executed shaders at power-of-two sizes: chains and frames without BLOOM bit for bit, BLOOM frames
    inside the interval."""
    g = golden(name)
    Wd, Hd, w, h = (int(g[k]) for k in ("Wd", "Hd", "w", "h"))
    half = bool(g["half"])
    flags = pkg.FLAG_NEAREST_FILTERING | ((pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX) if half else 0)
    s = make(pkg, Wd, Hd, w, h, flags, BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]))
    s.writeField("dye", g["in_dye"])
    dither = g["dither"].astype(F32)
    s.dithering = dither
    keys = {"target": "back", "checker": "checker", "bare": "bare"}
    for tag in (str(t) for t in g["sets"]):
        kw = M.SETS[tag]
        set_keywords(s, kw)
        for key, bg in keys.items():
            if f"{tag}_{key}" not in g:
                continue
            s.config["TRANSPARENT"] = MODES[bg][0]
            got = s.render(w, h, target=MODES[bg][1])
            for k, tex in (("bloom", s.last_bloom), ("sunrays", s.last_sunrays)):
                if tex is not None:
                    assert G.same_bits(tex, g[k]), (tag, k)
            if kw & M.BLOOM:
                d = M.display(g["in_dye"], w, h, kw, g["bloom"], g["sunrays"] if kw & M.SUNRAYS else None, dither,
                              BACK_RGB, BACKGROUNDS[bg], w / h, nearest=True)
                n, bad = G.check_display(got, d["lo"], d["hi"])
                assert n == 0 and G.check_display(g[f"{tag}_{key}"], d["lo"], d["hi"])[0] == 0, (tag, key, bad)
            else:
                assert G.same_bits(got, g[f"{tag}_{key}"]), (tag, key)
    s.close()


@pytest.mark.parametrize("handle", HANDLES)
@pytest.mark.parametrize("bg", ["back", "transparent"])
def test_captures(pkg, handle, bg):
    """The capture fixture's dye on every handle kind: bytes equal to the model without BLOOM (and, on the
    fp32 handle, to the executed shaders), inside the byte bracket with it."""
    g = golden(f"nearest_capture_64_canvas_128_{bg}")
    dye_in, w, h, cw, ch = g["in_dye"], int(g["w"]), int(g["h"]), int(g["canvas_w"]), int(g["canvas_h"])
    cfg = dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]))
    dither, transparent = g["dither"].astype(F32), bool(g["transparent"])
    s = make(pkg, 64, 64, cw, ch, flags_of(pkg, kind(handle)), CAPTURE_RESOLUTION=int(g["capture_res"]),
             TRANSPARENT=transparent, **cfg)
    s.writeField("dye", dye_in)
    s.dithering = dither
    dye = s.readField("dye")                           # fp16-rounded on a half-storage handle
    for tag in (str(t) for t in g["sets"]):
        kw = M.SETS[tag]
        if not allowed(kind(handle), kw):
            continue
        set_keywords(s, kw)
        got = s.captureScreenshot()
        check_capture(got, model_capture(kind(handle), dye, w, h, cw, ch, kw, dither, cfg, transparent), kw, (tag, handle))
        if handle == "fp32" and not kw & M.BLOOM:
            assert np.array_equal(got, g[f"{tag}_rgba8"]), tag
    s.close()


@pytest.mark.parametrize("half", [False, True])
def test_resize_copies_through_nearest(pkg, oracle, half):
    """fluid_resize up, down and ragged: velocity and dye are the model's NEAREST copy, rounded to fp16 on a
    half-storage handle; a field whose size did not change is kept bit for bit."""
    flags = pkg.FLAG_NEAREST_FILTERING | (pkg.FLAG_HALF_STORAGE if half else 0)
    s = make(pkg, 64, 64, 128, 128, flags)
    s._sizes = (32, 32, 64, 64); s.initFramebuffers()
    rng = np.random.default_rng(3)
    s.writeField("velocity", (rng.standard_normal((32, 32, 2)) * 50).astype(F32))
    s.writeField("dye", seeded_dye(64, 64, 4))
    for sizes in [(48, 48, 128, 96), (20, 30, 40, 28), (20, 30, 97, 51), (20, 30, 32, 32), (64, 16, 32, 32)]:
        v0, d0 = s.readField("velocity"), s.readField("dye")
        s._sizes = sizes; s.initFramebuffers()
        v1, d1 = s.readField("velocity"), s.readField("dye")
        Wv, Hv, Wd, Hd = sizes
        for old, new, W, H in ((v0, v1, Wv, Hv), (d0, d1, Wd, Hd)):
            if old.shape[:2] == (H, W):
                assert G.same_bits(new, old), sizes
            else:
                assert G.same_bits(new, M.resize(old, W, H, half=half)), sizes
    s.close()


def test_simulation_is_unchanged(pkg):
    """The same seeded session on a flagged and an unflagged handle (graph and FLAG_NO_GRAPH): every field bit
    for bit after every call, and the launch, Jacobi and graph counters equal."""
    fields = ("velocity", "dye", "pressure", "divergence", "curl")
    stats = ("launches", "jacobi_launches", "graph_captures", "graph_launches", "cvd_stream_launches",
             "gradient_stream_launches")
    for extra in (0, pkg.FLAG_NO_GRAPH, pkg.FLAG_HALF_STORAGE):
        sims = [pkg.FluidSimulation({"SIM_RESOLUTION": 64, "DYE_RESOLUTION": 128}, 256, 256, flags=extra | f,
                                    random=np.random.RandomState(11).random_sample) for f in (0, pkg.FLAG_NEAREST_FILTERING)]
        for s in sims:
            s.config.update(SHADING=True, DYE_RESOLUTION=128)
        rng = np.random.default_rng(5)
        d = rng.standard_normal((64, 64)).astype(F32)
        p = rng.standard_normal((64, 64)).astype(F32)
        rec = np.column_stack([rng.random((6, 2)), rng.standard_normal((6, 2)) * 500, rng.random((6, 3))]).astype(F32)
        calls = [lambda s: s.multipleSplats(3), lambda s: s.splat(0.3, 0.6, 120.0, -80.0, (0.2, 0.5, 0.9)),
                 lambda s: s.splats(rec), lambda s: s.step(0.016), lambda s: s.step(0.016),
                 lambda s: s.pressure_solve_host(d.copy(), p.copy(), 20), lambda s: s.pass_("pressure_solve"),
                 lambda s: s.step(0.01)]
        for k, call in enumerate(calls):
            for s in sims:
                call(s)
            for f in fields:
                assert G.same_bits(sims[0].readField(f), sims[1].readField(f)), (extra, k, f)
            assert [sims[0].stat(x) for x in stats] == [sims[1].stat(x) for x in stats], (extra, k)
        for s in sims:
            s.close()


@pytest.mark.parametrize("handle", ["fp32", "half_half_postfx"])
def test_frame_launches_equal_the_linear_frame(pkg, handle):
    linear_flags = flags_of(pkg, handle)
    counts = []
    for flags in (flags_of(pkg, kind(handle)), linear_flags):
        s = make(pkg, 64, 64, 128, 128, flags, CAPTURE_RESOLUTION=64)
        s.writeField("dye", seeded_dye(64, 64, 5))
        s.dithering = golden_dither()
        row = []
        for kw in range(8):
            set_keywords(s, kw)
            for call in (lambda: s.render(128, 128), s.captureScreenshot):
                call()
                n0 = s.launch_count()
                call()
                row.append(s.launch_count() - n0)
        counts.append(row)
        s.close()
    assert counts[0] == counts[1]


def test_half_storage_without_half_postfx_still_refuses_bloom(pkg):
    s = make(pkg, 64, 64, 64, 64, pkg.FLAG_HALF_STORAGE | pkg.FLAG_NEAREST_FILTERING)
    s.config.update(BLOOM=True, SUNRAYS=False)
    s.dithering = golden_dither()
    with pytest.raises(pkg.FluidError) as e:
        s.render(64, 64)
    assert e.value.code == -1 and "HALF_POSTFX" in str(e.value)
    s.close()


def test_slab_with_the_flag_is_refused(pkg):
    L = pkg.lib()
    cfg = pkg._lib.Config()
    L.fluid_config_default(C.byref(cfg))
    cfg.sim_w, cfg.sim_h, cfg.dye_w, cfg.dye_h = 64, 64, 64, 64
    cfg.flags = pkg.FLAG_NEAREST_FILTERING
    h = C.c_void_p()
    uid = C.create_string_buffer(128)
    assert L.fluid_create_slab(C.byref(cfg), 0, 2, uid, 128, C.byref(h)) == -1
    assert not h.value
