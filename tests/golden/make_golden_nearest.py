"""Cuts the fixtures of FLUID_FLAG_NEAREST_FILTERING, the reference on a device without float linear
filtering (`!ext.supportLinearFiltering`, S:127-134): dye (S:990), the bloom FBO and pyramid (S:1017),
sunrays and sunraysTemp (S:1039) are NEAREST textures, the dithering texture stays LINEAR + REPEAT
(createTextureAsync S:1131-1134).  By EXECUTING the reference's GLSL text with oracle/glsl_exec.py.

    WEBGL_FLUID_REFERENCE=<checkout> python tests/golden/make_golden_nearest.py

The orchestration is that of make_golden_keywords.render(), make_golden_half_postfx.render_half() and
make_golden_capture.capture_render(), run unchanged while glsl_exec's Texture is created NEAREST
(Texture(..., linear=False)) unless it is REPEAT-wrapped.  Render targets become NEAREST too, which
changes nothing: a target is written, never sampled.  The dye is drawn as in those generators.

Writes only these files (the other fixtures are left as they are):
  nearest_64_to_128_{plain,bloom}.npz     fp32 dye and chains, power of two: the four sets without BLOOM,
                                          the four with it (two files keep each small; same dye in both)
  nearest_48x32_to_50x75.npz              all eight sets on a ragged dye and portrait canvas
  nearest_half_64_to_128_{plain,bloom}.npz   fp16 dye, half-float chains and mask (HALF_STORAGE | HALF_POSTFX)
  nearest_transparent_64x32_to_128x64.npz three sets over the checkerboard and bare (TRANSPARENT)
  nearest_capture_64_canvas_128_{back,transparent}.npz   all eight sets, 64^2 capture of a 128^2 canvas
"""
import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_capture as CAP  # noqa: E402
import make_golden_half_postfx as HP  # noqa: E402
import make_golden_keywords as K  # noqa: E402
from make_golden_keywords import G  # noqa: E402

BACK = CAP.BACK
SETS = CAP.SETS          # all eight: none, shading, bloom, shading_bloom, sunrays, shading_sunrays, bloom_sunrays, all three
PLAIN = tuple(t for t, kw in SETS.items() if "BLOOM" not in kw)
WITH_BLOOM = tuple(t for t, kw in SETS.items() if "BLOOM" in kw)


class _NearestTexture(G.Texture):
    """createFBO with `filtering` = NEAREST (S:1045-1077); REPEAT textures (the dithering) stay LINEAR."""

    def __init__(self, w, h, ch, linear, half=False, repeat=False):
        super().__init__(w, h, ch, linear and repeat, half, repeat)


@contextlib.contextmanager
def nearest_samplers():
    linear = G.Texture
    G.Texture = _NearestTexture
    try:
        yield
    finally:
        G.Texture = linear


def seeded_dye(Wd, Hd, seed, scale, half):
    """The generators' dye, rng ** 4 * scale with alpha 1, rounded to fp16 for a half-storage handle."""
    rng = np.random.default_rng(seed)
    dye = (rng.random((Hd, Wd, 4), dtype=np.float32) ** 4 * np.float32(scale)).astype(np.float32); dye[..., 3] = 1
    if half:
        dye = dye.astype(np.float16).astype(np.float32)
    s = G.GLSLSim(16, 16, Wd, Hd); s.load(dye=dye)
    return s, dye


def keyword_fixture(name, Wd, Hd, w, h, seed, sets=tuple(SETS), half=False, transparent=False, bloom_res=64, sun_res=48):
    """Each set of `sets` over BACK_COLOR (<set>_target), or over the checkerboard (<set>_checker) and bare
    (<set>_bare) with `transparent`; the chains once (they do not depend on the keywords)."""
    dither = K.dithering()
    s, dye = seeded_dye(Wd, Hd, seed, 3.0, half)
    cfg = dict(BLOOM_RESOLUTION=bloom_res, SUNRAYS_RESOLUTION=sun_res)
    o = dict(Wd=Wd, Hd=Hd, w=w, h=h, bloom_res=bloom_res, sun_res=sun_res, in_dye=dye, dither=dither.astype(np.float16),
             back=np.array(BACK, np.float32), sets=np.array(list(sets)), half=half)
    modes = [("checker", True, True), ("bare", True, False)] if transparent else [("target", False, True)]
    for tag in sets:
        for key, tr, scr in modes:
            with nearest_samplers():
                if half:
                    assert not transparent
                    r = HP.render_half(s, w, h, dither, cfg, SETS[tag])
                else:
                    r = K.render(s, w, h, dither, cfg, BACK, SETS[tag], tr, scr)
            o[f"{tag}_{key}"] = r["target"]
            for k in ("bloom", "sunrays", "mask_alpha"):
                if r[k] is not None:
                    assert k not in o or np.array_equal(o[k], r[k]), k
                    o[k] = r[k].astype(np.float32)
            for k, t in enumerate(r["pyramid"]):
                o[f"pyr{k}"] = t
    np.savez_compressed(os.path.join(K.OUT, name + ".npz"), **o)


def capture_fixture(name, Wd, Hd, canvas_w, canvas_h, capture_res, bloom_res, sun_res, seed):
    """make_golden_capture.capture_fixture through NEAREST samplers."""
    w, h = CAP.get_resolution(capture_res, canvas_w, canvas_h)
    dither = K.dithering()
    s, dye = seeded_dye(Wd, Hd, seed, 1.0, False)
    cfg = dict(BLOOM_RESOLUTION=bloom_res, SUNRAYS_RESOLUTION=sun_res)
    for bg, transparent in (("back", False), ("transparent", True)):
        o = dict(Wd=Wd, Hd=Hd, canvas_w=canvas_w, canvas_h=canvas_h, w=w, h=h, capture_res=capture_res,
                 bloom_res=bloom_res, sun_res=sun_res, in_dye=dye, dither=dither.astype(np.float16),
                 back=np.array(BACK, np.float32), transparent=transparent, sets=np.array(list(SETS)))
        for tag, kw in SETS.items():
            with nearest_samplers():
                t = CAP.capture_render(s, w, h, canvas_w, canvas_h, dither, cfg, kw, transparent)
            assert np.array_equal(t.astype(np.float16).astype(np.float32), t), (name, tag, bg)   # stored as fp16
            assert np.array_equal(s.dye.read.data, dye), (name, tag, bg)                           # dye.read untouched
            o[f"{tag}_half"] = t.astype(np.float16)
            o[f"{tag}_rgba8"] = CAP.normalize_texture(t.astype(np.float16))
        np.savez_compressed(os.path.join(K.OUT, f"{name}_{bg}.npz"), **o)


if __name__ == "__main__":
    K.check_against_postfx_fixtures()            # the shared orchestration still cuts the LINEAR fixtures
    CAP.check_self_consistency()
    for part, sets in (("plain", PLAIN), ("bloom", WITH_BLOOM)):
        keyword_fixture(f"nearest_64_to_128_{part}", 64, 64, 128, 128, 41, sets=sets)
        keyword_fixture(f"nearest_half_64_to_128_{part}", 64, 64, 128, 128, 43, sets=sets, half=True)
    keyword_fixture("nearest_48x32_to_50x75", 48, 32, 50, 75, 42)
    keyword_fixture("nearest_transparent_64x32_to_128x64", 64, 32, 128, 64, 44,
                    sets=("none", "shading", "shading_bloom_sunrays"), transparent=True)
    capture_fixture("nearest_capture_64_canvas_128", 64, 64, 128, 128, 64, 64, 48, 45)
    print("NEAREST display vectors written to", K.OUT)
