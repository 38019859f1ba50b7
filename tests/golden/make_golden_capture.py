"""Cuts tests/golden/capture_*.npz: captureScreenshot() (S:287-299) up to normalizeTexture (S:309-327),
by EXECUTING the reference's GLSL text with oracle/glsl_exec.py.  The bloom and sunrays chains come from
make_golden_keywords.render() run on the canvas; the capture target is drawn here (capture_render).

    WEBGL_FLUID_REFERENCE=<checkout> python tests/golden/make_golden_capture.py

captureScreenshot renders into an RGBA half-float FBO of getResolution(CAPTURE_RESOLUTION) (S:288-290):
every store rounds to fp16 (glsl_exec rounds half textures to nearest even and blends in fp32 against
the stored destination), drawColor(BACK_COLOR) lands in fp16 before the display is blended over it, and
with TRANSPARENT the display is stored bare (no checkerboard: target != null, S:1303-1314).  The bloom and
sunrays FBOs keep the sizes initBloomFramebuffers / initSunraysFramebuffers give them from the drawing
buffer (S:1012-1043), so they are sized from the canvas, not from the target.  normalizeTexture clamps to
[0, 1], multiplies by 255 and stores into a Uint8Array (truncation; NaN -> 0), flipping the rows so that
the top row comes first.

Each geometry gets two files, capture_<geometry>_<bg>.npz with bg = "back" (over BACK_COLOR (10, 20, 30))
or "transparent" (config.TRANSPARENT), which keeps each under 400 KB.  Each holds the input dye, the fp16
dithering texture and the sizes, and for each of the eight keyword sets: <set>_half, the fp16 target
(row 0 = bottom), and <set>_rgba8, the uint8 image after normalizeTexture (row 0 = top).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_keywords as K  # noqa: E402
from make_golden_keywords import G  # noqa: E402

OUT = HERE
BACK = (10, 20, 30)
SETS = {"none": (), "shading": ("SHADING",), "bloom": ("BLOOM",), "shading_bloom": ("SHADING", "BLOOM"),
        "sunrays": ("SUNRAYS",), "shading_sunrays": ("SHADING", "SUNRAYS"), "bloom_sunrays": ("BLOOM", "SUNRAYS"),
        "shading_bloom_sunrays": ("SHADING", "BLOOM", "SUNRAYS")}


def get_resolution(res, w, h):
    """getResolution (S:1612-1624) on a w x h drawing buffer, in JS doubles."""
    ar = w / h
    if ar < 1: ar = 1.0 / ar
    mn, mx = int(np.floor(res + 0.5)), int(np.floor(res * ar + 0.5))
    return (mx, mn) if w > h else (mn, mx)


def capture_render(sim, width, height, canvas_w, canvas_h, dither, cfg, keywords, transparent):
    """render(target) of S:1296-1317 into captureScreenshot's width x height RGBA half-float target (S:289).
    applyBloom / applySunrays + blur are make_golden_keywords.render() on the canvas_w x canvas_h drawing
    buffer, whose sizes the reference's bloom and sunrays FBOs keep; its own frame is discarded.  Then
    drawColor(BACK_COLOR) unless TRANSPARENT (never the checkerboard: target != null) and drawDisplay at
    the target's size (texelSize, ditherScale: S:1332-1344), blended ONE / ONE_MINUS_SRC_ALPHA, or with
    blending off under TRANSPARENT (S:1303-1309).  Returns the stored fp16 target as float32."""
    js = open(G.REFERENCE_JS).read()
    P = lambda vs, fs, d=(): G.Program(js, vs, fs, d)                                 # noqa: E731
    dye = G.Texture(sim.dye.read.w, sim.dye.read.h, 4, True); dye.data = sim.dye.read.data
    chains = K.render(sim, canvas_w, canvas_h, dither, cfg, BACK, keywords) if {"BLOOM", "SUNRAYS"} & set(keywords) else None
    target = G.Texture(width, height, 4, True, half=True)
    if not transparent:                                                             # drawColor, S:1319-1323
        col = P("baseVertexShader", "colorShader")
        col.set(texelSize=(1.0 / width, 1.0 / height), color=(BACK[0] / 255, BACK[1] / 255, BACK[2] / 255, 1))
        col.blit(target)
    disp = P("baseVertexShader", "displayShaderSource", tuple(k for k in ("SHADING", "BLOOM", "SUNRAYS") if k in keywords))
    disp.set(texelSize=(1.0 / width, 1.0 / height), uTexture=dye)                   # S:1337-1338
    if "BLOOM" in keywords:
        bh, bw = chains["bloom"].shape[:2]
        bloom = G.Texture(bw, bh, 4, True); bloom.data = chains["bloom"]
        dith = G.Texture(dither.shape[1], dither.shape[0], 3, True, repeat=True)
        dith.data[..., :3] = dither
        disp.set(uBloom=bloom, uDithering=dith, ditherScale=(width / dith.w, height / dith.h))   # S:1339-1344, S:1626-1631
    if "SUNRAYS" in keywords:
        sh, sw = chains["sunrays"].shape
        sun = G.Texture(sw, sh, 1, True)                                            # an R texture reads as (r, 0, 0, 1)
        sun.data[..., 0] = chains["sunrays"]
        disp.set(uSunrays=sun)                                                      # S:1345-1346
    disp.blit(target, blend=None if transparent else "premult")
    return target.data.copy()


def normalize_texture(half):
    """normalizeTexture, S:309-327, in JS doubles: clamp01(v) * 255 into a Uint8Array (ToUint8: NaN -> 0,
    otherwise truncation), rows flipped so that the top row comes first."""
    v = half.astype(np.float64)
    x = np.minimum(np.maximum(v, 0.0), 1.0) * 255.0          # NaN stays NaN through Math.max / Math.min
    return np.where(np.isnan(x), 0.0, np.trunc(x)).astype(np.uint8)[::-1].copy()


def capture_fixture(name, Wd, Hd, canvas_w, canvas_h, capture_res, bloom_res, sun_res, seed):
    w, h = get_resolution(capture_res, canvas_w, canvas_h)
    dither = K.dithering()
    rng = np.random.default_rng(seed)
    s = G.GLSLSim(16, 16, Wd, Hd)
    # dimmer than the keyword fixtures' (** 4 * 3): there most bytes would saturate at 255 and pin nothing
    dye = (rng.random((Hd, Wd, 4), dtype=np.float32) ** 4).astype(np.float32); dye[..., 3] = 1
    s.load(dye=dye)
    cfg = dict(BLOOM_RESOLUTION=bloom_res, SUNRAYS_RESOLUTION=sun_res)
    files = {}
    for bg, transparent in (("back", False), ("transparent", True)):
        o = dict(Wd=Wd, Hd=Hd, canvas_w=canvas_w, canvas_h=canvas_h, w=w, h=h, capture_res=capture_res,
                 bloom_res=bloom_res, sun_res=sun_res, in_dye=dye, dither=dither.astype(np.float16),
                 back=np.array(BACK, np.float32), transparent=transparent, sets=np.array(list(SETS)))
        for tag, kw in SETS.items():
            t = capture_render(s, w, h, canvas_w, canvas_h, dither, cfg, kw, transparent)
            assert np.array_equal(t.astype(np.float16).astype(np.float32), t), (name, tag, bg)   # stored as fp16
            assert np.array_equal(s.dye.read.data, dye), (name, tag, bg)                           # dye.read untouched
            o[f"{tag}_half"] = t.astype(np.float16)
            o[f"{tag}_rgba8"] = normalize_texture(t.astype(np.float16))
        files[bg] = o
    for tag in SETS:                                # the backgrounds differ wherever the display is not opaque
        assert not np.array_equal(files["back"][f"{tag}_rgba8"], files["transparent"][f"{tag}_rgba8"]), (name, tag)
    for bg, o in files.items():
        np.savez_compressed(os.path.join(OUT, f"{name}_{bg}.npz"), **o)


def check_self_consistency():
    """The fp16 store rounds like numpy's float16; normalizeTexture's corner cases (S:309-327, ToUint8)."""
    v = np.array([np.nan, -np.inf, -1.0, 0.0, 1.0 / 255.0, 0.5, 1.0 - 2.0 ** -11, 1.0, 2.0, np.inf, 70000.0], np.float32)
    with np.errstate(over="ignore"):
        half = v.astype(np.float16)
    assert np.isinf(half[-1])                                                   # overflow goes to +Inf
    got = normalize_texture(half[None, :, None].repeat(4, 2))[0, :, 0]
    assert list(got) == [0, 0, 0, 0, 0, 127, 254, 255, 255, 255, 255], got      # 1/255 in fp16 is just below it


if __name__ == "__main__":
    K.check_against_postfx_fixtures()           # the chains' render() reproduces the committed postfx fixtures
    check_self_consistency()
    # power of two: 64^2 dye, 128^2 canvas, CAPTURE_RESOLUTION 64 -> 64^2 target
    capture_fixture("capture_64_canvas_128", 64, 64, 128, 128, 64, 64, 48, 31)
    # canvas != target: 807 x 640 canvas, CAPTURE_RESOLUTION 48 -> 61 x 48 target.  The bloom FBO is 40 x 32
    # from the canvas and would be 41 x 32 from the target; the sunrays FBO 50 x 40 against 51 x 40.
    # (A 48-texel capture keeps each file under 400 KB.)
    assert get_resolution(48, 807, 640) == (61, 48)
    assert get_resolution(32, 807, 640) == (40, 32) and get_resolution(32, 61, 48) == (41, 32)
    assert get_resolution(40, 807, 640) == (50, 40) and get_resolution(40, 61, 48) == (51, 40)
    capture_fixture("capture_48x32_canvas_807x640", 48, 32, 807, 640, 48, 32, 40, 32)
    print("capture vectors written to", OUT)
