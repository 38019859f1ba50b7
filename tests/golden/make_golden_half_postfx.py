"""Cuts the fixtures of FLUID_FLAG_HALF_STORAGE | FLUID_FLAG_HALF_POSTFX, the reference's desktop storage:
fp16 dye, and half-float bloom FBO, pyramid, sunrays, sunraysTemp and sunrays mask (S:138-147,
S:986-1006, S:1012-1043), by EXECUTING the reference's GLSL text with oracle/glsl_exec.py.

    WEBGL_FLUID_REFERENCE=<checkout> python tests/golden/make_golden_half_postfx.py

render_half() is make_golden_keywords.render() with the chains' textures created half-float (glsl_exec's
Texture(half=True) rounds every store to fp16 and blends in fp32 against the stored destination); the
render() frame target stays fp32.  capture_render_half() is make_golden_capture.capture_render() over
those chains.  The dye and its seeds are drawn as in those two generators and rounded to fp16 before they
are loaded, as a half-storage handle holds them.

Writes only these files (the other fixtures are left as they are):
  keywords_half_64_to_128.npz                 power of two, the five post-FX keyword sets
  keywords_half_48x32_to_50x75.npz            ragged dye, portrait canvas, the same five sets
  capture_half_64_canvas_128_{back,transparent}.npz   all eight sets, 64^2 capture of a 128^2 canvas
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_capture as CAP  # noqa: E402
import make_golden_keywords as K  # noqa: E402
from make_golden_keywords import G  # noqa: E402

BACK = CAP.BACK


def render_half(sim, width, height, dither, cfg, keywords, transparent=False, to_screen=True):
    """render(target) of S:1296-1317 with `keywords` over BACK_COLOR (or TRANSPARENT), the bloom FBO, the
    pyramid, sunrays, sunraysTemp and the mask (dye.write) being half-float textures."""
    js = open(G.REFERENCE_JS).read()
    c = dict(BLOOM_ITERATIONS=8, BLOOM_RESOLUTION=256, BLOOM_INTENSITY=0.8, BLOOM_THRESHOLD=0.6,
             BLOOM_SOFT_KNEE=0.7, SUNRAYS_RESOLUTION=196, SUNRAYS_WEIGHT=1.0)
    c.update(cfg)
    P = lambda vs, fs, d=(): G.Program(js, vs, fs, d)                                 # noqa: E731
    dye = G.Texture(sim.dye.read.w, sim.dye.read.h, 4, True); dye.data = sim.dye.read.data
    bloom, pyramid, sun, mask = None, [], None, None
    if "BLOOM" in keywords:                                                         # applyBloom(dye.read, bloom)
        bw, bh = CAP.get_resolution(c["BLOOM_RESOLUTION"], width, height)
        bloom = G.Texture(bw, bh, 4, True, half=True)
        for i in range(c["BLOOM_ITERATIONS"]):
            pw, ph = bw >> (i + 1), bh >> (i + 1)
            if pw < 2 or ph < 2: break
            pyramid.append(G.Texture(pw, ph, 4, True, half=True))
        if len(pyramid) >= 2:
            knee = c["BLOOM_THRESHOLD"] * c["BLOOM_SOFT_KNEE"] + 0.0001
            pre = P("baseVertexShader", "bloomPrefilterShader")
            pre.set(texelSize=(0.0, 0.0), curve=(c["BLOOM_THRESHOLD"] - knee, knee * 2, 0.25 / knee),
                    threshold=c["BLOOM_THRESHOLD"], uTexture=dye)
            pre.blit(bloom)
            last = bloom
            blurp = P("baseVertexShader", "bloomBlurShader")
            for dest in pyramid:
                blurp.set(texelSize=(last.texelSizeX, last.texelSizeY), uTexture=last)
                blurp.blit(dest); last = dest
            for i in range(len(pyramid) - 2, -1, -1):
                blurp.set(texelSize=(last.texelSizeX, last.texelSizeY), uTexture=last)
                blurp.blit(pyramid[i], blend="add"); last = pyramid[i]
            fin = P("baseVertexShader", "bloomFinalShader")
            fin.set(texelSize=(last.texelSizeX, last.texelSizeY), uTexture=last, intensity=c["BLOOM_INTENSITY"])
            fin.blit(bloom)
    if "SUNRAYS" in keywords:                                                       # applySunrays + blur(…, 1)
        sw, sh = CAP.get_resolution(c["SUNRAYS_RESOLUTION"], width, height)
        mask = G.Texture(dye.w, dye.h, 4, True, half=True)
        sun, tmp = G.Texture(sw, sh, 1, True, half=True), G.Texture(sw, sh, 1, True, half=True)
        mp = P("baseVertexShader", "sunraysMaskShader"); mp.set(texelSize=(0.0, 0.0), uTexture=dye); mp.blit(mask)
        sp = P("baseVertexShader", "sunraysShader"); sp.set(texelSize=(0.0, 0.0), weight=c["SUNRAYS_WEIGHT"], uTexture=mask); sp.blit(sun)
        bp = P("blurVertexShader", "blurShader")
        bp.set(texelSize=(sun.texelSizeX, 0.0), uTexture=sun); bp.blit(tmp)
        bp.set(texelSize=(0.0, sun.texelSizeY), uTexture=tmp); bp.blit(sun)
    target = G.Texture(width, height, 4, True)
    if not transparent:                                                             # drawColor, S:1319-1323
        col = P("baseVertexShader", "colorShader")
        col.set(texelSize=(1.0 / width, 1.0 / height), color=(BACK[0] / 255, BACK[1] / 255, BACK[2] / 255, 1))
        col.blit(target)
    elif to_screen:                                                                 # drawCheckerboard, S:1325-1329
        chk = P("baseVertexShader", "checkerboardShader")
        chk.set(texelSize=(1.0 / width, 1.0 / height), aspectRatio=width / height)
        chk.blit(target)
    disp = P("baseVertexShader", "displayShaderSource", tuple(k for k in ("SHADING", "BLOOM", "SUNRAYS") if k in keywords))
    disp.set(texelSize=(1.0 / width, 1.0 / height), uTexture=dye)                   # S:1337-1338
    if "BLOOM" in keywords:
        dith = G.Texture(dither.shape[1], dither.shape[0], 3, True, repeat=True)
        dith.data[..., :3] = dither
        disp.set(uBloom=bloom, uDithering=dith, ditherScale=(width / dith.w, height / dith.h))   # S:1339-1344, S:1626-1631
    if "SUNRAYS" in keywords:
        disp.set(uSunrays=sun)                                                      # S:1345-1346
    disp.blit(target, blend=None if transparent and not to_screen else "premult")  # S:1303-1308
    return dict(target=target.data.copy(), bloom=None if bloom is None else bloom.data.copy(),
                sunrays=None if sun is None else sun.data[..., 0].copy(),
                mask_alpha=None if mask is None else mask.data[..., 3].copy(), pyramid=[t.data.copy() for t in pyramid])


def capture_render_half(sim, width, height, canvas_w, canvas_h, dither, cfg, keywords, transparent):
    """make_golden_capture.capture_render with the half-float chains of render_half on the canvas."""
    js = open(G.REFERENCE_JS).read()
    P = lambda vs, fs, d=(): G.Program(js, vs, fs, d)                                 # noqa: E731
    dye = G.Texture(sim.dye.read.w, sim.dye.read.h, 4, True); dye.data = sim.dye.read.data
    chains = render_half(sim, canvas_w, canvas_h, dither, cfg, keywords) if {"BLOOM", "SUNRAYS"} & set(keywords) else None
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


def half_sim(Wd, Hd, seed, scale):
    """A GLSLSim holding the seeded dye (rng ** 4 * scale, alpha 1) rounded to fp16."""
    rng = np.random.default_rng(seed)
    dye = (rng.random((Hd, Wd, 4), dtype=np.float32) ** 4 * np.float32(scale)).astype(np.float32); dye[..., 3] = 1
    dye = dye.astype(np.float16).astype(np.float32)
    s = G.GLSLSim(16, 16, Wd, Hd); s.load(dye=dye)
    return s, dye


def keyword_fixture(name, Wd, Hd, w, h, seed, bloom_res=64, sun_res=48):
    """The five post-FX keyword sets of make_golden_keywords over BACK_COLOR: <set>_target, and the chains
    (stored once: they do not depend on the keywords)."""
    dither = K.dithering()
    s, dye = half_sim(Wd, Hd, seed, 3.0)
    cfg = dict(BLOOM_RESOLUTION=bloom_res, SUNRAYS_RESOLUTION=sun_res)
    sets = list(K.KEYWORD_SETS)
    o = dict(Wd=Wd, Hd=Hd, w=w, h=h, bloom_res=bloom_res, sun_res=sun_res, in_dye=dye, dither=dither.astype(np.float16),
             back=np.array(BACK, np.float32), sets=np.array(sets))
    for tag in sets:
        r = render_half(s, w, h, dither, cfg, K.KEYWORD_SETS[tag])
        o[f"{tag}_target"] = r["target"]
        for k in ("bloom", "sunrays", "mask_alpha"):
            if r[k] is not None:
                assert k not in o or np.array_equal(o[k], r[k]), k
                o[k] = r[k].astype(np.float32)
        for k, t in enumerate(r["pyramid"]):
            o[f"pyr{k}"] = t
    np.savez_compressed(os.path.join(K.OUT, name + ".npz"), **o)


def capture_fixture(name, Wd, Hd, canvas_w, canvas_h, capture_res, bloom_res, sun_res, seed):
    """make_golden_capture.capture_fixture with the fp16 dye and the half-float chains."""
    w, h = CAP.get_resolution(capture_res, canvas_w, canvas_h)
    dither = K.dithering()
    s, dye = half_sim(Wd, Hd, seed, 1.0)
    cfg = dict(BLOOM_RESOLUTION=bloom_res, SUNRAYS_RESOLUTION=sun_res)
    for bg, transparent in (("back", False), ("transparent", True)):
        o = dict(Wd=Wd, Hd=Hd, canvas_w=canvas_w, canvas_h=canvas_h, w=w, h=h, capture_res=capture_res,
                 bloom_res=bloom_res, sun_res=sun_res, in_dye=dye, dither=dither.astype(np.float16),
                 back=np.array(BACK, np.float32), transparent=transparent, sets=np.array(list(CAP.SETS)))
        for tag, kw in CAP.SETS.items():
            t = capture_render_half(s, w, h, canvas_w, canvas_h, dither, cfg, kw, transparent)
            assert np.array_equal(t.astype(np.float16).astype(np.float32), t), (name, tag, bg)   # stored as fp16
            assert np.array_equal(s.dye.read.data, dye), (name, tag, bg)                           # dye.read untouched
            o[f"{tag}_half"] = t.astype(np.float16)
            o[f"{tag}_rgba8"] = CAP.normalize_texture(t.astype(np.float16))
        np.savez_compressed(os.path.join(K.OUT, f"{name}_{bg}.npz"), **o)


if __name__ == "__main__":
    K.check_against_postfx_fixtures()
    CAP.check_self_consistency()
    keyword_fixture("keywords_half_64_to_128", 64, 64, 128, 128, 26)
    keyword_fixture("keywords_half_48x32_to_50x75", 48, 32, 50, 75, 27)
    capture_fixture("capture_half_64_canvas_128", 64, 64, 128, 128, 64, 64, 48, 33)
    print("half-float post-FX vectors written to", K.OUT)
