"""Cuts tests/golden/keywords_*.npz: render() with the display keyword sets that are neither none /
SHADING (display_*.npz) nor SHADING + BLOOM + SUNRAYS (postfx_*.npz), by EXECUTING the reference's
GLSL text with oracle/glsl_exec.py, like make_golden.py.

    WEBGL_FLUID_REFERENCE=<checkout> python tests/golden/make_golden_keywords.py

render() and drawDisplay (S:1296-1348) are restated here call for call for any keyword set:
applyBloom (S:1350-1394) only with BLOOM, applySunrays + blur (S:1396-1419) only with SUNRAYS, the
display program compiled with the keywords of updateKeywords (S:1160-1166) and given the bloom /
dithering / sunrays textures only for the keywords that are on (S:1339-1346).  With all three keywords
and BACK_COLOR this reproduces postfx_*.npz exactly (checked before anything is written).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import glsl_exec as G  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
KEYWORD_SETS = {"bloom": ("BLOOM",), "sunrays": ("SUNRAYS",), "bloom_sunrays": ("BLOOM", "SUNRAYS"),
                "shading_bloom": ("SHADING", "BLOOM"), "shading_sunrays": ("SHADING", "SUNRAYS")}


def render(sim, width, height, dither, cfg, back_color, keywords, transparent=False, to_screen=True):
    """render(target) of S:1296-1317 with `keywords` on the dye of a GLSLSim.  TRANSPARENT: the
    checkerboard under the display on the screen, the bare display (blending off) into a capture target."""
    js = open(G.REFERENCE_JS).read()
    c = dict(BLOOM_ITERATIONS=8, BLOOM_RESOLUTION=256, BLOOM_INTENSITY=0.8, BLOOM_THRESHOLD=0.6,
             BLOOM_SOFT_KNEE=0.7, SUNRAYS_RESOLUTION=196, SUNRAYS_WEIGHT=1.0)
    c.update(cfg)

    def get_resolution(res):                                                        # S:1612-1624
        ar = width / height
        if ar < 1: ar = 1.0 / ar
        mn, mx = int(np.floor(res + 0.5)), int(np.floor(res * ar + 0.5))
        return (mx, mn) if width > height else (mn, mx)

    P = lambda vs, fs, d=(): G.Program(js, vs, fs, d)                                 # noqa: E731
    dye = G.Texture(sim.dye.read.w, sim.dye.read.h, 4, True); dye.data = sim.dye.read.data
    bloom, pyramid, sun, mask = None, [], None, None
    if "BLOOM" in keywords:                                                         # applyBloom(dye.read, bloom)
        bw, bh = get_resolution(c["BLOOM_RESOLUTION"])
        bloom = G.Texture(bw, bh, 4, True)
        for i in range(c["BLOOM_ITERATIONS"]):
            pw, ph = bw >> (i + 1), bh >> (i + 1)
            if pw < 2 or ph < 2: break
            pyramid.append(G.Texture(pw, ph, 4, True))
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
        sw, sh = get_resolution(c["SUNRAYS_RESOLUTION"])
        mask = G.Texture(dye.w, dye.h, 4, True)
        sun, tmp = G.Texture(sw, sh, 1, True), G.Texture(sw, sh, 1, True)
        mp = P("baseVertexShader", "sunraysMaskShader"); mp.set(texelSize=(0.0, 0.0), uTexture=dye); mp.blit(mask)
        sp = P("baseVertexShader", "sunraysShader"); sp.set(texelSize=(0.0, 0.0), weight=c["SUNRAYS_WEIGHT"], uTexture=mask); sp.blit(sun)
        bp = P("blurVertexShader", "blurShader")
        bp.set(texelSize=(sun.texelSizeX, 0.0), uTexture=sun); bp.blit(tmp)
        bp.set(texelSize=(0.0, sun.texelSizeY), uTexture=tmp); bp.blit(sun)
    target = G.Texture(width, height, 4, True)
    if not transparent:                                                             # drawColor, S:1319-1323
        col = P("baseVertexShader", "colorShader")
        col.set(texelSize=(1.0 / width, 1.0 / height), color=(back_color[0] / 255, back_color[1] / 255, back_color[2] / 255, 1))
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


def dithering():
    """LDR_LLL1_0.png / 255, rounded through fp16 as the fixtures store it, so that the stored texture
    is exactly the one the executed shaders read."""
    from PIL import Image
    d = np.asarray(Image.open(os.path.join(G.REFERENCE_DIR, "LDR_LLL1_0.png")).convert("RGB"), dtype=np.float32) / np.float32(255.0)
    return d.astype(np.float16).astype(np.float32)


def keyword_fixture(name, Wd, Hd, w, h, seed, sets, transparent=False, bloom_res=64, sun_res=48):
    """One dye field drawn with each keyword set of `sets` (names of KEYWORD_SETS).  The bloom and sunrays
    chains do not depend on the keywords: their textures are stored once.  transparent: each set over the
    checkerboard on the screen (<set>_checker) and bare into a capture target (<set>_bare) instead of over
    BACK_COLOR (<set>_target)."""
    dither = dithering()
    rng = np.random.default_rng(seed)
    s = G.GLSLSim(16, 16, Wd, Hd)
    dye = (rng.random((Hd, Wd, 4), dtype=np.float32) ** 4 * 3).astype(np.float32); dye[..., 3] = 1
    s.load(dye=dye)
    cfg = dict(BLOOM_RESOLUTION=bloom_res, SUNRAYS_RESOLUTION=sun_res)
    o = dict(Wd=Wd, Hd=Hd, w=w, h=h, bloom_res=bloom_res, sun_res=sun_res, in_dye=dye, dither=dither.astype(np.float16),
             back=np.array([10, 20, 30], np.float32), sets=np.array(sets))
    modes = [("checker", True, True), ("bare", True, False)] if transparent else [("target", False, True)]
    for tag in sets:
        for key, tr, scr in modes:
            r = render(s, w, h, dither, cfg, (10, 20, 30), KEYWORD_SETS[tag], tr, scr)
            o[f"{tag}_{key}"] = r["target"]
            for k in ("bloom", "sunrays", "mask_alpha"):
                if r[k] is not None:
                    assert k not in o or np.array_equal(o[k], r[k]), k
                    o[k] = r[k].astype(np.float32)
            for k, t in enumerate(r["pyramid"]):
                o[f"pyr{k}"] = t
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **o)


def check_against_postfx_fixtures():
    """All three keywords over BACK_COLOR must give the committed postfx_*.npz bit for bit."""
    from PIL import Image
    full = np.asarray(Image.open(os.path.join(G.REFERENCE_DIR, "LDR_LLL1_0.png")).convert("RGB"), dtype=np.float32) / np.float32(255.0)
    for name in ("postfx_64_to_128", "postfx_48x32_to_50x75"):
        g = np.load(os.path.join(OUT, name + ".npz"))
        s = G.GLSLSim(16, 16, int(g["Wd"]), int(g["Hd"])); s.load(dye=g["in_dye"])
        r = render(s, int(g["w"]), int(g["h"]), full, dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"])),
                   (10, 20, 30), ("SHADING", "BLOOM", "SUNRAYS"))
        for k in ("target", "bloom", "sunrays", "mask_alpha"):
            assert np.array_equal(r[k], g[k]), (name, k)


if __name__ == "__main__":
    check_against_postfx_fixtures()
    for tag in KEYWORD_SETS:            # power-of-two target, dye and bloom FBO: one file per set keeps each small
        keyword_fixture(f"keywords_{tag}_64_to_128", 64, 64, 128, 128, 23, [tag])
    keyword_fixture("keywords_48x32_to_50x75", 48, 32, 50, 75, 24, list(KEYWORD_SETS))      # ragged, portrait canvas
    keyword_fixture("keywords_transparent_64x32_to_128x64", 64, 32, 128, 64, 25, ["bloom_sunrays"], transparent=True)
    print("display keyword vectors written to", OUT)
