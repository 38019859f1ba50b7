"""Cuts tests/golden/postfx_params_*.npz: render() with SHADING + BLOOM + SUNRAYS and the post-FX sliders
BLOOM_INTENSITY / BLOOM_THRESHOLD / BLOOM_SOFT_KNEE / SUNRAYS_WEIGHT away from their defaults, by EXECUTING the
reference's GLSL text with oracle/glsl_exec.py (make_golden_keywords.render: applyBloom derives knee and curve
in JS doubles and gl.uniform narrows them, S:1358-1363).

    WEBGL_FLUID_REFERENCE=<checkout> python tests/golden/make_golden_postfx_params.py

Three parameter sets of tests/test_postfx_params_cpu.py: t033_k07 (a slider position where deriving knee /
curve in fp32 gives other uniforms than the doubles), t0_k1 (threshold 0 with soft knee 1) and t1_k0_i2_w03
(intensity 2.0 and weight 0.3, over a hard step at threshold 1), each on that file's dye, every size a power
of two: 64 x 64 dye, 128 x 64 canvas, bloom FBO 64 x 32, sunrays 32 x 16.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import glsl_exec as G  # noqa: E402
from make_golden_keywords import dithering, render  # noqa: E402
import test_postfx_params_cpu as P  # noqa: E402

FIXTURE_SETS = ["t033_k07", "t0_k1", "t1_k0_i2_w03"]


def fixture(name):
    Wd, Hd, w, h, bloom_res, sun_res, _ = P.GEOMETRIES["pow2"]
    I, T, K, W = P.SETS[name]
    dither = dithering()
    dye = P.params_dye(Wd, Hd)
    s = G.GLSLSim(16, 16, Wd, Hd)
    s.load(dye=dye)
    cfg = dict(BLOOM_RESOLUTION=bloom_res, SUNRAYS_RESOLUTION=sun_res, BLOOM_INTENSITY=I, BLOOM_THRESHOLD=T,
               BLOOM_SOFT_KNEE=K, SUNRAYS_WEIGHT=W)
    r = render(s, w, h, dither, cfg, (10, 20, 30), ("SHADING", "BLOOM", "SUNRAYS"))
    np.savez_compressed(os.path.join(HERE, f"postfx_params_{name}_64_to_128x64.npz"), Wd=Wd, Hd=Hd, w=w, h=h,
                        bloom_res=bloom_res, sun_res=sun_res, set=name, intensity=I, threshold=T, soft_knee=K, weight=W,
                        in_dye=dye, dither=dither.astype(np.float16), back=np.array([10, 20, 30], np.float32),
                        target=r["target"], bloom=r["bloom"], sunrays=r["sunrays"].astype(np.float32))


if __name__ == "__main__":
    for n in FIXTURE_SETS:
        fixture(n)
    print("post-FX slider vectors written to", HERE)
