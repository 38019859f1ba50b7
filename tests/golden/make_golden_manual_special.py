"""Cuts the fixtures of the MANUAL_FILTERING advection (the reference on a device without float linear
filtering, S:758-770) with inf and NaN velocity: GLSLSim(linear_filtering=False) EXECUTES the reference's
advectionShader with oracle/glsl_exec.py.

    WEBGL_FLUID_REFERENCE=<checkout> python tests/golden/make_golden_manual_special.py

On power-of-two grids the shader's velocity sample at a cell centre is mix(mix(a,b,0), mix(c,d,0), 0): a +x,
+y or +xy neighbour that is inf or NaN makes it NaN (0 * inf), and with it the cell's back-trace and every
channel of its result.  These files pin that for the oracle (tests/test_manual_special_cpu.py), which the GPU
tests of the non-finite advection compare against.

Writes only manual_special_<W>x<H>_<Wd>x<Hd>.npz at 16x16/16x16, 32x32/64x64 and 128x16/128x16.  Each holds,
for v in (+inf, -inf, NaN) and component c in (x, y), the case `<k>_<c>` (k the index of v in
sim_harness.CENTRE_SPECIALS): velocity from sim_harness.centre_special_velocity (coarse) and its velocity
advection, and a coarse dye advected by that same velocity.  VELOCITY_DISSIPATION 0.2, DENSITY_DISSIPATION 1.

A back-trace from an inf or NaN velocity gives a NaN coordinate.  glsl_exec's Texture clamps tap indices with
np.clip, which keeps NaN and then cannot index; here such a tap reads texel 0 (the library's texel_index), as in
make_golden_linear.py.  The weights are NaN then, so the value is NaN whichever texel is read.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import glsl_exec as G  # noqa: E402
from sim_harness import CENTRE_SPECIALS, centre_special_velocity  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
DT = np.float32(0.016666)  # the calcDeltaTime clamp, S:1191
SHAPES = [(16, 16, 16, 16), (32, 32, 64, 64), (128, 16, 128, 16)]

_fetch = G.Texture._fetch


def _fetch_nan_to_texel0(self, ix, iy):
    return _fetch(self, np.where(np.isnan(ix), 0, ix), np.where(np.isnan(iy), 0, iy))


G.Texture._fetch = _fetch_nan_to_texel0


def coarse_dye(Wd, Hd, rng):
    """red constant over 4 x 4 texel blocks, k / 16 in [-8, 8); green and blue 0, alpha 1"""
    dye = np.zeros((Hd, Wd, 4), np.float32)
    dye[..., 0] = np.repeat(np.repeat(rng.integers(-128, 128, (Hd // 4, Wd // 4)) / 16.0, 4, 0), 4, 1)
    dye[..., 3] = 1.0
    return dye


def advect(W, H, Wd, Hd, v, dye, field):
    s = G.GLSLSim(W, H, Wd, Hd, linear_filtering=False, config=dict(VELOCITY_DISSIPATION=0.2, DENSITY_DISSIPATION=1))
    s.load(velocity=v, dye=dye)
    with np.errstate(all="ignore"):
        (s.run_advect_velocity if field == "velocity" else s.run_advect_dye)(DT)
    return s.fields()[field]


def cut(W, H, Wd, Hd, seed):
    o = dict(W=W, H=H, Wd=Wd, Hd=Hd, dt=DT, velocity_dissipation=np.float32(0.2), density_dissipation=np.float32(1.0))
    rng = np.random.default_rng(seed)
    o["in_dye"] = dye = coarse_dye(Wd, Hd, rng)
    for k, value in enumerate(CENTRE_SPECIALS):
        for c in (0, 1):
            v = centre_special_velocity(W, H, value, c, seed + 10 * k + c, coarse=True)
            o[f"{k}_{c}_in_velocity"] = v
            o[f"{k}_{c}_advect_velocity"] = advect(W, H, Wd, Hd, v, dye, "velocity")
            o[f"{k}_{c}_advect_dye"] = advect(W, H, Wd, Hd, v, dye, "dye")
    np.savez_compressed(os.path.join(OUT, f"manual_special_{W}x{H}_{Wd}x{Hd}.npz"), **o)


if __name__ == "__main__":
    for k, shp in enumerate(SHAPES):
        cut(*shp, 900 + 100 * k)
    print("golden vectors written to", OUT)
