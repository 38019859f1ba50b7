"""Cuts the fixtures of FLUID_FLAG_LINEAR_ADVECTION, the reference on a device WITH float linear
filtering (every desktop browser): the advectionShader's #else branch (S:776-779) samples uVelocity
and uSource through the LINEAR samplers of dye and velocity (S:990).  By EXECUTING the reference's
GLSL text with oracle/glsl_exec.py (GLSLSim(linear_filtering=True, half=...)).

    WEBGL_FLUID_REFERENCE=<checkout> python tests/golden/make_golden_linear.py

Writes only these files (the other fixtures are left as they are):
  linear_pass_{fp32,half}_<W>x<H>_<Wd>x<Hd>.npz   advect velocity, then dye, from written fields
      (VELOCITY_DISSIPATION 0.2, DENSITY_DISSIPATION 1) at 32x32/64x64, 64x32/128x64, 16x16/16x16,
      128x128/256x256 (coarser fields, see fields(), so that the file stays small) and the ragged
      24x16/40x28.  The 32x32/64x64 and 16x16/16x16 files also hold a
      `special_*` case: velocity with +inf and -inf texels and -0 next to finite ones, so that a cell
      whose LINEAR sample weighs an infinite neighbour by 0 gets NaN (0 * inf), as the GL spec's
      weighted sum gives it.
  linear_step_{fp32,half}_<W>x<H>_<Wd>x<Hd>.npz   two whole steps from written fields, no splats (so
      expf plays no part), CURL 30, 20 pressure iterations, at 32x32/64x64 and 64x32/128x64.
Half files hold fp16-representable inputs, and every texture stores fp16 like the real RGBA16F ones.

A back-trace from an infinite velocity gives a NaN coordinate.  glsl_exec's Texture clamps tap indices
with np.clip, which keeps NaN and then cannot index; here such a tap reads texel 0 (the library's
texel_index).  The weights are NaN then, so the value is NaN whichever texel is read.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import glsl_exec as G  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
DT = np.float32(0.016666)  # the calcDeltaTime clamp, S:1191

PASS_SHAPES = [(32, 32, 64, 64), (64, 32, 128, 64), (16, 16, 16, 16), (128, 128, 256, 256), (24, 16, 40, 28)]
SPECIAL_SHAPES = [(32, 32, 64, 64), (16, 16, 16, 16)]
STEP_SHAPES = [(32, 32, 64, 64), (64, 32, 128, 64)]

_fetch = G.Texture._fetch


def _fetch_nan_to_texel0(self, ix, iy):
    return _fetch(self, np.where(np.isnan(ix), 0, ix), np.where(np.isnan(iy), 0, iy))


G.Texture._fetch = _fetch_nan_to_texel0


def _store(a, half):
    a = np.asarray(a, np.float32)
    return a.astype(np.float16).astype(np.float32) if half else a


def fields(W, H, Wd, Hd, half, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((H, W, 2)) * 50
    dye = rng.standard_normal((Hd, Wd, 4)) * 100     # mixed signs: the weighted sums cancel
    if W >= 128:
        # keeps the file small (the results of random fields do not compress): velocity from 32 values per
        # component, multiples of 4 in [-64, 60] (dt = 0.016666 still scatters the back-traces); one dye
        # channel, constant over 4 x 4 texel blocks with values k / 16 in [-8, 8), green and blue 0, alpha 1
        v = rng.integers(-16, 16, (H, W, 2)) * 4.0
        red = np.repeat(np.repeat(rng.integers(-128, 128, (Hd // 4, Wd // 4)) / 16.0, 4, 0), 4, 1)
        dye = np.zeros((Hd, Wd, 4))
        dye[..., 0] = red
        dye[..., 3] = 1.0
    v, dye = _store(v, half), _store(dye, half)
    return v, dye


def special(v, dye, half):
    """+inf, -inf and -0 velocity texels beside finite ones; a NaN and inf in dye."""
    v = v.copy(); dye = dye.copy()
    H, W = v.shape[:2]
    v[H // 2, W // 2, 0] = np.inf
    v[H // 4, W // 3, 1] = -np.inf
    v[1, 1] = (-0.0, -0.0)
    v[H - 2, 2, 0] = -0.0
    dye[0, 0, 0] = np.nan
    dye[-1, -1, 2] = np.inf
    return _store(v, half), _store(dye, half)


def advect_pair(W, H, Wd, Hd, half, v, dye):
    s = G.GLSLSim(W, H, Wd, Hd, linear_filtering=True, half=half,
                  config=dict(VELOCITY_DISSIPATION=0.2, DENSITY_DISSIPATION=1))
    s.load(velocity=v, dye=dye)
    with np.errstate(all="ignore"):
        s.run_advect_velocity(DT); av = s.fields()["velocity"]
        s.run_advect_dye(DT); ad = s.fields()["dye"]
    return av, ad


def per_pass(W, H, Wd, Hd, half, seed):
    v, dye = fields(W, H, Wd, Hd, half, seed)
    o = dict(W=W, H=H, Wd=Wd, Hd=Hd, dt=DT, half=half, velocity_dissipation=np.float32(0.2),
             density_dissipation=np.float32(1.0), in_velocity=v, in_dye=dye)
    o["advect_velocity"], o["advect_dye"] = advect_pair(W, H, Wd, Hd, half, v, dye)
    if (W, H, Wd, Hd) in SPECIAL_SHAPES:
        sv, sd = special(v, dye, half)
        o["special_in_velocity"], o["special_in_dye"] = sv, sd
        o["special_advect_velocity"], o["special_advect_dye"] = advect_pair(W, H, Wd, Hd, half, sv, sd)
    tag = "half" if half else "fp32"
    np.savez_compressed(os.path.join(OUT, f"linear_pass_{tag}_{W}x{H}_{Wd}x{Hd}.npz"), **o)


def steps(W, H, Wd, Hd, half, seed, n=2):
    v, dye = fields(W, H, Wd, Hd, half, seed)
    s = G.GLSLSim(W, H, Wd, Hd, linear_filtering=True, half=half, config=dict(CURL=30, PRESSURE_ITERATIONS=20))
    s.load(velocity=v, dye=dye)
    o = dict(W=W, H=H, Wd=Wd, Hd=Hd, dt=DT, half=half, curl=np.float32(30), pressure_iterations=20, steps=n,
             init_velocity=v, init_dye=dye)
    for k in range(1, n + 1):
        s.step(DT)
        for name, a in s.fields().items():
            o[f"s{k}_{name}"] = a
    tag = "half" if half else "fp32"
    np.savez_compressed(os.path.join(OUT, f"linear_step_{tag}_{W}x{H}_{Wd}x{Hd}.npz"), **o)


if __name__ == "__main__":
    for half in (False, True):
        for k, shp in enumerate(PASS_SHAPES):
            per_pass(*shp, half, 700 + k)
        for k, shp in enumerate(STEP_SHAPES):
            steps(*shp, half, 800 + k)
    print("golden vectors written to", OUT)
