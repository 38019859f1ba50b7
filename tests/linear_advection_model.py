"""fp32 model of FLUID_FLAG_LINEAR_ADVECTION: the advectionShader's #else branch (S:776-779), where
texture2D(uVelocity, vUv) and texture2D(uSource, coord) go through the LINEAR samplers dye and velocity
are created with (S:990), as a browser with float linear filtering runs it.

TEST INFRASTRUCTURE ONLY.  Every operation is one numpy float32 ufunc, so it is rounded on its own
(no contraction), in the order include/fluid.h gives:
    L(tex, uv):  u = uv.x * n_x - .5, i0 = floor(u), a = u - i0 (v, b likewise), taps clamped like
                 texel_index (NaN and <= 0 -> 0, >= n - 1 -> n - 1),
                 ((w00 t00 + w10 t10) + w01 t01) + w11 t11, w00 = (1-a)(1-b), w10 = a(1-b), w01 = (1-a)b, w11 = ab
    velocity:    c = uv - (dt * L(vel, uv)) * ts;  L(vel, c) / (1 + VELOCITY_DISSIPATION * dt)
    dye:         c = uv - (dt * L(vel, uv)) * ts   (the SIM texel size, S:1276);  L(dye, c) / (1 + DENSITY_DISSIPATION * dt)
The rest of a step is the C oracle's (oracle/oracle.py), unchanged.

The keyword arguments of `advect` build the mutants that tests/test_linear_advection_cpu.py shows the
golden vectors reject: the manual shader's mix-of-mix weights, its uv / ts - .5 coordinate, and the own
texel in place of the velocity sample at a cell centre.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

F = np.float32
ROWS = 256          # rows per chunk: bounds the temporaries at 4096^2 dye
P4_HALF_GATE = 1e-6  # max_rel of the fp16 desktop scenario after one step (p4_linear_half_32), CPU and GPU


def texel_index(f, n):
    out = np.zeros(f.shape, np.int64)
    pos = f > 0                                    # NaN is not
    top = f >= F(n - 1)
    mid = pos & ~top
    out[mid] = f[mid].astype(np.int64)
    out[top] = n - 1
    return out


def cell_uv(n, uv="cell"):
    """Fragment centres of an n-texel axis.  "cell": (i + .5) / n, the library's (exact 2^-k multiples on
    power-of-two grids).  "raster": the vUv the executed shaders get, aPosition * .5 + .5 with aPosition
    the NDC centre (i + .5) / n * 2 - 1 (oracle/glsl_exec.py); it differs by an ulp on ragged grids."""
    c = (np.arange(n, dtype=F) + F(0.5)) / F(n)
    return c if uv == "cell" else (c * F(2) - F(1)) * F(0.5) + F(0.5)


def fetch(tex, uvx, uvy, weights="gl", coord="uvn"):
    """One sample of a (n_y, n_x, C) fp32 field at uv arrays of one shape.  weights='mix' and
    coord='uvts' are the MANUAL_FILTERING shader's (mutants here)."""
    H, W = tex.shape[:2]
    if coord == "uvn":
        u = uvx * F(W) - F(0.5); v = uvy * F(H) - F(0.5)
    else:
        u = uvx / F(1.0 / W) - F(0.5); v = uvy / F(1.0 / H) - F(0.5)
    fi = np.floor(u); fj = np.floor(v)
    a = (u - fi)[..., None]; b = (v - fj)[..., None]
    i0 = texel_index(fi, W); i1 = texel_index(fi + F(1), W)
    j0 = texel_index(fj, H); j1 = texel_index(fj + F(1), H)
    t00 = tex[j0, i0]; t10 = tex[j0, i1]; t01 = tex[j1, i0]; t11 = tex[j1, i1]
    one = F(1)
    if weights == "mix":
        return (t00 * (one - a) + t10 * a) * (one - b) + (t01 * (one - a) + t11 * a) * b
    w00 = (one - a) * (one - b); w10 = a * (one - b); w01 = (one - a) * b; w11 = a * b
    return ((w00 * t00 + w10 * t10) + w01 * t01) + w11 * t11


def advect(vel, src, dt, dissipation, weights="gl", coord="uvn", own_texel=False, uv="cell"):
    """One advection blit: velocity (H, W, 2) carries src (Hs, Ws, C); returns (Hs, Ws, C) fp32.
    uv: the fragment centres (cell_uv)."""
    vel = np.ascontiguousarray(vel, F); src = np.ascontiguousarray(src, F)
    H, W = vel.shape[:2]
    Hs, Ws, C = src.shape
    tsx, tsy = F(1.0 / W), F(1.0 / H)
    dt = F(dt)
    decay = F(1) + F(dissipation) * dt
    uvx_row = cell_uv(Ws, uv); uvy_all = cell_uv(Hs, uv)
    out = np.empty((Hs, Ws, C), F)
    with np.errstate(all="ignore"):
        for r0 in range(0, Hs, ROWS):
            r1 = min(r0 + ROWS, Hs)
            uvx = np.broadcast_to(uvx_row, (r1 - r0, Ws))
            uvy = np.broadcast_to(uvy_all[r0:r1, None], (r1 - r0, Ws))
            if own_texel and (Hs, Ws) == (H, W):
                vv = vel[r0:r1]
            else:
                vv = fetch(vel, uvx, uvy, weights, coord)
            cx = uvx - (dt * vv[..., 0]) * tsx
            cy = uvy - (dt * vv[..., 1]) * tsy
            out[r0:r1] = fetch(src, cx, cy, weights, coord) / decay
    return out


class LinearOracleSim(O.OracleSim):
    """OracleSim whose two advection blits are `advect` above: the reference's step() (S:1231-1294) on a
    device with float linear filtering.  Splats and every other pass are the C oracle's."""

    def step(self, dt):
        dt = float(np.float32(dt))
        self.curl = self._st(O.curl(self.velocity))
        self.velocity = self._st(O.vorticity(self.velocity, self.curl, self.CURL, dt))
        self.divergence = self._st(O.divergence(self.velocity))
        self.pressure = self._st(O.clear(self.pressure, self.PRESSURE))
        if self.half_storage:
            for _ in range(self.PRESSURE_ITERATIONS):
                self.pressure = self._st(O.jacobi(self.pressure, self.divergence, 1))
        else:
            self.pressure = O.jacobi(self.pressure, self.divergence, self.PRESSURE_ITERATIONS)
        self.velocity = self._st(O.gradient_subtract(self.pressure, self.velocity))
        self.velocity = self._st(advect(self.velocity, self.velocity, dt, self.VELOCITY_DISSIPATION))
        self.dye = self._st(advect(self.velocity, self.dye, dt, self.DENSITY_DISSIPATION))
