"""ctypes binding of the CPU oracle (oracle/libfluid_oracle.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  Nothing under webgl_fluid_simulation_b200/ imports it.

Parity status: UNPINNED BY THE REFERENCE (it has no tests or fixtures and cannot run here);
pinned against known-answer tests and against tests/golden/*.npz, which oracle/glsl_exec.py
produced by executing the reference's own GLSL source text (see that file).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfluid_oracle.so")


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "fluid_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


_lib = None
_f = C.POINTER(C.c_float)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO)
        i, f, sz = C.c_int, C.c_float, C.c_size_t
        L.oracle_curl.argtypes = [_f, _f, i, i]
        L.oracle_vorticity.argtypes = [_f, _f, _f, i, i, f, f]
        L.oracle_divergence.argtypes = [_f, _f, i, i]
        L.oracle_clear.argtypes = [_f, _f, sz, f]
        L.oracle_jacobi.argtypes = [_f, _f, _f, i, i]
        L.oracle_jacobi_iters.argtypes = [_f, _f, _f, i, i, i]
        L.oracle_copy_rows.argtypes = [_f, _f, i, i]; L.oracle_copy_rows.restype = None
        L.oracle_gradient_subtract.argtypes = [_f, _f, _f, i, i]
        L.oracle_advect.argtypes = [_f, i, i, _f, _f, i, i, i, f, f]
        L.oracle_splat.argtypes = [_f, _f, i, i, i, f, f, f, _f, f]
        L.oracle_resample.argtypes = [_f, i, i, _f, i, i, i]
        L.oracle_round_half.argtypes = [_f, sz]
        L.oracle_display.argtypes = [_f, i, i, _f, i, i, i, _f, i, f]; L.oracle_display.restype = None
        # the post-FX blits, one per shader pass (render_postfx, tests/display_model.py)
        L.oracle_bloom_prefilter.argtypes = [_f, i, i, _f, i, i, f, f, f, f]
        L.oracle_box4.argtypes = [_f, i, i, _f, i, i, f, i]
        L.oracle_sunrays_mask.argtypes = [_f, _f, i, i]
        L.oracle_sunrays.argtypes = [_f, i, i, _f, i, i, f]
        L.oracle_blur3.argtypes = [_f, _f, i, i, f, f]
        L.oracle_display_full.argtypes = [_f, i, i, _f, i, i, _f, i, i, _f, i, i, _f, i, i, _f, i, f]
        L.oracle_num_threads.restype = i
        for fn in (L.oracle_curl, L.oracle_vorticity, L.oracle_divergence, L.oracle_clear,
                   L.oracle_jacobi, L.oracle_jacobi_iters, L.oracle_gradient_subtract,
                   L.oracle_advect, L.oracle_splat, L.oracle_resample, L.oracle_round_half,
                   L.oracle_bloom_prefilter, L.oracle_box4, L.oracle_sunrays_mask, L.oracle_sunrays,
                   L.oracle_blur3, L.oracle_display_full):
            fn.restype = None
        _lib = L
    return _lib


def _p(a: np.ndarray):
    assert a.dtype == np.float32 and a.flags.c_contiguous
    return a.ctypes.data_as(_f)


def _c(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def num_threads() -> int:
    return int(lib().oracle_num_threads())


def usable_cores() -> int:
    """Cores this process can actually USE: the affinity mask, capped by the cgroup CPU quota
    (a container may see 128 CPUs in its mask and be throttled to a few cores' worth of time —
    an OpenMP team sized by the mask then runs 10-100x slower and erratically)."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    n = min(n, max(1, int(float(txt[0]) / float(txt[1]) + 0.5)))
            else:
                q = int(txt[0])
                if q > 0:
                    per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                    n = min(n, max(1, int(q / per + 0.5)))
            break
        except Exception:
            continue
    return n


def use_all_cores(n: int | None = None) -> int:
    """Size the OpenMP team to the cores this process may use (torchrun sets OMP_NUM_THREADS=1).
    Pass `n` when the count was taken earlier: with OMP_PROC_BIND set, an OpenMP runtime binds the
    initial thread when it loads, after which the affinity mask of this thread is a single core."""
    n = usable_cores() if n is None else int(n)
    L = lib()
    L.oracle_set_num_threads.argtypes = [C.c_int]; L.oracle_set_num_threads.restype = None
    L.oracle_set_num_threads(int(n))
    return num_threads()


# Array conventions: scalar fields are (H, W); velocity (H, W, 2); dye (Hd, Wd, 4); row 0 = bottom.

def curl(v):
    v = _c(v); H, W, _ = v.shape
    out = np.empty((H, W), np.float32)
    lib().oracle_curl(_p(v), _p(out), W, H)
    return out


def vorticity(v, curl_f, curl_k, dt):
    v = _c(v); curl_f = _c(curl_f); H, W, _ = v.shape
    out = np.empty_like(v)
    lib().oracle_vorticity(_p(v), _p(curl_f), _p(out), W, H, curl_k, dt)
    return out


def divergence(v):
    v = _c(v); H, W, _ = v.shape
    out = np.empty((H, W), np.float32)
    lib().oracle_divergence(_p(v), _p(out), W, H)
    return out


def clear(p, value):
    p = _c(p)
    out = np.empty_like(p)
    lib().oracle_clear(_p(p), _p(out), p.size, value)
    return out


def jacobi(p, div, iters=1):
    p = _c(p).copy(); div = _c(div); H, W = p.shape
    tmp = np.empty_like(p)
    lib().oracle_jacobi_iters(_p(p), _p(tmp), _p(div), W, H, int(iters))
    return p


def gradient_subtract(p, v):
    p = _c(p); v = _c(v); H, W = p.shape
    out = np.empty_like(v)
    lib().oracle_gradient_subtract(_p(p), _p(v), _p(out), W, H)
    return out


def advect(vel, src, dt, dissipation):
    vel = _c(vel); src = _c(src)
    H, W, _ = vel.shape
    Hs, Ws, Cc = src.shape
    out = np.empty_like(src)
    lib().oracle_advect(_p(vel), W, H, _p(src), _p(out), Ws, Hs, Cc, dt, dissipation)
    return out


def splat(base, aspect, x, y, color3, radius):
    base = _c(base); Hh, Ww, Cc = base.shape
    out = np.empty_like(base)
    col = np.asarray(color3, np.float32)
    lib().oracle_splat(_p(base), _p(out), Ww, Hh, Cc, aspect, x, y, _p(col), radius)
    return out


def resample(src, Wd, Hd):
    src = _c(src); Hs, Ws, Cc = src.shape
    out = np.empty((Hd, Wd, Cc), np.float32)
    lib().oracle_resample(_p(src), Ws, Hs, _p(out), Wd, Hd, Cc)
    return out


BG_COLOR, BG_CHECKERBOARD, BG_NONE = 0, 1, 2   # what drawDisplay is blended over (render(), S:1296-1317)


def display(dye, w, h, shading=True, back_rgb=(0.0, 0.0, 0.0), background=BG_COLOR, aspect=None):
    """render() with bloom / sunrays off: (h, w, 4) float RGBA, row 0 = bottom.  background:
    BG_COLOR = drawColor(BACK_COLOR); BG_CHECKERBOARD = TRANSPARENT on the screen (S:1325-1329);
    BG_NONE = TRANSPARENT into a capture target (blending disabled)."""
    dye = _c(dye); Hd, Wd, _ = dye.shape
    out = np.empty((h, w, 4), np.float32)
    back = np.asarray(back_rgb, np.float32)
    lib().oracle_display(_p(dye), Wd, Hd, _p(out), w, h, 1 if shading else 0, _p(back), int(background),
                         float(w / h if aspect is None else aspect))
    return out


def render_postfx(dye, w, h, dither, cfg=None, back_rgb=(0.0, 0.0, 0.0), background=0, aspect=None):
    """render(null) with SHADING + BLOOM + SUNRAYS (reference desktop defaults S:70-84): applyBloom
    (S:1350-1394), applySunrays + blur (S:1396-1419), drawColor + drawDisplay (S:1296-1348), FBO
    sizes from getResolution (S:1012-1043).  dither: (dh, dw, 3) float in [0,1], row 0 = first image row (no UNPACK_FLIP_Y)."""
    L = lib()
    c = dict(BLOOM_ITERATIONS=8, BLOOM_RESOLUTION=256, BLOOM_INTENSITY=0.8, BLOOM_THRESHOLD=0.6,
             BLOOM_SOFT_KNEE=0.7, SUNRAYS_RESOLUTION=196, SUNRAYS_WEIGHT=1.0)
    c.update(cfg or {})
    dye = _c(dye); Hd, Wd, _ = dye.shape
    dither = _c(dither)

    def get_resolution(res):                                  # S:1612-1624
        ar = w / h
        if ar < 1: ar = 1.0 / ar
        mn, mx = int(np.floor(res + 0.5)), int(np.floor(res * ar + 0.5))
        return (mx, mn) if w > h else (mn, mx)

    bw, bh = get_resolution(c["BLOOM_RESOLUTION"])
    bloom = np.zeros((bh, bw, 4), np.float32); bloom[..., 3] = 1.0        # createFBO clears to (0,0,0,1)
    sizes = []
    for k in range(c["BLOOM_ITERATIONS"]):
        pw, ph = bw >> (k + 1), bh >> (k + 1)
        if pw < 2 or ph < 2: break
        sizes.append((pw, ph))
    pyr = []
    if len(sizes) >= 2:
        knee = c["BLOOM_THRESHOLD"] * c["BLOOM_SOFT_KNEE"] + 0.0001
        L.oracle_bloom_prefilter(_p(dye), Wd, Hd, _p(bloom), bw, bh, c["BLOOM_THRESHOLD"] - knee, knee * 2,
                                 0.25 / knee, c["BLOOM_THRESHOLD"])
        last, lw, lh = bloom, bw, bh
        for pw, ph in sizes:
            t = np.empty((ph, pw, 4), np.float32)
            L.oracle_box4(_p(last), lw, lh, _p(t), pw, ph, 1.0, 0)
            pyr.append(t); last, lw, lh = t, pw, ph
        for k in range(len(pyr) - 2, -1, -1):
            pw, ph = sizes[k]
            L.oracle_box4(_p(last), lw, lh, _p(pyr[k]), pw, ph, 1.0, 1)
            last, lw, lh = pyr[k], pw, ph
        L.oracle_box4(_p(last), lw, lh, _p(bloom), bw, bh, c["BLOOM_INTENSITY"], 0)
    sw, sh = get_resolution(c["SUNRAYS_RESOLUTION"])
    mask = np.empty_like(dye)
    L.oracle_sunrays_mask(_p(dye), _p(mask), Wd, Hd)
    sun = np.empty((sh, sw), np.float32); tmp = np.empty_like(sun)
    L.oracle_sunrays(_p(mask), Wd, Hd, _p(sun), sw, sh, c["SUNRAYS_WEIGHT"])
    L.oracle_blur3(_p(sun), _p(tmp), sw, sh, 1.0 / sw, 0.0)
    L.oracle_blur3(_p(tmp), _p(sun), sw, sh, 0.0, 1.0 / sh)
    out = np.empty((h, w, 4), np.float32)
    back = np.asarray(back_rgb, np.float32)
    L.oracle_display_full(_p(dye), Wd, Hd, _p(bloom), bw, bh, _p(sun), sw, sh, _p(dither), dither.shape[1],
                          dither.shape[0], _p(out), w, h, _p(back), int(background), float(w / h if aspect is None else aspect))
    return dict(target=out, bloom=bloom, sunrays=sun, mask_alpha=mask[..., 3].copy(), pyramid=pyr)


def round_half(a):
    a = _c(a).copy()
    lib().oracle_round_half(_p(a), a.size)
    return a


def correct_radius(splat_radius: float, aspect: float) -> np.float32:
    """correctRadius(config.SPLAT_RADIUS / 100.0), S:1447 + S:1457-1462 (double math, fp32 uniform)."""
    r = float(splat_radius) / 100.0          # JS doubles all the way ...
    if aspect > 1:
        r *= float(aspect)
    return np.float32(r)                     # ... narrowed once, by gl.uniform1f


class OracleSim:
    """The reference's global simulation state + step()/splat(), on the CPU (S:950-954, S:1231-1294,
    S:1441-1455).  Orchestrated here in Python over the per-pass C functions so tests can peek at
    every intermediate field; the C oracle_sim_* twin (used for CPU timing) is checked against it."""

    def __init__(self, W, H, Wd, Hd, half_storage=False, **cfg):
        self.W, self.H, self.Wd, self.Hd = W, H, Wd, Hd
        self.DENSITY_DISSIPATION = 1.0
        self.VELOCITY_DISSIPATION = 0.2
        self.PRESSURE = 0.8
        self.PRESSURE_ITERATIONS = 20
        self.CURL = 30.0
        self.SPLAT_RADIUS = 0.25
        self.aspect = W / H
        self.half_storage = half_storage
        for k, v in cfg.items():
            assert hasattr(self, k), k
            setattr(self, k, v)
        self.velocity = np.zeros((H, W, 2), np.float32)
        self.dye = np.zeros((Hd, Wd, 4), np.float32)
        self.dye[..., 3] = 1.0  # clearColor (0,0,0,1): S:136, S:1059
        self.pressure = np.zeros((H, W), np.float32)
        self.divergence = np.zeros((H, W), np.float32)
        self.curl = np.zeros((H, W), np.float32)

    def _st(self, a):
        return round_half(a) if self.half_storage else a

    def step(self, dt):
        dt = float(np.float32(dt))
        self.curl = self._st(curl(self.velocity))
        self.velocity = self._st(vorticity(self.velocity, self.curl, self.CURL, dt))
        self.divergence = self._st(divergence(self.velocity))
        self.pressure = self._st(clear(self.pressure, self.PRESSURE))
        if self.half_storage:
            for _ in range(self.PRESSURE_ITERATIONS):
                self.pressure = self._st(jacobi(self.pressure, self.divergence, 1))
        else:
            self.pressure = jacobi(self.pressure, self.divergence, self.PRESSURE_ITERATIONS)
        self.velocity = self._st(gradient_subtract(self.pressure, self.velocity))
        self.velocity = self._st(advect(self.velocity, self.velocity, dt, self.VELOCITY_DISSIPATION))
        self.dye = self._st(advect(self.velocity, self.dye, dt, self.DENSITY_DISSIPATION))

    def splat(self, x, y, dx, dy, r, g, b):
        radius = correct_radius(self.SPLAT_RADIUS, self.aspect)
        self.velocity = self._st(splat(self.velocity, self.aspect, x, y, (dx, dy, 0.0), radius))
        self.dye = self._st(splat(self.dye, self.aspect, x, y, (r, g, b), radius))


class OracleSimC:
    """Thin handle over the C oracle_sim_* API (whole step in C; used for CPU timing)."""

    class _S(C.Structure):
        _fields_ = [("W", C.c_int), ("H", C.c_int), ("Wd", C.c_int), ("Hd", C.c_int),
                    ("density_dissipation", C.c_float), ("velocity_dissipation", C.c_float),
                    ("pressure", C.c_float), ("curl", C.c_float), ("splat_radius", C.c_float),
                    ("aspect", C.c_float), ("pressure_iterations", C.c_int),
                    ("half_storage", C.c_int),
                    ("v", _f), ("v2", _f), ("dye", _f), ("dye2", _f), ("p", _f), ("p2", _f),
                    ("div", _f), ("curl_f", _f)]

    def __init__(self, W, H, Wd, Hd):
        L = lib()
        L.oracle_sim_create.restype = C.POINTER(self._S)
        L.oracle_sim_create.argtypes = [C.c_int] * 4
        L.oracle_sim_destroy.argtypes = [C.POINTER(self._S)]
        L.oracle_sim_step.argtypes = [C.POINTER(self._S), C.c_float]
        L.oracle_sim_splat.argtypes = [C.POINTER(self._S)] + [C.c_float] * 7
        self._L = L
        self.s = L.oracle_sim_create(W, H, Wd, Hd)

    def step(self, dt):
        self._L.oracle_sim_step(self.s, dt)

    def splat(self, x, y, dx, dy, r, g, b):
        self._L.oracle_sim_splat(self.s, x, y, dx, dy, r, g, b)

    def field(self, name):
        s = self.s.contents
        shp = {"velocity": (s.H, s.W, 2), "dye": (s.Hd, s.Wd, 4), "pressure": (s.H, s.W),
               "divergence": (s.H, s.W), "curl": (s.H, s.W)}[name]
        ptr = {"velocity": s.v, "dye": s.dye, "pressure": s.p, "divergence": s.div,
               "curl": s.curl_f}[name]
        return np.ctypeslib.as_array(ptr, shape=(int(np.prod(shp)),)).reshape(shp).copy()

    def close(self):
        if self.s:
            self._L.oracle_sim_destroy(self.s)
            self.s = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
