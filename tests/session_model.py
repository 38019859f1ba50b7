"""The oracle side of one library handle over a whole session, and the seeded operation generator that
drives it.  Test infrastructure (CPU only).

A session is a list of operations, each a plain tuple, applied in order to a handle and to a
SessionModel in lockstep (tests/test_gpu_session.py).  The model holds what the handle should hold --
velocity, dye, pressure, divergence, curl, sizes, canvas, config, handle mode -- and has one method per
operation, built from what already exists:

  step                  oracle.OracleSim (fp32 or half_storage), its config attributes set live;
                        linear_advection_model.LinearOracleSim in the LINEAR modes
  resize                oracle.resample (+ round_half in half storage) when a size changes, the NEAREST
                        copy display_model.resize in the NEAREST modes; pressure, divergence and curl start
                        over at zero (fluid_resize, S:982-1010 + S:1116-1126)
  pressure_solve, jacobi, pressure_solve_host
                        oracle.clear + oracle.jacobi; in half storage every blit rounded to fp16, the
                        host inputs too (they travel through fluid_write)
  splat, splats         splat_model.splat_interval: the handle's result is checked against the interval,
                        then ADOPTED, so that later operations stay comparable bit for bit
  render, capture       display_model with the handle's storage and sampler; read-only

A handle mode (MODES) is its storage and its sampler.  The storage picks the schedule, the generated
operations and the data they write; the sampler changes only the model's step, resize and draws.

Every array an operation writes is derived from the operation tuple alone (op_data), so a logged
session can be replayed from its log.

Data: every session writes the special values of sim_harness.special_fields (+-0, subnormals, +-inf, NaN
and a band of large pressure) into velocity, pressure and divergence, rounded to fp16 in half storage; fp32
sessions add large finite values, and their dye may hold inf and NaN too.
"""
from __future__ import annotations

import numpy as np

import display_model as M
import splat_model as SM
from linear_advection_model import LinearOracleSim
from oracle import oracle as O
from sim_harness import nasty_fields, nasty_records, special_fields

F32 = np.float32
# handle modes: mode -> (half, sampler).  half: FLUID_FLAG_HALF_STORAGE | FLUID_FLAG_HALF_POSTFX (HALF_SCHEDULE);
# sampler "manual": the MANUAL advection and LINEAR draws of an ordinary handle, "linear":
# FLUID_FLAG_LINEAR_ADVECTION (with half storage the desktop browser's configuration), "nearest":
# FLUID_FLAG_NEAREST_FILTERING (a WebGL device without float linear filtering: NEAREST draws and resize copy)
MODES = {
    "fp32": (False, "manual"),
    "half": (True, "manual"),
    "linear": (False, "linear"),
    "desktop": (True, "linear"),
    "nearest": (False, "nearest"),
    "nearest_half": (True, "nearest"),
}


def is_half(mode: str) -> bool:
    return MODES[mode][0]
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
SIM_KEYS = ("DENSITY_DISSIPATION", "VELOCITY_DISSIPATION", "PRESSURE", "PRESSURE_ITERATIONS", "CURL", "SPLAT_RADIUS")
TINY = 2.0 ** -123          # divergence below this defeats the blocked Jacobi's contracted tail (jacobi.cuh)
BACK = {"r": 10, "g": 20, "b": 30}
BACK_RGB = (10 / 255, 20 / 255, 30 / 255)
# small post-FX targets keep the oracle's chains cheap; BLOOM_ITERATIONS 8 still builds a pyramid
FXCFG = dict(BLOOM_RESOLUTION=32, SUNRAYS_RESOLUTION=24, CAPTURE_RESOLUTION=40)
DT_CLAMP = 0.016666         # calcDeltaTime's min(dt, 0.016666), S:1188-1194

# ---- sizes -------------------------------------------------------------------------------------------
# (W, H, Wd, Hd, canvas_w, canvas_h, classes): classes name what fluid.cu selects at that size, as the
# suite's other tests establish it (sim_harness STREAM_SHAPES / TILED_SHAPES, test_gpu_parity HALF_SIZES,
# test_gpu_fast_paths ADVECT_SHAPES, test_host_pressure_solve_banded_pipeline).  They are labels, not
# a restatement of the selection rules: the GPU test checks them through fluid_stat.
#   stream / tiled       curl-vorticity-divergence + gradientSubtract kernels
#   adv4_same / adv4 / adv1_pow2 / ragged     velocity + dye advection kernels
#   blocked / scalar     fp32 Jacobi; half8 / half_scalar: hs::jacobi8_kernel / jacobi_scalar_kernel<StoreHalf>
#   banded / one_piece   fluid_pressure_solve_host at <= 64 iterations
#   degenerate           a grid of fewer than 8 columns or rows
FP32_SCHEDULE = [
    (64, 64, 64, 64, 160, 160, {"tiled", "adv1_pow2", "blocked", "one_piece"}),
    (1024, 512, 1024, 512, 200, 100, {"stream", "adv4_same", "blocked", "banded"}),
    (1024, 512, 2048, 1024, 200, 100, {"stream", "adv4", "blocked", "banded", "dye_only"}),
    (1024, 512, 2048, 1024, 200, 100, {"stream", "adv4", "blocked", "banded", "same_size"}),
    (520, 33, 2048, 1024, 180, 60, {"tiled", "ragged", "blocked", "one_piece", "sim_only"}),
    (130, 66, 195, 99, 130, 66, {"tiled", "ragged", "scalar", "one_piece"}),
    (964, 600, 964, 600, 160, 100, {"stream", "ragged", "blocked", "banded"}),
    (7, 5, 9, 6, 70, 50, {"tiled", "ragged", "scalar", "one_piece", "degenerate"}),
    (1, 9, 3, 27, 20, 180, {"tiled", "ragged", "scalar", "one_piece", "degenerate"}),
    (1024, 512, 1024, 512, 100, 200, {"stream", "adv4_same", "blocked", "banded", "earlier_size"}),
    (64, 64, 64, 64, 160, 160, {"tiled", "adv1_pow2", "blocked", "one_piece", "earlier_size"}),
]
HALF_SCHEDULE = [
    (64, 64, 128, 128, 160, 160, {"half8", "one_piece"}),
    (264, 40, 528, 80, 198, 30, {"half8", "one_piece"}),
    (520, 33, 780, 50, 180, 60, {"half8", "one_piece"}),
    (520, 33, 780, 50, 180, 60, {"half8", "one_piece", "same_size"}),
    (100, 60, 780, 50, 180, 60, {"half_scalar", "one_piece", "sim_only"}),
    (100, 60, 150, 90, 180, 60, {"half_scalar", "one_piece", "dye_only"}),
    (7, 5, 9, 6, 70, 50, {"half_scalar", "one_piece", "degenerate"}),
    (1, 9, 3, 27, 20, 180, {"half_scalar", "one_piece", "degenerate"}),
    (264, 40, 528, 80, 120, 160, {"half8", "one_piece", "earlier_size"}),
    (64, 64, 128, 128, 160, 160, {"half8", "one_piece", "earlier_size"}),
]


def schedule(half: bool):
    return HALF_SCHEDULE if half else FP32_SCHEDULE


# ---- operations --------------------------------------------------------------------------------------
# ("step", dt)                          ("splat", seed)              ("splats", n, seed)
# ("write", field, seed)                ("write_tiny_div", seed)     ("pressure_solve",)
# ("jacobi", k)                         ("host_solve", iters, seed)  ("config", key, value)
# ("jacobi_block", k)                   ("resize", schedule index)
# ("render", keywords, transparent, target)                          ("capture", keywords, transparent)
KINDS = ("step", "splat", "splats", "write", "write_tiny_div", "pressure_solve", "jacobi", "host_solve", "config",
         "jacobi_block", "resize", "render", "capture")
CONFIG_VALUES = {
    "CURL": (0.0, 12.5, 30.0, 55.0),
    "PRESSURE": (0.0, 0.8, 1.0, 0.33),
    "PRESSURE_ITERATIONS": (0, 1, 13, 14, 20, 50),
    "VELOCITY_DISSIPATION": (0.0, 0.2, 1.0, 4.0),
    "DENSITY_DISSIPATION": (0.0, 1.0, 0.5, 4.0),
    "SPLAT_RADIUS": (0.25, 0.1, 1.5),
}
JACOBI_BLOCKS = (0, 1, 7, 13)
SPLATS_N = (2, 5, 127, 128, 129, 200)
TINY_DT = 1e-30
# the committed sessions of each mode: together its seeds reach every class (test_session_model_cpu.py)
SEEDS = {
    "fp32": (3, 10, 76, 4, 5),
    "half": (1, 3, 12, 2, 4),
    "linear": (100, 103, 183),
    "desktop": (100, 101, 104),
    "nearest": (101, 104, 249),
    "nearest_half": (102, 103, 106),
}
N_OPS = 40


def random_dt(rng) -> float:
    k = int(rng.integers(4))
    if k == 0:
        return 0.0
    if k == 1:
        return TINY_DT
    if k == 2:
        return float(np.float32(rng.uniform(0.003, DT_CLAMP)))
    return DT_CLAMP


def generate(seed: int, half: bool, n_ops: int) -> list[tuple]:
    """A seeded session of about n_ops operations.  Resizes walk the storage mode's whole schedule in
    order (so every boundary is crossed both ways and the session ends at its starting size); the
    operations between them are drawn at random."""
    rng = np.random.default_rng(seed)
    sched = schedule(half)
    per = max(2, n_ops // len(sched))
    ops: list[tuple] = []
    si = 0
    weights = np.array([6, 2, 1.5, 2, 0 if half else 0.7, 1.5, 1, 1, 4, 1.5, 0, 1.2, 0.8])
    weights = weights / weights.sum()
    # config values and JACOBI_BLOCK come from shuffled decks, so that a session spreads over them
    deck = [(k, v) for k, vals in CONFIG_VALUES.items() for v in vals]
    deck = [deck[i] for i in rng.permutation(len(deck))]
    blocks = [JACOBI_BLOCKS[i] for i in rng.permutation(len(JACOBI_BLOCKS))]
    dealt = {"config": 0, "jacobi_block": 0}

    def draw():
        kind = KINDS[int(rng.choice(len(KINDS), p=weights))]
        s = int(rng.integers(1 << 30))
        if kind == "step":
            return ("step", random_dt(rng))
        if kind == "splat":
            return ("splat", s)
        if kind == "splats":
            W, H, Wd, Hd = sched[si][:4]
            big = Wd * Hd <= 1 << 16                 # the interval of 200 records costs O(records x texels)
            n = int(rng.choice(SPLATS_N if big else SPLATS_N[:2]))
            return ("splats", n, s)
        if kind == "write":
            return ("write", FIELDS[int(rng.integers(5))], s)
        if kind == "write_tiny_div":
            return ("write_tiny_div", s)
        if kind == "pressure_solve":
            return ("pressure_solve",)
        if kind == "jacobi":
            return ("jacobi", int(rng.choice([0, 1, 5, 13, 14, 27])))
        if kind == "host_solve":
            return ("host_solve", int(rng.choice([0, 1, 13, 20, 50])), s)
        if kind == "config":
            dealt["config"] += 1
            return ("config",) + deck[(dealt["config"] - 1) % len(deck)]
        if kind == "jacobi_block":
            dealt["jacobi_block"] += 1
            return ("jacobi_block", blocks[(dealt["jacobi_block"] - 1) % len(blocks)])
        kw = int(rng.integers(8))
        if kind == "render":
            return ("render", kw, bool(rng.integers(2)), bool(rng.integers(4) == 0))
        return ("capture", kw, bool(rng.integers(2)))

    for si in range(len(sched)):
        if si:
            ops.append(("resize", si))
        for _ in range(per):
            ops.append(draw())
        ops.append(("step", random_dt(rng)))        # every size is stepped at least once
    return ops


def op_classes(ops, half: bool) -> set:
    """What a session reaches: the operation kinds, config keys, JACOBI_BLOCK values, splat counts on both
    sides of the 128-record launch, dt kinds and the size classes of every size it steps at."""
    sched = schedule(half)
    out = set()
    si = 0
    stepped = set()
    for op in ops:
        out.add(op[0])
        if op[0] == "resize":
            si = op[1]
            W, H, Wd, Hd = sched[si][:4]
            pW, pH, pWd, pHd = sched[si - 1][:4]
            out.add("resize_up" if W * H > pW * pH else "resize_down" if W * H < pW * pH else "resize_same_sim")
            if sched[si][4] * sched[si - 1][5] != sched[si][5] * sched[si - 1][4]:
                out.add("canvas_aspect_change")
        elif op[0] == "config":
            out.add(f"config:{op[1]}")
            if op[1] == "PRESSURE_ITERATIONS":
                out.add(f"iters:{op[2]}")
        elif op[0] == "jacobi_block":
            out.add(f"jacobi_block:{op[1]}")
        elif op[0] == "splats":
            out.add("splats<=128" if op[1] <= 128 else "splats>128")
        elif op[0] == "step":
            out.add("dt:0" if op[1] == 0 else "dt:tiny" if op[1] == TINY_DT else "dt:clamp" if op[1] == DT_CLAMP else "dt:jitter")
            stepped.add(si)
        elif op[0] == "render":
            if op[1] & M.SUNRAYS:
                out.add("render:sunrays")
            if op[1] & M.BLOOM:
                out.add("render:bloom")
            if op[2]:
                out.add("render:transparent")
        elif op[0] == "write":
            out.add(f"write:{op[1]}")
    for si in stepped:
        out |= {f"size:{c}" for c in sched[si][6]}
    return out


# ---- the data an operation writes ---------------------------------------------------------------------
def fp32_special(a, rng, big):
    """Subnormals, signed zeros and large finite values sprinkled over `a` (finite only)."""
    flat = a.reshape(-1)
    specials = np.array([-0.0, 0.0, 1e-40, -3e-39, 1.4e-45, big, -big], F32)
    k = max(1, flat.size // 9)
    flat[rng.integers(0, flat.size, k)] = rng.choice(specials, k)
    return a


def field_data(name, W, H, Wd, Hd, seed, half: bool):
    """The array a ("write", name, seed) operation writes."""
    rng = np.random.default_rng(seed)
    if half:
        v, dye, p = special_fields(O, W, H, Wd, Hd, seed)
        if name == "velocity":
            return v
        if name == "dye":
            return dye
        if name == "pressure":
            return p
        v2, _, _ = nasty_fields(W, H, 1, 1, seed + 1)
        return O.round_half(v2[..., 0] if name == "divergence" else v2[..., 1] * F32(0.01))
    if name == "velocity":
        return fp32_special(special_fields(O, W, H, 1, 1, seed, half=False)[0], rng, F32(1e30))
    if name == "dye":
        _, dye, _ = nasty_fields(1, 1, Wd, Hd, seed)
        return dye
    if name == "pressure":
        return fp32_special(special_fields(O, W, H, 1, 1, seed, half=False)[2], rng, F32(1e20))
    if name == "divergence":
        v2, _, _ = nasty_fields(W, H, 1, 1, seed + 1)
        return fp32_special(v2[..., 0], rng, F32(1e20))
    _, _, c = nasty_fields(W, H, 1, 1, seed)                  # curl: recomputed before any pass reads it
    c.reshape(-1)[rng.integers(0, c.size, max(1, c.size // 9))] = np.nan
    return c


def tiny_divergence(W, H, seed):
    """Ordinary divergence with a patch (and a sprinkle) of values in (0, 2^-123)."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(-1, 1, (H, W)).astype(F32)
    tiny = (rng.integers(1, 2 ** 23, (H, W)) * 2.0 ** -149).astype(F32) * rng.choice([-1, 1], (H, W)).astype(F32)
    r0, c0 = H // 3, W // 4
    d[r0:r0 + max(1, H // 4), c0:c0 + max(1, W // 3)] = tiny[r0:r0 + max(1, H // 4), c0:c0 + max(1, W // 3)]
    pick = rng.random((H, W)) < 0.02
    d[pick] = tiny[pick]
    assert ((d != 0) & (np.abs(d) < F32(TINY))).any()
    return d


def splat_records(n, seed):
    """n records: ordinary pointer splats mixed with splat_model's nasty ones."""
    rng = np.random.default_rng(seed)
    r = np.empty((n, 7), F32)
    r[:, 0:2] = rng.uniform(0, 1, (n, 2))
    r[:, 2:4] = rng.uniform(-500, 500, (n, 2))
    r[:, 4:7] = rng.uniform(0, 1.5, (n, 3))
    nasty = rng.random(n) < 0.3
    r[nasty] = nasty_records(int(nasty.sum()), seed + 1)
    return r


def host_inputs(W, H, seed, half: bool):
    """(divergence, pressure) handed to fluid_pressure_solve_host."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(-1, 1, (H, W)).astype(F32)
    p = rng.standard_normal((H, W)).astype(F32)
    d[H // 2, W // 3] = F32(2.0 ** -130)                      # a tiny value: flagged by the scan of its band
    if half:
        d = d * F32(4.0)
    return d, p


# ---- the model ---------------------------------------------------------------------------------------
class SessionModel:
    """What one handle of `mode` (MODES) holds.  config: the simulation keys the host mirror pushes live
    (SIM_KEYS)."""

    def __init__(self, W, H, Wd, Hd, canvas, mode="fp32", config=None):
        self.mode = mode
        self.half, sampler = MODES[mode]
        self.nearest = sampler == "nearest"
        sim = LinearOracleSim if sampler == "linear" else O.OracleSim
        self.sim = sim(W, H, Wd, Hd, half_storage=self.half)
        self.canvas = tuple(canvas)
        self.config = {k: getattr(self.sim, k) for k in SIM_KEYS}
        self.config.update(config or {})
        self.jacobi_block = 0

    # sizes and fields
    @property
    def sizes(self):
        return self.sim.W, self.sim.H, self.sim.Wd, self.sim.Hd

    def field(self, name) -> np.ndarray:
        return getattr(self.sim, name)

    def _st(self, a):
        a = np.ascontiguousarray(a, F32)
        return O.round_half(a) if self.half else a.copy()

    def _sync(self):
        for k in SIM_KEYS:
            setattr(self.sim, k, self.config[k])
        self.sim.aspect = self.canvas[0] / self.canvas[1]

    # operations
    def step(self, dt):
        self._sync()
        self.sim.step(dt)

    def write(self, name, a):
        setattr(self.sim, name, self._st(a))

    def _solve(self, p, iters, clear=True):
        """clear (PRESSURE * p) then `iters` sweeps, in the storage format."""
        if clear:
            p = self._st(O.clear(p, self.config["PRESSURE"]))
        if self.half:
            for _ in range(iters):
                p = self._st(O.jacobi(p, self.sim.divergence, 1))
            return p
        return O.jacobi(p, self.sim.divergence, iters) if iters else p

    def pressure_solve(self):
        self.sim.pressure = self._solve(self.sim.pressure, int(self.config["PRESSURE_ITERATIONS"]))

    def jacobi(self, k):
        self.sim.pressure = self._solve(self.sim.pressure, int(k), clear=False)

    def pressure_solve_host(self, div, p, iters) -> np.ndarray:
        """The pressure fluid_pressure_solve_host hands back (and leaves in the handle)."""
        self.sim.divergence = self._st(div)
        self.sim.pressure = self._solve(self._st(p), int(iters))
        return self.sim.pressure

    def _copy(self, a, W, H):
        """resizeFBO's copy of a field into W x H through the handle's sampler, in the storage format."""
        return M.resize(a, W, H, half=self.half) if self.nearest else self._st(O.resample(a, W, H))

    def resize(self, W, H, Wd, Hd, canvas):
        s = self.sim
        if (W, H) != (s.W, s.H):
            s.velocity = self._copy(s.velocity, W, H)
        if (Wd, Hd) != (s.Wd, s.Hd):
            s.dye = self._copy(s.dye, Wd, Hd)
        s.W, s.H, s.Wd, s.Hd = W, H, Wd, Hd
        s.pressure = np.zeros((H, W), F32)
        s.divergence = np.zeros((H, W), F32)
        s.curl = np.zeros((H, W), F32)
        self.canvas = tuple(canvas)

    def splat_interval(self, recs):
        """[lo, hi] of velocity and dye after the records (splat_model), at the canvas aspect."""
        cw, ch = self.canvas
        aspect, rad = SM.aspect_of(cw, ch), SM.radius_of(self.config["SPLAT_RADIUS"], cw, ch)
        with np.errstate(invalid="ignore", over="ignore"):
            return {n: SM.splat_interval(self.field(n), recs, aspect, rad, half=self.half) for n in ("velocity", "dye")}

    def adopt(self, velocity, dye):
        """After a splat inside its interval: the handle's bits become the model's."""
        self.sim.velocity = np.ascontiguousarray(velocity, F32).copy()
        self.sim.dye = np.ascontiguousarray(dye, F32).copy()

    def render(self, keywords, background, dither, fxcfg):
        """render() at the canvas size: display_model.render with the handle's storage and sampler (chains,
        target, and the powf interval lo / hi with BLOOM)."""
        w, h = self.canvas
        return M.render(self.sim.dye, w, h, dither, keywords, fxcfg, back_rgb=BACK_RGB, background=background,
                        aspect=w / h, nearest=self.nearest, half_targets=self.half, half_mask=self.half)

    def capture_size(self, capture_res):
        return M.get_resolution(capture_res, *self.canvas)

    def capture(self, keywords, transparent, dither, fxcfg, capture_res):
        """captureScreenshot(): display_model.capture with the handle's storage and sampler (rgba8, and the
        byte bracket lo / hi with BLOOM)."""
        cw, ch = self.canvas
        w, h = self.capture_size(capture_res)
        return M.capture(self.sim.dye, w, h, cw, ch, dither, keywords, transparent, BACK_RGB, cfg=fxcfg,
                         nearest=self.nearest, half_targets=self.half, half_mask=self.half)
