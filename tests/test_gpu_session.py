"""Whole sessions on one handle against the oracle: a seeded sequence of API calls -- steps, splats,
writes, pressure solves on the device and from the host, live config, resizes, renders and captures --
runs on a library handle and, in lockstep, on session_model.SessionModel.  After every operation all
five fields are compared with the model (bitwise, NaN in the same places), splats and frames against
their intervals; the launch counters confirm which kernels each size selects.

Every session also runs on a FLAG_NO_GRAPH twin: after every operation it must hold the graph handle's
bits and have made as many launches, which tells a step-graph cache fault from a model fault.

Sessions run in every handle mode of session_model.MODES: fp32 and half storage (HALF_STORAGE |
HALF_POSTFX), each with the MANUAL advection and LINEAR draws of an ordinary handle, with
FLUID_FLAG_LINEAR_ADVECTION (linear; desktop, the configuration the reference runs on a desktop browser)
and with FLUID_FLAG_NEAREST_FILTERING (nearest, nearest_half).

On failure the message carries the session's mode and seed, the index of the failing operation and the
log of operations so far; replay(pkg, mode, ops) runs a logged session again."""
import numpy as np
import pytest

import display_harness as DH
import display_model as M
import gamma_model as G
import session_model as S
import splat_model as SM
from conftest import bits_equal
from oracle import oracle as O
from sim_harness import same_bits
from webgl_fluid_simulation_b200 import slab

pytestmark = pytest.mark.gpu
STATS = ("jacobi_launches", "cvd_stream_launches", "gradient_stream_launches", "graph_captures", "jacobi_exact_streams",
         "advect4_launches")
FX = {k: S.FXCFG[k] for k in ("BLOOM_RESOLUTION", "SUNRAYS_RESOLUTION")}


def mode_flags(pkg, mode):
    """The flags a handle of session_model mode `mode` is made with."""
    half, sampler = S.MODES[mode]
    return ((pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX if half else 0)
            | (pkg.FLAG_LINEAR_ADVECTION if sampler == "linear" else 0)
            | (pkg.FLAG_NEAREST_FILTERING if sampler == "nearest" else 0))


@pytest.fixture(scope="module")
def pkg():
    import webgl_fluid_simulation_b200 as p
    O.build()
    O.use_all_cores()                      # the model steps 2048 x 1024 dye: size the OpenMP team to the quota
    return p


class Session:
    """A graph handle, its FLAG_NO_GRAPH twin and the model, driven one operation at a time."""

    def __init__(self, pkg, mode):
        self.pkg, self.mode = pkg, mode
        self.half = S.is_half(mode)
        self.sched = S.schedule(self.half)
        self.si = 0
        self.dither = DH.golden_dither()
        W, H, Wd, Hd, cw, ch, _ = self.sched[0]
        flags = mode_flags(pkg, mode)
        self.sims = [self._make(flags), self._make(flags | pkg.FLAG_NO_GRAPH)]
        self.model = S.SessionModel(W, H, Wd, Hd, (cw, ch), mode=mode)
        self.fresh = True                                 # no step since the handle was made or resized

    def _make(self, flags):
        W, H, Wd, Hd, cw, ch, _ = self.sched[0]
        s = self.pkg.FluidSimulation({"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}, canvas_width=cw,
                                     canvas_height=ch, flags=flags, sizes=(W, H, Wd, Hd))
        s.config.update(BACK_COLOR=S.BACK, **S.FXCFG)
        s.dithering = self.dither
        return s

    def close(self):
        for s in self.sims:
            s.close()

    # ---- helpers --------------------------------------------------------------------------------------
    @property
    def classes(self):
        return self.sched[self.si][6]

    def stats(self):
        return [{k: s.stat(k) for k in STATS} for s in self.sims]

    def solve_launches(self, iters):
        """Jacobi launches of one solve: the library's launch plan (slab.py mirrors it) on the sizes that run
        the blocked kernel, one sweep per launch on the others."""
        if "blocked" in self.classes:
            H = self.model.sizes[1]
            return len(slab.jacobi_launches(iters, slab.SlabPlan(H, 8, 0, 1).block(self.model.jacobi_block)))
        return iters

    def tiny_divergence(self):
        d = np.abs(self.model.field("divergence"))
        return bool(((d > 0) & (d < np.float32(S.TINY))).any())

    def exact_expected(self, iters):
        """A blocked solve of tiny divergence must send some warps to the exact tail."""
        return ("blocked" in self.classes and self.model.jacobi_block != 1 and iters > 0 and self.tiny_divergence())

    def check_fields(self):
        g, t = self.sims
        for n in S.FIELDS:
            got = g.readField(n)
            assert got.shape == self.model.field(n).shape, (n, got.shape, self.model.field(n).shape)
            assert same_bits(got, self.model.field(n)), f"{n} differs from the model"
            assert bits_equal(t.readField(n), got), f"{n}: the FLAG_NO_GRAPH twin differs from the graph handle"
        assert g.launch_count() == t.launch_count(), ("launch counts", g.launch_count(), t.launch_count())

    # ---- operations -----------------------------------------------------------------------------------
    def run(self, op):
        getattr(self, "op_" + op[0])(*op[1:])
        self.check_fields()

    def op_step(self, dt):
        before = self.stats()
        for s in self.sims:
            s.step(dt)
        self.model.step(dt)
        after = self.stats()
        iters = int(self.model.config["PRESSURE_ITERATIONS"])
        for k, (b, a) in enumerate(zip(before, after)):
            d = {n: a[n] - b[n] for n in STATS}
            assert d["jacobi_launches"] == self.solve_launches(iters), (k, d, iters, self.model.jacobi_block)
            streamed = "stream" in self.classes and not self.half
            assert d["cvd_stream_launches"] == int(streamed), (k, d)
            assert d["gradient_stream_launches"] == int(streamed), (k, d)
            # the 4-cell velocity and dye kernels: fp32 power-of-two grids at least 128 wide, either sampler
            four = bool({"adv4", "adv4_same"} & self.classes) and not self.half
            assert d["advect4_launches"] == 2 * four, (k, d)
            if k == 0 and self.fresh:
                assert d["graph_captures"] == 1, ("the first step after a resize must capture a new graph", d)
            if k == 1:
                assert a["graph_captures"] == 0
        self.fresh = False

    def op_splat(self, seed):
        self._splat(S.splat_records(1, seed), one=True)

    def op_splats(self, n, seed):
        self._splat(S.splat_records(n, seed), one=False)

    def _splat(self, recs, one):
        for s in self.sims:
            if one:
                r = [float(x) for x in recs[0]]
                s.splat(*r[:4], tuple(r[4:]))
            else:
                s.splats(recs)
        # read from both handles: a half-storage read launches a widen kernel, and the launch counts must match
        got, _ = ({n: s.readField(n) for n in ("velocity", "dye")} for s in self.sims)
        for n, (lo, hi) in self.model.splat_interval(recs).items():
            bad, first = SM.check_splat(got[n], lo, hi)
            assert bad == 0, (n, bad, first)
        self.model.adopt(got["velocity"], got["dye"])

    def op_write(self, name, seed):
        a = S.field_data(name, *self.model.sizes, seed, self.half)
        for s in self.sims:
            s.writeField(name, a)
        self.model.write(name, a)

    def op_write_tiny_div(self, seed):
        W, H = self.model.sizes[:2]
        d = S.tiny_divergence(W, H, seed)
        for s in self.sims:
            s.writeField("divergence", d)
        self.model.write("divergence", d)

    def _solve(self, call, iters, want):
        before = self.stats()
        exact = self.exact_expected(iters)
        for s in self.sims:
            call(s)
        after = self.stats()
        for k, (b, a) in enumerate(zip(before, after)):
            assert a["jacobi_launches"] - b["jacobi_launches"] == want, (k, a, b, want)
            if exact:
                assert a["jacobi_exact_streams"] > b["jacobi_exact_streams"], ("tiny divergence ran contracted", k)

    def op_pressure_solve(self):
        iters = int(self.model.config["PRESSURE_ITERATIONS"])
        self._solve(lambda s: s.pass_("pressure_solve"), iters, self.solve_launches(iters))
        self.model.pressure_solve()

    def op_jacobi(self, k):
        self._solve(lambda s: s.pass_("jacobi", k), k, self.solve_launches(k))
        self.model.jacobi(k)

    def op_host_solve(self, iters, seed):
        W, H = self.model.sizes[:2]
        d, p = S.host_inputs(W, H, seed, self.half)
        bands = slab.host_bands(H, iters, block=self.model.jacobi_block) if "banded" in self.classes else []
        if bands and self.model.jacobi_block != 1:
            want = sum(len(b["launches"]) for b in bands)
        else:
            want = self.solve_launches(iters)
        outs = []
        self.model.write("divergence", d)                # the premise reads the divergence of the solve
        self._solve(lambda s: outs.append(self._host(s, d, p, iters)), iters, want)
        ref = self.model.pressure_solve_host(d, p, iters)
        assert same_bits(outs[0], ref), "fluid_pressure_solve_host result differs from the model"
        assert bits_equal(outs[1], outs[0])

    @staticmethod
    def _host(s, d, p, iters):
        ph = p.copy()
        s.pressure_solve_host(d.copy(), ph, iters)
        return ph

    def op_config(self, key, value):
        for s in self.sims:
            s.config[key] = value
        self.model.config[key] = value

    def op_jacobi_block(self, k):
        for s in self.sims:
            s.set_param("JACOBI_BLOCK", k)
        self.model.jacobi_block = k

    def op_resize(self, si):
        W, H, Wd, Hd, cw, ch, _ = self.sched[si]
        for s in self.sims:
            s.canvas = {"width": cw, "height": ch}
            s._sizes = (W, H, Wd, Hd)
            s.initFramebuffers()
            assert s._dims("velocity")[:2] == (W, H) and s._dims("dye")[:2] == (Wd, Hd)
        self.model.resize(W, H, Wd, Hd, (cw, ch))
        self.si = si
        self.fresh = True

    @staticmethod
    def _keywords(s, kw, transparent):
        DH.set_keywords(s, kw)
        s.config["TRANSPARENT"] = transparent

    def op_render(self, kw, transparent, target):
        frames = []
        for s in self.sims:
            self._keywords(s, kw, transparent)
            frames.append(s.render(target=target))
        g, t = self.sims
        bg = O.BG_NONE if transparent and target else O.BG_CHECKERBOARD if transparent else O.BG_COLOR
        DH.check_frame(g, frames[0], self.model.render(kw, bg, self.dither, FX), kw, ("render", kw, transparent, target))
        assert G.same_bits(frames[1], frames[0])

    def op_capture(self, kw, transparent):
        got = []
        for s in self.sims:
            self._keywords(s, kw, transparent)
            got.append(s.captureScreenshot())
        ref = self.model.capture(kw, transparent, self.dither, FX, S.FXCFG["CAPTURE_RESOLUTION"])
        DH.check_capture(got[0], ref, kw, ("capture", kw, transparent))
        assert np.array_equal(got[1], got[0])


def replay(pkg, mode, ops, seed=None):
    """Runs a logged session on a handle of `mode`; an AssertionError names the mode, the seed, the
    operation and the log up to it."""
    s = Session(pkg, mode)
    try:
        s.check_fields()
        for i, op in enumerate(ops):
            try:
                s.run(op)
            except AssertionError as e:
                log = "\n".join(f"  {k:3d} {o!r}" for k, o in enumerate(ops[:i + 1]))
                raise AssertionError(f"session seed={seed} mode={mode}: operation {i} {op!r} failed: {e}\n"
                                     f"replay(pkg, {mode!r}, ops) with ops =\n{log}") from e
    finally:
        s.close()


# ---- scripted hand-offs --------------------------------------------------------------------------------
ALL3 = M.SHADING | M.BLOOM | M.SUNRAYS
SCRIPTS = {
    # fluid_pressure_solve_host flips the pressure parity outside any step: the next replay must read the
    # buffer the solve left its result in (banded at 1024 x 512, one piece at 64 x 64)
    "host_solve_then_step": ("fp32", [
        ("write", "velocity", 1), ("write", "dye", 2), ("step", S.DT_CLAMP), ("host_solve", 20, 3), ("step", S.DT_CLAMP),
        ("resize", 1), ("step", S.DT_CLAMP), ("host_solve", 20, 4), ("step", S.DT_CLAMP), ("step", 0.01),
        ("host_solve", 50, 5), ("host_solve", 13, 6), ("step", S.DT_CLAMP), ("pressure_solve",), ("step", S.DT_CLAMP)]),
    # resize away and back: an earlier graph-cache key returns with new buffers
    "resize_and_back": ("fp32", [
        ("write", "velocity", 7), ("step", S.DT_CLAMP), ("resize", 1), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP),
        ("resize", 5), ("step", S.DT_CLAMP), ("resize", 9), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP),
        ("resize", 10), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP)]),
    "half_resize_and_back": ("half", [
        ("write", "velocity", 8), ("step", S.DT_CLAMP), ("resize", 1), ("step", S.DT_CLAMP), ("resize", 4),
        ("step", S.DT_CLAMP), ("resize", 8), ("step", S.DT_CLAMP), ("resize", 9), ("step", S.DT_CLAMP)]),
    # SUNRAYS draws its mask into dye.write (and, in half storage, widens dye into the shared scratch)
    "sunrays_frame_then_splat_and_step": ("fp32", [
        ("write", "dye", 9), ("render", M.SHADING | M.SUNRAYS, False, False), ("splat", 10), ("step", S.DT_CLAMP),
        ("render", M.BLOOM | M.SUNRAYS, True, False), ("splats", 5, 11), ("step", S.DT_CLAMP),
        ("capture", ALL3, False), ("step", S.DT_CLAMP), ("render", ALL3, True, True), ("step", S.DT_CLAMP)]),
    "half_sunrays_frame_then_splat_and_step": ("half", [
        ("write", "dye", 12), ("render", M.SHADING | M.SUNRAYS, False, False), ("splat", 13), ("step", S.DT_CLAMP),
        ("render", ALL3, False, False), ("write", "velocity", 14), ("splats", 129, 15), ("step", S.DT_CLAMP),
        ("capture", ALL3, True), ("step", S.DT_CLAMP)]),
    # a host write of tiny divergence rebuilds the tiny map: the next blocked solve must use the exact tail
    "tiny_divergence_write_then_solve_and_step": ("fp32", [
        ("write", "velocity", 16), ("write_tiny_div", 17), ("pressure_solve",), ("step", S.DT_CLAMP),
        ("write_tiny_div", 18), ("jacobi", 13), ("step", S.DT_CLAMP), ("resize", 1), ("write_tiny_div", 19),
        ("pressure_solve",), ("step", S.DT_CLAMP)]),
    # JACOBI_BLOCK changes the launches of a replayed step but not its bits: the launch counts catch a
    # graph key without it
    "live_jacobi_block_between_replays": ("fp32", [
        ("write", "velocity", 20), ("write", "pressure", 21), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP),
        ("jacobi_block", 7), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP), ("jacobi_block", 13), ("step", S.DT_CLAMP),
        ("jacobi_block", 1), ("step", S.DT_CLAMP), ("jacobi_block", 0), ("step", S.DT_CLAMP),
        ("config", "PRESSURE_ITERATIONS", 14), ("step", S.DT_CLAMP), ("config", "PRESSURE_ITERATIONS", 0),
        ("step", S.DT_CLAMP), ("config", "PRESSURE_ITERATIONS", 1), ("step", 0.0), ("jacobi_block", 7),
        ("step", S.DT_CLAMP), ("resize", 1), ("step", S.DT_CLAMP), ("jacobi_block", 13), ("step", S.DT_CLAMP)]),
    # LINEAR advection across the 4-cell kernels: one-cell -> adv4_same -> adv4 -> ragged -> adv4_same, two
    # steps at each size, and live dissipations, CURL, PRESSURE_ITERATIONS and JACOBI_BLOCK between replays
    # (changing a value back replays the graph captured before the change); splats and a host solve before steps
    "linear_resize_across_adv4_and_back": ("linear", [
        ("write", "velocity", 31), ("write", "dye", 32), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP),
        ("resize", 1), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP), ("config", "VELOCITY_DISSIPATION", 4.0),
        ("step", S.DT_CLAMP), ("config", "VELOCITY_DISSIPATION", 0.2), ("step", S.DT_CLAMP),
        ("config", "DENSITY_DISSIPATION", 0.0), ("step", S.DT_CLAMP), ("config", "CURL", 55.0), ("step", 0.01),
        ("host_solve", 20, 33), ("step", S.DT_CLAMP),
        ("resize", 2), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP), ("splats", 5, 34), ("config", "DENSITY_DISSIPATION", 1.0),
        ("step", S.DT_CLAMP), ("config", "PRESSURE_ITERATIONS", 13), ("jacobi_block", 7), ("step", S.DT_CLAMP),
        ("config", "CURL", 30.0), ("step", S.DT_CLAMP), ("config", "CURL", 55.0), ("step", S.DT_CLAMP),
        ("resize", 4), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP), ("config", "VELOCITY_DISSIPATION", 1.0),
        ("step", S.DT_CLAMP), ("splat", 35), ("step", S.DT_CLAMP),
        ("resize", 1), ("step", S.DT_CLAMP), ("step", S.DT_CLAMP), ("config", "DENSITY_DISSIPATION", 4.0),
        ("jacobi_block", 0), ("step", S.DT_CLAMP), ("config", "DENSITY_DISSIPATION", 1.0), ("step", S.DT_CLAMP)]),
    # the desktop configuration (HALF_STORAGE | HALF_POSTFX | LINEAR_ADVECTION) through the reference's update():
    # splats, a step at the clamped dt, a frame with all three keywords; a capture, a host solve, a resize and back
    "desktop_frame_loop": ("desktop", [
        ("write", "velocity", 41), ("write", "dye", 42),
        ("splats", 5, 43), ("step", S.DT_CLAMP), ("render", ALL3, False, False),
        ("splat", 44), ("step", S.DT_CLAMP), ("render", ALL3, False, False),
        ("splats", 2, 45), ("step", 0.0123), ("render", ALL3, False, False), ("capture", ALL3, False),
        ("splats", 3, 46), ("step", S.DT_CLAMP), ("render", ALL3, False, False),
        ("host_solve", 20, 47), ("step", S.DT_CLAMP), ("render", ALL3, False, False),
        ("resize", 1), ("splats", 2, 48), ("step", S.DT_CLAMP), ("render", ALL3, False, False),
        ("resize", 9), ("splat", 49), ("step", S.DT_CLAMP), ("render", ALL3, False, False),
        ("splats", 5, 50), ("step", S.DT_CLAMP), ("render", ALL3, True, False), ("capture", ALL3, True),
        ("splats", 129, 51), ("step", S.DT_CLAMP), ("render", ALL3, False, False)]),
    # NEAREST resize copies in half storage across the whole schedule; after each resize every keyword set is
    # drawn, a capture taken and one step run
    "nearest_half_resize_then_draw": ("nearest_half", [("write", "velocity", 61), ("write", "dye", 62)] + [
        op for si in range(1, len(S.HALF_SCHEDULE)) for op in
        [("resize", si)] + [("render", kw, bool(kw & 1), kw in (3, 6)) for kw in range(8)]
        + [("capture", ALL3 if si % 2 else si % 8, bool(si % 3 == 0)), ("step", S.DT_CLAMP)]]),
}


@pytest.mark.parametrize("name", list(SCRIPTS))
def test_scripted_hand_off(pkg, name):
    mode, ops = SCRIPTS[name]
    replay(pkg, mode, ops, seed=name)


# ---- seeded random sessions ----------------------------------------------------------------------------
@pytest.mark.parametrize("mode,seed", [(m, s) for m in S.MODES for s in S.SEEDS[m]])
def test_random_session(pkg, mode, seed):
    half = S.is_half(mode)
    replay(pkg, mode, S.generate(seed, half, S.N_OPS), seed=seed)
