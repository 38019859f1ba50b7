"""session_model.py on the CPU: the model against the oracle it is built from and the executed copy-shader
goldens, and the operation generator's determinism and reach over the seeds test_gpu_session.py runs."""
import numpy as np
import pytest

import display_model as M
import session_model as S
from conftest import bits_equal, golden, max_rel
from linear_advection_model import LinearOracleSim

# what the committed sessions of test_gpu_session.py must reach, per storage mode
OPS = {"step", "splat", "splats", "write", "pressure_solve", "jacobi", "host_solve", "config", "jacobi_block", "resize",
       "render", "capture"}
COMMON = (OPS | {f"config:{k}" for k in S.CONFIG_VALUES} | {f"jacobi_block:{k}" for k in S.JACOBI_BLOCKS}
          | {"splats<=128", "splats>128", "dt:0", "dt:tiny", "dt:jitter", "dt:clamp", "resize_up", "resize_down",
             "resize_same_sim", "canvas_aspect_change", "render:sunrays", "render:bloom", "render:transparent"}
          | {f"write:{n}" for n in S.FIELDS} | {f"iters:{k}" for k in S.CONFIG_VALUES["PRESSURE_ITERATIONS"]}
          | {"size:same_size", "size:sim_only", "size:dye_only", "size:earlier_size", "size:degenerate", "size:one_piece"})
REACH = {
    False: COMMON | {"write_tiny_div", "size:stream", "size:tiled", "size:adv4_same", "size:adv4", "size:adv1_pow2",
                     "size:ragged", "size:blocked", "size:scalar", "size:banded"},
    True: COMMON | {"size:half8", "size:half_scalar"},
}


def test_step_only_sequences_equal_oraclesim(oracle):
    """Writes, live config and steps through the model of every mode == the mode's simulation driven
    directly, bit for bit: OracleSim, and LinearOracleSim in the LINEAR modes (linear, desktop), whose
    steps differ from OracleSim's."""
    for mode, (half, sampler) in S.MODES.items():
        sim = LinearOracleSim if sampler == "linear" else oracle.OracleSim
        for W, H, Wd, Hd in ((36, 20, 54, 30), (128, 64, 256, 128)):
            m = S.SessionModel(W, H, Wd, Hd, (72, 40), mode=mode)
            ref = sim(W, H, Wd, Hd, half_storage=half)
            manual = oracle.OracleSim(W, H, Wd, Hd, half_storage=half)
            v = S.field_data("velocity", W, H, Wd, Hd, 1, half)
            dye = S.field_data("dye", W, H, Wd, Hd, 2, half)
            m.write("velocity", v); m.write("dye", dye)
            R = oracle.round_half if half else (lambda a: a.copy())
            ref.velocity, ref.dye = R(v), R(dye)
            manual.velocity, manual.dye = R(v), R(dye)
            for k, (key, val, dt) in enumerate([(None, None, S.DT_CLAMP), ("CURL", 12.5, 0.01), ("PRESSURE_ITERATIONS", 13, 0.0),
                                                ("VELOCITY_DISSIPATION", 4.0, S.TINY_DT), ("PRESSURE", 0.33, S.DT_CLAMP),
                                                ("PRESSURE_ITERATIONS", 0, S.DT_CLAMP)]):
                if key:
                    m.config[key] = val
                    setattr(ref, key, val)
                    setattr(manual, key, val)
                m.step(dt); ref.step(dt); manual.step(dt)
                for n in S.FIELDS:
                    a, b = m.field(n), getattr(ref, n)
                    assert a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)), (mode, k, n)
                    assert bits_equal(np.nan_to_num(a), np.nan_to_num(b)), (mode, k, n)
            differs = not bits_equal(np.nan_to_num(m.field("dye")), np.nan_to_num(manual.dye))
            assert differs == (sampler == "linear"), (mode, W, H)


def test_pressure_solves_equal_clear_and_jacobi(oracle):
    """pass_("pressure_solve"), pass_("jacobi", k) and the host solve: clear + jacobi of the oracle; in half
    storage every blit rounded to fp16, the host inputs included."""
    W, H = 24, 16
    rng = np.random.default_rng(3)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    m = S.SessionModel(W, H, W, H, (48, 32))
    m.write("pressure", p); m.write("divergence", d)
    m.pressure_solve()
    assert bits_equal(m.field("pressure"), oracle.jacobi(oracle.clear(p, 0.8), d, 20))
    m.jacobi(5)
    assert bits_equal(m.field("pressure"), oracle.jacobi(oracle.jacobi(oracle.clear(p, 0.8), d, 20), d, 5))
    assert bits_equal(m.pressure_solve_host(d, p, 13), oracle.jacobi(oracle.clear(p, 0.8), d, 13))
    h = S.SessionModel(W, H, W, H, (48, 32), mode="half")
    R = oracle.round_half
    want = R(oracle.clear(R(p), 0.8))
    for _ in range(3):
        want = R(oracle.jacobi(want, R(d), 1))
    assert bits_equal(h.pressure_solve_host(d, p, 3), want)
    assert bits_equal(h.field("divergence"), R(d))


def test_resize_equals_copy_shader_goldens(oracle):
    """The model's resize: the executed copyShader bit for bit on the power-of-two golden, within
    test_oracle_golden.py's 2e-6 on the ragged ones; pressure, divergence and curl start over at zero; an
    unchanged size keeps its field as it is."""
    g = golden("resample_dye_64_to_32")
    m = S.SessionModel(16, 16, 64, 64, (64, 64))
    m.write("dye", g["src"]); m.write("pressure", np.ones((16, 16), np.float32))
    m.resize(16, 16, 32, 32, (64, 64))
    assert bits_equal(m.field("dye"), g["linear"])
    assert not m.field("pressure").any() and m.field("pressure").shape == (16, 16)
    for name, vel in (("resample_v_32_to_48", True), ("resample_dye_40x28_to_64x48", False)):
        g = golden(name)
        Ws, Hs = g["src"].shape[1], g["src"].shape[0]
        Wd, Hd = int(g["Wd"]), int(g["Hd"])
        if vel:
            m = S.SessionModel(Ws, Hs, 8, 8, (Ws, Hs)); m.write("velocity", g["src"])
            keep = m.field("dye").copy()
            m.resize(Wd, Hd, 8, 8, (Wd, Hd))
            got = m.field("velocity")
            assert bits_equal(m.field("dye"), keep)
        else:
            m = S.SessionModel(8, 8, Ws, Hs, (Ws, Hs)); m.write("dye", g["src"])
            m.resize(8, 8, Wd, Hd, (Wd, Hd))
            got = m.field("dye")
        assert max_rel(got, g["linear"]) < 2e-6, name
        for n in ("pressure", "divergence", "curl"):
            assert not m.field(n).any()


def test_nearest_resize_equals_display_model_resize(oracle):
    """The resize of a NEAREST model (nearest, nearest_half): velocity and dye are display_model.resize's
    NEAREST copy (fp16-rounded in half storage), not the LINEAR copy of the other modes; a field whose size
    did not change keeps its bits; pressure, divergence and curl start over at zero."""
    for mode in ("nearest", "nearest_half"):
        half = S.is_half(mode)
        W, H, Wd, Hd = 36, 20, 54, 30
        m = S.SessionModel(W, H, Wd, Hd, (72, 40), mode=mode)
        lin = S.SessionModel(W, H, Wd, Hd, (72, 40), mode="half" if half else "fp32")
        for n in ("velocity", "dye"):
            a = S.field_data(n, W, H, Wd, Hd, 7, half)
            m.write(n, a); lin.write(n, a)
        m.write("pressure", np.ones((H, W), np.float32))
        # up, down, ragged; sim only, dye only; and back
        for sizes in ((72, 40, 108, 60), (17, 9, 108, 60), (17, 9, 25, 70), (64, 64, 25, 70), (36, 20, 54, 30)):
            v0, d0 = m.field("velocity").copy(), m.field("dye").copy()
            m.resize(*sizes, (72, 40)); lin.resize(*sizes, (72, 40))
            W, H, Wd, Hd = sizes
            for n, old, (w, h) in (("velocity", v0, (W, H)), ("dye", d0, (Wd, Hd))):
                got = m.field(n)
                if old.shape[:2] == (h, w):
                    assert bits_equal(np.nan_to_num(got), np.nan_to_num(old)), (mode, sizes, n)
                else:
                    want = M.resize(old, w, h, half=half)
                    assert got.shape == want.shape and np.array_equal(np.isnan(got), np.isnan(want)), (mode, sizes, n)
                    assert bits_equal(np.nan_to_num(got), np.nan_to_num(want)), (mode, sizes, n)
                    assert not bits_equal(np.nan_to_num(got), np.nan_to_num(lin.field(n))), (mode, sizes, n)
            for n in ("pressure", "divergence", "curl"):
                assert m.field(n).shape == (H, W) and not m.field(n).any(), (mode, sizes, n)
            for n in ("velocity", "dye"):
                lin.write(n, m.field(n))       # the next resize copies the same fields


def test_splat_interval_holds_the_oracle_splat(oracle):
    """The interval the model checks a splat against contains the oracle's own splat (glibc expf)."""
    m = S.SessionModel(48, 32, 96, 64, (150, 100))
    m.write("velocity", S.field_data("velocity", 48, 32, 96, 64, 4, False))
    recs = S.splat_records(3, 5)
    iv = m.splat_interval(recs)
    v = m.field("velocity")
    for r in recs:
        v = oracle.splat(v, np.float32(1.5), float(r[0]), float(r[1]), (float(r[2]), float(r[3]), 0.0),
                         S.SM.radius_of(0.25, 150, 100))
    lo, hi = iv["velocity"]
    assert S.SM.check_splat(v, lo, hi)[0] == 0


@pytest.mark.parametrize("mode", list(S.MODES))
def test_generator_is_deterministic_and_reaches_every_class(mode):
    """Same seed, same session; another seed, another session; and over the committed seeds of a mode in
    test_gpu_session.py every operation kind, config key, JACOBI_BLOCK value, dt kind, splat count class,
    resize direction and size class of its storage's schedule is reached, the session ending at its
    starting size."""
    half = S.is_half(mode)
    seeds = S.SEEDS[mode]
    assert len(seeds) >= 3, seeds
    a = S.generate(seeds[0], half, S.N_OPS)
    assert a == S.generate(seeds[0], half, S.N_OPS)
    assert a != S.generate(seeds[0] + 1000, half, S.N_OPS)
    reached = set()
    for seed in seeds:
        ops = S.generate(seed, half, S.N_OPS)
        assert 30 <= len(ops) <= 60, len(ops)
        resizes = [op[1] for op in ops if op[0] == "resize"]
        assert resizes == list(range(1, len(S.schedule(half))))
        assert S.schedule(half)[resizes[-1]][:4] == S.schedule(half)[0][:4]
        reached |= S.op_classes(ops, half)
    missing = REACH[half] - reached
    assert not missing, sorted(missing)


def test_schedules_cross_each_boundary_both_ways():
    """Each size class of the schedule is entered from a size without it and left for one without it."""
    for half in (False, True):
        sched = S.schedule(half)
        four = {"adv4", "adv4_same"}
        pairs = [({"stream"}, {"tiled"}), (four, {"adv1_pow2"}), (four, {"ragged"}), ({"blocked"}, {"scalar"}),
                 ({"banded"}, {"one_piece"})] if not half else [({"half8"}, {"half_scalar"})]
        seq = [c[6] for c in sched]
        assert sched[-1][:4] == sched[0][:4]
        for a, b in pairs:
            ab = any(a & x and b & y for x, y in zip(seq, seq[1:]))
            ba = any(b & x and a & y for x, y in zip(seq, seq[1:]))
            assert ab and ba, (half, a, b)
