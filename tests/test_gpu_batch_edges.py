"""Batch handles' step kernels at the data that reaches their data-dependent branches, member by member against
the oracle.

A batch handle (fluid_create_batch) steps through BATCH instantiations of the step kernels, the member as blockIdx.z:
cvd_stream_kernel<true>, gradient_stream_kernel<true>, jacobi_tb_kernel<K, SCALE, true> and the 4-cell advections.
They stream at every size and B, with a chunking that depends on B (fluid.cu stream_args, tb_rows), where an ordinary
handle of the same size may run the tiled kernels; they read CURL, PRESSURE, the dissipations and dt from the member
table; and a batch runs the blocked Jacobi kernel at every JACOBI_BLOCK, depth 1 included.

* The tiny-divergence guard (tests/test_gpu_tiny_guard.py) through the batch writer.  Each member has its own region
  of the tiny map, tiny_map_w(W) * tiny_map_h(H) bytes at blockIdx.z regions from the start: cvd_stream_kernel<true>
  flags it and the blocked Jacobi kernel reads it.  The placed sites of jacobi_tb_model go to different members in
  each step: member 0 clean while others carry sites, sites in member m's last map row beside sites in member
  m + 1's first.  A writer or reader that takes another member's region misses a flag, and that member's pressure
  differs from the oracle's.
* The data sets of tests/test_gpu_fast_paths.py (exponent-tiled, far-field, and special values with +-inf and NaN),
  one per member, each member with its own CURL, PRESSURE, dissipations and dt: vort_pre / quot_fast, div_n_by's fast
  quotient and its IEEE division in different members of one launch, tap_pair's clamp of far back-traces.
Every field of every member is checked bit for bit (NaN-aware where the data holds NaN) against the oracle's step
from that member's inputs."""
import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import (ITERS, JB, TINY, TINY_CH, cases, expected, first_sweep_differs, site_defeats_contraction,
                             sweeps)
from sim_harness import exp_tiled, far_field, jacobi_plan, make, nasty_fields, same_bits
from sim_harness import pkg  # noqa: F401 -- a fixture

F = np.float32
DT = 0.016666
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")

# (W, H, B, Wd, Hd) of the tiny-guard steps
EDGE_CASES = [
    (128, 2, 5, 256, 4),        # one partial map cell per member: each member's region is a single byte
    (128, 32, 3, 128, 32),      # exactly one map row; dye on the sim grid (advect_dye4_kernel<SAME>)
    (256, 64, 4, 512, 128),     # cvd windows end at columns 119/120/121 and 239/240/241; 2 x 2 map cells
    (1024, 512, 2, 1024, 512),  # 9 cvd windows, 8 x 16 map cells, 14 groups of sites
    (128, 2, 64, 128, 2),       # B = 64: each member's streams are one chunk of H rows, the grid 64 members deep
]
EDGE_IDS = [f"{W}x{H}-B{B}" for W, H, B, _, _ in EDGE_CASES]


def batch(pkg, B, W, H, Wd, Hd, flags=0, jb=0, **cfg):
    c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}
    c.update(cfg)
    b = pkg.FluidBatch(B, c, canvas_width=W, canvas_height=H, sizes=(W, H, Wd, Hd), flags=flags, jacobi_block=jb)
    assert b.members == B
    return b


def write_members(b, inputs):
    """inputs: one dict of velocity / pressure / dye per member."""
    for name in ("velocity", "pressure", "dye"):
        b.writeField(name, np.stack([x[name] for x in inputs]))


def growth(s, stats, fn):
    """{stat: growth} of handle s over fn()."""
    n0 = {k: s.stat(k) for k in stats}
    fn()
    return {k: s.stat(k) - n0[k] for k in stats}


# ---- 1. the tiny-divergence guard, member by member ----------------------------------------------------------
def map_rows(case):
    """The tiny-map rows a case's sites flag."""
    return {j // TINY_CH for s in case["sites"] for (j, _) in s[3]}


def rounds(W, H, B):
    """The case group each member carries in each step, None for clean data.
    * [None, 0, 1, ..., n - 1] dealt out B at a time: in the first step member 0 is clean while members 1.. carry
      groups, one step later every group has been carried, and the members of one step carry different groups
      (B <= n + 1) or all of them;
    * two steps in which every even member carries a group with a site in its last map row and every odd member one
      with a site in its first map row, then the other way round: for every m, some step has sites in member m's last
      map row and in member m + 1's first, the two rows that are neighbours in the map, and neighbouring members
      carry different groups, so that neither member's flags stand in for the other's;
    * a step of clean members only, after steps with sites: the map must have been cleared."""
    cs = cases(W, H)
    n, mh = len(cs), -(-H // TINY_CH)
    deal = [None] + list(range(n))
    out = [[deal[(r * B + m) % len(deal)] for m in range(B)] for r in range(-(-len(deal) // B))]
    last = [g for g in range(n) if mh - 1 in map_rows(cs[g])]
    first = [g for g in range(n) if 0 in map_rows(cs[g])]
    for par in (0, 1):
        pools = [last if (m + par) % 2 == 0 else first for m in range(B)]
        out.append([pool[m % len(pool)] for m, pool in enumerate(pools)])
    out.append([None] * B)
    return out


def clean_fields(W, H, m):
    """Velocity and pressure of a member that carries no site: ordinary magnitudes, whose divergence has no value
    in (0, 2^-123) (test_premise checks it)."""
    v = exp_tiled((H, W, 2), 7000 + 13 * m + W + H, lo=-20, hi=20, zeros=0.0)
    p = np.random.default_rng(9000 + m + W).standard_normal((H, W)).astype(F)
    return v, p


def member_inputs(O, W, H, Wd, Hd, case, m):
    """Velocity, pressure and dye of member m carrying `case` (None: clean data)."""
    v, p = clean_fields(W, H, m) if case is None else (case["v"], case["p0"])
    return {"velocity": v, "pressure": p, "dye": far_field(O, Wd, Hd, 4, 11 + m)}


def oracle_step(O, W, H, Wd, Hd, x):
    ref = O.OracleSim(W, H, Wd, Hd, PRESSURE_ITERATIONS=ITERS)
    ref.velocity, ref.pressure, ref.dye = x["velocity"].copy(), x["pressure"].copy(), x["dye"].copy()
    ref.step(DT)
    return ref


@pytest.mark.parametrize("W,H,B,Wd,Hd", EDGE_CASES, ids=EDGE_IDS)
def test_premise(oracle, W, H, B, Wd, Hd):
    """On the CPU: every placed site defeats the contraction at these shapes (exact rational arithmetic on the
    first sweep, whole solves on a crop, the CPU restatement of the solve equal to the oracle's), a whole step
    keeps each case's divergence, clean members have no tiny divergence, and rounds() keeps its promises."""
    O = oracle
    cs = cases(W, H)
    assert cs
    for c in cs:
        assert c["sites"]
        cleared = c["p0"] * F(0.8)
        for (_, _, _, cells) in c["sites"]:
            assert site_defeats_contraction(c["p0"], c["d"], cells)
            for (j, i) in cells:
                assert 0 < abs(float(c["d"][j, i])) < TINY
                assert first_sweep_differs(cleared, c["d"], j, i)
        assert bits_equal(sweeps(cleared, c["d"], ITERS), expected(O, c)[0])
        assert bits_equal(O.divergence(O.vorticity(c["v"], O.curl(c["v"]), 30.0, DT)), c["d"])
    for m in range(B):
        v, _ = clean_fields(W, H, m)
        d = O.divergence(O.vorticity(v, O.curl(v), 30.0, DT))
        assert not ((d != 0) & (np.abs(d) < F(TINY))).any(), m
    plan = rounds(W, H, B)
    n, mh = len(cs), -(-H // TINY_CH)
    assert {g for step in plan for g in step} == set(range(n)) | {None}
    assert plan[0][0] is None and any(g is not None for g in plan[0][1:])
    if B <= n + 1:
        assert all(len(set(step)) == B for step in plan[:-3])
    for m in range(B - 1):
        assert any(step[m] is not None and step[m + 1] is not None and mh - 1 in map_rows(cs[step[m]])
                   and 0 in map_rows(cs[step[m + 1]]) for step in plan), m
        assert all(step[m] != step[m + 1] for step in plan[-3:-1]), m
    assert plan[-1] == [None] * B and any(g is not None for g in plan[-2])


@pytest.mark.gpu
@pytest.mark.parametrize("jb", JB)
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("W,H,B,Wd,Hd", EDGE_CASES, ids=EDGE_IDS)
def test_batch_flags_every_placed_cell_per_member(pkg, oracle, W, H, B, Wd, Hd, graph, jb):
    """One step() per row of rounds() from written velocity, pressure and dye, as a CUDA graph and with
    FLAG_NO_GRAPH: every field of every member bitwise against the oracle's step from that member's inputs, the
    divergence of a member carrying a case equal to the case's; one cvd_stream_kernel launch and the blocked plan's
    Jacobi launches per step; exact streams in a step if and only if some member carries a site (a batch runs the
    blocked kernel at every depth, so at JACOBI_BLOCK 1 too)."""
    O = oracle
    cs = cases(W, H)
    b = batch(pkg, B, W, H, Wd, Hd, flags=0 if graph else pkg.FLAG_NO_GRAPH, jb=jb, PRESSURE_ITERATIONS=ITERS)
    plan = rounds(W, H, B)
    launches = len(jacobi_plan(W, H, False, ITERS, jb))
    for k, carried in enumerate(plan):
        inputs = [member_inputs(O, W, H, Wd, Hd, None if g is None else cs[g], m) for m, g in enumerate(carried)]
        write_members(b, inputs)
        n = growth(b, ("cvd_stream_launches", "jacobi_launches", "jacobi_exact_streams"), lambda: b.step(DT))
        got = {name: b.readField(name) for name in FIELDS}
        for m, (g, x) in enumerate(zip(carried, inputs)):
            ref = oracle_step(O, W, H, Wd, Hd, x)
            if g is not None:
                assert bits_equal(got["divergence"][m], cs[g]["d"]), (k, m, g)
            for name in FIELDS:
                assert bits_equal(got[name][m], getattr(ref, name)), (k, m, g, name)
        assert n["cvd_stream_launches"] == 1 and n["jacobi_launches"] == launches, (k, n)
        assert (n["jacobi_exact_streams"] > 0) == any(g is not None for g in carried), (k, carried, n)
    assert b.stat("graph_launches") == (len(plan) if graph else 0)
    b.close()


# ---- 2. the fast paths' data, one set and one set of values per member ---------------------------------------
ITERS_FAST = 20
BIG_DISS = 1e20     # 1 + diss * dt above 2^60 for dt >= 0.0116: div_n_by divides by IEEE in every cell of the member
# one row per member: data set, CURL, PRESSURE, VELOCITY_DISSIPATION, DENSITY_DISSIPATION, dt of each step
MEMBERS = [
    ("exp_tiled", 0.0, 0.8, 0.0, BIG_DISS, (0.016666, 0.1)),
    ("far_field", 1e4, 0.0, BIG_DISS, 0.0, (0.1, 0.016666)),
    ("special", 30.0, 0.0, 4.0, BIG_DISS, (0.016, 0.05)),
    ("exp_tiled", 1e4, 2.0, BIG_DISS, 4.0, (0.05, 0.0)),
    ("far_field", 0.0, 1.0, 0.2, 0.0, (0.0, 0.016)),
    ("special", 1e4, 0.8, 0.0, 1.0, (0.1, 0.1)),
]
KEYS = ("CURL", "PRESSURE", "VELOCITY_DISSIPATION", "DENSITY_DISSIPATION")
# (W, H, Wd, Hd): the batch streams at each; only the largest is large enough for an ordinary twin to stream too
FAST_SIZES = [(128, 2, 256, 4), (256, 64, 512, 128), (1024, 1024, 1024, 1024)]
TWIN_SIZE = (1024, 1024)


def fast_fields(O, W, H, Wd, Hd, data, seed):
    """velocity, dye, pressure of one data set of tests/test_gpu_fast_paths.py, with dye that reaches both sides of
    div_n_by's range split (exponents -149..100 tile by tile, far-field decay, specials)."""
    if data == "exp_tiled":
        return exp_tiled((H, W, 2), seed), exp_tiled((Hd, Wd, 4), seed + 2, tile=(4, 8)), exp_tiled((H, W), seed + 1)
    if data == "far_field":
        v = far_field(O, W, H, 2, seed)
        return v, far_field(O, Wd, Hd, 4, seed + 1), np.ascontiguousarray(v[..., 0] * F(0.01))
    return nasty_fields(W, H, Wd, Hd, seed)


def decay(diss, dt):
    """The advection's denominator 1 + diss * dt in fp32, as the kernels form it."""
    return F(1.0) + F(diss) * F(dt)


def test_member_values_reach_both_divisions():
    """In each step, for both dissipations, some member's decay lies above 2^60, where div_n_by divides by IEEE in
    every cell, and some inside [2^-20, 2^60], where it takes the fast quotient for numerators in range; the data sets
    all take part, CURL and PRESSURE take 0 and other values, and the dts differ."""
    for k in range(2):
        for col in (3, 4):
            dens = [decay(r[col], r[5][k]) for r in MEMBERS]
            assert any(d > F(2.0 ** 60) for d in dens) and any(F(2.0 ** -20) <= d <= F(2.0 ** 60) for d in dens)
        assert len({r[5][k] for r in MEMBERS}) > 3
    assert {r[0] for r in MEMBERS} == {"exp_tiled", "far_field", "special"}
    assert {0.0, 1e4} <= {r[1] for r in MEMBERS} and 0.0 in {r[2] for r in MEMBERS}


@pytest.mark.gpu
@pytest.mark.parametrize("W,H,Wd,Hd", FAST_SIZES)
def test_fast_path_data_per_member(pkg, oracle, W, H, Wd, Hd):
    """Two steps of a batch whose members hold different data sets and their own CURL, PRESSURE, dissipations and
    dt (fluid_set_param_members, fluid_step_members): every field of every member against the oracle's step with
    that member's values, and at TWIN_SIZE against an ordinary twin that runs the non-batch instantiations of the
    same streaming kernels.  The launch counters say which kernels ran."""
    O = oracle
    B = len(MEMBERS)
    twin = (W, H) == TWIN_SIZE
    b = batch(pkg, B, W, H, Wd, Hd, PRESSURE_ITERATIONS=ITERS_FAST)
    twins = [make(pkg, W, H, Wd, Hd, PRESSURE_ITERATIONS=ITERS_FAST) for _ in MEMBERS] if twin else []
    data = [fast_fields(O, W, H, Wd, Hd, r[0], 31 * m + W + H) for m, r in enumerate(MEMBERS)]
    for i, name in enumerate(("velocity", "dye", "pressure")):
        b.writeField(name, np.stack([d[i] for d in data]))
        for t, d in zip(twins, data):
            t.writeField(name, d[i])
    refs = []
    for m, r in enumerate(MEMBERS):
        values = dict(zip(KEYS, r[1:5]))
        b.member_config[m].update(values)
        if twin:
            twins[m].config.update(values)
        ref = O.OracleSim(W, H, Wd, Hd, PRESSURE_ITERATIONS=ITERS_FAST, **values)
        ref.velocity, ref.dye, ref.pressure = (a.copy() for a in data[m])
        refs.append(ref)
    stats = ("cvd_stream_launches", "gradient_stream_launches", "advect4_launches")
    want = {"cvd_stream_launches": 1, "gradient_stream_launches": 1, "advect4_launches": 2}
    for k in range(2):
        dts = np.array([r[5][k] for r in MEMBERS], F)
        assert growth(b, stats, lambda: b.step(dts)) == want, k
        for t, dt in zip(twins, dts):
            assert growth(t, stats, lambda: t.step(float(dt))) == want, k
        for ref, dt in zip(refs, dts):
            ref.step(float(dt))
        got = {name: b.readField(name) for name in FIELDS}
        for m, r in enumerate(MEMBERS):
            equal = same_bits if r[0] == "special" else bits_equal
            for name in FIELDS:
                assert equal(got[name][m], getattr(refs[m], name)), (k, m, r[0], name)
                if twin:
                    assert same_bits(got[name][m], twins[m].readField(name)), (k, m, r[0], name, "twin")
    for key, col in zip(KEYS, range(1, 5)):
        assert b.member_params(key).tolist() == [F(r[col]) for r in MEMBERS], key
    b.close()
    for t in twins:
        t.close()
