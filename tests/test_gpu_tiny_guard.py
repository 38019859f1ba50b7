"""The blocked Jacobi kernel's tiny-divergence guard against every writer of divergence.

jacobi_tb_kernel ends each update with the contracted tail fma(S, 0.25, -0.25 d), which is bit-exact only
where d == 0 or |d| >= 2^-123 (tests/test_fma_contraction_cpu.py).  Every cell with 0 < |d| < 2^-123 must be
flagged in the tiny map (one byte per 128 columns x 32 rows, global rows), so that the warp streams whose
footprint covers it run the un-contracted tail.  The map has one producer per writer of divergence, each
with its own indexing: cvd_stream_kernel (per lane, 120-column windows), the tiled fused kernel, the unfused
divergence_kernel, tiny_scan_kernel behind fluid_write(DIVERGENCE), the one-piece host solve and every
upload chunk of the banded host solve, and the map's allocation on create and resize.  The batch writer,
cvd_stream_kernel<true>, flags one region of the map per member, which the batch form of the blocked kernel
reads; tests/test_gpu_batch_edges.py places the same sites in different members of a batch step.

The data here places tiny divergence on purpose where that indexing can go wrong: the grid's walls, both
sides of every map-cell edge (columns 128k - 1 / 128k / 128k + 1, rows 32k - 1 / 32k / 32k + 1), both sides
of the streaming kernel's 120-column window edges, the last partial map column and row, the first and last
row of each banded upload chunk, and map cells that only exist after a resize.  Each placed cell comes with
a pressure neighbourhood for which the contracted tail gives different bits (checked on the CPU, first in
exact rational arithmetic for the first sweep, then through whole solves): a flag that is missing at any
placed cell makes the GPU solve differ from the oracle."""
from fractions import Fraction

import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import (ITERS, JB, NJ, ROW_GAP, SEP, TINY, TINY_CH, TINY_CW, _same_bits, blocked, cases,
                             expected, first_sweep_differs, first_sweep_sum, fma as kernel_tail, groups, isolated,
                             map_cells, placements, ref as exact_tail, rn32, site_defeats_contraction, sweeps)
from sim_harness import STREAM_SHAPES, exp_tiled, far_field, make
from sim_harness import pkg  # noqa: F401 -- a fixture
from webgl_fluid_simulation_b200 import slab

F = np.float32
DT = 0.016666
SMS = 132                          # SMs of an H100 SXM (fluid.cu tb_rows sizes the streams from it)
RAGGED_STREAM = [(1000, 520)]      # streaming, W % 128 = 104, W % 120 = 40, H % 32 = 8
TILED_EXTRA = [(1000, 37), (130, 66)]      # too few warps to stream; 130 % 4 = 2 (no blocked kernel)
STEP_SHAPES = [(964, 600), (1000, 37)]     # one streaming and one tiled size for whole steps
HOST_ONE_PIECE = (1000, 300)       # shorter than two bands: the one-piece host solve
HOST_BANDED = (256, 2000)          # 7 bands of 286 rows, the last one ragged (284)


def stream_map_rows(W, H, n_rows, K):
    """The most map rows one warp stream of a depth-K launch over n_rows output rows reads: fluid.cu tb_rows at
    one resident CTA per SM (the fewest chunks, so the longest streams), plus the 2K rows of its cone."""
    hx = (K + 3) // 4 * 4
    nxw = -(-W // (128 - 2 * hx))
    nch = max(1, max(nxw, SMS) // nxw)
    r = max(-(-n_rows // nch), 4 * K)
    r += (-(r + 2 * K)) % 3
    L = min(min(r, n_rows) + 2 * K, H)
    return max((s + L - 1) // TINY_CH - s // TINY_CH + 1 for s in range(TINY_CH))


def single_rounding(S, d):
    """The exact rational S*0.25 - 0.25*d rounded once to fp32 (nearest even).  Where S - d is exact -- as it
    is for every placed cell -- this IS the reference's value: what breaks the identity is the kernel's
    pre-scaled divergence rn(-0.25 d), rounded before the fma."""
    x = Fraction(float(S)) / 4 - Fraction(float(d)) / 4
    return F(0.0) if x == 0 else rn32(x)


class NewCells(tuple):
    """region predicate of the cells a resize added: rows from new_rows on or columns from new_cols on."""
    def __new__(cls, new_rows, new_cols):
        return super().__new__(cls, (new_rows, new_cols))

    def __call__(self, j, i):
        return j >= self[0] or i >= self[1]


STREAM_CASES = STREAM_SHAPES + RAGGED_STREAM
TILED_CASES = STREAM_SHAPES + TILED_EXTRA
ALL_SHAPES = list(dict.fromkeys(STREAM_CASES + TILED_CASES + STEP_SHAPES + [HOST_ONE_PIECE]))


def band_rows(W, H):
    """First and last row of every upload chunk of the banded host solve, and the first row of the ragged last
    band (slab.host_bands mirrors fluid.cu solve_host_banded)."""
    bands = slab.host_bands(H, ITERS)
    rows = [r for b in bands for r in (b["up_lo"], b["up_hi"] - 1)] + [bands[-1]["lo"]]
    return tuple(dict.fromkeys(rows))


# ---- CPU: the premise --------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H", ALL_SHAPES + [HOST_BANDED])
def test_placed_cells_defeat_the_contraction(oracle, W, H):
    """Every placed cell distinguishes the contracted tail from the reference's (exact rational arithmetic on
    the first sweep, whole solves on a crop), so a GPU solve that missed its flag would not be bitwise; the
    difference comes from rounding -0.25 d ahead of the fma (the once-rounded S/4 - d/4 agrees with the
    reference); and at the guard's boundary -- |d| = 2^-123 exactly, d = +-0 -- the same neighbourhoods give
    equal bits."""
    extra = band_rows(W, H) if (W, H) == HOST_BANDED else ()
    subnormal = normal = negative = positive = 0
    for c in cases(W, H, extra):
        assert c["sites"]
        cleared = c["p0"] * F(0.8)
        for (_, _, _, cells) in c["sites"]:
            assert site_defeats_contraction(c["p0"], c["d"], cells)
            for (j, i) in cells:
                dv = c["d"][j, i]
                assert 0 < abs(float(dv)) < TINY
                subnormal += abs(float(dv)) < 2.0 ** -126; normal += abs(float(dv)) >= 2.0 ** -126
                negative += dv < 0; positive += dv > 0
                S = first_sweep_sum(cleared, j, i)
                assert first_sweep_differs(cleared, c["d"], j, i)
                assert _same_bits(single_rounding(S, dv), exact_tail(S, dv))
                for edge in (F(TINY), F(-TINY), F(0.0), F(-0.0)):
                    assert _same_bits(kernel_tail(S, edge), exact_tail(S, edge)), (j, i, float(edge))
                    if edge != 0 and S != 0:              # (the once-rounded rational has no sign of zero)
                        assert _same_bits(single_rounding(S, edge), exact_tail(S, edge)), (j, i, float(edge))
        # the restatement of the sweep is the oracle's, bit for bit
        assert bits_equal(sweeps(cleared, c["d"], ITERS), expected(oracle, c)[0])
    assert subnormal and normal and negative and positive


@pytest.mark.parametrize("W,H", [(1024, 512), (1000, 520), (16900, 8), (8, 4096), (1000, 37), (130, 66)])
def test_placements_reach_every_edge(W, H):
    """The generator's promise: tiny cells on both walls, on both sides of the first map-cell edge in x and y
    and of the first cvd window edge, in the last partial map column / row, one site whose second cell lies
    across a map-cell edge; the sites of one group isolated from each other."""
    sites = placements(W, H)
    cells = [c for s in sites for c in s[3]]
    cs, rs = {c[1] for c in cells}, {c[0] for c in cells}
    assert {0, W - 1} <= cs and {0, H - 1} <= rs
    for x in (127, 128, 119, 120):
        assert x >= W or x in cs, x
    for y in (31, 32):
        assert y >= H or y in rs, y
    if W % TINY_CW:
        assert any(c >= W // TINY_CW * TINY_CW for c in cs)
    if H % TINY_CH:
        assert any(r >= H // TINY_CH * TINY_CH for r in rs)
    assert any(len(map_cells(s)) == 2 for s in sites)
    for a in range(len(sites)):
        for b in range(a):
            assert min(max(abs(p[0] - q[0]), abs(p[1] - q[1])) for p in sites[a][3] for q in sites[b][3]) >= SEP
    gs = groups(sites)
    assert sorted(q for g in gs for q in g) == list(range(len(sites)))
    for g in gs:
        for a in g:
            for b in g:
                assert a == b or isolated(map_cells(sites[a]), map_cells(sites[b])), (a, b)


def test_no_stream_reads_two_sites_of_a_group():
    """isolated() rests on the footprint of a blocked warp stream: 128 columns (two adjacent map columns) by
    its rows plus 2K, which must span at most ROW_GAP map rows for every blocked launch these tests make:
    pressure_solve and the NJ sweeps at each JACOBI_BLOCK, the banded host solve's launches, on every shape."""
    shapes = ALL_SHAPES + [HOST_BANDED, (1000, 200), (1024, 520), (256, 64), (1024, 32), (120, 600)]
    worst = 0
    for W, H in shapes:
        for jb in JB:
            if not blocked(W, H, jb):
                continue
            kb = min(jb or slab.KMAX, slab.KMAX)
            for n in (ITERS, NJ):
                for K in slab.jacobi_launches(n, kb):
                    worst = max(worst, stream_map_rows(W, H, H, K))
            for b in slab.host_bands(H, ITERS, block=jb):
                for K, lo, hi in b["launches"]:
                    worst = max(worst, stream_map_rows(W, H, hi - lo, K))
    assert 2 <= worst <= ROW_GAP, worst


def test_banded_placement_covers_every_upload_chunk_edge():
    W, H = HOST_BANDED
    bands = slab.host_bands(H, ITERS)
    assert len(bands) >= 3 and bands[-1]["hi"] - bands[-1]["lo"] < bands[0]["hi"] - bands[0]["lo"]
    rows = {c[0] for s in placements(W, H, band_rows(W, H)) for c in s[3]}
    for b in bands:
        assert b["up_lo"] in rows and b["up_hi"] - 1 in rows, b
    assert any(bands[-1]["lo"] <= r for r in rows)


# ---- GPU: every writer, bitwise against the oracle ---------------------------------------------------------
def solve_and_check(s, O, case, W, H, jb):
    """pressure_solve from the written pressure, then NJ sweeps from it written again: both bitwise against the
    oracle, and the blocked kernel ran flagged streams through the exact tail."""
    want_solve, want_jac = expected(O, case)
    for name, run, want in (("solve", lambda: s.pass_("pressure_solve"), want_solve),
                            ("jacobi", lambda: s.pass_("jacobi", NJ), want_jac)):
        s.writeField("pressure", case["p0"])
        e0 = s.stat("jacobi_exact_streams")
        run()
        assert bits_equal(s.readField("pressure"), want), (name, W, H, jb, case["sites"][0])
        n = s.stat("jacobi_exact_streams") - e0
        assert (n > 0) if blocked(W, H, jb) else (n == 0), (name, n)


@pytest.mark.gpu
@pytest.mark.parametrize("jb", JB)
@pytest.mark.parametrize("W,H", STREAM_CASES)
def test_streaming_cvd_flags_every_placed_cell(pkg, oracle, W, H, jb):
    """curl_vorticity_divergence on the row-streaming kernel (the launch counter says it ran) writes the tiny
    cells itself: divergence bitwise, then the solves, one group of isolated sites at a time."""
    s = make(pkg, W, H, 8, 8, jb=jb, PRESSURE_ITERATIONS=ITERS)
    for c in cases(W, H):
        s.writeField("velocity", c["v"])
        n0 = s.stat("cvd_stream_launches")
        s.pass_("curl_vorticity_divergence", DT)
        assert s.stat("cvd_stream_launches") - n0 == 1
        assert bits_equal(s.readField("divergence"), c["d"])
        solve_and_check(s, oracle, c, W, H, jb)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("jb", JB)
@pytest.mark.parametrize("mode", ["tiled", "unfused"])
@pytest.mark.parametrize("W,H", TILED_CASES)
def test_tiled_and_unfused_divergence_flag_every_placed_cell(pkg, oracle, W, H, mode, jb):
    """The tiled fused kernel (FLUID_FLAG_TILED_PASSES) and the unfused divergence_kernel (FLUID_FLAG_UNFUSED,
    the divergence pass) write the tiny cells themselves, at streaming-sized grids and at W % 4 != 0."""
    flags = pkg.FLAG_TILED_PASSES if mode == "tiled" else pkg.FLAG_UNFUSED
    s = make(pkg, W, H, 8, 8, flags=flags, jb=jb, PRESSURE_ITERATIONS=ITERS)
    for c in cases(W, H):
        s.writeField("velocity", c["v"])
        n0 = s.stat("cvd_stream_launches")
        s.pass_("curl_vorticity_divergence", DT) if mode == "tiled" else s.pass_("divergence")
        assert s.stat("cvd_stream_launches") == n0
        assert bits_equal(s.readField("divergence"), c["d"])
        solve_and_check(s, oracle, c, W, H, jb)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("jb", JB)
@pytest.mark.parametrize("W,H", [(1024, 512), (1000, 520), (1000, 37), (16900, 3)])
def test_written_divergence_flags_every_placed_cell(pkg, oracle, W, H, jb):
    """writeField("divergence"): tiny_scan_kernel over the written rows."""
    s = make(pkg, W, H, 8, 8, jb=jb, PRESSURE_ITERATIONS=ITERS)
    for c in cases(W, H):
        s.writeField("divergence", c["d"])
        solve_and_check(s, oracle, c, W, H, jb)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("jb", JB)
@pytest.mark.parametrize("where", ["one_piece", "banded"])
def test_host_solve_flags_every_placed_cell(pkg, oracle, where, jb):
    """pressure_solve_host: in one piece (a grid shorter than two bands) the whole written divergence is
    scanned; banded, each upload chunk is scanned as it arrives, and the tiny cells sit in the first and last
    row of every chunk and in the ragged last band; the launches are the ones slab.host_bands plans.  At
    JACOBI_BLOCK 1 the library does not band (one sweep per launch, no blocked kernel, no map): there the
    tall grid is solved in one piece and only checked bitwise."""
    W, H = HOST_ONE_PIECE if where == "one_piece" else HOST_BANDED
    s = make(pkg, W, H, 8, 8, jb=jb, PRESSURE_ITERATIONS=ITERS)
    bands = slab.host_bands(H, ITERS, block=jb)
    assert bool(bands) == (where == "banded")
    for c in cases(W, H, band_rows(W, H) if where == "banded" else ()):
        ph = c["p0"].copy()
        e0, l0 = s.stat("jacobi_exact_streams"), s.stat("jacobi_launches")
        s.pressure_solve_host(c["d"], ph, ITERS)
        assert bits_equal(ph, expected(oracle, c)[0]), (where, jb, c["sites"][0])
        assert bits_equal(s.readField("pressure"), ph)
        n = s.stat("jacobi_exact_streams") - e0
        assert (n > 0) if blocked(W, H, jb) else (n == 0), n
        launches = s.stat("jacobi_launches") - l0
        if not blocked(W, H, jb):
            assert launches == ITERS
        elif where == "banded":
            assert launches == sum(len(b["launches"]) for b in bands)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("jb", JB)
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("W,H", STEP_SHAPES)
def test_whole_step_flags_every_placed_cell(pkg, oracle, W, H, graph, jb):
    """One whole step() per group from the placed velocity and pressure, as a CUDA graph and with
    FLAG_NO_GRAPH: every field bitwise against the oracle's step."""
    O = oracle
    Wd, Hd = W // 2, H // 2 + 1
    dye = far_field(O, Wd, Hd, 4, 3)
    s = make(pkg, W, H, Wd, Hd, flags=0 if graph else pkg.FLAG_NO_GRAPH, jb=jb, PRESSURE_ITERATIONS=ITERS)
    steps = 0
    for c in cases(W, H):
        ref = O.OracleSim(W, H, Wd, Hd, PRESSURE_ITERATIONS=ITERS)
        s.writeField("velocity", c["v"]); s.writeField("pressure", c["p0"]); s.writeField("dye", dye)
        ref.velocity, ref.pressure, ref.dye = c["v"].copy(), c["p0"].copy(), dye.copy()
        e0 = s.stat("jacobi_exact_streams")
        s.step(DT); ref.step(DT)
        steps += 1
        assert bits_equal(ref.divergence, c["d"])
        assert bits_equal(ref.pressure, expected(O, c)[0])
        for n in ("pressure", "divergence", "velocity", "curl", "dye"):
            assert bits_equal(s.readField(n), getattr(ref, n)), n
        n = s.stat("jacobi_exact_streams") - e0
        assert (n > 0) if blocked(W, H, jb) else (n == 0), n
    assert s.stat("graph_launches") == (steps if graph else 0)
    s.close()


# ---- GPU: staleness and resize ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(1024, 512), (1000, 37)])
def test_map_follows_divergence_through_writers(pkg, oracle, W, H):
    """Divergence tiny, ordinary, tiny at other cells, ordinary, tiny again, each time through another writer
    on one handle: the solves stay bitwise, and after an ordinary divergence no stream runs the exact tail
    (the map was cleared, not left holding the earlier cells)."""
    O = oracle
    cs = cases(W, H)
    assert len(cs) >= 2
    a, b = cs[0], cs[1]
    ordinary_v = exp_tiled((H, W, 2), W + H, lo=-20, hi=20, zeros=0.0)
    ordinary_d = np.random.default_rng(W).uniform(-1, 1, (H, W)).astype(F)
    s = make(pkg, W, H, 8, 8, PRESSURE_ITERATIONS=ITERS)

    def ordinary_solve(d):
        p = np.random.default_rng(H).standard_normal((H, W)).astype(F)
        s.writeField("pressure", p)
        e0 = s.stat("jacobi_exact_streams")
        s.pass_("pressure_solve")
        assert bits_equal(s.readField("pressure"), O.jacobi(O.clear(p, 0.8), d, ITERS))
        assert s.stat("jacobi_exact_streams") == e0

    s.writeField("velocity", a["v"]); s.pass_("curl_vorticity_divergence", DT)
    solve_and_check(s, O, a, W, H, 0)
    s.writeField("divergence", ordinary_d)
    ordinary_solve(ordinary_d)
    s.writeField("velocity", b["v"]); s.pass_("divergence")
    assert bits_equal(s.readField("divergence"), b["d"])
    solve_and_check(s, O, b, W, H, 0)
    s.writeField("velocity", ordinary_v); s.pass_("curl_vorticity_divergence", DT)
    d2 = s.readField("divergence")
    assert bits_equal(d2, O.divergence(O.vorticity(ordinary_v, O.curl(ordinary_v), 30.0, DT)))
    assert not ((d2 != 0) & (np.abs(d2) < F(TINY))).any()
    ordinary_solve(d2)
    s.writeField("divergence", a["d"])
    solve_and_check(s, O, a, W, H, 0)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("writer", ["cvd", "write"])
@pytest.mark.parametrize("src,dst", [((256, 64), (1000, 200)), ((1024, 32), (1024, 520)), ((120, 600), (964, 600))])
def test_resize_flags_cells_in_new_map_columns_and_rows(pkg, oracle, src, dst, writer):
    """After a resize to a wider and / or taller grid the map has cells it did not have before: tiny cells
    placed only there (through the fused pass or a written divergence) must be flagged by the next solve."""
    O = oracle
    (w0, h0), (W, H) = src, dst
    first = cases(w0, h0)[0]
    s = make(pkg, w0, h0, 8, 8, PRESSURE_ITERATIONS=ITERS)
    s.writeField("divergence", first["d"])
    solve_and_check(s, O, first, w0, h0, 0)
    s._sizes = (W, H, 8, 8); s.initFramebuffers()
    new_cols, new_rows = -(-w0 // TINY_CW) * TINY_CW, -(-h0 // TINY_CH) * TINY_CH
    for c in cases(W, H, region=NewCells(new_rows, new_cols)):
        assert all(j >= new_rows or i >= new_cols for st in c["sites"] for (j, i) in st[3])
        if writer == "cvd":
            s.writeField("velocity", c["v"]); s.pass_("curl_vorticity_divergence", DT)
            assert bits_equal(s.readField("divergence"), c["d"])
        else:
            s.writeField("divergence", c["d"])
        solve_and_check(s, O, c, W, H, 0)
    s.close()
