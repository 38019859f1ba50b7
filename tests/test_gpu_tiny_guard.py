"""The blocked Jacobi kernel's tiny-divergence guard against every writer of divergence.

jacobi_tb_kernel ends each update with the contracted tail fma(S, 0.25, -0.25 d), which is bit-exact only
where d == 0 or |d| >= 2^-123 (tests/test_fma_contraction_cpu.py).  Every cell with 0 < |d| < 2^-123 must be
flagged in the tiny map (one byte per 128 columns x 32 rows, global rows), so that the warp streams whose
footprint covers it run the un-contracted tail.  The map has one producer per writer of divergence, each
with its own indexing: cvd_stream_kernel (per lane, 120-column windows), the tiled fused kernel, the unfused
divergence_kernel, tiny_scan_kernel behind fluid_write(DIVERGENCE), the one-piece host solve and every
upload chunk of the banded host solve, and the map's allocation on create and resize.

The data here places tiny divergence on purpose where that indexing can go wrong: the grid's walls, both
sides of every map-cell edge (columns 128k - 1 / 128k / 128k + 1, rows 32k - 1 / 32k / 32k + 1), both sides
of the streaming kernel's 120-column window edges, the last partial map column and row, the first and last
row of each banded upload chunk, and map cells that only exist after a resize.  Each placed cell comes with
a pressure neighbourhood for which the contracted tail gives different bits (checked on the CPU, first in
exact rational arithmetic for the first sweep, then through whole solves): a flag that is missing at any
placed cell makes the GPU solve differ from the oracle."""
import functools
from fractions import Fraction

import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import fma_tail
from test_fma_contraction_cpu import add32, fma as kernel_tail, ref as exact_tail, rn32
from test_gpu_fast_paths import exp_tiled, far_field
from test_gpu_parity import STREAM_SHAPES, make
from webgl_fluid_simulation_b200 import slab

F = np.float32
DT = 0.016666
TINY = 2.0 ** -123
TINY_CW, TINY_CH = 128, 32         # jacobi.cuh: one map byte per 128 columns x 32 rows
CVD_COLS = 120                     # stream_passes.cuh CVD2_VALID: output columns of a cvd_stream_kernel window
ITERS, NJ = 16, 9                  # sweeps of pressure_solve / of the pass_("jacobi", n) that follows it
JB = [0, 1, 7, 13]                 # JACOBI_BLOCK: the default depth, one sweep per launch, two explicit depths
SEP = 3                            # Chebyshev distance between the cells of different placed sites
ROW_GAP, COL_GAP = 4, 3            # map rows / columns between the flagged map cells of one group of sites
SMS = 132                          # SMs of an H100 SXM (fluid.cu tb_rows sizes the streams from it)
PATCH = 1                          # tiny pressure within this distance of a placed cell
RAGGED_STREAM = [(1000, 520)]      # streaming, W % 128 = 104, W % 120 = 40, H % 32 = 8
TILED_EXTRA = [(1000, 37), (130, 66)]      # too few warps to stream; 130 % 4 = 2 (no blocked kernel)
STEP_SHAPES = [(964, 600), (1000, 37)]     # one streaming and one tiled size for whole steps
HOST_ONE_PIECE = (1000, 300)       # shorter than two bands: the one-piece host solve
HOST_BANDED = (256, 2000)          # 7 bands of 286 rows, the last one ragged (284)


# ---- where to put tiny cells -------------------------------------------------------------------------------
def _edges(n, cell, window=None, extra=()):
    """Indices along one axis in priority order: `extra`, both walls, the three indices around the first
    map-cell edge, the first index of the last partial map cell, the first window edge, then every other
    map-cell edge (cell*k - 1, cell*k, cell*k + 1) and window edge (window*k - 1, window*k)."""
    out = list(extra) + [0, n - 1, cell - 1, cell, cell + 1]
    if n % cell:
        out.append(n // cell * cell)
    if window:
        out += [window - 1, window]
    for k in range(2, (n - 1) // cell + 1):
        out += [cell * k - 1, cell * k, cell * k + 1]
    if window:
        for k in range(2, (n - 1) // window + 1):
            out += [window * k - 1, window * k]
    return [x for x in dict.fromkeys(out) if 0 <= x < n]


def impulse_cells(comp, j, i, W, H):
    """The divergence cells a single velocity value of component comp (0: x, 1: y) at (j, i) makes nonzero:
    the cells before and after it along that axis, or the wall cell and its neighbour (the wall reflects the
    normal component, S:804-807).  None on an axis of length 1, where the two wall terms cancel."""
    n, a = (W, i) if comp == 0 else (H, j)
    if n < 2:
        return None
    idx = [0, 1] if a == 0 else [n - 2, n - 1] if a == n - 1 else [a - 1, a + 1]
    return [(j, k) for k in idx] if comp == 0 else [(k, i) for k in idx]


def impulse_at(comp, j, i, W, H):
    """Where to put the velocity value of component comp so that cell (j, i) is one of impulse_cells: on the
    cell itself at a wall, else one further along the axis (the target and the cell two further are tiny)."""
    n, a = (W, i) if comp == 0 else (H, j)
    a = a if a in (0, n - 1) else a + 1
    return (j, a) if comp == 0 else (a, i)


def placements(W, H, extra_rows=(), region=None):
    """Sites of tiny divergence for a W x H grid: a list of (comp, j, i, cells), one velocity value at (j, i)
    whose divergence is nonzero exactly at `cells` (two cells, opposite signs).  Column targets (walls, map
    and window edges) get an x-value beside them, so the target and the cell two columns further are tiny;
    at column 128k - 1 that second cell lies across the map edge, at row 32k - 1 (y-values for row targets)
    likewise.  The cells of different sites keep SEP apart; groups() then splits the sites into sets that are
    solved one at a time.  region(j, i) -> bool restricts the cells (the new part of a resized grid)."""
    cols = _edges(W, TINY_CW, CVD_COLS)
    rows = _edges(H, TINY_CH, extra=extra_rows)
    targets = []                                  # (axis, index): rows and columns interleaved, in priority order
    for q in range(max(len(cols), len(rows))):
        if q < len(rows):
            targets.append((1, rows[q]))
        if q < len(cols):
            targets.append((0, cols[q]))
    sites, cells_so_far = [], []
    for q, (axis, t) in enumerate(targets):
        for alt in range(12):                    # the free coordinate: spread over the grid, next try elsewhere
            if axis == 0:
                i, j = t, (H // 2 + 41 * (q + 7 * alt)) % H
                comp = 0 if W >= 2 else 1
            else:
                j, i = t, (W // 2 + 53 * (q + 7 * alt)) % W
                comp = 1 if H >= 2 else 0
            pos = impulse_at(comp, j, i, W, H)
            cells = impulse_cells(comp, pos[0], pos[1], W, H)
            if cells is None or (j, i) not in cells:
                continue
            if region is not None and not all(region(*c) for c in cells):
                continue
            if any(max(abs(c[0] - o[0]), abs(c[1] - o[1])) < SEP for c in cells for o in cells_so_far):
                continue
            sites.append((comp, pos[0], pos[1], cells))
            cells_so_far += cells
            break
    return sites


def map_cells(site):
    return {(j // TINY_CH, i // TINY_CW) for (j, i) in site[3]}


def isolated(a, b):
    """Map cells a and b are never read by one blocked stream: a stream reads at most two adjacent map
    columns and at most ROW_GAP map rows (test_no_stream_reads_two_sites_of_a_group)."""
    return all(abs(p[0] - q[0]) >= ROW_GAP or abs(p[1] - q[1]) >= COL_GAP for p in a for q in b)


def groups(sites):
    """Split sites (in order) into groups whose flagged map cells are pairwise isolated.  One solve per group:
    the streams that read a site's map cells read no other site's, so a flag its writer misplaces or drops is
    not covered by a correct flag of a neighbouring site, and most map cells of each solve stay clear."""
    out = []
    for q, s in enumerate(sites):
        m = map_cells(s)
        for g in out:
            if all(isolated(m, map_cells(sites[o])) for o in g):
                g.append(q)
                break
        else:
            out.append([q])
    return out


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


# ---- the CPU restatement of the solve --------------------------------------------------------------------
def sweeps(p, d, n, contracted=None):
    """n Jacobi sweeps in the reference's order ((((L + R) + B) + T) - d) * 0.25 with CLAMP_TO_EDGE; where the
    mask `contracted` is set, the blocked kernel's contracted tail fma(S, 0.25, rn(-0.25 d)) instead."""
    H, W = p.shape
    il = np.maximum(np.arange(W) - 1, 0); ir = np.minimum(np.arange(W) + 1, W - 1)
    jb = np.maximum(np.arange(H) - 1, 0); jt = np.minimum(np.arange(H) + 1, H - 1)
    dq = F(-0.25) * d
    for _ in range(n):
        S = ((p[:, il] + p[:, ir]) + p[jb, :]) + p[jt, :]
        e = (S - d) * F(0.25)
        p = e if contracted is None else np.where(contracted, fma_tail(S, dq), e)
    return p


def first_sweep_sum(p, j, i):
    """S of cell (j, i) in the first sweep, in the reference's order, through exact rational arithmetic."""
    H, W = p.shape
    L, R = p[j, max(i - 1, 0)], p[j, min(i + 1, W - 1)]
    B, T = p[max(j - 1, 0), i], p[min(j + 1, H - 1), i]
    return add32(add32(add32(L, R), B), T)


def single_rounding(S, d):
    """The exact rational S*0.25 - 0.25*d rounded once to fp32 (nearest even).  Where S - d is exact -- as it
    is for every placed cell -- this IS the reference's value: what breaks the identity is the kernel's
    pre-scaled divergence rn(-0.25 d), rounded before the fma."""
    x = Fraction(float(S)) / 4 - Fraction(float(d)) / 4
    return F(0.0) if x == 0 else rn32(x)


def _same_bits(a, b):
    return np.array([a], F).view(np.uint32)[0] == np.array([b], F).view(np.uint32)[0]


def first_sweep_differs(cleared, d, j, i):
    S, dv = first_sweep_sum(cleared, j, i), d[j, i]
    return not _same_bits(kernel_tail(S, dv), exact_tail(S, dv))


def site_defeats_contraction(p0, d, cells):
    """The premise of one placed site: (1) in the first sweep of pressure_solve, at each of its cells, the
    kernel's contracted value fma(S, 0.25, rn(-0.25 d)) differs from the reference's; (2) a solve that runs
    the contracted tail at these cells only -- the flag of this
    site missing -- ends with different bits than the exact one, for pressure_solve (clear + ITERS sweeps)
    and for NJ sweeps from the written pressure.  Checked on a crop that keeps every value it compares
    exact: the real walls, and ITERS + 4 cells on every other side."""
    H, W = p0.shape
    js = [c[0] for c in cells]; is_ = [c[1] for c in cells]
    R = max(ITERS, NJ) + 4
    j0, j1 = max(min(js) - R, 0), min(max(js) + R + 1, H)
    i0, i1 = max(min(is_) - R, 0), min(max(is_) + R + 1, W)
    pc, dc = p0[j0:j1, i0:i1], d[j0:j1, i0:i1]
    cleared = pc * F(0.8)
    if not all(first_sweep_differs(cleared, dc, j - j0, i - i0) for (j, i) in cells):
        return False
    mask = np.zeros(pc.shape, bool)
    for (j, i) in cells:
        mask[j - j0, i - i0] = True
    # cells whose final value is exact on the crop: more sweeps away from every side that is not a wall
    keep = np.zeros(pc.shape, bool)
    m = max(ITERS, NJ) + 1
    keep[(m if j0 else 0):pc.shape[0] - (m if j1 < H else 0), (m if i0 else 0):pc.shape[1] - (m if i1 < W else 0)] = True
    for start, n in ((cleared, ITERS), (pc, NJ)):
        a, b = sweeps(start, dc, n), sweeps(start, dc, n, mask)
        if bits_equal(a[keep], b[keep]):
            return False
    return True


@functools.lru_cache(maxsize=None)
def tiny_case(W, H, extra_rows=(), region=None, group=0):
    """Velocity, divergence and pressure of one group of placed sites: velocity zero but for one value per
    site, its divergence tiny exactly at the sites' cells (subnormal and normal magnitudes, both signs) and exact zeros
    elsewhere; pressure tiny near the sites (drawn until site_defeats_contraction holds for every site),
    ordinary far from them, zero in between."""
    from oracle import oracle as O
    rng = np.random.default_rng(group * 7919 + W * 31 + H)
    every = placements(W, H, extra_rows, region)
    index = groups(every)[group]
    sites = [every[q] for q in index]
    v = np.zeros((H, W, 2), F)
    mags = []
    for q, (comp, j, i, _) in enumerate(sites):
        # subnormal, or normal below 2^-124: from 2^-124 on, rn(-0.25 d) is exact and the contracted tail
        # cannot differ (the guard's bound 2^-123 is one binade conservative), so such a cell proves nothing
        # d = k * 2^-149 with k = 2 mod 4, so that rn(-0.25 d) is inexact too: where it is exact the
        # contracted tail equals the reference's whatever the neighbourhood
        e = int(rng.integers(-141, -127)) if index[q] % 2 == 0 else int(rng.integers(-126, -124))
        k = (int(np.ldexp(rng.uniform(1.0, 2.0), e + 149)) & ~3) | 2
        dm = F(np.ldexp(float(k), -149))
        v[j, i, comp] = F(2.0) * dm * F(rng.choice([-1.0, 1.0]))
        mags.append(float(dm))
    d = O.divergence(v)
    placed = {c for s in sites for c in s[3]}
    tiny = (d != 0) & (np.abs(d) < F(TINY))
    assert set(zip(*np.nonzero(tiny))) == placed and not d[~tiny].any()
    p0 = np.zeros((H, W), F)
    near = np.zeros((H, W), bool)
    R = max(ITERS, NJ) + 6
    for (_, _, _, cells) in sites:
        for (j, i) in cells:
            near[max(j - R, 0):j + R + 1, max(i - R, 0):i + R + 1] = True
    p0[~near] = rng.standard_normal(int((~near).sum())).astype(F)

    owner = np.full((H, W), -1)                  # each patch cell belongs to the first site that reaches it
    for q, (_, _, _, cells) in enumerate(sites):
        for (j, i) in cells:
            box = owner[max(j - PATCH, 0):j + PATCH + 1, max(i - PATCH, 0):i + PATCH + 1]
            box[box < 0] = q

    def draw(q):
        m = owner == q
        n = int(m.sum())
        p0[m] = (rng.uniform(0.1, 3.0, n) * mags[q] * rng.choice([-1.0, 1.0], n)).astype(F)

    for q in range(len(sites)):
        draw(q)
    # one site at a time until it holds; the crops of near sites overlap, so check those again afterwards
    reach = 2 * (max(ITERS, NJ) + 5)
    todo = list(range(len(sites)))
    for _ in range(50):
        bad = [q for q in todo if not site_defeats_contraction(p0, d, sites[q][3])]
        if not bad:
            break
        for q in bad:
            for _ in range(200):
                draw(q)
                if site_defeats_contraction(p0, d, sites[q][3]):
                    break
        todo = [q for q, s in enumerate(sites)
                if any(abs(s[1] - sites[b][1]) <= reach and abs(s[2] - sites[b][2]) <= reach for b in bad)]
    else:
        raise AssertionError(f"no pressure neighbourhood defeats the contraction at every site of {W}x{H}")
    return dict(v=v, d=d, p0=p0, sites=sites)


class NewCells(tuple):
    """region predicate of the cells a resize added: rows from new_rows on or columns from new_cols on."""
    def __new__(cls, new_rows, new_cols):
        return super().__new__(cls, (new_rows, new_cols))

    def __call__(self, j, i):
        return j >= self[0] or i >= self[1]


def cases(W, H, extra_rows=(), region=None):
    """tiny_case of every group of the placement."""
    n = len(groups(placements(W, H, extra_rows, region)))
    return [tiny_case(W, H, extra_rows, region, g) for g in range(n)]


def expected(O, case):
    """The oracle's pressure after pressure_solve and after NJ sweeps from the written pressure."""
    if "solve" not in case:
        case["solve"] = O.jacobi(O.clear(case["p0"], 0.8), case["d"], ITERS)
        case["jac"] = O.jacobi(case["p0"], case["d"], NJ)
    return case["solve"], case["jac"]


def blocked(W, H, jb):
    """fluid.cu tb_eligible and blocked(): only the blocked kernel reads the tiny map."""
    return W % 4 == 0 and W >= 16 and H >= 2 and jb != 1


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
@pytest.fixture(scope="module")
def pkg():
    import webgl_fluid_simulation_b200 as p
    return p


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
