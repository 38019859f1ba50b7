"""Lane-level numpy model of csrc/jacobi.cuh::jacobi_tb_kernel — same window geometry, mirrored
loads, staged 128-column boxes, 3-slot rotating windows, shifted K+3-slot div register ring, wall selects,
chunking and store predicate, statement for statement, and the same choice of tail per warp stream: the
contracted fma(S, 0.25, -0.25 d) unless the tiny-divergence map flags the stream's footprint (run exact
from the start) or its level-0 inputs reached BIG_IN (run again exact).  It exists so the kernel's index
logic and tail selection can be checked against the oracle on a machine without a GPU
(tests/test_jacobi_tb_model.py); it is not used by the product.

Beside it, what the CPU and GPU tests of that tail share: the two tails in exact rational arithmetic
(tests/test_fma_contraction_cpu.py), the data sets at the top of the fp32 range and on inf / NaN, and the
placements of tiny divergence on every edge of the tiny map (tests/test_gpu_tiny_guard.py)."""
import functools
from fractions import Fraction

import numpy as np

from conftest import bits_equal
from sim_harness import exp_tiled, jacobi_plan, same_bits

F = F32 = np.float32
TINY_CW, TINY_CH = 128, 32                 # jacobi.cuh: one tiny-map byte per 128 columns x 32 rows
TINY_DIV = F(2.0 ** -123)
BIG_IN = 2.0 ** 122

# which streams run the exact tail: "exact" all of them, "tiny" those whose footprint the tiny map flags
# (the selection before BIG_IN existed), "kernel" those plus the ones whose level-0 inputs reach BIG_IN
SELECT = ("exact", "tiny", "kernel")


def _shfl_up(x):      # lane l receives lane l-1 (lane 0 keeps its own value)
    return np.concatenate([x[:1], x[:-1]])


def _shfl_down(x):    # lane l receives lane l+1 (lane 31 keeps its own value)
    return np.concatenate([x[1:], x[-1:]])


def fma_tail(S, dq):
    """fp32 fma(S, 0.25, dq): S * 0.25 is exact in float64, the float64 sum rounds at most once, and that
    rounding followed by the fp32 one equals a single fp32 rounding (53 >= 2 * 24 + 2; checked against exact
    arithmetic in tests/test_fma_contraction_cpu.py)."""
    return (S.astype(np.float64) * 0.25 + dq.astype(np.float64)).astype(F)


def _jacobi4(below, c, above, d, exact):
    """exact: ((((L + R) + B) + T) - d) * 0.25;  else fma(((L + R) + B) + T, 0.25, d) with d = -0.25 div."""
    l = _shfl_up(c[:, 3]); r = _shfl_down(c[:, 0])
    S = np.empty_like(c)
    S[:, 0] = ((l + c[:, 1]) + below[:, 0]) + above[:, 0]
    S[:, 1] = ((c[:, 0] + c[:, 2]) + below[:, 1]) + above[:, 1]
    S[:, 2] = ((c[:, 1] + c[:, 3]) + below[:, 2]) + above[:, 2]
    S[:, 3] = ((c[:, 2] + r) + below[:, 3]) + above[:, 3]
    return (S - d) * F(0.25) if exact else fma_tail(S, d)


def tiny_map(div, W, H, row_off=0):
    """The kernel's map of divergence values in (0, 2^-123), GLOBAL rows (a local buffer from row_off)."""
    m = np.zeros(((H + TINY_CH - 1) // TINY_CH, (W + TINY_CW - 1) // TINY_CW), bool)
    for j, i in zip(*np.nonzero((div != 0) & (np.abs(div) < TINY_DIV))):
        m[(j + row_off) // TINY_CH, i // TINY_CW] = True
    return m


def jacobi_tb_model(pin, div, K, rows_per_chunk, scale=None, row_off=0, out_lo=None, out_hi=None,
                    H=None, pout=None, select="kernel", stats=None):
    """pin/div: local buffers (rows x W).  Returns pout (local buffer; untouched rows stay NaN).
    select: one of SELECT.  stats, a dict, gets "exact_streams": the streams that ran the exact tail."""
    assert select in SELECT
    rows_local, W = pin.shape
    H = rows_local if H is None else H
    out_lo = 0 if out_lo is None else out_lo
    out_hi = H if out_hi is None else out_hi
    HX = (K + 3) // 4 * 4; VALID = 128 - 2 * HX; RD = K + 3; U = 3
    assert W % 4 == 0 and W >= 16
    if pout is None:
        pout = np.full_like(pin, np.nan)
    nxw = (W + VALID - 1) // VALID
    nch = (out_hi - out_lo + rows_per_chunk - 1) // rows_per_chunk
    tmap = tiny_map(div, W, H, row_off)
    lane = np.arange(32)
    n_exact = 0
    for wid in range(nxw * nch):
        wx, cy = wid % nxw, wid // nxw
        gx = wx * VALID - HX + 4 * lane
        lc = gx.copy(); rev = np.zeros(32, bool)
        m = gx < 0; lc[m] = -gx[m] - 4; rev[m] = True
        m = gx >= W; lc[m] = 2 * W - 4 - gx[m]; rev[m] = True
        lc = np.minimum(np.maximum(lc, 0), W - 4)
        lane_out = (lane >= HX // 4) & (lane < 32 - HX // 4) & (gx >= 0) & (gx < W)
        y0 = out_lo + cy * rows_per_chunk
        y1 = min(y0 + rows_per_chunk, out_hi)
        ys = max(y0 - K, 0)
        ye = min(y1 - 1 + K, H - 1)
        nsteps = y1 - ys + K
        # TMA staging: step s takes row ys + s of the 128-column box from column x0, zero outside the
        # buffer's rows and the grid's columns; a lane reads its column group clamped into the box
        x0 = wx * VALID - HX
        # the tiny-map cells of the stream's footprint, as the kernel's prologue reads them
        cx0, cx1 = max(x0, 0) // TINY_CW, min(x0 + 127, W - 1) // TINY_CW
        flagged = tmap[ys // TINY_CH:ye // TINY_CH + 1, cx0:cx1 + 1].any()
        cols = np.minimum(np.maximum(lc, x0), x0 + 124)[:, None] + np.arange(4)[None, :]
        inside = (cols >= 0) & (cols < W)

        def load(buf, r):
            v = np.zeros((32, 4), F)
            if 0 <= r - row_off < buf.shape[0]:
                v[inside] = buf[r - row_off][cols[inside]]
            v[rev] = v[rev][:, ::-1]
            return v

        def stream(exact):
            """One pass of the warp over its rows; returns the largest level-0 magnitude (fmaxf: NaN drops out)."""
            big = F(0)
            w = np.zeros((K, 3, 32, 4), F)
            dr = np.full((RD, 32, 4), np.nan, F)
            rout = ys - K
            for s0 in range(0, nsteps, U):
                edge = (ys + s0 - K <= 0) or (ys + s0 + 2 >= H - 1)
                for ph in range(U):
                    inn = load(pin, ys + s0 + ph); dv = load(div, ys + s0 + ph)
                    if scale is not None:
                        inn = F(scale) * inn
                    if not exact:
                        big = np.fmax(big, np.fmax(np.fmax.reduce(np.abs(inn), axis=None),
                                                   np.fmax.reduce(np.abs(dv), axis=None)))
                        dv = F(-0.25) * dv
                    w[0, (ph + 2) % 3] = inn
                    dr[K + ph] = dv
                    for t in range(1, K + 1):
                        c = w[t - 1, (ph + 1) % 3]
                        below = w[t - 1, (ph + 0) % 3]
                        above = w[t - 1, (ph + 2) % 3]
                        if edge:
                            r = rout + (K - t)
                            if r == 0: below = c
                            if r == H - 1: above = c
                        d = dr[K + ph - t]
                        o = _jacobi4(below, c, above, d, exact)
                        if t < K:
                            w[t, (ph + 2) % 3] = o
                        elif y0 <= rout < y1:
                            for l in np.nonzero(lane_out)[0]:
                                pout[rout - row_off, gx[l]:gx[l] + 4] = o[l]
                    rout += 1
                for j in range(K):
                    dr[j] = dr[j + 3]
            return big

        with np.errstate(invalid="ignore", over="ignore"):
            exact = select == "exact" or flagged
            if not exact:
                # the kernel's rerun: the exact pass stores over the rows the contracted one stored
                exact = stream(False) >= BIG_IN and select == "kernel"
            if exact:
                stream(True)
                n_exact += 1
    if stats is not None:
        stats["exact_streams"] = n_exact
    return pout


# ---- the two tails in exact rational arithmetic ---------------------------------------------------------
def rn32(x: Fraction) -> np.float32:
    """Correctly rounded (nearest-even) fp32 of a nonzero exact rational, subnormals and overflow included.
    A result that underflows to zero keeps the sign of x."""
    s = -1 if x < 0 else 1
    a = abs(x)
    # exponent e with 2^e <= a < 2^(e+1)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    e = max(e, -126)                      # subnormals share the exponent of the smallest normal
    ulp = Fraction(2) ** (e - 23)
    q, r = divmod(a, ulp)
    q = int(q)
    if r * 2 > ulp or (r * 2 == ulp and (q & 1)):
        q += 1
    v = Fraction(q) * ulp
    if v >= Fraction(2) ** 128:
        return F32(s * np.inf)
    return F32(s * float(v))              # exactly representable: float() is exact


def _finite(*xs):
    return all(np.isfinite(x) for x in xs)


def _neg0(*signs):
    """An exact zero sum is -0 only when every addend is a zero of negative sign (round to nearest)."""
    return F32(-0.0) if all(signs) else F32(0.0)


def add32(a, b):
    """rn32(a + b) for fp32 a, b, with IEEE rules for inf / NaN and the sign of zero."""
    if not _finite(a, b):
        with np.errstate(invalid="ignore"):
            return F32(np.float64(a) + np.float64(b))      # inf +- finite, inf - inf = NaN, NaN: as IEEE
    s = Fraction(float(a)) + Fraction(float(b))
    if s == 0:
        return _neg0(np.signbit(a), np.signbit(b)) if a == 0 and b == 0 else F32(0.0)
    return rn32(s)


def mul32(a, b):
    if not _finite(a, b):
        with np.errstate(invalid="ignore"):
            return F32(np.float64(a) * np.float64(b))
    s = Fraction(float(a)) * Fraction(float(b))
    if s == 0:
        return F32(-0.0) if np.signbit(a) != np.signbit(b) else F32(0.0)
    return rn32(s)


def fma32(a, b, c):
    """rn32(a*b + c), one rounding.  float64 a*b of fp32 operands is exact, so the special cases follow IEEE."""
    if not _finite(a, b, c):
        with np.errstate(invalid="ignore"):
            return F32(np.float64(a) * np.float64(b) + np.float64(c))
    p = Fraction(float(a)) * Fraction(float(b))
    s = p + Fraction(float(c))
    if s == 0:
        return _neg0(np.signbit(a) != np.signbit(b), np.signbit(c)) if p == 0 and c == 0 else F32(0.0)
    return rn32(s)


def ref(S, d):     # the reference tail: (S - d) * 0.25, two roundings
    return mul32(add32(S, -d), F32(0.25))


def fma(S, d):     # the contracted tail: d' = rn(-0.25 d), then one rounding of S*0.25 + d'
    return fma32(S, F32(0.25), mul32(d, F32(-0.25)))


# ---- the top of the fp32 range, inf and NaN ------------------------------------------------------------
# Data sets the contracted tail must survive (shared with the GPU tests).  Stored pressure is divided by
# PRESSURE so that the fused clear brings the patch to the magnitude that overflows at once.
KINDS = ["near_max", "near_max_neg", "huge_div", "nonfinite", "full_range"]
NONFINITE_KINDS = {"nonfinite", "full_range"}          # inf / NaN in the inputs
# results that can hold NaN (inf - inf of overflowed neighbours), whose bits differ between x86 and the GPU:
# compared NaN-aware, the others bitwise
NAN_KINDS = NONFINITE_KINDS | {"huge_div"}


def special_fields(kind, W, H, seed, pressure=1.0):
    """(p, d) of one data set: ordinary fields with
    near_max      p = 8.5e37 / PRESSURE over a patch and d = -1e37 under it: four such neighbours sum to
                  3.4e38 and S - d rounds to +inf in the first sweep, while S/4 - d/4 is finite;
    near_max_neg  the same with both signs flipped;
    huge_div      |d| in [2^126, FLT_MAX] over a patch of ordinary p: the first sweep leaves p ~ -d/4 and
                  the second one overflows;
    nonfinite     +-inf and NaN sprinkled into both p and d;
    full_range    binary exponents -149..127 tile by tile for both (subnormals to inf)."""
    rng = np.random.default_rng(seed)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    r0, r1 = H // 4, min(H // 4 + max(3, H // 3), H)
    c0, c1 = W // 3, W // 3 + max(8, W // 4)
    if kind in ("near_max", "near_max_neg"):
        sg = np.float32(1.0 if kind == "near_max" else -1.0)
        p[r0:r1, c0:c1] = sg * np.float32(8.5e37 / pressure)
        d[max(r0 - 1, 0):r1 + 1, c0 - 1:c1 + 1] = -sg * np.float32(1e37)
    elif kind == "huge_div":
        mag = rng.uniform(2.0 ** 126, float(np.finfo(np.float32).max), (r1 - r0, c1 - c0))
        d[r0:r1, c0:c1] = (mag * rng.choice([-1.0, 1.0], mag.shape)).astype(np.float32)
    elif kind == "nonfinite":
        for a in (p, d):
            k = rng.choice(H * W, size=max(6, H * W // 500), replace=False)
            a.flat[k] = rng.choice(np.array([np.inf, -np.inf, np.nan], np.float32), k.size)
    else:
        p = exp_tiled((H, W), seed, lo=-149, hi=127, tile=(4, 16))
        d = exp_tiled((H, W), seed + 1, lo=-149, hi=127, tile=(4, 16))
    return p, d


def overflow_sweep(oracle, p, d, iters, pressure):
    """First sweep (1-based) of the oracle's clear + `iters` sweeps with a cell whose S and d are finite and
    whose rn(S - d) is infinite -- where the contracted tail would differ -- or None."""
    q = oracle.clear(p, pressure)
    for k in range(1, iters + 1):
        e = np.pad(q, 1, mode="edge")
        with np.errstate(invalid="ignore", over="ignore"):
            S = ((e[1:-1, :-2] + e[1:-1, 2:]) + e[:-2, 1:-1]) + e[2:, 1:-1]
            hit = np.isfinite(S) & np.isfinite(d) & np.isinf(S - d)
        if hit.any():
            return k
        q = oracle.jacobi(q, d, 1)
    return None


def equal(kind, a, b):
    return same_bits(a, b) if kind in NAN_KINDS else bits_equal(a, b)


# ---- tiny divergence on every edge of the tiny map ---------------------------------------------------------
TINY = 2.0 ** -123
CVD_COLS = 120                     # stream_passes.cuh CVD2_VALID: output columns of a cvd_stream_kernel window
ITERS, NJ = 16, 9                  # sweeps of pressure_solve / of the pass_("jacobi", n) that follows it
JB = [0, 1, 7, 13]                 # JACOBI_BLOCK: the default depth, one sweep per launch, two explicit depths
SEP = 3                            # Chebyshev distance between the cells of different placed sites
ROW_GAP, COL_GAP = 4, 3            # map rows / columns between the flagged map cells of one group of sites
PATCH = 1                          # tiny pressure within this distance of a placed cell


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


# the CPU restatement of the solve
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


def _same_bits(a, b):
    return np.array([a], F).view(np.uint32)[0] == np.array([b], F).view(np.uint32)[0]


def first_sweep_differs(cleared, d, j, i):
    S, dv = first_sweep_sum(cleared, j, i), d[j, i]
    return not _same_bits(fma(S, dv), ref(S, dv))


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
    """Whether the blocked kernel, the only reader of the tiny map, runs the solves of these tests."""
    return jacobi_plan(W, H, False, ITERS, jb) != [1] * ITERS
