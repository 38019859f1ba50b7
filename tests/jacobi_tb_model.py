"""Lane-level numpy model of csrc/jacobi.cuh::jacobi_tb_kernel — same window geometry, mirrored
loads, staged 128-column boxes, 3-slot rotating windows, shifted K+3-slot div register ring, wall selects,
chunking and store predicate, statement for statement, and the same choice of tail per warp stream: the
contracted fma(S, 0.25, -0.25 d) unless the tiny-divergence map flags the stream's footprint (run exact
from the start) or its level-0 inputs reached BIG_IN (run again exact).  It exists so the kernel's index
logic and tail selection can be checked against the oracle on a machine without a GPU
(tests/test_jacobi_tb_model.py); it is not used by the product."""
import numpy as np

F = np.float32
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
