"""Lane-level numpy model of csrc/jacobi.cuh::jacobi_tb_kernel — same window geometry, mirrored
loads, staged 128-column boxes, 3-slot rotating windows, shifted K+3-slot div register ring, wall selects,
chunking and store predicate, statement for statement.  It exists so the kernel's index logic can be checked against the oracle
on a machine without a GPU (tests/test_jacobi_tb_model.py); it is not used by the product."""
import numpy as np

F = np.float32


def _shfl_up(x):      # lane l receives lane l-1 (lane 0 keeps its own value)
    return np.concatenate([x[:1], x[:-1]])


def _shfl_down(x):    # lane l receives lane l+1 (lane 31 keeps its own value)
    return np.concatenate([x[1:], x[-1:]])


def _jacobi4(below, c, above, d):
    l = _shfl_up(c[:, 3]); r = _shfl_down(c[:, 0])
    o = np.empty_like(c)
    o[:, 0] = ((((l + c[:, 1]) + below[:, 0]) + above[:, 0]) - d[:, 0]) * F(0.25)
    o[:, 1] = ((((c[:, 0] + c[:, 2]) + below[:, 1]) + above[:, 1]) - d[:, 1]) * F(0.25)
    o[:, 2] = ((((c[:, 1] + c[:, 3]) + below[:, 2]) + above[:, 2]) - d[:, 2]) * F(0.25)
    o[:, 3] = ((((c[:, 2] + r) + below[:, 3]) + above[:, 3]) - d[:, 3]) * F(0.25)
    return o


def jacobi_tb_model(pin, div, K, rows_per_chunk, scale=None, row_off=0, out_lo=None, out_hi=None,
                    H=None, pout=None):
    """pin/div: local buffers (rows x W).  Returns pout (local buffer; untouched rows stay NaN)."""
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
    lane = np.arange(32)
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
        nsteps = y1 - ys + K
        # TMA staging: step s takes row ys + s of the 128-column box from column x0, zero outside the
        # buffer's rows and the grid's columns; a lane reads its column group clamped into the box
        x0 = wx * VALID - HX
        cols = np.minimum(np.maximum(lc, x0), x0 + 124)[:, None] + np.arange(4)[None, :]
        inside = (cols >= 0) & (cols < W)

        def load(buf, r):
            v = np.zeros((32, 4), F)
            if 0 <= r - row_off < buf.shape[0]:
                v[inside] = buf[r - row_off][cols[inside]]
            v[rev] = v[rev][:, ::-1]
            return v

        w = np.zeros((K, 3, 32, 4), F)
        dr = np.full((RD, 32, 4), np.nan, F)
        rout = ys - K
        for s0 in range(0, nsteps, U):
            edge = (ys + s0 - K <= 0) or (ys + s0 + 2 >= H - 1)
            for ph in range(U):
                inn = load(pin, ys + s0 + ph); dv = load(div, ys + s0 + ph)
                if scale is not None:
                    inn = F(scale) * inn
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
                    with np.errstate(invalid="ignore"):
                        o = _jacobi4(below, c, above, d)
                    if t < K:
                        w[t, (ph + 2) % 3] = o
                    elif y0 <= rout < y1:
                        for l in np.nonzero(lane_out)[0]:
                            pout[rout - row_off, gx[l]:gx[l] + 4] = o[l]
                rout += 1
            for j in range(K):
                dr[j] = dr[j + 3]
    return pout
