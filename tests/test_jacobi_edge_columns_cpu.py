"""Lane model of one window of the blocked Jacobi kernel: how far the shuffle garbage creeps.

A window is 128 columns; every level takes its x-neighbours from the adjacent lanes, and the outermost
columns have none (modelled as NaN).  If the level-0 column just outside each side of the window is supplied at
level 1 (the staged box holds it), level K is NaN-free exactly on [K - 1, 128 - (K - 1)), so a window needs
HX = roundup(K - 1, 4) halo columns per side; without it the range is [K, 128 - K) and HX = roundup(K, 4).
Walls mirror the loads (p[-1-m] = p[m], p[W+m] = p[W-1-m]), the edge columns included, and the valid columns
then equal K reference sweeps bit for bit, also with the clear pass fused into the level-0 loads."""
import numpy as np
import pytest

DEPTHS = range(1, 14)


def hx(K):
    return (K + 2) // 4 * 4


def mirror(c, W):
    c = np.where(c < 0, -1 - c, c)
    return np.where(c >= W, 2 * W - 1 - c, c)


def reference(p, d, K, scale=None):
    q = p if scale is None else np.float32(scale) * p
    for _ in range(K):
        e = np.pad(q, ((1, 1), (1, 1)), mode="edge")
        q = ((((e[1:-1, :-2] + e[1:-1, 2:]) + e[:-2, 1:-1]) + e[2:, 1:-1]) - d) * np.float32(0.25)
    return q


def window(p, d, x0, K, edge_columns, scale=None):
    """K levels of the 128 columns from x0 (all rows, y walls clamped): (level K, columns)"""
    H, W = p.shape
    cols = np.arange(x0 - 1, x0 + 129)                       # the window and its two edge columns
    ok = (mirror(cols, W) >= 0) & (mirror(cols, W) < W)      # a single reflection reaches the grid
    src = np.clip(mirror(cols, W), 0, W - 1)
    lvl0 = np.where(ok, p[:, src], np.float32(np.nan))
    if scale is not None:
        lvl0 = np.float32(scale) * lvl0
    dw = np.where(ok, d[:, src], np.float32(0))[:, 1:-1]
    q = lvl0[:, 1:-1]
    for t in range(1, K + 1):
        left = np.concatenate([np.full((H, 1), np.nan, np.float32), q[:, :-1]], axis=1)
        right = np.concatenate([q[:, 1:], np.full((H, 1), np.nan, np.float32)], axis=1)
        if t == 1 and edge_columns:
            left[:, 0], right[:, -1] = lvl0[:, 0], lvl0[:, -1]
        e = np.pad(q, ((1, 1), (0, 0)), mode="edge")
        q = ((((left + right) + e[:-2]) + e[2:]) - dw) * np.float32(0.25)
    return q, cols[1:-1]


def fields(W, H=9, seed=0):
    rng = np.random.default_rng(seed + W)
    return rng.standard_normal((H, W)).astype(np.float32), rng.uniform(-1, 1, (H, W)).astype(np.float32)


@pytest.mark.parametrize("K", DEPTHS)
def test_interior_window_valid_range_with_and_without_edge_columns(K):
    p, d = fields(512)
    with np.errstate(invalid="ignore"):
        new, _ = window(p, d, 200, K, True)
        old, _ = window(p, d, 200, K, False)
    fine = lambda q: ~np.isnan(q).any(axis=0)
    assert np.array_equal(fine(new), (np.arange(128) >= K - 1) & (np.arange(128) < 128 - (K - 1)))
    assert np.array_equal(fine(old), (np.arange(128) >= K) & (np.arange(128) < 128 - K))      # the premise
    want = reference(p, d, K)[:, 200:328]
    assert np.array_equal(new[:, fine(new)], want[:, fine(new)])
    assert hx(K) >= K - 1 and hx(K) % 4 == 0 and (hx(K) == 0 or hx(K) - 4 < K - 1)


@pytest.mark.parametrize("scale", [None, 0.8])
@pytest.mark.parametrize("K", DEPTHS)
def test_every_window_of_a_grid_equals_the_reference_on_its_payload(K, scale):
    valid = 128 - 2 * hx(K)
    for W in sorted({valid, valid + 4, 2 * valid - 4, 2 * valid, 3 * valid + 4, 16, 64}):
        if W < K:                       # a single reflection must reach the grid
            continue
        p, d = fields(W, seed=K)
        want = reference(p, d, K, scale)
        for wx in range(-(-W // valid)):
            x0 = wx * valid - hx(K)
            with np.errstate(invalid="ignore"):
                q, cols = window(p, d, x0, K, True, scale)
            out = (np.arange(128) >= hx(K)) & (np.arange(128) < 128 - hx(K)) & (cols >= 0) & (cols < W)
            assert out.any()
            assert np.array_equal(q[:, out].view(np.uint32), want[:, cols[out]].view(np.uint32)), (K, W, wx)
