"""The plan of a frame on row slabs (slab.draw_plan, mirrored by fluid.cu draw / draw_ghost_rows / post_fx_chains)
checked on CPU against brute-force enumeration of every LINEAR tap a slab rank's frame makes, in the kernels' fp32
arithmetic: the display and shading taps of its band of the target (display_kernel), the bloom prefilter's taps of
its band of the bloom FBO (bloom_prefilter_kernel), and the sunrays mask's taps of the dye rows it owns
(sunrays_mask_kernel).  Every tap must lie in the rank's owned dye rows plus the ghost rows the plan refreshes, and
the bands a gather assembles must tile the buffer."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

F = np.float32


def tap_rows(n_src, rows, n_tgt, shading=False):
    """Source rows read by the LINEAR fetches (passes.cuh linear_fetch: floor, then texel_index's clamp) at target
    rows `rows` of an n_tgt-row target: uv.y = (j + 0.5) / n_tgt, and with shading also uv.y +- 1 / n_tgt."""
    uv = (np.asarray(rows).astype(F) + F(0.5)) / F(n_tgt)
    uvs = [uv]
    if shading:
        ts = F(1.0 / n_tgt)                                   # texelSize: a JS double narrowed on the host
        uvs += [uv + ts, uv - ts]
    out = []
    for u in uvs:
        fj = np.floor(u * F(n_src) - F(0.5))
        out += [np.clip(fj, 0, n_src - 1), np.clip(fj + F(1), 0, n_src - 1)]
    return np.concatenate(out).astype(np.int64)


def reach(taps, d0, d1):
    """Rows beyond the owned dye rows [d0, d1) that `taps` read, on the farther side."""
    return max(d0 - int(taps.min()), int(taps.max()) - (d1 - 1), 0) if len(taps) else 0


def geometries(n, seed):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        world = int(rng.integers(2, 9))
        dye_h = int(rng.integers(28, 2500))
        height = int(rng.choice([rng.integers(world, 64), rng.integers(world, 4000)]))
        bloom_h = int(rng.choice([0, rng.integers(1, 40), rng.integers(1, 600)]))
        yield world, dye_h, height, bloom_h, bool(rng.integers(0, 2))


FIXED = [(2, 1024, 1080, 256, True), (3, 1536, 640, 196, True), (8, 2048, 1080, 256, True), (4, 369, 8, 0, False),
         (6, 369, 8, 0, False), (5, 4096, 2160, 13, True), (2, 128, 8, 4, True), (7, 300, 1081, 2, False)]


@pytest.mark.parametrize("seed", range(4))
def test_every_tap_lies_in_the_rows_the_plan_refreshes(seed):
    from webgl_fluid_simulation_b200.slab import draw_plan, rows
    slack = []
    cases = list(geometries(400, seed)) + (FIXED if seed == 0 else [])
    for world, dye_h, height, bloom_h, sunrays in cases:
        need = 0
        plans = [draw_plan(dye_h, height, r, world, bloom_h, sunrays) for r in range(world)]
        assert len({p["ghost"] for p in plans}) == 1                 # exchange sizes match on every rank
        for r, p in enumerate(plans):
            d0, d1 = rows(dye_h, r, world)                            # the dye rows the rank owns
            y0, y1 = p["band"]
            taps = [tap_rows(dye_h, np.arange(y0, y1), height, shading=True)]
            if bloom_h:
                b0, b1 = p["bloom_rows"]
                taps.append(tap_rows(dye_h, np.arange(b0, b1), bloom_h))
            if sunrays:
                assert p["mask_rows"] == (d0, d1)
                taps.append(tap_rows(dye_h, np.arange(d0, d1), dye_h))
            need = max(need, reach(np.concatenate(taps), d0, d1))
            assert p["gathers"] == (bloom_h > 0) + sunrays
        assert need <= plans[0]["ghost"], (world, dye_h, height, bloom_h, sunrays, need, plans[0]["ghost"])
        slack.append(plans[0]["ghost"] - need)
    assert min(slack) <= 2                                            # a bound, and not a loose one everywhere


def test_mask_and_bloom_alone():
    """The mask at dye texel centres reads one row beyond the owned ones (its +y tap has weight 0 but is read: an
    inf there gives NaN); the prefilter's reach follows the bloom FBO's height, not the target's."""
    from webgl_fluid_simulation_b200.slab import draw_ghost_rows, rows
    for world, dye_h in ((2, 128), (3, 1000), (8, 4096), (5, 777)):
        r = max(reach(tap_rows(dye_h, np.arange(*rows(dye_h, k, world)), dye_h), *rows(dye_h, k, world)) for k in range(world))
        assert r == 1
    for world, dye_h, bloom_h in ((2, 1024, 4), (4, 2048, 16), (3, 999, 7)):
        r = max(reach(tap_rows(dye_h, np.arange(*rows(bloom_h, k, world)), bloom_h), *rows(dye_h, k, world))
                for k in range(world))
        assert r <= draw_ghost_rows(dye_h, 10 ** 6, bloom_h) and draw_ghost_rows(dye_h, 10 ** 6, bloom_h) > draw_ghost_rows(dye_h, 10 ** 6)


def test_bands_tile_every_gathered_buffer():
    from webgl_fluid_simulation_b200.slab import draw_plan
    for world, dye_h, height, bloom_h in ((2, 1024, 1080, 256), (3, 225, 640, 13), (8, 512, 807, 5), (4, 150, 3, 2)):
        plans = [draw_plan(dye_h, height, r, world, bloom_h, True) for r in range(world)]
        for key, n in (("band", height), ("bloom_rows", bloom_h), ("mask_rows", dye_h)):
            b = [p[key] for p in plans]
            assert b[0][0] == 0 and b[-1][1] == n and all(x[1] == y[0] for x, y in zip(b, b[1:])), (key, b)


def test_gather_bytes_from_shapes():
    from webgl_fluid_simulation_b200.slab import gather_bytes
    # the desktop frame on a 1920 x 1080 canvas: a 455 x 256 bloom FBO, a 1820 x 1024 dye
    assert gather_bytes(1820, 1024, 455, 256, True) == 16 * 455 * 256 + 4 * 1820 * 1024
    assert gather_bytes(1820, 1024) == 0
