"""Depth 13, the single-GPU default of a TMA-staged pressure solve (50 sweeps in 4 launches of 13 / 12
instead of 5 of 10), one above the cap of 12 that row slabs, the banded host solve and the cp.async
staging keep.

CPU: the lane-level model at K = 13 against the oracle.  GPU: the library's blocked solve at depth 13
against one sweep per launch and the oracle, bit for bit, and the launch counts of each staging."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import bits_equal
from jacobi_tb_model import jacobi_tb_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_TMA = 13                          # csrc/fluid.cu: KMAX_TMA
K_MAX = 12                          # csrc/fluid.cu: KMAX (cp.async staging, row slabs, host bands)
TINY = 9.4039548e-38                # 2^-123: below it the contracted tail is not exact (EXACT streams)


# ---- CPU: the lane-level model at depth 13 ----------------------------------------------------------
@pytest.mark.parametrize("W,H,R", [(4 * 43, 47, 27), (96, 40, 52), (256, 31, 13), (388, 70, 30)])
def test_model_k13_equals_oracle_sweeps(oracle, W, H, R):
    """Walls, mirrored x-halos (W not a multiple of the 96-column payload) and chunk seams."""
    rng = np.random.default_rng(W + H + R)
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.standard_normal((H, W)).astype(np.float32)
    assert bits_equal(jacobi_tb_model(p, d, K_TMA, R), oracle.jacobi(p, d, K_TMA))


def test_model_k13_fused_clear_and_slab(oracle):
    K = K_TMA
    rng = np.random.default_rng(13)
    H, W = 3 * K + 20, 136
    p = rng.standard_normal((H, W)).astype(np.float32)
    d = rng.standard_normal((H, W)).astype(np.float32)
    assert bits_equal(jacobi_tb_model(p, d, K, 4 * K, scale=0.8), oracle.jacobi(oracle.clear(p, 0.8), d, K))
    full = oracle.jacobi(p, d, K)
    r0, r1 = K + 3, H - K - 2                          # an interior slab: local rows = owned +- K ghosts
    lo, hi = r0 - K, r1 + K
    got = jacobi_tb_model(p[lo:hi], d[lo:hi], K, 9, row_off=lo, out_lo=r0, out_hi=r1, H=H)
    assert bits_equal(got[r0 - lo:r1 - lo], full[r0:r1])


# ---- GPU: the library's blocked solve at depth 13 ---------------------------------------------------
# (W, H, iters, JACOBI_BLOCK, tiny): W = 4096 has the last window with mirrored lanes outside the staged
# box; the other widths are not multiples of the 96-column payload; short grids; iteration counts that
# are not multiples of 13; 0 = the library's default depth; tiny = a patch of divergence values in
# (0, 2^-123), so that the un-contracted (EXACT) streams run too.
DEEP_CASES = [(4096, 96, 50, 0, True), (4096, 64, 26, 13, False), (4096, 80, 50, 13, True),
              (1000, 45, 50, 0, False), (364, 30, 31, 13, True), (532, 7, 15, 0, False),
              (200, 300, 33, 13, True), (92, 3, 16, 0, False), (1028, 130, 39, 0, True)]
_RUN = """
import sys, numpy as np
import webgl_fluid_simulation_b200 as pkg
out = {}
for W, H, iters, jb, tiny in %r:
    rng = np.random.default_rng(W + 3 * H + iters + jb)
    p = rng.standard_normal((H, W)).astype(np.float32); d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    if tiny:
        r, c = min(4, H - H // 3), min(40, W - W // 2)
        d[H // 3:H // 3 + r, W // 2:W // 2 + c] = rng.uniform(0.5, 1, (r, c)).astype(np.float32) * np.float32(%r)
    s = pkg.FluidSimulation({"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": 8, "PRESSURE_ITERATIONS": iters},
                            canvas_width=W, canvas_height=H, jacobi_block=jb, sizes=(W, H, 8, 8))
    s.writeField("pressure", p); s.writeField("divergence", d); s.pass_("pressure_solve")
    k = f"{W}_{H}_{iters}_{jb}"
    out[k] = s.readField("pressure"); out[k + "_launches"] = np.array(s.stat("jacobi_launches"))
    out[k + "_p"] = p; out[k + "_d"] = d
    s.close()
np.savez(sys.argv[1], **out)
""" % (DEEP_CASES, TINY)


@pytest.mark.gpu
def test_depth13_bitwise_vs_naive_and_oracle(oracle, tmp_path):
    """TMA boxes (depth 13 by default) and the cp.async ring (capped at 12; the staging is chosen once
    per process, so each runs in its own) both equal one sweep per launch and the oracle bit for bit."""
    res = {}
    for stage in ("tma", "ldgsts", "naive"):
        f = str(tmp_path / f"{stage}.npz")
        env = dict(os.environ, FLUID_TB_STAGE="ldgsts" if stage == "ldgsts" else "tma",
                   PYTHONPATH=os.pathsep.join([ROOT] + [x for x in [os.environ.get("PYTHONPATH")] if x]))
        code = _RUN.replace("jacobi_block=jb", "jacobi_block=1, flags=pkg.FLAG_NAIVE_JACOBI") if stage == "naive" else _RUN
        r = subprocess.run([sys.executable, "-c", code, f], capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
        assert r.returncode == 0, r.stderr[-2000:]
        res[stage] = np.load(f)
    for W, H, iters, jb, tiny in DEEP_CASES:
        k = f"{W}_{H}_{iters}_{jb}"
        p, d = res["tma"][k + "_p"], res["tma"][k + "_d"]
        if tiny:
            assert np.any((d != 0) & (np.abs(d) < np.float32(TINY))), k
        want = oracle.jacobi(oracle.clear(p, 0.8), d, iters)
        for stage in ("tma", "ldgsts", "naive"):
            assert bits_equal(res[stage][k], want), (k, stage)
        assert int(res["tma"][k + "_launches"]) == -(-iters // K_TMA), k
        assert int(res["ldgsts"][k + "_launches"]) == -(-iters // (K_MAX if jb else 10)), k
