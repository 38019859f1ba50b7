"""Every contracted stream of the blocked Jacobi kernel runs one instantiation, whose level-0 loads
reverse the float4 of a lane that mirrors a column wall and leave every other lane as loaded
(csrc/jacobi.cuh, jacobi_tb_kernel).  At every block depth, with both stagings, the first and last
windows (mirrored lanes, the last one at widths that are and are not a multiple of the payload) and the
interior windows equal the oracle bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import bits_equal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(4096, 40), (1000, 61), (364, 50), (132, 37), (96, 20)]
DEPTHS = list(range(1, 14))
_RUN = """
import sys, numpy as np
import webgl_fluid_simulation_b200 as pkg
out = {}
for W, H in %r:
    rng = np.random.default_rng(W + H)
    p = rng.standard_normal((H, W)).astype(np.float32); d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    out[f"{W}_{H}_p"] = p; out[f"{W}_{H}_d"] = d
    for jb in %r:
        s = pkg.FluidSimulation({"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": 8, "PRESSURE_ITERATIONS": 2 * jb + 1},
                                canvas_width=W, canvas_height=H, jacobi_block=jb, sizes=(W, H, 8, 8))
        s.writeField("pressure", p); s.writeField("divergence", d); s.pass_("pressure_solve")
        out[f"{W}_{H}_{jb}"] = s.readField("pressure")
        s.close()
np.savez(sys.argv[1], **out)
""" % (SHAPES, DEPTHS)


@pytest.mark.gpu
@pytest.mark.parametrize("stage", ["tma", "ldgsts"])
def test_mirrored_and_interior_windows_bitwise_every_depth(oracle, tmp_path, stage):
    f = str(tmp_path / f"{stage}.npz")
    env = dict(os.environ, FLUID_TB_STAGE=stage,
               PYTHONPATH=os.pathsep.join([ROOT] + [x for x in [os.environ.get("PYTHONPATH")] if x]))
    r = subprocess.run([sys.executable, "-c", _RUN, f], capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    res = np.load(f)
    for W, H in SHAPES:
        p, d = res[f"{W}_{H}_p"], res[f"{W}_{H}_d"]
        for jb in DEPTHS:
            want = oracle.jacobi(oracle.clear(p, 0.8), d, 2 * jb + 1)
            assert bits_equal(res[f"{W}_{H}_{jb}"], want), (W, H, jb, stage)
