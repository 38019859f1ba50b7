"""Every contracted stream of the blocked Jacobi kernel runs one instantiation, whose level-0 loads
reverse the float4 of a lane that mirrors a column wall and leave every other lane as loaded
(csrc/jacobi.cuh, jacobi_tb_kernel).  At every block depth the first and last windows (mirrored lanes,
the last one at widths that are and are not a multiple of the payload) and the interior windows equal
the oracle bit for bit."""
import numpy as np
import pytest

from conftest import bits_equal

SHAPES = [(4096, 40), (1000, 61), (364, 50), (132, 37), (96, 20)]
DEPTHS = list(range(1, 14))


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", SHAPES)
def test_mirrored_and_interior_windows_bitwise_every_depth(oracle, W, H):
    import webgl_fluid_simulation_b200 as pkg
    rng = np.random.default_rng(W + H)
    p = rng.standard_normal((H, W)).astype(np.float32); d = rng.uniform(-1, 1, (H, W)).astype(np.float32)
    for jb in DEPTHS:
        s = pkg.FluidSimulation({"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": 8, "PRESSURE_ITERATIONS": 2 * jb + 1},
                                canvas_width=W, canvas_height=H, jacobi_block=jb, sizes=(W, H, 8, 8))
        s.writeField("pressure", p); s.writeField("divergence", d); s.pass_("pressure_solve")
        got = s.readField("pressure")
        assert s.stat("jacobi_exact_streams") == 0, (W, H, jb)
        s.close()
        assert bits_equal(got, oracle.jacobi(oracle.clear(p, 0.8), d, 2 * jb + 1)), (W, H, jb)
