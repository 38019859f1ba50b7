"""Half storage (FLUID_FLAG_HALF_STORAGE) on non-finite and overflowing data, against the oracle's
half mode: every pass once and one whole step.  The fields hold +-0, fp16 subnormals, +-inf and NaN,
and pressure of magnitude 6e4 next to the opposite sign, so that gradientSubtract's results overflow
fp16 when they are stored.  NaN-aware comparison: NaN in the same places, every other element bitwise
(CPU and GPU NaN payloads differ)."""
import numpy as np
import pytest

from sim_harness import make, same_bits, special_fields
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu
DT = 0.016666
SHAPES = [(64, 48, 128, 96), (128, 128, 256, 256), (100, 60, 150, 90)]


@pytest.mark.parametrize("W,H,Wd,Hd", SHAPES)
def test_half_storage_special_values_every_pass_vs_oracle(pkg, oracle, W, H, Wd, Hd):
    """The per-pass sequence of the half-storage parity test, rounded to fp16 after every blit.  The
    written pressure is put back before gradientSubtract, whose +-6e4 steps the clear pass and the
    Jacobi sweeps would otherwise smooth below the fp16 overflow."""
    O = oracle
    R = O.round_half
    v, dye, p = special_fields(O, W, H, Wd, Hd, W + H)
    s = make(pkg, W, H, Wd, Hd, flags=pkg.FLAG_HALF_STORAGE)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    assert same_bits(s.readField("velocity"), v)
    s.pass_("curl"); c = s.readField("curl"); assert same_bits(c, R(O.curl(v)))
    s.pass_("vorticity", DT); v2 = s.readField("velocity")
    assert same_bits(v2, R(O.vorticity(v, c, 30.0, DT)))
    s.pass_("divergence"); d = s.readField("divergence"); assert same_bits(d, R(O.divergence(v2)))
    s.pass_("clear_pressure"); p1 = s.readField("pressure"); assert same_bits(p1, R(O.clear(p, 0.8)))
    s.pass_("jacobi", 5); p2 = p1
    for _ in range(5):
        p2 = R(O.jacobi(p2, d, 1))
    assert same_bits(s.readField("pressure"), p2)
    s.writeField("pressure", p)
    s.pass_("gradient_subtract"); v3 = s.readField("velocity")
    ref_v3 = R(O.gradient_subtract(p, v2))
    assert same_bits(v3, ref_v3)
    assert np.isinf(ref_v3[H // 4:H // 2]).any()                     # the premise: stores that overflow fp16
    s.pass_("advect_velocity", DT); v4 = s.readField("velocity")
    assert same_bits(v4, R(O.advect(v3, v3, DT, 0.2)))
    s.pass_("advect_dye", DT); assert same_bits(s.readField("dye"), R(O.advect(v4, dye, DT, 1.0)))
    s.close()


@pytest.mark.parametrize("W,H,Wd,Hd", SHAPES)
def test_half_storage_special_values_whole_step_vs_oracle(pkg, oracle, W, H, Wd, Hd):
    """One whole step (graph replay, 20 iterations) from the same fields, every field."""
    O = oracle
    v, dye, p = special_fields(O, W, H, Wd, Hd, W + H + 1)
    s = make(pkg, W, H, Wd, Hd, flags=pkg.FLAG_HALF_STORAGE)
    ref = O.OracleSim(W, H, Wd, Hd, half_storage=True)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    s.step(DT); ref.step(DT)
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert same_bits(s.readField(n), getattr(ref, n)), n
    s.close()
