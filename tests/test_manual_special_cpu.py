"""The oracle's MANUAL advection (oracle.advect) against the executed MANUAL_FILTERING shader with inf and NaN
velocity (tests/golden/make_golden_manual_special.py -> manual_special_*.npz), bit for bit with NaN in the same
places, and the premise of that data: every placement class of sim_harness.centre_placements gives a cell that
is NaN in the reference and finite if the velocity sample at a cell centre were taken as the own texel alone."""
import numpy as np
import pytest

import linear_advection_model as M
from conftest import golden
from sim_harness import CENTRE_SPECIALS, centre_placements, same_bits

SHAPES = ["16x16_16x16", "32x32_64x64", "128x16_128x16"]
CASES = [f"{k}_{c}" for k in range(len(CENTRE_SPECIALS)) for c in (0, 1)]


def own_texel(v, src, g, diss):
    """the manual shader with the velocity sample at a cell centre replaced by the cell's own texel"""
    return M.advect(v, src, float(g["dt"]), diss, weights="mix", coord="uvts", own_texel=True)


@pytest.mark.parametrize("shape", SHAPES)
def test_oracle_matches_executed_manual_shader_with_nonfinite_velocity(oracle, shape):
    g = golden(f"manual_special_{shape}")
    dt, dv, dd = float(g["dt"]), float(g["velocity_dissipation"]), float(g["density_dissipation"])
    for case in CASES:
        v = g[f"{case}_in_velocity"]
        assert not np.isfinite(v).all()
        assert same_bits(oracle.advect(v, v, dt, dv), g[f"{case}_advect_velocity"]), case
        assert same_bits(oracle.advect(v, g["in_dye"], dt, dd), g[f"{case}_advect_dye"]), case


@pytest.mark.parametrize("shape", SHAPES)
def test_every_placement_separates_the_reference_from_the_own_texel_rule(oracle, shape):
    """For each placement class and case, one of the cells whose centre sample weighs the special by 0 is NaN in
    the golden and finite under the own-texel rule, in the velocity pass and (dye grid == sim grid) the dye pass."""
    g = golden(f"manual_special_{shape}")
    W, H, Wd, Hd = (int(g[k]) for k in ("W", "H", "Wd", "Hd"))
    dv, dd = float(g["velocity_dissipation"]), float(g["density_dissipation"])
    passes = [("velocity", None, dv)] + ([("dye", g["in_dye"], dd)] if (W, H) == (Wd, Hd) else [])
    for case in CASES:
        v = g[f"{case}_in_velocity"]
        for field, src, diss in passes:
            ref = g[f"{case}_advect_{field}"]
            own = own_texel(v, v if src is None else src, g, diss)
            for name, (r, c) in centre_placements(W, H).items():
                cells = [(r, c - 1), (r - 1, c), (r - 1, c - 1)]
                hit = [(y, x) for y, x in cells
                       if y >= 0 and x >= 0 and np.isnan(ref[y, x]).all() and np.isfinite(own[y, x]).all()]
                assert hit, (case, field, name)
