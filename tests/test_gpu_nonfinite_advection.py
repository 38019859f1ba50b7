"""fp32 MANUAL advection with inf and NaN velocity against the oracle, per pass, over whole steps and on batch
handles, NaN-aware bit for bit (sim_harness.same_bits).

On power-of-two grids the reference's velocity sample at a cell centre is mix(mix(a,b,0), mix(c,d,0), 0): the
own texel where the +x, +y and +xy neighbours (clamped to the edge) are finite, NaN where one is inf or NaN, and
then the cell's back-trace and every channel of its result are NaN.  The kernels that compute that sample without
a coordinate (kOwnTexel in passes.cuh) are the one-cell POW2 velocity and dye SAME kernels and the 4-cell
velocity and dye SAME kernels, plain and BATCH; FLUID_STAT_ADVECT4_LAUNCHES tells the 4-cell ones from the
others.  The special values sit where sim_harness.centre_placements puts them: interior, across the 4-cell
lane layout and block edges, on the last column and row, and on a batch member's first and last rows."""
import numpy as np
import pytest

import linear_advection_model as M
from sim_harness import CENTRE_SPECIALS, centre_special_velocity, make, rand_fields, same_bits
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu

DT = 0.016666
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
CASES = [(k, c) for k in range(len(CENTRE_SPECIALS)) for c in (0, 1)]

# (W, H, Wd, Hd, flag names, 4-cell launches per pass (velocity, dye)).  The first six run a kOwnTexel kernel in
# both passes, the next two in their velocity pass; every other pass is a control that samples velocity through a
# coordinate.
SHAPES = [
    (64, 64, 64, 64, (), (0, 0)),                       # one-cell POW2 velocity, one-cell dye SAME
    (128, 128, 128, 128, ("TILED_PASSES",), (0, 0)),    # the same kernels on a grid the 4-cell ones could take
    (128, 128, 128, 128, (), (1, 1)),                   # velocity4, dye4 SAME
    (256, 64, 256, 64, (), (1, 1)),
    (1024, 512, 1024, 512, (), (1, 1)),
    (256, 256, 256, 256, (), (1, 1)),
    (128, 128, 256, 256, (), (1, 1)),                   # velocity4; dye4 !SAME
    (32, 32, 64, 64, (), (0, 0)),                       # one-cell POW2 velocity; one-cell dye !SAME
    (36, 20, 54, 30, (), (0, 0)),                       # ragged
    (128, 128, 128, 128, ("LINEAR_ADVECTION",), (1, 1)),
    (64, 64, 64, 64, ("HALF_STORAGE",), (0, 0)),        # MANUAL half storage: the !POW2 forms
]


def flags_of(pkg, names):
    f = 0
    for n in names:
        f |= getattr(pkg, "FLAG_" + n)
    return f


def reference(O, names, v, src, diss):
    with np.errstate(all="ignore"):
        if "LINEAR_ADVECTION" in names:
            return M.advect(v, src, DT, diss)
        r = O.advect(v, src, DT, diss)
    return O.round_half(r) if "HALF_STORAGE" in names else r


@pytest.mark.parametrize("field", ["velocity", "dye"])
@pytest.mark.parametrize("W,H,Wd,Hd,names,n4", SHAPES)
def test_advection_pass_with_nonfinite_velocity_vs_oracle(pkg, oracle, W, H, Wd, Hd, names, n4, field):
    """One pass from written fields, every case: velocity advected by itself, or dye by the written velocity."""
    O = oracle
    s = make(pkg, W, H, Wd, Hd, flags=flags_of(pkg, names))
    _, dye, _ = rand_fields(W, H, Wd, Hd, W + Wd)
    if "HALF_STORAGE" in names:
        dye = O.round_half(dye)
    for k, c in CASES:
        v = centre_special_velocity(W, H, CENTRE_SPECIALS[k], c, 10 * W + H + 3 * k + c)
        if "HALF_STORAGE" in names:
            v = O.round_half(v)
        s.writeField("velocity", v); s.writeField("dye", dye)
        n0 = s.stat("advect4_launches")
        s.pass_("advect_" + field, DT)
        assert s.stat("advect4_launches") - n0 == n4[field == "dye"]
        want = reference(O, names, v, v, 0.2) if field == "velocity" else reference(O, names, v, dye, 1.0)
        assert same_bits(s.readField(field), want), (k, c)
    s.close()


def pre_advection_velocity(O, v, p, dt=DT):
    """The velocity the first step's advection reads (OracleSim.step up to gradientSubtract, default config)."""
    with np.errstate(all="ignore"):
        v = O.vorticity(v, O.curl(v), 30.0, float(np.float32(dt)))
        return O.gradient_subtract(O.jacobi(O.clear(p, 0.8), O.divergence(v), 20), v)


def reaches_advection(O, v, p, dt=DT):
    """Premise: finite and non-finite velocity side by side where the advection starts.  The vorticity pass
    clamps written velocity to [-1000, 1000]; an inf or NaN in pressure spreads through the Jacobi sweeps, and
    gradientSubtract turns it into inf or NaN velocity."""
    a = pre_advection_velocity(O, v, p, dt)
    bad = ~np.isfinite(a).all(axis=-1)
    return bad.any() and (~bad).any() and (bad[:, 1:] != bad[:, :-1]).any() and (bad[1:] != bad[:-1]).any()


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("W,H,Wd,Hd,k", [(64, 64, 64, 64, 0), (256, 256, 256, 256, 1), (128, 128, 256, 256, 2),
                                         (1024, 512, 1024, 512, 0)])
def test_whole_steps_from_nonfinite_fields_vs_oracle(pkg, oracle, W, H, Wd, Hd, k, graph):
    """Three steps from written velocity with the placements of one case and pressure holding the case's value at
    a few cells; all five fields after every step."""
    O = oracle
    v = centre_special_velocity(W, H, CENTRE_SPECIALS[k], k % 2, W + H)
    dye, p = rand_fields(W, H, Wd, Hd, W * 7)[1:]
    for r, c in ((H // 2, W // 3), (H - 1, W // 2), (H // 4, W - 1)):
        p[r, c] = np.float32(CENTRE_SPECIALS[k])
    assert reaches_advection(O, v, p)
    s = make(pkg, W, H, Wd, Hd, flags=0 if graph else pkg.FLAG_NO_GRAPH)
    ref = O.OracleSim(W, H, Wd, Hd)
    s.writeField("velocity", v); s.writeField("dye", dye); s.writeField("pressure", p)
    ref.velocity, ref.dye, ref.pressure = v.copy(), dye.copy(), p.copy()
    for step in range(3):
        s.step(DT)
        with np.errstate(all="ignore"):
            ref.step(DT)
        for n in FIELDS:
            assert same_bits(s.readField(n), getattr(ref, n)), (step, n)
    assert s.stat("graph_launches") == (3 if graph else 0)
    s.close()


def member_fields(B, W, H, seed):
    """(B, H, W, 2) velocity, (B, H, W, 4) dye and (B, H, W) pressure.  Member m's last row and member m + 1's
    first row hold a special value (cycling through the cases) in velocity, at columns 32, 128 and W - 1 beside a
    finite -0.0, and in pressure, at columns W / 4 and 3 W / 4: the first member's last-row velocity must not take
    the next member's first row as its +y neighbour."""
    rng = np.random.default_rng(seed)
    v = (rng.standard_normal((B, H, W, 2)) * 50).astype(np.float32)
    dye = rng.random((B, H, W, 4), dtype=np.float32)
    p = rng.standard_normal((B, H, W)).astype(np.float32)
    for m in range(B):
        k, c = CASES[m % len(CASES)]
        x = np.float32(CENTRE_SPECIALS[k])
        for mm, row, pc in ((m, H - 1, W // 4), ((m + 1) % B, 0, 3 * W // 4)):
            p[mm, row, pc] = x
            for col in (32, 128, W - 1):
                if col < W:
                    v[mm, row, col, c] = x
                    v[mm, row, col - 1, c] = np.float32(-0.0)
    return v, dye, p


@pytest.mark.parametrize("per_member_dt", [False, True])
@pytest.mark.parametrize("B,W,H", [(3, 128, 2), (5, 128, 2), (4, 256, 256)])
def test_batch_members_with_nonfinite_fields_vs_oracle(pkg, oracle, B, W, H, per_member_dt):
    """Every member of a batch against OracleSim given that member's fields and dt, two steps; a member's last
    row clamps its +y neighbour to itself and must never read the next member's first row."""
    O = oracle
    b = pkg.FluidBatch(B, {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(W, H)}, canvas_width=W,
                       canvas_height=H, sizes=(W, H, W, H))
    v, dye, p = member_fields(B, W, H, B * W + H)
    dts = [DT * (0.5 + 0.25 * m) for m in range(B)] if per_member_dt else [DT] * B
    for m in range(B):
        assert reaches_advection(O, v[m], p[m], dts[m]), m
    b.writeField("velocity", v); b.writeField("dye", dye); b.writeField("pressure", p)
    refs = []
    for m in range(B):
        r = O.OracleSim(W, H, W, H)
        r.velocity, r.dye, r.pressure = v[m].copy(), dye[m].copy(), p[m].copy()
        refs.append(r)
    n0 = b.stat("advect4_launches")
    for step in range(2):
        b.step(dts if per_member_dt else DT)
        with np.errstate(all="ignore"):
            for r, dt in zip(refs, dts):
                r.step(dt)
        for n in FIELDS:
            got = b.readField(n)
            for m, r in enumerate(refs):
                assert same_bits(got[m], getattr(r, n)), (step, n, m)
    assert b.stat("advect4_launches") - n0 == 4
    b.close()
