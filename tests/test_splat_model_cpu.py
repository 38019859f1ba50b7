"""Premises of the per-texel splat interval (tests/splat_model.py), on the CPU:

* the oracle (glibc expf, under 1 ulp) lies inside it on every grid, base, storage format, radius and
  canvas the GPU file checks;
* it is tight enough to catch real bugs: each mutant below -- the model's own arithmetic with one
  change -- falls outside it on hundreds of texels;
* the canvases the GPU file uses do what they are there for (a radius that depends on the narrowing
  of the aspect, an aspect below 1)."""
import numpy as np
import pytest

import splat_model as M
from splat_model import BASES, CANVASES, GRIDS, NARROWING_CANVAS, RADII, bases, records

F32 = np.float32
def oracle_splats(O, base, recs, aspect, radius, half):
    """The oracle's splat() per record on one plane, rounded to fp16 after each in half storage."""
    out = O.round_half(base) if half else base.copy()
    C = base.shape[-1]
    for r in recs.tolist():
        col = (r[2], r[3], 0.0) if C == 2 else tuple(r[4:7])
        out = O.splat(out, float(aspect), r[0], r[1], col, float(radius))
        if half:
            out = O.round_half(out)
    return out


def assert_inside(got, lo, hi, what):
    n, bad = M.check_splat(got, lo, hi)
    assert n == 0, (what, n, bad)


def check_oracle(O, W, H, Wd, Hd, kind, half, recs, canvas, splat_radius, seed):
    aspect = M.aspect_of(*canvas)
    radius = M.radius_of(splat_radius, *canvas)
    assert radius == O.correct_radius(splat_radius, canvas[0] / canvas[1])
    for name, base in zip(("velocity", "dye"), bases(kind, W, H, Wd, Hd, seed)):
        if half:
            base = M.store(base, True)
        got = oracle_splats(O, base, recs, aspect, radius, half)
        lo, hi = M.splat_interval(base, recs, aspect, radius, half=half)
        assert_inside(got, lo, hi, name)


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
@pytest.mark.parametrize("kind", BASES)
@pytest.mark.parametrize("W,H,Wd,Hd", GRIDS)
def test_oracle_inside_interval(oracle, W, H, Wd, Hd, kind, half):
    recs = records(24, W + H, [(W, H), (Wd, Hd)])
    check_oracle(oracle, W, H, Wd, Hd, kind, half, recs, (W, H), 0.25, seed=W * 3 + H)


@pytest.mark.parametrize("half", [False, True], ids=["fp32", "half"])
@pytest.mark.parametrize("canvas", CANVASES, ids=lambda c: f"{c[0]}x{c[1]}")
@pytest.mark.parametrize("splat_radius", RADII)
def test_oracle_inside_interval_radius_and_canvas(oracle, splat_radius, canvas, half):
    W, H, Wd, Hd = 114, 64, 228, 128
    recs = records(40, 7, [(W, H), (Wd, Hd)])
    check_oracle(oracle, W, H, Wd, Hd, "nasty", half, recs, canvas, splat_radius, seed=3)


def test_oracle_far_field_and_texel_centre_inside_interval(oracle):
    """One plane on a zero base, colour 1: the value is e itself, from 1 at a texel centre (q == -0)
    through the subnormal band to 0."""
    W, H = 228, 128
    aspect, radius = M.aspect_of(W, H), M.radius_of(0.25, W, H)
    for x, y in ((M.uv(W)[57], M.uv(H)[100]), (-0.45, 0.5), (0.5, 1.45)):
        rec = np.array([[x, y, 0, 0, 1, 1, 1]], F32)
        base = np.zeros((H, W, 4), F32)
        got = oracle_splats(oracle, base, rec, aspect, radius, False)
        lo, hi = M.splat_interval(base, rec, aspect, radius)
        assert_inside(got, lo, hi, (x, y))


# ---- the mutants -----------------------------------------------------------------------------------
# Each is the model's arithmetic with one change, on one channel of colour 1 over a zero base, where
# the value is e itself (a correctly rounded expf unless the mutant changes it).  The interval must reject each on hundreds of texels.
MUT_W, MUT_H = 228, 128          # ragged in both directions
MUT_RECS = [(0.3, 0.6), (0.5, 0.5), (-0.2, 0.1), (0.9, 1.3)]     # near and far: every magnitude of q


def rejected(mutant, canvas=(MUT_W, MUT_H), splat_radius=0.25, W=MUT_W, H=MUT_H):
    """How many texels the interval rejects, summed over MUT_RECS; `mutant(x, y, aspect, radius)`
    returns the mutant's (H, W) values."""
    aspect, radius = M.aspect_of(*canvas), M.radius_of(splat_radius, *canvas)
    total = 0
    for x, y in MUT_RECS:
        rec = np.array([[x, y, 0, 0, 1, 0, 0]], F32)
        lo, hi = M.splat_interval(np.zeros((H, W, 4), F32), rec, aspect, radius)
        got = np.zeros((H, W, 4), F32)
        got[..., 0] = mutant(x, y, aspect, radius)
        got[..., 3] = 1.0
        # the unmutated arithmetic is inside, everywhere
        exact = got.copy()
        exact[..., 0] = M.exp_rn(M.quotient(M.uv(W), M.uv(H), x, y, aspect, radius))
        assert M.check_splat(exact, lo, hi)[0] == 0
        total += M.check_splat(got, lo, hi)[0]
    return total


def test_narrowing_canvas_radius_differs_between_double_and_float_aspect():
    cw, ch = NARROWING_CANVAS
    assert cw / ch > 1
    good = M.radius_of(0.25, cw, ch)
    bad = F32(0.25 / 100.0 * float(F32(cw / ch)))
    assert good == F32(0.00355) and bad != good, (good, bad)
    assert M.aspect_of(cw, ch) == F32(cw) / F32(ch)


def test_aspect_below_one_does_not_scale_the_radius():
    for cw, ch in CANVASES:
        if cw < ch:
            assert M.radius_of(0.25, cw, ch) == F32(0.0025)
            assert M.radius_of(1.0, cw, ch) == F32(0.01)
            break
    else:
        pytest.fail("no canvas with aspect < 1")


def test_mutant_radius_from_float_aspect_is_rejected():
    cw, ch = NARROWING_CANVAS

    def mutant(x, y, aspect, radius):
        bad = F32(0.25 / 100.0 * float(F32(cw / ch)))
        assert bad != radius
        return M.exp_rn(M.quotient(M.uv(MUT_W), M.uv(MUT_H), x, y, aspect, bad))
    assert rejected(mutant, canvas=NARROWING_CANVAS) >= 5000


def test_mutant_uv_by_reciprocal_is_rejected():
    def mutant(x, y, aspect, radius):
        ux = (np.arange(MUT_W, dtype=F32) + F32(0.5)) * F32(1.0 / MUT_W)
        uy = (np.arange(MUT_H, dtype=F32) + F32(0.5)) * F32(1.0 / MUT_H)
        assert not np.array_equal(ux, M.uv(MUT_W))
        return M.exp_rn(M.quotient(ux, uy, x, y, aspect, radius))
    assert rejected(mutant) >= 1000


@pytest.mark.parametrize("direction", [1, -1], ids=["up", "down"])
def test_mutant_q_one_ulp_off_is_rejected(direction):
    def mutant(x, y, aspect, radius):
        return M.exp_rn(M.step_ulps(M.quotient(M.uv(MUT_W), M.uv(MUT_H), x, y, aspect, radius), direction))
    assert rejected(mutant) >= 5000


def test_mutant_e_eight_ulp_off_where_q_is_large_is_rejected():
    def mutant(x, y, aspect, radius):
        q = M.quotient(M.uv(MUT_W), M.uv(MUT_H), x, y, aspect, radius)
        e = M.exp_rn(q)
        return np.where(np.abs(q) > 8, M.step_ulps(e, 8), e)
    assert rejected(mutant) >= 5000


def test_mutant_flushing_subnormal_e_is_rejected():
    """expf compiled with -ftz=true: subnormal results become 0."""
    def mutant(x, y, aspect, radius):
        e = M.exp_rn(M.quotient(M.uv(MUT_W), M.uv(MUT_H), x, y, aspect, radius))
        return np.where(e < np.finfo(F32).tiny, F32(0.0), e)
    assert rejected(mutant) >= 1000


def test_check_splat_nan_inf_and_signed_zero():
    lo = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0], F32)
    hi = lo.copy()
    assert M.check_splat(lo.copy(), lo, hi)[0] == 0
    for k, wrong in enumerate([1.0, np.float32(3e38), np.nan, -0.0, 0.0, np.nan]):
        got = lo.copy()
        got[k] = wrong
        n, bad = M.check_splat(got, lo, hi)
        assert n == 1 and bad[0][0] == (k,), (k, bad)
    # -0 + e*c where e*c == +0 is +0; a -0 base with a -0 term stays -0
    lo, hi = M.apply(np.full((1, 1, 2), -0.0, F32), np.full((1, 1, 2), -0.0, F32),
                     np.zeros((1, 1), F32), np.zeros((1, 1), F32), (0.5, -0.5))
    assert not np.signbit(lo[0, 0, 0]) and not np.signbit(hi[0, 0, 0])
    assert np.signbit(lo[0, 0, 1]) and np.signbit(hi[0, 0, 1])
