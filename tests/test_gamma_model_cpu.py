"""Premises of the per-texel display interval (display_model.display, tests/gamma_model.py), on the CPU:

* the oracle (glibc powf, within 1 ulp) lies inside it at every texel, under every background, on the
  inputs the GPU file draws: the executed-shader goldens, seeded, zero and dim dye (bk across the knee
  of linearToGamma), dithering textures of other shapes, of a wide range and large enough that noise
  overflows, and dye holding +-inf, NaN, -2, subnormal and 1e30 texels;
* the display model equals the oracle bit for bit on that non-finite dye (C's fmaxf / fminf drop NaN);
* it is tight enough to catch real bugs: each mutant below -- the model's arithmetic with one change --
  falls outside it on hundreds of texels of at least one input.

Deleting fmaxf(bk, 0) is an equivalent mutant wherever bk is finite or NaN: powf of a negative bk or
of NaN is NaN, and the knee's fmaxf turns that into 0, as it does powf(0) = 0.  It differs only where
bk = -inf (powf(-inf, y) = +inf).  The bloom FBO never holds an inf (a LINEAR weight of 0 times an
inf is NaN), so only a dithering value below -FLT_MAX / 2, whose noise overflows to -inf, gets there.

The knee constants 1.055f or 0.055f moved by one ulp stay inside the interval on every input here: the
change is smaller than the width POWF_ULP gives 1.055 p, even where c = 0 and the frame is bare.  test_deleting_the_bk_clamp_is_equivalent_except_at_minus_inf
pins both halves."""
import numpy as np
import pytest

import display_model as M
import gamma_model as G
from conftest import golden
from display_harness import BACK_RGB, BACKGROUNDS, CASES
from oracle import oracle as O

F32 = np.float32
ALL3 = M.ALL3
def oracle_frame(O, c, background):
    return O.render_postfx(c["dye"], c["w"], c["h"], c["dither"], cfg=c["cfg"], back_rgb=BACK_RGB,
                           background=background, aspect=c["w"] / c["h"])


@pytest.mark.parametrize("bg", list(BACKGROUNDS))
@pytest.mark.parametrize("name", list(CASES))
def test_oracle_inside_interval(oracle, name, bg):
    c = CASES[name]
    r = oracle_frame(oracle, c, BACKGROUNDS[bg])
    d = M.display(c["dye"], c["w"], c["h"], ALL3, r["bloom"], r["sunrays"], c["dither"], BACK_RGB, BACKGROUNDS[bg],
                  c["w"] / c["h"])
    n, bad = G.check_display(r["target"], d["lo"], d["hi"])
    assert n == 0, (n, bad)


def unclamped_argument(c, bl):
    """bl + noise / 255 without fmaxf(bk, 0)."""
    w, h, dither = c["w"], c["h"], c["dither"]
    dsx, dsy = M.dither_scale(w, h, dither)
    uvx, uvy = M.uv_grid(w, h)
    noise = M.linear_fetch(dither, uvx * dsx, uvy * dsy, repeat=True)[..., :1] * F32(2) - F32(1)
    return bl + noise / F32(255)


def pow_argument(c, r, keywords=ALL3, unclamped=False):
    _, bl = M.colour_terms(c["dye"], c["w"], c["h"], keywords, r["bloom"], r["sunrays"])
    return unclamped_argument(c, bl) if unclamped else M.gamma_argument(bl, c["dither"], c["w"], c["h"])


def test_inputs_reach_what_they_are_there_for(oracle):
    """bk spans the knee (zero and dim dye), a wide range (wide dither), +inf and (before fmaxf) -inf
    (overflowing dither); the non-finite dye makes every colour of the bloom FBO NaN -- a LINEAR weight
    of 0 times an inf is NaN, so the bloom FBO never holds an inf -- and puts NaN into the oracle's frame."""
    knee = F32(0.055 / 1.055) ** F32(2.4)
    with np.errstate(invalid="ignore", over="ignore"):
        bk = {k: pow_argument(CASES[k], oracle_frame(oracle, CASES[k], 0)) for k in CASES}
        nf = oracle_frame(oracle, CASES["nonfinite"], 0)
    for k in ("zero", "dim"):
        assert np.count_nonzero((bk[k] > 0) & (bk[k] < knee)) > 1000, k
        assert np.count_nonzero(bk[k] > knee) > 1000, k
    assert np.count_nonzero(bk["zero"] == 0) > 10000
    assert bk["wide_dither"].max() > 2.0 ** 50 and bk["wide_dither"].min() < 8
    assert np.count_nonzero(np.isposinf(bk["overflow_dither"])) > 1000
    with np.errstate(over="ignore"):
        bl = pow_argument(CASES["overflow_dither"], oracle_frame(oracle, CASES["overflow_dither"], 0), unclamped=True)
    assert np.count_nonzero(np.isneginf(bl)) > 1000
    assert np.isnan(nf["bloom"][..., :3]).all() and np.isnan(nf["target"]).any()
    for k in ("postfx_64_to_128", "postfx_48x32_to_50x75", "seeded"):
        assert bk[k].min() > knee, k                            # the goldens never reach the knee


@pytest.mark.parametrize("bg", list(BACKGROUNDS))
@pytest.mark.parametrize("shading", [False, True])
def test_model_equals_oracle_on_nonfinite_dye(oracle, shading, bg):
    """none / SHADING: the model's display shader == oracle.display, NaN in the same places."""
    c = CASES["nonfinite"]
    with np.errstate(invalid="ignore", over="ignore"):
        mine = M.display(c["dye"], c["w"], c["h"], M.SHADING if shading else 0, None, None, None, BACK_RGB,
                         BACKGROUNDS[bg], c["w"] / c["h"])["target"]
    ref = oracle.display(c["dye"], c["w"], c["h"], shading, BACK_RGB, BACKGROUNDS[bg])
    assert np.isnan(ref).any()
    assert G.same_bits(mine, ref)


def test_check_display_and_same_bits():
    lo = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0], F32)
    assert G.check_display(lo.copy(), lo, lo.copy())[0] == 0
    got = lo.copy(); got[4] = 0.0
    assert G.check_display(got, lo, lo.copy())[0] == 1
    with pytest.raises(AssertionError):
        G.check_display(lo, lo, np.zeros_like(lo))
    a = np.array([np.nan, 1.0], F32)
    other_nan = np.array([0x7FFFFFFF, 0x3F800000], np.uint32).view(F32)
    assert G.same_bits(a, other_nan) and not G.same_bits(a, np.array([1.0, 1.0], F32))
    assert not G.same_bits(a, np.array([np.nan, np.nextafter(F32(1), F32(2))], F32))


def test_powf_bounds_special_cases():
    bk = np.array([0.0, 1.0, np.inf, 1e-45, 2.0], F32)
    lo, hi = G.powf_bounds(bk)
    assert list(lo[:3]) == [0.0, 1.0, np.inf] and list(hi[:3]) == [0.0, 1.0, np.inf]
    assert lo[3] > 0 and hi[4] == G.step_ulps(G.pow_rn(bk[4]), G.POWF_ULP) and lo[4] < hi[4]


# ---- the mutants -----------------------------------------------------------------------------------
# Each mutant is the model's arithmetic with one change.  restate() is that arithmetic, value by value;
# the interval must accept the unchanged restatement everywhere and reject each mutant on hundreds of
# texels of at least one input.
MUTANT_INPUTS = ["seeded", "zero", "dim", "wide_dither"]
MUTANT_BACKGROUNDS = [O.BG_COLOR, O.BG_NONE]


def restate(c, r, background, power=None, gamma=M.linear_to_gamma, repeat=True, alpha_before_bloom=False):
    """render() with all three keywords in the model's arithmetic; `power(bk)` defaults to numpy's pow."""
    w, h, dither = c["w"], c["h"], c["dither"]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        col, bl = M.colour_terms(c["dye"], w, h, ALL3, r["bloom"], r["sunrays"])
        bk = M.gamma_argument(bl, dither, w, h, repeat=repeat)
        p = np.power(bk, G.Y) if power is None else power(bk)
        out = col + gamma(p)
        a = M.alpha_of(col if alpha_before_bloom else out)
        return M.over_background(out, a, BACK_RGB, background, w / h)


def rejected(mutant_kwargs):
    """{input: texels rejected, summed over MUTANT_BACKGROUNDS}."""
    out = {}
    for name in MUTANT_INPUTS:
        c = CASES[name]
        r = oracle_frame(O, c, 0)
        n = 0
        for bg in MUTANT_BACKGROUNDS:
            d = M.display(c["dye"], c["w"], c["h"], ALL3, r["bloom"], r["sunrays"], c["dither"], BACK_RGB, bg,
                          c["w"] / c["h"])
            lo, hi = d["lo"], d["hi"]
            good = restate(c, r, bg)
            assert G.check_display(good, lo, hi)[0] == 0, name
            bad = restate(c, r, bg, **mutant_kwargs)
            n += G.check_display(bad, lo, hi)[0]
        out[name] = n
    return out


def pow_ulps_off(k):
    def power(bk):
        p = G.pow_rn(bk)
        return np.where((bk == 0) | (bk == 1) | np.isinf(bk), p, G.step_ulps(p, k))
    return power


def exp2_log2(bk):
    """fp32 exp2f(y * log2f(x)), each correctly rounded: what __powf / -use_fast_math compute, at best."""
    with np.errstate(divide="ignore"):
        t = G.Y * np.log2(bk.astype(np.float64)).astype(F32)
    return np.exp2(t.astype(np.float64)).astype(F32)


MUTANTS = {
    "powf_6_ulp_up": dict(power=pow_ulps_off(G.POWF_ULP + 2)),
    "powf_6_ulp_down": dict(power=pow_ulps_off(-(G.POWF_ULP + 2))),
    "exp2f_of_y_log2f": dict(power=exp2_log2),
    "exponent_one_ulp_up": dict(power=lambda bk: G.pow_rn(bk, np.nextafter(G.Y, F32(1)))),
    "exponent_one_ulp_down": dict(power=lambda bk: G.pow_rn(bk, np.nextafter(G.Y, F32(0)))),
    "knee_clamp_deleted": dict(gamma=lambda p: F32(1.055) * p - F32(0.055)),
    "dither_clamp_to_edge": dict(repeat=False),
    "alpha_before_bloom": dict(alpha_before_bloom=True),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutant_is_rejected(mutant):
    n = rejected(MUTANTS[mutant])
    assert max(n.values()) >= 300, n


def test_mutant_dither_scale_of_the_canvas_in_capture_is_rejected(oracle):
    """captureScreenshot: getTextureScale of the 128 x 128 canvas instead of the 64 x 64 target."""
    g = golden("capture_64_canvas_128_back")
    dye, dither = g["in_dye"], g["dither"].astype(F32)
    cfg = dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]))
    w, h, cw, ch = int(g["w"]), int(g["h"]), int(g["canvas_w"]), int(g["canvas_h"])
    assert (w, cw) == (64, 128)
    n = 0
    for transparent in (False, True):
        good = M.capture(dye, w, h, cw, ch, dither, ALL3, transparent, BACK_RGB, cfg=cfg)
        assert G.bytes_outside(good["rgba8"], good["lo"], good["hi"]) == 0
        bad = M.capture(dye, w, h, cw, ch, dither, ALL3, transparent, BACK_RGB, cfg=cfg,
                        scale=M.dither_scale(cw, ch, dither))["rgba8"]
        n += G.bytes_outside(bad, good["lo"], good["hi"])
    assert n >= 300, n


def test_deleting_the_bk_clamp_is_equivalent_except_at_minus_inf(oracle):
    """Without fmaxf(bk, 0) the frame is the same bits on every input but the one whose dithering overflows
    to -inf; there the texels where bk = -inf draw powf(-inf, y) = +inf."""
    def unclamped(c, r, bg):
        with np.errstate(invalid="ignore", over="ignore"):
            col, bl = M.colour_terms(c["dye"], c["w"], c["h"], ALL3, r["bloom"], r["sunrays"])
            out = col + M.linear_to_gamma(np.power(unclamped_argument(c, bl), G.Y))
            return M.over_background(out, M.alpha_of(out), BACK_RGB, bg, c["w"] / c["h"])
    for name, c in CASES.items():
        r = oracle_frame(oracle, c, 0)
        for bg in BACKGROUNDS.values():
            same = G.same_bits(unclamped(c, r, bg), restate(c, r, bg))
            assert same == (name != "overflow_dither"), (name, bg)
