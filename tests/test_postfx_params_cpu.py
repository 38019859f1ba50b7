"""The four post-FX sliders -- BLOOM_INTENSITY, BLOOM_THRESHOLD, BLOOM_SOFT_KNEE, SUNRAYS_WEIGHT (S:79-84, the
settings panel S:227-232) -- away from their defaults, on the CPU.  The parameter sets and the dye that
tests/test_gpu_postfx_params.py draws with them live in tests/display_harness.py; this file shows that they
are strong enough to catch a wrong kernel:

* branches: for every set, the bloom prefilter (bloomPrefilterShader S:614-631) sees enough texels below
  curve.x, inside the knee and above it, with rq winning and losing max(rq, br - threshold), and with br
  under the max(br, 0.0001) guard as zeros, fp32 subnormals and negatives;
* mutants: each one-change variant of the chain model below -- one slider replaced by its default, threshold
  and knee swapped, knee / curve derived in fp32 instead of in JS doubles, the intensity applied on the
  additive up-pass instead of the final blit -- changes the expected bloom FBO or sunrays bits and the
  expected frame of at least one set, and all but the fp32 curve (a few ulp of bloom) its capture and canvas
  bytes too;
* the oracle against the executed reference shaders with these sliders (postfx_params_*.npz, cut by
  tests/golden/make_golden_postfx_params.py): bloom FBO and sunrays bit for bit, the frame at the tolerance
  of the power-of-two post-FX goldens."""
import numpy as np
import pytest

import canvas_model as CV
import capture_model as CM
import display_model as M
import gamma_model as G
from conftest import golden, max_rel
from display_harness import (BACK_RGB, DEFAULTS, FIXTURES, GEOMETRIES, KEYS, SETS, cfg_of, fixture_cfg, golden_dither,
                             params_dye)
from oracle import oracle as O

F32 = np.float32
ALL3 = M.ALL3
MIN_TEXELS = 8                               # bloom texels each branch must get, per set and geometry


# ---- the chain model, with its mutants -------------------------------------------------------------------
MUTANTS = [f"default_{k}" for k in KEYS] + ["threshold_knee_swapped", "curve_in_fp32", "intensity_on_up_pass"]


def chains(dye, w, h, cfg, mutant=None, half_targets=False, half_mask=False):
    """The bloom and sunrays chains of render() on a w x h canvas (display_model.chains, the fp16 stores with
    `half_targets` / `half_mask`), with one change when `mutant` names one of MUTANTS."""
    assert mutant is None or mutant in MUTANTS, mutant
    c = dict(cfg)
    if mutant and mutant.startswith("default_"):
        c[mutant[len("default_"):]] = DEFAULTS[mutant[len("default_"):]]
    if mutant == "threshold_knee_swapped":
        c["BLOOM_THRESHOLD"], c["BLOOM_SOFT_KNEE"] = c["BLOOM_SOFT_KNEE"], c["BLOOM_THRESHOLD"]
    return M.chains(dye, w, h, M.BLOOM | M.SUNRAYS, c, half_targets=half_targets, half_mask=half_mask,
                    fp32_curve=mutant == "curve_in_fp32", intensity_on_up_pass=mutant == "intensity_on_up_pass")


def outputs(dye, geometry, name, mutant=None, kw=ALL3):
    """What the fp32 handle is checked on, from the chains: the frame over BACK_COLOR, the capture bytes and the
    canvas bytes over BACK_COLOR and over the checkerboard."""
    Wd, Hd, w, h = GEOMETRIES[geometry][:4]
    cfg = cfg_of(name, geometry)
    dither = golden_dither()
    with np.errstate(invalid="ignore", over="ignore"):
        r = chains(dye, w, h, cfg, mutant)
        frame = M.display(dye, w, h, kw, r["bloom"], r["sunrays"], dither, BACK_RGB, O.BG_COLOR, w / h)["target"]
        bare = M.display(dye, w, h, kw, r["bloom"], r["sunrays"], dither, BACK_RGB, O.BG_NONE, w / h)["target"]
        cw_, ch_ = M.get_resolution(cfg["CAPTURE_RESOLUTION"], w, h)
        pre = M.display(dye, cw_, ch_, kw, r["bloom"], r["sunrays"], dither, CM.back16(BACK_RGB), O.BG_COLOR,
                        cw_ / ch_)["target"]
        canvas = [CV.canvas(bare, BACK_RGB, t, w / h) for t in (False, True)]
    return dict(r, frame=frame, capture=CM.to_bytes(pre)[::-1], canvas=canvas)


# ---- the prefilter's branches ----------------------------------------------------------------------------
def fetched(dye, geometry, nearest=False):
    """The dye colour the prefilter fetches at every bloom texel (LINEAR or NEAREST, the library's vUv)."""
    Wd, Hd, w, h, bres = GEOMETRIES[geometry][:5]
    bw, bh = M.get_resolution(bres, w, h)
    return M.fetch(dye, *M.uv_grid(bw, bh), nearest)[..., :3].astype(F32)


def branches(c, threshold, soft_knee):
    """{branch: number of texels} of the prefilter on fetched colours c, in its fp32 arithmetic."""
    c0, c1, c2, th = M.curve(threshold, soft_knee)
    br = np.fmax(c[..., 0], np.fmax(c[..., 1], c[..., 2]))
    x = br - c0
    rq = np.fmin(np.fmax(x, F32(0)), c1)
    rq = (c2 * rq) * rq
    tiny = F32(np.finfo(F32).tiny)
    return dict(below_curve0=int(np.count_nonzero(x < 0)), in_knee=int(np.count_nonzero((x > 0) & (x < c1))),
                above_knee=int(np.count_nonzero(x > c1)), rq_wins=int(np.count_nonzero(rq > br - th)),
                rq_loses=int(np.count_nonzero(rq < br - th)), zero=int(np.count_nonzero(br == 0)),
                subnormal=int(np.count_nonzero((br > 0) & (br < tiny))), negative=int(np.count_nonzero(br < 0)),
                small=int(np.count_nonzero((br >= tiny) & (br < F32(0.0001)))))


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("nearest", [False, True])
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_every_set_reaches_every_prefilter_branch(geometry, nearest, half):
    """Every branch on at least MIN_TEXELS bloom texels of every set but `above`, whose br all lie below curve.x
    (its prefilter draws zeros, and so its bloom FBO is zero).  A half-storage dye has no fp32 subnormal left."""
    dye = params_dye(*GEOMETRIES[geometry][:2])
    if half:
        dye = O.round_half(dye)
    c = fetched(dye, geometry, nearest)
    for name, (_, T, K, _) in SETS.items():
        n = branches(c, T, K)
        if name == "above":
            assert n["below_curve0"] == c.shape[0] * c.shape[1], n
            continue
        for b, k in n.items():
            if b == "subnormal" and half:
                assert k == 0
            else:
                assert k >= MIN_TEXELS, (name, b, n)


def test_sets_cover_the_slider_values():
    I, T, K, W = (set(v[k] for v in SETS.values()) for k in range(4))
    assert {0.0, 0.05, 0.6, 1.0} <= T and max(T) > params_dye(64, 64)[..., :3].max() + max(T) * 0.2 + 1e-4
    assert {0.0, 1.0} <= K and {0.0, 0.1, 2.0} <= I and max(I) > 3000 and {0.0, 0.3} <= W and max(W) > 1
    differ = [n for n, (_, t, k, _) in SETS.items() if 0 < t <= 1 and 0 < k <= 1
              and not np.array_equal(np.array(M.curve(t, k), F32), np.array(M.curve(t, k, fp32=True), F32))]
    assert len(differ) >= 2, differ


def test_above_and_overflow_sets_do_what_they_are_for(oracle):
    """`above`: a zero bloom FBO.  `overflow`: +inf in the fp16 bloom FBO (not everywhere), finite in fp32."""
    Wd, Hd, w, h = GEOMETRIES["pow2"][:4]
    dye = params_dye(Wd, Hd)
    assert not chains(dye, w, h, cfg_of("above"))["bloom"][..., :3].any()
    with np.errstate(over="ignore"):
        half = chains(dye, w, h, cfg_of("overflow"), half_targets=True)["bloom"][..., :3]
    assert 0 < np.count_nonzero(np.isposinf(half)) < half.size
    assert np.isfinite(chains(dye, w, h, cfg_of("overflow"))["bloom"]).all()


@pytest.mark.parametrize("half", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_chain_model_is_the_models_chains(oracle, geometry, half):
    """Unmutated, chains() is display_model.render's chains bit for bit.  With fp32 targets those are
    oracle.render_postfx's bit for bit (bloom FBO, pyramid, sunrays, mask), and the oracle's frame lies inside
    the model's powf interval."""
    Wd, Hd, w, h = GEOMETRIES[geometry][:4]
    dye = params_dye(Wd, Hd)
    bits = lambda a, b: np.array_equal(a.view(np.uint32), b.view(np.uint32))          # noqa: E731
    for name in SETS:
        cfg = cfg_of(name, geometry)
        with np.errstate(over="ignore", invalid="ignore"):
            mine = chains(dye, w, h, cfg, half_targets=half[0], half_mask=half[1])
            ref = M.render(dye, w, h, golden_dither(), ALL3, cfg, back_rgb=BACK_RGB, half_targets=half[0],
                           half_mask=half[1])
        for k in ("bloom", "sunrays"):
            assert bits(mine[k], ref[k]), (name, k)
        if half[0]:
            continue
        o = O.render_postfx(dye, w, h, golden_dither(), cfg=cfg, back_rgb=BACK_RGB)
        for k in ("bloom", "sunrays", "mask_alpha"):
            assert bits(ref[k], o[k]), (name, k)
        assert len(ref["pyramid"]) == len(o["pyramid"]) and all(map(bits, ref["pyramid"], o["pyramid"])), name
        assert G.check_display(o["target"], ref["lo"], ref["hi"])[0] == 0, name


# Mutants whose change stays below one byte of every capture and canvas: curve_in_fp32 moves a curve
# component by an ulp, and so the bloom FBO by a few ulp.  The bloom FBO's bits and the frame catch it.
SUB_BYTE = {"curve_in_fp32"}


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutant_changes_the_expected_bits(oracle, mutant):
    """Each mutant changes the bloom FBO or the sunrays texture of at least one set, and the frame of at least
    one set; all but SUB_BYTE change the capture bytes and the canvas bytes of at least one set too."""
    hits = dict(chain=[], frame=[], capture=[], canvas=[])
    for geometry in GEOMETRIES:
        dye = params_dye(*GEOMETRIES[geometry][:2])
        for name in SETS:
            good, bad = outputs(dye, geometry, name), outputs(dye, geometry, name, mutant)
            same = lambda a, b: np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))  # noqa: E731
            if not (same(good["bloom"], bad["bloom"]) and same(good["sunrays"], bad["sunrays"])):
                hits["chain"].append((geometry, name))
            if not same(good["frame"], bad["frame"]):
                hits["frame"].append((geometry, name))
            if not same(good["capture"], bad["capture"]):
                hits["capture"].append((geometry, name))
            if not all(same(a, b) for a, b in zip(good["canvas"], bad["canvas"])):
                hits["canvas"].append((geometry, name))
    want = ("chain", "frame") if mutant in SUB_BYTE else tuple(hits)
    assert all(hits[k] for k in want), (mutant, hits)


# ---- the oracle against the executed shaders ------------------------------------------------------------
@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_executed_shaders(oracle, name):
    """Bloom FBO and sunrays bit for bit, the frame within the power-of-two post-FX goldens' 2e-6
    (test_oracle_golden.py: pow() is implementation-defined).  The fixture's sliders and dye are the set's."""
    g = golden(name)
    assert tuple(fixture_cfg(g)[k] for k in KEYS) == SETS[str(g["set"])]
    assert np.array_equal(g["in_dye"].view(np.uint32), params_dye(int(g["Wd"]), int(g["Hd"])).view(np.uint32))
    r = oracle.render_postfx(g["in_dye"], int(g["w"]), int(g["h"]), g["dither"].astype(F32), cfg=fixture_cfg(g),
                             back_rgb=tuple(float(x) / 255 for x in g["back"]))
    for k in ("bloom", "sunrays"):
        assert np.array_equal(r[k].view(np.uint32), g[k].view(np.uint32)), k
    assert max_rel(r["target"], g["target"]) < 2e-6


def test_fixtures_tell_the_fp32_curve_from_the_double_one(oracle):
    """On t033_k07's fixture the curve derived in fp32 gives another bloom FBO than the executed shaders'."""
    g = golden(FIXTURES[0])
    bad = chains(g["in_dye"], int(g["w"]), int(g["h"]), fixture_cfg(g), mutant="curve_in_fp32")["bloom"]
    assert not np.array_equal(bad.view(np.uint32), g["bloom"].view(np.uint32))
