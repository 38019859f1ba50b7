"""The storage of FLUID_FLAG_HALF_POSTFX on the CPU: display_model's chains with half-float
targets (and, for a half-storage handle, a half-float sunrays mask) against the executed reference shaders
with half-float textures (keywords_half_*.npz, capture_half_*.npz from tests/golden/make_golden_half_postfx.py),
and the frame tolerance the GPU tests use against those fixtures."""
import numpy as np
import pytest

import display_model as M
import gamma_model as G
from conftest import golden, max_rel
from gamma_model import CAPTURE_SETS, FRAME_TOL, POW2, RAGGED, RAGGED_CHAIN_TEXELS, cfg_of, fp16_ulps

F32 = np.float32
BACK_RGB = (10 / 255, 20 / 255, 30 / 255)
KEYWORDS = {"bloom": M.BLOOM, "sunrays": M.SUNRAYS, "bloom_sunrays": M.BLOOM | M.SUNRAYS,
            "shading_bloom": M.SHADING | M.BLOOM, "shading_sunrays": M.SHADING | M.SUNRAYS}
def half_chains(g, half_mask=True):
    w, h = int(g["w"]), int(g["h"])
    return M.chains(g["in_dye"], w, h, M.BLOOM | M.SUNRAYS, cfg_of(g), half_targets=True, half_mask=half_mask)


@pytest.mark.parametrize("name", [POW2, RAGGED])
def test_fixture_holds_fp16_chains(name):
    """The executed chains really are fp16 values, and so is the dye they read."""
    g = golden(name)
    for k in ["in_dye", "bloom", "sunrays", "mask_alpha"] + [f for f in g.files if f.startswith("pyr")]:
        assert np.array_equal(g[k].astype(np.float16).astype(F32), g[k]), k
    assert sorted(str(t) for t in g["sets"]) == sorted(KEYWORDS)


def test_power_of_two_chains_equal_executed_shaders(oracle):
    g = golden(POW2)
    r = half_chains(g)
    assert G.same_bits(r["bloom"], g["bloom"])
    assert G.same_bits(r["sunrays"], g["sunrays"])
    assert G.same_bits(r["mask_alpha"], g["mask_alpha"])
    assert len(r["pyramid"]) == 5
    for k, t in enumerate(r["pyramid"]):
        assert G.same_bits(t, g[f"pyr{k}"]), k


def test_ragged_chains_within_measured_bound(oracle):
    g = golden(RAGGED)
    r = half_chains(g)
    for k, t in enumerate(r["pyramid"]):
        assert G.same_bits(t, g[f"pyr{k}"]), k
    for k, n in RAGGED_CHAIN_TEXELS.items():
        assert np.count_nonzero(r[k] != g[k]) <= n, k
        assert fp16_ulps(r[k], g[k]) <= 1, k


@pytest.mark.parametrize("name", [POW2, RAGGED])
def test_frames_within_frame_tolerance(oracle, name):
    """The model's frames with the half-float chains against the executed frames: bit for bit on the
    power-of-two fixture, within FRAME_TOL on the ragged one; and further from them with fp32 chains."""
    g = golden(name)
    w, h = int(g["w"]), int(g["h"])
    worst = 0.0
    for tag in (str(t) for t in g["sets"]):
        kw = KEYWORDS[tag]
        ref = M.render(g["in_dye"], w, h, g["dither"].astype(F32), kw, cfg_of(g), back_rgb=BACK_RGB, half_targets=True,
                       half_mask=True)
        if name == POW2:
            assert G.same_bits(ref["target"], g[f"{tag}_target"]), tag
        worst = max(worst, max_rel(ref["target"], g[f"{tag}_target"]))
    assert worst < FRAME_TOL, worst
    if name == RAGGED:
        assert worst > 1e-4, worst            # the bound above is measured, not loose


def test_fp32_chains_are_not_the_half_float_frame(oracle):
    """Without half-float targets the model misses the executed half-float frame by more than FRAME_TOL on
    some set: the flag is needed to draw the reference's frame."""
    g = golden(POW2)
    w, h = int(g["w"]), int(g["h"])
    worst = max(max_rel(M.render(g["in_dye"], w, h, g["dither"].astype(F32), KEYWORDS[str(t)], cfg_of(g),
                                 back_rgb=BACK_RGB)["target"], g[f"{t}_target"]) for t in g["sets"])
    assert worst > FRAME_TOL, worst


def test_defaults_are_the_oracle(oracle):
    """The model without half-float storage is oracle.render_postfx: chains bit for bit, the oracle's frame (glibc
    powf) inside the model's powf interval at every value."""
    g = golden(POW2)
    w, h = int(g["w"]), int(g["h"])
    a = M.render(g["in_dye"], w, h, g["dither"].astype(F32), M.ALL3, cfg_of(g), back_rgb=BACK_RGB)
    b = oracle.render_postfx(g["in_dye"], w, h, g["dither"].astype(F32), cfg=cfg_of(g), back_rgb=BACK_RGB)
    for k in ("bloom", "sunrays", "mask_alpha"):
        assert G.same_bits(a[k], b[k]), k
    assert len(a["pyramid"]) == len(b["pyramid"]) and all(G.same_bits(x, y) for x, y in zip(a["pyramid"], b["pyramid"]))
    assert G.check_display(b["target"], a["lo"], a["hi"])[0] == 0


@pytest.mark.parametrize("bg", ["back", "transparent"])
def test_captures_equal_executed_shaders(oracle, bg):
    """display_model.capture with half-float chains gives the executed capture's bytes exactly, all eight sets."""
    g = golden(f"capture_half_64_canvas_128_{bg}")
    cfg = cfg_of(g)
    for kw, tag in enumerate(CAPTURE_SETS):
        c = M.capture(g["in_dye"], int(g["w"]), int(g["h"]), int(g["canvas_w"]), int(g["canvas_h"]),
                      g["dither"].astype(F32), kw, bool(g["transparent"]), BACK_RGB, cfg=cfg, half_targets=True,
                      half_mask=True)
        assert np.array_equal(c["rgba8"], g[f"{tag}_rgba8"]), tag


def test_overflow_rounds_to_inf(oracle):
    """Dye bright enough that the prefiltered bloom exceeds 65504: the fp16 bloom FBO holds +inf there and
    finite values elsewhere (the input of the GPU overflow test)."""
    dye = np.full((64, 64, 4), 0.5, F32); dye[..., 3] = 1
    dye[20:24, 30:34, 0] = 2.0e5
    cfg = dict(BLOOM_RESOLUTION=64, SUNRAYS_RESOLUTION=48)
    with np.errstate(invalid="ignore", over="ignore"):
        r = M.chains(dye, 128, 128, M.BLOOM, cfg, half_targets=True)
        r32 = M.chains(dye, 128, 128, M.BLOOM, cfg)
    assert np.isposinf(r["bloom"][..., 0]).any() and np.isfinite(r["bloom"][..., 1:3]).all()
    assert np.isfinite(r32["bloom"]).all() and r32["bloom"].max() > 65504
