"""The display keyword sets of render() (updateKeywords, S:1160-1166) on the CPU: the display model
(display_model.py, over the oracle's chains) against the executed reference shaders for the five sets
that are neither none / SHADING (test_oracle_golden's display tests) nor all three (its postfx tests),
and the host-side mapping from `config` to the keyword mask.  Runs without a GPU."""
import numpy as np
import pytest

import display_model as M
import webgl_fluid_simulation_b200 as pkg
from conftest import bits_equal, golden, max_rel

KEYWORDS = {"bloom": pkg.DISPLAY_BLOOM, "sunrays": pkg.DISPLAY_SUNRAYS,
            "bloom_sunrays": pkg.DISPLAY_BLOOM | pkg.DISPLAY_SUNRAYS,
            "shading_bloom": pkg.DISPLAY_SHADING | pkg.DISPLAY_BLOOM,
            "shading_sunrays": pkg.DISPLAY_SHADING | pkg.DISPLAY_SUNRAYS}


def _render(O, g, keywords, background=0):
    return M.render(g["in_dye"], int(g["w"]), int(g["h"]), g["dither"].astype(np.float32), keywords,
                    cfg=dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"])),
                    back_rgb=tuple(float(x) / 255 for x in g["back"]), background=background)


def _check_chains(r, g, keywords, pow2):
    """bloom FBO + pyramid and sunrays mask: bitwise on the power-of-two geometry (the sunrays FBO is
    48 wide there, so its texture is not); 3e-4 on the ragged one, as test_oracle_golden."""
    tol = 3e-4
    n = len([k for k in g.files if k.startswith("pyr")])
    if keywords & pkg.DISPLAY_BLOOM:
        assert len(r["pyramid"]) == n
        if pow2:
            assert bits_equal(r["bloom"], g["bloom"])
            assert all(bits_equal(r["pyramid"][k], g[f"pyr{k}"]) for k in range(n))
        else:
            assert max_rel(r["bloom"], g["bloom"]) < tol
    else:
        assert r["bloom"] is None and r["pyramid"] == []
    if keywords & pkg.DISPLAY_SUNRAYS:
        if pow2:
            assert bits_equal(r["mask_alpha"], g["mask_alpha"]) and max_rel(r["sunrays"], g["sunrays"]) < 2e-6
        else:
            assert max_rel(r["mask_alpha"], g["mask_alpha"]) < tol and max_rel(r["sunrays"], g["sunrays"]) < tol
    else:
        assert r["sunrays"] is None and r["mask_alpha"] is None


@pytest.mark.parametrize("tag", list(KEYWORDS))
@pytest.mark.parametrize("pow2", [True, False])
def test_keyword_sets_match_executed_reference_shaders(oracle, pow2, tag):
    """Each keyword set over BACK_COLOR.  Power-of-two geometry: bloom chain and mask bitwise; the frame
    within 2e-6 and not bitwise for any of the five sets (measured 1.2e-7 .. 2.0e-7): BLOOM goes through
    pow(), which numpy and glibc round differently, and SUNRAYS through the 48-wide sunrays texture.
    Ragged geometry: 3e-4 (vUv rounding amplified by br * 20 in the mask)."""
    g = golden(f"keywords_{tag}_64_to_128" if pow2 else "keywords_48x32_to_50x75")
    assert tag in [str(s) for s in g["sets"]]
    r = _render(oracle, g, KEYWORDS[tag])
    _check_chains(r, g, KEYWORDS[tag], pow2)
    assert max_rel(r["target"], g[f"{tag}_target"]) < (2e-6 if pow2 else 3e-4)


def test_keyword_set_transparent_matches_executed_reference_shaders(oracle):
    """config.TRANSPARENT with BLOOM + SUNRAYS: over the checkerboard on the screen and bare into a
    capture target (S:1303-1312), within 2e-6 of the executed shaders."""
    g = golden("keywords_transparent_64x32_to_128x64")
    kw = KEYWORDS["bloom_sunrays"]
    for key, bg in (("checker", oracle.BG_CHECKERBOARD), ("bare", oracle.BG_NONE)):
        r = _render(oracle, g, kw, bg)
        _check_chains(r, g, kw, True)
        assert max_rel(r["target"], g[f"bloom_sunrays_{key}"]) < 2e-6, key


@pytest.mark.parametrize("keywords", range(8))
def test_keyword_model_restates_the_oracle_display(oracle, keywords):
    """The model's numpy display shader against the oracle's C one where the oracle has it: without
    BLOOM and SUNRAYS bit for bit vs oracle.display, and with all three within pow()'s last places of
    oracle.render_postfx (numpy's and glibc's powf round differently).  This pins the restatement the model draws every set
    with."""
    g = golden("keywords_48x32_to_50x75")
    w, h = int(g["w"]), int(g["h"])
    full = oracle.render_postfx(g["in_dye"], w, h, g["dither"].astype(np.float32),
                                cfg=dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"])))
    for bg in (oracle.BG_COLOR, oracle.BG_CHECKERBOARD, oracle.BG_NONE):
        mine = M.display(g["in_dye"], w, h, keywords, full["bloom"], full["sunrays"], g["dither"].astype(np.float32),
                         tuple(float(x) / 255 for x in g["back"]), bg, w / h)["target"]
        if not keywords & (pkg.DISPLAY_BLOOM | pkg.DISPLAY_SUNRAYS):
            ref = oracle.display(g["in_dye"], w, h, bool(keywords & pkg.DISPLAY_SHADING),
                                 tuple(float(x) / 255 for x in g["back"]), bg)
            assert bits_equal(mine, ref), bg
        if keywords == 7:
            ref = oracle.render_postfx(g["in_dye"], w, h, g["dither"].astype(np.float32),
                                       cfg=dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"])),
                                       back_rgb=tuple(float(x) / 255 for x in g["back"]), background=bg)
            assert max_rel(mine, ref["target"]) < 1e-6, bg


@pytest.mark.parametrize("shading", [False, True])
@pytest.mark.parametrize("bloom", [False, True])
@pytest.mark.parametrize("sunrays", [False, True])
def test_config_to_keyword_mask_like_update_keywords(shading, bloom, sunrays):
    cfg = dict(pkg.default_config(), SHADING=shading, BLOOM=bloom, SUNRAYS=sunrays)
    want = (pkg.DISPLAY_SHADING if shading else 0) | (pkg.DISPLAY_BLOOM if bloom else 0) | (pkg.DISPLAY_SUNRAYS if sunrays else 0)
    assert pkg.display_keywords(cfg) == want
    dither = np.zeros((64, 64, 3), np.float32)
    kw, fx, dith = pkg.postfx_inputs(cfg, dither)
    assert kw == want
    assert (fx is None) == (not bloom and not sunrays)
    assert (dith is None) == (not bloom)
    if bloom:
        with pytest.raises(ValueError, match="dithering"):
            pkg.postfx_inputs(cfg, None)
        with pytest.raises(ValueError, match="dithering"):
            pkg.postfx_inputs(cfg, np.zeros((64, 64), np.float32))
    else:                                                       # no dithering texture needed
        kw, fx, dith = pkg.postfx_inputs(cfg, None)
        assert kw == want and dith is None and (fx is None) == (not sunrays)


def test_default_config_keeps_bloom_and_sunrays_off():
    c = pkg.default_config()
    assert c["BLOOM"] is False and c["SUNRAYS"] is False and c["SHADING"] is True
    assert pkg.display_keywords(c) == pkg.DISPLAY_SHADING
