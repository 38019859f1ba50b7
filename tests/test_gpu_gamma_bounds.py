"""render() and captureScreenshot() with BLOOM on the GPU against the per-texel interval of
display_model.display (tests/gamma_model.py): every value of the frame and every byte of the capture must lie within the fp32
arithmetic of the display shader with a powf inside POWF_ULP of float64 pow.  The interval of a frame is
built from the model's bloom FBO and sunrays texture (the oracle's blits), after checking the GPU's against
them bit for bit (NaN in the same places).

Inputs are display_harness.CASES, those of test_gamma_model_cpu.py (goldens, seeded, zero and dim dye, dithering of other
shapes, of a wide range and overflowing, non-finite dye) plus one frame at the reference's sizes; the
non-finite dye goes through all eight keyword sets, on fp32 and half-storage handles.  A readout of the
device powf itself closes the file."""
import numpy as np
import pytest

import display_harness as DH
import display_model as M
import gamma_model as G
from conftest import golden
from display_harness import BACK_RGB, BACKGROUNDS, MODES, golden_dither, make, nonfinite_dye, seeded_dye, set_keywords
from display_harness import CASES, DIM_CFG, FXCFG
from display_model import ALL3
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu
F32 = np.float32
BLOOM_SETS = [M.BLOOM, M.SHADING | M.BLOOM, M.BLOOM | M.SUNRAYS, ALL3]
NO_BLOOM_SETS = [0, M.SHADING, M.SUNRAYS, M.SHADING | M.SUNRAYS]
HALF = 0x10


def draw_and_check(pkg, c, sets=BLOOM_SETS):
    """Each keyword set with BLOOM x background: the chains equal the model's (the oracle's blits), the frame lies
    within the interval of display_model."""
    DH.draw_all(pkg, "fp32", c["dye"], c["w"], c["h"], c["dither"], cfg=c["cfg"], sets=sets)


@pytest.mark.parametrize("name", list(CASES))
def test_frames_within_interval(pkg, oracle, name):
    draw_and_check(pkg, CASES[name])


def test_reference_size_frame_within_interval(pkg, oracle):
    """A 1024^2 dye drawn to 1920 x 1080 with BLOOM_RESOLUTION 256 and SUNRAYS_RESOLUTION 196, all three
    keywords."""
    c = dict(dye=seeded_dye(1024, 1024, 1920), w=1920, h=1080, dither=golden_dither(),
             cfg=dict(BLOOM_RESOLUTION=256, SUNRAYS_RESOLUTION=196))
    draw_and_check(pkg, c, sets=[ALL3])


def capture_inputs():
    """name -> (dye, target w, h, canvas w, h, CAPTURE_RESOLUTION, dither, post-FX keys, transparent)."""
    out = {}
    for geometry in ("capture_64_canvas_128", "capture_48x32_canvas_807x640"):
        for bg in ("back", "transparent"):
            g = golden(f"{geometry}_{bg}")
            out[f"{geometry}_{bg}"] = (g["in_dye"], int(g["w"]), int(g["h"]), int(g["canvas_w"]), int(g["canvas_h"]),
                                       int(g["capture_res"]), g["dither"].astype(F32),
                                       dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"])),
                                       bool(g["transparent"]))
    for transparent in (False, True):
        t = "_transparent" if transparent else ""
        out["dim" + t] = (seeded_dye(64, 64, 192, scale=1.0) * F32(0.25), 64, 64, 128, 128, 64, golden_dither(), DIM_CFG,
                          transparent)
        out["nonfinite" + t] = (nonfinite_dye(64, 64, 8), 64, 64, 128, 128, 64, golden_dither(), FXCFG, transparent)
    return out


CAPTURES = capture_inputs()


@pytest.mark.parametrize("name", list(CAPTURES))
def test_captures_within_interval(pkg, name):
    """All eight sets: with BLOOM every byte within [B(lo), B(hi)]; without it the capture model's bytes
    exactly."""
    dye, w, h, cw, ch, res, dither, cfg, transparent = CAPTURES[name]
    s = make(pkg, dye.shape[1], dye.shape[0], cw, ch, CAPTURE_RESOLUTION=res, TRANSPARENT=transparent, **cfg)
    s.writeField("dye", dye)
    s.dithering = dither
    with np.errstate(invalid="ignore", over="ignore"):
        for kw in range(8):
            set_keywords(s, kw)
            got = s.captureScreenshot()
            assert got.shape == (h, w, 4)
            DH.check_capture(got, DH.model_capture("fp32", dye, w, h, cw, ch, kw, dither, cfg, transparent), kw, (name, kw))
    s.close()


def test_nonfinite_frames_without_bloom(pkg, oracle):
    """none, SHADING, SUNRAYS, SHADING + SUNRAYS on the non-finite dye, every background: the frame equals
    oracle.display / the display model bit for bit (NaN in the same places), the sunrays texture the
    oracle's."""
    c = CASES["nonfinite"]
    dye, w, h = c["dye"], c["w"], c["h"]
    s = make(pkg, dye.shape[1], dye.shape[0], w, h, **c["cfg"])
    s.writeField("dye", dye)
    with np.errstate(invalid="ignore", over="ignore"):
        for kw in NO_BLOOM_SETS:
            set_keywords(s, kw)
            for bg, (transparent, target) in MODES.items():
                s.config["TRANSPARENT"] = transparent
                got = s.render(w, h, target=target)
                ref = DH.model_frame("fp32", dye, w, h, kw, None, c["cfg"], BACKGROUNDS[bg])
                assert np.isnan(ref["target"]).any()
                assert G.same_bits(got, ref["target"]), (kw, bg)
                if kw & M.SUNRAYS:
                    assert G.same_bits(s.last_sunrays, ref["sunrays"]), (kw, bg)
    s.close()


def test_nonfinite_half_storage(pkg, oracle):
    """A half-storage handle holds the non-finite dye in fp16 (1e30 overflows to inf, the subnormal
    flushes to 0): none and SHADING frames and captures equal the oracle / capture model of that fp16 dye."""
    c = CASES["nonfinite"]
    w, h = c["w"], c["h"]
    dye16 = oracle.round_half(c["dye"])
    s = make(pkg, 64, 64, w, h, flags=HALF, CAPTURE_RESOLUTION=64)
    s.writeField("dye", c["dye"])
    assert G.same_bits(s.readField("dye"), dye16)
    assert np.count_nonzero(np.isinf(dye16)) > np.count_nonzero(np.isinf(c["dye"]))
    with np.errstate(invalid="ignore", over="ignore"):
        for kw in (0, M.SHADING):
            set_keywords(s, kw)
            for bg, (transparent, target) in MODES.items():
                s.config["TRANSPARENT"] = transparent
                ref = oracle.display(dye16, w, h, bool(kw), BACK_RGB, BACKGROUNDS[bg])
                assert G.same_bits(s.render(w, h, target=target), ref), (kw, bg)
            for transparent in (False, True):
                s.config["TRANSPARENT"] = transparent
                want = DH.model_capture("half", dye16, 64, 64, w, h, kw, None, None, transparent)["rgba8"]
                assert np.array_equal(s.captureScreenshot(), want), (kw, transparent)
    s.close()


RANGES = [(-14, -10), (-10, 0), (0, 10), (10, 40), (40, 80), (80, 120)]


def test_direct_powf_readout(pkg, capsys):
    """Zero dye, BLOOM only, bare: the bloom FBO is exactly zero, so each channel of the frame is
    fmaxf(1.055 powf(bk) - 0.055, 0) with bk = fmaxf((2d - 1) / 255, 0) from the dithering value d, read at
    its texel centre (dithering texture the size of the target).  For every texel, the smallest k such that
    some p within k ulp of pow(bk, y) rounded to fp32 gives the observed value: at most POWF_ULP.  The
    largest k is printed per binade range of bk; texels below the knee (value 0 whatever p) are counted
    apart."""
    W = H = 512
    rng = np.random.default_rng(2024)
    e = rng.uniform(-14, 120, (H, W))
    d = ((np.exp2(e) * 255 + 1) / 2).astype(F32)
    dither = np.repeat(d[..., None], 3, axis=-1)
    s = make(pkg, 64, 64, W, H, TRANSPARENT=True, BLOOM_RESOLUTION=256, SUNRAYS_RESOLUTION=196)
    s.writeField("dye", np.zeros((64, 64, 4), F32))
    s.dithering = dither
    set_keywords(s, M.BLOOM)
    got = s.render(W, H, target=True)
    assert np.all(s.last_bloom[..., :3] == 0)
    s.close()
    assert np.array_equal(got[..., 0], got[..., 1]) and np.array_equal(got[..., 0], got[..., 2])
    g = got[..., 0]
    bk = M.gamma_argument(np.zeros((H, W, 3), F32), dither, W, H)[..., 0]
    assert bk.min() < 2.0 ** -10 and bk.max() > 2.0 ** 119
    p = G.pow_rn(bk)
    dist = np.full(bk.shape, 99)
    for k in range(9):
        for sign in (1, -1):
            hit = (M.linear_to_gamma(G.step_ulps(p, sign * k)) == g) & (dist == 99)
            dist[hit] = k
    flat = (g == 0) & (M.linear_to_gamma(G.step_ulps(p, 8)) == 0)         # below the knee: no information
    lb = np.log2(bk.astype(np.float64))
    lines = []
    for a, b in RANGES:
        m = (lb >= a) & (lb < b)
        info = m & ~flat
        worst = int(dist[info].max()) if info.any() else None
        lines.append(f"2^{a}..2^{b}: max {worst} ulp over {int(info.sum())} texels"
                     + (f", {int((m & flat).sum())} below the knee" if (m & flat).any() else ""))
        assert b <= -10 or info.sum() > 1000, (a, b)
    with capsys.disabled():
        print("\n[powf] smallest ulp distance from pow(float64(bk), y) rounded to fp32 that explains the frame, "
              "by the range of bk: " + "; ".join(lines))
    assert dist[~flat].max() <= G.POWF_ULP, int(dist[~flat].max())
