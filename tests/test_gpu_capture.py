"""captureScreenshot() (S:287-327) on the GPU: fluid_capture against the CPU model (display_model.py) and the
executed reference shaders (capture_*.npz) under the byte tolerance rule, bit for bit against the fp32
render() path it fuses, the kernels it launches, what it leaves alone, and what it refuses."""
import ctypes as C

import numpy as np
import pytest

import capture_model as CM
import display_model as M
from conftest import bits_equal, golden
from display_harness import BACK_RGB, check_capture, make, model_capture, seeded_dye, set_keywords
from display_harness import dither  # noqa: F401 -- a fixture
from sim_harness import pkg  # noqa: F401 -- a fixture

pytestmark = pytest.mark.gpu
GEOMETRIES = ["capture_64_canvas_128", "capture_48x32_canvas_807x640"]


def outside_executed(got, half, delta):
    """The rule against an executed fixture, whose pre-store value p is known only through its fp16 store h:
    |p - h| <= ulp16(h) / 2, so an implementation within d of p lies in [h - d - ulp/2, h + d + ulp/2]."""
    h = half.astype(np.float64)
    u = np.spacing(np.abs(half)).astype(np.float64) / 2
    d = delta * np.maximum(1.0, np.abs(h))
    lo, hi = CM.to_bytes(h - d - u)[::-1], CM.to_bytes(h + d + u)[::-1]
    return int(np.count_nonzero((got < lo) | (got > hi)))


def expected_from_frame(frame):
    """flip(trunc(clamp01(float16(frame)) * 255)): the fp32 render() frame through the capture epilogue."""
    return CM.to_bytes(frame)[::-1]


@pytest.mark.parametrize("name", GEOMETRIES)
def test_capture_vs_model_and_executed_shaders(pkg, name):
    """All eight keyword sets x {BACK_COLOR (10, 20, 30), TRANSPARENT}: against the model (exact without
    BLOOM, within the per-texel powf interval of gamma_model.py with it) and against the executed shaders
    (exact for none / SHADING on the power-of-two geometry, 2e-6 for the others there, 3e-4 on the
    canvas != target geometry).  dye.read is untouched."""
    for bg in ("back", "transparent"):
        g = golden(f"{name}_{bg}")
        pow2 = int(g["canvas_w"]) == int(g["canvas_h"])
        s = make(pkg, int(g["Wd"]), int(g["Hd"]), int(g["canvas_w"]), int(g["canvas_h"]),
                 CAPTURE_RESOLUTION=int(g["capture_res"]), BLOOM_RESOLUTION=int(g["bloom_res"]),
                 SUNRAYS_RESOLUTION=int(g["sun_res"]), TRANSPARENT=bool(g["transparent"]))
        s.writeField("dye", g["in_dye"])
        s.dithering = g["dither"].astype(np.float32)
        for tag, kw in M.SETS.items():
            set_keywords(s, kw)
            got = s.captureScreenshot()
            assert got.dtype == np.uint8 and got.shape == (int(g["h"]), int(g["w"]), 4)
            cfg = dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"]))
            want = model_capture("fp32", g["in_dye"], int(g["w"]), int(g["h"]), int(g["canvas_w"]), int(g["canvas_h"]), kw,
                                 g["dither"].astype(np.float32), cfg, bool(g["transparent"]))
            check_capture(got, want, kw, (name, bg, tag))
            if pow2 and not kw & (M.BLOOM | M.SUNRAYS):
                assert np.array_equal(got, g[f"{tag}_rgba8"]), (name, bg, tag)
            else:
                delta = 2e-6 if pow2 else 3e-4
                assert outside_executed(got, g[f"{tag}_half"], delta) == 0, (name, bg, tag)
            assert bits_equal(s.readField("dye"), g["in_dye"]), (name, bg, tag)
        s.close()


@pytest.mark.parametrize("Wd,Hd,w,h", [(64, 64, 64, 64), (48, 32, 50, 75)])
def test_capture_equals_quantised_render_frame(pkg, dither, Wd, Hd, w, h):
    """Canvas = target: with BACK_COLOR (0, 0, 0) the capture is bit for bit the fp32 render() frame (over
    background 0) through fp16, clamp01 * 255, truncation and the flip; with TRANSPARENT, render(target=True)
    through the same.  All eight sets."""
    s = make(pkg, Wd, Hd, w, h, CAPTURE_RESOLUTION=min(w, h), BLOOM_RESOLUTION=32, SUNRAYS_RESOLUTION=24)
    s.config["BACK_COLOR"] = {"r": 0, "g": 0, "b": 0}
    s.writeField("dye", seeded_dye(Wd, Hd, 11, scale=1.0))
    s.dithering = dither
    assert pkg.capture_inputs(s.config, w, h, dither)["width"] == w
    for kw in range(8):
        set_keywords(s, kw)
        for transparent in (False, True):
            s.config["TRANSPARENT"] = transparent
            frame = s.render(w, h, target=True)
            got = s.captureScreenshot()
            assert np.array_equal(got, expected_from_frame(frame)), (kw, transparent)
    s.close()


@pytest.mark.parametrize("iterations,levels", [(8, 5), (1, 1)])
def test_capture_launches_what_render_launches(pkg, dither, iterations, levels):
    """Steady state: a capture launches exactly what render() launches for the same set (1, + 4 with
    SUNRAYS, + 2L + 1 with BLOOM).  A capture right after a render() on the same canvas launches no more:
    it reuses the post-FX targets (remaking the bloom FBO would add a fill_alpha_kernel launch)."""
    s = make(pkg, 64, 64, 128, 128, CAPTURE_RESOLUTION=64, BLOOM_RESOLUTION=64, SUNRAYS_RESOLUTION=48,
             BLOOM_ITERATIONS=iterations)
    s.writeField("dye", seeded_dye(64, 64, 5, scale=1.0))
    s.dithering = dither
    for kw in range(8):
        set_keywords(s, kw)
        want = 1 + (4 if kw & M.SUNRAYS else 0) + (2 * levels + 1 if kw & M.BLOOM and levels >= 2 else 0)
        s.render(128, 128)
        n0 = s.launch_count()
        s.render(128, 128)
        assert s.launch_count() - n0 == want, kw
        n0 = s.launch_count()
        s.captureScreenshot()
        assert s.launch_count() - n0 <= want, kw          # right after render() on the same canvas
        n0 = s.launch_count()
        s.captureScreenshot()
        assert s.launch_count() - n0 == want, kw          # steady state
    s.close()


def test_capture_leaves_dye_and_render_alone(pkg, dither):
    """dye.read is unchanged by a capture (SUNRAYS draws its mask into dye.write, as the reference does), and
    the render() after it is the render() before it: FLUID_BACKGROUND (the checkerboard here) is untouched."""
    dye = seeded_dye(64, 48, 9, scale=1.0)
    s = make(pkg, 64, 48, 128, 96, CAPTURE_RESOLUTION=48, BLOOM_RESOLUTION=32, SUNRAYS_RESOLUTION=24, TRANSPARENT=True)
    s.writeField("dye", dye)
    s.dithering = dither
    for kw in range(8):
        set_keywords(s, kw)
        before = s.render()
        bg = C.c_float()
        assert s._L.fluid_get_param(s._h, pkg.PARAM["BACKGROUND"], C.byref(bg)) == 0 and bg.value == 1
        s.captureScreenshot()
        assert bits_equal(s.readField("dye"), dye), kw
        assert s._L.fluid_get_param(s._h, pkg.PARAM["BACKGROUND"], C.byref(bg)) == 0 and bg.value == 1
        assert bits_equal(s.render(), before), kw
    s.close()


def test_half_storage_capture(pkg, oracle, dither):
    """A half-storage handle captures none and SHADING exactly as its own render() frame quantised; BLOOM or
    SUNRAYS are refused with FLUID_ERR_INVALID and the handle stays usable.  The capture launches the widen
    kernel and the display."""
    s = make(pkg, 64, 64, 64, 64, flags=pkg.FLAG_HALF_STORAGE, CAPTURE_RESOLUTION=64)
    s.config["BACK_COLOR"] = {"r": 0, "g": 0, "b": 0}
    s.writeField("dye", oracle.round_half(seeded_dye(64, 64, 3, scale=1.0)))
    s.dithering = dither
    for bloom, sunrays in ((True, False), (False, True), (True, True)):
        s.config.update(SHADING=True, BLOOM=bloom, SUNRAYS=sunrays)
        with pytest.raises(pkg.FluidError) as e:
            s.captureScreenshot()
        assert e.value.code == -1 and "HALF_STORAGE" in str(e.value)
    for shading in (False, True):
        s.config.update(SHADING=shading, BLOOM=False, SUNRAYS=False)
        for transparent in (False, True):
            s.config["TRANSPARENT"] = transparent
            frame = s.render(64, 64, target=True)
            n0 = s.launch_count()
            got = s.captureScreenshot()
            assert s.launch_count() - n0 == 2
            assert np.array_equal(got, expected_from_frame(frame)), (shading, transparent)
    s.close()


def test_refusals_leave_the_handle_usable(pkg, dither):
    """Every bad argument gets FLUID_ERR_INVALID, and the next good capture on the same handle succeeds."""
    s = make(pkg, 64, 64, 128, 128, CAPTURE_RESOLUTION=64, BLOOM_RESOLUTION=64, SUNRAYS_RESOLUTION=48)
    s.writeField("dye", seeded_dye(64, 64, 7, scale=1.0))
    s.dithering = dither
    s.config.update(SHADING=True, BLOOM=True, SUNRAYS=True)
    _, fx, dith = pkg.postfx_inputs(s.config, dither)
    good = s.captureScreenshot()
    out = np.empty((64, 64, 4), np.uint8)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)        # noqa: E731
    all3 = M.SHADING | M.BLOOM | M.SUNRAYS

    def call(w=64, h=64, cw=128, ch=128, kw=all3, fx_=C.byref(fx), d=ptr(dith), n=out.size, dst=ptr(out)):
        return s._L.fluid_capture(s._h, w, h, cw, ch, kw, 0, fx_, d, dith.shape[1], dith.shape[0], *BACK_RGB, dst, n)

    bad = [dict(kw=8), dict(kw=all3 | 0x10), dict(n=out.size - 1), dict(n=out.size + 4), dict(w=0), dict(h=0),
           dict(cw=0), dict(ch=-1), dict(kw=M.BLOOM, d=None), dict(kw=M.BLOOM, fx_=None), dict(kw=M.SUNRAYS, fx_=None),
           dict(dst=None)]
    for b in bad:
        assert call(**b) == -1, b
        assert call() == 0, b
        assert np.array_equal(out, good), b
    s.close()


def test_capture_writes_png(pkg, dither, tmp_path):
    """captureScreenshot(path) writes the returned bytes as an RGBA PNG."""
    import zlib
    s = make(pkg, 64, 64, 128, 128, CAPTURE_RESOLUTION=64)
    s.writeField("dye", seeded_dye(64, 64, 1, scale=1.0))
    p = tmp_path / "fluid.png"
    img = s.captureScreenshot(str(p))
    data = p.read_bytes()
    assert data[:8] == b"\x89PNG\r\n\x1a\n" and data[12:16] == b"IHDR"
    n = int.from_bytes(data[33:37], "big")
    assert data[37:41] == b"IDAT"
    raw = np.frombuffer(zlib.decompress(data[41:41 + n]), np.uint8).reshape(64, 1 + 64 * 4)
    assert np.all(raw[:, 0] == 0) and np.array_equal(raw[:, 1:].reshape(64, 64, 4), img)
    s.close()
