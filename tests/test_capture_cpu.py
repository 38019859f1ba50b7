"""captureScreenshot() (S:287-349) on the CPU: the capture model (display_model.py, capture_model.py) against the executed
reference shaders (capture_*.npz), a negative control for the canvas-sized post-FX, the PNG writer, and
the host-side mapping from `config` and the canvas to what fluid_capture is given.  Runs without a GPU."""
import struct
import zlib

import numpy as np
import pytest

import capture_model as CM
import display_model as M
import webgl_fluid_simulation_b200 as pkg
from conftest import golden

GEOMETRIES = {"pow2": "capture_64_canvas_128", "ragged": "capture_48x32_canvas_807x640"}
SETS = M.SETS


def executed_delta(geometry, kw):
    """The fp32 tolerance of the keyword tests against the executed shaders: exact for none / SHADING and
    2e-6 for the others on the power-of-two geometry (pow() and the 48-wide sunrays texture), 3e-4 on the
    ragged one."""
    if geometry == "ragged":
        return 3e-4
    return 0.0 if not kw & (M.BLOOM | M.SUNRAYS) else 2e-6


def model(g, kw, fx_size=None):
    return M.capture(g["in_dye"], int(g["w"]), int(g["h"]), int(g["canvas_w"]), int(g["canvas_h"]),
                     g["dither"].astype(np.float32), kw, bool(g["transparent"]),
                     tuple(float(x) / 255 for x in g["back"]),
                     cfg=dict(BLOOM_RESOLUTION=int(g["bloom_res"]), SUNRAYS_RESOLUTION=int(g["sun_res"])), fx_size=fx_size)


@pytest.mark.parametrize("bg", ["back", "transparent"])
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_capture_model_matches_executed_reference_shaders(oracle, geometry, bg):
    """All eight keyword sets: every byte of the executed capture lies in the rule's bracket around the
    model's pre-store value.  The fixture's bytes are normalizeTexture of its own fp16 target."""
    g = golden(f"{GEOMETRIES[geometry]}_{bg}")
    assert [str(s) for s in g["sets"]] == list(SETS)
    for tag, kw in SETS.items():
        half = g[f"{tag}_half"]
        assert half.dtype == np.float16 and half.shape == (int(g["h"]), int(g["w"]), 4)
        assert np.array_equal(CM.to_bytes(half)[::-1], g[f"{tag}_rgba8"]), tag
        m = model(g, kw)
        assert CM.bytes_outside(g[f"{tag}_rgba8"], m["pre"], executed_delta(geometry, kw)) == 0, tag
        if executed_delta(geometry, kw) == 0:
            assert np.array_equal(m["rgba8"], g[f"{tag}_rgba8"]), tag


@pytest.mark.parametrize("bg", ["back", "transparent"])
def test_target_sized_post_fx_fails_on_the_canvas_fixture(oracle, bg):
    """Negative control: the bloom and sunrays FBOs sized from the 61 x 48 target (41 x 32, 51 x 40) instead
    of the 807 x 640 canvas (40 x 32, 50 x 40) must fail the same rule for every set with BLOOM or SUNRAYS,
    so the fixture does pin the canvas sizes."""
    g = golden(f"{GEOMETRIES['ragged']}_{bg}")
    w, h = int(g["w"]), int(g["h"])
    assert (w, h) == (61, 48)
    assert pkg.getResolution(int(g["bloom_res"]), 807, 640) == {"width": 40, "height": 32}
    assert pkg.getResolution(int(g["bloom_res"]), w, h) == {"width": 41, "height": 32}
    assert pkg.getResolution(int(g["sun_res"]), 807, 640) == {"width": 50, "height": 40}
    assert pkg.getResolution(int(g["sun_res"]), w, h) == {"width": 51, "height": 40}
    for tag, kw in SETS.items():
        if not kw & (M.BLOOM | M.SUNRAYS):
            continue
        wrong = model(g, kw, fx_size=(w, h))
        assert CM.bytes_outside(g[f"{tag}_rgba8"], wrong["pre"], executed_delta("ragged", kw)) > 0, tag


def test_byte_rule_corner_cases():
    """B(x): fp16 store (nearest even, overflow to +-Inf), clamp01, * 255, truncation, NaN -> 0; monotone."""
    x = np.array([np.nan, -np.inf, -1.0, 0.0, 1 / 255, 0.5, 1 - 2.0 ** -11, 1.0, 65520.0, np.inf], np.float64)
    assert list(CM.to_bytes(x)) == [0, 0, 0, 0, 0, 127, 254, 255, 255, 255]
    r = np.sort(np.random.default_rng(1).normal(0.5, 0.6, 20000))
    assert np.all(np.diff(CM.to_bytes(r).astype(int)) >= 0)
    assert CM.back16((10 / 255, 20 / 255, 30 / 255)) == tuple(float(np.float16(np.float32(c / 255))) for c in (10, 20, 30))


def _read_png(path):
    """A minimal PNG reader: every chunk's CRC, IHDR, the concatenated IDAT stream inflated and un-filtered
    (filter types 0-4 of the PNG spec)."""
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, []
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert crc == zlib.crc32(tag + body) & 0xFFFFFFFF, tag
        chunks.append((tag, body))
        pos += 12 + n
    assert chunks[0][0] == b"IHDR" and chunks[-1] == (b"IEND", b"")
    w, h, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", chunks[0][1])
    assert (depth, ctype, comp, filt, inter) == (8, 6, 0, 0, 0)
    raw = zlib.decompress(b"".join(b for t, b in chunks if t == b"IDAT"))
    stride = 4 * w
    assert len(raw) == h * (stride + 1)
    out = np.zeros((h, stride), np.int64)
    for j in range(h):
        f, line = raw[j * (stride + 1)], np.frombuffer(raw, np.uint8, stride, j * (stride + 1) + 1).astype(np.int64)
        up = out[j - 1] if j else np.zeros(stride, np.int64)
        row = np.zeros(stride, np.int64)
        for i in range(stride):
            a = row[i - 4] if i >= 4 else 0
            c = up[i - 4] if i >= 4 else 0
            b = up[i]
            if f == 0: p = 0
            elif f == 1: p = a
            elif f == 2: p = b
            elif f == 3: p = (a + b) // 2
            else:
                pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                p = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
            row[i] = (line[i] + p) & 0xFF
        out[j] = row
    return out.astype(np.uint8).reshape(h, w, 4), [t for t, _ in chunks]


@pytest.mark.parametrize("shape", [(1, 1), (7, 13), (64, 81)])
def test_write_png_round_trip(tmp_path, shape):
    img = np.random.default_rng(shape[1]).integers(0, 256, shape + (4,), dtype=np.uint8)
    p = tmp_path / "fluid.png"
    pkg.write_png(str(p), img)
    got, tags = _read_png(str(p))
    assert tags == [b"IHDR", b"IDAT", b"IEND"]
    assert np.array_equal(got, img)


def test_write_png_refuses_other_images(tmp_path):
    for bad in (np.zeros((4, 4, 4), np.float32), np.zeros((4, 4, 3), np.uint8), np.zeros((4, 4), np.uint8)):
        with pytest.raises(ValueError):
            pkg.write_png(str(tmp_path / "x.png"), bad)


def test_product_writes_png_without_pil():
    import inspect
    import webgl_fluid_simulation_b200.sim as sim
    assert "PIL" not in inspect.getsource(sim)


@pytest.mark.parametrize("shading", [False, True])
@pytest.mark.parametrize("bloom", [False, True])
@pytest.mark.parametrize("sunrays", [False, True])
@pytest.mark.parametrize("transparent", [False, True])
def test_capture_inputs_from_config_and_canvas(shading, bloom, sunrays, transparent):
    """captureScreenshot's target is getResolution(CAPTURE_RESOLUTION) of the canvas (S:288); the keywords,
    TRANSPARENT, the post-FX keys and the dithering texture follow render() (postfx_inputs)."""
    cfg = dict(pkg.default_config(), SHADING=shading, BLOOM=bloom, SUNRAYS=sunrays, TRANSPARENT=transparent,
               CAPTURE_RESOLUTION=64)
    a = pkg.capture_inputs(cfg, 807, 640, np.zeros((64, 64, 3), np.float32))
    assert (a["width"], a["height"]) == (81, 64)
    assert a["keywords"] == pkg.display_keywords(cfg) and a["transparent"] is transparent
    assert (a["fx"] is None) == (not bloom and not sunrays)
    assert (a["dither"] is None) == (not bloom)
    if bloom:
        with pytest.raises(ValueError, match="dithering"):
            pkg.capture_inputs(cfg, 807, 640, None)
    else:
        assert pkg.capture_inputs(cfg, 807, 640, None)["dither"] is None
    b = pkg.capture_inputs(dict(cfg, CAPTURE_RESOLUTION=512), 1080, 1920, None if not bloom else np.zeros((2, 2, 3)))
    assert (b["width"], b["height"]) == (512, 910)


def test_default_config_has_capture_resolution():
    assert pkg.default_config()["CAPTURE_RESOLUTION"] == 512          # S:62
