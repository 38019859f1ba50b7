"""Batch draws with a look per image (fluid_render_canvas_looks / fluid_capture_looks), on the CPU:

* the ABI: include/fluid.h, the library's exports and the ctypes binding agree on the two entry points and on
  fluid_look;
* the look table: csrc/looks.h, the host code that turns a fluid_look into what the batch kernels read, compiled
  on its own and run on every display_harness.SETS slider set.  The prefilter's knee and curve must be the float64
  restatement narrowed once; at t033_k07, t039_k1 and t005 deriving them in fp32 gives other bits, so a table
  derived in fp32 fails here.  The backgrounds are the capture's fp16 BACK_COLOR and the canvas's u8(BACK_COLOR);
* FluidBatch's choice of call, against a stand-in library that records the calls: the shared-look calls of
  before while no member overrides a DISPLAY_MEMBER_KEYS key, the _looks calls with one fluid_look per image
  otherwise, and ValueError for any other key."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import webgl_fluid_simulation_b200 as pkg
from display_harness import SETS
from webgl_fluid_simulation_b200 import _lib, sim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "webgl_fluid_simulation_b200", "csrc")
F32 = np.float32
NEW = ("fluid_render_canvas_looks", "fluid_capture_looks")


@pytest.fixture(scope="module")
def L():
    pkg.build()
    return pkg.lib()


def header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "fluid.h")).read(), flags=re.S)


# ---- 1. header = library = binding -----------------------------------------------------------------------------
def test_header_library_and_binding_agree(L):
    hdr = header()
    body = re.search(r"typedef struct fluid_look \{(.*?)\} fluid_look;", hdr, re.S).group(1)
    fields = []
    for ctype, names in re.findall(r"(double|float|int32_t)\s+([^;]+);", body):
        fields += [(n.strip(), ctype) for n in names.split(",")]
    ctypes_of = {"double": C.c_double, "float": C.c_float, "int32_t": C.c_int32}
    assert [(n, ctypes_of[t]) for n, t in fields] == list(_lib.Look._fields_)
    assert C.sizeof(_lib.Look) == 48
    for name in NEW:
        assert name in _lib.SYMBOLS and hasattr(L, name), name
        params = re.search(name + r"\s*\((.*?)\);", hdr, re.S).group(1).split(",")
        assert len(getattr(L, name).argtypes) == len(params), name
        assert "const fluid_look* looks" in [p.strip() for p in params], name
    # the same as the shared-look calls, without transparent and back_*, with the looks before dst
    assert L.fluid_render_canvas_looks.argtypes[-6] is C.POINTER(_lib.Look)
    assert L.fluid_capture_looks.argtypes[-6] is C.POINTER(_lib.Look)


# ---- 2. the look table -----------------------------------------------------------------------------------------
DRIVER = r"""
#include <cstdio>
#include "looks.h"
// one fluid_look per input line; the ImageLook the library derives from it, each value's bits in hex
int main() {
    fluid_look l;
    while (std::scanf("%la %la %la %la %a %a %a %d", &l.bloom_intensity, &l.bloom_threshold, &l.bloom_soft_knee,
                      &l.sunrays_weight, &l.back_r, &l.back_g, &l.back_b, &l.transparent) == 8) {
        const fk::ImageLook e = fk::image_look(l);
        const float f[] = {e.curve[0], e.curve[1], e.curve[2], e.curve[3], e.intensity, e.weight,
                           e.back16[0], e.back16[1], e.back16[2]};
        for (float v : f) { unsigned u; std::memcpy(&u, &v, 4); std::printf("%08x ", u); }
        std::printf("%d %d %d %d\n", e.back8[0], e.back8[1], e.back8[2], e.transparent);
    }
}
"""


@pytest.fixture(scope="module")
def image_look(tmp_path_factory):
    """image_look of csrc/looks.h as a function of a list of looks (tuples in fluid_look's order)."""
    cxx = shutil.which(os.environ.get("CXX", "c++")) or shutil.which("g++")
    assert cxx, "a C++ compiler"
    d = tmp_path_factory.mktemp("looks")
    src, exe = d / "driver.cpp", d / "driver"
    src.write_text("#include <cstring>\n" + DRIVER)
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.run([cxx, "-O3", "-std=c++17", "-I", CSRC, "-I", os.path.join(cuda, "include"), str(src), "-o",
                    str(exe)], check=True)

    def run(looks):
        lines = [" ".join([float(v).hex() for v in lk[:4]] + [float(F32(v)).hex() for v in lk[4:7]] + [str(lk[7])])
                 for lk in looks]
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True,
                             check=True).stdout.split("\n")
        rows = []
        for line in out[:len(looks)]:
            v = line.split()
            rows.append(dict(f=np.array([int(x, 16) for x in v[:9]], np.uint32).view(F32),
                             back8=[int(x) for x in v[9:12]], transparent=int(v[12])))
        return rows

    return run


def curve64(threshold, soft_knee):
    """applyBloom's knee and curve (S:1358-1363) in float64, each narrowed once to fp32."""
    knee = threshold * soft_knee + 0.0001
    return np.array([threshold - knee, knee * 2, 0.25 / knee, threshold], np.float64).astype(F32)


def curve32(threshold, soft_knee):
    """The same derived in fp32: the mistake the table must not make."""
    t, k = F32(threshold), F32(soft_knee)
    knee = t * k + F32(0.0001)
    return np.array([t - knee, knee * F32(2), F32(0.25) / knee, t], F32)


def test_prefilter_constants_are_derived_in_double(image_look):
    names = list(SETS)
    rows = image_look([(*SETS[n], 0.1, 0.2, 0.3, 0) for n in names])
    for n, r in zip(names, rows):
        I, T, K, W = SETS[n]
        want = np.concatenate([curve64(T, K), np.array([I, W], np.float64).astype(F32)])
        assert np.array_equal(r["f"][:6].view(np.uint32), want.view(np.uint32)), (n, r["f"][:6], want)
    differ = {n for n in names if not np.array_equal(curve64(*SETS[n][1:3]).view(np.uint32),
                                                     curve32(*SETS[n][1:3]).view(np.uint32))}
    assert {"t033_k07", "t039_k1", "t005"} <= differ, differ


def u8(x):
    """u8 of the canvas: clamp01 (NaN 0), times 255 in fp32, rounded to nearest even."""
    c = np.fmin(np.fmax(F32(x), F32(0)), F32(1))
    return int(np.rint(c * F32(255)))


def test_backgrounds(image_look):
    """BACK_COLOR channels at 0 and 255 and between, and values outside [0, 1] and NaN as the C call may get them:
    the capture's fp16 store of the value and the canvas's byte; transparent is one bit."""
    backs = [(0.0, 1.0, 10 / 255), (20 / 255, 30 / 255, 127.5 / 255), (-0.5, 2.0, float("nan")),
             (float("inf"), -float("inf"), 0.5 / 255), (1.5 / 255, 2.5 / 255, 254.5 / 255)]
    for tr in (0, 1, 7):
        rows = image_look([(0.8, 0.6, 0.7, 1.0, *b, tr) for b in backs])
        for b, r in zip(backs, rows):
            f16 = np.array(b, F32).astype(np.float16).astype(F32)
            assert np.array_equal(r["f"][6:9], f16, equal_nan=True), (b, r["f"][6:9], f16)
            assert r["back8"] == [u8(x) for x in b], (b, r["back8"])
            assert r["transparent"] == (tr != 0)


# ---- 3. FluidBatch's calls -------------------------------------------------------------------------------------
class Recorder:
    """A stand-in library: records every draw with its arguments and the looks it was given."""

    def __init__(self, members):
        self.B = members
        self.calls = []

    def fluid_members(self, h):
        return self.B

    def fluid_set_param_f64(self, h, key, v):
        return 0

    def fluid_set_param_members(self, h, key, values, n):
        return 0

    def fluid_last_error(self, h):
        return b""

    def _record(self, name, args, looks_at=None, list_at=None):
        rec = {"name": name, "args": args}
        if looks_at is not None:
            n = args[-1]
            rec["looks"] = [tuple(getattr(args[looks_at][k], f) for f, _ in _lib.Look._fields_) for k in range(n)]
        if list_at is not None:
            mp, n = args[list_at], args[-1]
            rec["members"] = None if mp is None else np.ctypeslib.as_array(mp, (n,)).tolist()
        self.calls.append(rec)
        return 0

    def fluid_render_canvas_batch(self, *a):
        return self._record("canvas_batch", a)

    def fluid_render_canvas_members(self, *a):
        return self._record("canvas_members", a, list_at=-2)

    def fluid_render_canvas_looks(self, *a):
        return self._record("canvas_looks", a, looks_at=8, list_at=-2)

    def fluid_capture_batch(self, *a):
        return self._record("capture_batch", a)

    def fluid_capture_members(self, *a):
        return self._record("capture_members", a, list_at=-2)

    def fluid_capture_looks(self, *a):
        return self._record("capture_looks", a, looks_at=10, list_at=-2)

    def take(self):
        c, self.calls = self.calls, []
        return c


def stand_in(B):
    b = object.__new__(sim.FluidBatch)
    b.config = sim.default_config()
    b.config.update(SHADING=True, BLOOM=False, SUNRAYS=True, BACK_COLOR={"r": 10, "g": 20, "b": 30})
    b.canvas = {"width": 64, "height": 48}
    b._L = Recorder(B)
    b._h = C.c_void_p(1)
    b._pushed = {}
    b.member_config = [{} for _ in range(B)]
    return b


def look_of(c):
    """The fluid_look FluidBatch must pass for a member whose config is c, as the record holds it."""
    bc = c["BACK_COLOR"]
    return (float(c["BLOOM_INTENSITY"]), float(c["BLOOM_THRESHOLD"]), float(c["BLOOM_SOFT_KNEE"]),
            float(c["SUNRAYS_WEIGHT"]), *(float(F32(bc[k] / 255)) for k in "rgb"), 1 if c.get("TRANSPARENT") else 0)


def draw(b, call, members=None):
    return b.render_canvas(members=members) if call == "canvas" else b.captureScreenshot(members=members)


@pytest.mark.parametrize("call", ["canvas", "capture"])
def test_shared_look_calls_without_display_overrides(L, call):
    """MEMBER_KEYS overrides alone leave render_canvas() and captureScreenshot() on the calls they made before."""
    b = stand_in(3)
    b.member_config[1]["CURL"] = 5.0
    draw(b, call)
    draw(b, call, members=[2, 0])
    got = b._L.take()
    assert [c["name"] for c in got] == [call + "_batch", call + "_members"]
    assert got[1]["members"] == [2, 0]
    tr_at = 4 if call == "canvas" else 6                      # transparent, after (w, h[, canvas_w, canvas_h], kw)
    assert all(c["args"][tr_at] == 0 for c in got)
    assert got[0]["args"][tr_at + 5:tr_at + 8] == pytest.approx((10 / 255, 20 / 255, 30 / 255))


@pytest.mark.parametrize("call", ["canvas", "capture"])
def test_looks_calls_with_display_overrides(L, call):
    """One override of a DISPLAY_MEMBER_KEYS key sends every draw through the _looks call: one fluid_look per
    image, member_config over config, the shared call's other arguments unchanged, and the list as given."""
    B = 4
    b = stand_in(B)
    b.config["TRANSPARENT"] = False
    over = [{}, {"BLOOM_INTENSITY": 2.0, "BACK_COLOR": {"r": 0, "g": 255, "b": 7}},
            {"TRANSPARENT": True, "SUNRAYS_WEIGHT": 0.3, "CURL": 1.0},
            {"BLOOM_THRESHOLD": 0.33, "BLOOM_SOFT_KNEE": 0.7}]
    b.member_config = [dict(o) for o in over]
    draw(b, call)
    shared = b._L.take()
    b.member_config = [{} for _ in range(B)]
    draw(b, call)
    plain = b._L.take()[0]["args"]
    b.member_config = [dict(o) for o in over]
    draw(b, call, members=[3, 1])
    draw(b, call, members=[])
    got = shared + b._L.take()
    assert [c["name"] for c in got] == [call + "_looks"] * 3
    looks = [look_of({**b.config, **o}) for o in over]
    assert got[0]["looks"] == looks and got[0]["members"] is None and got[0]["args"][-1] == B
    assert got[1]["looks"] == [looks[3], looks[1]] and got[1]["members"] == [3, 1]
    assert got[2]["looks"] == [] and got[2]["args"][-1] == 0
    # sizes, keywords, fx and the dithering texture's size as the shared-look call passes them; its transparent
    # (plain[k]) and back_* are dropped
    k = 4 if call == "canvas" else 6
    a = got[0]["args"]
    assert a[:k] == plain[:k] and a[k + 2:k + 4] == plain[k + 3:k + 5]
    assert bytes(a[k]._obj) == bytes(plain[k + 1]._obj) and a[k + 1] is None is plain[k + 2]
    assert a[-4] == 4 * B * a[1] * a[2]


@pytest.mark.parametrize("key", ["PRESSURE_ITERATIONS", "ASPECT", "BLOOM_ITERATIONS", "BLOOM_RESOLUTION",
                                 "SUNRAYS_RESOLUTION", "CAPTURE_RESOLUTION", "SHADING", "BLOOM"])
def test_other_keys_raise(L, key):
    b = stand_in(2)
    b.member_config[1][key] = 1
    for call in ("canvas", "capture"):
        with pytest.raises(ValueError):
            draw(b, call)
    assert b._L.take() == []


def test_display_keys_are_not_pushed_as_member_values():
    b = stand_in(2)
    pushed = []
    b._L.fluid_set_param_members = lambda h, key, values, n: pushed.append(key) or 0
    b._L.fluid_step = lambda h, dt: 0
    for k in sim.FluidBatch.DISPLAY_MEMBER_KEYS:
        b.member_config[1][k] = {"r": 1, "g": 2, "b": 3} if k == "BACK_COLOR" else 0.5
    b.step(0.016)
    assert pushed == []
    assert set(sim.FluidBatch.DISPLAY_MEMBER_KEYS).isdisjoint(sim.FluidBatch.MEMBER_KEYS)
