"""Host-side mirror of the reference's simulation surface (script.js), over the C ABI.

The reference's interface is a set of globals in one classic script: `config` (S:59-85),
`step(dt)` (S:1231-1294), `splat(x,y,dx,dy,color)` (S:1441-1455), `multipleSplats(n)` (S:1427-1439),
`splatPointer(p)` (S:1421-1425), `initFramebuffers()` (S:982-1010), `generateColor()` (S:1565-1571),
`calcDeltaTime()` (S:1188-1194), `update()` (S:1176-1186) and the field objects
`velocity/dye/pressure/divergence/curl` (S:950-954).  `FluidSimulation` keeps those names,
argument meanings and the live-`config` behaviour (keys are read on every call), and forwards the
work to libfluid_b200 (hand-written sm_90a kernels).  js/fluid-sim.js is the same mirror in the
reference's own language for when Node is available; this Python twin is what the tests drive.

There is no CPU or PyTorch fallback: constructing a simulation without the built library or
without an H100 raises.

The host-side helpers (Pointer, HSVtoRGB, wrap, generateColor, multipleSplats, splatPointer,
calcDeltaTime, updateColors, applyInputs, updatePointer*Data, correctDelta*) follow script.js line
for line because mirroring that interface is the point; those parts are Copyright (c) 2017 Pavel
Dobryakov, MIT License (see LICENSE).
"""
from __future__ import annotations

import ctypes as C
import math
import random as _random
import struct
import time
import zlib

import numpy as np

from . import _lib
from ._lib import DISPLAY_BLOOM, DISPLAY_SHADING, DISPLAY_SUNRAYS, FIELD, PARAM, STAT, Config, FluidError, PostFX, Timing


def default_config(flags: int = 0) -> dict:
    """The simulation keys of the reference `config` literal, S:59-69 + S:73 (render keys are out of
    scope and kept only so a reference config object can be passed through unchanged).  With
    FLAG_NEAREST_FILTERING in `flags` the reference's override for a device without float linear
    filtering applies (S:109-114): DYE_RESOLUTION 512, SHADING / BLOOM / SUNRAYS off."""
    c = {
        "SIM_RESOLUTION": 128,
        "DYE_RESOLUTION": 1024,
        "CAPTURE_RESOLUTION": 512,   # S:62, captureScreenshot's target (S:288)
        "DENSITY_DISSIPATION": 1,
        "VELOCITY_DISSIPATION": 0.2,
        "PRESSURE": 0.8,
        "PRESSURE_ITERATIONS": 20,
        "CURL": 30,
        "SPLAT_RADIUS": 0.25,
        "SPLAT_FORCE": 6000,
        "SHADING": True,
        "COLORFUL": True,
        "COLOR_UPDATE_SPEED": 10,
        "PAUSED": False,
        "BACK_COLOR": {"r": 0, "g": 0, "b": 0},
        "TRANSPARENT": False,
        "BLOOM": False,          # reference default is true; needs `sim.dithering` (the 64x64 RGB texture), see render()
        "BLOOM_ITERATIONS": 8,
        "BLOOM_RESOLUTION": 256,
        "BLOOM_INTENSITY": 0.8,
        "BLOOM_THRESHOLD": 0.6,
        "BLOOM_SOFT_KNEE": 0.7,
        "SUNRAYS": False,        # reference default is true
        "SUNRAYS_RESOLUTION": 196,
        "SUNRAYS_WEIGHT": 1.0,
    }
    if flags & _lib.FLAG_NEAREST_FILTERING:
        c.update(DYE_RESOLUTION=512, SHADING=False, BLOOM=False, SUNRAYS=False)
    return c


class Pointer:
    """pointerPrototype, S:87-98."""

    def __init__(self):
        self.id = -1
        self.texcoordX = 0.0
        self.texcoordY = 0.0
        self.prevTexcoordX = 0.0
        self.prevTexcoordY = 0.0
        self.deltaX = 0.0
        self.deltaY = 0.0
        self.down = False
        self.moved = False
        self.color = {"r": 30, "g": 0, "b": 300}


def HSVtoRGB(h, s, v):
    """S:1573-1597."""
    i = math.floor(h * 6)
    f = h * 6 - i
    p = v * (1 - s)
    q = v * (1 - f * s)
    t = v * (1 - (1 - f) * s)
    r, g, b = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)][i % 6]
    return {"r": r, "g": g, "b": b}


def getResolution(resolution, canvas_w, canvas_h):
    """S:1612-1624 (via the C ABI so both hosts share one implementation)."""
    w, h = C.c_int(), C.c_int()
    _lib.lib().fluid_get_resolution(int(resolution), int(canvas_w), int(canvas_h), C.byref(w), C.byref(h))
    return {"width": w.value, "height": h.value}


def display_keywords(config) -> int:
    """updateKeywords, S:1160-1166: the display shader's keyword set as DISPLAY_* bits."""
    kw = 0
    if config.get("SHADING"):
        kw |= DISPLAY_SHADING
    if config.get("BLOOM"):
        kw |= DISPLAY_BLOOM
    if config.get("SUNRAYS"):
        kw |= DISPLAY_SUNRAYS
    return kw


def postfx_inputs(config, dithering):
    """What render() hands fluid_render_keywords besides the target: (keywords, PostFX or None without
    BLOOM and SUNRAYS, the float32 (dh, dw, 3) dithering texture or None without BLOOM).  The dithering
    texture is drawn only with BLOOM (S:1341-1344), so only then is it required."""
    kw = display_keywords(config)
    dith = None
    if kw & DISPLAY_BLOOM:
        if dithering is None:
            raise ValueError("BLOOM needs sim.dithering: the (64, 64, 3) float RGB dithering texture (LDR_LLL1_0.png / 255)")
        dith = np.ascontiguousarray(dithering, np.float32)
        if dith.ndim != 3 or dith.shape[2] != 3 or dith.shape[0] < 1 or dith.shape[1] < 1:
            raise ValueError(f"sim.dithering must be (height, width, 3) RGB, got shape {dith.shape}")
    if not kw & (DISPLAY_BLOOM | DISPLAY_SUNRAYS):
        return kw, None, None
    fx = PostFX(int(config["BLOOM_ITERATIONS"]), int(config["BLOOM_RESOLUTION"]), float(config["BLOOM_INTENSITY"]),
                float(config["BLOOM_THRESHOLD"]), float(config["BLOOM_SOFT_KNEE"]), int(config["SUNRAYS_RESOLUTION"]),
                float(config["SUNRAYS_WEIGHT"]))
    return kw, fx, dith


def capture_inputs(config, canvas_w, canvas_h, dithering):
    """What captureScreenshot (S:287-299) hands fluid_capture: the target size getResolution(CAPTURE_RESOLUTION)
    of the canvas, the display keywords, config.TRANSPARENT, and the PostFX / dithering texture of
    postfx_inputs (the dithering texture is required only with BLOOM)."""
    res = getResolution(config["CAPTURE_RESOLUTION"], canvas_w, canvas_h)
    kw, fx, dith = postfx_inputs(config, dithering)
    return dict(width=res["width"], height=res["height"], keywords=kw, transparent=bool(config.get("TRANSPARENT")),
                fx=fx, dither=dith)


def write_png(path, rgba8) -> None:
    """Writes an (h, w, 4) uint8 image, top row first, as an 8-bit RGBA PNG: signature, IHDR (colour type
    6), one zlib IDAT with filter 0 on every row, IEND.  It stands in for toDataURL + downloadURI
    (S:296-297).  The bytes are written as they are: browsers that keep 2-D canvases premultiplied change
    RGB wherever alpha < 255 on the way through putImageData / toDataURL, which is browser-defined and
    not emulated."""
    img = np.ascontiguousarray(rgba8)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 4:
        raise ValueError(f"write_png needs an (h, w, 4) uint8 image, got {img.dtype} {img.shape}")
    h, w = img.shape[:2]

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    raw = np.concatenate([np.zeros((h, 1), np.uint8), img.reshape(h, 4 * w)], axis=1).tobytes()
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n")
        f.write(chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 6, 0, 0, 0)))
        f.write(chunk(b"IDAT", zlib.compress(raw, 6)))
        f.write(chunk(b"IEND", b""))


class _Field:
    """What the reference exposes as `velocity.read`, `dye.read`, ...: size + texel size + data."""

    def __init__(self, sim, name):
        self._sim, self._name = sim, name

    @property
    def width(self):
        return self._sim._dims(self._name)[0]

    @property
    def height(self):
        return self._sim._dims(self._name)[1]

    @property
    def texelSizeX(self):
        return 1.0 / self.width

    @property
    def texelSizeY(self):
        return 1.0 / self.height

    def read(self) -> np.ndarray:
        return self._sim.readField(self._name)


class _Handle:
    """What FluidSimulation and FluidBatch share: a library handle `_h`, the live `config` pushed before each
    call, and the calls that take any handle."""

    def _check(self, rc):
        if rc != 0:
            msg = self._L.fluid_last_error(self._h if self._h else None)
            raise FluidError(rc, msg.decode() if msg else "")

    def _aspect(self):
        return self.canvas["width"] / self.canvas["height"]

    def _config(self, sim_w, sim_h, dye_w, dye_h):
        """The fluid_config of a new handle: the simulation keys as they stand now (a slab handle sizes its
        ghost zone from PRESSURE_ITERATIONS); later changes are pushed live by _push_config()."""
        cfg = Config()
        self._L.fluid_config_default(C.byref(cfg))
        cfg.sim_w, cfg.sim_h, cfg.dye_w, cfg.dye_h = sim_w, sim_h, dye_w, dye_h
        cfg.aspect = self._aspect()
        cfg.device, cfg.flags, cfg.jacobi_block = self._device, self._flags, self._jb
        cfg.density_dissipation = float(self.config["DENSITY_DISSIPATION"])
        cfg.velocity_dissipation = float(self.config["VELOCITY_DISSIPATION"])
        cfg.pressure = float(self.config["PRESSURE"])
        cfg.pressure_iterations = int(self.config["PRESSURE_ITERATIONS"])
        cfg.curl = float(self.config["CURL"])
        cfg.splat_radius = float(self.config["SPLAT_RADIUS"])
        return cfg

    def _live_values(self):
        """What _push_config pushes: each key's value as `config` and the canvas hold it now."""
        return {
            "DENSITY_DISSIPATION": self.config["DENSITY_DISSIPATION"],
            "VELOCITY_DISSIPATION": self.config["VELOCITY_DISSIPATION"],
            "PRESSURE": self.config["PRESSURE"],
            "PRESSURE_ITERATIONS": self.config["PRESSURE_ITERATIONS"],
            "CURL": self.config["CURL"],
            "SPLAT_RADIUS": self.config["SPLAT_RADIUS"],
            "ASPECT": self._aspect(),
        }

    def _push(self, key, value):
        # JS numbers are doubles: SPLAT_RADIUS and the aspect enter double arithmetic in
        # correctRadius (S:1457-1462) before the single fp32 narrowing of gl.uniform1f
        self._check(self._L.fluid_set_param_f64(self._h, PARAM[key], float(value)))

    def _push_config(self):
        """The reference reads `config` live inside step()/splat(); mirror that by pushing every
        changed scalar before the call."""
        for k, v in self._live_values().items():
            if self._pushed.get(k) != v:
                self._push(k, v)
                self._pushed[k] = v

    def _canvas_args(self):
        """What render(null) on the canvas hands fluid_render_canvas and fluid_render_canvas_batch: (width, height,
        the arguments from `keywords` to `back_b`).  config.SHADING / BLOOM / SUNRAYS / TRANSPARENT (the
        checkerboard) / BACK_COLOR and the post-FX sliders are read now; BLOOM needs `self.dithering`."""
        cfg = self.config
        w, h = self.canvas["width"], self.canvas["height"]
        self._push_config()                                  # the checkerboard uses canvas.width / canvas.height (S:1327)
        kw, fx, dith = postfx_inputs(cfg, getattr(self, "dithering", None))
        return w, h, (kw, 1 if cfg.get("TRANSPARENT") else 0, *_fx_args(fx, dith), *_back_rgb(cfg))

    def _capture_args(self):
        """What captureScreenshot hands fluid_capture, fluid_capture_device and fluid_capture_batch: (width, height,
        the arguments from `canvas_w` to `back_b`).  The target is getResolution(CAPTURE_RESOLUTION) of the canvas;
        config is read as in _canvas_args."""
        cfg = self.config
        cw, ch = self.canvas["width"], self.canvas["height"]
        a = capture_inputs(cfg, cw, ch, getattr(self, "dithering", None))
        return a["width"], a["height"], (cw, ch, a["keywords"], 1 if a["transparent"] else 0,
                                         *_fx_args(a["fx"], a["dither"]), *_back_rgb(cfg))

    def _dims(self, name):
        w, h, c, r0 = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        self._check(self._L.fluid_field_dims(self._h, FIELD[name], C.byref(w), C.byref(h), C.byref(c), C.byref(r0)))
        return w.value, h.value, c.value, r0.value

    def step(self, dt):
        """step(dt), S:1231-1294."""
        self._push_config()
        self._check(self._L.fluid_step(self._h, float(dt)))

    def sync(self):
        self._check(self._L.fluid_sync(self._h))

    def mark(self, slot):
        self._check(self._L.fluid_mark(self._h, slot))

    def elapsed_ms(self) -> float:
        ms = C.c_float()
        self._check(self._L.fluid_elapsed_ms(self._h, C.byref(ms)))
        return ms.value

    def timing(self) -> dict:
        t = Timing()
        self._check(self._L.fluid_timing_last(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in Timing._fields_}

    def launch_count(self) -> int:
        return int(self._L.fluid_launch_count(self._h))

    def stat(self, name) -> int:
        """Library counters (fluid_stat): launches, jacobi_launches, halo_launches, halo_exchanges,
        graph_captures, graph_launches, halo_transport_p2p, cvd_stream_launches and
        gradient_stream_launches (how many curl-vorticity-divergence / gradientSubtract passes ran
        the row-streaming kernel rather than the tiled one; graph replays included), and
        jacobi_exact_streams (warps of the blocked Jacobi kernel that ran the un-contracted tail, for
        tiny divergence or inputs near FLT_MAX; waits for the handle's queued work)."""
        return int(self._L.fluid_stat(self._h, STAT[name]))

    def device_ptr(self, name) -> int:
        return int(self._L.fluid_device_ptr(self._h, FIELD[name]) or 0)

    def set_param(self, key, value):
        self._check(self._L.fluid_set_param(self._h, PARAM[key], float(value)))

    def close(self):
        if self._h:
            self._L.fluid_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class FluidSimulation(_Handle):
    """The reference's simulation state and frame functions on one handle.  `flags` pick the device the
    reference runs on: FLAG_NEAREST_FILTERING is a device without float linear filtering (NEAREST display /
    post-FX / resize samplers, with its config override); FLAG_LINEAR_ADVECTION is a device with it, whose
    step() advects through LINEAR samplers (the advectionShader's #else branch, S:776-779) instead of the
    MANUAL_FILTERING bilerp every other handle runs.  FLAG_HALF_STORAGE | FLAG_HALF_POSTFX |
    FLAG_LINEAR_ADVECTION is the desktop browser's frame and step.  LINEAR_ADVECTION is single-GPU and
    refused with NEAREST_FILTERING; it adds no config override (the reference has none)."""

    def __init__(self, config: dict | None = None, canvas_width: int = 1024, canvas_height: int = 1024,
                 device: int = -1, flags: int = 0, jacobi_block: int = 0, random=None,
                 rank: int = 0, world: int = 1, nccl_uid: bytes | None = None,
                 sizes: tuple | None = None):
        self.config = default_config(flags)          # the caller's keys win, as later GUI edits do
        if config:
            self.config.update(config)
        self.canvas = {"width": int(canvas_width), "height": int(canvas_height)}
        self.random = random or _random.random          # Math.random stand-in (injectable, seedable)
        self.pointers = [Pointer()]                     # S:100-102
        self.splatStack = []
        self.lastUpdateTime = time.time() * 1000.0      # S:1172
        self.colorUpdateTimer = 0.0
        self._L = _lib.lib()
        self._h = C.c_void_p()
        self._device, self._flags, self._jb = device, flags, jacobi_block
        self._rank, self._world, self._uid = rank, world, nccl_uid
        # test hook: explicit (sim_w, sim_h, dye_w, dye_h) instead of getResolution(config.*)
        self._sizes = sizes
        self._pushed = {}
        self.velocity = _Field(self, "velocity")
        self.dye = _Field(self, "dye")
        self.pressure = _Field(self, "pressure")
        self.divergence = _Field(self, "divergence")
        self.curl = _Field(self, "curl")
        self.initFramebuffers()

    # ---- initFramebuffers, S:982-1010 --------------------------------------------------------------
    def initFramebuffers(self):
        simRes = getResolution(self.config["SIM_RESOLUTION"], self.canvas["width"], self.canvas["height"])
        dyeRes = getResolution(self.config["DYE_RESOLUTION"], self.canvas["width"], self.canvas["height"])
        if self._sizes is not None:
            simRes = {"width": self._sizes[0], "height": self._sizes[1]}
            dyeRes = {"width": self._sizes[2], "height": self._sizes[3]}
        if not self._h:                                  # `dye == null` branch: create
            cfg = self._config(simRes["width"], simRes["height"], dyeRes["width"], dyeRes["height"])
            if self._world > 1:
                uid = C.create_string_buffer(self._uid, len(self._uid))
                self._check(self._L.fluid_create_slab(C.byref(cfg), self._rank, self._world, uid,
                                                      len(self._uid), C.byref(self._h)))
            else:
                self._check(self._L.fluid_create(C.byref(cfg), C.byref(self._h)))
        else:                                            # resizeDoubleFBO branch, S:1116-1126
            self._check(self._L.fluid_resize(self._h, simRes["width"], simRes["height"],
                                             dyeRes["width"], dyeRes["height"]))
            if self._world > 1 and getattr(self, "halo_transport", "nccl") == "p2p":
                # the peer mappings died with the old arena: export / connect again (collective)
                from .distributed import connect_peers
                self.halo_transport = "p2p" if connect_peers(self) else "nccl"
        self._pushed = {}
        self._push_config()

    # ---- the hot path (step(dt): _Handle) ------------------------------------------------------------
    def splat(self, x, y, dx, dy, color):
        """splat(x, y, dx, dy, color), S:1441-1455; color is {r,g,b} like the reference's."""
        self._push_config()
        if isinstance(color, dict):
            r, g, b = color["r"], color["g"], color["b"]
        else:
            r, g, b = color
        self._check(self._L.fluid_splat(self._h, float(x), float(y), float(dx), float(dy),
                                        float(r), float(g), float(b)))

    def splats(self, records):
        """len(records) splat() calls in one: records is (n, 7) of (x, y, dx, dy, r, g, b), applied in
        order with the same bits as one splat() per row, in ceil(n/128) launches.  `records` may also be a
        C-contiguous (n, 7) float32 CUDA array on the handle's device (anything with __cuda_array_interface__,
        e.g. a torch tensor): the records are read on the GPU in one launch (fluid_splats_device), with the same
        bits and no host copy, after the waits of writeField."""
        if hasattr(records, "__cuda_array_interface__"):
            n = _records_rows(records)
            src = _device_array(records, "<f4", 7 * n, "splats")
            self._push_config()
            self._check(self._L.fluid_splats_device(self._h, src, n))
            self.sync()
            return
        a = np.asarray(records)
        if a.ndim != 2 or a.shape[1] != 7:
            raise ValueError(f"splats() takes an (n, 7) array of (x, y, dx, dy, r, g, b), got shape {a.shape}")
        a = np.ascontiguousarray(a, np.float32)        # round to nearest, as c_float does per argument
        self._push_config()
        self._check(self._L.fluid_splats(self._h, a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0]))

    def splatPointer(self, pointer):
        """S:1421-1425."""
        dx = pointer.deltaX * self.config["SPLAT_FORCE"]
        dy = pointer.deltaY * self.config["SPLAT_FORCE"]
        self.splat(pointer.texcoordX, pointer.texcoordY, dx, dy, pointer.color)

    def multipleSplats(self, amount):
        """S:1427-1439 (same draw order from the random stream as the reference)."""
        for _ in range(int(amount)):
            color = self.generateColor()
            color["r"] *= 10.0
            color["g"] *= 10.0
            color["b"] *= 10.0
            x = self.random()
            y = self.random()
            dx = 1000 * (self.random() - 0.5)
            dy = 1000 * (self.random() - 0.5)
            self.splat(x, y, dx, dy, color)

    def generateColor(self):
        """S:1565-1571."""
        c = HSVtoRGB(self.random(), 1.0, 1.0)
        c["r"] *= 0.15
        c["g"] *= 0.15
        c["b"] *= 0.15
        return c

    # ---- frame driver (the caller of the hot path), S:1176-1229 --------------------------------------
    def calcDeltaTime(self, now_ms=None):
        """S:1188-1194: dt = min(wall delta, 0.016666)."""
        now = time.time() * 1000.0 if now_ms is None else now_ms
        dt = (now - self.lastUpdateTime) / 1000.0
        dt = min(dt, 0.016666)
        self.lastUpdateTime = now
        return dt

    def updateColors(self, dt):
        """S:1207-1217."""
        if not self.config["COLORFUL"]:
            return
        self.colorUpdateTimer += dt * self.config["COLOR_UPDATE_SPEED"]
        if self.colorUpdateTimer >= 1:
            self.colorUpdateTimer = wrap(self.colorUpdateTimer, 0, 1)
            for p in self.pointers:
                p.color = self.generateColor()

    def applyInputs(self):
        """S:1219-1229."""
        if self.splatStack:
            self.multipleSplats(self.splatStack.pop())
        for p in self.pointers:
            if p.moved:
                p.moved = False
                self.splatPointer(p)

    def update(self, now_ms=None, canvas=None):
        """One iteration of update(), S:1176-1186, minus rAF.  With `canvas` (a destination render_canvas
        takes as `out`) it ends with render_canvas(out=canvas), as the reference's ends with render(null);
        without it nothing is drawn."""
        dt = self.calcDeltaTime(now_ms)
        self.updateColors(dt)
        self.applyInputs()
        if not self.config["PAUSED"]:
            self.step(dt)
        if canvas is not None:
            self.render_canvas(out=canvas)
        return dt

    # pointer helpers, S:1527-1563
    def updatePointerDownData(self, pointer, id_, posX, posY):
        pointer.id = id_
        pointer.down = True
        pointer.moved = False
        pointer.texcoordX = posX / self.canvas["width"]
        pointer.texcoordY = 1.0 - posY / self.canvas["height"]
        pointer.prevTexcoordX = pointer.texcoordX
        pointer.prevTexcoordY = pointer.texcoordY
        pointer.deltaX = 0
        pointer.deltaY = 0
        pointer.color = self.generateColor()

    def updatePointerMoveData(self, pointer, posX, posY):
        pointer.prevTexcoordX = pointer.texcoordX
        pointer.prevTexcoordY = pointer.texcoordY
        pointer.texcoordX = posX / self.canvas["width"]
        pointer.texcoordY = 1.0 - posY / self.canvas["height"]
        pointer.deltaX = self.correctDeltaX(pointer.texcoordX - pointer.prevTexcoordX)
        pointer.deltaY = self.correctDeltaY(pointer.texcoordY - pointer.prevTexcoordY)
        pointer.moved = abs(pointer.deltaX) > 0 or abs(pointer.deltaY) > 0

    def correctDeltaX(self, delta):
        a = self._aspect()
        return delta * a if a < 1 else delta

    def correctDeltaY(self, delta):
        a = self._aspect()
        return delta / a if a > 1 else delta

    # ---- data access (the reference hands textures to GL; a host mirror hands arrays) ----------------
    def readField(self, name, out: np.ndarray | None = None) -> np.ndarray:
        """framebufferToTexture (S:301-307) generalised: rows x width [x channels] float32, row 0 =
        bottom.  On a slab rank: the rows this rank owns.  `out`: a caller-owned float32 buffer of
        the right size (e.g. pinned host memory) to read into instead of allocating, or a C-contiguous
        float32 CUDA array on the handle's device (anything with __cuda_array_interface__, e.g. a torch
        tensor) of exactly that many elements: the field is copied (widened, in half storage) on the GPU,
        with no host copy, and the array is returned as it was passed.  The waits are render_canvas's:
        pending work that may use the array first, the handle's stream before returning."""
        w, h, c, _ = self._dims(name)
        n = w * h * c
        dst = _device_array(out, "<f4", n, "readField")
        if dst is not None:
            self._check(self._L.fluid_read_device(self._h, FIELD[name], dst, n))
            self.sync()
            return out
        shape = (h, w, c) if c > 1 else (h, w)
        if out is None:
            out = np.empty(shape, np.float32)
        else:
            assert out.dtype == np.float32 and out.flags.c_contiguous and out.size == n
            out = out.reshape(shape)
        self._check(self._L.fluid_read(self._h, FIELD[name], out.ctypes.data_as(C.c_void_p), out.size))
        return out

    def writeField(self, name, array):
        """Overwrites a field with `array` (rows x width [x channels], row 0 = bottom): anything numpy turns
        into float32, or a C-contiguous float32 CUDA array of exactly the field's element count, copied
        (narrowed, in half storage) on the GPU with render_canvas's waits."""
        if hasattr(array, "__cuda_array_interface__"):
            w, h, c, _ = self._dims(name)
            src = _device_array(array, "<f4", w * h * c, "writeField")
            self._check(self._L.fluid_write_device(self._h, FIELD[name], src, w * h * c))
            self.sync()
            return
        a = np.ascontiguousarray(array, np.float32)
        self._check(self._L.fluid_write(self._h, FIELD[name], a.ctypes.data_as(C.c_void_p), a.size))

    def render(self, width=None, height=None, target=False) -> np.ndarray:
        """render(target), S:1296-1317: (height, width, 4) float32 RGBA, row 0 = bottom.  Defaults
        to the canvas size (target == null branch, S:1332-1333).  config.TRANSPARENT: the display is
        drawn over the checkerboard on the screen (target=False, S:1311-1312) and bare, un-blended,
        into a capture target (target=True: what captureScreenshot renders into, S:287-299).
        config.SHADING / BLOOM / SUNRAYS pick the display keywords like updateKeywords (S:1160-1166);
        BLOOM needs `sim.dithering`.  BLOOM or SUNRAYS need an fp32 handle or one created with
        FLAG_HALF_POSTFX (then the bloom and sunrays targets are fp16, as are the reference's; with
        FLAG_HALF_STORAGE | FLAG_HALF_POSTFX this is the reference's desktop frame; FLAG_LINEAR_ADVECTION
        changes how step() advects, not how a frame is drawn).  last_bloom /
        last_sunrays hold the bloom FBO / sunrays texture of the frame (widened to float32), or None when
        that keyword is off.
        On a slab rank: the rank's band of the target, rows render_band = (y0, y1) (fluid_render_band), for
        every keyword set; bands concatenate in rank order.  With BLOOM or SUNRAYS every rank must call with
        the same arguments (the ranks gather the post-FX inputs), and last_bloom / last_sunrays are whole."""
        w = int(width or self.canvas["width"]); h = int(height or self.canvas["height"])
        bc = self.config["BACK_COLOR"]                       # normalizeColor, S:1599-1606
        out = np.empty((h, w, 4), np.float32)
        cfg = self.config
        bg = 0 if not cfg.get("TRANSPARENT") else (2 if target else 1)
        if self._pushed.get("BACKGROUND") != bg:
            self._check(self._L.fluid_set_param(self._h, PARAM["BACKGROUND"], float(bg)))
            self._pushed["BACKGROUND"] = bg
        self._push_config()                                  # the checkerboard uses canvas.width / canvas.height (S:1327)
        kw, fx, dith = postfx_inputs(cfg, getattr(self, "dithering", None))
        self.last_bloom = self.last_sunrays = None           # the bloom FBO / sunrays texture of this frame, if drawn
        if kw & DISPLAY_BLOOM:
            b = getResolution(cfg["BLOOM_RESOLUTION"], w, h)
            self.last_bloom = np.empty((b["height"], b["width"], 4), np.float32)
        if kw & DISPLAY_SUNRAYS:
            sr = getResolution(cfg["SUNRAYS_RESOLUTION"], w, h)
            self.last_sunrays = np.empty((sr["height"], sr["width"]), np.float32)
        y0, y1 = self._band(h)                               # a slab rank draws its band of the target only
        out = out[: y1 - y0]
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)   # noqa: E731
        self._check(self._L.fluid_render_keywords(
            self._h, w, h, kw, None if fx is None else C.byref(fx), ptr(dith),
            0 if dith is None else dith.shape[1], 0 if dith is None else dith.shape[0],
            bc["r"] / 255, bc["g"] / 255, bc["b"] / 255, ptr(out), out.size, ptr(self.last_bloom), ptr(self.last_sunrays)))
        return out

    def captureScreenshot(self, path=None, out=None) -> np.ndarray:
        """captureScreenshot(), S:287-299: render() into an RGBA half-float target of
        getResolution(CAPTURE_RESOLUTION) and normalizeTexture (S:309-327), all on the GPU.  Returns the
        (h, w, 4) uint8 image, TOP row first.  The bloom and sunrays FBOs keep the canvas sizes, as in the
        reference; config.TRANSPARENT stores the display bare (no checkerboard); BLOOM needs `sim.dithering`.
        BLOOM or SUNRAYS need the same handles as render().
        With `path`, also writes the image as a PNG (write_png: the bytes unchanged).
        `out`: a C-contiguous uint8 CUDA array on the handle's device of exactly 4 * w * h bytes (e.g. a torch
        tensor): the display kernel stores the image into it, with no host copy and render_canvas's waits, and
        the array is returned as it was passed.  A PNG needs host bytes, so `path` with `out` is refused.
        On a slab rank: the rank's band, (y1 - y0, w, 4) top row first, rows render_band = (y0, y1) of the
        bottom-up target; the whole image is the bands in reverse rank order (distributed.gather_image).  A PNG
        needs the whole image, so `path` is refused there."""
        w, h, args = self._capture_args()
        if out is not None:
            if not hasattr(out, "__cuda_array_interface__"):
                raise ValueError("captureScreenshot(out=...) takes a CUDA array; without `out` it returns a numpy image")
            if path is not None:
                raise ValueError("captureScreenshot writes a PNG from host bytes: pass `path` or a CUDA `out`, not both")
        if path is not None and self._world > 1:
            raise ValueError("captureScreenshot(path=...) needs the whole image: a slab rank draws only its band "
                             "(gather the bands with distributed.gather_image and write_png them)")
        y0, y1 = self._band(h)
        n = 4 * w * (y1 - y0)
        dst = _device_array(out, "|u1", n, "captureScreenshot")
        img = np.empty((y1 - y0, w, 4), np.uint8) if dst is None else None
        self._check((self._L.fluid_capture if dst is None else self._L.fluid_capture_device)(
            self._h, w, h, *args, img.ctypes.data_as(C.c_void_p) if dst is None else dst, n))
        if dst is not None:
            self.sync()
            return out
        if path is not None:
            write_png(path, img)
        return img

    def render_canvas(self, out=None):
        """render(null), S:1296-1317, on the canvas: canvas.width x canvas.height RGBA8, the bytes the
        drawing buffer holds after the frame (fluid_render_canvas in include/fluid.h states the rule:
        source and blend factors clamped, destination quantised, round to nearest even).  config.SHADING /
        BLOOM / SUNRAYS / TRANSPARENT (the checkerboard) / BACK_COLOR as in render(); BLOOM needs
        `sim.dithering`.  Returns the (height, width, 4) uint8 image, top row first (ImageData order).
        `out`: a C-contiguous uint8 numpy array of 4 * width * height bytes, or a C-contiguous uint8 CUDA
        array on the handle's device, 4-byte aligned (anything with __cuda_array_interface__, e.g. a torch
        tensor).  The display kernel writes a CUDA array directly, with no copy to the host.  The handle's
        stream does not order against other streams, so the call first waits for the work that may still
        use the array: the producer stream a version-3 interface names, or, where the interface names none
        (torch's is version 2), every queued kernel and copy of the array's device.  The handle's stream is
        synchronised before returning, so the array can be read at once.  A CUDA array is returned as it
        was passed.
        On a slab rank: the rank's band, (y1 - y0, width, 4) top row first, rows render_band = (y0, y1) of the
        bottom-up canvas; the whole canvas is the bands in reverse rank order (distributed.gather_image), and
        `out` holds the band.  With BLOOM or SUNRAYS every rank must call with the same config."""
        w, h, args = self._canvas_args()
        y0, y1 = self._band(h)
        dst, result, on_device = _u8_destination(out, (y1 - y0, w, 4), "render_canvas")
        self._check(self._L.fluid_render_canvas(self._h, w, h, *args, dst, 4 * w * (y1 - y0), 1 if on_device else 0))
        if on_device:
            self.sync()
        return result

    def _band(self, height):
        """(y0, y1): the rows of a `height`-row target this handle draws (fluid_render_band; all of them on one
        GPU), also kept as render_band."""
        y0, y1 = C.c_int(), C.c_int()
        self._check(self._L.fluid_render_band(self._h, int(height), C.byref(y0), C.byref(y1)))
        self.render_band = (y0.value, y1.value)
        return self.render_band

    @staticmethod
    def textureToCanvas(rgba: np.ndarray) -> np.ndarray:
        """normalizeTexture + textureToCanvas (S:309-349): clamp01 * 255 truncated into a Uint8
        image, flipped so that row 0 is the TOP (canvas order)."""
        img = (np.clip(rgba, 0.0, 1.0) * 255.0).astype(np.uint8)
        return img[::-1].copy()

    # ---- per-pass entry points (test surface; one reference blit each) -------------------------------
    def pass_(self, name, *args):
        self._push_config()
        fn = getattr(self._L, "fluid_pass_" + name)
        conv = [C.c_int(int(a)) if name == "jacobi" else C.c_float(float(a)) for a in args]
        self._check(fn(self._h, *conv))

    def pressure_solve_host(self, div_host: np.ndarray, p_host: np.ndarray, iters: int):
        assert div_host.dtype == np.float32 and p_host.dtype == np.float32
        self._push_config()
        self._check(self._L.fluid_pressure_solve_host(self._h, div_host.ctypes.data_as(C.c_void_p),
                                                      p_host.ctypes.data_as(C.c_void_p), int(iters)))



class FluidBatch(_Handle):
    """`members` independent simulations of one size and config in one handle (fluid_create_batch): step(),
    splats(), readField() and writeField() act on all of them through the same kernel launches, and member m
    holds the bits a FluidSimulation given member m's inputs would hold.  Sizes come from `sizes` (sim_w,
    sim_h, dye_w, dye_h) or from getResolution of config SIM_RESOLUTION / DYE_RESOLUTION on the canvas; they
    must be powers of two with widths >= 128 and heights >= 2.  `config` is read live before each call and
    applies to every member, except that `member_config[m]` (a dict per member, empty at creation) overrides the
    MEMBER_KEYS for member m: a parameter sweep.  step() takes one dt, or one per member.  flags: FLAG_NO_GRAPH or
    0.  render_canvas() and captureScreenshot() draw every member through one set of launches; render(), resize and
    the per-pass entry points are FluidSimulation's only.  readField(), writeField(), render_canvas() and
    captureScreenshot() take `members=`, a host list of distinct member indices, to act on those members only, and
    reset(members) puts members back to their state at creation.  `member_config[m]` may also override the
    DISPLAY_MEMBER_KEYS: render_canvas() and captureScreenshot() then draw member m with its own post-FX sliders and
    background, still through one set of launches."""

    # the config keys a member can hold a value of its own for (fluid_set_param_members)
    MEMBER_KEYS = ("DENSITY_DISSIPATION", "VELOCITY_DISSIPATION", "PRESSURE", "CURL", "SPLAT_RADIUS")
    # the config keys of a member's look in render_canvas() and captureScreenshot() (fluid_render_canvas_looks,
    # fluid_capture_looks): the post-FX sliders and the background
    DISPLAY_MEMBER_KEYS = ("BLOOM_INTENSITY", "BLOOM_THRESHOLD", "BLOOM_SOFT_KNEE", "SUNRAYS_WEIGHT", "BACK_COLOR",
                           "TRANSPARENT")

    def __init__(self, members: int, config: dict | None = None, canvas_width: int = 1024, canvas_height: int = 1024,
                 sizes: tuple | None = None, flags: int = 0, jacobi_block: int = 0, device: int = -1):
        self.config = default_config(flags)
        if config:
            self.config.update(config)
        self.canvas = {"width": int(canvas_width), "height": int(canvas_height)}
        self._L = _lib.lib()
        self._h = C.c_void_p()
        self._device, self._flags, self._jb = device, flags, jacobi_block
        self._pushed = {}
        if sizes is None:
            sim = getResolution(self.config["SIM_RESOLUTION"], canvas_width, canvas_height)
            dye = getResolution(self.config["DYE_RESOLUTION"], canvas_width, canvas_height)
            sizes = (sim["width"], sim["height"], dye["width"], dye["height"])
        self._check(self._L.fluid_create_batch(C.byref(self._config(*sizes)), int(members), C.byref(self._h)))
        self.member_config = [{} for _ in range(self.members)]
        self._push_config()

    @property
    def members(self) -> int:
        return int(self._L.fluid_members(self._h))

    def _check_member_config(self):
        """ValueError unless member_config holds one dict per member, each overriding MEMBER_KEYS and
        DISPLAY_MEMBER_KEYS only."""
        B = self.members
        if len(self.member_config) != B:
            raise ValueError(f"member_config holds {len(self.member_config)} dicts for {B} members")
        keys = self.MEMBER_KEYS + self.DISPLAY_MEMBER_KEYS
        for m, over in enumerate(self.member_config):
            bad = sorted(set(over) - set(keys))
            if bad:
                raise ValueError(f"member_config[{m}] sets {bad}: only {list(keys)} can differ between members")

    def _live_values(self):
        """A MEMBER_KEYS value is the float64 vector of every member's value, `member_config` over `config`."""
        self._check_member_config()
        vals = super()._live_values()
        for k in self.MEMBER_KEYS:
            vec = np.array([float(over.get(k, self.config[k])) for over in self.member_config], np.float64)
            vals[k] = vec.tobytes()                       # compared bit for bit: -0.0 is not 0.0
        return vals

    def _push(self, key, value):
        if key not in self.MEMBER_KEYS:
            return super()._push(key, value)
        vec = np.frombuffer(value, np.float64)
        bits = vec.view(np.int64)
        if (bits == bits[0]).all():                       # one value for every member: as a FluidSimulation pushes it
            return super()._push(key, vec[0])
        self._check(self._L.fluid_set_param_members(self._h, PARAM[key], vec.ctypes.data_as(C.POINTER(C.c_double)),
                                                     vec.size))

    def member_params(self, key):
        """The B values of a MEMBER_KEYS key the handle holds, float32, as FluidSimulation's get_param would
        return them (fluid_get_param_members)."""
        out = np.empty(self.members, np.float32)
        self._check(self._L.fluid_get_param_members(self._h, PARAM[key], out.ctypes.data_as(C.POINTER(C.c_float)),
                                                    out.size))
        return out

    def step(self, dt):
        """step(dt) of every member: one number for all of them, or a sequence of B numbers, dt[m] for member m."""
        if np.ndim(dt) == 0:
            return super().step(dt)
        d = np.ascontiguousarray(dt, np.float32)
        if d.ndim != 1 or d.size != self.members:
            raise ValueError(f"step() takes one dt or {self.members} of them, got shape {d.shape}")
        self._push_config()
        self._check(self._L.fluid_step_members(self._h, d.ctypes.data_as(C.POINTER(C.c_float)), d.size))

    def splats(self, members, records):
        """Row k of records ((n, 7): x, y, dx, dy, r, g, b) splatted into member members[k]; each member takes
        its rows in order, with the bits of FluidSimulation.splats, and members named by no row are untouched.
        Both may instead be CUDA arrays on the handle's device (an int32 vector of n and a C-contiguous (n, 7)
        float32 array): the records are grouped and applied on the GPU in two launches (fluid_splats_batch_device),
        with the same bits and no host copy, after the waits of writeField.  One on the host and the other on the
        device is a ValueError.  A member index outside [0, B) in a CUDA array makes the call splat nothing and is
        reported by the sync that ends it (FluidError)."""
        dev_m, dev_r = hasattr(members, "__cuda_array_interface__"), hasattr(records, "__cuda_array_interface__")
        if dev_m != dev_r:
            raise ValueError("splats() takes members and records both in host memory or both as CUDA arrays")
        if dev_m:
            n = _records_rows(records)
            mem = _device_array(members, "<i4", n, "splats")
            src = _device_array(records, "<f4", 7 * n, "splats")
            self._push_config()
            self._check(self._L.fluid_splats_batch_device(self._h, mem, src, n))
            self.sync()
            return
        m = np.ascontiguousarray(members, np.int32).reshape(-1)
        a = np.asarray(records)
        if a.ndim != 2 or a.shape[1] != 7 or a.shape[0] != m.size:
            raise ValueError(f"splats() takes n member indices and an (n, 7) array, got {m.size} and {a.shape}")
        a = np.ascontiguousarray(a, np.float32)
        self._push_config()
        self._check(self._L.fluid_splats_batch(self._h, m.ctypes.data_as(C.POINTER(C.c_int32)),
                                               a.ctypes.data_as(C.POINTER(C.c_float)), m.size))

    def _shape(self, name, n=None):
        """(n, H, W[, C]) of a field: n images, B of them when n is None."""
        w, h, c, _ = self._dims(name)
        n = self.members if n is None else n
        return (n, h, w, c) if c > 1 else (n, h, w)

    @staticmethod
    def _member_list(members):
        """`members` (a sequence or numpy array of member indices, or None) as a C-contiguous int32 vector and its
        ctypes pointer; (None, None) for None.  Member lists live on the host: a CUDA array is a ValueError.  The
        library checks the indices (distinct, in [0, B))."""
        if members is None:
            return None, None
        if hasattr(members, "__cuda_array_interface__"):
            raise ValueError("members must be a host sequence or numpy array of member indices, not a CUDA array")
        a = np.asarray(members)
        if a.ndim != 1 or (a.size and not np.issubdtype(a.dtype, np.integer)):
            raise ValueError(f"members must be a 1-D list of integer member indices, got {a.dtype} {a.shape}")
        m = np.ascontiguousarray(a, np.int32)
        if not np.array_equal(m, a):
            raise ValueError("members holds an index outside the int32 range")
        return m, m.ctypes.data_as(C.POINTER(C.c_int32))

    def readField(self, name, out=None, members=None) -> np.ndarray:
        """(B, H, W[, C]) float32, member by member, row 0 = bottom.  `out` as FluidSimulation.readField: a
        float32 host buffer of that size, or a C-contiguous float32 CUDA array of that many elements, filled on
        the GPU and returned as passed.  members: (n, H, W[, C]) of the listed members only, slot k member
        members[k] (fluid_read_members)."""
        m, mp = self._member_list(members)
        shape = self._shape(name, None if m is None else m.size)
        n = int(np.prod(shape))
        dst = _device_array(out, "<f4", n, "readField")
        if dst is not None:
            if m is None:
                self._check(self._L.fluid_read_device(self._h, FIELD[name], dst, n))
            else:
                self._check(self._L.fluid_read_members(self._h, FIELD[name], mp, m.size, dst, n, 1))
            self.sync()
            return out
        if out is None:
            out = np.empty(shape, np.float32)
        else:
            assert out.dtype == np.float32 and out.flags.c_contiguous and out.size == n
            out = out.reshape(shape)
        if m is None:
            self._check(self._L.fluid_read(self._h, FIELD[name], out.ctypes.data_as(C.c_void_p), out.size))
        else:
            self._check(self._L.fluid_read_members(self._h, FIELD[name], mp, m.size, out.ctypes.data_as(C.c_void_p),
                                                   out.size, 0))
        return out

    def writeField(self, name, array, members=None):
        """Overwrites a field of every member with `array` ((B, H, W[, C])): anything numpy turns into float32,
        or a C-contiguous float32 CUDA array of exactly that many elements.  members: only the listed members,
        `array` then (n, H, W[, C]) with slot k for member members[k] (fluid_write_members); the others keep
        every bit."""
        m, mp = self._member_list(members)
        n = int(np.prod(self._shape(name, None if m is None else m.size)))
        if hasattr(array, "__cuda_array_interface__"):
            src = _device_array(array, "<f4", n, "writeField")
            if m is None:
                self._check(self._L.fluid_write_device(self._h, FIELD[name], src, n))
            else:
                self._check(self._L.fluid_write_members(self._h, FIELD[name], mp, m.size, src, n, 1))
            self.sync()
            return
        a = np.ascontiguousarray(array, np.float32)
        if m is None:
            self._check(self._L.fluid_write(self._h, FIELD[name], a.ctypes.data_as(C.c_void_p), a.size))
        else:
            self._check(self._L.fluid_write_members(self._h, FIELD[name], mp, m.size, a.ctypes.data_as(C.c_void_p),
                                                    a.size, 0))

    def reset(self, members):
        """The listed members back to their state at creation: every field zero, dye alpha 1, in one launch
        (fluid_reset_members).  member_config is config and stays."""
        m, mp = self._member_list(members)
        if m is None:
            raise ValueError("reset() takes a list of member indices")
        self._check(self._L.fluid_reset_members(self._h, mp, m.size))

    def _looks(self, m):
        """None when no member overrides a DISPLAY_MEMBER_KEYS key: the draw takes one look from `config`.  Otherwise
        the fluid_look of each image, `member_config` over `config`: member k's for image k, or member m[k]'s for a
        member list m (an index outside [0, B) gets `config`'s look; the library refuses the list)."""
        self._check_member_config()
        if not any(k in over for over in self.member_config for k in self.DISPLAY_MEMBER_KEYS):
            return None
        B = self.members
        idx = range(B) if m is None else m.tolist()
        looks = (_lib.Look * len(idx))()
        for k, i in enumerate(idx):
            c = {**self.config, **(self.member_config[i] if 0 <= i < B else {})}
            looks[k] = _lib.Look(float(c["BLOOM_INTENSITY"]), float(c["BLOOM_THRESHOLD"]), float(c["BLOOM_SOFT_KNEE"]),
                                 float(c["SUNRAYS_WEIGHT"]), *_back_rgb(c), 1 if c.get("TRANSPARENT") else 0)
        return looks

    def _draw(self, fn_all, fn_members, fn_looks, what, w, h, args, look_args, out, members):
        """A whole-batch draw, or with `members` the draw of the listed members only, image k member members[k].
        When a member overrides a DISPLAY_MEMBER_KEYS key, fn_looks draws every image with its member's look; its
        arguments `look_args` are `args` without transparent and back_*."""
        m, mp = self._member_list(members)
        n = self.members if m is None else m.size
        looks = self._looks(m)
        dst, result, on_device = _u8_destination(out, (n, h, w, 4), what)
        tail = (dst, 4 * w * h * n, 1 if on_device else 0)
        if looks is not None:
            self._check(fn_looks(self._h, w, h, *look_args, looks, *tail, mp, n))
        else:
            self._check(fn_all(self._h, w, h, *args, *tail) if m is None else
                        fn_members(self._h, w, h, *args, *tail, mp, n))
        if on_device:
            self.sync()
        return result

    def render_canvas(self, out=None, members=None):
        """FluidSimulation.render_canvas for every member (fluid_render_canvas_batch): (B, canvas height, canvas
        width, 4) uint8, member by member, member m's image the bytes a FluidSimulation of this config and canvas
        draws from member m's dye.  Config, canvas and `self.dithering` as there.  `out`: a C-contiguous uint8 numpy
        array of that many bytes, or a C-contiguous uint8 CUDA array of them with render_canvas's waits, returned
        as it was passed.  members: the listed members' images only, (n, h, w, 4), image k member members[k]
        (fluid_render_canvas_members).  A member's DISPLAY_MEMBER_KEYS overrides give its image that member's
        sliders and background (fluid_render_canvas_looks)."""
        w, h, args = self._canvas_args()
        look_args = (args[0], *args[2:6])                    # keywords, fx, dither_rgb, dw, dh
        return self._draw(self._L.fluid_render_canvas_batch, self._L.fluid_render_canvas_members,
                          self._L.fluid_render_canvas_looks, "render_canvas", w, h, args, look_args, out, members)

    def captureScreenshot(self, out=None, members=None):
        """FluidSimulation.captureScreenshot for every member (fluid_capture_batch): (B, h, w, 4) uint8 at
        getResolution(CAPTURE_RESOLUTION) of the canvas, member by member, each top row first.  No PNG is written.
        `out`, `members` and the DISPLAY_MEMBER_KEYS overrides as in render_canvas (fluid_capture_members,
        fluid_capture_looks)."""
        w, h, args = self._capture_args()
        look_args = (*args[:3], *args[4:8])                  # canvas_w, canvas_h, keywords, fx, dither_rgb, dw, dh
        return self._draw(self._L.fluid_capture_batch, self._L.fluid_capture_members, self._L.fluid_capture_looks,
                          "captureScreenshot", w, h, args, look_args, out, members)


def _fx_args(fx, dith):
    """fx, dither_rgb, dw and dh of the draw calls, from the PostFX and dithering texture of postfx_inputs."""
    return (None if fx is None else C.byref(fx), None if dith is None else dith.ctypes.data_as(C.c_void_p),
            0 if dith is None else dith.shape[1], 0 if dith is None else dith.shape[0])


def _back_rgb(cfg):
    """back_r, back_g, back_b of the draw calls: normalizeColor(BACK_COLOR), S:1599-1606."""
    bc = cfg["BACK_COLOR"]
    return bc["r"] / 255, bc["g"] / 255, bc["b"] / 255


def _u8_destination(out, shape, what):
    """Where an 8-bit draw of `shape` goes: (dst pointer, the array to return, on_device).  `out` is None (a new
    numpy array), a C-contiguous uint8 numpy array of that many bytes (returned reshaped), or a C-contiguous
    uint8 CUDA array of them (waited for by _device_array, returned as passed)."""
    n = int(np.prod(shape))
    dst = _device_array(out, "|u1", n, what)
    if dst is not None:
        return dst, out, True
    if out is None:
        out = np.empty(shape, np.uint8)
    if not isinstance(out, np.ndarray) or out.dtype != np.uint8 or not out.flags.c_contiguous or out.size != n:
        raise ValueError(f"{what} needs a C-contiguous uint8 array of {n} bytes")
    return out.ctypes.data_as(C.c_void_p), out.reshape(shape), False


def _records_rows(records):
    """n of a CUDA array of splat records, which must have shape (n, 7)."""
    shape = tuple(records.__cuda_array_interface__["shape"])
    if len(shape) != 2 or shape[1] != 7:
        raise ValueError(f"splats() takes an (n, 7) array of (x, y, dx, dy, r, g, b), got shape {shape}")
    return int(shape[0])


_cuda = None
_TYPES = {"|u1": "uint8", "<i4": "int32", "<f4": "float32"}


def _device_array(a, typestr, n, what):
    """None unless `a` has __cuda_array_interface__.  For a CUDA array: ValueError unless it is C-contiguous
    with n elements of `typestr`; then, once _wait_for_users has returned, its device pointer."""
    cai = getattr(a, "__cuda_array_interface__", None)
    if cai is None:
        return None
    shape, strides = tuple(cai["shape"]), cai.get("strides")
    item = np.dtype(typestr).itemsize
    dense = strides is None or tuple(strides) == tuple(item * int(np.prod(shape[k + 1:])) for k in range(len(shape)))
    if cai["typestr"] != typestr or int(np.prod(shape)) != n or not dense:
        unit = "bytes" if item == 1 else "elements"
        raise ValueError(f"{what} needs a C-contiguous {_TYPES[typestr]} CUDA array of {n} {unit}, got "
                         f"{cai['typestr']} {shape} strides {strides}")
    _wait_for_users(cai)
    return C.c_void_p(cai["data"][0])


def _wait_for_users(cai):
    """Blocks until no queued GPU work can still read or write the CUDA array whose
    __cuda_array_interface__ is `cai`, so a kernel on the handle's non-blocking stream may overwrite it.
    A version-3 interface names the producer's stream ("stream": None means nothing is pending; 1 and 2
    are the legacy and per-thread default streams, which the driver API takes as handles): that stream is
    synchronised.  Without the key (version 2, torch's) the array's device is synchronised, every stream.
    A pointer the driver does not know is left alone: the library refuses it."""
    global _cuda
    if "stream" in cai and cai["stream"] is None:
        return
    if _cuda is None:
        L = C.CDLL("libcuda.so.1")
        L.cuPointerGetAttribute.argtypes = [C.c_void_p, C.c_int, C.c_uint64]
        L.cuCtxPushCurrent_v2.argtypes = [C.c_void_p]
        L.cuCtxPopCurrent_v2.argtypes = [C.POINTER(C.c_void_p)]
        L.cuStreamSynchronize.argtypes = [C.c_void_p]
        _cuda = L
    ctx = C.c_void_p()
    CU_POINTER_ATTRIBUTE_CONTEXT = 1
    if _cuda.cuPointerGetAttribute(C.byref(ctx), CU_POINTER_ATTRIBUTE_CONTEXT, int(cai["data"][0])) != 0 or not ctx:
        return
    if _cuda.cuCtxPushCurrent_v2(ctx) != 0:
        raise RuntimeError("cuCtxPushCurrent on the context of the destination failed")
    try:
        rc = _cuda.cuStreamSynchronize(C.c_void_p(int(cai["stream"]))) if "stream" in cai else _cuda.cuCtxSynchronize()
    finally:
        _cuda.cuCtxPopCurrent_v2(C.byref(C.c_void_p()))
    if rc != 0:
        raise RuntimeError(f"waiting for the pending work on the destination failed: CUresult {rc}")


def wrap(value, mn, mx):
    """S:1599-1603."""
    rng = mx - mn
    if rng == 0:
        return mn
    return (value - mn) % rng + mn
