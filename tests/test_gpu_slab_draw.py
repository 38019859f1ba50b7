"""Frames, canvases and captures on row slabs (DESIGN §7) with every display keyword set, on ONE GPU: `world` slab
handles of one process draw their bands, and the bands, put together, equal an ordinary handle's image bit for bit;
the bloom FBO and sunrays texture every rank holds equal the ordinary handle's.

The rank handles come from a test build of the library (tests/slab_loopback_gather.cu): fluid.cu compiled with
FLUID_TEST_LOOPBACK and FLUID_TEST_LOOPBACK_GATHER, whose halo exchange and row-band all-gather copy the other ranks'
rows by stream-ordered device copies instead of calling NCCL.  Everything else is the library's own slab code: the
dye ghost-row refresh of a frame, the prefilter on a band of the bloom FBO, the sunrays mask on the rank's own dye
rows, the pyramid, sunrays and blurs on the gathered inputs, and the display band.  Each rank is driven from its
own thread.  Not covered: the NCCL gather itself -- tools/slab_draw_check.py runs it where there are two or more
GPUs."""
import concurrent.futures as cf
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from sim_harness import same_bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "webgl_fluid_simulation_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "slab_loopback_gather.cu")
BUILD_DIR = os.path.join(ROOT, "tests", "slab_loopback_gather_build")
HALO_ERR, INVALID, OK = -5, -1, 0
DT = 0.016666
F = np.float32
KEYWORDS = [dict(SHADING=bool(k & 1), BLOOM=bool(k & 2), SUNRAYS=bool(k & 4)) for k in range(8)]
# (BLOOM_INTENSITY, BLOOM_THRESHOLD, BLOOM_SOFT_KNEE, SUNRAYS_WEIGHT): two slider positions of
# test_gpu_postfx_params.py (t0_k0_w4: sunrays above 1; t033_k07: knee and curve narrowed where fp32 and JS differ)
SLIDERS = {"t0_k0_w4": (0.1, 0.0, 0.0, 4.0), "t033_k07": (0.55, 0.33, 0.7, 0.45)}


# ---- the loopback build with the gather ----------------------------------------------------------------------------
def _nvflags():
    """NVFLAGS of csrc/Makefile, so that the test build compiles fluid.cu exactly as the library is compiled."""
    out = subprocess.run(["make", "-s", "--no-print-directory", "-C", CSRC, "-f", "Makefile", "-f", "-", "print-nvflags"],
                         input="print-nvflags: ; @echo $(NVFLAGS)\n", capture_output=True, text=True, check=True)
    return out.stdout.split()


def _build():
    """libfluid_slab_loopback_gather.so, rebuilt only when a source is newer.  Under tests/ when the tree is writable,
    else in the temporary directory."""
    srcs = [SRC, os.path.join(ROOT, "tests", "slab_loopback.cu"), os.path.join(ROOT, "include", "fluid.h"),
            os.path.join(CSRC, "Makefile")]
    srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))]
    newest = max(os.path.getmtime(s) for s in srcs)
    for d in (BUILD_DIR, os.path.join(tempfile.gettempdir(), f"fluid_slab_loopback_gather_{os.getuid()}")):
        so = os.path.join(d, "libfluid_slab_loopback_gather.so")
        if os.path.exists(so) and os.path.getmtime(so) >= newest:
            return so
        try:
            os.makedirs(d, exist_ok=True)
        except OSError:
            continue
        if not os.access(d, os.W_OK):
            continue
        nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
        tmp = so + f".{os.getpid()}.tmp"
        # -Bsymbolic: the test build's calls into itself never bind to the production library loaded beside it
        subprocess.run([nvcc, *_nvflags(), "-Xlinker", "-Bsymbolic", "-shared", "-o", tmp, SRC, "-lcudart", "-ldl"],
                       check=True, capture_output=True)
        os.replace(tmp, so)
        return so
    raise RuntimeError("no writable directory for the loopback gather build")


@pytest.fixture(scope="session")
def loop():
    """(package, loopback library, torch): the library bound like webgl_fluid_simulation_b200._lib binds the product."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import webgl_fluid_simulation_b200 as pkg
    from webgl_fluid_simulation_b200 import _lib
    pkg.build()
    so = _build()
    saved_path, saved_lib = _lib.SO_PATH, _lib._lib
    try:
        _lib.SO_PATH, _lib._lib = so, None
        L = _lib.lib()
    finally:
        _lib.SO_PATH, _lib._lib = saved_path, saved_lib
    L.fluid_loopback_link.argtypes = [C.POINTER(C.c_void_p), C.c_int]
    return pkg, L, torch


class Group:
    """`world` rank handles of the loopback build, linked into one group, and `one`, an ordinary handle of the
    product, all created with the same config, sizes and canvas, holding the same dithering texture."""

    def __init__(self, loop, world, W, H, Wd, Hd, canvas=(256, 256), halo_rows=None, **cfg):
        pkg, L, self.torch = loop
        from webgl_fluid_simulation_b200 import _lib
        self.L, self.world = L, world
        c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd), "PRESSURE_ITERATIONS": 20}
        c.update(cfg)
        kw = dict(canvas_width=canvas[0], canvas_height=canvas[1], sizes=(W, H, Wd, Hd))
        self.one = pkg.FluidSimulation(dict(c), **kw)
        old_env, saved = os.environ.get("FLUID_HALO_ROWS"), _lib._lib
        try:
            if halo_rows:
                os.environ["FLUID_HALO_ROWS"] = str(halo_rows)
            _lib._lib = L
            self.ranks = [pkg.FluidSimulation(dict(c), rank=r, world=world, nccl_uid=bytes(128), **kw) for r in range(world)]
        finally:
            _lib._lib = saved
            if halo_rows:
                if old_env is None:
                    del os.environ["FLUID_HALO_ROWS"]
                else:
                    os.environ["FLUID_HALO_ROWS"] = old_env
        arr = (C.c_void_p * world)(*[s._h.value for s in self.ranks])
        assert L.fluid_loopback_link(arr, world) == OK, L.fluid_last_error(None)
        dither = np.random.default_rng(64).random((64, 64, 3), dtype=F)
        for s in self.handles():
            s.dithering = dither
        self.pool = cf.ThreadPoolExecutor(world)

    def handles(self):
        return self.ranks + [self.one]

    def each(self, fn):
        """fn(rank handle) on every rank, each on its own thread; the results in rank order."""
        futs = [self.pool.submit(fn, s) for s in self.ranks]
        return [f.result() for f in futs]

    def all(self, fn):
        out = self.each(fn)
        return out, fn(self.one)

    def set(self, **cfg):
        for s in self.handles():
            s.config.update(cfg)

    def write(self, name, full):
        self.one.writeField(name, full)
        for s in self.ranks:
            w, n, _, r0 = s._dims(name)
            s.writeField(name, full[r0:r0 + n])

    def seams(self):
        return [s._dims("dye")[3] for s in self.ranks[1:]]

    def stat(self, name):
        vals = [s.stat(name) for s in self.ranks]
        assert len(set(vals)) == 1, (name, vals)                 # SPMD: every rank counts the same
        return vals[0]

    def close(self):
        self.pool.shutdown()
        for s in self.handles():
            s.close()


@pytest.fixture
def group(loop):
    made = []

    def make(*a, **kw):
        g = Group(loop, *a, **kw)
        made.append(g)
        return g
    yield make
    for g in made:
        g.close()


def same_u8(a, b):
    return a.shape == b.shape and np.array_equal(a, b)


def check_draws(g, what, frame_size=None):
    """Every keyword set over BACK_COLOR and the checkerboard / bare: render()'s frame bands in rank order, every
    rank's bloom FBO and sunrays texture, canvas bands (host and device) and capture bands (host and device) in
    reverse rank order, all against `one`; per frame one dye exchange and one gather per post-FX chain."""
    torch = g.torch
    fw, fh = frame_size or (g.one.canvas["width"], g.one.canvas["height"])
    for kw in KEYWORDS:
        for transparent in (False, True):
            g.set(TRANSPARENT=transparent, **kw)
            tag = f"{what} {kw} transparent={transparent}"
            n_ex, n_ga = g.stat("halo_exchanges"), g.stat("gathers")

            def frame(s):
                img = s.render(fw, fh)
                return img, s.last_bloom, s.last_sunrays, s.render_band
            mine, ref = g.all(frame)
            assert g.stat("halo_exchanges") - n_ex == 1, tag
            assert g.stat("gathers") - n_ga == kw["BLOOM"] + kw["SUNRAYS"], tag
            assert same_bits(np.concatenate([m[0] for m in mine], axis=0), ref[0]), tag + " frame"
            assert [m[3] for m in mine] == [((fh * r) // g.world, (fh * (r + 1)) // g.world) for r in range(g.world)]
            for k, name in ((1, "bloom"), (2, "sunrays")):
                assert all((m[k] is None) == (ref[k] is None) for m in mine), tag
                if ref[k] is not None:
                    for r, m in enumerate(mine):
                        assert same_bits(m[k], ref[k]), f"{tag} {name} of rank {r}"
            for on_device in (False, True):
                def canvas(s):
                    if not on_device:
                        return s.render_canvas()
                    y0, y1 = s._band(s.canvas["height"])
                    t = torch.empty((y1 - y0, s.canvas["width"], 4), dtype=torch.uint8, device="cuda")
                    return s.render_canvas(out=t).cpu().numpy()
                mine, ref = g.all(canvas)
                assert same_u8(np.concatenate(mine[::-1], axis=0), ref), f"{tag} canvas on_device={on_device}"

                def capture(s):
                    if not on_device:
                        return s.captureScreenshot()
                    w, h, _ = s._capture_args()
                    y0, y1 = s._band(h)
                    t = torch.empty((y1 - y0, w, 4), dtype=torch.uint8, device="cuda")
                    return s.captureScreenshot(out=t).cpu().numpy()
                mine, ref = g.all(capture)
                assert same_u8(np.concatenate(mine[::-1], axis=0), ref), f"{tag} capture on_device={on_device}"


# (world, W, H, Wd, Hd): power-of-two slabs with dye == sim and dye = 2 x sim, ragged and uneven slabs, 8 ranks
GEOMETRIES = [
    (2, 128, 128, 128, 128),
    (3, 256, 256, 512, 512),
    (4, 200, 150, 300, 225),
    (3, 200, 150, 400, 300),
    (8, 128, 256, 256, 512),
]
# canvases: the desktop's, a ragged one, a portrait one
CANVASES = [(1920, 1080), (807, 640), (480, 854)]


@pytest.mark.parametrize("canvas", CANVASES)
@pytest.mark.parametrize("world,W,H,Wd,Hd", GEOMETRIES)
def test_every_keyword_set_equals_one_gpu(group, world, W, H, Wd, Hd, canvas):
    """Seeded dye up to 10, every keyword set, against one GPU; the frame at the canvas size and at a short,
    wide target."""
    g = group(world, W, H, Wd, Hd, canvas=canvas)
    rng = np.random.default_rng(world * 100 + Hd)
    g.write("dye", rng.random((Hd, Wd, 4), dtype=F) * F(10))
    check_draws(g, f"canvas {canvas}")
    if canvas == CANVASES[0]:
        check_draws(g, "frame 333 x 97", frame_size=(333, 97))


def test_band_edges_on_dye_seams(group):
    """BLOOM_RESOLUTION and SUNRAYS_RESOLUTION equal to the dye height on a square canvas: the bands of the bloom
    FBO a rank prefilters start and end on the dye seams, and the sunrays texture has the dye's rows."""
    g = group(4, 256, 256, 512, 512, canvas=(512, 512), BLOOM_RESOLUTION=512, SUNRAYS_RESOLUTION=512)
    assert g.seams() == [128, 256, 384]
    rng = np.random.default_rng(5)
    g.write("dye", rng.random((512, 512, 4), dtype=F) * F(3))
    check_draws(g, "bands on seams")


@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("world,W,H,Wd,Hd", [(2, 128, 128, 128, 128), (3, 200, 150, 400, 300), (4, 128, 256, 256, 512)])
def test_nonfinite_dye_beside_the_seams(group, world, W, H, Wd, Hd, value):
    """NaN or +-inf dye on the row just below and the row just above each seam (on a few columns and channels): the
    mask's and the display's weight-0 taps across a seam read it, so it must travel with the ghost rows."""
    g = group(world, W, H, Wd, Hd, canvas=(W * 3, H * 3))
    rng = np.random.default_rng(23)
    dye = rng.random((Hd, Wd, 4), dtype=F)
    for k, s in enumerate(g.seams()):
        for c in range(4):
            col = (11 + 37 * k + 53 * c) % Wd
            dye[s - 1, col, c % 3] = F(value)
            dye[s, (col + 5) % Wd, (c + 1) % 3] = F(value)
    g.write("dye", dye)
    check_draws(g, f"{value} beside the seams")


@pytest.mark.parametrize("sliders", ["t0_k0_w4", "t033_k07"])
def test_post_fx_sliders(group, sliders):
    I, T, K, Wt = SLIDERS[sliders]
    g = group(3, 200, 150, 400, 300, canvas=(807, 640))
    g.set(BLOOM_INTENSITY=I, BLOOM_THRESHOLD=T, BLOOM_SOFT_KNEE=K, SUNRAYS_WEIGHT=Wt)
    g.write("dye", np.random.default_rng(8).random((300, 400, 4), dtype=F) * F(2))
    check_draws(g, sliders)


def test_frames_after_steps_splats_and_a_resize(group):
    """Splats on the seams and steps, the desktop frame, canvas and capture; a resize that grows; again.  The launches
    of a frame equal one GPU's, and a second frame of one size launches what the first launched less the targets'
    first clear (the post-FX targets are not made again)."""
    g = group(3, 128, 96, 256, 192, canvas=(640, 480))
    rng = np.random.default_rng(9)
    recs = [(rng.random(), s / 192 if k % 2 else rng.random(), 600 * (rng.random() - 0.5), 600 * (rng.random() - 0.5),
             2 * rng.random(), rng.random(), 2 * rng.random()) for k, s in enumerate(g.seams() * 3)]
    g.all(lambda s: s.splats(np.array(recs, F)))
    for _ in range(3):
        g.all(lambda s: s.step(DT))
    check_draws(g, "after steps")
    g.set(SHADING=True, BLOOM=True, SUNRAYS=True, TRANSPARENT=False)
    launches = []
    for _ in range(3):
        before = [s.stat("launches") for s in g.handles()]
        g.all(lambda s: s.render())
        launches.append([s.stat("launches") - b for s, b in zip(g.handles(), before)])
    assert launches[1] == launches[2] and len(set(launches[1])) == 1, launches

    def resize(s):
        s._sizes = (192, 144, 384, 288)
        s.initFramebuffers()
    g.all(resize)
    g.all(lambda s: s.splats(np.array(recs, F)))
    g.all(lambda s: s.step(DT))
    check_draws(g, "after a resize")


def test_refusals_make_no_exchange(group, loop):
    """A wrong n_floats / n_bytes and BLOOM without a dithering texture are refused on every rank before any
    exchange or gather, and the group draws afterwards."""
    from webgl_fluid_simulation_b200 import _lib
    g = group(4, 200, 150, 300, 225, canvas=(807, 640))
    g.write("dye", np.random.default_rng(2).random((225, 300, 4), dtype=F))
    fx = _lib.PostFX(8, 256, 0.8, 0.6, 0.7, 196, 1.0)
    dith = np.ascontiguousarray(g.one.dithering)
    kw = _lib.DISPLAY_SHADING | _lib.DISPLAY_BLOOM | _lib.DISPLAY_SUNRAYS
    n_ex, n_ga = g.stat("halo_exchanges"), g.stat("gathers")

    def refused(s):
        y0, y1 = s._band(640)
        n = 4 * 807 * (y1 - y0)
        buf = np.empty(n + 4, F)
        p = buf.ctypes.data_as(C.c_void_p)
        d = dith.ctypes.data_as(C.c_void_p)
        rcs = [s._L.fluid_render_keywords(s._h, 807, 640, kw, C.byref(fx), d, 64, 64, 0.0, 0.0, 0.0, p, n - 4, None, None),
               s._L.fluid_render_keywords(s._h, 807, 640, kw, C.byref(fx), None, 64, 64, 0.0, 0.0, 0.0, p, n, None, None),
               s._L.fluid_render_canvas(s._h, 807, 640, kw, 0, C.byref(fx), d, 64, 64, 0.0, 0.0, 0.0, p, n + 4, 0),
               s._L.fluid_capture(s._h, 807, 640, 807, 640, kw, 0, C.byref(fx), None, 64, 64, 0.0, 0.0, 0.0, p, n)]
        return rcs
    assert g.each(refused) == [[INVALID] * 4] * 4
    assert (g.stat("halo_exchanges"), g.stat("gathers")) == (n_ex, n_ga)
    g.set(SHADING=True, BLOOM=True, SUNRAYS=True)
    mine, ref = g.all(lambda s: s.render_canvas())
    assert same_u8(np.concatenate(mine[::-1], axis=0), ref)
    assert g.stat("gathers") == n_ga + 2


def test_ghost_rows_the_slab_does_not_keep(group):
    """A 14-row-halo slab (Gd = 14): a frame whose bloom prefilter (BLOOM_RESOLUTION 8: an 8-row FBO with a 2-level
    pyramid, 18 dye ghost rows) or display band (a 16-row target: 26) reaches further is refused with FLUID_ERR_HALO
    on every rank, after the exchange every rank makes; SUNRAYS alone and the canvas-sized frame draw, and equal one
    GPU."""
    from webgl_fluid_simulation_b200.slab import draw_ghost_rows
    g = group(2, 256, 256, 256, 256, canvas=(256, 256), halo_rows=14, BLOOM_RESOLUTION=8)
    assert draw_ghost_rows(256, 256, 8, True) == 18 and draw_ghost_rows(256, 16) == 26
    assert draw_ghost_rows(256, 256, 0, True) <= 14
    g.write("dye", np.random.default_rng(4).random((256, 256, 4), dtype=F))

    def rc_of(fn):
        def call(s):
            try:
                fn(s)
                return OK
            except Exception as e:                               # FluidError
                return e.code
        return call
    g.set(BLOOM=True, SUNRAYS=False)
    assert g.each(rc_of(lambda s: s.render())) == [HALO_ERR] * 2
    assert g.each(rc_of(lambda s: s.render_canvas())) == [HALO_ERR] * 2
    g.set(BLOOM=False, SUNRAYS=False)
    assert g.each(rc_of(lambda s: s.render(64, 16))) == [HALO_ERR] * 2
    g.set(SHADING=True, SUNRAYS=True)
    mine, ref = g.all(lambda s: s.render())
    assert same_bits(np.concatenate(mine, axis=0), ref)
    mine, ref = g.all(lambda s: s.captureScreenshot())
    assert same_u8(np.concatenate(mine[::-1], axis=0), ref)


def test_png_needs_the_whole_image(group, tmp_path):
    g = group(2, 128, 128, 128, 128)
    with pytest.raises(ValueError, match="whole image"):
        g.ranks[0].captureScreenshot(path=str(tmp_path / "band.png"))
