"""Row slabs (DESIGN §7) on ONE GPU: `world` slab handles of one process swap their halos by stream-ordered
device copies, and every rank's owned rows, concatenated, equal an ordinary handle's fields bit for bit.

The rank handles come from a test build of the library (tests/slab_loopback.cu): fluid.cu compiled with
FLUID_TEST_LOOPBACK, whose halo exchange copies the neighbours' boundary rows into this rank's ghost rows
instead of calling NCCL or the peer-memory push.  Everything else is the library's own slab code: the step, the
Jacobi plan (deep halo and per-launch fallback), the tiny-divergence scans of received strips, the 4-cell and
one-cell advection kernels with their ghost-zone checks, splats, resize and render bands.  Each rank is driven
from its own thread (ctypes releases the GIL), as one process per GPU would drive it.  Not covered: the real
transports (the NCCL calls, halo_push_kernel and its flag handshake) -- tests/test_gpu_multi.py runs those
where there are two or more GPUs."""
import concurrent.futures as cf
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from jacobi_tb_model import ITERS as TINY_ITERS
from jacobi_tb_model import TINY, groups, placements, tiny_case
from sim_harness import near_max_patch, same_bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "webgl_fluid_simulation_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "slab_loopback.cu")
BUILD_DIR = os.path.join(ROOT, "tests", "slab_loopback_build")
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
DT = 0.016666
HALO_ERR, OK = -5, 0
F = np.float32


# ---- the loopback build ------------------------------------------------------------------------------------------
def _nvflags():
    """NVFLAGS of csrc/Makefile, so that the test build compiles fluid.cu exactly as the library is compiled."""
    out = subprocess.run(["make", "-s", "--no-print-directory", "-C", CSRC, "-f", "Makefile", "-f", "-", "print-nvflags"],
                         input="print-nvflags: ; @echo $(NVFLAGS)\n", capture_output=True, text=True, check=True)
    return out.stdout.split()


def _build_loopback():
    """libfluid_slab_loopback.so, rebuilt only when a source is newer.  Under tests/ when the tree is writable,
    else in the temporary directory."""
    srcs = [SRC, os.path.join(ROOT, "include", "fluid.h"), os.path.join(CSRC, "Makefile")]
    srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))]
    newest = max(os.path.getmtime(s) for s in srcs)
    for d in (BUILD_DIR, os.path.join(tempfile.gettempdir(), f"fluid_slab_loopback_{os.getuid()}")):
        so = os.path.join(d, "libfluid_slab_loopback.so")
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
    raise RuntimeError("no writable directory for the loopback build")


@pytest.fixture(scope="session")
def loop():
    """(package, loopback library): the library bound like webgl_fluid_simulation_b200._lib binds the product."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import webgl_fluid_simulation_b200 as pkg
    from webgl_fluid_simulation_b200 import _lib
    pkg.build()
    so = _build_loopback()
    saved_path, saved_lib = _lib.SO_PATH, _lib._lib
    try:
        _lib.SO_PATH, _lib._lib = so, None
        L = _lib.lib()
    finally:
        _lib.SO_PATH, _lib._lib = saved_path, saved_lib
    L.fluid_loopback_link.argtypes = [C.POINTER(C.c_void_p), C.c_int]
    return pkg, L


# ---- a group of ranks beside an ordinary handle ------------------------------------------------------------------
def ghost_rows(H, Hd, world, iters, halo_rows=None):
    """G of fluid.cu slab_geometry."""
    g = max(14, halo_rows) if halo_rows else max(64, iters + 2)
    per = max(1, -(-Hd // H))
    return min(g, H // world, (Hd // world) // per)


class Group:
    """`world` rank handles of the loopback build, linked into one group, and `one`, an ordinary handle of the
    product, all created with the same config and sizes."""

    def __init__(self, loop, world, W, H, Wd, Hd, iters=20, flags=0, jb=0, halo_rows=None, **cfg):
        pkg, L = loop
        from webgl_fluid_simulation_b200 import _lib
        self.pkg, self.L, self.world = pkg, L, world
        c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd), "PRESSURE_ITERATIONS": iters}
        c.update(cfg)
        kw = dict(canvas_width=W, canvas_height=H, flags=flags, jacobi_block=jb, sizes=(W, H, Wd, Hd))
        self.one = pkg.FluidSimulation(dict(c), **kw)
        old_env = os.environ.get("FLUID_HALO_ROWS")
        saved = _lib._lib
        try:
            if halo_rows:
                os.environ["FLUID_HALO_ROWS"] = str(halo_rows)
            _lib._lib = L
            self.ranks = [pkg.FluidSimulation(dict(c), rank=r, world=world, nccl_uid=bytes(128), **kw)
                          for r in range(world)]
        finally:
            _lib._lib = saved
            if halo_rows:
                if old_env is None:
                    del os.environ["FLUID_HALO_ROWS"]
                else:
                    os.environ["FLUID_HALO_ROWS"] = old_env
        self.G = ghost_rows(H, Hd, world, iters, halo_rows)
        self.link()
        self.pool = cf.ThreadPoolExecutor(world)

    def link(self):
        arr = (C.c_void_p * self.world)(*[s._h.value for s in self.ranks])
        assert self.L.fluid_loopback_link(arr, self.world) == OK, self.L.fluid_last_error(None)

    def each(self, fn):
        """fn(rank handle) on every rank, each on its own thread; the results in rank order."""
        futs = [self.pool.submit(fn, s) for s in self.ranks]
        return [f.result() for f in futs]

    def all(self, fn):
        """fn on every rank and on the ordinary handle."""
        out = self.each(fn)
        fn(self.one)
        return out

    def rows(self, name):
        return [(s._dims(name)[3], s._dims(name)[1]) for s in self.ranks]

    def seams(self):
        return [r0 for r0, _ in self.rows("velocity")[1:]]

    def write(self, name, full):
        """The full array into `one`, each rank's owned rows into the rank."""
        self.one.writeField(name, full)
        for s, (r0, n) in zip(self.ranks, self.rows(name)):
            s.writeField(name, full[r0:r0 + n])

    def gathered(self, name):
        return np.concatenate(self.each(lambda s: s.readField(name)), axis=0)

    def assert_same(self, what, fields=FIELDS):
        for name in fields:
            got, want = self.gathered(name), self.one.readField(name)
            if not same_bits(got, want):
                bad = np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))
                raise AssertionError(f"{what}: {name} differs at {len(bad)} entries, first (row, col) "
                                     f"{bad[:4, :2].tolist()}, seams at rows {self.seams()}")

    def stat(self, name):
        vals = [s.stat(name) for s in self.ranks]
        assert len(set(vals)) == 1, (name, vals)                 # SPMD: every rank counts the same
        return vals[0]

    def close(self):
        self.pool.shutdown()
        for s in self.ranks:
            s.close()
        self.one.close()


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


def jacobi_exchanges(g, iters, jb=0, naive=False, W=None):
    """Halo exchanges of one pressure solve on a slab (DESIGN §7): ONE group when the ghost rows hold iters + 1
    rows (deep halo), else one for divergence and one before each launch."""
    if iters <= 0:
        return 0
    if iters + 1 <= g.G:
        return 1
    kb = max(1, min(jb if jb > 0 else 10, 13, g.G - 1))
    tb = (W % 4 == 0 and W >= 16) and not naive and kb != 1
    k = kb if tb else 1
    return 1 + -(-iters // k)


def records(rng, n, seams_y, force):
    """n splat records: half centred on a slab seam (y = seam row / H), half anywhere."""
    r = np.empty((n, 7), F)
    r[:, 0] = rng.random(n)
    r[:, 1] = rng.random(n)
    k = np.arange(n) % 2 == 0
    if len(seams_y):
        r[k, 1] = np.asarray(seams_y, F)[np.arange(int(k.sum())) % len(seams_y)]
    r[:, 2:4] = force * (rng.random((n, 2)) - 0.5)
    r[:, 4:7] = 1.5 * rng.random((n, 3))
    return r


# ---- whole sessions over the slab geometries ---------------------------------------------------------------------
# (world, W, H, Wd, Hd, FLUID_HALO_ROWS, splat force): 4-cell kernels on power-of-two grids at least 128 wide (dye ==
# sim and dye = 2 x sim), one-cell kernels with row offsets on ragged grids, uneven slabs, and minimal slabs of
# 14-16 rows with a 14- or 16-row ghost zone (the per-launch Jacobi fallback: 21 rows would be needed)
GEOMETRIES = [
    (2, 128, 128, 128, 128, None, 1000),
    (3, 256, 256, 512, 512, None, 1000),
    (8, 128, 256, 256, 512, None, 1000),
    (4, 200, 150, 300, 225, None, 1000),
    (3, 200, 150, 300, 225, None, 1000),
    (2, 36, 64, 36, 64, None, 1000),
    (4, 36, 64, 72, 128, None, 1000),
    (2, 128, 32, 128, 32, 14, 300),
    (3, 128, 44, 128, 44, 14, 300),
    (4, 128, 64, 256, 128, 16, 300),
]


@pytest.mark.parametrize("world,W,H,Wd,Hd,halo,force", GEOMETRIES)
def test_session_equals_one_gpu(group, world, W, H, Wd, Hd, halo, force):
    """Splats on the seams (one call each, then a burst of 150 records: two launches), steps with changing dt,
    a host write of every field followed by a step (velocity: the +-3 ghost rows are rebuilt first), render
    bands, a resize that grows and one that shrinks -- every field of every rank equal to one GPU after each
    call, and the halo exchanges of each step as DESIGN §7 counts them."""
    g = group(world, W, H, Wd, Hd, halo_rows=halo)
    rng = np.random.default_rng(world * 1000 + H)
    seams_y = [s / H for s in g.seams()]
    for rec in records(rng, 6, seams_y, force):
        g.all(lambda s: s.splat(*rec[:4], tuple(rec[4:])))
    g.assert_same("splat() x 6")
    assert g.stat("halo_transport_p2p") == 0
    deep = 20 + 1 <= g.G
    per_step = jacobi_exchanges(g, 20, W=W) + 2
    for k, dt in enumerate((DT, 0.011, 0.0073)):
        n0 = g.stat("halo_exchanges")
        g.all(lambda s: s.step(dt))
        assert g.stat("halo_exchanges") - n0 == per_step, (k, deep)
        g.assert_same(f"step {k} dt={dt}")
        if k == 0:
            burst = records(rng, 150, seams_y, force)
            g.all(lambda s: s.splats(burst))
            g.assert_same("splats(150)")
    v, dye, p = ((rng.standard_normal((H, W, 2)) * 0.2 * force).astype(F), rng.random((Hd, Wd, 4), dtype=F),
                 rng.standard_normal((H, W)).astype(F))
    for name, a in (("velocity", v), ("dye", dye), ("pressure", p), ("divergence", rng.standard_normal((H, W)).astype(F))):
        g.write(name, a)
        g.assert_same(f"write {name}")
        n0 = g.stat("halo_exchanges")
        g.all(lambda s: s.step(DT))
        assert g.stat("halo_exchanges") - n0 == per_step + (name == "velocity"), name
        g.assert_same(f"write {name} + step")
    for cfg in ({}, {"SHADING": True}, {"SHADING": True, "TRANSPARENT": True}):
        def draw(s):
            s.config.update({"SHADING": False, "TRANSPARENT": False, "BLOOM": False, "SUNRAYS": False}, **cfg)
            return s.render(W + 17, 2 * Hd + 1)
        bands = g.each(draw)
        assert same_bits(np.concatenate(bands, axis=0), draw(g.one)), cfg
    if halo is None:
        for sizes in ((2 * W, 2 * H, 2 * Wd, 2 * Hd), (W, H, Wd, Hd)):
            def resize(s):
                s._sizes = sizes
                s.initFramebuffers()
            g.all(resize)
            g.assert_same(f"resize to {sizes}", ("velocity", "dye"))
            g.all(lambda s: s.step(DT))
            g.assert_same(f"resize to {sizes} + step")


def test_slab_check_drive_sequence(group):
    """tools/slab_check.py's drive() on 2 ranks of its default 512 x 768 / 1024 x 1536 grid, 23 sweeps: seeded
    multipleSplats, a 2000 texel/s splat pair on the seam, 4 steps with a burst after the second, a 256 x 192
    frame, a resize to 256 x 384 / 512 x 768 and 2 more steps, then a host-written solve."""
    W, H, WD, HD, FAST = 512, 768, 1024, 1536, 2000.0
    g = group(2, W, H, WD, HD, iters=23)

    def drive(sim):
        rs = np.random.RandomState(5)
        sim.random = lambda: float(rs.random_sample())
        sim.multipleSplats(6)
        sim.splats([(0.5, 0.5, 0.3 * FAST, FAST, 0.9, 0.2, 0.1), (0.25, 0.5, 0.0, -FAST, 0.1, 0.8, 0.3)])
        for k in range(4):
            sim.step(0.016666)
            if k == 1:
                sim.splats([(rs.random_sample(), rs.random_sample(), 1000 * (rs.random_sample() - 0.5),
                             1000 * (rs.random_sample() - 0.5), 1.5 * rs.random_sample(), 0.0, 1.5 * rs.random_sample())
                            for _ in range(6)])
        out = {n: sim.readField(n) for n in ("velocity", "dye", "pressure", "divergence")}
        out["frame"] = sim.render(256, 192)
        sim._sizes = (256, 384, 512, 768)
        sim.initFramebuffers()
        out["resized_velocity"] = sim.readField("velocity"); out["resized_dye"] = sim.readField("dye")
        for _ in range(2):
            sim.step(0.016666)
        out["after_velocity"] = sim.readField("velocity"); out["after_dye"] = sim.readField("dye")
        return out

    mine = g.each(drive)
    ref = drive(g.one)
    rng = np.random.default_rng(1)
    pfull = rng.standard_normal((384, 256)).astype(F); dfull = rng.uniform(-1, 1, (384, 256)).astype(F)
    g.write("pressure", pfull); g.write("divergence", dfull)
    g.all(lambda s: s.pass_("pressure_solve"))
    for name, want in ref.items():
        assert same_bits(np.concatenate([m[name] for m in mine], axis=0), want), name
    g.assert_same("host-written solve", ("pressure",))


# ---- the pressure solve: every plan --------------------------------------------------------------------------------
@pytest.mark.parametrize("naive", [False, True])
@pytest.mark.parametrize("jb", [0, 1, 7])
@pytest.mark.parametrize("iters", [20, 50, 70])
def test_pressure_solve_plans(group, iters, jb, naive):
    """pressure_solve with iterations + 1 <= G (one deep exchange) and iterations raised above G - 1 after
    creation (a divergence exchange, then one before each launch), at JACOBI_BLOCK 1, 7 and the default and with
    naive Jacobi, on 4 uneven slabs of a ragged grid; the rank counters and the bits against one GPU."""
    from webgl_fluid_simulation_b200 import _lib
    W, H = 132, 259
    g = group(4, W, H, W, H, iters=20, flags=_lib.FLAG_NAIVE_JACOBI if naive else 0, jb=jb)
    assert g.G == 64
    rng = np.random.default_rng(iters + jb)
    g.write("pressure", rng.standard_normal((H, W)).astype(F))
    g.write("divergence", rng.uniform(-1, 1, (H, W)).astype(F))
    for s in g.ranks + [g.one]:
        s.config["PRESSURE_ITERATIONS"] = iters
    n0 = g.stat("halo_exchanges")
    g.all(lambda s: s.pass_("pressure_solve"))
    assert g.stat("halo_exchanges") - n0 == jacobi_exchanges(g, iters, jb, naive, W)
    g.assert_same(f"solve iters={iters} jb={jb} naive={naive}", ("pressure", "divergence"))
    # the same divergence again: a deep solve sends only pressure now, still one exchange
    n0 = g.stat("halo_exchanges")
    g.all(lambda s: s.pass_("pressure_solve"))
    assert g.stat("halo_exchanges") - n0 == jacobi_exchanges(g, iters, jb, naive, W)
    g.assert_same("second solve", ("pressure",))


def test_exact_streams_near_flt_max(group):
    """Pressure near FLT_MAX on both sides of every seam: the blocked kernel's exact tail runs on the slabs as it
    does on one GPU, and the bits agree."""
    W, H = 256, 256
    g = group(4, W, H, W, H)
    rng = np.random.default_rng(3)
    p = rng.standard_normal((H, W)).astype(F); d = rng.uniform(-1, 1, (H, W)).astype(F)
    for k, s in enumerate(g.seams()):
        near_max_patch(p, d, s - 3, s + 3, 20 + 60 * k, 28 + 60 * k, 0.8)
    g.write("pressure", p); g.write("divergence", d)
    g.all(lambda s: s.pass_("pressure_solve"))
    g.assert_same("near-FLT_MAX solve", ("pressure",))
    assert sum(s.stat("jacobi_exact_streams") for s in g.ranks) > 0
    assert g.one.stat("jacobi_exact_streams") > 0


@pytest.mark.parametrize("halo", [None, 14])
def test_tiny_divergence_reaches_a_rank_only_as_ghost_rows(group, halo):
    """Divergence with 0 < |d| < 2^-123 in pairs of cells two rows apart that lie on ONE side of the seam, next to
    it and at the far end of the strip: each pair is owned by one rank and reaches its neighbour only in the strips
    [row0 - n, row0) / [row1, row1 + n) that the exchange brings (deep halo: n = iters; FLUID_HALO_ROWS=14: the
    fallback's first launch depth), with no tiny cell of the neighbour's own rows in the same map cells.  Every
    placed cell defeats the contracted tail (jacobi_tb_model), so a strip that is not scanned after the exchange
    gives different bits."""
    W, H, world, iters = 256, 128, 2, TINY_ITERS
    s0 = H // 2
    depth = iters if halo is None else 8                     # deep halo / depth of the fallback's first launch
    extra = (s0 - 3, s0, s0 - depth, s0 + depth - 3)         # row targets: y-sites with cells at t and t + 2
    every = placements(W, H, extra)
    wanted = [g_ for g_ in groups(every) if any(every[q][3][0][0] in extra or every[q][3][1][0] in extra for q in g_)]
    assert wanted
    g = group(world, W, H, W, H, iters=iters, halo_rows=halo)
    assert (iters + 1 <= g.G) == (halo is None)
    below = above = 0
    for gi, q in enumerate(groups(every)):
        if q not in wanted:
            continue
        c = tiny_case(W, H, extra, None, gi)
        for (j, i) in (cell for site in c["sites"] for cell in site[3]):
            below += s0 - depth <= j < s0
            above += s0 <= j < s0 + depth
        assert not c["d"][(c["d"] != 0) & (np.abs(c["d"]) >= TINY)].any()
        g.write("pressure", c["p0"]); g.write("divergence", c["d"])
        g.all(lambda s: s.pass_("pressure_solve"))
        g.assert_same(f"tiny group {gi}", ("pressure",))
    assert below >= 4 and above >= 4, (below, above)


# ---- data at the seams -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,W,H,Wd,Hd", [(2, 128, 128, 128, 128), (3, 256, 256, 512, 512), (4, 200, 150, 200, 150),
                                             (2, 36, 64, 72, 128)])
@pytest.mark.parametrize("value", [np.inf, -np.inf, np.nan, -0.0])
def test_specials_beside_the_seams(group, world, W, H, Wd, Hd, value):
    """inf, NaN and -0.0 in velocity on the row just below and the row just above each seam (x on one column, y on
    another): the manual bilerp's +y neighbour of a rank's last row is its neighbour's first row, so the NaN the
    reference makes there must cross the seam.  Two steps, every field against one GPU."""
    g = group(world, W, H, Wd, Hd)
    rng = np.random.default_rng(17)
    v = (rng.standard_normal((H, W, 2)) * 30).astype(F)
    for k, s in enumerate(g.seams()):
        c = (7 + 41 * k) % (W - 2)
        v[s - 1, c, 0] = v[s, c + 1, 1] = F(value)
        v[s, c, 0] = v[s - 1, c + 1, 1] = F(value)
    g.write("velocity", v)
    g.write("dye", rng.random((Hd, Wd, 4), dtype=F))
    for k in range(2):
        g.all(lambda s: s.step(DT))
        g.assert_same(f"{value} beside the seams, step {k}")


# ---- the ghost-zone contract ---------------------------------------------------------------------------------------
def reach_verdict(V, j_lo, j_hi, lo, hi, H, dt, eps=1e-3):
    """From the velocity advection reads (float64): 'in' when every back-trace tap of output rows [j_lo, j_hi)
    lies in the valid rows [lo, hi) with eps to spare, 'out' when one leaves them by more than eps, else None."""
    vy = V[j_lo:j_hi, :, 1].astype(np.float64)
    j = np.arange(j_lo, j_hi, dtype=np.float64)[:, None]
    st = j - dt * vy                                          # (uv - dt v ts) * H - 0.5, in rows
    verdicts = set()
    for e in (-eps, eps):
        y = np.floor(st + e)
        j0 = np.clip(y, -1, H - 1); j1 = np.minimum(j0 + 1, H - 1); j0 = np.maximum(j0, 0)
        verdicts.add(bool(((j0 < lo) | (j1 >= hi)).any()))
    return None if len(verdicts) > 1 else ("out" if verdicts.pop() else "in")


@pytest.mark.parametrize("dy_sign", [1.0, -1.0])
def test_fast_splat_across_a_seam(group, dy_sign):
    """A splat on the seam of two 16-row-halo slabs, aimed across it, at a sweep of speeds.  The velocity that
    advection reads (after the projection) comes from the one-GPU handle's passes; from it, in float64, the reach
    of every back-trace: where all stay inside a rank's valid rows, that rank's sync returns OK and the step
    equals one GPU; where one leaves them, the sync returns FLUID_ERR_HALO.  No speed may give other bits
    without the error."""
    W = H = 128
    halo = 16
    seen = {"in": 0, "out": 0}
    # the projection keeps a fraction of a splat's force: the reach crosses G - 5 = 11 rows within this sweep
    for speed in (500, 1000, 2000, 3000, 4000, 5000, 6000, 7000, 8000, 10000, 14000, 20000, 40000):
        g = group(2, W, H, W, H, halo_rows=halo, CURL=0.0)
        probe = g.pkg.FluidSimulation(dict(g.one.config), canvas_width=W, canvas_height=H, sizes=(W, H, W, H))
        rec = np.array([[0.5, g.seams()[0] / H, 0.3 * speed, dy_sign * speed, 0.9, 0.2, 0.1],
                        [0.3, 0.62, -0.2 * speed, -dy_sign * speed, 0.1, 0.8, 0.3]], F)
        probe.splats(rec)
        probe.pass_("curl_vorticity_divergence", DT)
        probe.pass_("pressure_solve")
        probe.pass_("gradient_subtract")
        V = probe.readField("velocity")
        probe.pass_("advect_velocity", DT)                    # what the dye advection reads
        V2 = probe.readField("velocity")
        probe.close()
        g.all(lambda s: s.splats(rec))
        g.all(lambda s: s.step(DT))
        rcs = g.each(lambda s: g.L.fluid_sync(s._h))
        for s, rc, (r0, n) in zip(g.ranks, rcs, g.rows("velocity")):
            lo, hi = max(r0 - g.G, 0), min(r0 + n + g.G, H)
            # velocity: owned rows +- 3 from V; dye (same grid, Gd == G): owned rows from V2
            both = {reach_verdict(V, max(r0 - 3, 0), min(r0 + n + 3, H), lo, hi, H, DT),
                    reach_verdict(V2, r0, r0 + n, lo, hi, H, DT)}
            verdict = "out" if "out" in both else ("in" if both == {"in"} else None)
            assert rc in (OK, HALO_ERR), (speed, rc)
            if verdict == "out":
                assert rc == HALO_ERR, (speed, s._rank, "a back-trace left the ghost zone without FLUID_ERR_HALO")
            elif verdict == "in":
                assert rc == OK, (speed, s._rank, g.L.fluid_last_error(s._h))
            if verdict:
                seen[verdict] += 1
        if all(rc == OK for rc in rcs):
            g.assert_same(f"speed {speed}")
        g.close()
    assert seen["in"] >= 4 and seen["out"] >= 4, seen
