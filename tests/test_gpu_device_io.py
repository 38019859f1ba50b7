"""Fields and captures through the caller's device memory (fluid_read_device / fluid_write_device /
fluid_capture_device; readField(out=...), writeField and captureScreenshot(out=...) with a CUDA array) on the
GPU, with torch CUDA tensors as the arrays: the same bits as the host twins on every handle kind, a whole
session driven through each path in lockstep, the tiny-divergence map of the blocked solve rebuilt by a
device write of divergence, ordering against torch's streams, the field arena and the buffer's guard bytes
left alone, and every refusal."""
import ctypes as C

import numpy as np
import pytest

import display_harness as DH
from conftest import bits_equal
from jacobi_tb_model import ITERS, JB, blocked, cases, expected
from sim_harness import POISONS, SLEEP_CYCLES, V3, Arena, make, special_values
from sim_harness import pkg, torch  # noqa: F401 -- fixtures

pytestmark = pytest.mark.gpu
F = np.float32
DT = 0.016666
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
SIZES = [(128, 128, 1024, 1024), (1024, 1024, 2048, 2048), (36, 20, 54, 30), (1, 9, 3, 27), (9, 1, 27, 3)]
KINDS = ["fp32", "half", "desktop", "nearest"]
INVALID = -1


def flags_of(pkg, kind):
    return {"fp32": 0, "half": pkg.FLAG_HALF_STORAGE,
            "desktop": pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX | pkg.FLAG_LINEAR_ADVECTION,
            "nearest": pkg.FLAG_NEAREST_FILTERING}[kind]


def shape_of(s, f):
    w, h, c, _ = s._dims(f)
    return (h, w, c) if c > 1 else (h, w)


def on_gpu(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a, F).copy()).cuda()


def read_dev(torch, s, f):
    """readField into a fresh float32 CUDA tensor, back on the host."""
    t = torch.empty(shape_of(s, f), dtype=torch.float32, device="cuda")
    assert s.readField(f, out=t) is t
    return t.cpu().numpy()


def seeded(pkg, s, seed, steps=2):
    rs = np.random.RandomState(seed)
    s.random = lambda: float(rs.random_sample())
    s.multipleSplats(3)
    for _ in range(steps):
        s.step(DT)


# ---- 1. and 2.: the same bits as fluid_read / fluid_write --------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("W,H,Wd,Hd", SIZES)
def test_read_device_is_read(pkg, torch, kind, W, H, Wd, Hd):
    """After seeded splats and steps, and after fluid_write of special values, every field read into device
    memory has the bits fluid_read gives (half storage: exact widening; NaN in the same places)."""
    s = make(pkg, W, H, Wd, Hd, flags=flags_of(pkg, kind))
    seeded(pkg, s, W + Hd)
    for f in FIELDS:
        assert bits_equal(read_dev(torch, s, f), s.readField(f)), (kind, f)
    for k, f in enumerate(FIELDS):
        s.writeField(f, special_values(shape_of(s, f), k + W, bool(flags_of(pkg, kind) & pkg.FLAG_HALF_STORAGE)))
    for f in FIELDS:
        host = s.readField(f)
        assert np.isnan(host).any() and np.isinf(host).any()
        assert bits_equal(read_dev(torch, s, f), host), (kind, f)
    s.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("W,H,Wd,Hd", SIZES)
def test_write_device_is_write(pkg, torch, kind, W, H, Wd, Hd):
    """write_device of an array, read back, equals fluid_write of the same array on a twin handle, bit for bit:
    special values everywhere, and on half storage fp16 overflow and round-to-nearest-even ties."""
    flags = flags_of(pkg, kind)
    half = bool(flags & pkg.FLAG_HALF_STORAGE)
    a, b = make(pkg, W, H, Wd, Hd, flags=flags), make(pkg, W, H, Wd, Hd, flags=flags)
    for k, f in enumerate(FIELDS):
        x = special_values(shape_of(a, f), 7 * k + H, half)
        a.writeField(f, x)
        t = on_gpu(torch, x)
        assert b.writeField(f, t) is None
        assert bits_equal(t.cpu().numpy(), x)                        # the source is only read
        want = a.readField(f)
        assert bits_equal(b.readField(f), want), (kind, f)
        if half:
            assert np.isinf(want).sum() > np.isinf(x).sum()           # the overflowing values became +-inf
    a.close(); b.close()


# ---- 3.: a whole session through each path ------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("start", range(len(SIZES)), ids=[f"{s[0]}x{s[1]}" for s in SIZES])
def test_session_twin(pkg, torch, kind, start):
    """Two handles driven through splats, graph-replayed steps, writes of every field, pressure_solve, a
    render and a resize (to the next size of SIZES), one reading and writing through host memory and the
    other through device memory: after every call every field is bitwise equal between them and both have
    launched the same number of kernels."""
    flags = flags_of(pkg, kind)
    half = bool(flags & pkg.FLAG_HALF_STORAGE)
    src, dst = SIZES[start], SIZES[(start + 1) % len(SIZES)]
    hs, ds = make(pkg, *src, flags=flags), make(pkg, *src, flags=flags)
    for s in (hs, ds):
        rs = np.random.RandomState(5 + start)
        s.random = lambda rs=rs: float(rs.random_sample())

    def same(what):
        for f in FIELDS:
            assert bits_equal(read_dev(torch, ds, f), hs.readField(f)), (kind, what, f)
        assert hs.stat("launches") == ds.stat("launches"), (kind, what)

    def both(what, fn):
        fn(hs, "host"); fn(ds, "device")
        same(what)

    def writes(s, io, special_):
        for k, f in enumerate(FIELDS):
            rng = np.random.default_rng(k + 10 * special_)
            x = special_values(shape_of(s, f), k, half) if special_ else rng.standard_normal(shape_of(s, f)).astype(F)
            s.writeField(f, x if io == "host" else on_gpu(torch, x))

    same("create")
    both("splats", lambda s, io: s.multipleSplats(3))
    for k in range(3):
        both(f"step {k}", lambda s, io: s.step(DT))
    assert hs.stat("graph_launches") == ds.stat("graph_launches") == 3
    both("write ordinary", lambda s, io: writes(s, io, False))
    both("pressure_solve", lambda s, io: s.pass_("pressure_solve"))
    both("step after write", lambda s, io: s.step(DT))
    frames = []
    both("render", lambda s, io: frames.append(s.render()))
    assert bits_equal(frames[0], frames[1])

    def resize(s, io):
        s._sizes = dst
        s.initFramebuffers()
    both("resize", resize)
    both("write special", lambda s, io: writes(s, io, True))
    both("pressure_solve after resize", lambda s, io: s.pass_("pressure_solve"))
    both("step after resize", lambda s, io: s.step(DT))
    hs.close(); ds.close()


# ---- 4.: the tiny-divergence map -----------------------------------------------------------------------------
@pytest.mark.parametrize("jb", JB)
@pytest.mark.parametrize("W,H", [(1024, 512), (1000, 520), (1000, 37), (16900, 3)])
def test_device_written_divergence_flags_every_placed_cell(pkg, torch, oracle, W, H, jb):
    """Divergence written from device memory with the tiny-value placements of jacobi_tb_model: the solve
    equals the fluid_write twin's and the oracle bit for bit, and the blocked kernel ran the same number of
    exact-tail streams on both (none where the blocked kernel does not run)."""
    a = make(pkg, W, H, 8, 8, jb=jb, PRESSURE_ITERATIONS=ITERS)
    b = make(pkg, W, H, 8, 8, jb=jb, PRESSURE_ITERATIONS=ITERS)
    for c in cases(W, H):
        a.writeField("divergence", c["d"])
        b.writeField("divergence", on_gpu(torch, c["d"]))
        n = []
        for s in (a, b):
            s.writeField("pressure", c["p0"])
            e0 = s.stat("jacobi_exact_streams")
            s.pass_("pressure_solve")
            n.append(s.stat("jacobi_exact_streams") - e0)
        want = expected(oracle, c)[0]
        assert bits_equal(a.readField("pressure"), want) and bits_equal(read_dev(torch, b, "pressure"), want)
        assert n[0] == n[1] and ((n[1] > 0) if blocked(W, H, jb) else (n[1] == 0)), (n, jb)
    a.close(); b.close()


@pytest.mark.parametrize("W,H", [(1024, 512), (4096, 4096)])
def test_device_solve_is_the_host_solve(pkg, torch, W, H):
    """write_device(divergence) + write_device(pressure) + pressure_solve + read_device(pressure) gives the bits
    of fluid_pressure_solve_host, 50 sweeps (banded host solve at 4096^2)."""
    rng = np.random.default_rng(W)
    p = rng.standard_normal((H, W)).astype(F)
    d = rng.uniform(-1, 1, (H, W)).astype(F)
    d[H // 3:H // 3 + 40, W // 5:W // 5 + 200] = F(2.0 ** -130)             # tiny cells: the map must be right
    a = make(pkg, W, H, 8, 8, PRESSURE_ITERATIONS=50)
    want = p.copy()
    a.pressure_solve_host(d, want, 50)
    b = make(pkg, W, H, 8, 8, PRESSURE_ITERATIONS=50)
    b.writeField("divergence", on_gpu(torch, d))
    b.writeField("pressure", on_gpu(torch, p))
    b.pass_("pressure_solve")
    assert bits_equal(read_dev(torch, b, "pressure"), want)
    assert b.stat("jacobi_exact_streams") > 0
    a.close(); b.close()


# ---- 5.: ordering ---------------------------------------------------------------------------------------------
def test_ordering_against_torch_streams(pkg, torch):
    """A source filled on a side stream behind a long sleep, handed over with a version-3 interface naming that
    stream, is written with its final values; a field read into a tensor can be used by torch at once."""
    s = make(pkg, 256, 256, 512, 512)
    seeded(pkg, s, 3)
    x = np.random.default_rng(1).standard_normal((256, 256, 2)).astype(F)
    t = on_gpu(torch, np.zeros_like(x))
    final = on_gpu(torch, x)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        t.copy_(final)
    s.writeField("velocity", V3(t, side))
    assert bits_equal(s.readField("velocity"), x)
    dye = s.readField("dye")
    out = torch.full(dye.shape, -1.0, dtype=torch.float32, device="cuda")
    doubled = s.readField("dye", out=out) * 2                              # queued on torch's stream right away
    assert bits_equal(doubled.cpu().numpy(), dye * F(2))
    s.close()


# ---- 6.: the arena and the buffer's guard bytes ------------------------------------------------------------
GUARD = 64                                                                 # floats on either side of the buffer


def guarded(torch, n, value):
    buf = torch.full((n + 2 * GUARD,), value, dtype=torch.float32, device="cuda")
    return buf, buf[GUARD:GUARD + n]


def guards_intact(buf, value):
    b = buf.cpu().numpy()
    return bits_equal(b[:GUARD], np.full(GUARD, value, F)) and bits_equal(b[-GUARD:], np.full(GUARD, value, F))


@pytest.mark.parametrize("kind", ["fp32", "half"])
@pytest.mark.parametrize("W,H,Wd,Hd", [(36, 20, 54, 30), (1024, 512, 1024, 512)])
def test_device_io_writes_only_its_field(pkg, torch, kind, W, H, Wd, Hd):
    """Under both arena poisons: read_device changes no arena byte, write_device(f) only what may_change("write",
    f) allows, and the device buffer's guard bytes on both sides stay as they were."""
    half = kind == "half"
    s = make(pkg, W, H, Wd, Hd, flags=flags_of(pkg, kind))
    g = Arena(torch, s, half)
    R = (lambda a: a.astype(np.float16).astype(F)) if half else (lambda a: a)
    for k, f in enumerate(FIELDS):
        x = R(np.random.default_rng(k).standard_normal(shape_of(s, f)).astype(F))
        for value in POISONS:
            s.writeField(f, x)
            buf, view = guarded(torch, x.size, -3.5)
            got = g.run("read", lambda: s.readField(f, out=view), (f,), value, swaps=())
            assert got is view and bits_equal(view.cpu().numpy().reshape(x.shape), x) and guards_intact(buf, -3.5), (f, value)
            buf, view = guarded(torch, x.size, -3.5)
            view.copy_(torch.from_numpy(x.reshape(-1)))
            g.run("write", lambda: s.writeField(f, view), (), value, field=f, swaps=())
            assert bits_equal(s.readField(f), x) and guards_intact(buf, -3.5), (f, value)
    s.close()


@pytest.mark.parametrize("kind", ["fp32", "half_half_postfx"])
def test_capture_device_writes_nothing_in_the_arena(pkg, torch, kind):
    """Under both arena poisons a capture into device memory changes no arena byte outside what render() may
    write (dye.write under SUNRAYS), gives the bytes of the clean host capture, and leaves its guard bytes."""
    dye = DH.stored(kind, DH.seeded_dye(64, 48, 9))
    s = DH.make(pkg, 64, 48, 96, 80, DH.flags_of(pkg, kind))
    s.config["CAPTURE_RESOLUTION"] = 64
    s.writeField("dye", dye)
    s.dithering = DH.golden_dither()
    g = Arena(torch, s, kind.startswith("half"))
    for kw in range(8):
        DH.set_keywords(s, kw)
        clean = s.captureScreenshot()
        n = clean.size
        for value in POISONS:
            buf = torch.full((n + 2 * 256,), 0xA5, dtype=torch.uint8, device="cuda")
            view = buf[256:256 + n]
            call = "render_sunrays" if kw & pkg.DISPLAY_SUNRAYS else "render"
            assert g.run(call, lambda: s.captureScreenshot(out=view), ("dye",), value, swaps=()) is view
            b = buf.cpu().numpy()
            assert np.all(b[:256] == 0xA5) and np.all(b[256 + n:] == 0xA5), (kw, value)
            assert np.array_equal(b[256:256 + n].reshape(clean.shape), clean), (kw, value)
    s.close()


# ---- 7.: refusals ---------------------------------------------------------------------------------------------
def test_field_refusals_leave_buffer_and_fields_alone(pkg, torch):
    """Each refused read_device / write_device returns FLUID_ERR_INVALID, leaves a poisoned buffer and every
    field as they were, and the next good call succeeds."""
    s = make(pkg, 64, 48, 96, 72)
    seeded(pkg, s, 2)
    before = {f: s.readField(f) for f in FIELDS}
    L, h = s._L, s._h
    n = s._dims("velocity")[0] * s._dims("velocity")[1] * 2
    dev = torch.full((n + 4,), -7.25, dtype=torch.float32, device="cuda")
    dp = dev.data_ptr()
    host = np.full(n, -7.25, F)
    pinned = L.fluid_host_alloc(4 * n)
    assert pinned
    pinned_view = np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_float)), (n,))
    pinned_view[:] = -7.25
    base = s.device_ptr("velocity")
    g = Arena(torch, s)
    arena_base = g.base
    bad = [dict(n_=n - 1), dict(n_=n + 1), dict(n_=0), dict(buf=None), dict(field=-1), dict(field=5),
           dict(buf=host.ctypes.data), dict(buf=pinned), dict(buf=dp + 2), dict(buf=dp + 1),
           dict(buf=base), dict(buf=s.device_ptr("curl")), dict(buf=s.device_ptr("dye") + 4),
           dict(buf=arena_base + g.L.bytes - 4)]
    if torch.cuda.device_count() > 1:
        other = torch.full((n,), -7.25, dtype=torch.float32, device="cuda:1")
        bad.append(dict(buf=other.data_ptr()))
    torch.cuda.synchronize()
    for fn in (L.fluid_read_device, L.fluid_write_device):
        for b in bad:
            args = dict(field=0, buf=dp, n_=n)
            args.update(b)
            assert fn(h, args["field"], args["buf"], args["n_"]) == INVALID, (fn.__name__, b)
            assert L.fluid_sync(h) == 0
            torch.cuda.synchronize()
            assert bool((dev == -7.25).all()) and np.all(host == -7.25) and np.all(pinned_view == -7.25), b
            for f in FIELDS:
                assert bits_equal(s.readField(f), before[f]), (fn.__name__, b, f)
            assert s.readField("velocity", out=dev[:n]) is not None                    # the handle is usable
            assert bits_equal(dev[:n].cpu().numpy(), before["velocity"].reshape(-1))
            dev.fill_(-7.25)
            torch.cuda.synchronize()
    L.fluid_host_free(pinned)
    s.close()


def test_capture_refusals_leave_dst_and_the_handle_alone(pkg, torch):
    """Every refusal of fluid_capture and of a device buffer returns FLUID_ERR_INVALID with the poisoned dst
    unchanged; the next good capture gives the host capture's bytes."""
    s = DH.make(pkg, 64, 64, 64, 64, BLOOM_RESOLUTION=32, SUNRAYS_RESOLUTION=24, CAPTURE_RESOLUTION=64)
    s.writeField("dye", DH.seeded_dye(64, 64, 7))
    dither = DH.golden_dither()
    s.dithering = dither
    DH.set_keywords(s, 7)
    _, fx, dith = pkg.postfx_inputs(s.config, dither)
    good = s.captureScreenshot()
    w = h = 64
    n = 4 * w * h
    L = s._L
    dev = torch.full((n + 8,), 0x5A, dtype=torch.uint8, device="cuda")
    dp = dev.data_ptr()
    host = np.full(n, 0x5A, np.uint8)
    pinned = L.fluid_host_alloc(n)
    C.memset(pinned, 0x5A, n)
    g = Arena(torch, s)

    def call(w_=w, h_=h, cw=64, ch=64, kw=7, fx_=C.byref(fx), d=dith.ctypes.data_as(C.c_void_p), n_=n, dst=dp):
        return L.fluid_capture_device(s._h, w_, h_, cw, ch, kw, 0, fx_, d, dith.shape[1], dith.shape[0],
                                      *DH.BACK_RGB, dst, n_)

    bad = [dict(kw=8), dict(n_=n - 1), dict(n_=n + 4), dict(n_=0), dict(w_=0), dict(h_=0), dict(cw=0), dict(ch=0),
           dict(kw=2, d=None), dict(kw=2, fx_=None), dict(kw=4, fx_=None), dict(dst=None),
           dict(dst=host.ctypes.data), dict(dst=pinned), dict(dst=dp + 1), dict(dst=dp + 2),
           dict(dst=s.device_ptr("dye")), dict(dst=g.base + g.L.bytes - 4)]
    if torch.cuda.device_count() > 1:
        bad.append(dict(dst=torch.full((n,), 0x5A, dtype=torch.uint8, device="cuda:1").data_ptr()))
    torch.cuda.synchronize()
    dye = s.readField("dye")
    for b in bad:
        assert call(**b) == INVALID, b
        assert L.fluid_sync(s._h) == 0
        assert bool((dev == 0x5A).all()) and np.all(host == 0x5A), b
        assert np.all(np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_uint8)), (n,)) == 0x5A), b
        assert bits_equal(s.readField("dye"), dye), b
        img = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
        assert np.array_equal(s.captureScreenshot(out=img).cpu().numpy(), good), b
    assert call(dst=dp + 4) == 0 and L.fluid_sync(s._h) == 0
    assert np.array_equal(dev[4:4 + n].cpu().numpy().reshape(h, w, 4), good)
    L.fluid_host_free(pinned)
    s.close()
    # half storage without HALF_POSTFX refuses BLOOM / SUNRAYS captures into device memory as well
    s = DH.make(pkg, 64, 64, 64, 64, pkg.FLAG_HALF_STORAGE, CAPTURE_RESOLUTION=64)
    s.dithering = dither
    t = torch.full((64, 64, 4), 0x5A, dtype=torch.uint8, device="cuda")
    for kw in (2, 4, 7):
        DH.set_keywords(s, kw)
        with pytest.raises(pkg.FluidError) as e:
            s.captureScreenshot(out=t)
        assert e.value.code == INVALID
        assert bool((t == 0x5A).all())
    s.close()


def test_python_refuses_bad_arrays(pkg, torch, tmp_path):
    """ValueError before any call: wrong dtype, wrong size, a strided view, `path` together with a CUDA `out`,
    and a numpy `out` for captureScreenshot."""
    s = make(pkg, 32, 32, 64, 64)
    s.config["CAPTURE_RESOLUTION"] = 32
    n0 = s.stat("launches")
    bad_fields = [torch.zeros((32, 32, 2), dtype=torch.float64, device="cuda"),
                  torch.zeros((32, 32, 3), dtype=torch.float32, device="cuda"),
                  torch.zeros((32, 64, 2), dtype=torch.float32, device="cuda")[:, ::2]]
    for t in bad_fields:
        with pytest.raises(ValueError):
            s.readField("velocity", out=t)
        with pytest.raises(ValueError):
            s.writeField("velocity", t)
    w, h = pkg.getResolution(32, 64, 64)["width"], pkg.getResolution(32, 64, 64)["height"]
    for t in (torch.zeros((h, w, 4), dtype=torch.int32, device="cuda"), torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")):
        with pytest.raises(ValueError):
            s.captureScreenshot(out=t)
    with pytest.raises(ValueError):
        s.captureScreenshot(path=str(tmp_path / "x.png"), out=torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        s.captureScreenshot(out=np.zeros((h, w, 4), np.uint8))
    assert s.stat("launches") == n0
    s.close()


# ---- 8.: captures -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["fp32", "half_half_postfx", "nearest_fp32"])
@pytest.mark.parametrize("Wd,Hd,cw,ch", [(64, 64, 128, 128), (48, 32, 807, 640)])
def test_capture_device_is_capture(pkg, torch, kind, Wd, Hd, cw, ch):
    """All eight keyword sets, TRANSPARENT off and on: captureScreenshot(out=t) holds the bytes of
    captureScreenshot() and launches as many kernels."""
    s = DH.make(pkg, Wd, Hd, cw, ch, DH.flags_of(pkg, kind), CAPTURE_RESOLUTION=min(cw, ch) // 2 + 3)
    s.writeField("dye", DH.nonfinite_dye(Wd, Hd, Wd + cw))
    s.dithering = DH.golden_dither()
    for kw in range(8):
        DH.set_keywords(s, kw)
        for transparent in (False, True):
            s.config["TRANSPARENT"] = transparent
            s.captureScreenshot()                               # post-FX targets made for this canvas
            n0 = s.stat("launches")
            host = s.captureScreenshot()
            host_launches = s.stat("launches") - n0
            t = torch.full(host.shape, 0x5A, dtype=torch.uint8, device="cuda")
            n0 = s.stat("launches")
            assert s.captureScreenshot(out=t) is t
            assert s.stat("launches") - n0 == host_launches, (kind, kw, transparent)
            assert np.array_equal(t.cpu().numpy(), host), (kind, kw, transparent)
    s.close()
