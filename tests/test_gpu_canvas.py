"""render(null) on the RGBA8 canvas (fluid_render_canvas / FluidSimulation.render_canvas) on the GPU: bit for
bit the canvas rule of tests/canvas_model.py applied to the same handle's bare display fragment, the same
bytes into host and device memory, the kernels it launches, what it leaves alone in the field arena, what
it refuses, and update(canvas=...)."""
import ctypes as C

import numpy as np
import pytest

import arena_model as A
import canvas_model as CM
from display_harness import BACK, BACK_RGB, flags_of, make, set_keywords
from display_harness import dither  # noqa: F401 -- a fixture
from display_model import ALL3, BLOOM, SHADING, SUNRAYS
from sim_harness import POISONS, SLEEP_CYCLES, V3, Arena
from sim_harness import pkg, torch  # noqa: F401 -- fixtures

pytestmark = pytest.mark.gpu
F = np.float32
# (dye w, dye h, canvas w, canvas h, plant fused-rule witnesses): the capture goldens' geometries, and one
# where the canvas samples the dye at its texel centres, so planted texels reach the fragment unchanged
GEOMETRIES = [(64, 64, 128, 128, False), (48, 32, 807, 640, False), (64, 64, 64, 64, True)]
KINDS = {"fp32": "fp32", "half": "half_half_postfx", "nearest": "nearest_fp32"}


def mode_flags(pkg, mode):
    return flags_of(pkg, KINDS[mode])


def seeded_dye(Wd, Hd, seed, special=True):
    """Values up to 10 (display alpha above 1 on many texels, below 1 on others); with `special`, a few
    texels holding NaN and +-inf."""
    rng = np.random.default_rng(seed)
    dye = rng.random((Hd, Wd, 4), dtype=F) ** 3
    dye[rng.random((Hd, Wd)) < 0.4, :3] *= F(10)
    dye[..., 3] = 1
    if special:
        for k, v in enumerate((np.nan, np.inf, -np.inf, np.nan)):
            dye[(7 * k + 3) % Hd, (11 * k + 5) % Wd, k % 3] = v
    return dye


def plant_witnesses(dye, cw, ch, rng):
    """Texels (r, 0, a) whose red byte tells the rule from the fused one: row 1 over BACK_COLOR, row 3 over
    the checkerboard (destinations of those canvas texels).  fp16-representable, so half storage keeps them."""
    opaque = CM.destination_bytes(cw, ch, BACK_RGB, False, cw / ch)
    checker = CM.destination_bytes(cw, ch, BACK_RGB, True, cw / ch)
    for row, d8 in ((1, opaque), (3, checker)):
        for i in range(0, min(cw, dye.shape[1]), 2):
            r, g, a = CM.fused_witnesses(F(d8[row, i, 0]) / F(255), 1, rng)[0]
            dye[row, i, :3] = [r, g, a]


def first_mismatch(got, want):
    idx = np.argwhere(got != want)
    return len(idx), (idx[0].tolist(), got[tuple(idx[0])], want[tuple(idx[0])]) if len(idx) else None


@pytest.mark.parametrize("mode", ["fp32", "half", "nearest"])
def test_canvas_is_the_rule_applied_to_the_bare_fragment(pkg, dither, mode):
    """All eight keyword sets x {BACK_COLOR (10, 20, 30), TRANSPARENT}: the canvas equals canvas_model applied to
    render(w, h, target=True) with TRANSPARENT (FLUID_BACKGROUND 2: the same display kernel, no blend), bit
    for bit.  Across the geometries every wrong rule of the model changes at least one byte of the
    expected canvases, so none of them could pass."""
    hits = dict.fromkeys(CM.MUTANTS, 0)
    rng = np.random.default_rng(17)
    for Wd, Hd, cw, ch, plant in GEOMETRIES:
        s = make(pkg, Wd, Hd, cw, ch, mode_flags(pkg, mode))
        dye = seeded_dye(Wd, Hd, 5 + Wd, special=not plant)
        if plant:
            plant_witnesses(dye, cw, ch, rng)
        s.writeField("dye", dye)
        s.dithering = dither
        for kw in range(8):
            set_keywords(s, kw)
            s.config["TRANSPARENT"] = True
            frag = s.render(cw, ch, target=True)
            for transparent in (False, True):
                s.config["TRANSPARENT"] = transparent
                got = s.render_canvas()
                assert got.dtype == np.uint8 and got.shape == (ch, cw, 4)
                want = CM.canvas(frag, BACK_RGB, transparent, cw / ch)
                assert np.array_equal(got, want), (mode, cw, ch, kw, transparent, first_mismatch(got, want))
                for m in CM.MUTANTS:
                    hits[m] += int(np.count_nonzero(CM.canvas(frag, BACK_RGB, transparent, cw / ch, mutant=m) != want))
        s.close()
    assert all(hits.values()), hits


@pytest.mark.parametrize("mode", ["fp32", "half"])
def test_host_and_device_destinations_agree(pkg, torch, dither, mode):
    """A numpy array, the default host array and a slice of a torch uint8 CUDA tensor get the same bytes; the
    poisoned guard bytes on both sides of the slice do not move."""
    cw, ch, G = 96, 80, 64
    n = cw * ch * 4
    s = make(pkg, 64, 48, cw, ch, mode_flags(pkg, mode))
    s.writeField("dye", seeded_dye(64, 48, 3))
    s.dithering = dither
    buf = torch.empty(n + 2 * G, dtype=torch.uint8, device="cuda")
    for kw in (0, SHADING, SUNRAYS, ALL3):
        set_keywords(s, kw)
        for transparent in (False, True):
            s.config["TRANSPARENT"] = transparent
            host = s.render_canvas()
            flat = np.full(n, 0x5A, np.uint8)
            assert s.render_canvas(out=flat).base is flat and np.array_equal(flat.reshape(ch, cw, 4), host)
            buf.fill_(0xA5)
            torch.cuda.synchronize()
            dev = buf[G:G + n]
            assert s.render_canvas(out=dev) is dev
            b = buf.cpu().numpy()
            assert np.all(b[:G] == 0xA5) and np.all(b[G + n:] == 0xA5), (kw, transparent)
            assert np.array_equal(b[G:G + n].reshape(ch, cw, 4), host), (kw, transparent)
            img = torch.empty((ch, cw, 4), dtype=torch.uint8, device="cuda")
            s.render_canvas(out=img)
            assert np.array_equal(img.cpu().numpy(), host), (kw, transparent)
    s.close()


def test_device_destination_waits_for_pending_torch_work(pkg, torch, dither):
    """The handle's stream does not order against torch's, so render_canvas waits for the work still queued on
    the destination.  A fill queued behind a long sleep on torch's current stream, on a side stream, or on
    the stream a version-3 interface names, lands before the canvas; a clone queued behind a sleep reads the
    previous canvas, not the next one."""
    s = make(pkg, 64, 48, 96, 80)
    s.writeField("dye", seeded_dye(64, 48, 21))
    s.dithering = dither
    set_keywords(s, ALL3)
    first = s.render_canvas()
    set_keywords(s, SHADING)
    second = s.render_canvas()
    assert not np.array_equal(first, second)
    t = torch.empty((80, 96, 4), dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    for where in ("current", "side", "v3"):
        torch.cuda.synchronize()
        stream = side if where == "side" else torch.cuda.current_stream()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SLEEP_CYCLES)
            t.fill_(0xA5)
        s.render_canvas(out=V3(t, stream) if where == "v3" else t)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), second), where
    set_keywords(s, ALL3)
    s.render_canvas(out=t)
    torch.cuda._sleep(SLEEP_CYCLES)
    seen = t.clone()                                      # queued behind the sleep on torch's stream
    set_keywords(s, SHADING)
    s.render_canvas(out=t)
    torch.cuda.synchronize()
    assert np.array_equal(seen.cpu().numpy(), first) and np.array_equal(t.cpu().numpy(), second)
    s.close()


def test_canvas_launches_what_render_launches(pkg, torch, dither):
    """Steady state: a canvas launches exactly what render() launches for the same keywords, into host or
    device memory.  Right after render() on the same canvas it launches no more (no post-FX target is
    made again: remaking the bloom FBO would add a fill launch)."""
    s = make(pkg, 64, 64, 128, 128)
    s.writeField("dye", seeded_dye(64, 64, 5))
    s.dithering = dither
    t = torch.empty((128, 128, 4), dtype=torch.uint8, device="cuda")
    for transparent in (False, True):
        s.config["TRANSPARENT"] = transparent
        for kw in range(8):
            set_keywords(s, kw)
            s.render()
            n0 = s.launch_count()
            s.render()
            want = s.launch_count() - n0
            for out in (None, None, t, t):
                n0 = s.launch_count()
                s.render_canvas(out=out)
                assert s.launch_count() - n0 == want, (kw, transparent, out is None)
    s.close()


@pytest.mark.parametrize("mode", ["fp32", "half"])
def test_canvas_writes_nothing_else_in_the_arena(pkg, torch, dither, mode):
    """Under both poisons of the arena guard (every arena byte but dye.read's extent poisoned), a canvas into
    host or device memory changes no arena byte outside what render() may write: nothing, or dye.write
    under SUNRAYS; and its bytes do not depend on the poison."""
    s = make(pkg, 64, 48, 96, 80, mode_flags(pkg, mode))
    g = Arena(torch, s, half=mode == "half")
    s.writeField("dye", seeded_dye(64, 48, 13))
    s.dithering = dither
    t = torch.empty((80, 96, 4), dtype=torch.uint8, device="cuda")
    for kw in range(8):
        set_keywords(s, kw)
        call = "render_sunrays" if kw & SUNRAYS else "render"
        assert A.MAY_CHANGE[call] == (("dye.write",) if kw & SUNRAYS else ())
        for transparent in (False, True):
            s.config["TRANSPARENT"] = transparent
            runs = [g.run(call, lambda: s.render_canvas(), ("dye",), v) for v in POISONS]
            runs += [g.run(call, lambda: s.render_canvas(out=t).cpu().numpy(), ("dye",), v) for v in POISONS]
            assert all(np.array_equal(runs[0], r) for r in runs[1:]), (kw, transparent)
    s.close()


def test_refusals_leave_dst_and_the_handle_alone(pkg, torch, dither):
    """Every bad argument gets FLUID_ERR_INVALID with the poisoned destination unchanged, and the next good
    call on the same handle succeeds."""
    cw, ch = 64, 64
    n = cw * ch * 4
    s = make(pkg, 64, 64, cw, ch, BLOOM_RESOLUTION=32, SUNRAYS_RESOLUTION=24)
    s.writeField("dye", seeded_dye(64, 64, 7))
    s.dithering = dither
    set_keywords(s, ALL3)
    _, fx, dith = pkg.postfx_inputs(s.config, dither)
    good = s.render_canvas()
    L = s._L
    host = np.full(n, 0x5A, np.uint8)
    dev = torch.full((n + 8,), 0x5A, dtype=torch.uint8, device="cuda")
    pinned = L.fluid_host_alloc(n)
    assert pinned
    C.memset(pinned, 0x5A, n)
    torch.cuda.synchronize()
    hp, dp = host.ctypes.data_as(C.c_void_p), dev.data_ptr()
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)        # noqa: E731

    def call(w=cw, h=ch, kw=ALL3, fx_=C.byref(fx), d=ptr(dith), n_=n, dst=hp, on=0):
        return L.fluid_render_canvas(s._h, w, h, kw, 0, fx_, d, dith.shape[1], dith.shape[0], *BACK_RGB,
                                     dst, n_, on)

    bad = [dict(kw=8), dict(kw=ALL3 | 0x10), dict(n_=n - 1), dict(n_=n + 4), dict(n_=0), dict(w=0), dict(h=0),
           dict(w=-3), dict(kw=BLOOM, d=None), dict(kw=BLOOM, fx_=None), dict(kw=SUNRAYS, fx_=None), dict(dst=None),
           dict(on=1), dict(on=1, dst=pinned), dict(on=1, dst=dp + 1), dict(on=1, dst=dp + 2), dict(on=1, dst=dp, n_=n - 4),
           dict(on=1, dst=dp, kw=BLOOM, d=None)]
    if torch.cuda.device_count() > 1:
        other = torch.full((n,), 0x5A, dtype=torch.uint8, device="cuda:1")
        bad.append(dict(on=1, dst=other.data_ptr()))
    out = np.empty((ch, cw, 4), np.uint8)
    for b in bad:
        assert call(**b) == -1, b
        torch.cuda.synchronize()
        assert np.all(host == 0x5A) and bool((dev == 0x5A).all()), b
        assert np.all(np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_uint8)), (n,)) == 0x5A), b
        assert call(dst=ptr(out)) == 0, b
        assert np.array_equal(out, good), b
    assert call(on=1, dst=dp + 4) == 0 and s._L.fluid_sync(s._h) == 0
    assert np.array_equal(dev[4:4 + n].cpu().numpy().reshape(ch, cw, 4), good)
    L.fluid_host_free(pinned)
    s.close()
    # half storage without FLUID_FLAG_HALF_POSTFX draws none / SHADING only, as render() does
    s = make(pkg, 64, 64, cw, ch, pkg.FLAG_HALF_STORAGE)
    s.writeField("dye", seeded_dye(64, 64, 7))
    s.dithering = dither
    for kw in (BLOOM, SUNRAYS, ALL3):
        set_keywords(s, kw)
        with pytest.raises(pkg.FluidError) as e:
            s.render_canvas()
        assert e.value.code == -1 and "HALF_STORAGE" in str(e.value)
    set_keywords(s, SHADING)
    s.config["TRANSPARENT"] = True
    frag = s.render(cw, ch, target=True)
    assert np.array_equal(s.render_canvas(), CM.canvas(frag, BACK_RGB, True, cw / ch))
    s.close()


def test_update_with_canvas_is_update_then_render_canvas(pkg, torch, dither):
    """A seeded session (multipleSplats, a pointer drag, TRANSPARENT switched on half way): update(canvas=t)
    leaves in t, frame after frame, the bytes update() followed by render_canvas() returns."""

    def session(into_tensor):
        rs = np.random.RandomState(11)
        s = pkg.FluidSimulation({"SIM_RESOLUTION": 32, "DYE_RESOLUTION": 64, "SHADING": True, "BLOOM": True,
                                 "SUNRAYS": True, "BLOOM_RESOLUTION": 32, "SUNRAYS_RESOLUTION": 24, "BACK_COLOR": BACK},
                                canvas_width=96, canvas_height=64, random=lambda: float(rs.random_sample()))
        s.dithering = dither
        s.lastUpdateTime = 0.0
        s.splatStack.append(4)
        t = torch.zeros((64, 96, 4), dtype=torch.uint8, device="cuda")
        frames = []
        for k in range(8):
            if k == 2:
                s.updatePointerDownData(s.pointers[0], 0, 30.0, 20.0)
            if 2 <= k <= 4:
                s.updatePointerMoveData(s.pointers[0], 30.0 + 9 * k, 20.0 + 4 * k)
            if k == 5:
                s.config["TRANSPARENT"] = True
            now = 16.0 * (k + 1)
            if into_tensor:
                s.update(now_ms=now, canvas=t)
                frames.append(t.cpu().numpy())
            else:
                s.update(now_ms=now)
                frames.append(s.render_canvas())
        s.close()
        return frames

    a, b = session(True), session(False)
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), (k, first_mismatch(x, y))
    assert len({f.tobytes() for f in a}) == len(a)          # the frames move
