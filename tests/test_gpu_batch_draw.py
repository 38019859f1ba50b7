"""Drawing batch handles (fluid_render_canvas_batch / fluid_capture_batch, FluidBatch.render_canvas and
FluidBatch.captureScreenshot): every member of a batch drawn through one set of launches.  The oracle is an
ordinary handle of the same sizes, canvas and config, its twin, holding that member's dye: member m's image
equals the twin's bit for bit.  The twin's canvas and capture are checked against the display model elsewhere."""
import ctypes as C

import numpy as np
import pytest

import arena_model as A
from display_harness import BACK, BACK_RGB, KEYS, SETS, nonfinite_dye, seeded_dye, set_keywords
from display_harness import dither  # noqa: F401 -- a fixture
from display_model import ALL3, BLOOM, SHADING, SUNRAYS
from sim_harness import POISONS, SLEEP_CYCLES, V3, Arena, _DeviceBytes, address_range, rand_fields, same_bits
from sim_harness import pkg, torch  # noqa: F401 -- fixtures

pytestmark = pytest.mark.gpu

DEFAULT = (128, 128, 1024, 1024)
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
CALLS = ("canvas", "capture")
INVALID = -1


# ---- handles and draws ---------------------------------------------------------------------------------------
def config(size, sliders=None, fx_res=None, capture_res=512):
    """Config keys shared by a batch and its twins: BACK_COLOR (10, 20, 30), a slider set of display_harness.SETS
    (None: the defaults), (BLOOM_RESOLUTION, SUNRAYS_RESOLUTION) (None: the defaults) and CAPTURE_RESOLUTION."""
    W, H, Wd, Hd = size
    c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd), "BACK_COLOR": BACK, "CAPTURE_RESOLUTION": capture_res}
    if sliders is not None:
        c.update(zip(KEYS, SETS[sliders]))
    if fx_res is not None:
        c.update(BLOOM_RESOLUTION=fx_res[0], SUNRAYS_RESOLUTION=fx_res[1])
    return c


def batch(pkg, B, size, canvas, cfg, dither):
    b = pkg.FluidBatch(B, dict(cfg), canvas_width=canvas[0], canvas_height=canvas[1], sizes=size)
    assert b.members == B
    b.dithering = dither
    return b


def twin(pkg, size, canvas, cfg, dither):
    t = pkg.FluidSimulation(dict(cfg), canvas_width=canvas[0], canvas_height=canvas[1], sizes=size)
    assert t._dims("dye")[:2] == size[2:]
    t.dithering = dither
    return t


def draw(s, call, out=None):
    return s.render_canvas(out=out) if call == "canvas" else s.captureScreenshot(out=out)


def image_shape(pkg, s, call):
    """(h, w) of one image of `call` on the handle's canvas and config."""
    if call == "canvas":
        return s.canvas["height"], s.canvas["width"]
    r = pkg.getResolution(s.config["CAPTURE_RESOLUTION"], s.canvas["width"], s.canvas["height"])
    return r["height"], r["width"]


def device_out(torch, pkg, b, call):
    return torch.empty((b.members,) + image_shape(pkg, b, call) + (4,), dtype=torch.uint8, device="cuda")


def requests(kws=range(8)):
    """(keywords, TRANSPARENT, call) of the draws a test makes."""
    return [(kw, tr, call) for kw in kws for tr in (False, True) for call in CALLS]


def configure(s, kw, transparent):
    set_keywords(s, kw)
    s.config["TRANSPARENT"] = transparent


def first_mismatch(got, want):
    idx = np.argwhere(got != want)
    return len(idx), (idx[0].tolist(), got[tuple(idx[0])], want[tuple(idx[0])]) if len(idx) else None


def draw_batch(torch, pkg, b, reqs):
    """Every request into host memory and into a device tensor: the host images, after checking that both
    destinations got the same bytes."""
    images = {}
    for kw, tr, call in reqs:
        configure(b, kw, tr)
        host = draw(b, call)
        assert host.dtype == np.uint8 and host.shape == (b.members,) + image_shape(pkg, b, call) + (4,)
        dev = device_out(torch, pkg, b, call)
        assert draw(b, call, dev) is dev
        assert np.array_equal(dev.cpu().numpy(), host), (kw, tr, call)
        images[kw, tr, call] = host
    return images


def check_twins(t, dyes, images, members=None):
    """Member m of every image equals the twin's draw of the same request from dye m."""
    for m in range(len(dyes)) if members is None else members:
        t.writeField("dye", dyes[m])
        for (kw, tr, call), got in images.items():
            configure(t, kw, tr)
            want = draw(t, call)
            assert np.array_equal(got[m], want), (m, kw, tr, call, first_mismatch(got[m], want))


def member_dyes(size, B, salt):
    return [seeded_dye(size[2], size[3], 1000 * salt + m) for m in range(B)]


# ---- 1. every member against its twin ------------------------------------------------------------------------
# (B, size, canvas, slider set, (BLOOM_RESOLUTION, SUNRAYS_RESOLUTION), CAPTURE_RESOLUTION).  The reference
# desktop frame (1920 x 1080 at the default sizes, default post-FX, a 910 x 512 capture); ragged, tiny and
# one-texel canvases; captures whose target is larger or smaller than the canvas.
CASES = [
    (1, DEFAULT, (1920, 1080), None, None, 512),
    (2, DEFAULT, (1920, 1080), "overflow", None, 256),
    (5, (256, 256, 256, 256), (50, 75), "above", (64, 48), 64),
    (64, (128, 2, 256, 4), (128, 64), "t033_k07", (64, 48), 32),
    (2, (512, 128, 1024, 256), (1, 1), "t0_k1", (64, 48), 16),
    (5, (512, 128, 1024, 256), (128, 64), "t1_k0_i2_w03", None, 100),
    (64, (256, 256, 256, 256), (50, 75), "t0_k0_w4", (32, 24), 48),
    (2, (128, 2, 256, 4), (1, 1), "overflow", None, 8),
]


@pytest.mark.parametrize("B,size,canvas,sliders,fx_res,capture_res", CASES)
def test_members_equal_twins(pkg, torch, dither, B, size, canvas, sliders, fx_res, capture_res):
    """All eight keyword sets, TRANSPARENT off and on, canvas and capture, host and device destinations: a
    different seeded dye in every member, each member's image the twin's."""
    cfg = config(size, sliders, fx_res, capture_res)
    b, t = batch(pkg, B, size, canvas, cfg, dither), twin(pkg, size, canvas, cfg, dither)
    dyes = member_dyes(size, B, B)
    b.writeField("dye", np.stack(dyes))
    with np.errstate(invalid="ignore", over="ignore"):
        check_twins(t, dyes, draw_batch(torch, pkg, b, requests()))
    b.close(); t.close()


# ---- 2. member isolation -------------------------------------------------------------------------------------
def test_nonfinite_member_stays_in_its_images(pkg, torch, dither):
    """The middle member holds +-inf, NaN and 1e30 on its corners and edges, where the samplers clamp: its
    neighbours' images still equal their twins', and so does its own."""
    size, canvas, B = (128, 128, 256, 256), (96, 80), 3
    cfg = config(size, "t005", (64, 48), 64)
    b, t = batch(pkg, B, size, canvas, cfg, dither), twin(pkg, size, canvas, cfg, dither)
    dyes = member_dyes(size, B, 5)
    dyes[1] = nonfinite_dye(size[2], size[3], 8)
    b.writeField("dye", np.stack(dyes))
    with np.errstate(invalid="ignore", over="ignore"):
        check_twins(t, dyes, draw_batch(torch, pkg, b, requests()))
    b.close(); t.close()


# ---- 3. launch counts ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 64])
def test_launch_counts_are_the_twins(pkg, torch, dither, B):
    """A batch draw launches what the twin's draw of the same request launches, post-FX targets made on first use
    included, for every keyword set, into host or device memory."""
    size, canvas = (128, 128, 256, 256), (128, 64)
    cfg = config(size, None, (64, 48), 64)
    b, t = batch(pkg, B, size, canvas, cfg, dither), twin(pkg, size, canvas, cfg, dither)
    b.writeField("dye", np.stack(member_dyes(size, B, 3)))
    t.writeField("dye", seeded_dye(size[2], size[3], 3))
    outs = {call: device_out(torch, pkg, b, call) for call in CALLS}
    for kw, tr, call in requests():
        for s in (b, t):
            configure(s, kw, tr)
        for out in (None, outs[call]):
            n_b = b.launch_count()
            draw(b, call, out)
            n_t = t.launch_count()
            draw(t, call)
            assert b.launch_count() - n_b == t.launch_count() - n_t, (kw, tr, call, out is None)
    b.close(); t.close()


# ---- 4. state ------------------------------------------------------------------------------------------------
def test_draws_leave_every_field_alone(pkg, torch, dither):
    """After every request, each field's .read holds every member's bits from before."""
    size, canvas, B = (128, 128, 256, 256), (64, 48), 3
    b = batch(pkg, B, size, canvas, config(size, None, (32, 24), 32), dither)
    data = [rand_fields(*size, 70 + m) for m in range(B)]
    for k, name in enumerate(("velocity", "dye", "pressure")):
        b.writeField(name, np.stack([d[k] for d in data]))
    b.step(0.016)
    before = {n: b.readField(n) for n in FIELDS}
    for kw, tr, call in requests():
        configure(b, kw, tr)
        draw(b, call)
        for n in FIELDS:
            assert same_bits(b.readField(n), before[n]), (kw, tr, call, n)
    b.close()


def test_session(pkg, torch, dither):
    """splat -> step -> draw -> new sliders and canvas size -> draw -> step, on a batch and one twin per member:
    every field of every member and every image equal the twins' after each call.  The canvas change remakes
    every post-FX target."""
    size, B = (128, 128, 256, 256), 3
    cfg = config(size, None, (64, 48), 64)
    b = batch(pkg, B, size, (96, 80), cfg, dither)
    twins = [twin(pkg, size, (96, 80), cfg, dither) for _ in range(B)]
    handles = [b] + twins

    def same_fields(what):
        for n in FIELDS:
            got = b.readField(n)
            for m, t in enumerate(twins):
                assert same_bits(got[m], t.readField(n)), (what, n, m)

    def same_images(what):
        for kw in (ALL3, BLOOM | SUNRAYS, SHADING):
            for call in CALLS:
                for s in handles:
                    configure(s, kw, False)
                got = draw(b, call)
                for m, t in enumerate(twins):
                    assert np.array_equal(got[m], draw(t, call)), (what, kw, call, m)
        same_fields(what + " (fields)")

    rng = np.random.default_rng(9)
    recs = np.concatenate([rng.uniform(0.2, 0.8, (2 * B, 2)), rng.uniform(-300, 300, (2 * B, 2)),
                           rng.uniform(0, 2, (2 * B, 3))], axis=1).astype(np.float32)
    members = np.repeat(np.arange(B, dtype=np.int32), 2)
    b.splats(members, recs)
    for m, t in enumerate(twins):
        t.splats(recs[members == m])
    same_fields("splats")
    for s in handles:
        s.step(0.016)
    same_fields("step")
    same_images("draw")
    for s in handles:
        s.config.update(zip(KEYS, SETS["t039_k1"]))
        s.config.update(BLOOM_RESOLUTION=48, SUNRAYS_RESOLUTION=40, CAPTURE_RESOLUTION=40)
        s.canvas = {"width": 160, "height": 72}
    same_images("new sliders and canvas")
    for s in handles:
        s.step(0.016)
    same_fields("step after")
    for s in handles:
        s.close()


# ---- 5. arena guard ------------------------------------------------------------------------------------------
class BatchArena(Arena):
    """The guarded arena of a batch handle: its slots hold the B members back to back, the layout of an ordinary
    handle whose grids are the members stacked as rows."""

    def __init__(self, torch, s, members):
        self.members = members
        super().__init__(torch, s)

    def attach(self):
        s, B = self.s, self.members
        (W, H), (Wd, Hd) = s._dims("velocity")[:2], s._dims("dye")[:2]
        self.L = L = A.layout(W, B * H, Wd, B * Hd)
        s.sync()
        self.base, size = address_range(s.device_ptr("velocity"))
        assert size >= L.bytes, (size, L.bytes)
        assert self.base == s.device_ptr("velocity") - L.v[self.parity()["velocity"]]
        self.t = self.torch.as_tensor(_DeviceBytes(self.base, L.bytes), device="cuda")


def test_arena_guard(pkg, torch, dither):
    """Under both poisons (every arena byte but dye.read poisoned), a batch draw into host or device memory moves
    no arena byte outside dye.write, none at all without SUNRAYS, and its bytes do not depend on the poison."""
    size, canvas, B = (128, 128, 256, 256), (96, 80), 3
    b = batch(pkg, B, size, canvas, config(size, None, (64, 48), 64), dither)
    b.writeField("dye", np.stack(member_dyes(size, B, 13)))
    g = BatchArena(torch, b, B)
    for kw, tr, call in requests():
        configure(b, kw, tr)
        guard = "render_sunrays" if kw & SUNRAYS else "render"
        assert A.MAY_CHANGE[guard] == (("dye.write",) if kw & SUNRAYS else ())
        out = device_out(torch, pkg, b, call)
        runs = [g.run(guard, lambda: draw(b, call), ("dye",), v) for v in POISONS]
        runs += [g.run(guard, lambda: draw(b, call, out).cpu().numpy(), ("dye",), v) for v in POISONS]
        assert all(np.array_equal(runs[0], r) for r in runs[1:]), (kw, tr, call)
    b.close()


# ---- 6. more than 2^31 texels in one array -------------------------------------------------------------------
def test_offsets_past_2_31_texels(pkg, torch, dither):
    """4160 members on a 1024 x 512 canvas: the canvases hold 2.18e9 texels (8.7 GB), past 2^31, and the bloom FBO
    and pyramid (512 x 256 per member, fp32 RGBA) 11.6 GB, past 4 GiB.  An offset computed in 32 bits, in
    texels or in bytes, lands on the wrong member: the first and last members equal their twins."""
    size, canvas, B = (128, 2, 128, 2), (1024, 512), 4160
    cfg = config(size, None, None, 512)
    b, t = batch(pkg, B, size, canvas, cfg, dither), twin(pkg, size, canvas, cfg, dither)
    dyes = member_dyes(size, B, 17)
    b.writeField("dye", np.stack(dyes))
    out = torch.empty((B, 512, 1024, 4), dtype=torch.uint8, device="cuda")
    assert out.numel() // 4 > 2 ** 31
    check = (0, 1, 2, B - 3, B - 2, B - 1)
    for call in CALLS:
        assert image_shape(pkg, b, call) == (512, 1024)
        for s in (b, t):
            configure(s, BLOOM | SUNRAYS, False)
        out.fill_(0xA5)
        assert draw(b, call, out) is out
        for m in check:
            t.writeField("dye", dyes[m])
            assert np.array_equal(out[m].cpu().numpy(), draw(t, call)), (call, m)
    del out
    b.close(); t.close()


# ---- 7. ordering and guards ----------------------------------------------------------------------------------
def test_device_destination_ordering_and_guards(pkg, torch, dither):
    """A fill queued behind a long sleep on torch's current stream, on a side stream, or on the stream a version-3
    interface names, lands before the batch's images; poisoned guard bytes around a device slice do not move;
    host and device destinations get the same bytes."""
    size, canvas, B = (128, 128, 256, 256), (96, 80), 5
    b = batch(pkg, B, size, canvas, config(size, None, (64, 48), 64), dither)
    b.writeField("dye", np.stack(member_dyes(size, B, 21)))
    configure(b, ALL3, False)
    side = torch.cuda.Stream()
    for call in CALLS:
        host = draw(b, call)
        t = device_out(torch, pkg, b, call)
        for where in ("current", "side", "v3"):
            torch.cuda.synchronize()
            stream = side if where == "side" else torch.cuda.current_stream()
            with torch.cuda.stream(stream):
                torch.cuda._sleep(SLEEP_CYCLES)
                t.fill_(0xA5)
            draw(b, call, V3(t, stream) if where == "v3" else t)
            torch.cuda.synchronize()
            assert np.array_equal(t.cpu().numpy(), host), (call, where)
        n, G = host.size, 64
        buf = torch.full((n + 2 * G,), 0x5A, dtype=torch.uint8, device="cuda")
        dev = buf[G:G + n]
        assert draw(b, call, dev) is dev
        got = buf.cpu().numpy()
        assert np.all(got[:G] == 0x5A) and np.all(got[G + n:] == 0x5A), call
        assert np.array_equal(got[G:G + n].reshape(host.shape), host), call
        flat = np.full(n, 0x33, np.uint8)
        assert draw(b, call, flat).base is flat and np.array_equal(flat.reshape(host.shape), host), call
    b.close()


# ---- 8. refusals ---------------------------------------------------------------------------------------------
def test_refusals_leave_dst_and_the_handle_alone(pkg, torch, dither):
    """Every bad argument gets FLUID_ERR_INVALID with the poisoned host, pinned and device destinations unchanged;
    the batch still steps like its twins, and a good call then draws the same bytes into host and device memory."""
    size, canvas, B = (128, 128, 256, 256), (64, 64), 3
    cfg = config(size, None, (32, 24), 64)
    b = batch(pkg, B, size, canvas, cfg, dither)
    twins = [twin(pkg, size, canvas, cfg, dither) for _ in range(B)]
    data = [rand_fields(*size, 90 + m) for m in range(B)]
    for k, name in enumerate(("velocity", "dye", "pressure")):
        b.writeField(name, np.stack([d[k] for d in data]))
        for t, d in zip(twins, data):
            t.writeField(name, d[k])
    configure(b, ALL3, False)
    _, fx, dith = pkg.postfx_inputs(b.config, dither)
    w = h = 64
    n = B * 4 * w * h
    L = b._L
    host = np.full(n, 0x5A, np.uint8)
    dev = torch.full((n + 8,), 0x5A, dtype=torch.uint8, device="cuda")
    pinned = L.fluid_host_alloc(n)
    assert pinned
    C.memset(pinned, 0x5A, n)
    hp, dp = host.ctypes.data_as(C.c_void_p), dev.data_ptr()
    dptr = dith.ctypes.data_as(C.c_void_p)

    def call(which, hnd=None, w_=w, h_=h, cw=w, ch=h, kw=ALL3, fx_=C.byref(fx), d=dptr, n_=n, dst=hp, on=0):
        hnd = b._h if hnd is None else hnd
        tail = (kw, 0, fx_, d, dith.shape[1], dith.shape[0], *BACK_RGB, dst, n_, on)
        if which == "canvas":
            return L.fluid_render_canvas_batch(hnd, w_, h_, *tail)
        return L.fluid_capture_batch(hnd, w_, h_, cw, ch, *tail)

    bad = [dict(hnd=twins[0]._h), dict(hnd=twins[0]._h, n_=n // B), dict(n_=n // B), dict(n_=n - 4), dict(n_=0),
           dict(w_=0), dict(h_=0), dict(w_=-3), dict(kw=8), dict(kw=ALL3 | 0x10), dict(kw=BLOOM, d=None),
           dict(kw=BLOOM, fx_=None), dict(kw=SUNRAYS, fx_=None), dict(dst=None), dict(on=1), dict(on=1, dst=pinned),
           dict(on=1, dst=dp + 1), dict(on=1, dst=dp + 2), dict(on=1, dst=dp, n_=n // B),
           dict(on=1, dst=b.device_ptr("dye")), dict(on=1, dst=b.device_ptr("velocity") + 64)]
    for which in CALLS:
        dev.fill_(0x5A)                                      # the good call below writes into dev
        torch.cuda.synchronize()
        for k, bd in enumerate(bad + ([dict(cw=0), dict(ch=-1)] if which == "capture" else [])):
            assert call(which, **bd) == INVALID, (which, bd)
            torch.cuda.synchronize()
            assert np.all(host == 0x5A) and bool((dev == 0x5A).all()), (which, bd)
            assert np.all(np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_uint8)), (n,)) == 0x5A), (which, bd)
            if k % 4 == 0:                                   # the handle stays usable
                b.step(0.016)
                for t in twins:
                    t.step(0.016)
                got = b.readField("dye")
                for m, t in enumerate(twins):
                    assert same_bits(got[m], t.readField("dye")), (which, bd, m)
        assert call(which, on=1, dst=dp + 4) == 0 and L.fluid_sync(b._h) == 0
        out = np.empty((B, h, w, 4), np.uint8)
        assert call(which, dst=out.ctypes.data_as(C.c_void_p)) == 0
        assert np.array_equal(dev[4:4 + n].cpu().numpy().reshape(B, h, w, 4), out), which
    L.fluid_host_free(pinned)
    b.step(0.016)
    for t in twins:
        t.step(0.016)
    for name in FIELDS:
        got = b.readField(name)
        for m, t in enumerate(twins):
            assert same_bits(got[m], t.readField(name)), (name, m)
    b.close()
    for t in twins:
        t.close()
