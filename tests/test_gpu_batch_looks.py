"""Batch draws with a look per image (fluid_render_canvas_looks / fluid_capture_looks, and FluidBatch's
render_canvas() / captureScreenshot() with DISPLAY_MEMBER_KEYS in member_config): every image equals, byte for
byte, the draw of an ordinary twin (FluidSimulation) configured with that member's sliders, BACK_COLOR and
TRANSPARENT and holding that member's dye.  Also: equal looks give the shared-look draw's bytes, the launches are
the shared-look draw's, only the drawn members' dye.write moves in the field arena, and every refusal leaves dst
and the handle alone."""
import ctypes as C

import numpy as np
import pytest

import arena_model as A
from display_harness import BACK, KEYS, SETS, nonfinite_dye, seeded_dye, set_keywords
from display_harness import dither  # noqa: F401 -- a fixture
from display_model import ALL3, BLOOM, SUNRAYS
from sim_harness import POISONS, _DeviceBytes, address_range, delta, rand_fields, same_bits
from sim_harness import pkg, torch  # noqa: F401 -- fixtures
from webgl_fluid_simulation_b200 import _lib

pytestmark = pytest.mark.gpu

DEFAULT = (128, 128, 1024, 1024)
SIZES = [DEFAULT, (256, 256, 256, 256), (128, 2, 256, 4), (512, 128, 1024, 256)]     # test_gpu_batch_draw's
FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
CALLS = ("canvas", "capture")
INVALID = -1
NAMES = list(SETS)
# BACK_COLOR of the members in turn: every channel at 0 and at 255, and between
BACKS = [{"r": 0, "g": 255, "b": 0}, {"r": 255, "g": 0, "b": 255}, BACK, {"r": 0, "g": 0, "b": 0},
         {"r": 255, "g": 255, "b": 255}, {"r": 128, "g": 1, "b": 254}]


# ---- handles, looks and draws --------------------------------------------------------------------------------
def shared_config(size, capture_res, fx_res=(64, 48)):
    W, H, Wd, Hd = size
    return {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd), "BACK_COLOR": BACK,
            "CAPTURE_RESOLUTION": capture_res, "BLOOM_RESOLUTION": fx_res[0], "SUNRAYS_RESOLUTION": fx_res[1]}


def look(m, salt=0):
    """Member m's look: a slider set of display_harness.SETS (all ten across ten members, overflow and above
    included), a BACK_COLOR of BACKS, and TRANSPARENT on every third member."""
    k = m + salt
    out = dict(zip(KEYS, SETS[NAMES[k % len(NAMES)]]))
    out.update(BACK_COLOR=dict(BACKS[k % len(BACKS)]), TRANSPARENT=k % 3 == 1)
    return out


def batch(pkg, B, size, canvas, cfg, dither, salt=0):
    b = pkg.FluidBatch(B, dict(cfg), canvas_width=canvas[0], canvas_height=canvas[1], sizes=size)
    assert b.members == B
    b.dithering = dither
    for m in range(B):
        b.member_config[m].update(look(m, salt))
    return b


def twin(pkg, size, canvas, cfg, dither):
    t = pkg.FluidSimulation(dict(cfg), canvas_width=canvas[0], canvas_height=canvas[1], sizes=size)
    t.dithering = dither
    return t


def draw(s, call, out=None, members=None):
    if members is None:
        return s.render_canvas(out=out) if call == "canvas" else s.captureScreenshot(out=out)
    return s.render_canvas(out=out, members=members) if call == "canvas" else s.captureScreenshot(out=out, members=members)


def image_shape(pkg, s, call):
    if call == "canvas":
        return s.canvas["height"], s.canvas["width"]
    r = pkg.getResolution(s.config["CAPTURE_RESOLUTION"], s.canvas["width"], s.canvas["height"])
    return r["height"], r["width"]


def first_mismatch(got, want):
    idx = np.argwhere(got != want)
    return len(idx), (idx[0].tolist(), got[tuple(idx[0])], want[tuple(idx[0])]) if len(idx) else None


def member_dyes(size, B, salt):
    return [seeded_dye(size[2], size[3], 1000 * salt + m) for m in range(B)]


def draw_looks(torch, pkg, b, kws=range(8), members=None):
    """Every keyword set, canvas and capture, into host memory and into a torch uint8 tensor: the host images,
    after checking that both destinations got the same bytes and that the draw went through the _looks call."""
    images = {}
    n = b.members if members is None else len(members)
    for kw in kws:
        set_keywords(b, kw)
        for call in CALLS:
            assert b._looks(None) is not None
            host = draw(b, call, members=members)
            assert host.dtype == np.uint8 and host.shape == (n,) + image_shape(pkg, b, call) + (4,)
            dev = torch.full(host.shape, 0xA5, dtype=torch.uint8, device="cuda")
            assert draw(b, call, dev, members=members) is dev
            assert np.array_equal(dev.cpu().numpy(), host), (kw, call)
            images[kw, call] = host
    return images


def check_twins(t, b, dyes, images, members=None):
    """Image k equals the twin's draw from its member's dye with its member's look."""
    base = dict(t.config)
    for k, m in enumerate(range(len(dyes)) if members is None else members):
        t.writeField("dye", dyes[m])
        t.config.clear()
        t.config.update(base)
        t.config.update(b.member_config[m])
        for (kw, call), got in images.items():
            set_keywords(t, kw)
            want = draw(t, call)
            assert np.array_equal(got[k], want), (k, m, kw, call, first_mismatch(got[k], want))


# ---- 1. every image against its twin --------------------------------------------------------------------------
# (B, size, canvas, CAPTURE_RESOLUTION): B = 1, 5 and 64 on each batch size, ragged, tiny and one-texel canvases,
# captures larger and smaller than the canvas
CASES = [(B, size, canvas, cres) for B in (1, 5, 64) for size, canvas, cres in
         zip(SIZES, [(96, 80), (50, 75), (128, 64), (1, 1)] if B != 64 else [(64, 48), (50, 75), (128, 64), (1, 1)],
             [64, 100, 32, 16])]


@pytest.mark.parametrize("B,size,canvas,capture_res", CASES)
def test_images_equal_twins(pkg, torch, dither, B, size, canvas, capture_res):
    """All eight keyword sets, canvas and capture, host and device: a different dye and look in every member,
    transparent and opaque members in one call."""
    cfg = shared_config(size, capture_res)
    b, t = batch(pkg, B, size, canvas, cfg, dither, salt=B), twin(pkg, size, canvas, cfg, dither)
    dyes = member_dyes(size, B, B)
    b.writeField("dye", np.stack(dyes))
    with np.errstate(invalid="ignore", over="ignore"):
        check_twins(t, b, dyes, draw_looks(torch, pkg, b))
    b.close(); t.close()


def test_subsets_and_nonfinite_member(pkg, torch, dither):
    """Shuffled, single and empty lists: image k equals its member's twin and image members[k] of the whole-batch
    looks draw.  Member 2 holds +-inf, NaN and 1e30 on its corners and edges."""
    size, canvas, B = (256, 256, 256, 256), (96, 80), 7
    cfg = shared_config(size, 64)
    b, t = batch(pkg, B, size, canvas, cfg, dither, salt=3), twin(pkg, size, canvas, cfg, dither)
    dyes = member_dyes(size, B, 7)
    dyes[2] = nonfinite_dye(size[2], size[3], 8)
    b.writeField("dye", np.stack(dyes))
    with np.errstate(invalid="ignore", over="ignore"):
        whole = draw_looks(torch, pkg, b)
        check_twins(t, b, dyes, whole)
        for ms in ([5, 2, 0, 6, 3], [4], [2], []):
            got = draw_looks(torch, pkg, b, members=ms)
            for key, imgs in got.items():
                assert np.array_equal(imgs, whole[key][ms]), (ms, key)
    b.close(); t.close()


# ---- 2. against the shared-look draw --------------------------------------------------------------------------
def uniform_looks(B, c):
    bc = c["BACK_COLOR"]
    one = _lib.Look(c["BLOOM_INTENSITY"], c["BLOOM_THRESHOLD"], c["BLOOM_SOFT_KNEE"], c["SUNRAYS_WEIGHT"],
                    bc["r"] / 255, bc["g"] / 255, bc["b"] / 255, 1 if c["TRANSPARENT"] else 0)
    return (_lib.Look * B)(*([one] * B))


@pytest.mark.parametrize("sliders", ["t033_k07", "overflow"])
def test_equal_looks_give_the_shared_draw_with_its_launches(pkg, torch, dither, sliders):
    """Looks all equal to config's: the bytes of fluid_render_canvas_batch / fluid_capture_batch (and of the
    _members calls for a list), with their launch counts, for every keyword set and TRANSPARENT off and on.
    Distinct looks launch the same."""
    size, canvas, B = (128, 128, 256, 256), (96, 80), 5
    cfg = dict(shared_config(size, 64), **dict(zip(KEYS, SETS[sliders])))
    b = pkg.FluidBatch(B, cfg, canvas_width=canvas[0], canvas_height=canvas[1], sizes=size)
    b.dithering = dither
    b.writeField("dye", np.stack(member_dyes(size, B, 11)))
    ms = [3, 0]
    with np.errstate(invalid="ignore", over="ignore"):
        for kw in range(8):
            for tr in (False, True):
                set_keywords(b, kw)
                b.config["TRANSPARENT"] = tr
                for call in CALLS:
                    for members in (None, ms):
                        b.member_config = [{} for _ in range(B)]
                        shared = draw(b, call, members=members)
                        n_shared = delta(b, "launches", lambda: draw(b, call, members=members))
                        n = B if members is None else len(members)
                        out = np.full((n,) + image_shape(pkg, b, call) + (4,), 0x5A, np.uint8)
                        w, h, args = b._canvas_args() if call == "canvas" else b._capture_args()
                        look_args = (args[0], *args[2:6]) if call == "canvas" else (*args[:3], *args[4:8])
                        fn = b._L.fluid_render_canvas_looks if call == "canvas" else b._L.fluid_capture_looks
                        mp = None if members is None else (C.c_int32 * n)(*members)
                        looks = uniform_looks(n, b.config)
                        n_looks = delta(b, "launches", lambda: fn(b._h, w, h, *look_args, looks,
                                                                   out.ctypes.data_as(C.c_void_p), out.size, 0, mp, n))
                        assert np.array_equal(out, shared), (kw, tr, call, members, first_mismatch(out, shared))
                        assert n_looks == n_shared, (kw, tr, call, members)
                        for m in range(B):                   # distinct looks, through FluidBatch
                            b.member_config[m].update(look(m))
                        assert delta(b, "launches", lambda: draw(b, call, members=members)) == n_shared
    b.close()


# ---- 3. arena guard --------------------------------------------------------------------------------------------
class BatchArena:
    """A batch handle's arena as a uint8 torch tensor: the layout of an ordinary handle whose grids are the B
    members stacked as rows, so member m of a slot is the m-th B-th of the slot's extent."""

    def __init__(self, torch, s, B):
        self.torch, self.s, self.B = torch, s, B
        (W, H), (Wd, Hd) = s._dims("velocity")[:2], s._dims("dye")[:2]
        self.L = L = A.layout(W, B * H, Wd, B * Hd)
        s.sync()
        self.base, asize = address_range(s.device_ptr("velocity"))
        assert asize >= L.bytes
        self.t = torch.as_tensor(_DeviceBytes(self.base, L.bytes), device="cuda")

    def parity(self):
        par = {}
        for f in A.PAIRS:
            off = self.s.device_ptr(f) - self.base
            assert off in (self.L.slot(f, 0), self.L.slot(f, 1)), f
            par[f] = int(off == self.L.slot(f, 1))
        return par

    def run(self, fn, targets, ms, value):
        """Every byte but the .read extents poisoned, fn(), then nothing outside members ms of `targets` moved."""
        torch, L = self.torch, self.L
        par = self.parity()
        keep = [A.extent_range(L, f + ".read" if f in A.PAIRS else f, par) for f in FIELDS]
        saved = [self.t[lo:hi].clone() for lo, hi in keep]
        self.t.fill_(value)
        for (lo, hi), x in zip(keep, saved):
            self.t[lo:hi] = x
        before = self.t.clone()
        torch.cuda.synchronize()
        out = fn()
        self.s.sync()
        assert self.parity() == par
        moved = before != self.t
        for tg in targets:
            lo, hi = A.extent_range(L, tg, par)
            per = (hi - lo) // self.B
            for m in ms:
                moved[lo + m * per:lo + (m + 1) * per] = False
        n = int(moved.sum())
        offs = moved.nonzero()[:8, 0].cpu().numpy() if n else []
        del before, moved
        assert n == 0, (targets, ms, hex(value), n, A.report(L, offs))
        return out


def test_arena_guard(pkg, torch, dither):
    """Under both poisons, a looks draw of the whole batch or of a list moves no arena byte but the drawn members'
    dye.write, and only with SUNRAYS; its bytes do not depend on the poison."""
    size, canvas, B = (128, 128, 256, 256), (96, 80), 4
    b = batch(pkg, B, size, canvas, shared_config(size, 64), dither)
    b.writeField("dye", np.stack(member_dyes(size, B, 13)))
    g = BatchArena(torch, b, B)
    for kw in (ALL3, BLOOM, SUNRAYS, 0):
        set_keywords(b, kw)
        for call in CALLS:
            target = ("dye.write",) if kw & SUNRAYS else ()
            for ms in (None, [3, 1]):
                drawn = range(B) if ms is None else ms
                runs = [g.run(lambda: draw(b, call, members=ms), target, drawn, v) for v in POISONS]
                assert np.array_equal(runs[0], runs[1]), (kw, call, ms)
    b.close()


# ---- 4. refusals -----------------------------------------------------------------------------------------------
def test_refusals_leave_dst_and_the_handle_alone(pkg, torch, dither):
    """Every bad argument gets FLUID_ERR_INVALID with the poisoned host and device destinations unchanged; the batch
    still steps like its twins, and a good call then draws the twins' images."""
    size, canvas, B = (128, 128, 256, 256), (64, 64), 3
    cfg = shared_config(size, 64, (32, 24))
    b = batch(pkg, B, size, canvas, cfg, dither)
    twins = [twin(pkg, size, canvas, cfg, dither) for _ in range(B)]
    data = [rand_fields(*size, 90 + m) for m in range(B)]
    for k, name in enumerate(("velocity", "dye", "pressure")):
        b.writeField(name, np.stack([d[k] for d in data]))
        for t, d in zip(twins, data):
            t.writeField(name, d[k])
    set_keywords(b, ALL3)
    _, fx, dith = pkg.postfx_inputs(b.config, dither)
    looks = b._looks(None)
    w = h = 64
    n = B * 4 * w * h
    L = b._L
    host = np.full(n, 0x5A, np.uint8)
    dev = torch.full((n + 8,), 0x5A, dtype=torch.uint8, device="cuda")
    hp, dp = host.ctypes.data_as(C.c_void_p), dev.data_ptr()
    dptr = dith.ctypes.data_as(C.c_void_p)
    i32 = lambda *v: (C.c_int32 * len(v))(*v)                # noqa: E731

    def call(which, hnd=None, w_=w, h_=h, cw=w, ch=h, kw=ALL3, fx_=C.byref(fx), d=dptr, lk=looks, n_=n, dst=hp, on=0,
             ms=None, k=B):
        hnd = b._h if hnd is None else hnd
        tail = (kw, fx_, d, dith.shape[1], dith.shape[0], lk, dst, n_, on, ms, k)
        if which == "canvas":
            return L.fluid_render_canvas_looks(hnd, w_, h_, *tail)
        return L.fluid_capture_looks(hnd, w_, h_, cw, ch, *tail)

    one = n // B
    bad = [dict(hnd=twins[0]._h), dict(lk=None), dict(lk=None, ms=i32(0), k=1, n_=one), dict(k=B - 1),
           dict(k=B + 1), dict(k=0, n_=0), dict(k=-1), dict(ms=i32(0, 0), k=2, n_=2 * one), dict(ms=i32(B), k=1, n_=one),
           dict(ms=i32(-1), k=1, n_=one), dict(ms=i32(0), k=-1), dict(ms=i32(1, 2), k=2, n_=one),
           dict(n_=one), dict(n_=n - 4), dict(w_=0), dict(h_=-3), dict(kw=8), dict(kw=BLOOM, d=None),
           dict(kw=BLOOM, fx_=None), dict(kw=SUNRAYS, fx_=None), dict(dst=None), dict(on=1), dict(on=1, dst=dp + 1),
           dict(on=1, dst=dp, n_=one), dict(on=1, dst=b.device_ptr("dye"))]
    for which in CALLS:
        dev.fill_(0x5A)
        torch.cuda.synchronize()
        for j, bd in enumerate(bad + ([dict(cw=0), dict(ch=-1)] if which == "capture" else [])):
            assert call(which, **bd) == INVALID, (which, bd)
            torch.cuda.synchronize()
            assert np.all(host == 0x5A) and bool((dev == 0x5A).all()), (which, bd)
            if j % 5 == 0:                                   # the handle stays usable
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
        if which == "canvas":
            for m, t in enumerate(twins):
                t.config.update(b.member_config[m])
                set_keywords(t, ALL3)
                assert np.array_equal(out[m], t.render_canvas()), m
    for name in FIELDS:
        got = b.readField(name)
        for m, t in enumerate(twins):
            assert same_bits(got[m], t.readField(name)), (name, m)
    b.close()
    for t in twins:
        t.close()
