"""Member subsets of batch handles: fluid_read_members, fluid_write_members, fluid_reset_members,
fluid_render_canvas_members and fluid_capture_members, and FluidBatch's `members=` keywords and reset() over them.
A subset read or draw equals the matching members of the whole-batch call bit for bit; after a subset write or reset
each member equals its twin (an ordinary handle given that member's inputs) through later splats and steps; every
call writes only its members' extents of the field arena; every bad list or buffer is refused with nothing touched."""
import ctypes as C

import numpy as np
import pytest

import arena_model as A
from display_harness import BACK, BACK_RGB, seeded_dye, set_keywords
from display_harness import dither  # noqa: F401 -- a fixture
from display_model import ALL3, BLOOM, SUNRAYS
from sim_harness import (POISONS, SLEEP_CYCLES, V3, _DeviceBytes, address_range, delta, exp_tiled, make,
                         nasty_fields, nasty_records, rand_fields, same_bits)
from sim_harness import pkg, torch  # noqa: F401 -- fixtures

pytestmark = pytest.mark.gpu

FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
DEFAULT = (128, 128, 1024, 1024)
INVALID = -1
SIZES = [DEFAULT, (128, 2, 256, 4), (512, 128, 1024, 256), (256, 256, 256, 256)]
MEMBER_VALUES = {"CURL": (0.0, 30.0, 1e4, 5.0), "PRESSURE": (0.0, 0.8, 1.0, 2.0),
                 "VELOCITY_DISSIPATION": (0.0, 0.2, 1.0, 4.0), "DENSITY_DISSIPATION": (1.0, 0.0, 4.0, 0.5),
                 "SPLAT_RADIUS": (0.25, 0.01, 3.0, 0.5)}


# ---- handles and data ----------------------------------------------------------------------------------------
def batch(pkg, B, size, flags=0, canvas=None, **cfg):
    W, H, Wd, Hd = size
    c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}
    c.update(cfg)
    cw, ch = canvas or (W, H)
    b = pkg.FluidBatch(B, c, canvas_width=cw, canvas_height=ch, sizes=size, flags=flags)
    assert b.members == B
    return b


def twin(pkg, size, flags=0, **cfg):
    return make(pkg, *size, flags=flags, **cfg)


def give(b, twins, values):
    """Member m's values through member_config, twin m's through its config."""
    for m, t in enumerate(twins):
        for k, v in values.items():
            b.member_config[m][k] = v[m % len(v)]
            t.config[k] = v[m % len(v)]


def member_data(size, B, seed):
    """Five fields of B members: nasty_fields (+-0, subnormals, +-inf, NaN) rolled per member, so no two agree."""
    W, H, Wd, Hd = size
    v, d, p = nasty_fields(W, H, Wd, Hd, seed)
    base = {"velocity": v, "dye": d, "pressure": p, "divergence": np.roll(p, 7), "curl": -np.roll(p, 3)}
    return {n: np.stack([np.roll(a.reshape(-1), 13 * m).reshape(a.shape) for m in range(B)]) for n, a in base.items()}


def write_all(b, data, twins=()):
    for n, a in data.items():
        b.writeField(n, a)
        for m, t in enumerate(twins):
            t.writeField(n, a[m])


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def lists(B, rng):
    """single, all in order, all shuffled, the last, and none"""
    return [[B // 2], list(range(B)), [int(x) for x in rng.permutation(B)], [B - 1], []]


def assert_twins(b, twins, what):
    for n in FIELDS:
        got = b.readField(n)
        for m, t in enumerate(twins):
            assert same_bits(got[m], t.readField(n)), (what, n, m)


def splat_both(b, twins, seed_):
    rng = np.random.default_rng(seed_)
    B = len(twins)
    members = np.repeat(np.arange(B, dtype=np.int32), rng.integers(1, 3, B))
    recs = nasty_records(len(members), seed_)
    b.splats(members, recs)
    for m, t in enumerate(twins):
        t.splats(recs[members == m])


def step_both(b, twins, dts):
    b.step(dts)
    for t, d in zip(twins, dts):
        t.step(float(d))


def close(*handles):
    for h in handles:
        h.close()


# ---- 1. reads ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("B", [1, 5, 64])
def test_reads_equal_the_whole_batch(pkg, torch, B, size):
    """Every list, every field, into host numpy, pinned host, and 16-byte and 4-byte aligned torch memory: slot k is
    member members[k] of the whole-batch read, bit for bit.  A device read is one launch, a host read none; an empty
    list launches nothing."""
    b = batch(pkg, B, size)
    write_all(b, member_data(size, B, 11 * B))
    rng = np.random.default_rng(B)
    L = b._L
    for n in FIELDS:
        whole = b.readField(n)
        per = whole[0].size
        dev = torch.empty(B * per + 1, dtype=torch.float32, device="cuda")
        pinned = L.fluid_host_alloc(4 * B * per)
        assert pinned
        pin = np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_float)), (B * per,))
        for ms in lists(B, rng):
            want = whole[ms]
            k = len(ms) * per
            got = b.readField(n, members=ms)
            assert got.shape == want.shape and np.array_equal(bits(got), bits(want)), (n, ms)
            assert np.array_equal(bits(b.readField(n, out=pin[:k], members=np.array(ms, np.int64))), bits(want)), (n, ms)
            for off in (0, 1):                            # float4 and float copies
                out = dev[off:off + k]
                out.fill_(-7.0)
                launches = delta(b, "launches", lambda: b.readField(n, out=out, members=ms))
                assert launches == (1 if ms else 0), (n, ms, off)
                assert np.array_equal(bits(out.cpu().numpy()), bits(want).reshape(-1)), (n, ms, off)
            assert delta(b, "launches", lambda: b.readField(n, members=ms)) == 0
        L.fluid_host_free(pinned)
        del dev
    close(b)


# ---- 2. writes -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False])
def test_writes_then_splats_and_steps_equal_twins(pkg, torch, graph):
    """Writes of listed members from host memory and from aligned and misaligned device memory, at both parities of
    every pair, then splats and steps with per-member values and dts, under a graph or not: every member equals its
    twin after every call, and members no write lists keep every byte.  One write puts tiny divergence (velocity
    near 2^-130) into a member just before a step."""
    size, B = (128, 128, 256, 256), 5
    flags = 0 if graph else pkg.FLAG_NO_GRAPH
    b = batch(pkg, B, size, flags)
    twins = [twin(pkg, size, flags) for _ in range(B)]
    give(b, twins, MEMBER_VALUES)
    write_all(b, member_data(size, B, 3), twins)
    rng = np.random.default_rng(5)
    W, H, Wd, Hd = size
    plans = [("velocity", [3, 1], "host"), ("dye", [0], "dev"), ("pressure", [4, 2, 0], "dev1"),
             ("divergence", [1], "host"), ("curl", [2, 3], "dev"), ("velocity", [4], "tiny"), ("dye", [2, 4], "dev1")]
    for r, (n, ms, how) in enumerate(plans):
        shape = b.readField(n, members=ms).shape
        if how == "tiny":
            a = exp_tiled(shape[1:], 40 + r, lo=-140, hi=-125)[None]
        else:
            a = (rng.standard_normal(shape) * (0.5 if n == "dye" else 40)).astype(np.float32)
        before = b.readField(n)
        if how.startswith("dev"):
            off = 1 if how == "dev1" else 0
            buf = torch.empty(a.size + off, dtype=torch.float32, device="cuda")
            buf[off:] = torch.from_numpy(a.reshape(-1)).cuda()
            assert delta(b, "launches", lambda: b.writeField(n, buf[off:], members=ms)) == 1
        else:
            assert delta(b, "launches", lambda: b.writeField(n, a, members=ms)) == 0
        after = b.readField(n)
        for k, m in enumerate(ms):
            assert np.array_equal(bits(after[m]), bits(a[k])), (n, ms, m)
            twins[m].writeField(n, a[k])
        for m in set(range(B)) - set(ms):
            assert np.array_equal(bits(after[m]), bits(before[m])), (n, ms, m)
        assert_twins(b, twins, f"write {n} {ms}")
        splat_both(b, twins, 100 + r)
        assert_twins(b, twins, f"splats after {n} {ms}")
        step_both(b, twins, np.array([0.016, 0.01, 1 / 60, 0.0, 0.02], np.float32)[np.roll(np.arange(B), r)])
        assert_twins(b, twins, f"step after {n} {ms}")
    close(b, *twins)


# ---- 3. reset ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False])
def test_reset_members_equal_fresh_twins(pkg, torch, graph):
    """Reset members equal freshly created twins given their member values, through later splats and steps; other
    members are untouched; the reset is one launch and captures no graph, nor does the step after it."""
    size, B = (128, 128, 256, 256), 4
    flags = 0 if graph else pkg.FLAG_NO_GRAPH
    b = batch(pkg, B, size, flags)
    twins = [twin(pkg, size, flags) for _ in range(B)]
    give(b, twins, MEMBER_VALUES)
    write_all(b, {n: a for n, a in member_data(size, B, 8).items() if n in ("velocity", "dye", "pressure")}, twins)
    dts = np.array([0.016, 0.01, 1 / 60, 0.02], np.float32)
    for r in range(3):                                    # both parities of every pair, each with its graph
        splat_both(b, twins, 10 + r)
        step_both(b, twins, dts)
    assert_twins(b, twins, "before reset")
    for ms in ([2, 0], [3], [], list(range(B))):
        before = {n: b.readField(n) for n in FIELDS}
        captures = b.stat("graph_captures")
        assert delta(b, "launches", lambda: b.reset(ms)) == (1 if ms else 0), ms
        for m in ms:
            twins[m].close()
            twins[m] = twin(pkg, size, flags)
            for k, v in MEMBER_VALUES.items():
                twins[m].config[k] = v[m % len(v)]
        for n in FIELDS:
            got = b.readField(n)
            for m in set(range(B)) - set(ms):
                assert np.array_equal(bits(got[m]), bits(before[n][m])), (ms, n, m)
        assert_twins(b, twins, f"reset {ms}")
        splat_both(b, twins, 20 + len(ms))
        assert_twins(b, twins, f"splats after reset {ms}")
        step_both(b, twins, dts)
        assert_twins(b, twins, f"step after reset {ms}")
        assert b.stat("graph_captures") == captures, ms
    close(b, *twins)


# ---- 4. draws ------------------------------------------------------------------------------------------------
def draw(s, call, out=None, members=None):
    if call == "canvas":
        return s.render_canvas(out=out, members=members)
    return s.captureScreenshot(out=out, members=members)


def image_shape(pkg, s, call):
    if call == "canvas":
        return s.canvas["height"], s.canvas["width"]
    r = pkg.getResolution(s.config["CAPTURE_RESOLUTION"], s.canvas["width"], s.canvas["height"])
    return r["height"], r["width"]


def draw_batch(pkg, B, size, canvas, dither):
    b = batch(pkg, B, size, canvas=canvas, BACK_COLOR=BACK, CAPTURE_RESOLUTION=64, BLOOM_RESOLUTION=64,
              SUNRAYS_RESOLUTION=48)
    b.dithering = dither
    b.writeField("dye", np.stack([seeded_dye(size[2], size[3], 300 + m) for m in range(B)]))
    return b


def test_subset_draws_equal_the_whole_batch(pkg, torch, dither):
    """All eight keyword sets, BACK_COLOR and checkerboard / transparent, canvas and capture, into host and device
    memory: image k of a subset draw is image members[k] of the whole-batch draw, byte for byte, with the launches
    of a whole-batch draw; subset and whole draws alternate."""
    size, canvas, B = (256, 256, 256, 256), (50, 75), 5
    b = draw_batch(pkg, B, size, canvas, dither)
    subsets = ([3], [4, 0, 2], [1, 3, 0, 4, 2], [])
    for kw in range(8):
        for tr in (False, True):
            set_keywords(b, kw)
            b.config["TRANSPARENT"] = tr
            for call in ("canvas", "capture"):
                whole = draw(b, call)                     # first: it makes the targets a keyword set adds
                n_whole = delta(b, "launches", lambda: draw(b, call))
                for ms in subsets:
                    n_sub = delta(b, "launches", lambda: draw(b, call, members=ms))
                    assert n_sub == (n_whole if ms else 0), (kw, tr, call, ms)
                    got = draw(b, call, members=ms)
                    assert got.shape == (len(ms),) + image_shape(pkg, b, call) + (4,)
                    assert np.array_equal(got, whole[ms]), (kw, tr, call, ms)
                    dev = torch.full((len(ms),) + image_shape(pkg, b, call) + (4,), 0xA5, dtype=torch.uint8,
                                     device="cuda")
                    assert draw(b, call, dev, members=ms) is dev
                    assert np.array_equal(dev.cpu().numpy(), whole[ms]), (kw, tr, call, ms)
                    assert np.array_equal(draw(b, call), whole), (kw, tr, call, ms)
    close(b)


# ---- 5. arena guard ------------------------------------------------------------------------------------------
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
        assert self.base == s.device_ptr("velocity") - L.v[self.parity()["velocity"]]
        self.t = torch.as_tensor(_DeviceBytes(self.base, L.bytes), device="cuda")

    def parity(self):
        par = {}
        for f in A.PAIRS:
            off = self.s.device_ptr(f) - self.base
            assert off in (self.L.slot(f, 0), self.L.slot(f, 1)), f
            par[f] = int(off == self.L.slot(f, 1))
        return par

    def member_ranges(self, targets, ms, par):
        """Byte ranges of members ms in each of `targets` (field, field.read or field.write)."""
        out = []
        for t in targets:
            lo, hi = A.extent_range(self.L, t, par)
            per = (hi - lo) // self.B
            out += [(lo + m * per, lo + (m + 1) * per) for m in ms]
        return out

    def run(self, fn, targets, ms, value):
        """Every byte but the .read extents poisoned, fn(), then nothing outside members ms of `targets` moved.
        Returns fn()'s result."""
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
        for lo, hi in self.member_ranges(targets, ms, par):
            moved[lo:hi] = False
        n = int(moved.sum())
        offs = moved.nonzero()[:8, 0].cpu().numpy() if n else []
        del before, moved
        assert n == 0, (targets, ms, hex(value), n, A.report(L, offs))
        return out


def test_arena_guard(pkg, torch, dither):
    """Under both poisons: a read moves no arena byte, a write only the listed members' .read of its field, a reset
    both slots of every field of the listed members, a draw only the listed members' dye.write and only with
    SUNRAYS.  Device reads upload the list, so the list buffer lies outside the arena.  Results do not depend on
    the poison."""
    size, canvas, B = (128, 128, 256, 256), (96, 80), 4
    b = draw_batch(pkg, B, size, canvas, dither)
    write_all(b, member_data(size, B, 21))
    g = BatchArena(torch, b, B)
    ms = [3, 1]
    pairs = tuple(f + "." + s for f in A.PAIRS for s in ("read", "write")) + ("divergence", "curl")
    for n in FIELDS:
        dev = torch.empty(b.readField(n, members=ms).size, dtype=torch.float32, device="cuda")
        runs = [g.run(lambda: b.readField(n, members=ms), (), ms, v) for v in POISONS]
        runs += [g.run(lambda: b.readField(n, out=dev, members=ms).cpu().numpy(), (), ms, v) for v in POISONS]
        assert all(np.array_equal(bits(runs[0]), bits(r).reshape(runs[0].shape)) for r in runs[1:]), n
        a = np.random.default_rng(1).standard_normal(runs[0].shape).astype(np.float32)
        target = (n + ".read",) if n in A.PAIRS else (n,)
        for v in POISONS:
            g.run(lambda: b.writeField(n, a, members=ms), target, ms, v)
            assert np.array_equal(bits(b.readField(n, members=ms)), bits(a)), (n, hex(v))
            dev.copy_(torch.from_numpy(a.reshape(-1)))
            g.run(lambda: b.writeField(n, dev, members=ms), target, ms, v)
            assert np.array_equal(bits(b.readField(n, members=ms)), bits(a)), (n, hex(v))
    for v in POISONS:
        g.run(lambda: b.reset(ms), pairs, ms, v)
    write_all(b, member_data(size, B, 22))
    for kw in (ALL3, BLOOM, SUNRAYS, 0):
        set_keywords(b, kw)
        for call in ("canvas", "capture"):
            target = ("dye.write",) if kw & SUNRAYS else ()
            runs = [g.run(lambda: draw(b, call, members=ms), target, ms, v) for v in POISONS]
            assert np.array_equal(runs[0], runs[1]), (kw, call)
    close(b)


# ---- 6. ordering and refusals --------------------------------------------------------------------------------
def test_device_paths_wait_for_torch_streams(pkg, torch, dither):
    """A fill of the destination (read) or source (write) queued behind a long sleep on torch's current stream, a
    side stream, or the stream a version-3 interface names, lands before the call reads or writes it."""
    size, B = (128, 128, 256, 256), 5
    b = draw_batch(pkg, B, size, (96, 80), dither)
    ms = [4, 1]
    side = torch.cuda.Stream()
    want = b.readField("dye", members=ms)
    for where in ("current", "side", "v3"):
        stream = side if where == "side" else torch.cuda.current_stream()
        t = torch.empty(want.shape, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SLEEP_CYCLES)
            t.fill_(-5.0)
        b.readField("dye", out=V3(t, stream) if where == "v3" else t, members=ms)
        torch.cuda.synchronize()
        assert np.array_equal(bits(t.cpu().numpy()), bits(want)), where
        new = np.full(want.shape, 0.25, np.float32) + np.float32(len(where))
        src = torch.zeros(want.shape, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SLEEP_CYCLES)
            src.copy_(torch.from_numpy(new).cuda(non_blocking=False))
        b.writeField("dye", V3(src, stream) if where == "v3" else src, members=ms)
        torch.cuda.synchronize()
        assert np.array_equal(bits(b.readField("dye", members=ms)), bits(new)), where
        b.writeField("dye", want, members=ms)
    for call in ("canvas", "capture"):
        set_keywords(b, ALL3)
        host = draw(b, call, members=ms)
        t = torch.empty(host.shape, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP_CYCLES)
            t.fill_(0xA5)
        draw(b, call, V3(t, side), members=ms)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), host), call
    with pytest.raises(ValueError):
        b.readField("dye", members=torch.tensor(ms, dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):
        b.reset([0.5])
    close(b)


def test_refusals_leave_everything_alone(pkg, torch, dither):
    """Every bad list, size, field, handle and buffer is FLUID_ERR_INVALID: poisoned host, pinned and device
    buffers unchanged, every field of every member unchanged, and the batch still steps like its twins."""
    size, B = (128, 128, 256, 256), 4
    b = batch(pkg, B, size, canvas=(64, 64), BACK_COLOR=BACK, CAPTURE_RESOLUTION=64, BLOOM_RESOLUTION=32,
              SUNRAYS_RESOLUTION=24)
    b.dithering = dither
    twins = [twin(pkg, size) for _ in range(B)]
    data = [rand_fields(*size, 90 + m) for m in range(B)]
    for k, name in enumerate(("velocity", "dye", "pressure")):
        b.writeField(name, np.stack([d[k] for d in data]))
        for t, d in zip(twins, data):
            t.writeField(name, d[k])
    L = b._L
    per = 128 * 128                                       # pressure floats per member
    nbytes = 4 * 2 * per * 4                              # room for two members of velocity
    host = np.full(nbytes, 0x5A, np.uint8)
    dev = torch.full((nbytes + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    pinned = L.fluid_host_alloc(nbytes)
    assert pinned
    C.memset(pinned, 0x5A, nbytes)
    hp, dp = host.ctypes.data_as(C.c_void_p), dev.data_ptr()
    I32 = C.POINTER(C.c_int32)

    def lst(*ms):
        a = np.array(ms, np.int32)
        return a, a.ctypes.data_as(I32)

    def io(fn, hnd=None, field=2, ms=(1, 3), n=None, buf=hp, nf=None, on=0, null=False):
        a, p = lst(*ms)
        n = len(ms) if n is None else n
        nf = n * per if nf is None else nf
        return fn(b._h if hnd is None else hnd, field, None if null else p, n, buf, nf, on)

    def clean():
        torch.cuda.synchronize()
        pin = np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_uint8)), (nbytes,))
        return np.all(host == 0x5A) and bool((dev == 0x5A).all()) and np.all(pin == 0x5A)

    bad_io = [dict(ms=(1, 4)), dict(ms=(-1,)), dict(ms=(2, 2)), dict(ms=(0, 1, 0)), dict(n=-1, ms=()),
              dict(null=True), dict(nf=2 * per - 1), dict(nf=2 * per + 1), dict(nf=per), dict(field=5),
              dict(field=-1), dict(field=0, nf=2 * per), dict(hnd=twins[0]._h), dict(ms=tuple(range(B)) + (0,)),
              dict(on=1, buf=pinned), dict(on=1, buf=dp + 2), dict(on=1, buf=None),
              dict(on=1, buf=b.device_ptr("pressure")), dict(on=1, buf=b.device_ptr("velocity") + 64)]
    before = {n: b.readField(n) for n in FIELDS}

    def unchanged(what):
        for n in FIELDS:
            assert same_bits(b.readField(n), before[n]), (what, n)

    for k, bd in enumerate(bad_io):
        for fn in (L.fluid_read_members, L.fluid_write_members):
            assert io(fn, **bd) == INVALID, (fn.__name__, bd)
            assert clean(), (fn.__name__, bd)
    unchanged("io")
    for ms, n, null, hnd in [((4,), 1, False, None), ((1, 1), 2, False, None), ((), -1, False, None),
                             ((0,), 1, True, None), ((0,), 1, False, twins[0]._h)]:
        a, p = lst(*ms)
        assert L.fluid_reset_members(b._h if hnd is None else hnd, None if null else p, n) == INVALID, (ms, n, null)
    unchanged("reset")
    set_keywords(b, ALL3)
    _, fx, dith = pkg.postfx_inputs(b.config, dither)
    w = h = 64
    img = 4 * w * h

    def drw(which, ms=(2,), n=None, hnd=None, n_=None, dst=dp, on=1, null=False):
        a, p = lst(*ms)
        n = len(ms) if n is None else n
        tail = (ALL3, 0, C.byref(fx), dith.ctypes.data_as(C.c_void_p), dith.shape[1], dith.shape[0], *BACK_RGB, dst,
                n * img if n_ is None else n_, on, None if null else p, n)
        hnd = b._h if hnd is None else hnd
        if which == "canvas":
            return L.fluid_render_canvas_members(hnd, w, h, *tail)
        return L.fluid_capture_members(hnd, w, h, 64, 64, *tail)

    bad_draw = [dict(ms=(4,)), dict(ms=(-2,)), dict(ms=(1, 1)), dict(ms=(), n=-1), dict(null=True), dict(n_=B * img),
                dict(n_=img - 4), dict(hnd=twins[0]._h), dict(on=1, dst=dp + 1), dict(on=1, dst=pinned),
                dict(on=0, dst=None), dict(on=1, dst=b.device_ptr("dye"))]
    for which in ("canvas", "capture"):
        for bd in bad_draw:
            assert drw(which, **bd) == INVALID, (which, bd)
            assert clean(), (which, bd)
    unchanged("draw")
    b.sync()
    for r in range(2):
        step_both(b, twins, np.full(B, 0.016, np.float32))
    assert_twins(b, twins, "after refusals")
    L.fluid_host_free(pinned)
    close(b, *twins)
