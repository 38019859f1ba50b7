"""Splats from CUDA memory (fluid_splats_device / fluid_splats_batch_device, splats() with CUDA arrays).  The
oracle is a twin handle of the same kind and seeded state that takes the same records through the host path
(fluid_splats / fluid_splats_batch, pinned elsewhere against the oracle, the splat model and ordinary twins):
after every call every field equals the twin's bit for bit.  Also: one launch per ordinary call and a constant
per batch call, graphs replayed across device splats, the arena guard, out-of-range members reported by the next
sync with nothing splatted, ordering against a torch side stream, and every refusal."""
import ctypes as C

import numpy as np
import pytest

import arena_model as A
from sim_harness import (SLEEP_CYCLES, V3, Arena, _DeviceBytes, address_range, delta, make, nasty_fields,  # noqa: F401
                         nasty_records, pkg, rand_fields, same_bits, torch)
from splat_model import records

pytestmark = pytest.mark.gpu

FIELDS = ("velocity", "dye", "pressure", "divergence", "curl")
INVALID = -1
DEFAULT = (128, 128, 1024, 1024)


def dev(torch, a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda", dtype=dtype)


def assert_same(a, b, what, fields=FIELDS):
    for name in fields:
        assert same_bits(a.readField(name), b.readField(name)), (what, name)


# ---- ordinary handles ---------------------------------------------------------------------------------------
def kinds(pkg):
    return {"fp32": 0, "half": pkg.FLAG_HALF_STORAGE,
            "desktop": pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX | pkg.FLAG_LINEAR_ADVECTION,
            "nearest": pkg.FLAG_NEAREST_FILTERING}


def twins(pkg, size, flags, seed, **cfg):
    """A device-path handle and its host-path twin with the same nasty fields."""
    a, b = make(pkg, *size, flags=flags, **cfg), make(pkg, *size, flags=flags, **cfg)
    for name, f in zip(("velocity", "dye", "pressure"), nasty_fields(*size, seed)):
        a.writeField(name, f)
        b.writeField(name, f)
    return a, b


NS = (1, 127, 128, 129, 300, 5000)
SIZES = [DEFAULT, (36, 20, 54, 30), (1, 9, 3, 27), (9, 1, 27, 3)]


@pytest.mark.parametrize("kind", ["fp32", "half", "desktop", "nearest"])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s)))
def test_twins(pkg, torch, kind, size):
    """Every n of NS in turn on one pair: the same bits after every call, one launch per device call."""
    W, H, Wd, Hd = size
    a, b = twins(pkg, size, kinds(pkg)[kind], 7)
    for k, n in enumerate(NS):
        recs = records(n, 100 + k, [(W, H), (Wd, Hd)])
        t = dev(torch, recs)
        assert delta(a, "launches", lambda: a.splats(t)) == 1
        b.splats(recs)
        assert_same(a, b, (kind, size, n))
    a.close(); b.close()


def test_twins_4096(pkg, torch):
    size = (4096, 4096, 4096, 4096)
    a, b = twins(pkg, size, 0, 9)
    for k, n in enumerate((24, 129)):
        recs = records(n, 200 + k, [(4096, 4096)])
        a.splats(dev(torch, recs))
        b.splats(recs)
        assert_same(a, b, n, ("velocity", "dye"))
    a.close(); b.close()


@pytest.mark.parametrize("flags", [0, "half"])
def test_ieee_radius_and_aspect(pkg, torch, flags):
    """A canvas of aspect 1.8 (the radius scaled by it) and SPLAT_RADIUS 5e-5, where every warp takes the IEEE
    division; the radius and aspect changing between calls."""
    flags = pkg.FLAG_HALF_STORAGE if flags == "half" else 0
    size = (36, 20, 54, 30)
    a, b = twins(pkg, size, flags, 11)
    for k, rad in enumerate((5e-5, 0.25, 5e-5)):
        for s in (a, b):
            s.config["SPLAT_RADIUS"] = rad
        recs = records(129, 300 + k, [(36, 20), (54, 30)])
        a.splats(dev(torch, recs))
        b.splats(recs)
        assert_same(a, b, rad)
    a.close(); b.close()


def test_zero_records_launch_nothing(pkg, torch):
    a, b = twins(pkg, (36, 20, 54, 30), 0, 13)
    par = {f: a.device_ptr(f) for f in FIELDS}
    assert delta(a, "launches", lambda: a.splats(torch.empty((0, 7), device="cuda"))) == 0
    assert {f: a.device_ptr(f) for f in FIELDS} == par
    assert_same(a, b, "n = 0")
    a.close(); b.close()


@pytest.mark.parametrize("graph", [True, False])
def test_session_with_steps(pkg, torch, graph):
    """Device splats between steps, graph or NO_GRAPH: the twin's bits, and graph steps replay without a new
    capture once both parities have been captured."""
    flags = 0 if graph else pkg.FLAG_NO_GRAPH
    size = (128, 128, 256, 256)
    a, b = twins(pkg, size, flags, 15)
    for k in range(12):
        if k == 4:
            caps = a.stat("graph_captures")
        recs = records(3 + 40 * (k % 3), 400 + k, [(128, 128), (256, 256)])
        a.splats(dev(torch, recs))
        b.splats(recs)
        a.step(0.016 + 0.001 * k); b.step(0.016 + 0.001 * k)
        assert_same(a, b, k)
    if graph:
        assert a.stat("graph_captures") == caps
    a.close(); b.close()


@pytest.mark.parametrize("n,half", [(1, False), (300, False), (129, True)])
def test_arena_guard(pkg, torch, n, half):
    """With every other arena byte poisoned, a device splat call writes only velocity.write and dye.write and
    swaps both pairs; the result is the twin's under both poisons."""
    size = (128, 64, 256, 128)
    flags = pkg.FLAG_HALF_STORAGE if half else 0
    a, b = twins(pkg, size, flags, 17)
    inputs = {name: a.readField(name) for name in ("velocity", "dye")}
    recs = records(n, 500, [(128, 64), (256, 128)])
    t = dev(torch, recs)
    b.splats(recs)
    want = {name: b.readField(name) for name in ("velocity", "dye")}
    g = Arena(torch, a, half=half)
    for value in (0xFF, 0x3C):
        for name, x in inputs.items():
            a.writeField(name, x)
        g.run("splats", lambda: a.splats(t), tuple(inputs), value, swaps=("velocity", "dye"))
        for name in ("velocity", "dye"):
            assert same_bits(a.readField(name), want[name]), (name, hex(value))
    a.close(); b.close()


def test_ordering_against_a_side_stream(pkg, torch):
    """Records written on a torch side stream behind a long sleep: splats() waits for them."""
    size = (128, 128, 256, 256)
    a, b = twins(pkg, size, 0, 19)
    recs = records(200, 600, [(128, 128), (256, 256)])
    src = dev(torch, recs)
    t = torch.zeros((200, 7), device="cuda")
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        t.copy_(src)
    a.splats(t)
    b.splats(recs)
    assert_same(a, b, "torch v2")
    side2 = torch.cuda.Stream()
    with torch.cuda.stream(side2):
        torch.cuda._sleep(SLEEP_CYCLES)
        t.copy_(src.flip(0))
    a.splats(V3(t, side2))
    b.splats(recs[::-1])
    assert_same(a, b, "v3 producer stream")
    a.close(); b.close()


def test_refusals(pkg, torch):
    L = pkg.lib()
    a, b = twins(pkg, (36, 20, 54, 30), 0, 21)
    bt = pkg.FluidBatch(2, {}, sizes=(128, 2, 128, 2))
    recs = records(4, 700, [(36, 20)])
    good = dev(torch, recs)
    pinned = torch.from_numpy(recs).pin_memory()
    host = np.ascontiguousarray(recs)
    mis = torch.zeros(4 * 7 + 1, device="cuda")
    mis_ptr = mis.data_ptr() + 2
    ptrs = {f: a.device_ptr(f) for f in FIELDS}
    cases = [
        ("host", host.ctypes.data, 4), ("pinned", pinned.data_ptr(), 4), ("misaligned", mis_ptr, 4),
        ("arena", a.device_ptr("dye"), 4), ("negative n", good.data_ptr(), -1), ("NULL", None, 4),
    ]
    for what, p, n in cases:
        rc = L.fluid_splats_device(a._h, p, n)
        assert rc == INVALID, what
        assert L.fluid_last_error(a._h), what
        assert {f: a.device_ptr(f) for f in FIELDS} == ptrs, what
        assert_same(a, b, what)
    assert np.array_equal(pinned.numpy(), recs) and np.array_equal(good.cpu().numpy(), recs)
    assert L.fluid_splats_device(bt._h, good.data_ptr(), 4) == INVALID           # a batch handle
    mem = dev(torch, np.zeros(4, np.int32))
    assert L.fluid_splats_batch_device(a._h, mem.data_ptr(), good.data_ptr(), 4) == INVALID   # an ordinary handle
    assert_same(a, b, "wrong kind")
    # still usable
    a.splats(good); b.splats(recs)
    assert_same(a, b, "after refusals")
    bt.close(); a.close(); b.close()


# ---- batch handles ------------------------------------------------------------------------------------------
def batch(pkg, B, size, flags=0, **cfg):
    W, H, Wd, Hd = size
    c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}
    c.update(cfg)
    bt = pkg.FluidBatch(B, c, canvas_width=W, canvas_height=H, sizes=size, flags=flags)
    assert bt.members == B
    return bt


def batch_twins(pkg, B, size, seed, flags=0, radii=None):
    """A device-path batch and its host-path twin, different fields in every member, optional per-member radii."""
    a, b = batch(pkg, B, size, flags), batch(pkg, B, size, flags)
    data = [rand_fields(*size, 1000 * seed + m) for m in range(B)]
    for k, name in enumerate(("velocity", "dye", "pressure")):
        x = np.stack([d[k] for d in data])
        a.writeField(name, x)
        b.writeField(name, x)
    if radii is not None:
        for s in (a, b):
            for m in range(B):
                s.member_config[m]["SPLAT_RADIUS"] = radii[m % len(radii)]
    return a, b


def shuffled(B, n_max, seed):
    """0..n_max records per member in a shuffled call order: some members are named by none."""
    rng = np.random.default_rng(seed)
    members = np.repeat(np.arange(B, dtype=np.int32), rng.integers(0, n_max + 1, B))
    recs = nasty_records(len(members), seed)
    order = rng.permutation(len(members))
    return members[order], recs[order]


def splat_pair(torch, a, b, members, recs):
    """Device call on a, host call on b; members named by no record keep every byte.  Returns the launches."""
    before = {f: a.readField(f) for f in ("velocity", "dye")}
    n = delta(a, "launches", lambda: a.splats(dev(torch, members, torch.int32), dev(torch, recs)))
    b.splats(members, recs)
    assert_same(a, b, ("batch", len(members)))
    idle = np.setdiff1d(np.arange(a.members), members)
    for f, x in before.items():
        assert same_bits(a.readField(f)[idle], x[idle]), f
    return n


BATCH_SIZES = [DEFAULT, (256, 256, 256, 256), (512, 128, 1024, 256), (128, 2, 128, 2)]


@pytest.mark.parametrize("B", [1, 5, 64])
@pytest.mark.parametrize("size", BATCH_SIZES, ids=lambda s: "x".join(map(str, s)))
def test_batch_twins(pkg, torch, B, size):
    """Shuffled records (up to 3 per member, members with none), then every record to one member, with
    per-member radii (one on the IEEE division path); two launches per call whatever B and n."""
    a, b = batch_twins(pkg, B, size, B, radii=(0.25, 5e-5, 0.01, 3.0))
    members, recs = shuffled(B, 3, 10 + B)
    if len(members):
        assert splat_pair(torch, a, b, members, recs) == 2
    m = B // 2
    assert splat_pair(torch, a, b, np.full(300, m, np.int32), nasty_records(300, 20 + B)) == 2
    a.close(); b.close()


def test_batch_launches_are_constant(pkg, torch):
    counts = []
    for B in (1, 64):
        a, b = batch_twins(pkg, B, DEFAULT, 30)
        for n in (1, 5000):
            rng = np.random.default_rng(n)
            counts.append(splat_pair(torch, a, b, rng.integers(0, B, n).astype(np.int32), nasty_records(n, n)))
        a.close(); b.close()
    assert counts == [2, 2, 2, 2]


def test_batch_many_members_one_record_each(pkg, torch):
    B = 4096
    a, b = batch_twins(pkg, B, (128, 2, 128, 2), 40)
    rng = np.random.default_rng(41)
    splat_pair(torch, a, b, rng.permutation(B).astype(np.int32), nasty_records(B, 42))
    members, recs = shuffled(B, 2, 43)                      # and a second call, some members named by none
    splat_pair(torch, a, b, members, recs)
    a.close(); b.close()


@pytest.mark.parametrize("graph", [True, False])
def test_batch_session_with_steps(pkg, torch, graph):
    """Device splats between steps with changing dts: the twin's bits, and graph steps never recapture."""
    flags = 0 if graph else pkg.FLAG_NO_GRAPH
    B = 5
    a, b = batch_twins(pkg, B, DEFAULT, 50, flags=flags, radii=(0.25, 0.5))
    for _ in range(2):                                    # one graph per pressure parity
        a.step(0.016); b.step(0.016)
    caps = a.stat("graph_captures")
    for k in range(6):
        members, recs = shuffled(B, 4, 60 + k)
        if len(members):
            splat_pair(torch, a, b, members, recs)
        dts = [0.016 + 0.001 * (k + m) for m in range(B)]
        a.step(dts); b.step(dts)
        assert_same(a, b, ("step", k))
    assert a.stat("graph_captures") == caps == b.stat("graph_captures")
    a.close(); b.close()


class BatchArena(Arena):
    """The guarded arena of a batch handle: the layout of an ordinary handle whose grids are the B members
    stacked as rows (W x B*H and Wd x B*Hd)."""

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
        self.t = self.torch.as_tensor(_DeviceBytes(self.base, L.bytes), device="cuda")

    def member_range(self, field, side, m, par):
        lo, hi = A.extent_range(self.L, f"{field}.{side}", par)
        n = (hi - lo) // self.members
        return lo + m * n, lo + (m + 1) * n


def test_batch_arena_guard(pkg, torch):
    """Under both poisons a device batch call moves only the named members' .read regions and swaps nothing."""
    B, size = 4, (128, 128, 256, 256)
    a, b = batch_twins(pkg, B, size, 70)
    inputs = {f: a.readField(f) for f in ("velocity", "dye")}
    members, recs = np.array([2, 0, 2, 2], np.int32), nasty_records(4, 71)
    b.splats(members, recs)
    want = {f: b.readField(f) for f in ("velocity", "dye")}
    tm, tr = dev(torch, members, torch.int32), dev(torch, recs)
    g = BatchArena(torch, a, B)
    for value in (0xFF, 0x3C):
        for f, x in inputs.items():
            a.writeField(f, x)
        par = g.poison(tuple(inputs), value)
        before = g.image()
        a.splats(tm, tr)
        moved = np.flatnonzero(before != g.image())
        allowed = [g.member_range(f, "read", m, par) for f in ("velocity", "dye") for m in (0, 2)]
        out = A.outside(moved, allowed)
        assert len(out) == 0, (hex(value), A.report(g.L, out))
        for f in ("velocity", "dye"):
            assert same_bits(a.readField(f), want[f]), (f, hex(value))
    a.close(); b.close()


def test_batch_out_of_range_member(pkg, torch):
    """One bad index: nothing is splatted, the next sync reports it once, and the call after it works."""
    B = 5
    a, b = batch_twins(pkg, B, DEFAULT, 80)
    before = {f: a.readField(f) for f in FIELDS}
    for bad in (5, -1, 70000):
        members = np.array([0, 1, bad, 3, 1], np.int32)
        with pytest.raises(pkg.FluidError):
            a.splats(dev(torch, members, torch.int32), dev(torch, nasty_records(5, 81)))
        a.sync()                                          # reported once
        for f in FIELDS:
            assert same_bits(a.readField(f), before[f]), (bad, f)
    members, recs = shuffled(B, 3, 82)
    splat_pair(torch, a, b, members, recs)
    a.close(); b.close()


def test_batch_ordering_against_a_side_stream(pkg, torch):
    B = 5
    a, b = batch_twins(pkg, B, DEFAULT, 90)
    members, recs = shuffled(B, 6, 91)
    tm, tr = torch.zeros(len(members), dtype=torch.int32, device="cuda"), torch.zeros((len(members), 7), device="cuda")
    sm, sr = dev(torch, members, torch.int32), dev(torch, recs)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        tm.copy_(sm); tr.copy_(sr)
    a.splats(V3(tm, side), V3(tr, side))
    b.splats(members, recs)
    assert_same(a, b, "batch ordering")
    a.close(); b.close()


def test_batch_refusals(pkg, torch):
    L = pkg.lib()
    B = 3
    a, b = batch_twins(pkg, B, (128, 2, 128, 2), 95)
    recs = nasty_records(4, 96)
    members = np.array([0, 2, 1, 0], np.int32)
    gr, gm = dev(torch, recs), dev(torch, members, torch.int32)
    hr, hm = np.ascontiguousarray(recs), np.ascontiguousarray(members)
    mis = torch.zeros(4 * 7 + 1, device="cuda")
    arena = a.device_ptr("dye")
    cases = [
        ("host members", hm.ctypes.data, gr.data_ptr(), 4), ("host records", gm.data_ptr(), hr.ctypes.data, 4),
        ("misaligned members", mis.data_ptr() + 2, gr.data_ptr(), 4),
        ("misaligned records", gm.data_ptr(), mis.data_ptr() + 2, 4),
        ("arena members", arena, gr.data_ptr(), 4), ("arena records", gm.data_ptr(), arena, 4),
        ("negative n", gm.data_ptr(), gr.data_ptr(), -1), ("NULL members", None, gr.data_ptr(), 4),
        ("NULL records", gm.data_ptr(), None, 4),
    ]
    ptrs = {f: a.device_ptr(f) for f in FIELDS}
    for what, pm, pr, n in cases:
        assert L.fluid_splats_batch_device(a._h, pm, pr, n) == INVALID, what
        assert L.fluid_last_error(a._h), what
        assert {f: a.device_ptr(f) for f in FIELDS} == ptrs, what
        assert_same(a, b, what)
    assert np.array_equal(gr.cpu().numpy(), recs) and np.array_equal(gm.cpu().numpy(), members)
    assert L.fluid_splats_batch_device(a._h, None, None, 0) == 0
    assert L.fluid_sync(a._h) == 0
    splat_pair(torch, a, b, members, recs)
    a.close(); b.close()
