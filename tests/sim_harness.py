"""What the simulation tests share: the fixtures, handles made at exact sizes, their input data, the shape
tables that select each size-selected kernel, the NaN-aware bitwise comparison, the Jacobi launch rule, and
the arena guard -- a handle's field arena poisoned and snapshotted around a call (arena_model holds the
layout).  Test infrastructure; the handles and the arena need the built package and a GPU, the data does not.

Test modules take the fixtures by name (`from sim_harness import pkg, torch`): pytest registers the
fixtures it finds in a test module's namespace, with module scope per importing module."""
import ctypes as C

import numpy as np
import pytest

import arena_model as A
from conftest import bits_equal
from webgl_fluid_simulation_b200 import slab

F = np.float32
POISONS = (0xFF, 0x3C)


# ---- fixtures ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pkg():
    import webgl_fluid_simulation_b200 as p
    return p


@pytest.fixture(scope="module")
def torch():
    import torch as t
    assert t.cuda.is_available()
    return t


# ---- handles -------------------------------------------------------------------------------------------------
def make(pkg, W, H, Wd, Hd, flags=0, jb=0, **cfg):
    c = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd)}
    c.update(cfg)
    # canvas aspect = W/H like the reference; exact sizes are forced through the test hook because
    # getResolution rounds (e.g. a 9x6 dye grid is not reachable from a 7:5 canvas)
    s = pkg.FluidSimulation(c, canvas_width=W, canvas_height=H, flags=flags, jacobi_block=jb,
                            sizes=(W, H, Wd, Hd))
    assert s._dims("velocity")[:2] == (W, H), s._dims("velocity")
    assert s._dims("dye")[:2] == (Wd, Hd), s._dims("dye")
    return s


def solve(s, p, d, iters, pressure, jb=None):
    """fused clear + `iters` sweeps (pressure given) or `iters` sweeps alone (pressure None)"""
    if jb is not None:
        s.set_param("JACOBI_BLOCK", jb)
    s.config["PRESSURE_ITERATIONS"] = iters
    s.config["PRESSURE"] = 1.0 if pressure is None else pressure
    s.writeField("pressure", p); s.writeField("divergence", d)
    if pressure is None:
        s.pass_("jacobi", iters)
    else:
        s.pass_("pressure_solve")
    return s.readField("pressure")


# ---- comparison ----------------------------------------------------------------------------------------------
def same_bits(a, b) -> bool:
    """fp32 arrays equal bit for bit with NaN in the same places, NaN payloads ignored (the device's
    canonical NaN is 0x7fffffff, x86's default NaN 0xffc00000)."""
    a = np.ascontiguousarray(a, F); b = np.ascontiguousarray(b, F)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    keep = ~np.isnan(a)
    return np.array_equal(a.view(np.uint32)[keep], b.view(np.uint32)[keep])


# ---- field and record data -----------------------------------------------------------------------------------
def rand_fields(W, H, Wd, Hd, seed):
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal((H, W, 2)) * 50).astype(np.float32),
            rng.random((Hd, Wd, 4), dtype=np.float32),
            rng.standard_normal((H, W)).astype(np.float32))


def nasty_fields(W, H, Wd, Hd, seed):
    """Seeded fields with -0.0, subnormals, +-inf and NaN sprinkled over ordinary values."""
    rng = np.random.default_rng(seed)

    def sprinkle(a):
        flat = a.reshape(-1)
        specials = np.array([-0.0, 0.0, 1e-40, -3e-39, 1.4e-45, np.inf, -np.inf, np.nan], np.float32)
        k = max(1, flat.size // 7)
        flat[rng.integers(0, flat.size, k)] = rng.choice(specials, k)
        return a
    v = sprinkle((rng.standard_normal((H, W, 2)) * 50).astype(np.float32))
    d = sprinkle(rng.uniform(-1, 2, (Hd, Wd, 4)).astype(np.float32))
    p = rng.standard_normal((H, W)).astype(np.float32)
    return v, d, p


def nasty_records(n, seed):
    """Points inside and outside [0, 1], negative colours, large forces, and far points whose weights
    end in the subnormal range or at zero."""
    rng = np.random.default_rng(seed)
    r = np.empty((n, 7), np.float32)
    r[:, 0:2] = rng.uniform(-0.5, 1.5, (n, 2))
    r[:, 2:4] = rng.uniform(-1, 1, (n, 2)) * 10.0 ** rng.integers(0, 5, (n, 1))
    r[:, 4:7] = rng.uniform(-1.5, 1.5, (n, 3))
    far = rng.random(n) < 0.2
    r[far, 0] = rng.choice([-0.45, 1.45, 3.0, -40.0], far.sum())
    exact = rng.random(n) < 0.1                         # a point on a texel centre: d == 0 there
    r[exact, 0:2] = 0.5
    return r


def special(a, rng):
    """`a` with a quarter of its values replaced by +-0, fp32 and fp16 subnormals, +-inf and NaN (each present)."""
    specials = np.array([-0.0, 0.0, 1e-40, -3e-39, 1.4e-45, 6e-8, -3e-7, np.inf, -np.inf, np.nan], np.float32)
    flat = a.reshape(-1)
    k = flat.size // 4
    flat[rng.choice(flat.size, k, replace=False)] = np.resize(specials, k)
    return a


def special_values(shape, seed, half):
    """Seeded values with a quarter replaced by +-0, fp32 and fp16 subnormals, +-inf and NaN (special); for
    half storage also values that overflow fp16 or sit exactly between two fp16 values."""
    rng = np.random.default_rng(seed)
    a = special((rng.standard_normal(shape) * 50).astype(F), rng)
    if half:
        flat = a.reshape(-1)
        extra = np.array([65520.0, -65520.0, 1e5, -7e4, 65504.0, 65519.0, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11,
                          -(2.0 ** -24) * 1.5, 2.0 ** -25], F)
        k = min(flat.size, 3 * extra.size)
        flat[rng.choice(flat.size, k, replace=False)] = np.resize(extra, k)
    flat = a.reshape(-1)                        # a field of a few cells: NaN and inf all the same
    if not np.isnan(flat).any():
        flat[0] = np.nan
    if not np.isinf(flat).any():
        flat[-1] = -np.inf
    return a


def special_fields(O, W, H, Wd, Hd, seed, half=True):
    """nasty_fields with a band of +-6e4 pressure whose sign flips every two cells in x and y: the cells two
    apart across a flip differ by 1.2e5 (fp16 overflows).  half: rounded to fp16."""
    v, dye, p = nasty_fields(W, H, Wd, Hd, seed)
    s = lambda n: np.where((np.arange(n) // 2) % 2 == 0, 1.0, -1.0).astype(np.float32)
    big = np.float32(6e4) * s(H)[:, None] * s(W)[None, :]
    band = slice(H // 4, max(H // 2, H // 4 + 4))
    p[band] = big[band]
    return tuple(O.round_half(a) for a in (v, dye, p)) if half else (v, dye, p)


CENTRE_SPECIALS = (np.inf, -np.inf, np.nan)


def centre_placements(W, H):
    """{class: (row, col)} of the cells where centre_special_velocity puts its special value.  The manual
    bilerp's velocity sample at a cell centre weighs the +x, +y and +xy neighbours (clamped to the edge) by 0, so
    a special at (r, c) reaches the samples of (r, c - 1), (r - 1, c) and (r - 1, c - 1) and its own.  The
    classes cross the 4-cell kernels' lane layout (column 31 -> 32: lane 31, k = 0 -> lane 0, k = 1), their
    blocks in x (column 127 -> 128) and in y (row 7 -> 8), and sit on the last column and row, where the
    clamped neighbour is the cell itself."""
    p = {"interior": (min(5, H - 1), min(5, W - 1)), "last_col": (H // 2, W - 1), "last_row": (H - 1, min(9, W - 1)),
         "corner": (H - 1, W - 1)}
    if W > 40:
        p["lane"] = (min(3, H - 1), 32)
    if W > 136:
        p["block"] = (min(3, H - 1), 128)
    if H > 10:
        p["row_block"] = (8, min(12, W - 1))
    return p


def centre_special_velocity(W, H, value, comp, seed, coarse=False):
    """Ordinary velocity with `value` (+-inf or NaN) in component `comp` at every centre_placements cell.  The
    cells left of and below each one move up and right, so that their back-traces stay off the special texel and
    only their centre sample meets it; the cell right of it holds a finite -0.0.  coarse: multiples of 4 in
    [-64, 60], which compress (golden files)."""
    rng = np.random.default_rng(seed)
    if coarse:
        v = (rng.integers(-16, 16, (H, W, 2)) * 4).astype(F)
    else:
        v = (rng.standard_normal((H, W, 2)) * 50).astype(F)
    for r, c in centre_placements(W, H).values():
        v[max(r - 1, 0):r + 1, max(c - 1, 0):c + 1] = F(4.0)
        v[r, c, comp] = F(value)
        if c + 1 < W:
            v[r, c + 1, comp] = F(-0.0)
    return v


def exp_tiled(shape, seed, lo=-149, hi=100, tile=(16, 128), zeros=0.03):
    """Random signs and mantissas, one binary exponent in [lo, hi] per tile of (rows, columns) --
    a 128x16 tile is a warp's window of the streaming kernels -- plus exact +-0 cells.  Exponents near
    -149 give subnormals."""
    rng = np.random.default_rng(seed)
    H, W = shape[:2]
    e = rng.integers(lo, hi + 1, (-(-H // tile[0]), -(-W // tile[1])))
    e = np.repeat(np.repeat(e, tile[0], 0), tile[1], 1)[:H, :W]
    e = e.reshape(e.shape + (1,) * (len(shape) - 2))
    m = rng.uniform(1.0, 2.0, shape) * rng.choice([-1.0, 1.0], shape)
    a = np.ldexp(m, e).astype(np.float32)
    z = rng.random(shape) < zeros
    a[z] = np.where(rng.random(int(z.sum())) < 0.5, np.float32(0.0), np.float32(-0.0))
    return a


def far_field(O, W, H, C, seed):
    """Gaussian splats on a zero field (dye: alpha 1): the far field underflows gradually through the
    subnormal range to exact zeros."""
    rng = np.random.default_rng(seed)
    f = np.zeros((H, W, C), np.float32)
    if C == 4:
        f[..., 3] = 1.0
    rad = O.correct_radius(0.25, W / H)
    for _ in range(2):
        x, y = rng.uniform(0.2, 0.8, 2)
        col = rng.uniform(-400, 400, 3) if C == 2 else rng.uniform(0.2, 1.5, 3)
        f = O.splat(f, W / H, float(x), float(y), tuple(float(c) for c in col), rad)
    return f


def near_max_patch(p, d, r0, r1, c0, c1, pressure):
    p[r0:r1, c0:c1] = np.float32(8.5e37 / pressure)
    d[r0 - 1:r1 + 1, c0 - 1:c1 + 1] = np.float32(-1e37)


# ---- shapes --------------------------------------------------------------------------------------------------
SIZES = [(32, 32, 64, 64), (48, 32, 96, 64), (128, 128, 128, 128), (36, 20, 54, 30), (7, 5, 9, 6),
         (256, 64, 512, 128), (1, 9, 3, 27), (9, 1, 27, 3)]
# Grids too small to give every SM a warp stream run the tiled kernels of passes.cuh; these run
# curl_vorticity_divergence_kernel and gradient_subtract_kernel (and (16, 2) at 16 columns too).
TILED_SHAPES = [(64, 40), (128, 128), (256, 96), (16, 2), (132, 77), (520, 33)]
# Grids that select the row-streaming kernels of stream_passes.cuh (cvd: 120 output columns per
# warp, lanes 1..30; gradient: 128 columns, lanes 0..31).  Warp counts from stream_args, for 132 SMs:
#   8x4096    one window; both x walls inside one warp, only lanes 1 and 2 produce output
#   12x4093   W/4 odd; the last 16-row chunk is partial (4093 = 255*16 + 13)
#   124x2050  the second cvd window has one output lane; W % 128 = 124 for gradient
#   964x600   964 = 8*120 + 4: the last cvd window produces only its wall lane
#   132x2051  gradient: the last 128-column window has one live lane; H % 4 = 3, so the GS_U tail re-reads
#   16900xH   141 cvd / 133 gradient windows fill the SMs in one chunk; H = 1 puts both y walls on one
#             row; gradient's last window is a single wall lane
#   1024x512  an ordinary power-of-two grid
STREAM_SHAPES = [(8, 4096), (12, 4093), (124, 2050), (964, 600), (132, 2051), (16900, 1), (16900, 2),
                 (16900, 3), (1024, 512)]


# ---- the Jacobi launch rule ----------------------------------------------------------------------------------
def jacobi_plan(W, H, half, iters, jb=0, naive=False):
    """Depths of the Jacobi launches of a device solve (fluid.cu run_jacobi): JacobiPlan's balanced split
    (slab.jacobi_launches) when the blocked kernel runs (tb_eligible, not FLAG_NAIVE_JACOBI, depth != 1),
    otherwise one sweep per launch."""
    kb = min(jb if jb > 0 else slab.KMAX, slab.KMAX)
    if not half and W % 4 == 0 and W >= 16 and H >= 2 and not naive and kb != 1:
        return slab.jacobi_launches(iters, kb)
    return [1] * iters


def pressure_swaps(n):
    """The pressure pair after n swaps: .read changed slot iff n is odd."""
    return ("pressure",) if n % 2 else ()


# ---- the arena guard -----------------------------------------------------------------------------------------
def address_range(ptr):
    """cuMemGetAddressRange: (base, size) of the allocation holding device address `ptr`."""
    cuda = C.CDLL("libcuda.so.1")
    base, size = C.c_uint64(), C.c_size_t()
    rc = cuda.cuMemGetAddressRange_v2(C.byref(base), C.byref(size), C.c_uint64(ptr))
    assert rc == 0, rc
    return base.value, size.value


class _DeviceBytes:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class Arena:
    """A handle's arena as a uint8 torch tensor, and the guarded call."""

    def __init__(self, torch, s, half=False):
        self.torch, self.s, self.half = torch, s, half
        self.attach()

    def attach(self):
        """(Re)reads the layout from the handle's sizes: after creation and after fluid_resize."""
        s = self.s
        (W, H), (Wd, Hd) = s._dims("velocity")[:2], s._dims("dye")[:2]
        self.L = L = A.layout(W, H, Wd, Hd, self.half)
        s.sync()
        self.base, size = address_range(s.device_ptr("velocity"))
        assert size >= L.bytes, (size, L.bytes)
        par = self.parity()
        assert self.base == s.device_ptr("velocity") - L.v[par["velocity"]]
        self.t = self.torch.as_tensor(_DeviceBytes(self.base, L.bytes), device="cuda")

    def parity(self):
        """The slot each pair's .read is in, from fluid_device_ptr; every .read pointer must sit at a slot."""
        L, par = self.L, {}
        for f in A.PAIRS:
            off = self.s.device_ptr(f) - self.base
            assert off in (L.slot(f, 0), L.slot(f, 1)), (f, off)
            par[f] = int(off == L.slot(f, 1))
        for f in ("divergence", "curl"):
            assert self.s.device_ptr(f) - self.base == L.slot(f), f
        return par

    def poison(self, inputs, value):
        """Every byte but the .read extents of `inputs` set to `value`; returns the parity."""
        par = self.parity()
        self.s.sync()
        keep = [A.extent_range(self.L, f + ".read" if f in A.PAIRS else f, par) for f in inputs]
        saved = [self.t[lo:hi].clone() for lo, hi in keep]
        self.t.fill_(value)
        for (lo, hi), x in zip(keep, saved):
            self.t[lo:hi] = x
        return par

    def image(self):
        self.s.sync()
        return self.t.cpu().numpy()

    def run(self, call, fn, inputs, value, field=None, swaps=None):
        """Poison, snapshot, fn(), snapshot: nothing outside may_change(call) moved.  swaps: the pairs whose
        .read must have changed slot (None: not checked).  Returns fn()'s result."""
        torch, L = self.torch, self.L
        par = self.poison(inputs, value)
        before = self.t.clone()
        torch.cuda.synchronize()
        out = fn()
        self.s.sync()
        after = self.parity()
        if swaps is not None:
            assert after == {f: par[f] ^ (f in swaps) for f in A.PAIRS}, (call, par, after)
        moved = before != self.t
        for lo, hi in A.may_change(call, L, par, field):
            moved[lo:hi] = False
        n = int(moved.sum())
        offs = moved.nonzero()[:8, 0].cpu().numpy() if n else []
        del before, moved
        torch.cuda.synchronize()
        assert n == 0, (call, hex(value), n, A.report(L, offs))
        return out


def check(g, call, fn, inputs, expect, field=None, swaps=None, cmp=bits_equal):
    """g.run under both poisons, inputs written fresh before each; every field of `expect` read back equals
    it (or satisfies it, when callable) and is bit-identical between the two runs."""
    runs = []
    for value in POISONS:
        for n, a in inputs.items():
            g.s.writeField(n, a)
        torch = g.torch
        torch.cuda.synchronize()
        g.run(call, fn, tuple(inputs), value, field, swaps)
        got = {n: g.s.readField(n) for n in expect}
        for n, want in expect.items():
            assert want(got[n]) if callable(want) else cmp(got[n], want), (call, n, hex(value))
        runs.append(got)
    for n in expect:
        assert bits_equal(runs[0][n], runs[1][n]), (call, n)


def delta(s, stat, fn):
    n0 = s.stat(stat)
    fn()
    return s.stat(stat) - n0


# ---- ordering against torch streams ------------------------------------------------------------------------
SLEEP_CYCLES = 200_000_000                               # about 0.1 s of torch.cuda._sleep at 1.98 GHz


class V3:
    """A version-3 __cuda_array_interface__ of tensor `t` naming `stream` as its producer."""

    def __init__(self, t, stream):
        self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, version=3, stream=stream.cuda_stream or 1)
