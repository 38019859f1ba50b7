"""splat() / splats() on the GPU against the per-texel interval of tests/splat_model.py: every texel of
velocity and dye must lie within the fp32 arithmetic of the shader with an expf inside EXPF_ULP of
float64 exp, carried through every record and the storage format's rounding.  The base each check
starts from is the field as the library stores it (read back after the write).

Covers fp32 and half storage; the grids of sim_harness.SIZES plus partial 128x16 splat tiles in
both directions; 4096^2 on a subset of rows; one splat() per record and splats() with n = 1, 24 and 129
(across the 128-record launch boundary); SPLAT_RADIUS down to 5e-5, where div_fast_ok fails for every
texel; records on texel centres (d == 0) and far away (e subnormal or 0); canvases of aspect 1, > 1,
< 1 and the one where the radius depends on narrowing the aspect; zero, exponent-tiled and nasty bases.
A readout of the device expf itself closes the file."""
import numpy as np
import pytest

import splat_model as M
from sim_harness import make
from sim_harness import pkg  # noqa: F401 -- a fixture
from splat_model import BASES, CANVASES, GRIDS, NARROWING_CANVAS, RADII, bases, records

pytestmark = pytest.mark.gpu
F32 = np.float32
HALF = 0x10
STORAGE = pytest.mark.parametrize("flags", [0, HALF], ids=["fp32", "half"])


def apply_calls(s, recs, call):
    if call == "splat":
        for x, y, dx, dy, r, g, b in recs.tolist():
            s.splat(x, y, dx, dy, (r, g, b))
    else:
        s.splats(recs)


def check_planes(s, recs, canvas, splat_radius, half, before, rows=None):
    aspect, radius = M.aspect_of(*canvas), M.radius_of(splat_radius, *canvas)
    for name in ("velocity", "dye"):
        got = s.readField(name)
        H = got.shape[0]
        if rows is not None:
            got = got[rows]
        lo, hi = M.splat_interval(before[name], recs, aspect, radius, half=half, rows=rows, H=H)
        n, bad = M.check_splat(got, lo, hi)
        assert n == 0, (name, f"{n} elements outside", bad)


def run(pkg, W, H, Wd, Hd, flags, kind, recs, call, canvas=None, splat_radius=0.25, seed=0):
    s = make(pkg, W, H, Wd, Hd, flags=flags)
    canvas = canvas or (W, H)
    s.canvas = {"width": canvas[0], "height": canvas[1]}
    s.config["SPLAT_RADIUS"] = splat_radius
    v, d = bases(kind, W, H, Wd, Hd, seed)
    s.writeField("velocity", v); s.writeField("dye", d)
    before = {n: s.readField(n) for n in ("velocity", "dye")}
    apply_calls(s, recs, call)
    check_planes(s, recs, canvas, splat_radius, bool(flags & HALF), before)
    s.close()


CALLS = [("splat", 24), ("splats", 1), ("splats", 24), ("splats", 129)]


@STORAGE
@pytest.mark.parametrize("call,n", CALLS, ids=[f"{c}{n}" for c, n in CALLS])
@pytest.mark.parametrize("W,H,Wd,Hd", GRIDS)
def test_every_texel_within_interval(pkg, W, H, Wd, Hd, call, n, flags):
    recs = records(n, W * 5 + H + n, [(W, H), (Wd, Hd)])
    for k, kind in enumerate(BASES):
        run(pkg, W, H, Wd, Hd, flags, kind, recs, call, seed=W + H + k)


@STORAGE
@pytest.mark.parametrize("canvas", CANVASES, ids=lambda c: f"{c[0]}x{c[1]}")
@pytest.mark.parametrize("splat_radius", RADII)
def test_radius_and_canvas_within_interval(pkg, splat_radius, canvas, flags):
    """The radius narrowing canvas (142x100) on the grid where a one-ulp radius moves most texels."""
    W, H, Wd, Hd = 114, 64, 228, 128
    recs = records(129, 17, [(W, H), (Wd, Hd)])
    for k, kind in enumerate(BASES):
        run(pkg, W, H, Wd, Hd, flags, kind, recs, "splats", canvas=canvas, splat_radius=splat_radius, seed=k)


def rows_4096(seed):
    """First and last 16 rows, both sides of 16-row tile seams, and 64 seeded rows."""
    N = 4096
    seams = [s + d for s in (16, 1024, 2048, 2064, 4080) for d in (-1, 0)]
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([np.arange(16), np.arange(N - 16, N), seams, rng.integers(0, N, 64)]))


@STORAGE
@pytest.mark.parametrize("n,kind", [(1, "zero"), (129, "nasty")])
def test_4096_rows_within_interval(pkg, n, kind, flags):
    N = 4096
    recs = records(n, 40 + n, [(N, N)])
    s = make(pkg, N, N, N, N, flags=flags)
    v, d = bases(kind, N, N, N, N, seed=n)
    s.writeField("velocity", v); s.writeField("dye", d)
    del v, d
    rows = rows_4096(n)
    before = {m: s.readField(m)[rows] for m in ("velocity", "dye")}
    s.splats(recs)
    check_planes(s, recs, (N, N), 0.25, bool(flags & HALF), before, rows=rows)
    s.close()


def test_direct_expf_readout(pkg, capsys):
    """Zero dye, colour (1, 1, 1), fp32: dye.rgb is expf(q) itself.  Within EXPF_ULP of exp(float64(q))
    everywhere; the largest distance seen is printed for normal, subnormal and zero results."""
    W = H = 1024
    s = make(pkg, 256, 256, W, H)
    worst = {"normal": 0, "subnormal": 0, "zero": 0}
    count = {"normal": 0, "subnormal": 0, "zero": 0}
    cases = [((1024, 1024), r, xy) for r in RADII for xy in ((0.5, 0.5), (M.uv(W)[300], M.uv(H)[700]), (-0.1, 0.2))]
    cases += [(NARROWING_CANVAS, 0.25, (0.3, 0.6)), ((1024, 2048), 1.0, (0.9, 0.95))]
    for canvas, rad, (x, y) in cases:
        s.canvas = {"width": canvas[0], "height": canvas[1]}
        s.config["SPLAT_RADIUS"] = rad
        s.writeField("dye", np.zeros((H, W, 4), F32))
        s.splat(float(x), float(y), 0.0, 0.0, (1.0, 1.0, 1.0))
        got = s.readField("dye")[..., :3]
        q = M.quotient(M.uv(W), M.uv(H), x, y, M.aspect_of(*canvas), M.radius_of(rad, *canvas))
        ref = M.exp_rn(q)
        dist = np.abs(got.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64)[..., None])
        sub = ref < np.finfo(F32).tiny
        for key, m in (("normal", ~sub), ("subnormal", sub & (ref > 0)), ("zero", ref == 0)):
            if m.any():
                worst[key] = max(worst[key], int(dist[m].max()))
                count[key] += int(m.sum())
        assert not np.signbit(got).any()
        assert dist.max() <= M.EXPF_ULP, (canvas, rad, x, y, int(dist.max()))
    with capsys.disabled():
        print("\n[expf] max ulp distance to exp(float64(q)) rounded to fp32, by the class of that rounded value: " +
              ", ".join(f"{k} {worst[k]} ({count[k]} texels)" for k in worst))
    assert min(count.values()) > 0
    s.close()
