"""Device time of batch draws where every member has its own look (post-FX sliders, BACK_COLOR, TRANSPARENT): B = 64
and 256 thumbnails (128^2 sim, 256^2 dye and canvas, SHADING | BLOOM | SUNRAYS), canvas and capture, three ways:

  looks      one fluid_render_canvas_looks / fluid_capture_looks call, a look per image
  per-look   one fluid_render_canvas_members / fluid_capture_members call per member, each with that member's
             sliders and background: the only way to draw distinct looks without the _looks calls
  shared     one fluid_render_canvas_batch / fluid_capture_batch call, one look for every member: the floor

Every call draws into device memory.  Each row is timed with device events (fluid_mark around `--calls` rounds on the
handle's stream), repeated `--repeats` times after `--warmup` rounds: the median time per round, with the minimum and
maximum of the repeats as its spread.  Prints one JSON line per row, then a markdown table with the card's name and
power limit, read in the same run.

    python tools/bench_batch_looks.py [--calls 10] [--repeats 7] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import webgl_fluid_simulation_b200 as pkg  # noqa: E402
from tools.bench_batch import card  # noqa: E402

SIZE = (128, 128, 256, 256)
CANVAS = 256


def timed(b, fn, calls, repeats, warmup):
    """(median, min, max) device milliseconds per round of fn over `repeats` windows of `calls` rounds."""
    for _ in range(warmup):
        fn()
    b.sync()
    ms = []
    for _ in range(repeats):
        b.mark(0)
        for _ in range(calls):
            fn()
        b.mark(1)
        ms.append(b.elapsed_ms() / calls)
    return float(np.median(ms)), float(min(ms)), float(max(ms))


def looks_of(B, seed):
    """B distinct looks: sliders around the reference defaults, a random BACK_COLOR, every third member TRANSPARENT."""
    rng = np.random.default_rng(seed)
    out = []
    for m in range(B):
        out.append(dict(BLOOM_INTENSITY=float(rng.uniform(0.1, 2.0)), BLOOM_THRESHOLD=float(rng.uniform(0.0, 1.0)),
                        BLOOM_SOFT_KNEE=float(rng.uniform(0.0, 1.0)), SUNRAYS_WEIGHT=float(rng.uniform(0.0, 2.0)),
                        BACK_COLOR={k: int(v) for k, v in zip("rgb", rng.integers(0, 256, 3))},
                        TRANSPARENT=m % 3 == 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for B in (64, 256):
        cfg = {"SIM_RESOLUTION": 128, "DYE_RESOLUTION": 256, "SHADING": True, "BLOOM": True, "SUNRAYS": True,
               "CAPTURE_RESOLUTION": CANVAS}
        b = pkg.FluidBatch(B, cfg, canvas_width=CANVAS, canvas_height=CANVAS, sizes=SIZE)
        b.dithering = np.random.default_rng(0).random((64, 64, 3), dtype=np.float32)
        b.writeField("dye", torch.rand(B * SIZE[2] * SIZE[3] * 4, device="cuda") ** 4 * 3)
        looks = looks_of(B, B)
        L, h = b._L, b._h
        for call in ("canvas", "capture"):
            fns = ((L.fluid_render_canvas_batch, L.fluid_render_canvas_members, L.fluid_render_canvas_looks)
                   if call == "canvas" else (L.fluid_capture_batch, L.fluid_capture_members, L.fluid_capture_looks))
            b.member_config = [{} for _ in range(B)]
            w, hh, args = b._canvas_args() if call == "canvas" else b._capture_args()
            per = 4 * w * hh
            out = torch.empty(B * per, dtype=torch.uint8, device="cuda")
            optr = C.c_void_p(out.data_ptr())
            # one member's call with its own look: the shared call's arguments with its sliders and background
            single, base = [], dict(b.config)
            for m in range(B):
                b.config.update(looks[m])
                single.append((np.array([m], np.int32),) + (b._canvas_args() if call == "canvas" else b._capture_args()))
            b.config = base
            for m in range(B):
                b.member_config[m].update(looks[m])
            table = b._looks(None)
            look_args = (args[0], *args[2:6]) if call == "canvas" else (*args[:3], *args[4:8])

            def row(way, fn):
                med, lo, hi = timed(b, fn, a.calls, a.repeats, a.warmup)
                r = {"call": call, "members": B, "way": way, "median_ms": med, "min_ms": lo, "max_ms": hi,
                     "card": name, "power_limit": power}
                print(json.dumps(r), flush=True)
                rows.append(r)

            def per_look():
                for k, (m, _, _, ar) in enumerate(single):
                    b._check(fns[1](h, w, hh, *ar, C.c_void_p(out.data_ptr() + k * per), per, 1,
                                    m.ctypes.data_as(C.POINTER(C.c_int32)), 1))

            row("looks", lambda: b._check(fns[2](h, w, hh, *look_args, table, optr, B * per, 1, None, B)))
            row("per-look", per_look)
            row("shared", lambda: b._check(fns[0](h, w, hh, *args, optr, B * per, 1)))
            del out
        b.sync()
        b.close()
    print(f"\n{name}, power limit {power}; B thumbnails at 128^2 sim / 256^2 dye on a 256^2 canvas (capture 256^2), "
          f"SHADING | BLOOM | SUNRAYS, a look per member; device time per draw of all B images, median of "
          f"{a.repeats} x {a.calls} (min - max)\n")
    print("| call | B | way | ms | spread | µs per image |")
    print("|---|---:|---|---:|---|---:|")
    for r in rows:
        print(f"| {r['call']} | {r['members']} | {r['way']} | {r['median_ms']:.3f} | {r['min_ms']:.3f} - "
              f"{r['max_ms']:.3f} | {1000 * r['median_ms'] / r['members']:.1f} |")


if __name__ == "__main__":
    main()
