"""Device time of a batch handle's member-subset calls against the whole-batch calls they replace, at B = 256 members
of the reference default size (128^2 sim, 1024^2 dye: 16 MiB of dye per member).

  read / write of dye for 1, 16 and 256 members, into and from device memory (fluid_read_members /
      fluid_write_members with a torch tensor: one gather or scatter launch) and pinned host memory (one copy per
      member, then a sync), against fluid_read_device / fluid_write_device and fluid_read / fluid_write of all 256
  reset of 1, 16 and 256 members (fluid_reset_members: one launch)
  canvas and capture of 4 and 16 members on a 256^2 canvas with SHADING | BLOOM | SUNRAYS, into device memory,
      against the whole-batch draw of the same batch

Each row is timed with device events (fluid_mark around `--calls` calls on the handle's stream, host copies
included), repeated `--repeats` times after `--warmup` calls: the median time per call, with the minimum and maximum
of the repeats as its spread.  Prints one JSON line per row, then a markdown table with the card's name and power
limit, read in the same run.

    python tools/bench_batch_members.py [--calls 10] [--repeats 7] [--warmup 2]
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

B = 256
SIZE = (128, 128, 1024, 1024)
DYE = 1024 * 1024 * 4            # floats of dye per member


def timed(b, fn, calls, repeats, warmup):
    """(median, min, max) device milliseconds per call of fn over `repeats` windows of `calls` calls."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    name, power = card()
    W, H, Wd, Hd = SIZE
    cfg = {"SIM_RESOLUTION": 128, "DYE_RESOLUTION": 1024, "SHADING": True, "BLOOM": True, "SUNRAYS": True,
           "CAPTURE_RESOLUTION": 256}
    b = pkg.FluidBatch(B, cfg, canvas_width=256, canvas_height=256, sizes=SIZE)
    b.dithering = np.random.default_rng(0).random((64, 64, 3), dtype=np.float32)
    L, h, F = b._L, b._h, pkg.FIELD["dye"]
    dev = torch.rand(B * DYE, device="cuda")
    b.writeField("dye", dev)
    pinned = L.fluid_host_alloc(4 * B * DYE)
    assert pinned, "no pinned host memory for 256 members of dye"
    rng = np.random.default_rng(1)
    lists = {n: np.ascontiguousarray(rng.permutation(B)[:n], np.int32) for n in (1, 16, 256)}
    ip = lambda m: m.ctypes.data_as(C.POINTER(C.c_int32))
    dptr = lambda: C.c_void_p(dev.data_ptr())
    rows = []

    def row(op, where, n, fn):
        med, lo, hi = timed(b, fn, a.calls, a.repeats, a.warmup)
        r = {"op": op, "dst": where, "members": n, "median_ms": med, "min_ms": lo, "max_ms": hi,
             "card": name, "power_limit": power}
        print(json.dumps(r), flush=True)
        rows.append(r)

    for op, sub, whole_dev, whole_host in (("read", L.fluid_read_members, L.fluid_read_device, L.fluid_read),
                                           ("write", L.fluid_write_members, L.fluid_write_device, L.fluid_write)):
        for n, m in lists.items():
            row(op, "device", n, lambda m=m: b._check(sub(h, F, ip(m), m.size, dptr(), m.size * DYE, 1)))
            row(op, "pinned", n, lambda m=m: b._check(sub(h, F, ip(m), m.size, pinned, m.size * DYE, 0)))
        row(op + " (whole batch)", "device", B, lambda f=whole_dev: b._check(f(h, F, dptr(), B * DYE)))
        row(op + " (whole batch)", "pinned", B, lambda f=whole_host: b._check(f(h, F, pinned, B * DYE)))
    for n, m in lists.items():
        row("reset", "-", n, lambda m=m: b._check(L.fluid_reset_members(h, ip(m), m.size)))
    b.writeField("dye", dev)
    del dev
    for call in ("canvas", "capture"):
        w, hh, args = b._canvas_args() if call == "canvas" else b._capture_args()
        whole_fn, sub_fn = ((L.fluid_render_canvas_batch, L.fluid_render_canvas_members) if call == "canvas"
                            else (L.fluid_capture_batch, L.fluid_capture_members))
        out = torch.empty(B * hh * w * 4, dtype=torch.uint8, device="cuda")
        optr = C.c_void_p(out.data_ptr())
        for n in (4, 16):
            m = np.ascontiguousarray(rng.permutation(B)[:n], np.int32)
            row(call, "device", n, lambda m=m: b._check(sub_fn(h, w, hh, *args, optr, n * 4 * w * hh, 1, ip(m), n)))
        row(call + " (whole batch)", "device", B, lambda: b._check(whole_fn(h, w, hh, *args, optr, B * 4 * w * hh, 1)))
        del out
    b.sync()
    L.fluid_host_free(pinned)
    b.close()
    print(f"\n{name}, power limit {power}; B = {B} at 128^2 / 1024^2, dye (16 MiB per member); draws on a 256^2 canvas, "
          f"SHADING | BLOOM | SUNRAYS; device time per call, median of {a.repeats} x {a.calls} calls (min - max)\n")
    print("| call | buffer | members | ms per call | spread |")
    print("|---|---|---:|---:|---|")
    for r in rows:
        print(f"| {r['op']} | {r['dst']} | {r['members']} | {r['median_ms']:.3f} | {r['min_ms']:.3f} - {r['max_ms']:.3f} |")


if __name__ == "__main__":
    main()
