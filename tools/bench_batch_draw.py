"""Time per member-frame of a batch handle's draw (fluid_render_canvas_batch / fluid_capture_batch) into a device
tensor, against B ordinary handles each drawing into a device tensor of its own (fluid_render_canvas /
fluid_capture_device).

For each workload and B in its member list: a FluidBatch of B members and B FluidSimulation handles, each member
and handle holding its own seeded dye, warmed up, then K frames each.  Reported per member-frame:
  batch_device_us   device time between fluid_mark events around the batch's K draws
  batch_wall_us     host clock around the same K draws, ended by a sync
  handles_wall_us   host clock around K rounds of one draw per ordinary handle, ended by syncing them all
The draws are queued through the C calls with no sync between them (sim.py's render_canvas(out=...) synchronises
the device and the handle on every call).  The ordinary handles run on B streams of their own, which the device
may overlap, so their cost is the wall time of a round.  Prints one JSON line per row, then a markdown table with
the card's name and power limit, read in the same run.

    python tools/bench_batch_draw.py [--steps 20] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import webgl_fluid_simulation_b200 as pkg  # noqa: E402
from tools.bench_batch import card  # noqa: E402

# (name, (sim_w, sim_h, dye_w, dye_h), canvas, call, CAPTURE_RESOLUTION, members): the reference desktop frame
# with all three keywords, and 256^2 thumbnails for dataset generation
WORKLOADS = [
    ("desktop", (128, 128, 1024, 1024), (1920, 1080), "canvas", 512, (1, 8, 64)),
    ("thumbnail", (128, 128, 256, 256), (256, 256), "canvas", 256, (1, 64, 256)),
    ("thumbnail", (128, 128, 256, 256), (256, 256), "capture", 256, (1, 64, 256)),
]


def dither():
    return np.random.default_rng(0).random((64, 64, 3), dtype=np.float32)


def dye(Wd, Hd, seed):
    d = (np.random.default_rng(seed).random((Hd, Wd, 4), dtype=np.float32) ** 4 * np.float32(3)).astype(np.float32)
    d[..., 3] = 1
    return d


def frame(s, call, out, batch):
    """One draw of `s` into the device tensor `out`, queued on the handle's stream."""
    L = s._L
    if call == "canvas":
        w, h, args = s._canvas_args()
        fn = L.fluid_render_canvas_batch if batch else L.fluid_render_canvas
        rc = fn(s._h, w, h, *args, C.c_void_p(out.data_ptr()), out.numel(), 1)
    else:
        w, h, args = s._capture_args()
        ptr = C.c_void_p(out.data_ptr())
        rc = (L.fluid_capture_batch(s._h, w, h, *args, ptr, out.numel(), 1) if batch
              else L.fluid_capture_device(s._h, w, h, *args, ptr, out.numel()))
    s._check(rc)


def measure(size, canvas, call, capture_res, B, steps, warmup):
    W, H, Wd, Hd = size
    cfg = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd), "SHADING": True, "BLOOM": True,
           "SUNRAYS": True, "CAPTURE_RESOLUTION": capture_res}
    d = dither()
    b = pkg.FluidBatch(B, cfg, canvas_width=canvas[0], canvas_height=canvas[1], sizes=size)
    b.dithering = d
    dyes = [dye(Wd, Hd, m) for m in range(B)]
    b.writeField("dye", np.stack(dyes))
    if call == "canvas":
        h, w = canvas[1], canvas[0]
    else:
        r = pkg.getResolution(capture_res, *canvas)
        h, w = r["height"], r["width"]
    out = torch.empty((B, h, w, 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for _ in range(warmup):
        frame(b, call, out, True)
    b.sync()
    t0 = time.perf_counter()
    b.mark(0)
    for _ in range(steps):
        frame(b, call, out, True)
    b.mark(1)
    b.sync()
    wall = time.perf_counter() - t0
    dev = b.elapsed_ms() / 1e3
    b.close()
    del out

    hs, outs = [], []
    for m in range(B):
        s = pkg.FluidSimulation(cfg, canvas[0], canvas[1], sizes=size)
        s.dithering = d
        s.writeField("dye", dyes[m])
        hs.append(s)
        outs.append(torch.empty((h, w, 4), dtype=torch.uint8, device="cuda"))
    torch.cuda.synchronize()
    for _ in range(warmup):
        for s, o in zip(hs, outs):
            frame(s, call, o, False)
    for s in hs:
        s.sync()
    t0 = time.perf_counter()
    for _ in range(steps):
        for s, o in zip(hs, outs):
            frame(s, call, o, False)
    for s in hs:
        s.sync()
    hwall = time.perf_counter() - t0
    for s in hs:
        s.close()
    n = steps * B
    return {"size": f"{W}x{H}/{Wd}x{Hd}", "canvas": f"{canvas[0]}x{canvas[1]}", "call": call, "image": f"{w}x{h}",
            "members": B, "steps": steps, "batch_device_us": dev / n * 1e6, "batch_wall_us": wall / n * 1e6,
            "handles_wall_us": hwall / n * 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for _, size, canvas, call, cres, members in WORKLOADS:
        for B in members:
            r = measure(size, canvas, call, cres, B, a.steps, a.warmup)
            r.update(card=name, power_limit=power)
            print(json.dumps(r), flush=True)
            rows.append(r)
    print(f"\n{name}, power limit {power}; microseconds per member-frame, SHADING | BLOOM | SUNRAYS\n")
    print("| sim / dye | canvas | call (image) | B | batch, device | batch, wall | B handles, wall | handles / batch (wall) |")
    print("|---|---|---|---:|---:|---:|---:|---:|")
    for r in rows:
        print(f"| {r['size']} | {r['canvas']} | {r['call']} ({r['image']}) | {r['members']} | {r['batch_device_us']:.1f} | "
              f"{r['batch_wall_us']:.1f} | {r['handles_wall_us']:.1f} | {r['handles_wall_us'] / r['batch_wall_us']:.1f} |")


if __name__ == "__main__":
    main()
