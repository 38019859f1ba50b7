"""Time per member-step of a batch handle (fluid_create_batch) against B ordinary handles stepped in turn.

For each size and B in --members: a FluidBatch of B members and B FluidSimulation handles (graphs both), seeded
with splats, warmed up, then K steps each.  Reported per member-step:
  batch_device_us   device time between fluid_mark events around the batch's K steps
  batch_wall_us     host clock around the same K steps, ended by a sync
  handles_wall_us   host clock around K rounds of one step per ordinary handle, ended by syncing them all
The ordinary handles run on B streams of their own, which the device may overlap, so their cost is the wall
time of a round; there is no single stream to put device events on.  Prints one JSON line per row, then a
markdown table with the card's name and power limit, read in the same run.

    python tools/bench_batch.py [--members 1,8,64,256] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import webgl_fluid_simulation_b200 as pkg  # noqa: E402

# (sim_w, sim_h, dye_w, dye_h, PRESSURE_ITERATIONS): the reference default, and a SAME-dye grid at 50 sweeps
SIZES = [(128, 128, 1024, 1024, 20), (256, 256, 256, 256, 50)]
DT = 0.016666


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in q.split(","))
    except Exception as e:                                   # the table still says what it could not read
        import torch
        name, power = torch.cuda.get_device_name(0), f"unknown ({e.__class__.__name__})"
    return name, power


def records(n, seed):
    rng = np.random.default_rng(seed)
    r = np.empty((n, 7), np.float32)
    r[:, 0:2] = rng.uniform(0.1, 0.9, (n, 2))
    r[:, 2:4] = rng.uniform(-500, 500, (n, 2))
    r[:, 4:7] = rng.uniform(0, 1.5, (n, 3))
    return r


def measure(size, B, steps, warmup):
    W, H, Wd, Hd, iters = size
    cfg = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd), "PRESSURE_ITERATIONS": iters}
    b = pkg.FluidBatch(B, cfg, canvas_width=W, canvas_height=H, sizes=(W, H, Wd, Hd))
    recs = records(4 * B, B)
    b.splats(np.repeat(np.arange(B, dtype=np.int32), 4), recs)
    for _ in range(warmup):
        b.step(DT)
    b.sync()
    t0 = time.perf_counter()
    b.mark(0)
    for _ in range(steps):
        b.step(DT)
    b.mark(1)
    b.sync()
    wall = time.perf_counter() - t0
    dev = b.elapsed_ms() / 1e3
    b.close()

    hs = [pkg.FluidSimulation(cfg, W, H, sizes=(W, H, Wd, Hd)) for _ in range(B)]
    for m, s in enumerate(hs):
        s.splats(recs[4 * m:4 * m + 4])
    for _ in range(warmup):
        for s in hs:
            s.step(DT)
    for s in hs:
        s.sync()
    t0 = time.perf_counter()
    for _ in range(steps):
        for s in hs:
            s.step(DT)
    for s in hs:
        s.sync()
    hwall = time.perf_counter() - t0
    for s in hs:
        s.close()
    n = steps * B
    return {"size": f"{W}x{H}/{Wd}x{Hd} x{iters}", "members": B, "steps": steps,
            "batch_device_us": dev / n * 1e6, "batch_wall_us": wall / n * 1e6, "handles_wall_us": hwall / n * 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", default="1,8,64,256")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for size in SIZES:
        for B in (int(x) for x in a.members.split(",")):
            r = measure(size, B, a.steps, a.warmup)
            r.update(card=name, power_limit=power)
            print(json.dumps(r), flush=True)
            rows.append(r)
    print(f"\n{name}, power limit {power}; microseconds per member-step\n")
    print("| size | B | batch, device | batch, wall | B handles, wall | handles / batch (wall) |")
    print("|---|---:|---:|---:|---:|---:|")
    for r in rows:
        print(f"| {r['size']} | {r['members']} | {r['batch_device_us']:.1f} | {r['batch_wall_us']:.1f} | "
              f"{r['handles_wall_us']:.1f} | {r['handles_wall_us'] / r['batch_wall_us']:.1f} |")


if __name__ == "__main__":
    main()
