"""Time per member-step of a parameter sweep on a batch handle (each member its own CURL, PRESSURE, dissipations,
SPLAT_RADIUS and dt, all changed at every step) against a uniform batch (one config and dt for all members).

For each size and B in --members, --rounds rounds alternate the two, so that both see the same state of a shared
machine.  With --parent DIR, each round also times the uniform batch with the package in DIR (another build of this
project, such as the commit before per-member values) in a subprocess, to show what the member table costs a
uniform batch.  Each measurement: a batch seeded with splats, warmed up, then K steps between fluid_mark events
(device time).  Prints one JSON line per measurement, then a markdown table of medians with the card's name and
power limit, read in the same run.

    python tools/bench_batch_sweep.py [--members 64,256] [--steps 20] [--warmup 5] [--rounds 3] [--parent DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.environ.get("BENCH_PKG_ROOT") or os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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


def measure(size, B, steps, warmup, sweep):
    """Device microseconds per member-step."""
    W, H, Wd, Hd, iters = size
    cfg = {"SIM_RESOLUTION": min(W, H), "DYE_RESOLUTION": min(Wd, Hd), "PRESSURE_ITERATIONS": iters}
    b = pkg.FluidBatch(B, cfg, canvas_width=W, canvas_height=H, sizes=(W, H, Wd, Hd))
    L, h = b._L, b._h
    rng = np.random.default_rng(B)
    sweeps = []
    for _ in range(warmup + steps):                          # values and dts of every step, made before timing
        vals = {"CURL": (0, 60), "PRESSURE": (0.5, 1.0), "VELOCITY_DISSIPATION": (0, 1), "DENSITY_DISSIPATION": (0, 2),
                "SPLAT_RADIUS": (0.1, 0.5)}
        arrays = [(pkg.PARAM[k], np.ascontiguousarray(rng.uniform(lo, hi, B))) for k, (lo, hi) in vals.items()]
        dts = (DT * rng.uniform(0.5, 1.0, B)).astype(np.float32)
        sweeps.append(([(k, a.ctypes.data_as(C.POINTER(C.c_double)), a) for k, a in arrays],
                       dts.ctypes.data_as(C.POINTER(C.c_float)), dts))

    def step(k):                                             # the C calls, so that the host stays ahead of the device
        if not sweep:
            return b.step(DT)
        vals, dtp, _ = sweeps[k]
        for key, ptr, _ in vals:
            assert L.fluid_set_param_members(h, key, ptr, B) == 0
        assert L.fluid_step_members(h, dtp, B) == 0

    b.splats(np.repeat(np.arange(B, dtype=np.int32), 4), records(4 * B, B))
    for k in range(warmup):
        step(k)
    b.sync()
    b.mark(0)
    for k in range(steps):
        step(warmup + k)
    b.mark(1)
    b.sync()
    us = b.elapsed_ms() * 1e3 / (steps * B)
    b.close()
    return us


def measure_parent(parent, size, B, steps, warmup):
    env = dict(os.environ, BENCH_PKG_ROOT=os.path.abspath(parent))
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--uniform-once", ",".join(map(str, size)), str(B),
                          str(steps), str(warmup)], env=env, capture_output=True, text=True, check=True).stdout
    return float(out.strip().splitlines()[-1])


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--uniform-once":  # a --parent measurement, in that package
        size = tuple(int(x) for x in sys.argv[2].split(","))
        print(measure(size, int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), sweep=False))
        return
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", default="64,256")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for size in SIZES:
        for B in (int(x) for x in a.members.split(",")):
            t = {"sweep": [], "uniform": [], "uniform_parent": []}
            for r in range(a.rounds):
                t["sweep"].append(measure(size, B, a.steps, a.warmup, sweep=True))
                t["uniform"].append(measure(size, B, a.steps, a.warmup, sweep=False))
                if a.parent:
                    t["uniform_parent"].append(measure_parent(a.parent, size, B, a.steps, a.warmup))
                print(json.dumps({"size": list(size), "members": B, "round": r, "card": name, "power_limit": power,
                                  **{k: v[-1] for k, v in t.items() if v}}), flush=True)
            rows.append((size, B, {k: float(np.median(v)) if v else float("nan") for k, v in t.items()}))
    print(f"\n{name}, power limit {power}; device microseconds per member-step, median of {a.rounds} alternating rounds\n")
    print("| size | B | sweep | uniform | uniform, parent | sweep / uniform |")
    print("|---|---:|---:|---:|---:|---:|")
    for (W, H, Wd, Hd, it), B, m in rows:
        print(f"| {W}x{H}/{Wd}x{Hd} x{it} | {B} | {m['sweep']:.2f} | {m['uniform']:.2f} | {m['uniform_parent']:.2f} | "
              f"{m['sweep'] / m['uniform']:.3f} |")


if __name__ == "__main__":
    main()
