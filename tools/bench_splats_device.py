"""Splats from host arrays against splats from CUDA arrays, on one handle and on a batch handle.

usage: python tools/bench_splats_device.py [--quick] [--out FILE.json]

  * one handle, fp32, at 4096^2 / 4096^2 and at the reference default 128^2 / 1024^2, n in {1, 24, 128, 1024,
    8192}: fluid_splats (records in the kernel parameter block, ceil(n/128) launches, each reading and writing
    velocity and dye) against fluid_splats_device (one launch, records staged from device memory);
  * a batch of 256 members at 128^2 / 1024^2, with 1 and with 64 records per member in shuffled order:
    fluid_splats_batch (host sort, one launch per 128 records or 64 members) against fluid_splats_batch_device
    (a grouping launch and a splat launch);
  * device time per call between fluid_mark events over windows of >= 0.3 s (one call at least), the two paths
    alternated, 3 rounds: median and range.  Records are already where each path takes them, so the columns
    compare the GPU work; the host path's copy of GPU-made records to the host is not counted here;
  * launches per call, and the seeded results of both paths compared bit for bit at every size.
The card name and power limit come from nvidia-smi (read-only query) and are printed with the numbers."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import webgl_fluid_simulation_b200 as pkg  # noqa: E402

SINGLE = [(4096, 4096, 4096, 4096), (128, 128, 1024, 1024)]
COUNTS = [1, 24, 128, 1024, 8192]
BATCH_B, BATCH_SIZE, PER_MEMBER = 256, (128, 128, 1024, 1024), [1, 64]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                               # the numbers still mean something with the torch name
        import torch
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


def records(n, seed):
    rng = np.random.default_rng(seed)
    r = np.empty((n, 7), np.float32)
    r[:, 0:2] = rng.random((n, 2))
    r[:, 2:4] = rng.uniform(-1000, 1000, (n, 2))
    r[:, 4:7] = rng.uniform(0, 1.5, (n, 3))
    return r


class Timer:
    def __init__(self, s):
        self.s, self.L = s, pkg.lib()

    def per_call(self, call, min_s=0.3):
        """ms of device time per call over a window of >= min_s (one call at least), and launches per call."""
        s, L = self.s, self.L
        call(); s.sync()
        t0 = time.perf_counter(); call(); s.sync()
        reps = max(1, int(min_s / max(time.perf_counter() - t0, 1e-6)))
        l0 = L.fluid_launch_count(s._h)
        s.mark(0)
        for _ in range(reps):
            call()
        s.mark(1)
        s.sync()
        return s.elapsed_ms() / reps, (L.fluid_launch_count(s._h) - l0) / reps


def compare(host_fn, dev_fn, rounds):
    """median / min / max ms of both, alternated; launches per call"""
    h, d = [], []
    for _ in range(rounds):
        t, lh = host_fn(); h.append(t)
        t, ld = dev_fn(); d.append(t)
    st = lambda x: {"median_ms": statistics.median(x), "min_ms": min(x), "max_ms": max(x)}  # noqa: E731
    return {"host": st(h), "device": st(d), "launches": {"host": lh, "device": ld},
            "device_over_host": statistics.median(d) / statistics.median(h)}


def single(torch, size, counts, rounds):
    L = pkg.lib()
    out = []
    a = pkg.FluidSimulation({}, size[0], size[1], device=0, sizes=size)
    b = pkg.FluidSimulation({}, size[0], size[1], device=0, sizes=size)
    ta, tb = Timer(a), Timer(b)
    for n in counts:
        recs = records(n, n)
        t = torch.as_tensor(recs, device="cuda")
        hp, dp = recs.ctypes.data_as(C.POINTER(C.c_float)), t.data_ptr()
        # the same state, one call each: the same bits
        for name in ("velocity", "dye"):
            b.writeField(name, a.readField(name))
        a._check(L.fluid_splats(a._h, hp, n)); b._check(L.fluid_splats_device(b._h, dp, n)); b.sync()
        same = all(np.array_equal(a.readField(f).view(np.uint32), b.readField(f).view(np.uint32)) for f in ("velocity", "dye"))
        r = compare(lambda: ta.per_call(lambda: a._check(L.fluid_splats(a._h, hp, n))),
                    lambda: tb.per_call(lambda: b._check(L.fluid_splats_device(b._h, dp, n))), rounds)
        r.update(size=list(size), n=n, bitwise_equal=bool(same))
        print(json.dumps(r), flush=True)
        out.append(r)
    a.close(); b.close()
    return out


def batch(torch, per_member, rounds, B=BATCH_B):
    L = pkg.lib()
    size = BATCH_SIZE
    a = pkg.FluidBatch(B, {}, sizes=size, device=0)
    b = pkg.FluidBatch(B, {}, sizes=size, device=0)
    ta, tb = Timer(a), Timer(b)
    out = []
    for k in per_member:
        rng = np.random.default_rng(k)
        members = rng.permutation(np.repeat(np.arange(B, dtype=np.int32), k))
        recs = records(len(members), 100 + k)
        n = len(members)
        tm, tr = torch.as_tensor(members, device="cuda"), torch.as_tensor(recs, device="cuda")
        hm, hr = members.ctypes.data_as(C.POINTER(C.c_int32)), recs.ctypes.data_as(C.POINTER(C.c_float))
        for name in ("velocity", "dye"):
            b.writeField(name, a.readField(name))
        a._check(L.fluid_splats_batch(a._h, hm, hr, n))
        b._check(L.fluid_splats_batch_device(b._h, tm.data_ptr(), tr.data_ptr(), n)); b.sync()
        same = all(np.array_equal(a.readField(f).view(np.uint32), b.readField(f).view(np.uint32)) for f in ("velocity", "dye"))
        r = compare(lambda: ta.per_call(lambda: a._check(L.fluid_splats_batch(a._h, hm, hr, n))),
                    lambda: tb.per_call(lambda: b._check(L.fluid_splats_batch_device(b._h, tm.data_ptr(), tr.data_ptr(), n))),
                    rounds)
        r.update(size=list(size), members=B, per_member=k, n=n, bitwise_equal=bool(same))
        print(json.dumps(r), flush=True)
        out.append(r)
    a.close(); b.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--quick", action="store_true", help="small sizes and counts, one round (a rehearsal)")
    ap.add_argument("--out", help="write the results as JSON")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_splats_device needs a CUDA device")
    res = {"card": card(), "single": [], "batch": []}
    print("card:", res["card"], flush=True)
    if args.quick:
        res["single"] += single(torch, (128, 128, 256, 256), [1, 129], 1)
        res["batch"] += batch(torch, [1, 4], 1, B=8)
    else:
        for size in SINGLE:
            res["single"] += single(torch, size, COUNTS, 3)
        res["batch"] += batch(torch, PER_MEMBER, 3)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
