"""What moving a field costs: fluid_read_device / fluid_write_device against fluid_read / fluid_write into pinned
host memory.

usage: python tools/bench_device_io.py [--calls K] [--host-calls KH] [--repeats R] [--out FILE.json]

  * sizes: the reference default (128^2 sim, 1024^2 dye) and 4096^2 / 4096^2; fields velocity (float2) and dye
    (float4); storage fp32 and FLUID_FLAG_HALF_STORAGE;
  * device path: K calls between two fluid_mark events on the handle's stream, device ms per call (the calls
    return without synchronising; one fluid_elapsed_ms waits for the window), into or out of a torch float32
    CUDA tensor;
  * host path: KH calls of fluid_read / fluid_write into or out of fluid_host_alloc memory, host ms per call
    (perf_counter; every call synchronises the stream itself);
  * bytes per device call, computed from the shapes: the fp32 field read plus written (8 B per element), or
    the fp16 field and the fp32 buffer (6 B per element) in half storage; that over the device time, and as a
    share of the H100 SXM data-sheet HBM3 figure of 3.35 TB/s (a data-sheet number, not one this run reached);
  * median and range over R repeats after a warm-up, the paths interleaved; the device read is checked bit for
    bit against the host read.
The card name and power limit come from nvidia-smi (read-only query) in the same run."""
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

DATASHEET_HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet, HBM3
SIZES = {"128^2/1024^2": (128, 128, 1024, 1024), "4096^2/4096^2": (4096, 4096, 4096, 4096)}
STORAGE = {"fp32": 0, "half_storage": pkg.FLAG_HALF_STORAGE}
FIELDS = ("velocity", "dye")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                  # the timing below still needs the GPU
        return {"name": "unknown", "error": str(e)}


def summary(xs):
    return {"median": round(statistics.median(xs), 5), "min": round(min(xs), 5), "max": round(max(xs), 5)}


def device_ms(s, fn, k):
    s.sync()
    s.mark(0)
    for _ in range(k):
        fn()
    s.mark(1)
    return s.elapsed_ms() / k


def host_ms(s, fn, k):
    s.sync()
    t0 = time.perf_counter()
    for _ in range(k):
        fn()
    return (time.perf_counter() - t0) * 1e3 / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--host-calls", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    L = pkg.lib()
    result = {"card": card(), "calls_per_window": a.calls, "host_calls_per_window": a.host_calls, "repeats": a.repeats,
              "datasheet_hbm_TB_s": DATASHEET_HBM_BYTES_PER_S / 1e12, "cases": {}}
    for size_name, sizes in SIZES.items():
        for storage, flags in STORAGE.items():
            s = pkg.FluidSimulation({}, canvas_width=sizes[0], canvas_height=sizes[1], flags=flags, sizes=sizes)
            for field in FIELDS:
                fid = pkg.FIELD[field]
                w, h, c, _ = s._dims(field)
                n = w * h * c
                src = torch.rand(n, dtype=torch.float32, device="cuda") * 8 - 4
                dst = torch.empty(n, dtype=torch.float32, device="cuda")
                pinned = C.c_void_p(L.fluid_host_alloc(4 * n))
                assert pinned.value, "fluid_host_alloc failed"
                torch.cuda.synchronize()
                sp, dp = C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr())
                paths = {
                    "read_device": (device_ms, lambda: s._check(L.fluid_read_device(s._h, fid, dp, n)), a.calls),
                    "write_device": (device_ms, lambda: s._check(L.fluid_write_device(s._h, fid, sp, n)), a.calls),
                    "read_host_pinned": (host_ms, lambda: s._check(L.fluid_read(s._h, fid, pinned, n)), a.host_calls),
                    "write_host_pinned": (host_ms, lambda: s._check(L.fluid_write(s._h, fid, pinned, n)), a.host_calls),
                }
                for clock, fn, _ in paths.values():
                    clock(s, fn, 3)                          # warm-up: modules loaded, scratch made
                times = {k: [] for k in paths}
                for _ in range(a.repeats):
                    for name, (clock, fn, k) in paths.items():
                        times[name].append(clock(s, fn, k))
                bytes_per_call = n * (6 if flags & pkg.FLAG_HALF_STORAGE else 8)
                out = {"elements": n, "bytes_per_device_call": bytes_per_call}
                for name, ts in times.items():
                    out[name + "_ms"] = summary(ts)
                    if name.endswith("_device"):
                        bw = bytes_per_call / (statistics.median(ts) * 1e-3)
                        out[name + "_GB_s"] = round(bw / 1e9, 1)
                        out[name + "_share_of_datasheet_hbm"] = round(bw / DATASHEET_HBM_BYTES_PER_S, 3)
                s._check(L.fluid_read_device(s._h, fid, dp, n))
                s.sync()
                s._check(L.fluid_read(s._h, fid, pinned, n))
                host = np.ctypeslib.as_array(C.cast(pinned, C.POINTER(C.c_float)), (n,))
                out["device_read_equals_host_read"] = bool(np.array_equal(host.view(np.uint32),
                                                                          dst.cpu().numpy().view(np.uint32)))
                result["cases"][f"{size_name} {storage} {field}"] = out
                L.fluid_host_free(pinned)
                del src, dst
            s.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
