"""Device time of the two advection passes with the MANUAL_FILTERING shader (the default) and with
FLUID_FLAG_LINEAR_ADVECTION, on twin handles in one process, alternating.
usage: python tools/bench_advection.py [--quick] [--reps N] [--out FILE.json]

  * sizes: 4096^2 / 4096^2 (dye4<SAME>), 2048^2 / 4096^2 (dye4<!SAME>), 128^2 / 1024^2 (the reference's
    default SIM / DYE_RESOLUTION), fp32 and fp16 storage;
  * a repeat is `iters` back-to-back fluid_pass_advect_velocity (or _dye) calls between two fluid_mark
    events on the handle's stream; the MANUAL and LINEAR handles take turns repeat by repeat after a
    warm-up, and the median and spread (min, max) of the per-pass times are reported;
  * bytes moved per pass (each field read once, written once) over the median give an HBM rate.
The card name, power limit and maximum SM clock come from nvidia-smi (read-only query) in the same run.
Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from webgl_fluid_simulation_b200 import _lib  # noqa: E402

SIZES = [(4096, 4096, 4096, 4096), (2048, 2048, 4096, 4096), (128, 128, 1024, 1024)]
DT = 0.016666


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                     # the measurement itself does not depend on it
        return {"error": str(e)}


class Handle:
    def __init__(self, L, W, H, Wd, Hd, flags):
        self.L = L
        cfg = _lib.Config()
        L.fluid_config_default(C.byref(cfg))
        cfg.sim_w, cfg.sim_h, cfg.dye_w, cfg.dye_h = W, H, Wd, Hd
        cfg.flags = flags
        self.h = C.c_void_p()
        self.ok(L.fluid_create(C.byref(cfg), C.byref(self.h)))
        rng = np.random.default_rng(W + Wd)
        v = (rng.standard_normal((H, W, 2)) * 50).astype(np.float32)
        d = rng.random((Hd, Wd, 4), dtype=np.float32)
        for f, a in ((0, v), (1, d)):
            self.ok(L.fluid_write(self.h, f, a.ctypes.data_as(C.POINTER(C.c_float)), a.size))

    def ok(self, rc):
        if rc != 0:
            raise RuntimeError(f"fluid call failed ({rc}): {self.L.fluid_last_error(self.h if hasattr(self, 'h') else None)}")

    def window(self, which, iters):
        """ms per pass over `iters` back-to-back passes."""
        L, h = self.L, self.h
        fn = L.fluid_pass_advect_velocity if which == "velocity" else L.fluid_pass_advect_dye
        self.ok(L.fluid_mark(h, 0))
        for _ in range(iters):
            self.ok(fn(h, C.c_float(DT)))
        self.ok(L.fluid_mark(h, 1))
        ms = C.c_float()
        self.ok(L.fluid_elapsed_ms(h, C.byref(ms)))
        return ms.value / iters

    def close(self):
        self.L.fluid_destroy(self.h)


def pass_bytes(W, H, Wd, Hd, half, which):
    e = 2 if half else 4
    if which == "velocity":
        return 2 * W * H * 2 * e                       # read + write
    return W * H * 2 * e + 2 * Wd * Hd * 4 * e         # velocity read, dye read + write


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out")
    a = ap.parse_args()
    L = _lib.lib()
    L.fluid_pass_advect_velocity.argtypes = L.fluid_pass_advect_dye.argtypes = [C.c_void_p, C.c_float]
    L.fluid_mark.argtypes = [C.c_void_p, C.c_int]
    L.fluid_elapsed_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    reps = 3 if a.quick else a.reps
    res = {"card": card(), "reps": reps, "cases": []}
    for W, H, Wd, Hd in SIZES:
        for half in (False, True):
            base = _lib.FLAG_HALF_STORAGE if half else 0
            hs = {"manual": Handle(L, W, H, Wd, Hd, base), "linear": Handle(L, W, H, Wd, Hd, base | _lib.FLAG_LINEAR_ADVECTION)}
            for which in ("velocity", "dye"):
                nbytes = pass_bytes(W, H, Wd, Hd, half, which)
                iters = max(5, min(200, int(2e10 / nbytes)))      # a window of roughly 20 GB moved
                for h in hs.values():                              # warm-up
                    h.window(which, iters)
                t = {k: [] for k in hs}
                for _ in range(reps):
                    for k, h in hs.items():
                        t[k].append(h.window(which, iters))
                case = {"sim": f"{W}x{H}", "dye": f"{Wd}x{Hd}", "storage": "fp16" if half else "fp32", "pass": which,
                        "iters": iters, "bytes": nbytes}
                for k, xs in t.items():
                    med = statistics.median(xs)
                    case[k] = {"median_ms": round(med, 5), "min_ms": round(min(xs), 5), "max_ms": round(max(xs), 5),
                               "GB_per_s": round(nbytes / med / 1e6, 1)}
                case["linear_over_manual"] = round(case["linear"]["median_ms"] / case["manual"]["median_ms"], 4)
                res["cases"].append(case)
            for h in hs.values():
                h.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
