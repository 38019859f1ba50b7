"""Splat bursts on one GPU: n x fluid_splat() against one fluid_splats(n), at three grid sizes.

usage: python tools/bench_splats.py [--old-so PATH] [--quick] [--out FILE.json]

  * configurations: 128^2 sim / 1024^2 dye (the reference default on a 1024^2 canvas), 1024^2 / 2048^2,
    4096^2 / 4096^2; record counts n in {1, 4, 10, 24, 128}; fp32 storage;
  * (a) n x splat() and (b) one splats(n), device time between fluid_mark events, after a warm-up,
    over windows of >= 0.5 s, 5 repeats: median and range of the time per burst;
  * launches per burst (fluid_launch_count), HBM bytes from the shapes (every launch reads and writes
    velocity and dye once) and the achieved GB/s;
  * from the SASS of the splats kernel (cuobjdump): instructions and MUFU per texel and record on the
    fast path of its record loop, and which of issue, MUFU and HBM bounds each burst;
  * --old-so: another build of the library (the parent commit's, which has no fluid_splats), loaded
    next to this one.  At n = 1 the two are timed alternately, and a seeded 24-splat burst is dumped
    from both (fp32 and half storage) and compared bit for bit.
The card name, power limit and maximum SM clock come from nvidia-smi (read-only query)."""
import argparse
import ctypes as C
import json
import math
import os
import re
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from webgl_fluid_simulation_b200 import _lib  # noqa: E402

CONFIGS = [(128, 128, 1024, 1024), (1024, 1024, 2048, 2048), (4096, 4096, 4096, 4096)]
COUNTS = [1, 4, 10, 24, 128]
PER_LAUNCH = 128                  # SPLATS_PER_LAUNCH of csrc/passes.cuh
TILE = 8                          # texels per thread of splats_kernel (SPL_TX x SPL_TY)
HBM_BPS = 3.35e12                 # H100 SXM data sheet
SMS, ISSUE_LANES, MUFU_LANES = 132, 128, 16   # per SM and clock: 4 schedulers x 32 lanes; 16 SFU lanes
FLAG_HALF = 0x10


class Lib:
    """The few entry points this tool needs, on any build of the library (ctypes, RTLD_LOCAL)."""

    def __init__(self, path):
        self.path = path
        L = C.CDLL(path)
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        L.fluid_config_default.argtypes = [C.POINTER(_lib.Config)]; L.fluid_config_default.restype = None
        L.fluid_create.argtypes = [C.POINTER(_lib.Config), C.POINTER(vp)]
        L.fluid_destroy.argtypes = [vp]; L.fluid_destroy.restype = None
        L.fluid_splat.argtypes = [vp] + [f] * 7
        L.fluid_mark.argtypes = [vp, i]
        L.fluid_elapsed_ms.argtypes = [vp, C.POINTER(f)]
        L.fluid_launch_count.argtypes = [vp]; L.fluid_launch_count.restype = C.c_uint64
        L.fluid_sync.argtypes = [vp]
        L.fluid_read.argtypes = [vp, i, vp, C.c_size_t]
        L.fluid_write.argtypes = [vp, i, vp, C.c_size_t]
        L.fluid_last_error.argtypes = [vp]; L.fluid_last_error.restype = C.c_char_p
        self.has_splats = hasattr(L, "fluid_splats")
        if self.has_splats:
            L.fluid_splats.argtypes = [vp, C.POINTER(f), i]
        self.L = L

    def create(self, W, H, Wd, Hd, flags=0):
        cfg = _lib.Config()
        self.L.fluid_config_default(C.byref(cfg))
        cfg.sim_w, cfg.sim_h, cfg.dye_w, cfg.dye_h = W, H, Wd, Hd
        cfg.aspect, cfg.device, cfg.flags = W / H, 0, flags
        h = C.c_void_p()
        self.ok(None, self.L.fluid_create(C.byref(cfg), C.byref(h)))
        return h

    def ok(self, h, rc):
        if rc != 0:
            raise RuntimeError(f"{self.path}: {rc} {self.L.fluid_last_error(h)}")

    def burst(self, h, recs, batched):
        if batched:
            self.ok(h, self.L.fluid_splats(h, recs.ctypes.data_as(C.POINTER(C.c_float)), len(recs)))
        else:
            for x, y, dx, dy, r, g, b in recs.tolist():
                self.ok(h, self.L.fluid_splat(h, x, y, dx, dy, r, g, b))

    def window(self, h, recs, batched, reps):
        """ms per burst over `reps` bursts, and launches per burst"""
        l0 = self.L.fluid_launch_count(h)
        self.ok(h, self.L.fluid_mark(h, 0))
        for _ in range(reps):
            self.burst(h, recs, batched)
        self.ok(h, self.L.fluid_mark(h, 1))
        ms = C.c_float()
        self.ok(h, self.L.fluid_elapsed_ms(h, C.byref(ms)))
        return ms.value / reps, (self.L.fluid_launch_count(h) - l0) / reps

    def read(self, h, field, shape):
        out = np.empty(shape, np.float32)
        self.ok(h, self.L.fluid_read(h, field, out.ctypes.data_as(C.c_void_p), out.size))
        return out

    def write(self, h, field, a):
        a = np.ascontiguousarray(a, np.float32)
        self.ok(h, self.L.fluid_write(h, field, a.ctypes.data_as(C.c_void_p), a.size))


def records(n, seed):
    """multipleSplats-like records: points in [0, 1], forces of +-500, colours up to 1.5"""
    rng = np.random.default_rng(seed)
    r = np.empty((n, 7), np.float32)
    r[:, 0:2] = rng.uniform(0, 1, (n, 2))
    r[:, 2:4] = rng.uniform(-500, 500, (n, 2))
    r[:, 4:7] = rng.uniform(0, 1.5, (n, 3))
    return r


def timed(lib, h, recs, batched, quick):
    """warm-up, then reps per window so that a window lasts >= 0.5 s; 5 windows"""
    min_s, repeats = (0.1, 3) if quick else (0.5, 5)
    lib.window(h, recs, batched, 3)
    t, _ = lib.window(h, recs, batched, 3)
    reps = max(3, math.ceil(min_s * 1e3 / max(t, 1e-4)))
    ms, launches = zip(*[lib.window(h, recs, batched, reps) for _ in range(repeats)])
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "reps": reps,
            "launches": launches[0]}


def pass_bytes(W, H, Wd, Hd, half=False):
    """one read and one write of velocity and dye"""
    return 2 * (W * H * (4 if half else 8) + Wd * Hd * (8 if half else 16))


def sass_loops(so):
    """Fast-path instructions and MUFU per texel-record of each record loop of each splats_kernel."""
    try:
        sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    except (OSError, subprocess.CalledProcessError) as e:
        return {"error": f"cuobjdump failed: {e}"}
    out, cur, ins = {}, None, []

    def flush():
        if not cur or "splats_kernel" not in cur:
            return
        loops = []
        for a, t in ins:
            m = re.search(r"BRA (0x[0-9a-f]+)", t)
            if not m or int(m.group(1), 16) >= a:
                continue
            lo = int(m.group(1), 16)
            body = [(b, x) for b, x in ins if lo <= b <= a]
            skip = set()                   # the all-lanes-fast vote jumps over the compiler-division variant
            for j, (b, x) in enumerate(body):
                if x.startswith("VOTE.ALL") and j + 1 < len(body):
                    mm = re.search(r"@P\d BRA (0x[0-9a-f]+)", body[j + 1][1])
                    if mm:
                        skip |= {bb for bb, _ in body if body[j + 1][0] < bb < int(mm.group(1), 16)}
            fast = [x for b, x in body if b not in skip]
            ops = [re.match(r"(?:@!?U?P\w+\s+)?([A-Z0-9_]+)", x).group(1) for x in fast]
            loops.append({"static": len(body), "fast_path": len(fast), "mufu": ops.count("MUFU"),
                          "instr_per_texel_record": len(fast) / TILE, "mufu_per_texel_record": ops.count("MUFU") / TILE})
        loops.sort(key=lambda d: -d["fast_path"])   # dye (3 colour channels) before velocity
        out["half" if "Half" in cur else "fp32"] = dict(zip(("dye", "velocity"), loops))

    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            flush(); cur, ins = m.group(1), []
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if m and cur:
            ins.append((int(m.group(1), 16), m.group(2).strip()))
    flush()
    return out


def bound(n_launch, texel_records, nbytes, sass, clock_mhz):
    """least time of a burst (ms) by issue, MUFU and HBM, and which one bounds it"""
    if "fp32" not in sass or not clock_mhz:
        return None
    ipt = max(d["instr_per_texel_record"] for d in sass["fp32"].values())
    mpt = max(d["mufu_per_texel_record"] for d in sass["fp32"].values())
    hz = clock_mhz * 1e6
    t = {"issue": texel_records * ipt / (SMS * ISSUE_LANES * hz) * 1e3,
         "mufu": texel_records * mpt / (SMS * MUFU_LANES * hz) * 1e3,
         "hbm": n_launch * nbytes / HBM_BPS * 1e3}
    t["bound_by"] = max(t, key=t.get)
    return t


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, subprocess.CalledProcessError, ValueError, IndexError) as e:
        return {"error": str(e)}


def old_vs_new(new, old, quick):
    res = {"timing_n1": [], "bitwise_24": []}
    one = records(1, 5)
    for W, H, Wd, Hd in CONFIGS:
        hs = {lib: lib.create(W, H, Wd, Hd) for lib in (old, new)}
        for lib in (old, new):
            timed(lib, hs[lib], one, False, True)   # warm-up of both before the alternation
        rounds = {"old": [], "new": []}
        for _ in range(3 if quick else 5):
            for tag, lib in (("old", old), ("new", new)):
                rounds[tag].append(timed(lib, hs[lib], one, False, True)["median_ms"])
        res["timing_n1"].append({"config": [W, H, Wd, Hd], **{k: {"median_ms": statistics.median(v), "min_ms": min(v),
                                                                  "max_ms": max(v), "windows": v} for k, v in rounds.items()}})
        for lib, h in hs.items():
            lib.L.fluid_destroy(h)
        for flags in (0, FLAG_HALF):
            rng = np.random.default_rng(W + flags)
            v = (rng.standard_normal((H, W, 2)) * 50).astype(np.float32)
            d = rng.uniform(-1, 2, (Hd, Wd, 4)).astype(np.float32)
            v.reshape(-1)[:: 97] = -0.0
            recs = records(24, 99)
            out = {}
            for tag, lib, batched in (("old", old, False), ("new_splat", new, False), ("new_splats", new, True)):
                h = lib.create(W, H, Wd, Hd, flags)
                lib.write(h, 0, v); lib.write(h, 1, d)
                lib.burst(h, recs, batched)
                out[tag] = (lib.read(h, 0, (H, W, 2)), lib.read(h, 1, (Hd, Wd, 4)))
                lib.L.fluid_destroy(h)
            same = {k: all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(out["old"], out[k]))
                    for k in ("new_splat", "new_splats")}
            res["bitwise_24"].append({"config": [W, H, Wd, Hd], "storage": "half" if flags else "fp32",
                                      "old_vs_new_splat_bitwise": same["new_splat"],
                                      "old_vs_new_splats_bitwise": same["new_splats"]})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old-so", help="another build of libfluid_b200.so to compare with at n = 1")
    ap.add_argument("--quick", action="store_true", help="0.1 s windows, 3 repeats (a rehearsal, not a measurement)")
    ap.add_argument("--out", help="also write the JSON result here")
    args = ap.parse_args()
    new = Lib(_lib.SO_PATH)
    if not new.has_splats:
        sys.exit(f"{_lib.SO_PATH} has no fluid_splats")
    result = {"card": card(), "library": _lib.SO_PATH, "sass": sass_loops(_lib.SO_PATH), "rows": []}
    clock = re.match(r"\d+", result["card"].get("max_sm_clock", ""))
    clock_mhz = int(clock.group(0)) if clock else None
    for W, H, Wd, Hd in CONFIGS:
        lib = new
        h = lib.create(W, H, Wd, Hd)
        nbytes = pass_bytes(W, H, Wd, Hd)
        for n in COUNTS:
            recs = records(n, n)
            row = {"config": [W, H, Wd, Hd], "n": n}
            for tag, batched in (("a_n_x_splat", False), ("b_splats", True)):
                t = timed(lib, h, recs, batched, args.quick)
                t["hbm_bytes"] = int(round(t["launches"])) * nbytes
                t["gb_per_s"] = t["hbm_bytes"] / (t["median_ms"] * 1e-3) / 1e9
                row[tag] = t
            row["speedup"] = row["a_n_x_splat"]["median_ms"] / row["b_splats"]["median_ms"]
            row["b_least_ms"] = bound(math.ceil(n / PER_LAUNCH), n * (W * H + Wd * Hd), nbytes, result["sass"], clock_mhz)
            result["rows"].append(row)
            print(json.dumps(row), flush=True)
        lib.L.fluid_destroy(h)
    if args.old_so:
        result["old_vs_new"] = old_vs_new(new, Lib(args.old_so), args.quick)
        print(json.dumps(result["old_vs_new"]), flush=True)
    print(json.dumps({"card": result["card"], "sass": result["sass"]}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
