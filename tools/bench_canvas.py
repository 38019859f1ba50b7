"""What a displayed frame costs: render() read back as fp32 against render_canvas() into host or device memory.

usage: python tools/bench_canvas.py [--frames K] [--repeats R] [--out FILE.json]

  * the reference desktop frame: 128^2 sim, 1024^2 dye, a 1920 x 1080 canvas, SHADING + BLOOM + SUNRAYS
    (BLOOM_RESOLUTION 256 / 8 iterations, SUNRAYS_RESOLUTION 196), over a dye stirred by seeded splats;
  * storage: fp32, and FLUID_FLAG_HALF_STORAGE | FLUID_FLAG_HALF_POSTFX (the reference's half-float FBOs);
  * per frame, (a) fluid_render_keywords into pinned host memory (the fp32 frame, 16 B per texel copied),
    (b) fluid_render_canvas into pinned host memory (4 B per texel copied), (c) fluid_render_canvas into a
    torch uint8 CUDA tensor (nothing copied; one fluid_sync after the K frames);
  * device time between fluid_mark events and host time (perf_counter around K frames ending in a
    sync), median and range over R repeats after a warm-up; (b) and (c) are checked byte for byte.
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

W, H = 1920, 1080
MODES = {"fp32": 0, "half_storage+half_postfx": pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                  # the timing below still needs the GPU
        return {"name": "unknown", "error": str(e)}


def stirred(flags):
    rs = np.random.RandomState(3)
    s = pkg.FluidSimulation({"SHADING": True, "BLOOM": True, "SUNRAYS": True}, canvas_width=W, canvas_height=H,
                            flags=flags, sizes=(128, 128, 1024, 1024), random=lambda: float(rs.random_sample()))
    s.dithering = np.random.default_rng(1).random((64, 64, 3), dtype=np.float32)
    s.multipleSplats(12)
    for _ in range(10):
        s.step(0.016666)
    s.sync()
    return s


def timed(s, frame, k, repeats):
    """(device ms per frame, host ms per frame) lists over `repeats` windows of k frames."""
    dev, host = [], []
    for _ in range(repeats):
        s.sync()
        t0 = time.perf_counter()
        s.mark(0)
        for _ in range(k):
            frame()
        s.mark(1)
        s.sync()
        host.append((time.perf_counter() - t0) * 1e3 / k)
        dev.append(s.elapsed_ms() / k)
    return dev, host


def summary(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    L = pkg.lib()
    n = W * H * 4
    result = {"card": card(), "canvas": [W, H], "sim": [128, 128], "dye": [1024, 1024], "keywords": "SHADING+BLOOM+SUNRAYS",
              "frames_per_window": a.frames, "repeats": a.repeats,
              "bytes_copied_per_frame": {"render_fp32_pinned": n * 4, "canvas_pinned": n, "canvas_device": 0}, "modes": {}}
    for mode, flags in MODES.items():
        s = stirred(flags)
        kw, fx, dith = pkg.postfx_inputs(s.config, s.dithering)
        s._push_config()
        s.set_param("BACKGROUND", 0)
        frame32 = C.cast(L.fluid_host_alloc(n * 4), C.c_void_p)
        canvas8 = C.cast(L.fluid_host_alloc(n), C.c_void_p)
        assert frame32.value and canvas8.value, "fluid_host_alloc failed"
        t = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        dp = dith.ctypes.data_as(C.c_void_p)

        def render():
            s._check(L.fluid_render_keywords(s._h, W, H, kw, C.byref(fx), dp, 64, 64, 0.0, 0.0, 0.0, frame32, n, None, None))

        def canvas(dst, on):
            return lambda: s._check(L.fluid_render_canvas(s._h, W, H, kw, 0, C.byref(fx), dp, 64, 64, 0.0, 0.0, 0.0, dst, n, on))

        paths = {"render_fp32_pinned": render, "canvas_pinned": canvas(canvas8, 0),
                 "canvas_device": canvas(C.c_void_p(t.data_ptr()), 1)}
        for fn in paths.values():
            timed(s, fn, 5, 1)                              # warm-up: targets made, modules loaded
        dev, host = {k: [] for k in paths}, {k: [] for k in paths}
        for _ in range(a.repeats):
            for name, fn in paths.items():                  # interleaved so drift hits all three alike
                d, h = timed(s, fn, a.frames, 1)
                dev[name] += d
                host[name] += h
        out = {name: {"device_ms": summary(dev[name]), "host_ms": summary(host[name])} for name in paths}
        s.sync()
        got = np.ctypeslib.as_array(C.cast(canvas8, C.POINTER(C.c_uint8)), (n,)).copy()
        out["canvas_host_equals_device"] = bool(np.array_equal(got, t.cpu().numpy().reshape(-1)))
        result["modes"][mode] = out
        L.fluid_host_free(frame32)
        L.fluid_host_free(canvas8)
        s.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
