"""Sweeps the temporal-block depth and the rows-per-warp-stream of jacobi_tb_kernel on an H100.
usage: python tools/tune_jacobi.py [W] [iters] > tune.txt"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import webgl_fluid_simulation_b200 as pkg  # noqa: E402

W = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
ITERS = int(sys.argv[2]) if len(sys.argv) > 2 else 50
rng = np.random.default_rng(0)
p = rng.standard_normal((W, W)).astype(np.float32)
d = rng.uniform(-1, 1, (W, W)).astype(np.float32)
print(f"# {W}x{W}, {ITERS} iterations; ms per solve, G updates/s")
for kb in (1, 2, 4, 6, 8, 9, 10, 11, 12):
    for rows in ((0,) if kb == 1 else (0, 32, 48, 64, 96, 128, 192, 256, 512)):
        os.environ["FLUID_JACOBI_ROWS"] = str(rows)
        flags = pkg.FLAG_NAIVE_JACOBI if kb == 1 else 0
        s = pkg.FluidSimulation({"SIM_RESOLUTION": W, "DYE_RESOLUTION": 64, "PRESSURE_ITERATIONS": ITERS},
                                1024, 1024, flags=flags, jacobi_block=kb)
        s.writeField("pressure", p); s.writeField("divergence", d)
        for _ in range(3):
            s.pass_("pressure_solve")
        s.sync()
        n = 20
        s.mark(0)
        for _ in range(n):
            s.pass_("pressure_solve")
        s.mark(1)
        ms = s.elapsed_ms() / n
        print(f"kb={kb:2d} rows={rows:4d}  {ms:8.4f} ms  {W*W*ITERS/ms/1e6:9.1f} G/s", flush=True)
        s.close()
