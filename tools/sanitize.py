"""Small end-to-end run for compute-sanitizer (memcheck / racecheck / initcheck):
    compute-sanitizer --tool memcheck python tools/sanitize.py
Exercises every kernel on grids that hit the wall / mirror / ragged-tile paths."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import webgl_fluid_simulation_b200 as pkg  # noqa: E402

for (W, H, Wd, Hd, flags, jb) in [(132, 45, 200, 70, 0, 5), (64, 64, 128, 128, pkg.FLAG_NO_GRAPH, 10),
                                  (36, 20, 54, 30, pkg.FLAG_UNFUSED, 3), (256, 130, 256, 130, 0, 12)]:
    rs = np.random.RandomState(3)
    s = pkg.FluidSimulation({"PRESSURE_ITERATIONS": 23}, W, H, flags=flags, jacobi_block=jb,
                            sizes=(W, H, Wd, Hd), random=rs.random_sample)
    s.multipleSplats(3)
    for _ in range(3):
        s.step(0.016666)
    s.config["SIM_RESOLUTION"] = 48
    for n in ("velocity", "dye", "pressure", "divergence", "curl"):
        assert np.isfinite(s.readField(n)).all(), n
    s.close()
# streaming curl/vorticity/divergence + gradient, 4-cell advection (power-of-two widths >= 128), the
# banded host solve, half-float storage, TRANSPARENT display, the post-FX chain
rs = np.random.RandomState(5)
s = pkg.FluidSimulation({"PRESSURE_ITERATIONS": 20}, 256, 640, sizes=(256, 640, 256, 640), random=rs.random_sample)
s.multipleSplats(3)
for _ in range(2):
    s.step(0.016666)
d = rs.uniform(-1, 1, (640, 256)).astype(np.float32); p = rs.standard_normal((640, 256)).astype(np.float32)
s.pressure_solve_host(d, p, 20)                  # 2 bands
assert np.isfinite(p).all()
s.config["TRANSPARENT"] = True; s.canvas = {"width": 96, "height": 64}
assert np.isfinite(s.render(96, 64)).all()
s.config.update(TRANSPARENT=False, BLOOM=True, SUNRAYS=True, SHADING=True, BLOOM_RESOLUTION=64, SUNRAYS_RESOLUTION=48)
s.dithering = rs.random_sample((64, 64, 3)).astype(np.float32)
assert np.isfinite(s.render(96, 64)).all()
s.close()
s = pkg.FluidSimulation({"PRESSURE_ITERATIONS": 9}, 96, 72, sizes=(96, 72, 144, 108), flags=pkg.FLAG_HALF_STORAGE, random=rs.random_sample)
s.multipleSplats(2)
for _ in range(2):
    s.step(0.016666)
assert np.isfinite(s.readField("dye")).all()
s.close()
# the reference's desktop frame: fp16 dye and fp16 post-FX targets, the sunrays mask stored into the fp16 dye.write
s = pkg.FluidSimulation({"PRESSURE_ITERATIONS": 9}, 96, 72, sizes=(96, 72, 144, 108),
                        flags=pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX, random=rs.random_sample)
s.multipleSplats(2)
s.step(0.016666)
s.config.update(BLOOM=True, SUNRAYS=True, SHADING=True, BLOOM_RESOLUTION=64, SUNRAYS_RESOLUTION=48)
s.dithering = rs.random_sample((64, 64, 3)).astype(np.float32)
assert np.isfinite(s.render(96, 72)).all()
s.close()
# the same frame on a device without float linear filtering: NEAREST dye, bloom, pyramid and sunrays samplers
s = pkg.FluidSimulation({"PRESSURE_ITERATIONS": 9}, 96, 72, sizes=(96, 72, 144, 108),
                        flags=pkg.FLAG_HALF_STORAGE | pkg.FLAG_HALF_POSTFX | pkg.FLAG_NEAREST_FILTERING,
                        random=rs.random_sample)
s.multipleSplats(2)
s.step(0.016666)
s.config.update(BLOOM=True, SUNRAYS=True, SHADING=True, BLOOM_RESOLUTION=64, SUNRAYS_RESOLUTION=48)
s.dithering = rs.random_sample((64, 64, 3)).astype(np.float32)
assert np.isfinite(s.render(96, 72)).all()
s.close()
print("sanitize run complete")
