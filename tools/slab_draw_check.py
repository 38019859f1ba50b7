"""Multi-GPU check of frames, canvases and captures on row slabs, launched with one rank per GPU:
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/slab_draw_check.py
Every rank runs its slab of a W x H simulation (seeded splats + steps through the public API) and draws the
reference's desktop frame (SHADING + BLOOM + SUNRAYS), render(null) on the RGBA8 canvas and captureScreenshot: its
band of each, with the bloom and sunrays inputs gathered over NCCL.  Rank 0 assembles the bands
(distributed.gather_image), runs the same simulation on ONE GPU and compares bit for bit, together with every
rank's bloom FBO and sunrays texture.  Prints 'SLAB_DRAW_CHECK ok' / 'SLAB_DRAW_CHECK FAIL ...' on rank 0."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import webgl_fluid_simulation_b200 as pkg  # noqa: E402
from webgl_fluid_simulation_b200.distributed import create_slab_simulation, gather_image  # noqa: E402

W = int(os.environ.get("SLAB_W", 256)); H = int(os.environ.get("SLAB_H", 256))
WD = int(os.environ.get("SLAB_WD", 1024)); HD = int(os.environ.get("SLAB_HD", 1024))
CW = int(os.environ.get("SLAB_CANVAS_W", 1920)); CH = int(os.environ.get("SLAB_CANVAS_H", 1080))
STEPS = int(os.environ.get("SLAB_STEPS", 4))


def drive(sim, seed=5):
    rs = np.random.RandomState(seed)
    sim.random = lambda: float(rs.random_sample())
    sim.dithering = np.random.default_rng(64).random((64, 64, 3), dtype=np.float32)
    sim.multipleSplats(8)
    for _ in range(STEPS):
        sim.step(0.016666)
    sim.config.update(SHADING=True, BLOOM=True, SUNRAYS=True, TRANSPARENT=False)
    out = {"frame": sim.render(), "bloom": sim.last_bloom, "sunrays": sim.last_sunrays}
    out["canvas"] = sim.render_canvas()
    out["capture"] = sim.captureScreenshot()
    return out


def same(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype == np.float32:
        return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a.view(np.uint32)[~np.isnan(a)],
                                                                          b.view(np.uint32)[~np.isnan(b)])
    return np.array_equal(a, b)


def main():
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, world = dist.get_rank(), dist.get_world_size()
    cfg = {"SIM_RESOLUTION": W, "DYE_RESOLUTION": WD}
    sim = create_slab_simulation(cfg, CW, CH, device=local, sizes=(W, H, WD, HD))
    mine = drive(sim)
    gathers = sim.stat("gathers")
    sim.close()
    whole = {"frame": gather_image(mine["frame"], bottom_first=True),
             "canvas": gather_image(mine["canvas"]), "capture": gather_image(mine["capture"])}
    targets = [None] * world
    dist.all_gather_object(targets, (mine["bloom"], mine["sunrays"]))
    ok, msgs = True, []
    if rank == 0:
        one = pkg.FluidSimulation(cfg, CW, CH, device=local, sizes=(W, H, WD, HD))
        ref = drive(one)
        one.close()
        for name in ("frame", "canvas", "capture"):
            if not same(whole[name], ref[name]):
                ok = False
                msgs.append(f"{name}: {whole[name].shape} vs {ref[name].shape}")
        for r, (bloom, sun) in enumerate(targets):
            if not same(bloom, ref["bloom"]) or not same(sun, ref["sunrays"]):
                ok = False
                msgs.append(f"bloom / sunrays of rank {r}")
        if gathers != 6:
            ok = False
            msgs.append(f"{gathers} gathers, expected 6 (three BLOOM + SUNRAYS draws)")
        print(("SLAB_DRAW_CHECK ok" if ok else "SLAB_DRAW_CHECK FAIL " + "; ".join(msgs)) +
              f" world={world} grid={W}x{H} dye={WD}x{HD} canvas={CW}x{CH}", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
