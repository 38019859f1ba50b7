"""Multi-GPU correctness check, launched with one rank per GPU:
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/slab_check.py
Every rank runs its slab of a W x H simulation (seeded splats + steps through the public API);
rank 0 additionally runs the same simulation on ONE GPU and compares bit for bit (SURVEY §8e bar:
k-GPU == 1-GPU bitwise).  Prints 'SLAB_CHECK ok' / 'SLAB_CHECK FAIL ...' on rank 0."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import webgl_fluid_simulation_b200 as pkg  # noqa: E402
from webgl_fluid_simulation_b200.distributed import create_slab_simulation  # noqa: E402

W = int(os.environ.get("SLAB_W", 512)); H = int(os.environ.get("SLAB_H", 768))
WD = int(os.environ.get("SLAB_WD", 1024)); HD = int(os.environ.get("SLAB_HD", 1536))
ITERS = int(os.environ.get("SLAB_ITERS", 23)); STEPS = int(os.environ.get("SLAB_STEPS", 4))
RESIZE = os.environ.get("SLAB_RESIZE")             # "W,H,WD,HD": initFramebuffers() to these sizes after the steps, then 2 more steps
FAST = float(os.environ.get("SLAB_FAST", 0))     # texels/s of an extra splat placed ON a slab edge (back-trace reach test)


def drive(sim, seed=5):
    rs = np.random.RandomState(seed)
    sim.random = lambda: float(rs.random_sample())
    sim.multipleSplats(6)                                # one splat() per record ...
    if FAST:   # the fastest thing a pointer flick produces, right on the boundary between two slabs, aimed across it
        sim.splats([(0.5, 0.5, 0.3 * FAST, FAST, 0.9, 0.2, 0.1), (0.25, 0.5, 0.0, -FAST, 0.1, 0.8, 0.3)])
    for k in range(STEPS):
        sim.step(0.016666)
        if k == 1:                                       # ... and a burst in one splats() call
            sim.splats([(rs.random_sample(), rs.random_sample(), 1000 * (rs.random_sample() - 0.5),
                         1000 * (rs.random_sample() - 0.5), 1.5 * rs.random_sample(), 0.0, 1.5 * rs.random_sample())
                        for _ in range(6)])
    out = {n: sim.readField(n) for n in ("velocity", "dye", "pressure", "divergence")}
    out["frame_"] = sim.render(256, 192)                 # a slab rank returns its band of the 256 x 192 target
    if RESIZE:                                           # resizeDoubleFBO on a live simulation (S:1116-1126), slab or not
        sim._sizes = tuple(int(x) for x in RESIZE.split(","))
        sim.initFramebuffers()
        out["resized_velocity"] = sim.readField("velocity"); out["resized_dye"] = sim.readField("dye")
        for _ in range(2):
            sim.step(0.016666)
        out["after_velocity"] = sim.readField("velocity"); out["after_dye"] = sim.readField("dye")
    return out


def main():
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, world = dist.get_rank(), dist.get_world_size()
    cfg = {"SIM_RESOLUTION": W, "DYE_RESOLUTION": WD, "PRESSURE_ITERATIONS": ITERS}
    sim = create_slab_simulation(cfg, W, H, device=local, sizes=(W, H, WD, HD))
    mine = drive(sim)
    # also the bench metric's entry point on slabs
    Ws, Hs = (tuple(int(x) for x in RESIZE.split(","))[:2]) if RESIZE else (W, H)      # the grid the handles hold by now
    rng = np.random.default_rng(1)
    pfull = rng.standard_normal((Hs, Ws)).astype(np.float32); dfull = rng.uniform(-1, 1, (Hs, Ws)).astype(np.float32)
    r0 = sim._dims("pressure")[3]; rows = sim._dims("pressure")[1]
    sim.writeField("pressure", pfull[r0:r0 + rows]); sim.writeField("divergence", dfull[r0:r0 + rows])
    sim.pass_("pressure_solve"); mine["solve"] = sim.readField("pressure")
    sim.close()
    mine["frame"] = mine.pop("frame_")
    gathered = [None] * world
    dist.all_gather_object(gathered, {k: (v, ) for k, v in mine.items()})
    ok, msgs = True, []
    if rank == 0:
        one = pkg.FluidSimulation(cfg, W, H, device=local, sizes=(W, H, WD, HD))
        ref = drive(one)
        one.writeField("pressure", pfull); one.writeField("divergence", dfull)
        one.pass_("pressure_solve"); ref["solve"] = one.readField("pressure")
        one.close()
        ref["frame"] = ref.pop("frame_")
        for name, full in ref.items():
            got = np.concatenate([g[name][0] for g in gathered], axis=0)
            same = got.shape == full.shape and np.array_equal(got.view(np.uint32), full.view(np.uint32))
            if not same:
                ok = False
                bad = np.argwhere(got.view(np.uint32) != full.view(np.uint32)) if got.shape == full.shape else []
                msgs.append(f"{name}: shape {got.shape} vs {full.shape}, {len(bad)} differing words, first {bad[:3].tolist() if len(bad) else ''}")
        print(("SLAB_CHECK ok" if ok else "SLAB_CHECK FAIL " + "; ".join(msgs)) + f" world={world} grid={W}x{H} dye={WD}x{HD}", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
