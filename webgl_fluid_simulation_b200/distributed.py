"""One-process-per-GPU launcher glue: torch.distributed is only the plumbing (rendezvous +
broadcast of the ncclUniqueId); the halo exchange itself runs inside libfluid_b200 over NCCL."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _lib
from .sim import FluidSimulation


def nccl_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    rc = _lib.lib().fluid_nccl_unique_id(buf, 128)
    if rc != 0:
        raise _lib.FluidError(rc, (_lib.lib().fluid_last_error(None) or b"").decode())
    return buf.raw


def create_slab_simulation(config=None, canvas_width=1024, canvas_height=1024, device=-1, **kw) -> FluidSimulation:
    """Every rank of an initialised torch.distributed group calls this; returns the rank's slab."""
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    box = [nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    sim = FluidSimulation(config, canvas_width, canvas_height, device=device, rank=rank, world=world,
                          nccl_uid=box[0], **kw)
    sim.halo_transport = "nccl"
    if os.environ.get("FLUID_HALO", "p2p") != "nccl" and world > 1:
        if connect_peers(sim):
            sim.halo_transport = "p2p"
    return sim


def connect_peers(sim: FluidSimulation) -> bool:
    """Switch a slab handle to the peer-memory halo path: all-gather the 256-byte IPC exports and
    connect each rank to rank-1 / rank+1 (single NVLink / NVSwitch box).  If ANY rank cannot export
    or map (IPC not permitted, different boxes), EVERY rank falls back to the NCCL transport, so
    the group never mixes the two.  Returns True when the peer-memory path is active."""
    import torch.distributed as dist
    L = _lib.lib()
    rank, world = dist.get_rank(), dist.get_world_size()
    blob = C.create_string_buffer(256)
    ok = L.fluid_p2p_export(sim._h, blob, 256) == 0
    blobs = [None] * world
    dist.all_gather_object(blobs, blob.raw if ok else None)
    if ok and all(b is not None for b in blobs):
        below = C.create_string_buffer(blobs[rank - 1], 256) if rank > 0 else None
        above = C.create_string_buffer(blobs[rank + 1], 256) if rank + 1 < world else None
        ok = L.fluid_p2p_connect(sim._h, below, above) == 0
    else:
        ok = False
    flags = [None] * world
    dist.all_gather_object(flags, bool(ok))          # also the barrier: nobody pushes before everyone has mapped
    if not all(flags):
        sim._check(L.fluid_p2p_disable(sim._h))
        return False
    return True


def gather_image(band, bottom_first: bool = False):
    """Every rank of the group calls this with the band its slab drew; rank 0 gets the whole image, the others
    None.  bottom_first: render()'s fp32 frame (row 0 at the bottom), whose bands stack in rank order; otherwise a
    canvas or capture (top row first), whose bands stack in reverse rank order."""
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    parts = [None] * world if rank == 0 else None
    dist.gather_object(np.ascontiguousarray(band), parts, dst=0)
    if rank != 0:
        return None
    return np.concatenate(parts if bottom_first else parts[::-1], axis=0)
