"""Multi-GPU launch helpers (one process per GPU, SURVEY.md §8e).

The partition of the film and the reduce of the per-rank films live in the library: pb2_render_path[_device] with
``tile_count == 0`` renders this rank's 16x16 tiles (tile t belongs to rank t % world) and sums the films onto rank 0
with one ncclReduce (include/pb2.h, pb2_dist_*).  What is left for Python is the rendezvous: handing rank 0's NCCL
unique id to the other ranks over the process group torchrun has already set up.
"""
import ctypes as C

import numpy as np

from . import PathParams, check, lib, ptr

PB2_DIST_ID_BYTES = 128


def dist_init_from_torch():
    """pb2_dist_init over torch.distributed's default process group (call after pb2_init / pbrt_v3_b200.init).
    Returns (rank, world); a no-op returning (0, 1) when no process group is initialised."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return 0, 1
    L = lib()
    rank, world = dist.get_rank(), dist.get_world_size()
    uid = np.zeros(PB2_DIST_ID_BYTES, np.uint8)
    if rank == 0:
        check(L.pb2_dist_unique_id(ptr(uid)))
    device = "cuda" if dist.get_backend() == "nccl" else "cpu"
    t = torch.from_numpy(uid).to(device)
    dist.broadcast(t, src=0)
    uid = np.ascontiguousarray(t.cpu().numpy())
    check(L.pb2_dist_init(rank, world, ptr(uid)))
    return rank, world


def work_items(film, params, tile_rank=0, tile_count=1):
    """(pixel x, pixel y, sample number) of every work item of one rank's partition, as the render kernels enumerate them
    (pb2_work_items: the kernels' own decode function compiled for the host); skipped items are dropped."""
    L = lib()
    p = PathParams()
    C.memmove(C.byref(p), params if isinstance(params, C._Pointer) else C.byref(params), C.sizeof(PathParams))
    p.tile_rank, p.tile_count = tile_rank, tile_count
    n = C.c_int64()
    check(L.pb2_work_items(film, C.byref(p), 0, 0, None, C.byref(n)))
    out = np.zeros((n.value, 3), np.int32)
    check(L.pb2_work_items(film, C.byref(p), 0, n.value, ptr(out), None))
    # a skipped item is (-1, -1, -1); a pixel coordinate alone may be negative (filters wider than a pixel extend the sample
    # bounds beyond the film), a sample number never is
    return out[out[:, 2] >= 0]
