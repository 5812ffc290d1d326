"""Two processes, two GPUs: the partition + NCCL film reduce INSIDE pb2_render_path (pb2_dist_init).  Needs >= 2 devices
(skipped on a machine with one GPU; run on two or more with `python -m pytest tests/test_gpu_multi.py -m gpu`)."""
import os
import socket
import subprocess
import sys

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

WORKER = r'''
import ctypes as C, os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
import pbrt_v3_b200 as pb
from pbrt_v3_b200 import multigpu
local = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group(backend="nccl", device_id=torch.device("cuda", local))
pb.init(local)
rank, world = multigpu.dist_init_from_torch()
assert (rank, world) == (dist.get_rank(), 2)
L = pb.lib()
for make in (lambda: pb.HostScene.soup(20000, xres=100, yres=70, spp=4),
             lambda: pb.HostScene.from_file(os.path.join(sys.argv[1], "tests", "scenes", "materials.pbrt"))):
    hs = make()
    dev = hs.device_scene()
    h, w = hs.film_shape()
    merged = np.full((h, w, 4), -1, np.float32)
    st = pb.Stats()
    # collective: tile_count = 0
    pb.check(L.pb2_render_path(dev, hs.camera, hs.film, hs.params_copy(tile_rank=0, tile_count=0), pb.ptr(merged) if rank == 0 else None, C.byref(st)))
    cam = torch.tensor([int(st.camera_rays)], device="cuda")
    dist.all_reduce(cam)
    spp = hs.params.contents.samples_per_pixel
    assert int(cam) == h * w * spp and 0 < st.camera_rays < h * w * spp      # every rank rendered a part, together everything
    if rank == 0:
        alone = np.zeros((h, w, 4), np.float32)
        pb.check(L.pb2_render_path(dev, hs.camera, hs.film, hs.params_copy(tile_rank=0, tile_count=1), pb.ptr(alone), None))
        assert np.array_equal(merged[..., 3], alone[..., 3]), "filter weight sums of the merged film must equal the single-GPU film's"
        assert np.allclose(merged, alone, rtol=1e-4, atol=1e-4)
    # the device-resident form reduces onto rank 0's film too
    film = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    pb.check(L.pb2_render_path_device(dev, hs.camera, hs.film, hs.params_copy(tile_rank=0, tile_count=0), C.c_void_p(film.data_ptr()), 1,
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream), None))
    torch.cuda.synchronize()
    if rank == 0:
        assert np.allclose(film.cpu().numpy(), merged, rtol=1e-4, atol=1e-4)
    dist.barrier()
L.pb2_dist_shutdown()
dist.destroy_process_group()
print("rank", rank, "ok")
'''


def test_two_processes_render_and_reduce_inside_the_library(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script), ROOT]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0 and res.stdout.count(" ok") == 2, res.stdout[-4000:]


GROUP_WORKER = r'''
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import pbrt_v3_b200 as pb
L = pb.lib()
pb.check(L.pb2_init_devices(0, None))            # every visible device, one process
n = L.pb2_device_count()
assert n >= 2, n
for make in (lambda: pb.HostScene.soup(20000, xres=100, yres=70, spp=4),
             lambda: pb.HostScene.instanced_soup(2000, grid=4, xres=64, yres=36, spp=4),
             lambda: pb.HostScene.from_file(os.path.join(sys.argv[1], "tests", "scenes", "killeroo_like.pbrt"))):
    hs = make()
    group, sg = hs.render_rgbw(hs.params_copy(tile_rank=0, tile_count=0))      # tiles dealt to the devices, films merged on the first
    alone, sa = hs.render_rgbw(hs.params_copy(tile_rank=0, tile_count=1))      # the primary device alone
    assert (sg.camera_rays, sg.regular_rays, sg.shadow_rays) == (sa.camera_rays, sa.regular_rays, sa.shadow_rays)
    assert np.array_equal(group[..., 3], alone[..., 3]) and np.allclose(group, alone, rtol=1e-4, atol=1e-4)
    img, st = hs.render()                                                     # Integrator::Render of the host classes: the group as well
    assert st.camera_rays == sa.camera_rays and np.allclose(img, hs.resolve(alone), rtol=1e-4, atol=1e-5)
print("group of", n, "ok")
'''


def test_one_process_renders_on_every_visible_device(tmp_path):
    """pb2_init_devices: scene replicas, one host thread per device, the film merge on the primary device over peer access."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    script = tmp_path / "group.py"
    script.write_text(GROUP_WORKER)
    res = subprocess.run([sys.executable, str(script), ROOT], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0 and " ok" in res.stdout, res.stdout[-4000:]
