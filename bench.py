#!/usr/bin/env python
"""Benchmark of the path-tracing hot path (BASELINE.json metric: Msamples/sec at 1920x1080x64spp).

    python bench.py --gpus N --steps K --warmup W            # this repo's CUDA path
    python bench.py ... --dump-outputs DIR                   # ... and the film of the last timed step (see below)
    python bench.py --impl reference --gpus N --steps K ...  # the reference's CPU path (oracle/_ref)

A "step" is one pass of the hot path over the whole workload: SamplerIntegrator::Render with
PathIntegrator::Li for every pixel sample of BASELINE.json's configs[1] — synthetic 1 M random
triangles, 1920x1080, 64 spp (Halton), maxdepth 8, 1 H100 per rank.  The scene (BVH, triangles,
materials, lights, light-distribution tables, Halton tables) is resident in HBM before the timed
region; with N ranks the film's 16x16 tiles are dealt round-robin to the ranks, every rank renders
its tiles into its own film and one ncclReduce(sum) to rank 0 merges them (SURVEY.md §8e) - partition
and reduce happen INSIDE pb2_render_path[_device] (pb2_dist_init; torch.distributed only launches the
ranks, carries the NCCL id and takes the max over ranks of the timings).

One JSON line is printed by rank 0:
  value        whole-job Msamples/s from the device-timed steps (inputs resident, film left on device)
  e2e          the same metric through the public host-buffer call pb2_render_path: camera/film/params
               structs go in, the merged film comes back to host memory inside the timed region
  roofline     the BVH traversal kernel (k_wf_trace_w): algorithmic bytes (32 B x node visits + 36 B x
               primitive tests, counted on the device in the reference's traversal order) / its summed
               launch time, against MEASURED_PEAKS.json's HBM copy bandwidth (else the H100 SXM data sheet's)
  cpu_baseline the reference's own CPU implementation (oracle/_ref, every host thread this process may
               use) on a bounded sample of the same workload: the first k of the spp Halton samples of EVERY
               pixel of the frame (k chosen so that the sample takes --ref-seconds), so both arms trace the
               same mix of rays (rays_per_sample is printed by both)

--dump-outputs DIR writes the rgbw film (float32, height x width x 4) of the last timed step as DIR/film.npy when it
is at most 64 MB (1920x1080: 33 MB); a larger film (3840x2160: 133 MB) is written as a fixed sample of 2^21 pixels drawn
with seed 0: DIR/film_pixels.npy (float64 row-major pixel indices y * width + x, ascending) and DIR/film_sample.npy
(float32, their rgbw).  The inputs are seeded, so the same arguments give comparable files from two builds.

Workloads (BASELINE.json configs): soup = configs[1] (default; --tris 10000000 / 50000000 for the scenes
beyond L2), killeroo = configs[2] (the reference's scenes/killeroo-simple.pbrt at 1920x1080x256, stored in
tests/golden/killeroo_simple.npz), instanced = configs[3].
"""
import argparse
import ctypes as C
import json
import math
import os
import re
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOAD = dict(tris=1000000, seed=1234, jitter=0.02, xres=1920, yres=1080, spp=64, maxdepth=8)
HBM_FALLBACK_GBS = 3350.0  # H100 SXM data sheet (HBM3), not a measured figure
DUMP_LIMIT_BYTES = 64 << 20   # --dump-outputs writes at most this much
DUMP_SAMPLE_PIXELS = 1 << 21  # pixels of the seeded sample of a larger film: 16 MB of indices + 32 MB of rgbw


def measured_hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "MEASURED_PEAKS.json hbm_gbs"
        except Exception:
            pass
    return HBM_FALLBACK_GBS, "fallback (H100 SXM data sheet)"


class ClockSampler:
    """nvidia-smi clock / throttle-reason sampling during the timed region."""

    def __init__(self, index):
        self.index = index
        self.samples = []
        self.proc = None

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            parts = [x.strip() for x in line.split(",")]
            if len(parts) >= 7:
                self.samples.append(parts)

    def stop(self):
        if self.proc:
            self.proc.terminate()
        sm = sorted(int(float(s[0])) for s in self.samples if s[0].replace(".", "").isdigit())
        mx = [int(float(s[1])) for s in self.samples if s[1].replace(".", "").isdigit()]
        reasons = []
        for name, col in (("hw_slowdown", 3), ("hw_thermal_slowdown", 4), ("sw_thermal_slowdown", 5), ("sw_power_cap", 6)):
            if any(s[col].lower().startswith("active") for s in self.samples):
                reasons.append(name)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": reasons,
                "samples": len(self.samples)}


KILLEROO_NPZ = os.path.join(ROOT, "tests", "golden", "killeroo_simple.npz")   # the reference's scene file and the geometry it includes


def build_scene(args):
    import pbrt_v3_b200 as pb
    if args.workload == "instanced":
        # BASELINE.json configs[3]: one args.tris-triangle object instanced grid x grid times (SURVEY.md §8d C4)
        return pb.HostScene.instanced_soup(args.tris, grid=args.grid, xres=args.xres, yres=args.yres, spp=args.spp, maxdepth=args.maxdepth)
    if args.workload == "killeroo":
        # BASELINE.json configs[2]: the reference's own scenes/killeroo-simple.pbrt, only film size and sample count changed
        import numpy as np
        stored = np.load(KILLEROO_NPZ)
        text = stored["scene"].tobytes().decode()
        text, n1 = re.subn(r'"integer xresolution" \[\d+\] "integer yresolution" \[\d+\]',
                           '"integer xresolution" [%d] "integer yresolution" [%d]' % (args.xres, args.yres), text, count=1)
        text, n2 = re.subn(r'"integer pixelsamples" \[\d+\]', '"integer pixelsamples" [%d]' % args.spp, text, count=1)
        text, n3 = re.subn(r'Integrator "path"', 'Integrator "path" "integer maxdepth" [%d]' % args.maxdepth, text, count=1)
        assert n1 == 1 and n2 == 1 and n3 == 1
        # outside the tree (it may be read-only): the scene next to geometry/ (its Include is relative)
        with tempfile.TemporaryDirectory() as d:
            os.makedirs(os.path.join(d, "geometry"))
            with open(os.path.join(d, "geometry", "killeroo.pbrt"), "wb") as f:
                f.write(stored["geometry"].tobytes())
            dst = os.path.join(d, "killeroo-%dx%dx%d.pbrt" % (args.xres, args.yres, args.spp))
            with open(dst, "w") as f:
                f.write(text)
            return pb.HostScene.from_file(dst)
    return pb.HostScene.soup(args.tris, seed=args.seed, jitter=args.jitter, xres=args.xres, yres=args.yres,
                             spp=args.spp, maxdepth=args.maxdepth)


def host_threads():
    """Threads this process may really use: CPU affinity, capped by the cgroup CPU quota (not os.cpu_count())."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]            # cgroup v2
        if quota != "max":
            n = min(n, max(1, int(math.ceil(int(quota) / int(period)))))
    except Exception:
        try:
            quota = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())             # cgroup v1
            period = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if quota > 0 and period > 0:
                n = min(n, max(1, int(math.ceil(quota / period))))
        except Exception:
            pass
    return max(1, n)


def time_reference(hs, args, target_seconds, threads=0, scene=None):
    """Times the reference CPU path (oracle/_ref: the reference's own SamplerIntegrator::Render + PathIntegrator; the
    C++ port if _ref was not built) on a bounded sample of the workload: samples 0 .. k-1 of every pixel of the frame.
    A HaltonSampler's sample i of a pixel does not depend on the total count, so this is a subset of the very samples
    the full render takes, spread uniformly over the frame; the sample's rays per camera sample are printed."""
    from oracle import pyoracle
    checker = pyoracle.reference() or pyoracle.port()
    if checker is None:
        return None, None
    if threads <= 0:
        threads = host_threads()
    if scene is None:
        scene = checker.scene(hs)   # builds the reference's own BVH (seconds for 1 M triangles; outside the timing)
    spp = hs.params.contents.samples_per_pixel
    pixels = args.xres * args.yres
    _, secs, _ = scene.render(n_threads=threads, params=hs.params_copy(samples_per_pixel=1))
    rate = pixels / max(secs, 1e-6)
    k = int(max(1, min(spp, rate * target_seconds // pixels)))
    _, secs, st = scene.render(n_threads=threads, params=hs.params_copy(samples_per_pixel=k))
    nsamp = pixels * k
    rays = int(st.regular_rays + st.shadow_rays)
    return {"value": nsamp / secs / 1e6, "unit": "Msamples/s", "cores": threads, "host_cpus": os.cpu_count(),
            "kind": checker.kind, "seconds": secs, "mrays_per_s": rays / secs / 1e6, "rays_per_sample": rays / nsamp,
            "sample": "samples 0..%d of the %d Halton samples of every pixel of the %dx%d frame (%d camera samples), %d host threads; "
                      "scene generated and flattened by this repo's host front end, rendered by the reference's SamplerIntegrator::Render"
                      % (k - 1, spp, args.xres, args.yres, nsamp, threads)}, scene


def run_reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    hs = build_scene(args)
    vals = []
    info = None
    scene = None
    # every step is a bounded sample of the workload; the whole run stays within ~2.5 minutes of rendering
    per_step = min(args.ref_seconds, 150.0 / max(1, args.warmup + args.steps))
    for i in range(args.warmup + args.steps):
        info, scene = time_reference(hs, args, target_seconds=per_step, scene=scene)
        if info is None:
            print(json.dumps({"impl": "reference", "unavailable": "neither oracle/_ref nor the oracle port is built"}))
            return 0
        if i >= args.warmup:
            vals.append(info)
    # the steps are equal-sized samples of the workload: the value is the mean rate over the timed steps
    best = dict(vals[-1])
    best["value"] = sum(v["value"] * v["seconds"] for v in vals) / sum(v["seconds"] for v in vals)
    best["mrays_per_s"] = sum(v["mrays_per_s"] * v["seconds"] for v in vals) / sum(v["seconds"] for v in vals)
    best["rays_per_sample"] = sum(v["rays_per_sample"] * v["seconds"] for v in vals) / sum(v["seconds"] for v in vals)
    ms = 1e3 * sum(v["seconds"] for v in vals) / len(vals)
    line = {"metric": "Msamples/sec", "value": best["value"], "unit": "Msamples/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic", "impl": "reference",
            "config": workload_config(args, "cpu"),
            "cpu_baseline": {k: best[k] for k in ("value", "unit", "cores", "host_cpus", "kind", "sample", "rays_per_sample")},
            "e2e": {"value": best["value"], "unit": "Msamples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "mrays_per_s": best["mrays_per_s"], "rays_per_sample": best["rays_per_sample"], "gpu_launches": 0}
    print(json.dumps(line))
    return 0


def workload_config(args, parallelism):
    common = {"resolution": [args.xres, args.yres], "spp": args.spp, "maxdepth": args.maxdepth, "parallelism": parallelism}
    if args.workload == "instanced":
        return dict(common, workload="synthetic instanced triangles (SURVEY.md §8d C4): one %d-triangle soup object x %d instances, "
                                     "%dx%dx%dspp Halton, PathIntegrator maxdepth %d, matte Kd .6, 2-triangle area light"
                                     % (args.tris, args.grid * args.grid, args.xres, args.yres, args.spp, args.maxdepth),
                    triangles=args.tris * args.grid * args.grid,
                    l2_note="inputs larger than L2: every step streams the 1 GiB path-context pool through the 50 MB L2; no explicit flush")
    if args.workload == "killeroo":
        return dict(common, workload="scenes/killeroo-simple.pbrt of the reference (SURVEY.md §8d C3): 66 533 primitives (two loop-subdivided "
                                     "killeroos with normals, plastic; sphere area light), %dx%dx%dspp Halton, PathIntegrator maxdepth %d"
                                     % (args.xres, args.yres, args.spp, args.maxdepth),
                    triangles=66532,
                    l2_note="inputs larger than L2: every step streams the 1 GiB path-context pool and the film through the 50 MB L2; "
                            "the scene itself (a few MB) is L2-resident; no explicit flush")
    scene_mb = args.tris * (61 + 48) / 1e6
    return dict(common, workload="synthetic %d random triangles (soup, SURVEY.md §8d C2%s), %dx%dx%dspp Halton, PathIntegrator maxdepth %d, "
                                 "matte Kd .6, 2-triangle area light"
                                 % (args.tris, "" if args.tris == WORKLOAD["tris"] else " generator at another size", args.xres, args.yres, args.spp,
                                    args.maxdepth),
                triangles=args.tris,
                l2_note="inputs larger than L2: every step streams the 1 GiB path-context pool and the film through the 50 MB L2 "
                        "next to the scene (node records + leaf records = %.0f MB); no explicit flush" % scene_mb)


def dump_film(directory, rgbw):
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    if rgbw.nbytes <= DUMP_LIMIT_BYTES:
        np.save(os.path.join(directory, "film.npy"), rgbw)
        return
    pixels = np.sort(np.random.RandomState(0).choice(rgbw.shape[0] * rgbw.shape[1], DUMP_SAMPLE_PIXELS, replace=False))
    np.save(os.path.join(directory, "film_pixels.npy"), pixels.astype(np.float64))
    np.save(os.path.join(directory, "film_sample.npy"), rgbw.reshape(-1, 4)[pixels])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="soup", choices=["soup", "instanced", "killeroo"],
                    help="soup = BASELINE.json configs[1], the headline (default; --tris for the 10 M / 50 M variants); "
                         "killeroo = configs[2]; instanced = configs[3]'s generator")
    ap.add_argument("--tris", type=int, default=None, help="triangles (soup: 1 000 000) / triangles of the instanced object (100 000)")
    ap.add_argument("--seed", type=int, default=WORKLOAD["seed"])
    ap.add_argument("--jitter", type=float, default=None, help="soup: half edge of a triangle's vertex cube (0.02; SURVEY's 50 M scene: 0.005)")
    ap.add_argument("--grid", type=int, default=10, help="instanced: grid x grid instances")
    ap.add_argument("--xres", type=int, default=WORKLOAD["xres"])
    ap.add_argument("--yres", type=int, default=WORKLOAD["yres"])
    ap.add_argument("--spp", type=int, default=None)
    ap.add_argument("--maxdepth", type=int, default=None)
    ap.add_argument("--ref-seconds", type=float, default=15.0, help="CPU seconds per reference sample")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the film (rgb + filter-weight sum, float32) of the last timed step to DIR/film.npy; a film over "
                         "64 MB as a seeded sample of 2^21 pixels: DIR/film_pixels.npy (indices) + DIR/film_sample.npy (rgbw)")
    args = ap.parse_args()
    inst, kill = args.workload == "instanced", args.workload == "killeroo"
    if args.tris is None: args.tris = 100000 if inst else WORKLOAD["tris"]
    if args.spp is None: args.spp = 128 if inst else 256 if kill else WORKLOAD["spp"]
    if args.maxdepth is None: args.maxdepth = 5 if (inst or kill) else WORKLOAD["maxdepth"]
    if args.jitter is None: args.jitter = WORKLOAD["jitter"]
    args.warmup = max(args.warmup, 3)   # timing rule: at least three untimed steps

    if args.impl == "reference":
        return run_reference_arm(args)

    import numpy as np
    import torch
    import torch.distributed as dist

    import pbrt_v3_b200 as pb

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group(backend="nccl", device_id=torch.device("cuda", local_rank))
    pb.init(local_rank)
    L = pb.lib()
    if world > 1:
        # the library's own NCCL communicator (pb2_dist_init): torch.distributed only carries rank 0's unique id to the others
        from pbrt_v3_b200 import multigpu
        multigpu.dist_init_from_torch()

    hs = build_scene(args)
    dev = hs.device_scene()  # BVH + triangles + tables resident in HBM from here on
    h, w = hs.film_shape()
    film = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    # tile_count = 0: the render call is a collective - every rank renders the tiles t with t % world == rank and the
    # library sums the per-rank films onto rank 0 with one ncclReduce on the same stream (the distributed MergeFilmTile)
    params = hs.params_copy(tile_rank=0, tile_count=0)
    stream = torch.cuda.current_stream().cuda_stream
    n_samples = w * h * args.spp

    def step(stats=None):
        pb.check(L.pb2_render_path_device(dev, hs.camera, hs.film, params, C.c_void_p(film.data_ptr()), 1, C.c_void_p(stream), stats))

    def sync():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # algorithmic bytes of one frame: one untimed frame with the counting traversal kernel
    st = pb.Stats()
    count_params = hs.params_copy(tile_rank=0, tile_count=0, flags=1)
    pb.check(L.pb2_render_path_device(dev, hs.camera, hs.film, count_params, C.c_void_p(film.data_ptr()), 1, C.c_void_p(stream), C.byref(st)))
    node_visits, prim_tests = int(st.node_visits), int(st.prim_tests)
    rays_frame = int(st.regular_rays + st.shadow_rays)

    for _ in range(max(args.warmup, 3)):
        step()
    sync()
    clocks = ClockSampler(local_rank)
    clocks.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    launches = 0
    trace_ms = 0.0
    sync()
    e0.record()
    for _ in range(args.steps):
        s = pb.Stats()
        step(s)
        launches += int(s.kernel_launches)
        trace_ms += float(s.trace_ms)
    e1.record()
    sync()
    ms_total = e0.elapsed_time(e1)
    if args.dump_outputs and rank == 0:   # rank 0 holds the merged film of the last timed step
        dump_film(args.dump_outputs, film.cpu().numpy())
    clock_info = clocks.stop()
    t = torch.tensor([ms_total, trace_ms], dtype=torch.float64, device="cuda")
    counts = torch.tensor([float(node_visits), float(prim_tests), float(rays_frame), float(launches)], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(counts, op=dist.ReduceOp.SUM)
    ms_total, trace_ms = float(t[0]), float(t[1])
    node_visits, prim_tests, rays_frame, launches = (int(x) for x in counts.tolist())
    ms_per_step = ms_total / args.steps
    value = n_samples / ms_per_step / 1e3

    # end to end through the host-buffer ABI call pb2_render_path, at every N: structs in, this rank's tiles rendered, the
    # NCCL reduce inside the call, and the merged film copied into rank 0's page-locked host buffer inside the call
    host_ptr = C.c_void_p()
    pb.check(L.pb2_host_alloc(h * w * 16, C.byref(host_ptr)))
    host_film = np.ctypeslib.as_array(C.cast(host_ptr, C.POINTER(C.c_float)), shape=(h, w, 4))
    e2e_ms = []
    for i in range(2 + args.steps):
        sync()
        t0 = time.perf_counter()
        pb.check(L.pb2_render_path(dev, hs.camera, hs.film, params, host_ptr if rank == 0 else None, None))
        sync()
        if i >= 2:
            e2e_ms.append((time.perf_counter() - t0) * 1e3)
    if rank == 0:
        wsum = float(host_film[..., 3].sum())
        assert n_samples <= wsum <= 1.02 * n_samples, "the merged film must hold every camera sample (weight sum %r)" % wsum
    e2e_t = torch.tensor([sum(e2e_ms) / len(e2e_ms)], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(e2e_t, op=dist.ReduceOp.MAX)
    e2e_ms_step = float(e2e_t[0])
    in_bytes = C.sizeof(pb.Camera) + C.sizeof(pb.FilmDesc) + C.sizeof(pb.PathParams)

    if rank == 0:
        peak, peak_src = measured_hbm_peak()
        alg_bytes = 32 * node_visits + 36 * prim_tests  # SURVEY.md §8d, whole frame, all ranks
        trace_s = trace_ms / args.steps / 1e3           # max over ranks of the summed trace-kernel time per frame
        achieved = (alg_bytes / world) / trace_s / 1e9 if trace_s > 0 else None
        line = {
            "metric": "Msamples/sec", "value": value, "unit": "Msamples/s", "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic", "config": workload_config(args, "tiles-dp%d" % world),
            "mrays_per_s": rays_frame / ms_per_step / 1e3, "rays_per_sample": rays_frame / n_samples,
            "e2e": {"value": n_samples / e2e_ms_step / 1e3, "unit": "Msamples/s", "ms_per_step": e2e_ms_step,
                    "h2d_bytes_per_step": in_bytes, "d2h_bytes_per_step": int(host_film.nbytes),
                    "note": "scene upload happens once at pb2_scene_create (outside, like the reference's scene construction); "
                            "per step the camera/film/integrator structs go in and the merged rgbw film comes back"},
            "gpu_launches": launches, "clocks": clock_info,
            "roofline": {"kernel": "k_wf_trace_w (BVH traversal + ray/triangle tests)", "bound": "hbm", "achieved": achieved, "peak": peak,
                         "unit": "GB/s", "frac": (achieved / peak) if achieved else None, "peak_source": peak_src,
                         "basis": "NOMINAL: `achieved` divides the reference traversal's algorithmic bytes (SURVEY.md 8d: 32 B x node visits + 36 B x "
                                  "primitive tests, counted on the device) by the kernel's time; much of that traffic is served from L2, "
                                  "so it is not the kernel's DRAM traffic",
                         "algorithmic_bytes_per_frame": alg_bytes, "node_visits": node_visits, "prim_tests": prim_tests,
                         "bytes_per_ray": alg_bytes / max(rays_frame, 1), "trace_ms_per_frame": trace_ms / args.steps,
                         "trace_share_of_step": (trace_ms / args.steps) / ms_per_step,
                         "concurrency_note": "the renderer runs two wavefront pipelines on two streams: a trace launch shares the GPU with the other "
                                             "pipeline's kernels, so the summed launch durations (trace_ms_per_frame) can exceed the kernel's share of "
                                             "the step and `achieved` is the per-launch figure under that sharing",
                         "frac_of_step": (alg_bytes / world) / (ms_per_step / 1e3) / 1e9 / peak},
        }
        if not args.no_cpu_baseline and world == 1:   # the CPU side-by-side is reported by the N = 1 run only
            try:
                cb, _ = time_reference(hs, args, target_seconds=args.ref_seconds)
                if cb:
                    line["cpu_baseline"] = {k: cb[k] for k in ("value", "unit", "cores", "host_cpus", "kind", "sample", "rays_per_sample")}
                    line["cpu_baseline"]["mrays_per_s"] = cb["mrays_per_s"]
            except Exception as e:  # the baseline is reporting only; never lose the GPU line
                line["cpu_baseline"] = {"error": repr(e)}
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        L.pb2_dist_shutdown()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
