"""Developer script (runs on a GPU machine): what giving up trace blocks costs, and what sharing the SMs gains.

    python tools/coresident_sweep.py [--workload soup|killeroo|instanced] [--spp N] [--frames F] [--json FILE]

Builds the scene bench.py builds (tools/kernel_times.py's defaults) and, for each persistent trace grid of 8, 7, 6 and
5 blocks per SM (PB2_TRACE_BLOCKS) and the grid renderWavefront sizes itself (the list-kernel reserve):
  1. one pipeline (PB2_PIPES=1): the per-kernel times of one frame under torch.profiler, after warm-up frames, and the
     frame's device time unprofiled;
  2. two pipelines: the frame's device time unprofiled.
PB2_PIPES is read once per process, so each pipeline count runs in a worker process of its own; PB2_TRACE_BLOCKS is
read at every render.  Frame times are the median of --frames frames, device events around each.  The
card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SETTINGS = ["8", "7", "6", "5", "auto"]   # PB2_TRACE_BLOCKS ("auto": unset)


def worker(args):
    import ctypes as C

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    import kernel_times
    import pbrt_v3_b200 as pb

    pipes = int(os.environ["PB2_PIPES"])
    inst, kill = args.workload == "instanced", args.workload == "killeroo"
    w = bench.WORKLOAD
    scene_args = argparse.Namespace(
        workload=args.workload, seed=w["seed"], jitter=w["jitter"], xres=w["xres"], yres=w["yres"], grid=10,
        tris=100000 if inst else w["tris"], spp=args.spp if args.spp is not None else (128 if inst else 256 if kill else w["spp"]),
        maxdepth=5 if (inst or kill) else w["maxdepth"])
    torch.cuda.set_device(0)
    pb.init(0)
    L = pb.lib()
    hs = bench.build_scene(scene_args)
    dev = hs.device_scene()
    h, wd = hs.film_shape()
    film = torch.zeros((h, wd, 4), dtype=torch.float32, device="cuda")
    params = hs.params_copy(tile_rank=0, tile_count=0)
    stream = torch.cuda.current_stream().cuda_stream

    def frame():
        pb.check(L.pb2_render_path_device(dev, hs.camera, hs.film, params, C.c_void_p(film.data_ptr()), 1, C.c_void_p(stream), None))

    def frame_ms():
        times = []
        for _ in range(args.frames):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            frame()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        return sorted(times)[len(times) // 2], times

    rows = []
    for blocks in SETTINGS:
        if blocks == "auto":
            os.environ.pop("PB2_TRACE_BLOCKS", None)
        else:
            os.environ["PB2_TRACE_BLOCKS"] = blocks
        for _ in range(args.warmup):
            frame()
        torch.cuda.synchronize()
        med, times = frame_ms()
        row = {"pipes": pipes, "trace_blocks": blocks, "frame_ms": med, "frames_ms": times}
        if pipes == 1:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                frame()
                torch.cuda.synchronize()
            per = {}
            for ev in prof.events():
                if ev.device_type != torch.autograd.DeviceType.CUDA or "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
                    continue
                k = kernel_times.kernel_name(ev.name)
                per[k] = per.get(k, 0.0) + ev.time_range.elapsed_us() / 1e3
            row["kernels_ms"] = per
        rows.append(row)
        print(json.dumps({k: v for k, v in row.items() if k != "frames_ms"}), flush=True)
    with open(args.out, "w") as f:
        json.dump({"workload": vars(scene_args), "rows": rows}, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="soup", choices=["soup", "instanced", "killeroo"])
    ap.add_argument("--spp", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write every row as JSON to this file")
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)

    import tempfile

    import kernel_times
    card = kernel_times.card_info(0)
    print("card: %s" % json.dumps(card), flush=True)
    rows, workload = [], None
    with tempfile.TemporaryDirectory() as d:
        for pipes in (1, 2):
            out = os.path.join(d, "pipes%d.json" % pipes)
            env = dict(os.environ, PB2_PIPES=str(pipes))
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "1", "--out", out, "--workload", args.workload,
                   "--warmup", str(args.warmup), "--frames", str(args.frames)] + (["--spp", str(args.spp)] if args.spp else [])
            subprocess.run(cmd, env=env, check=True)
            with open(out) as f:
                r = json.load(f)
            rows += r["rows"]
            workload = r["workload"]
    print("workload: %s" % json.dumps(workload))
    kernels = []
    for r in rows:
        for k in r.get("kernels_ms", {}):
            if k not in kernels:
                kernels.append(k)
    one = [r for r in rows if r["pipes"] == 1]
    print("one pipeline, ms per frame (kernels: one profiled frame; frame: median of %d, device events, unprofiled)" % args.frames)
    print("%-60s" % "trace blocks per SM" + "".join("%10s" % r["trace_blocks"] for r in one))
    for k in kernels:
        print("%-60s" % k[:60] + "".join("%10.1f" % r["kernels_ms"].get(k, 0.0) for r in one))
    print("%-60s" % "frame" + "".join("%10.1f" % r["frame_ms"] for r in one))
    two = [r for r in rows if r["pipes"] == 2]
    print("two pipelines, frame ms (median of %d, device events, unprofiled)" % args.frames)
    print("%-60s" % "trace blocks per SM" + "".join("%10s" % r["trace_blocks"] for r in two))
    print("%-60s" % "frame" + "".join("%10.1f" % r["frame_ms"] for r in two))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card, "workload": workload, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
