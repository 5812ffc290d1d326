"""Developer script (runs on a GPU machine): where one frame of the bench workload spends its device time, per kernel.

    python tools/kernel_times.py [--workload soup|killeroo|instanced] [--spp N] [--warmup W] [--json FILE]

Builds the scene bench.py builds (same defaults: BASELINE.json configs[1], 1 M triangles, 1920x1080x64), renders
--warmup frames, then records ONE frame with torch.profiler (CUDA activities only) and prints, per kernel name (template
arguments kept, parameter list dropped), the number of launches, the summed launch durations and their share of the
summed durations of all kernels.  The two wavefront pipelines run on two streams, so the summed durations exceed the
frame's wall time; the frame's device time is measured in a separate, unprofiled frame and printed too.  The card's name
and power limit are read in the same run: a time is a time on that card at that limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (build_scene and the workload defaults)


def card_info(index):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"error": repr(e)}


def kernel_name(name):
    name = name.split("(")[0]
    return name[5:] if name.startswith("void ") else name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="soup", choices=["soup", "instanced", "killeroo"])
    ap.add_argument("--tris", type=int, default=None)
    ap.add_argument("--spp", type=int, default=None)
    ap.add_argument("--maxdepth", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the table as JSON to this file")
    args = ap.parse_args()
    inst, kill = args.workload == "instanced", args.workload == "killeroo"
    w = bench.WORKLOAD
    scene_args = argparse.Namespace(
        workload=args.workload, seed=w["seed"], jitter=w["jitter"], xres=w["xres"], yres=w["yres"], grid=10,
        tris=args.tris if args.tris is not None else (100000 if inst else w["tris"]),
        spp=args.spp if args.spp is not None else (128 if inst else 256 if kill else w["spp"]),
        maxdepth=args.maxdepth if args.maxdepth is not None else (5 if (inst or kill) else w["maxdepth"]))

    import torch
    from torch.profiler import ProfilerActivity, profile

    import pbrt_v3_b200 as pb

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

    for _ in range(max(1, args.warmup)):
        frame()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    frame()
    e1.record()
    torch.cuda.synchronize()
    frame_ms = e0.elapsed_time(e1)

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        frame()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
            continue
        k = kernel_name(ev.name)
        n, us = per.get(k, (0, 0.0))
        per[k] = (n + 1, us + ev.time_range.elapsed_us())
    total_us = sum(us for _, us in per.values())
    rows = sorted(((k, n, us) for k, (n, us) in per.items()), key=lambda r: -r[2])

    card = card_info(0)
    print("card: %s" % json.dumps(card))
    print("workload: %s %dx%dx%d spp, maxdepth %d; frame %.1f ms (device events, unprofiled)"
          % (args.workload, scene_args.xres, scene_args.yres, scene_args.spp, scene_args.maxdepth, frame_ms))
    print("%-70s %8s %11s %7s" % ("kernel", "launches", "total ms", "share"))
    for k, n, us in rows:
        print("%-70s %8d %11.2f %6.1f%%" % (k[:70], n, us / 1e3, 100.0 * us / total_us))
    print("%-70s %8d %11.2f" % ("all kernels (summed launch durations, two streams)", sum(r[1] for r in rows), total_us / 1e3))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card, "workload": vars(scene_args), "frame_ms": frame_ms, "kernels_total_ms": total_us / 1e3,
                       "kernels": [{"name": k, "launches": n, "ms": us / 1e3, "share": us / total_us} for k, n, us in rows]}, f, indent=1)


if __name__ == "__main__":
    main()
