"""The render kernels' own radiance, bit for bit: one-sample frames.

Elsewhere a rendered film is held to the model of its samples only within k * 2^-24 * sum |L * w|, the bound of float32
additions in any order (the film is summed with atomics).  That bound lets one sample of a pixel be several ulps off, or
every sample of a frame one ulp off.  At one sample per pixel with the box filter of radius 0.5, FilmTile::AddSample puts
a sample into the one pixel its pFilm lies in, so a pixel's RGB is 0 + L of ONE path exactly as the wavefront kernels
computed it, and its weight is 1.  Those kernels are k_wf_advance's shade and light steps of every shade class and
instantiation, the chained light step of the trace kernel, k_wf_finish and the re-shade of lazily lit vertices.  A sample
whose pFilm coordinate is an integer (Halton index below baseScales[0] for x, below baseScales[1] for y) lands in 2 or 4
pixels.  A pixel with two deposits holds (0 + a) + b, which does not depend on the order of a and b.  Checks:

  1. every configuration of the round loop renders every case at one sample per pixel, each configuration in a worker
     process of its own (the knobs are read once per process): test_gpu_wavefront_schedules.SCHEDULES with every flag of
     case_flags, and PB2_SHADE_GENERAL=1 with and without the tail kernel.  The pipe schedules need 65 536 work items or
     more: they render at a raised film resolution (about 160 000 pixels) instead of a raised sample count;
  2. the weight channel equals the number of deposits in every pixel; the RGB of every pixel with at most two deposits
     equals float32(0) + a (+ b) of pb2_li_samples' L bit for bit; pixels with three or more deposits (a handful) get the
     float32 bound;
  3. ray counters are equal in every configuration, and camera rays equal the work items;
  4. the benchmark's shapes as bench.build_scene makes them (the 1 M-triangle soup, killeroo-simple, the instanced
     generator; 1920 x 1080) with the shipped settings: class-0 kernels, two pipelines, the real pool;
  5. the films of a three-way tile partition, summed, and with two devices both multi-GPU forms, give the film bit for bit;
  6. pb2_li_samples of the native-resolution one-sample frames equals the reference's PathIntegrator::Li, recorded in
     device-math mode by tests/make_golden.py (record_reference below) into tests/golden/one_sample.npz.  The sample count
     sets the scale of the ray differentials (1 / sqrt(spp)), so test_gpu_exact_parity's frames do not cover these.
"""
import argparse
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import golden_cases as gc
import test_gpu_shade_classes as sc_t
import test_gpu_wavefront_schedules as ws
from conftest import GOLDEN, ROOT, SCENES

TESTS = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(GOLDEN, "one_sample.npz")

CASES = ws.CASES + ["matte_box", "matte_mesh_lights"]
CONFIGS = {name: env for name, (env, _) in ws.SCHEDULES.items()}
CONFIGS.update({"general": {"PB2_SHADE_GENERAL": "1"}, "general_rounds": {"PB2_SHADE_GENERAL": "1", "PB2_FINISH": "0"}})
PIPED = tuple(name for name, (_, pipes) in ws.SCHEDULES.items() if pipes)
PARTITION_CASES = ("params", "soup")
KNOBS = ("PB2_POOL", "PB2_PIPES", "PB2_FINISH", "PB2_SYNC_EVERY", "PB2_LIGHTDIST_LAZY", "PB2_SHADE_GENERAL")
MAX_CROWDED = 8        # pixels with three or more deposits allowed in one frame


# ---------------------------------------------------------------------------------------------------------------------
# Cases at one sample per pixel, at the native film resolution or scaled up
# ---------------------------------------------------------------------------------------------------------------------
def case_text(case):
    """The scene text of a case, with every file it reads named by absolute path."""
    if case in ws.GOLDEN_CASES:
        return gc.scene_file_text(SCENES, case)
    if case == "gaussian":     # its filter is modelled by test_gpu_wavefront_schedules; here it renders with the box filter
        text = ws.case_text(case)
        assert text.count('PixelFilter "gaussian"') == 1
        return text.replace('PixelFilter "gaussian"', 'PixelFilter "box"')
    return sc_t.case_text(case)


def scaled(text, s):
    """The scene with its film resolution (and the integrator's pixel bounds) s times larger in x and y."""
    text, n = re.subn(r'("integer [xy]resolution"\s*\[?\s*)(\d+)', lambda m: m.group(1) + str(int(m.group(2)) * s), text)
    assert n == 2, n
    return re.sub(r'("integer pixelbounds"\s*\[)([\d\s]+)\]', lambda m: m.group(1) + " ".join(str(int(v) * s) for v in m.group(2).split()) + "]", text)


def make_case(pb, case, s=1):
    """A case's scene; s > 1: its film s times larger in x and y (the files under tests/scenes are read, never written)."""
    if case == "soup":
        return gc.soup_scene(pb, xres=gc.SOUP["xres"] * s, yres=gc.SOUP["yres"] * s)
    if case == "instanced_soup":
        return pb.HostScene.instanced_soup(2000, grid=4, xres=64 * s, yres=36 * s, spp=4)
    if s == 1 and case != "gaussian":
        return sc_t.make_case(pb, case)
    return pb.HostScene.from_string(scaled(case_text(case), s))


def one_sample(hs, **over):
    return hs.params_copy(samples_per_pixel=1, **over)


def pipe_scale(pb, case):
    """Film scale that gives a pipe schedule about ws.PIPE_ITEMS work items at one sample per pixel."""
    from pbrt_v3_b200 import multigpu
    hs = make_case(pb, case)
    return math.ceil(math.sqrt(ws.PIPE_ITEMS / len(multigpu.work_items(hs.film, one_sample(hs)))))


# ---------------------------------------------------------------------------------------------------------------------
# What the film of one-sample frames must hold (host arithmetic only)
# ---------------------------------------------------------------------------------------------------------------------
def expected_film(film, li, pfilm):
    """Per pixel of the box-filtered film: the deposits k (FilmTile::AddSample's range, test_gpu_wavefront_schedules.deposits),
    the first and second sample deposited there (-1: none) and, where k <= 2, the float32 RGB 0 + a (+ b) of the clamped L."""
    x0, y0, x1, y1 = (int(v) for v in film.cropped_pixel_bounds)
    h, w = y1 - y0, x1 - x0
    L = ws.clamped_samples(film, li)
    pix, smp = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    for sel, xs, ys, tab in ws.deposits(film, pfilm):
        assert tab is None, "one-sample frames are rendered with the box filter"
        pix.append((ys - y0) * w + (xs - x0))
        smp.append(sel)
    pix, smp = np.concatenate(pix), np.concatenate(smp)
    order = np.argsort(pix, kind="stable")
    pix, smp = pix[order], smp[order]
    k = np.bincount(pix, minlength=h * w)
    start = np.cumsum(k) - k
    first, second = np.full(h * w, -1), np.full(h * w, -1)
    first[k >= 1] = smp[start[k >= 1]]
    second[k >= 2] = smp[start[k >= 2] + 1]
    rgb = np.zeros((h * w, 3), np.float32)
    rgb[k >= 1] = np.float32(0) + L[first[k >= 1]]
    rgb[k == 2] = rgb[k == 2] + L[second[k == 2]]
    return {"k": k.reshape(h, w), "rgb": rgb.reshape(h, w, 3), "first": first.reshape(h, w), "second": second.reshape(h, w), "L": L}


def ulps(a, b):
    """Distance in float32 ulps (across zero too)."""
    ia, ib = (np.int64(np.float32(v).view(np.int32)) for v in (a, b))
    ia, ib = (v if v >= 0 else -(v & 0x7fffffff) for v in (ia, ib))
    return int(abs(ia - ib))


def film_check(film, rgbw, exp, items, model_bound):
    """Compares one rendered film with expected_film.  Returns (summary, message): summary = [pixels, pixels compared bit for
    bit (k <= 2), pixels with 2 deposits, pixels with 3+, pixels that differ, weight channel equal]; message is None or why
    the film differs, with the first differing pixel, its work item, both L values and their ulp distance."""
    k, want = exp["k"], exp["rgb"]
    x0, y0 = int(film.cropped_pixel_bounds[0]), int(film.cropped_pixel_bounds[1])
    rgbw = np.asarray(rgbw, np.float32)
    exact = k <= 2
    weight_ok = np.array_equal(rgbw[..., 3], k.astype(np.float32))
    differ = exact & (rgbw[..., :3].view(np.uint32) != want.view(np.uint32)).any(-1)
    crowded = ~exact
    if crowded.any():
        model, bound = model_bound()
        differ |= crowded & (np.abs(rgbw[..., :3].astype(np.float64) - model[..., :3]) > bound[..., :3]).any(-1)
    summary = [k.size, int(exact.sum()), int((k == 2).sum()), int(crowded.sum()), int(differ.sum()), int(weight_ok)]
    why = []
    if not weight_ok:
        bad = np.argwhere(rgbw[..., 3] != k)[0]
        why.append("weight channel differs from the deposit count in %d pixels (first x %d y %d: %g, %d deposits)"
                   % ((rgbw[..., 3] != k).sum(), bad[1] + x0, bad[0] + y0, rgbw[tuple(bad) + (3,)], k[tuple(bad)]))
    if differ.any():
        y, x = np.argwhere(differ)[0]
        c = int(np.flatnonzero(rgbw[y, x, :3].view(np.uint32) != want[y, x].view(np.uint32))[0]) if exact[y, x] else 0
        i = exp["first"][y, x]
        msg = ("%d pixels differ (first x %d y %d, %d deposits, channel %d): film %r, expected %r (%d ulps); work item %s, "
               "pb2_li_samples L %r" % (differ.sum(), x + x0, y + y0, k[y, x], c, rgbw[y, x, :3].tolist(), want[y, x].tolist(),
                                        ulps(rgbw[y, x, c], want[y, x, c]), items[i].tolist() if i >= 0 else None,
                                        exp["L"][i].tolist() if i >= 0 else None))
        if exp["second"][y, x] >= 0:
            msg += "; second work item %s, L %r" % (items[exp["second"][y, x]].tolist(), exp["L"][exp["second"][y, x]].tolist())
        why.append(msg)
    return np.array(summary, np.int64), ("; ".join(why) or None)


# ---------------------------------------------------------------------------------------------------------------------
# The workers: one process per configuration
# ---------------------------------------------------------------------------------------------------------------------
def frame(pb, hs, flags_list, partition=False):
    """Renders hs at one sample per pixel under every flag and checks each film; the samples come from pb2_li_samples."""
    from pbrt_v3_b200 import multigpu
    film = hs.film.contents
    params = one_sample(hs)
    items = multigpu.work_items(hs.film, params)
    li, pfilm = hs.li_samples(items[:, :2], items[:, 2].astype(np.int64), params)
    exp = expected_film(film, li, pfilm)
    memo = []

    def model_bound():
        if not memo:
            memo.append(ws.film_model(film, li, pfilm))
        return memo[0]
    out = {"flags": np.array(flags_list), "items": np.int64(len(items))}
    summaries, messages, stats = [], [], []
    for f in flags_list:
        rgbw, st = hs.render_rgbw(one_sample(hs, flags=f))
        s, why = film_check(film, rgbw, exp, items, model_bound)
        summaries.append(s)
        messages.append(why or "")
        stats.append([st.camera_rays, st.regular_rays, st.shadow_rays])
    out.update({"summary": np.array(summaries), "message": np.array(messages), "stats": np.array(stats, np.int64)})
    if partition:
        s, m = [], []
        for f in flags_list[:2]:
            parts = sum(hs.render_rgbw(one_sample(hs, flags=f, tile_rank=r, tile_count=3))[0].astype(np.float64) for r in range(3))
            a, why = film_check(film, parts.astype(np.float32), exp, items, model_bound)
            s.append(a)
            m.append(why or "")
        out.update({"parts_summary": np.array(s), "parts_message": np.array(m)})
    return out, items, li, pfilm


def render_config(name, out):
    import pbrt_v3_b200 as pb
    res = {}
    for case in CASES:
        env = ws.CASE_ENV.get(case, {})
        os.environ.update(env)
        try:
            hs = make_case(pb, case, pipe_scale(pb, case) if name in PIPED else 1)
            r, items, li, pfilm = frame(pb, hs, ws.case_flags(pb, case), partition=case in PARTITION_CASES and name in ws.PARTITION_SCHEDULES)
            if name == "shipped":
                r["pixels"], r["digest"] = gc.pixel_digests(items, li, pfilm)
            res.update({case + ":" + k: v for k, v in r.items()})
        finally:
            for key in env:
                os.environ.pop(key, None)
    np.savez(out, **res)


BENCH_SHAPES = ("soup", "killeroo", "instanced")


def bench_args(workload):
    import bench
    a = dict(bench.WORKLOAD, workload=workload, grid=10, spp=1)
    if workload != "soup":
        a.update(tris=100000, maxdepth=5)
    return argparse.Namespace(**a)


def render_bench(out):
    import bench
    import pbrt_v3_b200 as pb
    res = {}
    for w in BENCH_SHAPES:
        hs = bench.build_scene(bench_args(w))
        r, _, _, _ = frame(pb, hs, [0])
        res.update({w + ":" + k: v for k, v in r.items()})
        del hs
    np.savez(out, **res)


WORKER = r'''
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_gpu_sample_films as t
if sys.argv[3] == "bench":
    t.render_bench(sys.argv[4])
else:
    t.render_config(sys.argv[3], sys.argv[4])
print(sys.argv[3], "ok")
'''


@pytest.fixture(scope="module")
def config(tmp_path_factory):
    """config(name) -> {case: {field: array}} of that configuration's worker (run once per module, on first use)."""
    d = tmp_path_factory.mktemp("sample_films")
    script = d / "worker.py"
    script.write_text(WORKER)
    done = {}

    def get(name):
        if name not in done:
            out = d / (name + ".npz")
            env = dict(os.environ)
            for knob in KNOBS:
                env.pop(knob, None)
            env.update(CONFIGS.get(name, {}))
            res = subprocess.run([sys.executable, str(script), ROOT, TESTS, name, str(out)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                 text=True, timeout=1200, cwd=ROOT, env=env)
            if res.returncode != 0:
                done[name] = "worker for %s failed:\n%s" % (name, res.stdout[-4000:])
            else:
                z = np.load(out)
                cases = {}
                for key in z.files:
                    case, field = key.split(":")
                    cases.setdefault(case, {})[field] = z[key]
                done[name] = cases
        if isinstance(done[name], str):
            pytest.fail(done[name])
        return done[name]
    return get


def assert_films(r, what, summary="summary", message="message"):
    for f, s, m in zip(r["flags"], r[summary], r[message]):
        pixels, exact, two, crowded, differ, weight_ok = (int(v) for v in s)
        assert not m, "%s, flags %d: %s" % (what, f, m)
        assert weight_ok and differ == 0
        assert exact > 0.99 * pixels, "%s, flags %d: only %d of %d pixels compared bit for bit" % (what, f, exact, pixels)
        assert crowded <= MAX_CROWDED, "%s, flags %d: %d pixels with three or more deposits" % (what, f, crowded)


# ---------------------------------------------------------------------------------------------------------------------
# Checks 1-3: every configuration, every case, every flag
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_one_sample_film_is_the_samples_bit_for_bit(config, name, case):
    r = config(name)[case]
    assert_films(r, "%s / %s" % (name, case))
    assert (r["stats"][:, 0] == r["items"]).all(), ("camera rays", r["stats"][:, 0].tolist(), int(r["items"]))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_ray_counters_of_one_sample_frames_do_not_depend_on_the_configuration(config, case):
    for names in ([n for n in CONFIGS if n not in PIPED], list(PIPED)):
        seen = {(n, int(f)): tuple(int(v) for v in st) for n in names for f, st in zip(config(n)[case]["flags"], config(n)[case]["stats"])}
        assert len(set(seen.values())) == 1, seen


# ---------------------------------------------------------------------------------------------------------------------
# Check 4: the benchmark's shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("workload", BENCH_SHAPES)
def test_benchmark_shapes_at_one_sample_are_the_samples_bit_for_bit(config, workload):
    r = config("bench")[workload]
    assert int(r["items"]) == 1920 * 1080
    assert_films(r, workload)
    assert int(r["stats"][0][0]) == int(r["items"])


# ---------------------------------------------------------------------------------------------------------------------
# Check 5: partitions of the frame
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", PARTITION_CASES)
@pytest.mark.parametrize("name", ws.PARTITION_SCHEDULES)
def test_tile_partition_of_one_sample_frames_is_bit_for_bit(config, name, case):
    """Each rank film holds 0 + a (+ b) of its own deposits; their float64 sum rounded to float32 is (0 + a) + b."""
    r = config(name)[case]
    assert_films(dict(r, flags=r["flags"][:2]), "%s / %s, tile_count = 3" % (name, case), "parts_summary", "parts_message")


MULTI_WORKER = r'''
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import pbrt_v3_b200 as pb
import test_gpu_sample_films as t
dist = sys.argv[3] == "dist"
if dist:
    import torch, torch.distributed as td
    from pbrt_v3_b200 import multigpu
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    td.init_process_group(backend="nccl", device_id=torch.device("cuda", local))
    pb.init(local)
    rank, world = multigpu.dist_init_from_torch()
else:
    pb.check(pb.lib().pb2_init_devices(0, None))
    rank = 0
L = pb.lib()
for case in ("soup", "killeroo_like", "instanced_soup"):
    hs = t.make_case(pb, case, 4)
    dev = hs.device_scene()
    h, w = hs.film_shape()
    group = np.zeros((h, w, 4), np.float32)
    pb.check(L.pb2_render_path(dev, hs.camera, hs.film, t.one_sample(hs, tile_rank=0, tile_count=0), pb.ptr(group) if rank == 0 else None, None))
    if rank == 0:
        alone = np.zeros((h, w, 4), np.float32)
        pb.check(L.pb2_render_path(dev, hs.camera, hs.film, t.one_sample(hs, tile_rank=0, tile_count=1), pb.ptr(alone), None))
        k = t.expected_film(hs.film.contents, *hs.li_samples(*t.sample_ids(hs)))["k"]
        assert np.array_equal(group[k <= 2].view(np.uint32), alone[k <= 2].view(np.uint32)), case
        assert np.allclose(group, alone, rtol=1e-6, atol=1e-6), case
    if dist:
        td.barrier()
if dist:
    L.pb2_dist_shutdown()
    td.destroy_process_group()
print("rank", rank, "ok")
'''


def sample_ids(hs):
    """(pixel xy, sample number, params) of every work item of a one-sample frame: pb2_li_samples' arguments."""
    from pbrt_v3_b200 import multigpu
    params = one_sample(hs)
    items = multigpu.work_items(hs.film, params)
    return items[:, :2], items[:, 2].astype(np.int64), params


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["dist", "group"])
def test_multi_gpu_one_sample_films_equal_the_single_gpu_film(tmp_path, form):
    """pb2_dist_init (two processes, the NCCL reduce) and pb2_init_devices (one process, every visible device): the merged
    film equals the single-GPU film bit for bit in every pixel with at most two deposits."""
    import socket

    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    script = tmp_path / "multi.py"
    script.write_text(MULTI_WORKER)
    if form == "group":
        cmd = [sys.executable, str(script), ROOT, TESTS, form]
    else:
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
               "--master-port", str(port), str(script), ROOT, TESTS, form]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0 and " ok" in res.stdout, res.stdout[-4000:]


# ---------------------------------------------------------------------------------------------------------------------
# Check 6: the one-sample frames' samples against the reference
# ---------------------------------------------------------------------------------------------------------------------
def record_reference(ref, path):
    """Per-pixel digests of the sample number, L and pFilm of every work item of every case's native-resolution one-sample
    frame, as the compiled reference computes them in device-math mode (run by tests/make_golden.py)."""
    import pbrt_v3_b200 as pb
    out = {}
    with ref.device_math():
        for case in CASES:
            hs = make_case(pb, case)
            pix, sn, params = sample_ids(hs)
            li, pfilm = ref.scene(hs).li_samples(pix, sn, params)
            out[case + ":pixels"], out[case + ":digest"] = gc.pixel_digests(np.c_[pix, sn], li, pfilm)
    np.savez_compressed(path, **out)


@pytest.fixture(scope="module")
def want():
    if not os.path.exists(FIXTURE):
        pytest.fail("%s is missing: tests/make_golden.py records it from the compiled reference" % FIXTURE)
    z = np.load(FIXTURE)
    return {k: z[k] for k in z.files}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_one_sample_frames_equal_the_reference(config, want, case):
    """pb2_li_samples' samples of the frames rendered above (the shipped worker) against the reference's, pixel by pixel;
    no exceptions."""
    r = config("shipped")[case]
    assert np.array_equal(r["pixels"], want[case + ":pixels"]), "the work items cover other pixels than the reference's"
    bad = r["pixels"][r["digest"] != want[case + ":digest"]]
    assert len(bad) == 0, "samples of %d of %d pixels differ from the reference's (first pixels %s)" % (len(bad), len(r["pixels"]), bad[:10].tolist())


def test_fixture_is_what_the_reference_records(pb, tmp_path):
    """tests/golden/one_sample.npz is what record_reference gives with the compiled reference, where it is built."""
    from oracle import pyoracle
    ref = pyoracle.reference()
    if ref is None or not ref.has_device_math:
        pytest.skip("the compiled reference (oracle/_ref) with device math is not built here")
    record_reference(ref, str(tmp_path / "one_sample.npz"))
    got, fixture = np.load(tmp_path / "one_sample.npz"), np.load(FIXTURE)
    assert sorted(got.files) == sorted(fixture.files)
    for key in got.files:
        assert np.array_equal(got[key], fixture[key]), key


@pytest.mark.parametrize("case", CASES)
def test_cases_render_with_the_box_filter_and_scale_for_the_pipes(pb, case):
    """The premises of the checks, on the host: every case's film has the box filter of radius 0.5, and its scaled-up film
    gives the pipe schedules 65 536 work items or more at one sample per pixel, in the same scene (the same shade class)."""
    from pbrt_v3_b200 import multigpu
    hs = make_case(pb, case)
    film = hs.film.contents
    assert film.filter_type == pb.PB2_FILTER_BOX and tuple(film.filter_radius) == (.5, .5)
    native = (len(multigpu.work_items(hs.film, one_sample(hs))), sc_t.shade_class(pb, hs), hs.desc.contents.n_prims)
    s = pipe_scale(pb, case)
    big = make_case(pb, case, s)
    assert len(multigpu.work_items(big.film, one_sample(big))) >= max(65536, native[0] * s * s * 9 // 10)
    assert (sc_t.shade_class(pb, big), big.desc.contents.n_prims) == native[1:]
