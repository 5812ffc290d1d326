"""The wavefront round loop (renderWavefront: k_wf_gen, the trace kernel, k_wf_advance<light>, k_wf_advance<shade>,
k_wf_finish, k_wf_reset) under schedules that the golden scenes never reach with the shipped settings.

A golden scene has at most 49 152 work items, so with the shipped settings every sample gets a context of its own in
round 0 (no context is ever recycled), one pipeline runs, and k_wf_finish walks every path to its end right after the
first round: the tuned trace kernels see camera rays only and the light step never runs.  The schedule knobs
(PB2_POOL, PB2_PIPES, PB2_FINISH, PB2_SYNC_EVERY) are read once per process, so each schedule renders every case in a
worker process of its own; the tests read what the workers wrote.

Checks:
  1. per-pixel model: every work item's L and pFilm from pb2_li_samples (one thread per sample, the same lane functions),
     clamped like addSample and deposited in float64 with FilmTile::AddSample's pixel range.  The weight channel of a
     box-filtered film must equal the model's exactly; every RGB value must lie within k * 2^-24 * sum |L * w| of the
     model, k = deposits in the pixel: the error bound of float32 additions in any order.  This rests on a path's L being
     bit-identical in the wavefront and in pb2_li_samples, which tests/test_gpu_sample_films.py checks: at one sample per
     pixel the film holds each path's L itself, in every schedule and configuration of this file.
  2. ray counters: camera rays = valid work items; regular and shadow rays equal in every schedule and under every flag.
  3. the golden scenes at native spp, with the rounds forced, against the reference's image and ray counts.
  4. PB2_FLAG_CHAIN: checks 1-3 everywhere, fewer launches, and the reference's emissive-sphere furnace.
  5. tile partitions: the films of tile_count = 3 sum to the model of the full film.
"""
import ctypes as C
import ctypes.util
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import golden_cases as gc
from conftest import GOLDEN, ROOT, SCENES

TESTS = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -24   # unit roundoff of float32

# name: (environment, pipelines).  Pipelines need a pool of 65 536 contexts, so the pipe schedules render every case at
# a raised sample count (about 160 000 valid work items): each pipeline's pool is refilled at least twice.
SCHEDULES = {
    "shipped": ({}, False),
    "rounds": ({"PB2_FINISH": "0"}, False),                                           # every bounce through the round kernels
    "refill": ({"PB2_FINISH": "0", "PB2_POOL": "2048"}, False),                        # contexts recycled many times
    "refill_tail": ({"PB2_POOL": "2048"}, False),                                     # k_wf_finish on recycled contexts
    "tiny": ({"PB2_FINISH": "0", "PB2_POOL": "256", "PB2_SYNC_EVERY": "1"}, False),    # hundreds of rounds, checked every round
    "pipes2": ({"PB2_POOL": "65536", "PB2_PIPES": "2"}, True),
    "pipes2_rounds": ({"PB2_POOL": "65536", "PB2_PIPES": "2", "PB2_FINISH": "0"}, True),
    "pipes3": ({"PB2_POOL": "65536", "PB2_PIPES": "3"}, True),                         # 65 536 is not a multiple of 3
    "pipes3_rounds": ({"PB2_POOL": "65536", "PB2_PIPES": "3", "PB2_FINISH": "0"}, True),
    "pipes4": ({"PB2_POOL": "65536", "PB2_PIPES": "4"}, True),
    "pipes4_rounds": ({"PB2_POOL": "65536", "PB2_PIPES": "4", "PB2_FINISH": "0"}, True),
}
PIPE_ITEMS = 160000
GOLDEN_SCHEDULES = ("rounds", "refill", "tiny")
PARTITION_SCHEDULES = ("refill", "pipes2")

GOLDEN_CASES = ["soup", "killeroo_like", "materials", "instances", "specular", "substrate", "metal", "uber", "roughglass", "lights", "params",
                "envlight", "textured", "textured_lens", "sobol", "envmap", "bumpmap", "texcombine", "checker"]
EXTRA_CASES = ["lights_spatial_lazy", "emissive_mesh", "emissive_sphere", "instanced_soup", "gaussian", "one_sided_lights"]
CASES = GOLDEN_CASES + EXTRA_CASES
CASE_ENV = {"lights_spatial_lazy": {"PB2_LIGHTDIST_LAZY": "1"}}
KERNEL_CASES = ("killeroo_like", "instances", "specular", "soup")    # rendered with every trace-kernel variant too
PARTITION_CASES = ("params", "soup", "instances", "one_sided_lights")
# the chained trace kernel is selected for these (triangle / sphere / instanced scenes with two-child records, no alpha)
CHAIN_CASES = ("soup", "killeroo_like", "materials", "instances", "specular", "lights", "emissive_sphere", "one_sided_lights",
               "instanced_soup", "lights_spatial_lazy", "emissive_mesh")

# A one-sided emissive quad whose per-vertex normals point against its winding (it emits downwards, its winding says
# upwards) above a matte floor and a glossy box, and a one-sided emissive sphere, cut open at the top, that stands in
# the floor: it lights the floor around it and not the floor inside it.  A MIS ray that reaches either light counts only
# if the light's surface at the hit faces the ray.  The quad's side comes from its interpolated normals, so the chained
# light step must hand the stored barycentrics to lightAdvance (a sphere's surface is recomputed from the ray).
ONE_SIDED_LIGHTS = """
LookAt 0 -5 1.6  0 0 .3  0 0 1
Camera "perspective" "float fov" [45]
Film "image" "integer xresolution" [48] "integer yresolution" [32]
Sampler "halton" "integer pixelsamples" [8]
Integrator "path" "integer maxdepth" [5]
WorldBegin
AttributeBegin
  AreaLightSource "diffuse" "rgb L" [4 4 4]
  Shape "trianglemesh" "point P" [-1 -1 2.2  1 -1 2.2  1 1 2.2  -1 1 2.2] "integer indices" [0 1 2 0 2 3]
    "normal N" [0 0 -1  0 0 -1  0 0 -1  0 0 -1]
AttributeEnd
AttributeBegin
  Translate 1.3 .6 .2
  AreaLightSource "diffuse" "rgb L" [2 1.5 1]
  Shape "sphere" "float radius" [.7] "float zmax" [.35]
AttributeEnd
Material "matte" "rgb Kd" [.6 .6 .6]
Shape "trianglemesh" "point P" [-4 -4 0 4 -4 0 4 4 0 -4 4 0] "integer indices" [0 1 2 0 2 3]
Material "plastic" "rgb Kd" [.2 .3 .5] "rgb Ks" [.5 .5 .5] "float roughness" [.05]
Shape "trianglemesh" "point P" [-1.2 -.4 0 -.4 -.4 0 -.4 .4 0 -1.2 .4 0 -1.2 -.4 .8 -.4 -.4 .8 -.4 .4 .8 -1.2 .4 .8]
  "integer indices" [0 1 5 0 5 4 1 2 6 1 6 5 2 3 7 2 7 6 3 0 4 3 4 7 4 5 6 4 6 7]
WorldEnd
"""


def case_text(case):
    """The scene text of a case that is not a golden scene file or a synthetic generator."""
    from test_gpu_parity import emissive_mesh_scene
    if case == "lights_spatial_lazy":
        return gc.lights_text(SCENES, "spatial")
    if case == "emissive_mesh":
        return emissive_mesh_scene(40)          # 3200 lights: the spatial table is built on demand
    if case == "emissive_sphere":
        return gc.analytic_scene_text("emissive_sphere")
    if case == "gaussian":
        return gc.filter_scene_text(SCENES, "gaussian")
    if case == "one_sided_lights":
        return ONE_SIDED_LIGHTS
    raise KeyError(case)


def make_case(pb, case):
    from test_oracle import load_scene
    if case in GOLDEN_CASES:
        return load_scene(pb, case)
    if case == "instanced_soup":
        return pb.HostScene.instanced_soup(2000, grid=4, xres=64, yres=36, spp=4)
    return pb.HostScene.from_string(case_text(case))


def case_flags(pb, case):
    flags = [0, pb.PB2_FLAG_CHAIN]
    if case in KERNEL_CASES:
        flags += [pb.PB2_FLAG_WIDE4, pb.PB2_FLAG_LINEAR_NODES, pb.PB2_FLAG_PLAIN_TRACE, pb.PB2_FLAG_SMALL_STACK, pb.PB2_FLAG_LD128,
                  pb.PB2_FLAG_LEAF_TMA, pb.PB2_FLAG_POOL]
    return flags


# ---------------------------------------------------------------------------------------------------------------------
# The per-pixel model (host arithmetic only)
# ---------------------------------------------------------------------------------------------------------------------
def filter_table(film):
    """Film's 16 x 16 filter weight table as the library's host code builds it (computeFilterTable: Filter::Evaluate in
    float, in the same order, with libm's expf and sinf), or None for the box filter."""
    import pbrt_v3_b200 as pb
    if film.filter_type == pb.PB2_FILTER_BOX:
        return None
    libm = C.CDLL(ctypes.util.find_library("m"))
    libm.expf.restype, libm.expf.argtypes = C.c_float, [C.c_float]
    libm.sinf.restype, libm.sinf.argtypes = C.c_float, [C.c_float]
    f32 = np.float32
    expf = lambda v: f32(libm.expf(float(v)))
    sinf = lambda v: f32(libm.sinf(float(v)))
    rx, ry = f32(film.filter_radius[0]), f32(film.filter_radius[1])
    p0, p1 = f32(film.filter_param[0]), f32(film.filter_param[1])
    if film.filter_type == pb.PB2_FILTER_GAUSSIAN:           # gaussian.h:50-66
        alpha = p0
        exp_x, exp_y = expf(-alpha * rx * rx), expf(-alpha * ry * ry)
        g = lambda d, e: max(f32(0), f32(expf(-alpha * d * d) - e))
        evaluate = lambda x, y: g(x, exp_x) * g(y, exp_y)
    elif film.filter_type == pb.PB2_FILTER_MITCHELL:         # mitchell.h:53-63
        B, Cm = p0, p1

        def m1(v):
            v = abs(f32(2) * v)
            if v > f32(1):
                return ((-B - f32(6) * Cm) * v * v * v + (f32(6) * B + f32(30) * Cm) * v * v + (f32(-12) * B - f32(48) * Cm) * v
                        + (f32(8) * B + f32(24) * Cm)) * (f32(1) / f32(6))
            return ((f32(12) - f32(9) * B - f32(6) * Cm) * v * v * v + (f32(-18) + f32(12) * B + f32(6) * Cm) * v * v
                    + (f32(6) - f32(2) * B)) * (f32(1) / f32(6))
        inv_rx, inv_ry = f32(1) / rx, f32(1) / ry
        evaluate = lambda x, y: m1(x * inv_rx) * m1(y * inv_ry)
    elif film.filter_type == pb.PB2_FILTER_SINC:             # sinc.h:53-63
        tau, pi = p0, f32(3.14159265358979323846)

        def sinc(v):
            v = abs(v)
            if float(v) < 1e-5:                                  # a float against a double literal
                return f32(1)
            return sinf(pi * v) / (pi * v)

        def windowed(v, radius):
            v = abs(v)
            if v > radius:
                return f32(0)
            lanczos = sinc(v / tau)
            return sinc(v) * lanczos
        evaluate = lambda x, y: windowed(x, rx) * windowed(y, ry)
    elif film.filter_type == pb.PB2_FILTER_TRIANGLE:         # triangle.cpp:40-43
        evaluate = lambda x, y: max(f32(0), rx - abs(x)) * max(f32(0), ry - abs(y))
    else:
        raise NotImplementedError("filter type %d is not modelled" % film.filter_type)
    table = np.zeros(256, np.float32)
    for y in range(16):
        for x in range(16):
            table[y * 16 + x] = evaluate((f32(x) + f32(.5)) * rx / f32(16), (f32(y) + f32(.5)) * ry / f32(16))
    return table


def clamped_samples(film, li):
    """L as addSample deposits it: scaled down to maxSampleLuminance where its luminance is above it (float32)."""
    f32 = np.float32
    L = np.array(li, np.float32)
    lum = f32(0.212671) * L[:, 0] + f32(0.715160) * L[:, 1] + f32(0.072169) * L[:, 2]
    m = f32(film.max_sample_luminance)
    over = lum > m
    L[over] = L[over] * (m / lum[over])[:, None]
    return L


def deposits(film, pfilm):
    """FilmTile::AddSample's pixel range of every sample, clipped to the cropped bounds: yields (sample indices, pixel x,
    pixel y, filter-table index) once per offset inside the ranges (the table index is None for the box filter)."""
    f32 = np.float32
    x0, y0, x1, y1 = (int(v) for v in film.cropped_pixel_bounds)
    box = filter_table(film) is None
    rx, ry = f32(film.filter_radius[0]), f32(film.filter_radius[1])
    inv_rx, inv_ry = f32(1) / rx, f32(1) / ry
    pf = np.asarray(pfilm, np.float32)
    dx, dy = pf[:, 0] - f32(.5), pf[:, 1] - f32(.5)
    p0x, p0y = np.maximum(np.ceil(dx - rx).astype(np.int64), x0), np.maximum(np.ceil(dy - ry).astype(np.int64), y0)
    p1x, p1y = np.minimum(np.floor(dx + rx).astype(np.int64) + 1, x1), np.minimum(np.floor(dy + ry).astype(np.int64) + 1, y1)
    for oy in range(max(0, int((p1y - p0y).max(initial=0)))):
        for ox in range(max(0, int((p1x - p0x).max(initial=0)))):
            xx, yy = p0x + ox, p0y + oy
            sel = np.flatnonzero((xx < p1x) & (yy < p1y))
            xs, ys = xx[sel], yy[sel]
            tab = None
            if not box:
                fx = np.abs((xs.astype(np.float32) - dx[sel]) * inv_rx * f32(16))
                fy = np.abs((ys.astype(np.float32) - dy[sel]) * inv_ry * f32(16))
                tab = np.minimum(np.floor(fy).astype(np.int64), 15) * 16 + np.minimum(np.floor(fx).astype(np.int64), 15)
            yield sel, xs, ys, tab


def film_model(film, li, pfilm):
    """The film that depositing the samples (li, pfilm) must give: addSample's maxSampleLuminance clamp in float32, then
    FilmTile::AddSample's pixel range and filter-table look-up in float32 and the sum in float64.  Returns (rgbw, bound):
    rgbw (h, w, 4) float64, bound (h, w, 4) = k * 2^-24 * sum |L * w| per channel, k = deposits in the pixel."""
    x0, y0, x1, y1 = (int(v) for v in film.cropped_pixel_bounds)
    h, w = y1 - y0, x1 - x0
    L = clamped_samples(film, li)
    table = filter_table(film)
    total = np.zeros((h * w, 4), np.float64)
    absum = np.zeros((h * w, 4), np.float64)
    k = np.zeros(h * w, np.float64)
    for sel, xs, ys, tab in deposits(film, pfilm):
        wt = np.ones(len(xs), np.float32) if table is None else table[tab]
        contrib = np.concatenate([L[sel] * wt[:, None], wt[:, None]], 1).astype(np.float64)
        idx = (ys - y0) * w + (xs - x0)
        np.add.at(total, idx, contrib)
        np.add.at(absum, idx, np.abs(contrib))
        np.add.at(k, idx, 1)
    return total.reshape(h, w, 4), (k[:, None] * U * absum).reshape(h, w, 4)


def model_mismatch(film, model, bound, box):
    """Why `film` (float32 rgbw) is not the model, or None."""
    film = np.asarray(film, np.float64)
    if box and not np.array_equal(film[..., 3], model[..., 3]):
        bad = film[..., 3] != model[..., 3]
        return "weight channel differs in %d pixels (first %s)" % (bad.sum(), np.argwhere(bad)[0].tolist())
    err = np.abs(film - model)
    bad = err > bound
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        return "%d values outside k * 2^-24 * sum|L w| (first %s: film %.9g model %.9g bound %.3g)" % (bad.sum(), list(i), film[i], model[i], bound[i])
    return None


# ---------------------------------------------------------------------------------------------------------------------
# The worker: one process per schedule (the schedule knobs are read once per process)
# ---------------------------------------------------------------------------------------------------------------------
def render_schedule(schedule, out):
    import pbrt_v3_b200 as pb
    from pbrt_v3_b200 import multigpu
    pipes = SCHEDULES[schedule][1]
    res = {}
    for case in CASES:
        env = CASE_ENV.get(case, {})
        os.environ.update(env)
        try:
            hs = make_case(pb, case)
            base = hs.params_copy()
            spp = base.samples_per_pixel
            if pipes:
                per_spp = len(multigpu.work_items(hs.film, hs.params_copy(samples_per_pixel=1)))
                spp = math.ceil(PIPE_ITEMS / per_spp)
                if base.sampler == pb.PB2_SAMPLER_SOBOL:
                    spp = 1 << (spp - 1).bit_length()
            flags = case_flags(pb, case)
            films, images, stats = [], [], []
            for f in flags:
                film, st = hs.render_rgbw(hs.params_copy(flags=f, samples_per_pixel=spp))
                films.append(film)
                images.append(hs.resolve(film))
                stats.append([st.camera_rays, st.regular_rays, st.shadow_rays, st.kernel_launches])
            params = hs.params_copy(samples_per_pixel=spp)
            items = multigpu.work_items(hs.film, params)
            li, pfilm = hs.li_samples(items[:, :2], items[:, 2].astype(np.int64), params)
            model, bound = film_model(hs.film.contents, li, pfilm)
            res.update({case + ":flags": np.array(flags), case + ":film": np.array(films), case + ":image": np.array(images),
                        case + ":stats": np.array(stats, np.int64), case + ":items": np.int64(len(items)), case + ":spp": np.int64(spp),
                        case + ":model": model, case + ":bound": bound,
                        case + ":box": np.bool_(hs.film.contents.filter_type == pb.PB2_FILTER_BOX)})
            if case in PARTITION_CASES and schedule in PARTITION_SCHEDULES:
                parts = []
                for f in flags[:2]:
                    parts.append(sum(hs.render_rgbw(hs.params_copy(flags=f, samples_per_pixel=spp, tile_rank=r, tile_count=3))[0].astype(np.float64)
                                     for r in range(3)))
                res[case + ":parts"] = np.array(parts)
        finally:
            for key in env:
                os.environ.pop(key, None)
    np.savez(out, **res)


WORKER = r'''
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_gpu_wavefront_schedules as t
t.render_schedule(sys.argv[3], sys.argv[4])
print("schedule", sys.argv[3], "ok")
'''


@pytest.fixture(scope="module")
def schedule(tmp_path_factory):
    """schedule(name) -> {case: {field: array}} of that schedule's worker (run once per module, on first use)."""
    d = tmp_path_factory.mktemp("schedules")
    script = d / "worker.py"
    script.write_text(WORKER)
    done = {}

    def get(name):
        if name not in done:
            out = d / (name + ".npz")
            env = dict(os.environ)
            for knob in ("PB2_POOL", "PB2_PIPES", "PB2_FINISH", "PB2_SYNC_EVERY", "PB2_LIGHTDIST_LAZY"):
                env.pop(knob, None)
            env.update(SCHEDULES[name][0])
            res = subprocess.run([sys.executable, str(script), ROOT, TESTS, name, str(out)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                 text=True, timeout=1200, cwd=ROOT, env=env)
            if res.returncode != 0:
                done[name] = "worker for schedule %s failed:\n%s" % (name, res.stdout[-4000:])
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


# ---------------------------------------------------------------------------------------------------------------------
# Check 1 (and 4): every film against its per-sample model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("name", list(SCHEDULES))
def test_film_equals_the_sum_of_its_samples(schedule, name, case):
    r = schedule(name)[case]
    for f, film in zip(r["flags"], r["film"]):
        why = model_mismatch(film, r["model"], r["bound"], bool(r["box"]))
        assert why is None, "flags %d: %s" % (f, why)


# ---------------------------------------------------------------------------------------------------------------------
# Check 2: ray counters
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_ray_counters_do_not_depend_on_the_schedule(schedule, case):
    for pipes in (False, True):
        seen = {}
        for name, (_, p) in SCHEDULES.items():
            if p != pipes:
                continue
            r = schedule(name)[case]
            for f, st in zip(r["flags"], r["stats"]):
                assert st[0] == r["items"], (name, int(f), "camera rays", int(st[0]), int(r["items"]))
                seen[(name, int(f))] = (int(st[1]), int(st[2]))
        assert len(set(seen.values())) == 1, seen


# ---------------------------------------------------------------------------------------------------------------------
# Check 3: the golden scenes at depth, against the reference's image and ray counts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", GOLDEN_CASES)
@pytest.mark.parametrize("name", GOLDEN_SCHEDULES)
def test_rounds_at_depth_match_the_reference(schedule, name, case):
    from test_gpu_parity import image_metrics
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    r = schedule(name)[case]
    cam, reg, sh = (int(x) for x in g["rays"])
    for f, img, st in zip(r["flags"][:2], r["image"][:2], r["stats"][:2]):
        frac, mean_rel = image_metrics(img, g["image"])
        assert frac >= 0.999 and mean_rel <= 1e-4, (int(f), frac, mean_rel)
        assert abs(float(img.mean()) - float(g["image"].mean())) <= 1e-4 * float(g["image"].mean()), int(f)
        assert st[0] == cam, int(f)
        assert abs(int(st[1]) - reg) <= max(2, reg // 1000) and abs(int(st[2]) - sh) <= max(2, sh // 1000), (int(f), st.tolist(), reg, sh)


# ---------------------------------------------------------------------------------------------------------------------
# Check 4: the chained light step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CHAIN_CASES)
def test_chain_takes_fewer_launches_when_the_rounds_run(schedule, case):
    import pbrt_v3_b200 as pb
    r = schedule("rounds")[case]
    launches = {int(f): int(st[3]) for f, st in zip(r["flags"], r["stats"])}
    assert launches[pb.PB2_FLAG_CHAIN] < launches[0], launches


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCHEDULES))
def test_emissive_sphere_furnace_in_every_schedule(schedule, name):
    """The reference's analytic scene (camera inside a reverse-oriented emissive sphere): radiance 1 within 0.02 with
    every flag.  A chained MIS ray that reaches the sphere is counted only if the sphere's inner side faces it."""
    r = schedule(name)["emissive_sphere"]
    means = {int(f): float(img.mean()) for f, img in zip(r["flags"], r["image"])}
    assert all(abs(m - gc.ANALYTIC_EXPECTED) <= gc.ANALYTIC_DELTA for m in means.values()), means


# ---------------------------------------------------------------------------------------------------------------------
# Check 5: tile partitions
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", PARTITION_CASES)
@pytest.mark.parametrize("name", PARTITION_SCHEDULES)
def test_tile_partition_sums_to_the_model(schedule, name, case):
    """The films of tile_count = 3 (the params scene's pixel bounds make a lane draw several items) sum to the full
    film's model: each rank film is within its own bound, so their float64 sum is within the full film's."""
    r = schedule(name)[case]
    for f, parts in zip(r["flags"][:2], r["parts"]):
        why = model_mismatch(parts, r["model"], r["bound"], True)
        assert why is None, "flags %d: %s" % (f, why)


# ---------------------------------------------------------------------------------------------------------------------
# The model itself, on the CPU: the oracle port's samples through it give the port's own render
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["soup"] + list(gc.FILTER_CASES))
def test_model_reproduces_the_port_render(port, case):
    """Every reconstruction filter of golden_cases.FILTER_CASES ("gaussian" is also this file's gaussian case)."""
    import pbrt_v3_b200 as pb
    from pbrt_v3_b200 import multigpu
    hs = make_case(pb, case) if case in CASES else pb.HostScene.from_string(gc.filter_scene_text(SCENES, case))
    sc = port.scene(hs)
    items = multigpu.work_items(hs.film, hs.params)
    li, pfilm = sc.li_samples(items[:, :2], items[:, 2].astype(np.int64))
    model, bound = film_model(hs.film.contents, li, pfilm)
    want, _, _ = sc.render(n_threads=1)
    got = hs.resolve(model.astype(np.float32))
    rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-3)
    table = filter_table(hs.film.contents)
    if table is not None and (table < 0).any():
        # negative lobes (mitchell, sinc): where they nearly cancel, the port's own float32 sums are off by up to their
        # bounds relative to the small sums that remain.  Such values may exceed 1e-5 by that much, and only a few may
        # (1 of the 13 440 values of the four cases does, the sinc case's).
        part = lambda b, m: b / np.maximum(np.abs(m), 1e-30)
        allowance = (part(bound[..., :3], model[..., :3]) + part(bound[..., 3:], model[..., 3:])) * np.abs(want) / np.maximum(np.abs(want), 1e-3)
        loose = rel > 1e-5
        assert loose.sum() <= rel.size // 1000, int(loose.sum())
        rel = np.where(loose, rel - allowance, rel)
    assert rel.max() <= 1e-5, float(rel.max())
    assert (model[..., 3] > 0).all() and (bound >= 0).all()
