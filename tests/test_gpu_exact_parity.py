"""The CUDA path against the compiled reference run with the device's transcendentals: BIT FOR BIT.

The device computes its six transcendentals as (float)f((double)x) (pb2_math.cuh: psinf, pcosf, psincosf, plogf, patan2f,
pacosf); the reference calls glibc's sinf / cosf / sincosf / logf / atan2f / acosf.  That is the one source of difference
the tolerances of test_gpu_parity.py allow for.  In device-math mode the reference evaluates those six functions the
device's way (oracle/ref_devmath.cpp), so what is left is CUDA's double-precision routines against glibc's, a couple of
double ulps that reach a float result only when the double value lies next to a float rounding boundary.  So this file
demands equality with what the reference computes in that mode, recorded by tests/make_golden.py (record_reference below)
into tests/golden/exact_parity.npz as 32-bit digests of every bit (the values themselves would make a fixture of tens of MB):

  * every work item of every frame: pb2_li_samples' sample number, L and pFilm, one digest per pixel;
  * golden scenes: pb2_intersect's every field (spheres' n, ns, dpdu, uv included; not the barycentrics, which the
    reference does not expose), pb2_intersect_p, the light distributions and the textured scene's MIPMap look-ups;
  * films of the benchmarked kernels, with the shipped settings and with every bounce through the round kernels
    (PB2_FINISH=0), against the float64 film model of the samples (test_gpu_wavefront_schedules.film_model), which the first
    check makes the reference's: weight channel of box-filtered films exact, every RGB value within k * 2^-24 * sum |L w|;
  * camera, regular and shadow ray counters equal to the reference's SamplerIntegrator::Render;
  * the full-size benchmark scene on 32 x 32 blocks of five crop windows.

A pixel whose samples differ because CUDA's double routine rounds a call differently from glibc's is listed in EXCEPTIONS
below, keyed by (scene, pixel x, pixel y), with the sample, the function and the argument a host replay exhibits.  Any
other mismatch is a bug of the kernels or of the harness.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import golden_cases as gc
from conftest import GOLDEN, ROOT, SCENES
from test_gpu_parity import SCENE_CASES, emissive_mesh_scene
from test_gpu_wavefront_schedules import ONE_SIDED_LIGHTS, film_model, model_mismatch
from test_oracle import load_scene

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))

# (scene, pixel x, pixel y) -> "sample n: function(argument)": pixels whose samples differ because CUDA's double routine and
# glibc's round the named call differently.  None are known.
EXCEPTIONS = {}

EXTRA_CASES = ["analytic_" + c for c in sorted(gc.ANALYTIC_SCENES)] + ["filter_" + c for c in sorted(gc.FILTER_CASES)] + \
              ["soup20k", "instanced_soup", "emissive_mesh", "lights_spatial", "lights_uniform", "one_sided_lights"]
CASES = SCENE_CASES + EXTRA_CASES
MODELLED_FILTERS = ("box", "gaussian")    # film_model's filter tables


def make_case(pb, case):
    if case in SCENE_CASES:
        return load_scene(pb, case)
    if case.startswith("analytic_"):
        return pb.HostScene.from_string(gc.analytic_scene_text(case[len("analytic_"):]))
    if case.startswith("filter_"):
        return pb.HostScene.from_string(gc.filter_scene_text(SCENES, case[len("filter_"):]))
    if case == "soup20k":
        return pb.HostScene.soup(20000, xres=96, yres=54, spp=8)
    if case == "instanced_soup":
        return pb.HostScene.instanced_soup(2000, grid=4, xres=64, yres=36, spp=4)
    if case == "emissive_mesh":
        return pb.HostScene.from_string(emissive_mesh_scene(40))
    if case in ("lights_spatial", "lights_uniform"):
        return pb.HostScene.from_string(gc.lights_text(SCENES, case.split("_")[1]))
    if case == "one_sided_lights":
        return pb.HostScene.from_string(ONE_SIDED_LIGHTS)
    raise KeyError(case)


FIXTURE = os.path.join(GOLDEN, "exact_parity.npz")
XRES, YRES, TRIS, SPP = 1920, 1080, 1000000, 64
CROPS = [(256, 128), (1408, 208), (832, 496), (320, 880), (1600, 864)]   # test_gpu_fullsize.py's 128 x 72 windows
BLOCK = 32


def counters(st):
    return int(st.camera_rays), int(st.regular_rays), int(st.shadow_rays)


def frame_items(hs, params=None):
    from pbrt_v3_b200 import multigpu
    items = multigpu.work_items(hs.film, params if params is not None else hs.params)
    return items, items[:, :2], items[:, 2].astype(np.int64)


def block_params(hs, x0, y0):
    """The 32 x 32 block inside the crop window at (x0, y0), and the window itself, as pixel bounds."""
    block, crop = hs.params_copy(), hs.params_copy()
    bx, by = x0 + 48, y0 + 20
    block.pixel_bounds[0], block.pixel_bounds[1], block.pixel_bounds[2], block.pixel_bounds[3] = bx, by, bx + BLOCK, by + BLOCK
    crop.pixel_bounds[0], crop.pixel_bounds[1], crop.pixel_bounds[2], crop.pixel_bounds[3] = x0, y0, x0 + 128, y0 + 72
    return block, crop


def hit_rows(hits):
    """Hit records without the barycentrics (the reference's SurfaceInteraction has none)."""
    h = hits.copy()
    h["b"] = 0
    return h


def record_reference(ref, path):
    """What the compiled reference computes in device-math mode for every check of this file (run by tests/make_golden.py):
    per-pixel digests of every work item's L and pFilm, ray counters, hit / light-distribution / look-up digests."""
    import pbrt_v3_b200 as pb
    out = {}
    with ref.device_math():
        for case in CASES:
            hs = make_case(pb, case)
            _, pix, sn = frame_items(hs)
            sc = ref.scene(hs)
            li, pfilm = sc.li_samples(pix, sn)
            out[case + ":pixels"], out[case + ":digest"] = gc.pixel_digests(np.c_[pix, sn], li, pfilm)
            out[case + ":rays"] = np.array(counters(sc.render(n_threads=0)[2]), np.int64)
            if case in SCENE_CASES:
                nodes = hs.nodes()
                out[case + ":hits"] = gc.row_digest(hit_rows(sc.intersect(gc.rays_for(pb, nodes, 1500, 11))))
                out[case + ":occluded"] = sc.intersect_p(gc.rays_for(pb, nodes, 1500, 12, shadow=True))
                out[case + ":light_distribution"] = gc.row_digest(sc.light_distribution(gc.points_for(nodes, 400, 15)))
            del sc
        for i, t in enumerate(make_case(pb, "textured").textures()):
            st, dst = gc.texture_lookup_inputs(3000, 100 + i)
            out["lookup_%d" % i] = gc.row_digest(ref.texture_lookup(t, st, dst))
        hs = pb.HostScene.soup(TRIS, xres=XRES, yres=YRES, spp=SPP, maxdepth=8)
        sc = ref.scene(hs)
        for x0, y0 in CROPS:
            block, _ = block_params(hs, x0, y0)
            _, pix, sn = frame_items(hs, block)
            li, pfilm = sc.li_samples(pix, sn, block)
            key = "fullsize_%d_%d" % (x0, y0)
            out[key + ":pixels"], out[key + ":digest"] = gc.pixel_digests(np.c_[pix, sn], li, pfilm)
            out[key + ":rays"] = np.array(counters(sc.render(n_threads=0, params=block)[2]), np.int64)
    np.savez_compressed(path, **out)


# ---------------------------------------------------------------------------------------------------------------------
# The round kernels on every bounce: a worker process (PB2_FINISH is read once per process)
# ---------------------------------------------------------------------------------------------------------------------
def render_rounds(out):
    import pbrt_v3_b200 as pb
    res = {}
    for case in CASES:
        hs = make_case(pb, case)
        film, st = hs.render_rgbw()
        res[case + ":film"] = film
        res[case + ":stats"] = np.array(counters(st), np.int64)
    np.savez(out, **res)


WORKER = r'''
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_gpu_exact_parity as t
t.render_rounds(sys.argv[3])
print("rounds ok")
'''


@pytest.fixture(scope="module")
def rounds(tmp_path_factory):
    d = tmp_path_factory.mktemp("exact_rounds")
    script, out = d / "worker.py", d / "rounds.npz"
    script.write_text(WORKER)
    env = dict(os.environ)
    for knob in ("PB2_POOL", "PB2_PIPES", "PB2_SYNC_EVERY", "PB2_LIGHTDIST_LAZY"):
        env.pop(knob, None)
    env["PB2_FINISH"] = "0"
    res = subprocess.run([sys.executable, str(script), ROOT, TESTS, str(out)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         timeout=1200, cwd=ROOT, env=env)
    if res.returncode != 0:
        pytest.fail("worker with PB2_FINISH=0 failed:\n" + res.stdout[-4000:])
    z = np.load(out)
    return {key: z[key] for key in z.files}


@pytest.fixture(scope="module")
def want():
    """The reference's results in device-math mode, recorded by tests/make_golden.py (record_reference above)."""
    if not os.path.exists(FIXTURE):
        pytest.fail("%s is missing: tests/make_golden.py records it from the compiled reference" % FIXTURE)
    z = np.load(FIXTURE)
    return {k: z[k] for k in z.files}


def check_samples(want, key, case, items, li, pfilm):
    """Every work item's L and pFilm against the reference's, pixel by pixel; EXCEPTIONS removed."""
    pixels, digest = gc.pixel_digests(items, li, pfilm)
    assert np.array_equal(pixels, want[key + ":pixels"]), "%s: the work items cover other pixels than the reference's" % key
    bad = [tuple(int(v) for v in p) for p in pixels[digest != want[key + ":digest"]]]
    bad = [p for p in bad if (case,) + p not in EXCEPTIONS]
    assert not bad, "%s: samples of %d of %d pixels differ from the reference's (first pixels %s)" % (key, len(bad), len(pixels), bad[:10])


# ---------------------------------------------------------------------------------------------------------------------
# Every work item, the films and the ray counters
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_every_sample_film_and_counter_equals_the_reference(pb, want, rounds, case):
    hs = make_case(pb, case)
    items, pix, sn = frame_items(hs)
    li, pfilm = hs.li_samples(pix, sn)
    check_samples(want, case, case, items, li, pfilm)
    ref_rays = tuple(int(v) for v in want[case + ":rays"])
    shipped, st = hs.render_rgbw()
    assert counters(st) == ref_rays, "shipped settings: ray counters"
    assert tuple(int(v) for v in rounds[case + ":stats"]) == ref_rays, "PB2_FINISH=0: ray counters"
    film = hs.film.contents
    kind = {pb.PB2_FILTER_BOX: "box", pb.PB2_FILTER_GAUSSIAN: "gaussian"}.get(film.filter_type)
    if kind not in MODELLED_FILTERS:
        return    # mitchell / sinc / triangle: the samples and the counters above are what this file checks
    # the samples equal the reference's (above), so this is the model of the reference's samples
    model, bound = film_model(film, li, pfilm)
    for name, f in (("shipped", shipped), ("PB2_FINISH=0", rounds[case + ":film"])):
        why = model_mismatch(f, model, bound, kind == "box")
        assert why is None, "%s: %s" % (name, why)


# ---------------------------------------------------------------------------------------------------------------------
# Hits, any-hits, light distributions, texture look-ups
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SCENE_CASES)
def test_hits_and_light_distributions_are_the_reference_bits(pb, want, name):
    hs = load_scene(pb, name)
    nodes = hs.nodes()
    rays = gc.rays_for(pb, nodes, 1500, 11)
    bad = np.flatnonzero(gc.row_digest(hit_rows(hs.intersect(rays))) != want[name + ":hits"])
    assert len(bad) == 0, "%d of %d hit records differ in some field (first rays %s)" % (len(bad), len(rays), bad[:10].tolist())
    assert np.array_equal(hs.intersect_p(gc.rays_for(pb, nodes, 1500, 12, shadow=True)), want[name + ":occluded"])
    bad = np.flatnonzero(gc.row_digest(hs.light_distribution(gc.points_for(nodes, 400, 15))) != want[name + ":light_distribution"])
    assert len(bad) == 0, "light distributions differ at %d points" % len(bad)


def test_texture_lookups_are_the_reference_bits(pb, want):
    textures = load_scene(pb, "textured").textures()
    assert len(textures) == 10
    for i, t in enumerate(textures):
        st, dst = gc.texture_lookup_inputs(3000, 100 + i)
        bad = gc.row_digest(pb.texture_lookup(t, st, dst)) != want["lookup_%d" % i]
        assert not bad.any(), "texture %d: %d of %d look-ups differ (first st %s dst %s)" % (i, bad.sum(), len(bad), st[bad][0], dst[bad][0])


# ---------------------------------------------------------------------------------------------------------------------
# The benchmark scene at full size: 32 x 32 blocks inside five crop windows
# ---------------------------------------------------------------------------------------------------------------------
def test_full_size_blocks_equal_the_reference(pb, want):
    hs = pb.HostScene.soup(TRIS, xres=XRES, yres=YRES, spp=SPP, maxdepth=8)
    film = hs.film.contents
    for x0, y0 in CROPS:
        block, crop = block_params(hs, x0, y0)
        bx, by = block.pixel_bounds[0], block.pixel_bounds[1]
        items, pix, sn = frame_items(hs, block)
        assert len(items) == BLOCK * BLOCK * SPP
        li, pfilm = hs.li_samples(pix, sn, block)
        key = "fullsize_%d_%d" % (x0, y0)
        check_samples(want, key, "fullsize", items, li, pfilm)
        model, bound = film_model(film, li, pfilm)
        # the block rendered alone: every deposit of the film comes from the block's samples
        rgbw, st = hs.render_rgbw(block)
        assert counters(st) == tuple(int(v) for v in want[key + ":rays"]), (bx, by)
        why = model_mismatch(rgbw, model, bound, True)
        assert why is None, "block at %s rendered alone: %s" % ((bx, by), why)
        # the 128 x 72 window: pixels one inside the block's edge receive samples of block pixels only
        rgbw, st = hs.render_rgbw(crop)
        assert st.camera_rays == 128 * 72 * SPP
        inner = (slice(by + 1, by + BLOCK - 1), slice(bx + 1, bx + BLOCK - 1))
        why = model_mismatch(rgbw[inner], model[inner], bound[inner], True)
        assert why is None, "window at %s: %s" % ((x0, y0), why)
