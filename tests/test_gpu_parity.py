"""CUDA path (through the C ABI) against the CPU checker and the golden vectors of the reference.

Tolerances (also stated in DESIGN.md):
  * Scene::Intersect / IntersectP, Halton samples, light-sampling distributions, CameraSample::pFilm:
    BIT-EXACT (integer / IEEE +-*/ sqrt arithmetic only, compiled with -fmad=false).
  * PathIntegrator::Li per sample: |dL| <= 1e-4 * max(1, |L|) for >= 99.9 % of the samples (transcendentals are
    evaluated in double and rounded, which almost always equals glibc's float result; a one-ulp difference in a
    sampled direction can flip an edge decision or move a sharp microfacet lobe).
  * images: >= 99.9 % of the pixels within 1 % relative, mean relative error <= 1e-4, image mean within 1e-4.
  * Scene::Intersect / IntersectP call counters: equal to the reference's within 0.1 % (edge flips).
These pin the device to the glibc goldens and to the port.  The transcendentals are the only reason for them:
test_gpu_exact_parity.py runs the compiled reference with the device's definitions of sinf / cosf / sincosf / logf / atan2f /
acosf and asserts per-sample Li, every hit field, look-ups, light distributions and ray counters EQUAL, and films within the
float32 summation bound of the reference's samples.  Measured effect (test_ref_device_math.py): the device's definitions
change Li in 1032 of the 57 000 golden samples (1 to 445 of 3000 per scene, most on the environment-lit scenes).
"""
import ctypes as C
import os

import numpy as np
import pytest

import golden_cases as gc
from conftest import GOLDEN, SCENES
from test_oracle import load_scene, same_bvh, tessellated_sphere_scene

pytestmark = pytest.mark.gpu

SCENE_CASES = ["soup", "killeroo_like", "materials", "instances", "specular", "substrate", "metal", "uber", "roughglass", "lights", "params",
               "envlight", "textured", "textured_lens", "sobol", "envmap", "bumpmap", "texcombine", "checker"]


def li_ok(got, want):
    err = np.abs(got - want).max(axis=1) / np.maximum(1, np.abs(want).max(axis=1))
    return float((err <= 1e-4).mean())


def image_metrics(got, want):
    rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-3)
    return float((rel.max(axis=2) <= 0.01).mean()), float(rel.mean())


@pytest.mark.parametrize("case", sorted(gc.ANALYTIC_SCENES))
def test_reference_analytic_scenes_on_gpu(pb, checker, case):
    """The reference's own end-to-end tests of the path (src/tests/analytic_scenes.cpp, Path / perspective / Halton 256):
    the furnace scenes must average to radiance 1 within 0.02 - and match the CPU checker like every other scene."""
    hs = pb.HostScene.from_string(gc.analytic_scene_text(case))
    img, st = hs.render()
    assert abs(float(img.mean()) - gc.ANALYTIC_EXPECTED) <= gc.ANALYTIC_DELTA, float(img.mean())
    ref_img, _, ref_st = checker.scene(hs).render(n_threads=0)
    frac, mean_rel = image_metrics(img, ref_img)
    assert frac >= 0.99 and mean_rel <= 1e-4, (frac, mean_rel)
    assert st.camera_rays == ref_st.camera_rays == 25600


@pytest.mark.parametrize("case", sorted(gc.FILTER_CASES))
def test_gpu_filters_match_reference_golden(pb, case):
    """Film::AddSample through the filter weight table on the device against the reference's image.  The device adds
    the weighted samples to a pixel in a different order than the CPU's tile merges, so this is a tolerance test: 1 %
    per pixel for 99.9 % of the pixels, 1e-4 on the mean relative error (the same bar as the box-filter images)."""
    g = np.load(os.path.join(GOLDEN, "filters.npz"))
    hs = pb.HostScene.from_string(gc.filter_scene_text(SCENES, case))
    img, st = hs.render()
    want = g["image_" + case]
    assert img.shape == want.shape
    frac, mean_rel = image_metrics(img, want)
    assert frac >= 0.999 and mean_rel <= 1e-4, (case, frac, mean_rel)
    cam, reg, sh = (int(x) for x in g["rays_" + case])
    assert st.camera_rays == cam
    assert abs(int(st.regular_rays) - reg) <= max(2, reg // 1000) and abs(int(st.shadow_rays) - sh) <= max(2, sh // 1000)


def test_filter_type_outside_the_enum_is_refused(pb):
    hs = pb.HostScene.from_string(gc.filter_scene_text(SCENES, "gaussian"))
    dev = hs.device_scene()
    film = pb.FilmDesc.from_buffer_copy(hs.film.contents)
    film.filter_type = 9
    h, w = hs.film_shape()
    out = np.zeros((h, w, 4), np.float32)
    st = pb.Stats()
    rc = hs.L.pb2_render_path(dev, hs.camera, C.byref(film), hs.params, pb.ptr(out), C.byref(st))
    assert rc == pb.PB2_ERR_INVALID


@pytest.mark.parametrize("name", SCENE_CASES)
def test_gpu_matches_reference_golden(pb, name):
    check_scene_against_golden(pb, name)


def check_scene_against_golden(pb, name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    hs = load_scene(pb, name)
    nodes = hs.nodes()
    xres, yres = hs.film.contents.full_resolution[0], hs.film.contents.full_resolution[1]
    spp = hs.params.contents.samples_per_pixel
    hits = hs.intersect(gc.rays_for(pb, nodes, 1500, 11))
    gh = g["hits"]
    assert np.array_equal(hits["prim"], gh["prim"])
    d = hs.desc.contents
    prim_type = np.ctypeslib.as_array(d.prim_type, shape=(d.n_prims,))
    on_sphere = (hits["prim"] >= 0) & (prim_type[np.maximum(hits["prim"], 0)] == pb.PB2_PRIM_SPHERE)
    for f in ("t", "p", "p_error", "n", "ns", "dpdu", "uv"):
        # triangles: everything is +-*/sqrt -> bit-identical.  Spheres: t, p, pError likewise; the normal / dpdu / uv
        # go through acos, sin, atan2 (sphere.cpp:107-117), where glibc and the device may differ in the last bit.
        exact = ~on_sphere if f in ("n", "ns", "dpdu", "uv") else np.ones(len(hits), bool)
        assert np.array_equal(gc.bits(hits[f][exact]), gc.bits(gh[f][exact])), "hit field %s must be bit-identical to the reference" % f
        assert np.allclose(hits[f][~exact], gh[f][~exact], rtol=2e-6, atol=1e-6), f
    assert np.array_equal(hs.intersect_p(gc.rays_for(pb, nodes, 1500, 12, shadow=True)), g["occluded"])
    hpix, hsn, hdim = gc.sample_ids(xres, yres, spp, 4000, 14, max_dim=200)
    assert np.array_equal(gc.bits(hs.halton(hpix, hsn, hdim)), gc.bits(g["halton"]))
    assert np.array_equal(gc.bits(hs.light_distribution(gc.points_for(nodes, 400, 15))), gc.bits(g["light_distribution"]))
    pix, sn = gc.sample_ids(xres, yres, spp, 3000, 13)
    li, pfilm = hs.li_samples(pix, sn)
    assert np.array_equal(gc.bits(pfilm), gc.bits(g["pfilm"]))
    assert li_ok(li, g["li"]) >= 0.999
    img, st = hs.render()
    frac, mean_rel = image_metrics(img, g["image"])
    assert frac >= 0.999 and mean_rel <= 1e-4, (frac, mean_rel)
    assert abs(float(img.mean()) - float(g["image"].mean())) <= 1e-4 * float(g["image"].mean())
    cam, reg, sh = (int(x) for x in g["rays"])
    assert st.camera_rays == cam
    assert abs(int(st.regular_rays) - reg) <= max(2, reg // 1000) and abs(int(st.shadow_rays) - sh) <= max(2, sh // 1000)
    assert st.kernel_launches > 0


def test_gpu_matches_checker_on_a_larger_scene(pb, checker):
    """20 000 random triangles at 96x54x8: sizes the CPU checker finishes in seconds."""
    hs = pb.HostScene.soup(20000, xres=96, yres=54, spp=8)
    sc = checker.scene(hs)
    nodes = hs.nodes()
    rays = gc.rays_for(pb, nodes, 20000, 21)
    assert hs.intersect(rays).tobytes() == _without_b(sc.intersect(rays), hs.intersect(rays))
    srays = gc.rays_for(pb, nodes, 20000, 22, shadow=True)
    assert np.array_equal(hs.intersect_p(srays), sc.intersect_p(srays))
    pix, sn = gc.sample_ids(96, 54, 8, 20000, 23)
    li, _ = hs.li_samples(pix, sn)
    ref_li, _ = sc.li_samples(pix, sn)
    assert li_ok(li, ref_li) >= 0.999
    img, st = hs.render()
    ref_img, _, ref_st = sc.render(n_threads=0)
    frac, mean_rel = image_metrics(img, ref_img)
    assert frac >= 0.999 and mean_rel <= 1e-4
    assert st.camera_rays == ref_st.camera_rays == 96 * 54 * 8
    assert abs(int(st.regular_rays) - int(ref_st.regular_rays)) <= ref_st.regular_rays // 1000 + 2


@pytest.mark.parametrize("strategy", ["spatial", "uniform"])
def test_delta_lights_under_other_light_sampling_strategies(pb, checker, strategy):
    """The golden case `lights` uses "power"; the spatial distribution calls every light's Sample_Li from voxel sample
    points (lightdistrib.cpp:232-300) and must come out bit-identical, delta lights included."""
    text = open(os.path.join(SCENES, "lights.pbrt")).read().replace('"string lightsamplestrategy" "power"', '"string lightsamplestrategy" "%s"' % strategy)
    hs = pb.HostScene.from_string(text)
    sc = checker.scene(hs)
    pts = gc.points_for(hs.nodes(), 400, 15)
    assert np.array_equal(gc.bits(hs.light_distribution(pts)), gc.bits(sc.light_distribution(pts)))
    pix, sn = gc.sample_ids(64, 48, 8, 3000, 13)
    li, pfilm = hs.li_samples(pix, sn)
    ref_li, ref_pfilm = sc.li_samples(pix, sn)
    assert np.array_equal(gc.bits(pfilm), gc.bits(ref_pfilm)) and li_ok(li, ref_li) >= 0.999
    img, st = hs.render()
    ref_img, _, ref_st = sc.render(n_threads=0)
    frac, mean_rel = image_metrics(img, ref_img)
    assert frac >= 0.999 and mean_rel <= 1e-4
    assert abs(int(st.shadow_rays) - int(ref_st.shadow_rays)) <= ref_st.shadow_rays // 1000 + 2


@pytest.mark.parametrize("name,maxprims", [("killeroo_like", 4), ("killeroo_like", 1), ("killeroo_like", 16), ("random20k", 4)])
def test_device_hlbvh_build_equals_reference(pb, name, maxprims, monkeypatch):
    """pb2_hlbvh_build: Morton codes, the sort, the treelets, the SAH tree over the treelet roots and the depth-first layout,
    all by CUDA kernels, give the reference's LinearBVHNode array and primitive order (the fixtures tests/test_host.py checks
    the host build against) - and so does pb2_hlbvh_treelets with the upper tree and the flatten on the host."""
    g = np.load(os.path.join(GOLDEN, "hlbvh.npz"))
    text = gc.random_mesh_scene_text(20000, 5) if name == "random20k" else open(os.path.join(SCENES, name + ".pbrt")).read()
    for upper in ("device", "host"):
        monkeypatch.setenv("PB2_DEVICE_BVH_UPPER", upper)
        hs = pb.HostScene.from_string(gc.with_accelerator(text, "hlbvh", maxprims, device_build=True))
        assert same_bvh(hs.nodes(), g["nodes_%s_%d" % (name, maxprims)]), upper
        assert np.array_equal(hs.bvh_prims(0), g["prims_%s_%d" % (name, maxprims)]), upper


def test_device_hlbvh_build_equals_host_build_on_a_larger_mesh(pb):
    text = gc.random_mesh_scene_text(200000, 9)
    hs = pb.HostScene.from_string(gc.with_accelerator(text, "hlbvh", 4))
    nodes, prims = hs.nodes().copy(), hs.bvh_prims(0).copy()
    hs = pb.HostScene.from_string(gc.with_accelerator(text, "hlbvh", 4, device_build=True))
    assert len(nodes) > 100000 and same_bvh(hs.nodes(), nodes) and np.array_equal(hs.bvh_prims(0), prims)
    rays = gc.rays_for(pb, nodes, 2000, 3)
    hits = hs.intersect(rays)
    assert (hits["prim"] >= 0).sum() > 100


def test_hlbvh_tree_traces_and_renders_like_the_sah_tree(pb):
    """A different BVH over the same primitives changes the traversal, not the answers: closest hits and the image of
    the golden case killeroo_like (recorded with the default SAH tree) must come out of the HLBVH tree as well."""
    g = np.load(os.path.join(GOLDEN, "killeroo_like.npz"))
    rays = gc.rays_for(pb, load_scene(pb, "killeroo_like").nodes(), 1500, 11)    # the rays the golden hits were recorded for
    hs = pb.HostScene.from_string(gc.with_accelerator(open(os.path.join(SCENES, "killeroo_like.pbrt")).read(), "hlbvh", 4))
    hits = hs.intersect(rays)
    same = hits["prim"] == g["hits"]["prim"]
    assert same.mean() >= 0.999                      # ties on shared edges may go to the neighbouring triangle
    assert np.array_equal(gc.bits(hits["t"][same]), gc.bits(g["hits"]["t"][same]))
    img, st = hs.render()
    frac, mean_rel = image_metrics(img, g["image"])
    assert frac >= 0.999 and mean_rel <= 1e-4, (frac, mean_rel)


@pytest.mark.parametrize("maxprims,split", [(16, "sah"), (40, "equal"), (1, "middle")])
def test_other_bvh_shapes_match_checker(pb, checker, maxprims, split):
    """Leaves of up to 16 primitives still fit the two-child records, 40 do not (the 32-byte-node kernel takes over),
    1 gives the deepest tree; every variant must trace and render like the checker's BVHAccel built the same way."""
    text = open(os.path.join(SCENES, "killeroo_like.pbrt")).read().replace(
        "WorldBegin", 'Accelerator "bvh" "string splitmethod" "%s" "integer maxnodeprims" [%d]\nWorldBegin' % (split, maxprims))
    hs = pb.HostScene.from_string(text)
    sm = {"sah": 0, "middle": 2, "equal": 3}[split]
    sc = checker.scene(hs, max_prims_in_node=maxprims, split_method=sm)
    rays = gc.rays_for(pb, hs.nodes(), 20000, 61)
    assert hs.intersect(rays).tobytes() == _without_b(sc.intersect(rays), hs.intersect(rays))
    img, st = hs.render()
    ref_img, _, ref_st = sc.render(n_threads=0)
    frac, mean_rel = image_metrics(img, ref_img)
    assert frac >= 0.999 and mean_rel <= 1e-4
    assert abs(int(st.regular_rays) - int(ref_st.regular_rays)) <= ref_st.regular_rays // 1000 + 2


def test_instanced_soup_matches_checker(pb, checker):
    """A soup object instanced 4 x 4 times with random rotations (the generator of BASELINE.json configs[3] at a size the
    CPU checker renders in a second): hits bit-identical, any-hits equal, image and ray counters as for every scene."""
    hs = pb.HostScene.instanced_soup(2000, grid=4, xres=64, yres=36, spp=4)
    sc = checker.scene(hs)
    rays = gc.rays_for(pb, hs.nodes(), 20000, 51)
    assert hs.intersect(rays).tobytes() == _without_b(sc.intersect(rays), hs.intersect(rays))
    srays = gc.rays_for(pb, hs.nodes(), 20000, 52, shadow=True)
    assert np.array_equal(hs.intersect_p(srays), sc.intersect_p(srays))
    img, st = hs.render()
    ref_img, _, ref_st = sc.render(n_threads=0)
    frac, mean_rel = image_metrics(img, ref_img)
    assert frac >= 0.999 and mean_rel <= 1e-4
    assert st.camera_rays == ref_st.camera_rays == 64 * 36 * 4
    assert abs(int(st.regular_rays) - int(ref_st.regular_rays)) <= ref_st.regular_rays // 1000 + 2
    assert abs(int(st.shadow_rays) - int(ref_st.shadow_rays)) <= ref_st.shadow_rays // 1000 + 2
    # traversal counters: both BVH levels count like the reference's STAT_COUNTERs would
    dev = hs.device_scene()
    film = np.zeros((36, 64, 4), np.float32)
    cst = pb.Stats()
    pb.check(pb.lib().pb2_render_path(dev, hs.camera, hs.film, hs.params_copy(flags=1), pb.ptr(film), C.byref(cst)))
    if checker.kind == "port":
        assert abs(int(cst.node_visits) - int(ref_st.node_visits)) <= ref_st.node_visits // 1000 + 10
        assert abs(int(cst.prim_tests) - int(ref_st.prim_tests)) <= ref_st.prim_tests // 1000 + 10


def _without_b(ref_hits, gpu_hits):
    """The checker's SurfaceInteraction has no barycentrics; take the GPU's so that every other byte is compared."""
    h = ref_hits.copy()
    h["b"] = gpu_hits["b"]
    return h.tobytes()


def test_traversal_counters_equal_the_reference_order(pb, port):
    """PB2_FLAG_COUNT_TRAVERSAL counts LinearBVHNode fetches / primitive tests like STAT_COUNTERs around bvh.cpp:672/677/710/714
    would; the port counts the same events on the CPU: identical traversal order => identical counts."""
    hs = pb.HostScene.soup(5000, xres=48, yres=27, spp=4)
    dev = hs.device_scene()
    film = np.zeros((27, 48, 4), np.float32)
    st = pb.Stats()
    pb.check(pb.lib().pb2_render_path(dev, hs.camera, hs.film, hs.params_copy(flags=1), pb.ptr(film), C.byref(st)))
    _, _, pst = port.scene(hs).render(n_threads=1)
    assert st.node_visits > 0 and st.prim_tests > 0
    assert abs(int(st.node_visits) - int(pst.node_visits)) <= pst.node_visits // 1000 + 10
    assert abs(int(st.prim_tests) - int(pst.prim_tests)) <= pst.prim_tests // 1000 + 10
    # the counting kernel and the tuned kernel produce the same film
    film2, st2 = hs.render_rgbw()
    assert np.allclose(film, film2, rtol=1e-5, atol=1e-5)
    assert st2.regular_rays == st.regular_rays and st2.shadow_rays == st.shadow_rays
    # ... and so do the other kernels (two-child records, the 32-byte LinearBVHNode array, the small-stack builds).  At this
    # size k_wf_finish takes over after round 0, so they trace camera rays only; test_gpu_wavefront_schedules.py renders
    # them with the rounds forced
    for kname, flags in wf_kernels(pb).items():
        film3 = np.zeros((27, 48, 4), np.float32)
        st3 = pb.Stats()
        pb.check(pb.lib().pb2_render_path(dev, hs.camera, hs.film, hs.params_copy(flags=flags), pb.ptr(film3), C.byref(st3)))
        assert np.allclose(film, film3, rtol=1e-5, atol=1e-5), kname
        assert st3.regular_rays == st.regular_rays and st3.shadow_rays == st.shadow_rays, kname


def wf_kernels(pb):
    """Every traversal kernel of the render path (selected by pb2_path_params.flags)."""
    return {"wide2": 0, "wide4": pb.PB2_FLAG_WIDE4, "linear": pb.PB2_FLAG_LINEAR_NODES, "plain": pb.PB2_FLAG_PLAIN_TRACE,
            "wide2_spill": pb.PB2_FLAG_SMALL_STACK, "wide4_spill": pb.PB2_FLAG_SMALL_STACK | pb.PB2_FLAG_WIDE4,
            "wide2_ld128": pb.PB2_FLAG_LD128, "wide4_ld128": pb.PB2_FLAG_LD128 | pb.PB2_FLAG_WIDE4,
            "wide2_leaf_tma": pb.PB2_FLAG_LEAF_TMA, "ray_pool": pb.PB2_FLAG_POOL}


def check_wavefront_records(pb, hs, rays, srays, want_hits, want_occluded):
    """pb2_trace_wavefront (the persistent-warp kernels the renderer launches) against Scene::Intersect / IntersectP
    results: found flag, primitive, t and the barycentrics BIT FOR BIT, for every kernel variant, with the two ray
    classes alone and mixed inside the same warps."""
    hit = want_hits["prim"] >= 0
    mixed = np.concatenate([rays, srays])
    cls = np.concatenate([np.zeros(len(rays), np.uint8), np.ones(len(srays), np.uint8)])
    perm = np.random.RandomState(5).permutation(len(mixed))
    for kname, flags in wf_kernels(pb).items():
        for batch in ("split", "mixed"):
            if batch == "split":
                r = hs.trace_wavefront(rays, flags=flags)
                q = hs.trace_wavefront(srays, any_hit=np.ones(len(srays), np.uint8), flags=flags)
            else:
                m = hs.trace_wavefront(mixed[perm], any_hit=cls[perm], flags=flags)
                back = np.empty_like(m)
                back[perm] = m
                r, q = back[: len(rays)], back[len(rays):]
            assert np.array_equal(r["found"] > 0, hit), kname
            assert np.array_equal(r["prim"], want_hits["prim"]), kname
            assert np.array_equal(gc.bits(r["t"]), gc.bits(want_hits["t"])), kname
            assert np.array_equal(gc.bits(r["b"][hit]), gc.bits(want_hits["b"][hit])), kname
            assert (r["listed"] == 1).all() and (q["listed"] == 2).all(), kname
            assert np.array_equal(q["found"] > 0, want_occluded != 0), kname


@pytest.mark.parametrize("name", SCENE_CASES)
def test_wavefront_trace_kernels_write_the_reference_hit_records(pb, name):
    """The kernels that are BENCHMARKED (k_wf_trace_w<2>, <4>, k_wf_trace) leave the reference's closest hit in the path
    contexts: same rays as the golden hit test, compared with the golden prim / t recorded from the compiled reference
    and with every bit of pb2_intersect's (t, b0, b1, b2), which that test pins to the reference."""
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    hs = load_scene(pb, name)
    nodes = hs.nodes()
    rays, srays = gc.rays_for(pb, nodes, 1500, 11), gc.rays_for(pb, nodes, 1500, 12, shadow=True)
    hits = hs.intersect(rays)
    assert np.array_equal(hits["prim"], g["hits"]["prim"]) and np.array_equal(gc.bits(hits["t"]), gc.bits(g["hits"]["t"]))
    check_wavefront_records(pb, hs, rays, srays, hits, g["occluded"])


def test_wavefront_trace_kernels_on_instances_and_deep_stacks(pb, checker):
    """Instanced soup (two BVH levels, the instance frame on the kernel's stack) and a BVH with one primitive per leaf
    (deepest stacks): hit records of every kernel variant against the CPU checker's Scene::Intersect."""
    deep = open(os.path.join(SCENES, "killeroo_like.pbrt")).read().replace(
        "WorldBegin", 'Accelerator "bvh" "string splitmethod" "middle" "integer maxnodeprims" [1]\nWorldBegin')
    for make, kw in ((lambda: pb.HostScene.instanced_soup(2000, grid=4, xres=64, yres=36, spp=4), {}),
                     (lambda: pb.HostScene.from_string(deep), dict(max_prims_in_node=1, split_method=2))):
        hs = make()   # the host front end holds one scene at a time
        sc = checker.scene(hs, **kw)
        rays, srays = gc.rays_for(pb, hs.nodes(), 20000, 61), gc.rays_for(pb, hs.nodes(), 20000, 62, shadow=True)
        want = sc.intersect(rays)
        got = hs.intersect(rays)
        assert np.array_equal(got["prim"], want["prim"]) and np.array_equal(gc.bits(got["t"]), gc.bits(want["t"]))
        check_wavefront_records(pb, hs, rays, srays, got, sc.intersect_p(srays))


@pytest.mark.parametrize("partial", [False, True])
def test_sphere_spawned_rays_do_not_reintersect_on_gpu(pb, port, partial):
    """FullSphere.Reintersect / PartialSphere.Reintersect (src/tests/shapes.cpp:427-497) through pb2_intersect / pb2_intersect_p,
    and the hits themselves against the CPU checker."""
    found = 0
    for i in range(12):
        text, rays, rng = gc.sphere_reintersect_case(pb, i, partial)
        hs = pb.HostScene.from_string(text)
        h = hs.intersect(rays)
        want = port.scene(hs).intersect(rays)
        assert np.array_equal(h["prim"], want["prim"]) and np.array_equal(gc.bits(h["t"]), gc.bits(want["t"]))
        assert np.array_equal(gc.bits(h["p"]), gc.bits(want["p"])) and np.array_equal(gc.bits(h["p_error"]), gc.bits(want["p_error"]))
        h = h[h["prim"] >= 0]
        found += len(h)
        if len(h) == 0:
            continue
        out = gc.spawned_rays(pb, h, rng)
        assert (hs.intersect(out)["prim"] == -1).all() and not hs.intersect_p(out).any()
    assert found > 300


def test_watertight_on_gpu(pb):
    hs, verts = tessellated_sphere_scene(pb)
    rng = np.random.RandomState(1)
    n = 50000
    rays = np.zeros(n, pb.RAY_DTYPE)
    rays["o"] = rng.uniform(-0.5, 0.5, (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3))
    rays["d"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    rays["d"][: n // 2] = verts[rng.randint(0, len(verts), n // 2)] - rays["o"][: n // 2]
    rays["t_max"] = np.inf
    assert (hs.intersect(rays)["prim"] >= 0).all()
    assert hs.intersect_p(rays).all()


def test_edge_cases(pb):
    hs = gc.soup_scene(pb)
    assert len(hs.intersect(np.zeros(0, pb.RAY_DTYPE))) == 0            # empty batch
    rays = np.zeros(4, pb.RAY_DTYPE)
    rays["o"] = (0, 0, 50)
    rays["d"] = [(0, 0, -1), (0, 0, 1), (0, 0, -1), (0, 0, 0)]
    rays["t_max"] = [np.inf, np.inf, 0.0, np.inf]                         # tMax 0 and a zero direction (NaN slabs) must miss
    h = hs.intersect(rays)
    assert h["prim"][0] >= 0 and (h["prim"][1:] == -1).all()
    # maxdepth 0: only emitted light seen directly; spp 1; pixel bounds smaller than the film
    p = hs.params_copy(max_depth=0, samples_per_pixel=1)
    p.pixel_bounds[0], p.pixel_bounds[1], p.pixel_bounds[2], p.pixel_bounds[3] = 4, 2, 20, 10
    film, st = hs.render_rgbw(p)
    assert st.camera_rays == 16 * 8 and st.shadow_rays == 0 and st.regular_rays == st.camera_rays
    w = film[..., 3]
    assert w[2:10, 4:20].sum() >= 16 * 8 - 1e-3 and w[12:, :].sum() == 0
    # invalid arguments are refused with PB2_ERR_INVALID, not crashes
    bad = hs.params_copy(samples_per_pixel=0)
    with pytest.raises(pb.Pb2Error):
        hs.render_rgbw(bad)
    bad = hs.params_copy(tile_rank=3, tile_count=2)
    with pytest.raises(pb.Pb2Error):
        hs.render_rgbw(bad)


def test_tile_partition_sums_to_the_full_film(pb):
    """Multi-GPU contract (SURVEY.md §8e): the films of the tile subsets t % n == r add up to the single-GPU film."""
    hs = pb.HostScene.soup(3000, xres=80, yres=45, spp=4)   # ragged 16x16 tiling
    full, st = hs.render_rgbw()
    for n in (2, 3):
        parts, rays = [], 0
        for r in range(n):
            f, s = hs.render_rgbw(hs.params_copy(tile_rank=r, tile_count=n))
            parts.append(f)
            rays += int(s.camera_rays)
        assert rays == st.camera_rays == 80 * 45 * 4
        assert np.allclose(sum(parts), full, rtol=1e-5, atol=1e-5)
        assert np.array_equal(sum(p[..., 3] for p in parts), full[..., 3])
    # a filter wider than a pixel: samples of one rank's tiles reach into pixels of the other ranks' tiles, so the sum of
    # the per-rank films (the NCCL reduce) is what merges them, as Film::MergeFilmTile merges overlapping tiles
    hs = pb.HostScene.from_string(gc.filter_scene_text(SCENES, "gaussian").replace('"integer xresolution" [40]', '"integer xresolution" [72]'))
    full, st = hs.render_rgbw()
    parts = [hs.render_rgbw(hs.params_copy(tile_rank=r, tile_count=3))[0] for r in range(3)]
    assert np.allclose(sum(parts), full, rtol=1e-4, atol=1e-5)
    assert sum(int((p[..., 3] > 0).sum()) for p in parts) > int((full[..., 3] > 0).sum())   # the per-rank supports overlap


def test_reference_shaped_api_and_cli(pb, tmp_path):
    """Integrator::Render through the host C++ classes writes the image the ABI call produced; the CLI runs a scene file."""
    import subprocess
    hs = pb.HostScene.from_file(os.path.join(SCENES, "materials.pbrt"))
    img, st = hs.render()
    film, _ = hs.render_rgbw()
    assert np.allclose(hs.resolve(film), img, rtol=1e-5, atol=1e-6)
    out = tmp_path / "out.pfm"
    exe = os.path.join(os.path.dirname(pb.LIB_PATH), "pb2_pbrt")
    res = subprocess.run([exe, "--outfile", str(out), os.path.join(SCENES, "materials.pbrt")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert res.returncode == 0, res.stdout
    data = open(out, "rb").read()
    assert data.startswith(b"PF\n48 32\n-1.000000\n")
    cli = np.frombuffer(data[len(b"PF\n48 32\n-1.000000\n"):], "<f4").reshape(32, 48, 3)[::-1]
    assert np.allclose(cli, img, rtol=1e-5, atol=1e-6)
    # the reference's default container: half-float EXR (imageio.cpp:164-190), read back by hand
    import struct
    out = tmp_path / "out.exr"
    res = subprocess.run([exe, "--outfile", str(out), os.path.join(SCENES, "materials.pbrt")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert res.returncode == 0, res.stdout
    data = open(out, "rb").read()
    assert struct.unpack_from("<I", data, 0)[0] == 20000630
    body = np.frombuffer(data[-32 * (8 + 48 * 6):], np.uint8).reshape(32, 8 + 48 * 6)[:, 8:].copy().view(np.float16).reshape(32, 3, 48)
    exr = body[:, ::-1, :].transpose(0, 2, 1).astype(np.float32)
    assert np.allclose(exr, img, rtol=2e-3, atol=1e-4)      # half precision: 11 significant bits


def test_single_shape_intersect_goes_to_the_device(pb):
    """Shape::Intersect on the host classes is answered by the same kernels through a one-primitive aggregate:
    exercised here through a scene with a single triangle (BVH of one leaf)."""
    text = 'Camera "perspective"\nFilm "image" "integer xresolution" [4] "integer yresolution" [4]\nWorldBegin\n' \
           'Shape "trianglemesh" "integer indices" [0 1 2] "point P" [0 0 0  1 0 0  0 1 0]\nWorldEnd\n'
    hs = pb.HostScene.from_string(text)
    rays = np.zeros(2, pb.RAY_DTYPE)
    rays["o"] = [(0.25, 0.25, 1), (2, 2, 1)]
    rays["d"] = (0, 0, -1)
    rays["t_max"] = np.inf
    h = hs.intersect(rays)
    assert h["prim"][0] == 0 and h["prim"][1] == -1 and h["t"][0] == 1.0
    assert np.allclose(h["b"][0], (0.5, 0.25, 0.25)) and np.allclose(h["p"][0], (0.25, 0.25, 0))


def emissive_mesh_scene(n_side, res=(48, 32), spp=4):
    """A grid of 2 * n_side^2 emissive triangles (each one a DiffuseAreaLight, api.cpp:1394-1400) over a matte floor and a
    plastic box: 'spatial' light sampling with thousands of lights."""
    pts, idx = [], []
    for j in range(n_side + 1):
        for i in range(n_side + 1):
            pts += [-1 + 2 * i / n_side, -1 + 2 * j / n_side, 1.6 + 0.1 * np.sin(3.0 * i / n_side) * np.cos(2.0 * j / n_side)]
    for j in range(n_side):
        for i in range(n_side):
            a = j * (n_side + 1) + i
            idx += [a, a + n_side + 1, a + 1, a + 1, a + n_side + 1, a + n_side + 2]
    fmt = lambda v: " ".join("%.6g" % x for x in v)
    return """
LookAt 0 -4 1.2  0 0 .5  0 0 1
Camera "perspective" "float fov" [40]
Film "image" "integer xresolution" [%d] "integer yresolution" [%d] "string filename" "emissive.pfm"
Sampler "halton" "integer pixelsamples" [%d]
Integrator "path" "integer maxdepth" [4]
WorldBegin
AttributeBegin
  AreaLightSource "diffuse" "rgb L" [6 5 4]
  Shape "trianglemesh" "point P" [%s] "integer indices" [%s]
AttributeEnd
Material "matte" "rgb Kd" [.6 .6 .6]
Shape "trianglemesh" "point P" [-3 -3 0 3 -3 0 3 3 0 -3 3 0] "integer indices" [0 1 2 0 2 3]
Material "plastic" "rgb Kd" [.3 .5 .3] "rgb Ks" [.4 .4 .4] "float roughness" [.1]
Shape "trianglemesh" "point P" [-.5 -.5 0 .5 -.5 0 .5 .5 0 -.5 .5 0 -.5 -.5 .8 .5 -.5 .8 .5 .5 .8 -.5 .5 .8]
  "integer indices" [0 1 5 0 5 4 1 2 6 1 6 5 2 3 7 2 7 6 3 0 4 3 4 7 4 5 6 4 6 7]
WorldEnd
""" % (res[0], res[1], spp, fmt(pts), " ".join(str(i) for i in idx))


@pytest.mark.parametrize("name", ["soup", "materials", "lights_spatial"])
def test_lazy_light_distribution_equals_the_eager_one(pb, name, monkeypatch):
    """PB2_LIGHTDIST_LAZY=1: voxel records are built on demand (requested by the first vertex that falls into the voxel,
    built between two kernels, the vertex shaded again).  Everything that depends on them must come out as with the eager
    table: the distributions themselves bit for bit, per-sample Li, the film and the ray counters."""
    def make():
        if name == "lights_spatial":
            return pb.HostScene.from_string(open(os.path.join(SCENES, "lights.pbrt")).read().replace('"power"', '"spatial"'))
        return load_scene(pb, name)
    results = []
    for lazy in ("0", "1"):
        monkeypatch.setenv("PB2_LIGHTDIST_LAZY", lazy)
        hs = make()
        nodes = hs.nodes()
        xres, yres = hs.film.contents.full_resolution[0], hs.film.contents.full_resolution[1]
        spp = hs.params.contents.samples_per_pixel
        pix, sn = gc.sample_ids(xres, yres, spp, 3000, 13)
        results.append((hs.light_distribution(gc.points_for(nodes, 400, 15)), hs.li_samples(pix, sn)[0]) + hs.render_rgbw())
    (d0, l0, f0, s0), (d1, l1, f1, s1) = results
    assert np.array_equal(gc.bits(d0), gc.bits(d1))
    assert np.array_equal(gc.bits(l0), gc.bits(l1))
    assert np.array_equal(f0[..., 3], f1[..., 3]) and np.allclose(f0, f1, rtol=1e-5, atol=1e-5)
    assert (s0.camera_rays, s0.regular_rays, s0.shadow_rays) == (s1.camera_rays, s1.regular_rays, s1.shadow_rays)


def test_emissive_mesh_with_thousands_of_lights(pb, checker):
    """Every emissive triangle is a light (2 x 40 x 40 = 3200 here).  A spatial-distribution record is 25 KB then: the table
    for all 64^3 voxels would take 6 GB and 10^11 light samples; built on demand only the voxels path vertices fall into
    exist - as in the reference, whose results this must match."""
    hs = pb.HostScene.from_string(emissive_mesh_scene(40))
    assert hs.desc.contents.n_lights == 3200
    sc = checker.scene(hs)
    nodes = hs.nodes()
    pts = gc.points_for(nodes, 60, 15)
    assert np.array_equal(gc.bits(hs.light_distribution(pts)), gc.bits(sc.light_distribution(pts)))
    pix, sn = gc.sample_ids(48, 32, 4, 1500, 13)
    li, _ = hs.li_samples(pix, sn)
    ref_li, _ = sc.li_samples(pix, sn)
    assert li_ok(li, ref_li) >= 0.999
    img, st = hs.render()
    ref_img, _, ref_st = sc.render(n_threads=0)
    frac, mean_rel = image_metrics(img, ref_img)
    assert frac >= 0.999 and mean_rel <= 1e-4, (frac, mean_rel)
    assert st.camera_rays == ref_st.camera_rays
    assert abs(int(st.regular_rays) - int(ref_st.regular_rays)) <= ref_st.regular_rays // 1000 + 2


def test_render_after_a_standalone_intersect_sees_the_lights(pb):
    """Scene::Intersect before Render flattens the aggregate without lights; Render must not reuse that copy (a scene lit
    by delta lights only would come out black, one with area lights would fail to flatten)."""
    for name in ("lights", "materials"):
        first, _ = pb.HostScene.from_file(os.path.join(SCENES, name + ".pbrt")).render()
        hs = pb.HostScene.from_file(os.path.join(SCENES, name + ".pbrt"))
        o, d, t = np.array([0, 0, 5], np.float32), np.array([0, 0, -1], np.float32), np.zeros(1, np.float32)
        nodes = hs.nodes()
        o[:] = 0.5 * (nodes["bmin"][0] + nodes["bmax"][0]) + np.float32([0, 0, 2 * (nodes["bmax"][0][2] - nodes["bmin"][0][2])])
        assert hs.L.pb2h_scene_intersect(pb.ptr(o), pb.ptr(d), pb.ptr(t)) in (0, 1)
        img, st = hs.render()
        assert img.mean() > 0 and np.allclose(img, first, rtol=1e-5, atol=1e-6)


def test_maxdepth_beyond_the_halton_tables_is_refused(pb):
    hs = gc.soup_scene(pb)
    dev = hs.device_scene()
    out = np.zeros(hs.film_shape() + (4,), np.float32)
    rc = hs.L.pb2_render_path(dev, hs.camera, hs.film, hs.params_copy(max_depth=124), pb.ptr(out), None)
    assert rc == pb.PB2_ERR_UNSUPPORTED and b"1000 dimensions" in hs.L.pb2_last_error()
    pb.check(hs.L.pb2_render_path(dev, hs.camera, hs.film, hs.params_copy(max_depth=123), pb.ptr(out), None))


def test_texture_lookups_match_the_reference_mipmap(pb):
    """MIPMap::Lookup on the device (EWA and trilinear filtering, three wrap modes, resampled pyramids) against look-ups
    recorded from the compiled reference, for every texture of tests/scenes/textured.pbrt.  The arithmetic is the
    reference's operation for operation; the level of detail goes through log(), where the device's logf and glibc's may
    differ in the last bit: nearly every look-up must be bit-identical, all of them within 2e-6 (relative to the value 1)."""
    g = np.load(os.path.join(GOLDEN, "textures.npz"))
    hs = load_scene(pb, "textured")
    textures = hs.textures()
    assert len(textures) == 10
    for i, t in enumerate(textures):
        st, dst = gc.texture_lookup_inputs(3000, 100 + i)
        got = pb.texture_lookup(t, st, dst)
        want = g["lookup_%d" % i]
        same = (gc.bits(got) == gc.bits(want)).all(axis=1).mean()
        err = np.abs(got - want).max() / max(1.0, float(np.abs(want).max()))
        assert same >= 0.995 and err <= 2e-6, (i, same, err)


def test_alpha_masked_meshes_through_every_render_kernel(pb):
    """The alpha test (triangle.cpp:333-338, 531-569) inside the tuned trace kernel and inside the one-thread-per-ray
    traversal give the same film: the cut-out scene rendered with the default kernel selection and with
    PB2_FLAG_PLAIN_TRACE / PB2_FLAG_LINEAR_NODES (both end in the plain traversal for such scenes)."""
    hs = load_scene(pb, "textured")
    base, st0 = hs.render_rgbw(hs.params_copy(flags=0))
    for flags in (pb.PB2_FLAG_PLAIN_TRACE, pb.PB2_FLAG_LINEAR_NODES):
        film, st = hs.render_rgbw(hs.params_copy(flags=flags))
        assert np.array_equal(film[..., 3], base[..., 3])
        assert np.allclose(film, base, rtol=1e-4, atol=1e-5)
        assert st.regular_rays == st0.regular_rays and st.shadow_rays == st0.shadow_rays


@pytest.mark.parametrize("name", ["soup", "materials", "instances", "specular", "lights"])
def test_chained_light_step_renders_the_same_film(pb, name):
    """PB2_FLAG_CHAIN selects the chained trace kernel and the render still gives the same film and ray counts.  These scenes
    are small enough for k_wf_finish to take over after round 0, before any shadow or MIS ray is in a trace list, so the
    chained light step itself hardly runs here: test_gpu_wavefront_schedules.py checks it with the rounds forced."""
    hs = load_scene(pb, name)
    base, st0 = hs.render_rgbw(hs.params_copy(flags=0))
    film, st = hs.render_rgbw(hs.params_copy(flags=pb.PB2_FLAG_CHAIN))
    assert np.array_equal(film[..., 3], base[..., 3])
    assert np.allclose(film, base, rtol=1e-4, atol=1e-5)
    assert (st.camera_rays, st.regular_rays, st.shadow_rays) == (st0.camera_rays, st0.regular_rays, st0.shadow_rays)
    assert st.kernel_launches < st0.kernel_launches
