"""The shade feature class (pb2_shade_class, SHADE_* in device/pb2_shade.cuh).

A scene whose surfaces are all Lambertian (matte, sigma 0) and whose lights are all area lights gets a shade step, light
step and tail kernel compiled for that class alone: the Oren-Nayar and microfacet lobes and the delta / infinite lights
are compiled out, nothing else changes.  Checks:
  1. each scene selects the class its material and light records call for; PB2_SHADE_GENERAL=1 selects the general one.
  2. with PB2_SHADE_GENERAL=1 and without it, the ray counters are equal and every film equals the per-sample model
     (pb2_li_samples, the general lane functions) within k * 2^-24 * sum |L * w|, the weight channel exactly, both when
     the tail kernel walks the paths and when every bounce goes through the round kernels.  The knobs are read once
     per process, so every configuration renders in a worker process of its own.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

TESTS = os.path.dirname(os.path.abspath(__file__))

SHADE_OREN_NAYAR, SHADE_MICROFACET, SHADE_NON_AREA, SHADE_ALL = 1, 2, 4, 7

# A one-sided emissive quad whose normals point against its winding, over a matte floor and a matte box: every surface
# Lambertian, every light an area light (class 0), no spheres.
MATTE_BOX = """
LookAt 0 -5 1.6  0 0 .3  0 0 1
Camera "perspective" "float fov" [45]
Film "image" "integer xresolution" [48] "integer yresolution" [32]
Sampler "halton" "integer pixelsamples" [8]
Integrator "path" "integer maxdepth" [6]
WorldBegin
AttributeBegin
  AreaLightSource "diffuse" "rgb L" [4 4 4]
  Shape "trianglemesh" "point P" [-1 -1 2.2  1 -1 2.2  1 1 2.2  -1 1 2.2] "integer indices" [0 1 2 0 2 3]
    "normal N" [0 0 -1  0 0 -1  0 0 -1  0 0 -1]
AttributeEnd
Material "matte" "rgb Kd" [.6 .6 .6]
Shape "trianglemesh" "point P" [-4 -4 0 4 -4 0 4 4 0 -4 4 0] "integer indices" [0 1 2 0 2 3]
Material "matte" "rgb Kd" [.2 .3 .5] "float sigma" [0]
Shape "trianglemesh" "point P" [-1.2 -.4 0 -.4 -.4 0 -.4 .4 0 -1.2 .4 0 -1.2 -.4 .8 -.4 -.4 .8 -.4 .4 .8 -1.2 .4 .8]
  "integer indices" [0 1 5 0 5 4 1 2 6 1 6 5 2 3 7 2 7 6 3 0 4 3 4 7 4 5 6 4 6 7]
WorldEnd
"""

# case: the class its records call for
EXPECTED = {
    "soup": 0,                                              # matte Kd .6, two triangle area lights (the bench scene's kind)
    "instanced_soup": 0,
    "matte_box": 0,
    "matte_mesh_lights": 0,                                 # 3200 emissive triangles over matte: the lazy light distribution
    "killeroo_like": SHADE_MICROFACET,                      # plastic killeroos
    "emissive_mesh": SHADE_MICROFACET,                      # a plastic box
    "one_sided_lights": SHADE_MICROFACET,
    "killeroo_simple": SHADE_MICROFACET,                    # the reference's killeroo-simple.pbrt (bench --workload killeroo)
    "materials": SHADE_OREN_NAYAR | SHADE_MICROFACET,       # matte with sigma, plastic
    "instances": SHADE_OREN_NAYAR | SHADE_MICROFACET,
    "params": SHADE_OREN_NAYAR | SHADE_MICROFACET,
    "gaussian": SHADE_OREN_NAYAR | SHADE_MICROFACET,
    "lights": SHADE_ALL,                                    # point, spot and distant lights, and an uber material
    "specular": SHADE_ALL,                                  # mirror / glass
    "substrate": SHADE_ALL,
    "metal": SHADE_ALL,
    "uber": SHADE_ALL,
    "roughglass": SHADE_ALL,
    "envlight": SHADE_ALL,
}
# rendered under both classes: the class-0 scenes, and scenes of other classes as controls
RENDER_CASES = ["soup", "instanced_soup", "matte_box", "matte_mesh_lights", "killeroo_like", "params", "lights"]
CONFIGS = {
    "general": {"PB2_SHADE_GENERAL": "1"},
    "class": {},
    "general_rounds": {"PB2_SHADE_GENERAL": "1", "PB2_FINISH": "0"},
    "class_rounds": {"PB2_FINISH": "0"},
}


def case_text(case):
    """The scene text of this file's own cases (the others: test_gpu_wavefront_schedules.case_text)."""
    if case == "matte_box":
        return MATTE_BOX
    if case == "matte_mesh_lights":
        from test_gpu_parity import emissive_mesh_scene
        text = emissive_mesh_scene(40)
        assert text.count('Material "plastic"') == 1
        return text.replace('Material "plastic"', 'Material "matte"')
    import test_gpu_wavefront_schedules as ws
    return ws.case_text(case)


def make_case(pb, case):
    if case == "killeroo_simple":
        import argparse
        import bench
        return bench.build_scene(argparse.Namespace(workload="killeroo", xres=32, yres=18, spp=1, maxdepth=5))
    if case in ("matte_box", "matte_mesh_lights"):
        return pb.HostScene.from_string(case_text(case))
    import test_gpu_wavefront_schedules as ws
    return ws.make_case(pb, case)


def shade_class(pb, hs):
    L = pb.lib()
    L.pb2_shade_class.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
    out = C.c_int32(-1)
    pb.check(L.pb2_shade_class(C.cast(hs.desc, C.c_void_p), C.byref(out)))
    return out.value


# ---------------------------------------------------------------------------------------------------------------------
# Check 1: the host's choice (no device needed)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(EXPECTED))
def test_scene_selects_its_class(pb, case):
    assert shade_class(pb, make_case(pb, case)) == EXPECTED[case]


CLASS_WORKER = r'''
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import pbrt_v3_b200 as pb
import test_gpu_shade_classes as t
print(" ".join(str(t.shade_class(pb, t.make_case(pb, c))) for c in sys.argv[3:]))
'''


def test_general_switch_selects_the_general_class(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(CLASS_WORKER)
    env = dict(os.environ, PB2_SHADE_GENERAL="1")
    res = subprocess.run([sys.executable, str(script), ROOT, TESTS, "soup", "lights"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, timeout=600, cwd=ROOT, env=env)
    assert res.returncode == 0, res.stdout[-4000:]
    assert res.stdout.split()[-2:] == [str(SHADE_ALL), str(SHADE_ALL)], res.stdout[-4000:]


# ---------------------------------------------------------------------------------------------------------------------
# Check 2: renders under both classes
# ---------------------------------------------------------------------------------------------------------------------
def render_config(out):
    import pbrt_v3_b200 as pb
    from pbrt_v3_b200 import multigpu
    from test_gpu_wavefront_schedules import film_model
    res = {}
    for case in RENDER_CASES:
        hs = make_case(pb, case)
        params = hs.params_copy()
        film, st = hs.render_rgbw(params)
        items = multigpu.work_items(hs.film, params)
        li, pfilm = hs.li_samples(items[:, :2], items[:, 2].astype(np.int64), params)
        model, bound = film_model(hs.film.contents, li, pfilm)
        res.update({case + ":film": film, case + ":stats": np.array([st.camera_rays, st.regular_rays, st.shadow_rays], np.int64),
                    case + ":items": np.int64(len(items)), case + ":model": model, case + ":bound": bound,
                    case + ":class": np.int64(shade_class(pb, hs)),
                    case + ":box": np.bool_(hs.film.contents.filter_type == pb.PB2_FILTER_BOX)})
    np.savez(out, **res)


RENDER_WORKER = r'''
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_gpu_shade_classes as t
t.render_config(sys.argv[3])
print("ok")
'''


@pytest.fixture(scope="module")
def config(tmp_path_factory):
    """config(name) -> {case: {field: array}} of that configuration's worker (run once per module, on first use)."""
    d = tmp_path_factory.mktemp("shade_classes")
    script = d / "worker.py"
    script.write_text(RENDER_WORKER)
    done = {}

    def get(name):
        if name not in done:
            out = d / (name + ".npz")
            env = dict(os.environ)
            for knob in ("PB2_SHADE_GENERAL", "PB2_POOL", "PB2_PIPES", "PB2_FINISH", "PB2_SYNC_EVERY", "PB2_LIGHTDIST_LAZY"):
                env.pop(knob, None)
            env.update(CONFIGS[name])
            res = subprocess.run([sys.executable, str(script), ROOT, TESTS, str(out)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
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


@pytest.mark.gpu
@pytest.mark.parametrize("case", RENDER_CASES)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_film_equals_the_sum_of_its_samples(config, name, case):
    from test_gpu_wavefront_schedules import model_mismatch
    r = config(name)[case]
    assert int(r["stats"][0]) == int(r["items"])
    why = model_mismatch(r["film"], r["model"], r["bound"], bool(r["box"]))
    assert why is None, why


@pytest.mark.gpu
@pytest.mark.parametrize("case", RENDER_CASES)
@pytest.mark.parametrize("tail", ["", "_rounds"])
def test_ray_counters_do_not_depend_on_the_class(config, tail, case):
    general, narrow = config("general" + tail)[case], config("class" + tail)[case]
    assert int(general["class"]) == SHADE_ALL
    if case in EXPECTED:
        assert int(narrow["class"]) == EXPECTED[case]
    assert np.array_equal(general["stats"], narrow["stats"]), (general["stats"].tolist(), narrow["stats"].tolist())
    box = bool(general["box"])
    if box:
        assert np.array_equal(general["film"][..., 3], narrow["film"][..., 3])
