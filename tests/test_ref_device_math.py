"""The compiled reference's device-math mode (oracle/ref_devmath.cpp, `Oracle.device_math()`), on the CPU.

libpbrt_ref.so routes the reference's sinf / cosf / sincosf / logf / atan2f / acosf through wrappers.  With the mode off
they are glibc's functions, so the reference computes what it always computed; with it on they are (float)f((double)x),
the device's definitions (pb2_math.cuh), and test_gpu_exact_parity.py compares the CUDA path with the reference bit for
bit.  These tests check the wrappers themselves, that they reach the path's code, and that the mode leaves the tables built
at construction (which the library builds on the host with glibc) alone.
"""
import ctypes as C
import ctypes.util
import os

import numpy as np
import pytest

import golden_cases as gc
from conftest import GOLDEN
from test_gpu_parity import SCENE_CASES
from test_oracle import load_scene

F32 = np.float32


@pytest.fixture(scope="module")
def ref():
    from oracle import pyoracle
    r = pyoracle.reference()
    if r is None:
        pytest.skip("the compiled reference (oracle/_ref) is not built here")
    if not r.has_device_math:
        # a library from before the wrappers: where the reference's sources are, __graft_entry__.build() relinks it
        pytest.skip("oracle/_ref/libpbrt_ref.so predates the device-math wrappers and the reference's sources are not here to relink it")
    return r


@pytest.fixture(scope="module")
def libm():
    m = C.CDLL(ctypes.util.find_library("m"))
    for name in ("sinf", "cosf", "logf", "acosf"):
        getattr(m, name).restype, getattr(m, name).argtypes = C.c_float, [C.c_float]
    m.atan2f.restype, m.atan2f.argtypes = C.c_float, [C.c_float, C.c_float]
    for name in ("sin", "cos", "log", "acos"):
        getattr(m, name).restype, getattr(m, name).argtypes = C.c_double, [C.c_double]
    m.atan2.restype, m.atan2.argtypes = C.c_double, [C.c_double, C.c_double]
    m.sincos.restype, m.sincos.argtypes = None, [C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    m.sincosf.restype, m.sincosf.argtypes = None, [C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    return m


def awkward(rng, n, lo_exp=-45, hi_exp=38):
    """Random floats of every magnitude and sign, with +-0, the smallest subnormals, the largest finite values."""
    mag = 10.0 ** rng.uniform(lo_exp, hi_exp, n)
    x = (np.sign(rng.uniform(-1, 1, n)) * mag).astype(F32)
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754942e-38, 1.1754944e-38, 3.4028235e38, -3.4028235e38,
                        1e30, -1e30, 1e20, 65536.0, np.pi, -np.pi, np.pi / 2, 2 * np.pi], F32)
    return np.concatenate([special, x, rng.uniform(-10, 10, n).astype(F32)])


def host(libm, name, a, b=None):
    """glibc's float function and the device's definition (float)f((double)x), one argument at a time."""
    g, d = [], []
    for i, x in enumerate(a):
        x = float(x)
        if name == "sincosf":
            s, c = C.c_float(), C.c_float()
            libm.sincosf(x, C.byref(s), C.byref(c))
            g.append((s.value, c.value))
            ds, dc = C.c_double(), C.c_double()
            libm.sincos(x, C.byref(ds), C.byref(dc))
            d.append((ds.value, dc.value))
        elif name == "atan2f":
            g.append(libm.atan2f(x, float(b[i])))
            d.append(libm.atan2(x, float(b[i])))
        else:
            g.append(getattr(libm, name)(x))
            d.append(getattr(libm, name[:-1])(x))
    return np.array(g, F32), np.array(d, np.float64).astype(F32)


def test_wrappers_are_exported(ref):
    for name in ("sinf", "cosf", "sincosf", "logf", "atan2f", "acosf"):
        assert hasattr(ref.L, "__wrap_" + name), name


@pytest.mark.parametrize("name", ["sinf", "cosf", "sincosf", "logf", "atan2f", "acosf"])
def test_wrapped_function_is_glibc_or_the_device_definition(ref, libm, name):
    rng = np.random.RandomState(7)
    b = None
    if name == "logf":
        a = np.abs(awkward(rng, 3000))                              # +0 and -0 kept: log gives -inf for both
        a = np.concatenate([a, np.array([-0.0, 1.0, 2.0, 0.5], F32)])
    elif name == "acosf":
        a = np.concatenate([np.array([1, -1, 0, -0.0, 1e-45, -1e-45, 0.5, -0.5, 0.99999994, -0.99999994], F32),
                            rng.uniform(-1, 1, 3000).astype(F32), (np.sign(rng.uniform(-1, 1, 1000)) * 10.0 ** rng.uniform(-45, 0, 1000)).astype(F32)])
    elif name == "atan2f":
        y, x = awkward(rng, 1500, -40, 38), awkward(rng, 1500, -40, 38)[::-1]
        zeros = np.array([0.0, -0.0], F32)
        ones = np.array([1.0, -1.0, 1e-45, -3e38], F32)
        q = [(a0, b0) for a0 in np.concatenate([zeros, ones]) for b0 in np.concatenate([zeros, ones])]   # four quadrants, axes, zeros
        a = np.concatenate([y, np.array([p[0] for p in q], F32)])
        b = np.concatenate([x, np.array([p[1] for p in q], F32)])
    else:
        a = awkward(rng, 3000)
    glibc, device = host(libm, name, a, b)
    with ref.device_math(False):
        off = ref.transcendental(name, a, b)
    with ref.device_math(True):
        on = ref.transcendental(name, a, b)
    assert np.array_equal(gc.bits(off), gc.bits(glibc)), "mode off: not glibc's %s" % name
    assert np.array_equal(gc.bits(on), gc.bits(device)), "mode on: not (float)%s((double)x)" % name[:-1]
    # the two definitions do differ now and then: the mode is not a no-op
    if name in ("sinf", "cosf", "sincosf", "logf", "atan2f"):
        assert not np.array_equal(gc.bits(glibc), gc.bits(device)), name


def test_device_math_mode_is_restored_and_refused_on_the_port(ref, libm, port):
    x = awkward(np.random.RandomState(3), 500)
    glibc, device = host(libm, "sinf", x)
    with ref.device_math():
        with ref.device_math(False):
            inner = ref.transcendental("sinf", x)
        outer = ref.transcendental("sinf", x)
    after = ref.transcendental("sinf", x)
    assert np.array_equal(gc.bits(inner), gc.bits(glibc)) and np.array_equal(gc.bits(after), gc.bits(glibc))
    assert np.array_equal(gc.bits(outer), gc.bits(device))
    with pytest.raises(RuntimeError):
        with port.device_math():
            pass


def test_device_math_reaches_the_path_and_nothing_else(pb, ref):
    """Mode off, the golden scenes' Li and Halton samples are the recorded ones bit for bit; mode on, some Li samples change
    (the transcendentals run in sampling, shading and sphere hits) while the Halton samples (no transcendentals) do not.
    The counts printed are the size of the effect that the tolerances of test_gpu_parity.py budget for."""
    changed = {}
    for name in SCENE_CASES:
        g = np.load(os.path.join(GOLDEN, name + ".npz"))
        hs = load_scene(pb, name)
        sc = ref.scene(hs)
        f = hs.film.contents
        xres, yres, spp = f.full_resolution[0], f.full_resolution[1], hs.params.contents.samples_per_pixel
        pix, sn = gc.sample_ids(xres, yres, spp, 3000, 13)
        hpix, hsn, hdim = gc.sample_ids(xres, yres, spp, 4000, 14, max_dim=200)
        li_off, pf_off = sc.li_samples(pix, sn)
        with ref.device_math():
            li_on, pf_on = sc.li_samples(pix, sn)
            halton_on = ref.halton(hs.film, hs.params, hpix, hsn, hdim)
        assert np.array_equal(gc.bits(li_off), gc.bits(g["li"])), name
        assert np.array_equal(gc.bits(halton_on), gc.bits(g["halton"])), name
        assert np.array_equal(gc.bits(pf_on), gc.bits(pf_off)), name
        changed[name] = int((gc.bits(li_on) != gc.bits(li_off)).any(axis=1).sum())
    print("Li samples (of 3000) that change when the reference uses the device's transcendentals:", changed)
    assert sum(changed.values()) > 0, changed


def test_construction_tables_are_built_with_glibc_in_device_math_mode(pb, ref):
    """InfiniteAreaLight's Distribution2D and MIPMap's Lanczos-resampled pyramids are built by the library on the host with
    glibc; in device-math mode the reference still builds them the same way, bit for bit as recorded."""
    with ref.device_math():
        g = np.load(os.path.join(GOLDEN, "env_distribution.npz"))
        hs = pb.HostScene.from_file(os.path.join(os.path.dirname(GOLDEN), "scenes", "envmap.pbrt"))
        d = hs.desc.contents
        env = [d.delta_lights[i].env_tex for i in range(d.n_lights) if d.lights[i].type == pb.PB2_LIGHT_INFINITE][0]
        nu, nv, table = ref.env_distribution(d.textures[env - 1])
        assert (nu, nv) == (int(g["nu"]), int(g["nv"])) and np.array_equal(gc.bits(table), gc.bits(g["table"]))
        g = np.load(os.path.join(GOLDEN, "texture_pyramids.npz"))
        for i, t in enumerate(gc.awkward_textures(pb)):
            levels = ref.texture_pyramid(t)
            assert np.array_equal(gc.bits(np.concatenate([lv.ravel() for lv in levels])), gc.bits(g["pyramid_%d" % i])), i
