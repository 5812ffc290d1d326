"""TEST INFRASTRUCTURE ONLY — ctypes view of the two CPU checkers.

* ``oracle/_ref/libpbrt_ref.so``  (``kind == "reference"``): the unmodified reference sources compiled
  by ``oracle/Makefile.ref`` behind ``oracle/ref_harness.cpp``.
* ``oracle/lib/libpb2_oracle.so`` (``kind == "port"``): the plain C++ restatement ``oracle/pb2_oracle.cpp``.

Both export the same entry points (prefix ``ref_`` / ``orc_``) over the same ``pb2_scene_desc`` the CUDA
library consumes.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module; the product (pbrt_v3_b200/) never does.
"""
import contextlib
import ctypes as C
import os

import numpy as np

from pbrt_v3_b200 import (Camera, FilmDesc, HIT_DTYPE, NODE_DTYPE, PathParams, RAY_DTYPE, SceneDesc, Stats, ptr)

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_PATH = os.path.join(_HERE, "_ref", "libpbrt_ref.so")
PORT_PATH = os.path.join(_HERE, "lib", "libpb2_oracle.so")


class Oracle:
    def __init__(self, path, prefix, kind):
        self.kind = kind
        self.L = C.CDLL(path)
        self.p = prefix
        vp = C.c_void_p
        f = self._f
        f("scene_create").restype = vp
        f("scene_create").argtypes = [C.POINTER(SceneDesc), C.c_int, C.c_int]
        f("scene_destroy").argtypes = [vp]
        f("bvh_dump").restype = C.c_int64
        f("bvh_dump").argtypes = [vp, vp, C.c_int64, vp]
        f("intersect").argtypes = [vp, vp, C.c_int64, vp]
        f("intersect_p").argtypes = [vp, vp, C.c_int64, vp]
        f("render").argtypes = [vp, C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), C.c_int, vp,
                                C.POINTER(C.c_double), C.POINTER(Stats)]
        f("li_samples").argtypes = [vp, C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), vp, vp, C.c_int64, vp, vp]
        f("halton_samples").argtypes = [C.POINTER(FilmDesc), C.POINTER(PathParams), vp, vp, vp, C.c_int64, vp]
        f("radical_inverse").argtypes = [C.c_int, vp, C.c_int64, C.c_int, vp]
        f("light_distribution").argtypes = [vp, vp, C.c_int64, vp]
        f("loop_subdivide").argtypes = [C.c_int, C.c_int, vp, C.c_int, vp, C.POINTER(C.c_int), C.POINTER(C.c_int), vp, vp, vp]
        f("camera_derived").argtypes = [C.POINTER(Camera), C.POINTER(FilmDesc), vp, vp, vp]
        f("transform").argtypes = [C.c_int, vp, vp, vp]

    def _f(self, name):
        return getattr(self.L, self.p + name)

    def scene(self, host_scene, max_prims_in_node=4, split_method=0):
        return OracleScene(self, host_scene, max_prims_in_node, split_method)

    def halton(self, film, params, pixel_xy, sample_num, dim):
        pixel_xy = np.ascontiguousarray(pixel_xy, np.int32)
        sample_num = np.ascontiguousarray(sample_num, np.int64)
        dim = np.ascontiguousarray(dim, np.int32)
        out = np.zeros(len(dim), np.float32)
        if self._f("halton_samples")(film, params, ptr(pixel_xy), ptr(sample_num), ptr(dim), len(dim), ptr(out)):
            raise RuntimeError("the %s oracle does not restate this sampler" % self.kind)
        return out

    def radical_inverse(self, base_index, a, scrambled=False):
        a = np.ascontiguousarray(a, np.uint64)
        out = np.zeros(len(a), np.float32)
        self._f("radical_inverse")(base_index, ptr(a), len(a), 1 if scrambled else 0, ptr(out))
        return out

    def loop_subdivide(self, n_levels, indices, P):
        indices = np.ascontiguousarray(indices, np.int32)
        P = np.ascontiguousarray(P, np.float32)
        nv, ni = C.c_int(), C.c_int()
        fn = self._f("loop_subdivide")
        fn(n_levels, len(indices), ptr(indices), len(P), ptr(P), C.byref(nv), C.byref(ni), None, None, None)
        oP = np.zeros((nv.value, 3), np.float32)
        oN = np.zeros((nv.value, 3), np.float32)
        oI = np.zeros(ni.value, np.int32)
        fn(n_levels, len(indices), ptr(indices), len(P), ptr(P), C.byref(nv), C.byref(ni), ptr(oP), ptr(oN), ptr(oI))
        return oP, oN, oI

    def camera_derived(self, camera, film):
        r2c = np.zeros(16, np.float32)
        dx = np.zeros(3, np.float32)
        dy = np.zeros(3, np.float32)
        self._f("camera_derived")(camera, film, ptr(r2c), ptr(dx), ptr(dy))
        return r2c, dx, dy

    def texture_pyramid(self, texture):
        """MIPMap::pyramid of the reference for one pb2_texture: list of (h, w, channels) arrays (reference only)."""
        import pbrt_v3_b200 as pb
        fn = self._f("texture_pyramid")
        fn.argtypes = [C.POINTER(pb.Texture), C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_void_p]
        return pb.texture_pyramid(texture, fn)

    def texture_lookup(self, texture, st, dst):
        """MIPMap::Lookup(st, dst0, dst1) of the reference for a batch (reference only)."""
        import pbrt_v3_b200 as pb
        st = np.ascontiguousarray(st, np.float32)
        dst = np.ascontiguousarray(dst, np.float32)
        out = np.zeros((len(st), 3), np.float32)
        fn = self._f("texture_lookup")
        fn.argtypes = [C.POINTER(pb.Texture), C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
        fn(C.byref(texture), len(st), ptr(st), ptr(dst), ptr(out))
        return out

    def sobol_tables(self, m):
        """The reference's VdCSobolMatrices[m - 1] / VdCSobolMatricesInv[m - 1] (104 entries) and SobolMatrices32 (reference only)."""
        tab = np.zeros(104, np.uint64)
        mats = np.zeros((1024, 52), np.uint32)
        fn = self._f("sobol_tables")
        fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        if fn(m, ptr(tab), ptr(mats)):
            raise ValueError("resolution 2^%d outside the reference's tables" % m)
        return tab, mats

    def bsdf_eval(self, material, frames):
        """The reference's own BSDF (Material::ComputeScatteringFunctions, BSDF::f / Pdf / Sample_f) for a material record at
        given shading frames (reference only; layout as pb2_bsdf_eval_host)."""
        import pbrt_v3_b200 as pb
        fn = self._f("bsdf_eval")
        fn.argtypes = [C.POINTER(pb.Material), C.c_int64, C.c_void_p, C.c_void_p]
        return pb.bsdf_eval_host(material, frames, fn)

    def texture_evaluate(self, textures, n_textures, tex_id, uv, duv):
        """Texture::Evaluate of the reference's own texture objects built from a description's texture array (reference only)."""
        import pbrt_v3_b200 as pb
        fn = self._f("texture_evaluate")
        fn.argtypes = [C.POINTER(pb.Texture), C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
        return pb.texture_eval_host(textures, n_textures, tex_id, uv, duv, fn)

    def env_distribution(self, texture):
        """InfiniteAreaLight::distribution for an environment map given as a pb2_texture: (nu, nv, table) in the layout of
        pb2_env_distribution (reference only)."""
        import pbrt_v3_b200 as pb
        fn = self._f("env_distribution")
        fn.argtypes = [C.POINTER(pb.Texture), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_void_p]
        return pb.env_distribution(texture, fn)

    def copper_rgb(self):
        """(eta, k) RGB of the metal material's default copper spectra (reference only)."""
        eta = np.zeros(3, np.float32)
        k = np.zeros(3, np.float32)
        self._f("copper_rgb")(ptr(eta), ptr(k))
        return eta, k

    @property
    def has_device_math(self):
        """True when this library was linked by oracle/Makefile.ref with the device-math wrappers (a reference library built
        by an older recipe has neither the wrappers nor the switch)."""
        return self.kind == "reference" and hasattr(self.L, "ref_set_device_math") and hasattr(self.L, "__wrap_sinf")

    @contextlib.contextmanager
    def device_math(self, on=True):
        """Within the block the reference evaluates sinf / cosf / sincosf / logf / atan2f / acosf as the device does,
        (float)f((double)x) (oracle/ref_devmath.cpp), while it traces, samples, shades and looks textures up; scenes, lights,
        films, cameras and textures are still built with glibc's functions.  The previous setting is restored on exit
        (reference only: the port has no such switch)."""
        if self.kind != "reference":
            raise RuntimeError("device math is a mode of the compiled reference, not of the %s oracle" % self.kind)
        if not self.has_device_math:
            raise RuntimeError("%s was built without the device-math wrappers: rebuild it with oracle/Makefile.ref" % self.L._name)
        fn = self._f("set_device_math")
        fn.argtypes, fn.restype = [C.c_int], C.c_int
        was = fn(1 if on else 0)
        try:
            yield self
        finally:
            fn(was)

    TRANSCENDENTALS = {"sinf": 0, "cosf": 1, "sincosf": 2, "logf": 3, "atan2f": 4, "acosf": 5}

    def transcendental(self, name, a, b=None):
        """One of the six wrapped float functions, called from the reference's harness under the current device-math setting:
        (n,) results, (n, 2) = (sin, cos) for sincosf; atan2f takes y = a, x = b (reference only)."""
        a = np.ascontiguousarray(a, np.float32)
        b = np.ascontiguousarray(a if b is None else b, np.float32)
        out = np.zeros((len(a), 2) if name == "sincosf" else len(a), np.float32)
        fn = self._f("transcendentals")
        fn.argtypes = [C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
        if fn(self.TRANSCENDENTALS[name], len(a), ptr(a), ptr(b), ptr(out)):
            raise ValueError(name)
        return out

    def transform(self, kind, args):
        args = np.ascontiguousarray(args, np.float32)
        m = np.zeros(16, np.float32)
        mi = np.zeros(16, np.float32)
        self._f("transform")(kind, ptr(args), ptr(m), ptr(mi))
        return m, mi


class OracleScene:
    def __init__(self, oracle, host_scene, max_prims_in_node, split_method):
        self.o = oracle
        self.hs = host_scene
        self.h = oracle._f("scene_create")(host_scene.desc, max_prims_in_node, split_method)
        if not self.h:
            raise RuntimeError("oracle could not build the scene")
        self.n_lights = host_scene.desc.contents.n_lights
        self.n_prims = host_scene.bvh_range(0)[3]   # primitives of the scene-level BVH

    def __del__(self):
        try:
            if self.h:
                self.o._f("scene_destroy")(self.h)
                self.h = None
        except Exception:
            pass

    def bvh(self):
        n = self.o._f("bvh_dump")(self.h, None, 0, None)
        nodes = np.zeros(n, NODE_DTYPE)
        prims = np.zeros(self.n_prims, np.int32)
        self.o._f("bvh_dump")(self.h, ptr(nodes), n, ptr(prims))
        return nodes, prims

    def intersect(self, rays):
        rays = np.ascontiguousarray(rays, RAY_DTYPE)
        hits = np.zeros(len(rays), HIT_DTYPE)
        self.o._f("intersect")(self.h, ptr(rays), len(rays), ptr(hits))
        return hits

    def intersect_p(self, rays):
        rays = np.ascontiguousarray(rays, RAY_DTYPE)
        occ = np.zeros(len(rays), np.uint8)
        self.o._f("intersect_p")(self.h, ptr(rays), len(rays), ptr(occ))
        return occ

    def render(self, n_threads=0, params=None):
        h, w = self.hs.film_shape()
        out = np.zeros((h, w, 3), np.float32)
        secs = C.c_double()
        st = Stats()
        rc = self.o._f("render")(self.h, self.hs.camera, self.hs.film, params if params is not None else self.hs.params,
                                 n_threads, ptr(out), C.byref(secs), C.byref(st))
        if rc:
            raise RuntimeError("the %s oracle does not cover this frame (sampler outside its restatement)" % self.o.kind)
        return out, secs.value, st

    def li_samples(self, pixel_xy, sample_num, params=None):
        pixel_xy = np.ascontiguousarray(pixel_xy, np.int32)
        sample_num = np.ascontiguousarray(sample_num, np.int64)
        n = len(sample_num)
        rgb = np.zeros((n, 3), np.float32)
        pfilm = np.zeros((n, 2), np.float32)
        if self.o._f("li_samples")(self.h, self.hs.camera, self.hs.film, params if params is not None else self.hs.params,
                                   ptr(pixel_xy), ptr(sample_num), n, ptr(rgb), ptr(pfilm)):
            raise RuntimeError("the %s oracle does not cover this frame (sampler outside its restatement)" % self.o.kind)
        return rgb, pfilm

    def camera_differentials(self, pixel_xy, sample_num, params=None):
        """Camera rays with their differentials, the first hit and its (u, v) differentials as the reference computes them:
        (n, 39) records (layout in oracle/ref_harness.cpp, ref_camera_differentials; reference only)."""
        pixel_xy = np.ascontiguousarray(pixel_xy, np.int32)
        sample_num = np.ascontiguousarray(sample_num, np.int64)
        out = np.zeros((len(sample_num), 39), np.float32)
        fn = self.o._f("camera_differentials")
        fn.argtypes = [C.c_void_p, C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        fn(self.h, self.hs.camera, self.hs.film, params if params is not None else self.hs.params, ptr(pixel_xy), ptr(sample_num),
           len(sample_num), ptr(out))
        return out

    def light_distribution(self, points):
        points = np.ascontiguousarray(points, np.float32)
        out = np.zeros((len(points), 2 * self.n_lights + 1), np.float32)
        self.o._f("light_distribution")(self.h, ptr(points), len(points), ptr(out))
        return out


_cache = {}


def reference():
    """The compiled reference (oracle/_ref); None when it has not been built (no /root/reference)."""
    if "ref" not in _cache:
        _cache["ref"] = Oracle(REF_PATH, "ref_", "reference") if os.path.exists(REF_PATH) else None
    return _cache["ref"]


def port():
    """The C++ restatement (oracle/pb2_oracle.cpp)."""
    if "port" not in _cache:
        _cache["port"] = Oracle(PORT_PATH, "orc_", "port") if os.path.exists(PORT_PATH) else None
    return _cache["port"]


def best():
    return reference() or port()
