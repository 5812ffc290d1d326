"""pbrt_v3_b200 — H100-native path-tracing hot path behind pbrt-v3's plugin API.

Python is only the driver here (tests, bench.py, multi-GPU launch through torch.distributed):
everything below is a thin ctypes view of

* ``lib/libpb2.so`` — the C ABI of ``include/pb2.h`` (CUDA kernels, sm_90a) plus the C++ host-side
  scene front end (``csrc/host``: .pbrt parser, pbrt's Shape/Primitive/BVHAccel/Film/... classes,
  SAH BVH build), exported for scripting through the ``pb2h_*`` helpers of ``csrc/host/capi.cpp``.

There is no CPU implementation of the path in this package: without a CUDA device every compute
entry point fails with ``Pb2Error`` (``PB2_ERR_NO_DEVICE``).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PB2_LIB") or os.path.join(_HERE, "lib", "libpb2.so")   # PB2_LIB: A/B builds during tuning

c_float_p = C.POINTER(C.c_float)
c_int32_p = C.POINTER(C.c_int32)
c_int64_p = C.POINTER(C.c_int64)
c_uint8_p = C.POINTER(C.c_uint8)

PB2_OK, PB2_ERR_NO_DEVICE, PB2_ERR_CUDA, PB2_ERR_INVALID, PB2_ERR_UNSUPPORTED, PB2_ERR_NCCL = range(6)
PB2_PRIM_TRIANGLE, PB2_PRIM_SPHERE, PB2_PRIM_INSTANCE = 0, 1, 2
PB2_FILTER_BOX, PB2_FILTER_GAUSSIAN, PB2_FILTER_MITCHELL, PB2_FILTER_SINC, PB2_FILTER_TRIANGLE = 0, 1, 2, 3, 4
PB2_MAT_NONE, PB2_MAT_MATTE, PB2_MAT_PLASTIC, PB2_MAT_MIRROR, PB2_MAT_GLASS, PB2_MAT_SUBSTRATE, PB2_MAT_METAL, PB2_MAT_UBER = range(8)
PB2_ABI_VERSION = 10   # include/pb2.h (tests/test_abi.py checks that header, this mirror and the library agree)
PB2_LIGHTDIST_UNIFORM, PB2_LIGHTDIST_POWER, PB2_LIGHTDIST_SPATIAL = 0, 1, 2
PB2_LIGHT_AREA, PB2_LIGHT_POINT, PB2_LIGHT_SPOT, PB2_LIGHT_DISTANT, PB2_LIGHT_INFINITE = 0, 1, 2, 3, 4


class BvhNode(C.Structure):
    _fields_ = [("bmin", C.c_float * 3), ("bmax", C.c_float * 3), ("offset", C.c_int32),
                ("n_prims", C.c_uint16), ("axis", C.c_uint8), ("pad", C.c_uint8)]


class Mesh(C.Structure):
    _fields_ = [("first_tri", C.c_int32), ("n_tris", C.c_int32), ("first_vertex", C.c_int32),
                ("n_vertices", C.c_int32), ("has_n", C.c_int32), ("has_uv", C.c_int32), ("has_s", C.c_int32),
                ("reverse_orientation", C.c_int32), ("transform_swaps_handedness", C.c_int32),
                ("alpha_tex", C.c_int32), ("shadow_alpha_tex", C.c_int32), ("pad", C.c_int32)]


class Sphere(C.Structure):
    _fields_ = [("object_to_world", C.c_float * 16), ("world_to_object", C.c_float * 16),
                ("radius", C.c_float), ("z_min", C.c_float), ("z_max", C.c_float), ("theta_min", C.c_float),
                ("theta_max", C.c_float), ("phi_max", C.c_float), ("reverse_orientation", C.c_int32),
                ("transform_swaps_handedness", C.c_int32)]


class Material(C.Structure):
    _fields_ = [("type", C.c_int32), ("kd", C.c_float * 3), ("sigma", C.c_float), ("ks", C.c_float * 3),
                ("roughness", C.c_float), ("remap_roughness", C.c_int32), ("pad", C.c_int32 * 2),
                ("kr", C.c_float * 3), ("kt", C.c_float * 3), ("eta", C.c_float), ("uroughness", C.c_float),
                ("vroughness", C.c_float), ("opacity", C.c_float * 3), ("metal_eta", C.c_float * 3),
                ("metal_k", C.c_float * 3), ("pad3", C.c_int32 * 2), ("tex", C.c_int32 * 16)]


PB2_WRAP_REPEAT, PB2_WRAP_BLACK, PB2_WRAP_CLAMP = 0, 1, 2
PB2_SAMPLER_HALTON, PB2_SAMPLER_SOBOL = 0, 1
(PB2_TEX_KD, PB2_TEX_KS, PB2_TEX_KR, PB2_TEX_KT, PB2_TEX_OPACITY, PB2_TEX_SIGMA, PB2_TEX_ROUGHNESS, PB2_TEX_UROUGHNESS,
 PB2_TEX_VROUGHNESS, PB2_TEX_ETA, PB2_TEX_METAL_ETA, PB2_TEX_METAL_K, PB2_TEX_BUMP) = range(13)


class Texture(C.Structure):
    _fields_ = [("channels", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("wrap", C.c_int32),
                ("do_trilinear", C.c_int32), ("max_anisotropy", C.c_float), ("su", C.c_float), ("sv", C.c_float),
                ("du", C.c_float), ("dv", C.c_float), ("kind", C.c_int32), ("pad", C.c_int32), ("texels", c_float_p),
                ("child", C.c_int32 * 3), ("value", C.c_float * 3)]


PB2_TEXKIND_IMAGE, PB2_TEXKIND_CONSTANT, PB2_TEXKIND_SCALE, PB2_TEXKIND_MIX, PB2_TEXKIND_CHECKERBOARD, PB2_TEXKIND_UV = 0, 1, 2, 3, 4, 5


class Light(C.Structure):
    _fields_ = [("prim", C.c_int32), ("L", C.c_float * 3), ("two_sided", C.c_int32), ("area", C.c_float),
                ("type", C.c_int32), ("pad", C.c_int32)]


class DeltaLight(C.Structure):
    _fields_ = [("p", C.c_float * 3), ("total_width_deg", C.c_float), ("falloff_start_deg", C.c_float),
                ("world_radius", C.c_float), ("world_to_light", C.c_float * 9), ("pad", C.c_float),
                ("light_to_world", C.c_float * 9), ("env_tex", C.c_int32), ("pad2", C.c_float * 2)]


class Bvh(C.Structure):
    _fields_ = [("node_offset", C.c_int64), ("n_nodes", C.c_int64), ("prim_offset", C.c_int64), ("n_prims", C.c_int64)]


class Instance(C.Structure):
    _fields_ = [("instance_to_world", C.c_float * 16), ("world_to_instance", C.c_float * 16), ("bvh", C.c_int32),
                ("lone_prim", C.c_int32), ("pad", C.c_int32 * 2)]


class SceneDesc(C.Structure):
    _fields_ = [("n_vertices", C.c_int64), ("P", c_float_p), ("N", c_float_p), ("UV", c_float_p), ("S", c_float_p),
                ("n_tris", C.c_int64), ("tri_index", c_int32_p), ("tri_mesh", c_int32_p),
                ("n_meshes", C.c_int32), ("meshes", C.POINTER(Mesh)),
                ("n_spheres", C.c_int32), ("spheres", C.POINTER(Sphere)),
                ("n_prims", C.c_int64), ("prim_type", c_uint8_p), ("prim_index", c_int32_p),
                ("prim_material", c_int32_p), ("prim_light", c_int32_p),
                ("n_nodes", C.c_int64), ("nodes", C.POINTER(BvhNode)), ("bvh_prims", c_int32_p),
                ("n_materials", C.c_int32), ("materials", C.POINTER(Material)),
                ("n_lights", C.c_int32), ("lights", C.POINTER(Light)),
                ("light_strategy", C.c_int32), ("spatial_max_voxels", C.c_int32),
                ("n_instances", C.c_int32), ("n_bvhs", C.c_int32), ("instances", C.POINTER(Instance)),
                ("bvhs", C.POINTER(Bvh)), ("n_bvh_prims", C.c_int64), ("delta_lights", C.POINTER(DeltaLight)),
                ("n_textures", C.c_int32), ("pad_textures", C.c_int32), ("textures", C.POINTER(Texture))]


class Camera(C.Structure):
    _fields_ = [("camera_to_world", C.c_float * 16), ("world_to_camera", C.c_float * 16),
                ("screen_window", C.c_float * 4), ("fov", C.c_float), ("lens_radius", C.c_float),
                ("focal_distance", C.c_float), ("shutter_open", C.c_float), ("shutter_close", C.c_float),
                ("raster_to_camera", C.c_float * 16), ("dx_camera", C.c_float * 3), ("dy_camera", C.c_float * 3)]


class FilmDesc(C.Structure):
    _fields_ = [("full_resolution", C.c_int32 * 2), ("cropped_pixel_bounds", C.c_int32 * 4),
                ("filter_radius", C.c_float * 2), ("max_sample_luminance", C.c_float), ("scale", C.c_float),
                ("filter_type", C.c_int32), ("filter_param", C.c_float * 2), ("pad", C.c_int32)]


class PathParams(C.Structure):
    _fields_ = [("samples_per_pixel", C.c_int32), ("sample_at_pixel_center", C.c_int32), ("max_depth", C.c_int32),
                ("rr_threshold", C.c_float), ("pixel_bounds", C.c_int32 * 4), ("tile_rank", C.c_int32),
                ("tile_count", C.c_int32), ("flags", C.c_int32), ("sampler", C.c_int32)]


class Ray(C.Structure):
    _fields_ = [("o", C.c_float * 3), ("d", C.c_float * 3), ("t_max", C.c_float)]


class Hit(C.Structure):
    _fields_ = [("prim", C.c_int32), ("t", C.c_float), ("b", C.c_float * 3), ("p", C.c_float * 3),
                ("p_error", C.c_float * 3), ("n", C.c_float * 3), ("ns", C.c_float * 3), ("dpdu", C.c_float * 3),
                ("uv", C.c_float * 2)]


class WfHit(C.Structure):
    _fields_ = [("found", C.c_int32), ("leaf", C.c_int32), ("prim", C.c_int32), ("t", C.c_float), ("b", C.c_float * 3),
                ("listed", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("camera_rays", C.c_uint64), ("regular_rays", C.c_uint64), ("shadow_rays", C.c_uint64),
                ("node_visits", C.c_uint64), ("prim_tests", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("render_ms", C.c_double), ("h2d_ms", C.c_double), ("d2h_ms", C.c_double), ("trace_ms", C.c_double)]


RAY_DTYPE = np.dtype([("o", np.float32, 3), ("d", np.float32, 3), ("t_max", np.float32)])
HIT_DTYPE = np.dtype([("prim", np.int32), ("t", np.float32), ("b", np.float32, 3), ("p", np.float32, 3),
                      ("p_error", np.float32, 3), ("n", np.float32, 3), ("ns", np.float32, 3),
                      ("dpdu", np.float32, 3), ("uv", np.float32, 2)])
WFHIT_DTYPE = np.dtype([("found", np.int32), ("leaf", np.int32), ("prim", np.int32), ("t", np.float32), ("b", np.float32, 3),
                        ("listed", np.int32)])
PB2_FLAG_COUNT_TRAVERSAL, PB2_FLAG_LINEAR_NODES, PB2_FLAG_WIDE4, PB2_FLAG_PLAIN_TRACE, PB2_FLAG_SMALL_STACK, PB2_FLAG_LD128, PB2_FLAG_LEAF_TMA, PB2_FLAG_POOL = 1, 2, 4, 8, 16, 32, 64, 128
PB2_FLAG_CHAIN = 256
NODE_DTYPE = np.dtype([("bmin", np.float32, 3), ("bmax", np.float32, 3), ("offset", np.int32),
                       ("n_prims", np.uint16), ("axis", np.uint8), ("pad", np.uint8)])
assert WFHIT_DTYPE.itemsize == C.sizeof(WfHit)
assert RAY_DTYPE.itemsize == C.sizeof(Ray) and HIT_DTYPE.itemsize == C.sizeof(Hit) and NODE_DTYPE.itemsize == 32


class Pb2Error(RuntimeError):
    def __init__(self, code, message):
        super().__init__("pb2 status %d: %s" % (code, message))
        self.code = code


_lib = None


def lib():
    """Loads lib/libpb2.so (built in-tree by __graft_entry__.build()); fails loudly if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(the CUDA extension is required; there is no fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.pb2_last_error.restype = C.c_char_p
    L.pb2_scene_create.argtypes = [C.POINTER(SceneDesc), C.POINTER(vp)]
    L.pb2_scene_destroy.argtypes = [vp]
    L.pb2_intersect.argtypes = [vp, vp, C.c_int64, vp]
    L.pb2_intersect_p.argtypes = [vp, vp, C.c_int64, vp]
    L.pb2_trace_wavefront.argtypes = [vp, vp, vp, C.c_int64, C.c_int32, vp]
    L.pb2_work_items.argtypes = [C.POINTER(FilmDesc), C.POINTER(PathParams), C.c_int64, C.c_int64, vp, C.POINTER(C.c_int64)]
    L.pb2_init_devices.argtypes = [C.c_int, C.POINTER(C.c_int)]
    L.pb2_dist_unique_id.argtypes = [vp]
    L.pb2_dist_init.argtypes = [C.c_int, C.c_int, vp]
    L.pb2_dist_info.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pb2_host_alloc.argtypes = [C.c_size_t, C.POINTER(vp)]
    L.pb2_host_free.argtypes = [vp]
    L.pb2_render_path.argtypes = [vp, C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), vp, C.POINTER(Stats)]
    L.pb2_render_path_device.argtypes = [vp, C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), vp,
                                         C.c_int, vp, C.POINTER(Stats)]
    L.pb2_li_samples.argtypes = [vp, C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), vp, vp, C.c_int64, vp, vp]
    L.pb2_halton_samples.argtypes = [C.POINTER(FilmDesc), C.POINTER(PathParams), vp, vp, vp, C.c_int64, vp]
    L.pb2_light_distribution.argtypes = [vp, vp, C.c_int64, vp]
    L.pb2_sobol_samples_host.argtypes = [C.POINTER(FilmDesc), C.POINTER(PathParams), vp, vp, vp, C.c_int64, vp, vp]
    L.pb2_texture_pyramid.argtypes = [C.POINTER(Texture), C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), vp]
    L.pb2_texture_lookup.argtypes = [C.POINTER(Texture), C.c_int64, vp, vp, vp]
    L.pb2_env_distribution.argtypes = [C.POINTER(Texture), C.POINTER(C.c_int32), C.POINTER(C.c_int32), vp]
    L.pb2_texture_eval_host.argtypes = [C.POINTER(Texture), C.c_int32, C.c_int32, C.c_int64, vp, vp, vp]
    L.pb2_bsdf_eval_host.argtypes = [C.POINTER(Material), C.c_int64, vp, vp]
    L.pb2_camera_differentials_host.argtypes = [C.POINTER(Camera), C.POINTER(FilmDesc), C.POINTER(PathParams), C.c_int64, vp, vp]
    L.pb2_uv_differentials_host.argtypes = [C.c_int64, vp, vp]
    L.pb2h_parse_file.argtypes = [C.c_char_p, C.c_char_p]
    L.pb2h_parse_string.argtypes = [C.c_char_p]
    L.pb2h_synth_soup.argtypes = [C.c_int64, C.c_uint64, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p]
    L.pb2h_synth_instanced.argtypes = [C.c_int64, C.c_int, C.c_uint64, C.c_uint64, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int]
    L.pb2h_scene_desc.restype = C.POINTER(SceneDesc)
    L.pb2h_camera.restype = C.POINTER(Camera)
    L.pb2h_film.restype = C.POINTER(FilmDesc)
    L.pb2h_path_params.restype = C.POINTER(PathParams)
    L.pb2h_render.argtypes = [C.c_int, C.POINTER(Stats)]
    L.pb2h_image.restype = c_float_p
    L.pb2h_image.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pb2h_resolve_film.argtypes = [vp, vp]
    L.pb2h_device_scene.restype = vp
    L.pb2h_write_pfm.argtypes = [C.c_char_p, vp, C.c_int, C.c_int]
    L.pb2h_write_image.argtypes = [C.c_char_p, vp] + [C.c_int] * 6
    L.pb2h_read_image.argtypes = [C.c_char_p, vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pb2h_loop_subdivide.argtypes = [C.c_int, C.c_int, vp, C.c_int, vp, C.POINTER(C.c_int), C.POINTER(C.c_int), vp, vp, vp]
    L.pb2h_set_light_strategy.argtypes = [C.c_int]
    L.pb2h_scene_intersect.argtypes = [vp, vp, vp]
    _lib = L
    return L


def check(code):
    if code != PB2_OK:
        raise Pb2Error(code, lib().pb2_last_error().decode("utf-8", "replace"))


def ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


_initialised_device = None


def init(device=None):
    """pb2_init on this process's GPU (LOCAL_RANK under torchrun). Raises Pb2Error without a device."""
    global _initialised_device
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", os.environ.get("PB2_DEVICE", "0")))
    if _initialised_device == device:
        return
    check(lib().pb2_init(device))
    _initialised_device = device


def sobol_samples_host(film, params, pixel_xy, sample_num, dim, tables=False):
    """SobolSampler sample values computed on the host by the kernels' own source functions (pb2_sobol_samples_host)."""
    pixel_xy = np.ascontiguousarray(pixel_xy, np.int32)
    sample_num = np.ascontiguousarray(sample_num, np.int64)
    dim = np.ascontiguousarray(dim, np.int32)
    out = np.zeros(len(dim), np.float32)
    tab = np.zeros(104, np.uint64)
    check(lib().pb2_sobol_samples_host(film, params, ptr(pixel_xy), ptr(sample_num), ptr(dim), len(dim), ptr(out), ptr(tab)))
    return (out, tab) if tables else out


def texture_pyramid(texture, fn=None):
    """The levels of the MIP pyramid the library builds for one pb2_texture (host code, no device): list of (h, w, channels)
    arrays, finest first.  fn: the entry point (default pb2_texture_pyramid; the oracle passes its own)."""
    fn = fn or lib().pb2_texture_pyramid
    nl, w, h = C.c_int32(), C.c_int32(), C.c_int32()
    check(fn(C.byref(texture), 0, C.byref(nl), C.byref(w), C.byref(h), None))
    levels = []
    for lv in range(nl.value):
        check(fn(C.byref(texture), lv, C.byref(nl), C.byref(w), C.byref(h), None))
        a = np.zeros((h.value, w.value, texture.channels), np.float32)
        check(fn(C.byref(texture), lv, C.byref(nl), C.byref(w), C.byref(h), ptr(a)))
        levels.append(a)
    return levels


def bsdf_eval_host(material, frames, fn=None):
    """The BSDF of one pb2_material record at n shading frames (n, 17): n, ns, dpdu, wo, wi, u -> (n, 19): f, pdf, the non-specular
    sample (wi, f, pdf), the continuation sample (wi, f, pdf, flags); on the host by the shade kernel's own functions (or, with
    fn, by the oracle).  Layout: include/pb2.h, pb2_bsdf_eval_host."""
    fn = fn or lib().pb2_bsdf_eval_host
    frames = np.ascontiguousarray(frames, np.float32)
    out = np.zeros((len(frames), 19), np.float32)
    check(fn(C.byref(material), len(frames), ptr(frames), ptr(out)))
    return out


def texture_eval_host(textures, n_textures, tex_id, uv, duv, fn=None):
    """Texture::Evaluate of texture tex_id (0-based) of a description's texture array at points (u, v) with differentials
    (dudx, dvdx, dudy, dvdy), on the host by the kernels' own functions (or, with fn, by the oracle): (n, 3)."""
    fn = fn or lib().pb2_texture_eval_host
    uv = np.ascontiguousarray(uv, np.float32)
    duv = np.ascontiguousarray(duv, np.float32)
    out = np.zeros((len(uv), 3), np.float32)
    check(fn(textures, n_textures, tex_id, len(uv), ptr(uv), ptr(duv), ptr(out)))
    return out


def env_distribution(texture, fn=None):
    """The Distribution2D the library derives for an InfiniteAreaLight with this environment map (host code): (nu, nv, table)."""
    fn = fn or lib().pb2_env_distribution
    nu, nv = C.c_int32(), C.c_int32()
    check(fn(C.byref(texture), C.byref(nu), C.byref(nv), None))
    table = np.zeros(nv.value * (2 * nu.value + 2) + 2 * nv.value + 2, np.float32)
    check(fn(C.byref(texture), C.byref(nu), C.byref(nv), ptr(table)))
    return nu.value, nv.value, table


def read_image(path):
    """The host front end's ReadImage (PFM / PNG / TGA / OpenEXR): (h, w, 3) float32, row 0 at the top."""
    w, h = C.c_int(), C.c_int()
    if lib().pb2h_read_image(path.encode(), None, C.byref(w), C.byref(h)) != 0:
        raise RuntimeError("cannot read %s" % path)
    out = np.zeros((h.value, w.value, 3), np.float32)
    lib().pb2h_read_image(path.encode(), ptr(out), C.byref(w), C.byref(h))
    return out


def texture_lookup(texture, st, dst):
    """MIPMap::Lookup(st, dst0, dst1) on the device for a batch: st (n, 2), dst (n, 4) -> (n, 3)."""
    init()
    st = np.ascontiguousarray(st, np.float32)
    dst = np.ascontiguousarray(dst, np.float32)
    out = np.zeros((len(st), 3), np.float32)
    check(lib().pb2_texture_lookup(C.byref(texture), len(st), ptr(st), ptr(dst), ptr(out)))
    return out


class HostScene:
    """A scene held by the C++ host front end (one at a time: it mirrors pbrt's global API state)."""

    _generation = 0

    def __init__(self):
        self.L = lib()
        HostScene._generation += 1
        self._gen = HostScene._generation   # a later parse replaces the C++ side's scene: this object then refuses to be used

    def _current(self):
        if self._gen != HostScene._generation:
            raise RuntimeError("this HostScene was replaced by a later HostScene (the host front end holds one scene at a time)")

    @classmethod
    def from_file(cls, path, outfile=None):
        s = cls()
        if s.L.pb2h_parse_file(path.encode(), outfile.encode() if outfile else None) != 0:
            raise RuntimeError("could not parse %s" % path)
        return s

    @classmethod
    def from_string(cls, text):
        s = cls()
        if s.L.pb2h_parse_string(text.encode()) != 0:
            raise RuntimeError("could not parse scene text")
        return s

    @classmethod
    def soup(cls, n_tris, seed=1234, jitter=0.02, xres=1920, yres=1080, spp=64, maxdepth=8, light_strategy=None):
        """SURVEY.md §8d synthetic triangle soup (config 2 with the defaults and n_tris=1_000_000)."""
        s = cls()
        if s.L.pb2h_synth_soup(n_tris, seed, jitter, xres, yres, spp, maxdepth,
                               light_strategy.encode() if light_strategy else None) != 0:
            raise RuntimeError("could not build the synthetic scene")
        return s

    @classmethod
    def instanced_soup(cls, n_object_tris, grid=10, seed=4321, seed_instances=99, jitter=0.05, xres=1920, yres=1080, spp=128, maxdepth=5):
        """SURVEY.md §8d config 4: one soup object instanced grid x grid times (100 000 triangles x 100 with the defaults)."""
        s = cls()
        if s.L.pb2h_synth_instanced(n_object_tris, grid, seed, seed_instances, jitter, xres, yres, spp, maxdepth) != 0:
            raise RuntimeError("could not build the synthetic instanced scene")
        return s

    # flattened descriptions (host memory owned by the C++ side)
    @property
    def desc(self):
        self._current()
        p = self.L.pb2h_scene_desc()
        if not p:
            raise RuntimeError("scene could not be flattened (see stderr)")
        return p

    @property
    def camera(self):
        self._current()
        return self.L.pb2h_camera()

    @property
    def film(self):
        self._current()
        return self.L.pb2h_film()

    @property
    def params(self):
        return self.L.pb2h_path_params()

    def params_copy(self, **overrides):
        p = PathParams()
        C.memmove(C.byref(p), self.params, C.sizeof(PathParams))
        for k, v in overrides.items():
            setattr(p, k, v)
        return p

    def film_shape(self):
        b = self.film.contents.cropped_pixel_bounds
        return (b[3] - b[1], b[2] - b[0])

    def bvh_range(self, k=0):
        """(node_offset, n_nodes, prim_offset, n_prims) of BVH k: 0 = the scene BVH, k >= 1 = an instanced object's."""
        d = self.desc.contents
        if d.n_bvhs == 0:
            return 0, d.n_nodes, 0, d.n_prims
        b = d.bvhs[k]
        return b.node_offset, b.n_nodes, b.prim_offset, b.n_prims

    def nodes(self, k=0):
        d = self.desc.contents
        no, nn, _, _ = self.bvh_range(k)
        return np.ctypeslib.as_array(C.cast(d.nodes, C.POINTER(C.c_uint8)), shape=(d.n_nodes * 32,)).view(NODE_DTYPE)[no:no + nn].copy()

    def bvh_prims(self, k=0):
        d = self.desc.contents
        _, _, po, pn = self.bvh_range(k)
        total = d.n_bvh_prims if d.n_bvhs > 0 else d.n_prims
        return np.ctypeslib.as_array(d.bvh_prims, shape=(total,))[po:po + pn].copy()

    # device side
    def device_scene(self):
        init()
        h = self.L.pb2h_device_scene()
        if not h:
            raise Pb2Error(PB2_ERR_CUDA, "device scene could not be created: " + self.L.pb2_last_error().decode())
        return h

    def render(self, write_image=False):
        """Integrator::Render through the reference-shaped host API. Returns (rgb[h,w,3], Stats)."""
        init()
        st = Stats()
        rc = self.L.pb2h_render(1 if write_image else 0, C.byref(st))
        if rc != 0:
            raise Pb2Error(rc, "render failed: " + self.L.pb2_last_error().decode())
        w, h = C.c_int(), C.c_int()
        p = self.L.pb2h_image(C.byref(w), C.byref(h))
        img = np.ctypeslib.as_array(p, shape=(h.value, w.value, 3)).copy()
        return img, st

    def render_rgbw(self, params=None):
        """pb2_render_path with host buffers: returns (rgbw[h,w,4], Stats)."""
        dev = self.device_scene()
        h, w = self.film_shape()
        out = np.zeros((h, w, 4), np.float32)
        st = Stats()
        check(self.L.pb2_render_path(dev, self.camera, self.film, params if params is not None else self.params,
                                     ptr(out), C.byref(st)))
        return out, st

    def resolve(self, rgbw):
        """Film::MergeFilmTile + WriteImage arithmetic on an rgbw film. Returns rgb[h,w,3]."""
        h, w = self.film_shape()
        rgbw = np.ascontiguousarray(rgbw, np.float32)
        out = np.zeros((h, w, 3), np.float32)
        if self.L.pb2h_resolve_film(ptr(rgbw), ptr(out)) != 0:
            raise RuntimeError("resolve failed")
        return out

    def intersect(self, rays):
        dev = self.device_scene()
        rays = np.ascontiguousarray(rays, RAY_DTYPE)
        hits = np.zeros(len(rays), HIT_DTYPE)
        check(self.L.pb2_intersect(dev, ptr(rays), len(rays), ptr(hits)))
        return hits

    def intersect_p(self, rays):
        dev = self.device_scene()
        rays = np.ascontiguousarray(rays, RAY_DTYPE)
        occ = np.zeros(len(rays), np.uint8)
        check(self.L.pb2_intersect_p(dev, ptr(rays), len(rays), ptr(occ)))
        return occ

    def trace_wavefront(self, rays, any_hit=None, flags=0):
        """The render path's traversal kernel over a ray batch (pb2_trace_wavefront): raw (found, leaf, prim, t, b) records."""
        dev = self.device_scene()
        rays = np.ascontiguousarray(rays, RAY_DTYPE)
        out = np.zeros(len(rays), WFHIT_DTYPE)
        if any_hit is not None:
            any_hit = np.ascontiguousarray(any_hit, np.uint8)
        check(self.L.pb2_trace_wavefront(dev, ptr(rays), ptr(any_hit), len(rays), flags, ptr(out)))
        return out

    def textures(self):
        """The scene description's image textures (ctypes pb2_texture records; valid while this scene is the current one)."""
        d = self.desc.contents
        return [d.textures[i] for i in range(d.n_textures)]

    def li_samples(self, pixel_xy, sample_num, params=None):
        dev = self.device_scene()
        pixel_xy = np.ascontiguousarray(pixel_xy, np.int32)
        sample_num = np.ascontiguousarray(sample_num, np.int64)
        n = len(sample_num)
        rgb = np.zeros((n, 3), np.float32)
        pfilm = np.zeros((n, 2), np.float32)
        check(self.L.pb2_li_samples(dev, self.camera, self.film, params if params is not None else self.params,
                                    ptr(pixel_xy), ptr(sample_num), n, ptr(rgb), ptr(pfilm)))
        return rgb, pfilm

    def halton(self, pixel_xy, sample_num, dim):
        init()
        pixel_xy = np.ascontiguousarray(pixel_xy, np.int32)
        sample_num = np.ascontiguousarray(sample_num, np.int64)
        dim = np.ascontiguousarray(dim, np.int32)
        out = np.zeros(len(dim), np.float32)
        check(self.L.pb2_halton_samples(self.film, self.params, ptr(pixel_xy), ptr(sample_num), ptr(dim), len(dim), ptr(out)))
        return out

    def light_distribution(self, points):
        dev = self.device_scene()
        points = np.ascontiguousarray(points, np.float32)
        nl = self.desc.contents.n_lights
        out = np.zeros((len(points), 2 * nl + 1), np.float32)
        check(self.L.pb2_light_distribution(dev, ptr(points), len(points), ptr(out)))
        return out


def loop_subdivide(n_levels, indices, P):
    L = lib()
    indices = np.ascontiguousarray(indices, np.int32)
    P = np.ascontiguousarray(P, np.float32)
    nv, ni = C.c_int(), C.c_int()
    L.pb2h_loop_subdivide(n_levels, len(indices), ptr(indices), len(P), ptr(P), C.byref(nv), C.byref(ni), None, None, None)
    oP = np.zeros((nv.value, 3), np.float32)
    oN = np.zeros((nv.value, 3), np.float32)
    oI = np.zeros(ni.value, np.int32)
    L.pb2h_loop_subdivide(n_levels, len(indices), ptr(indices), len(P), ptr(P), C.byref(nv), C.byref(ni), ptr(oP), ptr(oN), ptr(oI))
    return oP, oN, oI
