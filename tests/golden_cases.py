"""Seeded inputs shared by tests/make_golden.py (which records the reference's outputs for them) and the tests."""
import os

import numpy as np

SOUP = dict(n_tris=2000, seed=77, jitter=0.05, xres=32, yres=18, spp=4, maxdepth=5)


def soup_scene(pb, **over):
    kw = dict(SOUP)
    kw.update(over)
    return pb.HostScene.soup(kw.pop("n_tris"), **kw)


def rays_for(pb, nodes, n, seed, shadow=False):
    rng = np.random.RandomState(seed)
    lo, hi = nodes["bmin"][0], nodes["bmax"][0]
    ext = hi - lo
    rays = np.zeros(n, pb.RAY_DTYPE)
    rays["o"] = rng.uniform(lo - 0.1 * ext, hi + 0.1 * ext, (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    # a few axis-parallel directions: zero components make invDir infinite (bvh.cpp:666)
    d[: n // 50, 0] = 0
    d[n // 50: n // 25, 1:] = 0
    if shadow:
        rays["d"] = (d * 0.3 * float(ext.max())).astype(np.float32)
        rays["t_max"] = np.float32(1 - 1e-4)
    else:
        rays["d"] = d
        rays["t_max"] = np.inf
    return rays


def sample_ids(xres, yres, spp, n, seed, max_dim=None):
    rng = np.random.RandomState(seed)
    pix = np.stack([rng.randint(0, xres, n), rng.randint(0, yres, n)], 1).astype(np.int32)
    sn = rng.randint(0, spp, n).astype(np.int64)
    if max_dim is None:
        return pix, sn
    return pix, sn, rng.randint(0, max_dim, n).astype(np.int32)


def points_for(nodes, n, seed):
    rng = np.random.RandomState(seed)
    lo, hi = nodes["bmin"][0], nodes["bmax"][0]
    ext = hi - lo
    return rng.uniform(lo - 0.05 * ext, hi + 0.05 * ext, (n, 3)).astype(np.float32)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def nan_canonical(hits):
    """Hit records with every NaN as 0x7fc00000: a NaN's sign and payload are not specified by IEEE 754 (x86 produces
    0xffc00000, the device 0x7fffffff), so only NaN-ness is compared.  The reference reports hits at t = NaN for rays from
    origins near 1e30 (the edge functions overflow); the device reports the same hits."""
    h = hits.copy()
    for f in h.dtype.names:
        if h.dtype[f].base == np.float32:
            h[f] = np.where(np.isnan(h[f]), np.float32(np.nan), h[f])
    return h


def row_digest(a):
    """A 32-bit digest of every bit of each row of an array of 4-byte values (FNV-1a over the words, folded): fixtures keep
    these instead of the values where the values would make them large."""
    w = np.ascontiguousarray(a).view(np.uint32).reshape(len(a), -1).astype(np.uint64)
    h = np.full(len(a), 0xcbf29ce484222325, np.uint64)
    for j in range(w.shape[1]):
        h = (h ^ w[:, j]) * np.uint64(0x100000001b3)
    return (h ^ (h >> np.uint64(32))).astype(np.uint32)


def pixel_digests(items, li, pfilm):
    """Per pixel of the work items (x, y, sample): the pixels in sorted order and a digest of every bit of every sample's
    sample number, L and pFilm there."""
    rows = np.concatenate([np.ascontiguousarray(items[:, 2:3], np.int32).view(np.float32), np.asarray(li, np.float32),
                           np.asarray(pfilm, np.float32)], 1)
    pixels, inv = np.unique(np.asarray(items[:, :2], np.int32), axis=0, return_inverse=True)
    acc = np.zeros(len(pixels), np.uint64)
    np.add.at(acc, inv.ravel(), row_digest(rows).astype(np.uint64))
    return pixels, (acc ^ (acc >> np.uint64(32))).astype(np.uint32)


# Reconstruction filters (src/filters/): the PixelFilter line and the Film line of each case; geometry, lights and
# materials are tests/scenes/materials.pbrt's.  Wider-than-a-pixel filters make neighbouring tiles overlap in the film,
# so the order in which tiles are merged shows in the last bit: these cases are rendered by ONE thread on the CPU side.
FILTER_CASES = {
    "gaussian": ('PixelFilter "gaussian"', ""),
    "mitchell": ('PixelFilter "mitchell"', ""),
    "sinc": ('PixelFilter "sinc"', ""),
    "triangle": ('PixelFilter "triangle"', ""),
    "gaussian_aniso_crop": ('PixelFilter "gaussian" "float xwidth" [1.25] "float ywidth" [3] "float alpha" [1]',
                            ' "float cropwindow" [.2 .9 .1 .7]'),
    "mitchell_sharp": ('PixelFilter "mitchell" "float B" [0] "float C" [.5] "float xwidth" [2.5] "float ywidth" [1.5]', ""),
    "sinc_narrow": ('PixelFilter "sinc" "float xwidth" [2] "float ywidth" [3] "float tau" [2]', ""),
    "box_wide": ('PixelFilter "box" "float xwidth" [1.5] "float ywidth" [.75]', ""),
}


def filter_scene_text(scene_dir, case):
    import os
    import re
    pixel_filter, film_extra = FILTER_CASES[case]
    text = open(os.path.join(scene_dir, "materials.pbrt")).read()
    text, n = re.subn(r'Film "image"[^\n]*', 'Film "image" "integer xresolution" [40] "integer yresolution" [28]' + film_extra, text)
    assert n == 1
    text, n = re.subn(r'"integer pixelsamples" \[8\]', '"integer pixelsamples" [4]', text)
    assert n == 1
    return text.replace("WorldBegin", pixel_filter + "\nWorldBegin", 1)


def scene_file_text(scene_dir, name):
    """tests/scenes/<name>.pbrt as one text that parses from anywhere: its Includes inlined, the files it reads (textures/)
    named by absolute path."""
    import re
    text = open(os.path.join(scene_dir, name + ".pbrt")).read()
    text = re.sub(r'Include "([^"]+)"', lambda m: open(os.path.join(scene_dir, m.group(1))).read(), text)
    return text.replace('"textures/', '"%s/' % os.path.join(scene_dir, "textures"))


def with_accelerator(text, split, maxprims, device_build=False):
    extra = ' "bool devicebuild" "true"' if device_build else ""
    return text.replace("WorldBegin", 'Accelerator "bvh" "string splitmethod" "%s" "integer maxnodeprims" [%d]%s\nWorldBegin' % (split, maxprims, extra), 1)


def random_mesh_scene_text(n_tris, seed):
    """A scene file with one trianglemesh of n_tris small random triangles inside the unit cube (for BVH-build tests)."""
    rng = np.random.RandomState(seed)
    c = rng.rand(n_tris, 1, 3).astype(np.float32)
    P = (c + 0.03 * (rng.rand(n_tris, 3, 3).astype(np.float32) - 0.5)).reshape(-1, 3)
    idx = np.arange(3 * n_tris)
    return ('LookAt .5 -2 .5  .5 .5 .5  0 0 1\nCamera "perspective" "float fov" 40\nSampler "halton" "integer pixelsamples" 1\n'
            'Film "image" "integer xresolution" 16 "integer yresolution" 16\nWorldBegin\n'
            'AttributeBegin\nAreaLightSource "diffuse" "rgb L" [5 5 5]\nShape "trianglemesh" "integer indices" [0 1 2] "point P" [0 0 2 1 0 2 0 1 2]\nAttributeEnd\n'
            'Shape "trianglemesh" "integer indices" [%s] "point P" [%s]\nWorldEnd\n'
            % (" ".join(map(str, idx)), " ".join("%.9g" % v for v in P.ravel())))


# The reference's own end-to-end tests of this path (src/tests/analytic_scenes.cpp:68-248, 270-296, 54-66): furnace scenes
# inside a unit sphere seen by a perspective camera at its centre, PathIntegrator depth 8, Halton 256 spp, 10 x 10 film;
# the average pixel value must be 1 within 0.02.
ANALYTIC_SCENES = {
    "one_point_light": 'LightSource "point" "rgb I" [3.14159265358979 3.14159265358979 3.14159265358979]\n'
                       'Material "matte" "rgb Kd" [.5 .5 .5]\n',
    "four_point_lights": 'LightSource "point" "rgb I" [.785398163397448 .785398163397448 .785398163397448]\n' * 4
                         + 'Material "matte" "rgb Kd" [.5 .5 .5]\n',
    "emissive_sphere": 'Material "matte" "rgb Kd" [.5 .5 .5]\nAreaLightSource "diffuse" "rgb L" [.5 .5 .5]\n',
    "uber_kd_kr": 'LightSource "point" "rgb I" [9.42477796076938 9.42477796076938 9.42477796076938]\n'
                  'Material "uber" "rgb Kd" [.25 .25 .25] "rgb Ks" [0 0 0] "rgb Kr" [.5 .5 .5] "rgb Kt" [0 0 0] "float roughness" 0 '
                  '"rgb opacity" [1 1 1] "float index" 1 "bool remaproughness" "false"\n',
}
ANALYTIC_EXPECTED, ANALYTIC_DELTA = 1.0, 0.02


def analytic_scene_text(case):
    return ('Camera "perspective" "float fov" 45 "float screenwindow" [-1 1 -1 1]\n'
            'Film "image" "integer xresolution" 10 "integer yresolution" 10 "float diagonal" 1\n'
            'Sampler "halton" "integer pixelsamples" 256\nIntegrator "path" "integer maxdepth" 8\nWorldBegin\n'
            + ANALYTIC_SCENES[case] + 'ReverseOrientation\nShape "sphere" "float radius" 1\nWorldEnd\n')


def sphere_reintersect_case(pb, i, partial):
    """One case of FullSphere.Reintersect / PartialSphere.Reintersect (src/tests/shapes.cpp:427-497): a sphere whose radius
    spans eight decades, rays from far-away origins (coordinates up to 1e8) into its bounding box.  Returns (scene text, rays)."""
    rng = np.random.RandomState(1000 + i)

    def pexp(e=8):   # shapes.cpp:18-25: +- 10^[-e, e]
        return (1 if rng.rand() < .5 else -1) * 10.0 ** rng.uniform(-e, e)
    radius = abs(pexp(4))
    zmin, zmax, phimax = -radius, radius, 360.0
    if partial:
        if rng.rand() >= .5:
            zmin = rng.uniform(-radius, radius)
        if rng.rand() >= .5:
            zmax = rng.uniform(-radius, radius)
        if rng.rand() >= .5:
            phimax = rng.rand() * 360
    text = ('Camera "perspective"\nFilm "image" "integer xresolution" [4] "integer yresolution" [4]\nWorldBegin\n'
            'Shape "sphere" "float radius" %.9g "float zmin" %.9g "float zmax" %.9g "float phimax" %.9g\nWorldEnd\n' % (radius, zmin, zmax, phimax))
    n = 400
    rays = np.zeros(n, pb.RAY_DTYPE)
    rays["o"] = np.array([[pexp() for _ in range(3)] for _ in range(n)], np.float32)
    lo, hi = np.float32(min(zmin, zmax)), np.float32(max(zmin, zmax))
    box_lo, box_hi = np.array([-radius, -radius, lo], np.float32), np.array([radius, radius, hi], np.float32)
    target = (box_lo + rng.rand(n, 3).astype(np.float32) * (box_hi - box_lo)).astype(np.float32)
    d = target - rays["o"]
    norm = rng.rand(n) < .5
    d[norm] /= np.linalg.norm(d[norm], axis=1, keepdims=True)
    rays["d"] = d
    rays["t_max"] = np.inf
    return text, rays, rng


def spawned_rays(pb, hits, rng):
    """Interaction::SpawnRay (interaction.h:64-67, OffsetRayOrigin geometry.h:1440-1454) in a random direction on the
    normal's side of every hit."""
    n = len(hits)
    w = rng.normal(size=(n, 3)).astype(np.float32)
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    nrm, p, pe = hits["n"], hits["p"], hits["p_error"]
    w[(w * nrm).sum(axis=1) < 0] *= -1                     # Faceforward(w, isect.n)
    d = (np.abs(nrm) * pe).sum(axis=1, keepdims=True)
    off = (d * nrm).astype(np.float32)
    po = (p + off).astype(np.float32)
    up, dn = off > 0, off < 0
    po[up] = np.nextafter(po[up], np.float32(np.inf))
    po[dn] = np.nextafter(po[dn], np.float32(-np.inf))
    rays = np.zeros(n, pb.RAY_DTYPE)
    rays["o"], rays["d"], rays["t_max"] = po, w, np.inf
    return rays


def texture_lookup_inputs(n, seed):
    """(st, dst) batches for MIPMap::Lookup: footprints from none at all to several times the whole image, isotropic
    and up to 60 : 1 anisotropic (beyond every maxanisotropy in use), one derivative zero, st outside [0, 1] for the wrap modes."""
    rs = np.random.RandomState(seed)
    st = rs.uniform(-0.6, 1.6, (n, 2)).astype(np.float32)
    kind = rs.randint(0, 7, n)
    size = np.exp(rs.uniform(np.log(1e-4), np.log(3.0), n))
    ang = rs.uniform(0, 2 * np.pi, n)
    ratio = np.exp(rs.uniform(0, np.log(60.0), n))
    d0 = np.stack([np.cos(ang), np.sin(ang)], 1) * size[:, None]
    ang1 = ang + np.where(kind == 5, rs.uniform(0, np.pi, n), np.pi / 2)   # kind 5: not orthogonal
    d1 = np.stack([np.cos(ang1), np.sin(ang1)], 1) * (size / ratio)[:, None]
    d1[kind == 1] = d0[kind == 1][:, ::-1] * [1, -1]    # isotropic
    d0[kind == 0] = 0                                  # no differentials at all
    d1[kind == 0] = 0
    d1[kind == 2] = 0                                  # one derivative zero
    swap = kind == 3                                   # the second one is the longer
    d0[swap], d1[swap] = d1[swap].copy(), d0[swap].copy()
    exact = kind == 6                                  # footprints of exactly 2^-k texture widths
    d0[exact] = np.stack([2.0 ** -rs.randint(0, 8, exact.sum()), np.zeros(exact.sum())], 1)
    d1[exact] = d0[exact][:, ::-1]
    return st, np.concatenate([d0, d1], 1).astype(np.float32)


TEXTURE_EVAL_SCENES = ("textured", "texcombine", "checker")


def texture_eval_inputs(n, seed):
    """(u, v) in [-1, 3]^2 and (dudx, dvdx, dudy, dvdy) from 1e-4 to 0.7, every fifth point without differentials."""
    rs = np.random.RandomState(seed)
    uv = rs.uniform(-1, 3, (n, 2)).astype(np.float32)
    mag = np.exp(rs.uniform(np.log(1e-4), np.log(.7), (n, 1)))
    duv = (rs.normal(size=(n, 4)) * mag).astype(np.float32)
    duv[::5] = 0
    return uv, duv

DIFFERENTIAL_SCENES = ("textured", "textured_lens", "bumpmap", "instances")


BSDF_SCENES = ("materials", "specular", "substrate", "metal", "uber", "roughglass")
BSDF_FRAMES = 1000   # shading frames per material record (the fixture stays under 1 MB)


def bsdf_frames(n, seed):
    """Random shading frames for BSDF evaluation: geometric normal, a shading normal near it (a third of them equal), a shading
    dpdu (a quarter of them not perpendicular to ns), wo and wi anywhere on the sphere, a 2D sample."""
    rs = np.random.RandomState(seed)

    def unit(v):
        return v / np.linalg.norm(v, axis=1, keepdims=True)
    nrm = unit(rs.normal(size=(n, 3)))
    ns = unit(nrm + 0.3 * rs.normal(size=(n, 3)))
    ns[::3] = nrm[::3]
    t = rs.normal(size=(n, 3))
    dpdu = (t - ns * (t * ns).sum(1, keepdims=True)) * rs.uniform(.2, 3, (n, 1))
    dpdu[::4] += 0.2 * ns[::4]
    wo, wi = unit(rs.normal(size=(n, 3))), unit(rs.normal(size=(n, 3)))
    return np.ascontiguousarray(np.concatenate([nrm, ns, dpdu, wo, wi, rs.uniform(0, 1, (n, 2))], 1), np.float32)


def lights_text(scene_dir, strategy):
    """tests/scenes/lights.pbrt under another light-sampling strategy ("spatial", "uniform")."""
    text = open(os.path.join(scene_dir, "lights.pbrt")).read()
    return text.replace('"string lightsamplestrategy" "power"', '"string lightsamplestrategy" "%s"' % strategy)


def awkward_textures(pb):
    """Random images of awkward sizes (1 x N, N x 1, primes, already a power of two) as pb2_texture records; the texel
    arrays are kept alive on the records."""
    import ctypes as C
    rs = np.random.RandomState(9)
    out = []
    for (w, h, ch, wrap) in [(1, 1, 1, 0), (1, 7, 3, 0), (5, 1, 1, 2), (13, 31, 3, 1), (16, 4, 1, 0), (33, 64, 3, 2), (100, 3, 1, 1)]:
        texels = rs.uniform(0, 2, (h, w, ch)).astype(np.float32)
        t = pb.Texture(channels=ch, width=w, height=h, wrap=wrap, do_trilinear=0, max_anisotropy=8.0, su=1, sv=1, du=0, dv=0,
                       texels=texels.ctypes.data_as(C.POINTER(C.c_float)))
        t._texels = texels
        out.append(t)
    return out


# the reference's scenes/killeroo-simple.pbrt and the file it includes, stored in tests/golden/killeroo_simple.npz
KILLEROO_FILES = {"scene": "killeroo-simple.pbrt", "geometry": os.path.join("geometry", "killeroo.pbrt")}


def killeroo_scene(directory, golden_dir):
    """Writes the stored killeroo-simple scene into `directory` (its Include is relative) and returns the scene file's path."""
    g = np.load(os.path.join(golden_dir, "killeroo_simple.npz"))
    for key, rel in KILLEROO_FILES.items():
        path = os.path.join(directory, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(g[key].tobytes())
    return os.path.join(directory, KILLEROO_FILES["scene"])


# ---------------------------------------------------------------------------------------------------------------------
# Edge scenes and rays for the trace kernels (tests/make_golden.py record_trace_edges, tests/test_gpu_trace_edges.py):
# geometry and rays where a traversal that is only nearly the reference's gives another answer - coincident primitives
# (the first one the reference's order reaches wins, `t < tMax` is strict), box planes shared by many nodes and flat boxes,
# origins on box planes, rays through box corners and triangle vertices, signed zeros and infinite 1 / d, t_max at a hit's t.
# ---------------------------------------------------------------------------------------------------------------------
EDGE_HEADER = ('LookAt %s  %s  0 0 1\nCamera "perspective" "float fov" 45\nSampler "halton" "integer pixelsamples" 4\n'
               'Integrator "path" "integer maxdepth" 3\nFilm "image" "integer xresolution" 32 "integer yresolution" 24\nWorldBegin\n'
               'AttributeBegin\nAreaLightSource "diffuse" "rgb L" [6 6 6]\n'
               'Shape "trianglemesh" "integer indices" [0 1 2 0 2 3] "point P" [%s]\nAttributeEnd\n')


def _fmt(v):
    return " ".join("%.9g" % x for x in np.asarray(v, np.float32).ravel())


def _mesh(P, I, material=None):
    m = 'Material "matte" "rgb Kd" [%s]\n' % material if material else ""
    return m + 'Shape "trianglemesh" "integer indices" [%s] "point P" [%s]\n' % (" ".join(str(int(i)) for i in np.ravel(I)), _fmt(P))


def _edge_header(eye, at, light_z, off=0.0):
    lo, hi = -1 + off, 4 + off
    light = [[lo, lo, light_z], [hi, lo, light_z], [hi, hi, light_z], [lo, hi, light_z]]
    return EDGE_HEADER % (_fmt(eye), _fmt(at), _fmt(light))


def _grid(n, rng, z_jitter, scale=1.0):
    """An n x n tessellated height field over [0, 3]^2 with shared vertices: (P, I)."""
    xs = np.linspace(0, 3, n + 1, dtype=np.float32)
    X, Y = np.meshgrid(xs, xs)
    Z = (1 + z_jitter * rng.uniform(-1, 1, X.shape)).astype(np.float32) * scale
    P = np.stack([X, Y, Z], -1).reshape(-1, 3)
    I = []
    for j in range(n):
        for i in range(n):
            a = j * (n + 1) + i
            I += [[a, a + 1, a + n + 2], [a, a + n + 2, a + n + 1]]
    return P, np.array(I, np.int32)


def edge_scene_text(name):
    rng = np.random.RandomState({"coincident": 1, "coincident_wide": 2, "axis_grid": 3, "axis_grid_far": 3, "fan": 4, "spheres": 5,
                                 "instances": 6}[name])
    floor = _mesh([[-2, -2, 0], [5, -2, 0], [5, 5, 0], [-2, 5, 0]], [[0, 1, 2], [0, 2, 3]], ".5 .5 .5")
    if name in ("coincident", "coincident_wide"):
        # a mesh, then copies of it: identical with another material, reversed winding, vertex order rotated
        P, I = _grid(8 if name == "coincident" else 4, rng, 0.2)
        text = _edge_header((1.5, -4, 4), (1.5, 1.5, 1), 4) + floor + _mesh(P, I, ".7 .2 .2") + _mesh(P, I, ".2 .7 .2")
        text += _mesh(P, I[:, ::-1], ".2 .2 .7") + _mesh(P, I[:, [1, 2, 0]], ".7 .7 .2")
        if name == "coincident_wide":
            # 18 more copies of three triangles: their centroid bounds are degenerate, so each ends in a leaf of 22 (> 16)
            for k in range(18):
                text += _mesh(P, I[[0, 7, 20]][:, [[0, 1, 2], [1, 2, 0], [2, 0, 1]][k % 3]], "%.2f .5 .5" % (0.1 + 0.04 * k))
        return text + "WorldEnd\n"
    if name in ("axis_grid", "axis_grid_far"):
        # unit cubes and axis-aligned quads on an integer lattice: node boxes share planes, quads make flat boxes
        off = 1e5 if name == "axis_grid_far" else 0.0
        cube_P = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]], np.float32)
        cube_I = np.array([[0, 2, 1], [0, 3, 2], [4, 5, 6], [4, 6, 7], [0, 1, 5], [0, 5, 4], [1, 2, 6], [1, 6, 5], [2, 3, 7], [2, 7, 6],
                           [3, 0, 4], [3, 4, 7]], np.int32)
        quad_I = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
        text = _edge_header((1.5 + off, -5 + off, 5), (1.5 + off, 1.5 + off, 1), 5, off)
        text += _mesh(np.float32([[-2, -2, 0], [5, -2, 0], [5, 5, 0], [-2, 5, 0]]) + np.float32([off, off, 0]), quad_I, ".5 .5 .5")
        cells = [(x, y, z) for x in range(4) for y in range(4) for z in range(3)]
        for k in rng.permutation(len(cells))[:22]:
            x, y, z = cells[k]
            text += _mesh(cube_P + np.float32([x + off, y + off, z]), cube_I, "%.2f .4 .6" % (0.2 + 0.02 * x))
        for k in range(24):
            axis, c = rng.randint(3), rng.randint(0, 4)
            a0, b0 = rng.randint(0, 3, 2)
            sa, sb = rng.randint(1, 3, 2)
            q = np.zeros((4, 3), np.float32)
            u, v = (axis + 1) % 3, (axis + 2) % 3
            q[:, axis] = c
            q[:, u] = [a0, a0 + sa, a0 + sa, a0]
            q[:, v] = [b0, b0, b0 + sb, b0 + sb]
            text += _mesh(q + np.float32([off, off, 0]), quad_I, ".6 .6 %.2f" % (0.1 + 0.03 * k))
        return text + "WorldEnd\n"
    if name == "fan":
        # a tessellated grid and triangle fans: many triangles share a vertex, rays go through shared vertices and edges
        P, I = _grid(12, rng, 0.0)
        text = _edge_header((1.5, -4, 4), (1.5, 1.5, 1), 4) + floor + _mesh(P, I, ".6 .3 .3")
        for k in range(6):
            c = np.float32([rng.uniform(0, 3), rng.uniform(0, 3), rng.uniform(1.5, 2.5)])
            m = 8 + 4 * k
            ang = np.linspace(0, 2 * np.pi, m, endpoint=False)
            r = rng.uniform(0.3, 0.7)
            ring = np.stack([c[0] + r * np.cos(ang), c[1] + r * np.sin(ang), c[2] + 0.2 * np.sin(3 * ang)], 1)
            FP = np.concatenate([c[None], ring]).astype(np.float32)
            FI = [[0, 1 + i, 1 + (i + 1) % m] for i in range(m)]
            text += _mesh(FP, FI, ".3 .6 .%d" % k)
        return text + "WorldEnd\n"
    if name == "spheres":
        text = _edge_header((1.5, -5, 4), (1.5, 1.5, 1), 5) + floor
        shapes = [(0.5, 0.5, 1, 'Shape "sphere" "float radius" .8'),
                  (2.5, 0.5, 1, 'Shape "sphere" "float radius" .8 "float phimax" 270'),
                  (0.5, 2.5, 1, 'Shape "sphere" "float radius" .8 "float zmin" -.5 "float zmax" .6'),
                  (2.5, 2.5, 1, 'Shape "sphere" "float radius" .8 "float zmin" -.7 "float zmax" .3 "float phimax" 200'),
                  (1.5, 1.5, 2, 'Shape "sphere" "float radius" .6'),
                  (1.5, 1.5, 2, 'Shape "sphere" "float radius" .6')]   # two coincident spheres
        for k, (x, y, z, s) in enumerate(shapes):
            text += 'AttributeBegin\nTranslate %g %g %g\nMaterial "matte" "rgb Kd" [.%d .5 .5]\n%s\nAttributeEnd\n' % (x, y, z, k + 1, s)
        return text + "WorldEnd\n"
    if name == "instances":
        P, I = _grid(3, rng, 0.3, 0.5)
        text = _edge_header((1.5, -5, 4), (1.5, 1.5, 1), 5) + floor
        text += 'ObjectBegin "patch"\n' + _mesh(P * np.float32(0.5), I, ".6 .4 .2") + 'Shape "sphere" "float radius" .2\nObjectEnd\n'
        for tr in ("Translate 0 0 .5", "Translate 0 0 .5", "Translate 3 0 .5\nScale -1 1 1", "Translate 1 1.5 1\nRotate 30 0 0 1"):
            text += "AttributeBegin\n%s\nObjectInstance \"patch\"\nAttributeEnd\n" % tr
        return text + "WorldEnd\n"
    raise KeyError(name)


# name -> maxnodeprims of the SAH build
EDGE_SCENES = {"coincident": 4, "coincident_wide": 4, "axis_grid": 4, "axis_grid_far": 4, "fan": 4, "spheres": 4, "instances": 4}
SHADOW_EPSILON = np.float32(0.0001)
SLAB_SCALE = np.float32(1) + np.float32(2) * ((np.float32(3) * np.float32(2.0 ** -24)) / (np.float32(1) - np.float32(3) * np.float32(2.0 ** -24)))


def edge_scene(pb, name):
    return pb.HostScene.from_string(with_accelerator(edge_scene_text(name), "sah", EDGE_SCENES[name]))


def slab_events(o, d, bmin, bmax, t_max):
    """Bounds3::IntersectP (geometry.h:1412-1438) in float32 without FMA for rays (n, 3) against boxes (m, 3), (n, m) each:
    the verdict, and whether the test met an exact equality - an entry parameter equal to the exit parameter it is compared
    with, or the origin on one of the box's planes (slab value 0 * inf = NaN for axis-parallel rays)."""
    f = np.float32
    with np.errstate(all="ignore"):
        inv = (f(1) / d.astype(f))[:, None, :]
        neg = inv < 0
        o = o.astype(f)[:, None, :]
        near = np.where(neg, bmax[None], bmin[None]).astype(f)
        far = np.where(neg, bmin[None], bmax[None]).astype(f)
        dn, df = (near - o).astype(f), (far - o).astype(f)
        t0 = (dn * inv).astype(f)
        t1 = ((df * inv).astype(f) * SLAB_SCALE).astype(f)
        on_plane = ((dn == 0) | (df == 0)).any(-1)
        tmin, tmax = t0[..., 0], t1[..., 0]
        eq = (tmin == t1[..., 1]) | (t0[..., 1] == tmax)
        ok = ~((tmin > t1[..., 1]) | (t0[..., 1] > tmax))
        tmin = np.where(t0[..., 1] > tmin, t0[..., 1], tmin)
        tmax = np.where(t1[..., 1] < tmax, t1[..., 1], tmax)
        eq |= (tmin == t1[..., 2]) | (t0[..., 2] == tmax)
        ok &= ~((tmin > t1[..., 2]) | (t0[..., 2] > tmax))
        tmin = np.where(t0[..., 2] > tmin, t0[..., 2], tmin)
        tmax = np.where(t1[..., 2] < tmax, t1[..., 2], tmax)
        ok &= (tmin < np.asarray(t_max, f)[:, None]) & (tmax > 0)
    return ok, eq | on_plane


def reached_box_equalities(nodes, rays, t_final):
    """Per ray: some box test of the reference's traversal met an exact equality (slab_events).  The boxes counted are the
    root's and those of children of nodes the ray passes with its final tMax: every one of them the reference tests."""
    ok, eq = slab_events(rays["o"], rays["d"], nodes["bmin"], nodes["bmax"], t_final)
    parent = np.full(len(nodes), -1)
    interior = np.flatnonzero(nodes["n_prims"] == 0)
    parent[interior + 1] = interior
    parent[nodes["offset"][interior]] = interior
    reached = np.ones_like(ok)
    reached[:, 1:] = ok[:, parent[1:]]
    return (eq & reached).any(1)


def slow_rays(rays):
    """Rays whose origin or 1 / d is not finite: the kernels test their boxes with the reference's exact sequence."""
    with np.errstate(divide="ignore", over="ignore"):
        return ~(np.isfinite(np.float32(1) / rays["d"]).all(1) & np.isfinite(rays["o"]).all(1))


def _unit(v):
    return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(np.float32)


def edge_rays(pb, hs, closest, n_per_family=200, seed=0):
    """Path rays and shadow rays of the edge families for a scene (closest: Scene::Intersect of the reference, for the
    t_max family and the shadow segments).  Returns (rays, shadow rays, family of each ray)."""
    rng = np.random.RandomState(seed)
    f = np.float32
    nodes = hs.nodes()
    lo, hi = nodes["bmin"][0], nodes["bmax"][0]
    ext = (hi - lo).astype(f)
    d = hs.desc.contents
    tri_type = np.ctypeslib.as_array(d.prim_type, shape=(d.n_prims,))
    P = np.ctypeslib.as_array(d.P, shape=(d.n_vertices, 3)).copy() if d.n_vertices else np.zeros((0, 3), f)
    TI = np.ctypeslib.as_array(d.tri_index, shape=(d.n_tris, 3)).copy() if d.n_tris else np.zeros((0, 3), np.int32)
    n = n_per_family

    def inside(k, margin=0.1):
        return rng.uniform(lo - margin * ext, hi + margin * ext, (k, 3)).astype(f)

    def aim(o, target):
        with np.errstate(all="ignore"):
            return (target.astype(f) - o.astype(f)).astype(f)

    fams = []
    # 1. origins with one or two coordinates exactly on a node's bmin / bmax plane
    k = rng.randint(0, len(nodes), n)
    o = inside(n)
    for j in range(n):
        for ax in rng.choice(3, 1 + (j % 2), replace=False):
            o[j, ax] = (nodes["bmin"] if rng.rand() < .5 else nodes["bmax"])[k[j], ax]
    dd = _unit(rng.normal(size=(n, 3)))
    half = n // 2
    dd[:half] = aim(o[:half], inside(half, 0.0))
    fams.append(("box_planes", o, dd))
    # 2. +0 / -0 components, exactly axis-parallel, 1e-30 components (finite 1 / d, overflowing products), denormals
    o = inside(n)
    dd = _unit(aim(o, inside(n, 0.0)))
    kind = np.arange(n) % 6
    for j in range(n):
        ax = rng.randint(3)
        if kind[j] == 0:
            dd[j, ax] = f(0.0)
        elif kind[j] == 1:
            dd[j, ax] = f(-0.0)
        elif kind[j] == 2:
            s = f(1.0) if rng.rand() < .5 else f(-1.0)
            dd[j] = f(-0.0) if rng.rand() < .5 else f(0.0)
            dd[j, ax] = s
        elif kind[j] == 3:
            dd[j, ax] = f(1e-30) * (1 if rng.rand() < .5 else -1)
        elif kind[j] == 4:
            dd[j, ax] = f(1e-40) * (1 if rng.rand() < .5 else -1)
    fams.append(("directions", o, dd))
    # 3. aimed at node-box corners and edge points, nudged by ulps until an entry parameter EQUALS an exit parameter
    k = rng.randint(0, len(nodes), n)
    corner_sel = rng.randint(0, 2, (n, 3))
    tgt = np.where(corner_sel == 0, nodes["bmin"][k], nodes["bmax"][k]).astype(f)
    edge = np.arange(n) % 2 == 1
    ax = rng.randint(0, 3, n)
    mid = ((nodes["bmin"][k] + nodes["bmax"][k]) * f(0.5)).astype(f)
    tgt[edge, ax[edge]] = mid[edge, ax[edge]]
    o = (tgt + _unit(rng.normal(size=(n, 3))) * ext.max() * f(0.6)).astype(f)
    dd = aim(o, tgt)
    best = dd.copy()
    for j in range(n):
        bmin, bmax = nodes["bmin"][k[j]][None], nodes["bmax"][k[j]][None]
        cand = np.repeat(dd[j][None], 3 * 33, 0)
        steps = np.tile(np.arange(-16, 17), 3)
        axes = np.repeat(np.arange(3), 33)
        vals = cand[np.arange(len(cand)), axes]
        for s in range(len(cand)):
            v = vals[s]
            for _ in range(abs(steps[s])):
                v = np.nextafter(v, f(np.inf) if steps[s] > 0 else f(-np.inf))
            cand[s, axes[s]] = v
        ok, eq = slab_events(np.repeat(o[j][None], len(cand), 0), cand, bmin, bmax, np.full(len(cand), np.inf, f))
        hitq = np.flatnonzero(eq[:, 0] & ok[:, 0])
        if len(hitq):
            best[j] = cand[hitq[np.argmin(np.abs(steps[hitq]))]]
    fams.append(("corners", o, best))
    # 4. aimed at triangle vertices and at float midpoints of triangle edges
    if len(TI):
        t = rng.randint(0, len(TI), n)
        v = rng.randint(0, 3, n)
        tgt = P[TI[t, v]].astype(f)
        m = np.arange(n) % 2 == 1
        tgt[m] = ((P[TI[t, v]][m] + P[TI[t, (v + 1) % 3]][m]) * f(0.5)).astype(f)
        o = (tgt + _unit(rng.normal(size=(n, 3))) * ext.max() * f(0.5)).astype(f)
        fams.append(("vertices", o, aim(o, tgt)))
    # 5. t_max at a reference hit's t, one ulp either side of it, +0, -0, negative
    o = inside(n, 0.0)
    dd = _unit(aim(o, inside(n, 0.0)))
    fams.append(("tmax", o, dd))
    # 6. non-finite origins, and far origins (|o| ~ 1e30) aimed at the scene
    o = inside(n)
    dd = _unit(aim(o, inside(n, 0.0)))
    m = np.arange(n) % 2 == 0
    o[m, rng.randint(0, 3, m.sum())] = np.where(rng.rand(m.sum()) < .5, f(np.inf), f(-np.inf))
    far = ~m
    w = _unit(rng.normal(size=(far.sum(), 3)))
    c = ((lo + hi) * f(0.5)).astype(f)
    o[far] = (c + w * f(1e30)).astype(f)
    dd[far] = -w
    fams.append(("nonfinite", o, dd))

    names = [nm for nm, _, _ in fams]
    fam = np.concatenate([np.full(len(a), i, np.int32) for i, (_, a, _) in enumerate(fams)])
    rays = np.zeros(len(fam), pb.RAY_DTYPE)
    rays["o"] = np.concatenate([a for _, a, _ in fams])
    rays["d"] = np.concatenate([b for _, _, b in fams])
    rays["t_max"] = np.inf
    tm = fam == names.index("tmax")
    h = closest(rays)
    t = h["t"][tm]
    choice = np.arange(tm.sum()) % 6
    with np.errstate(all="ignore"):
        tmax = np.select([choice == 0, choice == 1, choice == 2, choice == 3, choice == 4],
                         [t, np.nextafter(t, f(np.inf)), np.nextafter(t, f(-np.inf)), f(0.0), f(-0.0)], f(-1.0)).astype(f)
    tmax[(h["prim"][tm] < 0) & (choice < 3)] = np.inf
    rays["t_max"][tm] = tmax
    h = closest(rays)
    # shadow rays: the same origins, segments that end exactly at the reference's hit point (or far beyond a miss)
    srays = rays.copy()
    srays["t_max"] = f(1) - SHADOW_EPSILON
    hit = h["prim"] >= 0
    with np.errstate(all="ignore"):
        srays["d"][hit] = (h["p"][hit] - rays["o"][hit]).astype(f)
        srays["d"][~hit] = (rays["d"][~hit] * ext.max() * f(2)).astype(f)
    return rays, srays, fam, names


def coincident_prims(hs):
    """Per scene primitive: another primitive covers exactly the same triangle (same three vertex positions in any order)
    or is the same sphere."""
    d = hs.desc.contents
    ptype = np.ctypeslib.as_array(d.prim_type, shape=(d.n_prims,))
    pidx = np.ctypeslib.as_array(d.prim_index, shape=(d.n_prims,))
    out = np.zeros(d.n_prims, bool)
    keys = {}
    P = np.ctypeslib.as_array(d.P, shape=(d.n_vertices, 3)) if d.n_vertices else None
    TI = np.ctypeslib.as_array(d.tri_index, shape=(d.n_tris, 3)) if d.n_tris else None
    for i in range(d.n_prims):
        if ptype[i] == 0:
            key = (0,) + tuple(sorted(P[TI[pidx[i]]].astype(np.float32).tobytes()[12 * j:12 * j + 12] for j in range(3)))
        elif ptype[i] == 1:
            s = d.spheres[pidx[i]]
            key = (1, bytes(s))
        else:
            continue
        keys.setdefault(key, []).append(i)
    for v in keys.values():
        if len(v) > 1:
            out[v] = True
    return out


def edge_coverage(hs, nodes, rays, hits):
    """What the edge rays of a scene reach (floors on these keep the fixture from being weakened quietly)."""
    prim = hits["prim"]
    coinc = coincident_prims(hs)
    on_coincident = (prim >= 0) & coinc[np.clip(prim, 0, len(coinc) - 1)]
    t_final = np.where(prim >= 0, hits["t"], rays["t_max"]).astype(np.float32)
    return {"coincident_hits": int(on_coincident.sum()),
            "box_equalities": int(reached_box_equalities(nodes, rays, t_final).sum()),
            "negative_zero": int((np.signbit(rays["d"]) & (rays["d"] == 0)).any(1).sum()),
            "slow": int(slow_rays(rays).sum()),
            "hits": int((prim >= 0).sum())}
