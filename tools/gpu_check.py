"""Developer script (runs on a GPU machine): CUDA path vs the CPU checker.

Prints one line per check; tests/ holds the asserted versions of the same comparisons.
usage: python tools/gpu_check.py [n_tris | scene.pbrt] [--perf]
"""
import sys
import time

import numpy as np

sys.path.insert(0, ".")
import pbrt_v3_b200 as pb  # noqa: E402
from oracle import pyoracle  # noqa: E402


def random_rays(n, seed=1, lo=(-1.5, -1.5, -1.5), hi=(1.5, 1.5, 1.5)):
    rng = np.random.RandomState(seed)
    rays = np.zeros(n, pb.RAY_DTYPE)
    o = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays["o"] = o
    rays["d"] = d.astype(np.float32)
    rays["t_max"] = np.inf
    return rays


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def main():
    n_tris = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 20000
    ref = pyoracle.best()
    print("oracle kind:", ref.kind)
    scene_file = [a for a in sys.argv[1:] if a.endswith(".pbrt")]
    if scene_file:
        hs = pb.HostScene.from_file(scene_file[0])
    else:
        hs = pb.HostScene.soup(n_tris, xres=96, yres=54, spp=8)
    xres, yres = hs.film.contents.full_resolution[0], hs.film.contents.full_resolution[1]
    spp = hs.params.contents.samples_per_pixel
    rs = ref.scene(hs)
    nodes = hs.nodes()
    lo, hi = nodes["bmin"][0], nodes["bmax"][0]
    ext = hi - lo
    lo, hi = lo - 0.1 * ext, hi + 0.1 * ext

    rays = random_rays(20000, 1, lo, hi)
    t0 = time.time()
    g = hs.intersect(rays)
    print("gpu intersect %.2fs" % (time.time() - t0))
    r = rs.intersect(rays)
    same_prim = g["prim"] == r["prim"]
    hit = r["prim"] >= 0
    print("intersect: prim equal %d/%d, hits %d" % (same_prim.sum(), len(rays), hit.sum()))
    both = same_prim & hit
    for f in ("t", "p", "p_error", "n", "ns", "dpdu", "uv"):
        eq = bits(g[f][both]) == bits(r[f][both])
        close = np.isclose(g[f][both], r[f][both], rtol=1e-5, atol=1e-6)
        print("  %-8s bit-equal %d/%d (close %d)" % (f, eq.all(axis=-1).sum() if eq.ndim > 1 else eq.sum(), both.sum(),
                                                    close.all(axis=-1).sum() if close.ndim > 1 else close.sum()))
    rays2 = random_rays(20000, 2, lo, hi)
    rays2["d"] *= 0.7 * float(ext.max()) / 3
    rays2["t_max"] = 1 - 1e-4
    go, ro = hs.intersect_p(rays2), rs.intersect_p(rays2)
    print("intersect_p: equal %d/%d, occluded %d" % ((go == ro).sum(), len(go), ro.sum()))

    rng = np.random.RandomState(3)
    n = 20000
    pix = np.stack([rng.randint(0, xres, n), rng.randint(0, yres, n)], 1).astype(np.int32)
    sn = rng.randint(0, spp, n).astype(np.int64)
    dim = rng.randint(0, 150, n).astype(np.int32)
    gh, rh = hs.halton(pix, sn, dim), ref.halton(hs.film, hs.params, pix, sn, dim)
    print("halton: bit-equal %d/%d" % ((bits(gh) == bits(rh)).sum(), n))

    pts = rng.uniform(lo, hi, (2000, 3)).astype(np.float32)
    gl, rl = hs.light_distribution(pts), rs.light_distribution(pts)
    print("light distribution: bit-equal rows %d/%d, max abs diff %.3g" % ((bits(gl) == bits(rl)).all(axis=1).sum(), len(pts), np.abs(gl - rl).max()))

    gL, gp = hs.li_samples(pix, sn)
    rL, rp = rs.li_samples(pix, sn)
    err = np.abs(gL - rL).max(axis=1) / np.maximum(1, np.abs(rL).max(axis=1))
    print("li: pfilm bit-equal %d/%d; |dL| <= 1e-4 rel: %d/%d; bit-equal %d; max rel err %.3g; mean ref L %.4f mean gpu L %.4f"
          % ((bits(gp) == bits(rp)).all(axis=1).sum(), n, (err <= 1e-4).sum(), n, (bits(gL) == bits(rL)).all(axis=1).sum(), err.max(), rL.mean(), gL.mean()))
    for i in np.where(err > 1e-4)[0][:5]:
        print("   sample", pix[i], sn[i], "gpu", gL[i], "ref", rL[i])

    img_g, st = hs.render()
    img_r, secs, st_r = rs.render(n_threads=0)
    rel = np.abs(img_g - img_r) / np.maximum(np.abs(img_r), 1e-3)
    print("image: gpu %.1f ms, ref %.2f s; rays gpu %d/%d/%d ref %d/%d/%d" % (st.render_ms, secs, st.camera_rays, st.regular_rays, st.shadow_rays, st_r.camera_rays, st_r.regular_rays, st_r.shadow_rays))
    print("image: mean gpu %.5f ref %.5f; pixels within 1%%: %.4f; mean rel err %.3g; max abs diff %.3g"
          % (img_g.mean(), img_r.mean(), (rel.max(axis=2) <= 0.01).mean(), rel.mean(), np.abs(img_g - img_r).max()))


if __name__ == "__main__":
    main()
