"""The trace kernels on the rays where a traversal that is only nearly the reference's gives another answer: exact ties of
coincident primitives, origins on box planes, entry parameters equal to exit parameters at box corners, rays through
triangle vertices, +-0 / 1e-30 / denormal direction components, t_max at a hit's t and one ulp either side, non-finite
and far origins (tests/golden_cases.py edge_scene / edge_rays).  Every result is compared BIT FOR BIT with what the
compiled reference recorded in device-math mode (tests/golden/trace_edges.npz, tests/make_golden.py record_trace_edges):
pb2_intersect / pb2_intersect_p, and every kernel variant of the render path through check_wavefront_records, with three
batch compositions - finite rays only (every box test of the record kernels takes slabTestPairFast), finite rays with a
ray of non-finite 1 / d among every four (nearly every warp takes the exact compare sequence), all rays."""
import os
import subprocess
import sys

import numpy as np
import pytest

import golden_cases as gc
from conftest import GOLDEN, ROOT
from test_gpu_exact_parity import hit_rows
from test_gpu_parity import check_wavefront_records
from test_oracle import same_bvh

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def g():
    z = np.load(os.path.join(GOLDEN, "trace_edges.npz"))
    return {k: z[k] for k in z.files}


def checked_hits(pb, g, name):
    """The scene, and pb2_intersect's hits of the edge rays after checking every field against the reference's bits (NaNs
    compared as NaNs: golden_cases.nan_canonical)."""
    hs = gc.edge_scene(pb, name)
    assert same_bvh(hs.nodes(), g[name + ":nodes"])
    hits = hs.intersect(g[name + ":rays"])
    assert np.array_equal(hits["prim"], g[name + ":prim"])
    want = gc.nan_canonical(np.rec.fromarrays([g[name + ":t"]], names="t"))["t"]
    assert np.array_equal(gc.bits(gc.nan_canonical(hits)["t"]), gc.bits(want))
    bad = np.flatnonzero(gc.row_digest(hit_rows(gc.nan_canonical(hits))) != g[name + ":digest"])
    assert len(bad) == 0, "%d of %d hit records differ in some field (first rays %s)" % (len(bad), len(hits), bad[:10].tolist())
    return hs, hits


@pytest.mark.parametrize("name", list(gc.EDGE_SCENES))
def test_intersect_is_the_reference_bits_on_edge_rays(pb, g, name):
    hs, _ = checked_hits(pb, g, name)
    assert np.array_equal(hs.intersect_p(g[name + ":srays"]), g[name + ":occluded"])


def interleaved(rays, slow):
    """Indices: the finite rays in order, after every three of them one of the slow rays (cycled through)."""
    fin, slo = np.flatnonzero(~slow), np.flatnonzero(slow)
    out = []
    for i in range(0, len(fin), 3):
        out += list(fin[i:i + 3]) + [slo[(i // 3) % len(slo)]]
    return np.array(out)


@pytest.mark.parametrize("batch", ["finite", "interleaved", "all"])
@pytest.mark.parametrize("name", list(gc.EDGE_SCENES))
def test_wavefront_kernels_on_edge_rays(pb, g, name, batch):
    """Found flag, primitive, t and barycentrics of every kernel variant equal pb2_intersect's (checked above against the
    reference), any-hits equal the reference's, path and shadow rays alone and mixed in the same warps."""
    hs, hits = checked_hits(pb, g, name)
    rays, srays, occ = g[name + ":rays"], g[name + ":srays"], g[name + ":occluded"]
    slow, sslow = gc.slow_rays(rays), gc.slow_rays(srays)
    if batch == "finite":
        i, j = np.flatnonzero(~slow), np.flatnonzero(~sslow)
    elif batch == "interleaved":
        i, j = interleaved(rays, slow), interleaved(srays, sslow)
        assert gc.slow_rays(rays[i])[3::4].all()
    else:
        i, j = np.arange(len(rays)), np.arange(len(srays))
    check_wavefront_records(pb, hs, rays[i], srays[j], hits[i], occ[j])


KERNEL_PROBE = r'''
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import numpy as np
import golden_cases as gc
import pbrt_v3_b200 as pb
from test_gpu_parity import wf_kernels
z = np.load(sys.argv[4])
hs = gc.edge_scene(pb, sys.argv[3])
for flags in wf_kernels(pb).values():
    hs.trace_wavefront(z[sys.argv[3] + ":rays"][:64], flags=flags)
print("probe ok")
'''


@pytest.mark.parametrize("name,kernel", [("coincident_wide", "k_wf_trace:"), ("coincident", "k_wf_trace_w<2>:")])
def test_leaves_beyond_sixteen_primitives_take_the_linear_node_kernel(pb, tmp_path, name, kernel):
    """A degenerate-centroid leaf of more than 16 primitives does not fit the two- and four-child records: every variant
    of the render path then traces the scene with k_wf_trace over the 32-B LinearBVHNode array (and the edge tests above
    check that kernel's hits).  The library names the kernel it selects under PB2_VERBOSE (read once per process)."""
    script = tmp_path / "probe.py"
    script.write_text(KERNEL_PROBE)
    env = dict(os.environ, PB2_VERBOSE="1")
    res = subprocess.run([sys.executable, str(script), ROOT, TESTS, name, os.path.join(GOLDEN, "trace_edges.npz")], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, timeout=600, cwd=ROOT, env=env)
    assert res.returncode == 0 and "probe ok" in res.stdout, res.stdout[-4000:]
    selected = [line.split("trace kernel ")[1].split(" ")[0] for line in res.stdout.splitlines() if "pb2: trace kernel " in line]
    plain = ("k_wf_trace_plain",)
    assert selected and kernel in selected, selected
    if name == "coincident_wide":
        assert all(k == "k_wf_trace:" or k.startswith(plain) for k in selected), selected
