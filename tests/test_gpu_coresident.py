"""Several wavefront pipelines sharing the SMs: the trace grid's size changes no result.

With several pipelines and the class-0 shade step renderWavefront sizes the persistent trace grid so that one
list-kernel block fits beside it on every SM and gives every kernel of the frame one shared-memory carve-out.  A launch may then be only partly resident,
and the pipelines' kernels interleave in new ways.  None of that may change a path's radiance or a ray count.  Every
case of the schedule tests renders at one sample per pixel (tests/test_gpu_sample_films.py's check: a box-filtered
pixel holds 0 + L of one path, bit for bit against pb2_li_samples, and its weight is its deposit count) with
PB2_TRACE_BLOCKS at 8, 7 and 6 blocks per SM on two and three pipelines, and so do the benchmark's shapes at
1920 x 1080 with the shipped pool and pipelines.  The ray counters of every setting equal those of the shipped render
(no knob set).

PB2_PIPES and PB2_POOL are read once per process, so each pipeline count renders in a worker process of its own;
PB2_TRACE_BLOCKS is read at every render.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import test_gpu_sample_films as sf
import test_gpu_wavefront_schedules as ws
from conftest import ROOT

TESTS = os.path.dirname(os.path.abspath(__file__))

SETTINGS = ("8", "7", "6")   # PB2_TRACE_BLOCKS
WORKERS = {
    "pipes2": {"PB2_POOL": "65536", "PB2_PIPES": "2"},
    "pipes3": {"PB2_POOL": "65536", "PB2_PIPES": "3"},
    "bench": {},
}
KNOBS = sf.KNOBS + ("PB2_TRACE_BLOCKS",)


def render_settings(pb, hs, flags):
    """The one-sample frame of hs under every setting and flag, checked against pb2_li_samples, and the ray counters of
    the shipped render (no knob set) and of every setting."""
    from pbrt_v3_b200 import multigpu
    film = hs.film.contents
    params = sf.one_sample(hs)
    items = multigpu.work_items(hs.film, params)
    li, pfilm = hs.li_samples(items[:, :2], items[:, 2].astype(np.int64), params)
    exp = sf.expected_film(film, li, pfilm)
    memo = []

    def model_bound():
        if not memo:
            memo.append(ws.film_model(film, li, pfilm))
        return memo[0]
    shipped = []
    for f in flags:
        _, st = hs.render_rgbw(sf.one_sample(hs, flags=f))
        shipped.append([st.camera_rays, st.regular_rays, st.shadow_rays])
    summaries, messages, stats = [], [], []
    try:
        for blocks in SETTINGS:
            os.environ["PB2_TRACE_BLOCKS"] = blocks
            for f in flags:
                rgbw, st = hs.render_rgbw(sf.one_sample(hs, flags=f))
                s, why = sf.film_check(film, rgbw, exp, items, model_bound)
                summaries.append(s)
                messages.append(why or "")
                stats.append([st.camera_rays, st.regular_rays, st.shadow_rays])
    finally:
        os.environ.pop("PB2_TRACE_BLOCKS", None)
    return {"flags": np.array(flags * len(SETTINGS)), "items": np.int64(len(items)), "summary": np.array(summaries),
            "message": np.array(messages), "stats": np.array(stats, np.int64), "shipped": np.array(shipped * len(SETTINGS), np.int64)}


def render_worker(name, out):
    import pbrt_v3_b200 as pb
    res = {}
    if name == "bench":
        import bench
        for w in sf.BENCH_SHAPES:
            hs = bench.build_scene(sf.bench_args(w))
            res.update({w + ":" + k: v for k, v in render_settings(pb, hs, [0]).items()})
            del hs
    else:
        for case in ws.CASES:
            env = ws.CASE_ENV.get(case, {})
            os.environ.update(env)
            try:
                hs = sf.make_case(pb, case, sf.pipe_scale(pb, case))
                res.update({case + ":" + k: v for k, v in render_settings(pb, hs, [0, pb.PB2_FLAG_CHAIN]).items()})
            finally:
                for key in env:
                    os.environ.pop(key, None)
    np.savez(out, **res)


WORKER = r'''
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_gpu_coresident as t
t.render_worker(sys.argv[3], sys.argv[4])
print(sys.argv[3], "ok")
'''


@pytest.fixture(scope="module")
def worker(tmp_path_factory):
    """worker(name) -> {case: {field: array}} of that worker (run once per module, on first use)."""
    d = tmp_path_factory.mktemp("coresident")
    script = d / "worker.py"
    script.write_text(WORKER)
    done = {}

    def get(name):
        if name not in done:
            out = d / (name + ".npz")
            env = dict(os.environ)
            for knob in KNOBS:
                env.pop(knob, None)
            env.update(WORKERS[name])
            res = subprocess.run([sys.executable, str(script), ROOT, TESTS, name, str(out)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                 text=True, timeout=1800, cwd=ROOT, env=env)
            if res.returncode != 0:
                done[name] = "worker %s failed:\n%s" % (name, res.stdout[-4000:])
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


def check(r, what):
    sf.assert_films(r, what)
    assert (r["stats"][:, 0] == r["items"]).all(), (what, "camera rays", r["stats"][:, 0].tolist(), int(r["items"]))
    assert np.array_equal(r["stats"], r["shipped"]), (what, "ray counters differ from the shipped render", r["stats"].tolist(), r["shipped"].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("case", ws.CASES)
@pytest.mark.parametrize("name", ["pipes2", "pipes3"])
def test_shared_sms_change_no_sample(worker, name, case):
    check(worker(name)[case], "%s / %s" % (name, case))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sf.BENCH_SHAPES)
def test_shared_sms_change_no_sample_of_the_bench_shapes(worker, shape):
    check(worker("bench")[shape], shape)
