"""The shade step draws a path vertex's sampler dimensions in one batch (haltonSampleBatch, device/pb2_sampler.cuh): every
value must be the bits the per-dimension evaluation gives, or the renders would change."""
import ctypes as C

import numpy as np
import pytest

BATCH = 8          # kSampleBatch
MAX_DIMS = 1000    # kMaxHaltonDims


def _primes(n):
    out = []
    k = 2
    while len(out) < n:
        if all(k % p for p in out if p * p <= k):
            out.append(k)
        k += 1
    return out


def _table_block(b):
    """B = b^m, the largest power of b <= 8192 with m <= 5 (HaltonDimTab::B)."""
    B, m = b, 1
    while B * b <= 8192 and m < 5:
        B, m = B * b, m + 1
    return B


def _bench_scene(pb):
    # the DHalton of the bench frame: 1920x1080, 64 spp
    return pb.HostScene.soup(10, xres=1920, yres=1080, spp=64, maxdepth=8)


def test_batch_equals_the_digit_tables_on_the_host(pb):
    """Every window [dim0, dim0 + 8) from dimension 2 up to the last one, at random 32-bit indices and at each window
    base's block edges (0, B - 1, B, B^2, B^2 + 1, 2^32 - 1): the batch gives scrambledRadicalInverseTab's bits."""
    L = pb.lib()
    hs = _bench_scene(pb)
    primes = _primes(MAX_DIMS)
    rng = np.random.RandomState(7)
    idx, dim0 = [], []
    for d0 in range(2, MAX_DIMS - BATCH + 1):
        edges = {0, 2 ** 32 - 1}
        for b in primes[d0:d0 + BATCH]:
            B = _table_block(b)
            edges |= {B - 1, B, B * B, B * B + 1}
        window = np.concatenate([np.array(sorted(edges), np.uint64), rng.randint(0, 2 ** 32, 16, dtype=np.uint64),
                                 rng.randint(0, 2 * 10 ** 6, 16, dtype=np.uint64)])   # (the bench frame's indices are below 2^21)
        idx.append(window)
        dim0.append(np.full(len(window), d0, np.int32))
    idx = np.concatenate(idx).astype(np.uint32)
    dim0 = np.concatenate(dim0)
    batch = np.zeros((len(idx), BATCH), np.float32)
    tab = np.zeros((len(idx), BATCH), np.float32)
    fn = L.pb2_debug_halton_batch
    fn.argtypes = [C.POINTER(pb.FilmDesc), C.POINTER(pb.PathParams), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    assert fn(hs.film, hs.params, pb.ptr(idx), pb.ptr(dim0), len(idx), pb.ptr(batch), pb.ptr(tab)) == 0
    assert np.array_equal(batch.view(np.uint32), tab.view(np.uint32))
    assert 0 <= batch.min() and batch.max() < 1


@pytest.mark.gpu
def test_batch_on_the_device_equals_halton_samples(pb):
    """On the device, the batch of a (pixel, sample number) over dimensions [dim0, dim0 + 8) equals pb2_halton_samples of
    each of those dimensions: table windows, windows that start at dimensions 0 and 1, and indices of 2^32 and above."""
    L = pb.lib()
    hs = _bench_scene(pb)
    rng = np.random.RandomState(11)
    dim0 = np.concatenate([np.arange(0, MAX_DIMS - BATCH + 1), rng.randint(2, 40, 4000)]).astype(np.int32)
    n = len(dim0)
    pixel_xy = np.stack([rng.randint(0, 1920, n), rng.randint(0, 1080, n)], 1).astype(np.int32)
    sample_num = rng.randint(0, 64, n).astype(np.int64)
    sample_num[::97] = rng.randint(2 ** 18, 2 ** 22, len(sample_num[::97]))   # indices of 2^32 and above (sample stride 31104)
    batch = np.zeros((n, BATCH), np.float32)
    fn = L.pb2_debug_halton_batch_device
    fn.argtypes = [C.POINTER(pb.FilmDesc), C.POINTER(pb.PathParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    pb.init(0)
    assert fn(hs.film, hs.params, pb.ptr(pixel_xy), pb.ptr(sample_num), pb.ptr(dim0), n, pb.ptr(batch)) == 0
    rep = np.repeat(np.arange(n), BATCH)
    dims = (dim0[rep] + np.tile(np.arange(BATCH), n)).astype(np.int32)
    want = hs.halton(pixel_xy[rep], sample_num[rep], dims).reshape(n, BATCH)
    assert np.array_equal(batch.view(np.uint32), want.view(np.uint32))
