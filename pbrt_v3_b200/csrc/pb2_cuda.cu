// CUDA kernels and the C ABI (include/pb2.h) of the path-tracing hot path, sm_90a only.
//
// Kernels
//   k_build_leaf_records      scene upload: gather triangle vertices into BVH-ordered 48-B leaf records
//   k_spatial_light_dist      scene upload: SpatialLightDistribution::ComputeDistribution for every voxel
//   k_intersect / k_intersect_p   Scene::Intersect / IntersectP for a batch of rays (1 thread = 1 ray)
//   k_wf_gen / k_wf_trace* / k_wf_advance<>   the wavefront renderer (pb2_wavefront.cuh):
//                             SamplerIntegrator::Render + PathIntegrator::Li + FilmTile::AddSample
//   k_li_samples, k_halton_samples, k_light_distribution   parity / debug entry points
//   k_hlbvh_centroid_bounds / k_hlbvh_morton / k_hlbvh_treelet_starts / k_hlbvh_emit   the O(n) stages of
//                             BVHAccel::HLBVHBuild behind pb2_hlbvh_treelets (with cub's radix sort between them)
//
// Compile flags that matter for parity: -fmad=false (the reference has no FMA contraction),
// default IEEE division and square root, no fast-math.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <dlfcn.h>
#include <nccl.h>   // types and prototypes only: libnccl is loaded at run time by pb2_dist_init (no link-time dependency)

#include <algorithm>
#include <mutex>
#include <chrono>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "device/pb2_path.cuh"
#include "device/pb2_wide4.cuh"
#include "host/core.h"  // pbrt::RNG for the Halton permutation table
#include "pb2.h"

using namespace pb2;

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
static thread_local std::string g_lastError;
static int setError(int code, const std::string &msg) {
    g_lastError = msg;
    return code;
}
#define CUDA_TRY(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            return setError(PB2_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));           \
    } while (0)

// Devices bound by pb2_init / pb2_init_devices.  g_devs[0] is the primary one (every single-device entry point, the root of
// a multi-device render); a render over several local devices runs one host thread per device, each with t_dev set to its
// entry, so that the code below - written for "the current device" - needs no device argument.
struct DeviceState {
    int id = -1;
    int numSMs = 0;
    int32_t *primes = nullptr, *primeSums = nullptr;   // Halton tables in this device's memory
    uint16_t *perms = nullptr;
    ulonglong2 *dimRecs = nullptr;
    HaltonDimTab *dimTabs = nullptr;
    uint16_t *digitTab = nullptr;
    uint32_t *sobol = nullptr;        // SobolMatrices32 (uploaded on the first frame that uses the SobolSampler)
    uint64_t *sobolVdc = nullptr;     // the two SobolIntervalToIndex tables of the frame being rendered (104 entries)
    bool peerOfPrimary = false;   // the primary device can read this one's memory directly (NVLink / PCIe peer access)
};
static std::vector<DeviceState> g_devs;
static thread_local int t_dev = 0;
static bool g_initialised = false;
static DeviceState &cur() {
    static DeviceState none;   // before pb2_init: null tables (host-only entry points such as pb2_work_items never read them)
    return (size_t)t_dev < g_devs.size() ? g_devs[(size_t)t_dev] : none;
}
#define g_numSMs (cur().numSMs)

// ---------------------------------------------------------------------------------------------
// Multi-GPU: one process per GPU, the film reduce over NCCL (SURVEY.md §8e).  The communicator spans the processes
// that called pb2_dist_init with the same unique id; rank r renders the tiles t with t % world == r and
// Film::MergeFilmTile across GPUs is one ncclReduce(sum) of the W x H x 4 floats to rank 0.
// ---------------------------------------------------------------------------------------------
struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Reduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int *) = nullptr;
};
static NcclApi g_nccl;
static struct {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1;
} g_dist;

static int loadNccl() {
    if (g_nccl.handle) return PB2_OK;
    // a libnccl.so.2 that is already mapped into the process (torch's bundled copy under torchrun) is found by its soname
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return setError(PB2_ERR_NCCL, std::string("libnccl.so.2 could not be loaded: ") + dlerror());
    NcclApi a;
    a.handle = h;
    a.GetUniqueId = (decltype(a.GetUniqueId))dlsym(h, "ncclGetUniqueId");
    a.CommInitRank = (decltype(a.CommInitRank))dlsym(h, "ncclCommInitRank");
    a.CommDestroy = (decltype(a.CommDestroy))dlsym(h, "ncclCommDestroy");
    a.Reduce = (decltype(a.Reduce))dlsym(h, "ncclReduce");
    a.GetErrorString = (decltype(a.GetErrorString))dlsym(h, "ncclGetErrorString");
    a.GetVersion = (decltype(a.GetVersion))dlsym(h, "ncclGetVersion");
    if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.Reduce || !a.GetErrorString)
        return setError(PB2_ERR_NCCL, "libnccl.so.2 lacks a required symbol");
    g_nccl = a;
    return PB2_OK;
}
#define NCCL_TRY(expr)                                                                                        \
    do {                                                                                                      \
        ncclResult_t _r = (expr);                                                                             \
        if (_r != ncclSuccess) return setError(PB2_ERR_NCCL, std::string(#expr) + ": " + g_nccl.GetErrorString(_r)); \
    } while (0)

static int envInt(const char *name, int def) {
    const char *v = std::getenv(name);
    return v ? std::atoi(v) : def;
}

// ---------------------------------------------------------------------------------------------
// Halton tables (lowdiscrepancy.cpp:40,124,2490-2504; halton.cpp:65-93)
// ---------------------------------------------------------------------------------------------
struct HaltonTables {   // host copies; the device copies live in DeviceState (dimRecs: per dimension {ceil(2^64 / prime), prime | primeSum << 32})
    std::vector<int32_t> hPrimes, hPrimeSums;
    std::vector<HaltonDimTab> hDimTabs;   // digit tables of the scrambled radical inverse (pb2_sampler.cuh)
    std::vector<uint16_t> hDigitTab;
    std::vector<ulonglong2> hDimRecs;
    std::vector<uint16_t> hPerms;
};
static HaltonTables g_halton;

static void buildHaltonHostTables() {
    if (!g_halton.hPrimes.empty()) return;
    std::vector<int32_t> &primes = g_halton.hPrimes;
    for (int n = 2; (int)primes.size() < kMaxHaltonDims; ++n) {
        bool isPrime = true;
        for (int p : primes) {
            if (p * p > n) break;
            if (n % p == 0) { isPrime = false; break; }
        }
        if (isPrime) primes.push_back(n);
    }
    g_halton.hPrimeSums.resize(kMaxHaltonDims);
    int sum = 0;
    for (int i = 0; i < kMaxHaltonDims; ++i) {
        g_halton.hPrimeSums[i] = sum;
        sum += primes[i];
    }
    // ComputeRadicalInversePermutations with a default-constructed RNG; Shuffle() from sampling.h:150-157
    g_halton.hPerms.resize(sum);
    pbrt::RNG rng;
    uint16_t *p = g_halton.hPerms.data();
    for (int i = 0; i < kMaxHaltonDims; ++i) {
        int count = primes[i];
        for (int j = 0; j < count; ++j) p[j] = (uint16_t)j;
        for (int j = 0; j < count; ++j) {
            int other = j + (int)rng.UniformUInt32((uint32_t)(count - j));
            std::swap(p[j], p[other]);
        }
        p += count;
    }
    // exact division by the base in the digit loops: floor(a / d) == umul64hi(a, ceil(2^64 / d)) for a < 2^32
    g_halton.hDimRecs.resize(kMaxHaltonDims);
    for (int i = 0; i < kMaxHaltonDims; ++i) {
        uint64_t d = (uint64_t)primes[i];
        uint64_t magic = ~0ull / d + 1;   // d is never a power of two above 2, and base 2 does not use it
        g_halton.hDimRecs[i] = make_ulonglong2(magic, (uint64_t)(uint32_t)primes[i] | ((uint64_t)(uint32_t)g_halton.hPrimeSums[i] << 32));
    }
    // digit tables: the digit loop of ScrambledRadicalInverseSpecialized (lowdiscrepancy.cpp:405-424) run once per table
    // entry, over exactly m digits (full) and until the value is used up (nat)
    g_halton.hDimTabs.resize(kMaxHaltonDims);
    for (int i = 0; i < kMaxHaltonDims; ++i) {
        HaltonDimTab &t = g_halton.hDimTabs[i];
        memset(&t, 0, sizeof(t));
        const uint32_t base = (uint32_t)primes[i];
        const uint16_t *perm = g_halton.hPerms.data() + g_halton.hPrimeSums[i];
        uint32_t B = base, m = 1;
        while ((uint64_t)B * base <= kHaltonTabMax && m < 5) {   // n must fit the 3 bits above the 13 of the reversed digits
            B *= base;
            ++m;
        }
        t.B = B;
        t.m = m;
        t.magicB = ~0ull / B + 1;
        t.tabOffset = (uint32_t)g_halton.hDigitTab.size();
        uint32_t p = 1;
        for (int k = 0; k < 6; ++k) {
            t.pow[k] = p;
            p = (uint64_t)p * base > 0xffffffffull ? 0u : p * base;
        }
        const float invBase = 1.f / (float)base;
        float invBaseN = 1;
        for (int k = 0; k < 16; ++k) {
            t.invPow[k] = invBaseN;
            invBaseN *= invBase;
        }
        t.tail = invBase * perm[0] / (1 - invBase);
        g_halton.hDigitTab.resize(g_halton.hDigitTab.size() + 2 * (size_t)B);
        uint16_t *nat = g_halton.hDigitTab.data() + t.tabOffset, *full = nat + B;
        for (uint32_t x = 0; x < B; ++x) {
            uint32_t a = x, rev = 0, n = 0, revFull = 0;
            for (uint32_t k = 0; k < m; ++k) {
                const uint32_t next = a / base, digit = a - next * base;
                revFull = revFull * base + perm[digit];
                if (a) {
                    rev = revFull;
                    n = k + 1;
                }
                a = next;
            }
            // (rev: the state when the loop stops at the last non-zero digit = revFull as of that digit)
            nat[x] = (uint16_t)(rev | (n << 13));
            full[x] = (uint16_t)revFull;
        }
    }
}

static void extendedGCD(uint64_t a, uint64_t b, int64_t *x, int64_t *y) {
    if (b == 0) {
        *x = 1;
        *y = 0;
        return;
    }
    int64_t d = a / b, xp, yp;
    extendedGCD(b, a % b, &xp, &yp);
    *x = yp;
    *y = xp - (d * yp);
}
static uint64_t multiplicativeInverse(int64_t a, int64_t n) {
    int64_t x, y;
    extendedGCD(a, n, &x, &y);
    int64_t r = x - (x / n) * n;
    return (uint64_t)(r < 0 ? r + n : r);
}

struct SampleBounds { int x0, y0, x1, y1; };
static SampleBounds filmSampleBounds(const pb2_film_desc *f) {  // Film::GetSampleBounds (film.cpp:80-86)
    SampleBounds b;
    b.x0 = (int)std::floor((float)f->cropped_pixel_bounds[0] + 0.5f - f->filter_radius[0]);
    b.y0 = (int)std::floor((float)f->cropped_pixel_bounds[1] + 0.5f - f->filter_radius[1]);
    b.x1 = (int)std::ceil((float)f->cropped_pixel_bounds[2] - 0.5f + f->filter_radius[0]);
    b.y1 = (int)std::ceil((float)f->cropped_pixel_bounds[3] - 0.5f + f->filter_radius[1]);
    return b;
}

static DHalton makeHalton(const pb2_film_desc *film, const pb2_path_params *pp) {
    DHalton h;
    SampleBounds sb = filmSampleBounds(film);
    int res[2] = {sb.x1 - sb.x0, sb.y1 - sb.y0};
    for (int i = 0; i < 2; ++i) {
        int base = (i == 0) ? 2 : 3;
        int scale = 1, exp = 0;
        while (scale < std::min(res[i], kMaxResolution)) {
            scale *= base;
            ++exp;
        }
        h.baseScales[i] = scale;
        h.baseExponents[i] = exp;
    }
    h.sampleStride = h.baseScales[0] * h.baseScales[1];
    h.multInverse[0] = (int)multiplicativeInverse(h.baseScales[1], h.baseScales[0]);
    h.multInverse[1] = (int)multiplicativeInverse(h.baseScales[0], h.baseScales[1]);
    h.sampleAtPixelCenter = pp->sample_at_pixel_center;
    h.samplesPerPixel = pp->samples_per_pixel;
    h.perms = cur().perms;
    h.primes = cur().primes;
    h.primeSums = cur().primeSums;
    h.dimRecs = cur().dimRecs;
    // digit tables (pb2_sampler.cuh): +7.8 % on the shading-bound killeroo-like scene, +0.8 % on the 1 M soup, bit-identical
    // values; PB2_HALTON_LOOP=1 selects the digit loop (A/B)
    h.dimTabs = envInt("PB2_HALTON_LOOP", 0) ? nullptr : cur().dimTabs;
    h.digitTab = cur().digitTab;
    h.sobol = nullptr;
    h.sobolVdc = nullptr;
    h.sobolLog2Res = h.sobolRes = 0;
    h.sbx0 = sb.x0;
    h.sby0 = sb.y0;
    return h;
}

// ---- SobolSampler (src/samplers/sobol.{h,cpp}) ---------------------------------------------------------------------------
// The generator matrices (1024 dimensions x 52 columns of 32-bit fractions) are read once from sobol_matrices32.bin next to
// this library (tools/make_sobol_tables.py).  The two tables SobolIntervalToIndex needs (the reference's VdCSobolMatrices /
// VdCSobolMatricesInv, sobolmatrices.cpp) follow from dimensions 0 and 1 and are derived here for the frame's resolution
// 2^m: the pixel a sample falls into is the upper m bits of its first two dimensions, i.e. a GF(2)-linear map A of the
// index bits; column (2m + c) of A is the pixel offset that bit c of the sample number ("frame") adds - VdCSobolMatrices[m-1][c]
// - and the inverse of A's first 2m columns turns a pixel back into the low index bits - VdCSobolMatricesInv[m-1][c] is the
// c-th column of that inverse.
static std::vector<uint32_t> g_sobolMatrices;
static std::mutex g_sobolMutex;
static int loadSobolMatrices() {
    std::lock_guard<std::mutex> lock(g_sobolMutex);
    if (!g_sobolMatrices.empty()) return PB2_OK;
    Dl_info info;
    std::string dir = ".";
    if (dladdr((void *)&loadSobolMatrices, &info) && info.dli_fname) {
        dir = info.dli_fname;
        size_t slash = dir.find_last_of('/');
        dir = slash == std::string::npos ? "." : dir.substr(0, slash);
    }
    const std::string path = dir + "/sobol_matrices32.bin";
    FILE *f = fopen(path.c_str(), "rb");
    std::vector<uint32_t> m((size_t)kSobolDims * kSobolMatrixSize);
    if (!f || fread(m.data(), sizeof(uint32_t), m.size(), f) != m.size()) {
        if (f) fclose(f);
        return setError(PB2_ERR_UNSUPPORTED, "SobolSampler: cannot read " + path + " (run tools/make_sobol_tables.py or __graft_entry__.build())");
    }
    fclose(f);
    // dimension 0 must be the van der Corput sequence and dimension 1 start with the all-ones row: a cheap sanity check of the file
    for (int k = 0; k < 32; ++k)
        if (m[k] != (0x80000000u >> k) || !(m[kSobolMatrixSize + k] & 0x80000000u))
            return setError(PB2_ERR_INVALID, "SobolSampler: " + path + " does not hold Sobol' generator matrices");
    g_sobolMatrices.swap(m);
    return PB2_OK;
}
// (px << m | py) offset that index bit k adds, for resolution 2^m (m <= 26: the columns' upper 32 bits are enough)
static uint64_t sobolPixelColumn(int k, int m) {
    const uint64_t c0 = g_sobolMatrices[k], c1 = g_sobolMatrices[kSobolMatrixSize + k];
    return ((c0 >> (32 - m)) << m) | (c1 >> (32 - m));
}
static void sobolIntervalTables(int m, uint64_t out[2 * kSobolMatrixSize]) {
    memset(out, 0, 2 * kSobolMatrixSize * sizeof(uint64_t));
    if (m <= 0) return;
    const int n = 2 * m;
    for (int c = 0; c + n < kSobolMatrixSize; ++c) out[c] = sobolPixelColumn(n + c, m);
    // invert the n x n matrix whose column k is sobolPixelColumn(k, m): Gauss-Jordan on rows {A row | identity row}
    std::vector<uint64_t> a((size_t)n, 0), id((size_t)n);
    for (int r = 0; r < n; ++r) {
        for (int k = 0; k < n; ++k)
            if ((sobolPixelColumn(k, m) >> r) & 1) a[r] |= 1ull << k;
        id[r] = 1ull << r;
    }
    for (int k = 0, rr = 0; k < n; ++k, ++rr) {
        int p = rr;
        while (p < n && !((a[p] >> k) & 1)) ++p;   // (always found: the first two Sobol' dimensions form a (0, 2)-sequence)
        if (p == n) return;
        std::swap(a[rr], a[p]);
        std::swap(id[rr], id[p]);
        for (int r = 0; r < n; ++r)
            if (r != rr && ((a[r] >> k) & 1)) {
                a[r] ^= a[rr];
                id[r] ^= id[rr];
            }
    }
    // now a[k] == 1 << k: index bit k = parity(id[k] & pixel bits); column c of the inverse collects the k with bit c set
    for (int c = 0; c < n; ++c) {
        uint64_t v = 0;
        for (int k = 0; k < n; ++k)
            if ((id[k] >> c) & 1) v |= 1ull << k;
        out[kSobolMatrixSize + c] = v;
    }
}
// Completes a DHalton for a frame that uses the SobolSampler, on the current device.
static int attachSobol(DHalton *h, const pb2_film_desc *film) {
    int rc = loadSobolMatrices();
    if (rc) return rc;
    DeviceState &dev = cur();
    if (!dev.sobol) {
        CUDA_TRY(cudaMalloc((void **)&dev.sobol, g_sobolMatrices.size() * sizeof(uint32_t)));
        CUDA_TRY(cudaMemcpy(dev.sobol, g_sobolMatrices.data(), g_sobolMatrices.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    if (!dev.sobolVdc) CUDA_TRY(cudaMalloc((void **)&dev.sobolVdc, 2 * kSobolMatrixSize * sizeof(uint64_t)));
    // SobolSampler's constructor (sobol.h:52-57): resolution = RoundUpPow2(max extent of the sample bounds)
    SampleBounds sb = filmSampleBounds(film);
    int extent = std::max(sb.x1 - sb.x0, sb.y1 - sb.y0), res = 1, log2Res = 0;
    while (res < extent) {
        res <<= 1;
        ++log2Res;
    }
    if (log2Res > 26) return setError(PB2_ERR_UNSUPPORTED, "SobolSampler: sample bounds beyond 2^26 pixels in one direction");
    uint64_t tables[2 * kSobolMatrixSize];
    sobolIntervalTables(log2Res, tables);
    CUDA_TRY(cudaMemcpy(dev.sobolVdc, tables, sizeof(tables), cudaMemcpyHostToDevice));
    h->sobol = dev.sobol;
    h->sobolVdc = dev.sobolVdc;
    h->sobolLog2Res = log2Res;
    h->sobolRes = res;
    h->sampleAtPixelCenter = 0;
    return PB2_OK;
}

// ---------------------------------------------------------------------------------------------
// scene
// ---------------------------------------------------------------------------------------------
struct pb2_scene {
    DScene d;
    std::vector<void *> allocations;
    float *film = nullptr;  // cached device film for pb2_render_path
    float *filterTable = nullptr;  // 16 x 16 filter weights of the frame being rendered (non-box filters)
    size_t filmFloats = 0;
    unsigned long long *counters = nullptr;  // CTR_*
    int64_t nPrims = 0;
    int nLights = 0;
    int bvhDepth = 0;  // maximum number of simultaneously pending far children = tree depth (scene BVH)
    int instDepth = 0; // the same for the deepest instanced object's BVH
    int shadeFeatures = SHADE_GENERAL;   // recordShadeFeatures: the lobes, lights and specular materials of the records
    int devIndex = 0;             // entry of g_devs this copy lives on
    std::vector<pb2_scene *> replicas;   // primary only: the copies on g_devs[1..] (pb2_init_devices with several devices)
    bool lazyLightDist = false;   // spatial light distribution built on demand (DLightDist::slots)
    int *ldHostCounters = nullptr;   // pinned copy of DLightDist::counters
    // wavefront pool (allocated on first render)
    void *wfCtx = nullptr;
    int *wfQueues = nullptr;
    unsigned *wfCounts = nullptr;
    unsigned *wfHostCounts = nullptr;  // pinned
    int wfCapacity = 0;
    std::vector<cudaEvent_t> traceEvents;
    int2 *wfSpill = nullptr;                 // k_wf_trace_pool: stack entries beyond its shared-memory depth
    void *paramBuf = nullptr;                // device copies of {DScene, DRenderParams} of the render in flight (renderWavefront)
    cudaStream_t pipeStreams[4] = {nullptr, nullptr, nullptr, nullptr};   // streams of the wavefront pipelines 1.. (renderWavefront)
    cudaEvent_t forkEvent = nullptr, joinEvents[4] = {nullptr, nullptr, nullptr, nullptr};
};

template <typename T>
static int upload(pb2_scene *s, const T *host, size_t count, const T **dev) {
    *dev = nullptr;
    if (count == 0 || host == nullptr) return PB2_OK;
    void *p = nullptr;
    CUDA_TRY(cudaMalloc(&p, count * sizeof(T)));
    s->allocations.push_back(p);
    CUDA_TRY(cudaMemcpy(p, host, count * sizeof(T), cudaMemcpyHostToDevice));
    *dev = (const T *)p;
    return PB2_OK;
}
template <typename T>
static int allocate(pb2_scene *s, size_t count, T **dev) {
    void *p = nullptr;
    CUDA_TRY(cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T)));
    s->allocations.push_back(p);
    *dev = (T *)p;
    return PB2_OK;
}

__global__ void k_build_leaf_records(DScene sc, const int32_t *prims, int64_t n, float4 *out) {
    int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n) return;
    int prim = prims[j];
    float4 a, b, c;
    if (sc.primType[prim] == PB2_PRIM_SPHERE) {
        a = make_float4(0, 0, 0, __int_as_float(prim));
        b = make_float4(0, 0, 0, __uint_as_float(LEAF_SPHERE));
        c = make_float4(0, 0, 0, __int_as_float(sc.primIndex[prim]));
    } else if (sc.primType[prim] == PB2_PRIM_INSTANCE) {
        a = make_float4(0, 0, 0, __int_as_float(prim));
        b = make_float4(0, 0, 0, __uint_as_float(LEAF_INSTANCE));
        c = make_float4(0, 0, 0, __int_as_float(sc.primIndex[prim]));
    } else {
        int tri = sc.primIndex[prim];
        TriVerts t = triVerts(sc, tri);
        uint32_t flags = 0;
        V2 uv[3];
        const pb2_mesh mesh = sc.meshes[sc.triMesh[tri]];
        triUVs(sc, tri, mesh, uv);
        V3 dpdu, dpdv;
        if (!triPartials(t.p0, t.p1, t.p2, uv, &dpdu, &dpdv)) flags |= LEAF_DEGENERATE;
        if ((mesh.reverse_orientation != 0) ^ (mesh.transform_swaps_handedness != 0)) flags |= LEAF_FLIP;
        if (mesh.has_n || mesh.has_s || mesh.has_uv) flags |= LEAF_ATTR;
        if (mesh.alpha_tex || mesh.shadow_alpha_tex) flags |= LEAF_ALPHA;
        a = make_float4(t.p0.x, t.p0.y, t.p0.z, __int_as_float(prim));
        b = make_float4(t.p1.x, t.p1.y, t.p1.z, __uint_as_float(flags));
        c = make_float4(t.p2.x, t.p2.y, t.p2.z, __int_as_float(sc.primLight[prim]));
    }
    out[3 * j] = a;
    out[3 * j + 1] = b;
    out[3 * j + 2] = c;
}

__global__ void k_spatial_light_dist(DScene sc, DHalton h, float *table) {
    int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const DLightDist &ld = sc.lightDist;
    int64_t total = (int64_t)ld.nVoxels[0] * ld.nVoxels[1] * ld.nVoxels[2];
    if (v >= total) return;
    int pz = (int)(v % ld.nVoxels[2]);
    int py = (int)((v / ld.nVoxels[2]) % ld.nVoxels[1]);
    int px = (int)(v / ((int64_t)ld.nVoxels[2] * ld.nVoxels[1]));
    computeVoxelDistribution(sc, h, ld, px, py, pz, table + v * ld.stride);
}

// ---------------------------------------------------------------------------------------------
// intersection kernels
// ---------------------------------------------------------------------------------------------
__global__ void k_intersect(DScene sc, const pb2_ray *rays, int64_t n, pb2_hit *hits) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    DRay r;
    r.o = mk3(rays[i].o[0], rays[i].o[1], rays[i].o[2]);
    r.d = mk3(rays[i].d[0], rays[i].d[1], rays[i].d[2]);
    r.tMax = rays[i].t_max;
    DHit h;
    h.leaf = -1;
    h.b0 = h.b1 = h.b2 = 0;
    h.inst = -1;
    float tMax = r.tMax;
    bool found = traverse<false>(sc, r, &tMax, &h, nullptr);
    pb2_hit out;
    memset(&out, 0, sizeof(out));
    out.prim = -1;
    out.t = tMax;
    if (found) {
        DInteraction it = hitInteraction<SHADE_SPHERES>(sc, h, r, tMax);
        out.prim = it.prim;
        out.b[0] = h.b0; out.b[1] = h.b1; out.b[2] = h.b2;
        out.p[0] = it.p.x; out.p[1] = it.p.y; out.p[2] = it.p.z;
        out.p_error[0] = it.pError.x; out.p_error[1] = it.pError.y; out.p_error[2] = it.pError.z;
        out.n[0] = it.n.x; out.n[1] = it.n.y; out.n[2] = it.n.z;
        out.ns[0] = it.ns.x; out.ns[1] = it.ns.y; out.ns[2] = it.ns.z;
        out.dpdu[0] = it.dpdus.x; out.dpdu[1] = it.dpdus.y; out.dpdu[2] = it.dpdus.z;
        out.uv[0] = it.uv.x; out.uv[1] = it.uv.y;
    }
    hits[i] = out;
}

__global__ void k_intersect_p(DScene sc, const pb2_ray *rays, int64_t n, uint8_t *occluded) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    DRay r;
    r.o = mk3(rays[i].o[0], rays[i].o[1], rays[i].o[2]);
    r.d = mk3(rays[i].d[0], rays[i].d[1], rays[i].d[2]);
    r.tMax = rays[i].t_max;
    DHit h;
    h.leaf = -1;
    h.inst = -1;
    float tMax = r.tMax;
    occluded[i] = traverse<true>(sc, r, &tMax, &h, nullptr) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// render
// ---------------------------------------------------------------------------------------------
struct DRenderParams {
    DCamera cam;
    DHalton halton;
    DPathParams path;
    int sbx0, sby0, sbx1, sby1;  // sample bounds (Film::GetSampleBounds)
    int pbx0, pby0, pbx1, pby1;  // PathIntegrator::pixelBounds
    int cx0, cy0, cx1, cy1;      // Film::croppedPixelBounds
    float filterRadiusX, filterRadiusY;
    float invFilterRadiusX, invFilterRadiusY;
    const float *filterTable;    // 16 x 16 weights of Film::filterTable, nullptr for the box filter (all ones)
    float maxSampleLuminance;
    int nTilesX, nTilesY;
    int tileRank, tileCount;
    long long nOwnedTiles;
    long long nWorkItems;        // nOwnedTiles * 256 * spp
    int spp;
    float diffScale;             // 1 / sqrt(spp): RayDifferential::ScaleDifferentials in SamplerIntegrator::Render (integrator.cpp:273-274)
};

enum { CTR_WORK = 0, CTR_CAMERA = 1, CTR_REGULAR = 2, CTR_SHADOW = 3, CTR_NODES = 4, CTR_PRIMS = 5, CTR_COUNT = 8 };

PB2_HD int compact1by1(unsigned x) {
    x &= 0x55555555u;
    x = (x ^ (x >> 1)) & 0x33333333u;
    x = (x ^ (x >> 2)) & 0x0f0f0f0fu;
    x = (x ^ (x >> 4)) & 0x00ff00ffu;
    return (int)x;
}

// Work item -> (pixel, sample number).  Items are ordered tile by tile (the reference's 16x16 tiles,
// integrator.cpp:235-240), then by sample number, then in Morton order inside the tile, so 32
// consecutive items are one sample number of an 8x4 pixel block: coherent camera rays for a warp.
// Tile t belongs to this call when t % tileCount == tileRank (multi-GPU partition, SURVEY.md §8e).
PB2_HD bool decodeWork(const DRenderParams &rp, long long item, int *px, int *py, int *sample) {
    long long perTile = 256LL * rp.spp;
    long long owned = item / perTile;
    int r = (int)(item - owned * perTile);
    long long tile = (long long)rp.tileRank + owned * rp.tileCount;
    int ty = (int)(tile / rp.nTilesX), tx = (int)(tile - (long long)ty * rp.nTilesX);
    int s = r >> 8, m = r & 255;
    int x = rp.sbx0 + tx * 16 + compact1by1((unsigned)m);
    int y = rp.sby0 + ty * 16 + compact1by1((unsigned)m >> 1);
    *px = x;
    *py = y;
    *sample = s;
    if (x >= rp.sbx1 || y >= rp.sby1) return false;
    // integrator.cpp:274: pixels outside pixelBounds are skipped
    return x >= rp.pbx0 && x < rp.pbx1 && y >= rp.pby0 && y < rp.pby1;
}

// FilmTile::AddSample (film.h:121-161) with a box filter, accumulated straight into the merged film
// (MergeFilmTile's sum, film.cpp:117-130).  For every tile the tile's pixel bounds contain the
// support of each of its samples, so the clamp to the tile bounds is the clamp to the cropped bounds.
// FilmTile::AddSample with a filter weight table (film.h:121-161); out of line so that the kernels
// that call it do not carry its registers on their main path.
__device__ __noinline__ void addSampleFiltered(const DRenderParams &rp, float4 *film, V2 pFilm, V3 L) {
    float dx = pFilm.x - 0.5f, dy = pFilm.y - 0.5f;
    int p0x = (int)ceilf(dx - rp.filterRadiusX), p0y = (int)ceilf(dy - rp.filterRadiusY);
    int p1x = (int)floorf(dx + rp.filterRadiusX) + 1, p1y = (int)floorf(dy + rp.filterRadiusY) + 1;
    p0x = max(p0x, rp.cx0);
    p0y = max(p0y, rp.cy0);
    p1x = min(p1x, rp.cx1);
    p1y = min(p1y, rp.cy1);
    int width = rp.cx1 - rp.cx0;
    for (int yy = p0y; yy < p1y; ++yy) {
        float fy = fabsf(((float)yy - dy) * rp.invFilterRadiusY * 16.f);
        int ify = min((int)floorf(fy), 15);
        for (int xx = p0x; xx < p1x; ++xx) {
            float fx = fabsf(((float)xx - dx) * rp.invFilterRadiusX * 16.f);
            int ifx = min((int)floorf(fx), 15);
            float w = rp.filterTable[ify * 16 + ifx];
            float4 *px = film + ((size_t)(yy - rp.cy0) * width + (xx - rp.cx0));
            atomicAdd(px, make_float4(L.x * w, L.y * w, L.z * w, w));   // contribSum += L * sampleWeight(1) * w
        }
    }
}

__device__ __forceinline__ void addSample(const DRenderParams &rp, float4 *film, V2 pFilm, V3 L) {
    float y = luminance(L);
    if (y > rp.maxSampleLuminance) L = L * (rp.maxSampleLuminance / y);
    if (rp.filterTable) {
        addSampleFiltered(rp, film, pFilm, L);
        return;
    }
    float dx = pFilm.x - 0.5f, dy = pFilm.y - 0.5f;
    int p0x = (int)ceilf(dx - rp.filterRadiusX), p0y = (int)ceilf(dy - rp.filterRadiusY);
    int p1x = (int)floorf(dx + rp.filterRadiusX) + 1, p1y = (int)floorf(dy + rp.filterRadiusY) + 1;
    p0x = max(p0x, rp.cx0);
    p0y = max(p0y, rp.cy0);
    p1x = min(p1x, rp.cx1);
    p1y = min(p1y, rp.cy1);
    int width = rp.cx1 - rp.cx0;
    for (int yy = p0y; yy < p1y; ++yy)
        for (int xx = p0x; xx < p1x; ++xx) {
            // box filter: filterTable[...] == 1 everywhere; L * sampleWeight(1) * filterWeight(1)
            float4 *px = film + ((size_t)(yy - rp.cy0) * width + (xx - rp.cx0));
            atomicAdd(px, make_float4(L.x, L.y, L.z, 1.f));
        }
}

#include "pb2_wavefront.cuh"

// PathIntegrator::Li for explicit (pixel, sample) pairs: the same lane functions, one thread per sample.
__global__ void k_li_samples(DScene sc, DRenderParams rp, const int32_t *pixelXY, const int64_t *sampleNum, int64_t n,
                             float *outRGB, float *outPFilm, int *deferred) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int px = pixelXY[2 * i], py = pixelXY[2 * i + 1];
    DSampler smp;
    smp.index = sampleIndex<true>(rp.halton, px, py, sampleNum[i]);
    smp.dim = 0;
    V2 pFilm;
    DRay ray = generateCameraRay<true>(rp.cam, rp.halton, smp, px, py, &pFilm);
    DLane ln;
    laneStartPath(ln, ray, smp);
    while (ln.state != LS_IDLE) {
        DHit hit;
        float tMax;
        bool found = traceLane(sc, ln, &tMax, &hit, nullptr);
        DTexCtx tc;
        tc.cam = &rp.cam;
        tc.pFilm = pFilm;
        tc.diffScale = rp.diffScale;
        laneAdvance<SHADE_FULL>(sc, rp.halton, rp.path, ln, found, hit, tMax, &tc);
        if (ln.state == LS_DEFER) {   // lazy light distribution: the voxel has been requested; the host builds it and runs the sample again
            atomicAdd(deferred, 1);
            return;
        }
    }
    V3 L = guardRadiance(ln.L);
    outRGB[3 * i] = L.x;
    outRGB[3 * i + 1] = L.y;
    outRGB[3 * i + 2] = L.z;
    if (outPFilm) {
        outPFilm[2 * i] = pFilm.x;
        outPFilm[2 * i + 1] = pFilm.y;
    }
}

// pb2_trace_wavefront: rays -> path contexts of the wavefront pool (state + ray, what the trace kernels read) ...
__global__ void k_wf_debug_fill(WfPool pool, const pb2_ray *rays, const uint8_t *anyHit, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        for (int q = 0; q < WQ_COUNT; ++q) pool.counts[q] = 0;
        pool.counts[WQ_TRACE0] = (unsigned)n;
    }
    if (i >= n) return;
    WfCtx &cx = pool.ctx[i];
    cx.ln.state = (anyHit && anyHit[i]) ? LS_SHADOW : LS_PATH;
    cx.ln.ray.o = mk3(rays[i].o[0], rays[i].o[1], rays[i].o[2]);
    cx.ln.ray.d = mk3(rays[i].d[0], rays[i].d[1], rays[i].d[2]);
    cx.ln.ray.tMax = rays[i].t_max;
    cx.hit = make_float4(__int_as_float(-1), 0.f, 0.f, 0.f);
    cx.tHit = 0.f;
    cx.found = -1;
    pool.queue[WQ_TRACE0][i] = i;
}
// ... and the records the trace kernel left in them -> pb2_wf_hit
__global__ void k_wf_debug_read(DScene sc, WfPool pool, int n, pb2_wf_hit *out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const WfCtx &cx = pool.ctx[i];
    pb2_wf_hit h;
    h.found = cx.found;
    h.t = cx.tHit;
    h.leaf = __float_as_int(cx.hit.x);
    h.b[0] = cx.hit.y; h.b[1] = cx.hit.z; h.b[2] = cx.hit.w;
    h.prim = (cx.found > 0 && h.leaf >= 0) ? asInt(ldg4(&sc.leafPrims[3 * (size_t)h.leaf]).w) : -1;
    h.listed = 0;
    out[i] = h;
}
__global__ void k_wf_debug_lists(WfPool pool, pb2_wf_hit *out) {
    // which list the kernel appended each context to: 1 = shade list (path rays), 2 = light list (shadow rays)
    unsigned ns = pool.counts[WQ_SHADE], nl = pool.counts[WQ_LIGHT];
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < ns + nl; i += gridDim.x * blockDim.x) {
        int c = i < ns ? pool.queue[WQ_SHADE][i] : pool.queue[WQ_LIGHT][i - ns];
        atomicAdd(&out[c].listed, i < ns ? 1 : 2);
    }
}

__global__ void k_halton_samples(DHalton h, const int32_t *pixelXY, const int64_t *sampleNum, const int32_t *dim, int64_t n,
                                 float *out) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int px = pixelXY[2 * i], py = pixelXY[2 * i + 1];
    int64_t index = sampleIndex<true>(h, px, py, sampleNum[i]);
    // (SobolSampler::SampleDimension turns its two pixel dimensions into the offset inside the current pixel)
    if (h.sobol && dim[i] < 2) out[i] = sobolPixelSample(h, index, dim[i], dim[i] == 0 ? px : py);
    else out[i] = sampleDimension<true>(h, index, dim[i]);
}

// the sampler batch of the shade step (haltonSampleBatch) for explicit (pixel, sample, first dimension) triples
__global__ void k_halton_batch(DHalton h, const int32_t *pixelXY, const int64_t *sampleNum, const int32_t *dim0, int64_t n, float *out) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t index = sampleIndex<true>(h, pixelXY[2 * i], pixelXY[2 * i + 1], sampleNum[i]);
    float u[kSampleBatch];
    haltonSampleBatch<true>(h, index, dim0[i], kSampleBatch, u);
#pragma unroll
    for (int k = 0; k < kSampleBatch; ++k) out[kSampleBatch * i + k] = u[k];
}

__global__ void k_light_distribution(DScene sc, const float *points, int64_t n, float *out) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *rec = lightDistLookup(sc.lightDist, mk3(points[3 * i], points[3 * i + 1], points[3 * i + 2]));
    if (!rec) return;   // lazy: requested; the host builds the record and launches again
    int stride = 2 * sc.nLights + 1;
    for (int k = 0; k < stride; ++k) out[i * stride + k] = rec[k];
}

// ---------------------------------------------------------------------------------------------
// host side of the ABI
// ---------------------------------------------------------------------------------------------
static DHalton haltonTablesOnly() {   // what radicalInverse() needs: the tables, no film geometry
    DHalton h;
    memset(&h, 0, sizeof(h));
    h.primes = cur().primes;
    h.primeSums = cur().primeSums;
    h.perms = cur().perms;
    h.dimRecs = cur().dimRecs;
    h.dimTabs = cur().dimTabs;
    h.digitTab = cur().digitTab;
    return h;
}

// Lazy light distribution: build the records requested so far (no host synchronisation: the kernel reads the count).
static void launchLightDistBuild(const pb2_scene *scene, cudaStream_t stream) {
    k_lightdist_build<<<g_numSMs * 4, 128, 0, stream>>>(scene->d, haltonTablesOnly());
    k_lightdist_done<<<1, 32, 0, stream>>>(scene->d);
}
static int lightDistOverflowed(pb2_scene *scene, cudaStream_t stream, bool *overflowed) {
    *overflowed = false;
    if (!scene->lazyLightDist) return PB2_OK;
    CUDA_TRY(cudaMemcpyAsync(scene->ldHostCounters, scene->d.lightDist.counters, 4 * sizeof(int), cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    *overflowed = scene->ldHostCounters[2] != 0;
    return PB2_OK;
}
static int lightDistOverflowError() {
    return setError(PB2_ERR_UNSUPPORTED, "the on-demand pool of spatial light distributions is exhausted (very many lights x very many voxels touched): "
                                         "raise PB2_LIGHTDIST_POOL_MB or use lightsamplestrategy \"power\" / \"uniform\"");
}

static int requireDevice() {
    if (!g_initialised) return setError(PB2_ERR_NO_DEVICE, "pb2_init() has not succeeded: no CUDA device is bound (there is no CPU fallback)");
    return PB2_OK;
}

// Film's filter weight table (film.cpp:68-77): filter->Evaluate at the centres of a 16 x 16 grid over
// the positive quadrant of the filter's support.  Filter::Evaluate of src/filters/{gaussian,mitchell,sinc,
// triangle}.{h,cpp}, evaluated on the host in float like the reference does.
static bool computeFilterTable(const pb2_film_desc *f, float table[256]) {
    const float rx = f->filter_radius[0], ry = f->filter_radius[1];
    const float p0 = f->filter_param[0], p1 = f->filter_param[1];
    auto eval = [&](float x, float y) -> float {
        switch (f->filter_type) {
        case PB2_FILTER_GAUSSIAN: {   // gaussian.h:50-66
            const float alpha = p0, expX = std::exp(-alpha * rx * rx), expY = std::exp(-alpha * ry * ry);
            auto g = [&](float d, float expv) { return std::max((float)0, float(std::exp(-alpha * d * d) - expv)); };
            return g(x, expX) * g(y, expY);
        }
        case PB2_FILTER_MITCHELL: {   // mitchell.h:53-63
            const float B = p0, C = p1;
            auto m1 = [&](float v) {
                v = std::abs(2 * v);
                if (v > 1)
                    return ((-B - 6 * C) * v * v * v + (6 * B + 30 * C) * v * v + (-12 * B - 48 * C) * v + (8 * B + 24 * C)) * (1.f / 6.f);
                return ((12 - 9 * B - 6 * C) * v * v * v + (-18 + 12 * B + 6 * C) * v * v + (6 - 2 * B)) * (1.f / 6.f);
            };
            const float invRx = 1 / rx, invRy = 1 / ry;
            return m1(x * invRx) * m1(y * invRy);
        }
        case PB2_FILTER_SINC: {       // sinc.h:53-63
            const float tau = p0, Pi = 3.14159265358979323846f;
            auto sinc = [&](float v) -> float {
                v = std::abs(v);
                if (v < 1e-5) return 1;
                return std::sin(Pi * v) / (Pi * v);
            };
            auto ws = [&](float v, float radius) -> float {
                v = std::abs(v);
                if (v > radius) return 0;
                float lanczos = sinc(v / tau);
                return sinc(v) * lanczos;
            };
            return ws(x, rx) * ws(y, ry);
        }
        case PB2_FILTER_TRIANGLE:     // triangle.cpp:40-43
            return std::max((float)0, rx - std::abs(x)) * std::max((float)0, ry - std::abs(y));
        default:
            return 1.f;               // box.cpp:40
        }
    };
    int offset = 0;
    for (int y = 0; y < 16; ++y)
        for (int x = 0; x < 16; ++x, ++offset) table[offset] = eval((x + 0.5f) * rx / 16, (y + 0.5f) * ry / 16);
    return f->filter_type != PB2_FILTER_BOX;
}

static DRenderParams makeRenderParams(const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp) {
    DRenderParams rp;
    memset(&rp, 0, sizeof(rp));
    memcpy(rp.cam.rasterToCamera.m, cam->raster_to_camera, sizeof(float) * 16);
    memcpy(rp.cam.cameraToWorld.m, cam->camera_to_world, sizeof(float) * 16);
    rp.cam.lensRadius = cam->lens_radius;
    rp.cam.focalDistance = cam->focal_distance;
    rp.cam.dxCamera = mk3(cam->dx_camera[0], cam->dx_camera[1], cam->dx_camera[2]);
    rp.cam.dyCamera = mk3(cam->dy_camera[0], cam->dy_camera[1], cam->dy_camera[2]);
    rp.diffScale = 1 / std::sqrt((float)pp->samples_per_pixel);
    rp.halton = makeHalton(film, pp);
    rp.path.maxDepth = pp->max_depth;
    rp.path.rrThreshold = pp->rr_threshold;
    SampleBounds sb = filmSampleBounds(film);
    rp.sbx0 = sb.x0; rp.sby0 = sb.y0; rp.sbx1 = sb.x1; rp.sby1 = sb.y1;
    rp.pbx0 = pp->pixel_bounds[0]; rp.pby0 = pp->pixel_bounds[1]; rp.pbx1 = pp->pixel_bounds[2]; rp.pby1 = pp->pixel_bounds[3];
    rp.cx0 = film->cropped_pixel_bounds[0]; rp.cy0 = film->cropped_pixel_bounds[1];
    rp.cx1 = film->cropped_pixel_bounds[2]; rp.cy1 = film->cropped_pixel_bounds[3];
    rp.filterRadiusX = film->filter_radius[0];
    rp.filterRadiusY = film->filter_radius[1];
    rp.invFilterRadiusX = 1.f / film->filter_radius[0];   // Filter::invRadius (filter.h:55)
    rp.invFilterRadiusY = 1.f / film->filter_radius[1];
    rp.filterTable = nullptr;
    rp.maxSampleLuminance = film->max_sample_luminance;
    rp.nTilesX = (sb.x1 - sb.x0 + 15) / 16;
    rp.nTilesY = (sb.y1 - sb.y0 + 15) / 16;
    rp.tileCount = std::max(1, pp->tile_count);
    rp.tileRank = pp->tile_rank;
    long long nTiles = (long long)std::max(0, rp.nTilesX) * std::max(0, rp.nTilesY);
    rp.nOwnedTiles = nTiles > rp.tileRank ? (nTiles - rp.tileRank + rp.tileCount - 1) / rp.tileCount : 0;
    rp.spp = pp->samples_per_pixel;
    rp.nWorkItems = rp.nOwnedTiles * 256LL * rp.spp;
    return rp;
}

static int validateRenderArgs(const pb2_scene *scene, const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp) {
    if (!scene || !cam || !film || !pp) return setError(PB2_ERR_INVALID, "null argument");
    if (pp->samples_per_pixel <= 0 || pp->max_depth < 0) return setError(PB2_ERR_INVALID, "bad samples_per_pixel / max_depth");
    // a path vertex consumes up to 8 sampler dimensions after the camera sample's 5; the reference aborts with
    // "HaltonSampler can only sample 1000 dimensions" (lowdiscrepancy.cpp:2506 via halton.cpp:112) when a path gets there -
    // here the tables end at the same place, so a maxdepth that could reach it is refused up front
    if (5 + 8 * ((long long)pp->max_depth + 1) > kMaxHaltonDims)
        return setError(PB2_ERR_UNSUPPORTED, "maxdepth above 123: HaltonSampler can only sample 1000 dimensions");
    if (pp->tile_count < 0 || pp->tile_rank < 0 || (pp->tile_count > 0 && pp->tile_rank >= pp->tile_count))
        return setError(PB2_ERR_INVALID, "bad tile_rank / tile_count");
    if (pp->sampler != PB2_SAMPLER_HALTON && pp->sampler != PB2_SAMPLER_SOBOL) return setError(PB2_ERR_INVALID, "unknown sampler");
    if (pp->sampler == PB2_SAMPLER_SOBOL && (pp->samples_per_pixel & (pp->samples_per_pixel - 1)))
        return setError(PB2_ERR_INVALID, "SobolSampler: samples_per_pixel must be the power of two its constructor rounds up to (sobol.h:52)");
    if (film->cropped_pixel_bounds[2] < film->cropped_pixel_bounds[0] || film->cropped_pixel_bounds[3] < film->cropped_pixel_bounds[1])
        return setError(PB2_ERR_INVALID, "bad cropped pixel bounds");
    if (!(film->filter_radius[0] > 0) || !(film->filter_radius[1] > 0)) return setError(PB2_ERR_INVALID, "bad filter radius");
    if (film->filter_type < PB2_FILTER_BOX || film->filter_type > PB2_FILTER_TRIANGLE) return setError(PB2_ERR_INVALID, "unknown filter type");
    return PB2_OK;
}

enum { kMaxPipes = 4 };   // wavefront pipelines (renderWavefront)
typedef void (*TraceKernel)(DScene, WfPool, int, WfChain);
typedef void (*AdvanceKernel)(const DScene *, const DRenderParams *, WfPool, int, int, int, float4 *, unsigned long long *);

// The launch shape of the trace kernel a scene is traced with.
struct TraceLaunch {
    TraceKernel fn = nullptr;
    int block = 128;
    size_t smem = 0;
    int grid = 0;          // SMs x resident blocks: every trace kernel loops over its list
    bool chain = false;    // the kernel advances shadow / MIS rays itself (no k_wf_advance<light> launch)
    int carveout = 0;      // the shared-memory carve-out set on the kernel (percent)
    bool reserved = false; // the grid leaves room for a list-kernel block on every SM
    const char *name = "";
};

// The trace kernels (pb2_wavefront.cuh): k_wf_trace_plain, BVHAccel::Intersect as written (TK_COUNT: with node / primitive
// counters), the ray-pool kernel, and the persistent warps over the two-child records (the default), the four-child records
// and the reference's 32-B LinearBVHNode array (k_wf_trace).
enum TraceKernelForm { TK_COUNT, TK_PLAIN, TK_POOL, TK_WIDE2, TK_WIDE4, TK_LINEAR };
// One instantiation of a trace kernel and the trace features (TRACE_*) it is compiled for.
struct TraceKernelEntry {
    TraceKernelForm form;
    int features;
    TraceKernel fn;
    const char *name;   // on the PB2_VERBOSE line
    size_t smem;        // dynamic shared memory per block
};
template <int WIDTH, int T>
static TraceKernelEntry wideTrace() {
    const char *name = WIDTH == 4              ? "k_wf_trace_w<4>"
                       : (T & TRACE_ALPHA) ? "k_wf_trace_w<2,alpha>"
                       : (T & TRACE_CHAIN) ? "k_wf_trace_w<2,chain>"
                                           : "k_wf_trace_w<2>";
    return {WIDTH == 4 ? TK_WIDE4 : TK_WIDE2, T, k_wf_trace_w<WIDTH, T>, name, 0};
}
template <int T>
static TraceKernelEntry linearTrace() { return {TK_LINEAR, T, k_wf_trace<T>, "k_wf_trace", 0}; }

// The trace kernel for a scene and the PB2_FLAG_* of a call: its form and the features it must be compiled for.  The
// first rule that matches wins, and a flag a rule does not name is ignored.  render: the caller is a render (the
// contexts are whole paths); pb2_trace_wavefront's contexts are bare rays, which cannot be chained.
struct TraceKey {
    TraceKernelForm form;
    int features;
};
static TraceKey chooseTraceKernel(const pb2_scene *scene, int flags, bool render) {
    const bool instanced = scene->d.instances != nullptr;
    // the two- and four-child records exist for scenes within their limits (2^27 primitives, 16 per leaf)
    const bool records = scene->d.wide4 != nullptr && !(flags & PB2_FLAG_LINEAR_NODES);
    // the two levels of an instanced scene must fit the 64-entry stack of the 32-B-node kernel
    const bool linearFits = !instanced || scene->bvhDepth + 3 + scene->instDepth <= 64;
    int sceneBits = scene->d.spheres ? TRACE_SPHERES : 0;
    if (instanced) sceneBits |= TRACE_SPHERES | TRACE_INST;   // an instanced kernel compiles the sphere code as well
    if (flags & PB2_FLAG_COUNT_TRAVERSAL) return {TK_COUNT, 0};
    if ((flags & PB2_FLAG_PLAIN_TRACE) || (!records && !linearFits)) return {TK_PLAIN, 0};
    // alpha masks: the two-child kernel with the alpha test, whatever the other flags
    if (scene->d.hasAlpha) return records ? TraceKey{TK_WIDE2, sceneBits | TRACE_ALPHA} : TraceKey{TK_PLAIN, 0};
    // the spheres tuning always has the local-memory spill
    if (!records) return {TK_LINEAR, sceneBits | (sceneBits || scene->bvhDepth > 32 ? TRACE_DEEP : 0)};
    if ((flags & PB2_FLAG_POOL) && !sceneBits) return {TK_POOL, 0};
    const bool ld128 = (flags & PB2_FLAG_LD128) != 0;
    int features = sceneBits | (ld128 ? TRACE_LD128 : 0) | ((flags & PB2_FLAG_SMALL_STACK) ? TRACE_SMALL_STACK : 0);
    if (flags & PB2_FLAG_WIDE4) return {TK_WIDE4, features};
    // the two-child kernel with 32-byte loads: LEAF_TMA on a triangle scene overrides SMALL_STACK; CHAIN in a render unless
    // SMALL_STACK or LEAF_TMA is set
    if (!ld128 && (flags & PB2_FLAG_LEAF_TMA) && !sceneBits) features = TRACE_LEAF_TMA;
    if (!ld128 && render && (flags & PB2_FLAG_CHAIN) && !(flags & (PB2_FLAG_SMALL_STACK | PB2_FLAG_LEAF_TMA))) features |= TRACE_CHAIN;
    return {TK_WIDE2, features};
}

// One H100 SM (sm_90): what the trace grid and a list-kernel block share.
constexpr int kSmRegs = 65536, kSmThreads = 2048, kSmBlocks = 32, kRegUnit = 256;
constexpr int kSmSmem = 233472, kBlockSmemReserved = 1024;   // 228 KB of shared memory; 1 KB of it per resident block

static int blockRegs(int regsPerThread, int threads) {
    return (threads + 31) / 32 * ((regsPerThread * 32 + kRegUnit - 1) / kRegUnit * kRegUnit);
}

// the shared-memory carve-out (percent of kSmSmem) that holds `bytes` of blocks' shared memory
static int carveoutPercent(size_t bytes) { return (int)std::min<size_t>(100, (bytes * 100 + kSmSmem - 1) / kSmSmem); }

extern "C" int pb2_trace_blocks_with_reserve(int32_t traceRegs, int32_t traceSmem, int32_t listRegs, int32_t listSmem, int32_t maxBlocks) {
    const int list = blockRegs(listRegs, 128), trace = blockRegs(traceRegs, 128);
    int n = std::min(maxBlocks, kSmBlocks - 1);
    while (n > 0 && (n * trace + list > kSmRegs || (n + 1) * 128 > kSmThreads ||
                     n * (traceSmem + kBlockSmemReserved) + listSmem + kBlockSmemReserved > kSmSmem))
        --n;
    return std::max(n, 0);
}

// The block of the frame's list kernels (gen, light, shade) that the trace grid leaves room for on every SM when
// several pipelines share the GPU: the largest registers and static shared memory of the three.
struct ListReserve {
    int regs = 0;
    int smem = 0;
};

// steps: the render's other kernels, for the PB2_VERBOSE line.  reserve (a render with several pipelines): size the
// persistent grid so that one list-kernel block fits beside it on every SM, and set the carve-out that holds both.  Only
// a kernel with registers for 8 blocks per SM (the triangle kernels) gives blocks up: on an H100 the instanced kernel, at
// 6 blocks, lost more than the overlap gained (DESIGN.md section 3).  PB2_TRACE_BLOCKS=n fixes the blocks per SM (at
// most what the kernel's occupancy allows).
static int selectTraceKernel(pb2_scene *scene, int flags, TraceLaunch *out, bool render = false, const char *steps = "",
                             const ListReserve *reserve = nullptr) {
    static const TraceKernelEntry kernels[] = {
        {TK_COUNT, 0, k_wf_trace_plain<true>, "k_wf_trace_plain<count>", 0},
        {TK_PLAIN, 0, k_wf_trace_plain<false>, "k_wf_trace_plain", 0},
        {TK_POOL, 0, k_wf_trace_pool, "k_wf_trace_pool", 4 * sizeof(PoolWarp)},
        wideTrace<2, 0>(), wideTrace<2, TRACE_SMALL_STACK>(),
        wideTrace<2, TRACE_LD128>(), wideTrace<2, TRACE_LD128 | TRACE_SMALL_STACK>(),
        wideTrace<2, TRACE_SPHERES>(), wideTrace<2, TRACE_SPHERES | TRACE_SMALL_STACK>(),
        wideTrace<2, TRACE_SPHERES | TRACE_LD128>(), wideTrace<2, TRACE_SPHERES | TRACE_LD128 | TRACE_SMALL_STACK>(),
        wideTrace<2, TRACE_SPHERES | TRACE_INST>(), wideTrace<2, TRACE_SPHERES | TRACE_INST | TRACE_SMALL_STACK>(),
        wideTrace<2, TRACE_SPHERES | TRACE_INST | TRACE_LD128>(), wideTrace<2, TRACE_SPHERES | TRACE_INST | TRACE_LD128 | TRACE_SMALL_STACK>(),
        wideTrace<2, TRACE_LEAF_TMA>(),
        wideTrace<2, TRACE_CHAIN>(), wideTrace<2, TRACE_SPHERES | TRACE_CHAIN>(), wideTrace<2, TRACE_SPHERES | TRACE_INST | TRACE_CHAIN>(),
        wideTrace<2, TRACE_ALPHA>(), wideTrace<2, TRACE_SPHERES | TRACE_ALPHA>(), wideTrace<2, TRACE_SPHERES | TRACE_INST | TRACE_ALPHA>(),
        wideTrace<4, 0>(), wideTrace<4, TRACE_SMALL_STACK>(),
        wideTrace<4, TRACE_LD128>(), wideTrace<4, TRACE_LD128 | TRACE_SMALL_STACK>(),
        wideTrace<4, TRACE_SPHERES>(), wideTrace<4, TRACE_SPHERES | TRACE_SMALL_STACK>(),
        wideTrace<4, TRACE_SPHERES | TRACE_LD128>(), wideTrace<4, TRACE_SPHERES | TRACE_LD128 | TRACE_SMALL_STACK>(),
        wideTrace<4, TRACE_SPHERES | TRACE_INST>(), wideTrace<4, TRACE_SPHERES | TRACE_INST | TRACE_SMALL_STACK>(),
        wideTrace<4, TRACE_SPHERES | TRACE_INST | TRACE_LD128>(), wideTrace<4, TRACE_SPHERES | TRACE_INST | TRACE_LD128 | TRACE_SMALL_STACK>(),
        linearTrace<0>(), linearTrace<TRACE_DEEP>(),
        linearTrace<TRACE_SPHERES | TRACE_DEEP>(), linearTrace<TRACE_SPHERES | TRACE_INST | TRACE_DEEP>(),
    };
    const TraceKey want = chooseTraceKernel(scene, flags, render);
    const TraceKernelEntry *k = nullptr;
    for (const TraceKernelEntry &e : kernels)
        if (e.form == want.form && e.features == want.features) k = &e;
    if (!k)
        return setError(PB2_ERR_CUDA, "no trace kernel of form " + std::to_string(want.form) + " is compiled for the trace features " +
                                          std::to_string(want.features));
    TraceLaunch t;
    t.fn = k->fn;
    t.smem = k->smem;
    t.chain = (k->features & TRACE_CHAIN) != 0;
    t.name = k->name;
    if (k->form == TK_POOL && !scene->wfSpill)   // per pipeline: up to 8 resident blocks per SM x 4 warps x PL_R slots x PL_SPILL entries
        CUDA_TRY(cudaMalloc((void **)&scene->wfSpill, (size_t)kMaxPipes * g_numSMs * 8 * 4 * PL_R * PL_SPILL * sizeof(int2)));
    if (t.smem) CUDA_TRY(cudaFuncSetAttribute(t.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)t.smem));
    int blocksPerSM = 1;
    // the occupancy calculator honours the kernel's carve-out preference: ask with all of the shared memory, not with the
    // carve-out an earlier render set for fewer blocks
    CUDA_TRY(cudaFuncSetAttribute(t.fn, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocksPerSM, t.fn, t.block, t.smem));
    // the persistent grid: at most 8 blocks per SM (the pool kernel's spill buffer is sized for 8)
    const int maxBlocks = std::max(1, std::min(blocksPerSM, 8));
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, t.fn));
    const int traceSmem = (int)(fa.sharedSizeBytes + t.smem);
    if (maxBlocks < 8) reserve = nullptr;
    t.reserved = reserve != nullptr;
    blocksPerSM = reserve ? std::max(1, pb2_trace_blocks_with_reserve(fa.numRegs, traceSmem, reserve->regs, reserve->smem, maxBlocks)) : maxBlocks;
    // (read at every render, so that one process can compare settings)
    const int fixedBlocks = envInt("PB2_TRACE_BLOCKS", 0);
    if (fixedBlocks > 0) blocksPerSM = std::min(fixedBlocks, maxBlocks);
    // ask for exactly the shared-memory carve-out the resident blocks (and the reserved list block) need; the rest stays L1
    size_t need = (size_t)blocksPerSM * (traceSmem + kBlockSmemReserved);
    if (reserve) need += reserve->smem + kBlockSmemReserved;
    t.carveout = carveoutPercent(need);
    CUDA_TRY(cudaFuncSetAttribute(t.fn, cudaFuncAttributePreferredSharedMemoryCarveout, t.carveout));
    static const int verbose = envInt("PB2_VERBOSE", 0);
    if (verbose) {
        char room[96] = "";
        if (reserve) snprintf(room, sizeof(room), " (reserve: one list block of %d regs, %d B smem)", reserve->regs, reserve->smem);
        fprintf(stderr, "pb2: trace kernel %s: %d regs, %d B smem, %d blocks/SM%s, carve-out %d %%, BVH depth %d%s\n", t.name, fa.numRegs,
                traceSmem, blocksPerSM, room, t.carveout, scene->bvhDepth, steps);
    }
    t.grid = g_numSMs * blocksPerSM;
    *out = t;
    return PB2_OK;
}

static int ensurePool(pb2_scene *scene, int capacity) {
    if (scene->wfCapacity < capacity) {
        if (scene->wfCtx) cudaFree(scene->wfCtx);
        if (scene->wfQueues) cudaFree(scene->wfQueues);
        scene->wfCtx = nullptr;
        scene->wfQueues = nullptr;
        scene->wfCapacity = 0;
        CUDA_TRY(cudaMalloc(&scene->wfCtx, (size_t)capacity * sizeof(WfCtx)));
        CUDA_TRY(cudaMalloc((void **)&scene->wfQueues, (size_t)capacity * WQ_COUNT * sizeof(int)));
        scene->wfCapacity = capacity;
    }
    if (!scene->wfCounts) CUDA_TRY(cudaMalloc((void **)&scene->wfCounts, kMaxPipes * WQ_COUNT * sizeof(unsigned)));
    if (!scene->wfHostCounts) CUDA_TRY(cudaMallocHost((void **)&scene->wfHostCounts, (kMaxPipes * WQ_COUNT + 2) * sizeof(unsigned long long)));
    return PB2_OK;
}

// Pipeline `pipe` of `nPipes`: an equal slice of the context pool with queues and counters of its own.
static WfPool poolOf(const pb2_scene *scene, int capacity, int pipe = 0, int nPipes = 1) {
    WfPool pool;
    const int cap = capacity / nPipes;
    pool.capacity = cap;
    pool.ctx = (WfCtx *)scene->wfCtx + (size_t)pipe * cap;
    for (int q = 0; q < WQ_COUNT; ++q) pool.queue[q] = scene->wfQueues + ((size_t)pipe * WQ_COUNT + q) * cap;
    pool.counts = scene->wfCounts + (size_t)pipe * WQ_COUNT;
    pool.ctr = scene->counters;
    pool.spill = scene->wfSpill ? scene->wfSpill + (size_t)pipe * g_numSMs * 8 * 4 * PL_R * PL_SPILL : nullptr;
    return pool;
}

// Resident blocks per SM of the SHADE_LAMBERT_AREA shade step (__launch_bounds__ minimum; DESIGN.md section 3)
constexpr int kShadeLambertAreaMinBlocks = 4;

typedef void (*GenKernel)(const DRenderParams *, WfPool, int, int);
typedef void (*FinishKernel)(const DScene *, const DRenderParams *, WfPool, int, unsigned, float4 *);

// One instantiation of a wavefront step's kernel and the shade features (SHADE_*) it is compiled for.
template <typename K>
struct StepKernel {
    int features;
    K fn;
};
template <bool SHADE, int MINB, int F>
static StepKernel<AdvanceKernel> advanceStep() { return {F, k_wf_advance<SHADE, MINB, F>}; }

// The instantiation compiled for the fewest features that contain the frame's, counting only the features the step reads:
// those of its widest instantiation, which every table holds.
template <typename K, size_t N>
static const StepKernel<K> &stepKernel(const StepKernel<K> (&table)[N], int frame) {
    int reads = 0;
    for (const StepKernel<K> &k : table) reads |= k.features;
    const StepKernel<K> *best = nullptr;
    for (const StepKernel<K> &k : table)
        if (!(frame & reads & ~k.features) && (!best || __builtin_popcount(k.features) < __builtin_popcount(best->features))) best = &k;
    return *best;
}

// The shade features of a frame (SHADE_* in device/pb2_shade.cuh): those of the scene's material and light records
// (recordShadeFeatures), and its spheres, its lazy light distribution, its image textures and the frame's sampler.
static int frameShadeFeatures(const pb2_scene *scene, const DRenderParams &rp) {
    int f = scene->shadeFeatures;
    if (scene->d.spheres) f |= SHADE_SPHERES;
    if (scene->lazyLightDist) f |= SHADE_LAZY;
    if (scene->d.nTextures > 0) f |= SHADE_TEXTURES;
    if (rp.halton.sobol) f |= SHADE_SOBOL;
    return f;
}

// Host driver of the wavefront rounds (see pb2_wavefront.cuh).
static int renderWavefront(pb2_scene *scene, const DRenderParams &rp, float4 *film, cudaStream_t stream, int flags,
                           bool timeTrace, unsigned long long *launches, double *traceMs) {
    const bool lazyLights = scene->lazyLightDist;   // k_wf_finish cannot defer a vertex: the rounds run to the end instead
    // 4 M contexts (1 GiB) at most: enough paths in flight to keep the SMs busy at 1920x1080
    static const int maxCapacity = envInt("PB2_POOL", 1 << 22);
    long long want = std::min<long long>(maxCapacity, std::max<long long>(rp.nWorkItems, 1024));
    int capacity = (int)((want + 255) / 256 * 256);
    int rc = ensurePool(scene, capacity);
    if (rc) return rc;
    // Each step runs the kernel compiled for the frame's shade features (stepKernel): Lambertian surfaces lit by area lights
    // (the bench scene) get the class-0 kernels.
    static const StepKernel<GenKernel> genSteps[] = {{0, k_wf_gen<0>}, {SHADE_SOBOL, k_wf_gen<SHADE_SOBOL>}};
    // light step: 7 resident blocks, as many as the shared-memory stage leaves room for (29 KB per block)
    static const StepKernel<AdvanceKernel> lightSteps[] = {
        advanceStep<false, 7, SHADE_LAMBERT_AREA>(),
        advanceStep<false, 7, SHADE_GENERAL>(),
        advanceStep<false, 7, SHADE_GENERAL | SHADE_SPHERES>(),
    };
    // image textures or the SobolSampler: one shade kernel with everything compiled in (3 resident blocks, its register
    // budget is not the bench scene's)
    static const StepKernel<AdvanceKernel> shadeSteps[] = {
        advanceStep<true, kShadeLambertAreaMinBlocks, SHADE_LAMBERT_AREA>(),
        advanceStep<true, 4, SHADE_GENERAL>(),
        advanceStep<true, 4, SHADE_GENERAL | SHADE_SPHERES>(),
        advanceStep<true, 4, SHADE_GENERAL | SHADE_SPECULAR>(),
        advanceStep<true, 4, SHADE_GENERAL | SHADE_SPHERES | SHADE_SPECULAR>(),
        advanceStep<true, 4, SHADE_GENERAL | SHADE_LAZY>(),
        advanceStep<true, 4, SHADE_GENERAL | SHADE_SPHERES | SHADE_LAZY>(),
        advanceStep<true, 4, SHADE_GENERAL | SHADE_SPECULAR | SHADE_LAZY>(),
        advanceStep<true, 4, SHADE_GENERAL | SHADE_SPHERES | SHADE_SPECULAR | SHADE_LAZY>(),
        advanceStep<true, 3, SHADE_FULL>(),
    };
    static const StepKernel<FinishKernel> finishSteps[] = {
        {SHADE_LAMBERT_AREA, k_wf_finish<SHADE_LAMBERT_AREA>},
        {SHADE_GENERAL, k_wf_finish<SHADE_GENERAL>},
        {SHADE_GENERAL | SHADE_SPHERES, k_wf_finish<SHADE_GENERAL | SHADE_SPHERES>},
        {SHADE_GENERAL | SHADE_SPECULAR, k_wf_finish<SHADE_GENERAL | SHADE_SPECULAR>},
        {SHADE_GENERAL | SHADE_SPHERES | SHADE_SPECULAR, k_wf_finish<SHADE_GENERAL | SHADE_SPHERES | SHADE_SPECULAR>},
    };
    const int features = frameShadeFeatures(scene, rp);
    const StepKernel<GenKernel> &gen = stepKernel(genSteps, features);
    const StepKernel<AdvanceKernel> &advLight = stepKernel(lightSteps, features), &advShade = stepKernel(shadeSteps, features);
    const StepKernel<FinishKernel> &finish = stepKernel(finishSteps, features);
    char steps[96];
    snprintf(steps, sizeof(steps), "; shade features %d: gen %d, light %d, shade %d, tail %d", features, gen.features,
             advLight.features, advShade.features, finish.features);
    // Two pipelines, each with half of the contexts and its own lists, on two streams: one pipeline's list kernels run on
    // the SMs beside the other pipeline's trace kernel.  Both draw samples from the one work counter.
    // Lazily lit scenes share one request list: one pipeline.  On an H100 two are faster than four on the traversal-bound
    // soup, the shading-bound killeroo scene and the instanced scene alike.  PB2_PIPES fixes the number (1 ... 4).
    static const int pipesEnv = envInt("PB2_PIPES", 0);
    const int pipesWanted = std::min((int)kMaxPipes, pipesEnv > 0 ? pipesEnv : 2);
    const int nPipes = (lazyLights || capacity < 65536) ? 1 : pipesWanted;
    // With several pipelines and the class-0 shade step the persistent trace grid leaves room for one block of the
    // largest list kernel on every SM, and every kernel of the frame asks for the same shared-memory carve-out: an SM
    // changes its L1 / shared-memory split only when it is idle, so a block whose kernel prefers another split waits
    // until the SM drains.  (The shading-bound frames of the general shade step were slower so on an H100.)
    const bool share = nPipes > 1 && advShade.features == SHADE_LAMBERT_AREA;
    ListReserve reserve;
    if (share) {
        for (const void *fn : {(const void *)gen.fn, (const void *)advLight.fn, (const void *)advShade.fn}) {
            cudaFuncAttributes fa;
            CUDA_TRY(cudaFuncGetAttributes(&fa, fn));
            reserve.regs = std::max(reserve.regs, fa.numRegs);
            reserve.smem = std::max(reserve.smem, (int)fa.sharedSizeBytes);
        }
    }
    TraceLaunch trace;
    if ((rc = selectTraceKernel(scene, flags, &trace, true, steps, share ? &reserve : nullptr))) return rc;
    // no reserve: the list kernels keep the driver's choice of carve-out
    const int listCarveout = trace.reserved ? trace.carveout : (int)cudaSharedmemCarveoutDefault;
    for (const void *fn : {(const void *)gen.fn, (const void *)advLight.fn, (const void *)advShade.fn, (const void *)finish.fn, (const void *)k_wf_reset})
        CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, listCarveout));
    // the scene and this frame's parameters as objects in device memory, read by the gen / advance / finish kernels and
    // wfChainLight.  One buffer per scene, and so per device: every device of a group renders its own replica.
    if (!scene->paramBuf) CUDA_TRY(cudaMalloc(&scene->paramBuf, sizeof(DScene) + sizeof(DRenderParams)));
    const DScene *dSc = reinterpret_cast<const DScene *>(scene->paramBuf);
    const DRenderParams *dRp = reinterpret_cast<const DRenderParams *>((char *)scene->paramBuf + sizeof(DScene));
    CUDA_TRY(cudaMemcpyAsync((void *)dSc, &scene->d, sizeof(DScene), cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync((void *)dRp, &rp, sizeof(DRenderParams), cudaMemcpyHostToDevice, stream));
    WfChain chain;
    memset(&chain, 0, sizeof(chain));
    if (trace.chain) {
        chain.sc = dSc;
        chain.rp = dRp;
        chain.film = film;
    }
    // the frame's last paths are walked to their end by one thread each once this few are left (k_wf_finish)
    static const int finishPerSM = envInt("PB2_FINISH", 256);
    // (image textures or the SobolSampler: the tail kernels are compiled without them, so the rounds run to the end)
    const bool textured = (features & (SHADE_TEXTURES | SHADE_SOBOL)) != 0;
    const unsigned finishThreshold = ((flags & PB2_FLAG_COUNT_TRAVERSAL) || lazyLights || textured) ? 0u : (unsigned)(g_numSMs * std::max(0, finishPerSM));
    const int finishBlocks = std::max(1, (int)((finishThreshold + 127) / 128));
    static const int syncEvery = std::max(1, envInt("PB2_SYNC_EVERY", 8));
    cudaStream_t streams[kMaxPipes] = {stream, stream, stream, stream};
    if (nPipes > 1) {
        if (!scene->forkEvent) CUDA_TRY(cudaEventCreateWithFlags(&scene->forkEvent, cudaEventDisableTiming));
        CUDA_TRY(cudaEventRecord(scene->forkEvent, stream));            // the film clear / counter reset of the caller's stream
        for (int p = 1; p < nPipes; ++p) {
            if (!scene->pipeStreams[p]) CUDA_TRY(cudaStreamCreateWithFlags(&scene->pipeStreams[p], cudaStreamNonBlocking));
            if (!scene->joinEvents[p]) CUDA_TRY(cudaEventCreateWithFlags(&scene->joinEvents[p], cudaEventDisableTiming));
            streams[p] = scene->pipeStreams[p];
            CUDA_TRY(cudaStreamWaitEvent(streams[p], scene->forkEvent, 0));
        }
    }
    WfPool pools[kMaxPipes];
    for (int p = 0; p < nPipes; ++p) pools[p] = poolOf(scene, capacity / nPipes * nPipes, p, nPipes);
    const int capP = pools[0].capacity;
    // The list kernels' grid-stride grids stay oversubscribed: grids of resident size (SMs x occupancy) for gen, light and
    // shade were not faster on C2 (173.5 against 173.9 Msamples/s, medians of three, H100 80GB HBM3 at 700 W)
    const int blocks128 = std::min((capP + 127) / 128, g_numSMs * 32);
    for (int p = 0; p < nPipes; ++p) k_wf_init<<<(capP + 255) / 256, 256, 0, streams[p]>>>(pools[p]);
    unsigned long long nLaunch = nPipes;
    size_t nEvents = 0;
    int cur = 0;
    volatile unsigned *hc = scene->wfHostCounts;
    unsigned long long *hWork = reinterpret_cast<unsigned long long *>(scene->wfHostCounts + kMaxPipes * WQ_COUNT);
    for (long long round = 0;; ++round) {
        int next = 1 - cur;
        for (int p = 0; p < nPipes; ++p) {
            const WfPool &pool = pools[p];
            cudaStream_t st = streams[p];
            gen.fn<<<blocks128, 128, 0, st>>>(dRp, pool, WQ_FREE0 + cur, WQ_TRACE0 + cur);
            if (timeTrace) {
                if (scene->traceEvents.size() < nEvents + 2) {
                    cudaEvent_t e0, e1;
                    CUDA_TRY(cudaEventCreate(&e0));
                    CUDA_TRY(cudaEventCreate(&e1));
                    scene->traceEvents.push_back(e0);
                    scene->traceEvents.push_back(e1);
                }
                CUDA_TRY(cudaEventRecord(scene->traceEvents[nEvents], st));
            }
            chain.freeQ = WQ_FREE0 + next;
            trace.fn<<<trace.grid, trace.block, trace.smem, st>>>(scene->d, pool, WQ_TRACE0 + cur, chain);
            if (timeTrace) {
                CUDA_TRY(cudaEventRecord(scene->traceEvents[nEvents + 1], st));
                nEvents += 2;
            }
            if (!trace.chain) advLight.fn<<<blocks128, 128, 0, st>>>(dSc, dRp, pool, WQ_LIGHT, WQ_TRACE0 + next, WQ_FREE0 + next, film, scene->counters);
            else --nLaunch;
            advShade.fn<<<blocks128, 128, 0, st>>>(dSc, dRp, pool, WQ_SHADE, WQ_TRACE0 + next, WQ_FREE0 + next, film, scene->counters);
            if (lazyLights) {
                // vertices that fell into voxels without a light distribution yet were put aside: build those records, shade again
                launchLightDistBuild(scene, st);
                advShade.fn<<<blocks128, 128, 0, st>>>(dSc, dRp, pool, WQ_RETRY, WQ_TRACE0 + next, WQ_FREE0 + next, film, scene->counters);
                nLaunch += 3;
            }
            if (finishThreshold) finish.fn<<<finishBlocks, 128, 0, st>>>(dSc, dRp, pool, WQ_TRACE0 + next, finishThreshold, film);
            k_wf_reset<<<1, 32, 0, st>>>(pool, WQ_FREE0 + cur, WQ_TRACE0 + cur, WQ_TRACE0 + next, finishThreshold);
            nLaunch += finishThreshold ? 6 : 5;
        }
        cur = next;
        // The host looks at the counters only every `syncEvery` rounds; rounds enqueued after the frame
        // has drained find empty lists and cost a few microseconds each.
        if ((round + 1) % syncEvery != 0) continue;
        for (int p = 0; p < nPipes; ++p)
            CUDA_TRY(cudaMemcpyAsync((void *)(scene->wfHostCounts + p * WQ_COUNT), pools[p].counts, WQ_COUNT * sizeof(unsigned), cudaMemcpyDeviceToHost, streams[p]));
        for (int p = 1; p < nPipes; ++p) CUDA_TRY(cudaStreamSynchronize(streams[p]));
        CUDA_TRY(cudaMemcpyAsync(hWork, &scene->counters[CTR_WORK], sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        bool overflowed = false;
        if ((rc = lightDistOverflowed(scene, stream, &overflowed))) return rc;
        if (overflowed) return lightDistOverflowError();
        const bool workLeft = (long long)*hWork < rp.nWorkItems;
        bool done = true;
        for (int p = 0; p < nPipes; ++p) {
            const unsigned traceNext = hc[p * WQ_COUNT + WQ_TRACE0 + cur], freeNext = hc[p * WQ_COUNT + WQ_FREE0 + cur];
            if (!(traceNext == 0 && !(workLeft && freeNext > 0))) done = false;
        }
        if (done) break;
        if (round > 100000000LL) return setError(PB2_ERR_CUDA, "wavefront did not terminate");
    }
    if (nPipes > 1) {   // what follows on the caller's stream (film reduce, copies) comes after both pipelines
        for (int p = 1; p < nPipes; ++p) {
            CUDA_TRY(cudaEventRecord(scene->joinEvents[p], streams[p]));
            CUDA_TRY(cudaStreamWaitEvent(stream, scene->joinEvents[p], 0));
        }
    }
    CUDA_TRY(cudaGetLastError());
    *launches = nLaunch;
    *traceMs = 0;
    for (size_t e = 0; e + 1 < nEvents; e += 2) {
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, scene->traceEvents[e], scene->traceEvents[e + 1]));
        *traceMs += ms;
    }
    // (with two pipelines this is the sum of launch durations of kernels that each shared the GPU with the other pipeline's
    // kernels: algorithmic bytes / this time is the per-launch figure the roofline contract asks for, a conservative one)
    return PB2_OK;
}

extern "C" {

int pb2_abi_version(void) { return PB2_ABI_VERSION; }
const char *pb2_last_error(void) { return g_lastError.c_str(); }

static void freeDeviceTables() {
    for (DeviceState &d : g_devs) {
        cudaSetDevice(d.id);
        cudaFree(d.primes);
        cudaFree(d.primeSums);
        cudaFree(d.perms);
        cudaFree(d.dimRecs);
        cudaFree(d.dimTabs);
        cudaFree(d.digitTab);
        cudaFree(d.sobol);
        cudaFree(d.sobolVdc);
    }
    g_devs.clear();
    g_initialised = false;
}

int pb2_init_devices(int n, const int *device_ids) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        cudaGetLastError();
        return setError(PB2_ERR_NO_DEVICE, std::string("no CUDA device available (") +
                                               (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") +
                                               "); the path-tracing hot path has no CPU fallback");
    }
    std::vector<int> ids;
    if (n <= 0) for (int i = 0; i < count; ++i) ids.push_back(i);   // every visible device
    else {
        if (!device_ids) return setError(PB2_ERR_INVALID, "null device list");
        ids.assign(device_ids, device_ids + n);
    }
    for (size_t i = 0; i < ids.size(); ++i) {
        if (ids[i] < 0 || ids[i] >= count) return setError(PB2_ERR_INVALID, "device id out of range");
        for (size_t j = 0; j < i; ++j)
            if (ids[j] == ids[i]) return setError(PB2_ERR_INVALID, "device listed twice");
    }
    if (g_initialised && g_devs.size() == ids.size()) {
        bool same = true;
        for (size_t i = 0; i < ids.size(); ++i) same &= g_devs[i].id == ids[i];
        if (same) return PB2_OK;
    }
    if (g_dist.comm) return setError(PB2_ERR_INVALID, "pb2_init: shut the communicator down (pb2_dist_shutdown) before rebinding devices");
    freeDeviceTables();
    buildHaltonHostTables();
    t_dev = 0;
    for (int id : ids) {
        CUDA_TRY(cudaSetDevice(id));
        cudaDeviceProp prop;
        CUDA_TRY(cudaGetDeviceProperties(&prop, id));
        if (prop.major != 9 || prop.minor != 0) {   // sm_90a code loads on compute capability 9.0 only
            freeDeviceTables();
            return setError(PB2_ERR_NO_DEVICE, std::string("device \"") + prop.name + "\" is not sm_90 (Hopper); this library is built for sm_90a only");
        }
        g_devs.emplace_back();
        DeviceState &d = g_devs.back();
        d.id = id;
        d.numSMs = prop.multiProcessorCount;
        CUDA_TRY(cudaMalloc((void **)&d.primes, g_halton.hPrimes.size() * sizeof(int32_t)));
        CUDA_TRY(cudaMalloc((void **)&d.primeSums, g_halton.hPrimeSums.size() * sizeof(int32_t)));
        CUDA_TRY(cudaMalloc((void **)&d.perms, g_halton.hPerms.size() * sizeof(uint16_t)));
        CUDA_TRY(cudaMalloc((void **)&d.dimRecs, g_halton.hDimRecs.size() * sizeof(ulonglong2)));
        CUDA_TRY(cudaMemcpy(d.dimRecs, g_halton.hDimRecs.data(), g_halton.hDimRecs.size() * sizeof(ulonglong2), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(d.primes, g_halton.hPrimes.data(), g_halton.hPrimes.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(d.primeSums, g_halton.hPrimeSums.data(), g_halton.hPrimeSums.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(d.perms, g_halton.hPerms.data(), g_halton.hPerms.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMalloc((void **)&d.dimTabs, g_halton.hDimTabs.size() * sizeof(HaltonDimTab)));
        CUDA_TRY(cudaMalloc((void **)&d.digitTab, g_halton.hDigitTab.size() * sizeof(uint16_t)));
        CUDA_TRY(cudaMemcpy(d.dimTabs, g_halton.hDimTabs.data(), g_halton.hDimTabs.size() * sizeof(HaltonDimTab), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(d.digitTab, g_halton.hDigitTab.data(), g_halton.hDigitTab.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
    }
    // the film merge of a multi-device render reads the other devices' films from the primary one over NVLink
    CUDA_TRY(cudaSetDevice(g_devs[0].id));
    for (size_t i = 1; i < g_devs.size(); ++i) {
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, g_devs[0].id, g_devs[i].id) == cudaSuccess && can) {
            cudaError_t pe = cudaDeviceEnablePeerAccess(g_devs[i].id, 0);
            g_devs[i].peerOfPrimary = pe == cudaSuccess || pe == cudaErrorPeerAccessAlreadyEnabled;
        }
        cudaGetLastError();
    }
    g_initialised = true;
    return PB2_OK;
}

int pb2_init(int device_id) { return pb2_init_devices(1, &device_id); }

int pb2_device_count(void) { return g_initialised ? (int)g_devs.size() : 0; }

int pb2_shutdown(void) {
    if (!g_initialised) return PB2_OK;
    pb2_dist_shutdown();
    freeDeviceTables();
    return PB2_OK;
}

// Host-side check of the digit tables (tests, no device): ScrambledRadicalInverse of index[i] in dimension dim[i] by the
// digit loop (out_loop) and through the tables (out_tab); the two must agree bit for bit.
int pb2_debug_radical_inverse_tables(const uint32_t *index, const int32_t *dim, int64_t n, float *out_loop, float *out_tab) {
    if (!index || !dim || !out_loop || !out_tab) return setError(PB2_ERR_INVALID, "null argument");
    buildHaltonHostTables();
    for (int64_t i = 0; i < n; ++i) {
        if (dim[i] < 2 || dim[i] >= kMaxHaltonDims) return setError(PB2_ERR_INVALID, "dimension out of range");
        const uint32_t base = (uint32_t)g_halton.hPrimes[dim[i]];
        const uint16_t *perm = g_halton.hPerms.data() + g_halton.hPrimeSums[dim[i]];
        const uint64_t magic = g_halton.hDimRecs[dim[i]].x;
        out_loop[i] = scrambledRadicalInverse32(base, magic, index[i], perm);
        out_tab[i] = scrambledRadicalInverseTab(g_halton.hDimTabs[dim[i]], g_halton.hDigitTab.data(), base, magic, index[i], perm);
    }
    return PB2_OK;
}

// Host-side check of the shade step's sampler batch (tests, no device): with the host tables, haltonSampleBatch of
// index[i] over dimensions dim0[i] .. dim0[i] + 7 (out_batch, 8 per item) and scrambledRadicalInverseTab of each of those
// dimensions (out_tab); the two must agree bit for bit.  The film and parameters give the DHalton a render would use.
int pb2_debug_halton_batch(const pb2_film_desc *film, const pb2_path_params *pp, const uint32_t *index, const int32_t *dim0, int64_t n,
                           float *out_batch, float *out_tab) {
    if (!film || !pp || !index || !dim0 || !out_batch || !out_tab) return setError(PB2_ERR_INVALID, "null argument");
    buildHaltonHostTables();
    DHalton h = makeHalton(film, pp);
    h.perms = g_halton.hPerms.data();
    h.primes = g_halton.hPrimes.data();
    h.primeSums = g_halton.hPrimeSums.data();
    h.dimRecs = g_halton.hDimRecs.data();
    h.dimTabs = g_halton.hDimTabs.data();
    h.digitTab = g_halton.hDigitTab.data();
    for (int64_t i = 0; i < n; ++i) {
        if (dim0[i] < 2 || dim0[i] + kSampleBatch > kMaxHaltonDims) return setError(PB2_ERR_INVALID, "dimension out of range");
        haltonSampleBatch(h, (int64_t)index[i], dim0[i], kSampleBatch, out_batch + kSampleBatch * i);
        for (int k = 0; k < kSampleBatch; ++k) {
            const int d = dim0[i] + k;
            const uint32_t base = (uint32_t)g_halton.hPrimes[d];
            const uint16_t *perm = g_halton.hPerms.data() + g_halton.hPrimeSums[d];
            out_tab[kSampleBatch * i + k] = scrambledRadicalInverseTab(g_halton.hDimTabs[d], g_halton.hDigitTab.data(), base,
                                                                       g_halton.hDimRecs[d].x, index[i], perm);
        }
    }
    return PB2_OK;
}

// Device-side check of the same batch: for each (pixel, sample number) the sample's index as a render computes it, then
// haltonSampleBatch over dimensions dim0[i] .. dim0[i] + 7 on the device (8 values per item in out), to be compared with
// pb2_halton_samples of the same dimensions.
int pb2_debug_halton_batch_device(const pb2_film_desc *film, const pb2_path_params *pp, const int32_t *pixel_xy,
                                  const int64_t *sample_num, const int32_t *dim0, int64_t n, float *out) {
    int rc = requireDevice();
    if (rc) return rc;
    if (!film || !pp || (n > 0 && (!pixel_xy || !sample_num || !dim0 || !out))) return setError(PB2_ERR_INVALID, "null argument");
    if (n <= 0) return PB2_OK;
    for (int64_t i = 0; i < n; ++i)
        if (dim0[i] < 0 || dim0[i] + kSampleBatch > kMaxHaltonDims) return setError(PB2_ERR_INVALID, "dimension out of range");
    DHalton h = makeHalton(film, pp);
    if (pp->sampler == PB2_SAMPLER_SOBOL && (rc = attachSobol(&h, film))) return rc;
    int32_t *dXY = nullptr, *dDim = nullptr;
    int64_t *dS = nullptr;
    float *dOut = nullptr;
    cudaError_t e = cudaMalloc((void **)&dXY, n * 2 * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dS, n * sizeof(int64_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dDim, n * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dOut, n * kSampleBatch * sizeof(float));
    if (e == cudaSuccess) e = cudaMemcpy(dXY, pixel_xy, n * 2 * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dS, sample_num, n * sizeof(int64_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dDim, dim0, n * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        k_halton_batch<<<(unsigned)((n + 127) / 128), 128>>>(h, dXY, dS, dDim, n, dOut);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dOut, n * kSampleBatch * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(dXY);
    cudaFree(dS);
    cudaFree(dDim);
    cudaFree(dOut);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, std::string("pb2_debug_halton_batch_device: ") + cudaGetErrorString(e));
    return PB2_OK;
}

int pb2_work_items(const pb2_film_desc *film, const pb2_path_params *pp, int64_t first, int64_t n, int32_t *out, int64_t *n_items) {
    if (!film || !pp) return setError(PB2_ERR_INVALID, "null argument");
    if (pp->samples_per_pixel <= 0 || pp->tile_count < 0 || pp->tile_rank < 0 || (pp->tile_count > 0 && pp->tile_rank >= pp->tile_count))
        return setError(PB2_ERR_INVALID, "bad samples_per_pixel / tile_rank / tile_count");
    pb2_camera cam;
    memset(&cam, 0, sizeof(cam));
    const DRenderParams rp = makeRenderParams(&cam, film, pp);   // the partition does not depend on the camera
    if (n_items) *n_items = rp.nWorkItems;
    for (int64_t i = 0; i < n && out; ++i) {
        int px = -1, py = -1, sample = -1;
        const bool inside = first + i >= 0 && first + i < rp.nWorkItems && decodeWork(rp, first + i, &px, &py, &sample);
        out[3 * i] = inside ? px : -1;
        out[3 * i + 1] = inside ? py : -1;
        out[3 * i + 2] = inside ? sample : -1;
    }
    return PB2_OK;
}

int pb2_dist_unique_id(void *id128) {
    if (!id128) return setError(PB2_ERR_INVALID, "null argument");
    int rc = loadNccl();
    if (rc) return rc;
    static_assert(sizeof(ncclUniqueId) == PB2_DIST_ID_BYTES, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    NCCL_TRY(g_nccl.GetUniqueId(&id));
    memcpy(id128, &id, sizeof(id));
    return PB2_OK;
}

int pb2_dist_init(int rank, int world, const void *id128) {
    int rc = requireDevice();
    if (rc) return rc;
    if (world < 1 || rank < 0 || rank >= world || (world > 1 && !id128)) return setError(PB2_ERR_INVALID, "bad rank / world / id");
    if (g_dist.comm) return setError(PB2_ERR_INVALID, "pb2_dist_init: a communicator already exists (call pb2_dist_shutdown first)");
    g_dist.rank = rank;
    g_dist.world = world;
    if (world == 1) return PB2_OK;
    if ((rc = loadNccl())) return rc;
    ncclUniqueId id;
    memcpy(&id, id128, sizeof(id));
    if (g_devs.size() != 1) return setError(PB2_ERR_INVALID, "pb2_dist_init: one device per process (pb2_init), not a local device group");
    CUDA_TRY(cudaSetDevice(g_devs[0].id));
    NCCL_TRY(g_nccl.CommInitRank(&g_dist.comm, world, id, rank));
    return PB2_OK;
}

int pb2_dist_info(int *rank, int *world) {
    if (rank) *rank = g_dist.rank;
    if (world) *world = g_dist.world;
    return PB2_OK;
}

int pb2_dist_shutdown(void) {
    if (g_dist.comm) g_nccl.CommDestroy(g_dist.comm);
    g_dist.comm = nullptr;
    g_dist.rank = 0;
    g_dist.world = 1;
    return PB2_OK;
}

int pb2_host_alloc(size_t bytes, void **out) {
    if (!out) return setError(PB2_ERR_INVALID, "null argument");
    *out = nullptr;
    int rc = requireDevice();
    if (rc) return rc;
    CUDA_TRY(cudaMallocHost(out, std::max<size_t>(bytes, 1)));
    return PB2_OK;
}

int pb2_host_free(void *p) {
    if (p) cudaFreeHost(p);
    return PB2_OK;
}

int pb2_scene_destroy(pb2_scene *s) {
    if (!s) return PB2_OK;
    for (pb2_scene *r : s->replicas) pb2_scene_destroy(r);
    s->replicas.clear();
    if (g_initialised && (size_t)s->devIndex < g_devs.size()) cudaSetDevice(g_devs[(size_t)s->devIndex].id);
    for (void *p : s->allocations) cudaFree(p);
    if (s->film) cudaFree(s->film);
    if (s->filterTable) cudaFree(s->filterTable);
    if (s->wfCtx) cudaFree(s->wfCtx);
    if (s->wfQueues) cudaFree(s->wfQueues);
    if (s->wfCounts) cudaFree(s->wfCounts);
    if (s->wfHostCounts) cudaFreeHost(s->wfHostCounts);
    if (s->ldHostCounters) cudaFreeHost(s->ldHostCounters);
    for (cudaEvent_t e : s->traceEvents) cudaEventDestroy(e);
    if (s->wfSpill) cudaFree(s->wfSpill);
    if (s->paramBuf) cudaFree(s->paramBuf);
    for (int p = 0; p < 4; ++p) {
        if (s->pipeStreams[p]) cudaStreamDestroy(s->pipeStreams[p]);
        if (s->joinEvents[p]) cudaEventDestroy(s->joinEvents[p]);
    }
    if (s->forkEvent) cudaEventDestroy(s->forkEvent);
    delete s;
    if (g_initialised) cudaSetDevice(g_devs[0].id);
    return PB2_OK;
}

static int createSceneOnCurrentDevice(const pb2_scene_desc *d, pb2_scene **out);

// One copy of the scene per bound device (the BVH and every table are replicated, SURVEY.md section 8e); the handle is the
// primary device's copy, which owns the others.
int pb2_scene_create(const pb2_scene_desc *d, pb2_scene **out) {
    if (!d || !out) return setError(PB2_ERR_INVALID, "null argument");
    *out = nullptr;
    int rc = requireDevice();
    if (rc) return rc;
    t_dev = 0;
    CUDA_TRY(cudaSetDevice(g_devs[0].id));
    pb2_scene *primary = nullptr;
    if ((rc = createSceneOnCurrentDevice(d, &primary))) return rc;
    for (size_t i = 1; i < g_devs.size() && rc == PB2_OK; ++i) {
        t_dev = (int)i;
        pb2_scene *rep = nullptr;
        if (cudaSetDevice(g_devs[i].id) != cudaSuccess) rc = setError(PB2_ERR_CUDA, "cudaSetDevice failed");
        else if ((rc = createSceneOnCurrentDevice(d, &rep)) == PB2_OK) {
            rep->devIndex = (int)i;
            primary->replicas.push_back(rep);
        }
    }
    t_dev = 0;
    cudaSetDevice(g_devs[0].id);
    if (rc) {
        pb2_scene_destroy(primary);
        return rc;
    }
    *out = primary;
    return PB2_OK;
}

static int recordShadeFeatures(const pb2_scene_desc *d);
int pb2_shade_class(const pb2_scene_desc *d, int32_t *out) {
    if (!d || !out) return setError(PB2_ERR_INVALID, "null argument");
    if (d->n_materials < 0 || (d->n_materials > 0 && !d->materials) || d->n_lights < 0 || (d->n_lights > 0 && !d->lights))
        return setError(PB2_ERR_INVALID, "bad material or light records");
    *out = recordShadeFeatures(d) & SHADE_GENERAL;
    return PB2_OK;
}

// ---- image textures: the MIPMap constructor (src/core/mipmap.h:112-203) on the host --------------------------------------
// Lanczos (src/core/texture.cpp:254-262) with the default tau = 2
static float texLanczos(float x) {
    const float tau = 2;
    x = std::abs(x);
    if (x < 1e-5f) return 1;
    if (x > 1.f) return 0;
    x *= 3.14159265358979323846f;
    float sv = std::sin(x * tau) / (x * tau);
    float lanczos = std::sin(x) / x;
    return sv * lanczos;
}
struct TexResampleWeight {
    int firstTexel;
    float weight[4];
};
// MIPMap::resampleWeights (mipmap.h:75-94)
static std::vector<TexResampleWeight> texResampleWeights(int oldRes, int newRes) {
    std::vector<TexResampleWeight> wt((size_t)newRes);
    const float filterwidth = 2.f;
    for (int i = 0; i < newRes; ++i) {
        float center = (i + .5f) * oldRes / newRes;
        wt[i].firstTexel = (int)std::floor((center - filterwidth) + 0.5f);
        for (int j = 0; j < 4; ++j) {
            float pos = wt[i].firstTexel + j + .5f;
            wt[i].weight[j] = texLanczos((pos - center) / filterwidth);
        }
        float invSumWts = 1 / (wt[i].weight[0] + wt[i].weight[1] + wt[i].weight[2] + wt[i].weight[3]);
        for (int j = 0; j < 4; ++j) wt[i].weight[j] *= invSumWts;
    }
    return wt;
}
static int texWrapIndex(int i, int n, int wrap) {   // the index a wrap mode turns i into, or -1 (black)
    if (wrap == PB2_WRAP_REPEAT) return texMod(i, n);
    if (wrap == PB2_WRAP_CLAMP) return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
    return (i >= 0 && i < n) ? i : -1;
}
// Appends the levels of one texture to `pool` (finest first) and fills its DTexture.
static int buildTexturePyramid(const pb2_texture &in, std::vector<float> &pool, DTexture *out) {
    if (in.kind != PB2_TEXKIND_IMAGE) return setError(PB2_ERR_INVALID, "texture: not an image (a constant or a combinator has no pyramid)");
    if ((in.channels != 1 && in.channels != 3) || in.width <= 0 || in.height <= 0 || !in.texels)
        return setError(PB2_ERR_INVALID, "texture: channels must be 1 or 3, the resolution positive, texels not null");
    if (in.wrap < PB2_WRAP_REPEAT || in.wrap > PB2_WRAP_CLAMP) return setError(PB2_ERR_INVALID, "texture: unknown wrap mode");
    if (in.width > 32768 || in.height > 32768) return setError(PB2_ERR_UNSUPPORTED, "texture larger than 32768 in one direction");
    const int C = in.channels;
    int rw = in.width, rh = in.height;
    std::vector<float> level0;
    auto isPow2 = [](int v) { return v && !(v & (v - 1)); };
    auto roundUpPow2 = [](int v) { int p = 1; while (p < v) p <<= 1; return p; };
    if (!isPow2(rw) || !isPow2(rh)) {
        // resample to a power of two: first in s, then in t (mipmap.h:128-176)
        const int pw = roundUpPow2(rw), ph = roundUpPow2(rh);
        std::vector<float> img((size_t)pw * ph * C, 0.f);
        std::vector<TexResampleWeight> sW = texResampleWeights(rw, pw);
        for (int t = 0; t < rh; ++t)
            for (int sx = 0; sx < pw; ++sx)
                for (int c = 0; c < C; ++c) {
                    float v = 0.f;
                    for (int j = 0; j < 4; ++j) {
                        int origS = texWrapIndex(sW[sx].firstTexel + j, rw, in.wrap);
                        if (origS >= 0 && origS < rw) v += sW[sx].weight[j] * in.texels[((size_t)t * rw + origS) * C + c];
                    }
                    img[((size_t)t * pw + sx) * C + c] = v;
                }
        std::vector<TexResampleWeight> tW = texResampleWeights(rh, ph);
        std::vector<float> work((size_t)ph);
        for (int sx = 0; sx < pw; ++sx)
            for (int c = 0; c < C; ++c) {
                for (int t = 0; t < ph; ++t) {
                    float v = 0.f;
                    for (int j = 0; j < 4; ++j) {
                        int offset = texWrapIndex(tW[t].firstTexel + j, rh, in.wrap);
                        if (offset >= 0 && offset < rh) v += tW[t].weight[j] * img[((size_t)offset * pw + sx) * C + c];
                    }
                    work[t] = v;
                }
                for (int t = 0; t < ph; ++t) img[((size_t)t * pw + sx) * C + c] = work[t] < 0.f ? 0.f : work[t];   // clamp(v, 0, Infinity)
            }
        level0.swap(img);
        rw = pw;
        rh = ph;
    } else
        level0.assign(in.texels, in.texels + (size_t)rw * rh * C);
    int nLevels = 1;
    for (int m = std::max(rw, rh); m > 1; m >>= 1) ++nLevels;   // 1 + Log2Int(max)
    memset(out, 0, sizeof(*out));
    out->channels = C;
    out->nLevels = nLevels;
    out->w = rw;
    out->h = rh;
    out->wrap = in.wrap;
    out->doTrilinear = in.do_trilinear != 0;
    out->maxAniso = in.max_anisotropy;
    out->su = in.su; out->sv = in.sv; out->du = in.du; out->dv = in.dv;
    out->levelOfs[0] = (long long)pool.size();
    pool.insert(pool.end(), level0.begin(), level0.end());
    int pw = rw, ph = rh;
    for (int i = 1; i < nLevels; ++i) {
        // each coarser level: the mean of four texels of the finer one, fetched through the wrap mode (mipmap.h:186-194)
        const int sRes = std::max(1, pw / 2), tRes = std::max(1, ph / 2);
        const size_t prev = (size_t)out->levelOfs[i - 1];
        out->levelOfs[i] = (long long)pool.size();
        pool.resize(pool.size() + (size_t)sRes * tRes * C);
        float *dst = pool.data() + out->levelOfs[i];
        const float *src = pool.data() + prev;
        auto texel = [&](int sx, int t, int c) -> float {
            sx = texWrapIndex(sx, pw, in.wrap);
            t = texWrapIndex(t, ph, in.wrap);
            if (sx < 0 || t < 0) return 0.f;
            return src[((size_t)t * pw + sx) * C + c];
        };
        for (int t = 0; t < tRes; ++t)
            for (int sx = 0; sx < sRes; ++sx)
                for (int c = 0; c < C; ++c)
                    dst[((size_t)t * sRes + sx) * C + c] =
                        .25f * (texel(2 * sx, 2 * t, c) + texel(2 * sx + 1, 2 * t, c) + texel(2 * sx, 2 * t + 1, c) + texel(2 * sx + 1, 2 * t + 1, c));
        pw = sRes;
        ph = tRes;
    }
    return PB2_OK;
}

static void texWeightLut(std::vector<float> &pool);
// The pyramids as they are uploaded, kept on the host while the scene is being created (an infinite light with an
// environment map derives its sampling distribution from them).
struct HostTextures {
    std::vector<float> pool;
    std::vector<DTexture> tex;
};
static int buildHostTextures(const pb2_scene_desc *d, HostTextures *host);
static int uploadTextures(pb2_scene *s, const pb2_scene_desc *d, HostTextures *host) {
    DScene &sc = s->d;
    if (d->n_textures <= 0) return PB2_OK;
    int rc = buildHostTextures(d, host);
    if (rc) return rc;
    if ((rc = upload(s, host->tex.data(), host->tex.size(), &sc.textures))) return rc;
    if ((rc = upload(s, host->pool.data(), host->pool.size(), &sc.texels))) return rc;
    sc.nTextures = d->n_textures;
    return PB2_OK;
}
// The pyramids of the image textures and the records of all textures, in host memory
static int buildHostTextures(const pb2_scene_desc *d, HostTextures *host) {
    if (!d->textures) return setError(PB2_ERR_INVALID, "n_textures > 0 but textures is null");
    std::vector<float> &pool = host->pool;
    texWeightLut(pool);
    std::vector<DTexture> &tex = host->tex;
    tex.resize((size_t)d->n_textures);
    std::vector<int> depth((size_t)d->n_textures, 0);
    for (int i = 0; i < d->n_textures; ++i) {
        const pb2_texture &in = d->textures[i];
        if (in.kind == PB2_TEXKIND_IMAGE) {
            int rc = buildTexturePyramid(in, pool, &tex[i]);
            if (rc) return rc;
            continue;
        }
        // a constant or a combinator (scale.h, mix.h): children must come before it, agree in channels, stay TEX_MAX_DEPTH deep
        DTexture &t = tex[i];
        memset(&t, 0, sizeof(t));
        if (in.channels != 1 && in.channels != 3) return setError(PB2_ERR_INVALID, "texture: channels must be 1 or 3");
        t.channels = in.channels;
        t.kind = in.kind;
        for (int c = 0; c < 3; ++c) t.value[c] = in.value[in.channels == 3 ? c : 0];
        if (in.kind == PB2_TEXKIND_CONSTANT) continue;
        t.su = in.su; t.sv = in.sv; t.du = in.du; t.dv = in.dv;   // the UVMapping2D of a checkerboard / uv texture
        if (in.kind == PB2_TEXKIND_UV) {
            if (in.channels != 3) return setError(PB2_ERR_INVALID, "texture: a uv texture has three channels");
            continue;
        }
        if (in.kind == PB2_TEXKIND_CHECKERBOARD) t.value[0] = in.value[0];   // the antialiasing mode, not a colour
        else if (in.kind != PB2_TEXKIND_SCALE && in.kind != PB2_TEXKIND_MIX) return setError(PB2_ERR_INVALID, "texture: unknown kind");
        const int nChildren = in.kind == PB2_TEXKIND_MIX ? 3 : 2;
        for (int c = 0; c < nChildren; ++c) {
            const int id = in.child[c];
            if (id < 1 || id > i) return setError(PB2_ERR_INVALID, "texture combinator: a child must precede its parent in the texture array");
            const int want = (in.kind == PB2_TEXKIND_MIX && c == 2) ? 1 : in.channels;
            if (d->textures[id - 1].channels != want) return setError(PB2_ERR_INVALID, "texture combinator: child with the wrong number of channels");
            t.child[c] = id;
            depth[i] = std::max(depth[i], depth[(size_t)id - 1] + 1);
        }
        if (depth[i] > TEX_MAX_DEPTH) return setError(PB2_ERR_UNSUPPORTED, "texture combinators nested more than three levels deep");
    }
    return PB2_OK;
}

// Texture::Evaluate for texture `id` of a texture array at n points given by (u, v) and (dudx, dvdx, dudy, dvdy), evaluated on
// the HOST by the functions the kernels compile (texEvaluateNode): parity / debug entry point, no device needed.
extern "C" int pb2_texture_eval_host(const pb2_texture *textures, int32_t n_textures, int32_t id, int64_t n, const float *uv,
                                     const float *duv, float *out) {
    if (!textures || n_textures <= 0 || id < 0 || id >= n_textures || (n > 0 && (!uv || !duv || !out))) return setError(PB2_ERR_INVALID, "bad argument");
    pb2_scene_desc d;
    memset(&d, 0, sizeof(d));
    d.n_textures = n_textures;
    d.textures = textures;
    HostTextures host;
    int rc = buildHostTextures(&d, &host);
    if (rc) return rc;
    for (int64_t i = 0; i < n; ++i) {
        DUvDiff dd;
        dd.dudx = duv[4 * i];
        dd.dvdx = duv[4 * i + 1];
        dd.dudy = duv[4 * i + 2];
        dd.dvdy = duv[4 * i + 3];
        const V3 v = texEvaluateNode(host.tex.data(), host.pool.data(), id, mk2(uv[2 * i], uv[2 * i + 1]), dd);
        out[3 * i] = v.x;
        out[3 * i + 1] = v.y;
        out[3 * i + 2] = v.z;
    }
    return PB2_OK;
}

static void texWeightLut(std::vector<float> &pool) {   // MIPMap::weightLut (mipmap.h:196-202)
    pool.assign((size_t)TEX_LUT_SIZE, 0.f);
    for (int i = 0; i < TEX_LUT_SIZE; ++i) {
        float alpha = 2;
        float r2 = float(i) / float(TEX_LUT_SIZE - 1);
        pool[i] = std::exp(-alpha * r2) - std::exp(-alpha);
    }
}

extern "C" int pb2_texture_pyramid(const pb2_texture *texture, int32_t level, int32_t *n_levels, int32_t *w, int32_t *h, float *out) {
    if (!texture || !n_levels || !w || !h) return setError(PB2_ERR_INVALID, "null argument");
    std::vector<float> pool;
    DTexture t;
    int rc = buildTexturePyramid(*texture, pool, &t);
    if (rc) return rc;
    if (level < 0 || level >= t.nLevels) return setError(PB2_ERR_INVALID, "texture level out of range");
    *n_levels = t.nLevels;
    *w = std::max(1, t.w >> level);
    *h = std::max(1, t.h >> level);
    if (out) memcpy(out, pool.data() + t.levelOfs[level], (size_t)*w * *h * t.channels * sizeof(float));
    return PB2_OK;
}

__global__ void k_texture_lookup(DTexture tx, const float *pool, int64_t n, const float *st, const float *dst, float *out) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    V3 v = texLookup(tx, pool, mk2(st[2 * i], st[2 * i + 1]), mk2(dst[4 * i], dst[4 * i + 1]), mk2(dst[4 * i + 2], dst[4 * i + 3]));
    out[3 * i] = v.x;
    out[3 * i + 1] = v.y;
    out[3 * i + 2] = v.z;
}

extern "C" int pb2_texture_lookup(const pb2_texture *texture, int64_t n, const float *st, const float *dst, float *out) {
    if (!g_initialised) return setError(PB2_ERR_NO_DEVICE, "pb2_init was not called or failed (no CUDA device: this library has no CPU fallback)");
    if (!texture || n < 0 || (n > 0 && (!st || !dst || !out))) return setError(PB2_ERR_INVALID, "null argument");
    std::vector<float> pool;
    texWeightLut(pool);
    DTexture t;
    int rc = buildTexturePyramid(*texture, pool, &t);
    if (rc || n == 0) return rc;
    float *dPool = nullptr, *dSt = nullptr, *dDst = nullptr, *dOut = nullptr;
    cudaError_t e = cudaMalloc((void **)&dPool, pool.size() * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dSt, (size_t)n * 2 * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dDst, (size_t)n * 4 * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dOut, (size_t)n * 3 * sizeof(float));
    if (e == cudaSuccess) e = cudaMemcpy(dPool, pool.data(), pool.size() * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dSt, st, (size_t)n * 2 * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dDst, dst, (size_t)n * 4 * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        k_texture_lookup<<<(unsigned)((n + 127) / 128), 128>>>(t, dPool, n, dSt, dDst, dOut);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dOut, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(dPool);
    cudaFree(dSt);
    cudaFree(dDst);
    cudaFree(dOut);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, cudaGetErrorString(e));
    return PB2_OK;
}

// The Distribution2D of an InfiniteAreaLight over its environment map (infinite.cpp:64-82, sampling.cpp:52-62) as one table:
// 2h rows of [func(2w) | cdf(2w + 1) | funcInt], then the marginal [func(2h) | cdf(2h + 1) | funcInt].
static int buildEnvDistribution(const DTexture &tx, const float *pool, std::vector<float> *out) {
    const int width = 2 * tx.w, height = 2 * tx.h;
    if ((size_t)width * height > ((size_t)1 << 27)) return setError(PB2_ERR_UNSUPPORTED, "environment map too large for its sampling table");
    const size_t rowStride = 2 * (size_t)width + 2;
    std::vector<float> &table = *out;
    table.assign((size_t)height * rowStride + 2 * (size_t)height + 2, 0.f);
    const float fwidth = 0.5f / std::min(width, height);
    for (int v = 0; v < height; ++v) {
        const float vp = (v + .5f) / (float)height;
        const float sinTheta = std::sin(3.14159265358979323846f * (v + .5f) / height);
        float *row = table.data() + (size_t)v * rowStride;
        for (int u = 0; u < width; ++u) {
            const float up = (u + .5f) / (float)width;
            const V3 c = texLookupWidth(tx, pool, mk2(up, vp), fwidth);
            row[u] = 0.212671f * c.x + 0.715160f * c.y + 0.072169f * c.z;   // RGBSpectrum::y()
            row[u] *= sinTheta;
        }
        finishVoxelDistribution(width, row);   // Distribution1D's constructor over [func | cdf | funcInt] (sampling.h:57-70)
    }
    float *marginal = table.data() + (size_t)height * rowStride;
    for (int v = 0; v < height; ++v) marginal[v] = table[(size_t)v * rowStride + 2 * (size_t)width + 1];
    finishVoxelDistribution(height, marginal);
    return PB2_OK;
}

extern "C" int pb2_env_distribution(const pb2_texture *texture, int32_t *nu, int32_t *nv, float *out) {
    if (!texture || !nu || !nv) return setError(PB2_ERR_INVALID, "null argument");
    std::vector<float> pool;
    texWeightLut(pool);
    DTexture t;
    int rc = buildTexturePyramid(*texture, pool, &t);
    if (rc) return rc;
    *nu = 2 * t.w;
    *nv = 2 * t.h;
    if (!out) return PB2_OK;
    std::vector<float> table;
    if ((rc = buildEnvDistribution(t, pool.data(), &table))) return rc;
    memcpy(out, table.data(), table.size() * sizeof(float));
    return PB2_OK;
}

// The shade features of the scene's material and light records (SHADE_* in device/pb2_shade.cuh): a bit stays clear only
// when no record of the scene can take the branch it stands for, so kernels compiled without it compute what the general
// ones do.  PB2_SHADE_GENERAL=1 gives every scene the general class (tests compare the two).
static int recordShadeFeatures(const pb2_scene_desc *d) {
    static const bool forceGeneral = envInt("PB2_SHADE_GENERAL", 0) != 0;
    int fc = forceGeneral ? SHADE_GENERAL : 0;
    for (int i = 0; i < d->n_materials; ++i) {
        const pb2_material &m = d->materials[i];
        if (m.type == PB2_MAT_NONE) continue;
        if (m.type == PB2_MAT_MATTE) {
            // makeBsdf: an Oren-Nayar lobe unless clamp(sigma, 0, 90) == 0 (sigma <= 0; a NaN or textured sigma counts)
            if (m.tex[PB2_TEX_SIGMA] || !(m.sigma <= 0.f)) fc |= SHADE_OREN_NAYAR;
        } else if (m.type == PB2_MAT_PLASTIC)
            fc |= SHADE_MICROFACET;
        else
            fc |= SHADE_SPECULAR | SHADE_GENERAL;   // the specular family: its kernels are compiled for the general class
    }
    for (int i = 0; i < d->n_lights; ++i)
        if (d->lights[i].type != PB2_LIGHT_AREA) fc |= SHADE_NON_AREA;
    return fc;
}

static int createSceneOnCurrentDevice(const pb2_scene_desc *d, pb2_scene **out) {
    int rc = PB2_OK;
    if (d->n_prims <= 0 || d->n_nodes <= 0 || !d->nodes || !d->bvh_prims || !d->prim_type || !d->prim_index)
        return setError(PB2_ERR_INVALID, "scene has no primitives / BVH");
    if (d->n_prims > 0x7fffffffLL || d->n_nodes > 0x7fffffffLL) return setError(PB2_ERR_UNSUPPORTED, "more than 2^31 primitives/nodes");
    for (int i = 0; i < d->n_materials; ++i)
        if (d->materials[i].type < PB2_MAT_NONE || d->materials[i].type > PB2_MAT_UBER)
            return setError(PB2_ERR_UNSUPPORTED, "material type outside the path's scope (matte, plastic, substrate, metal, uber, mirror, glass)");
    // texture references: in range, one channel for float parameters and alpha masks, three for spectra
    for (int i = 0; i < d->n_materials; ++i)
        for (int k = 0; k < PB2_TEX_SLOTS; ++k) {
            const int id = d->materials[i].tex[k];
            if (!id) continue;
            if (id < 0 || id > d->n_textures || !d->textures) return setError(PB2_ERR_INVALID, "material texture index out of range");
            const bool spectrum = k == PB2_TEX_KD || k == PB2_TEX_KS || k == PB2_TEX_KR || k == PB2_TEX_KT || k == PB2_TEX_OPACITY ||
                                  k == PB2_TEX_METAL_ETA || k == PB2_TEX_METAL_K;
            if (d->textures[id - 1].channels != (spectrum ? 3 : 1))
                return setError(PB2_ERR_INVALID, "material texture has the wrong number of channels for its parameter");
        }
    bool hasAlpha = false;
    for (int i = 0; i < d->n_meshes; ++i)
        for (int id : {d->meshes[i].alpha_tex, d->meshes[i].shadow_alpha_tex}) {
            if (!id) continue;
            if (id < 0 || id > d->n_textures || !d->textures || d->textures[id - 1].channels != 1)
                return setError(PB2_ERR_INVALID, "mesh alpha texture: index out of range or not a one-channel texture");
            hasAlpha = true;
        }
    struct Guard {
        pb2_scene *s;
        ~Guard() { if (s) pb2_scene_destroy(s); }
    } guard{new pb2_scene()};
    pb2_scene *s = guard.s;
    s->devIndex = t_dev;
    s->shadeFeatures = recordShadeFeatures(d);
    DScene &sc = s->d;
    memset(&sc, 0, sizeof(sc));
    sc.nNodes = d->n_nodes;
    sc.nPrims = d->n_prims;
    sc.nTris = d->n_tris;
    sc.nLights = d->n_lights;
    s->nPrims = d->n_prims;
    s->nLights = d->n_lights;
    // the scene's BVHs: one, or the scene BVH followed by one per instanced object
    std::vector<pb2_bvh> bvhs;
    int64_t nBvhPrims = d->n_prims;
    if (d->n_bvhs >= 1) {
        if (!d->bvhs) return setError(PB2_ERR_INVALID, "n_bvhs > 0 but bvhs is null");
        bvhs.assign(d->bvhs, d->bvhs + d->n_bvhs);
        nBvhPrims = d->n_bvh_prims;
        if (nBvhPrims <= 0 || nBvhPrims > d->n_prims) return setError(PB2_ERR_INVALID, "bad n_bvh_prims");
    } else
        bvhs.push_back(pb2_bvh{0, d->n_nodes, 0, d->n_prims});
    if (d->n_instances < 0 || (d->n_instances > 0 && !d->instances)) return setError(PB2_ERR_INVALID, "bad instances");
    for (const pb2_bvh &b : bvhs)
        if (b.node_offset < 0 || b.n_nodes <= 0 || b.node_offset + b.n_nodes > d->n_nodes || b.prim_offset < 0 || b.n_prims <= 0 ||
            b.prim_offset + b.n_prims > nBvhPrims)
            return setError(PB2_ERR_INVALID, "BVH range out of bounds");
    // device copy of the nodes with every index made global (secondChildOffset += node_offset,
    // primitivesOffset += prim_offset); bvhs[0] starts at 0, so a scene without instances is uploaded verbatim
    std::vector<pb2_bvh_node> rebased;
    if (bvhs.size() > 1) rebased.assign(d->nodes, d->nodes + d->n_nodes);
    s->bvhDepth = 0;
    for (size_t k = 0; k < bvhs.size(); ++k) {
        // depth of the tree = deepest traversal stack any ray can need (selects the shared-memory-stack kernel)
        const pb2_bvh &b = bvhs[k];
        std::vector<std::pair<int64_t, int>> todo{{0, 0}};
        int depth = 0;
        while (!todo.empty()) {
            std::pair<int64_t, int> nd = todo.back();
            todo.pop_back();
            if (nd.first < 0 || nd.first >= b.n_nodes) return setError(PB2_ERR_INVALID, "BVH child index out of range");
            depth = std::max(depth, nd.second);
            const pb2_bvh_node &node = d->nodes[b.node_offset + nd.first];
            if (node.n_prims == 0) {
                if (nd.second > 4096) return setError(PB2_ERR_INVALID, "BVH is not a tree");
                todo.push_back({nd.first + 1, nd.second + 1});
                todo.push_back({(int64_t)node.offset, nd.second + 1});
                if (!rebased.empty()) rebased[b.node_offset + nd.first].offset = (int32_t)(node.offset + b.node_offset);
            } else {
                if ((int64_t)node.offset + node.n_prims > b.n_prims || node.offset < 0)
                    return setError(PB2_ERR_INVALID, "BVH leaf range out of bounds");
                if (!rebased.empty()) rebased[b.node_offset + nd.first].offset = (int32_t)(node.offset + b.prim_offset);
            }
        }
        if (depth > 64) return setError(PB2_ERR_UNSUPPORTED, "BVH deeper than the reference's 64-entry traversal stack (bvh.cpp:671)");
        if (k == 0) s->bvhDepth = depth;
        else s->instDepth = std::max(s->instDepth, depth);
    }
    for (int64_t j = 0; j < nBvhPrims; ++j)
        if (d->bvh_prims[j] < 0 || d->bvh_prims[j] >= d->n_prims) return setError(PB2_ERR_INVALID, "bvh_prims entry out of range");
    for (int64_t i = 0; i < d->n_prims; ++i) {
        if (d->prim_type[i] == PB2_PRIM_INSTANCE) {
            if (d->prim_index[i] < 0 || d->prim_index[i] >= d->n_instances) return setError(PB2_ERR_INVALID, "instance index out of range");
        } else if (d->prim_type[i] != PB2_PRIM_TRIANGLE && d->prim_type[i] != PB2_PRIM_SPHERE)
            return setError(PB2_ERR_UNSUPPORTED, "primitive type outside the path's scope");
    }
    const pb2_bvh_node *nodes;
    if ((rc = upload(s, rebased.empty() ? d->nodes : rebased.data(), (size_t)d->n_nodes, &nodes))) return rc;
    sc.instances = nullptr;
    sc.nInstances = d->n_instances;
    std::vector<DInstance> inst((size_t)std::max(0, d->n_instances));   // uploaded below, once the record numbers are known
    if (d->n_instances > 0) {
        const float identity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
        for (int i = 0; i < d->n_instances; ++i) {
            const pb2_instance &pi = d->instances[i];
            memcpy(inst[i].i2w.m, pi.instance_to_world, sizeof(float) * 16);
            memcpy(inst[i].w2i.m, pi.world_to_instance, sizeof(float) * 16);
            inst[i].identity = memcmp(pi.instance_to_world, identity, sizeof(identity)) == 0;   // Transform::IsIdentity (transform.h:137-143)
            inst[i].wroot = pi.bvh >= 0 ? pi.bvh : -1;   // the pseudo record above the object BVH's root (two-child records)
            inst[i].wroot4 = -1;
            if (pi.bvh >= 0) {
                if (pi.bvh == 0 || pi.bvh >= (int)bvhs.size()) return setError(PB2_ERR_INVALID, "instance BVH out of range");
                inst[i].root = (int)bvhs[pi.bvh].node_offset;
                inst[i].lone = -1;
            } else {
                if (pi.lone_prim < 0 || pi.lone_prim >= nBvhPrims) return setError(PB2_ERR_INVALID, "instance primitive out of range");
                if (d->prim_type[d->bvh_prims[pi.lone_prim]] == PB2_PRIM_INSTANCE) return setError(PB2_ERR_INVALID, "instance of an instance");
                inst[i].root = -1;
                inst[i].lone = pi.lone_prim;
            }
        }
        for (size_t k = 1; k < bvhs.size(); ++k)
            for (int64_t j = 0; j < bvhs[k].n_prims; ++j)
                if (d->prim_type[d->bvh_prims[bvhs[k].prim_offset + j]] == PB2_PRIM_INSTANCE)
                    return setError(PB2_ERR_INVALID, "instance inside an object BVH (api.cpp:1554-1557 forbids it)");
    }
    sc.nodes = reinterpret_cast<const float4 *>(nodes);
    sc.wide = nullptr;
    sc.wide4 = nullptr;
    if (d->n_nodes > 0 && d->n_prims < (int64_t)WIDE_MAX_PRIMS) {
        // two-child records (pb2_scene.cuh): interior nodes keep their depth-first order; records
        // 0 .. nBvh-1 are the pseudo nodes above the root of each BVH (scene BVH, then instanced objects)
        const pb2_bvh_node *src = rebased.empty() ? d->nodes : rebased.data();   // indices global across BVHs
        const int32_t nBvh = (int32_t)bvhs.size();
        std::vector<int32_t> wideOf((size_t)d->n_nodes, -1);
        int32_t nWide = nBvh;
        bool fits = true;
        for (int64_t i = 0; i < d->n_nodes; ++i) {
            if (src[i].n_prims == 0) wideOf[i] = nWide++;
            else if (src[i].n_prims > WIDE_MAX_LEAF) fits = false;
        }
        if (fits) {
            struct WideRec { float b[12]; uint32_t ref0, ref1, meta, pad; };
            static_assert(sizeof(WideRec) == 64, "wide record is 64 bytes");
            std::vector<WideRec> wide((size_t)nWide);
            auto childRef = [&](int64_t i) -> uint32_t {
                const pb2_bvh_node &n = src[i];
                return n.n_prims == 0 ? (uint32_t)wideOf[i] : (WIDE_LEAF | ((uint32_t)(n.n_prims - 1) << WIDE_LEAF_COUNT_SHIFT) | (uint32_t)n.offset);
            };
            auto putBox = [&](float *dst, const pb2_bvh_node &n) {
                dst[0] = n.bmin[0]; dst[1] = n.bmin[1]; dst[2] = n.bmin[2];
                dst[3] = n.bmax[0]; dst[4] = n.bmax[1]; dst[5] = n.bmax[2];
            };
            memset(wide.data(), 0, wide.size() * sizeof(WideRec));
            for (int32_t k = 0; k < nBvh; ++k) {
                const int64_t root = bvhs[(size_t)k].node_offset;
                putBox(wide[(size_t)k].b, src[root]);
                putBox(wide[(size_t)k].b + 6, src[root]);
                wide[(size_t)k].ref0 = wide[(size_t)k].ref1 = childRef(root);
                wide[(size_t)k].meta = WIDE_SINGLE;
            }
            for (int64_t i = 0; i < d->n_nodes; ++i) {
                const pb2_bvh_node &n = src[i];
                if (n.n_prims != 0) continue;
                WideRec &w = wide[(size_t)wideOf[i]];
                putBox(w.b, src[i + 1]);
                putBox(w.b + 6, src[n.offset]);
                w.ref0 = childRef(i + 1);
                w.ref1 = childRef(n.offset);
                w.meta = (uint32_t)n.axis & 3u;
            }
            const WideRec *dWide;
            if ((rc = upload(s, wide.data(), wide.size(), &dWide))) return rc;
            sc.wide = reinterpret_cast<const float4 *>(dWide);
            // four-child records (device/pb2_wide4.cuh): every BVH's root gets a record of its own
            std::vector<int64_t> roots(bvhs.size());
            for (size_t k = 0; k < bvhs.size(); ++k) roots[k] = bvhs[k].node_offset;
            std::vector<int32_t> rootRecord(bvhs.size(), 0);
            const std::vector<float4> wide4 = buildWide4Records(src, roots.data(), roots.size(), rootRecord.data());
            const float4 *dWide4;
            if ((rc = upload(s, wide4.data(), wide4.size(), &dWide4))) return rc;
            sc.wide4 = dWide4;
            for (int i = 0; i < d->n_instances; ++i)
                inst[(size_t)i].wroot4 = d->instances[i].bvh >= 0 ? rootRecord[(size_t)d->instances[i].bvh] : -1;
        }
    }
    if (d->n_instances > 0) {
        const DInstance *dInst;
        if ((rc = upload(s, inst.data(), inst.size(), &dInst))) return rc;
        sc.instances = dInst;
    }
    if ((rc = upload(s, d->P, 3 * (size_t)d->n_vertices, &sc.P))) return rc;
    if ((rc = upload(s, d->N, d->N ? 3 * (size_t)d->n_vertices : 0, &sc.N))) return rc;
    if ((rc = upload(s, d->UV, d->UV ? 2 * (size_t)d->n_vertices : 0, &sc.UV))) return rc;
    if ((rc = upload(s, d->S, d->S ? 3 * (size_t)d->n_vertices : 0, &sc.S))) return rc;
    if ((rc = upload(s, d->tri_index, 3 * (size_t)d->n_tris, &sc.triIndex))) return rc;
    if ((rc = upload(s, d->tri_mesh, (size_t)d->n_tris, &sc.triMesh))) return rc;
    if ((rc = upload(s, d->meshes, (size_t)d->n_meshes, &sc.meshes))) return rc;
    if ((rc = upload(s, d->spheres, (size_t)d->n_spheres, &sc.spheres))) return rc;
    if ((rc = upload(s, d->prim_type, (size_t)d->n_prims, &sc.primType))) return rc;
    if ((rc = upload(s, d->prim_index, (size_t)d->n_prims, &sc.primIndex))) return rc;
    if ((rc = upload(s, d->prim_material, (size_t)d->n_prims, &sc.primMaterial))) return rc;
    if ((rc = upload(s, d->prim_light, (size_t)d->n_prims, &sc.primLight))) return rc;
    if ((rc = upload(s, d->materials, (size_t)d->n_materials, &sc.materials))) return rc;
    HostTextures hostTextures;
    if ((rc = uploadTextures(s, d, &hostTextures))) return rc;
    sc.hasAlpha = hasAlpha ? 1 : 0;
    if ((rc = upload(s, d->lights, (size_t)d->n_lights, &sc.lights))) return rc;
    sc.deltaLights = nullptr;
    for (int i = 0; i < d->n_lights; ++i) {
        if (d->lights[i].type < PB2_LIGHT_AREA || d->lights[i].type > PB2_LIGHT_INFINITE) return setError(PB2_ERR_INVALID, "unknown light type");
        if (d->lights[i].type != PB2_LIGHT_AREA && !d->delta_lights) return setError(PB2_ERR_INVALID, "a delta light without delta_lights");
    }
    std::vector<DDeltaLight> deltaLights;
    if (d->delta_lights && d->n_lights > 0) {
        deltaLights.resize(d->n_lights);
        memset(deltaLights.data(), 0, deltaLights.size() * sizeof(DDeltaLight));
        for (int i = 0; i < d->n_lights; ++i) {
            const pb2_delta_light &in = d->delta_lights[i];
            DDeltaLight &o = deltaLights[i];
            V3 p = mk3(in.p[0], in.p[1], in.p[2]);
            if (d->lights[i].type == PB2_LIGHT_DISTANT) p = normalize(p);   // distant.cpp:46
            o.p[0] = p.x; o.p[1] = p.y; o.p[2] = p.z;
            const float radPerDeg = 3.14159265358979323846f / 180;           // Radians() (pbrt.h:353), then std::cos(float) (spot.cpp:49-50)
            o.cosTotalWidth = std::cos(radPerDeg * in.total_width_deg);
            o.cosFalloffStart = std::cos(radPerDeg * in.falloff_start_deg);
            o.worldRadius = in.world_radius;
            for (int k = 0; k < 9; ++k) o.worldToLight[k] = in.world_to_light[k];
            for (int k = 0; k < 9; ++k) o.lightToWorld[k] = in.light_to_world[k];
            if (d->lights[i].type == PB2_LIGHT_INFINITE && in.env_tex) {
                // Environment map.  Lmap = MIPMap<RGBSpectrum>(resolution, texels) with the default filter parameters
                // (infinite.cpp:62): texture env_tex - 1 of the pool.  The sampling distribution (infinite.cpp:64-82): a
                // 2w x 2h image of Lmap->Lookup((u + .5) / width, (v + .5) / height, fwidth).y() * sin(theta), trilinear
                // look-ups evaluated here on the host by the functions the kernels use, then one Distribution1D per row
                // and the marginal over the rows' integrals (Distribution2D, sampling.cpp:52-62).
                if (sc.nInfinite >= 4) return setError(PB2_ERR_UNSUPPORTED, "more than four infinite lights");
                sc.infinite[sc.nInfinite++] = i;
                if (in.env_tex < 0 || in.env_tex > d->n_textures || d->textures[in.env_tex - 1].channels != 3)
                    return setError(PB2_ERR_INVALID, "infinite light: env_tex out of range or not a three-channel texture");
                const pb2_texture &pt = d->textures[in.env_tex - 1];
                if (pt.kind != PB2_TEXKIND_IMAGE) return setError(PB2_ERR_INVALID, "infinite light: the environment map must be an image");
                if (pt.wrap != PB2_WRAP_REPEAT || pt.do_trilinear || pt.max_anisotropy != 8.f)
                    return setError(PB2_ERR_INVALID, "infinite light: the environment map must carry MIPMap's default parameters (repeat, EWA, 8)");
                const DTexture &tx = hostTextures.tex[(size_t)in.env_tex - 1];
                const float *pool = hostTextures.pool.data();
                const int width = 2 * tx.w, height = 2 * tx.h;
                std::vector<float> table;
                if ((rc = buildEnvDistribution(tx, pool, &table))) return rc;
                const float *dTable = nullptr;
                if ((rc = upload(s, table.data(), table.size(), &dTable))) return rc;
                o.envDist = dTable;
                o.envNu = width;
                o.envNv = height;
                o.envTex = in.env_tex;
                // InfiniteAreaLight::Power's radiance (infinite.cpp:84-88), kept in dist[0..2] for the power light distribution
                const V3 pw = texLookupWidth(tx, pool, mk2(.5f, .5f), .5f);
                o.dist[0] = pw.x; o.dist[1] = pw.y; o.dist[2] = pw.z;
            } else if (d->lights[i].type == PB2_LIGHT_INFINITE) {
                if (sc.nInfinite >= 4) return setError(PB2_ERR_UNSUPPORTED, "more than four infinite lights");
                sc.infinite[sc.nInfinite++] = i;
                // The sampling distribution of the constructor (infinite.cpp:61-82) for the 1 x 1 map: a 2 x 2 image of
                // Lmap->Lookup((u + .5) / 2, (v + .5) / 2, width .25).y() * sin(Pi (v + .5) / 2); the look-up is
                // MIPMap::triangle(0, st) (level = log2(.25) < 0), evaluated in float as written (mipmap.h:264-274)
                const pb2_light &pl = d->lights[i];
                float img[4];
                for (int v = 0; v < 2; ++v) {
                    const float vp = (v + .5f) / (float)2;
                    const float sinTheta = std::sin(3.14159265358979323846f * (v + .5f) / 2);
                    for (int u = 0; u < 2; ++u) {
                        const float up = (u + .5f) / (float)2;
                        const float s_ = up * 1 - 0.5f, t_ = vp * 1 - 0.5f;
                        const int s0 = (int)std::floor(s_), t0 = (int)std::floor(t_);
                        const float ds = s_ - s0, dt = t_ - t0;
                        float rgb[3];
                        for (int c = 0; c < 3; ++c)
                            rgb[c] = ((1 - ds) * (1 - dt)) * pl.L[c] + ((1 - ds) * dt) * pl.L[c] + (ds * (1 - dt)) * pl.L[c] + (ds * dt) * pl.L[c];
                        img[u + v * 2] = 0.212671f * rgb[0] + 0.715160f * rgb[1] + 0.072169f * rgb[2];   // RGBSpectrum::y()
                        img[u + v * 2] *= sinTheta;
                    }
                }
                auto dist1D = [](const float *f, int n, float *rec) {   // Distribution1D ctor (sampling.h:57-70)
                    for (int k = 0; k < n; ++k) rec[k] = f[k];
                    float *cdf = rec + n;
                    cdf[0] = 0;
                    for (int k = 1; k < n + 1; ++k) cdf[k] = cdf[k - 1] + f[k - 1] / n;
                    const float funcInt = cdf[n];
                    if (funcInt == 0) for (int k = 1; k < n + 1; ++k) cdf[k] = float(k) / float(n);
                    else for (int k = 1; k < n + 1; ++k) cdf[k] /= funcInt;
                    rec[2 * n + 1] = funcInt;
                };
                dist1D(img, 2, o.dist);
                dist1D(img + 2, 2, o.dist + 6);
                const float marginal[2] = {o.dist[5], o.dist[6 + 5]};
                dist1D(marginal, 2, o.dist + 12);
            }
        }
        if ((rc = upload(s, deltaLights.data(), deltaLights.size(), &sc.deltaLights))) return rc;
    }
    for (int m = 0; m < d->n_meshes; ++m) {
        if (d->meshes[m].has_n && !d->N) return setError(PB2_ERR_INVALID, "mesh has_n but N is null");
        if (d->meshes[m].has_uv && !d->UV) return setError(PB2_ERR_INVALID, "mesh has_uv but UV is null");
        if (d->meshes[m].has_s && !d->S) return setError(PB2_ERR_INVALID, "mesh has_s but S is null");
    }
    // leaf records in BVH order
    const int32_t *bvhPrims;
    if ((rc = upload(s, d->bvh_prims, (size_t)nBvhPrims, &bvhPrims))) return rc;
    float4 *leaf;
    if ((rc = allocate(s, 3 * (size_t)nBvhPrims, &leaf))) return rc;
    {
        int threads = 256;
        int64_t blocks = (nBvhPrims + threads - 1) / threads;
        k_build_leaf_records<<<(unsigned)blocks, threads>>>(sc, bvhPrims, nBvhPrims, leaf);
        CUDA_TRY(cudaGetLastError());
    }
    sc.leafPrims = leaf;
    sc.lightRecs = nullptr;
    if (d->n_lights > 0) {
        // the same record for every area light's shape, in light order
        std::vector<int32_t> lightPrims(d->n_lights);
        for (int i = 0; i < d->n_lights; ++i) {
            if (d->lights[i].type != PB2_LIGHT_AREA) {
                lightPrims[i] = 0;   // delta lights have no shape; the record is never read
                continue;
            }
            if (d->lights[i].prim < 0 || d->lights[i].prim >= d->n_prims) return setError(PB2_ERR_INVALID, "light primitive out of range");
            lightPrims[i] = d->lights[i].prim;
        }
        const int32_t *dLightPrims;
        if ((rc = upload(s, lightPrims.data(), lightPrims.size(), &dLightPrims))) return rc;
        float4 *lrec;
        if ((rc = allocate(s, 3 * (size_t)d->n_lights, &lrec))) return rc;
        k_build_leaf_records<<<(unsigned)((d->n_lights + 255) / 256), 256>>>(sc, dLightPrims, d->n_lights, lrec);
        CUDA_TRY(cudaGetLastError());
        sc.lightRecs = lrec;
    }

    // light-sampling distribution (lightdistrib.cpp:48-66)
    DLightDist &ld = sc.lightDist;
    memset(&ld, 0, sizeof(ld));
    int nl = d->n_lights;
    ld.stride = 2 * nl + 2;
    ld.strategy = (nl <= 1) ? PB2_LIGHTDIST_UNIFORM : d->light_strategy;
    ld.boundsMin = mk3(d->nodes[0].bmin[0], d->nodes[0].bmin[1], d->nodes[0].bmin[2]);
    ld.boundsMax = mk3(d->nodes[0].bmax[0], d->nodes[0].bmax[1], d->nodes[0].bmax[2]);
    if (nl > 0 && ld.strategy != PB2_LIGHTDIST_SPATIAL) {
        // Distribution1D over constant 1 (uniform) or over Light::Power().y() (power)
        std::vector<float> rec(ld.stride);
        for (int i = 0; i < nl; ++i) {
            if (ld.strategy == PB2_LIGHTDIST_UNIFORM)
                rec[i] = 1.f;
            else {
                // DiffuseAreaLight::Power (diffuse.cpp:64-66): (twoSided ? 2 : 1) * Lemit * area * Pi, then y()
                const pb2_light &l = d->lights[i];
                const float Pi = 3.14159265358979323846f;
                float s2 = l.two_sided ? 2.f : 1.f;
                float p[3];
                for (int c = 0; c < 3; ++c) {
                    if (l.type == PB2_LIGHT_POINT)          // point.cpp:54: 4 * Pi * I
                        p[c] = l.L[c] * (4 * Pi);
                    else if (l.type == PB2_LIGHT_SPOT)      // spot.cpp:74-76: I * 2 * Pi * (1 - .5f * (cosFalloffStart + cosTotalWidth))
                        p[c] = ((l.L[c] * 2) * Pi) * (1 - .5f * (deltaLights[i].cosFalloffStart + deltaLights[i].cosTotalWidth));
                    else if (l.type == PB2_LIGHT_DISTANT)   // distant.cpp:61-63: L * Pi * worldRadius * worldRadius
                        p[c] = ((l.L[c] * Pi) * deltaLights[i].worldRadius) * deltaLights[i].worldRadius;
                    else if (l.type == PB2_LIGHT_INFINITE)  // infinite.cpp:84-88: Pi * r * r * Lookup((.5, .5), .5) (constant: the texel itself)
                        p[c] = ((Pi * deltaLights[i].worldRadius) * deltaLights[i].worldRadius) * (deltaLights[i].envTex ? deltaLights[i].dist[c] : l.L[c]);
                    else
                        p[c] = ((s2 * l.L[c]) * l.area) * Pi;
                }
                rec[i] = 0.212671f * p[0] + 0.715160f * p[1] + 0.072169f * p[2];
            }
        }
        float *cdf = rec.data() + nl;
        cdf[0] = 0;
        for (int i = 1; i < nl + 1; ++i) cdf[i] = cdf[i - 1] + rec[i - 1] / nl;
        float funcInt = cdf[nl];
        if (funcInt == 0) {
            for (int i = 1; i < nl + 1; ++i) cdf[i] = float(i) / float(nl);
        } else {
            for (int i = 1; i < nl + 1; ++i) cdf[i] /= funcInt;
        }
        rec[2 * nl + 1] = funcInt;
        if ((rc = upload(s, rec.data(), rec.size(), &ld.table))) return rc;
    } else if (nl > 0) {
        // SpatialLightDistribution ctor (lightdistrib.cpp:96-122)
        float diag[3] = {ld.boundsMax.x - ld.boundsMin.x, ld.boundsMax.y - ld.boundsMin.y, ld.boundsMax.z - ld.boundsMin.z};
        int maxExtent = (diag[0] > diag[1] && diag[0] > diag[2]) ? 0 : (diag[1] > diag[2] ? 1 : 2);
        float bmax = diag[maxExtent];
        int maxVoxels = d->spatial_max_voxels > 0 ? d->spatial_max_voxels : 64;
        for (int i = 0; i < 3; ++i) ld.nVoxels[i] = std::max(1, int(std::round(diag[i] / bmax * maxVoxels)));
        size_t nVox = (size_t)ld.nVoxels[0] * ld.nVoxels[1] * ld.nVoxels[2];
        const size_t recordBytes = (size_t)ld.stride * sizeof(float);
        // One record per voxel up front when that is small (a few lights: 6 MB for the bench scene); otherwise - every
        // emissive triangle is a light, a mesh of them makes records of kilobytes - records only for the voxels that path
        // vertices fall into, built on demand into a bounded pool (the reference's lazily filled hash table,
        // lightdistrib.cpp:141-230).  PB2_LIGHTDIST_LAZY=1 forces the lazy form (tests).
        const size_t eagerLimit = (size_t)std::max(1, envInt("PB2_LIGHTDIST_EAGER_MB", 256)) << 20;
        const bool lazy = envInt("PB2_LIGHTDIST_LAZY", 0) != 0 || nVox * recordBytes > eagerLimit;
        if (!lazy) {
            float *table;
            if ((rc = allocate(s, nVox * ld.stride, &table))) return rc;
            ld.table = table;
            int threads = 128;
            k_spatial_light_dist<<<(unsigned)((nVox + threads - 1) / threads), threads>>>(sc, haltonTablesOnly(), table);
            CUDA_TRY(cudaGetLastError());
        } else {
            const size_t poolLimit = (size_t)std::max(1, envInt("PB2_LIGHTDIST_POOL_MB", 2048)) << 20;
            const size_t records = std::max<size_t>(1, std::min(nVox, poolLimit / recordBytes));
            float *table;
            if ((rc = allocate(s, records * ld.stride, &table))) return rc;
            ld.table = table;
            ld.poolRecords = (int)records;
            if ((rc = allocate(s, nVox, &ld.slots))) return rc;
            if ((rc = allocate(s, nVox, &ld.requests))) return rc;
            if ((rc = allocate(s, (size_t)4, &ld.counters))) return rc;
            CUDA_TRY(cudaMemset(ld.slots, 0xff, nVox * sizeof(int)));   // LD_ABSENT
            CUDA_TRY(cudaMemset(ld.counters, 0, 4 * sizeof(int)));
            CUDA_TRY(cudaMallocHost((void **)&s->ldHostCounters, 4 * sizeof(int)));
            s->lazyLightDist = true;
        }
    }
    if ((rc = allocate(s, (size_t)CTR_COUNT, &s->counters))) return rc;
    CUDA_TRY(cudaDeviceSynchronize());
    guard.s = nullptr;
    *out = s;
    return PB2_OK;
}

int pb2_intersect(pb2_scene *scene, const pb2_ray *rays, int64_t n, pb2_hit *hits) {
    int rc = requireDevice();
    if (rc) return rc;
    if (!scene || (n > 0 && (!rays || !hits))) return setError(PB2_ERR_INVALID, "null argument");
    if (n <= 0) return PB2_OK;
    pb2_ray *dRays = nullptr;
    pb2_hit *dHits = nullptr;
    CUDA_TRY(cudaMalloc((void **)&dRays, n * sizeof(pb2_ray)));
    cudaError_t e = cudaMalloc((void **)&dHits, n * sizeof(pb2_hit));
    if (e != cudaSuccess) { cudaFree(dRays); return setError(PB2_ERR_CUDA, cudaGetErrorString(e)); }
    e = cudaMemcpy(dRays, rays, n * sizeof(pb2_ray), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        k_intersect<<<(unsigned)((n + 127) / 128), 128>>>(scene->d, dRays, n, dHits);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(hits, dHits, n * sizeof(pb2_hit), cudaMemcpyDeviceToHost);
    cudaFree(dRays);
    cudaFree(dHits);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, std::string("pb2_intersect: ") + cudaGetErrorString(e));
    return PB2_OK;
}

int pb2_intersect_p(pb2_scene *scene, const pb2_ray *rays, int64_t n, uint8_t *occluded) {
    int rc = requireDevice();
    if (rc) return rc;
    if (!scene || (n > 0 && (!rays || !occluded))) return setError(PB2_ERR_INVALID, "null argument");
    if (n <= 0) return PB2_OK;
    pb2_ray *dRays = nullptr;
    uint8_t *dOcc = nullptr;
    CUDA_TRY(cudaMalloc((void **)&dRays, n * sizeof(pb2_ray)));
    cudaError_t e = cudaMalloc((void **)&dOcc, n);
    if (e != cudaSuccess) { cudaFree(dRays); return setError(PB2_ERR_CUDA, cudaGetErrorString(e)); }
    e = cudaMemcpy(dRays, rays, n * sizeof(pb2_ray), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        k_intersect_p<<<(unsigned)((n + 127) / 128), 128>>>(scene->d, dRays, n, dOcc);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(occluded, dOcc, n, cudaMemcpyDeviceToHost);
    cudaFree(dRays);
    cudaFree(dOcc);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, std::string("pb2_intersect_p: ") + cudaGetErrorString(e));
    return PB2_OK;
}

int pb2_trace_wavefront(pb2_scene *scene, const pb2_ray *rays, const uint8_t *any_hit, int64_t n, int32_t flags, pb2_wf_hit *out) {
    int rc = requireDevice();
    if (rc) return rc;
    if (!scene || (n > 0 && (!rays || !out))) return setError(PB2_ERR_INVALID, "null argument");
    if (n <= 0) return PB2_OK;
    if (n > (1 << 24)) return setError(PB2_ERR_INVALID, "at most 2^24 rays per call");
    const int N = (int)n;
    if ((rc = ensurePool(scene, (N + 255) / 256 * 256))) return rc;
    TraceLaunch trace;
    if ((rc = selectTraceKernel(scene, flags, &trace))) return rc;
    WfPool pool = poolOf(scene, scene->wfCapacity);
    pb2_ray *dRays = nullptr;
    uint8_t *dAny = nullptr;
    pb2_wf_hit *dOut = nullptr;
    cudaError_t e = cudaMalloc((void **)&dRays, n * sizeof(pb2_ray));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dOut, n * sizeof(pb2_wf_hit));
    if (e == cudaSuccess && any_hit) e = cudaMalloc((void **)&dAny, n);
    if (e == cudaSuccess) e = cudaMemcpy(dRays, rays, n * sizeof(pb2_ray), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && any_hit) e = cudaMemcpy(dAny, any_hit, n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        const int blocks = (N + 127) / 128;
        k_wf_debug_fill<<<blocks, 128>>>(pool, dRays, dAny, N);
        WfChain noChain;
        memset(&noChain, 0, sizeof(noChain));
        trace.fn<<<trace.grid, trace.block, trace.smem>>>(scene->d, pool, WQ_TRACE0, noChain);
        k_wf_debug_read<<<blocks, 128>>>(scene->d, pool, N, dOut);
        k_wf_debug_lists<<<std::min(blocks, g_numSMs * 8), 128>>>(pool, dOut);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dOut, n * sizeof(pb2_wf_hit), cudaMemcpyDeviceToHost);
    cudaFree(dRays);
    cudaFree(dAny);
    cudaFree(dOut);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, std::string("pb2_trace_wavefront: ") + cudaGetErrorString(e));
    return PB2_OK;
}

// film[i] += sum over the peers' films: the Film::MergeFilmTile of a multi-device render, run on the primary device, which
// reads the other devices' memory directly (peer access over NVLink): 33 MB per peer at 1080p
__global__ void k_film_sum_peers(float4 *film, const float4 *p0, const float4 *p1, const float4 *p2, const float4 *p3, const float4 *p4,
                                 const float4 *p5, const float4 *p6, int nPeers, size_t nPixels) {
    const float4 *peers[7] = {p0, p1, p2, p3, p4, p5, p6};
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nPixels; i += (size_t)gridDim.x * blockDim.x) {
        float4 a = film[i];
        for (int k = 0; k < nPeers; ++k) {
            const float4 b = peers[k][i];
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        film[i] = a;
    }
}

static int ensureFilm(pb2_scene *scene, size_t nFloats) {
    if (scene->filmFloats < nFloats) {
        if (scene->film) cudaFree(scene->film);
        scene->film = nullptr;
        scene->filmFloats = 0;
        CUDA_TRY(cudaMalloc((void **)&scene->film, nFloats * sizeof(float)));
        scene->filmFloats = nFloats;
    }
    return PB2_OK;
}

static int renderPathDeviceOne(pb2_scene *scene, const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp,
                               float *film_rgbw_device, int clear, void *stream_, pb2_stats *stats);

// A render over the local device group (pb2_init_devices with n > 1, params.tile_count == 0): one host thread per device
// renders the tiles t with t % n == its index into its own copy of the scene and its own film; the primary device then adds
// the other films to its own.
static int renderPathDeviceGroup(pb2_scene *scene, const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp,
                                 float *film_rgbw_device, int clear, cudaStream_t stream, pb2_stats *stats) {
    const int n = (int)g_devs.size();
    if (n > 8) return setError(PB2_ERR_UNSUPPORTED, "at most 8 local devices");
    if ((int)scene->replicas.size() != n - 1) return setError(PB2_ERR_INVALID, "the scene was created before pb2_init_devices bound this device group");
    const size_t nPixels = (size_t)(film->cropped_pixel_bounds[2] - film->cropped_pixel_bounds[0]) *
                           (size_t)(film->cropped_pixel_bounds[3] - film->cropped_pixel_bounds[1]);
    std::vector<int> rcs((size_t)n, PB2_OK);
    std::vector<std::string> errs((size_t)n);
    std::vector<pb2_stats> sts((size_t)n);
    std::vector<std::thread> workers;
    CUDA_TRY(cudaStreamSynchronize(stream));   // the caller's earlier work on the film
    for (int i = 0; i < n; ++i)
        workers.emplace_back([&, i] {
            t_dev = i;
            pb2_scene *rep = i == 0 ? scene : scene->replicas[(size_t)i - 1];
            int rc = cudaSetDevice(g_devs[(size_t)i].id) == cudaSuccess ? PB2_OK : setError(PB2_ERR_CUDA, "cudaSetDevice failed");
            float *target = film_rgbw_device;
            if (rc == PB2_OK && i > 0) {
                rc = ensureFilm(rep, nPixels * 4);
                target = rep->film;
            }
            pb2_path_params p = *pp;
            p.tile_rank = i;
            p.tile_count = n;
            memset(&sts[(size_t)i], 0, sizeof(pb2_stats));
            if (rc == PB2_OK) rc = renderPathDeviceOne(rep, cam, film, &p, target, i == 0 ? clear : 1, nullptr, &sts[(size_t)i]);
            if (rc == PB2_OK && cudaDeviceSynchronize() != cudaSuccess) rc = setError(PB2_ERR_CUDA, "device synchronisation failed after the render");
            rcs[(size_t)i] = rc;
            errs[(size_t)i] = g_lastError;
        });
    for (std::thread &w : workers) w.join();
    t_dev = 0;
    CUDA_TRY(cudaSetDevice(g_devs[0].id));
    for (int i = 0; i < n; ++i)
        if (rcs[(size_t)i]) return setError(rcs[(size_t)i], "device " + std::to_string(g_devs[(size_t)i].id) + ": " + errs[(size_t)i]);
    // merge
    const float4 *peers[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    std::vector<float *> staged;
    for (int i = 1; i < n; ++i) {
        pb2_scene *rep = scene->replicas[(size_t)i - 1];
        if (g_devs[(size_t)i].peerOfPrimary) peers[i - 1] = reinterpret_cast<const float4 *>(rep->film);
        else {   // no peer access between the two devices: stage the film through a copy
            float *tmp = nullptr;
            CUDA_TRY(cudaMalloc((void **)&tmp, nPixels * 16));
            staged.push_back(tmp);
            CUDA_TRY(cudaMemcpyPeerAsync(tmp, g_devs[0].id, rep->film, g_devs[(size_t)i].id, nPixels * 16, stream));
            peers[i - 1] = reinterpret_cast<const float4 *>(tmp);
        }
    }
    const int blocks = (int)std::min<size_t>((nPixels + 255) / 256, (size_t)g_numSMs * 8);
    k_film_sum_peers<<<blocks, 256, 0, stream>>>(reinterpret_cast<float4 *>(film_rgbw_device), peers[0], peers[1], peers[2], peers[3], peers[4],
                                                 peers[5], peers[6], n - 1, nPixels);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(stream));
    for (float *t : staged) cudaFree(t);
    if (stats) {
        memset(stats, 0, sizeof(*stats));
        for (const pb2_stats &st : sts) {
            stats->camera_rays += st.camera_rays;
            stats->regular_rays += st.regular_rays;
            stats->shadow_rays += st.shadow_rays;
            stats->node_visits += st.node_visits;
            stats->prim_tests += st.prim_tests;
            stats->kernel_launches += st.kernel_launches;
            stats->render_ms = std::max(stats->render_ms, st.render_ms);   // the devices run concurrently
            stats->trace_ms = std::max(stats->trace_ms, st.trace_ms);
        }
        stats->kernel_launches += 1;
    }
    return PB2_OK;
}

int pb2_render_path_device(pb2_scene *scene, const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp,
                           float *film_rgbw_device, int clear, void *stream_, pb2_stats *stats) {
    int rc = requireDevice();
    if (rc) return rc;
    if ((rc = validateRenderArgs(scene, cam, film, pp))) return rc;
    if (!film_rgbw_device) return setError(PB2_ERR_INVALID, "null film pointer");
    if (pp->tile_count == 0 && g_devs.size() > 1) return renderPathDeviceGroup(scene, cam, film, pp, film_rgbw_device, clear, (cudaStream_t)stream_, stats);
    return renderPathDeviceOne(scene, cam, film, pp, film_rgbw_device, clear, stream_, stats);
}

static int renderPathDeviceOne(pb2_scene *scene, const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp,
                               float *film_rgbw_device, int clear, void *stream_, pb2_stats *stats) {
    int rc = PB2_OK;
    cudaStream_t stream = (cudaStream_t)stream_;
    // tile_count == 0: the partition of the communicator (every rank renders its tiles, the films are summed on rank 0);
    // a caller that sets tile_count >= 1 partitions by hand and gets exactly the tiles it asked for, unreduced
    const bool distributed = pp->tile_count == 0 && g_dist.world > 1;
    pb2_path_params ppLocal = *pp;
    if (distributed) {
        ppLocal.tile_rank = g_dist.rank;
        ppLocal.tile_count = g_dist.world;
        pp = &ppLocal;
    }
    DRenderParams rp = makeRenderParams(cam, film, pp);
    if (pp->sampler == PB2_SAMPLER_SOBOL && (rc = attachSobol(&rp.halton, film))) return rc;
    {
        float table[256];
        if (computeFilterTable(film, table)) {
            if (!scene->filterTable) CUDA_TRY(cudaMalloc((void **)&scene->filterTable, sizeof(table)));
            CUDA_TRY(cudaMemcpyAsync(scene->filterTable, table, sizeof(table), cudaMemcpyHostToDevice, stream));
            CUDA_TRY(cudaStreamSynchronize(stream));   // `table` is on this stack frame
            rp.filterTable = scene->filterTable;
        }
    }
    size_t nPixels = (size_t)(rp.cx1 - rp.cx0) * (size_t)(rp.cy1 - rp.cy0);
    if (clear) CUDA_TRY(cudaMemsetAsync(film_rgbw_device, 0, nPixels * 4 * sizeof(float), stream));
    CUDA_TRY(cudaMemsetAsync(scene->counters, 0, CTR_COUNT * sizeof(unsigned long long), stream));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (stats) {
        CUDA_TRY(cudaEventCreate(&e0));
        CUDA_TRY(cudaEventCreate(&e1));
        CUDA_TRY(cudaEventRecord(e0, stream));
    }
    unsigned long long launches = 0;
    double traceMs = 0;
    if (rp.nWorkItems > 0) {
        rc = renderWavefront(scene, rp, (float4 *)film_rgbw_device, stream, pp->flags, stats != nullptr, &launches, &traceMs);
        if (rc) {
            if (e0) cudaEventDestroy(e0);
            if (e1) cudaEventDestroy(e1);
            return rc;
        }
    }
    if (distributed)   // the distributed Film::MergeFilmTile (film.cpp:117-130): in place, the sum lands in rank 0's film
        NCCL_TRY(g_nccl.Reduce(film_rgbw_device, film_rgbw_device, nPixels * 4, ncclFloat, ncclSum, 0, g_dist.comm, stream));
    if (stats) {
        CUDA_TRY(cudaEventRecord(e1, stream));
        CUDA_TRY(cudaEventSynchronize(e1));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, e0, e1));
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        unsigned long long c[CTR_COUNT];
        CUDA_TRY(cudaMemcpyAsync(c, scene->counters, sizeof(c), cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        memset(stats, 0, sizeof(*stats));
        stats->camera_rays = c[CTR_CAMERA];
        stats->regular_rays = c[CTR_REGULAR];
        stats->shadow_rays = c[CTR_SHADOW];
        stats->node_visits = c[CTR_NODES];
        stats->prim_tests = c[CTR_PRIMS];
        stats->kernel_launches = launches;
        stats->render_ms = ms;
        stats->trace_ms = traceMs;
    }
    return PB2_OK;
}

int pb2_render_path(pb2_scene *scene, const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp,
                    float *film_rgbw, pb2_stats *stats) {
    int rc = requireDevice();
    if (rc) return rc;
    if ((rc = validateRenderArgs(scene, cam, film, pp))) return rc;
    if (!film_rgbw && !(pp->tile_count == 0 && g_dist.world > 1 && g_dist.rank != 0)) return setError(PB2_ERR_INVALID, "null film pointer");
    size_t nFloats = 4 * (size_t)(film->cropped_pixel_bounds[2] - film->cropped_pixel_bounds[0]) *
                     (size_t)(film->cropped_pixel_bounds[3] - film->cropped_pixel_bounds[1]);
    if (nFloats == 0) return PB2_OK;
    if ((rc = ensureFilm(scene, nFloats))) return rc;
    pb2_stats local;
    memset(&local, 0, sizeof(local));
    rc = pb2_render_path_device(scene, cam, film, pp, scene->film, 1, nullptr, stats ? &local : nullptr);
    if (rc) return rc;
    const bool receives = !(pp->tile_count == 0 && g_dist.world > 1 && g_dist.rank != 0);   // the merged film lands on rank 0
    if (receives) {
        // full PCIe rate when film_rgbw is page-locked (pb2_host_alloc); staged by the driver otherwise
        auto t0 = std::chrono::steady_clock::now();
        CUDA_TRY(cudaMemcpyAsync(film_rgbw, scene->film, nFloats * sizeof(float), cudaMemcpyDeviceToHost, nullptr));
        CUDA_TRY(cudaStreamSynchronize(nullptr));
        local.d2h_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    } else
        CUDA_TRY(cudaStreamSynchronize(nullptr));
    if (stats) *stats = local;
    return PB2_OK;
}

int pb2_li_samples(pb2_scene *scene, const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp,
                   const int32_t *pixel_xy, const int64_t *sample_num, int64_t n, float *out_rgb, float *out_pfilm) {
    int rc = requireDevice();
    if (rc) return rc;
    if ((rc = validateRenderArgs(scene, cam, film, pp))) return rc;
    if (n <= 0) return PB2_OK;
    if (!pixel_xy || !sample_num || !out_rgb) return setError(PB2_ERR_INVALID, "null argument");
    DRenderParams rp = makeRenderParams(cam, film, pp);
    if (pp->sampler == PB2_SAMPLER_SOBOL && (rc = attachSobol(&rp.halton, film))) return rc;
    int32_t *dXY = nullptr;
    int64_t *dS = nullptr;
    float *dRGB = nullptr, *dPF = nullptr;
    cudaError_t e = cudaMalloc((void **)&dXY, n * 2 * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dS, n * sizeof(int64_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dRGB, n * 3 * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dPF, n * 2 * sizeof(float));
    if (e == cudaSuccess) e = cudaMemcpy(dXY, pixel_xy, n * 2 * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dS, sample_num, n * sizeof(int64_t), cudaMemcpyHostToDevice);
    int *dDeferred = nullptr;
    if (e == cudaSuccess) e = cudaMalloc((void **)&dDeferred, sizeof(int));
    for (int pass = 0; e == cudaSuccess; ++pass) {
        // lazy light distribution: a sample that meets a voxel without a record stops; the records are built and ALL samples
        // run again (a pure function of pixel and sample number), until none stops - at most one pass per path vertex
        int deferred = 0;
        e = cudaMemset(dDeferred, 0, sizeof(int));
        if (e == cudaSuccess) {
            k_li_samples<<<(unsigned)((n + 63) / 64), 64>>>(scene->d, rp, dXY, dS, n, dRGB, dPF, dDeferred);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpy(&deferred, dDeferred, sizeof(int), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess || deferred == 0) break;
        launchLightDistBuild(scene, nullptr);
        bool overflowed = false;
        if (lightDistOverflowed(scene, nullptr, &overflowed) != PB2_OK || overflowed || pass > 4096) {
            cudaFree(dXY); cudaFree(dS); cudaFree(dRGB); cudaFree(dPF); cudaFree(dDeferred);
            return overflowed ? lightDistOverflowError() : setError(PB2_ERR_CUDA, "pb2_li_samples: light distribution build failed");
        }
    }
    cudaFree(dDeferred);
    if (e == cudaSuccess) e = cudaMemcpy(out_rgb, dRGB, n * 3 * sizeof(float), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && out_pfilm) e = cudaMemcpy(out_pfilm, dPF, n * 2 * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(dXY);
    cudaFree(dS);
    cudaFree(dRGB);
    cudaFree(dPF);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, std::string("pb2_li_samples: ") + cudaGetErrorString(e));
    return PB2_OK;
}

int pb2_halton_samples(const pb2_film_desc *film, const pb2_path_params *pp, const int32_t *pixel_xy,
                       const int64_t *sample_num, const int32_t *dim, int64_t n, float *out) {
    int rc = requireDevice();
    if (rc) return rc;
    if (!film || !pp || (n > 0 && (!pixel_xy || !sample_num || !dim || !out))) return setError(PB2_ERR_INVALID, "null argument");
    if (n <= 0) return PB2_OK;
    for (int64_t i = 0; i < n; ++i)
        if (dim[i] < 0 || dim[i] >= kMaxHaltonDims) return setError(PB2_ERR_INVALID, "HaltonSampler can only sample 1000 dimensions");
    DHalton h = makeHalton(film, pp);
    if (pp->sampler == PB2_SAMPLER_SOBOL && (rc = attachSobol(&h, film))) return rc;
    int32_t *dXY = nullptr, *dDim = nullptr;
    int64_t *dS = nullptr;
    float *dOut = nullptr;
    cudaError_t e = cudaMalloc((void **)&dXY, n * 2 * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dS, n * sizeof(int64_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dDim, n * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dOut, n * sizeof(float));
    if (e == cudaSuccess) e = cudaMemcpy(dXY, pixel_xy, n * 2 * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dS, sample_num, n * sizeof(int64_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dDim, dim, n * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        k_halton_samples<<<(unsigned)((n + 127) / 128), 128>>>(h, dXY, dS, dDim, n, dOut);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dOut, n * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(dXY);
    cudaFree(dS);
    cudaFree(dDim);
    cudaFree(dOut);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, std::string("pb2_halton_samples: ") + cudaGetErrorString(e));
    return PB2_OK;
}

int pb2_sobol_samples_host(const pb2_film_desc *film, const pb2_path_params *pp, const int32_t *pixel_xy, const int64_t *sample_num,
                           const int32_t *dim, int64_t n, float *out, uint64_t *tablesOut) {
    if (!film || !pp || (n > 0 && (!pixel_xy || !sample_num || !dim || !out))) return setError(PB2_ERR_INVALID, "null argument");
    int rc = loadSobolMatrices();
    if (rc) return rc;
    DHalton h;
    memset(&h, 0, sizeof(h));
    SampleBounds sb = filmSampleBounds(film);
    int extent = std::max(sb.x1 - sb.x0, sb.y1 - sb.y0), res = 1, log2Res = 0;
    while (res < extent) {
        res <<= 1;
        ++log2Res;
    }
    if (log2Res > 26) return setError(PB2_ERR_UNSUPPORTED, "SobolSampler: sample bounds beyond 2^26 pixels in one direction");
    uint64_t tables[2 * kSobolMatrixSize];
    sobolIntervalTables(log2Res, tables);
    if (tablesOut) memcpy(tablesOut, tables, sizeof(tables));
    h.sobol = g_sobolMatrices.data();
    h.sobolVdc = tables;
    h.sobolLog2Res = log2Res;
    h.sobolRes = res;
    h.sbx0 = sb.x0;
    h.sby0 = sb.y0;
    for (int64_t i = 0; i < n; ++i) {
        if (dim[i] < 0 || dim[i] >= kSobolDims) return setError(PB2_ERR_INVALID, "SobolSampler can only sample up to 1024 dimensions");
        const int px = pixel_xy[2 * i], py = pixel_xy[2 * i + 1];
        const int64_t index = sampleIndex<true>(h, px, py, sample_num[i]);
        out[i] = dim[i] < 2 ? sobolPixelSample(h, index, dim[i], dim[i] == 0 ? px : py) : sampleDimension<true>(h, index, dim[i]);
    }
    return PB2_OK;
}

int pb2_bsdf_eval_host(const pb2_material *material, int64_t n, const float *in, float *out) {
    if (!material || (n > 0 && (!in || !out))) return setError(PB2_ERR_INVALID, "null argument");
    DScene sc;
    memset(&sc, 0, sizeof(sc));
    const int32_t primMaterial = 0;
    sc.primMaterial = &primMaterial;
    sc.materials = material;
    for (int64_t i = 0; i < n; ++i) {
        const float *q = in + 17 * i;
        float *o = out + 19 * i;
        for (int k = 0; k < 19; ++k) o[k] = 0;
        DInteraction it;
        memset(&it, 0, sizeof(it));
        it.n = mk3(q[0], q[1], q[2]);
        it.ns = mk3(q[3], q[4], q[5]);
        it.dpdus = mk3(q[6], q[7], q[8]);
        const V3 wo = mk3(q[9], q[10], q[11]), wi = mk3(q[12], q[13], q[14]);
        it.wo = wo;
        it.prim = 0;
        // every lobe of every material; the texture slots are not evaluated
        constexpr int F = SHADE_GENERAL | SHADE_SPECULAR;
        DBsdf bsdf;
        if (!makeBsdf<F>(sc, it, &bsdf)) continue;
        if (bsdf.nLobes > 0) {   // (EstimateDirect is only entered with non-specular lobes: path.cpp:119-126)
            const V3 f = bsdfF<F>(bsdf, wo, wi);
            o[0] = f.x; o[1] = f.y; o[2] = f.z;
            o[3] = bsdfPdf<F>(bsdf, wo, wi);
            V3 wiS;
            float pdfS;
            const V3 fS = bsdfSampleF<F>(bsdf, wo, &wiS, mk2(q[15], q[16]), &pdfS, nullptr, true);
            if (pdfS != 0) { o[4] = wiS.x; o[5] = wiS.y; o[6] = wiS.z; }
            o[7] = fS.x; o[8] = fS.y; o[9] = fS.z;
            o[10] = pdfS;
        }
        V3 wiC;
        float pdfC;
        int flags = 0;
        const V3 fC = bsdfSampleF<F>(bsdf, wo, &wiC, mk2(q[15], q[16]), &pdfC, &flags);
        if (pdfC != 0) { o[11] = wiC.x; o[12] = wiC.y; o[13] = wiC.z; }
        o[14] = fC.x; o[15] = fC.y; o[16] = fC.z;
        o[17] = pdfC;
        o[18] = (float)flags;
    }
    return PB2_OK;
}

int pb2_camera_differentials_host(const pb2_camera *cam, const pb2_film_desc *film, const pb2_path_params *pp, int64_t n, const float *in,
                                  float *out) {
    if (!cam || !film || !pp || pp->samples_per_pixel <= 0 || (n > 0 && (!in || !out))) return setError(PB2_ERR_INVALID, "bad argument");
    DCamera c;
    memcpy(c.rasterToCamera.m, cam->raster_to_camera, sizeof(float) * 16);
    memcpy(c.cameraToWorld.m, cam->camera_to_world, sizeof(float) * 16);
    c.lensRadius = cam->lens_radius;
    c.focalDistance = cam->focal_distance;
    c.dxCamera = mk3(cam->dx_camera[0], cam->dx_camera[1], cam->dx_camera[2]);
    c.dyCamera = mk3(cam->dy_camera[0], cam->dy_camera[1], cam->dy_camera[2]);
    const float scale = 1 / std::sqrt((float)pp->samples_per_pixel);
    for (int64_t i = 0; i < n; ++i) {
        const float *q = in + 10 * i;
        const DRayDiff rd = cameraRayDifferentials(c, mk2(q[0], q[1]), mk2(q[2], q[3]), scale, mk3(q[4], q[5], q[6]), mk3(q[7], q[8], q[9]));
        float *o = out + 12 * i;
        o[0] = rd.rxo.x; o[1] = rd.rxo.y; o[2] = rd.rxo.z;
        o[3] = rd.rxd.x; o[4] = rd.rxd.y; o[5] = rd.rxd.z;
        o[6] = rd.ryo.x; o[7] = rd.ryo.y; o[8] = rd.ryo.z;
        o[9] = rd.ryd.x; o[10] = rd.ryd.y; o[11] = rd.ryd.z;
    }
    return PB2_OK;
}

int pb2_uv_differentials_host(int64_t n, const float *in, float *out) {
    if (n > 0 && (!in || !out)) return setError(PB2_ERR_INVALID, "null argument");
    for (int64_t i = 0; i < n; ++i) {
        const float *q = in + 24 * i;
        DRayDiff rd;
        rd.rxo = mk3(q[12], q[13], q[14]);
        rd.rxd = mk3(q[15], q[16], q[17]);
        rd.ryo = mk3(q[18], q[19], q[20]);
        rd.ryd = mk3(q[21], q[22], q[23]);
        const DUvDiff d = computeUvDifferentials(mk3(q[0], q[1], q[2]), mk3(q[3], q[4], q[5]), mk3(q[6], q[7], q[8]), mk3(q[9], q[10], q[11]), rd);
        out[4 * i] = d.dudx;
        out[4 * i + 1] = d.dvdx;
        out[4 * i + 2] = d.dudy;
        out[4 * i + 3] = d.dvdy;
    }
    return PB2_OK;
}

int pb2_light_distribution(pb2_scene *scene, const float *points_xyz, int64_t n, float *out) {
    int rc = requireDevice();
    if (rc) return rc;
    if (!scene || (n > 0 && (!points_xyz || !out))) return setError(PB2_ERR_INVALID, "null argument");
    if (n <= 0 || scene->nLights == 0) return PB2_OK;
    size_t stride = 2 * (size_t)scene->nLights + 1;
    float *dP = nullptr, *dOut = nullptr;
    cudaError_t e = cudaMalloc((void **)&dP, n * 3 * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc((void **)&dOut, n * stride * sizeof(float));
    if (e == cudaSuccess) e = cudaMemcpy(dP, points_xyz, n * 3 * sizeof(float), cudaMemcpyHostToDevice);
    for (int pass = 0; pass < (scene->lazyLightDist ? 2 : 1) && e == cudaSuccess; ++pass) {
        k_light_distribution<<<(unsigned)((n + 127) / 128), 128>>>(scene->d, dP, n, dOut);
        e = cudaGetLastError();
        if (scene->lazyLightDist && pass == 0 && e == cudaSuccess) {   // first pass requested the missing voxels
            launchLightDistBuild(scene, nullptr);
            bool overflowed = false;
            if (lightDistOverflowed(scene, nullptr, &overflowed) != PB2_OK || overflowed) {
                cudaFree(dP);
                cudaFree(dOut);
                return lightDistOverflowError();
            }
        }
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, dOut, n * stride * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(dP);
    cudaFree(dOut);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, std::string("pb2_light_distribution: ") + cudaGetErrorString(e));
    return PB2_OK;
}

}  // extern "C"

// ---------------------------------------------------------------- four-child records: host-side check (pb2_wide4.cuh)
// Not part of the ABI: replays BVHAccel::Intersect's traversal (bvh.cpp:662-700) over the 32-byte nodes and the traversal
// of the four-child records over the same tree, with the slab test the kernels use, and returns the sequence of primitive
// numbers each of them tests.  A primitive is stood in for by its bounding box (prim_bounds: n x 6, by primitive number; a
// box hit shrinks tMax to its entry distance), which is all the traversal order depends on.  Runs on the host.
extern "C" int pb2_debug_wide4_sequences(const pb2_bvh_node *nodes, int64_t n_nodes, const int32_t *bvh_prims, const float *prim_bounds,
                                         const float *rays_od, int64_t n_rays, int32_t max_len, int32_t *seq_binary,
                                         int32_t *seq_wide4, int32_t *len_binary, int32_t *len_wide4) {
    if (!nodes || n_nodes <= 0 || !bvh_prims || !prim_bounds || !rays_od) return PB2_ERR_INVALID;
    const int64_t root0 = 0;
    int32_t rootRecord = 0;
    const std::vector<float4> recs = buildWide4Records(nodes, &root0, 1, &rootRecord);
    for (int64_t i = 0; i < n_rays; ++i) {
        const float *rd = rays_od + 6 * i;
        const DRaySetup r = setupRay(mk3(rd[0], rd[1], rd[2]), mk3(rd[3], rd[4], rd[5]));
        auto leafTests = [&](int32_t first, int32_t count, float *tMax, int32_t *seq, int32_t *len) {
            for (int32_t j = first; j < first + count; ++j) {
                const int32_t prim = bvh_prims[j];
                if (*len < max_len) seq[*len] = prim;
                ++*len;
                const float *b = prim_bounds + 6 * (size_t)prim;
                float t;
                if (slabTestT(b[0], b[1], b[2], b[3], b[4], b[5], r, *tMax, &t) && t > 0) *tMax = t;
            }
        };
        {   // the reference's loop over the linear nodes
            float tMax = PB2_INFINITY;
            int32_t *seq = seq_binary + (size_t)i * max_len, len = 0, stack[64], sp = 0, cur = 0;
            for (;;) {
                const pb2_bvh_node &n = nodes[cur];
                float t;
                if (slabTestT(n.bmin[0], n.bmin[1], n.bmin[2], n.bmax[0], n.bmax[1], n.bmax[2], r, tMax, &t)) {
                    if (n.n_prims > 0) {
                        leafTests(n.offset, n.n_prims, &tMax, seq, &len);
                        if (sp == 0) break;
                        cur = stack[--sp];
                    } else {
                        const int neg = n.axis == 0 ? r.neg0 : (n.axis == 1 ? r.neg1 : r.neg2);
                        if (neg) { stack[sp++] = cur + 1; cur = n.offset; }
                        else { stack[sp++] = n.offset; cur = cur + 1; }
                    }
                } else {
                    if (sp == 0) break;
                    cur = stack[--sp];
                }
            }
            len_binary[i] = len;
        }
        {   // four-child records, walked as k_wf_trace_w<4> walks them (the root's own box is not tested: see pb2_wide4.cuh)
            float tMax = PB2_INFINITY;
            int32_t *seq = seq_wide4 + (size_t)i * max_len, len = 0, sp = 0;
            struct Entry { uint32_t ref; float tMin; } stack[3 * 64];
            bool have = true;
            uint32_t cur = (uint32_t)rootRecord;
            while (have) {
                if (cur & WIDE_LEAF) {
                    leafTests((int32_t)(cur & WIDE_LEAF_OFFSET_MASK), (int32_t)((cur >> WIDE_LEAF_COUNT_SHIFT) & 0xf) + 1, &tMax, seq, &len);
                    have = false;
                } else {
                    const float4 *w = &recs[8 * (size_t)cur];
                    uint32_t meta;
                    memcpy(&meta, &w[7].x, 4);
                    const Wide4Visit v = wide4Visit(w[0], w[1], w[2], w[3], w[4], w[5], w[6], meta, r, tMax);
                    uint32_t refs[4];
                    memcpy(refs, &w[6], sizeof(refs));
                    have = v.nPass > 0;
                    for (int k = 0; k < 4; ++k) {
                        if (!v.pass[k]) continue;
                        if (v.after[k] == v.nPass - 1) cur = refs[k];
                        else stack[sp + v.after[k]] = Entry{refs[k], v.tMin[k]};
                    }
                    if (v.nPass > 1) sp += v.nPass - 1;
                }
                while (!have && sp > 0) {
                    const Entry e = stack[--sp];
                    if (e.tMin < tMax) {   // the deferred child's box against the tMax of this moment
                        cur = e.ref;
                        have = true;
                    }
                }
            }
            len_wide4[i] = len;
        }
    }
    return PB2_OK;
}

// ---------------------------------------------------------------- HLBVH treelets on the device (bvh.cpp:404-539)
namespace {
__device__ __forceinline__ unsigned hlbvhLeftShift3(unsigned x) {   // bvh.cpp:106-130
    if (x == (1u << 10)) --x;
    x = (x | (x << 16)) & 0x30000ffu;
    x = (x | (x << 8)) & 0x300f00fu;
    x = (x | (x << 4)) & 0x30c30c3u;
    x = (x | (x << 2)) & 0x9249249u;
    return x;
}
// order-preserving map float <-> unsigned for atomicMin / atomicMax on floats
__device__ __forceinline__ unsigned floatOrdered(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float orderedFloat(unsigned u) {
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
// BVHPrimitiveInfo::centroid (bvh.cpp:57-58) and the bounds of all centroids (bvh.cpp:409-411): min / max are exact,
// so a block reduction followed by six atomics gives the sequential Union's result
__global__ void k_hlbvh_centroid_bounds(const float *bounds, int n, unsigned *box /* min xyz, max xyz, ordered */) {
    float lo[3] = {PB2_INFINITY, PB2_INFINITY, PB2_INFINITY}, hi[3] = {-PB2_INFINITY, -PB2_INFINITY, -PB2_INFINITY};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        for (int k = 0; k < 3; ++k) {
            float c = .5f * bounds[6 * (size_t)i + k] + .5f * bounds[6 * (size_t)i + 3 + k];
            lo[k] = fminf(lo[k], c);
            hi[k] = fmaxf(hi[k], c);
        }
    for (int k = 0; k < 3; ++k) {
        for (int o = 16; o > 0; o >>= 1) {
            lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
            hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&box[k], floatOrdered(lo[k]));
            atomicMax(&box[3 + k], floatOrdered(hi[k]));
        }
    }
}
// bvh.cpp:414-423: mortonCode = EncodeMorton3(bounds.Offset(centroid) * 1024)
__global__ void k_hlbvh_morton(const float *bounds, int n, const unsigned *box, unsigned *codes, int *index) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned v[3];
    for (int k = 0; k < 3; ++k) {
        float c = .5f * bounds[6 * (size_t)i + k] + .5f * bounds[6 * (size_t)i + 3 + k];
        float lo = orderedFloat(box[k]), hi = orderedFloat(box[3 + k]);
        float o = c - lo;                       // Bounds3::Offset (geometry.h:756-763)
        if (hi > lo) o /= hi - lo;
        v[k] = (unsigned)(o * 1024.f);
    }
    codes[i] = (hlbvhLeftShift3(v[2]) << 2) | (hlbvhLeftShift3(v[1]) << 1) | hlbvhLeftShift3(v[0]);
    index[i] = i;
}
// bvh.cpp:431-448: a treelet starts where the top 12 bits change; at most 4096 of them, one slot per prefix
__global__ void k_hlbvh_treelet_starts(const unsigned *codes, int n, int *start /* 4096, preset to -1 */) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned mask = 0x3ffc0000u;
    if (i == 0 || (codes[i] & mask) != (codes[i - 1] & mask)) start[(codes[i] & mask) >> 18] = i;
}
// emitLBVH (bvh.cpp:472-539), one thread per treelet, the recursion unrolled over an explicit stack.  Nodes are
// numbered in the reference's allocation order (a node before its subtrees, the first subtree before the second)
// inside the treelet's 2 * nPrimitives slots; interior bounds are filled bottom-up afterwards.
__global__ void k_hlbvh_emit(const float *bounds, const unsigned *codes, const int *sorted, const int2 *treelets /* start, count */,
                             int nTreelets, int maxPrimsInNode, pb2_build_node *pool, int *roots, int *treeletNodes = nullptr) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nTreelets) return;
    const int first = treelets[t].x, count = treelets[t].y;
    const unsigned *mp = codes + first;
    pb2_build_node *nodes = pool + 2 * (size_t)first;
    const int base = 2 * first;
    int next = 0;
    struct Item { int lo, n, bit, parent, side; };
    Item stack[40];
    int sp = 0;
    stack[sp++] = Item{0, count, 29 - 12, -1, 0};
    while (sp > 0) {
        Item it = stack[--sp];
        // levels without a split are passed through (bvh.cpp:496-501); the leaf test precedes them at every level
        bool leaf = false;
        for (;;) {
            if (it.bit == -1 || it.n < maxPrimsInNode) {
                leaf = true;
                break;
            }
            unsigned mask = 1u << it.bit;
            if ((mp[it.lo] & mask) != (mp[it.lo + it.n - 1] & mask)) break;
            --it.bit;
        }
        int me = next++;
        if (it.parent >= 0) nodes[it.parent].child[it.side] = base + me;
        pb2_build_node &nd = nodes[me];
        if (leaf) {
            float lo[3] = {PB2_INFINITY, PB2_INFINITY, PB2_INFINITY}, hi[3] = {-PB2_INFINITY, -PB2_INFINITY, -PB2_INFINITY};
            for (int i = 0; i < it.n; ++i) {
                const float *b = bounds + 6 * (size_t)sorted[first + it.lo + i];
                for (int k = 0; k < 3; ++k) {
                    lo[k] = fminf(lo[k], b[k]);
                    hi[k] = fmaxf(hi[k], b[3 + k]);
                }
            }
            for (int k = 0; k < 3; ++k) { nd.bmin[k] = lo[k]; nd.bmax[k] = hi[k]; }
            nd.child[0] = nd.child[1] = -1;
            nd.split_axis = 0;
            nd.first_prim_offset = first + it.lo;
            nd.n_primitives = it.n;
            continue;
        }
        unsigned mask = 1u << it.bit;
        int searchStart = 0, searchEnd = it.n - 1;   // bvh.cpp:503-517
        while (searchStart + 1 != searchEnd) {
            int mid = (searchStart + searchEnd) / 2;
            if ((mp[it.lo + searchStart] & mask) == (mp[it.lo + mid] & mask)) searchStart = mid;
            else searchEnd = mid;
        }
        int splitOffset = searchEnd;
        nd.child[0] = nd.child[1] = -1;
        nd.split_axis = it.bit % 3;
        nd.first_prim_offset = 0;
        nd.n_primitives = 0;
        // the first subtree is emitted first: push the second one below it
        stack[sp++] = Item{it.lo + splitOffset, it.n - splitOffset, it.bit - 1, me, 1};
        stack[sp++] = Item{it.lo, splitOffset, it.bit - 1, me, 0};
    }
    for (int i = next - 1; i >= 0; --i) {   // children carry larger numbers than their parent
        pb2_build_node &nd = nodes[i];
        if (nd.n_primitives > 0) continue;
        const pb2_build_node &a = pool[nd.child[0]], &b = pool[nd.child[1]];
        for (int k = 0; k < 3; ++k) {
            nd.bmin[k] = fminf(a.bmin[k], b.bmin[k]);
            nd.bmax[k] = fmaxf(a.bmax[k], b.bmax[k]);
        }
    }
    roots[t] = base;
    if (treeletNodes) treeletNodes[t] = next;
}

// ---- the upper half of HLBVHBuild on the device: buildUpperSAH (bvh.cpp:541-638) and flattenBVHTree (bvh.cpp:640-658) ----
// Working set of k_hlbvh_upper (at most 4096 treelets, hence at most 4095 nodes above them).
struct HlbvhUpper {
    int *order;            // the treelets as buildUpperSAH permutes them (std::partition)
    float *box;            // 6 floats per treelet: the bounds of its root
    int4 *stack;           // pending ranges {start, end, parent, side}
    pb2_build_node *nodes; // the nodes above the treelets, a parent before its children, the first subtree before the second;
                           // child >= 0: another of these nodes, child < 0: treelet -(child + 1)
    int *size, *offset;    // per upper node: nodes in its subtree, its place in the linear array
    int *treeletBase;      // per treelet: where its first node lands in the linear array
    int *counts;           // [0] upper nodes, [1] total nodes
};
// One thread: the SAH tree over the treelet roots is small (<= 4096 leaves) and sequential by nature (every split partitions
// the range the next ones work on).  The arithmetic is buildUpperSAH's, operation for operation, including libstdc++'s
// bidirectional std::partition (the order it leaves the elements in decides the tree).  Because a parent is numbered before
// its children and the first subtree is finished before the second starts, the numbering is the depth-first order
// flattenBVHTree walks: subtree sizes follow from one backward pass, offsets from one forward pass.
__global__ void k_hlbvh_upper(const pb2_build_node *pool, const int *roots, const int *treeletNodes, int nTreelets, HlbvhUpper w,
                              pb2_bvh_node *linear) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    for (int t = 0; t < nTreelets; ++t) {
        w.order[t] = t;
        const pb2_build_node &r = pool[roots[t]];
        for (int k = 0; k < 3; ++k) {
            w.box[6 * t + k] = r.bmin[k];
            w.box[6 * t + 3 + k] = r.bmax[k];
        }
    }
    int nUpper = 0, sp = 0;
    if (nTreelets == 1) w.treeletBase[0] = 0;
    else w.stack[sp++] = make_int4(0, nTreelets, -1, 0);
    constexpr int nBuckets = 12;
    while (sp > 0) {
        const int4 f = w.stack[--sp];
        const int start = f.x, end = f.y;
        if (end - start == 1) {
            w.nodes[f.z].child[f.w] = -(w.order[start] + 1);
            continue;
        }
        const int u = nUpper++;
        if (f.z >= 0) w.nodes[f.z].child[f.w] = u;
        float bmin[3] = {PB2_INFINITY, PB2_INFINITY, PB2_INFINITY}, bmax[3] = {-PB2_INFINITY, -PB2_INFINITY, -PB2_INFINITY};
        float cmin[3] = {PB2_INFINITY, PB2_INFINITY, PB2_INFINITY}, cmax[3] = {-PB2_INFINITY, -PB2_INFINITY, -PB2_INFINITY};
        for (int i = start; i < end; ++i) {
            const float *b = w.box + 6 * w.order[i];
            for (int k = 0; k < 3; ++k) {
                bmin[k] = fminf(bmin[k], b[k]);
                bmax[k] = fmaxf(bmax[k], b[3 + k]);
                const float c = (b[k] + b[3 + k]) * 0.5f;
                cmin[k] = fminf(cmin[k], c);
                cmax[k] = fmaxf(cmax[k], c);
            }
        }
        // Bounds3::MaximumExtent (geometry.h:733-741)
        const float dx = cmax[0] - cmin[0], dy = cmax[1] - cmin[1], dz = cmax[2] - cmin[2];
        const int dim = (dx > dy && dx > dz) ? 0 : (dy > dz ? 1 : 2);
        int count[nBuckets];
        float lo[nBuckets][3], hi[nBuckets][3];
        for (int b = 0; b < nBuckets; ++b) {
            count[b] = 0;
            for (int k = 0; k < 3; ++k) {
                lo[b][k] = PB2_INFINITY;
                hi[b][k] = -PB2_INFINITY;
            }
        }
        const float c0 = cmin[dim], c1 = cmax[dim];
        auto bucketOf = [&](int t) {
            const float centroid = (w.box[6 * t + dim] + w.box[6 * t + 3 + dim]) * 0.5f;
            int b = (int)(nBuckets * ((centroid - c0) / (c1 - c0)));
            if (b == nBuckets) b = nBuckets - 1;
            return b;
        };
        for (int i = start; i < end; ++i) {
            const int t = w.order[i], b = bucketOf(t);
            count[b]++;
            for (int k = 0; k < 3; ++k) {
                lo[b][k] = fminf(lo[b][k], w.box[6 * t + k]);
                hi[b][k] = fmaxf(hi[b][k], w.box[6 * t + 3 + k]);
            }
        }
        auto area = [](const float *mn, const float *mx) {   // Bounds3::SurfaceArea (geometry.h:723-726)
            const float ex = mx[0] - mn[0], ey = mx[1] - mn[1], ez = mx[2] - mn[2];
            return 2 * (ex * ey + ex * ez + ey * ez);
        };
        float minCost = 0;
        int minCostSplitBucket = 0;
        for (int i = 0; i < nBuckets - 1; ++i) {
            float l0[3] = {PB2_INFINITY, PB2_INFINITY, PB2_INFINITY}, h0[3] = {-PB2_INFINITY, -PB2_INFINITY, -PB2_INFINITY};
            float l1[3] = {PB2_INFINITY, PB2_INFINITY, PB2_INFINITY}, h1[3] = {-PB2_INFINITY, -PB2_INFINITY, -PB2_INFINITY};
            int count0 = 0, count1 = 0;
            for (int j = 0; j <= i; ++j) {
                for (int k = 0; k < 3; ++k) {
                    l0[k] = fminf(l0[k], lo[j][k]);
                    h0[k] = fmaxf(h0[k], hi[j][k]);
                }
                count0 += count[j];
            }
            for (int j = i + 1; j < nBuckets; ++j) {
                for (int k = 0; k < 3; ++k) {
                    l1[k] = fminf(l1[k], lo[j][k]);
                    h1[k] = fmaxf(h1[k], hi[j][k]);
                }
                count1 += count[j];
            }
            const float cost = .125f + (count0 * area(l0, h0) + count1 * area(l1, h1)) / area(bmin, bmax);
            if (i == 0 || cost < minCost) {
                minCost = cost;
                minCostSplitBucket = i;
            }
        }
        // std::partition for bidirectional iterators as libstdc++ writes it (bits/stl_algo.h __partition): the order of
        // the two halves it leaves behind is part of the result
        int first = start, last = end;
        for (;;) {
            for (;;) {
                if (first == last) break;
                if (bucketOf(w.order[first]) <= minCostSplitBucket) ++first;
                else break;
            }
            if (first == last) break;
            --last;
            for (;;) {
                if (first == last) break;
                if (!(bucketOf(w.order[last]) <= minCostSplitBucket)) --last;
                else break;
            }
            if (first == last) break;
            const int tmp = w.order[first];
            w.order[first] = w.order[last];
            w.order[last] = tmp;
            ++first;
        }
        const int mid = first;
        pb2_build_node &nd = w.nodes[u];
        for (int k = 0; k < 3; ++k) {
            nd.bmin[k] = bmin[k];   // == Union of the two children's bounds (min / max are exact)
            nd.bmax[k] = bmax[k];
        }
        nd.split_axis = dim;
        nd.n_primitives = 0;
        nd.first_prim_offset = 0;
        w.stack[sp++] = make_int4(mid, end, u, 1);
        w.stack[sp++] = make_int4(start, mid, u, 0);   // the first subtree is built (and numbered) first
    }
    auto sizeOf = [&](int child) { return child >= 0 ? w.size[child] : treeletNodes[-(child + 1)]; };
    for (int u = nUpper - 1; u >= 0; --u) w.size[u] = 1 + sizeOf(w.nodes[u].child[0]) + sizeOf(w.nodes[u].child[1]);
    if (nUpper > 0) w.offset[0] = 0;
    for (int u = 0; u < nUpper; ++u) {
        const int a = w.nodes[u].child[0], b = w.nodes[u].child[1];
        const int offA = w.offset[u] + 1, offB = offA + sizeOf(a);
        if (a >= 0) w.offset[a] = offA;
        else w.treeletBase[-(a + 1)] = offA;
        if (b >= 0) w.offset[b] = offB;
        else w.treeletBase[-(b + 1)] = offB;
        pb2_bvh_node out;
        for (int k = 0; k < 3; ++k) {
            out.bmin[k] = w.nodes[u].bmin[k];
            out.bmax[k] = w.nodes[u].bmax[k];
        }
        out.offset = offB;    // secondChildOffset
        out.n_prims = 0;
        out.axis = (uint8_t)w.nodes[u].split_axis;
        out.pad = 0;
        linear[w.offset[u]] = out;
    }
    w.counts[0] = nUpper;
    w.counts[1] = nUpper > 0 ? w.size[0] : treeletNodes[0];
}
// flattenBVHTree for the treelets: emitLBVH numbered each treelet's nodes in depth-first order already, so a treelet lands
// in the linear array as one block and only the child references change base.  One block per treelet.
__global__ void k_hlbvh_flatten(const pb2_build_node *pool, const int2 *treelets, const int *treeletNodes, const int *treeletBase,
                                int nTreelets, pb2_bvh_node *linear) {
    for (int t = blockIdx.x; t < nTreelets; t += gridDim.x) {
        const int poolBase = 2 * treelets[t].x, n = treeletNodes[t], linBase = treeletBase[t];
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const pb2_build_node &nd = pool[poolBase + i];
            pb2_bvh_node out;
            for (int k = 0; k < 3; ++k) {
                out.bmin[k] = nd.bmin[k];
                out.bmax[k] = nd.bmax[k];
            }
            if (nd.n_primitives > 0) {
                out.offset = nd.first_prim_offset;
                out.n_prims = (uint16_t)nd.n_primitives;
                out.axis = 0;
            } else {
                out.offset = linBase + (nd.child[1] - poolBase);
                out.n_prims = 0;
                out.axis = (uint8_t)nd.split_axis;
            }
            out.pad = 0;
            linear[linBase + i] = out;
        }
    }
}
}  // namespace

// Both HLBVH entry points.  nodes == nullptr: pb2_hlbvh_treelets (the treelets come back as build nodes, the caller builds
// the tree above them); otherwise pb2_hlbvh_build (everything on the device, the finished LinearBVHNode array comes back).
static int hlbvhOnDevice(const float *prim_bounds, int64_t n, int32_t max_prims_in_node, pb2_build_node *pool, int32_t *ordered_prims,
                         int32_t *treelet_roots, int32_t *n_treelets, pb2_bvh_node *nodes, int64_t *n_nodes, double *device_ms) {
    int rc = requireDevice();
    if (rc) return rc;
    if (n <= 0 || n >= (int64_t)1 << 30) return setError(PB2_ERR_INVALID, "primitive count out of range");
    const int N = (int)n;
    float *dBounds = nullptr;
    unsigned *dBox = nullptr, *dCodes = nullptr, *dCodesSorted = nullptr;
    int *dIndex = nullptr, *dSorted = nullptr, *dStart = nullptr, *dRoots = nullptr;
    int2 *dTreelets = nullptr;
    pb2_build_node *dPool = nullptr;
    int *dTreeletNodes = nullptr;
    pb2_bvh_node *dLinear = nullptr;
    HlbvhUpper up;
    memset(&up, 0, sizeof(up));
    void *dTemp = nullptr;
    size_t tempBytes = 0;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    std::vector<int> start(4096);
    std::vector<int2> treelets;
    cudaError_t e = cudaSuccess;
    auto step = [&](cudaError_t r) { if (e == cudaSuccess) e = r; return e == cudaSuccess; };
    step(cudaMalloc((void **)&dBounds, (size_t)N * 6 * sizeof(float)));
    step(cudaMalloc((void **)&dBox, 6 * sizeof(unsigned)));
    step(cudaMalloc((void **)&dCodes, (size_t)N * sizeof(unsigned)));
    step(cudaMalloc((void **)&dCodesSorted, (size_t)N * sizeof(unsigned)));
    step(cudaMalloc((void **)&dIndex, (size_t)N * sizeof(int)));
    step(cudaMalloc((void **)&dSorted, (size_t)N * sizeof(int)));
    step(cudaMalloc((void **)&dStart, 4096 * sizeof(int)));
    step(cudaMalloc((void **)&dRoots, 4096 * sizeof(int)));
    step(cudaMalloc((void **)&dTreelets, 4096 * sizeof(int2)));
    step(cudaMalloc((void **)&dPool, (size_t)2 * N * sizeof(pb2_build_node)));
    step(cudaMalloc((void **)&dTreeletNodes, 4096 * sizeof(int)));
    if (nodes) {
        step(cudaMalloc((void **)&dLinear, ((size_t)2 * N + 4096) * sizeof(pb2_bvh_node)));
        step(cudaMalloc((void **)&up.order, 4096 * sizeof(int)));
        step(cudaMalloc((void **)&up.box, 4096 * 6 * sizeof(float)));
        step(cudaMalloc((void **)&up.stack, 8192 * sizeof(int4)));
        step(cudaMalloc((void **)&up.nodes, 4096 * sizeof(pb2_build_node)));
        step(cudaMalloc((void **)&up.size, 4096 * sizeof(int)));
        step(cudaMalloc((void **)&up.offset, 4096 * sizeof(int)));
        step(cudaMalloc((void **)&up.treeletBase, 4096 * sizeof(int)));
        step(cudaMalloc((void **)&up.counts, 2 * sizeof(int)));
    }
    if (e == cudaSuccess) step(cub::DeviceRadixSort::SortPairs(nullptr, tempBytes, dCodes, dCodesSorted, dIndex, dSorted, N, 0, 30));
    step(cudaMalloc(&dTemp, tempBytes ? tempBytes : 1));
    step(cudaEventCreate(&e0));
    step(cudaEventCreate(&e1));
    step(cudaMemcpy(dBounds, prim_bounds, (size_t)N * 6 * sizeof(float), cudaMemcpyHostToDevice));
    if (e == cudaSuccess) {
        const unsigned init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
        step(cudaMemcpy(dBox, init, sizeof(init), cudaMemcpyHostToDevice));
        step(cudaMemset(dStart, 0xff, 4096 * sizeof(int)));
        step(cudaEventRecord(e0));
        const int threads = 256, blocks = (N + threads - 1) / threads;
        k_hlbvh_centroid_bounds<<<std::min(blocks, g_numSMs * 8), threads>>>(dBounds, N, dBox);
        k_hlbvh_morton<<<blocks, threads>>>(dBounds, N, dBox, dCodes, dIndex);
        // the reference's LSD radix sort over all 30 bits is a stable sort by the code; so is this one
        step(cub::DeviceRadixSort::SortPairs(dTemp, tempBytes, dCodes, dCodesSorted, dIndex, dSorted, N, 0, 30));
        k_hlbvh_treelet_starts<<<blocks, threads>>>(dCodesSorted, N, dStart);
        step(cudaGetLastError());
        step(cudaMemcpy(start.data(), dStart, 4096 * sizeof(int), cudaMemcpyDeviceToHost));
    }
    if (e == cudaSuccess) {
        for (int v = 0; v < 4096; ++v)
            if (start[v] >= 0) treelets.push_back(make_int2(start[v], 0));
        for (size_t i = 0; i < treelets.size(); ++i) treelets[i].y = (i + 1 < treelets.size() ? treelets[i + 1].x : N) - treelets[i].x;
        step(cudaMemcpy(dTreelets, treelets.data(), treelets.size() * sizeof(int2), cudaMemcpyHostToDevice));
        const int nT = (int)treelets.size();
        k_hlbvh_emit<<<(nT + 31) / 32, 32>>>(dBounds, dCodesSorted, dSorted, dTreelets, nT, max_prims_in_node, dPool, dRoots, dTreeletNodes);
        step(cudaGetLastError());
        if (nodes && e == cudaSuccess) {
            // the SAH tree over the treelet roots and the depth-first layout, without leaving the device
            k_hlbvh_upper<<<1, 32>>>(dPool, dRoots, dTreeletNodes, nT, up, dLinear);
            k_hlbvh_flatten<<<std::min(nT, g_numSMs * 8), 128>>>(dPool, dTreelets, dTreeletNodes, up.treeletBase, nT, dLinear);
            step(cudaGetLastError());
        }
        step(cudaEventRecord(e1));
        if (nodes) {
            int counts[2] = {0, 0};
            step(cudaMemcpy(counts, up.counts, sizeof(counts), cudaMemcpyDeviceToHost));
            if (e == cudaSuccess) {
                *n_nodes = counts[1];
                step(cudaMemcpy(nodes, dLinear, (size_t)counts[1] * sizeof(pb2_bvh_node), cudaMemcpyDeviceToHost));
            }
        } else {
            step(cudaMemcpy(pool, dPool, (size_t)2 * N * sizeof(pb2_build_node), cudaMemcpyDeviceToHost));
            step(cudaMemcpy(treelet_roots, dRoots, treelets.size() * sizeof(int), cudaMemcpyDeviceToHost));
        }
        step(cudaMemcpy(ordered_prims, dSorted, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost));
        float ms = 0;
        if (e == cudaSuccess && cudaEventElapsedTime(&ms, e0, e1) == cudaSuccess && device_ms) *device_ms = ms;
        if (n_treelets) *n_treelets = (int32_t)treelets.size();
    }
    for (void *p : {(void *)dBounds, (void *)dBox, (void *)dCodes, (void *)dCodesSorted, (void *)dIndex, (void *)dSorted, (void *)dStart,
                    (void *)dRoots, (void *)dTreelets, (void *)dPool, dTemp, (void *)dTreeletNodes, (void *)dLinear, (void *)up.order,
                    (void *)up.box, (void *)up.stack, (void *)up.nodes, (void *)up.size, (void *)up.offset, (void *)up.treeletBase,
                    (void *)up.counts})
        cudaFree(p);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (e != cudaSuccess) return setError(PB2_ERR_CUDA, std::string("HLBVH build on the device: ") + cudaGetErrorString(e));
    return PB2_OK;
}

extern "C" int pb2_hlbvh_treelets(const float *prim_bounds, int64_t n, int32_t max_prims_in_node, pb2_build_node *pool,
                                  int32_t *ordered_prims, int32_t *treelet_roots, int32_t *n_treelets, double *device_ms) {
    if (!prim_bounds || !pool || !ordered_prims || !treelet_roots || !n_treelets) return setError(PB2_ERR_INVALID, "null argument");
    return hlbvhOnDevice(prim_bounds, n, max_prims_in_node, pool, ordered_prims, treelet_roots, n_treelets, nullptr, nullptr, device_ms);
}

extern "C" int pb2_hlbvh_build(const float *prim_bounds, int64_t n, int32_t max_prims_in_node, pb2_bvh_node *nodes, int64_t *n_nodes,
                               int32_t *ordered_prims, double *device_ms) {
    if (!prim_bounds || !nodes || !n_nodes || !ordered_prims) return setError(PB2_ERR_INVALID, "null argument");
    return hlbvhOnDevice(prim_bounds, n, max_prims_in_node, nullptr, ordered_prims, nullptr, nullptr, nodes, n_nodes, device_ms);
}
