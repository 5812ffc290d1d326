// Wavefront organisation of SamplerIntegrator::Render + PathIntegrator::Li (included by pb2_cuda.cu).
//
// A pool of N path contexts (one camera sample in flight each) lives in HBM.  Every context holds
// the per-lane state machine of device/pb2_path.cuh: at any time it owns exactly one ray of one of
// three classes (path ray, shadow ray, MIS ray).  One ROUND is
//
//   k_wf_gen            contexts on the free list take the next work item (pixel, sample number),
//                       generate the camera ray (Halton dims 0-4, perspective camera) and join the
//                       trace list
//   k_wf_trace*         every listed context's ray is traced through the BVH (closest hit or any
//                       hit); the context is appended to the shade list (path ray) or the light list
//                       (shadow / MIS ray)                                  <- the dominant kernel
//   k_wf_advance<false> (light list) adds ldLight / misTerm, then starts the next ray of the vertex
//                       or finishes the vertex: next path ray, or the sample is deposited in the film
//                       and the context goes to the free list
//   k_wf_advance<true>  (shade list) evaluates the whole path vertex (SurfaceInteraction, BSDF, light
//                       pick, light sample + MIS sample, continuation + Russian roulette), queues its rays
//
// so every kernel runs with all lanes of a warp in the same code, the trace kernel keeps only ray
// state in registers, and a finished sample is replaced immediately (the pool stays full until the
// work counter runs out).  Lists are plain index arrays with device-side counters; the host only
// reads two counters per round to detect the end.
#ifndef PB2_WAVEFRONT_CUH
#define PB2_WAVEFRONT_CUH

struct alignas(32) WfCtx {
    DLane ln;              // starts with {int state; DRay ray;} = 32 bytes: what the trace kernels read
    alignas(16) float4 hit;  // (leaf record, b0, b1, b2): written by the trace kernels as one 16-byte store
    float tHit;
    int found;               // 0 = miss, 1 = hit, 2 + i = hit inside instance i
    V2 pFilm;
};
static_assert(offsetof(WfCtx, ln) == 0 && offsetof(DLane, state) == 0 && offsetof(DLane, ray) == 4 && sizeof(DRay) == 28,
              "the trace kernels read the first 32 bytes of a context as {state, o, d, tMax}");
static_assert(offsetof(WfCtx, tHit) % 8 == 0 && offsetof(WfCtx, found) == offsetof(WfCtx, tHit) + 4, "tHit/found are stored as one float2");
static_assert(sizeof(DLane) == 192 && offsetof(WfCtx, hit) == 192 && offsetof(WfCtx, tHit) == 208 && offsetof(WfCtx, pFilm) == 216 &&
                  sizeof(WfCtx) == 224 && sizeof(WfCtx) % 32 == 0,
              "a context is seven whole 32-byte sectors: the lane (six), then hit, tHit / found and pFilm (one)");

// ---------------------------------------------------------------------------------------------
// The list kernels (gen, light step, shade step) do not work on a context in place.  The 32 lanes of a warp hold 32
// unrelated contexts, so every scalar field access would be an instruction that touches 32 sectors of HBM, and every
// store of 4-12 bytes would leave a partial sector in L2.  Instead the warp copies its 32 contexts into shared memory with
// 16-byte streaming loads (each instruction: 512 contiguous bytes of ~2.3 contexts, every fetched sector used whole),
// each thread works on its copy, and the warp writes back the sectors the kernel can change with 16-byte streaming
// stores.  Streaming (evict-first) because a context is touched once per kernel: the BVH, which the other pipeline's
// trace launch is reading at the same time, should keep the L2.
// ---------------------------------------------------------------------------------------------
// A context in shared memory: WfCtx's bytes, padded from 224 to 232.  At 56 words per slot the 32 lanes of a warp
// reach 4 of the 32 banks with a 4-byte access (8-way conflicts); at 58 words, 16 with a 4-byte access and all 32 with
// an 8-byte one.
struct WfSlot {
    DLane ln;
    float hit[4];   // (leaf record, b0, b1, b2)
    float tHit;
    int found;
    V2 pFilm;
    int pad[2];
};
static_assert(offsetof(WfSlot, hit) == offsetof(WfCtx, hit) && offsetof(WfSlot, tHit) == offsetof(WfCtx, tHit) &&
                  offsetof(WfSlot, found) == offsetof(WfCtx, found) && offsetof(WfSlot, pFilm) == offsetof(WfCtx, pFilm) &&
                  sizeof(WfSlot) == 232 && alignof(WfSlot) == 8,
              "a slot holds a context's bytes at the context's offsets, 8-byte aligned, 58 words apart");

// Bytes at the start of a lane that a kernel can change and writes back (whole sectors):
//   WF_OUT_START  k_wf_gen: laneStartPath sets every field before lightNum; lightNum and pick (the rest of the third
//                 sector) are set by the shade step before anything reads them
//   WF_OUT_LIGHT  k_wf_advance<light>: lightAdvance changes state, ray, L, beta, bounces and ldSum, all below misTerm
//   WF_OUT_SHADE  k_wf_advance<shade>: the whole lane
enum { WF_OUT_START = 96, WF_OUT_LIGHT = 128, WF_OUT_SHADE = (int)sizeof(DLane) };
static_assert(offsetof(DLane, lightNum) == 88 && offsetof(DLane, pick) == 92 && offsetof(DLane, ldSum) == 96 && offsetof(DLane, ldLight) == 108 &&
                  offsetof(DLane, bounces) < 96 && offsetof(DLane, misTerm) == 120,
              "the written-back prefixes above cover the fields their kernels change");

// The lane index, read anew at every call: derived from threadIdx, the chunk addresses of the copies below are loop
// invariants of a list kernel's grid-stride loop, and the compiler hoists all ~50 of them out of it (the shade step then
// spills ~500 bytes).
__device__ __forceinline__ int wfLaneId() {
    int lane;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
    return lane;
}

// Sectors of a context that a kernel reads (bit s: bytes 32 s .. 32 s + 31), staged in by wfStageIn:
//   WF_IN_ALL    the light step: every field
//   WF_IN_SHADE  the shade step: sectors 0-2 (state, ray, L, beta, smp, bounces, specularBounce, camRay, etaScale) and 6
//                (hit, tHit, found, pFilm).  Sectors 3-5 (ldSum, ldLight, misTerm, misO / misD, nextO / nextD, betaNext) are
//                dead on entry to shadeVertex: each is written by the vertex before anything reads it (lightAdvance and
//                finishVertex read them only under the doNEE / hasMis / hasNext flags this vertex sets).  The write-back is
//                still WF_OUT_SHADE: where the vertex does not write them, the slot's stale bytes go back to dead fields.
enum { WF_IN_ALL = 0x7f, WF_IN_SHADE = 0x47 };
static_assert(offsetof(DLane, etaScale) + sizeof(float) <= 96 && offsetof(DLane, smp) + sizeof(DSampler) <= 96 &&
                  offsetof(DLane, ldSum) == 96 && offsetof(DLane, betaNext) + sizeof(V3) <= 192 && offsetof(WfCtx, hit) == 192 &&
                  offsetof(WfCtx, pFilm) + sizeof(V2) <= 224,
              "WF_IN_SHADE: the fields shadeVertex reads on entry lie in sectors 0-2 and 6, the dead ones in sectors 3-5");

// The 16-byte chunk of a context that is the kk-th of those SECTORS cover.
template <unsigned SECTORS>
__device__ __forceinline__ int wfStagedChunk(int kk) {
    if (SECTORS == WF_IN_ALL) return kk;
    const int n = kk >> 1;
    int s = 0, seen = 0;
#pragma unroll
    for (int t = 0; t < 7; ++t)
        if ((SECTORS >> t) & 1u) {
            s = n == seen ? t : s;
            ++seen;
        }
    return 2 * s + (kk & 1);
}

// Warp-collective (all 32 lanes, converged): the SECTORS of lane l's context c (c < 0: none) are copied into
// warpSlots[l], at their offsets.  16-byte loads in two batches per lane, all of a batch in flight at once (WF_IN_ALL:
// seven loads each; WF_IN_SHADE: four).
template <unsigned SECTORS = WF_IN_ALL>
__device__ __forceinline__ void wfStageIn(const WfCtx *ctx, WfSlot *warpSlots, int c) {
    constexpr int NSECT = ((SECTORS >> 0) & 1) + ((SECTORS >> 1) & 1) + ((SECTORS >> 2) & 1) + ((SECTORS >> 3) & 1) +
                          ((SECTORS >> 4) & 1) + ((SECTORS >> 5) & 1) + ((SECTORS >> 6) & 1);
    static_assert(SECTORS <= WF_IN_ALL && NSECT > 0, "sectors of a 224-byte context");
    constexpr int CHUNKS = 2 * NSECT, BATCH = NSECT;
    const int lane = wfLaneId();
    __syncwarp();
#pragma unroll
    for (int b = 0; b < 2; ++b) {
        uint4 v[BATCH];
        int cs[BATCH];
#pragma unroll
        for (int it = 0; it < BATCH; ++it) {
            const int q = (b * BATCH + it) * 32 + lane, j = q / CHUNKS, kk = q % CHUNKS;
            const int k = wfStagedChunk<SECTORS>(kk);
            cs[it] = __shfl_sync(0xffffffffu, c, j);
            if (cs[it] >= 0) v[it] = __ldcs(reinterpret_cast<const uint4 *>(ctx + cs[it]) + k);
        }
#pragma unroll
        for (int it = 0; it < BATCH; ++it) {
            const int q = (b * BATCH + it) * 32 + lane, j = q / CHUNKS, kk = q % CHUNKS;
            const int k = wfStagedChunk<SECTORS>(kk);
            if (cs[it] >= 0) {
                uint2 *s = reinterpret_cast<uint2 *>(reinterpret_cast<char *>(&warpSlots[j]) + 16 * k);
                s[0] = make_uint2(v[it].x, v[it].y);
                s[1] = make_uint2(v[it].z, v[it].w);
            }
        }
    }
    __syncwarp();
}

// Warp-collective: the first BYTES bytes of lane l's slot go back to its context c (c < 0: none).
template <int BYTES>
__device__ __forceinline__ void wfStageOut(WfCtx *ctx, const WfSlot *warpSlots, int c) {
    static_assert(BYTES % 32 == 0 && BYTES <= (int)sizeof(DLane), "whole sectors of the lane");
    constexpr int CHUNKS = BYTES / 16;
    const int lane = wfLaneId();
    __syncwarp();
#pragma unroll
    for (int it = 0; it < CHUNKS; ++it) {
        const int q = it * 32 + lane, j = q / CHUNKS, k = q % CHUNKS;
        const int cj = __shfl_sync(0xffffffffu, c, j);
        if (cj >= 0) {
            const uint2 *s = reinterpret_cast<const uint2 *>(reinterpret_cast<const char *>(&warpSlots[j]) + 16 * k);
            const uint2 lo = s[0], hi = s[1];
            __stcs(reinterpret_cast<uint4 *>(ctx + cj) + k, make_uint4(lo.x, lo.y, hi.x, hi.y));
        }
    }
    __syncwarp();
}

// WQ_RETRY: path vertices deferred by the shade step (lazy light distribution), shaded again after k_lightdist_build
enum { WQ_TRACE0 = 0, WQ_TRACE1 = 1, WQ_SHADE = 2, WQ_LIGHT = 3, WQ_FREE0 = 4, WQ_FREE1 = 5, WQ_CURSOR = 6, WQ_RETRY = 7, WQ_COUNT = 8 };
// WQ_FINISH: the counter that holds k_wf_finish's decision of the round (0 = not taken yet), read by k_wf_reset.  It is
// WQ_RETRY's: frames with a tail kernel are never lazily lit, so their retry list is never used.
enum { WQ_FINISH = WQ_RETRY, WF_FINISH_WAIT = 1, WF_FINISH_GO = 2 };

struct WfPool {
    int capacity;
    WfCtx *ctx;
    int *queue[WQ_COUNT];     // capacity entries each; WQ_CURSOR is a counter only, WQ_RETRY exists for lazy scenes only
    unsigned *counts;         // WQ_COUNT counters
    unsigned long long *ctr;  // the scene's CTR_* counters (ray / traversal statistics)
    int2 *spill;              // k_wf_trace_pool: stack entries beyond its shared-memory depth, [warp][slot][PL_SPILL]
};

// pool.queue[q] for a q known only at run time, as selects over the kernel parameter: indexing the parameter's array
// directly copies the whole WfPool to every thread's stack at kernel entry.  The empty asm hides each entry from the
// compiler, which would otherwise fold the selects back into that indexed load.
__device__ __forceinline__ int *wfQueue(const WfPool &pool, int q) {
    int *list = pool.queue[0];
#pragma unroll
    for (int k = 1; k < WQ_COUNT; ++k) {
        int *entry = pool.queue[k];
        asm("" : "+l"(entry));
        list = q == k ? entry : list;
    }
    return list;
}

// warp-aggregated append of one index per participating lane
__device__ __forceinline__ void wfPush(int *queue, unsigned *counter, int value, bool participate) {
    unsigned mask = __ballot_sync(0xffffffffu, participate);
    if (!mask) return;
    int lane = threadIdx.x & 31;
    int leader = __ffs(mask) - 1;
    unsigned base = 0;
    if (lane == leader) base = atomicAdd(counter, (unsigned)__popc(mask));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (participate) queue[base + __popc(mask & ((1u << lane) - 1u))] = value;
}

__device__ __forceinline__ void wfCountRays(unsigned long long *counters, unsigned regular, unsigned shadow) {
    for (int o = 16; o > 0; o >>= 1) {
        regular += __shfl_down_sync(0xffffffffu, regular, o);
        shadow += __shfl_down_sync(0xffffffffu, shadow, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (regular) atomicAdd(&counters[CTR_REGULAR], (unsigned long long)regular);
        if (shadow) atomicAdd(&counters[CTR_SHADOW], (unsigned long long)shadow);
    }
}

// What a CHAIN instantiation of the trace kernel needs to advance a context itself when a shadow or MIS ray ends (the work of
// k_wf_advance<light>): the scene and the frame's parameters as objects in device memory, the film, the list of freed contexts.
struct WfChain {
    const DScene *sc;
    const DRenderParams *rp;
    float4 *film;
    int freeQ;
    int pad;
};

// The light step for ONE context, inside the trace kernel: lightAdvance (shadow ray: add the light sample if unoccluded;
// MIS ray: add the BSDF sample if it reached the light), then the vertex's next ray - the MIS ray, or the continuation of
// the path - or the end of the path (the sample goes to the film).  Returns the lane's new state.  Out of line: the
// traversal loop must not carry its registers.
// The hit is the one the trace kernel has just stored in the context ((leaf, b0, b1, b2), tHit, the found code), decoded
// as k_wf_advance does: a MIS ray that reaches a one-sided area light is counted only when the light's surface at the
// hit faces the ray, and a triangle's surface is built from the hit's barycentrics (its shading normals) and instance.
template <int F>
__device__ __noinline__ int wfChainLight(const WfChain &ch, WfCtx *cx, bool found) {
    DLane &ln = cx->ln;
    const float4 h4 = cx->hit;
    const int foundCode = cx->found;
    DHit hit;
    hit.leaf = __float_as_int(h4.x);
    hit.b0 = h4.y;
    hit.b1 = h4.z;
    hit.b2 = h4.w;
    hit.inst = foundCode >= 2 ? foundCode - 2 : -1;
    lightAdvance<F>(*ch.sc, ln, found, hit, cx->tHit);
    if (ln.state == LS_IDLE) addSample(*ch.rp, ch.film, cx->pFilm, guardRadiance(ln.L));
    return ln.state;
}

// A context takes the next work item (pixel, sample number) and starts its camera ray: GetCameraSample + GenerateRay
// (Halton dims 0-4, perspective camera).  Warp-collective: all 32 lanes call it, `want` says which of them take part; work
// items that map outside the sample bounds / pixel bounds are skipped (integrator.cpp:274), so a lane may draw several.
// Returns false for a lane that did not want a sample or found the work counter exhausted (its context retires).
// The new lane and pFilm are built in `slot`.
template <bool GENERAL>
__device__ __forceinline__ bool wfStartSample(const DRenderParams &rp, const WfPool &pool, WfSlot &slot, bool want, unsigned *cameraRays) {
    bool started = false;
    while (__any_sync(0xffffffffu, want && !started)) {
        const bool draw = want && !started;
        const unsigned mask = __ballot_sync(0xffffffffu, draw);
        const int lane = threadIdx.x & 31, leader = __ffs(mask) - 1;
        unsigned long long w0 = 0;
        if (lane == leader) w0 = atomicAdd(&pool.ctr[CTR_WORK], (unsigned long long)__popc(mask));
        w0 = __shfl_sync(0xffffffffu, w0, leader);
        if (draw) {
            const long long item = (long long)w0 + __popc(mask & ((1u << lane) - 1u));
            if (item >= rp.nWorkItems) {
                want = false;  // no work left
            } else {
                int px, py, sample;
                if (decodeWork(rp, item, &px, &py, &sample)) {
                    DSampler smp;
                    smp.index = sampleIndex<GENERAL>(rp.halton, px, py, sample);
                    smp.dim = 0;
                    V2 pFilm;
                    DRay ray = generateCameraRay<GENERAL>(rp.cam, rp.halton, smp, px, py, &pFilm);
                    laneStartPath(slot.ln, ray, smp);
                    slot.pFilm = pFilm;
                    ++*cameraRays;
                    started = true;
                }
            }
        }
    }
    return started;
}

// Contexts on the free list take their next sample.  (Not inside k_wf_advance: there the few lanes of a warp that end a
// path would run this code alone inside the register-heavy, low-occupancy shade kernel.)
// The scene and the frame's parameters come as objects in device memory (renderWavefront uploads them once per render):
// a struct passed by value whose address reaches a device function is copied to every thread's stack at kernel entry.
// The new lanes are built in shared memory and written out as whole sectors (WF_OUT_START), pFilm as one 8-byte store.
template <int F>
__global__ void __launch_bounds__(128) k_wf_gen(const DRenderParams *__restrict__ rpp, WfPool pool, int freeQ, int traceQ) {
    __shared__ WfSlot stage[128];
    WfSlot &slot = stage[threadIdx.x];
    WfSlot *warpSlots = stage + (threadIdx.x & ~31u);
    const DRenderParams &rp = *rpp;
    const int *freeList = wfQueue(pool, freeQ);
    int *traceList = wfQueue(pool, traceQ);
    const unsigned n = pool.counts[freeQ];
    unsigned stride = gridDim.x * blockDim.x;
    unsigned cameraRays = 0;
    for (unsigned base = blockIdx.x * blockDim.x; base < n; base += stride) {
        unsigned i = base + threadIdx.x;
        const bool have = i < n;
        const int c = have ? freeList[i] : -1;
        const bool started = wfStartSample<(F & SHADE_SOBOL) != 0>(rp, pool, slot, have, &cameraRays);
        if (started) {
            slot.ln.lightNum = 0;   // (not read before the shade step sets them: written only to store no stale shared memory)
            slot.ln.pick = 0;
            __stcs(reinterpret_cast<float2 *>(&pool.ctx[c].pFilm), make_float2(slot.pFilm.x, slot.pFilm.y));
        }
        wfStageOut<WF_OUT_START>(pool.ctx, warpSlots, started ? c : -1);
        wfPush(traceList, &pool.counts[traceQ], c, started);
    }
    for (int o = 16; o > 0; o >>= 1) cameraRays += __shfl_down_sync(0xffffffffu, cameraRays, o);
    if ((threadIdx.x & 31) == 0 && cameraRays) {
        atomicAdd(&pool.ctr[CTR_CAMERA], (unsigned long long)cameraRays);
        atomicAdd(&pool.ctr[CTR_REGULAR], (unsigned long long)cameraRays);  // every camera ray is a Scene::Intersect call
    }
}

// Trace feature mask: what an instantiation of k_wf_trace_w or k_wf_trace is compiled for (its template argument T).
// The scene bits compile a primitive or a test into the leaf step; an instanced kernel compiles the sphere code as well.
// The variant bits choose among implementations that return the same records.  selectTraceKernel (pb2_cuda.cu) turns a
// scene and its PB2_FLAG_* into the mask wanted; every instantiation is listed once there.
enum {
    TRACE_SPHERES = 1,
    TRACE_INST = 2,
    TRACE_ALPHA = 4,            // alpha-masked triangles: a hit on a texel of value 0 is no hit
    TRACE_LD128 = 8,            // a record as 16-byte loads; clear: pairs of them as one 32-byte load (ldg256)
    TRACE_SMALL_STACK = 16,     // 4 instead of 16 stack entries per lane in shared memory (the spill path runs)
    TRACE_LEAF_TMA = 32,        // leaf records staged into shared memory by the TMA unit (triangles, two-child records)
    TRACE_CHAIN = 64,           // the light step runs inside the trace kernel (WfChain)
    TRACE_DEEP = 128,           // k_wf_trace: stack entries beyond the 32 in shared memory spill to local memory
};

// ---------------------------------------------------------------------------------------------
// Trace kernel, plain form: one thread per listed ray, BVHAccel::Intersect[P] exactly as written in
// device/pb2_scene.cuh.  Used when PB2_FLAG_COUNT_TRAVERSAL asks for node / primitive counters
// (COUNT) and as the simplest statement of what the tuned kernels below compute.
// ---------------------------------------------------------------------------------------------
template <bool COUNT>
__global__ void __launch_bounds__(128) k_wf_trace_plain(DScene sc, WfPool pool, int traceQ, WfChain) {
    unsigned long long *counters = pool.ctr;
    unsigned n = pool.counts[traceQ];
    unsigned stride = gridDim.x * blockDim.x;
    DCounters ctr;
    ctr.nodes = ctr.prims = 0;
    for (unsigned base = blockIdx.x * blockDim.x; base < n; base += stride) {
        unsigned i = base + threadIdx.x;
        bool have = i < n;
        int c = have ? pool.queue[traceQ][i] : 0;
        int state = LS_IDLE;
        if (have) {
            const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
            float4 a = p[0], b = p[1];
            state = __float_as_int(a.x);
            DRay ray;
            ray.o = mk3(a.y, a.z, a.w);
            ray.d = mk3(b.x, b.y, b.z);
            ray.tMax = b.w;
            float tMax = ray.tMax;
            DHit hit;
            hit.leaf = -1;
            hit.b0 = hit.b1 = hit.b2 = 0;
            hit.inst = -1;
            bool found = traverseAnyOrClosest(sc, ray, state == LS_SHADOW, &tMax, &hit, COUNT ? &ctr : nullptr);
            WfCtx &cx = pool.ctx[c];
            cx.hit = make_float4(__int_as_float(hit.leaf), hit.b0, hit.b1, hit.b2);
            cx.tHit = tMax;
            cx.found = found ? (state != LS_SHADOW && hit.inst >= 0 ? 2 + hit.inst : 1) : 0;
        }
        wfPush(pool.queue[WQ_SHADE], &pool.counts[WQ_SHADE], c, have && state == LS_PATH);
        wfPush(pool.queue[WQ_LIGHT], &pool.counts[WQ_LIGHT], c, have && state != LS_PATH);
    }
    if (COUNT) {
        unsigned long long n0 = ctr.nodes, n1 = ctr.prims;
        for (int o = 16; o > 0; o >>= 1) {
            n0 += __shfl_down_sync(0xffffffffu, n0, o);
            n1 += __shfl_down_sync(0xffffffffu, n1, o);
        }
        if ((threadIdx.x & 31) == 0) {
            atomicAdd(&counters[CTR_NODES], n0);
            atomicAdd(&counters[CTR_PRIMS], n1);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Trace kernel, tuned form: persistent warps.  Each lane walks its own ray through the BVH with
// the reference's visiting order (near child first, explicit stack, every primitive of a reached
// leaf), but the WARP decides by ballot which of three steps to run next, so that the lanes inside
// a step are mostly all busy:
//   node step   lanes that stand at a node: fetch the 32-byte node (two 16-byte loads), slab test,
//               descend / pop; NSUB visits per scheduling round
//   leaf step   lanes that reached a leaf wait until LEAF_T lanes did (or nobody can walk any
//               more), then test their leaf's primitives together (three 16-byte loads each)
//   fetch step  lanes whose ray is finished wait until FETCH_T lanes are (or nothing else is
//               left), then store their results, append their context to the shade / light list,
//               and take the next rays of the trace list (one warp-aggregated atomic)
// Node-visit and primitive-test counts per ray are the reference's; only the interleaving across
// lanes differs.  Details:
//   * the traversal stack lives in shared memory, [depth][thread] (conflict-free), not in local
//     memory, where it competes with node fetches for L1; entries beyond SDEPTH spill to a small local array
//     (TRACE_DEEP), or the host picks this kernel only when the BVH depth fits;
//   * the closest hit so far is written straight into the context (it changes ~1.5 times per ray);
//     only tMax stays in a register -> 54 registers for triangles, 8 blocks of 128 threads per SM;
//   * the descend / pop tail of the node step touches one stack slot with selects instead of
//     diverging into push and pop branches;
//   * context words are read / written with streaming hints so nodes + leaf records stay in L2.
// Two tunings: triangles, and spheres (instanced kernels included; always with TRACE_DEEP).
// ---------------------------------------------------------------------------------------------
// TRACE_INST: object instances (TransformedPrimitive).  An instance is a leaf primitive: the lane saves
// (tMax, rest of the leaf) in a 3-entry frame on its stack, takes the ray to instance space
// (Transform::operator()(Ray), transform.h:251-264) and walks the object's BVH with `instBase` as
// the stack floor; when that walk ends it comes back through the leaf step (F_EXIT), restores the
// world-space ray from its context and continues with the rest of the leaf - r.tMax = ray.tMax
// (primitive.cpp:83) if something was hit inside, the saved tMax otherwise.
template <int T>
__global__ void __launch_bounds__(128, (T & TRACE_SPHERES) ? 6 : 8) k_wf_trace(DScene sc, WfPool pool, int traceQ, WfChain) {
    // static: for plain constexpr locals that the lambdas below read, nvcc generates other code than for template arguments
    static constexpr bool SPHERES = (T & TRACE_SPHERES) != 0, INST = (T & TRACE_INST) != 0, DEEP = (T & TRACE_DEEP) != 0;
    static constexpr int LEAF_T = SPHERES ? 8 : 12, FETCH_T = 8, NSUB = SPHERES ? 2 : 4, SDEPTH = 32;
    __shared__ int sstack[SDEPTH][128];
    int lstack[DEEP ? 64 - SDEPTH : 1];
    const unsigned FULL = 0xffffffffu;
    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const unsigned n = pool.counts[traceQ];
    enum { M_FETCH = 0, M_NODE = 1, M_LEAF = 2 };
    enum { F_ANY = 1, F_FOUND = 2, F_EXHAUSTED = 4, F_EXIT = 8, F_HITIN = 16 };
    int inst = -1, hitInst = -1, instBase = 0;   // INST only; instBase = 0 outside an instance
    int mode = M_FETCH;
    int c = -1;
    int flags = 0;
    DRaySetup rs;
    rs.o = rs.invDir = mk3(0, 0, 0);
    rs.neg0 = rs.neg1 = rs.neg2 = 0;
    rs.kx = rs.ky = rs.kz = 0;
    rs.Sx = rs.Sy = rs.Sz = 0;
    float tMax = 0;
    int cur = 0, sp = 0, leafFirst = 0, leafN = 0;
    auto stackGet = [&](int slot) -> int { return (!DEEP || slot < SDEPTH) ? sstack[slot][tid] : lstack[DEEP ? slot - SDEPTH : 0]; };
    auto stackPut = [&](int slot, int v) {
        if (!DEEP || slot < SDEPTH) sstack[slot][tid] = v;
        else lstack[DEEP ? slot - SDEPTH : 0] = v;
    };
    while (true) {
        unsigned mNode = __ballot_sync(FULL, mode == M_NODE);
        unsigned mLeaf = __ballot_sync(FULL, mode == M_LEAF);
        unsigned mFetch = __ballot_sync(FULL, mode == M_FETCH && !((flags & F_EXHAUSTED) && c < 0));
        int nNode = __popc(mNode), nLeaf = __popc(mLeaf), nFetch = __popc(mFetch);
        int step;
        if (nFetch >= FETCH_T || (nFetch > 0 && nNode == 0 && nLeaf == 0)) step = M_FETCH;
        else if (nLeaf >= LEAF_T || (nLeaf > 0 && nNode == 0)) step = M_LEAF;
        else if (nNode > 0) step = M_NODE;
        else break;

        if (step == M_NODE) {
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub) {
                if (mode == M_NODE) {
                    float4 n0 = ldg4(&sc.nodes[2 * (size_t)cur]);
                    float4 n1 = ldg4(&sc.nodes[2 * (size_t)cur + 1]);
                    bool pass = slabTest(n0, n1, rs, tMax);
                    uint32_t meta = floatBits(n1.w);
                    int nPrims = (int)(meta & 0xffffu);
                    int axis = (int)((meta >> 16) & 0xffu);
                    int isNeg = axis == 0 ? rs.neg0 : (axis == 1 ? rs.neg1 : rs.neg2);
                    int second = asInt(n1.z);
                    bool interior = pass && nPrims == 0;
                    bool leaf = pass && nPrims > 0;
                    int far = isNeg ? cur + 1 : second;
                    int near = isNeg ? second : cur + 1;
                    // one stack slot per visit: interior nodes store the far child at sp, every
                    // other outcome reads the slot below (the node it would pop)
                    int slot = interior ? sp : (sp > 0 ? sp - 1 : 0);
                    int top = stackGet(slot);
                    if (interior) stackPut(slot, far);
                    if (interior) {
                        cur = near;
                        ++sp;
                    } else if (leaf) {
                        leafFirst = second;
                        leafN = nPrims;
                        mode = M_LEAF;
                    } else if (sp == instBase) {
                        if (INST && inst >= 0) {
                            mode = M_LEAF;   // the object's BVH is exhausted: leave the instance in the leaf step
                            flags |= F_EXIT;
                            leafN = 0;
                        } else
                            mode = M_FETCH;
                    } else {
                        cur = top;
                        --sp;
                    }
                }
            }
        } else if (step == M_LEAF) {
            if (mode == M_LEAF) {
                if (INST && (flags & F_EXIT)) {
                    // back to world space (TransformedPrimitive::Intersect returns, primitive.cpp:82-86)
                    flags &= ~F_EXIT;
                    sp -= 3;
                    float saved = __int_as_float(stackGet(sp));
                    leafFirst = stackGet(sp + 1);
                    leafN = stackGet(sp + 2);
                    if (!(flags & F_HITIN)) tMax = saved;
                    const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                    float4 ra = p[0], rb = p[1];
                    rs = setupRay(mk3(ra.y, ra.z, ra.w), mk3(rb.x, rb.y, rb.z));
                    inst = -1;
                    instBase = 0;
                }
                bool finished = false, entered = false;
                const bool any = (flags & F_ANY) != 0;
                while (leafN > 0) {
                    const int idx = leafFirst;
                    ++leafFirst;
                    --leafN;
                    const float4 *rec = &sc.leafPrims[3 * (size_t)idx];
                    float4 a = ldg4(rec), b = ldg4(rec + 1), c4 = ldg4(rec + 2);
                    uint32_t pf = floatBits(b.w);
                    if (INST && (pf & LEAF_INSTANCE)) {
                        const int id = asInt(c4.w);
                        const DInstance &in = sc.instances[id];
                        const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                        float4 ra = p[0], rb = p[1];
                        DRay ray;
                        ray.o = mk3(ra.y, ra.z, ra.w);
                        ray.d = mk3(rb.x, rb.y, rb.z);
                        ray.tMax = rb.w;
                        DRay r2 = xfRay(in.w2i, ray, tMax);
                        stackPut(sp, __float_as_int(tMax));
                        stackPut(sp + 1, leafFirst);
                        stackPut(sp + 2, leafN);
                        sp += 3;
                        instBase = sp;
                        inst = id;
                        flags &= ~F_HITIN;
                        rs = setupRay(r2.o, r2.d);
                        tMax = r2.tMax;
                        if (in.root >= 0) {
                            cur = in.root;
                            mode = M_NODE;
                            leafN = 0;
                            entered = true;
                            break;
                        }
                        leafFirst = in.lone;   // one-primitive object: its record is the whole "leaf"
                        leafN = 1;
                        continue;
                    }
                    if (SPHERES && (pf & LEAF_SPHERE)) {
                        const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                        float4 ra = p[0], rb = p[1];
                        DRay ray;
                        ray.o = mk3(ra.y, ra.z, ra.w);
                        ray.d = mk3(rb.x, rb.y, rb.z);
                        ray.tMax = rb.w;
                        if (INST && inst >= 0) ray = xfRay(sc.instances[inst].w2i, ray, tMax);
                        float t, phi;
                        if (sphereLeafTest(sc, asInt(c4.w), ray, tMax, &t, &phi)) {
                            flags |= F_FOUND;
                            if (any) { finished = true; break; }
                            tMax = t;
                            if (INST) {
                                hitInst = inst;
                                if (inst >= 0) flags |= F_HITIN;
                            }
                            __stcs(reinterpret_cast<float4 *>(&pool.ctx[c].hit), make_float4(__int_as_float(idx), phi, 0.f, 0.f));
                        }
                        continue;
                    }
                    float t, b0, b1, b2;
                    if (triangleTest(mk3(a.x, a.y, a.z), mk3(b.x, b.y, b.z), mk3(c4.x, c4.y, c4.z), rs, tMax, &t, &b0, &b1, &b2)) {
                        if (any) { flags |= F_FOUND; finished = true; break; }
                        if (pf & LEAF_DEGENERATE) continue;
                        flags |= F_FOUND;
                        tMax = t;
                        if (INST) {
                            hitInst = inst;
                            if (inst >= 0) flags |= F_HITIN;
                        }
                        __stcs(reinterpret_cast<float4 *>(&pool.ctx[c].hit), make_float4(__int_as_float(idx), b0, b1, b2));
                    }
                }
                if (!entered) {
                    leafN = 0;
                    if (finished) mode = M_FETCH;
                    else if (sp == instBase) {
                        if (INST && inst >= 0) flags |= F_EXIT;   // stays a leaf lane: the next leaf step leaves the instance
                        else mode = M_FETCH;
                    } else {
                        --sp;
                        cur = stackGet(sp);
                        mode = M_NODE;
                    }
                }
            }
        } else {  // M_FETCH: flush finished rays, then take new ones
            bool flush = mode == M_FETCH && c >= 0;
            int state = LS_IDLE;
            if (flush) {
                WfCtx &cx = pool.ctx[c];
                state = (flags & F_ANY) ? LS_SHADOW : __ldcs(&cx.ln.state);
                const int foundCode = (flags & F_FOUND) ? ((INST && !(flags & F_ANY) && hitInst >= 0) ? 2 + hitInst : 1) : 0;
                __stcs(reinterpret_cast<float2 *>(&cx.tHit), make_float2(tMax, __int_as_float(foundCode)));
            }
            wfPush(pool.queue[WQ_SHADE], &pool.counts[WQ_SHADE], c, flush && state == LS_PATH);
            wfPush(pool.queue[WQ_LIGHT], &pool.counts[WQ_LIGHT], c, flush && state != LS_PATH);
            if (flush) c = -1;
            bool want = mode == M_FETCH && !(flags & F_EXHAUSTED);
            unsigned wantMask = __ballot_sync(FULL, want);
            if (wantMask) {
                int leader = __ffs(wantMask) - 1;
                unsigned base = 0;
                if (lane == leader) base = atomicAdd(&pool.counts[WQ_CURSOR], (unsigned)__popc(wantMask));
                base = __shfl_sync(FULL, base, leader);
                if (want) {
                    unsigned i = base + __popc(wantMask & ((1u << lane) - 1u));
                    if (i >= n)
                        flags |= F_EXHAUSTED;
                    else {
                        c = pool.queue[traceQ][i];
                        const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                        float4 ra = __ldcs(p), rb = __ldcs(p + 1);
                        flags = (__float_as_int(ra.x) == LS_SHADOW) ? F_ANY : 0;
                        rs = setupRay(mk3(ra.y, ra.z, ra.w), mk3(rb.x, rb.y, rb.z));
                        tMax = rb.w;
                        cur = 0;
                        sp = 0;
                        leafN = 0;
                        mode = M_NODE;
                        if (INST) {
                            inst = hitInst = -1;
                            instBase = 0;
                        }
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Trace kernel over the two-child records (DScene::wide, triangle scenes).  Same persistent-warp
// scheduling as k_wf_trace; what changes is the node step.  A lane stands at an INTERIOR node whose
// own box it has already passed, fetches that node's 64-B record and tests BOTH children's boxes:
//   * the near child (by the node's split axis and the ray's direction sign, bvh.cpp:684-690) is
//     entered at once when its box passes - the reference tests that box next, with the same tMax;
//   * the far child is pushed only if its box passes, together with its entry parameter tMin.  The
//     reference tests the far box when it pops it, possibly against a smaller tMax; the only term of
//     Bounds3::IntersectP that depends on ray.tMax is `tMin < ray.tMax` (geometry.h:1437), so a pop
//     re-evaluates exactly that with the stored tMin and skips the entry otherwise.
// Every box is therefore tested once per ray with the reference's verdict, leaves are reached in
// the reference's order, and the primitive tests are the reference's - but a ray makes one
// dependent fetch per interior node it descends into instead of one per node it touches
// (82 -> ~41 on the bench scene), and the two slab tests of a step are independent instructions.
// ---------------------------------------------------------------------------------------------
// WIDTH = 2: the two-child records (DScene::wide); WIDTH = 4: the four-child records (DScene::wide4,
// device/pb2_wide4.cuh) - two levels of the reference's tree per fetch: a visit tests the four
// grandchildren's boxes, continues with the first entered one in the reference's visiting order and
// defers the others (up to three stack entries, the next one to visit on top).
// T: the trace features (TRACE_*).  With TRACE_LEAF_TMA (an experiment, DESIGN.md section 3) the leaf records of the lanes
// that take a leaf step are staged into shared memory by the TMA unit - one cp.async.bulk (UBLKCP) of up to four 48-byte
// records per lane, completion counted by one mbarrier per warp - and the triangle tests read them from there.
// The resident blocks per SM an instantiation asks of the compiler (__launch_bounds__).
constexpr int traceMinBlocks(int width, int t) {
    if (width == 4) return (t & TRACE_SPHERES) ? 5 : 7;
    if (t & TRACE_LEAF_TMA) return 5;
    return (t & (TRACE_SPHERES | TRACE_ALPHA)) ? 6 : 9;
}
template <int WIDTH, int T>
__global__ void __launch_bounds__(128, traceMinBlocks(WIDTH, T)) k_wf_trace_w(DScene sc, WfPool pool, int traceQ, WfChain chain) {
    static_assert(WIDTH == 2 || WIDTH == 4, "two- or four-child records");
    static constexpr bool SPHERES = (T & TRACE_SPHERES) != 0, INST = (T & TRACE_INST) != 0, ALPHA = (T & TRACE_ALPHA) != 0;
    static constexpr bool LD128 = (T & TRACE_LD128) != 0, LEAFTMA = (T & TRACE_LEAF_TMA) != 0, CHAIN = (T & TRACE_CHAIN) != 0;
    static_assert(!LEAFTMA || (!SPHERES && !INST), "the staging experiment covers triangle scenes");
    // LEAF_T = 1: a warp turns to its leaves as soon as one lane holds one
    static constexpr int LEAF_T = 1, FETCH_T = 8, NSUB = 4, SDEPTH = (T & TRACE_SMALL_STACK) ? 4 : 16;
    constexpr int STAGED = 4;   // records staged per lane and leaf step (the reference's default maxnodeprims)
    __shared__ alignas(16) float4 sleaf[LEAFTMA ? 128 * 3 * STAGED : 1];
    __shared__ alignas(8) unsigned long long sbar[LEAFTMA ? 4 : 1];
    unsigned barPhase = 0;
    if (LEAFTMA) {
        if ((threadIdx.x & 31) == 0) {
            const unsigned bar = (unsigned)__cvta_generic_to_shared(&sbar[threadIdx.x >> 5]);
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    constexpr int BLOCK = 128;
    __shared__ int2 sstack[SDEPTH * BLOCK];   // [SDEPTH][BLOCK] of (child reference, tMin bits)
    __shared__ unsigned sCount[2];            // CHAIN: Scene::Intersect / IntersectP calls started in this block (regular, shadow)
    if (CHAIN) {
        if (threadIdx.x < 2) sCount[threadIdx.x] = 0;
        __syncthreads();
    }
    // entries beyond SDEPTH (rare: only passing far children are pushed).  Worst case: one entry per level of the
    // reference's <= 64-level stack for WIDTH 2, three per two levels for WIDTH 4, plus the instance frame
    int2 lstack[(WIDTH == 4 ? 100 : 66) - SDEPTH];
    const unsigned FULL = 0xffffffffu;
    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const unsigned n = pool.counts[traceQ];
    enum { M_FETCH = 0, M_NODE = 1, M_LEAF = 2 };
    enum { F_ANY = 1, F_FOUND = 2, F_EXHAUSTED = 4, F_EXIT = 8, F_HITIN = 16 };
    // INST (object instances): as in k_wf_trace - an instance is a leaf primitive; the lane pushes a
    // frame of two entries ((rest of the leaf), (tMax, -)), walks the object's records from the pseudo
    // record above its root with `instBase` as stack floor, and leaves through the leaf step (F_EXIT).
    int inst = -1, hitInst = -1, instBase = 0;
    auto stGet = [&](int i) -> int2 { return i < SDEPTH ? sstack[i * BLOCK + tid] : lstack[i - SDEPTH]; };
    auto stPut = [&](int i, int2 e) {
        if (i < SDEPTH) sstack[i * BLOCK + tid] = e;
        else lstack[i - SDEPTH] = e;
    };
    int mode = M_FETCH;
    int c = -1;
    int flags = 0;
    DRaySetup rs;
    rs.o = rs.invDir = mk3(0, 0, 0);
    rs.neg0 = rs.neg1 = rs.neg2 = 0;
    rs.kx = rs.ky = rs.kz = 0;
    rs.Sx = rs.Sy = rs.Sz = 0;
    rs.slow = 0;
    float tMax = 0;
    int cur = 0, sp = 0, leafFirst = 0, leafN = 0;
    while (true) {
        unsigned mNode = __ballot_sync(FULL, mode == M_NODE);
        unsigned mLeaf = __ballot_sync(FULL, mode == M_LEAF);
        unsigned mFetch = __ballot_sync(FULL, mode == M_FETCH && !((flags & F_EXHAUSTED) && c < 0));
        int nNode = __popc(mNode), nLeaf = __popc(mLeaf), nFetch = __popc(mFetch);
        int step;
        if (nFetch >= FETCH_T || (nFetch > 0 && nNode == 0 && nLeaf == 0)) step = M_FETCH;
        else if (nLeaf >= LEAF_T || (nLeaf > 0 && nNode == 0)) step = M_LEAF;
        else if (nNode > 0) step = M_NODE;
        else break;

        if (step == M_NODE) {
            // min / max slab tests unless some lane's ray has a non-finite origin or 1 / d (see slabTestPairFast)
            const bool warpSlow = __any_sync(FULL, rs.slow != 0);
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub) {
                {
                    // A lane whose last visit (or leaf) left nothing to descend into (cur < 0) takes its next
                    // pending far child.  Straight-line predicated code for the whole warp: nearly every visit
                    // has SOME lane that must pop, and those few lanes would otherwise run ~25 instructions
                    // alone while the rest of the warp waited.  A popped entry whose tMin no longer beats
                    // tMax is dropped (the reference's box test at the pop, bvh.cpp:694-697); the next visit
                    // pops again.
                    const bool need = (mode == M_NODE) & (cur < 0);
                    const bool empty = need & (sp == instBase);
                    const bool pop = need & !empty;
                    const int slot = pop ? sp - 1 : 0;
                    const int2 e = slot < SDEPTH ? sstack[slot * BLOCK + tid] : lstack[slot - SDEPTH];
                    sp = pop ? sp - 1 : sp;
                    const bool take = pop & (__int_as_float(e.y) < tMax);
                    const bool leafRef = take & (e.x < 0);
                    leafFirst = leafRef ? (e.x & (int)WIDE_LEAF_OFFSET_MASK) : leafFirst;
                    leafN = leafRef ? (((e.x >> WIDE_LEAF_COUNT_SHIFT) & 0xf) + 1) : leafN;
                    cur = (take & !leafRef) ? e.x : cur;
                    mode = leafRef ? (int)M_LEAF : mode;
                    if (empty) {
                        if (INST && inst >= 0) {
                            mode = M_LEAF;   // the object is exhausted: leave the instance in the leaf step
                            flags |= F_EXIT;
                            leafN = 0;
                        } else
                            mode = M_FETCH;
                    }
                }
                if (WIDTH == 4) {
                    if (mode == M_NODE && cur >= 0) {
                        const float4 *w = &sc.wide4[8 * (size_t)cur];
                        float4 q0, q1, q2, q3, q4, q5, q6, q7;
                        if (!LD128) {
                            ldg256(w, q0, q1);
                            ldg256(w + 2, q2, q3);
                            ldg256(w + 4, q4, q5);
                            ldg256(w + 6, q6, q7);
                        } else {
                            q0 = ldg4(w); q1 = ldg4(w + 1); q2 = ldg4(w + 2); q3 = ldg4(w + 3); q4 = ldg4(w + 4); q5 = ldg4(w + 5);
                            q6 = ldg4(w + 6);
                            q7.x = __uint_as_float(__ldg(reinterpret_cast<const unsigned *>(w + 7)));
                        }
                        const uint32_t meta = floatBits(q7.x);
                        const Wide4Visit v = warpSlow ? wide4Visit<false>(q0, q1, q2, q3, q4, q5, q6, meta, rs, tMax)
                                                      : wide4Visit<true>(q0, q1, q2, q3, q4, q5, q6, meta, rs, tMax);
                        const int refs[4] = {asInt(q6.x), asInt(q6.y), asInt(q6.z), asInt(q6.w)};
                        const int last = v.nPass - 1;
                        int ref = -1;
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const bool first = v.pass[k] & (v.after[k] == last);
                            ref = first ? refs[k] : ref;
                            // deferred: stack position sp + after puts the next one to visit on top.  One predicated
                            // shared-memory store; the local-memory spill is a branch that is almost never taken
                            const bool deferred = v.pass[k] & !first;
                            const int slot = sp + v.after[k];
                            const int2 e = make_int2(refs[k], __float_as_int(v.tMin[k]));
                            if (deferred & (slot < SDEPTH)) sstack[slot * BLOCK + tid] = e;
                            if (deferred & (slot >= SDEPTH)) lstack[slot - SDEPTH] = e;
                        }
                        sp += last > 0 ? last : 0;
                        const bool have = v.nPass > 0;
                        const bool isLeaf = have & (ref < 0);
                        leafFirst = isLeaf ? (ref & (int)WIDE_LEAF_OFFSET_MASK) : leafFirst;
                        leafN = isLeaf ? (((ref >> WIDE_LEAF_COUNT_SHIFT) & 0xf) + 1) : leafN;
                        mode = isLeaf ? (int)M_LEAF : (int)M_NODE;
                        cur = (have & !isLeaf) ? ref : -1;
                    }
                } else if (mode == M_NODE && cur >= 0) {
                    const float4 *w = &sc.wide[4 * (size_t)cur];
                    float4 q0, q1, q2, q3;
                    if (!LD128) {
                        ldg256(w, q0, q1);
                        ldg256(w + 2, q2, q3);
                    } else {
                        q0 = ldg4(w); q1 = ldg4(w + 1); q2 = ldg4(w + 2); q3 = ldg4(w + 3);
                    }
                    float t0, t1;
                    bool p0, p1;
                    if (warpSlow) slabTestPair(q0, q1, q2, rs, tMax, &p0, &p1, &t0, &t1);
                    else slabTestPairFast(q0, q1, q2, rs, tMax, &p0, &p1, &t0, &t1);
                    const uint32_t meta = floatBits(q3.z);
                    if (meta & WIDE_SINGLE) p1 = false;
                    const int axis = (int)(meta & 3u);
                    const bool isNeg = (axis == 0 ? rs.neg0 : (axis == 1 ? rs.neg1 : rs.neg2)) != 0;
                    const int ref0 = asInt(q3.x), ref1 = asInt(q3.y);
                    // straight-line tail: push the far child if both pass, continue with the near one (or with
                    // the only one that passed); with none, the pop is left to the next visit
                    const bool both = p0 & p1;
                    {
                        const int2 e = make_int2(isNeg ? ref0 : ref1, __float_as_int(isNeg ? t0 : t1));
                        if (both & (sp < SDEPTH)) sstack[sp * BLOCK + tid] = e;
                        if (both & (sp >= SDEPTH)) lstack[sp - SDEPTH] = e;
                        sp += both ? 1 : 0;
                    }
                    const int ref = (both ? isNeg : !p0) ? ref1 : ref0;
                    const bool have = p0 | p1;
                    const bool isLeaf = have & (ref < 0);
                    leafFirst = isLeaf ? (ref & (int)WIDE_LEAF_OFFSET_MASK) : leafFirst;
                    leafN = isLeaf ? (((ref >> WIDE_LEAF_COUNT_SHIFT) & 0xf) + 1) : leafN;
                    mode = isLeaf ? (int)M_LEAF : (int)M_NODE;
                    cur = (have & !isLeaf) ? ref : -1;
                }
            }
        } else if (step == M_LEAF) {
            int stagedN = 0;
            if (LEAFTMA) {
                // every lane of the warp takes part in the barrier protocol; lanes with a leaf issue one bulk copy each
                const unsigned bar = (unsigned)__cvta_generic_to_shared(&sbar[tid >> 5]);
                stagedN = (mode == M_LEAF) ? min(leafN, STAGED) : 0;
                unsigned bytes = (unsigned)stagedN * 48u;
                for (int o = 16; o > 0; o >>= 1) bytes += __shfl_xor_sync(FULL, bytes, o);
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the slots were read by ordinary loads in the last leaf step
                if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
                __syncwarp();
                if (stagedN > 0) {
                    const unsigned dst = (unsigned)__cvta_generic_to_shared(&sleaf[tid * STAGED * 3]);
                    const float4 *src = &sc.leafPrims[3 * (size_t)leafFirst];
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                                 "r"((unsigned)stagedN * 48u), "r"(bar)
                                 : "memory");
                }
                unsigned done = 0;
                while (!done)
                    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                 : "=r"(done)
                                 : "r"(bar), "r"(barPhase)
                                 : "memory");
                barPhase ^= 1u;
            }
            if (mode == M_LEAF) {
                if (INST && (flags & F_EXIT)) {
                    // back to world space (TransformedPrimitive::Intersect returns, primitive.cpp:82-86)
                    flags &= ~F_EXIT;
                    sp -= 2;
                    const int2 rest = stGet(sp), saved = stGet(sp + 1);
                    leafFirst = rest.x;
                    leafN = rest.y;
                    if (!(flags & F_HITIN)) tMax = __int_as_float(saved.x);
                    const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                    float4 ra = p[0], rb = p[1];
                    rs = setupRay(mk3(ra.y, ra.z, ra.w), mk3(rb.x, rb.y, rb.z));
                    inst = -1;
                    instBase = 0;
                }
                bool finished = false, entered = false;
                const bool any = (flags & F_ANY) != 0;
                int staged = 0;
                while (leafN > 0) {
                    const int idx = leafFirst;
                    ++leafFirst;
                    --leafN;
                    const float4 *rec = &sc.leafPrims[3 * (size_t)idx];
                    float4 a, b, c4;
                    if (LEAFTMA && staged < stagedN) {
                        const float4 *sl = &sleaf[(tid * STAGED + staged) * 3];
                        a = sl[0]; b = sl[1]; c4 = sl[2];
                        ++staged;
                    } else {
                        a = ldg4(rec); b = ldg4(rec + 1); c4 = ldg4(rec + 2);
                    }
                    uint32_t pf = floatBits(b.w);
                    if (INST && (pf & LEAF_INSTANCE)) {
                        const int id = asInt(c4.w);
                        const DInstance &in = sc.instances[id];
                        const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                        float4 ra = p[0], rb = p[1];
                        DRay ray;
                        ray.o = mk3(ra.y, ra.z, ra.w);
                        ray.d = mk3(rb.x, rb.y, rb.z);
                        ray.tMax = rb.w;
                        DRay r2 = xfRay(in.w2i, ray, tMax);
                        stPut(sp, make_int2(leafFirst, leafN));
                        stPut(sp + 1, make_int2(__float_as_int(tMax), 0));
                        sp += 2;
                        instBase = sp;
                        inst = id;
                        flags &= ~F_HITIN;
                        rs = setupRay(r2.o, r2.d);
                        tMax = r2.tMax;
                        if (in.wroot >= 0) {
                            cur = WIDTH == 4 ? in.wroot4 : in.wroot;
                            mode = M_NODE;
                            leafN = 0;
                            entered = true;
                            break;
                        }
                        leafFirst = in.lone;   // one-primitive object: its record is the whole "leaf"
                        leafN = 1;
                        continue;
                    }
                    if (SPHERES && (pf & LEAF_SPHERE)) {
                        const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                        float4 ra = p[0], rb = p[1];
                        DRay ray;
                        ray.o = mk3(ra.y, ra.z, ra.w);
                        ray.d = mk3(rb.x, rb.y, rb.z);
                        ray.tMax = rb.w;
                        if (INST && inst >= 0) ray = xfRay(sc.instances[inst].w2i, ray, tMax);
                        float t, phi;
                        if (sphereLeafTest(sc, asInt(c4.w), ray, tMax, &t, &phi)) {
                            flags |= F_FOUND;
                            if (any) { finished = true; break; }
                            tMax = t;
                            if (INST) {
                                hitInst = inst;
                                if (inst >= 0) flags |= F_HITIN;
                            }
                            __stcs(reinterpret_cast<float4 *>(&pool.ctx[c].hit), make_float4(__int_as_float(idx), phi, 0.f, 0.f));
                        }
                        continue;
                    }
                    float t, b0, b1, b2;
                    if (triangleTest(mk3(a.x, a.y, a.z), mk3(b.x, b.y, b.z), mk3(c4.x, c4.y, c4.z), rs, tMax, &t, &b0, &b1, &b2)) {
                        // alpha-masked meshes (TRACE_ALPHA instantiations only): a hit on a texel of value 0 is no hit
                        if (ALPHA && (pf & LEAF_ALPHA) && alphaRejects(sc, asInt(a.w), b0, b1, b2, any)) continue;
                        if (any) { flags |= F_FOUND; finished = true; break; }
                        if (pf & LEAF_DEGENERATE) continue;
                        flags |= F_FOUND;
                        tMax = t;
                        if (INST) {
                            hitInst = inst;
                            if (inst >= 0) flags |= F_HITIN;
                        }
                        __stcs(reinterpret_cast<float4 *>(&pool.ctx[c].hit), make_float4(__int_as_float(idx), b0, b1, b2));
                    }
                }
                if (!entered) {
                    leafN = 0;
                    if (finished) mode = M_FETCH;
                    else if (sp == instBase) {
                        if (INST && inst >= 0) flags |= F_EXIT;   // stays a leaf lane: the next leaf step leaves the instance
                        else mode = M_FETCH;
                    } else {
                        mode = M_NODE;   // the next node visit pops
                        cur = -1;
                    }
                }
            }
        } else {  // M_FETCH: flush finished rays, then take new ones
            bool flush = mode == M_FETCH && c >= 0;
            int state = LS_IDLE;
            if (flush) {
                WfCtx &cx = pool.ctx[c];
                state = (flags & F_ANY) ? LS_SHADOW : __ldcs(&cx.ln.state);
                const int foundCode = (flags & F_FOUND) ? ((INST && !(flags & F_ANY) && hitInst >= 0) ? 2 + hitInst : 1) : 0;
                __stcs(reinterpret_cast<float2 *>(&cx.tHit), make_float2(tMax, __int_as_float(foundCode)));
            }
            wfPush(pool.queue[WQ_SHADE], &pool.counts[WQ_SHADE], c, flush && state == LS_PATH);
            bool again = false;   // CHAIN: the context goes on with its next ray in this lane
            if (CHAIN) {
                // a shadow or MIS ray ended: the light step right here, and the vertex's next ray (MIS ray, or the path's
                // continuation) in this lane, in this launch - one round per bounce instead of up to three
                int next = LS_PATH;
                if (flush && state != LS_PATH) {
                    next = wfChainLight<SHADE_GENERAL | (SPHERES ? SHADE_SPHERES : 0)>(chain, &pool.ctx[c], (flags & F_FOUND) != 0);
                    again = next != LS_IDLE;
                }
                const unsigned mShadow = __ballot_sync(FULL, again && next == LS_SHADOW), mRegular = __ballot_sync(FULL, again && next != LS_SHADOW);
                if (lane == 0) {
                    if (mShadow) atomicAdd(&sCount[1], (unsigned)__popc(mShadow));
                    if (mRegular) atomicAdd(&sCount[0], (unsigned)__popc(mRegular));
                }
                wfPush(pool.queue[chain.freeQ], &pool.counts[chain.freeQ], c, flush && state != LS_PATH && !again);
            } else
                wfPush(pool.queue[WQ_LIGHT], &pool.counts[WQ_LIGHT], c, flush && state != LS_PATH);
            if (again) {
                const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                const float4 ra = p[0], rb = p[1];
                flags = (__float_as_int(ra.x) == LS_SHADOW) ? F_ANY : 0;
                rs = setupRay(mk3(ra.y, ra.z, ra.w), mk3(rb.x, rb.y, rb.z));
                tMax = rb.w;
                cur = 0;
                if (INST) {
                    inst = hitInst = -1;
                    instBase = 0;
                }
                sp = 0;
                leafN = 0;
                mode = M_NODE;
            } else if (flush)
                c = -1;
            bool want = mode == M_FETCH && !(flags & F_EXHAUSTED);
            unsigned wantMask = __ballot_sync(FULL, want);
            if (wantMask) {
                int leader = __ffs(wantMask) - 1;
                unsigned base = 0;
                if (lane == leader) base = atomicAdd(&pool.counts[WQ_CURSOR], (unsigned)__popc(wantMask));
                base = __shfl_sync(FULL, base, leader);
                if (want) {
                    unsigned i = base + __popc(wantMask & ((1u << lane) - 1u));
                    if (i >= n)
                        flags |= F_EXHAUSTED;
                    else {
                        c = pool.queue[traceQ][i];
                        const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                        float4 ra = __ldcs(p), rb = __ldcs(p + 1);
                        flags = (__float_as_int(ra.x) == LS_SHADOW) ? F_ANY : 0;
                        rs = setupRay(mk3(ra.y, ra.z, ra.w), mk3(rb.x, rb.y, rb.z));
                        tMax = rb.w;
                        cur = 0;   // WIDTH 2: the pseudo node above the root; WIDTH 4: the root's record
                        if (INST) {
                            inst = hitInst = -1;
                            instBase = 0;
                        }
                        sp = 0;
                        leafN = 0;
                        mode = M_NODE;
                    }
                }
            }
        }
    }
    if (CHAIN) {
        __syncthreads();
        if (threadIdx.x == 0) {
            if (sCount[0]) atomicAdd(&pool.ctr[CTR_REGULAR], (unsigned long long)sCount[0]);
            if (sCount[1]) atomicAdd(&pool.ctr[CTR_SHADOW], (unsigned long long)sCount[1]);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Trace kernel with a per-warp POOL of rays (triangle scenes, two-child records; PB2_FLAG_POOL).  k_wf_trace_w binds a ray
// to a lane for its whole life, so a step runs with the lanes that happen to be in that phase: ~21 of 32 in node steps, ~6 in
// leaf steps.  Here a warp owns PL_RAYS = 48 rays whose state lives in shared memory (structure of arrays, one column per ray: ray
// constants, tMax, current record, stack pointer, leaf range, flags; the stack of pending far children next to it), and every
// step the warp picks up to 32 rays THAT ARE IN THE PHASE BEING RUN, loads their state, runs the step in registers and stores
// what changed.  Per ray the traversal is the one of k_wf_trace_w, operation for operation (same records, same order, same
// pops against the tMax of the moment): only which lane executes a step of which ray differs.
// Slot flags: bit 0 any-hit, 1 found, 2-4 direction signs, 5-6 / 7-8 / 9-10 kx ky kz, 11 slow (non-finite), 12-13 phase.
// ---------------------------------------------------------------------------------------------
enum { PL_EMPTY = 0, PL_NODE = 1, PL_LEAF = 2, PL_DONE = 3, PL_R = 64, PL_SPILL = 64 };   // PL_R: the most slots a warp can have
// PL_SD stack entries per ray in shared memory: with PL_RAYS rays per warp, 25 KB per block, 8 resident blocks per SM
enum { PL_RAYS = 48, PL_SD = 8 };
struct PoolWarp {   // one warp's slice of shared memory
    float f[10][PL_RAYS];        // ox oy oz ix iy iz tMax Sx Sy Sz
    int i[6][PL_RAYS];           // cur, sp, ctx, flags, leafFirst, leafN
    int2 stk[PL_SD][PL_RAYS];    // (child reference, tMin bits); deeper entries go to WfPool::spill
    int list[PL_RAYS];           // slots chosen for the step, in rank order
};

__global__ void __launch_bounds__(128, 8) k_wf_trace_pool(DScene sc, WfPool pool, int traceQ, WfChain) {
    static_assert(PL_RAYS > 32 && PL_RAYS <= PL_R, "a warp owns 33 .. 64 slots");
    // node visits per node step; rays that must hold a leaf before a leaf step, be done or empty before a flush-and-fill step
    static constexpr int NSUB = 4, LEAF_T = 16, FILL_T = 12;
    extern __shared__ unsigned char poolSmemRaw[];
    PoolWarp &pw = reinterpret_cast<PoolWarp *>(poolSmemRaw)[threadIdx.x >> 5];
    const bool second = (threadIdx.x & 31) + 32 < PL_RAYS;   // this lane also looks after slot lane + 32
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned ltMask = (1u << lane) - 1u;
    const unsigned n = pool.counts[traceQ];
    int2 *spill = pool.spill + ((size_t)(blockIdx.x * 4 + (threadIdx.x >> 5)) * PL_R) * PL_SPILL;   // [slot][PL_SPILL]
    pw.i[3][lane] = 0;
    if (second) pw.i[3][lane + 32] = 0;
    __syncwarp();
    bool exhausted = false;
    // stack access of slot s
    auto stGet = [&](int s, int d) -> int2 { return d < PL_SD ? pw.stk[d][s] : spill[(size_t)s * PL_SPILL + (d - PL_SD)]; };
    auto stPut = [&](int s, int d, int2 e) {
        if (d < PL_SD) pw.stk[d][s] = e;
        else spill[(size_t)s * PL_SPILL + (d - PL_SD)] = e;
    };
    while (true) {
        // ---- census of the slots
        const int fl0 = pw.i[3][lane], fl1 = second ? pw.i[3][lane + 32] : -1;
        const int m0 = (fl0 >> 12) & 3, m1 = second ? ((fl1 >> 12) & 3) : -1;   // -1: no such slot
        const unsigned bN0 = __ballot_sync(FULL, m0 == PL_NODE), bN1 = __ballot_sync(FULL, m1 == PL_NODE);
        const unsigned bL0 = __ballot_sync(FULL, m0 == PL_LEAF), bL1 = __ballot_sync(FULL, m1 == PL_LEAF);
        const unsigned bD0 = __ballot_sync(FULL, m0 == PL_DONE), bD1 = __ballot_sync(FULL, m1 == PL_DONE);
        const int nN = __popc(bN0) + __popc(bN1), nL = __popc(bL0) + __popc(bL1), nD = __popc(bD0) + __popc(bD1);
        const int nE = PL_RAYS - nN - nL - nD;
        int phase;
        if (nD + (exhausted ? 0 : nE) >= FILL_T || (nN == 0 && nL == 0 && (nD > 0 || (!exhausted && nE > 0)))) phase = PL_DONE;   // flush + fill
        else if (nL >= LEAF_T || (nL > 0 && nN == 0)) phase = PL_LEAF;
        else if (nN > 0) phase = PL_NODE;
        else break;   // nothing in flight, nothing to flush, the list is exhausted

        if (phase == PL_DONE) {
#pragma unroll 1
            for (int h = 0; h < 2; ++h) {
                const bool exists = h == 0 || second;
                const int s = exists ? lane + 32 * h : lane;
                const int fl = exists ? pw.i[3][s] : (PL_NODE << 12);   // a lane without a second slot just takes part in the votes
                const int mode = (fl >> 12) & 3;
                const bool flush = mode == PL_DONE;
                int c = flush ? pw.i[2][s] : -1;
                int state = LS_IDLE;
                if (flush) {
                    WfCtx &cx = pool.ctx[c];
                    state = (fl & 1) ? LS_SHADOW : __ldcs(&cx.ln.state);
                    __stcs(reinterpret_cast<float2 *>(&cx.tHit), make_float2(pw.f[6][s], __int_as_float((fl & 2) ? 1 : 0)));
                }
                wfPush(pool.queue[WQ_SHADE], &pool.counts[WQ_SHADE], c, flush && state == LS_PATH);
                wfPush(pool.queue[WQ_LIGHT], &pool.counts[WQ_LIGHT], c, flush && state != LS_PATH);
                bool want = (flush || mode == PL_EMPTY) && !exhausted;
                const unsigned wantMask = __ballot_sync(FULL, want);
                int newFlags = 0;   // PL_EMPTY
                if (wantMask) {
                    const int leader = __ffs(wantMask) - 1;
                    unsigned base = 0;
                    if (lane == leader) base = atomicAdd(&pool.counts[WQ_CURSOR], (unsigned)__popc(wantMask));
                    base = __shfl_sync(FULL, base, leader);
                    const unsigned idx = base + __popc(wantMask & ltMask);
                    if (want && idx < n) {
                        c = pool.queue[traceQ][idx];
                        const float4 *p = reinterpret_cast<const float4 *>(&pool.ctx[c]);
                        const float4 ra = __ldcs(p), rb = __ldcs(p + 1);
                        const DRaySetup rs = setupRay(mk3(ra.y, ra.z, ra.w), mk3(rb.x, rb.y, rb.z));
                        pw.f[0][s] = rs.o.x; pw.f[1][s] = rs.o.y; pw.f[2][s] = rs.o.z;
                        pw.f[3][s] = rs.invDir.x; pw.f[4][s] = rs.invDir.y; pw.f[5][s] = rs.invDir.z;
                        pw.f[6][s] = rb.w;
                        pw.f[7][s] = rs.Sx; pw.f[8][s] = rs.Sy; pw.f[9][s] = rs.Sz;
                        pw.i[0][s] = 0;   // the pseudo node above the root
                        pw.i[1][s] = 0;
                        pw.i[2][s] = c;
                        newFlags = ((__float_as_int(ra.x) == LS_SHADOW) ? 1 : 0) | (rs.neg0 << 2) | (rs.neg1 << 3) | (rs.neg2 << 4) | (rs.kx << 5) |
                                   (rs.ky << 7) | (rs.kz << 9) | (rs.slow << 11) | (PL_NODE << 12);
                    }
                    if (__any_sync(FULL, want && idx >= n)) exhausted = true;
                }
                if (flush || want) pw.i[3][s] = newFlags;
            }
            __syncwarp();
            continue;
        }

        // ---- hand the slots of the chosen phase to the lanes: slot `lane` first, then slot `lane + 32`, in rank order
        const unsigned b0 = phase == PL_NODE ? bN0 : bL0, b1 = phase == PL_NODE ? bN1 : bL1;
        const int c0 = __popc(b0);
        if (b0 & (1u << lane)) pw.list[__popc(b0 & ltMask)] = lane;
        if (b1 & (1u << lane)) pw.list[c0 + __popc(b1 & ltMask)] = lane + 32;
        __syncwarp();
        const int nSel = min(c0 + __popc(b1), 32);
        const bool active = lane < nSel;
        const int s = active ? pw.list[lane] : 0;
        __syncwarp();

        if (phase == PL_NODE) {
            DRaySetup rs;
            rs.o = mk3(pw.f[0][s], pw.f[1][s], pw.f[2][s]);
            rs.invDir = mk3(pw.f[3][s], pw.f[4][s], pw.f[5][s]);
            float tMax = pw.f[6][s];
            int cur = pw.i[0][s], sp = pw.i[1][s];
            int fl = pw.i[3][s];
            rs.neg0 = (fl >> 2) & 1; rs.neg1 = (fl >> 3) & 1; rs.neg2 = (fl >> 4) & 1;
            rs.kx = rs.ky = rs.kz = 0;
            rs.Sx = rs.Sy = rs.Sz = 0;
            rs.slow = (fl >> 11) & 1;
            int mode = active ? (int)PL_NODE : (int)PL_EMPTY;   // lanes without a slot idle through the step
            int leafFirst = 0, leafN = 0;
            const bool warpSlow = __any_sync(FULL, active && rs.slow != 0);
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub) {
                {
                    // take the next pending far child when the last visit left nothing to descend into (cur < 0)
                    const bool need = (mode == PL_NODE) & (cur < 0);
                    const bool empty = need & (sp == 0);
                    const bool pop = need & !empty;
                    int2 e = make_int2(0, 0);
                    if (pop) e = stGet(s, sp - 1);
                    sp = pop ? sp - 1 : sp;
                    const bool take = pop & (__int_as_float(e.y) < tMax);
                    const bool leafRef = take & (e.x < 0);
                    leafFirst = leafRef ? (e.x & (int)WIDE_LEAF_OFFSET_MASK) : leafFirst;
                    leafN = leafRef ? (((e.x >> WIDE_LEAF_COUNT_SHIFT) & 0xf) + 1) : leafN;
                    cur = (take & !leafRef) ? e.x : cur;
                    mode = leafRef ? (int)PL_LEAF : mode;
                    if (empty) mode = PL_DONE;
                }
                if (mode == PL_NODE && cur >= 0) {
                    const float4 *w = &sc.wide[4 * (size_t)cur];
                    float4 q0, q1, q2, q3;
                    ldg256(w, q0, q1);
                    ldg256(w + 2, q2, q3);
                    float t0, t1;
                    bool p0, p1;
                    if (warpSlow) slabTestPair(q0, q1, q2, rs, tMax, &p0, &p1, &t0, &t1);
                    else slabTestPairFast(q0, q1, q2, rs, tMax, &p0, &p1, &t0, &t1);
                    const uint32_t meta = floatBits(q3.z);
                    if (meta & WIDE_SINGLE) p1 = false;
                    const int axis = (int)(meta & 3u);
                    const bool isNeg = (axis == 0 ? rs.neg0 : (axis == 1 ? rs.neg1 : rs.neg2)) != 0;
                    const int ref0 = asInt(q3.x), ref1 = asInt(q3.y);
                    const bool both = p0 & p1;
                    if (both) stPut(s, sp, make_int2(isNeg ? ref0 : ref1, __float_as_int(isNeg ? t0 : t1)));
                    sp += both ? 1 : 0;
                    const int ref = (both ? isNeg : !p0) ? ref1 : ref0;
                    const bool have = p0 | p1;
                    const bool isLeaf = have & (ref < 0);
                    leafFirst = isLeaf ? (ref & (int)WIDE_LEAF_OFFSET_MASK) : leafFirst;
                    leafN = isLeaf ? (((ref >> WIDE_LEAF_COUNT_SHIFT) & 0xf) + 1) : leafN;
                    mode = isLeaf ? (int)PL_LEAF : (int)PL_NODE;
                    cur = (have & !isLeaf) ? ref : -1;
                }
            }
            if (active) {
                pw.i[0][s] = cur;
                pw.i[1][s] = sp;
                pw.i[3][s] = (fl & 0xfff) | (mode << 12);
                pw.i[4][s] = leafFirst;
                pw.i[5][s] = leafN;
            }
        } else {   // PL_LEAF: every primitive of the leaf, in order (GeometricPrimitive::Intersect[P] + Triangle)
            if (active) {
                DRaySetup rs;
                rs.o = mk3(pw.f[0][s], pw.f[1][s], pw.f[2][s]);
                rs.invDir = mk3(0, 0, 0);
                float tMax = pw.f[6][s];
                rs.Sx = pw.f[7][s]; rs.Sy = pw.f[8][s]; rs.Sz = pw.f[9][s];
                int fl = pw.i[3][s];
                rs.neg0 = rs.neg1 = rs.neg2 = 0;
                rs.kx = (fl >> 5) & 3; rs.ky = (fl >> 7) & 3; rs.kz = (fl >> 9) & 3;
                rs.slow = 0;
                const int c = pw.i[2][s];
                int leafFirst = pw.i[4][s], leafN = pw.i[5][s];
                const bool any = (fl & 1) != 0;
                bool finished = false;
                while (leafN > 0) {
                    const int idx = leafFirst;
                    ++leafFirst;
                    --leafN;
                    const float4 *rec = &sc.leafPrims[3 * (size_t)idx];
                    const float4 a = ldg4(rec), b = ldg4(rec + 1), c4 = ldg4(rec + 2);
                    const uint32_t pf = floatBits(b.w);
                    float t, b0, b1, b2;
                    if (triangleTest(mk3(a.x, a.y, a.z), mk3(b.x, b.y, b.z), mk3(c4.x, c4.y, c4.z), rs, tMax, &t, &b0, &b1, &b2)) {
                        if (any) { fl |= 2; finished = true; break; }
                        if (pf & LEAF_DEGENERATE) continue;
                        fl |= 2;
                        tMax = t;
                        __stcs(reinterpret_cast<float4 *>(&pool.ctx[c].hit), make_float4(__int_as_float(idx), b0, b1, b2));
                    }
                }
                const int sp = pw.i[1][s];
                const int mode = (finished || sp == 0) ? (int)PL_DONE : (int)PL_NODE;
                pw.f[6][s] = tMax;
                pw.i[0][s] = -1;   // the next node step pops
                pw.i[3][s] = (fl & 0xfff) | (mode << 12);
            }
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// laneAdvance for every context of one list.  SHADE = true: the shade list (path rays: the whole
// vertex is evaluated); SHADE = false: the light list (shadow / MIS rays: a few adds and the next
// ray).  Two instantiations so that the light kernel is small and the warps of each stay converged.
// F: the shade features (SHADE_* in device/pb2_shade.cuh) the step is compiled for.  With SHADE_TEXTURES the camera ray's
// differentials are rebuilt from the context's pFilm.
// ---------------------------------------------------------------------------------------------
template <bool SHADE, int MINB, int F>
__global__ void __launch_bounds__(128, MINB) k_wf_advance(const DScene *__restrict__ scp, const DRenderParams *__restrict__ rpp, WfPool pool,
                                                          int srcQ, int traceQ, int freeQ, float4 *film, unsigned long long *counters) {
    __shared__ WfSlot stage[128];
    // the shade step's sampler batch (shadeVertex): one row per thread, padded to 9 words so that a warp's 32 rows fall
    // in 32 different banks
    __shared__ float sampleRows[SHADE ? 128 * (kSampleBatch + 1) : 1];
    WfSlot &slot = stage[threadIdx.x];
    WfSlot *warpSlots = stage + (threadIdx.x & ~31u);
    float *u = sampleRows + (SHADE ? threadIdx.x * (kSampleBatch + 1) : 0);
    const DScene &sc = *scp;
    const DRenderParams &rp = *rpp;
    const int *srcList = wfQueue(pool, srcQ);
    int *traceList = wfQueue(pool, traceQ), *freeList = wfQueue(pool, freeQ);
    unsigned n = pool.counts[srcQ];
    unsigned stride = gridDim.x * blockDim.x;
    unsigned regular = 0, shadow = 0;
    for (unsigned base = blockIdx.x * blockDim.x; base < n; base += stride) {
        unsigned i = base + threadIdx.x;
        bool have = i < n;
        int c = have ? srcList[i] : 0;
        bool ended = false, deferred = false;
        wfStageIn<SHADE ? WF_IN_SHADE : WF_IN_ALL>(pool.ctx, warpSlots, have ? c : -1);
        if (have) {
            DLane &ln = slot.ln;
            const int foundCode = slot.found;
            DHit hit;
            hit.leaf = __float_as_int(slot.hit[0]);
            hit.b0 = slot.hit[1];
            hit.b1 = slot.hit[2];
            hit.b2 = slot.hit[3];
            hit.inst = foundCode >= 2 ? foundCode - 2 : -1;
            bool found = foundCode != 0;
            float tHit = slot.tHit;
            if (SHADE && (F & SHADE_TEXTURES)) {
                DTexCtx tc;
                tc.cam = &rp.cam;
                tc.pFilm = slot.pFilm;
                tc.diffScale = rp.diffScale;
                shadeVertex<F>(sc, rp.halton, rp.path, ln, found, hit, tHit, u, &tc);
            } else if (SHADE) shadeVertex<F>(sc, rp.halton, rp.path, ln, found, hit, tHit, u);
            else lightAdvance<F>(sc, ln, found, hit, tHit);
            if (SHADE && (F & SHADE_LAZY) && ln.state == LS_DEFER) {
                ln.state = LS_PATH;   // untouched: shaded again from the retry list once its voxel's record exists
                deferred = true;
            } else {
                ended = ln.state == LS_IDLE;
                if (ended) addSample(rp, film, slot.pFilm, guardRadiance(ln.L));
                else if (ln.state == LS_SHADOW) shadow++;   // Scene::IntersectP call (scene.cpp:51-55)
                else regular++;                             // Scene::Intersect call (scene.cpp:45-49)
            }
        }
        // (an ended path's lane is not written back: its context goes to the free list, and k_wf_gen starts a new lane in it)
        wfStageOut<SHADE ? WF_OUT_SHADE : WF_OUT_LIGHT>(pool.ctx, warpSlots, have && !ended ? c : -1);
        if (SHADE && (F & SHADE_LAZY)) wfPush(pool.queue[WQ_RETRY], &pool.counts[WQ_RETRY], c, deferred);
        wfPush(traceList, &pool.counts[traceQ], c, have && !ended && !deferred);
        wfPush(freeList, &pool.counts[freeQ], c, have && ended);
    }
    wfCountRays(counters, regular, shadow);
}

// ---------------------------------------------------------------------------------------------
// End of a frame.  Once the work counter has run out the pool is no longer refilled and the number of paths in
// flight decays round by round: many more rounds, each a handful of launches over a few thousand rays that cannot
// fill the machine - a fixed cost per frame whatever the GPU count, so a growing share of the frame on several GPUs.
// k_wf_finish runs after the shade step of every round and does nothing until (a) no work item is left and (b) at
// most `threshold` contexts are still in flight; then every thread takes ONE of them and walks it to the end of its
// path with the per-lane state machine (traceLane + laneAdvance, the code of k_li_samples / pb2_li_samples), deposits
// the sample, and the frame is over.  Same functions, same order of operations per path as the wavefront kernels.
// k_wf_reset (below) empties the list when k_wf_finish has walked it.
// No block waits for another: the decision is one atomicCAS on WQ_FINISH.  With several pipelines the trace grid can leave
// room for one list-kernel block per SM, so a launch of any wavefront kernel may be only partly resident beside another
// pipeline's kernels: none of them (the trace kernels pull rays from an atomic cursor, the list kernels are grid-stride
// loops) may spin on another block of its own grid.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool wfFinishNow(const DRenderParams &rp, const WfPool &pool, int traceQ, unsigned threshold) {
    const unsigned n = pool.counts[traceQ];
    return n > 0 && n <= threshold && (long long)pool.ctr[CTR_WORK] >= rp.nWorkItems;
}

template <int F>
__global__ void __launch_bounds__(128) k_wf_finish(const DScene *__restrict__ scp, const DRenderParams *__restrict__ rpp, WfPool pool, int traceQ,
                                                   unsigned threshold, float4 *film) {
    const DScene &sc = *scp;
    const DRenderParams &rp = *rpp;
    // One decision for the whole launch and for this round's k_wf_reset.  The work counter is shared by the pipelines: it
    // can run out while the blocks of this launch look at it, so each block deciding for itself could walk some of the
    // listed paths and not others, and k_wf_reset could then empty a list whose paths were never walked.  The first block
    // to look decides; the others and k_wf_reset follow it.
    __shared__ bool sGo;
    if (threadIdx.x == 0) {
        const unsigned mine = wfFinishNow(rp, pool, traceQ, threshold) ? WF_FINISH_GO : WF_FINISH_WAIT;
        const unsigned first = atomicCAS(&pool.counts[WQ_FINISH], 0u, mine);
        sGo = (first ? first : mine) == WF_FINISH_GO;
    }
    __syncthreads();
    if (!sGo) return;
    const unsigned n = pool.counts[traceQ];
    const int *traceList = wfQueue(pool, traceQ);
    unsigned regular = 0, shadow = 0;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        WfCtx &cx = pool.ctx[traceList[i]];
        DLane &ln = cx.ln;
        while (ln.state != LS_IDLE) {
            DHit hit;
            float tMax;
            const bool found = traceLane(sc, ln, &tMax, &hit, nullptr);
            laneAdvance<F>(sc, rp.halton, rp.path, ln, found, hit, tMax);
            if (ln.state == LS_DEFER) break;            // (never: this kernel is not launched for lazily lit scenes)
            if (ln.state == LS_SHADOW) shadow++;        // the next ray is a Scene::IntersectP call
            else if (ln.state != LS_IDLE) regular++;    // ... a Scene::Intersect call
        }
        addSample(rp, film, cx.pFilm, guardRadiance(ln.L));
    }
    wfCountRays(pool.ctr, regular, shadow);
}

// ---------------------------------------------------------------------------------------------
// Lazy SpatialLightDistribution: the records of the voxels requested since the last build (lightDistLookup), one block
// per voxel.  Thread t owns lights t, t + 128, ...: a light's contribution is a sum over the 128 sample points in their
// order, so any assignment of lights to threads gives the eager builder's (and the reference's) bits; thread 0 then runs
// the sequential floor + cdf and publishes the record's index in the voxel's slot.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_lightdist_build(DScene sc, DHalton h) {
    const DLightDist &ld = sc.lightDist;
    const int nReq = ld.counters[0];
    __shared__ int sRecord;
    for (int r = blockIdx.x; r < nReq; r += gridDim.x) {
        const int voxel = ld.requests[r];
        if (threadIdx.x == 0) {
            int k = atomicAdd(&ld.counters[1], 1);
            if (k >= ld.poolRecords) {
                ld.counters[2] = 1;   // pool exhausted: the host fails the render loudly
                k = -1;
            }
            sRecord = k;
        }
        __syncthreads();
        const int k = sRecord;
        if (k >= 0) {
            float *rec = const_cast<float *>(ld.table) + (size_t)k * ld.stride;
            const int pz = voxel % ld.nVoxels[2], py = (voxel / ld.nVoxels[2]) % ld.nVoxels[1], px = voxel / (ld.nVoxels[2] * ld.nVoxels[1]);
            const DVoxelBounds vb = voxelBounds(ld, px, py, pz);
            for (int j = threadIdx.x; j < sc.nLights; j += blockDim.x) rec[j] = voxelLightContribution(sc, h, vb, j);
            __syncthreads();
            if (threadIdx.x == 0) {
                finishVoxelDistribution(sc.nLights, rec);
                __threadfence();
                ld.slots[voxel] = k;
            }
        }
        __syncthreads();
    }
}
__global__ void k_lightdist_done(DScene sc) {
    if (threadIdx.x == 0 && blockIdx.x == 0) sc.lightDist.counters[0] = 0;
}

__global__ void k_wf_init(WfPool pool) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (unsigned)pool.capacity) pool.queue[WQ_FREE0][i] = (int)i;
    if (i < WQ_COUNT) pool.counts[i] = (i == WQ_FREE0) ? (unsigned)pool.capacity : 0u;
}

// end of a round: the lists consumed in it are emptied (and the next trace list, if k_wf_finish has just run it dry)
__global__ void k_wf_reset(WfPool pool, int a, int b, int traceNext, unsigned threshold) {
    if (threadIdx.x == 0) {
        if (threshold && pool.counts[WQ_FINISH] == WF_FINISH_GO) pool.counts[traceNext] = 0;
        pool.counts[WQ_RETRY] = 0;   // (and WQ_FINISH)
        pool.counts[WQ_CURSOR] = 0;
        pool.counts[WQ_SHADE] = 0;
        pool.counts[WQ_LIGHT] = 0;
        pool.counts[a] = 0;
        pool.counts[b] = 0;
    }
}

#endif
