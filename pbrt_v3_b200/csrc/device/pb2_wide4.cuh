// Four-child node records: the layout the four-child trace kernel (k_wf_trace_w<4, T>, pb2_wavefront.cuh) walks.
//
// One 128-B record per interior node of every second level of the reference's binary tree (src/accelerators/bvh.cpp:
// 95-104, 640-658): the boxes of the node's grandchildren in the canonical slot order [LL, LR, RL, RR]; a child that is a
// leaf keeps its own box in the first slot of its pair and leaves the second empty.  Boxes are stored component-wise for
// two slots at a time, so that the packed FP32x2 slab test (slabTestPair4) takes its operands as the register pairs the
// 16-byte loads deliver:
//   q0 = (min.x[0], min.x[1], min.y[0], min.y[1])   q3 = the same for slots 2, 3
//   q1 = (min.z[0], min.z[1], max.x[0], max.x[1])   q4
//   q2 = (max.y[0], max.y[1], max.z[0], max.z[1])   q5
//   q6 = the four child references (int bits): index of the child's record, a WIDE_LEAF reference as in the two-child
//        records (pb2_scene.cuh), or WIDE4_EMPTY
//   q7.x = meta (int bits): split axis of the node (bits 0-1), of its first child (2-3), of its second child (4-5)
// Records are numbered in depth-first order of the collapsed tree (a record, then the subtrees of its slots in slot
// order), so a subtree is one contiguous range of memory, like the reference's depth-first LinearBVHNode array.
//
// Visiting order = the reference's (bvh.cpp:682-690): at each of the two collapsed levels the child on the ray's near side
// of the split axis first.  A child box is tested with the tMax of the visit; the caller re-checks a deferred child's
// entry distance against the tMax of the moment it is taken up.  Since a child's slab interval lies inside its parent's
// (the parent's planes are the min / max of its children's, and the slab arithmetic is monotonic in the plane) and tMax
// only shrinks, every leaf is reached iff the binary traversal reaches it, in the same order, and the root's own box need
// not be tested at all: a ray that misses it misses all four grandchildren.
// tests/test_host.py::test_wide4_records_keep_the_reference_order replays both traversals on the host with the functions
// below; tests/test_gpu_parity.py compares the kernel's hit records bit for bit.
#ifndef PB2_WIDE4_CUH
#define PB2_WIDE4_CUH

#include <cstring>
#include <vector>

#include "pb2_scene.cuh"

namespace pb2 {

enum : uint32_t { WIDE4_EMPTY = 0x7fffffffu };

// Host: collapse the binary trees rooted at roots[] (indices into nodes[], whose child / primitive offsets are global)
// into four-child records.  rootRecord[k] receives the record of roots[k]; a tree that is a single leaf gets one record
// whose first slot is that leaf.
inline std::vector<float4> buildWide4Records(const pb2_bvh_node *nodes, const int64_t *roots, size_t nRoots, int32_t *rootRecord) {
    std::vector<float4> out;
    struct Item { int64_t node; int32_t parent, slot; };
    std::vector<Item> todo;
    auto leafRef = [&](const pb2_bvh_node &n) { return WIDE_LEAF | ((uint32_t)(n.n_prims - 1) << WIDE_LEAF_COUNT_SHIFT) | (uint32_t)n.offset; };
    for (size_t k = 0; k < nRoots; ++k) {
        todo.push_back(Item{roots[k], -1, 0});
        bool first = true;
        while (!todo.empty()) {
            const Item it = todo.back();
            todo.pop_back();
            const int64_t i = it.node;
            const int32_t me = (int32_t)(out.size() / 8);
            if (first) rootRecord[k] = me;
            first = false;
            if (it.parent >= 0) {
                uint32_t ref = (uint32_t)me;
                std::memcpy(reinterpret_cast<char *>(&out[8 * (size_t)it.parent + 6]) + 4 * it.slot, &ref, 4);
            }
            float mn[4][3], mx[4][3];
            uint32_t refs[4] = {WIDE4_EMPTY, WIDE4_EMPTY, WIDE4_EMPTY, WIDE4_EMPTY};
            int64_t interior[4] = {-1, -1, -1, -1};
            for (int s = 0; s < 4; ++s)
                for (int c = 0; c < 3; ++c) {
                    mn[s][c] = PB2_INFINITY;
                    mx[s][c] = -PB2_INFINITY;
                }
            uint32_t meta = 0;
            auto put = [&](int slot, int64_t node) {
                const pb2_bvh_node &n = nodes[node];
                for (int c = 0; c < 3; ++c) {
                    mn[slot][c] = n.bmin[c];
                    mx[slot][c] = n.bmax[c];
                }
                if (n.n_prims > 0) refs[slot] = leafRef(n);
                else interior[slot] = node;   // its record number is patched in when the record is created
            };
            if (nodes[i].n_prims > 0)
                put(0, i);   // the whole tree is one leaf
            else {
                meta = nodes[i].axis & 3u;
                const int64_t child[2] = {i + 1, (int64_t)nodes[i].offset};
                for (int g = 0; g < 2; ++g) {
                    const pb2_bvh_node &c = nodes[child[g]];
                    if (c.n_prims > 0)
                        put(2 * g, child[g]);
                    else {
                        meta |= ((uint32_t)c.axis & 3u) << (2 + 2 * g);
                        put(2 * g, child[g] + 1);
                        put(2 * g + 1, (int64_t)c.offset);
                    }
                }
            }
            float f[32];
            std::memset(f, 0, sizeof(f));
            for (int h = 0; h < 2; ++h) {   // slots 2h, 2h + 1
                float *q = f + 12 * h;
                for (int j = 0; j < 2; ++j) {
                    const int s = 2 * h + j;
                    q[0 + j] = mn[s][0]; q[2 + j] = mn[s][1]; q[4 + j] = mn[s][2];
                    q[6 + j] = mx[s][0]; q[8 + j] = mx[s][1]; q[10 + j] = mx[s][2];
                }
            }
            std::memcpy(f + 24, refs, sizeof(refs));
            std::memcpy(f + 28, &meta, sizeof(meta));
            const size_t base = out.size();
            out.resize(base + 8);
            std::memcpy(&out[base], f, sizeof(f));
            for (int s = 3; s >= 0; --s)   // depth-first: slot 0's subtree follows the record directly
                if (interior[s] >= 0) todo.push_back(Item{interior[s], me, s});
        }
    }
    return out;
}

// Bounds3::IntersectP (geometry.h:1412-1438) for two slots of a four-child record at once; the arithmetic of slabTestPair
// (pb2_scene.cuh) with the operands already paired by the record layout.
PB2_HD void slabTestPair4(float4 a, float4 b, float4 c, const DRaySetup &r, float rayTMax, bool *pass0, bool *pass1, float *tMin0,
                          float *tMin1) {
#if defined(__CUDA_ARCH__)
    const float2 minX = make_float2(a.x, a.y), minY = make_float2(a.z, a.w), minZ = make_float2(b.x, b.y);
    const float2 maxX = make_float2(b.z, b.w), maxY = make_float2(c.x, c.y), maxZ = make_float2(c.z, c.w);
    const float2 nearX = r.neg0 ? maxX : minX, farX = r.neg0 ? minX : maxX;
    const float2 nearY = r.neg1 ? maxY : minY, farY = r.neg1 ? minY : maxY;
    const float2 nearZ = r.neg2 ? maxZ : minZ, farZ = r.neg2 ? minZ : maxZ;
    const float2 nox = make_float2(-r.o.x, -r.o.x), noy = make_float2(-r.o.y, -r.o.y), noz = make_float2(-r.o.z, -r.o.z);
    const float2 ix = make_float2(r.invDir.x, r.invDir.x), iy = make_float2(r.invDir.y, r.invDir.y), iz = make_float2(r.invDir.z, r.invDir.z);
    const float2 sc2 = make_float2(kSlabScale, kSlabScale);
    const float2 tMin = fmul2(fadd2(nearX, nox), ix);
    const float2 tMax = fmul2(fmul2(fadd2(farX, nox), ix), sc2);
    const float2 tyMin = fmul2(fadd2(nearY, noy), iy);
    const float2 tyMax = fmul2(fmul2(fadd2(farY, noy), iy), sc2);
    const float2 tzMin = fmul2(fadd2(nearZ, noz), iz);
    const float2 tzMax = fmul2(fmul2(fadd2(farZ, noz), iz), sc2);
    {
        const bool miss1 = (tMin.x > tyMax.x) | (tyMin.x > tMax.x);
        float lo = (tyMin.x > tMin.x) ? tyMin.x : tMin.x, hi = (tyMax.x < tMax.x) ? tyMax.x : tMax.x;
        const bool miss2 = (lo > tzMax.x) | (tzMin.x > hi);
        lo = (tzMin.x > lo) ? tzMin.x : lo;
        hi = (tzMax.x < hi) ? tzMax.x : hi;
        *tMin0 = lo;
        *pass0 = !miss1 & !miss2 & (lo < rayTMax) & (hi > 0);
    }
    {
        const bool miss1 = (tMin.y > tyMax.y) | (tyMin.y > tMax.y);
        float lo = (tyMin.y > tMin.y) ? tyMin.y : tMin.y, hi = (tyMax.y < tMax.y) ? tyMax.y : tMax.y;
        const bool miss2 = (lo > tzMax.y) | (tzMin.y > hi);
        lo = (tzMin.y > lo) ? tzMin.y : lo;
        hi = (tzMax.y < hi) ? tzMax.y : hi;
        *tMin1 = lo;
        *pass1 = !miss1 & !miss2 & (lo < rayTMax) & (hi > 0);
    }
#else
    *pass0 = slabTestT(a.x, a.z, b.x, b.z, c.x, c.z, r, rayTMax, tMin0);
    *pass1 = slabTestT(a.y, a.w, b.y, b.w, c.y, c.w, r, rayTMax, tMin1);
#endif
}

// slabTestPairFast (pb2_scene.cuh) for two slots of a four-child record: rays with finite origin and 1 / d only.
PB2_HD void slabTestPair4Fast(float4 a, float4 b, float4 c, const DRaySetup &r, float rayTMax, bool *pass0, bool *pass1, float *tMin0,
                              float *tMin1) {
#if defined(__CUDA_ARCH__)
    const float2 minX = make_float2(a.x, a.y), minY = make_float2(a.z, a.w), minZ = make_float2(b.x, b.y);
    const float2 maxX = make_float2(b.z, b.w), maxY = make_float2(c.x, c.y), maxZ = make_float2(c.z, c.w);
    const float2 nearX = r.neg0 ? maxX : minX, farX = r.neg0 ? minX : maxX;
    const float2 nearY = r.neg1 ? maxY : minY, farY = r.neg1 ? minY : maxY;
    const float2 nearZ = r.neg2 ? maxZ : minZ, farZ = r.neg2 ? minZ : maxZ;
    const float2 nox = make_float2(-r.o.x, -r.o.x), noy = make_float2(-r.o.y, -r.o.y), noz = make_float2(-r.o.z, -r.o.z);
    const float2 ix = make_float2(r.invDir.x, r.invDir.x), iy = make_float2(r.invDir.y, r.invDir.y), iz = make_float2(r.invDir.z, r.invDir.z);
    const float2 sc2 = make_float2(kSlabScale, kSlabScale);
    const float2 tMin = fmul2(fadd2(nearX, nox), ix);
    const float2 tMax = fmul2(fmul2(fadd2(farX, nox), ix), sc2);
    const float2 tyMin = fmul2(fadd2(nearY, noy), iy);
    const float2 tyMax = fmul2(fmul2(fadd2(farY, noy), iy), sc2);
    const float2 tzMin = fmul2(fadd2(nearZ, noz), iz);
    const float2 tzMax = fmul2(fmul2(fadd2(farZ, noz), iz), sc2);
    const float lo0 = fmaxf(fmaxf(tMin.x, tyMin.x), tzMin.x), hi0 = fminf(fminf(tMax.x, tyMax.x), tzMax.x);
    const float lo1 = fmaxf(fmaxf(tMin.y, tyMin.y), tzMin.y), hi1 = fminf(fminf(tMax.y, tyMax.y), tzMax.y);
    *tMin0 = lo0;
    *tMin1 = lo1;
    *pass0 = (lo0 <= hi0) & (lo0 < rayTMax) & (hi0 > 0);
    *pass1 = (lo1 <= hi1) & (lo1 < rayTMax) & (hi1 > 0);
#else
    slabTestPair4(a, b, c, r, rayTMax, pass0, pass1, tMin0, tMin1);
#endif
}

// One visit of a four-child record: which slots' boxes the ray enters (pass, tMin) and, for each entered slot, how many
// entered slots the reference's order visits AFTER it (`after`).  The slot with after == nPass - 1 is the one to continue
// with; every other entered slot goes on the stack at position sp + after[slot], which puts the next one to visit on top.
// The order: the node's near child first (by its split axis and the ray's direction sign), inside each child its own near
// child first - slot s = 2 g + j is visited before slot s' = 2 g' + j' iff g is the near child (g != g'), or j the near
// grandchild (g == g').
struct Wide4Visit {
    bool pass[4];
    float tMin[4];
    int after[4];
    int nPass;
};
template <bool FAST = false>
PB2_HD Wide4Visit wide4Visit(float4 q0, float4 q1, float4 q2, float4 q3, float4 q4, float4 q5, float4 q6, uint32_t meta, const DRaySetup &r,
                             float tMax) {
    Wide4Visit v;
    if (FAST) {
        slabTestPair4Fast(q0, q1, q2, r, tMax, &v.pass[0], &v.pass[1], &v.tMin[0], &v.tMin[1]);
        slabTestPair4Fast(q3, q4, q5, r, tMax, &v.pass[2], &v.pass[3], &v.tMin[2], &v.tMin[3]);
    } else {
        slabTestPair4(q0, q1, q2, r, tMax, &v.pass[0], &v.pass[1], &v.tMin[0], &v.tMin[1]);
        slabTestPair4(q3, q4, q5, r, tMax, &v.pass[2], &v.pass[3], &v.tMin[2], &v.tMin[3]);
    }
    // an empty slot's box is (+inf, -inf), which no ray enters; the explicit test keeps NaNs of 0 * inf out of the verdict
    v.pass[1] &= floatBits(q6.y) != WIDE4_EMPTY;
    v.pass[3] &= floatBits(q6.w) != WIDE4_EMPTY;
    v.pass[0] &= floatBits(q6.x) != WIDE4_EMPTY;
    v.pass[2] &= floatBits(q6.z) != WIDE4_EMPTY;
    const uint32_t negMask = (uint32_t)r.neg0 | ((uint32_t)r.neg1 << 1) | ((uint32_t)r.neg2 << 2);
    const bool nT = (negMask >> (meta & 3u)) & 1u, nA = (negMask >> ((meta >> 2) & 3u)) & 1u, nB = (negMask >> ((meta >> 4) & 3u)) & 1u;
    const int cntA = (int)v.pass[0] + (int)v.pass[1], cntB = (int)v.pass[2] + (int)v.pass[3];
    const int afterPairA = nT ? 0 : cntB, afterPairB = nT ? cntA : 0;   // the far child's slots come after the near child's
    v.after[0] = (int)(v.pass[1] & !nA) + afterPairA;
    v.after[1] = (int)(v.pass[0] & nA) + afterPairA;
    v.after[2] = (int)(v.pass[3] & !nB) + afterPairB;
    v.after[3] = (int)(v.pass[2] & nB) + afterPairB;
    v.nPass = cntA + cntB;
    return v;
}

}  // namespace pb2
#endif
