// Device-resident scene layout and the ray/box, ray/triangle and BVH traversal code.
//
// HBM layout (all arrays are uploaded once per scene and read-only during rendering):
//   nodes      pb2_bvh_node[n_nodes], 32 B each, byte-for-byte the reference's LinearBVHNode
//              (src/accelerators/bvh.cpp:95-104); a node is fetched as two 16-B vector loads.
//   wide       the same tree with the boxes moved up one level: one 64-B record per INTERIOR node,
//              float4 q0 = (c0.min.xyz, c0.max.x), q1 = (c0.max.yz, c1.min.xy), q2 = (c1.min.z, c1.max.xyz),
//              q3 = (ref0, ref1, meta, -) with c0 = the node's first child (index + 1), c1 = its second;
//              ref = index of the child's wide record, or WIDE_LEAF | (nPrims - 1) << 27 | primitivesOffset;
//              meta = the node's split axis (bits 0-1) | WIDE_SINGLE.  Record 0 is a pseudo node whose
//              only child is the root.  One fetch tests both children's boxes, so the render kernel
//              makes half the dependent memory round trips of the 32-B layout; every box is still
//              tested exactly once per ray, with the verdict the reference reaches (see k_wf_trace_w).
//   wide4      two levels of the tree per record: one 128-B record per interior node of every second level with the
//              boxes of its four grandchildren (device/pb2_wide4.cuh) - what the default trace kernel walks.
//   leafPrims  one 48-B record per primitive IN BVH ORDER (= BVHAccel::primitives order):
//              float4 a = (p0.xyz, primNumber), b = (p1.xyz, flags),
//              c = (p2.xyz, area-light number or -1 | sphereIndex for a sphere);
//              triangle vertices are pre-gathered through the index buffer so a leaf test is three
//              16-B loads from consecutive addresses instead of the reference's
//              primitive -> shape -> mesh -> index -> vertex pointer chase.  Shading rebuilds the
//              SurfaceInteraction of a plain triangle (no per-vertex N/S/UV) from the same record.
//   lightRecs  the same 48-B record for the shape of every area light, in light order (light sampling).
//   everything else (P/N/UV/indices, per-primitive material ids, materials, lights,
//   light-distribution tables, Halton permutations) is only touched at shading time.
#ifndef PB2_SCENE_CUH
#define PB2_SCENE_CUH

#include "pb2.h"
#include "pb2_math.cuh"
#include "pb2_texture.cuh"

namespace pb2 {

enum : uint32_t {
    LEAF_SPHERE = 1u,         // record describes a sphere, not a triangle
    LEAF_DEGENERATE = 2u,     // Triangle::Intersect rejects every hit (triangle.cpp:308-314); IntersectP does not
    LEAF_FLIP = 4u,           // reverseOrientation ^ transformSwapsHandedness of the triangle's mesh
    LEAF_ATTR = 8u,           // the mesh has per-vertex N, S or UV: shading must go through the index buffer
    LEAF_INSTANCE = 16u,      // record describes a TransformedPrimitive: c.w = instance number
    LEAF_ALPHA = 32u,         // the triangle's mesh has an alpha or shadow-alpha texture (triangle.cpp:333-338, 531-569)
};
enum : uint32_t {
    WIDE_LEAF = 0x80000000u,  // child reference: bits 0-26 primitivesOffset, bits 27-30 nPrimitives - 1
    WIDE_LEAF_COUNT_SHIFT = 27,
    WIDE_LEAF_OFFSET_MASK = (1u << 27) - 1,
    WIDE_SINGLE = 4u,         // meta: the record has only child 0 (the pseudo node above the root)
    WIDE_MAX_PRIMS = 1u << 27,   // 134 M primitives (config 5 has 50 M)
    WIDE_MAX_LEAF = 16u,         // primitives per leaf (the reference's default maxnodeprims is 4)
};

struct DLightDist {
    int strategy;             // PB2_LIGHTDIST_*
    int nVoxels[3];
    V3 boundsMin, boundsMax;  // Scene::WorldBound()
    const float *table;       // uniform/power: one record; spatial: one record per voxel (eager) / per touched voxel (lazy)
    int stride;               // floats per record: nLights func, nLights+1 cdf, 1 funcInt
    // Lazy spatial distribution (scenes with so many lights that a record for every voxel would not fit: every emissive
    // triangle is a light).  Like the reference's hash table (lightdistrib.cpp:141-230) a voxel's distribution is computed
    // when a path vertex first falls into it - here without waiting inside a kernel: the lookup of a missing voxel puts it
    // on a request list and returns null, the vertex is deferred, k_lightdist_build computes the requested records
    // between two kernels of the round, and the deferred vertices are shaded again.
    int *slots;               // nullptr = eager.  Per voxel: LD_ABSENT, LD_REQUESTED, or the record's index in `table`
    int *requests;            // voxels asked for since the last build (each voxel is asked for at most once)
    int *counters;            // [0] number of requests, [1] records allocated, [2] set when the pool overflowed
    int poolRecords;          // capacity of `table` in records
};
enum { LD_ABSENT = -1, LD_REQUESTED = -2 };

// TransformedPrimitive with a static transform (pb2_instance).
struct DInstance {
    M44 i2w, w2i;
    int root;       // global index of the object BVH's root node, or -1
    int lone;       // root < 0: leaf record of the object's only primitive
    int identity;   // Transform::IsIdentity(): the interaction is then not transformed (primitive.cpp:85-86)
    int wroot;      // two-child records: the pseudo record whose only child is the object BVH's root, or -1
    int wroot4;     // four-child records: the record of the object BVH's root
};

// A delta light as its constructor leaves it (point.h:52, spot.cpp:43-50, distant.cpp:43-46), derived from pb2_delta_light at upload
struct DDeltaLight {
    float p[3];                 // pLight, or the normalised wLight of a distant light
    float cosTotalWidth, cosFalloffStart;
    float worldRadius;
    float worldToLight[9];
    float pad;
    // InfiniteAreaLight with constant radiance (infinite.cpp:43-83 without a texture map): its 1 x 1 radiance map is
    // pb2_light::L; the sampling distribution over the 2 x 2 image the constructor derives from it, as three
    // Distribution1D records [func(2) | cdf(3) | funcInt]: row v = 0, row v = 1, the marginal over the rows
    float lightToWorld[9];
    float dist[18];
    float pad2;
    // ... with an environment map (pb2_delta_light::env_tex): Lmap is texture envTex - 1 of the scene's texture pool, the
    // Distribution2D over its 2w x 2h image is envDist: envNv rows of [func(envNu) | cdf(envNu + 1) | funcInt], then the
    // marginal [func(envNv) | cdf(envNv + 1) | funcInt] over the rows' integrals
    const float *envDist;
    int envNu, envNv;
    int envTex;
    int pad3;
};

struct DScene {
    const float4 *nodes;
    const float4 *wide;       // two-child nodes (below), nullptr when the scene exceeds their limits
    const float4 *wide4;      // four-child records (pb2_wide4.cuh), nullptr under the same condition
    const float4 *leafPrims;
    const float4 *lightRecs;
    int64_t nNodes, nPrims, nTris;
    const float *P, *N, *UV, *S;
    const int32_t *triIndex, *triMesh;
    const pb2_mesh *meshes;
    const pb2_sphere *spheres;
    const uint8_t *primType;
    const int32_t *primIndex, *primMaterial, *primLight;
    const pb2_material *materials;
    const pb2_light *lights;
    const DDeltaLight *deltaLights;       // parallel to lights, nullptr when every light is an area light
    int nLights;
    int nInfinite;            // Scene::infiniteLights (scene.h:66): entries of `lights` that escaped rays see
    int infinite[4];
    const DInstance *instances;   // nullptr: no object instancing in this scene
    int nInstances;
    DLightDist lightDist;
    const DTexture *textures;     // image textures (pb2_texture.cuh); nullptr: a scene of constant textures
    const float *texels;          // [0, 128): MIPMap::weightLut, then the pyramids
    int nTextures;
    int hasAlpha;                 // some mesh carries an alpha or shadow-alpha texture
};

struct DRay {
    V3 o, d;
    float tMax;
};

// Result of a closest-hit query: enough to rebuild the reference's SurfaceInteraction lazily.
struct DHit {
    int leaf;       // index into leafPrims (BVH order), -1 = miss
    float b0, b1, b2;
    int inst;       // instance the hit primitive was reached through, -1 = none
};

// Device analogue of the reference's STAT_COUNTERs around bvh.cpp:672/677/710/714: nodes fetched and
// primitives tested.  Pass nullptr to traverse without counting (the branch folds away after inlining).
struct DCounters { unsigned long long nodes, prims; };
#define PB2_COUNT_NODE(c) do { if (c) (c)->nodes++; } while (0)
#define PB2_COUNT_PRIM(c) do { if (c) (c)->prims++; } while (0)

// Per-ray constants of the watertight test (triangle.cpp:206-222) and of the slab test
// (bvh.cpp:666-667), computed once per ray instead of once per primitive.
struct DRaySetup {
    V3 o;
    V3 invDir;
    int neg0, neg1, neg2;
    int kx, ky, kz;
    float Sx, Sy, Sz;
    int slow;   // origin or 1 / d not finite: slab tests may meet NaNs (0 * inf) and must take the reference's exact compare sequence
};

PB2_HD float permuted(V3 v, int k) { return k == 0 ? v.x : (k == 1 ? v.y : v.z); }

PB2_HD DRaySetup setupRay(V3 o, V3 d) {
    DRaySetup s;
    s.o = o;
    s.invDir = mk3(1 / d.x, 1 / d.y, 1 / d.z);
    s.neg0 = s.invDir.x < 0;
    s.neg1 = s.invDir.y < 0;
    s.neg2 = s.invDir.z < 0;
    V3 ad = vabs(d);
    // MaxDimension (geometry.h:998-1001)
    s.kz = (ad.x > ad.y) ? ((ad.x > ad.z) ? 0 : 2) : ((ad.y > ad.z) ? 1 : 2);
    s.kx = s.kz + 1;
    if (s.kx == 3) s.kx = 0;
    s.ky = s.kx + 1;
    if (s.ky == 3) s.ky = 0;
    float dx = permuted(d, s.kx), dy = permuted(d, s.ky), dz = permuted(d, s.kz);
    s.Sx = -dx / dz;
    s.Sy = -dy / dz;
    s.Sz = 1.f / dz;
    // |x| < inf is false for NaN and infinities alike
    s.slow = !((fabsf(s.invDir.x) < PB2_INFINITY) & (fabsf(s.invDir.y) < PB2_INFINITY) & (fabsf(s.invDir.z) < PB2_INFINITY) &
               (fabsf(o.x) < PB2_INFINITY) & (fabsf(o.y) < PB2_INFINITY) & (fabsf(o.z) < PB2_INFINITY));
    return s;
}

// Bounds3::IntersectP(ray, invDir, dirIsNeg), geometry.h:1412-1438.
// The same test with the box given as six floats; also returns the entry parameter tMin, the only
// quantity the verdict compares with ray.tMax - a caller that keeps tMin can re-evaluate the test
// for a smaller ray.tMax later without the box (`pass && tMin < newTMax`).
PB2_HD bool slabTestT(float minx, float miny, float minz, float maxx, float maxy, float maxz, const DRaySetup &r,
                      float rayTMax, float *tMinOut) {
    float bx0 = r.neg0 ? maxx : minx, bx1 = r.neg0 ? minx : maxx;
    float by0 = r.neg1 ? maxy : miny, by1 = r.neg1 ? miny : maxy;
    float bz0 = r.neg2 ? maxz : minz, bz1 = r.neg2 ? minz : maxz;
    float tMin = (bx0 - r.o.x) * r.invDir.x;
    float tMax = (bx1 - r.o.x) * r.invDir.x;
    float tyMin = (by0 - r.o.y) * r.invDir.y;
    float tyMax = (by1 - r.o.y) * r.invDir.y;
    tMax *= kSlabScale;
    tyMax *= kSlabScale;
    // The reference's early returns, evaluated without branches (lanes of a warp test different
    // boxes; diverging here costs more than the few instructions an early exit would skip).  Each
    // comparison and update is the reference's, so every value that reaches the verdict is too.
    const bool miss1 = (tMin > tyMax) | (tyMin > tMax);
    tMin = (tyMin > tMin) ? tyMin : tMin;
    tMax = (tyMax < tMax) ? tyMax : tMax;
    float tzMin = (bz0 - r.o.z) * r.invDir.z;
    float tzMax = (bz1 - r.o.z) * r.invDir.z;
    tzMax *= kSlabScale;
    const bool miss2 = (tMin > tzMax) | (tzMin > tMax);
    tMin = (tzMin > tMin) ? tzMin : tMin;
    tMax = (tzMax < tMax) ? tzMax : tMax;
    *tMinOut = tMin;
    return !miss1 & !miss2 & (tMin < rayTMax) & (tMax > 0);
}

// Pairs of floats, lane 0 = child 0, lane 1 = child 1.  sm_90 has no packed FP32x2 add / multiply: each
// pair is two IEEE operations, never contracted into an FMA.
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
#endif

// Both children of a two-child record at once.  On the device the subtractions, multiplications and
// the far-plane scaling run on pairs (fadd2 / fmul2) - per component these are the IEEE operations of
// slabTestT, so the verdicts and tMin values are bit-identical to two slabTestT calls.
PB2_HD void slabTestPair(float4 q0, float4 q1, float4 q2, const DRaySetup &r, float rayTMax, bool *pass0, bool *pass1,
                         float *tMin0, float *tMin1) {
#if defined(__CUDA_ARCH__)
    // child 0: min = (q0.x, q0.y, q0.z), max = (q0.w, q1.x, q1.y); child 1: min = (q1.z, q1.w, q2.x), max = (q2.y, q2.z, q2.w)
    const float2 minX = make_float2(q0.x, q1.z), minY = make_float2(q0.y, q1.w), minZ = make_float2(q0.z, q2.x);
    const float2 maxX = make_float2(q0.w, q2.y), maxY = make_float2(q1.x, q2.z), maxZ = make_float2(q1.y, q2.w);
    const float2 nearX = r.neg0 ? maxX : minX, farX = r.neg0 ? minX : maxX;
    const float2 nearY = r.neg1 ? maxY : minY, farY = r.neg1 ? minY : maxY;
    const float2 nearZ = r.neg2 ? maxZ : minZ, farZ = r.neg2 ? minZ : maxZ;
    const float2 nox = make_float2(-r.o.x, -r.o.x), noy = make_float2(-r.o.y, -r.o.y), noz = make_float2(-r.o.z, -r.o.z);
    const float2 ix = make_float2(r.invDir.x, r.invDir.x), iy = make_float2(r.invDir.y, r.invDir.y), iz = make_float2(r.invDir.z, r.invDir.z);
    const float2 sc2 = make_float2(kSlabScale, kSlabScale);
    float2 tMin = fmul2(fadd2(nearX, nox), ix);
    float2 tMax = fmul2(fmul2(fadd2(farX, nox), ix), sc2);
    const float2 tyMin = fmul2(fadd2(nearY, noy), iy);
    const float2 tyMax = fmul2(fmul2(fadd2(farY, noy), iy), sc2);
    const float2 tzMin = fmul2(fadd2(nearZ, noz), iz);
    const float2 tzMax = fmul2(fmul2(fadd2(farZ, noz), iz), sc2);
    {
        const bool miss1 = (tMin.x > tyMax.x) | (tyMin.x > tMax.x);
        float a = (tyMin.x > tMin.x) ? tyMin.x : tMin.x, b = (tyMax.x < tMax.x) ? tyMax.x : tMax.x;
        const bool miss2 = (a > tzMax.x) | (tzMin.x > b);
        a = (tzMin.x > a) ? tzMin.x : a;
        b = (tzMax.x < b) ? tzMax.x : b;
        *tMin0 = a;
        *pass0 = !miss1 & !miss2 & (a < rayTMax) & (b > 0);
    }
    {
        const bool miss1 = (tMin.y > tyMax.y) | (tyMin.y > tMax.y);
        float a = (tyMin.y > tMin.y) ? tyMin.y : tMin.y, b = (tyMax.y < tMax.y) ? tyMax.y : tMax.y;
        const bool miss2 = (a > tzMax.y) | (tzMin.y > b);
        a = (tzMin.y > a) ? tzMin.y : a;
        b = (tzMax.y < b) ? tzMax.y : b;
        *tMin1 = a;
        *pass1 = !miss1 & !miss2 & (a < rayTMax) & (b > 0);
    }
#else
    *pass0 = slabTestT(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, r, rayTMax, tMin0);
    *pass1 = slabTestT(q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, r, rayTMax, tMin1);
#endif
}

// The same verdicts with min / max instructions, for rays whose origin and 1 / d are finite (DRaySetup::slow == 0).
// Without NaNs the reference's compare-and-assign steps ARE maxima and minima: tMin = max(tx0, ty0, tz0), tMax =
// min(tx1, ty1, tz1) (values equal up to the sign of a zero, which no comparison sees), and its two early returns reject
// exactly the boxes where some entry parameter exceeds ANOTHER axis' exit parameter.  `tMin <= tMax` also compares the
// two parameters of the same axis; they can only be out of order when the exit parameter is negative (the far-plane
// scaling by 1 + 2 gamma(3) moves it away from zero), and then the reference's final `tMax > 0` rejects the box as well.
// Four min / max instructions per box after the multiplications instead of ~16 compare-and-selects.
PB2_HD void slabTestPairFast(float4 q0, float4 q1, float4 q2, const DRaySetup &r, float rayTMax, bool *pass0, bool *pass1,
                             float *tMin0, float *tMin1) {
#if defined(__CUDA_ARCH__)
    const float2 minX = make_float2(q0.x, q1.z), minY = make_float2(q0.y, q1.w), minZ = make_float2(q0.z, q2.x);
    const float2 maxX = make_float2(q0.w, q2.y), maxY = make_float2(q1.x, q2.z), maxZ = make_float2(q1.y, q2.w);
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
    slabTestPair(q0, q1, q2, r, rayTMax, pass0, pass1, tMin0, tMin1);
#endif
}

PB2_HD bool slabTest(float4 n0, float4 n1, const DRaySetup &r, float rayTMax) {
    // n0 = (min.x, min.y, min.z, max.x), n1 = (max.y, max.z, offset, meta)
    float bx0 = r.neg0 ? n0.w : n0.x, bx1 = r.neg0 ? n0.x : n0.w;
    float by0 = r.neg1 ? n1.x : n0.y, by1 = r.neg1 ? n0.y : n1.x;
    float bz0 = r.neg2 ? n1.y : n0.z, bz1 = r.neg2 ? n0.z : n1.y;
    float tMin = (bx0 - r.o.x) * r.invDir.x;
    float tMax = (bx1 - r.o.x) * r.invDir.x;
    float tyMin = (by0 - r.o.y) * r.invDir.y;
    float tyMax = (by1 - r.o.y) * r.invDir.y;
    tMax *= kSlabScale;
    tyMax *= kSlabScale;
    if (tMin > tyMax || tyMin > tMax) return false;
    if (tyMin > tMin) tMin = tyMin;
    if (tyMax < tMax) tMax = tyMax;
    float tzMin = (bz0 - r.o.z) * r.invDir.z;
    float tzMax = (bz1 - r.o.z) * r.invDir.z;
    tzMax *= kSlabScale;
    if (tMin > tzMax || tzMin > tMax) return false;
    if (tzMin > tMin) tMin = tzMin;
    if (tzMax < tMax) tMax = tzMax;
    return (tMin < rayTMax) && (tMax > 0);
}

// The geometric part shared by Triangle::Intersect and IntersectP (triangle.cpp:197-291 / 435-527):
// translate, permute, shear, edge functions (double fallback on exact zeros), scaled-t range test,
// conservative t > deltaT test.  Returns true and t,b0,b1,b2 when the ray hits within (0, rayTMax).
PB2_HD bool triangleTest(V3 p0, V3 p1, V3 p2, const DRaySetup &r, float rayTMax, float *tOut, float *b0Out,
                         float *b1Out, float *b2Out) {
    V3 q0 = p0 - r.o, q1 = p1 - r.o, q2 = p2 - r.o;
    float p0x = permuted(q0, r.kx), p0y = permuted(q0, r.ky), p0z = permuted(q0, r.kz);
    float p1x = permuted(q1, r.kx), p1y = permuted(q1, r.ky), p1z = permuted(q1, r.kz);
    float p2x = permuted(q2, r.kx), p2y = permuted(q2, r.ky), p2z = permuted(q2, r.kz);
    p0x += r.Sx * p0z;
    p0y += r.Sy * p0z;
    p1x += r.Sx * p1z;
    p1y += r.Sy * p1z;
    p2x += r.Sx * p2z;
    p2y += r.Sy * p2z;
    float e0 = p1x * p2y - p1y * p2x;
    float e1 = p2x * p0y - p2y * p0x;
    float e2 = p0x * p1y - p0y * p1x;
    if (e0 == 0.0f || e1 == 0.0f || e2 == 0.0f) {
        double p2txp1ty = (double)p2x * (double)p1y;
        double p2typ1tx = (double)p2y * (double)p1x;
        e0 = (float)(p2typ1tx - p2txp1ty);
        double p0txp2ty = (double)p0x * (double)p2y;
        double p0typ2tx = (double)p0y * (double)p2x;
        e1 = (float)(p0typ2tx - p0txp2ty);
        double p1txp0ty = (double)p1x * (double)p0y;
        double p1typ0tx = (double)p1y * (double)p0x;
        e2 = (float)(p1typ0tx - p1txp0ty);
    }
    if ((e0 < 0 || e1 < 0 || e2 < 0) && (e0 > 0 || e1 > 0 || e2 > 0)) return false;
    float det = e0 + e1 + e2;
    if (det == 0) return false;
    p0z *= r.Sz;
    p1z *= r.Sz;
    p2z *= r.Sz;
    float tScaled = e0 * p0z + e1 * p1z + e2 * p2z;
    if (det < 0 && (tScaled >= 0 || tScaled < rayTMax * det)) return false;
    else if (det > 0 && (tScaled <= 0 || tScaled > rayTMax * det)) return false;
    float invDet = 1 / det;
    float b0 = e0 * invDet, b1 = e1 * invDet, b2 = e2 * invDet;
    float t = tScaled * invDet;
    float maxZt = maxComponent(vabs(mk3(p0z, p1z, p2z)));
    float deltaZ = kGamma3 * maxZt;
    float maxXt = maxComponent(vabs(mk3(p0x, p1x, p2x)));
    float maxYt = maxComponent(vabs(mk3(p0y, p1y, p2y)));
    float deltaX = kGamma5 * (maxXt + maxZt);
    float deltaY = kGamma5 * (maxYt + maxZt);
    float deltaE = 2 * (kGamma2 * maxXt * maxYt + deltaY * maxXt + deltaX * maxYt);
    float maxE = maxComponent(vabs(mk3(e0, e1, e2)));
    float deltaT = 3 * (kGamma3 * maxE * maxZt + deltaE * maxZt + deltaZ * maxE) * fabsf(invDet);
    if (t <= deltaT) return false;
    *tOut = t;
    *b0Out = b0;
    *b1Out = b1;
    *b2Out = b2;
    return true;
}

PB2_HD float4 ldg4(const float4 *p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
PB2_HD int asInt(float f) { return (int)floatBits(f); }
// 32 bytes of a node record.  sm_90's widest global load is 16 bytes per lane: two read-only 16-byte loads.
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ void ldg256(const float4 *p, float4 &a, float4 &b) {
    a = __ldg(p);
    b = __ldg(p + 1);
}
#else
inline void ldg256(const float4 *p, float4 &a, float4 &b) { a = p[0]; b = p[1]; }
#endif

struct SphereHit;  // pb2_sphere.cuh
PB2_HDN bool sphereLeafTest(const DScene &sc, int sphereIndex, const DRay &ray, float rayTMax, float *tHit, float *phi);

// Transform::operator()(const Ray &) (transform.h:251-264): the ray in the space of `t`, its origin
// moved along d to the edge of the transformed origin's error box and tMax shortened by the same dt.
PB2_HD DRay xfRay(const M44 &t, const DRay &r, float tMax) {
    V3 oError;
    V3 o = xfPointErr(t, r.o, &oError);
    V3 d = xfVector(t, r.d);
    float lengthSq = lengthSquared(d);
    if (lengthSq > 0) {
        float dt = dot(vabs(d), oError) / lengthSq;
        o = o + d * dt;
        tMax -= dt;
    }
    DRay out;
    out.o = o;
    out.d = d;
    out.tMax = tMax;
    return out;
}

// The alpha test of Triangle::Intersect (triangle.cpp:333-338) and IntersectP (triangle.cpp:531-569) for a hit at
// barycentrics (b0, b1, b2) of scene primitive `prim`: true when the hit does not count.  The look-up has no differentials
// (isectLocal is built without any), so both MIPMap filters reduce to the bilinear one at the finest level.
PB2_HDN bool alphaRejects(const DScene &sc, int prim, float b0, float b1, float b2, bool anyHit) {
    const int tri = sc.primIndex[prim];
    const pb2_mesh &mesh = sc.meshes[sc.triMesh[tri]];
    if (!mesh.alpha_tex && !(anyHit && mesh.shadow_alpha_tex)) return false;
    V2 uv0 = mk2(0, 0), uv1 = mk2(1, 0), uv2 = mk2(1, 1);   // Triangle::GetUVs (triangle.h:98-108)
    if (mesh.has_uv) {
        const int64_t v0 = sc.triIndex[3 * (int64_t)tri], v1 = sc.triIndex[3 * (int64_t)tri + 1], v2 = sc.triIndex[3 * (int64_t)tri + 2];
        uv0 = mk2(sc.UV[2 * v0], sc.UV[2 * v0 + 1]);
        uv1 = mk2(sc.UV[2 * v1], sc.UV[2 * v1 + 1]);
        uv2 = mk2(sc.UV[2 * v2], sc.UV[2 * v2 + 1]);
    }
    const V2 uvHit = mk2(b0 * uv0.x + b1 * uv1.x + b2 * uv2.x, b0 * uv0.y + b1 * uv1.y + b2 * uv2.y);
    DUvDiff none;   // (zero footprint: both MIPMap filters reduce to the bilinear look-up at the finest level)
    none.dudx = none.dvdx = none.dudy = none.dvdy = 0;
    if (mesh.alpha_tex && texEvaluateNode(sc.textures, sc.texels, mesh.alpha_tex - 1, uvHit, none).x == 0) return true;
    if (anyHit && mesh.shadow_alpha_tex && texEvaluateNode(sc.textures, sc.texels, mesh.shadow_alpha_tex - 1, uvHit, none).x == 0) return true;
    return false;
}

template <int LEVEL>
PB2_HD bool traverseLevel(const DScene &sc, int root, const DRay &ray, const DRaySetup &rs, const bool ANY, float *tMaxInOut,
                          DHit *hit, DCounters *ctr, int instId);

// One primitive of a leaf (GeometricPrimitive::Intersect[P], primitive.cpp:112-130; LEVEL 0 also
// TransformedPrimitive::Intersect[P], primitive.cpp:76-96).  Returns true when the primitive was
// hit within tMax: for ANY the caller stops, otherwise *tMax and *hit are the new closest hit.
template <int LEVEL>
PB2_HD bool testLeafRecord(const DScene &sc, int recIndex, const DRay &ray, const DRaySetup &rs, const bool ANY, float *tMax,
                           DHit *hit, DCounters *ctr, int instId) {
    const float4 *rec = &sc.leafPrims[3 * (size_t)recIndex];
    float4 a = ldg4(rec), b = ldg4(rec + 1), c = ldg4(rec + 2);
    PB2_COUNT_PRIM(ctr);
    uint32_t flags = floatBits(b.w);
    if (flags & LEAF_SPHERE) {
        float t, phi;
        if (!sphereLeafTest(sc, asInt(c.w), ray, *tMax, &t, &phi)) return false;
        if (ANY) return true;
        *tMax = t;
        hit->leaf = recIndex;
        hit->b0 = phi;
        hit->b1 = hit->b2 = 0;
        hit->inst = instId;
        return true;
    }
    if (flags & LEAF_INSTANCE) {
        if (LEVEL != 0) return false;   // pbrtObjectInstance inside an object definition is an error (api.cpp:1554-1557)
        const int id = asInt(c.w);
        const DInstance &inst = sc.instances[id];
        DRay r2 = xfRay(inst.w2i, ray, *tMax);
        DRaySetup rs2 = setupRay(r2.o, r2.d);
        float t2 = r2.tMax;
        bool f = inst.root >= 0 ? traverseLevel<1>(sc, inst.root, r2, rs2, ANY, &t2, hit, ctr, id)
                                : testLeafRecord<1>(sc, inst.lone, r2, rs2, ANY, &t2, hit, nullptr, id);   // counted once, above
        if (!f) return false;
        *tMax = t2;                      // r.tMax = ray.tMax (primitive.cpp:83)
        return true;
    }
    float t, b0, b1, b2;
    if (!triangleTest(mk3(a.x, a.y, a.z), mk3(b.x, b.y, b.z), mk3(c.x, c.y, c.z), rs, *tMax, &t, &b0, &b1, &b2)) return false;
    if ((flags & LEAF_ALPHA) && alphaRejects(sc, asInt(a.w), b0, b1, b2, ANY)) return false;
    if (ANY) return true;
    if (flags & LEAF_DEGENERATE) return false;
    *tMax = t;
    hit->leaf = recIndex;
    hit->b0 = b0;
    hit->b1 = b1;
    hit->b2 = b2;
    hit->inst = instId;
    return true;
}

// BVHAccel::Intersect (ANY=false, bvh.cpp:662-700) and IntersectP (ANY=true, bvh.cpp:702-738):
// depth-first, near child first by dirIsNeg[axis], explicit stack of far children, every primitive
// of a reached leaf tested, closest hit shrinks tMax.  Node visit order and the set of primitive
// tests are exactly the reference's, so device counters equal the instrumented reference's.
template <int LEVEL>
PB2_HD bool traverseLevel(const DScene &sc, int root, const DRay &ray, const DRaySetup &rs, const bool ANY, float *tMaxInOut,
                          DHit *hit, DCounters *ctr, int instId) {
    (void)ctr;
    float tMax = *tMaxInOut;
    bool found = false;
    int stack[64];
    int sp = 0, cur = root;
    while (true) {
        float4 n0 = ldg4(&sc.nodes[2 * (size_t)cur]);
        float4 n1 = ldg4(&sc.nodes[2 * (size_t)cur + 1]);
        PB2_COUNT_NODE(ctr);
        bool descend = false;
        if (slabTest(n0, n1, rs, tMax)) {
            uint32_t meta = floatBits(n1.w);
            int nPrims = (int)(meta & 0xffffu);
            if (nPrims > 0) {
                int first = asInt(n1.z);
                for (int i = 0; i < nPrims; ++i) {
                    if (testLeafRecord<LEVEL>(sc, first + i, ray, rs, ANY, &tMax, hit, ctr, instId)) {
                        if (ANY) return true;
                        found = true;
                    }
                }
            } else {
                int axis = (int)((meta >> 16) & 0xffu);
                int isNeg = axis == 0 ? rs.neg0 : (axis == 1 ? rs.neg1 : rs.neg2);
                int second = asInt(n1.z);
                if (isNeg) {
                    stack[sp++] = cur + 1;
                    cur = second;
                } else {
                    stack[sp++] = second;
                    cur = cur + 1;
                }
                descend = true;
            }
        }
        if (!descend) {
            if (sp == 0) break;
            cur = stack[--sp];
        }
    }
    *tMaxInOut = tMax;
    return found;
}

// Scene::Intersect / IntersectP (scene.cpp:45-55)
PB2_HD bool traverseAnyOrClosest(const DScene &sc, const DRay &ray, const bool ANY, float *tMaxInOut, DHit *hit,
                                 DCounters *ctr) {
    if (sc.nNodes == 0) return false;
    DRaySetup rs = setupRay(ray.o, ray.d);
    return traverseLevel<0>(sc, 0, ray, rs, ANY, tMaxInOut, hit, ctr, -1);
}

template <bool ANY>
PB2_HD bool traverse(const DScene &sc, const DRay &ray, float *tMaxInOut, DHit *hit, DCounters *ctr) {
    return traverseAnyOrClosest(sc, ray, ANY, tMaxInOut, hit, ctr);
}

}  // namespace pb2
#endif
