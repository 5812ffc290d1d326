// Everything that happens at a path vertex, per lane, in registers: rebuilding the
// SurfaceInteraction of the hit, the matte/plastic BSDFs, diffuse area lights, the light-sampling
// distributions, one-light next-event estimation with MIS, BSDF sampling, Russian roulette — and the
// perspective camera that starts a path.  Restates, on flat POD records instead of arena-allocated
// polymorphic objects:
//
//   Triangle::Intersect (post-hit part) / Sample / Area   src/shapes/triangle.cpp:293-424, 574-607
//   Shape::Sample(ref) / Pdf(ref,wi)                       src/core/shape.cpp:61-95
//   SurfaceInteraction, SetShadingGeometry, SpawnRay[To]   src/core/interaction.{h,cpp}
//   BSDF, LambertianReflection, OrenNayar, MicrofacetReflection, FrDielectric
//                                                          src/core/reflection.{h,cpp}
//   TrowbridgeReitzDistribution                            src/core/microfacet.{h,cpp}
//   MatteMaterial / PlasticMaterial                        src/materials/matte.cpp:45-62, plastic.cpp:45-70
//   DiffuseAreaLight                                       src/lights/diffuse.{h,cpp}
//   Uniform/Power/SpatialLightDistribution                 src/core/lightdistrib.cpp
//   UniformSampleOneLight / EstimateDirect                 src/core/integrator.cpp:85-215
//   PathIntegrator::Li                                     src/integrators/path.cpp:64-188
//   PerspectiveCamera::GenerateRayDifferential             src/cameras/perspective.cpp:95-144
#ifndef PB2_SHADE_CUH
#define PB2_SHADE_CUH

#include "pb2_sampler.cuh"
#include "pb2_scene.cuh"

namespace pb2 {

// ---------------------------------------------------------------- interactions
struct DInteraction {   // the part of (Surface)Interaction that Li and EstimateDirect read
    V3 p, pError, n;    // n == 0 marks a non-surface point (Interaction::IsSurfaceInteraction)
    V3 wo;              // Normalize(-ray.d) (interaction.h:61)
    V3 ns;              // shading.n
    V3 dpdus;           // shading.dpdu
    V2 uv;
    int prim;           // scene-order primitive number
};

// What SurfaceInteraction::ComputeDifferentials reads besides p and n: the (geometric) dpdu, dpdv of the hit
// ... and what Material::Bump reads: the shading dpdv, dndu, dndv (shading.dpdu is DInteraction::dpdus)
struct DTexGeom { V3 dpdu, dpdv, dpdvs, dndus, dndvs; };

struct TriVerts { V3 p0, p1, p2; };

PB2_HD V3 ld3(const float *a, int64_t i) { return mk3(a[3 * i], a[3 * i + 1], a[3 * i + 2]); }

PB2_HD TriVerts triVerts(const DScene &sc, int tri) {
    TriVerts t;
    t.p0 = ld3(sc.P, sc.triIndex[3 * (int64_t)tri]);
    t.p1 = ld3(sc.P, sc.triIndex[3 * (int64_t)tri + 1]);
    t.p2 = ld3(sc.P, sc.triIndex[3 * (int64_t)tri + 2]);
    return t;
}

// Triangle::GetUVs (triangle.h:98-108)
PB2_HD void triUVs(const DScene &sc, int tri, const pb2_mesh &mesh, V2 uv[3]) {
    if (mesh.has_uv) {
        for (int k = 0; k < 3; ++k) {
            int64_t v = sc.triIndex[3 * (int64_t)tri + k];
            uv[k] = mk2(sc.UV[2 * v], sc.UV[2 * v + 1]);
        }
    } else {
        uv[0] = mk2(0, 0);
        uv[1] = mk2(1, 0);
        uv[2] = mk2(1, 1);
    }
}

// dpdu/dpdv of a triangle (triangle.cpp:293-317).  Returns false when the triangle is degenerate
// (the reference then rejects the hit).
PB2_HD bool triPartials(V3 p0, V3 p1, V3 p2, const V2 uv[3], V3 *dpdu, V3 *dpdv) {
    float duv02x = uv[0].x - uv[2].x, duv02y = uv[0].y - uv[2].y;
    float duv12x = uv[1].x - uv[2].x, duv12y = uv[1].y - uv[2].y;
    V3 dp02 = p0 - p2, dp12 = p1 - p2;
    float determinant = duv02x * duv12y - duv02y * duv12x;
    bool degenerateUV = (double)fabsf(determinant) < 1e-8;
    *dpdu = mk3(0, 0, 0);
    *dpdv = mk3(0, 0, 0);
    if (!degenerateUV) {
        float invdet = 1 / determinant;
        *dpdu = (duv12y * dp02 - duv02y * dp12) * invdet;
        *dpdv = (-duv12x * dp02 + duv02x * dp12) * invdet;
    }
    if (degenerateUV || lengthSquared(cross(*dpdu, *dpdv)) == 0) {
        V3 ng = cross(p2 - p0, p1 - p0);
        if (lengthSquared(ng) == 0) return false;
        coordinateSystem(normalize(ng), dpdu, dpdv);
    }
    return true;
}

// The SurfaceInteraction Triangle::Intersect fills in for a hit with barycentrics (b0,b1,b2)
// (triangle.cpp:319-419).
// A 48-B leaf / light record (pb2_scene.cuh) unpacked: the triangle's world-space vertices, its
// LEAF_* flags, the scene-order primitive number and the area-light number (-1: not emissive).
struct TriRec {
    TriVerts tv;
    uint32_t flags;
    int prim, light;
};

PB2_HD TriRec loadTriRec(const float4 *recs, size_t i) {
    float4 a = ldg4(&recs[3 * i]), b = ldg4(&recs[3 * i + 1]), c = ldg4(&recs[3 * i + 2]);
    TriRec r;
    r.tv.p0 = mk3(a.x, a.y, a.z);
    r.tv.p1 = mk3(b.x, b.y, b.z);
    r.tv.p2 = mk3(c.x, c.y, c.z);
    r.prim = asInt(a.w);
    r.flags = floatBits(b.w);
    r.light = asInt(c.w);
    return r;
}

PB2_HD DInteraction triangleInteraction(const DScene &sc, const TriRec &rec, float b0, float b1, float b2, V3 rayD, DTexGeom *tg = nullptr) {
    DInteraction it;
    const int prim = rec.prim;
    const TriVerts tv = rec.tv;   // bitwise the vertices the index buffer leads to
    // meshes without per-vertex attributes never leave the record
    int tri = 0;
    pb2_mesh mesh;
    mesh.has_n = mesh.has_s = mesh.has_uv = 0;
    mesh.reverse_orientation = 0;
    mesh.transform_swaps_handedness = (rec.flags & LEAF_FLIP) ? 1 : 0;
    if (rec.flags & LEAF_ATTR) {
        tri = sc.primIndex[prim];
        mesh = sc.meshes[sc.triMesh[tri]];
    }
    V2 uv[3];
    triUVs(sc, tri, mesh, uv);
    V3 dpdu, dpdv;
    triPartials(tv.p0, tv.p1, tv.p2, uv, &dpdu, &dpdv);
    if (tg) {
        tg->dpdu = dpdu;
        tg->dpdv = dpdv;
        tg->dpdvs = dpdv;   // without per-vertex N / S the shading geometry is the geometric one, dndu = dndv = 0
        tg->dndus = tg->dndvs = mk3(0, 0, 0);
    }
    float xAbsSum = (fabsf(b0 * tv.p0.x) + fabsf(b1 * tv.p1.x) + fabsf(b2 * tv.p2.x));
    float yAbsSum = (fabsf(b0 * tv.p0.y) + fabsf(b1 * tv.p1.y) + fabsf(b2 * tv.p2.y));
    float zAbsSum = (fabsf(b0 * tv.p0.z) + fabsf(b1 * tv.p1.z) + fabsf(b2 * tv.p2.z));
    it.pError = kGamma7 * mk3(xAbsSum, yAbsSum, zAbsSum);
    it.p = b0 * tv.p0 + b1 * tv.p1 + b2 * tv.p2;
    it.uv = mk2(b0 * uv[0].x + b1 * uv[1].x + b2 * uv[2].x, b0 * uv[0].y + b1 * uv[1].y + b2 * uv[2].y);
    it.wo = normalize(-rayD);
    it.prim = prim;
    V3 dp02 = tv.p0 - tv.p2, dp12 = tv.p1 - tv.p2;
    it.n = it.ns = normalize(cross(dp02, dp12));
    if ((mesh.reverse_orientation != 0) ^ (mesh.transform_swaps_handedness != 0)) it.n = it.ns = -it.n;
    it.dpdus = dpdu;
    if (mesh.has_n || mesh.has_s) {
        int64_t v0 = sc.triIndex[3 * (int64_t)tri], v1 = sc.triIndex[3 * (int64_t)tri + 1], v2 = sc.triIndex[3 * (int64_t)tri + 2];
        V3 ns;
        if (mesh.has_n) {
            ns = (b0 * ld3(sc.N, v0) + b1 * ld3(sc.N, v1) + b2 * ld3(sc.N, v2));
            if (lengthSquared(ns) > 0) ns = normalize(ns);
            else ns = it.n;
        } else
            ns = it.n;
        V3 ss;
        if (mesh.has_s) {
            ss = (b0 * ld3(sc.S, v0) + b1 * ld3(sc.S, v1) + b2 * ld3(sc.S, v2));
            if (lengthSquared(ss) > 0) ss = normalize(ss);
            else ss = normalize(dpdu);
        } else
            ss = normalize(dpdu);
        V3 ts = cross(ss, ns);
        if (lengthSquared(ts) > 0.f) {
            ts = normalize(ts);
            ss = cross(ts, ns);
        } else
            coordinateSystem(ns, &ss, &ts);
        if (mesh.reverse_orientation) ts = -ts;
        // SetShadingGeometry(ss, ts, dndu, dndv, orientationIsAuthoritative = true), interaction.cpp:73-90
        it.ns = normalize(cross(ss, ts));
        it.n = faceforward(it.n, it.ns);
        it.dpdus = ss;
        if (tg) {
            tg->dpdvs = ts;
            if (mesh.has_n) {
                // dndu, dndv of the interpolated normal (triangle.cpp:383-413)
                const float duv02x = uv[0].x - uv[2].x, duv02y = uv[0].y - uv[2].y;
                const float duv12x = uv[1].x - uv[2].x, duv12y = uv[1].y - uv[2].y;
                const V3 n0 = ld3(sc.N, v0), n1 = ld3(sc.N, v1), n2 = ld3(sc.N, v2);
                const V3 dn1 = n0 - n2, dn2 = n1 - n2;
                const float determinant = duv02x * duv12y - duv02y * duv12x;
                if ((double)fabsf(determinant) < 1e-8) {
                    const V3 dn = cross(n2 - n0, n1 - n0);
                    if (lengthSquared(dn) == 0) tg->dndus = tg->dndvs = mk3(0, 0, 0);
                    else coordinateSystem(dn, &tg->dndus, &tg->dndvs);
                } else {
                    const float invDet = 1 / determinant;
                    tg->dndus = (duv12y * dn1 - duv02y * dn2) * invDet;
                    tg->dndvs = (-duv12x * dn1 + duv02x * dn2) * invDet;
                }
            }
        }
    }
    return it;
}

}  // namespace pb2

#include "pb2_sphere.cuh"

namespace pb2 {

// Shade features (the F template argument of the path functions and kernels): what a frame's scene records and parameters
// can reach.  A bit that is clear compiles away the branches whose run-time condition is false for every record of the
// scene and every parameter of the frame; the code that remains is the same, in the same order.  The host computes a
// frame's mask (frameShadeFeatures in pb2_cuda.cu) and runs the kernel compiled for the fewest bits that contain it.
//   SHADE_OREN_NAYAR   a matte material with sigma != 0 (diffuseKind 2)
//   SHADE_MICROFACET   a plastic material (its Trowbridge-Reitz lobe, hasMicrofacet)
//   SHADE_NON_AREA     a point, spot, distant or infinite light (DScene::deltaLights, nInfinite)
//   SHADE_SPHERES      sphere primitives and sphere area lights (LEAF_SPHERE; the interval-arithmetic code and its call frames)
//   SHADE_SPECULAR     a mirror, glass, substrate, metal or uber material (specKind, blend, general)
//   SHADE_LAZY         the lazy light distribution (DLightDist::slots): a vertex can be handed back (LS_DEFER)
//   SHADE_TEXTURES     image textures: materials' texture slots and bump maps, and the camera ray's differentials
//   SHADE_SOBOL        the frame draws from the SobolSampler (the sampler functions' GENERAL)
// The first three are the shade class that pb2_shade_class reports; SHADE_GENERAL is the class with every lobe and light.
enum { SHADE_OREN_NAYAR = 1, SHADE_MICROFACET = 2, SHADE_NON_AREA = 4, SHADE_SPHERES = 8, SHADE_SPECULAR = 16, SHADE_LAZY = 32,
       SHADE_TEXTURES = 64, SHADE_SOBOL = 128, SHADE_LAMBERT_AREA = 0, SHADE_GENERAL = 7, SHADE_FULL = 255 };

// *light receives the area-light number of the primitive that was hit (-1: not emissive).
// A hit inside an instanced object was found with the ray in instance space (hit.inst >= 0): the
// interaction is built there and then taken to world space as TransformedPrimitive::Intersect does
// with Transform::operator()(const SurfaceInteraction &) (primitive.cpp:85-86, transform.cpp:262-297).
template <int F>
PB2_HD DInteraction hitInteraction(const DScene &sc, const DHit &hit, const DRay &ray, float tHit, int *light = nullptr, DTexGeom *tg = nullptr) {
    TriRec rec = loadTriRec(sc.leafPrims, (size_t)hit.leaf);
    const DInstance *inst = nullptr;
    DRay r = ray;
    if (hit.inst >= 0 && sc.instances) {
        inst = &sc.instances[hit.inst];
        r = xfRay(inst->w2i, ray, ray.tMax);
    }
    DInteraction it;
    if ((F & SHADE_SPHERES) && (rec.flags & LEAF_SPHERE)) {
        if (light) *light = sc.primLight[rec.prim];
        it = sphereInteraction(sc, rec.prim, r, tHit, hit.b0, tg);
    } else {
        if (light) *light = rec.light;
        it = triangleInteraction(sc, rec, hit.b0, hit.b1, hit.b2, r.d, tg);
    }
    if (inst && !inst->identity) {
        V3 pError;
        it.p = xfPointErrIn(inst->i2w, it.p, it.pError, &pError);
        it.pError = pError;
        it.n = normalize(xfNormalInv(inst->w2i, it.n));
        it.wo = normalize(xfVector(inst->i2w, it.wo));
        it.ns = normalize(xfNormalInv(inst->w2i, it.ns));
        it.dpdus = xfVector(inst->i2w, it.dpdus);
        it.ns = faceforward(it.ns, it.n);
        if (tg) {
            tg->dpdu = xfVector(inst->i2w, tg->dpdu);
            tg->dpdv = xfVector(inst->i2w, tg->dpdv);
            tg->dpdvs = xfVector(inst->i2w, tg->dpdvs);
            tg->dndus = xfNormalInv(inst->w2i, tg->dndus);
            tg->dndvs = xfNormalInv(inst->w2i, tg->dndvs);
        }
    }
    return it;
}

// Interaction::SpawnRay (interaction.h:64-67)
PB2_HD DRay spawnRay(const DInteraction &it, V3 d) {
    DRay r;
    r.o = offsetRayOrigin(it.p, it.pError, it.n, d);
    r.d = d;
    r.tMax = PB2_INFINITY;
    return r;
}
// Interaction::SpawnRayTo(const Interaction&) (interaction.h:73-78)
PB2_HD DRay spawnRayTo(const DInteraction &from, V3 toP, V3 toPError, V3 toN) {
    DRay r;
    r.o = offsetRayOrigin(from.p, from.pError, from.n, toP - from.p);
    V3 target = offsetRayOrigin(toP, toPError, toN, r.o - toP);
    r.d = target - r.o;
    r.tMax = 1 - kShadowEpsilon;
    return r;
}

// ---------------------------------------------------------------- BSDF
struct DBsdf {
    V3 ns, ng, ss, ts;     // reflection.h:167-172
    int nLobes;            // 0, 1 or 2
    int diffuseKind;       // 0 none, 1 Lambertian, 2 Oren-Nayar
    V3 R;                  // diffuse reflectance
    float A, B;            // Oren-Nayar terms
    int hasMicrofacet;
    V3 Ks;
    float alpha;           // TrowbridgeReitz alphax == alphay
    // perfectly specular BxDF (not counted in nLobes, which is NumComponents(~BSDF_SPECULAR)):
    int specKind;          // 0 none, 1 SpecularReflection + FresnelNoOp (mirror), 2 FresnelSpecular (smooth glass)
    V3 specR, specT;
    float eta;             // BSDF::eta (reflection.h:216): the glass index, 1 otherwise
    // FresnelBlend (substrate): the one glossy lobe of the BSDF, Rd in R, Rs in Ks, anisotropic Trowbridge-Reitz
    int blend;
    float alphaX, alphaY;
    // BSDFs that are a LIST of BxDFs (uber.cpp:45-104, metal.cpp:60-80): bit i of `general` = lobe i is present,
    // in the order the material adds them.  nLobes counts the non-specular ones (GEN_LAMBERT, GEN_MICROFACET).
    int general;
    int conductor;         // the microfacet lobe's Fresnel: FresnelConductor(1, condEta, condK) instead of FresnelDielectric(1, e)
    V3 T0;                 // GEN_OPACITY: SpecularTransmission(T0, 1, 1)
    V3 condEta, condK;
    float e;               // the index the lobes' Fresnel terms use (BSDF::eta is 1 when GEN_OPACITY is present)
};
enum { BSDF_SAMPLED_SPECULAR = 1, BSDF_SAMPLED_TRANSMISSION = 2 };
enum { GEN_OPACITY = 1, GEN_LAMBERT = 2, GEN_MICROFACET = 4, GEN_SPEC_REFLECTION = 8, GEN_SPEC_TRANSMISSION = 16,
       GEN_MICRO_TRANSMISSION = 32,   // MicrofacetTransmission(specT, TrowbridgeReitz(alphaX, alphaY), 1, e): rough glass
       GEN_LOBES = 6, GEN_NON_SPECULAR = GEN_LAMBERT | GEN_MICROFACET | GEN_MICRO_TRANSMISSION };

PB2_HD V3 clampSpectrum(const float c[3]) {  // Spectrum::Clamp(0, Infinity), spectrum.h:126-132
    return mk3(clampf(c[0], 0.f, PB2_INFINITY), clampf(c[1], 0.f, PB2_INFINITY), clampf(c[2], 0.f, PB2_INFINITY));
}

// TrowbridgeReitzDistribution::RoughnessToAlpha (microfacet.h:127-132)
PB2_HD float roughnessToAlpha(float roughness) {
    roughness = pmax(roughness, (float)1e-3);
    float x = plogf(roughness);
    return 1.62142f + 0.819955f * x + 0.1734f * x * x + 0.0171201f * x * x * x + 0.000640711f * x * x * x * x;
}

// The textured parameters of a material at one shaded point: every slot of pb2_material::tex that names a texture is
// evaluated (Texture::Evaluate(*si), e.g. matte.cpp:53-54) and written over the constant.
PB2_HDN void applyTextures(const DScene &sc, V2 uv, const DUvDiff &d, pb2_material *mat) {
    for (int k = 0; k < PB2_TEX_SLOTS; ++k) {
        const int id = mat->tex[k];
        if (!id) continue;
        const V3 v = texEvaluateNode(sc.textures, sc.texels, id - 1, uv, d);
        float *dst3 = nullptr;
        switch (k) {
        case PB2_TEX_KD: dst3 = mat->kd; break;
        case PB2_TEX_KS: dst3 = mat->ks; break;
        case PB2_TEX_KR: dst3 = mat->kr; break;
        case PB2_TEX_KT: dst3 = mat->kt; break;
        case PB2_TEX_OPACITY: dst3 = mat->opacity; break;
        case PB2_TEX_METAL_ETA: dst3 = mat->metal_eta; break;
        case PB2_TEX_METAL_K: dst3 = mat->metal_k; break;
        case PB2_TEX_SIGMA: mat->sigma = v.x; break;
        case PB2_TEX_ROUGHNESS: mat->roughness = v.x; break;
        case PB2_TEX_UROUGHNESS: mat->uroughness = v.x; break;
        case PB2_TEX_VROUGHNESS: mat->vroughness = v.x; break;
        case PB2_TEX_ETA: mat->eta = v.x; break;
        }
        if (dst3) {
            dst3[0] = v.x;
            dst3[1] = v.y;
            dst3[2] = v.z;
        }
    }
}

// Material::Bump (material.cpp:45-82): the displacement texture evaluated at (u, v), (u + du, v) and (u, v + dv) tilts the
// shading frame.  Only what an ImageTexture with a UVMapping2D reads is shifted (uv; the look-ups share the point's
// differentials); the new shading normal is flipped to the side of the geometric one (SetShadingGeometry with
// orientationIsAuthoritative = false).
PB2_HDN void bumpShading(const DScene &sc, int tex, const DTexGeom &tg, const DUvDiff &d, DInteraction *it) {
    float du = .5f * (fabsf(d.dudx) + fabsf(d.dudy));
    if (du == 0) du = .0005f;
    const float uDisplace = texEvaluateNode(sc.textures, sc.texels, tex, mk2(it->uv.x + du, it->uv.y + 0.f), d).x;
    float dv = .5f * (fabsf(d.dvdx) + fabsf(d.dvdy));
    if (dv == 0) dv = .0005f;
    const float vDisplace = texEvaluateNode(sc.textures, sc.texels, tex, mk2(it->uv.x + 0.f, it->uv.y + dv), d).x;
    const float displace = texEvaluateNode(sc.textures, sc.texels, tex, it->uv, d).x;
    const V3 dpdu = it->dpdus + ((uDisplace - displace) / du) * it->ns + displace * tg.dndus;
    const V3 dpdv = tg.dpdvs + ((vDisplace - displace) / dv) * it->ns + displace * tg.dndvs;
    it->ns = faceforward(normalize(cross(dpdu, dpdv)), it->n);
    it->dpdus = dpdu;
}

// Material::ComputeScatteringFunctions for matte (matte.cpp:45-62) and plastic (plastic.cpp:45-70).
// Returns false when the primitive has no material (null BSDF: the path skips the surface).
// uvDiff: the point's (u, v) differentials, which image textures are evaluated with.
template <int F>
PB2_HD bool makeBsdf(const DScene &sc, const DInteraction &it, DBsdf *bsdf, const DUvDiff *uvDiff = nullptr) {
    int m = sc.primMaterial[it.prim];
    if (m < 0) return false;
    pb2_material mat = sc.materials[m];
    if (mat.type == PB2_MAT_NONE) return false;
    if ((F & SHADE_TEXTURES) && sc.textures && uvDiff) applyTextures(sc, it.uv, *uvDiff, &mat);
    bsdf->ns = it.ns;
    bsdf->ng = it.n;
    bsdf->ss = normalize(it.dpdus);
    bsdf->ts = cross(bsdf->ns, bsdf->ss);
    bsdf->nLobes = 0;
    bsdf->diffuseKind = 0;
    bsdf->hasMicrofacet = 0;
    bsdf->R = mk3(0, 0, 0);
    bsdf->Ks = mk3(0, 0, 0);
    bsdf->A = bsdf->B = 0;
    bsdf->alpha = 0;
    bsdf->specKind = 0;
    bsdf->specR = bsdf->specT = mk3(0, 0, 0);
    bsdf->eta = 1;
    bsdf->blend = 0;
    bsdf->alphaX = bsdf->alphaY = 0;
    bsdf->general = 0;
    bsdf->conductor = 0;
    bsdf->T0 = bsdf->condEta = bsdf->condK = mk3(0, 0, 0);
    bsdf->e = 1;
    if ((F & SHADE_SPECULAR) && mat.type == PB2_MAT_METAL) {
        // metal.cpp:60-80: one MicrofacetReflection(1, TrowbridgeReitz(uRough, vRough), FresnelConductor(1, eta, k))
        float uRough = mat.uroughness, vRough = mat.vroughness;
        if (mat.remap_roughness) {
            uRough = roughnessToAlpha(uRough);
            vRough = roughnessToAlpha(vRough);
        }
        bsdf->Ks = mk3(1, 1, 1);
        bsdf->alphaX = pmax(0.001f, uRough);
        bsdf->alphaY = pmax(0.001f, vRough);
        bsdf->conductor = 1;
        bsdf->condEta = mk3(mat.metal_eta[0], mat.metal_eta[1], mat.metal_eta[2]);
        bsdf->condK = mk3(mat.metal_k[0], mat.metal_k[1], mat.metal_k[2]);
        bsdf->general = GEN_MICROFACET;
        bsdf->nLobes = 1;
        return true;
    }
    if ((F & SHADE_SPECULAR) && mat.type == PB2_MAT_UBER) {
        // uber.cpp:45-104
        const float e = mat.eta;
        V3 op = clampSpectrum(mat.opacity);
        V3 t = mk3(clampf(-op.x + 1.f, 0.f, PB2_INFINITY), clampf(-op.y + 1.f, 0.f, PB2_INFINITY), clampf(-op.z + 1.f, 0.f, PB2_INFINITY));
        bsdf->e = e;
        if (!isBlack(t)) {
            bsdf->T0 = t;
            bsdf->general |= GEN_OPACITY;
        } else
            bsdf->eta = e;
        V3 kd = op * clampSpectrum(mat.kd);
        if (!isBlack(kd)) {
            bsdf->R = kd;
            bsdf->diffuseKind = 1;
            bsdf->general |= GEN_LAMBERT;
            bsdf->nLobes++;
        }
        V3 ks = op * clampSpectrum(mat.ks);
        if (!isBlack(ks)) {
            float roughu = mat.uroughness, roughv = mat.vroughness;
            if (mat.remap_roughness) {
                roughu = roughnessToAlpha(roughu);
                roughv = roughnessToAlpha(roughv);
            }
            bsdf->Ks = ks;
            bsdf->alphaX = pmax(0.001f, roughu);
            bsdf->alphaY = pmax(0.001f, roughv);
            bsdf->general |= GEN_MICROFACET;
            bsdf->nLobes++;
        }
        V3 kr = op * clampSpectrum(mat.kr);
        if (!isBlack(kr)) {
            bsdf->specR = kr;
            bsdf->general |= GEN_SPEC_REFLECTION;
        }
        V3 kt = op * clampSpectrum(mat.kt);
        if (!isBlack(kt)) {
            bsdf->specT = kt;
            bsdf->general |= GEN_SPEC_TRANSMISSION;
        }
        return true;
    }
    if ((F & SHADE_SPECULAR) && mat.type == PB2_MAT_SUBSTRATE) {
        // substrate.cpp:45-65
        V3 d = clampSpectrum(mat.kd), sp = clampSpectrum(mat.ks);
        if (!isBlack(d) || !isBlack(sp)) {
            float roughu = mat.uroughness, roughv = mat.vroughness;
            if (mat.remap_roughness) {
                roughu = roughnessToAlpha(roughu);
                roughv = roughnessToAlpha(roughv);
            }
            bsdf->R = d;
            bsdf->Ks = sp;
            bsdf->alphaX = pmax(0.001f, roughu);
            bsdf->alphaY = pmax(0.001f, roughv);
            bsdf->blend = 1;
            bsdf->nLobes = 1;
        }
        return true;
    }
    if ((F & SHADE_SPECULAR) && mat.type == PB2_MAT_MIRROR) {
        // mirror.cpp:45-58
        V3 r = clampSpectrum(mat.kr);
        if (!isBlack(r)) {
            bsdf->specKind = 1;
            bsdf->specR = r;
        }
        return true;
    }
    if ((F & SHADE_SPECULAR) && mat.type == PB2_MAT_GLASS && !(mat.uroughness == 0 && mat.vroughness == 0)) {
        // glass.cpp:45-93, rough: MicrofacetReflection(R, distrib, FresnelDielectric(1, eta)) + MicrofacetTransmission(T, distrib, 1, eta)
        V3 r = clampSpectrum(mat.kr), t = clampSpectrum(mat.kt);
        bsdf->eta = mat.eta;
        bsdf->e = mat.eta;
        if (isBlack(r) && isBlack(t)) return true;
        float urough = mat.uroughness, vrough = mat.vroughness;
        if (mat.remap_roughness) {
            urough = roughnessToAlpha(urough);
            vrough = roughnessToAlpha(vrough);
        }
        bsdf->alphaX = pmax(0.001f, urough);
        bsdf->alphaY = pmax(0.001f, vrough);
        if (!isBlack(r)) {
            bsdf->Ks = r;
            bsdf->general |= GEN_MICROFACET;
            bsdf->nLobes++;
        }
        if (!isBlack(t)) {
            bsdf->specT = t;
            bsdf->general |= GEN_MICRO_TRANSMISSION;
            bsdf->nLobes++;
        }
        return true;
    }
    if ((F & SHADE_SPECULAR) && mat.type == PB2_MAT_GLASS) {
        // glass.cpp:45-68 with urough == vrough == 0 and allowMultipleLobes (path.cpp:106): one FresnelSpecular
        V3 r = clampSpectrum(mat.kr), t = clampSpectrum(mat.kt);
        bsdf->eta = mat.eta;
        if (!(isBlack(r) && isBlack(t))) {
            bsdf->specKind = 2;
            bsdf->specR = r;
            bsdf->specT = t;
        }
        return true;
    }
    V3 kd = clampSpectrum(mat.kd);
    if (mat.type == PB2_MAT_MATTE) {
        float sig = clampf(mat.sigma, 0.f, 90.f);
        if (!isBlack(kd)) {
            bsdf->R = kd;
            if (!(F & SHADE_OREN_NAYAR) || sig == 0)
                bsdf->diffuseKind = 1;
            else {
                bsdf->diffuseKind = 2;
                float sigma = (kPi / 180) * sig;  // Radians()
                float sigma2 = sigma * sigma;
                bsdf->A = 1.f - (sigma2 / (2.f * (sigma2 + 0.33f)));
                bsdf->B = 0.45f * sigma2 / (sigma2 + 0.09f);
            }
            bsdf->nLobes = 1;
        }
    } else {
        if (!isBlack(kd)) {
            bsdf->R = kd;
            bsdf->diffuseKind = 1;
            bsdf->nLobes++;
        }
        V3 ks = clampSpectrum(mat.ks);
        if ((F & SHADE_MICROFACET) && !isBlack(ks)) {
            float rough = mat.roughness;
            if (mat.remap_roughness) rough = roughnessToAlpha(rough);
            bsdf->Ks = ks;
            bsdf->alpha = pmax(0.001f, rough);  // microfacet.h:109-113
            bsdf->hasMicrofacet = 1;
            bsdf->nLobes++;
        }
    }
    return true;
}

PB2_HD V3 worldToLocal(const DBsdf &b, V3 v) { return mk3(dot(v, b.ss), dot(v, b.ts), dot(v, b.ns)); }
PB2_HD V3 localToWorld(const DBsdf &b, V3 v) {
    return mk3(b.ss.x * v.x + b.ts.x * v.y + b.ns.x * v.z, b.ss.y * v.x + b.ts.y * v.y + b.ns.y * v.z,
               b.ss.z * v.x + b.ts.z * v.y + b.ns.z * v.z);
}

// reflection.h:55-86
PB2_HD float cosTheta(V3 w) { return w.z; }
PB2_HD float cos2Theta(V3 w) { return w.z * w.z; }
PB2_HD float absCosTheta(V3 w) { return fabsf(w.z); }
PB2_HD float sin2Theta(V3 w) { return pmax(0.f, 1.f - cos2Theta(w)); }
PB2_HD float sinTheta(V3 w) { return sqrtf(sin2Theta(w)); }
PB2_HD float tanTheta(V3 w) { return sinTheta(w) / cosTheta(w); }
PB2_HD float tan2Theta(V3 w) { return sin2Theta(w) / cos2Theta(w); }
PB2_HD float cosPhi(V3 w) { float s = sinTheta(w); return (s == 0) ? 1 : clampf(w.x / s, -1.f, 1.f); }
PB2_HD float sinPhi(V3 w) { float s = sinTheta(w); return (s == 0) ? 0 : clampf(w.y / s, -1.f, 1.f); }
PB2_HD float cos2Phi(V3 w) { return cosPhi(w) * cosPhi(w); }
PB2_HD float sin2Phi(V3 w) { return sinPhi(w) * sinPhi(w); }
PB2_HD bool sameHemisphere(V3 w, V3 wp) { return w.z * wp.z > 0; }

// FrDielectric(cosThetaI, 1.5, 1) (reflection.cpp:47-68)
PB2_HD float frDielectric(float cosThetaI, float etaI, float etaT) {
    cosThetaI = clampf(cosThetaI, -1.f, 1.f);
    bool entering = cosThetaI > 0.f;
    if (!entering) {
        float t = etaI; etaI = etaT; etaT = t;
        cosThetaI = fabsf(cosThetaI);
    }
    float sinThetaI = sqrtf(pmax(0.f, 1 - cosThetaI * cosThetaI));
    float sinThetaT = etaI / etaT * sinThetaI;
    if (sinThetaT >= 1) return 1;
    float cosThetaT = sqrtf(pmax(0.f, 1 - sinThetaT * sinThetaT));
    float Rparl = ((etaT * cosThetaI) - (etaI * cosThetaT)) / ((etaT * cosThetaI) + (etaI * cosThetaT));
    float Rperp = ((etaI * cosThetaI) - (etaT * cosThetaT)) / ((etaI * cosThetaI) + (etaT * cosThetaT));
    return (Rparl * Rparl + Rperp * Rperp) / 2;
}

// TrowbridgeReitzDistribution (microfacet.cpp:155-184, 338-344)
PB2_HD float trD(float alpha, V3 wh) {
    float t2 = tan2Theta(wh);
    if (isinf(t2)) return 0.;
    const float cos4Theta = cos2Theta(wh) * cos2Theta(wh);
    float e = (cos2Phi(wh) / (alpha * alpha) + sin2Phi(wh) / (alpha * alpha)) * t2;
    return 1 / (kPi * alpha * alpha * cos4Theta * (1 + e) * (1 + e));
}
PB2_HD float trLambda(float alpha, V3 w) {
    float absTanTheta = fabsf(tanTheta(w));
    if (isinf(absTanTheta)) return 0.;
    float a = sqrtf(cos2Phi(w) * alpha * alpha + sin2Phi(w) * alpha * alpha);
    float alpha2Tan2Theta = (a * absTanTheta) * (a * absTanTheta);
    return (-1 + sqrtf(1.f + alpha2Tan2Theta)) / 2;
}
PB2_HD float trG1(float alpha, V3 w) { return 1 / (1 + trLambda(alpha, w)); }
PB2_HD float trG(float alpha, V3 wo, V3 wi) { return 1 / (1 + trLambda(alpha, wo) + trLambda(alpha, wi)); }
PB2_HD float trPdf(float alpha, V3 wo, V3 wh) {  // sampleVisibleArea == true
    return trD(alpha, wh) * trG1(alpha, wo) * absDot(wo, wh) / absCosTheta(wo);
}

// TrowbridgeReitzSample11 (microfacet.cpp:238-282).  The normal-incidence branch runs in double,
// as the reference's unqualified sqrt/cos/sin do.
PB2_HDN void trSample11(float cosThetaV, float U1, float U2, float *slope_x, float *slope_y) {
    if ((double)cosThetaV > .9999) {
        float r = (float)sqrt((double)(U1 / (1 - U1)));
        float phi = (float)(6.28318530718 * (double)U2);
        double sPhi, cPhi;
        sincos((double)phi, &sPhi, &cPhi);
        *slope_x = (float)((double)r * cPhi);
        *slope_y = (float)((double)r * sPhi);
        return;
    }
    float sinThetaV = sqrtf(pmax(0.f, 1.f - cosThetaV * cosThetaV));
    float tanThetaV = sinThetaV / cosThetaV;
    float a = 1 / tanThetaV;
    float G1 = 2 / (1 + sqrtf(1.f + 1.f / (a * a)));
    float A = 2 * U1 / G1 - 1;
    float tmp = 1.f / (A * A - 1.f);
    if (tmp > 1e10) tmp = 1e10;
    float B = tanThetaV;
    float D = sqrtf(pmax((float)(B * B * tmp * tmp - (A * A - B * B) * tmp), 0.f));
    float slope_x_1 = B * tmp - D;
    float slope_x_2 = B * tmp + D;
    *slope_x = (A < 0 || slope_x_2 > 1.f / tanThetaV) ? slope_x_1 : slope_x_2;
    float S;
    if (U2 > 0.5f) {
        S = 1.f;
        U2 = 2.f * (U2 - .5f);
    } else {
        S = -1.f;
        U2 = 2.f * (.5f - U2);
    }
    float z = (U2 * (U2 * (U2 * 0.27385f - 0.73369f) + 0.46341f)) /
              (U2 * (U2 * (U2 * 0.093073f + 0.309420f) - 1.000000f) + 0.597999f);
    *slope_y = S * z * sqrtf(1.f + *slope_x * *slope_x);
}
// TrowbridgeReitzSample + Sample_wh, visible-area branch (microfacet.cpp:284-336)
PB2_HD V3 trSampleWh(float alpha, V3 wo, V2 u) {
    bool flip = wo.z < 0;
    V3 wi = flip ? -wo : wo;
    V3 wiStretched = normalize(mk3(alpha * wi.x, alpha * wi.y, wi.z));
    float slope_x, slope_y;
    trSample11(cosTheta(wiStretched), u.x, u.y, &slope_x, &slope_y);
    float tmp = cosPhi(wiStretched) * slope_x - sinPhi(wiStretched) * slope_y;
    slope_y = sinPhi(wiStretched) * slope_x + cosPhi(wiStretched) * slope_y;
    slope_x = tmp;
    slope_x = alpha * slope_x;
    slope_y = alpha * slope_y;
    V3 wh = normalize(mk3(-slope_x, -slope_y, 1.f));
    if (flip) wh = -wh;
    return wh;
}

// The same distribution with alphax != alphay (microfacet.cpp:155-184, 284-344), used by FresnelBlend
PB2_HD float trD2(float ax, float ay, V3 wh) {
    float t2 = tan2Theta(wh);
    if (isinf(t2)) return 0.;
    const float cos4Theta = cos2Theta(wh) * cos2Theta(wh);
    float e = (cos2Phi(wh) / (ax * ax) + sin2Phi(wh) / (ay * ay)) * t2;
    return 1 / (kPi * ax * ay * cos4Theta * (1 + e) * (1 + e));
}
PB2_HD float trLambda2(float ax, float ay, V3 w) {
    float absTanTheta = fabsf(tanTheta(w));
    if (isinf(absTanTheta)) return 0.;
    float a = sqrtf(cos2Phi(w) * ax * ax + sin2Phi(w) * ay * ay);
    float alpha2Tan2Theta = (a * absTanTheta) * (a * absTanTheta);
    return (-1 + sqrtf(1.f + alpha2Tan2Theta)) / 2;
}
PB2_HD float trPdf2(float ax, float ay, V3 wo, V3 wh) {
    return trD2(ax, ay, wh) * (1 / (1 + trLambda2(ax, ay, wo))) * absDot(wo, wh) / absCosTheta(wo);
}
PB2_HD V3 trSampleWh2(float ax, float ay, V3 wo, V2 u) {
    bool flip = wo.z < 0;
    V3 wi = flip ? -wo : wo;
    V3 wiStretched = normalize(mk3(ax * wi.x, ay * wi.y, wi.z));
    float slope_x, slope_y;
    trSample11(cosTheta(wiStretched), u.x, u.y, &slope_x, &slope_y);
    float tmp = cosPhi(wiStretched) * slope_x - sinPhi(wiStretched) * slope_y;
    slope_y = sinPhi(wiStretched) * slope_x + cosPhi(wiStretched) * slope_y;
    slope_x = tmp;
    slope_x = ax * slope_x;
    slope_y = ay * slope_y;
    V3 wh = normalize(mk3(-slope_x, -slope_y, 1.f));
    if (flip) wh = -wh;
    return wh;
}
// FresnelBlend::f / Pdf (reflection.cpp:290-303, 480-485)
PB2_HD float pow5f(float v) { return (v * v) * (v * v) * v; }
PB2_HD V3 blendF(const DBsdf &b, V3 wo, V3 wi) {
    V3 one = mk3(1, 1, 1);
    V3 diffuse = (28.f / (23.f * kPi)) * b.R * (one - b.Ks) * (1 - pow5f(1 - .5f * absCosTheta(wi))) * (1 - pow5f(1 - .5f * absCosTheta(wo)));
    V3 wh = wi + wo;
    if (wh.x == 0 && wh.y == 0 && wh.z == 0) return mk3(0, 0, 0);
    wh = normalize(wh);
    float cosT = dot(wi, wh);
    V3 schlick = b.Ks + pow5f(1 - cosT) * (one - b.Ks);
    V3 specular = (trD2(b.alphaX, b.alphaY, wh) / (4 * absDot(wi, wh) * pmax(absCosTheta(wi), absCosTheta(wo)))) * schlick;
    return diffuse + specular;
}
PB2_HD float blendPdf(const DBsdf &b, V3 wo, V3 wi) {
    if (!sameHemisphere(wo, wi)) return 0;
    V3 wh = normalize(wo + wi);
    float pdf_wh = trPdf2(b.alphaX, b.alphaY, wo, wh);
    return .5f * (absCosTheta(wi) * kInvPi + pdf_wh / (4 * dot(wo, wh)));
}

// individual BxDFs (local frame)
template <int F>
PB2_HD V3 diffuseF(const DBsdf &b, V3 wo, V3 wi) {
    if (!(F & SHADE_OREN_NAYAR) || b.diffuseKind == 1) return b.R * kInvPi;
    // OrenNayar::f (reflection.cpp:197-219)
    float sinThetaI = sinTheta(wi), sinThetaO = sinTheta(wo);
    float maxCos = 0;
    if ((double)sinThetaI > 1e-4 && (double)sinThetaO > 1e-4) {
        float sinPhiI = sinPhi(wi), cosPhiI = cosPhi(wi);
        float sinPhiO = sinPhi(wo), cosPhiO = cosPhi(wo);
        float dCos = cosPhiI * cosPhiO + sinPhiI * sinPhiO;
        maxCos = pmax(0.f, dCos);
    }
    float sinAlpha, tanBeta;
    if (absCosTheta(wi) > absCosTheta(wo)) {
        sinAlpha = sinThetaO;
        tanBeta = sinThetaI / absCosTheta(wi);
    } else {
        sinAlpha = sinThetaI;
        tanBeta = sinThetaO / absCosTheta(wo);
    }
    return b.R * kInvPi * (b.A + b.B * maxCos * sinAlpha * tanBeta);
}
PB2_HD float diffusePdf(V3 wo, V3 wi) { return sameHemisphere(wo, wi) ? absCosTheta(wi) * kInvPi : 0; }

// MicrofacetReflection::f (reflection.cpp:226-238) with FresnelDielectric(1.5, 1)
PB2_HD V3 microfacetF(const DBsdf &b, V3 wo, V3 wi) {
    float cosThetaO = absCosTheta(wo), cosThetaI = absCosTheta(wi);
    V3 wh = wi + wo;
    if (cosThetaI == 0 || cosThetaO == 0) return mk3(0, 0, 0);
    if (wh.x == 0 && wh.y == 0 && wh.z == 0) return mk3(0, 0, 0);
    wh = normalize(wh);
    float F = frDielectric(dot(wi, faceforward(wh, mk3(0, 0, 1))), 1.5f, 1.f);
    // R * D * G * F / (4 cosI cosO): Spectrum*float products left to right, then one division
    V3 num = b.Ks * trD(b.alpha, wh) * trG(b.alpha, wo, wi) * mk3(F, F, F);
    float den = (4 * cosThetaI * cosThetaO);
    return mk3(num.x / den, num.y / den, num.z / den);
}
PB2_HD float microfacetPdf(const DBsdf &b, V3 wo, V3 wi) {
    if (!sameHemisphere(wo, wi)) return 0;
    V3 wh = normalize(wo + wi);
    return trPdf(b.alpha, wo, wh) / (4 * dot(wo, wh));
}

// FrConductor (reflection.cpp:71-95): the Spectrum arithmetic per channel, in the reference's order.
PB2_HD float frConductor1(float cosThetaI, float cosThetaI2, float sinThetaI2, float etat, float k) {
    float eta = etat / 1.f, etak = k / 1.f;   // etai == 1 (metal.cpp:75)
    float eta2 = eta * eta, etak2 = etak * etak;
    float t0 = eta2 - etak2 - sinThetaI2;
    float a2plusb2 = sqrtf(t0 * t0 + 4 * eta2 * etak2);
    float t1 = a2plusb2 + cosThetaI2;
    float a = sqrtf(0.5f * (a2plusb2 + t0));
    float t2 = (2 * cosThetaI) * a;
    float Rs = (t1 - t2) / (t1 + t2);
    float t3 = cosThetaI2 * a2plusb2 + sinThetaI2 * sinThetaI2;
    float t4 = t2 * sinThetaI2;
    float Rp = Rs * (t3 - t4) / (t3 + t4);
    return 0.5f * (Rp + Rs);
}
PB2_HD V3 frConductor(float cosThetaI, V3 etat, V3 k) {
    cosThetaI = clampf(cosThetaI, -1.f, 1.f);
    float cosThetaI2 = cosThetaI * cosThetaI;
    float sinThetaI2 = (float)(1. - (double)cosThetaI2);
    return mk3(frConductor1(cosThetaI, cosThetaI2, sinThetaI2, etat.x, k.x), frConductor1(cosThetaI, cosThetaI2, sinThetaI2, etat.y, k.y),
               frConductor1(cosThetaI, cosThetaI2, sinThetaI2, etat.z, k.z));
}
// MicrofacetReflection::f / Pdf (reflection.cpp:226-238, 425-429) over TrowbridgeReitz(alphaX, alphaY) with the
// lobe's own Fresnel term
PB2_HD V3 microfacetFGen(const DBsdf &b, V3 wo, V3 wi) {
    float cosThetaO = absCosTheta(wo), cosThetaI = absCosTheta(wi);
    V3 wh = wi + wo;
    if (cosThetaI == 0 || cosThetaO == 0) return mk3(0, 0, 0);
    if (wh.x == 0 && wh.y == 0 && wh.z == 0) return mk3(0, 0, 0);
    wh = normalize(wh);
    float c = dot(wi, faceforward(wh, mk3(0, 0, 1)));
    V3 F;
    if (b.conductor) F = frConductor(fabsf(c), b.condEta, b.condK);
    else {
        float Fd = frDielectric(c, 1.f, b.e);
        F = mk3(Fd, Fd, Fd);
    }
    float G = 1 / (1 + trLambda2(b.alphaX, b.alphaY, wo) + trLambda2(b.alphaX, b.alphaY, wi));
    V3 num = b.Ks * trD2(b.alphaX, b.alphaY, wh) * G * F;
    float den = (4 * cosThetaI * cosThetaO);
    return mk3(num.x / den, num.y / den, num.z / den);
}
PB2_HD float microfacetPdfGen(const DBsdf &b, V3 wo, V3 wi) {
    if (!sameHemisphere(wo, wi)) return 0;
    V3 wh = normalize(wo + wi);
    return trPdf2(b.alphaX, b.alphaY, wo, wh) / (4 * dot(wo, wh));
}
// MicrofacetTransmission::f / Pdf (reflection.cpp:246-270, 444-458), etaA = 1, etaB = e, TransportMode::Radiance
PB2_HD V3 microTransF(const DBsdf &b, V3 wo, V3 wi) {
    if (sameHemisphere(wo, wi)) return mk3(0, 0, 0);
    float cosThetaO = cosTheta(wo), cosThetaI = cosTheta(wi);
    if (cosThetaI == 0 || cosThetaO == 0) return mk3(0, 0, 0);
    float eta = cosTheta(wo) > 0 ? (b.e / 1.f) : (1.f / b.e);
    V3 wh = normalize(wo + wi * eta);
    if (wh.z < 0) wh = -wh;
    if (dot(wo, wh) * dot(wi, wh) > 0) return mk3(0, 0, 0);
    float F = frDielectric(dot(wo, wh), 1.f, b.e);
    float sqrtDenom = dot(wo, wh) + eta * dot(wi, wh);
    float factor = 1 / eta;
    float G = 1 / (1 + trLambda2(b.alphaX, b.alphaY, wo) + trLambda2(b.alphaX, b.alphaY, wi));
    float v = fabsf(trD2(b.alphaX, b.alphaY, wh) * G * eta * eta * absDot(wi, wh) * absDot(wo, wh) * factor * factor /
                    (cosThetaI * cosThetaO * sqrtDenom * sqrtDenom));
    return mk3(1.f - F, 1.f - F, 1.f - F) * b.specT * v;
}
PB2_HD float microTransPdf(const DBsdf &b, V3 wo, V3 wi) {
    if (sameHemisphere(wo, wi)) return 0;
    float eta = cosTheta(wo) > 0 ? (b.e / 1.f) : (1.f / b.e);
    V3 wh = normalize(wo + wi * eta);
    if (dot(wo, wh) * dot(wi, wh) > 0) return 0;
    float sqrtDenom = dot(wo, wh) + eta * dot(wi, wh);
    float dwh_dwi = fabsf((eta * eta * dot(wi, wh)) / (sqrtDenom * sqrtDenom));
    return trPdf2(b.alphaX, b.alphaY, wo, wh) * dwh_dwi;
}
// BSDF::f over the lobe list (reflection.cpp:680-693): reflective lobes when wi and wo are on the same side of the
// geometric normal, transmissive ones otherwise; the specular lobes return 0
PB2_HD V3 genF(const DBsdf &b, V3 wo, V3 wi, bool reflect) {
    V3 f = mk3(0, 0, 0);
    if (reflect) {
        if (b.general & GEN_LAMBERT) f = f + b.R * kInvPi;
        if (b.general & GEN_MICROFACET) f = f + microfacetFGen(b, wo, wi);
    } else if (b.general & GEN_MICRO_TRANSMISSION)
        f = f + microTransF(b, wo, wi);
    return f;
}

// BSDF::f (reflection.cpp:680-693).  All lobes in scope are reflective and non-specular, so they
// match both BSDF_ALL and BSDF_ALL & ~BSDF_SPECULAR.
template <int F>
PB2_HD V3 bsdfF(const DBsdf &b, V3 woW, V3 wiW) {
    V3 wi = worldToLocal(b, wiW), wo = worldToLocal(b, woW);
    if (wo.z == 0) return mk3(0, 0, 0);
    bool reflect = dot(wiW, b.ng) * dot(woW, b.ng) > 0;
    V3 f = mk3(0, 0, 0);
    if ((F & SHADE_SPECULAR) && b.blend) return reflect ? blendF(b, wo, wi) : f;
    if ((F & SHADE_SPECULAR) && b.general) return genF(b, wo, wi, reflect);
    if (reflect) {
        if (b.diffuseKind) f = f + diffuseF<F>(b, wo, wi);
        if ((F & SHADE_MICROFACET) && b.hasMicrofacet) f = f + microfacetF(b, wo, wi);
    }
    return f;
}
// BSDF::Pdf (reflection.cpp:781-796)
template <int F>
PB2_HD float bsdfPdf(const DBsdf &b, V3 woW, V3 wiW) {
    if (b.nLobes == 0) return 0.f;
    V3 wo = worldToLocal(b, woW), wi = worldToLocal(b, wiW);
    if (wo.z == 0) return 0.;
    if ((F & SHADE_SPECULAR) && b.blend) return blendPdf(b, wo, wi);
    if ((F & SHADE_SPECULAR) && b.general) {
        // the callers ask with BSDF_ALL & ~BSDF_SPECULAR (integrator.cpp:134): matchingComps == nLobes
        float pdf = 0.f;
        if (b.general & GEN_LAMBERT) pdf += diffusePdf(wo, wi);
        if (b.general & GEN_MICROFACET) pdf += microfacetPdfGen(b, wo, wi);
        if (b.general & GEN_MICRO_TRANSMISSION) pdf += microTransPdf(b, wo, wi);
        return pdf / b.nLobes;
    }
    float pdf = 0.f;
    if (b.diffuseKind) pdf += diffusePdf(wo, wi);
    if ((F & SHADE_MICROFACET) && b.hasMicrofacet) pdf += microfacetPdf(b, wo, wi);
    return pdf / b.nLobes;
}
// BSDF::Sample_f (reflection.cpp:714-779).  Returns f; *pdf == 0 means no sample.
// Refract (reflection.h:97-109)
PB2_HD bool refract(V3 wi, V3 n, float eta, V3 *wt) {
    float cosThetaI = dot(n, wi);
    float sin2ThetaI = pmax(0.f, 1 - cosThetaI * cosThetaI);
    float sin2ThetaT = eta * eta * sin2ThetaI;
    if (sin2ThetaT >= 1) return false;
    float cosThetaT = sqrtf(1 - sin2ThetaT);
    *wt = eta * (-wi) + (eta * cosThetaI - cosThetaT) * n;
    return true;
}

// BSDF::Sample_f (reflection.cpp:714-779) over a lobe list.  nonSpecularOnly: the `type` argument is
// BSDF_ALL & ~BSDF_SPECULAR (EstimateDirect, integrator.cpp:165) instead of BSDF_ALL (path.cpp:133).
PB2_HDN V3 genSampleF(const DBsdf &b, V3 woW, V3 *wiW, V2 u, float *pdf, int *sampledFlags, bool nonSpecularOnly) {
    const int mask = nonSpecularOnly ? (b.general & GEN_NON_SPECULAR) : b.general;
    int matching = 0;
    for (int i = 0; i < GEN_LOBES; ++i) matching += (mask >> i) & 1;
    if (matching == 0) return mk3(0, 0, 0);
    int comp = (int)floorf(u.x * matching);
    if (comp > matching - 1) comp = matching - 1;
    int lobe = 0, count = comp;
    for (int i = 0; i < GEN_LOBES; ++i)
        if ((mask >> i) & 1) {
            if (count-- == 0) {
                lobe = 1 << i;
                break;
            }
        }
    V2 uRemapped = mk2(pmin(u.x * matching - comp, kOneMinusEpsilon), u.y);
    V3 wo = worldToLocal(b, woW), wi = mk3(0, 0, 0);
    if (wo.z == 0) return mk3(0, 0, 0);
    V3 f = mk3(0, 0, 0);
    int flags = 0;
    if (lobe == GEN_LAMBERT) {
        wi = cosineSampleHemisphere(uRemapped);   // BxDF::Sample_f (reflection.cpp:383-390)
        if (wo.z < 0) wi.z *= -1;
        *pdf = diffusePdf(wo, wi);
    } else if (lobe == GEN_MICROFACET) {
        // MicrofacetReflection::Sample_f (reflection.cpp:410-423)
        V3 wh = trSampleWh2(b.alphaX, b.alphaY, wo, uRemapped);
        if (dot(wo, wh) < 0) return mk3(0, 0, 0);
        wi = -wo + 2 * dot(wo, wh) * wh;  // Reflect
        if (!sameHemisphere(wo, wi)) return mk3(0, 0, 0);
        *pdf = trPdf2(b.alphaX, b.alphaY, wo, wh) / (4 * dot(wo, wh));
    } else if (lobe == GEN_MICRO_TRANSMISSION) {
        // MicrofacetTransmission::Sample_f (reflection.cpp:431-442)
        V3 wh = trSampleWh2(b.alphaX, b.alphaY, wo, uRemapped);
        if (dot(wo, wh) < 0) return mk3(0, 0, 0);
        float eta = cosTheta(wo) > 0 ? (1.f / b.e) : (b.e / 1.f);
        if (!refract(wo, wh, eta, &wi)) return mk3(0, 0, 0);
        *pdf = microTransPdf(b, wo, wi);
        flags = BSDF_SAMPLED_TRANSMISSION;
    } else if (lobe == GEN_SPEC_REFLECTION) {
        // SpecularReflection::Sample_f with FresnelDielectric(1, e) (reflection.cpp:136-143)
        wi = mk3(-wo.x, -wo.y, wo.z);
        *pdf = 1;
        float F = frDielectric(cosTheta(wi), 1.f, b.e);
        V3 fr = mk3(F, F, F) * b.specR;
        f = mk3(fr.x / absCosTheta(wi), fr.y / absCosTheta(wi), fr.z / absCosTheta(wi));
        flags = BSDF_SAMPLED_SPECULAR;
    } else {
        // SpecularTransmission::Sample_f (reflection.cpp:151-166), TransportMode::Radiance
        const float etaA = 1.f, etaB = (lobe == GEN_OPACITY) ? 1.f : b.e;
        const V3 T = (lobe == GEN_OPACITY) ? b.T0 : b.specT;
        bool entering = cosTheta(wo) > 0;
        float etaI = entering ? etaA : etaB;
        float etaT = entering ? etaB : etaA;
        V3 nn = mk3(0, 0, 1);
        if (dot(nn, wo) < 0) nn = -nn;  // Faceforward
        if (!refract(wo, nn, etaI / etaT, &wi)) return mk3(0, 0, 0);
        *pdf = 1;
        float F = frDielectric(cosTheta(wi), etaA, etaB);
        V3 ft = T * mk3(1.f - F, 1.f - F, 1.f - F);
        ft = ft * ((etaI * etaI) / (etaT * etaT));
        f = mk3(ft.x / absCosTheta(wi), ft.y / absCosTheta(wi), ft.z / absCosTheta(wi));
        flags = BSDF_SAMPLED_SPECULAR | BSDF_SAMPLED_TRANSMISSION;
    }
    if (*pdf == 0) return mk3(0, 0, 0);
    *wiW = localToWorld(b, wi);
    const bool specular = (lobe & GEN_NON_SPECULAR) == 0;
    if (!specular && matching > 1) {
        // the other matching lobes' Pdf(); specular ones return 0 (reflection.cpp:758-761)
        if (lobe != GEN_LAMBERT && (mask & GEN_LAMBERT)) *pdf += diffusePdf(wo, wi);
        if (lobe != GEN_MICROFACET && (mask & GEN_MICROFACET)) *pdf += microfacetPdfGen(b, wo, wi);
        if (lobe != GEN_MICRO_TRANSMISSION && (mask & GEN_MICRO_TRANSMISSION)) *pdf += microTransPdf(b, wo, wi);
    }
    if (matching > 1) *pdf /= matching;
    if (!specular) {
        bool reflect = dot(*wiW, b.ng) * dot(woW, b.ng) > 0;
        f = genF(b, wo, wi, reflect);
    }
    if (sampledFlags) *sampledFlags = flags;
    return f;
}

// *sampledFlags (optional): BSDF_SAMPLED_* of the BxDF that was sampled.
template <int F>
PB2_HD V3 bsdfSampleF(const DBsdf &b, V3 woW, V3 *wiW, V2 u, float *pdf, int *sampledFlags = nullptr, bool nonSpecularOnly = false) {
    *pdf = 0;
    if (sampledFlags) *sampledFlags = 0;
    if ((F & SHADE_SPECULAR) && b.general) return genSampleF(b, woW, wiW, u, pdf, sampledFlags, nonSpecularOnly);
    if ((F & SHADE_SPECULAR) && b.specKind) {
        // the BSDF holds exactly one BxDF, a specular one: matchingComps == 1, u is handed through
        // (uRemapped[0] = min(u[0], OneMinusEpsilon)), no pdf averaging and no re-evaluation of f
        // (reflection.cpp:725-775)
        V3 wo = worldToLocal(b, woW), wi;
        if (wo.z == 0) return mk3(0, 0, 0);
        V3 f;
        int flags = BSDF_SAMPLED_SPECULAR;
        if (b.specKind == 1) {
            // SpecularReflection::Sample_f with FresnelNoOp (reflection.cpp:136-143)
            wi = mk3(-wo.x, -wo.y, wo.z);
            *pdf = 1;
            f = mk3(b.specR.x / absCosTheta(wi), b.specR.y / absCosTheta(wi), b.specR.z / absCosTheta(wi));
        } else {
            // FresnelSpecular::Sample_f (reflection.cpp:487-521), etaA = 1, etaB = eta, TransportMode::Radiance
            float u0 = pmin(u.x, kOneMinusEpsilon);
            float Fr = frDielectric(cosTheta(wo), 1.f, b.eta);
            if (u0 < Fr) {
                wi = mk3(-wo.x, -wo.y, wo.z);
                *pdf = Fr;
                V3 fr = Fr * b.specR;
                f = mk3(fr.x / absCosTheta(wi), fr.y / absCosTheta(wi), fr.z / absCosTheta(wi));
            } else {
                bool entering = cosTheta(wo) > 0;
                float etaI = entering ? 1.f : b.eta;
                float etaT = entering ? b.eta : 1.f;
                V3 nn = mk3(0, 0, 1);
                if (dot(nn, wo) < 0) nn = -nn;  // Faceforward
                if (!refract(wo, nn, etaI / etaT, &wi)) return mk3(0, 0, 0);
                V3 ft = b.specT * (1 - Fr);
                ft = ft * ((etaI * etaI) / (etaT * etaT));
                flags |= BSDF_SAMPLED_TRANSMISSION;
                *pdf = 1 - Fr;
                f = mk3(ft.x / absCosTheta(wi), ft.y / absCosTheta(wi), ft.z / absCosTheta(wi));
            }
        }
        if (*pdf == 0) return mk3(0, 0, 0);
        *wiW = localToWorld(b, wi);
        if (sampledFlags) *sampledFlags = flags;
        return f;
    }
    int matching = b.nLobes;
    if (matching == 0) return mk3(0, 0, 0);
    if ((F & SHADE_SPECULAR) && b.blend) {
        // one glossy BxDF: comp 0, uRemapped[0] = min(u[0], OneMinusEpsilon); FresnelBlend::Sample_f
        // (reflection.cpp:460-478); f is then re-evaluated by the BSDF (reflection.cpp:767-775)
        V3 wo = worldToLocal(b, woW), wi;
        if (wo.z == 0) return mk3(0, 0, 0);
        V2 uu = mk2(pmin(u.x, kOneMinusEpsilon), u.y);
        if ((double)uu.x < .5) {
            uu.x = pmin(2 * uu.x, kOneMinusEpsilon);
            wi = cosineSampleHemisphere(uu);
            if (wo.z < 0) wi.z *= -1;
        } else {
            uu.x = pmin(2 * (uu.x - .5f), kOneMinusEpsilon);
            V3 wh = trSampleWh2(b.alphaX, b.alphaY, wo, uu);
            wi = -wo + 2 * dot(wo, wh) * wh;  // Reflect
            if (!sameHemisphere(wo, wi)) return mk3(0, 0, 0);
        }
        *pdf = blendPdf(b, wo, wi);
        if (*pdf == 0) return mk3(0, 0, 0);
        *wiW = localToWorld(b, wi);
        bool reflect = dot(*wiW, b.ng) * dot(woW, b.ng) > 0;
        return reflect ? blendF(b, wo, wi) : mk3(0, 0, 0);
    }
    int comp = (int)floorf(u.x * matching);
    if (comp > matching - 1) comp = matching - 1;
    // lobe order: diffuse first, then microfacet (plastic.cpp:53-68)
    bool sampleMicro = (F & SHADE_MICROFACET) && b.hasMicrofacet && (comp == matching - 1) && !(b.diffuseKind && comp == 0);
    V2 uRemapped = mk2(pmin(u.x * matching - comp, kOneMinusEpsilon), u.y);
    V3 wo = worldToLocal(b, woW), wi;
    if (wo.z == 0) return mk3(0, 0, 0);
    V3 f;
    if (!sampleMicro) {
        // BxDF::Sample_f (reflection.cpp:383-390)
        wi = cosineSampleHemisphere(uRemapped);
        if (wo.z < 0) wi.z *= -1;
        *pdf = diffusePdf(wo, wi);
        f = diffuseF<F>(b, wo, wi);
    } else {
        // MicrofacetReflection::Sample_f (reflection.cpp:410-423); wo.z == 0 handled above
        V3 wh = trSampleWh(b.alpha, wo, uRemapped);
        if (dot(wo, wh) < 0) return mk3(0, 0, 0);
        wi = -wo + 2 * dot(wo, wh) * wh;  // Reflect
        if (!sameHemisphere(wo, wi)) return mk3(0, 0, 0);
        *pdf = trPdf(b.alpha, wo, wh) / (4 * dot(wo, wh));
        f = microfacetF(b, wo, wi);
    }
    if (*pdf == 0) return mk3(0, 0, 0);
    *wiW = localToWorld(b, wi);
    if ((F & SHADE_MICROFACET) && matching > 1) {   // (two lobes: plastic's)
        if (sampleMicro) *pdf += diffusePdf(wo, wi);
        else *pdf += microfacetPdf(b, wo, wi);
        *pdf /= matching;
    }
    // non-specular lobes: f is re-evaluated over all matching lobes (reflection.cpp:767-775)
    bool reflect = dot(*wiW, b.ng) * dot(woW, b.ng) > 0;
    f = mk3(0, 0, 0);
    if (reflect) {
        if (b.diffuseKind) f = f + diffuseF<F>(b, wo, wi);
        if ((F & SHADE_MICROFACET) && b.hasMicrofacet) f = f + microfacetF(b, wo, wi);
    }
    return f;
}

// ---------------------------------------------------------------- area lights
struct DLightSample {
    V3 p, pError, n;   // pShape
    V3 wi;
    V3 Li;
    float pdf;
    bool delta;        // IsDeltaLight(light.flags) (light.h:57-60)
};

// Triangle::Area (triangle.cpp:574-580)
PB2_HD float triangleArea(const TriVerts &t) { return (float)(0.5 * (double)length(cross(t.p1 - t.p0, t.p2 - t.p0))); }

// DiffuseAreaLight::L (diffuse.h:56-58)
PB2_HD V3 lightL(const pb2_light &l, V3 n, V3 w) {
    return (l.two_sided || dot(n, w) > 0) ? mk3(l.L[0], l.L[1], l.L[2]) : mk3(0, 0, 0);
}

// Sphere::Sample(u, pdf) (sphere.cpp:219-230): uniform over the whole sphere, area measure.
PB2_HD void sphereSampleArea(const pb2_sphere &s, V2 u, V3 *p, V3 *pError, V3 *n, float *pdf) {
    M44 o2w = loadM44(s.object_to_world), w2o = loadM44(s.world_to_object);
    V3 pObj = mk3(0, 0, 0) + s.radius * uniformSampleSphere(u);
    *n = normalize(xfNormalInv(w2o, pObj));
    if (s.reverse_orientation) *n = *n * -1.f;
    pObj = pObj * (s.radius / length(pObj));
    V3 pObjError = kGamma5 * vabs(pObj);
    *p = xfPointErrIn(o2w, pObj, pObjError, pError);
    *pdf = 1 / (s.phi_max * s.radius * (s.z_max - s.z_min));
}

// DiffuseAreaLight::Sample_Li over Sphere::Sample(ref, u, pdf) (sphere.cpp:232-301)
PB2_HDN DLightSample sampleSphereLight(const DScene &sc, const pb2_light &l, const DInteraction &ref, V2 u) {
    DLightSample ls;
    const pb2_sphere s = sc.spheres[sc.primIndex[l.prim]];
    M44 o2w = loadM44(s.object_to_world);
    V3 pCenter = xfPoint(o2w, mk3(0, 0, 0));
    V3 pOrigin = offsetRayOrigin(ref.p, ref.pError, ref.n, pCenter - ref.p);
    if (lengthSquared(pOrigin - pCenter) <= s.radius * s.radius) {
        sphereSampleArea(s, u, &ls.p, &ls.pError, &ls.n, &ls.pdf);
        V3 wi = ls.p - ref.p;
        if (lengthSquared(wi) == 0)
            ls.pdf = 0;
        else {
            wi = normalize(wi);
            ls.pdf *= lengthSquared(ref.p - ls.p) / absDot(ls.n, -wi);
        }
        if (isinf(ls.pdf)) ls.pdf = 0.f;
    } else {
        float dc = length(ref.p - pCenter);
        float invDc = 1 / dc;
        V3 wc = (pCenter - ref.p) * invDc;
        V3 wcX, wcY;
        coordinateSystem(wc, &wcX, &wcY);
        float sinThetaMax = s.radius * invDc;
        float sinThetaMax2 = sinThetaMax * sinThetaMax;
        float invSinThetaMax = 1 / sinThetaMax;
        float cosThetaMax = sqrtf(pmax(0.f, 1 - sinThetaMax2));
        float cosThetaV = (cosThetaMax - 1) * u.x + 1;
        float sinTheta2 = 1 - cosThetaV * cosThetaV;
        if (sinThetaMax2 < 0.00068523f) {
            sinTheta2 = sinThetaMax2 * u.x;
            cosThetaV = sqrtf(1 - sinTheta2);
        }
        float cosAlpha = sinTheta2 * invSinThetaMax +
                         cosThetaV * sqrtf(pmax(0.f, 1.f - sinTheta2 * invSinThetaMax * invSinThetaMax));
        float sinAlpha = sqrtf(pmax(0.f, 1.f - cosAlpha * cosAlpha));
        float phi = u.y * 2 * kPi;
        // SphericalDirection(sinAlpha, cosAlpha, phi, -wcX, -wcY, -wc) (geometry.h:1461-1466)
        float sinPhiS, cosPhiS;
        psincosf(phi, &sinPhiS, &cosPhiS);
        V3 nWorld = sinAlpha * cosPhiS * (-wcX) + sinAlpha * sinPhiS * (-wcY) + cosAlpha * (-wc);
        V3 pWorld = pCenter + s.radius * nWorld;
        ls.p = pWorld;
        ls.pError = kGamma5 * vabs(pWorld);
        ls.n = nWorld;
        if (s.reverse_orientation) ls.n = ls.n * -1.f;
        ls.pdf = 1 / (2 * kPi * (1 - cosThetaMax));
    }
    if (ls.pdf == 0 || lengthSquared(ls.p - ref.p) == 0) {
        ls.pdf = 0;
        ls.Li = mk3(0, 0, 0);
        ls.wi = mk3(0, 0, 0);
        return ls;
    }
    ls.wi = normalize(ls.p - ref.p);
    ls.Li = lightL(l, ls.n, -ls.wi);
    return ls;
}

// Sphere::Pdf(ref, wi) (sphere.cpp:303-315); the inside case falls back to Shape::Pdf (shape.cpp:78-95)
PB2_HDN float sphereLightPdf(const DScene &sc, const pb2_light &l, const DInteraction &ref, V3 wi) {
    const pb2_sphere s = sc.spheres[sc.primIndex[l.prim]];
    M44 o2w = loadM44(s.object_to_world);
    V3 pCenter = xfPoint(o2w, mk3(0, 0, 0));
    V3 pOrigin = offsetRayOrigin(ref.p, ref.pError, ref.n, pCenter - ref.p);
    if (lengthSquared(pOrigin - pCenter) <= s.radius * s.radius) {
        DRay ray;
        ray.o = offsetRayOrigin(ref.p, ref.pError, ref.n, wi);
        ray.d = wi;
        ray.tMax = PB2_INFINITY;
        SphereRayHit h;
        if (!sphereTest(s, ray, ray.tMax, &h)) return 0;
        DInteraction li = sphereInteraction(sc, l.prim, ray, h.tHit, h.phi);
        float pdf = lengthSquared(ref.p - li.p) / (absDot(li.n, -wi) * (s.phi_max * s.radius * (s.z_max - s.z_min)));
        if (isinf(pdf)) pdf = 0.f;
        return pdf;
    }
    float sinThetaMax2 = s.radius * s.radius / lengthSquared(ref.p - pCenter);
    float cosThetaMax = sqrtf(pmax(0.f, 1 - sinThetaMax2));
    return 1 / (2 * kPi * (1 - cosThetaMax));
}

// DiffuseAreaLight::Sample_Li (diffuse.cpp:68-81) for a triangle shape: Triangle::Sample(u)
// (triangle.cpp:582-607) + Shape::Sample(ref,u,pdf) (shape.cpp:61-76).
PB2_HD DLightSample sampleTriangleLight(const DScene &sc, const pb2_light &l, const TriRec &rec, V3 refP, V2 u) {
    DLightSample s;
    const TriVerts t = rec.tv;
    V2 b = uniformSampleTriangle(u);
    float b2 = (1 - b.x - b.y);
    s.p = b.x * t.p0 + b.y * t.p1 + b2 * t.p2;
    s.n = normalize(cross(t.p1 - t.p0, t.p2 - t.p0));
    bool hasN = false;
    if (rec.flags & LEAF_ATTR) {
        int tri = sc.primIndex[rec.prim];
        if (sc.meshes[sc.triMesh[tri]].has_n) {
            hasN = true;
            int64_t v0 = sc.triIndex[3 * (int64_t)tri], v1 = sc.triIndex[3 * (int64_t)tri + 1], v2 = sc.triIndex[3 * (int64_t)tri + 2];
            V3 ns = b.x * ld3(sc.N, v0) + b.y * ld3(sc.N, v1) + b2 * ld3(sc.N, v2);
            s.n = faceforward(s.n, ns);
        }
    }
    if (!hasN && (rec.flags & LEAF_FLIP)) s.n = s.n * -1.f;
    V3 pAbsSum = vabs(b.x * t.p0) + vabs(b.y * t.p1) + vabs(b2 * t.p2);
    s.pError = kGamma6 * pAbsSum;
    s.pdf = 1 / triangleArea(t);
    // Shape::Sample(ref, u, pdf)
    V3 wi = s.p - refP;
    if (lengthSquared(wi) == 0)
        s.pdf = 0;
    else {
        wi = normalize(wi);
        s.pdf *= lengthSquared(refP - s.p) / absDot(s.n, -wi);
        if (isinf(s.pdf)) s.pdf = 0.f;
    }
    // DiffuseAreaLight::Sample_Li
    if (s.pdf == 0 || lengthSquared(s.p - refP) == 0) {
        s.pdf = 0;
        s.Li = mk3(0, 0, 0);
        s.wi = mk3(0, 0, 0);
        return s;
    }
    s.wi = normalize(s.p - refP);
    s.Li = lightL(l, s.n, -s.wi);
    return s;
}

// PointLight / SpotLight / DistantLight::Sample_Li (point.cpp:44-53, spot.cpp:52-72, distant.cpp:48-58).  The
// VisibilityTester's second point carries no normal and no error bounds, so SpawnRayTo aims at it exactly.
PB2_HDN DLightSample sampleDeltaLight(const pb2_light &l, const DDeltaLight &dl, V3 refP) {
    DLightSample s;
    s.delta = true;
    s.pError = s.n = mk3(0, 0, 0);
    s.pdf = 1.f;
    const V3 I = mk3(l.L[0], l.L[1], l.L[2]);
    if (l.type == PB2_LIGHT_DISTANT) {
        V3 wLight = mk3(dl.p[0], dl.p[1], dl.p[2]);
        s.wi = wLight;
        s.p = refP + wLight * (2 * dl.worldRadius);
        s.Li = I;
        return s;
    }
    V3 pLight = mk3(dl.p[0], dl.p[1], dl.p[2]);
    s.p = pLight;
    s.wi = normalize(pLight - refP);
    float d2 = lengthSquared(pLight - refP);
    if (l.type == PB2_LIGHT_POINT) {
        s.Li = mk3(I.x / d2, I.y / d2, I.z / d2);
        return s;
    }
    // SpotLight::Falloff(-wi)
    V3 w = -s.wi;
    const float *m = dl.worldToLight;
    V3 wl = normalize(mk3(m[0] * w.x + m[1] * w.y + m[2] * w.z, m[3] * w.x + m[4] * w.y + m[5] * w.z, m[6] * w.x + m[7] * w.y + m[8] * w.z));
    float cosT = wl.z, falloff;
    if (cosT < dl.cosTotalWidth) falloff = 0;
    else if (cosT >= dl.cosFalloffStart) falloff = 1;
    else {
        float delta = (cosT - dl.cosTotalWidth) / (dl.cosFalloffStart - dl.cosTotalWidth);
        falloff = (delta * delta) * (delta * delta);
    }
    V3 If = I * falloff;
    s.Li = mk3(If.x / d2, If.y / d2, If.z / d2);
    return s;
}

// ---------------------------------------------------------------- InfiniteAreaLight with constant radiance
// MIPMap<RGBSpectrum>::Lookup(st, width = 0) on the light's 1 x 1 map: Levels() - 1 + Log2(1e-8) < 0, i.e.
// MIPMap::triangle(0, st) (mipmap.h:245-274) - a bilinear blend of four copies of the one texel under ImageWrap::Repeat,
// whose weights sum to one only up to rounding, so the blend is evaluated as written there.
PB2_HD V3 infiniteLookup(const pb2_light &l, V2 st) {
    const V3 T = mk3(l.L[0], l.L[1], l.L[2]);
    const float s = st.x * 1 - 0.5f, t = st.y * 1 - 0.5f;
    const float s0 = floorf(s), t0 = floorf(t);
    const float ds = s - (float)(int)s0, dt = t - (float)(int)t0;
    return ((1 - ds) * (1 - dt)) * T + ((1 - ds) * dt) * T + (ds * (1 - dt)) * T + (ds * dt) * T;
}
// Distribution1D::SampleContinuous (sampling.h:73-89) over a record [func(n) | cdf(n+1) | funcInt]
PB2_HD float sampleContinuous1D(const float *rec, int n, float u, float *pdf, int *off) {
    const float *func = rec, *cdf = rec + n;
    const float funcInt = rec[2 * n + 1];
    int first = 0, len = n + 1;   // FindInterval(size = n + 1, cdf[i] <= u), pbrt.h:403-415
    while (len > 0) {
        int half = len >> 1, middle = first + half;
        if (cdf[middle] <= u) {
            first = middle + 1;
            len -= half + 1;
        } else
            len = half;
    }
    int offset = first - 1;
    offset = offset < 0 ? 0 : (offset > n - 1 ? n - 1 : offset);   // Clamp(first - 1, 0, size - 2)
    *off = offset;
    float du = u - cdf[offset];
    if ((cdf[offset + 1] - cdf[offset]) > 0) du /= (cdf[offset + 1] - cdf[offset]);
    *pdf = (funcInt > 0) ? func[offset] / funcInt : 0;
    return (offset + du) / n;
}
// InfiniteAreaLight::Le (infinite.cpp:90-94): SphericalPhi / SphericalTheta of the direction in light space (geometry.h:1456-1465)
// Lmap->Lookup(st) of a light with an environment map: MIPMap::Lookup(st, width = 0) is the bilinear look-up at the finest
// level (mipmap.h:227-235: level = Levels - 1 + log2(1e-8) < 0), wrap mode repeat
PB2_HD V3 envLookup(const DScene &sc, const pb2_light &l, const DDeltaLight &dl, V2 st) {
    if (dl.envTex) return texTriangle(sc.textures[dl.envTex - 1], sc.texels, 0, st);
    return infiniteLookup(l, st);
}
PB2_HDN V3 infiniteLe(const DScene &sc, const pb2_light &l, const DDeltaLight &dl, V3 d) {
    const float *m = dl.worldToLight;
    const V3 w = normalize(mk3(m[0] * d.x + m[1] * d.y + m[2] * d.z, m[3] * d.x + m[4] * d.y + m[5] * d.z, m[6] * d.x + m[7] * d.y + m[8] * d.z));
    float phi = patan2f(w.y, w.x);
    if (phi < 0) phi = phi + 2 * kPi;
    const float theta = pacosf(clampf(w.z, -1.f, 1.f));
    return envLookup(sc, l, dl, mk2(phi * (0.5f * kInvPi), theta * kInvPi));
}
// InfiniteAreaLight::Sample_Li (infinite.cpp:96-122); the VisibilityTester's far point has neither normal nor error bounds
PB2_HDN DLightSample sampleInfiniteLight(const DScene &sc, const pb2_light &l, const DDeltaLight &dl, V3 refP, V2 u) {
    DLightSample s;
    s.delta = false;
    s.pError = s.n = mk3(0, 0, 0);
    s.p = refP;
    s.wi = mk3(0, 0, 1);
    s.pdf = 0;
    s.Li = mk3(0, 0, 0);
    // Distribution2D::SampleContinuous (sampling.h:117-125): the row from the marginal with u[1], then inside the row with u[0]
    float pdf1, pdf0;
    int v, uo;
    float d0, d1;
    if (dl.envTex) {
        const int nu = dl.envNu, nv = dl.envNv;
        d1 = sampleContinuous1D(dl.envDist + (size_t)nv * (2 * nu + 2), nv, u.y, &pdf1, &v);
        d0 = sampleContinuous1D(dl.envDist + (size_t)v * (2 * nu + 2), nu, u.x, &pdf0, &uo);
    } else {
        d1 = sampleContinuous1D(dl.dist + 12, 2, u.y, &pdf1, &v);
        d0 = sampleContinuous1D(dl.dist + 6 * v, 2, u.x, &pdf0, &uo);
    }
    const float mapPdf = pdf0 * pdf1;
    if (mapPdf == 0) return s;
    const float theta = d1 * kPi, phi = d0 * 2 * kPi;
    const float cosTheta = pcosf(theta), sinTheta = psinf(theta);
    const float sinPhi = psinf(phi), cosPhi = pcosf(phi);
    const V3 vl = mk3(sinTheta * cosPhi, sinTheta * sinPhi, cosTheta);
    const float *m = dl.lightToWorld;
    s.wi = mk3(m[0] * vl.x + m[1] * vl.y + m[2] * vl.z, m[3] * vl.x + m[4] * vl.y + m[5] * vl.z, m[6] * vl.x + m[7] * vl.y + m[8] * vl.z);
    s.pdf = mapPdf / (2 * kPi * kPi * sinTheta);
    if (sinTheta == 0) s.pdf = 0;
    s.p = refP + s.wi * (2 * dl.worldRadius);
    s.Li = envLookup(sc, l, dl, mk2(d0, d1));
    return s;
}
// InfiniteAreaLight::Pdf_Li (infinite.cpp:124-132), Distribution2D::Pdf (sampling.h:126-132)
PB2_HDN float infinitePdfLi(const DDeltaLight &dl, V3 w) {
    const float *m = dl.worldToLight;
    const V3 wi = mk3(m[0] * w.x + m[1] * w.y + m[2] * w.z, m[3] * w.x + m[4] * w.y + m[5] * w.z, m[6] * w.x + m[7] * w.y + m[8] * w.z);
    const float theta = pacosf(clampf(wi.z, -1.f, 1.f));
    float phi = patan2f(wi.y, wi.x);
    if (phi < 0) phi = phi + 2 * kPi;
    const float sinTheta = psinf(theta);
    if (sinTheta == 0) return 0;
    const float px = phi * (0.5f * kInvPi), py = theta * kInvPi;
    if (dl.envTex) {
        const int nu = dl.envNu, nv = dl.envNv;
        int iu = (int)(px * nu), iv = (int)(py * nv);
        iu = iu < 0 ? 0 : (iu > nu - 1 ? nu - 1 : iu);
        iv = iv < 0 ? 0 : (iv > nv - 1 ? nv - 1 : iv);
        const float marginalInt = dl.envDist[(size_t)nv * (2 * nu + 2) + 2 * nv + 1];
        return (dl.envDist[(size_t)iv * (2 * nu + 2) + iu] / marginalInt) / (2 * kPi * kPi * sinTheta);
    }
    int iu = (int)(px * 2), iv = (int)(py * 2);
    iu = iu < 0 ? 0 : (iu > 1 ? 1 : iu);
    iv = iv < 0 ? 0 : (iv > 1 ? 1 : iv);
    return (dl.dist[6 * iv + iu] / dl.dist[12 + 5]) / (2 * kPi * kPi * sinTheta);
}

// `rec` is the light's record out of DScene::lightRecs, lightNum its index in Scene::lights.
template <int F>
PB2_HD DLightSample sampleLight(const DScene &sc, int lightNum, const pb2_light &l, const TriRec &rec, const DInteraction &ref, V2 u) {
    const bool nonArea = (F & SHADE_NON_AREA) && sc.deltaLights;
    if (nonArea && l.type == PB2_LIGHT_INFINITE) return sampleInfiniteLight(sc, l, sc.deltaLights[lightNum], ref.p, u);
    if (nonArea && l.type != PB2_LIGHT_AREA) return sampleDeltaLight(l, sc.deltaLights[lightNum], ref.p);
    DLightSample s;
    if ((F & SHADE_SPHERES) && (rec.flags & LEAF_SPHERE)) s = sampleSphereLight(sc, l, ref, u);
    else s = sampleTriangleLight(sc, l, rec, ref.p, u);
    s.delta = false;
    return s;
}

// DiffuseAreaLight::Pdf_Li -> Shape::Pdf(ref, wi) (shape.cpp:78-95): re-intersect the light's own
// shape with the spawned ray and convert the area density to solid angle.
template <int F>
PB2_HD float lightPdfLi(const DScene &sc, const pb2_light &l, const TriRec &rec, const DInteraction &ref, V3 wi, int lightNum = -1) {
    if ((F & SHADE_NON_AREA) && sc.deltaLights && l.type == PB2_LIGHT_INFINITE) return infinitePdfLi(sc.deltaLights[lightNum], wi);
    if ((F & SHADE_SPHERES) && (rec.flags & LEAF_SPHERE)) return sphereLightPdf(sc, l, ref, wi);
    DRay ray = spawnRay(ref, wi);
    const TriVerts t = rec.tv;
    DRaySetup rs = setupRay(ray.o, ray.d);
    float tHit, b0, b1, b2;
    if (!triangleTest(t.p0, t.p1, t.p2, rs, ray.tMax, &tHit, &b0, &b1, &b2)) return 0;
    if (rec.flags & LEAF_DEGENERATE) return 0;   // triPartials failed at upload (triangle.cpp:308-314)
    DInteraction li = triangleInteraction(sc, rec, b0, b1, b2, ray.d);
    float pdf = lengthSquared(ref.p - li.p) / (absDot(li.n, -wi) * triangleArea(t));
    if (isinf(pdf)) pdf = 0.f;
    return pdf;
}

// ---------------------------------------------------------------- light distributions
// LightDistribution::Lookup(p): returns the Distribution1D record for p.
PB2_HD const float *lightDistLookup(const DLightDist &ld, V3 p) {
    if (ld.strategy != PB2_LIGHTDIST_SPATIAL) return ld.table;
    // SpatialLightDistribution::Lookup (lightdistrib.cpp:141-147): Bounds3::Offset, then clamp(int(o*n))
    V3 o = p - ld.boundsMin;
    if (ld.boundsMax.x > ld.boundsMin.x) o.x /= ld.boundsMax.x - ld.boundsMin.x;
    if (ld.boundsMax.y > ld.boundsMin.y) o.y /= ld.boundsMax.y - ld.boundsMin.y;
    if (ld.boundsMax.z > ld.boundsMin.z) o.z /= ld.boundsMax.z - ld.boundsMin.z;
    int pi[3];
    float of[3] = {o.x, o.y, o.z};
    for (int i = 0; i < 3; ++i) {
        float v = of[i] * ld.nVoxels[i];
        int iv = (v != v) ? 0 : (v >= 2147483648.f ? ld.nVoxels[i] - 1 : (v <= -2147483648.f ? 0 : (int)v));
        pi[i] = iv < 0 ? 0 : (iv > ld.nVoxels[i] - 1 ? ld.nVoxels[i] - 1 : iv);
    }
    int64_t voxel = ((int64_t)pi[0] * ld.nVoxels[1] + pi[1]) * ld.nVoxels[2] + pi[2];
    if (!ld.slots) return ld.table + voxel * ld.stride;
#if defined(__CUDA_ARCH__)
    int s = ld.slots[voxel];
    if (s >= 0) return ld.table + (size_t)s * ld.stride;
    if (s == LD_ABSENT && atomicCAS(&ld.slots[voxel], (int)LD_ABSENT, (int)LD_REQUESTED) == LD_ABSENT)
        ld.requests[atomicAdd(&ld.counters[0], 1)] = (int)voxel;
#endif
    return nullptr;   // not built yet: the caller defers the vertex
}

// SpatialLightDistribution::ComputeDistribution (lightdistrib.cpp:232-300) for one voxel, written
// into rec = [func(n) | cdf(n+1) | funcInt] (Distribution1D ctor, sampling.h:57-70).  Three pieces, so that the
// eager builder (one thread per voxel) and the lazy one (one block per voxel, one thread per light) share every line
// of arithmetic: the voxel's bounds, the contribution of ONE light summed over the 128 Halton points in their order,
// and the floor + cdf over all lights in their order.
struct DVoxelBounds { V3 vMin, vMax; };
PB2_HD DVoxelBounds voxelBounds(const DLightDist &ld, int px, int py, int pz) {
    V3 p0 = mk3((float)px / (float)ld.nVoxels[0], (float)py / (float)ld.nVoxels[1], (float)pz / (float)ld.nVoxels[2]);
    V3 p1 = mk3((float)(px + 1) / (float)ld.nVoxels[0], (float)(py + 1) / (float)ld.nVoxels[1], (float)(pz + 1) / (float)ld.nVoxels[2]);
    // Bounds3f(WorldBound().Lerp(p0), WorldBound().Lerp(p1)): the two-point ctor takes min/max
    V3 a = mk3(lerpf(p0.x, ld.boundsMin.x, ld.boundsMax.x), lerpf(p0.y, ld.boundsMin.y, ld.boundsMax.y), lerpf(p0.z, ld.boundsMin.z, ld.boundsMax.z));
    V3 b = mk3(lerpf(p1.x, ld.boundsMin.x, ld.boundsMax.x), lerpf(p1.y, ld.boundsMin.y, ld.boundsMax.y), lerpf(p1.z, ld.boundsMin.z, ld.boundsMax.z));
    DVoxelBounds vb;
    vb.vMin = mk3(pmin(a.x, b.x), pmin(a.y, b.y), pmin(a.z, b.z));
    vb.vMax = mk3(pmax(a.x, b.x), pmax(a.y, b.y), pmax(a.z, b.z));
    return vb;
}
constexpr int kVoxelSamples = 128;
// light j's importance for the voxel: sum over the sample points of Li.y() / pdf, visibility ignored (lightdistrib.cpp:255-276)
PB2_HD float voxelLightContribution(const DScene &sc, const DHalton &h, const DVoxelBounds &vb, int j) {
    const pb2_light light = sc.lights[j];
    const TriRec rec = loadTriRec(sc.lightRecs, (size_t)j);
    float contrib = 0;
    for (int i = 0; i < kVoxelSamples; ++i) {
        V3 t = mk3(radicalInverse(h, 0, i), radicalInverse(h, 1, i), radicalInverse(h, 2, i));
        DInteraction intr;
        intr.p = mk3(lerpf(t.x, vb.vMin.x, vb.vMax.x), lerpf(t.y, vb.vMin.y, vb.vMax.y), lerpf(t.z, vb.vMin.z, vb.vMax.z));
        intr.pError = mk3(0, 0, 0);
        intr.n = mk3(0, 0, 0);
        intr.wo = mk3(1, 0, 0);
        intr.ns = mk3(0, 0, 0);
        intr.dpdus = mk3(0, 0, 0);
        intr.uv = mk2(0, 0);
        intr.prim = -1;
        V2 u = mk2(radicalInverse(h, 3, i), radicalInverse(h, 4, i));
        DLightSample ls = sampleLight<SHADE_GENERAL | SHADE_SPHERES>(sc, j, light, rec, intr, u);
        if (ls.pdf > 0) contrib += luminance(ls.Li) / ls.pdf;
    }
    return contrib;
}
// rec[0 .. n) holds the contributions: floor them (lightdistrib.cpp:278-294) and build the Distribution1D
PB2_HD void finishVoxelDistribution(int n, float *rec) {
    float sumContrib = 0;
    for (int j = 0; j < n; ++j) sumContrib += rec[j];
    float avgContrib = sumContrib / (kVoxelSamples * n);
    float minContrib = (avgContrib > 0) ? (float)(.001 * (double)avgContrib) : 1;
    for (int j = 0; j < n; ++j) rec[j] = pmax(rec[j], minContrib);
    float *cdf = rec + n;
    cdf[0] = 0;
    for (int i = 1; i < n + 1; ++i) cdf[i] = cdf[i - 1] + rec[i - 1] / n;
    float funcInt = cdf[n];
    if (funcInt == 0) {
        for (int i = 1; i < n + 1; ++i) cdf[i] = (float)i / (float)n;
    } else {
        for (int i = 1; i < n + 1; ++i) cdf[i] /= funcInt;
    }
    rec[2 * n + 1] = funcInt;
}
PB2_HD void computeVoxelDistribution(const DScene &sc, const DHalton &h, const DLightDist &ld, int px, int py, int pz,
                                     float *rec) {
    const DVoxelBounds vb = voxelBounds(ld, px, py, pz);
    for (int j = 0; j < sc.nLights; ++j) rec[j] = voxelLightContribution(sc, h, vb, j);
    finishVoxelDistribution(sc.nLights, rec);
}

// ---------------------------------------------------------------- camera
struct DCamera {
    M44 rasterToCamera, cameraToWorld;
    float lensRadius, focalDistance;
    V3 dxCamera, dyCamera;    // ProjectiveCamera: the camera-space step of one pixel in x / y (perspective.cpp:59-62)
};

// A camera ray's differentials (world space).
struct DRayDiff { V3 rxo, rxd, ryo, ryd; };

// The offset rays PerspectiveCamera::GenerateRayDifferential adds to a camera ray (perspective.cpp:117-144), taken to world
// space (Transform::operator()(RayDifferential), transform.h:266-275: the auxiliary origins are NOT moved along the ray as
// the main one is) and scaled as SamplerIntegrator::Render does (integrator.cpp:273-274, geometry.h:908-913).
// (o, d): the main ray in world space as it was traced; uLens: the lens sample of this camera sample.
PB2_HD DRayDiff cameraRayDifferentials(const DCamera &cam, V2 pFilm, V2 uLens, float scale, V3 o, V3 d) {
    V3 pCamera = xfPoint(cam.rasterToCamera, mk3(pFilm.x, pFilm.y, 0));
    V3 rxo = mk3(0, 0, 0), ryo = mk3(0, 0, 0), rxd, ryd;
    if (cam.lensRadius > 0) {
        V2 dsk = concentricSampleDisk(uLens);
        V2 pLens = mk2(cam.lensRadius * dsk.x, cam.lensRadius * dsk.y);
        V3 dx = normalize(pCamera + cam.dxCamera);
        float ft = cam.focalDistance / dx.z;
        V3 pFocus = mk3(0, 0, 0) + (ft * dx);
        rxo = mk3(pLens.x, pLens.y, 0);
        rxd = normalize(pFocus - rxo);
        V3 dy = normalize(pCamera + cam.dyCamera);
        ft = cam.focalDistance / dy.z;
        pFocus = mk3(0, 0, 0) + (ft * dy);
        ryo = mk3(pLens.x, pLens.y, 0);
        ryd = normalize(pFocus - ryo);
    } else {
        rxd = normalize(pCamera + cam.dxCamera);
        ryd = normalize(pCamera + cam.dyCamera);
    }
    DRayDiff r;
    r.rxo = xfPoint(cam.cameraToWorld, rxo);
    r.ryo = xfPoint(cam.cameraToWorld, ryo);
    r.rxd = xfVector(cam.cameraToWorld, rxd);
    r.ryd = xfVector(cam.cameraToWorld, ryd);
    r.rxo = o + (r.rxo - o) * scale;
    r.ryo = o + (r.ryo - o) * scale;
    r.rxd = d + (r.rxd - d) * scale;
    r.ryd = d + (r.ryd - d) * scale;
    return r;
}

// SurfaceInteraction::ComputeDifferentials (interaction.cpp:101-147): the (u, v) footprint of the pixel at a hit
PB2_HD DUvDiff computeUvDifferentials(V3 p, V3 n, V3 dpdu, V3 dpdv, const DRayDiff &rd) {
    DUvDiff z;
    z.dudx = z.dvdx = z.dudy = z.dvdy = 0;
    float dd = dot(n, p);
    float tx = -(dot(n, rd.rxo) - dd) / dot(n, rd.rxd);
    if (isinf(tx) || tx != tx) return z;
    V3 px = rd.rxo + tx * rd.rxd;
    float ty = -(dot(n, rd.ryo) - dd) / dot(n, rd.ryd);
    if (isinf(ty) || ty != ty) return z;
    V3 py = rd.ryo + ty * rd.ryd;
    int d0, d1;
    if (fabsf(n.x) > fabsf(n.y) && fabsf(n.x) > fabsf(n.z)) {
        d0 = 1;
        d1 = 2;
    } else if (fabsf(n.y) > fabsf(n.z)) {
        d0 = 0;
        d1 = 2;
    } else {
        d0 = 0;
        d1 = 1;
    }
    const float A00 = comp(dpdu, d0), A01 = comp(dpdv, d0), A10 = comp(dpdu, d1), A11 = comp(dpdv, d1);
    const float Bx0 = comp(px, d0) - comp(p, d0), Bx1 = comp(px, d1) - comp(p, d1);
    const float By0 = comp(py, d0) - comp(p, d0), By1 = comp(py, d1) - comp(p, d1);
    // SolveLinearSystem2x2 (transform.cpp:41-49)
    float det = A00 * A11 - A01 * A10;
    if (!(fabsf(det) < 1e-10f)) {
        DUvDiff r = z;
        r.dudx = (A11 * Bx0 - A01 * Bx1) / det;
        r.dvdx = (A00 * Bx1 - A10 * Bx0) / det;
        if (r.dudx != r.dudx || r.dvdx != r.dvdx) r.dudx = r.dvdx = 0;
        r.dudy = (A11 * By0 - A01 * By1) / det;
        r.dvdy = (A00 * By1 - A10 * By0) / det;
        if (r.dudy != r.dudy || r.dvdy != r.dvdy) r.dudy = r.dvdy = 0;
        return r;
    }
    return z;
}

// Sampler::GetCameraSample (sampler.cpp:46-52) + PerspectiveCamera::GenerateRayDifferential
// (perspective.cpp:95-144) + Transform::operator()(Ray) (transform.h:251-264).  Differentials are
// not carried: nothing on this path reads them (constant textures only).
template <bool GENERAL = false>
PB2_HD DRay generateCameraRay(const DCamera &cam, const DHalton &h, DSampler &smp, int px, int py, V2 *pFilmOut) {
    V2 uf;
    if (GENERAL && h.sobol) {
        uf = mk2(sobolPixelSample(h, smp.index, 0, px), sobolPixelSample(h, smp.index, 1, py));
        smp.dim += 2;
    } else
        uf = get2D(h, smp);
    V2 pFilm = mk2((float)px + uf.x, (float)py + uf.y);
    // CameraSample::time and pLens (sampler.cpp:46-52) take dimensions 2-4.  The sample values are pure
    // functions of (index, dimension): what is not read is not computed - time never is (static scenes),
    // pLens only with a finite aperture.
    smp.dim += 1;
    V2 uLens = mk2(0, 0);
    if (cam.lensRadius > 0) uLens = get2D<GENERAL>(h, smp);
    else smp.dim += 2;
    *pFilmOut = pFilm;
    V3 pCamera = xfPoint(cam.rasterToCamera, mk3(pFilm.x, pFilm.y, 0));
    DRay ray;
    ray.o = mk3(0, 0, 0);
    ray.d = normalize(pCamera);
    ray.tMax = PB2_INFINITY;
    if (cam.lensRadius > 0) {
        V2 d = concentricSampleDisk(uLens);
        V2 pLens = mk2(cam.lensRadius * d.x, cam.lensRadius * d.y);
        float ft = cam.focalDistance / ray.d.z;
        V3 pFocus = ray.o + ray.d * ft;
        ray.o = mk3(pLens.x, pLens.y, 0);
        ray.d = normalize(pFocus - ray.o);
    }
    V3 oError;
    V3 o = xfPointErr(cam.cameraToWorld, ray.o, &oError);
    V3 d = xfVector(cam.cameraToWorld, ray.d);
    float l2 = lengthSquared(d);
    float tMax = ray.tMax;
    if (l2 > 0) {
        float dt = dot(vabs(d), oError) / l2;
        o = o + d * dt;
        tMax -= dt;
    }
    ray.o = o;
    ray.d = d;
    ray.tMax = tMax;
    return ray;
}

// ---------------------------------------------------------------- PathIntegrator::Li
struct DPathParams {
    int maxDepth;
    float rrThreshold;
};

// The per-sample guard of SamplerIntegrator::Render (integrator.cpp:294-315)
PB2_HD V3 guardRadiance(V3 L) {
    if (L.x != L.x || L.y != L.y || L.z != L.z) return mk3(0, 0, 0);
    float y = luminance(L);
    if ((double)y < -1e-5) return mk3(0, 0, 0);
    if (isinf(y)) return mk3(0, 0, 0);
    return L;
}

}  // namespace pb2
#endif
