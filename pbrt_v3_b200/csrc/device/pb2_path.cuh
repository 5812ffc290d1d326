// PathIntegrator::Li as a per-lane state machine with ONE ray-tracing site.
//
// The reference's bounce loop (src/integrators/path.cpp:81-185) traces up to three rays per path
// vertex, at three different places: the path ray (closest hit), the next-event-estimation shadow
// ray (any hit, src/core/integrator.cpp:146) and the MIS ray of the BSDF sample (closest hit,
// integrator.cpp:202).  None of the sampler dimensions, BSDF values or ray origins of a vertex
// depends on the RESULT of the shadow or MIS ray, so a lane evaluates everything of the vertex up
// front (shadeVertex), queues the rays, and then only adds `ldLight` if the shadow ray was
// unoccluded and `misTerm` if the MIS ray reached the sampled light (lightAdvance).  Every ray of
// every class therefore goes through the same traversal kernel, and the heavy vertex code runs
// in its own kernel with all lanes doing the same thing.
// Sampler dimensions are consumed in the reference's order and the radiance is accumulated with
// the reference's operation order (Ld = (light + mis) / pickPdf; L += beta * Ld).
#ifndef PB2_PATH_CUH
#define PB2_PATH_CUH

#include "pb2_shade.cuh"

namespace pb2 {

// LS_DEFER: only ever seen between shadeVertex and its caller - the vertex fell into a voxel whose light distribution is
// not built yet (lazy SpatialLightDistribution); nothing of the lane was touched, the caller shades it again later.
enum { LS_IDLE = 0, LS_PATH = 1, LS_SHADOW = 2, LS_MIS = 3, LS_DEFER = 4 };

struct DLane {
    int state;
    DRay ray;            // ray to trace next (class given by state)
    // path
    V3 L, beta;
    DSampler smp;
    int bounces;
    bool specularBounce;
    bool camRay;         // the ray to shade next is the camera ray itself: the only one with differentials (path.cpp:130-131)
    float etaScale;
    // pending at the current vertex
    bool doNEE, hasMis, hasNext;
    int lightNum;
    float pick;          // light-pick pdf; 0 = UniformSampleOneLight returned black
    V3 ldSum, ldLight, misTerm;
    V3 misO, misD;       // MIS ray (tMax = inf)
    V3 nextO, nextD;     // continuation ray
    V3 betaNext;
};

PB2_HD void laneStartPath(DLane &ln, const DRay &ray, const DSampler &smp) {
    ln.state = LS_PATH;
    ln.ray = ray;
    ln.L = mk3(0, 0, 0);
    ln.beta = mk3(1, 1, 1);
    ln.smp = smp;
    ln.bounces = 0;
    ln.specularBounce = false;
    ln.camRay = true;
    ln.etaScale = 1;
    ln.doNEE = ln.hasMis = ln.hasNext = false;
}

// End of a vertex: fold the direct lighting in, then continue or stop (path.cpp:119-150,176-185).
PB2_HD void finishVertex(DLane &ln) {
    if (ln.doNEE) {
        V3 Ld = mk3(0, 0, 0);
        if (ln.pick != 0) Ld = mk3(ln.ldSum.x / ln.pick, ln.ldSum.y / ln.pick, ln.ldSum.z / ln.pick);
        ln.L = ln.L + ln.beta * Ld;
    }
    if (ln.hasNext) {
        ln.beta = ln.betaNext;
        ln.ray.o = ln.nextO;
        ln.ray.d = ln.nextD;
        ln.ray.tMax = PB2_INFINITY;
        ln.bounces++;
        ln.state = LS_PATH;
    } else
        ln.state = LS_IDLE;
}

PB2_HD void startMisOrFinish(DLane &ln) {
    if (ln.hasMis) {
        ln.ray.o = ln.misO;
        ln.ray.d = ln.misD;
        ln.ray.tMax = PB2_INFINITY;
        ln.state = LS_MIS;
    } else
        finishVertex(ln);
}

// What the camera ray's differentials are rebuilt from when image textures are evaluated.
struct DTexCtx {
    const DCamera *cam;
    V2 pFilm;           // of this camera sample
    float diffScale;    // 1 / sqrt(samples per pixel)
};

// The path ray has been traced: one iteration of the bounce loop up to (not including) the results
// of the two direct-lighting rays.
// F: the shade features (SHADE_* in pb2_shade.cuh) the vertex is compiled for.
// u: room for the vertex's kSampleBatch sampler values (the caller's: shared memory in the shade step).
template <int F>
PB2_HD void shadeVertex(const DScene &sc, const DHalton &h, const DPathParams &pp, DLane &ln, bool found, const DHit &hit,
                        float tMax, float *u, const DTexCtx *tc = nullptr) {
    constexpr bool SOBOL = (F & SHADE_SOBOL) != 0;
    // Every dimension this vertex can draw, [smp.dim, smp.dim + kSampleBatch), evaluated up front: the values are a pure
    // function of (index, dimension), and drawn here their table loads overlap the hit's leaf-record loads instead of
    // forming a chain of round trips each where its value is used.  A vertex that draws nothing skips it.
    const int dim0 = ln.smp.dim;
    if (found && ln.bounces < pp.maxDepth) haltonSampleBatch<SOBOL>(h, ln.smp.index, dim0, kSampleBatch, u);
    DInteraction isect;
    int li = -1;
    DTexGeom tg;
    DUvDiff uvDiff;
    uvDiff.dudx = uvDiff.dvdx = uvDiff.dudy = uvDiff.dvdy = 0;
    if (found) isect = hitInteraction<F>(sc, hit, ln.ray, tMax, &li, ((F & SHADE_TEXTURES) && tc) ? &tg : nullptr);
    if ((F & SHADE_TEXTURES) && tc && sc.textures) {
        if (found && ln.camRay) {
            // the camera ray's differentials are a pure function of the camera sample: rebuilt here, not carried in the lane
            V2 uLens = mk2(0, 0);
            if (tc->cam->lensRadius > 0) {
                DSampler ls = ln.smp;
                ls.dim = 3;   // CameraSample::pLens (sampler.cpp:46-52)
                uLens = get2D<SOBOL>(h, ls);
            }
            const DRayDiff rd = cameraRayDifferentials(*tc->cam, tc->pFilm, uLens, tc->diffScale, ln.ray.o, ln.ray.d);
            uvDiff = computeUvDifferentials(isect.p, isect.n, tg.dpdu, tg.dpdv, rd);
        }
        if (found && ln.bounces < pp.maxDepth) {
            // the material's bump map (e.g. matte.cpp:50: before its other textures are evaluated)
            const int m = sc.primMaterial[isect.prim];
            const int bump = m >= 0 ? sc.materials[m].tex[PB2_TEX_BUMP] : 0;
            if (bump) bumpShading(sc, bump - 1, tg, uvDiff, &isect);
        }
    }
    const float *lazyDistrib = nullptr;
    if ((F & SHADE_LAZY) && sc.lightDist.slots && found && ln.bounces < pp.maxDepth) {
        // lazy light distribution: look the voxel up before anything of the lane changes, so that a miss can hand the
        // vertex back untouched (the record is a pure function of the voxel: when it is built does not matter)
        lazyDistrib = lightDistLookup(sc.lightDist, isect.p);
        if (!lazyDistrib) {
            ln.state = LS_DEFER;
            return;
        }
    }
    if (ln.bounces == 0 || ln.specularBounce) {
        if (found) {
            if (li >= 0) ln.L = ln.L + ln.beta * lightL(sc.lights[li], isect.n, -ln.ray.d);
        } else {
            // the ray escaped: every infinite light is seen directly (path.cpp:96-98)
            if (F & SHADE_NON_AREA)
                for (int k = 0; k < sc.nInfinite; ++k)
                    ln.L = ln.L + ln.beta * infiniteLe(sc, sc.lights[sc.infinite[k]], sc.deltaLights[sc.infinite[k]], ln.ray.d);
        }
    }
    if (!found || ln.bounces >= pp.maxDepth) {
        ln.state = LS_IDLE;
        return;
    }
    if (F & SHADE_TEXTURES) ln.camRay = false;   // every ray spawned from here on is a plain Ray
    DBsdf bsdf;
    if (!makeBsdf<F>(sc, isect, &bsdf, (F & SHADE_TEXTURES) ? &uvDiff : nullptr)) {
        ln.ray = spawnRay(isect, ln.ray.d);  // null BSDF: skip the surface, same bounce count
        return;
    }
    const float *distrib = ((F & SHADE_LAZY) && lazyDistrib) ? lazyDistrib : lightDistLookup(sc.lightDist, isect.p);
    // The lane lives in HBM and is updated in place, the sampler's dimension counter included (a
    // register copy of ln.smp across this function would not fit: the 128-register budget is full).
    DSampler &smp = ln.smp;

    ln.doNEE = bsdf.nLobes > 0;
    ln.hasMis = false;
    ln.pick = 0;
    ln.ldSum = mk3(0, 0, 0);
    bool hasShadow = false;
    DRay shadow;
    shadow.o = shadow.d = mk3(0, 0, 0);
    shadow.tMax = 0;
    if (ln.doNEE && sc.nLights > 0) {
        // UniformSampleOneLight (integrator.cpp:85-106)
        float lightPickPdf;
        int lightNum = sampleDiscrete(distrib, sc.nLights, get1D<SOBOL>(h, smp, u, dim0), &lightPickPdf);
        if (lightPickPdf != 0) {
            ln.pick = lightPickPdf;
            ln.lightNum = lightNum;
            const pb2_light light = sc.lights[lightNum];
            const TriRec lightRec = loadTriRec(sc.lightRecs, (size_t)lightNum);
            V2 uLight = get2D<SOBOL>(h, smp, u, dim0);
            V2 uScattering = get2D<SOBOL>(h, smp, u, dim0);
            // EstimateDirect, light-sampling half (integrator.cpp:116-160)
            DLightSample ls = sampleLight<F>(sc, lightNum, light, lightRec, isect, uLight);
            float lightPdf = ls.pdf, scatteringPdf = 0;
            if (lightPdf > 0 && !isBlack(ls.Li)) {
                V3 f = bsdfF<F>(bsdf, isect.wo, ls.wi) * absDot(ls.wi, isect.ns);
                scatteringPdf = bsdfPdf<F>(bsdf, isect.wo, ls.wi);
                if (!isBlack(f)) {
                    shadow = spawnRayTo(isect, ls.p, ls.pError, ls.n);
                    hasShadow = true;
                    // a delta light's sample is not weighted (integrator.cpp:150-151): f * Li / lightPdf
                    float weight = ls.delta ? 1.f : powerHeuristic(lightPdf, scatteringPdf);
                    V3 fl = f * ls.Li * weight;
                    ln.ldLight = mk3(fl.x / lightPdf, fl.y / lightPdf, fl.z / lightPdf);
                }
            }
            // BSDF-sampling half (integrator.cpp:162-213), skipped for delta lights
            V3 wi;
            V3 f = mk3(0, 0, 0);
            if (!ls.delta) {
                f = bsdfSampleF<F>(bsdf, isect.wo, &wi, uScattering, &scatteringPdf, nullptr, true);
                if (scatteringPdf != 0) f = f * absDot(wi, isect.ns);
                else f = mk3(0, 0, 0);
            }
            if (!isBlack(f) && scatteringPdf > 0) {
                lightPdf = lightPdfLi<F>(sc, light, lightRec, isect, wi, lightNum);
                if (lightPdf != 0) {
                    float weight = powerHeuristic(scatteringPdf, lightPdf);
                    // Li is the light's Lemit when the MIS ray reaches its emitting side (checked after
                    // the trace); f * Li * Tr(=1) * weight / scatteringPdf.  An infinite light is seen when the ray
                    // escapes instead (integrator.cpp:209-211): its Le along wi is known here already.
                    V3 Lmis = mk3(light.L[0], light.L[1], light.L[2]);
                    if ((F & SHADE_NON_AREA) && sc.deltaLights && light.type == PB2_LIGHT_INFINITE) Lmis = infiniteLe(sc, light, sc.deltaLights[lightNum], wi);
                    V3 fl = f * Lmis * weight;
                    ln.misTerm = mk3(fl.x / scatteringPdf, fl.y / scatteringPdf, fl.z / scatteringPdf);
                    DRay mr = spawnRay(isect, wi);
                    ln.misO = mr.o;
                    ln.misD = mr.d;
                    ln.hasMis = true;
                }
            }
        }
    }

    // continuation (path.cpp:130-150, 176-184)
    ln.hasNext = false;
    {
        V3 wo = -ln.ray.d, wi;
        float pdf;
        int sampled = 0;
        V3 f = bsdfSampleF<F>(bsdf, wo, &wi, get2D<SOBOL>(h, smp, u, dim0), &pdf, &sampled);
        if (!(isBlack(f) || pdf == 0.f)) {
            V3 s = f * absDot(wi, isect.ns);
            V3 beta = ln.beta * mk3(s.x / pdf, s.y / pdf, s.z / pdf);
            ln.specularBounce = (sampled & BSDF_SAMPLED_SPECULAR) != 0;
            if ((sampled & BSDF_SAMPLED_SPECULAR) && (sampled & BSDF_SAMPLED_TRANSMISSION)) {
                // radiance scaling of refraction, tracked for Russian roulette only (path.cpp:142-149)
                float eta = bsdf.eta;
                ln.etaScale *= (dot(wo, isect.n) > 0) ? (eta * eta) : 1 / (eta * eta);
            }
            DRay nr = spawnRay(isect, wi);
            bool survive = true;
            V3 rrBeta = beta * ln.etaScale;
            if (maxComponentValue(rrBeta) < pp.rrThreshold && ln.bounces > 3) {
                float q = pmax(.05f, 1 - maxComponentValue(rrBeta));
                if (get1D<SOBOL>(h, smp, u, dim0) < q) survive = false;
                else {
                    float d = 1 - q;
                    beta = mk3(beta.x / d, beta.y / d, beta.z / d);
                }
            }
            if (survive) {
                ln.hasNext = true;
                ln.nextO = nr.o;
                ln.nextD = nr.d;
                ln.betaNext = beta;
            }
        }
    }

    if (hasShadow) {
        ln.ray = shadow;
        ln.state = LS_SHADOW;
    } else
        startMisOrFinish(ln);
}

// A shadow or MIS ray has been traced: add its term, then start the vertex's next ray or finish it.
template <int F>
PB2_HD void lightAdvance(const DScene &sc, DLane &ln, bool found, const DHit &hit, float tMax) {
    const bool nonArea = (F & SHADE_NON_AREA) && sc.deltaLights;
    if (ln.state == LS_SHADOW) {
        if (!found) ln.ldSum = ln.ldSum + ln.ldLight;  // VisibilityTester::Unoccluded
        startMisOrFinish(ln);
    } else {
        if (!found) {
            // the MIS ray escaped: Li = light.Le(ray), which is zero for every light but an infinite one (integrator.cpp:209-211)
            if (nonArea && sc.lights[ln.lightNum].type == PB2_LIGHT_INFINITE) ln.ldSum = ln.ldSum + ln.misTerm;
        } else if (!(nonArea && sc.lights[ln.lightNum].type == PB2_LIGHT_INFINITE)) {
            // the hit primitive's light number rides in its leaf record (spheres: via primLight)
            float4 b = ldg4(&sc.leafPrims[3 * (size_t)hit.leaf + 1]), c = ldg4(&sc.leafPrims[3 * (size_t)hit.leaf + 2]);
            int hitLight = asInt(c.w);
            if ((F & SHADE_SPHERES) && (floatBits(b.w) & LEAF_SPHERE)) hitLight = sc.primLight[asInt(ldg4(&sc.leafPrims[3 * (size_t)hit.leaf]).w)];
            if (hitLight == ln.lightNum) {
                const pb2_light light = sc.lights[ln.lightNum];
                // lightIsect.Le(-wi): DiffuseAreaLight::L with the hit's (face-forwarded) normal
                if (light.two_sided) ln.ldSum = ln.ldSum + ln.misTerm;
                else {
                    DInteraction lightIsect = hitInteraction<F>(sc, hit, ln.ray, tMax);
                    if (dot(lightIsect.n, -ln.ray.d) > 0) ln.ldSum = ln.ldSum + ln.misTerm;
                }
            }
        }
        finishVertex(ln);
    }
}

// Advance a lane after its current ray was traced.  Returns true when the path ended in this call
// (ln.L is then final and ln.state == LS_IDLE).  The vertex can always be handed back (SHADE_LAZY): the caller checks LS_DEFER.
template <int F>
PB2_HD bool laneAdvance(const DScene &sc, const DHalton &h, const DPathParams &pp, DLane &ln, bool found, const DHit &hit,
                        float tMax, const DTexCtx *tc = nullptr) {
    if (ln.state == LS_PATH) {
        float u[kSampleBatch];
        shadeVertex<F | SHADE_LAZY>(sc, h, pp, ln, found, hit, tMax, u, tc);
    } else
        lightAdvance<F>(sc, ln, found, hit, tMax);
    return ln.state == LS_IDLE;
}

// Traces the lane's current ray with the one-thread-per-ray traversal.
PB2_HD bool traceLane(const DScene &sc, const DLane &ln, float *tMax, DHit *hit, DCounters *ctr) {
    *tMax = ln.ray.tMax;
    hit->leaf = -1;
    hit->b0 = hit->b1 = hit->b2 = 0;
    hit->inst = -1;
    return traverseAnyOrClosest(sc, ln.ray, ln.state == LS_SHADOW, tMax, hit, ctr);
}

}  // namespace pb2
#endif
