// TEST INFRASTRUCTURE ONLY — never linked into or called by the product (pbrt_v3_b200/).
//
// C-ABI harness around the UNMODIFIED reference sources, compiled where they lie under
// /root/reference by oracle/Makefile.ref into oracle/_ref/libpbrt_ref.so.  It rebuilds a reference
// Scene (TriangleMesh/Sphere shapes, GeometricPrimitives, matte/plastic materials, DiffuseAreaLights,
// BVHAccel) from the same flattened pb2_scene_desc the CUDA library receives, and exposes the
// reference's own Scene::Intersect/IntersectP, HaltonSampler, SpatialLightDistribution,
// PathIntegrator::Li and SamplerIntegrator::Render on it.  Used (a) by tests as the parity oracle,
// (b) to pin the restatement in oracle/pb2_oracle.cpp, (c) by bench.py's `--impl reference` arm and
// `cpu_baseline` leg as the reference's CPU implementation of the path.
//
// The three symbols the reference's build would take from files we do not compile are defined
// here: PbrtOptions (src/core/api.cpp:141), parserLoc (src/core/parser.cpp:57) and WriteImage
// (src/core/imageio.cpp:81) — the last one captures the final RGB buffer instead of encoding a file.
#include <chrono>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <sstream>
#include <string>
#include <unordered_map>
#include <vector>
#include <atomic>
#include <thread>
#include <condition_variable>
#include <functional>
#include <set>
#include <algorithm>
#include <cmath>

// The reference keeps the linear BVH, the sphere's derived angles and the camera matrices private;
// a checker is allowed to look (and, for two const members that the flattened description stores
// already evaluated, to overwrite them so both sides see identical inputs).
#define private public
#define protected public
#include "pbrt.h"
#include "accelerators/bvh.h"
#include "cameras/perspective.h"
#include "core/api.h"
#include "core/film.h"
#include "core/imageio.h"
#include "core/light.h"
#include "core/lightdistrib.h"
#include "core/parallel.h"
#include "core/paramset.h"
#include "core/parser.h"
#include "core/primitive.h"
#include "core/sampling.h"
#include "core/scene.h"
#include "core/stats.h"
#include "filters/box.h"
#include "filters/gaussian.h"
#include "filters/mitchell.h"
#include "filters/sinc.h"
#include "filters/triangle.h"
#include "integrators/path.h"
#include "lights/diffuse.h"
#include "lights/distant.h"
#include "lights/infinite.h"
#include "lights/point.h"
#include "lights/spot.h"
#include "materials/matte.h"
#include "materials/plastic.h"
#include "materials/mirror.h"
#include "materials/glass.h"
#include "materials/substrate.h"
#include "materials/metal.h"
#include "materials/uber.h"
#include "samplers/halton.h"
#include "samplers/sobol.h"
#include "shapes/loopsubdiv.h"
#include "shapes/sphere.h"
#include "shapes/triangle.h"
#include "textures/checkerboard.h"
#include "textures/constant.h"
#include "textures/uv.h"
#include "textures/mix.h"
#include "textures/scale.h"
#include "mipmap.h"
#include "texture.h"
#undef private
#undef protected

#include "pb2.h"

namespace pbrt {
Options PbrtOptions;
Loc *parserLoc = nullptr;

static std::mutex g_imageMutex;
static std::vector<Float> g_lastImage;
static Bounds2i g_lastBounds;
// imageio.cpp is not compiled (it needs OpenEXR).  ReadImage serves images that ref_scene_create registered under a name
// of its own: the environment map of an InfiniteAreaLight travels in the scene description (pb2_delta_light::env_tex) as
// the texels ReadImage(mapname) * L, and the reference's constructor reads them back through this function.
static std::mutex g_registryMutex;
struct RegisteredImage { int w, h; std::vector<float> rgb; };
static std::map<std::string, RegisteredImage> g_imageRegistry;
std::unique_ptr<RGBSpectrum[]> ReadImage(const std::string &name, Point2i *resolution) {
    std::lock_guard<std::mutex> lock(g_registryMutex);
    auto it = g_imageRegistry.find(name);
    if (it == g_imageRegistry.end()) return nullptr;
    const RegisteredImage &im = it->second;
    resolution->x = im.w;
    resolution->y = im.h;
    std::unique_ptr<RGBSpectrum[]> out(new RGBSpectrum[(size_t)im.w * im.h]);
    for (size_t i = 0; i < (size_t)im.w * im.h; ++i) out[i] = RGBSpectrum::FromRGB(&im.rgb[3 * i]);
    return out;
}
void WriteImage(const std::string &, const Float *rgb, const Bounds2i &outputBounds, const Point2i &) {
    std::lock_guard<std::mutex> lock(g_imageMutex);
    g_lastBounds = outputBounds;
    g_lastImage.assign(rgb, rgb + 3 * (size_t)outputBounds.Area());
}

// Layout-identical restatement of the struct that exists only inside src/accelerators/bvh.cpp:95-104,
// so that BVHAccel::nodes can be read.
struct LinearBVHNode {
    Bounds3f bounds;
    union {
        int primitivesOffset;
        int secondChildOffset;
    };
    uint16_t nPrimitives;
    uint8_t axis;
    uint8_t pad[1];
};
}  // namespace pbrt

using namespace pbrt;

// Device math.  libpbrt_ref.so routes the reference's sinf / cosf / sincosf / logf / atan2f / acosf through
// ref_devmath.cpp, which computes them as the device does while ref_devmath_active is set.  ref_set_device_math(1) makes
// the entry points below set it around evaluation only (tracing, sampling, Li, look-ups), never while scenes, lights,
// films, cameras or textures are built: the tables those constructors fill (MIPMap's Lanczos weights, the infinite light's
// Distribution2D, the sinc filter's table) are built by the library on the host with glibc, as here.  The spatial light
// distribution, which the reference fills lazily during Li, is evaluation; the device builds it with its own functions.
// libb200_overlay.so includes this file but links glibc's functions directly, so the flag changes nothing there.
std::atomic<int> ref_devmath_active{0};

namespace {

int g_deviceMathMode = 0;

struct DeviceMathScope {
    DeviceMathScope() { ref_devmath_active.store(g_deviceMathMode); }
    ~DeviceMathScope() { ref_devmath_active.store(0); }
};

struct RefScene {
    std::vector<std::unique_ptr<Transform>> transforms;
    std::vector<std::shared_ptr<Primitive>> prims;  // scene order
    std::unordered_map<const Primitive *, int> primNumber;
    std::vector<std::shared_ptr<Light>> lights;
    std::shared_ptr<BVHAccel> bvh;
    std::unique_ptr<Scene> scene;
    int lightStrategy = PB2_LIGHTDIST_SPATIAL;
    std::unique_ptr<LightDistribution> distrib;  // for ref_light_distribution
};

Transform fromMatrices(const float m[16], const float mi[16]) {
    Matrix4x4 a, b;
    std::memcpy(a.m, m, sizeof(a.m));
    std::memcpy(b.m, mi, sizeof(b.m));
    return Transform(a, b);
}

const char *strategyName(int s) {
    return s == PB2_LIGHTDIST_UNIFORM ? "uniform" : (s == PB2_LIGHTDIST_POWER ? "power" : "spatial");
}

struct RenderObjects {
    Film *film = nullptr;  // owned by the camera (Camera::~Camera deletes it, camera.cpp:42)
    std::shared_ptr<const Camera> camera;
    std::shared_ptr<Sampler> sampler;
    std::unique_ptr<PathIntegrator> integrator;
    std::unique_ptr<Transform> c2w;
};

RenderObjects makeRenderObjects(const RefScene &rs, const pb2_camera *cam, const pb2_film_desc *fd,
                                const pb2_path_params *pp) {
    RenderObjects ro;
    Point2i res(fd->full_resolution[0], fd->full_resolution[1]);
    // Film takes a fractional crop window and ceil()s it (film.cpp:55-60); aim half a pixel low so
    // that the ceil lands exactly on the integer bounds of the description.
    Bounds2f crop(Point2f((fd->cropped_pixel_bounds[0] - 0.5f) / res.x, (fd->cropped_pixel_bounds[1] - 0.5f) / res.y),
                  Point2f((fd->cropped_pixel_bounds[2] - 0.5f) / res.x, (fd->cropped_pixel_bounds[3] - 0.5f) / res.y));
    crop.pMin.x = std::max(crop.pMin.x, 0.f);
    crop.pMin.y = std::max(crop.pMin.y, 0.f);
    const Vector2f radius(fd->filter_radius[0], fd->filter_radius[1]);
    std::unique_ptr<Filter> filter;
    switch (fd->filter_type) {
    case PB2_FILTER_GAUSSIAN: filter.reset(new GaussianFilter(radius, fd->filter_param[0])); break;
    case PB2_FILTER_MITCHELL: filter.reset(new MitchellFilter(radius, fd->filter_param[0], fd->filter_param[1])); break;
    case PB2_FILTER_SINC: filter.reset(new LanczosSincFilter(radius, fd->filter_param[0])); break;
    case PB2_FILTER_TRIANGLE: filter.reset(new TriangleFilter(radius)); break;
    default: filter.reset(new BoxFilter(radius)); break;
    }
    ro.film = new Film(res, crop, std::move(filter), 35.f, "ref.pfm", fd->scale, fd->max_sample_luminance);
    CHECK_EQ(ro.film->croppedPixelBounds.pMin.x, fd->cropped_pixel_bounds[0]);
    CHECK_EQ(ro.film->croppedPixelBounds.pMin.y, fd->cropped_pixel_bounds[1]);
    CHECK_EQ(ro.film->croppedPixelBounds.pMax.x, fd->cropped_pixel_bounds[2]);
    CHECK_EQ(ro.film->croppedPixelBounds.pMax.y, fd->cropped_pixel_bounds[3]);
    ro.c2w.reset(new Transform(fromMatrices(cam->camera_to_world, cam->world_to_camera)));
    AnimatedTransform ac2w(ro.c2w.get(), 0.f, ro.c2w.get(), 1.f);
    Bounds2f screen(Point2f(cam->screen_window[0], cam->screen_window[2]), Point2f(cam->screen_window[1], cam->screen_window[3]));
    ro.camera.reset(new PerspectiveCamera(ac2w, screen, cam->shutter_open, cam->shutter_close, cam->lens_radius,
                                          cam->focal_distance, cam->fov, ro.film, nullptr));
    if (pp->sampler == PB2_SAMPLER_SOBOL) ro.sampler.reset(new SobolSampler(pp->samples_per_pixel, ro.film->GetSampleBounds()));
    else ro.sampler.reset(new HaltonSampler(pp->samples_per_pixel, ro.film->GetSampleBounds(), pp->sample_at_pixel_center != 0));
    Bounds2i pb(Point2i(pp->pixel_bounds[0], pp->pixel_bounds[1]), Point2i(pp->pixel_bounds[2], pp->pixel_bounds[3]));
    ro.integrator.reset(new PathIntegrator(pp->max_depth, ro.camera, ro.sampler, pb, pp->rr_threshold,
                                           strategyName(rs.lightStrategy)));
    return ro;
}

void setThreads(int n) {
    static int current = -1;
    if (n <= 0) n = (int)std::max(1u, std::thread::hardware_concurrency());
    if (n == current) return;
    if (current != -1) ParallelCleanup();
    else std::atexit([] { ParallelCleanup(); });  // worker threads must be joined before static destructors run
    PbrtOptions.nThreads = n;
    PbrtOptions.quiet = true;
    ParallelInit();
    current = n;
}

uint64_t parseStat(const std::string &text, const char *label) {
    size_t p = text.find(label);
    if (p == std::string::npos) return 0;
    p += std::strlen(label);
    while (p < text.size() && (text[p] == ' ' || text[p] == '\t')) ++p;
    return std::strtoull(text.c_str() + p, nullptr, 10);
}

}  // namespace

// One pb2_texture as a reference texture: the reference's own MIPMap (pyramid construction, trilinear / EWA look-up) behind
// the reference's UVMapping2D, evaluated the way ImageTexture::Evaluate does (imagemap.h:83-89).  ImageTexture itself is
// not used because its constructor reads a file (ReadImage: imageio.cpp needs OpenEXR and is not compiled here); the
// description already holds what ImageTexture::GetTexture would hand to the MIPMap constructor.
template <typename Tmem, typename Tret>
class DescImageTexture : public Texture<Tret> {
  public:
    explicit DescImageTexture(const pb2_texture &t) : mapping(new UVMapping2D(t.su, t.sv, t.du, t.dv)) {
        std::vector<Tmem> texels((size_t)t.width * t.height);
        for (size_t i = 0; i < texels.size(); ++i) texels[i] = load(t.texels + i * t.channels);
        const ImageWrap wrap = t.wrap == PB2_WRAP_BLACK ? ImageWrap::Black : t.wrap == PB2_WRAP_CLAMP ? ImageWrap::Clamp : ImageWrap::Repeat;
        mipmap.reset(new MIPMap<Tmem>(Point2i(t.width, t.height), texels.data(), t.do_trilinear != 0, t.max_anisotropy, wrap));
    }
    Tret Evaluate(const SurfaceInteraction &si) const override {
        Vector2f dstdx, dstdy;
        Point2f st = mapping->Map(si, &dstdx, &dstdy);
        return convertOut(mipmap->Lookup(st, dstdx, dstdy));
    }

  private:
    static Float load(const float *p) { return *p; }
    static Float convertOut(Float v) { return v; }
    static Spectrum convertOut(const RGBSpectrum &from) {   // imagemap.h:107-111
        Float rgb[3];
        from.ToRGB(rgb);
        return Spectrum::FromRGB(rgb);
    }
    std::unique_ptr<TextureMapping2D> mapping;
    std::unique_ptr<MIPMap<Tmem>> mipmap;
};
template <>
DescImageTexture<RGBSpectrum, Spectrum>::DescImageTexture(const pb2_texture &t) : mapping(new UVMapping2D(t.su, t.sv, t.du, t.dv)) {
    std::vector<RGBSpectrum> texels((size_t)t.width * t.height);
    for (size_t i = 0; i < texels.size(); ++i) texels[i] = RGBSpectrum::FromRGB(t.texels + 3 * i);
    const ImageWrap wrap = t.wrap == PB2_WRAP_BLACK ? ImageWrap::Black : t.wrap == PB2_WRAP_CLAMP ? ImageWrap::Clamp : ImageWrap::Repeat;
    mipmap.reset(new MIPMap<RGBSpectrum>(Point2i(t.width, t.height), texels.data(), t.do_trilinear != 0, t.max_anisotropy, wrap));
}

// The reference's texture objects for a description's texture array (images through the reference's MIPMap, the other kinds
// as the reference's own ConstantTexture / ScaleTexture / MixTexture / Checkerboard2DTexture / UVTexture)
static void buildRefTextures(const pb2_scene_desc *d, std::vector<std::shared_ptr<Texture<Float>>> &floatTex,
                             std::vector<std::shared_ptr<Texture<Spectrum>>> &specTex) {
    // image textures (the MIPMap constructor runs ParallelFors: the thread pool must exist, parallel.cpp:186)
    floatTex.assign(d->n_textures, nullptr);
    specTex.assign(d->n_textures, nullptr);
    if (d->n_textures > 0) setThreads(0);
    for (int i = 0; i < d->n_textures; ++i) {
        const pb2_texture &pt = d->textures[i];
        const bool one = pt.channels == 1;
        if (pt.kind == PB2_TEXKIND_CONSTANT) {
            if (one) floatTex[i] = std::make_shared<ConstantTexture<Float>>(pt.value[0]);
            else specTex[i] = std::make_shared<ConstantTexture<Spectrum>>(Spectrum::FromRGB(pt.value));
        } else if (pt.kind == PB2_TEXKIND_SCALE) {   // the reference's own ScaleTexture / MixTexture over the children
            if (one) floatTex[i] = std::make_shared<ScaleTexture<Float, Float>>(floatTex[pt.child[0] - 1], floatTex[pt.child[1] - 1]);
            else specTex[i] = std::make_shared<ScaleTexture<Spectrum, Spectrum>>(specTex[pt.child[0] - 1], specTex[pt.child[1] - 1]);
        } else if (pt.kind == PB2_TEXKIND_MIX) {
            if (one) floatTex[i] = std::make_shared<MixTexture<Float>>(floatTex[pt.child[0] - 1], floatTex[pt.child[1] - 1], floatTex[pt.child[2] - 1]);
            else specTex[i] = std::make_shared<MixTexture<Spectrum>>(specTex[pt.child[0] - 1], specTex[pt.child[1] - 1], floatTex[pt.child[2] - 1]);
        } else if (pt.kind == PB2_TEXKIND_CHECKERBOARD) {
            const AAMethod aa = pt.value[0] == 0 ? AAMethod::None : AAMethod::ClosedForm;
            std::unique_ptr<TextureMapping2D> map(new UVMapping2D(pt.su, pt.sv, pt.du, pt.dv));
            if (one) floatTex[i] = std::make_shared<Checkerboard2DTexture<Float>>(std::move(map), floatTex[pt.child[0] - 1], floatTex[pt.child[1] - 1], aa);
            else specTex[i] = std::make_shared<Checkerboard2DTexture<Spectrum>>(std::move(map), specTex[pt.child[0] - 1], specTex[pt.child[1] - 1], aa);
        } else if (pt.kind == PB2_TEXKIND_UV) {
            specTex[i] = std::make_shared<UVTexture>(std::unique_ptr<TextureMapping2D>(new UVMapping2D(pt.su, pt.sv, pt.du, pt.dv)));
        } else if (one) floatTex[i] = std::make_shared<DescImageTexture<Float, Float>>(pt);
        else specTex[i] = std::make_shared<DescImageTexture<RGBSpectrum, Spectrum>>(pt);
    }

}
// The reference's Material object for one record: every parameter is the record's constant, or the texture its slot names
static std::shared_ptr<Material> makeRefMaterial(const pb2_material &pm, const std::vector<std::shared_ptr<Texture<Float>>> &floatTex,
                                                 const std::vector<std::shared_ptr<Texture<Spectrum>>> &specTex) {
    auto spec = [&](int slot, const float *c) -> std::shared_ptr<Texture<Spectrum>> {
        if (pm.tex[slot]) return specTex[pm.tex[slot] - 1];
        return std::make_shared<ConstantTexture<Spectrum>>(Spectrum::FromRGB(c));
    };
    auto flt = [&](int slot, float v) -> std::shared_ptr<Texture<Float>> {
        if (pm.tex[slot]) return floatTex[pm.tex[slot] - 1];
        return std::make_shared<ConstantTexture<Float>>(v);
    };
    auto kd = spec(PB2_TEX_KD, pm.kd);
    std::shared_ptr<Texture<Float>> bump = pm.tex[PB2_TEX_BUMP] ? floatTex[pm.tex[PB2_TEX_BUMP] - 1] : nullptr;
    if (pm.type == PB2_MAT_MATTE) {
        return std::make_shared<MatteMaterial>(kd, flt(PB2_TEX_SIGMA, pm.sigma), bump);
    } else if (pm.type == PB2_MAT_PLASTIC) {
        return std::make_shared<PlasticMaterial>(kd, spec(PB2_TEX_KS, pm.ks), flt(PB2_TEX_ROUGHNESS, pm.roughness), bump,
                                                         pm.remap_roughness != 0);
    } else if (pm.type == PB2_MAT_MIRROR) {
        return std::make_shared<MirrorMaterial>(spec(PB2_TEX_KR, pm.kr), bump);
    } else if (pm.type == PB2_MAT_SUBSTRATE) {
        return std::make_shared<SubstrateMaterial>(kd, spec(PB2_TEX_KS, pm.ks), flt(PB2_TEX_UROUGHNESS, pm.uroughness),
                                                           flt(PB2_TEX_VROUGHNESS, pm.vroughness), bump, pm.remap_roughness != 0);
    } else if (pm.type == PB2_MAT_UBER) {
        // the description carries the resolved u / v roughness (pb2.h); "roughness" itself is then never read
        return std::make_shared<UberMaterial>(kd, spec(PB2_TEX_KS, pm.ks), spec(PB2_TEX_KR, pm.kr), spec(PB2_TEX_KT, pm.kt),
                                                      flt(PB2_TEX_UROUGHNESS, pm.uroughness), flt(PB2_TEX_UROUGHNESS, pm.uroughness),
                                                      flt(PB2_TEX_VROUGHNESS, pm.vroughness), spec(PB2_TEX_OPACITY, pm.opacity),
                                                      flt(PB2_TEX_ETA, pm.eta), bump, pm.remap_roughness != 0);
    } else if (pm.type == PB2_MAT_METAL) {
        return std::make_shared<MetalMaterial>(spec(PB2_TEX_METAL_ETA, pm.metal_eta), spec(PB2_TEX_METAL_K, pm.metal_k),
                                                       flt(PB2_TEX_UROUGHNESS, pm.uroughness), flt(PB2_TEX_UROUGHNESS, pm.uroughness),
                                                       flt(PB2_TEX_VROUGHNESS, pm.vroughness), bump, pm.remap_roughness != 0);
    } else if (pm.type == PB2_MAT_GLASS) {
        return std::make_shared<GlassMaterial>(spec(PB2_TEX_KR, pm.kr), spec(PB2_TEX_KT, pm.kt), flt(PB2_TEX_UROUGHNESS, pm.uroughness),
                                                       flt(PB2_TEX_VROUGHNESS, pm.vroughness), flt(PB2_TEX_ETA, pm.eta), bump,
                                                       pm.remap_roughness != 0);
    }
    return nullptr;
}
extern "C" {

const char *ref_kind(void) { return "reference"; }

// Device math for the evaluation entry points (see DeviceMathScope); returns the previous setting
int ref_set_device_math(int on) {
    const int was = g_deviceMathMode;
    g_deviceMathMode = on != 0;
    return was;
}

// The six wrapped functions as the reference's own code calls them, under the current device-math setting.
// fn: 0 sinf, 1 cosf, 2 sincosf (sin, cos per element), 3 logf, 4 atan2f(y = a, x = b), 5 acosf.
int ref_transcendentals(int fn, int64_t n, const float *a, const float *b, float *out) {
    DeviceMathScope dm;
    for (int64_t i = 0; i < n; ++i) {
        switch (fn) {
        case 0: out[i] = sinf(a[i]); break;
        case 1: out[i] = cosf(a[i]); break;
        case 2: sincosf(a[i], &out[2 * i], &out[2 * i + 1]); break;
        case 3: out[i] = logf(a[i]); break;
        case 4: out[i] = atan2f(a[i], b[i]); break;
        case 5: out[i] = acosf(a[i]); break;
        default: return 1;
        }
    }
    return 0;
}

// MIPMap<T>::pyramid[level] of the reference for one texture description (row-major, channels floats per texel)
int ref_texture_pyramid(const pb2_texture *t, int level, int *n_levels, int *w, int *h, float *out) {
    setThreads(0);
    const ImageWrap wrap = t->wrap == PB2_WRAP_BLACK ? ImageWrap::Black : t->wrap == PB2_WRAP_CLAMP ? ImageWrap::Clamp : ImageWrap::Repeat;
    const size_t n = (size_t)t->width * t->height;
    if (t->channels == 1) {
        MIPMap<Float> mm(Point2i(t->width, t->height), t->texels, t->do_trilinear != 0, t->max_anisotropy, wrap);
        *n_levels = mm.Levels();
        if (level < 0 || level >= mm.Levels()) return 1;
        *w = mm.pyramid[level]->uSize();
        *h = mm.pyramid[level]->vSize();
        if (out)
            for (int y = 0; y < *h; ++y)
                for (int x = 0; x < *w; ++x) out[(size_t)y * *w + x] = (*mm.pyramid[level])(x, y);
    } else {
        std::vector<RGBSpectrum> texels(n);
        for (size_t i = 0; i < n; ++i) texels[i] = RGBSpectrum::FromRGB(t->texels + 3 * i);
        MIPMap<RGBSpectrum> mm(Point2i(t->width, t->height), texels.data(), t->do_trilinear != 0, t->max_anisotropy, wrap);
        *n_levels = mm.Levels();
        if (level < 0 || level >= mm.Levels()) return 1;
        *w = mm.pyramid[level]->uSize();
        *h = mm.pyramid[level]->vSize();
        if (out)
            for (int y = 0; y < *h; ++y)
                for (int x = 0; x < *w; ++x) (*mm.pyramid[level])(x, y).ToRGB(out + 3 * ((size_t)y * *w + x));
    }
    return 0;
}
// InfiniteAreaLight::distribution of the reference for an environment map given as a texture description, in the layout of
// pb2_env_distribution: nv rows of [func | cdf | funcInt], then the marginal
int ref_env_distribution(const pb2_texture *t, int *nu, int *nv, float *out) {
    setThreads(0);
    const std::string name = "pb2env:probe";
    {
        std::lock_guard<std::mutex> lock(g_registryMutex);
        RegisteredImage &im = g_imageRegistry[name];
        im.w = t->width;
        im.h = t->height;
        im.rgb.assign(t->texels, t->texels + (size_t)3 * t->width * t->height);
    }
    InfiniteAreaLight light(Transform(), Spectrum(1.f), 1, name);
    {
        std::lock_guard<std::mutex> lock(g_registryMutex);
        g_imageRegistry.erase(name);
    }
    const Distribution2D &d2 = *light.distribution;
    *nu = d2.pConditionalV[0]->Count();
    *nv = d2.pMarginal->Count();
    if (!out) return 0;
    auto put = [&](const Distribution1D &d, float *dst) {
        const int n = d.Count();
        for (int i = 0; i < n; ++i) dst[i] = d.func[i];
        for (int i = 0; i <= n; ++i) dst[n + i] = d.cdf[i];
        dst[2 * n + 1] = d.funcInt;
    };
    const size_t stride = 2 * (size_t)*nu + 2;
    for (int v = 0; v < *nv; ++v) put(*d2.pConditionalV[v], out + (size_t)v * stride);
    put(*d2.pMarginal, out + (size_t)*nv * stride);
    return 0;
}

// MIPMap<T>::Lookup(st, dst0, dst1) of the reference for a batch (st: 2 floats, dst: 4, out: 3 per look-up)
int ref_texture_lookup(const pb2_texture *t, int64_t n, const float *st, const float *dst, float *out) {
    setThreads(0);
    const ImageWrap wrap = t->wrap == PB2_WRAP_BLACK ? ImageWrap::Black : t->wrap == PB2_WRAP_CLAMP ? ImageWrap::Clamp : ImageWrap::Repeat;
    const size_t nt = (size_t)t->width * t->height;
    if (t->channels == 1) {
        MIPMap<Float> mm(Point2i(t->width, t->height), t->texels, t->do_trilinear != 0, t->max_anisotropy, wrap);
        DeviceMathScope dm;
        for (int64_t i = 0; i < n; ++i) {
            Float v = mm.Lookup(Point2f(st[2 * i], st[2 * i + 1]), Vector2f(dst[4 * i], dst[4 * i + 1]), Vector2f(dst[4 * i + 2], dst[4 * i + 3]));
            out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = v;
        }
    } else {
        std::vector<RGBSpectrum> texels(nt);
        for (size_t i = 0; i < nt; ++i) texels[i] = RGBSpectrum::FromRGB(t->texels + 3 * i);
        MIPMap<RGBSpectrum> mm(Point2i(t->width, t->height), texels.data(), t->do_trilinear != 0, t->max_anisotropy, wrap);
        DeviceMathScope dm;
        for (int64_t i = 0; i < n; ++i)
            mm.Lookup(Point2f(st[2 * i], st[2 * i + 1]), Vector2f(dst[4 * i], dst[4 * i + 1]), Vector2f(dst[4 * i + 2], dst[4 * i + 3])).ToRGB(out + 3 * i);
    }
    return 0;
}

// Texture::Evaluate of the reference for texture `id` at points given by (u, v) and (dudx, dvdx, dudy, dvdy)
int ref_texture_evaluate(const pb2_texture *textures, int n_textures, int id, int64_t n, const float *uv, const float *duv, float *out) {
    pb2_scene_desc d;
    std::memset(&d, 0, sizeof(d));
    d.n_textures = n_textures;
    d.textures = textures;
    std::vector<std::shared_ptr<Texture<Float>>> floatTex;
    std::vector<std::shared_ptr<Texture<Spectrum>>> specTex;
    buildRefTextures(&d, floatTex, specTex);
    DeviceMathScope dm;
    for (int64_t i = 0; i < n; ++i) {
        SurfaceInteraction si;
        si.uv = Point2f(uv[2 * i], uv[2 * i + 1]);
        si.dudx = duv[4 * i];
        si.dvdx = duv[4 * i + 1];
        si.dudy = duv[4 * i + 2];
        si.dvdy = duv[4 * i + 3];
        if (textures[id].channels == 1) out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = floatTex[id]->Evaluate(si);
        else specTex[id]->Evaluate(si).ToRGB(out + 3 * i);
    }
    return 0;
}

// The reference's BSDF for one material record at given shading frames (Material::ComputeScatteringFunctions with
// allowMultipleLobes = true, path.cpp:106), evaluated the way EstimateDirect and the path's continuation do.  Layout of
// in / out: pb2_bsdf_eval_host (include/pb2.h).
int ref_bsdf_eval(const pb2_material *pm, int64_t n, const float *in, float *out) {
    std::vector<std::shared_ptr<Texture<Float>>> floatTex;
    std::vector<std::shared_ptr<Texture<Spectrum>>> specTex;
    std::shared_ptr<Material> material = makeRefMaterial(*pm, floatTex, specTex);
    MemoryArena arena;
    const BxDFType nonSpecular = BxDFType(BSDF_ALL & ~BSDF_SPECULAR);
    DeviceMathScope dm;
    for (int64_t i = 0; i < n; ++i) {
        const float *q = in + 17 * i;
        float *o = out + 19 * i;
        for (int k = 0; k < 19; ++k) o[k] = 0;
        if (!material) continue;
        SurfaceInteraction si;
        si.n = Normal3f(q[0], q[1], q[2]);
        si.shading.n = Normal3f(q[3], q[4], q[5]);
        si.dpdu = si.shading.dpdu = Vector3f(q[6], q[7], q[8]);
        const Vector3f wo(q[9], q[10], q[11]), wi(q[12], q[13], q[14]);
        si.wo = wo;
        const Point2f u(q[15], q[16]);
        material->ComputeScatteringFunctions(&si, arena, TransportMode::Radiance, true);
        if (!si.bsdf) continue;
        Float rgb[3];
        if (si.bsdf->NumComponents(nonSpecular) > 0) {
            si.bsdf->f(wo, wi, nonSpecular).ToRGB(rgb);
            o[0] = rgb[0]; o[1] = rgb[1]; o[2] = rgb[2];
            o[3] = si.bsdf->Pdf(wo, wi, nonSpecular);
            Vector3f wiS;
            Float pdfS = 0;
            BxDFType sampled;
            Spectrum fS = si.bsdf->Sample_f(wo, &wiS, u, &pdfS, nonSpecular, &sampled);
            if (pdfS != 0) { o[4] = wiS.x; o[5] = wiS.y; o[6] = wiS.z; }
            fS.ToRGB(rgb);
            o[7] = rgb[0]; o[8] = rgb[1]; o[9] = rgb[2];
            o[10] = pdfS;
        }
        Vector3f wiC;
        Float pdfC = 0;
        BxDFType flags = BxDFType(0);
        Spectrum fC = si.bsdf->Sample_f(wo, &wiC, u, &pdfC, BSDF_ALL, &flags);
        if (pdfC != 0) { o[11] = wiC.x; o[12] = wiC.y; o[13] = wiC.z; }
        fC.ToRGB(rgb);
        o[14] = rgb[0]; o[15] = rgb[1]; o[16] = rgb[2];
        o[17] = pdfC;
        o[18] = (Float)(((flags & BSDF_SPECULAR) ? 1 : 0) | ((flags & BSDF_TRANSMISSION) ? 2 : 0));
        arena.Reset();
    }
    return 0;
}

void *ref_scene_create(const pb2_scene_desc *d, int max_prims_in_node, int split_method) {
    std::unique_ptr<RefScene> rs(new RefScene);
    rs->transforms.emplace_back(new Transform());
    const Transform *identity = rs->transforms.back().get();
    rs->lightStrategy = d->light_strategy;
    std::vector<std::shared_ptr<Texture<Float>>> floatTex;
    std::vector<std::shared_ptr<Texture<Spectrum>>> specTex;
    buildRefTextures(d, floatTex, specTex);
    // shapes
    std::vector<std::vector<std::shared_ptr<Shape>>> meshShapes(d->n_meshes);
    for (int m = 0; m < d->n_meshes; ++m) {
        const pb2_mesh &pm = d->meshes[m];
        std::vector<int> local(3 * (size_t)pm.n_tris);
        for (size_t i = 0; i < local.size(); ++i) local[i] = d->tri_index[3 * (size_t)pm.first_tri + i] - pm.first_vertex;
        const Point3f *P = reinterpret_cast<const Point3f *>(d->P) + pm.first_vertex;
        const Normal3f *N = (pm.has_n && d->N) ? reinterpret_cast<const Normal3f *>(d->N) + pm.first_vertex : nullptr;
        const Point2f *UV = (pm.has_uv && d->UV) ? reinterpret_cast<const Point2f *>(d->UV) + pm.first_vertex : nullptr;
        const Vector3f *S = (pm.has_s && d->S) ? reinterpret_cast<const Vector3f *>(d->S) + pm.first_vertex : nullptr;
        // Vertices/normals in the description are already in world space, so the mesh is rebuilt
        // under the identity transform (which maps every finite float to itself).
        meshShapes[m] = CreateTriangleMesh(identity, identity, pm.reverse_orientation != 0, pm.n_tris, local.data(),
                                           pm.n_vertices, P, S, N, UV, pm.alpha_tex ? floatTex[pm.alpha_tex - 1] : nullptr,
                                           pm.shadow_alpha_tex ? floatTex[pm.shadow_alpha_tex - 1] : nullptr, nullptr);
        for (auto &s : meshShapes[m])
            const_cast<bool &>(s->transformSwapsHandedness) = pm.transform_swaps_handedness != 0;
    }
    std::vector<std::shared_ptr<Shape>> sphereShapes(d->n_spheres);
    for (int s = 0; s < d->n_spheres; ++s) {
        const pb2_sphere &ps = d->spheres[s];
        rs->transforms.emplace_back(new Transform(fromMatrices(ps.object_to_world, ps.world_to_object)));
        const Transform *o2w = rs->transforms.back().get();
        rs->transforms.emplace_back(new Transform(fromMatrices(ps.world_to_object, ps.object_to_world)));
        const Transform *w2o = rs->transforms.back().get();
        auto sp = std::make_shared<Sphere>(o2w, w2o, ps.reverse_orientation != 0, ps.radius, ps.z_min, ps.z_max, 360.f);
        const_cast<Float &>(sp->thetaMin) = ps.theta_min;
        const_cast<Float &>(sp->thetaMax) = ps.theta_max;
        const_cast<Float &>(sp->phiMax) = ps.phi_max;
        const_cast<bool &>(sp->transformSwapsHandedness) = ps.transform_swaps_handedness != 0;
        sphereShapes[s] = sp;
    }
    // materials
    std::vector<std::shared_ptr<Material>> materials(d->n_materials);
    for (int i = 0; i < d->n_materials; ++i) materials[i] = makeRefMaterial(d->materials[i], floatTex, specTex);
    // primitives + lights (lights indexed as in the description = Scene::lights order)
    rs->lights.resize(d->n_lights);
    rs->prims.resize(d->n_prims);
    for (int64_t i = 0; i < d->n_prims; ++i) {
        if (d->prim_type[i] == PB2_PRIM_INSTANCE) continue;   // TransformedPrimitives are made below
        std::shared_ptr<Shape> shape;
        if (d->prim_type[i] == PB2_PRIM_TRIANGLE) {
            int tri = d->prim_index[i];
            int m = d->tri_mesh[tri];
            shape = meshShapes[m][tri - d->meshes[m].first_tri];
        } else
            shape = sphereShapes[d->prim_index[i]];
        std::shared_ptr<Material> mtl = d->prim_material[i] >= 0 ? materials[d->prim_material[i]] : nullptr;
        std::shared_ptr<AreaLight> area;
        if (d->prim_light[i] >= 0) {
            const pb2_light &pl = d->lights[d->prim_light[i]];
            area = std::make_shared<DiffuseAreaLight>(*identity, MediumInterface(), Spectrum::FromRGB(pl.L), 1, shape,
                                                      pl.two_sided != 0);
            rs->lights[d->prim_light[i]] = area;
        }
        rs->prims[i] = std::make_shared<GeometricPrimitive>(shape, mtl, area, MediumInterface());
        rs->primNumber[rs->prims[i].get()] = (int)i;
    }
    BVHAccel::SplitMethod sm = split_method == 1 ? BVHAccel::SplitMethod::HLBVH
                             : split_method == 2 ? BVHAccel::SplitMethod::Middle
                             : split_method == 3 ? BVHAccel::SplitMethod::EqualCounts
                                                 : BVHAccel::SplitMethod::SAH;
    const int maxPrims = max_prims_in_node > 0 ? max_prims_in_node : 4;
    if (d->n_instances > 0) {
        // Object instancing as pbrtObjectInstance does it (api.cpp:1547-1588): one accelerator per
        // instanced object over its GeometricPrimitives in creation order (= ascending primitive
        // number), or the lone primitive itself; one TransformedPrimitive per instance.
        std::vector<std::shared_ptr<Primitive>> objectAccel(d->n_bvhs > 0 ? d->n_bvhs : 1);
        for (int k = 1; k < d->n_bvhs; ++k) {
            std::vector<int32_t> numbers(d->bvh_prims + d->bvhs[k].prim_offset, d->bvh_prims + d->bvhs[k].prim_offset + d->bvhs[k].n_prims);
            std::sort(numbers.begin(), numbers.end());
            std::vector<std::shared_ptr<Primitive>> objPrims;
            for (int32_t n : numbers) objPrims.push_back(rs->prims[n]);
            objectAccel[k] = std::make_shared<BVHAccel>(objPrims, maxPrims, sm);
        }
        for (int64_t i = 0; i < d->n_prims; ++i) {
            if (d->prim_type[i] != PB2_PRIM_INSTANCE) continue;
            const pb2_instance &pi = d->instances[d->prim_index[i]];
            rs->transforms.emplace_back(new Transform(fromMatrices(pi.instance_to_world, pi.world_to_instance)));
            const Transform *i2w = rs->transforms.back().get();
            std::shared_ptr<Primitive> inner = pi.bvh >= 1 ? objectAccel[pi.bvh] : rs->prims[d->bvh_prims[pi.lone_prim]];
            AnimatedTransform anim(i2w, 0, i2w, 1);
            rs->prims[i] = std::make_shared<TransformedPrimitive>(inner, anim);
            rs->primNumber[rs->prims[i].get()] = (int)i;
        }
        // Scene::aggregate is built over the scene-level primitives only: the first bvhs[0].n_prims numbers
        std::vector<std::shared_ptr<Primitive>> top(rs->prims.begin(), rs->prims.begin() + d->bvhs[0].n_prims);
        rs->bvh = std::make_shared<BVHAccel>(top, maxPrims, sm);
    } else
        rs->bvh = std::make_shared<BVHAccel>(rs->prims, maxPrims, sm);
    // delta lights, built through the reference's own constructors.  The description carries what the constructors
    // derive from LightToWorld (pLight; the 3x3 of WorldToLight; LightToWorld(from - to)), so LightToWorld is rebuilt as
    // a translation to pLight whose inverse holds the recorded WorldToLight rows (Falloff only transforms a vector).
    for (int i = 0; i < d->n_lights; ++i) {
        const pb2_light &pl = d->lights[i];
        if (pl.type == PB2_LIGHT_AREA) continue;
        const pb2_delta_light &dl = d->delta_lights[i];
        Spectrum I = Spectrum::FromRGB(pl.L);
        if (pl.type == PB2_LIGHT_POINT)
            rs->lights[i] = std::make_shared<PointLight>(Translate(Vector3f(dl.p[0], dl.p[1], dl.p[2])), MediumInterface(), I);
        else if (pl.type == PB2_LIGHT_SPOT) {
            Matrix4x4 m = Translate(Vector3f(dl.p[0], dl.p[1], dl.p[2])).GetMatrix(), mInv;
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) mInv.m[r][c] = dl.world_to_light[3 * r + c];
            rs->lights[i] = std::make_shared<SpotLight>(Transform(m, mInv), MediumInterface(), I, dl.total_width_deg, dl.falloff_start_deg);
        } else if (pl.type == PB2_LIGHT_INFINITE) {
            // the reference's own InfiniteAreaLight without a texture map; Le / Sample_Li / Pdf_Li only transform vectors.
            // Its constructor runs a ParallelFor (infinite.cpp:71-81): the thread pool must exist (parallel.cpp:186)
            setThreads(0);
            Matrix4x4 m, mInv;
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) {
                    m.m[r][c] = dl.light_to_world[3 * r + c];
                    mInv.m[r][c] = dl.world_to_light[3 * r + c];
                }
            std::string mapName;
            Spectrum Linf = I;
            if (dl.env_tex) {
                // the description's texels are already ReadImage(mapname) * L: the constructor multiplies them by L = 1
                const pb2_texture &pt = d->textures[dl.env_tex - 1];
                mapName = "pb2env:" + std::to_string((long long)(size_t)rs.get()) + ":" + std::to_string(i);
                std::lock_guard<std::mutex> lock(g_registryMutex);
                RegisteredImage &im = g_imageRegistry[mapName];
                im.w = pt.width;
                im.h = pt.height;
                im.rgb.assign(pt.texels, pt.texels + (size_t)3 * pt.width * pt.height);
                Linf = Spectrum(1.f);
            }
            rs->lights[i] = std::make_shared<InfiniteAreaLight>(Transform(m, mInv), Linf, 1, mapName);
            if (dl.env_tex) {
                std::lock_guard<std::mutex> lock(g_registryMutex);
                g_imageRegistry.erase(mapName);
            }
        } else
            rs->lights[i] = std::make_shared<DistantLight>(Transform(), I, Vector3f(dl.p[0], dl.p[1], dl.p[2]));
    }
    rs->scene.reset(new Scene(rs->bvh, rs->lights));
    return rs.release();
}

void ref_scene_destroy(void *h) { delete static_cast<RefScene *>(h); }

// Copies the reference's own LinearBVHNode array and ordered primitive numbers.
int64_t ref_bvh_dump(void *h, pb2_bvh_node *out_nodes, int64_t max_nodes, int32_t *out_prims) {
    RefScene *rs = static_cast<RefScene *>(h);
    // node count: walk depth first
    const LinearBVHNode *nodes = reinterpret_cast<const LinearBVHNode *>(rs->bvh->nodes);
    if (!nodes) return 0;
    int64_t count = 0;
    {
        std::vector<int> stack{0};
        while (!stack.empty()) {
            int i = stack.back();
            stack.pop_back();
            count = std::max<int64_t>(count, i + 1);
            if (nodes[i].nPrimitives == 0) {
                stack.push_back(i + 1);
                stack.push_back(nodes[i].secondChildOffset);
            }
        }
    }
    static_assert(sizeof(LinearBVHNode) == sizeof(pb2_bvh_node), "node layouts differ");
    if (out_nodes) std::memcpy(out_nodes, nodes, sizeof(pb2_bvh_node) * (size_t)std::min(count, max_nodes));
    if (out_prims)
        for (size_t j = 0; j < rs->bvh->primitives.size(); ++j) out_prims[j] = rs->primNumber[rs->bvh->primitives[j].get()];
    return count;
}

int ref_intersect(void *h, const pb2_ray *rays, int64_t n, pb2_hit *hits) {
    RefScene *rs = static_cast<RefScene *>(h);
    DeviceMathScope dm;
    for (int64_t i = 0; i < n; ++i) {
        Ray ray(Point3f(rays[i].o[0], rays[i].o[1], rays[i].o[2]), Vector3f(rays[i].d[0], rays[i].d[1], rays[i].d[2]),
                rays[i].t_max);
        SurfaceInteraction isect;
        pb2_hit &o = hits[i];
        std::memset(&o, 0, sizeof(o));
        if (!rs->scene->Intersect(ray, &isect)) {
            o.prim = -1;
            o.t = ray.tMax;
            continue;
        }
        o.prim = rs->primNumber[isect.primitive];
        o.t = ray.tMax;
        for (int k = 0; k < 3; ++k) {
            o.p[k] = isect.p[k];
            o.p_error[k] = isect.pError[k];
            o.n[k] = isect.n[k];
            o.ns[k] = isect.shading.n[k];
            o.dpdu[k] = isect.shading.dpdu[k];
        }
        o.uv[0] = isect.uv[0];
        o.uv[1] = isect.uv[1];
        // barycentrics are not part of SurfaceInteraction; with the default (0,0),(1,0),(1,1)
        // parameterisation (triangle.h:98-108) uv = (b1+b2, b2), which tests use instead.
    }
    return 0;
}

int ref_intersect_p(void *h, const pb2_ray *rays, int64_t n, uint8_t *occluded) {
    RefScene *rs = static_cast<RefScene *>(h);
    DeviceMathScope dm;
    for (int64_t i = 0; i < n; ++i) {
        Ray ray(Point3f(rays[i].o[0], rays[i].o[1], rays[i].o[2]), Vector3f(rays[i].d[0], rays[i].d[1], rays[i].d[2]),
                rays[i].t_max);
        occluded[i] = rs->scene->IntersectP(ray) ? 1 : 0;
    }
    return 0;
}

// SamplerIntegrator::Render with the reference's thread pool.  out_rgb: 3 floats per cropped pixel
// (what Film::WriteImage hands to the image encoder).  seconds: wall time of Render().
int ref_render(void *h, const pb2_camera *cam, const pb2_film_desc *fd, const pb2_path_params *pp, int n_threads,
               float *out_rgb, double *seconds, pb2_stats *stats) {
    RefScene *rs = static_cast<RefScene *>(h);
    setThreads(n_threads);
    RenderObjects ro = makeRenderObjects(*rs, cam, fd, pp);
    ReportThreadStats();  // flush this thread's counters from earlier calls, then start from zero
    ClearStats();
    auto t0 = std::chrono::steady_clock::now();
    {
        DeviceMathScope dm;
        ro.integrator->Render(*rs->scene);
    }
    auto t1 = std::chrono::steady_clock::now();
    if (seconds) *seconds = std::chrono::duration<double>(t1 - t0).count();
    {
        std::lock_guard<std::mutex> lock(g_imageMutex);
        if (out_rgb) std::memcpy(out_rgb, g_lastImage.data(), g_lastImage.size() * sizeof(float));
    }
    if (stats) {
        std::memset(stats, 0, sizeof(*stats));
        MergeWorkerThreadStats();
        ReportThreadStats();
        char *buf = nullptr;
        size_t len = 0;
        FILE *f = open_memstream(&buf, &len);
        PrintStats(f);
        std::fclose(f);
        std::string text(buf, len);
        free(buf);
        stats->camera_rays = parseStat(text, "Camera rays traced");
        stats->regular_rays = parseStat(text, "Regular ray intersection tests");
        stats->shadow_rays = parseStat(text, "Shadow ray intersection tests");
        stats->render_ms = seconds ? *seconds * 1e3 : 0;
        ClearStats();
    }
    return 0;
}

int ref_li_samples(void *h, const pb2_camera *cam, const pb2_film_desc *fd, const pb2_path_params *pp,
                   const int32_t *pixel_xy, const int64_t *sample_num, int64_t n, float *out_rgb, float *out_pfilm) {
    RefScene *rs = static_cast<RefScene *>(h);
    setThreads(1);
    RenderObjects ro = makeRenderObjects(*rs, cam, fd, pp);
    ro.integrator->Preprocess(*rs->scene, *ro.sampler);
    MemoryArena arena;
    std::unique_ptr<Sampler> sampler = ro.sampler->Clone(0);
    DeviceMathScope dm;
    for (int64_t i = 0; i < n; ++i) {
        Point2i pixel(pixel_xy[2 * i], pixel_xy[2 * i + 1]);
        sampler->StartPixel(pixel);
        sampler->SetSampleNumber(sample_num[i]);
        CameraSample cs = sampler->GetCameraSample(pixel);
        RayDifferential ray;
        Float rayWeight = ro.camera->GenerateRayDifferential(cs, &ray);
        ray.ScaleDifferentials(1 / std::sqrt((Float)sampler->samplesPerPixel));
        Spectrum L(0.f);
        if (rayWeight > 0) L = ro.integrator->Li(ray, *rs->scene, *sampler, arena, 0);
        // integrator.cpp:294-315
        if (L.HasNaNs()) L = Spectrum(0.f);
        else if (L.y() < -1e-5) L = Spectrum(0.f);
        else if (std::isinf(L.y())) L = Spectrum(0.f);
        Float rgb[3];
        L.ToRGB(rgb);
        for (int k = 0; k < 3; ++k) out_rgb[3 * i + k] = rgb[k];
        if (out_pfilm) {
            out_pfilm[2 * i] = cs.pFilm.x;
            out_pfilm[2 * i + 1] = cs.pFilm.y;
        }
        arena.Reset();
    }
    return 0;
}

// The camera ray of each (pixel, sample) with its differentials as SamplerIntegrator::Render hands it to Li, the first
// intersection and what SurfaceInteraction::ComputeDifferentials derives there.  39 floats per sample:
// pFilm(2) pLens(2) o(3) d(3) rxOrigin(3) rxDirection(3) ryOrigin(3) ryDirection(3) hit(1) p(3) n(3) dpdu(3) dpdv(3) dudx dvdx dudy dvdy
int ref_camera_differentials(void *h, const pb2_camera *cam, const pb2_film_desc *fd, const pb2_path_params *pp,
                             const int32_t *pixel_xy, const int64_t *sample_num, int64_t n, float *out) {
    RefScene *rs = static_cast<RefScene *>(h);
    setThreads(1);
    RenderObjects ro = makeRenderObjects(*rs, cam, fd, pp);
    std::unique_ptr<Sampler> sampler = ro.sampler->Clone(0);
    DeviceMathScope dm;
    for (int64_t i = 0; i < n; ++i) {
        float *o = out + 39 * i;
        std::memset(o, 0, 39 * sizeof(float));
        Point2i pixel(pixel_xy[2 * i], pixel_xy[2 * i + 1]);
        sampler->StartPixel(pixel);
        sampler->SetSampleNumber(sample_num[i]);
        CameraSample cs = sampler->GetCameraSample(pixel);
        RayDifferential ray;
        ro.camera->GenerateRayDifferential(cs, &ray);
        ray.ScaleDifferentials(1 / std::sqrt((Float)sampler->samplesPerPixel));
        o[0] = cs.pFilm.x; o[1] = cs.pFilm.y; o[2] = cs.pLens.x; o[3] = cs.pLens.y;
        const Float v[18] = {ray.o.x, ray.o.y, ray.o.z, ray.d.x, ray.d.y, ray.d.z, ray.rxOrigin.x, ray.rxOrigin.y, ray.rxOrigin.z,
                             ray.rxDirection.x, ray.rxDirection.y, ray.rxDirection.z, ray.ryOrigin.x, ray.ryOrigin.y, ray.ryOrigin.z,
                             ray.ryDirection.x, ray.ryDirection.y, ray.ryDirection.z};
        for (int k = 0; k < 18; ++k) o[4 + k] = v[k];
        SurfaceInteraction isect;
        if (!rs->scene->Intersect(ray, &isect)) continue;
        isect.ComputeDifferentials(ray);
        o[22] = 1;
        const Float w[16] = {isect.p.x, isect.p.y, isect.p.z, isect.n.x, isect.n.y, isect.n.z, isect.dpdu.x, isect.dpdu.y, isect.dpdu.z,
                             isect.dpdv.x, isect.dpdv.y, isect.dpdv.z, isect.dudx, isect.dvdx, isect.dudy, isect.dvdy};
        for (int k = 0; k < 16; ++k) o[23 + k] = w[k];
    }
    return 0;
}

int ref_halton_samples(const pb2_film_desc *fd, const pb2_path_params *pp, const int32_t *pixel_xy,
                       const int64_t *sample_num, const int32_t *dim, int64_t n, float *out) {
    // sample bounds as Film::GetSampleBounds() computes them (film.cpp:80-86)
    Bounds2i sb(Point2i((int)std::floor(fd->cropped_pixel_bounds[0] + 0.5f - fd->filter_radius[0]),
                        (int)std::floor(fd->cropped_pixel_bounds[1] + 0.5f - fd->filter_radius[1])),
                Point2i((int)std::ceil(fd->cropped_pixel_bounds[2] - 0.5f + fd->filter_radius[0]),
                        (int)std::ceil(fd->cropped_pixel_bounds[3] - 0.5f + fd->filter_radius[1])));
    DeviceMathScope dm;
    if (pp->sampler == PB2_SAMPLER_SOBOL) {
        SobolSampler ss(pp->samples_per_pixel, sb);
        for (int64_t i = 0; i < n; ++i) {
            ss.StartPixel(Point2i(pixel_xy[2 * i], pixel_xy[2 * i + 1]));
            out[i] = ss.SampleDimension(ss.GetIndexForSample(sample_num[i]), dim[i]);
        }
        return 0;
    }
    HaltonSampler hs(pp->samples_per_pixel, sb, pp->sample_at_pixel_center != 0);
    for (int64_t i = 0; i < n; ++i) {
        hs.StartPixel(Point2i(pixel_xy[2 * i], pixel_xy[2 * i + 1]));
        int64_t index = hs.GetIndexForSample(sample_num[i]);
        out[i] = hs.SampleDimension(index, dim[i]);
    }
    return 0;
}

// The reference's own tables behind SobolIntervalToIndex for resolution 2^m (sobolmatrices.cpp): 52 entries of
// VdCSobolMatrices[m - 1], then 52 of VdCSobolMatricesInv[m - 1]; and SobolMatrices32 (1024 x 52) when asked for.
int ref_sobol_tables(int m, uint64_t *out104, uint32_t *matrices32) {
    if (m < 1 || m > 25) return 1;
    for (int c = 0; c < SobolMatrixSize; ++c) {
        out104[c] = VdCSobolMatrices[m - 1][c];
        out104[SobolMatrixSize + c] = VdCSobolMatricesInv[m - 1][c];
    }
    if (matrices32) std::memcpy(matrices32, SobolMatrices32, sizeof(uint32_t) * NumSobolDimensions * SobolMatrixSize);
    return 0;
}

// RadicalInverse / ScrambledRadicalInverse (src/core/lowdiscrepancy.cpp:427, 2506) with the
// sampler's permutation table; scrambled=0 -> RadicalInverse.
int ref_radical_inverse(int base_index, const uint64_t *a, int64_t n, int scrambled, float *out) {
    if (HaltonSampler::radicalInversePermutations.empty()) {
        RNG rng;
        HaltonSampler::radicalInversePermutations = ComputeRadicalInversePermutations(rng);
    }
    for (int64_t i = 0; i < n; ++i)
        out[i] = scrambled ? ScrambledRadicalInverse(base_index, a[i], &HaltonSampler::radicalInversePermutations[PrimeSums[base_index]])
                           : RadicalInverse(base_index, a[i]);
    return 0;
}

// For each point: n_lights func values then n_lights+1 cdf values of LightDistribution::Lookup(p).
int ref_light_distribution(void *h, const float *points, int64_t n, float *out) {
    RefScene *rs = static_cast<RefScene *>(h);
    if (!rs->distrib) rs->distrib = CreateLightSampleDistribution(strategyName(rs->lightStrategy), *rs->scene);
    size_t nl = rs->lights.size(), stride = 2 * nl + 1;
    DeviceMathScope dm;
    for (int64_t i = 0; i < n; ++i) {
        const Distribution1D *d = rs->distrib->Lookup(Point3f(points[3 * i], points[3 * i + 1], points[3 * i + 2]));
        for (size_t k = 0; k < nl; ++k) out[i * stride + k] = d->func[k];
        for (size_t k = 0; k <= nl; ++k) out[i * stride + nl + k] = d->cdf[k];
    }
    return 0;
}

// CreateLoopSubdiv (src/shapes/loopsubdiv.cpp:389-410) under the identity transform.
int ref_loop_subdivide(int n_levels, int n_indices, const int *indices, int n_vertices, const float *P,
                       int *out_n_vertices, int *out_n_indices, float *out_P, float *out_N, int *out_indices) {
    ParamSet ps;
    std::unique_ptr<int[]> idx(new int[n_indices]);
    std::memcpy(idx.get(), indices, n_indices * sizeof(int));
    ps.AddInt("indices", std::move(idx), n_indices);
    std::unique_ptr<Point3f[]> pts(new Point3f[n_vertices]);
    for (int i = 0; i < n_vertices; ++i) pts[i] = Point3f(P[3 * i], P[3 * i + 1], P[3 * i + 2]);
    ps.AddPoint3f("P", std::move(pts), n_vertices);
    std::unique_ptr<int[]> lv(new int[1]);
    lv[0] = n_levels;
    ps.AddInt("levels", std::move(lv), 1);
    Transform identity;
    std::vector<std::shared_ptr<Shape>> shapes = CreateLoopSubdiv(&identity, &identity, false, ps);
    if (shapes.empty()) return 1;
    const Triangle *t0 = static_cast<const Triangle *>(shapes[0].get());
    const TriangleMesh *mesh = t0->mesh.get();
    *out_n_vertices = mesh->nVertices;
    *out_n_indices = 3 * mesh->nTriangles;
    if (out_P)
        for (int i = 0; i < mesh->nVertices; ++i)
            for (int k = 0; k < 3; ++k) out_P[3 * i + k] = mesh->p[i][k];
    if (out_N)
        for (int i = 0; i < mesh->nVertices; ++i)
            for (int k = 0; k < 3; ++k) out_N[3 * i + k] = mesh->n[i][k];
    if (out_indices) std::memcpy(out_indices, mesh->vertexIndices.data(), sizeof(int) * 3 * mesh->nTriangles);
    return 0;
}

// PerspectiveCamera's derived matrices for a description (tests compare with the host's).
int ref_camera_derived(const pb2_camera *cam, const pb2_film_desc *fd, float *raster_to_camera16, float *dx3, float *dy3) {
    RefScene dummy;
    pb2_path_params pp;
    std::memset(&pp, 0, sizeof(pp));
    pp.samples_per_pixel = 1;
    pp.max_depth = 1;
    pp.pixel_bounds[2] = fd->full_resolution[0];
    pp.pixel_bounds[3] = fd->full_resolution[1];
    RenderObjects ro = makeRenderObjects(dummy, cam, fd, &pp);
    const PerspectiveCamera *pc = static_cast<const PerspectiveCamera *>(ro.camera.get());
    std::memcpy(raster_to_camera16, pc->RasterToCamera.m.m, 16 * sizeof(float));
    for (int k = 0; k < 3; ++k) {
        dx3[k] = pc->dxCamera[k];
        dy3[k] = pc->dyCamera[k];
    }
    return 0;
}

// Transform helpers of src/core/transform.cpp for host-math tests: kind 0 LookAt(9 args),
// 1 Rotate(angle, axis), 2 Perspective(fov, n, f), 3 Translate, 4 Scale. Returns m and mInv.
int ref_transform(int kind, const float *args, float *m16, float *minv16) {
    Transform t;
    switch (kind) {
    case 0: t = LookAt(Point3f(args[0], args[1], args[2]), Point3f(args[3], args[4], args[5]), Vector3f(args[6], args[7], args[8])); break;
    case 1: t = Rotate(args[0], Vector3f(args[1], args[2], args[3])); break;
    case 2: t = Perspective(args[0], args[1], args[2]); break;
    case 3: t = Translate(Vector3f(args[0], args[1], args[2])); break;
    case 4: t = Scale(args[0], args[1], args[2]); break;
    default: return 1;
    }
    std::memcpy(m16, t.GetMatrix().m, 16 * sizeof(float));
    std::memcpy(minv16, t.GetInverseMatrix().m, 16 * sizeof(float));
    return 0;
}

}  // extern "C"
