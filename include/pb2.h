/*
 * pb2.h — C ABI of the H100-native pbrt-v3 path-tracing hot path.
 *
 * pbrt-v3 has no dlopen plugin ABI: its "plugins" are C++ classes selected by name in
 * src/core/api.cpp.  The hot path sits behind these reference interfaces:
 *
 *   Integrator::Render(const Scene&)                      src/core/integrator.h:53-58
 *   SamplerIntegrator::Render / PathIntegrator::Li        src/core/integrator.cpp:228-339, src/integrators/path.cpp:64-188
 *   Aggregate / BVHAccel::Intersect / IntersectP          src/core/primitive.h:119-127, src/accelerators/bvh.cpp:662-738
 *   Shape / Triangle::Intersect / IntersectP              src/core/shape.h:51-89, src/shapes/triangle.cpp:188-572
 *   Scene::Intersect / IntersectP                         src/core/scene.cpp:45-55
 *   FilmTile::AddSample / Film::MergeFilmTile             src/core/film.h:121-161, src/core/film.cpp:117-130
 *
 * The host C++ classes in pbrt_v3_b200/csrc/host (same names, same virtual signatures) flatten a
 * scene into a pb2_scene_desc and call the entry points below; INTEGRATION.md shows the binding a
 * reference maintainer would add.  Plain pointers and sizes only; every function returns 0 on
 * success and a non-zero pb2_status otherwise (never throws); pb2_last_error() describes the
 * failure.  Calls are blocking.  The caller keeps ownership of every host pointer; device copies
 * are made inside.  There is NO CPU fallback: without a CUDA device every compute entry point
 * returns PB2_ERR_NO_DEVICE.
 */
#ifndef PB2_H
#define PB2_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB2_ABI_VERSION 10   /* 2: instancing block in pb2_scene_desc; 3: mirror / glass fields in pb2_material; 4: filter type in pb2_film_desc;
                             * 5: uber / metal fields in pb2_material (128 bytes); 6: point / spot / distant lights
                             * (pb2_light.type, pb2_scene_desc.delta_lights); 7: pb2_trace_wavefront, kernel-selector flags;
                             * 8: pb2_dist_* (NCCL film reduce inside the render calls), pb2_host_alloc;
                             * 9: PB2_LIGHT_INFINITE, pb2_delta_light.light_to_world (112 bytes);
                             * 10: image textures (pb2_texture, pb2_material.tex, pb2_mesh.alpha_tex / shadow_alpha_tex), pb2_path_params.sampler */

typedef enum pb2_status {
    PB2_OK = 0,
    PB2_ERR_NO_DEVICE = 1,   /* no CUDA device / driver: the product path fails loudly */
    PB2_ERR_CUDA = 2,        /* a CUDA runtime call failed */
    PB2_ERR_INVALID = 3,     /* bad argument / inconsistent scene description */
    PB2_ERR_UNSUPPORTED = 4, /* feature of the reference outside this path's scope (SURVEY.md §8) */
    PB2_ERR_NCCL = 5         /* libnccl could not be loaded, or an NCCL call failed */
} pb2_status;

/* ---- scene description (host memory, flattened by the host-side Scene) ------------------- */

/* Exactly the reference's LinearBVHNode, src/accelerators/bvh.cpp:95-104 (32 bytes,
 * depth-first order: the first child of interior node i is i+1). */
typedef struct pb2_bvh_node {
    float bmin[3];
    float bmax[3];
    int32_t offset;   /* leaf: primitivesOffset into bvh_prims; interior: secondChildOffset */
    uint16_t n_prims; /* 0 -> interior */
    uint8_t axis;
    uint8_t pad;
} pb2_bvh_node;

enum { PB2_PRIM_TRIANGLE = 0, PB2_PRIM_SPHERE = 1, PB2_PRIM_INSTANCE = 2 };
enum { PB2_MAT_NONE = 0, PB2_MAT_MATTE = 1, PB2_MAT_PLASTIC = 2, PB2_MAT_MIRROR = 3, PB2_MAT_GLASS = 4, PB2_MAT_SUBSTRATE = 5, PB2_MAT_METAL = 6,
       PB2_MAT_UBER = 7 };
enum { PB2_LIGHTDIST_UNIFORM = 0, PB2_LIGHTDIST_POWER = 1, PB2_LIGHTDIST_SPATIAL = 2 };
enum { PB2_FILTER_BOX = 0, PB2_FILTER_GAUSSIAN = 1, PB2_FILTER_MITCHELL = 2, PB2_FILTER_SINC = 3, PB2_FILTER_TRIANGLE = 4 };

/* One TriangleMesh (src/shapes/triangle.h:46-68).  Vertices are already in world space
 * (src/shapes/triangle.cpp:73-74); normals already transformed (triangle.cpp:83). */
typedef struct pb2_mesh {
    int32_t first_tri, n_tris;        /* range in tri_index[] */
    int32_t first_vertex, n_vertices; /* range in P/N/UV/S */
    int32_t has_n, has_uv, has_s;
    int32_t reverse_orientation;
    int32_t transform_swaps_handedness;
    /* TriangleMesh::alphaMask / shadowAlphaMask (triangle.h:61, triangle.cpp:333-338, 531-569): 0 = none, else 1 + index
     * into pb2_scene_desc.textures of a one-channel texture; a hit where it evaluates to exactly 0 is no hit
     * (alpha_tex: Intersect and IntersectP; shadow_alpha_tex: IntersectP only). */
    int32_t alpha_tex, shadow_alpha_tex;
    int32_t pad;
} pb2_mesh;

/* An ImageTexture (src/textures/imagemap.h:72-128) with a UVMapping2D (src/core/texture.cpp:93-99), described by what its
 * constructor hands to MIPMap (src/core/mipmap.h:112-119): the texels AFTER ReadImage, the flip in y (imagemap.cpp:77-84) and
 * convertIn (scale, inverse gamma, luminance for one-channel textures; imagemap.h:97-106).  The library resamples to a power
 * of two and builds the pyramid as the MIPMap constructor does (mipmap.h:121-203) and filters as MIPMap::Lookup does
 * (trilinear: mipmap.h:227-245; EWA: mipmap.h:263-350).  Texture differentials come from the camera ray's differentials
 * (perspective.cpp:117-144, scaled by 1/sqrt(spp), integrator.cpp:273-274) through SurfaceInteraction::ComputeDifferentials
 * (interaction.cpp:101-147); rays after the first bounce carry none (path.cpp:130-131), as in the reference. */
enum { PB2_WRAP_REPEAT = 0, PB2_WRAP_BLACK = 1, PB2_WRAP_CLAMP = 2 };
typedef struct pb2_texture {
    int32_t channels;        /* 1: ImageTexture<Float, Float>; 3: ImageTexture<RGBSpectrum, Spectrum> */
    int32_t width, height;   /* resolution of texels[] (any size; not yet a power of two) */
    int32_t wrap;            /* PB2_WRAP_* ("wrap") */
    int32_t do_trilinear;    /* "trilinear" */
    float max_anisotropy;    /* "maxanisotropy" */
    float su, sv, du, dv;    /* UVMapping2D: "uscale" "vscale" "udelta" "vdelta" */
    int32_t kind;            /* PB2_TEXKIND_*; zero-initialised = an image */
    int32_t pad;
    const float *texels;     /* PB2_TEXKIND_IMAGE: channels * width * height, row 0 is t = 0; NULL otherwise */
    /* the combinators over other textures of the array (1 + index, each smaller than the texture's own index, at most three
     * levels deep): PB2_TEXKIND_SCALE = child[0] * child[1] (ScaleTexture, src/textures/scale.h:50-64), PB2_TEXKIND_MIX =
     * (1 - a) * child[0] + a * child[1] with a = the one-channel texture child[2] (MixTexture, src/textures/mix.h:50-66);
     * children have the texture's own channel count.  PB2_TEXKIND_CONSTANT = value[0 .. channels) (ConstantTexture). */
    int32_t child[3];
    float value[3];
} pb2_texture;
/* PB2_TEXKIND_CHECKERBOARD: Checkerboard2DTexture (src/textures/checkerboard.h:52-107) over child[0] / child[1] with the
 * UVMapping2D in su .. dv; value[0] = 0: "aamode" "none", 1: "closedform".  PB2_TEXKIND_UV: UVTexture (src/textures/uv.h:48-63),
 * three channels, the mapping in su .. dv. */
enum { PB2_TEXKIND_IMAGE = 0, PB2_TEXKIND_CONSTANT = 1, PB2_TEXKIND_SCALE = 2, PB2_TEXKIND_MIX = 3, PB2_TEXKIND_CHECKERBOARD = 4,
       PB2_TEXKIND_UV = 5 };

/* slots of pb2_material.tex: which parameter a texture replaces */
enum { PB2_TEX_KD = 0, PB2_TEX_KS = 1, PB2_TEX_KR = 2, PB2_TEX_KT = 3, PB2_TEX_OPACITY = 4, PB2_TEX_SIGMA = 5, PB2_TEX_ROUGHNESS = 6,
       PB2_TEX_UROUGHNESS = 7, PB2_TEX_VROUGHNESS = 8, PB2_TEX_ETA = 9, PB2_TEX_METAL_ETA = 10, PB2_TEX_METAL_K = 11,
       /* the "bumpmap" displacement (a one-channel texture): Material::Bump (src/core/material.cpp:45-82) perturbs the shading
        * geometry before the material's other textures are evaluated */
       PB2_TEX_BUMP = 12, PB2_TEX_SLOTS = 13 };

/* Sphere (src/shapes/sphere.h:47-77). Matrices are row-major 4x4 (Matrix4x4::m). */
typedef struct pb2_sphere {
    float object_to_world[16];
    float world_to_object[16];
    float radius, z_min, z_max, theta_min, theta_max, phi_max;
    int32_t reverse_orientation;
    int32_t transform_swaps_handedness;
} pb2_sphere;

/* MatteMaterial (src/materials/matte.cpp:45-62) / PlasticMaterial (src/materials/plastic.cpp:45-70)
 * with constant textures (src/textures/constant.h:54). */
typedef struct pb2_material {
    int32_t type;
    float kd[3];
    float sigma;
    float ks[3];
    float roughness;
    int32_t remap_roughness;
    int32_t pad[2];
    /* MirrorMaterial (src/materials/mirror.cpp:45-58): kr.  GlassMaterial (src/materials/glass.cpp:45-93): kr, kt, eta
     * (the "index"/"eta" parameter), uroughness, vroughness, remap_roughness; both roughnesses zero = one FresnelSpecular,
     * otherwise the MicrofacetReflection + MicrofacetTransmission pair.
     * SubstrateMaterial (src/materials/substrate.cpp:45-65): kd, ks, uroughness, vroughness, remap_roughness. */
    float kr[3];
    float kt[3];
    float eta;
    float uroughness, vroughness;
    /* UberMaterial (src/materials/uber.cpp:45-104): kd, ks, kr, kt, opacity, eta, remap_roughness and
     * uroughness / vroughness already resolved ("uroughness" else "roughness"; "vroughness" else the u value).
     * MetalMaterial (src/materials/metal.cpp:60-80): metal_eta, metal_k, remap_roughness and uroughness /
     * vroughness resolved the same way (each falls back to "roughness"). */
    float opacity[3];
    float metal_eta[3];
    float metal_k[3];
    int32_t pad3[2];
    /* tex[PB2_TEX_*]: 0 = the constant above, else 1 + index into pb2_scene_desc.textures of the texture that is evaluated
     * at every shaded point instead (Kd->Evaluate(*si) etc., matte.cpp:53-54); spectrum parameters take three-channel
     * textures, float parameters one-channel ones.  The u / v roughness slots hold what the material's fall-back rules
     * resolve to ("uroughness" else "roughness", uber.cpp:82-85). */
    int32_t tex[16];            /* PB2_TEX_SLOTS of them are used */
} pb2_material;

/* One entry of Scene::lights, in the scene's order.  PB2_LIGHT_AREA: a DiffuseAreaLight (src/lights/diffuse.h:49-79)
 * attached to one primitive.  The other types are the delta lights (src/lights/{point,spot,distant}.cpp): L holds
 * I (point, spot) or L (distant), prim is -1, and delta_lights[same index] the geometry.  PB2_LIGHT_INFINITE: an
 * InfiniteAreaLight (src/lights/infinite.cpp): constant radiance L = "L" * "scale" from every direction, or an environment map
 * (pb2_delta_light.env_tex);
 * prim is -1, delta_lights[same index] carries its two 3x3 matrices and world_radius (Preprocess, infinite.h:61-63).  Rays
 * that leave the scene see it (path.cpp:96-98). */
enum { PB2_LIGHT_AREA = 0, PB2_LIGHT_POINT = 1, PB2_LIGHT_SPOT = 2, PB2_LIGHT_DISTANT = 3, PB2_LIGHT_INFINITE = 4 };
typedef struct pb2_light {
    int32_t prim;       /* index into prim_type[]/prim_index[] */
    float L[3];         /* Lemit = L * scale */
    int32_t two_sided;
    float area;         /* Shape::Area() of that primitive (DiffuseAreaLight::area, diffuse.cpp:52) */
    int32_t type;       /* PB2_LIGHT_* */
    int32_t pad;
} pb2_light;

typedef struct pb2_delta_light {
    float p[3];                 /* point, spot: pLight (point.h:52, spot.h:54); distant: LightToWorld(from - to), NOT normalised
                                 * (the constructor argument of distant.cpp:43-46; the library normalises it as the constructor does) */
    float total_width_deg;      /* spot: the constructor's totalWidth / falloffStart in degrees (spot.cpp:43-50); the library takes */
    float falloff_start_deg;    /*       their cosines as the constructor does */
    float world_radius;         /* distant: DistantLight::Preprocess (distant.h:55-57), from the scene bounds */
    float world_to_light[9];    /* spot, infinite: upper-left 3x3 of WorldToLight, row-major (SpotLight::Falloff, spot.cpp:63-72;
                                 * InfiniteAreaLight::Le / Pdf_Li, infinite.cpp:90-94, 124-132) */
    float pad;
    float light_to_world[9];    /* infinite: upper-left 3x3 of LightToWorld (InfiniteAreaLight::Sample_Li, infinite.cpp:96-122) */
    int32_t env_tex;            /* infinite: 0 = constant radiance pb2_light.L; else 1 + index into pb2_scene_desc.textures of the
                                 * environment map - a three-channel texture holding ReadImage(mapname) * L (infinite.cpp:50-57;
                                 * NOT flipped in y, wrap repeat), pb2_light.L is then ignored.  The library builds Lmap's pyramid
                                 * and the Distribution2D over the 2w x 2h luminance * sin(theta) image (infinite.cpp:61-82) */
    float pad2[2];
} pb2_delta_light;

/* One BVHAccel of the scene: bvhs[0] is Scene::aggregate, bvhs[k > 0] the accelerator that
 * pbrtObjectInstance builds over the primitives of an instanced object (src/core/api.cpp:1565-1573).
 * Node indices (secondChildOffset) and primitivesOffset values inside a BVH are LOCAL to it. */
typedef struct pb2_bvh {
    int64_t node_offset, n_nodes;   /* range in nodes[] */
    int64_t prim_offset, n_prims;   /* range in bvh_prims[] */
} pb2_bvh;

/* TransformedPrimitive (src/core/primitive.cpp:69-96) with a static transform: an instance of an
 * object.  Matrices are row-major 4x4: InstanceToWorld = the CTM at pbrtObjectInstance. */
typedef struct pb2_instance {
    float instance_to_world[16];
    float world_to_instance[16];
    int32_t bvh;        /* >= 1: bvhs[] entry of the object's accelerator; -1: the object is ONE primitive */
    int32_t lone_prim;  /* bvh == -1: position in bvh_prims[] (past every BVH's range) of that primitive */
    int32_t pad[2];
} pb2_instance;

typedef struct pb2_scene_desc {
    /* geometry */
    int64_t n_vertices;
    const float *P;        /* 3*n_vertices, world space */
    const float *N;        /* 3*n_vertices or NULL (only read for meshes with has_n) */
    const float *UV;       /* 2*n_vertices or NULL */
    const float *S;        /* 3*n_vertices or NULL */
    int64_t n_tris;
    const int32_t *tri_index; /* 3*n_tris, indices into the GLOBAL vertex arrays */
    const int32_t *tri_mesh;  /* n_tris, mesh of each triangle */
    int32_t n_meshes;
    const pb2_mesh *meshes;
    int32_t n_spheres;
    const pb2_sphere *spheres;

    /* primitives in scene order (GeometricPrimitive, src/core/primitive.cpp:98-130) */
    int64_t n_prims;
    const uint8_t *prim_type;     /* PB2_PRIM_* */
    const int32_t *prim_index;    /* triangle id or sphere id */
    const int32_t *prim_material; /* index into materials[], -1 = no material (null BSDF) */
    const int32_t *prim_light;    /* index into lights[], -1 = not emissive */

    /* BVHAccel (src/accelerators/bvh.cpp:183-225) built on the host */
    int64_t n_nodes;
    const pb2_bvh_node *nodes;
    const int32_t *bvh_prims;     /* n_prims: ordered primitive numbers (BVHAccel::primitives) */

    int32_t n_materials;
    const pb2_material *materials;
    int32_t n_lights;
    const pb2_light *lights;      /* Scene::lights order (src/core/api.cpp:1394-1400) */

    int32_t light_strategy;       /* PB2_LIGHTDIST_*; src/core/lightdistrib.cpp:48-66 */
    int32_t spatial_max_voxels;   /* 64, src/core/lightdistrib.h:104 */

    /* Object instancing (optional; all zero / NULL for a scene without ObjectInstance).
     * prim_type[i] == PB2_PRIM_INSTANCE: prim_index[i] = entry of instances[]; such primitives
     * appear only in bvhs[0].  The scene-level primitives are numbered 0 .. bvhs[0].n_prims-1 in
     * scene order; the GeometricPrimitives inside objects are ordinary entries of the prim_* arrays
     * after them (object by object, creation order) and appear only in their object's BVH, or - for a
     * one-primitive object - past all BVH ranges of bvh_prims.  With n_bvhs == 0 the arrays
     * nodes[n_nodes] / bvh_prims[n_prims] are the one scene BVH as before. */
    int32_t n_instances;
    int32_t n_bvhs;
    const pb2_instance *instances;
    const pb2_bvh *bvhs;
    int64_t n_bvh_prims;          /* length of bvh_prims when n_bvhs > 0 */
    /* n_lights entries, read for lights[i].type != PB2_LIGHT_AREA; NULL when every light is an area light */
    const pb2_delta_light *delta_lights;
    /* image textures named by pb2_material.tex and pb2_mesh.alpha_tex (NULL / 0: a scene of constant textures) */
    int32_t n_textures;
    int32_t pad_textures;
    const pb2_texture *textures;
} pb2_scene_desc;

/* PerspectiveCamera (src/cameras/perspective.cpp:45-67, 95-144). */
typedef struct pb2_camera {
    /* high-level parameters (what CreatePerspectiveCamera sees) */
    float camera_to_world[16];   /* row-major */
    float world_to_camera[16];
    float screen_window[4];      /* xmin xmax ymin ymax */
    float fov;
    float lens_radius, focal_distance;
    float shutter_open, shutter_close;
    /* derived by the host exactly as ProjectiveCamera does (src/core/camera.h:84-115) */
    float raster_to_camera[16];
    float dx_camera[3], dy_camera[3];
} pb2_camera;

/* Film (src/core/film.cpp:45-78) and its reconstruction filter (src/filters/{box,gaussian,mitchell,sinc,triangle}.cpp). */
typedef struct pb2_film_desc {
    int32_t full_resolution[2];
    int32_t cropped_pixel_bounds[4]; /* x0 y0 x1 y1 (Film::croppedPixelBounds) */
    float filter_radius[2];          /* Filter::radius */
    float max_sample_luminance;
    float scale;
    /* reconstruction filter (one of src/filters/); zero-initialised = box.  filter_param: gaussian {alpha, -},
     * mitchell {B, C}, sinc {tau, -}.  The 16x16 weight table of Film (film.cpp:68-77) is computed inside. */
    int32_t filter_type;             /* PB2_FILTER_* */
    float filter_param[2];
    int32_t pad;
} pb2_film_desc;

/* HaltonSampler (src/samplers/halton.cpp:65-131) + PathIntegrator parameters
 * (src/integrators/path.cpp:190-213). */
typedef struct pb2_path_params {
    int32_t samples_per_pixel;
    int32_t sample_at_pixel_center;
    int32_t max_depth;
    float rr_threshold;
    int32_t pixel_bounds[4];  /* x0 y0 x1 y1: PathIntegrator::pixelBounds */
    /* work partition for multi-GPU (SURVEY.md §8e): this call renders only the 16x16 sample
     * tiles t of SamplerIntegrator::Render (integrator.cpp:235-240) with t % tile_count == tile_rank */
    int32_t tile_rank, tile_count;
    int32_t flags;            /* PB2_FLAG_* */
    int32_t sampler;          /* PB2_SAMPLER_*; zero-initialised = the HaltonSampler */
} pb2_path_params;

/* The two GlobalSamplers of the reference.  PB2_SAMPLER_SOBOL: SobolSampler (src/samplers/sobol.cpp:41-60,
 * src/core/lowdiscrepancy.h:229-274): samples_per_pixel must already be the power of two its constructor rounds up to
 * (sobol.h:52); sample_at_pixel_center does not exist there and is ignored.  The generator matrices come from
 * pbrt_v3_b200/lib/sobol_matrices32.bin next to the library (tools/make_sobol_tables.py, run by build()). */
enum { PB2_SAMPLER_HALTON = 0, PB2_SAMPLER_SOBOL = 1 };

/* Count LinearBVHNode fetches and primitive tests (pb2_stats.node_visits / prim_tests) with the
 * one-thread-per-ray traversal kernel instead of the tuned one: the device analogue of the
 * reference's STAT_COUNTERs, used to obtain the algorithmic bytes of a frame (SURVEY.md §8d). */
#define PB2_FLAG_COUNT_TRAVERSAL 1
/* Trace with the kernel that reads the 32-byte LinearBVHNode array directly instead of the derived
 * two-child records (same results; kept selectable so both kernels stay under test). */
#define PB2_FLAG_LINEAR_NODES 2
/* Trace with the kernel over the four-child records (two tree levels per fetch) instead of the default two-child
 * records (same results; measured slightly slower, kept selectable and under test). */
#define PB2_FLAG_WIDE4 4
/* Trace with the one-thread-per-ray kernel (BVHAccel::Intersect as written) instead of the persistent-warp kernels. */
#define PB2_FLAG_PLAIN_TRACE 8
/* Give the record kernels 4 instead of 16 shared-memory stack entries per lane (tests: exercises the spill path). */
#define PB2_FLAG_SMALL_STACK 16
/* Fetch node records with 16-byte instead of 32-byte loads per lane (same results). */
#define PB2_FLAG_LD128 32
/* Experiment kept for the record (DESIGN.md section 3): stage leaf records into shared memory with TMA bulk copies
 * (cp.async.bulk / UBLKCP + mbarrier) before the triangle tests; triangle scenes, two-child kernel.  Same results, slower. */
#define PB2_FLAG_LEAF_TMA 64
/* Trace triangle scenes with the kernel that keeps a pool of 48 rays per warp in shared memory and picks, for every step,
 * the rays that are in the phase being run (k_wf_trace_pool).  Same results. */
#define PB2_FLAG_POOL 128
/* Experiment kept for the record (DESIGN.md section 3): the default trace kernels with the light step inside - when a shadow
 * or MIS ray ends, its lane adds the term, starts the vertex's next ray (MIS ray, continuation of the path) and traces it in
 * the same launch, so that a bounce takes one round instead of up to three.  Same results, fewer launches, slower. */
#define PB2_FLAG_CHAIN 256

typedef struct pb2_ray {
    float o[3];
    float d[3];
    float t_max;
} pb2_ray;

typedef struct pb2_hit {
    int32_t prim;      /* scene-order primitive number, -1 = miss */
    float t;           /* ray.tMax after Intersect (primitive.cpp:120) */
    float b[3];        /* triangle barycentrics b0,b1,b2 (triangle.cpp:263-268); sphere: phi,0,0 */
    float p[3];        /* SurfaceInteraction::p */
    float p_error[3];
    float n[3];        /* geometric normal after orientation/face-forward */
    float ns[3];       /* shading.n */
    float dpdu[3];     /* shading.dpdu */
    float uv[2];
} pb2_hit;

typedef struct pb2_stats {
    uint64_t camera_rays;     /* integrator.cpp:287 nCameraRays */
    uint64_t regular_rays;    /* scene.cpp:46 nIntersectionTests */
    uint64_t shadow_rays;     /* scene.cpp:52 nShadowTests */
    uint64_t node_visits;     /* LinearBVHNode records fetched (only with PB2_FLAG_COUNT_TRAVERSAL) */
    uint64_t prim_tests;      /* leaf primitive tests (only with PB2_FLAG_COUNT_TRAVERSAL) */
    uint64_t kernel_launches; /* number of our kernels launched by the call */
    double render_ms;         /* device time of the whole render (CUDA events on the launching stream) */
    double h2d_ms, d2h_ms;
    double trace_ms;          /* summed device time of the BVH traversal kernel launches */
} pb2_stats;

typedef struct pb2_scene pb2_scene; /* opaque: device-resident scene */

/* ---- entry points ----------------------------------------------------------------------- */

int pb2_abi_version(void);
const char *pb2_last_error(void);

/* Binds the calling process to one CUDA device (one process per GPU).  Replaces the reference's
 * ParallelInit() (src/core/parallel.cpp:301-336) as "bring up the execution resource". */
int pb2_init(int device_id);
/* Binds the calling process to a GROUP of local devices (n = 0: every visible device); device_ids[0] is the primary one.
 * pb2_scene_create then keeps one copy of the scene per device, and a render call whose params.tile_count is 0 deals the
 * film's 16x16 tiles round-robin to the devices (one host thread each) and adds the per-device films on the primary device,
 * which reads the others' memory over NVLink peer access - Film::MergeFilmTile (src/core/film.cpp:117-130) across GPUs
 * without leaving the process.  This is what the pb2_pbrt command line uses; one process per GPU + pb2_dist_init (below)
 * is the other way to use several GPUs, and the two do not combine. */
int pb2_init_devices(int n_devices, const int *device_ids);
int pb2_device_count(void);   /* devices bound by pb2_init / pb2_init_devices (0 before) */
int pb2_shutdown(void);

/* Multi-GPU (SURVEY.md section 8e): one process per GPU; the film's 16x16 sample tiles are dealt round-robin to the ranks,
 * the scene is replicated, and the distributed Film::MergeFilmTile (src/core/film.cpp:117-130) is ONE ncclReduce(sum) of
 * the W x H x 4 floats to rank 0, issued by pb2_render_path[_device] itself.  NCCL (libnccl.so.2) is loaded at run time.
 *   pb2_dist_unique_id   rank 0: a fresh communicator id (PB2_DIST_ID_BYTES bytes) to hand to every rank (any transport:
 *                        bench.py broadcasts it over torch.distributed, pb2_pbrt passes it through the environment)
 *   pb2_dist_init        collective over all ranks, after pb2_init: joins the communicator on this process's device
 * After that a render call whose params.tile_count is 0 is a COLLECTIVE: every rank renders its own tiles, rank 0
 * receives the merged film (the other ranks' film_rgbw may be NULL and is left untouched).  tile_count >= 1 keeps its
 * meaning of an explicit, unreduced partition.  Without pb2_dist_init (or with world 1) nothing changes. */
#define PB2_DIST_ID_BYTES 128
int pb2_dist_unique_id(void *id);
int pb2_dist_init(int rank, int world, const void *id);
int pb2_dist_info(int *rank, int *world);
int pb2_dist_shutdown(void);

/* The work partition of the render kernels, evaluated on the host (no device needed; the kernels run the same function):
 * for work items first .. first + n - 1 of the partition (params->tile_rank, params->tile_count) writes (pixel x, pixel y,
 * sample number) per item, or (-1, -1, -1) for an item that falls outside the sample bounds / pixelbounds and is skipped;
 * *n_items receives the number of work items of that partition.  Items are ordered tile by tile (the reference's 16 x 16
 * tiles, src/core/integrator.cpp:235-240; tile t belongs to rank t % tile_count), then by sample number, then along a
 * Morton curve inside the tile.  Used by the multi-process tests; `out` may be NULL to query the count. */
int pb2_work_items(const pb2_film_desc *film, const pb2_path_params *params, int64_t first, int64_t n, int32_t *out,
                   int64_t *n_items);

/* Page-locked host memory for film buffers: pb2_render_path copies the film back at the full PCIe rate into such a
 * buffer (cudaMemcpy into pageable memory is staged by the driver). */
int pb2_host_alloc(size_t bytes, void **out);
int pb2_host_free(void *p);

/* Uploads a flattened Scene (src/core/scene.h:50-80).  Builds the spatial light-distribution
 * tables (src/core/lightdistrib.cpp:232-300) on the device. */
int pb2_scene_create(const pb2_scene_desc *desc, pb2_scene **out);
int pb2_scene_destroy(pb2_scene *scene);
/* The shade feature class pb2_scene_create gives the scene described by desc (host only, no device needed): a bit
 * mask of what the scene's material and light records can produce, 1 = an Oren-Nayar lobe (matte, sigma != 0),
 * 2 = a plastic Trowbridge-Reitz lobe, 4 = a point, spot, distant or infinite light; 7 when a specular-family material
 * (mirror, glass, substrate, metal, uber) is present or the environment sets PB2_SHADE_GENERAL=1.  A scene of class 0
 * (Lambertian surfaces lit by area lights) gets a shade step compiled for that class alone, unless it also has spheres,
 * image textures, the SobolSampler or the lazily built light distribution. */
int pb2_shade_class(const pb2_scene_desc *desc, int32_t *out);

/* Scene::Intersect for a batch of rays (src/core/scene.cpp:45-49). rays/hits are HOST pointers. */
int pb2_intersect(pb2_scene *scene, const pb2_ray *rays, int64_t n, pb2_hit *hits);
/* Scene::IntersectP for a batch (src/core/scene.cpp:51-55). */
int pb2_intersect_p(pb2_scene *scene, const pb2_ray *rays, int64_t n, uint8_t *occluded);

/* SamplerIntegrator::Render with PathIntegrator::Li (src/core/integrator.cpp:228-339,
 * src/integrators/path.cpp:64-188).  film_rgbw (HOST, 4 floats per pixel of croppedPixelBounds,
 * row-major) receives what the reference's FilmTile pixels hold after all tiles were merged:
 * contribSum RGB and filterWeightSum (src/core/film.h:109-113); the host Film applies
 * MergeFilmTile's RGB->XYZ and WriteImage (src/core/film.cpp:117-130,169-211).
 * Host buffers in, host buffer out: copies are inside the call. */
int pb2_render_path(pb2_scene *scene, const pb2_camera *camera, const pb2_film_desc *film,
                    const pb2_path_params *params, float *film_rgbw, pb2_stats *stats);

/* Same computation with the film left resident in device memory (used by bench.py's device-timed
 * `value` and by the multi-GPU reduce).  film_rgbw_device is a DEVICE pointer to
 * 4*width*height floats, zeroed by the call when `clear` is non-zero.  `stream` is a cudaStream_t
 * (0 = default stream).  The call BLOCKS: the host reads the wavefront's counters every few rounds to detect the
 * end of the frame (work enqueued after the last of those reads may still be running on `stream` at return unless
 * stats != NULL).  A pb2_scene carries the scratch of ONE render at a time (path-context pool, queues, counters):
 * concurrent render calls on the same scene from different threads or streams are not supported. */
int pb2_render_path_device(pb2_scene *scene, const pb2_camera *camera, const pb2_film_desc *film,
                           const pb2_path_params *params, float *film_rgbw_device, int clear,
                           void *stream, pb2_stats *stats);

/* The traversal kernel of the RENDER path over a batch of rays (parity / debug entry point).  pb2_intersect[_p] run
 * BVHAccel::Intersect[P] one thread per ray as the reference writes it; the renderer traces with persistent-warp
 * kernels over derived node records (`flags`: the PB2_FLAG_* kernel selectors of pb2_path_params.flags).  This call puts
 * the rays into path contexts exactly as the renderer does, launches the kernel the renderer would launch for this scene
 * and these flags, and returns the raw records it leaves in the contexts.  any_hit[i] != 0 (may be NULL): ray i is
 * traced as a shadow ray (Scene::IntersectP, early exit), otherwise as a path ray (Scene::Intersect).  HOST pointers. */
typedef struct pb2_wf_hit {
    int32_t found;   /* 0 = miss, 1 = hit, 2 + i = hit inside instance i (path rays) */
    int32_t leaf;    /* position of the hit primitive in BVHAccel::primitives order (path rays), -1 = none */
    int32_t prim;    /* its scene-order primitive number, -1 = miss / shadow ray */
    float t;         /* ray.tMax after the traversal */
    float b[3];      /* barycentrics of the closest hit (sphere: phi, 0, 0) */
    int32_t listed;  /* 1 = the kernel queued the context for shading, 2 = for the light step (exactly one of them) */
} pb2_wf_hit;
int pb2_trace_wavefront(pb2_scene *scene, const pb2_ray *rays, const uint8_t *any_hit, int64_t n, int32_t flags,
                        pb2_wf_hit *out);

/* The persistent trace grid's blocks per SM when several wavefront pipelines share the GPU: the most 128-thread blocks of
 * the trace kernel (trace_regs registers per thread, trace_smem bytes of shared memory per block) that fit one H100 SM
 * together with one 128-thread block of the largest list kernel (list_regs, list_smem), at most max_blocks.  Registers
 * are allocated per warp in units of 256 from the SM's 65 536; an SM holds 2048 threads, 32 blocks and 228 KB of shared
 * memory, of which 1 KB per block is reserved.  Pure arithmetic, no device needed; 0 when not even one block fits. */
int pb2_trace_blocks_with_reserve(int32_t trace_regs, int32_t trace_smem, int32_t list_regs, int32_t list_smem, int32_t max_blocks);

/* PathIntegrator::Li for explicit (pixel, sample number) pairs, after the NaN/negative/infinite
 * guard of integrator.cpp:294-315: out_rgb gets 3 floats per sample, out_pfilm 2 floats
 * (CameraSample::pFilm).  Parity/debug entry point; HOST pointers. */
int pb2_li_samples(pb2_scene *scene, const pb2_camera *camera, const pb2_film_desc *film,
                   const pb2_path_params *params, const int32_t *pixel_xy, const int64_t *sample_num,
                   int64_t n, float *out_rgb, float *out_pfilm);

/* HaltonSampler::SampleDimension(GetIndexForSample(sample_num), dim) for a batch, evaluated on the
 * device (src/samplers/halton.cpp:96-127).  HOST pointers. */
int pb2_halton_samples(const pb2_film_desc *film, const pb2_path_params *params,
                       const int32_t *pixel_xy, const int64_t *sample_num, const int32_t *dim,
                       int64_t n, float *out);

/* SobolSampler::SampleDimension(GetIndexForSample(sample_num), dim) for a batch, evaluated on the HOST by the same source
 * functions the kernels compile (sobolIntervalToIndex, sobolSampleFloat; device/pb2_sampler.cuh) - no device needed; with
 * tables != NULL also the two SobolIntervalToIndex tables derived for this film's resolution (2 x 52 entries:
 * VdCSobolMatrices[m - 1], VdCSobolMatricesInv[m - 1], zero-padded).  Parity/debug entry point. */
int pb2_sobol_samples_host(const pb2_film_desc *film, const pb2_path_params *params, const int32_t *pixel_xy,
                           const int64_t *sample_num, const int32_t *dim, int64_t n, float *out, uint64_t *tables);

/* Distribution1D of SpatialLightDistribution::Lookup(p) (src/core/lightdistrib.cpp:141-230):
 * for each point writes n_lights func values followed by n_lights+1 cdf values. HOST pointers. */
int pb2_light_distribution(pb2_scene *scene, const float *points_xyz, int64_t n, float *out);

/* The MIP pyramid the library builds for one texture (the MIPMap constructor, src/core/mipmap.h:112-203: Lanczos
 * resampling to a power of two, then box-filtered levels).  Host code only - no device needed.  *n_levels, *w and *h
 * (resolution of `level`) are always written; `out` (channels * w * h floats, row-major) may be NULL.  Parity/debug. */
int pb2_texture_pyramid(const pb2_texture *texture, int32_t level, int32_t *n_levels, int32_t *w, int32_t *h, float *out);

/* Texture::Evaluate(si) for texture `id` (0-based) of a texture array - any kind: image, constant, scale, mix, checkerboard,
 * uv - at n points given by their (u, v) (2 floats each) and (dudx, dvdx, dudy, dvdy) (4 floats each), evaluated on the HOST by
 * the functions the kernels compile.  out: 3 floats per point (one-channel textures repeat their value).  Parity/debug. */
int pb2_texture_eval_host(const pb2_texture *textures, int32_t n_textures, int32_t id, int64_t n, const float *uv, const float *duv,
                          float *out);

/* The BSDF of one material record at given shading frames, evaluated on the HOST by the source the shade kernel compiles
 * (makeBsdf, bsdfF, bsdfPdf, bsdfSampleF; device/pb2_shade.cuh).  Parity/debug.  Per sample in: n (3), shading n (3), shading
 * dpdu (3), wo (3), wi (3), u (2) = 17 floats.  out, 19 floats: f(wo, wi) and Pdf(wo, wi) over the non-specular lobes as
 * EstimateDirect asks for them (integrator.cpp:127-130); Sample_f over the non-specular lobes (wi, f, pdf: integrator.cpp:166-169);
 * Sample_f over all lobes as the path continues (wi, f, pdf, flags: path.cpp:130-131; flags = BSDF_SAMPLED_* of pb2_shade.cuh). */
int pb2_bsdf_eval_host(const pb2_material *material, int64_t n, const float *in, float *out);

/* The two functions behind texture filtering footprints, evaluated on the HOST by the source the kernels compile.  Parity/debug.
 * pb2_camera_differentials_host: the offset rays PerspectiveCamera::GenerateRayDifferential adds to a camera ray
 * (perspective.cpp:117-144), in world space and scaled by 1 / sqrt(samples_per_pixel) (integrator.cpp:273-274).  Per sample in:
 * p_film (2), u_lens (2: CameraSample::pLens), the main ray's world o (3) and d (3) as traced = 10 floats; out: rxOrigin,
 * rxDirection, ryOrigin, ryDirection = 12 floats.
 * pb2_uv_differentials_host: SurfaceInteraction::ComputeDifferentials (interaction.cpp:101-147).  Per point in: p, n, dpdu,
 * dpdv (12 floats) and the four offset-ray vectors (12 floats) = 24 floats; out: dudx, dvdx, dudy, dvdy. */
int pb2_camera_differentials_host(const pb2_camera *camera, const pb2_film_desc *film, const pb2_path_params *params, int64_t n,
                                  const float *in, float *out);
int pb2_uv_differentials_host(int64_t n, const float *in, float *out);

/* The sampling distribution the library derives for an InfiniteAreaLight whose environment map is `texture` (infinite.cpp:64-82:
 * the Distribution2D over the 2w x 2h image of luminance * sin(theta)).  Host code only.  *nu = 2w, *nv = 2h (w, h: the map's
 * resolution after MIPMap's power-of-two resampling) are always written; `out` (may be NULL) receives nv rows of
 * [func(nu) | cdf(nu + 1) | funcInt] followed by the marginal [func(nv) | cdf(nv + 1) | funcInt].  Parity/debug. */
int pb2_env_distribution(const pb2_texture *texture, int32_t *nu, int32_t *nv, float *out);

/* MIPMap::Lookup(st, dst0, dst1) (mipmap.h:260-287: trilinear or EWA as the texture says) for a batch, evaluated on the
 * device with the code the shade kernel uses.  st: 2 floats per look-up, dst: 4 (dst0.x dst0.y dst1.x dst1.y), out: 3
 * (one-channel textures repeat their value).  The UVMapping2D parameters of the texture are NOT applied.  HOST pointers. */
int pb2_texture_lookup(const pb2_texture *texture, int64_t n, const float *st, const float *dst, float *out);

/* The lower half of BVHAccel::HLBVHBuild on the device (src/accelerators/bvh.cpp:404-470): Morton codes of the primitive
 * centroids over the centroid bounds (bvh.cpp:408-423), the stable sort by the 30-bit code (RadixSort, bvh.cpp:139-180),
 * and one LBVH treelet per distinct top-12-bit prefix (bvh.cpp:428-466, emitLBVH 472-539).  The caller finishes with
 * buildUpperSAH over the treelet roots (bvh.cpp:541-638) and flattens.
 *   prim_bounds      n x 6 floats, (pMin, pMax) of each primitive's world bound, in primitive order
 *   pool             2n records; treelet t's nodes occupy pool[2*start_t ...], children are pool indices
 *   ordered_prims    n primitive numbers in sorted (= BVHAccel::primitives) order; a leaf's first_prim_offset indexes it
 *   treelet_roots    up to 4096 pool indices in sorted order, *n_treelets of them
 * HOST pointers; blocking.  The result equals the host build (and the reference run by one thread) bit for bit. */
typedef struct pb2_build_node {
    float bmin[3], bmax[3];
    int32_t child[2];          /* -1, -1 for a leaf */
    int32_t split_axis;
    int32_t first_prim_offset;
    int32_t n_primitives;      /* 0 for an interior node */
} pb2_build_node;
int pb2_hlbvh_treelets(const float *prim_bounds, int64_t n, int32_t max_prims_in_node, pb2_build_node *pool,
                       int32_t *ordered_prims, int32_t *treelet_roots, int32_t *n_treelets, double *device_ms);

/* All of BVHAccel::HLBVHBuild and flattenBVHTree on the device (bvh.cpp:404-658): the stages above, then buildUpperSAH over
 * the treelet roots (bvh.cpp:541-638; one thread - at most 4096 leaves, each split partitions the range the next ones work
 * on - with libstdc++'s std::partition order) and the depth-first LinearBVHNode layout (bvh.cpp:640-658; a treelet's nodes
 * are numbered depth-first when they are emitted, so each lands as one block).  Only the finished array crosses the bus:
 *   nodes            room for 2n LinearBVHNodes; *n_nodes of them are written
 *   ordered_prims    n primitive numbers in BVHAccel::primitives order
 * HOST pointers; blocking.  Bit for bit the nodes the host build (and the reference run by one thread) produces. */
int pb2_hlbvh_build(const float *prim_bounds, int64_t n, int32_t max_prims_in_node, pb2_bvh_node *nodes, int64_t *n_nodes,
                    int32_t *ordered_prims, double *device_ms);

#ifdef __cplusplus
}
#endif
#endif /* PB2_H */
