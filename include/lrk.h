/*
 * lrk.h — C-ABI of the CUDA radiance kernel library (libb200pt.so).
 *
 * This is the drop-in boundary below LuisaRender's integrator interface
 * (SURVEY.md §8b).  The reference's Integrator/Surface/Light/Sampler classes are
 * DSL-staging objects (they record an AST, they are not callable at run time), so
 * the run-time boundary sits one level lower: the host (scene parsing, flattening,
 * BVH build, film I/O — include/lrh.h) hands a flattened, POD scene to this
 * library, which owns all device memory and runs the per-sample radiance loop in
 * hand-written sm_90a CUDA.
 *
 * What each entry point replaces in the reference (paths relative to /root/reference):
 *   lrk_create          <- Context::create_device + Device::create_stream      src/apps/cli.cpp:167-181
 *   lrk_upload_scene    <- Pipeline::create (Geometry::build, register_surface/light,
 *                          Integrator::build)                                    src/base/pipeline.cpp:44-99
 *   lrk_set_shard       <- (none: the reference is single device)               SURVEY.md §8e
 *   lrk_comm_unique_id / lrk_comm_init / lrk_reduce_film
 *                       <- (none; sums the film of src/films/color.cpp:107-130 over ranks)  SURVEY.md §8e
 *   lrk_film_clear      <- Film::Instance::prepare / clear                      src/films/color.cpp:132-144
 *   lrk_render          <- ProgressiveIntegrator::Instance::_render_one_camera  src/integrators/wave_path.cpp:220-567
 *   lrk_render_adaptive / lrk_download_sample_counts / lrk_download_film_variance
 *                       <- (none: an extension, the reference has no adaptive sampling)  DESIGN.md §4 (Adaptive sampling)
 *   option "gbuffer" / lrk_download_gbuffer / lrk_denoise
 *                       <- (none: an extension, the reference has no G-buffer and no denoiser)  DESIGN.md §4 (G-buffer and denoiser)
 *   lrk_download_film   <- Film::Instance::download (convert_image + copy)      src/films/color.cpp:87-105
 *   lrk_download_film_raw / lrk_film_device_ptr
 *                       <- the raw (sum rgb, sum weight) float4 film buffer     src/films/color.cpp:107-130
 *   lrk_trace           <- Geometry::trace_closest / trace_any                  src/base/geometry.cpp:218-279
 *   lrk_get_stats       <- "Rendering finished in {} ms." + device counters     src/integrators/wave_path.cpp:565-566
 *   lrk_last_error      <- LUISA_ERROR (log + abort)                            src/compute/include/luisa/core/logging.h:63
 *
 * Conventions: every function is extern "C", takes plain pointers and sizes, never
 * throws; returns 0 on success or a negative lrk_status.  All host arrays passed to
 * lrk_upload_scene are copied; the caller keeps ownership.  One lrk_ctx per GPU; calls
 * on one ctx must come from one thread at a time.
 */
#ifndef LRK_H
#define LRK_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LRK_ABI_VERSION 8u /* 7: lrk_render_adaptive, lrk_download_sample_counts, lrk_download_film_variance;
                              8: option "gbuffer", lrk_download_gbuffer, lrk_denoise */

typedef enum lrk_status {
    LRK_OK = 0,
    LRK_ERR_INVALID_ARGUMENT = -1,
    LRK_ERR_NO_DEVICE = -2,
    LRK_ERR_CUDA = -3,
    LRK_ERR_NO_SCENE = -4,
    LRK_ERR_UNSUPPORTED = -5,
    LRK_ERR_OUT_OF_MEMORY = -6
} lrk_status;

/* ---- geometry records (layouts follow SURVEY.md App. B) ---------------------------- */

/* Vertex, 32 B: src/util/vertex.h:37-56 */
typedef struct lrk_vertex {
    float p[3];
    float n[3];
    float uv[2];
} lrk_vertex;

/* Triangle, 12 B: src/compute/include/luisa/runtime/rtx/triangle.h:7-11 */
typedef struct lrk_triangle {
    uint32_t i0, i1, i2;
} lrk_triangle;

/* AliasEntry, 8 B: src/util/sampling.h:29-32 */
typedef struct lrk_alias_entry {
    float prob;
    uint32_t alias;
} lrk_alias_entry;

/* Ray, 32 B: src/compute/include/luisa/runtime/rtx/ray.h:10-16 */
typedef struct lrk_ray {
    float o[3];
    float tmin;
    float d[3];
    float tmax;
} lrk_ray;

/* Hit, 16 B: src/base/geometry.h:16-27; miss <=> inst == ~0u */
typedef struct lrk_hit {
    uint32_t inst;
    uint32_t prim;
    float bary[2];
} lrk_hit;

/* One unique mesh (= one BLAS).  Mirrors the four bindless slots of
 * src/base/geometry.cpp:68-84: vertices, triangles, alias table, pdf. Offsets index the
 * scene-global arrays of lrk_scene_desc. */
typedef struct lrk_mesh {
    uint32_t vertex_offset;
    uint32_t vertex_count;
    uint32_t triangle_offset; /* also the offset into alias[] and pdf[] */
    uint32_t triangle_count;
    uint32_t bvh_root;        /* index of this BLAS's root node in bvh_nodes[] */
    uint32_t tri_slot_offset; /* first BVH-ordered triangle slot of this mesh in tri_verts[] */
    uint32_t reserved[2];
} lrk_mesh;

/* BVH2 node, 64 B: both children's boxes + two child references.
 * ref: bit31 = leaf.  BLAS leaf: bits 28..30 = triangle count - 1, bits 0..27 = first
 * triangle slot (scene-global, indexes tri_verts[3*slot .. 3*slot+2]).  TLAS leaf:
 * bits 0..30 = instance index.  An unused child has an inverted box (lo=+inf, hi=-inf)
 * and ref LRK_BVH_EMPTY. */
typedef struct lrk_bvh_node {
    float lo0[3], hi0[3];
    float lo1[3], hi1[3];
    uint32_t ref0, ref1;
    uint32_t parent; /* index of the parent node (root: ~0u) */
    uint32_t reserved;
} lrk_bvh_node;

#define LRK_BVH_LEAF 0x80000000u
#define LRK_BVH_EMPTY 0xffffffffu
#define LRK_BVH_MAX_LEAF_TRIS 4u

/* One TLAS instance = one mesh leaf of the flattened shape graph
 * (src/base/geometry.cpp:29-163).  `handle` is exactly Shape::Handle::encode
 * (src/base/shape.cpp:46-70) with buffer_base = 4 * mesh index. */
typedef struct lrk_instance {
    uint32_t handle[4];
    float object_to_world[12]; /* row-major 3x4 */
    float world_to_object[12]; /* row-major 3x4 */
    uint32_t mesh;
    uint32_t visible; /* src/base/geometry.cpp:130-131: invisible instances are skipped by all rays */
    uint32_t reserved[2];
} lrk_instance;

/* Shape property flags: src/base/shape.h:34-39 */
#define LRK_SHAPE_HAS_VERTEX_NORMAL 1u
#define LRK_SHAPE_HAS_VERTEX_UV 2u
#define LRK_SHAPE_HAS_SURFACE 4u
#define LRK_SHAPE_HAS_LIGHT 8u
#define LRK_SHAPE_HAS_MEDIUM 16u
#define LRK_SHAPE_MAYBE_NON_OPAQUE 32u

/* ---- materials, lights ---------------------------------------------------------------- */

#define LRK_SURFACE_MATTE 0u  /* src/surfaces/matte.cpp */
#define LRK_SURFACE_DISNEY 1u /* src/surfaces/disney.cpp: closure class "disney", or "disney_trans" / "disney_thin" by the flags below */
#define LRK_SURFACE_MIRROR 2u  /* src/surfaces/mirror.cpp */
#define LRK_SURFACE_GLASS 3u   /* src/surfaces/glass.cpp (non-dispersive: fixed sRGB spectrum) */
#define LRK_SURFACE_PLASTIC 4u /* src/surfaces/plastic.cpp */
#define LRK_SURFACE_METAL 5u   /* src/surfaces/metal.cpp */
#define LRK_SURFACE_MIX 6u     /* src/surfaces/mix.cpp: two constant, non-Disney surface records mixed by a ratio */
#define LRK_SURFACE_LAYERED 7u /* src/surfaces/layered.cpp: two constant, non-Disney interfaces around a scattering slab */
#define LRK_SURFACE_TYPE_COUNT 8u

/* Surface::event_*: src/base/surface.h:37-41 */
#define LRK_EVENT_REFLECT 0u
#define LRK_EVENT_ENTER 1u
#define LRK_EVENT_EXIT 2u
#define LRK_EVENT_THROUGH 4u /* transmission through a thin surface: the path stays in its medium, no eta scale */

/* Disney lobe bits: src/surfaces/disney.cpp:326-333 */
#define LRK_DISNEY_LOBE_DIFFUSE 1u
#define LRK_DISNEY_LOBE_RETRO 2u
#define LRK_DISNEY_LOBE_FAKE_SS 4u
#define LRK_DISNEY_LOBE_SHEEN 8u
#define LRK_DISNEY_LOBE_CLEARCOAT 16u
#define LRK_DISNEY_LOBE_SPECULAR 32u
#define LRK_DISNEY_LOBE_DIFF_TRANS 64u
#define LRK_DISNEY_LOBE_SPEC_TRANS 128u

/* One surface node (tag = index), constants already decoded the way the reference's
 * constant textures + sRGB spectrum decode them (src/base/texture.cpp:15-80,
 * src/spectra/srgb.cpp:34-40).
 *   MATTE : p[0..2] = Kd, p[3] = sigma in degrees (saturate(v)*90, 0 if absent)
 *   DISNEY: p[0..2] = color, p[3] = color_lum, p[4] = metallic, p[5] = eta, p[6] = roughness
 *           (already remapped to alpha when remap_roughness), p[7] = specular_tint,
 *           p[8] = anisotropic, p[9] = sheen, p[10] = sheen_tint, p[11] = clearcoat,
 *           p[12] = clearcoat_gloss, p[13] = specular_trans, p[14] = flatness,
 *           p[15] = diffuse_trans; lobes = union of enabled lobes over all disney surface nodes of the scene
 *           that share the record's closure class (opaque / LRK_SURFACE_DISNEY_TRANSMISSIVE / LRK_SURFACE_DISNEY_THIN; the reference ORs them
 *           into one shared closure per class, src/surfaces/disney.cpp:869,994-995).
 *   MIRROR : p[0..2] = reflectance colour, p[3..4] = alpha (roughness after the optional remap; 0 without a roughness
 *            node: the distribution clamps it to 1e-4) — MirrorClosure::Context, mirror.cpp:84-88,142-162
 *   GLASS  : p[0..2] = Kr, p[3..5] = Kt, p[6] = eta_t (default 1.5; eta_i is 1), p[7..8] = alpha,
 *            p[9] = Kr_ratio = lum(Kr) / (lum(Kr) + lum(Kt)) — GlassClosure::Context, glass.cpp:133-142,229-279
 *   PLASTIC: p[0..2] = Kd / (1 - Kd * fresnel_dielectric_integral(eta)), p[3] = Kd_weight = lum(Kd) * exp(-2 lum(sigma_a)
 *            thickness), p[4..6] = sigma_a (NOT scaled by thickness, as the reference binds it), p[7] = eta,
 *            p[8..9] = alpha — PlasticContext, plastic.cpp:107-114,252-291
 *   METAL  : p[0..2] = n, p[3..5] = k (complex index at the spectrum's three wavelengths), p[6..8] = Kd reflectance tint,
 *            p[9..10] = alpha (default 0.5) — MetalClosure::Context, metal.cpp:208-215,273-310
 *   MIX    : p[0] = ratio = clamp(ratio.x, 0, 1) (default 0.5); mix_a / mix_b = indices of the two mixed surface records, which
 *            the host appends behind the tagged surfaces (surface_count counts them; instance handles never name them) —
 *            MixSurfaceClosure::Context, mix.cpp:88-91,195-211.  The closure reproduces the reference's arithmetic including
 *            its second sampling branch, which samples surface `a` again and weights the two evaluations the other way
 *            round (mix.cpp:170-176).
 *   LAYERED: p[0] = thickness (>= FLT_MIN), p[1] = g, p[2..4] = albedo, lobes = max_depth | samples << 16; mix_a / mix_b = record
 *            indices of the top / bottom interface (constant Matte / Mirror / Glass / Plastic / Metal records appended like a Mix's) —
 *            LayeredSurfaceClosure::Context, layered.cpp:205-212,478-503
 *   With image-textured parameters the four records use the raw layouts of LRK_SURFACE_RAW_PARAMS below.
 *
 * Image-textured parameters (SURVEY.md §8 row f1): tex[k] != 0 means parameter slot k is NOT the constant p[k] but is
 * evaluated per hit from image texture (tex[k] - 1) at the hit's uv, exactly as populate_closure does
 * (src/surfaces/matte.cpp:117-131, src/surfaces/disney.cpp:932-956):
 *   colour slots (MATTE 0, DISNEY 0): rgb = saturate(extend_color_to_rgb(v.xyz, channels)) -> p[0..2] (+ luminance ->
 *   p[3] for DISNEY); MATTE slot 3: saturate(v.x) * 90; DISNEY scalar slots 4..15: v.x, slot 6 additionally remapped
 *   max(v.x^2, 1e-4) when LRK_SURFACE_REMAP_ROUGHNESS is set in flags.
 *
 * Wrappers every surface node carries (NormalMapWrapper<OpacitySurfaceWrapper<...>>, src/base/surface.h:160-275):
 *   opacity   : LRK_SURFACE_MAYBE_NON_OPAQUE set when an `alpha` / `opacity` texture exists whose static value is < 1 (:177-181);
 *               alpha at a candidate hit = opacity_tex ? image(opacity_tex - 1, uv).x : opacity; the candidate is skipped when
 *               xxhash32(inst, prim, bary bits) * 2^-32 > alpha (Geometry::_alpha_skip, src/base/geometry.cpp:165-192), in
 *               closest-hit and any-hit traversal alike (:218-279).  Instances of such surfaces carry
 *               LRK_SHAPE_MAYBE_NON_OPAQUE in their handle flags (:123-126).
 *   normal map: LRK_SURFACE_HAS_NORMAL_MAP: n_local = 2 * rgb - 1 (rgb = image(normal_tex - 1, uv) or normal_value), x and y
 *               scaled by normal_strength when != 1, shading frame rebuilt around clamp_shading_normal (surface.h:236-253). */
#define LRK_SURFACE_HAS_TEXTURES 1u
#define LRK_SURFACE_REMAP_ROUGHNESS 2u
#define LRK_SURFACE_MAYBE_NON_OPAQUE 4u
#define LRK_SURFACE_HAS_NORMAL_MAP 8u
/* DISNEY only: the node is transmissive (`specular_trans` given and not black, not `thin`): the reference builds the closure
 * class "disney_trans" for it (src/surfaces/disney.cpp:61-75,925-930,1001-1007) - a fourth sampling technique with a
 * MicrofacetTransmission lobe (:452-464), a one-sided DisneyFresnel (:425), eta() = eta_t for the Russian-roulette scale
 * (:531-533).  `lobes` of such records is the union over the TRANSMISSIVE Disney nodes of the scene (each closure class
 * collects its own, :994-995). */
#define LRK_SURFACE_DISNEY_TRANSMISSIVE 16u
/* MIRROR / GLASS / PLASTIC / METAL with an image-textured parameter: p[] holds the node's RAW parameters and the closure context
 * above is derived per hit (colour slots: saturate(extend_color_to_rgb(texel)), as populate_closure's evaluate_albedo_spectrum;
 * alpha slots: a 1-channel roughness texture feeds both axes, a 2-channel one x and y, remapped max(r^2, 1e-4) when
 * LRK_SURFACE_REMAP_ROUGHNESS is set - a slot WITHOUT a texture already holds the final alpha):
 *   MIRROR : p[0..2] colour (tex[0]), p[3..4] alpha (tex[3])                                          mirror.cpp:142-162
 *   GLASS  : p[0..2] Kr (tex[0]), p[3..5] Kt (tex[3]), p[6] eta_t, p[7..8] alpha (tex[7]); p[9] = Kr_ratio from the luminances  glass.cpp:236-279
 *   PLASTIC: p[0..2] Kd (tex[0]), p[4..6] sigma_a (tex[4]), p[7] eta, p[8..9] alpha (tex[8]), p[10] thickness (tex[10]);
 *            p[0..2] <- Kd / (1 - Kd Fdr(eta)), p[3] <- lum(Kd) exp(-2 lum(sigma_a) thickness)        plastic.cpp:252-291
 *   METAL  : p[0..5] n, k (never textured), p[6..8] Kd (tex[6]), p[9..10] alpha (tex[9])               metal.cpp:273-310 */
#define LRK_SURFACE_RAW_PARAMS 32u
/* DISNEY only: a `thin` node with a non-black `specular_trans` or `diffuse_trans` (src/surfaces/disney.cpp:61-69): the closure class
 * "disney_thin" (ThinDisneyClosureImpl, :590-845) - five sampling techniques: the diffuse-like lobes weighted by
 * (1 - diffuse_trans), specular, clearcoat, a MicrofacetTransmission lobe through a distribution rescaled by
 * (0.65 eta - 0.35) (:686-701) and a Lambertian diffuse-transmission lobe weighted by p[15] = diffuse_trans (:703-710); both
 * transmissions report LRK_EVENT_THROUGH, and the closure has no eta().  `lobes` is the union over the THIN Disney nodes.
 * A `thin` node with neither transmission is an ordinary opaque Disney record. */
#define LRK_SURFACE_DISNEY_THIN 64u
typedef struct lrk_surface {
    uint32_t type;
    uint32_t lobes;
    uint32_t flags;
    uint32_t mix_a; /* MIX: record index of surface `a` */
    float p[16];
    uint32_t tex[16];
    uint32_t opacity_tex; /* 0 = constant `opacity` */
    float opacity;
    uint32_t normal_tex; /* 0 = constant `normal_value` */
    float normal_strength;
    float normal_value[3];
    uint32_t mix_b; /* MIX: record index of surface `b` */
} lrk_surface;

/* One image texture (src/textures/image.cpp:16-151).  Texels are RGBA float (8/16-bit sources converted with x/255,
 * x/65535: cpu_texture.h:63), row-major, row 0 first as stored in the file; sampling follows the reference's software
 * sampler (src/compute/src/rust/luisa_compute_backend_impl/src/cpu/codegen/cpu_texture.h:418-464,489-493), level 0 only
 * (the reference's evaluate() samples without LOD, image.cpp:165). */
#define LRK_TEX_ADDRESS_EDGE 0u
#define LRK_TEX_ADDRESS_REPEAT 1u
#define LRK_TEX_ADDRESS_MIRROR 2u
#define LRK_TEX_ADDRESS_ZERO 3u
#define LRK_TEX_FILTER_POINT 0u
#define LRK_TEX_FILTER_LINEAR 1u
#define LRK_TEX_ENCODING_LINEAR 0u
#define LRK_TEX_ENCODING_SRGB 1u
#define LRK_TEX_ENCODING_GAMMA 2u
typedef struct lrk_texture {
    uint64_t texel_offset; /* index of the first float4 texel in lrk_scene_desc::texels */
    uint32_t width, height;
    uint32_t channels; /* channels of the source image (1..4) */
    uint32_t address, filter, encoding;
    float scale, gamma;
    float uv_scale[2], uv_offset[2];
    uint32_t reserved[2];
} lrk_texture;

/* One light node (tag = index): src/lights/diffuse.cpp:23-26. emission is the decoded
 * illuminant (max(rgb,0)), L = emission * scale.
 * emission_tex != 0: the emission is image texture (emission_tex - 1), L = max(texel.xyz, 0) * scale
 * (Texture::Instance::evaluate_illuminant_spectrum, src/base/texture.cpp:47-57: no channel extension on this path), looked up
 * at the uv of the emitter hit or of the sampled light point (the light sampler builds that interaction with the full shading
 * attributes, src/lightsamplers/uniform.cpp:108-123). */
typedef struct lrk_light {
    float emission[3];
    float scale;
    uint32_t two_sided;
    uint32_t emission_tex;
    uint32_t reserved[2];
} lrk_light;

/* Light::Handle, 8 B: src/base/light.h:26-29 */
typedef struct lrk_light_handle {
    uint32_t instance_id;
    uint32_t light_tag;
} lrk_light_handle;

/* ---- camera, film, integrator ------------------------------------------------------- */

#define LRK_FILTER_LUT_SIZE 64u /* src/base/filter.h:18 */

typedef struct lrk_camera {
    float camera_to_world[12]; /* row-major 3x4 */
    uint32_t resolution[2];
    float tan_half_fov;     /* src/cameras/pinhole.cpp:56-57 */
    float filter_radius;    /* src/base/filter.cpp:13 */
    float filter_shift[2];
    uint32_t spp;           /* src/base/camera.cpp:28 */
    uint32_t reserved;
    float filter_lut[LRK_FILTER_LUT_SIZE];              /* src/base/filter.cpp:24-48 */
    float filter_pdf[LRK_FILTER_LUT_SIZE];              /* 63 used */
    float filter_alias_probs[LRK_FILTER_LUT_SIZE];      /* 63 used */
    uint32_t filter_alias_indices[LRK_FILTER_LUT_SIZE]; /* 63 used */
} lrk_camera;

typedef struct lrk_film {
    float scale[3]; /* 2^exposure, src/films/color.cpp:38-40 */
    float clamp;    /* src/films/color.cpp:41 */
} lrk_film;

#define LRK_INTEGRATOR_PATH 0u       /* src/integrators/wave_path.cpp (== mega_path.cpp estimator) */
#define LRK_INTEGRATOR_VOLUME_PATH 1u /* src/integrators/mega_vpt_naive.cpp (config C4) */

typedef struct lrk_integrator {
    uint32_t type;
    uint32_t max_depth;        /* src/integrators/wave_path.cpp:43 */
    uint32_t rr_depth;         /* :44 */
    float rr_threshold;        /* :45 */
    uint32_t samples_per_pass; /* :46 (a hint: the pass size is chosen by the library) */
    uint32_t sampler_seed;     /* src/base/sampler.cpp:11 */
    uint32_t reserved[2];
} lrk_integrator;

/* A participating medium (row a22): src/media/homogeneous.cpp, src/media/vacuum.cpp.  `present` is the kind: a vacuum medium has
 * priority LRK_MEDIUM_VACUUM_PRIORITY and never becomes the current medium of a path (src/util/medium_tracker.cpp:23-43). */
#define LRK_MEDIUM_NONE 0u
#define LRK_MEDIUM_HOMOGENEOUS 1u
#define LRK_MEDIUM_VACUUM 2u
#define LRK_MEDIUM_VACUUM_PRIORITY 0xffffffffu /* Medium::VACUUM_PRIORITY, src/base/medium.h:29 */
#define LRK_MEDIUM_INVALID_TAG 0xffffffffu     /* Medium::INVALID_TAG, src/base/medium.h:28 */
typedef struct lrk_medium {
    uint32_t present;
    uint32_t priority;
    float eta;
    float g; /* Henyey-Greenstein */
    float sigma_a[3];
    float sigma_s[3];
    float le[3];
    float reserved[3];
} lrk_medium;

/* The environment light (SURVEY.md §8 rows a12 / f3): src/environments/spherical.cpp with the uniform light sampler's
 * environment handling (src/lightsamplers/uniform.cpp:40-47,67-76,78-101,139-146).
 *   L(w)  = max(rgb, 0) * scale, rgb = emission texture at direction_to_uv(world_to_env * w) (spherical.cpp:51-58,70-75;
 *           illuminant decode src/spectra/srgb.cpp:48-54) or the constant `emission`
 *   image emission: importance sampling from a map_width x map_height (2048 x 1024) table built on the host exactly like
 *           Spherical::build (:140-236): Gaussian-filtered luminance * sin(theta), optional MIS compensation, one alias table
 *           per row + the marginal one.  alias = [map_height marginal entries][map_height * map_width conditional entries],
 *           pdf[y * map_width + x] = p(x,y) * pixel_count; directional pdf = pdf / sin(theta) / (2 pi^2) (:77-81)
 *   constant emission: uniform sphere sampling, pdf = 1 / (4 pi)
 *   env_prob: probability with which next-event estimation picks the environment (1 when there are no area lights, else
 *           clamp(environment_weight, 0.01, 0.99), uniform.cpp:40-47); area-light pdfs are scaled by (1 - env_prob). */
typedef struct lrk_environment {
    uint32_t present;
    uint32_t emission_tex; /* 0 = constant emission, else image texture id + 1 */
    float emission[3];     /* constant emission (already max(rgb, 0)) */
    float scale;
    float env_prob;
    float to_world[9]; /* row-major 3x3: environment -> world (make_float3x3 of the node's transform) */
    uint32_t map_width, map_height; /* 0 x 0 for constant emission */
    uint32_t reserved;
    const lrk_alias_entry *alias; /* map_height + map_height * map_width entries */
    const float *pdf;             /* map_height * map_width */
} lrk_environment;

/* The sampler (SURVEY.md §8 rows a1 / f2): src/base/sampler.h:42-48 as implemented by src/samplers/{independent,pmj02bn,sobol,
 * padded_sobol,zsobol}.cpp.  INDEPENDENT needs nothing but integrator.sampler_seed.  The quasi-Monte-Carlo samplers are
 * table driven; the host passes the tables (luisarender_b200/data/sampler_tables.bin, tools/extract_sampler_tables.py) and
 * what Sampler::Instance::reset(resolution, spp) derives from them on the host:
 *   PMJ02BN      pmj_samples u32[5][65536][2], blue_noise u16[48][128][128]; spp (<= 65536), w = the bit mask covering spp - 1,
 *                tile = pixel_tile_size, pmj_pixel_samples float2[tile * tile * spp] (the sorted first set, pmj02bn.cpp:132-162)
 *   SOBOL        sobol_matrices u32[1024][52]; scale = next_pow2(max(resolution)), vdc / vdc_inv u64[52] = the rows m - 1 of the
 *                van-der-Corput matrices for m = log2(scale) (sobol.cpp:112-131)
 *   PADDED_SOBOL sobol_matrices (the first two dimensions are read); spp
 *   ZSOBOL       sobol_matrices (first two dimensions); log2_spp, num_base4_digits (zsobol.cpp:96-103),
 *                zsobol_hash uint2[1024] = hash_value((seed << 32) | i) (zsobol.cpp:71-79)
 * Every sampler draws in the order the integrator asks (generate_pixel_2d for the filter, then 1D / 2D per bounce, App. A). */
#define LRK_SAMPLER_INDEPENDENT 0u
#define LRK_SAMPLER_PMJ02BN 1u
#define LRK_SAMPLER_SOBOL 2u
#define LRK_SAMPLER_PADDED_SOBOL 3u
#define LRK_SAMPLER_ZSOBOL 4u
typedef struct lrk_sampler {
    uint32_t type;
    uint32_t spp;
    uint32_t w;                /* PMJ02BN */
    uint32_t tile;             /* PMJ02BN: pixel_tile_size */
    uint32_t scale;            /* SOBOL */
    uint32_t log2_spp;         /* ZSOBOL */
    uint32_t num_base4_digits; /* ZSOBOL */
    uint32_t reserved;
    const uint32_t *sobol_matrices;
    const uint64_t *vdc;
    const uint64_t *vdc_inv;
    const uint32_t *pmj_samples;
    const uint16_t *blue_noise;
    const float *pmj_pixel_samples;
    uint64_t pmj_pixel_sample_count; /* float2 entries */
    const uint32_t *zsobol_hash;
} lrk_sampler;

typedef struct lrk_scene_desc {
    uint32_t abi_version; /* LRK_ABI_VERSION */
    uint32_t reserved0;

    const lrk_vertex *vertices;
    uint64_t vertex_count;
    const lrk_triangle *triangles;
    const lrk_alias_entry *alias;
    const float *pdf;
    uint64_t triangle_count;

    const lrk_mesh *meshes;
    uint32_t mesh_count;
    uint32_t instance_count;
    const lrk_instance *instances;

    const lrk_bvh_node *bvh_nodes;
    uint64_t bvh_node_count;
    uint32_t tlas_root;
    uint32_t reserved1;
    const float *tri_verts; /* 12 floats per BVH-ordered slot: v0.xyz, as_float(prim id), v1.xyz, 0, v2.xyz, 0 */
    uint64_t tri_slot_count;

    const lrk_surface *surfaces;
    uint32_t surface_count;
    uint32_t light_count; /* number of distinct light NODES */
    const lrk_light *lights;
    const lrk_light_handle *light_handles; /* first light_count per-instance handles (src/lightsamplers/uniform.cpp:34-38) */

    const lrk_texture *textures; /* image textures referenced by lrk_surface::tex (may be NULL when texture_count == 0) */
    uint32_t texture_count;
    uint32_t reserved2;
    const float *texels; /* RGBA float texels of all textures, 4 floats each */
    uint64_t texel_count;

    lrk_camera camera;
    lrk_film film;
    lrk_integrator integrator;
    lrk_medium environment_medium; /* copy of media[environment_medium_tag]; present = 0 when the scene has none */
    lrk_environment environment;
    lrk_sampler sampler;
    /* every medium of the scene, indexed by the medium tag of the shape handles: shape media in the order Geometry::build meets
     * them (src/base/geometry.cpp:134-142), then the environment medium (src/base/pipeline.cpp:72-79).  The order is part of the
     * result: MediumTracker::true_hit is called with a TAG where it expects a priority (src/integrators/mega_vpt_naive.cpp:387). */
    const lrk_medium *media;
    uint32_t medium_count;
    uint32_t environment_medium_tag; /* LRK_MEDIUM_INVALID_TAG: none */
} lrk_scene_desc;

/* ---- device control ----------------------------------------------------------------- */

typedef struct lrk_device_cfg {
    int32_t device_index;      /* -1: current device */
    uint32_t reserved;
    uint64_t max_paths_per_pass; /* 0: default (8 Mi) */
} lrk_device_cfg;

typedef struct lrk_stats {
    double render_ms;        /* device time of all lrk_render calls since the last lrk_film_clear */
    uint64_t samples;        /* camera samples started */
    uint64_t closest_rays;   /* rays traced by the closest-hit kernel */
    uint64_t shadow_rays;    /* rays traced by the any-hit kernel */
    uint64_t kernel_launches;
    uint64_t passes;
    /* filled only when counting is enabled (lrk_set_option("count_traversal", 1)) */
    uint64_t closest_nodes;  /* N_int of the closest-hit kernel (SURVEY.md §8d): 128-byte 4-wide nodes visited */
    uint64_t closest_tris;   /* N_tri */
    uint64_t closest_xforms; /* N_xform */
    uint64_t shadow_nodes;   /* the same three for the any-hit kernel */
    uint64_t shadow_tris;
    uint64_t shadow_xforms;
    double trace_closest_ms; /* CUDA-event time of the closest-hit kernel launches (when "time_kernels" = 1) */
    double trace_shadow_ms;
    double shade_ms;
    double other_ms;
    double reduce_ms; /* CUDA-event time of the lrk_reduce_film calls */
} lrk_stats;

typedef struct lrk_ctx lrk_ctx;

int lrk_abi_version(void);
int lrk_create(const lrk_device_cfg *cfg, lrk_ctx **out);
void lrk_destroy(lrk_ctx *ctx);
const char *lrk_last_error(const lrk_ctx *ctx);

int lrk_upload_scene(lrk_ctx *ctx, const lrk_scene_desc *scene);

/* Pixel-tile sharding for multi-GPU (SURVEY.md §8e): this ctx renders the tiles with
 * lrk_tile_owner(tile_id, world) == rank, tiles are tile_size x tile_size pixels in row-major tile order.
 *
 * Every run of `world` consecutive tiles hands one tile to each rank (exact balance of the tile COUNT), and the order inside
 * a run is rotated by a hash of the run's index: a plain tile_id % world makes every rank own fixed columns or diagonals of
 * the image whenever world and the number of tile columns share a factor (60 columns, 8 ranks: two column stripes per rank),
 * and the cost of a tile follows the image's structure. */
static inline uint32_t lrk_tile_owner(uint32_t tile_id, uint32_t world) {
    uint32_t run = tile_id / world, h = run * 0x9E3779B1u;
    h ^= h >> 15;
    h *= 0x85EBCA77u;
    h ^= h >> 13;
    return (tile_id % world + h % world) % world;
}
int lrk_set_shard(lrk_ctx *ctx, uint32_t rank, uint32_t world, uint32_t tile_size);

/* Cost-balanced sharding.  The static map above balances the tile COUNT; the cost of a tile follows the image (sky vs. geometry),
 * and at 8 ranks the slowest rank of the benchmark frame was 9 % over the mean.  lrk_balance_shards renders `probe_spp` samples of
 * the WHOLE frame on this context (every rank does the same, independently: the probe is deterministic, so all ranks arrive at the
 * same table without talking to each other), counts the rays traced for the pixels of every tile, assigns the tiles to ranks with
 * lrk_assign_tiles, and makes this context render rank `rank`'s tiles from then on (until the next lrk_set_shard /
 * lrk_upload_scene); the film is cleared.  The probe costs probe_spp / spp of a frame; the reduced film is bit-identical to a
 * single-GPU render whatever the assignment.
 * lrk_assign_tiles (host only, no GPU): longest-processing-time-first - tiles in order of decreasing cost (ties: lower tile id)
 * each go to the rank with the smallest load so far (ties: lower rank); owner[t] = rank of tile t. */
int lrk_balance_shards(lrk_ctx *ctx, uint32_t rank, uint32_t world, uint32_t tile_size, uint32_t probe_spp);
int lrk_assign_tiles(const uint32_t *cost, uint32_t tile_count, uint32_t world, uint32_t *owner);

/* The film reduce of the multi-GPU path (SURVEY.md §8e; the reference is single-device, its film is src/films/color.cpp:107-130).
 * One process per GPU.  One rank calls lrk_comm_unique_id and hands the LRK_COMM_ID_BYTES to the others by any means (a file,
 * MPI, torch.distributed); every rank then calls lrk_comm_init (collective) once, renders its tiles (lrk_set_shard), and calls
 * lrk_reduce_film (collective): the raw film of rank `root` becomes the sum over ranks - bit-identical to a single-GPU render,
 * since every pixel has exactly one owner - and the other ranks' films are left as they were.  NCCL is opened at run time
 * (libnccl.so.2; the copy already loaded into the process, if any); without it these calls return LRK_ERR_UNSUPPORTED. */
#define LRK_COMM_ID_BYTES 128
int lrk_comm_unique_id(uint8_t *id);
int lrk_comm_init(lrk_ctx *ctx, const uint8_t *id, uint32_t rank, uint32_t world);
int lrk_reduce_film(lrk_ctx *ctx, uint32_t root);

/* Options (unknown name -> LRK_ERR_INVALID_ARGUMENT):
 *   "count_traversal" (0/1)   traversal kernels count wide nodes / triangles / instance entries into lrk_stats
 *   "time_kernels" (0/1)      CUDA-event time per kernel category into lrk_stats
 *   "max_paths_per_pass" (n)  path-state capacity of one pass
 *   "refill_below", "inner_min" (1..32)  warp scheduling of the traversal kernels (results do not depend on them)
 *   "strict_math" (0/1)       closure kernels in IEEE arithmetic without FMA contraction (films then equal the CPU oracle's to
 *                             rel-L2 ~ 1e-7) instead of the fast-math arithmetic the reference's own CUDA backend compiles its
 *                             kernels with (the default; ~15 % faster on the headline scene).  Traversal, ray generation and the
 *                             film are IEEE either way; the near-specular closures (Mirror .. Mix), Layered and thin Disney too
 *   "device_bvh" (0/1)        build the hierarchy on the GPU at the next lrk_upload_scene instead of taking the caller's
 *   "pin_host_buffers" (0/1)  the caller promises that the host arrays it passes to lrk_upload_scene / lrk_download_film*
 *                             stay allocated until lrk_destroy (or until the option is cleared); the library page-locks each
 *                             of them once (cudaHostRegister), so that every later transfer of the same buffer is a
 *                             full-speed DMA: the per-frame path of an animation, and of bench.py's end-to-end leg
 *   "gbuffer" (0/1)           G-buffer mode, for lrk_denoise and external denoisers (see lrk_download_gbuffer).  The value the
 *                             option has at a film clear (lrk_film_clear, lrk_upload_scene, lrk_balance_shards, the start of
 *                             lrk_render_adaptive) decides whether the renders add to the G-buffer until the next clear, so that
 *                             every sample of a G-buffer film has its G-buffer entry.  The film itself is bit-identical either
 *                             way.  Surface integrator only: lrk_render / lrk_render_adaptive return LRK_ERR_UNSUPPORTED for
 *                             the volume integrator with the option on
 *   "light_tree" (0/1)        light selection of next-event estimation from a light tree (bounds, power and normal cone per node)
 *                             over every instance that carries a light, instead of the reference's uniform sampler over the light
 *                             nodes.  Read at lrk_upload_scene; the tree is built there from the scene description.  Another value
 *                             -> LRK_ERR_INVALID_ARGUMENT.  Surface integrator only: lrk_upload_scene returns LRK_ERR_UNSUPPORTED
 *                             for the volume integrator with the option on.  A scene with one emissive instance renders bit for bit
 *                             as without it.  LRK_ABI_VERSION stays 8: no layout or signature changed
 *   "light_solid_angle" (0/1) point sampling of next-event estimation: the point of the chosen emissive triangle is sampled
 *                             uniformly in the solid angle the triangle subtends at the shading point (Arvo's spherical-triangle
 *                             sampling) where that solid angle is in [3e-4, 6.22] sr, and uniformly by area, the reference's
 *                             sampler, elsewhere.  Less noise where a light is large or close.  Read at lrk_upload_scene; another
 *                             value -> LRK_ERR_INVALID_ARGUMENT.  Combines with "light_tree".  Surface integrator only:
 *                             lrk_upload_scene returns LRK_ERR_UNSUPPORTED for the volume integrator with the option on.
 *                             LRK_ABI_VERSION stays 8: no layout or signature changed
 *   "light_tree_triangles" (0/1) the bottom level of "light_tree": the tree also picks the triangle of the chosen emitter, from a
 *                             tree over the triangles of its mesh in object space (power = area, the triangle's normal as its
 *                             cone), instead of by area.  Less noise from curved one-sided lights, whose far side emits nothing
 *                             towards the point.  Read at lrk_upload_scene, which builds one such tree per emissive mesh and side
 *                             (about 14 us per triangle on the host); another value -> LRK_ERR_INVALID_ARGUMENT; on without
 *                             "light_tree" -> LRK_ERR_INVALID_ARGUMENT at lrk_upload_scene.  Combines with "light_solid_angle".
 *                             Surface integrator only, as "light_tree".  LRK_ABI_VERSION stays 8: no layout or signature changed
 *   "light_candidates" (0..32) resampled next-event estimation: for M = 2 .. 32, each surface vertex draws M candidates from the
 *                             light sampling the three options above configure, weights each by the luminance of its unshadowed
 *                             contribution (closure value x cosine x emission x MIS weight) over its pdf, and traces the shadow
 *                             ray of one, chosen in proportion to its weight (resampled importance sampling without reuse across
 *                             pixels).  Unbiased for every M; less noise where the closure or the receiver's orientation matters,
 *                             at the cost of M light samples and M closure evaluations per vertex.  0 (the default) and 1: one
 *                             light sample, as without the option.  Read at lrk_upload_scene; another value ->
 *                             LRK_ERR_INVALID_ARGUMENT.  Surface integrator only: lrk_upload_scene returns LRK_ERR_UNSUPPORTED for
 *                             the volume integrator with M >= 2.  LRK_ABI_VERSION stays 8: no layout or signature changed */
int lrk_set_option(lrk_ctx *ctx, const char *name, int64_t value);

int lrk_film_clear(lrk_ctx *ctx);

/* Render sample indices [spp_begin, spp_end) of every pixel of this ctx's shard and add
 * them to the film.  Asynchronous work is synchronised before returning. */
int lrk_render(lrk_ctx *ctx, uint32_t spp_begin, uint32_t spp_end);

/* Adaptive sampling (an extension: the reference has none; DESIGN.md §4 (Adaptive sampling)).  lrk_render_adaptive clears the film and renders
 * every pixel of this ctx's shard with a sample count of its own, n_p: sample indices [0, n_p), exactly the samples lrk_render(ctx,
 * 0, n_p) would add to that pixel, so the pixel's raw film entry is bit-identical to it.
 *   Rounds: every pixel gets [0, min_spp); after each round the pixels still active get [c, min(2c, max_spp)), c = their count.
 *           The render ends when no pixel is active or c == max_spp; a pixel that stops never restarts.  Counts are therefore
 *           min_spp * 2^k or max_spp.  Passes are sized like lrk_render's, for the active pixels.
 *   Error:  per pixel, from the film weight n (the samples the film kept, see the NaN / Inf filter) and the moments S1 = sum Y,
 *           S2 = sum Y^2 of those samples, Y = 0.2126 r + 0.7152 g + 0.0722 b of the clamped contribution times film.scale:
 *           m = S1 / n, v = max(S2 / n - m^2, 0) / (n - 1), e = sqrt(v) / max(m, 0.01) in IEEE fp32 (e = v = +inf when n < 2).
 *   Rule:   the unit is the 8x4 pixel block of the shard's pixel order (smaller at tile edges; blocks never cross tiles): a block
 *           stops when the maximum e over its pixels is strictly below `threshold`.  threshold = 0 never stops a block before
 *           max_spp, even one without any noise.  Decisions depend on the block's own pixels only, so a sharded, reduced render
 *           equals a single-GPU one bit for bit.
 * LRK_ERR_INVALID_ARGUMENT: min_spp < 2, max_spp < min_spp, a negative or non-finite threshold.  lrk_stats::samples counts the
 * samples rendered.  The moments buffer (8 B per pixel) and the count buffer are allocated by the first call. */
typedef struct lrk_adaptive {
    uint32_t min_spp, max_spp;
    float threshold;
    uint32_t reserved;
} lrk_adaptive;
int lrk_render_adaptive(lrk_ctx *ctx, const lrk_adaptive *p);
/* The sample count n_p of every pixel of the last adaptive render: W*H uint32, 0 outside this ctx's shard.
 * LRK_ERR_INVALID_ARGUMENT when no adaptive render ran since the last lrk_film_clear / lrk_upload_scene / lrk_render. */
int lrk_download_sample_counts(lrk_ctx *ctx, uint32_t *counts);
/* v above (the variance of the pixel's mean luminance: a noise map) for every pixel of the last adaptive render: W*H float,
 * 0 outside this ctx's shard.  Same error as lrk_download_sample_counts. */
int lrk_download_film_variance(lrk_ctx *ctx, float *v);

/* G-buffer and denoiser (an extension: the reference has neither; DESIGN.md §4 (G-buffer and denoiser)).
 * A G-buffer film holds per pixel, over its S samples in sample order: the sums of the first hit's albedo, of its shading normal
 * (vertex normal face-forwarded to the geometric one, before any normal map, turned against the camera ray) and of its
 * distance from the camera, and the number H of samples that hit a surface.  A miss adds zeros.  The albedo is the colour the
 * hit's closure scales: Matte Kd, Disney colour, Mirror colour, Glass Kt, saturate(Plastic p[0..2]), Metal Kd tint, a Mix's two
 * children weighted as the closure weights them, a Layered surface's bottom interface, 0 for a shape without a surface;
 * image-textured slots are evaluated at the hit.  It also holds the luminance moments of include/lrk.h's adaptive mode.
 * lrk_download_gbuffer: per pixel, albedo_cov = (sum albedo / S, H / S) and normal_depth = (normalize(sum n) or 0, sum t / H
 * or 0) as W*H float4 each, and variance = v of the adaptive mode (+inf below two samples) as W*H float; all 0 for pixels without
 * samples.  LRK_ERR_INVALID_ARGUMENT without a G-buffer film. */
int lrk_download_gbuffer(lrk_ctx *ctx, float *albedo_cov, float *normal_depth, float *variance);
/* The denoised film as W*H float4 in lrk_download_film's layout, alpha 1: an edge-avoiding à-trous filter over the
 * albedo-demodulated colour, guided by the G-buffer and the variance (five steps; denoise.h).  The film is not modified.
 * LRK_ERR_INVALID_ARGUMENT without a G-buffer film, LRK_ERR_UNSUPPORTED on a sharded context (world > 1): the other ranks hold the
 * neighbouring pixels and the G-buffer is not reduced. */
int lrk_denoise(lrk_ctx *ctx, float *rgba);

/* rgba = (sum_rgb / max(sum_w, 1)) * scale, a = 1 : W*H float4 (src/films/color.cpp:87-93) */
int lrk_download_film(lrk_ctx *ctx, float *rgba);
/* raw (sum r, sum g, sum b, sum w) : W*H float4 */
int lrk_download_film_raw(lrk_ctx *ctx, float *rgba);
/* device pointer of the raw film buffer (for the NCCL reduce of config C5) and its size */
int lrk_film_device_ptr(lrk_ctx *ctx, void **ptr, uint64_t *bytes);
/* overwrite the raw film with the (reduced) content of a device buffer of the same size */
int lrk_film_normalize_to_host(lrk_ctx *ctx, const void *device_raw, float *rgba);

/* Stand-alone ray queries against the uploaded scene (parity tests of rows a5/a7):
 * n rays in host memory -> n hits (any_hit == 0) or n occlusion flags in hits[i].inst
 * (0 = free, 1 = occluded; any_hit != 0). */
int lrk_trace(lrk_ctx *ctx, const lrk_ray *rays, uint64_t n, int any_hit, lrk_hit *hits);

/* Device-resident variant used by bench.py for the roofline measurement: traces the
 * same n device rays `repeat` times and returns the average kernel time in ms. */
int lrk_trace_device(lrk_ctx *ctx, const void *d_rays, uint64_t n, int any_hit, void *d_hits,
                     uint32_t repeat, float *avg_ms);

int lrk_get_stats(lrk_ctx *ctx, lrk_stats *stats);

/* the CUDA stream all work of this ctx is launched on (cudaStream_t as void*) */
void *lrk_stream(lrk_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* LRK_H */
