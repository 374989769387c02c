// volume_host.cpp — the DEVICE code of the general volume integrator (luisarender_b200/csrc/device/volume_general.cuh: medium
// tracker, surface events, transmittance walks, the per-sample loop, with the closures, light sampling and traversal it calls)
// compiled for the host, so that it can be compared with the oracle sample by sample without a GPU
// (tests/test_device_volume_on_host.py).  TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>

template<typename T>
static inline T __ldg(const T *p) { return *p; }
static inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
#ifndef __noinline__
#define __noinline__
#endif
#include <algorithm>
using std::isinf;
using std::isnan;
using std::max;
using std::min;
static inline void sincosf_host(float x, float *s, float *c) { *s = std::sin(x); *c = std::cos(x); }
#define sincosf sincosf_host

#include "../../luisarender_b200/csrc/device/volume_general.cuh"

using namespace lrk;

// film: width * height * 4 floats, the raw (sum rgb, weight) film of samples [spp_begin, spp_end) - accumulated like
// accumulate_kernel does (src/films/color.cpp:107-130); rays: {closest, shadow}
extern "C" int volume_general_host(const lrk_scene_desc *s, uint32_t spp_begin, uint32_t spp_end, float *film, uint64_t *rays) {
    std::vector<float4> xform(static_cast<size_t>(s->instance_count) * 4u), o2w(static_cast<size_t>(s->instance_count) * 3u);
    std::vector<uint4> handles(s->instance_count);
    std::vector<uint32_t> kinds(s->instance_count);
    bool alpha = false;
    for (uint32_t i = 0; i < s->instance_count; i++) {// as lrk_upload_scene lays the instance records out
        const auto &inst = s->instances[i];
        std::memcpy(&xform[i * 4u], inst.world_to_object, 48);
        xform[i * 4u + 3u] = make_float4(__uint_as_float(s->meshes[inst.mesh].bvh_root), 0.f, 0.f, 0.f);
        std::memcpy(&o2w[i * 3u], inst.object_to_world, 48);
        std::memcpy(&handles[i], inst.handle, 16);
        const uint32_t flags = inst.handle[0] & 1023u, surface_tag = (inst.handle[1] >> 12u) & 4095u;
        kinds[i] = (flags & LRK_SHAPE_HAS_SURFACE) ? hit_kind_of(s->surfaces[surface_tag]) : kHitEmitter;
        if ((flags & LRK_SHAPE_MAYBE_NON_OPAQUE) && (flags & LRK_SHAPE_HAS_SURFACE)) alpha = true;
    }
    uint32_t overflow = 0u;
    DeviceScene sc{};
    sc.self = &sc;
    sc.vertices = s->vertices;
    sc.triangles = s->triangles;
    sc.alias = s->alias;
    sc.pdf = s->pdf;
    sc.meshes = s->meshes;
    sc.inst_handles = handles.data();
    sc.inst_kind = kinds.data();
    sc.inst_o2w = o2w.data();
    sc.inst_xform = xform.data();
    sc.bvh_nodes = reinterpret_cast<const float4 *>(s->bvh_nodes);
    sc.traversal_overflow = &overflow;
    sc.tri_verts = reinterpret_cast<const float4 *>(s->tri_verts);
    sc.surfaces = s->surfaces;
    sc.textures = s->textures;
    sc.texels = reinterpret_cast<const float4 *>(s->texels);
    sc.env_present = 0u;
    sc.env_prob = 0.f;
    sc.lights = s->lights;
    sc.light_handles = s->light_handles;
    sc.camera = &s->camera;
    sc.tlas_root = s->tlas_root;
    sc.light_count = s->light_count;
    sc.instance_count = s->instance_count;
    sc.surface_count = s->surface_count;
    sc.max_depth = s->integrator.max_depth;
    sc.rr_depth = s->integrator.rr_depth;
    sc.rr_threshold = s->integrator.rr_threshold;
    sc.sampler_seed = s->integrator.sampler_seed;
    sc.sampler_type = LRK_SAMPLER_INDEPENDENT;
    sc.film_clamp = s->film.clamp;
    sc.width = s->camera.resolution[0];
    sc.height = s->camera.resolution[1];
    sc.media = s->media;
    sc.medium_count = s->medium_count;
    sc.env_medium_tag = s->environment_medium_tag;
    // the environment light, as lrk_upload_scene hands it to the kernels (lrk.cu)
    sc.env_alias = s->environment.alias;
    sc.env_pdf = s->environment.pdf;
    sc.env_present = s->environment.present ? 1u : 0u;
    sc.env_emission_tex = s->environment.present ? s->environment.emission_tex : 0u;
    sc.env_map_width = s->environment.map_width;
    sc.env_map_height = s->environment.map_height;
    sc.env_scale = s->environment.scale;
    sc.env_prob = s->environment.present ? s->environment.env_prob : 0.f;
    for (int k = 0; k < 3; k++) sc.env_emission[k] = s->environment.emission[k];
    for (int k = 0; k < 9; k++) sc.env_to_world[k] = s->environment.to_world[k];
    if (s->sampler.type != LRK_SAMPLER_INDEPENDENT) return -1;
    uint64_t closest = 0u, shadow = 0u;
    bool tracker_overflow = false;
    const float threshold = sc.film_clamp * std::fmax(1.f, 1.f);
    for (uint32_t py = 0; py < sc.height; py++) {
        for (uint32_t px = 0; px < sc.width; px++) {
            float *acc = film + (static_cast<size_t>(py) * sc.width + px) * 4u;
            for (uint32_t k = spp_begin; k < spp_end; k++) {
                uint32_t c = 0u, sh = 0u;
                const V3 rgb = alpha ? volume_general_li<true>(sc, px, py, k, c, sh, tracker_overflow)
                                     : volume_general_li<false>(sc, px, py, k, c, sh, tracker_overflow);
                closest += c;
                shadow += sh;
                const bool bad = isnan(rgb.x) || isnan(rgb.y) || isnan(rgb.z) || isinf(rgb.x) || isinf(rgb.y) || isinf(rgb.z);
                if (bad) continue;
                const float strength = std::fmax(std::fmax(std::fmax(std::fabs(rgb.x), std::fabs(rgb.y)), std::fabs(rgb.z)), 0.f);
                const V3 cl = rgb * (threshold / std::fmax(strength, threshold));
                if (cl.x != 0.f || cl.y != 0.f || cl.z != 0.f) {
                    acc[0] += cl.x;
                    acc[1] += cl.y;
                    acc[2] += cl.z;
                }
                acc[3] += 1.f;
            }
        }
    }
    if (rays) {
        rays[0] = closest;
        rays[1] = shadow;
    }
    return (overflow != 0u ? 1 : 0) | (tracker_overflow ? 2 : 0);
}
