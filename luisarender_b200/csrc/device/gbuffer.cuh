// The G-buffer mode's kernel (option "gbuffer", DESIGN.md §4 (G-buffer and denoiser)): per pixel, the sums over its samples of
// the first hit's albedo, shading normal and distance, with the sample and hit counts, accumulated with the film.
//
// It runs once per pass, right after the depth-0 closest-hit trace: at that point pb.hit[id] and ray_o / ray_d[0][id] are the
// camera sample's hit and ray for every generation slot id = s * npix + k.  Depth 1's trace overwrites the hits and depth 1's
// shade overwrites ray_d[0].  One thread per pixel adds the pass's samples in sample order, like accumulate_kernel, so the sums do
// not depend on how the samples are split into passes, chunks or shards.
#pragma once
#include "shading.cuh"

namespace lrk {

// The albedo of a resolved surface record: the colour its closure scales (include/lrk.h's record layouts).
__device__ __forceinline__ V3 gbuffer_record_albedo(const lrk_surface &s) {
    switch (s.type) {
        case LRK_SURFACE_GLASS: return v3(s.p[3], s.p[4], s.p[5]);// Kt
        case LRK_SURFACE_PLASTIC: return v3(saturate(s.p[0]), saturate(s.p[1]), saturate(s.p[2]));
        case LRK_SURFACE_METAL: return v3(s.p[6], s.p[7], s.p[8]);// Kd tint
        default: return v3(s.p[0], s.p[1], s.p[2]);// Matte Kd, Disney colour, Mirror colour
    }
}

// The albedo of a hit: the surface record the shade kernels use (image-textured slots evaluated at the hit's uv), a Mix's children
// weighted as MixClosure weights their evaluations, a Layered surface's bottom interface.  0 for a shape without a surface.
__device__ __forceinline__ V3 gbuffer_albedo(const DeviceScene &sc, const Interaction &it) {
    if (!it.shape.has_surface()) return v3(0.f);
    const lrk_surface *node = sc.surfaces + it.shape.surface_tag;
    if (node->type == LRK_SURFACE_MIX)
        return lerp(gbuffer_record_albedo(sc.surfaces[node->mix_a]), gbuffer_record_albedo(sc.surfaces[node->mix_b]), 1.f - node->p[0]);
    if (node->type == LRK_SURFACE_LAYERED) return gbuffer_record_albedo(sc.surfaces[node->mix_b]);
    if (node->flags & LRK_SURFACE_HAS_TEXTURES) {
        lrk_surface s = *node;
        resolve_surface_textures(sc, s, it.u, it.v);
        return gbuffer_record_albedo(s);
    }
    return gbuffer_record_albedo(*node);
}

// albedo[pixel] += (albedo, 1) per sample; normal[pixel] += (n, t) and hits[pixel] += 1 per sample that hit a surface, where n is
// the shading normal before any normal map facing the camera ray and t the distance from the ray origin.  A miss adds zeros.
__global__ void __launch_bounds__(kBlock) gbuffer_kernel(DeviceScene sc, const float4 *__restrict__ ray_o, const float4 *__restrict__ ray_d,
                                                         const uint4 *__restrict__ hits, const uint32_t *__restrict__ pixel_list, uint32_t pixel_offset,
                                                         uint32_t npix, uint32_t spp, float4 *__restrict__ albedo, float4 *__restrict__ normal,
                                                         float *__restrict__ hit_count) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= npix) return;
    const uint32_t pixel = __ldg(pixel_list + pixel_offset + k);
    const size_t pid = static_cast<size_t>(pixel >> 16u) * sc.width + (pixel & 0xffffu);
    float4 a = albedo[pid], n = normal[pid];
    float h = hit_count[pid];
    for (uint32_t s = 0; s < spp; s++) {
        const size_t id = static_cast<size_t>(s) * npix + k;
        a.w += 1.f;
        const uint4 hit = hits[id];
        if (hit.x == ~0u) continue;
        const float bu = __uint_as_float(hit.z), bv = __uint_as_float(hit.w);
        const Interaction it = make_interaction(sc, hit.x, hit.y, v3(1.f - bu - bv, bu, bv));
        const float4 ro = ray_o[id], rd = ray_d[id];
        V3 ns = it.shading.n;
        if (dot(ns, v3(rd.x, rd.y, rd.z)) > 0.f) ns = -ns;
        const float t = length(it.pg - v3(ro.x, ro.y, ro.z));
        const V3 c = gbuffer_albedo(sc, it);
        a.x += c.x;
        a.y += c.y;
        a.z += c.z;
        n.x += ns.x;
        n.y += ns.y;
        n.z += ns.z;
        n.w += t;
        h += 1.f;
    }
    albedo[pid] = a;
    normal[pid] = n;
    hit_count[pid] = h;
}

}// namespace lrk
