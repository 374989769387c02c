// The wavefront kernels (sm_90a).  One pass renders S samples of a chunk of pixels:
//
//   generate_rays                                   (reference wave_path.cpp:254-272)
//   for depth in 0 .. max_depth-1:
//       trace_closest   ray queue  -> hits          (wave_path.cpp:275-302, geometry.cpp:218-223)
//       shade           hits -> emitter MIS, light sample + shadow-ray record, closure evaluate/sample,
//                       Russian roulette, compacted next ray queue
//                                                   (wave_path.cpp:326-459 = evaluate_lights + sample_lights
//                                                    + evaluate_surfaces fused; hit reconstruction once)
//       trace_shadow    shadow queue -> Li[path] += contribution if unoccluded   (geometry.cpp:262-266)
//   accumulate          Li -> film, per-sample clamp (wave_path.cpp:462-469, films/color.cpp:107-130)
//
// Queues are dense SoA arrays of float4/uint2 records, ping-ponged per bounce; queue sizes live in device
// memory and every kernel is a grid-stride loop over `*count`, so the host never synchronises inside a
// pass (the reference's v2 reads six counters back per step, wave_path_v2.cpp:396-405).  Compaction uses
// warp ballots + one atomic per block iteration.  Radiance is carried in Li[path_id] (path_id is the
// generation slot), so film accumulation needs no atomics and is run-to-run deterministic.
#pragma once
#include <type_traits>
#include <utility>
#include "samplers.cuh"
#include "shading.cuh"
#include "traverse.cuh"
#include "pathcommon.cuh"
#include "pathstate.cuh"

namespace lrk {

__global__ void __launch_bounds__(kBlock) generate_rays_kernel(DeviceScene sc, PathBuffers pb, const uint32_t *__restrict__ pixel_list,
                                                               uint32_t pixel_offset, uint32_t npix, uint32_t spp_begin, uint32_t n) {
    uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id == 0u) {
        pb.counts[0] = n;
        for (uint32_t d = 1u; d < kCountSlots * kMaxDepthSlots; d++) pb.counts[d] = 0u;// sizes + the traversal kernels' fetch cursors
    }
    if (id >= n) return;
    uint32_t k = id % npix;
    uint32_t s = id / npix;
    uint32_t pixel = __ldg(pixel_list + pixel_offset + k);
    uint32_t px = pixel & 0xffffu, py = pixel >> 16u;
    PathSampler smp;
    smp.start(sampler_ref(sc), px, py, spp_begin + s);
    const float2 uf = smp.pixel2d(sampler_ref(sc));
    float4 ro, rd;
    float weight;
    camera_ray(sc.camera, px, py, uf.x, uf.y, ro, rd, weight);
    pb.ray_o[0][id] = ro;
    pb.ray_d[0][id] = rd;
    pb.beta_pdf[0][id] = make_float4(weight, weight, weight, 1e16f);
    pb.id_rng[0][id] = make_uint2(id, smp.state);
    pb.li[id] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---- traversal kernels -------------------------------------------------------------------------------
template<bool COUNT, bool ALPHA = false>
__global__ void __launch_bounds__(kTraceBlock, LRK_TRACE_MIN_BLOCKS) trace_closest_kernel(DeviceScene sc, const float4 *__restrict__ ray_o,
                                                               const float4 *__restrict__ ray_d, uint4 *__restrict__ hits,
                                                               const uint32_t *__restrict__ count, uint32_t *cursor,
                                                               unsigned long long *stats) {
    const uint32_t n = *count;
    TraversalCounters tc{0u, 0u, 0u};
    trace_queue<false, COUNT, 1, ALPHA>(sc, ray_o, ray_d, n, cursor, tc, [&](bool finished, uint32_t i, uint4 h) {
        if (finished) store_result_record(hits + i, h);
    });
    if (COUNT) {
        atomicAdd(stats + 2, static_cast<unsigned long long>(tc.nodes));
        atomicAdd(stats + 3, static_cast<unsigned long long>(tc.tris));
        atomicAdd(stats + 4, static_cast<unsigned long long>(tc.xforms));
    }
}

// Sorted-by-material dispatch, step 1: bucket the hits of this bounce by closure kind (the reference sorts its
// SURFACE queue by surface tag, wave_path_v2.cpp:891-928,1255-1260, with a one-thread prefix sum; here a near-stable
// block-aggregated partition).  Escaped rays are dropped, so the shade kernels only ever see real work; every bucket
// keeps the ray-queue order inside a block chunk, which keeps the shade kernels' gathers coalesced.  The kinds: hit_kinds.h.
__global__ void __launch_bounds__(kBlock) classify_hits_kernel(DeviceScene sc, PathBuffers pb, uint32_t depth) {
    const uint32_t n = *path_count(pb.counts, depth);
    for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        uint32_t kind = ~0u;
        if (i < n) {
            const uint32_t inst = pb.hit[i].x;
            if (inst != ~0u) kind = __ldg(sc.inst_kind + inst);
            if (pb.tile_cost != nullptr) {// lrk_balance_shards' probe: one unit per traced ray, two more per hit that gets shaded
                const uint32_t id = pb.id_rng[depth & 1u][i].x;
                const uint32_t pixel = __ldg(pb.pass_pixel_list + pb.pass_pixel_offset + id % pb.pass_npix);
                const uint32_t tile = ((pixel >> 16u) / pb.tile_cost_size) * pb.tile_cost_tiles_x + (pixel & 0xffffu) / pb.tile_cost_size;
                atomicAdd(pb.tile_cost + tile, inst != ~0u ? 3u : 1u);
            }
        }
        block_append<kBlock, kHitKinds>(kind != ~0u ? 1u << kind : 0u, [&](uint32_t k) { return bucket_count(pb.counts, k, depth); },
                                        [&](uint32_t k, uint32_t slot) { pb.hit_index[k][slot] = i; });
    }
}

template<bool COUNT, bool ALPHA = false>
__global__ void __launch_bounds__(kTraceBlock, LRK_SHADOW_MIN_BLOCKS) trace_shadow_kernel(DeviceScene sc, PathBuffers pb, const uint32_t *__restrict__ count,
                                                              uint32_t *cursor) {
    const uint32_t n = *count;
    TraversalCounters tc{0u, 0u, 0u};
    trace_queue<true, COUNT, 1, ALPHA>(sc, pb.sray_o, pb.sray_d, n, cursor, tc, [&](bool finished, uint32_t i, uint4 h) {
        if (finished && h.x == ~0u) {// unoccluded: add the pending next-event contribution to the path's radiance
            float4 c = pb.scontrib[i];
            uint32_t path = __float_as_uint(c.w);
            float4 li = pb.li[path];
            li.x += c.x;
            li.y += c.y;
            li.z += c.z;
            pb.li[path] = li;
        }
    });
    if (COUNT) {
        atomicAdd(pb.stats + 5, static_cast<unsigned long long>(tc.nodes));
        atomicAdd(pb.stats + 6, static_cast<unsigned long long>(tc.tris));
        atomicAdd(pb.stats + 7, static_cast<unsigned long long>(tc.xforms));
    }
}

// stand-alone queries (lrk_trace) on interleaved lrk_ray records: any-hit result is written as inst = 1 (occluded) / 0 (free)
template<bool ANY_HIT, bool ALPHA = false>
__global__ void __launch_bounds__(kTraceBlock) trace_query_kernel(DeviceScene sc, const float4 *__restrict__ rays, uint4 *__restrict__ hits,
                                                             uint32_t n, uint32_t *cursor) {
    TraversalCounters tc{0u, 0u, 0u};
    trace_queue<ANY_HIT, false, 2, ALPHA>(sc, rays, rays + 1, n, cursor, tc, [&](bool finished, uint32_t i, uint4 h) {
        if (ANY_HIT) h = make_uint4(h.x != ~0u ? 1u : 0u, 0u, 0u, 0u);
        if (finished) hits[i] = h;
    });
}

// ---- escaped rays -----------------------------------------------------------------------------------------
// Only launched for scenes with an environment light: environment radiance with MIS for every ray of the depth that left the
// scene (mega_path.cpp:68-75, UniformLightSamplerInstance::evaluate_miss uniform.cpp:67-76).  Without an environment the
// escaped rays are simply never looked at again (classify_hits_kernel buckets hits only).
__global__ void __launch_bounds__(kBlock) shade_miss_kernel(DeviceScene sc, PathBuffers pb, uint32_t depth) {
    const uint32_t n = *path_count(pb.counts, depth);
    const int in = depth & 1u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (pb.hit[i].x != ~0u) continue;
        float4 rd = pb.ray_d[in][i];
        float4 bp = pb.beta_pdf[in][i];
        uint2 ir = pb.id_rng[in][i];
        LightEval e = environment_evaluate(*sc.self, v3(rd.x, rd.y, rd.z));
        e.pdf *= sc.env_prob;
        V3 add = v3(bp.x, bp.y, bp.z) * e.L * balance_heuristic(bp.w, e.pdf);
        float4 li = pb.li[ir.x];
        li.x += add.x;
        li.y += add.y;
        li.z += add.z;
        pb.li[ir.x] = li;
    }
}

// ---- volume path (config C4): mega_vpt_naive.cpp:170-485 for ONE homogeneous environment medium ------------------------
// Scope and the reference quirks that are reproduced on purpose are listed next to the oracle's volume_path_li
// (oracle/oracle.cpp).  For opaque closures every transmittance ray ends at the first surface with f = 0, so both
// shadow rays of a bounce reduce to any-hit queries whose only side effect on the path is three PCG32 draws when
// they hit something (homogeneous.cpp:119-125).
//
// Wavefront schedule per depth d:   T1 any-hit(s1 rays) -> occl1 | T0 closest(main rays) -> hits |
//   volume_shade(d): PCG catch-up (occl2 of d-1, occl1 of d), distance sampling, scatter/absorb or surface shading,
//                    next ray + next bounce's s1 ray + surface NEE shadow record | T2 any-hit(shadow records) -> Li, occl2
__global__ void __launch_bounds__(kBlock) generate_rays_volume_kernel(DeviceScene sc, PathBuffers pb, const uint32_t *__restrict__ pixel_list,
                                                                      uint32_t pixel_offset, uint32_t npix, uint32_t spp_begin, uint32_t n) {
    uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id == 0u) {
        pb.counts[0] = n;
        for (uint32_t d = 1u; d < kCountSlots * kMaxDepthSlots; d++) pb.counts[d] = 0u;
    }
    if (id >= n) return;
    uint32_t k = id % npix;
    uint32_t s = id / npix;
    uint32_t pixel = __ldg(pixel_list + pixel_offset + k);
    uint32_t px = pixel & 0xffffu, py = pixel >> 16u;
    uint32_t state = xxhash32_uint4(px, py, sc.sampler_seed, spp_begin + s);
    float ux = lcg(state);
    float uy = lcg(state);
    float4 ro, rd;
    float weight;
    camera_ray(sc.camera, px, py, ux, uy, ro, rd, weight);
    // PCG32 rng(U64(as<UInt2>(generate_2d()))): first float = high word (src/util/u64.h:48,58-59)
    float s0 = lcg(state), s1 = lcg(state);
    PCG32 rng;
    rng.set_sequence((static_cast<unsigned long long>(__float_as_uint(s0)) << 32u) | __float_as_uint(s1));
    float u_rr = 0.f;
    if (1u >= sc.rr_depth) u_rr = lcg(state);
    float u_sel = lcg(state), ul0 = lcg(state), ul1 = lcg(state);
    float4 so, sd;
    medium_light_shadow_ray(sc, v3(ro.x, ro.y, ro.z), u_sel, ul0, ul1, so, sd);
    pb.ray_o[0][id] = ro;
    pb.ray_d[0][id] = rd;
    pb.beta_pdf[0][id] = make_float4(weight, weight, weight, 1e16f);
    pb.id_rng[0][id] = make_uint2(id, state);
    pb.li[id] = make_float4(0.f, 0.f, 0.f, 0.f);
    pb.pcg[0][id] = make_ulonglong2(rng.state, rng.inc);
    pb.u_rr[0][id] = u_rr;
    pb.s1ray_o[id] = so;
    pb.s1ray_d[id] = sd;
    pb.occl2[0][id] = 0u;
}

// T1 / T2: any-hit queries that record occlusion.  T2 also applies the pending surface NEE contribution.
template<bool COUNT>
__global__ void __launch_bounds__(kTraceBlock) trace_medium_shadow_kernel(DeviceScene sc, PathBuffers pb, const uint32_t *__restrict__ count,
                                                                     uint32_t *cursor) {
    const uint32_t n = *count;
    TraversalCounters tc{0u, 0u, 0u};
    trace_queue<true, COUNT, 1>(sc, pb.s1ray_o, pb.s1ray_d, n, cursor, tc, [&](bool finished, uint32_t i, uint4 h) {
        if (finished) pb.occl1[i] = h.x != ~0u ? 1u : 0u;
    });
    if (COUNT) {
        atomicAdd(pb.stats + 5, static_cast<unsigned long long>(tc.nodes));
        atomicAdd(pb.stats + 6, static_cast<unsigned long long>(tc.tris));
        atomicAdd(pb.stats + 7, static_cast<unsigned long long>(tc.xforms));
    }
}

template<bool COUNT>
__global__ void __launch_bounds__(kTraceBlock) trace_volume_nee_kernel(DeviceScene sc, PathBuffers pb, const uint32_t *__restrict__ count,
                                                                  uint32_t *cursor, uint32_t *__restrict__ occl_out) {
    const uint32_t n = *count;
    TraversalCounters tc{0u, 0u, 0u};
    trace_queue<true, COUNT, 1>(sc, pb.sray_o, pb.sray_d, n, cursor, tc, [&](bool finished, uint32_t i, uint4 h) {
        if (!finished) return;
        const bool occluded = h.x != ~0u;
        const uint32_t target = pb.s2_target[i];
        if (target != ~0u) occl_out[target] = occluded ? 1u : 0u;
        if (!occluded) {
            float4 c = pb.scontrib[i];
            if (c.x != 0.f || c.y != 0.f || c.z != 0.f) {
                uint32_t path = __float_as_uint(c.w);
                float4 li = pb.li[path];
                li.x += c.x;
                li.y += c.y;
                li.z += c.z;
                pb.li[path] = li;
            }
        }
    });
    if (COUNT) {
        atomicAdd(pb.stats + 5, static_cast<unsigned long long>(tc.nodes));
        atomicAdd(pb.stats + 6, static_cast<unsigned long long>(tc.tris));
        atomicAdd(pb.stats + 7, static_cast<unsigned long long>(tc.xforms));
    }
}

// ---- film ---------------------------------------------------------------------------------------------------
// One thread per pixel of the chunk: adds the S samples of this pass in sample order (deterministic).
// Per-sample clamp / NaN filter: src/films/color.cpp:107-130 with effective_spp = 1.
// MOMENTS (the adaptive mode, adaptive.cuh): also adds Y and Y^2 of every sample the film keeps to moments[pixel], where Y is the
// display luminance of the clamped contribution times film.scale.
template<bool MOMENTS>
__global__ void __launch_bounds__(kBlock) accumulate_kernel(DeviceScene sc, const float4 *__restrict__ li, float4 *__restrict__ film,
                                                            const uint32_t *__restrict__ pixel_list, uint32_t pixel_offset, uint32_t npix,
                                                            uint32_t spp, const uint32_t *__restrict__ counts, unsigned long long *stats,
                                                            float2 *__restrict__ moments) {
    uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0u) {// ray totals of this pass = sum of the per-depth queue sizes
        unsigned long long closest = 0ull, shadow = 0ull;
        for (uint32_t d = 0; d < sc.max_depth; d++) {
            closest += counts[d];
            shadow += counts[kMaxDepthSlots + d];
        }
        stats[0] += closest;
        stats[1] += shadow;
    }
    if (k >= npix) return;
    uint32_t pixel = __ldg(pixel_list + pixel_offset + k);
    uint32_t px = pixel & 0xffffu, py = pixel >> 16u;
    size_t pid = static_cast<size_t>(py) * sc.width + px;
    float4 acc = film[pid];
    float2 mom = MOMENTS ? moments[pid] : make_float2(0.f, 0.f);
    const float threshold = sc.film_clamp * fmaxf(1.f, 1.f);
    for (uint32_t s = 0; s < spp; s++) {
        float4 v = li[static_cast<size_t>(s) * npix + k];
        V3 rgb = v3(v.x, v.y, v.z) * 1.0f;// shutter weight
        bool bad = isnan(rgb.x) || isnan(rgb.y) || isnan(rgb.z) || isinf(rgb.x) || isinf(rgb.y) || isinf(rgb.z);
        if (bad) continue;
        float strength = fmaxf(fmaxf(fmaxf(fabsf(rgb.x), fabsf(rgb.y)), fabsf(rgb.z)), 0.f);
        V3 c = rgb * (threshold / fmaxf(strength, threshold));
        if (c.x != 0.f || c.y != 0.f || c.z != 0.f) {
            acc.x += c.x;
            acc.y += c.y;
            acc.z += c.z;
        }
        acc.w += 1.f;
        if (MOMENTS) {
            const float y = 0.2126f * (c.x * sc.film_scale[0]) + 0.7152f * (c.y * sc.film_scale[1]) + 0.0722f * (c.z * sc.film_scale[2]);
            mom.x += y;
            mom.y += y * y;
        }
    }
    film[pid] = acc;
    if (MOMENTS) moments[pid] = mom;
}

// convert_image: src/films/color.cpp:87-93
__global__ void __launch_bounds__(kBlock) convert_film_kernel(DeviceScene sc, const float4 *__restrict__ raw, float4 *__restrict__ out, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 c = raw[i];
    float nrm = fmaxf(c.w, 1.f);
    float inv = 1.f / nrm;
    out[i] = make_float4((inv * sc.film_scale[0]) * c.x, (inv * sc.film_scale[1]) * c.y, (inv * sc.film_scale[2]) * c.z, 1.f);
}

}// namespace lrk

#include "volume_general.cuh"
