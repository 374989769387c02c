// The volume path integrator with media bound to shapes (SURVEY.md §8 row a22 beyond config C4): MegakernelVolumePathTracingNaive::Li
// (src/integrators/mega_vpt_naive.cpp:170-485) with its medium tracker (src/util/medium_tracker.{h,cpp}), surface events (:68-94)
// and the transmittance walk through transmissive surfaces (:96-168).
//
// One thread per camera sample runs the whole path - the reference's own structure for this integrator (a megakernel).  The
// wavefront volume kernels (kernels.cuh) stay the fast path for config C4's shape: one homogeneous environment medium around
// opaque closures, where every transmittance ray ends at its first surface and reduces to an any-hit query.  Here a transmittance
// ray is a LOOP of closest-hit queries whose length depends on the surfaces it meets, interleaved with draws from the path's own
// PCG32 stream: there is no queue to compact between the steps, so each thread traces its rays itself (trace_single, traverse.cuh).
//
// Scope: homogeneous and vacuum media with eta = 1 (closures are built with eta_i = 1, as everywhere in this library), every
// closure kind of the surface integrator, the Independent sampler.  The reference's quirks are restated next to the oracle's
// volume_path_li (oracle/oracle.cpp), which this kernel follows statement by statement.
#pragma once
#include "pathcommon.cuh"
#include "traverse.cuh"

namespace lrk {

// MediumTracker: the reference keeps 32 (priority, medium) slots per path; 8 are stored here.  `size` keeps the reference's
// meaning (it also counts entries that were never stored, and refuses to enter at 32); an entry that would sort behind the
// eighth stored one raises the overflow flag (lrk_render fails) instead of being lost silently.
constexpr uint32_t kTrackerSlots = 8u;
constexpr uint32_t kTrackerCapacity = 32u;
struct DeviceMediumTracker {
    uint32_t priority[kTrackerSlots], tag[kTrackerSlots];
    uint32_t size;
    bool overflow;
    __device__ __forceinline__ void init() {
#pragma unroll
        for (uint32_t i = 0; i < kTrackerSlots; i++) {
            priority[i] = LRK_MEDIUM_VACUUM_PRIORITY;
            tag[i] = LRK_MEDIUM_INVALID_TAG;
        }
        size = 0u;
        overflow = false;
    }
    __device__ __forceinline__ bool vacuum() const { return priority[0] == LRK_MEDIUM_VACUUM_PRIORITY; }
    __device__ __forceinline__ bool true_hit(uint32_t p) const { return p <= priority[0]; }
    __device__ __forceinline__ uint32_t current_tag() const { return vacuum() ? LRK_MEDIUM_INVALID_TAG : tag[0]; }
    __device__ __forceinline__ void enter(uint32_t p, uint32_t t) {
        if (size == kTrackerCapacity) return;
        size += 1u;
        uint32_t x = p, v = t;
#pragma unroll
        for (uint32_t i = 0; i < kTrackerSlots; i++) {
            const uint32_t pi = priority[i], ti = tag[i];
            const bool swap = pi > x;
            priority[i] = swap ? x : pi;
            tag[i] = swap ? v : ti;
            x = swap ? pi : x;
            v = swap ? ti : v;
        }
        if (x != LRK_MEDIUM_VACUUM_PRIORITY) overflow = true;// a stored entry fell off the end
    }
    __device__ __forceinline__ void exit(uint32_t p, uint32_t t) {
        uint32_t removed = 0u;
#pragma unroll
        for (uint32_t i = 0; i < kTrackerSlots; i++) {
            const bool should_remove = priority[i] == p && tag[i] == t && removed == 0u;
            removed += should_remove ? 1u : 0u;
            const bool last = i + removed >= kTrackerSlots;
            priority[i] = last ? LRK_MEDIUM_VACUUM_PRIORITY : priority[(i + removed) & (kTrackerSlots - 1u)];
            tag[i] = last ? LRK_MEDIUM_INVALID_TAG : tag[(i + removed) & (kTrackerSlots - 1u)];
        }
        if (removed != 0u) {
            size -= 1u;
            if (size < kTrackerSlots) {
                priority[size] = LRK_MEDIUM_VACUUM_PRIORITY;
                tag[size] = LRK_MEDIUM_INVALID_TAG;
            }
        }
    }
};

// _event (mega_vpt_naive.cpp:68-94) in the closure's shading frame
__device__ __forceinline__ uint32_t surface_event_of(const Frame &shading, V3 wo, V3 wi) {
    const V3 wo_local = shading.world_to_local(wo), wi_local = shading.world_to_local(wi);
    return wo_local.z * wi_local.z > 0.f ? LRK_EVENT_REFLECT : wi_local.z > 0.f ? LRK_EVENT_EXIT : LRK_EVENT_ENTER;
}

// Runs f(closure, shading) with the closure of the hit's kind (the bucket key of the wavefront integrator's material sort).  Nothing
// for emitter-only hits and for Layered, which lrk_upload_scene refuses in the volume integrator.
template<typename F>
__device__ __forceinline__ void with_closure(const DeviceScene &sc, uint32_t kind, const lrk_surface *surf, const Interaction &it, const Frame &shading,
                                             V3 wo, F &&f) {
    with_hit_kind(kind, [&](auto k) {
        constexpr uint32_t K = decltype(k)::value;
        if constexpr (K != kHitLayered) with_hit_closure<K, true>(sc, surf, it, wo, [&] { return shading; }, f);
    });
}

template<typename Closure, typename = void>
struct has_event_member : std::false_type {};
template<typename Closure>
struct has_event_member<Closure, std::void_t<decltype(std::declval<const Closure &>().event)>> : std::true_type {};

// Surface::Closure::evaluate (src/base/surface.cpp:35-68) of the hit's closure
__device__ __noinline__ inline SurfEval general_surface_evaluate(const DeviceScene &sc, uint32_t kind, const lrk_surface *surf, const Interaction &it,
                                                          Frame shading, V3 wo, V3 wi) {
    SurfEval e;
    e.f = v3(0.f);
    e.pdf = 0.f;
    with_closure(sc, kind, surf, it, shading, wo, [&](auto &cl, const Frame &) {
        const V3 wo_local = shading.world_to_local(wo), wi_local = shading.world_to_local(wi);
        cl.prepare(wo_local);
        e = cl.evaluate_local(wo_local, wi_local);
        if (!validate_surface_sides(it.ng, shading.n, wo, wi)) {
            e.f = v3(0.f);
            e.pdf = 0.f;
        }
    });
    return e;
}

struct GeneralSurfaceSample {
    SurfEval light;// evaluate(wo, wi_light), zero when the light sample is invalid
    V3 wi, f;      // the closure's own sample
    float pdf;
    uint32_t event;
};
__device__ __noinline__ inline GeneralSurfaceSample general_surface_shade(const DeviceScene &sc, uint32_t kind, const lrk_surface *surf, const Interaction &it,
                                                                   Frame shading, V3 wo, LightSample ls, float u_lobe, float ub0, float ub1) {
    GeneralSurfaceSample out;
    out.light.f = out.f = v3(0.f);
    out.light.pdf = out.pdf = 0.f;
    out.wi = v3(0.f, 0.f, 1.f);
    out.event = LRK_EVENT_REFLECT;
    with_closure(sc, kind, surf, it, shading, wo, [&](auto &cl, const Frame &) {
        shade_surface_eval(cl, it, shading, wo, ls, u_lobe, ub0, ub1, out.light, out.wi, out.f, out.pdf);
        if constexpr (has_event_member<std::remove_reference_t<decltype(cl)>>::value) out.event = cl.event;
    });
    return out;
}

struct DeviceTransmittance {
    V3 f;
    float pdf;
};

__device__ __forceinline__ Interaction interaction_of_hit(const DeviceScene &sc, uint4 hit, V3 ray_d) {
    const float bu = __uint_as_float(hit.z), bv = __uint_as_float(hit.w);
    Interaction it = make_interaction(sc, hit.x, hit.y, v3(1.f - bu - bv, bu, bv));
    it.back_facing = dot(-ray_d, it.ng) < 0.0f;
    return it;
}

// _transmittance (mega_vpt_naive.cpp:96-168); the tracker is a copy (taken by value)
template<bool ALPHA>
__device__ __noinline__ inline DeviceTransmittance general_transmittance(const DeviceScene &sc, PCG32 &rng, DeviceMediumTracker tracker, float4 ray_o, float4 ray_d,
                                                                 uint32_t &rays, bool &tracker_overflow) {
    const float t_max = ray_d.w;
    const V3 dir = v3(ray_d.x, ray_d.y, ray_d.z);
    const V3 light_p = v3(ray_o.x, ray_o.y, ray_o.z) + dir * t_max;
    DeviceTransmittance T;
    T.f = v3(1.f);
    T.pdf = 0.f;
    while (T.f.x > 0.f || T.f.y > 0.f || T.f.z > 0.f) {
        const uint4 hit = trace_single<false, ALPHA>(sc, ray_o, ray_d);
        rays++;
        if (hit.x == ~0u) break;
        const Interaction it = interaction_of_hit(sc, hit, dir);
        const float t2surface = length(it.pg - v3(ray_o.x, ray_o.y, ray_o.z));
        const V3 wo = -dir, wi = dir;
        const uint32_t kind = __ldg(sc.inst_kind + hit.x);
        const lrk_surface *surf = sc.surfaces + it.shape.surface_tag;
        Frame shading = it.shading;
        if (it.shape.has_surface()) shading = closure_frame<true>(sc, surf, it, wo);
        const uint32_t surface_event = surface_event_of(shading, wo, wi);
        if (!tracker.vacuum()) {// HomogeneousMediumClosure::transmittance, homogeneous.cpp:119-133
            const lrk_medium m = sc.media[tracker.current_tag()];
            const V3 sigma_t = v3(m.sigma_a[0] + m.sigma_s[0], m.sigma_a[1] + m.sigma_s[1], m.sigma_a[2] + m.sigma_s[2]);
            V3 pc;
            pc.x = rng.uniform_float();
            pc.y = rng.uniform_float();
            pc.z = rng.uniform_float();
            const float ps = pc.x + pc.y + pc.z;
            pc = v3(pc.x / ps, pc.y / ps, pc.z / ps);
            const V3 Tr = exp3(-sigma_t * t2surface);
            T.f = T.f * Tr;
            const V3 pp = pc * Tr;
            T.pdf += pp.x + pp.y + pp.z;
        }
        if (it.shape.has_medium()) {
            const uint32_t tag = it.shape.medium_tag, priority = sc.media[tag].priority;
            if (surface_event == LRK_EVENT_EXIT) tracker.exit(priority, tag);
            else tracker.enter(priority, tag);
        }
        if (it.shape.has_surface()) {
            const SurfEval ev = general_surface_evaluate(sc, kind, surf, it, shading, wo, wi);
            T.f = T.f * ev.f;
            T.pdf += ev.pdf;
        }
        // Interaction::spawn_ray_to, src/base/interaction.cpp:25-30
        const V3 p_from = p_robust(it, light_p - it.pg);
        const V3 Lv = light_p - p_from;
        const float d = length(Lv);
        const V3 nd = Lv * (1.f / d);
        ray_o = make_float4(p_from.x, p_from.y, p_from.z, 0.f);
        ray_d = make_float4(nd.x, nd.y, nd.z, d * .9999f);
    }
    tracker_overflow = tracker_overflow || tracker.overflow;
    return T;
}

// One camera sample of the volume integrator: pixel (px, py), sample `sample_index`.  Returns Li; adds the rays it traced to the
// two counters and reports a medium-tracker overflow.
template<bool ALPHA>
__device__ __forceinline__ V3 volume_general_li(const DeviceScene &sc, uint32_t px, uint32_t py, uint32_t sample_index, uint32_t &closest_rays,
                                                uint32_t &shadow_rays, bool &tracker_overflow) {
    uint32_t state = xxhash32_uint4(px, py, sc.sampler_seed, sample_index);
    const float ux = lcg(state);
    const float uy = lcg(state);
    float4 ro, rd;
    float weight;
    camera_ray(sc.camera, px, py, ux, uy, ro, rd, weight);
    // PCG32 rng(U64(as<UInt2>(generate_2d()))): first float = high word (src/util/u64.h:48,58-59)
    const float s0 = lcg(state), s1 = lcg(state);
    PCG32 rng;
    rng.set_sequence((static_cast<unsigned long long>(__float_as_uint(s0)) << 32u) | __float_as_uint(s1));
    DeviceMediumTracker tracker;
    tracker.init();
    if (sc.env_medium_tag != LRK_MEDIUM_INVALID_TAG) tracker.enter(sc.media[sc.env_medium_tag].priority, sc.env_medium_tag);
    V3 beta = v3(weight), Li = v3(0.f);
    float pdf_bsdf = 1e16f, eta_scale = 1.f;
    for (uint32_t depth = 0; depth < sc.max_depth; depth++) {
        float eta = 1.f;
        float u_rr = 0.f;
        if (depth + 1u >= sc.rr_depth) u_rr = lcg(state);
        const uint4 hit = trace_single<false, ALPHA>(sc, ro, rd);
        closest_rays++;
        const bool valid = hit.x != ~0u;
        V3 o = v3(ro.x, ro.y, ro.z), d = v3(rd.x, rd.y, rd.z);
        Interaction it{};
        if (valid) it = interaction_of_hit(sc, hit, d);
        const bool has_medium = valid && it.shape.has_medium();
        const float t_max = valid ? length(it.pg - o) : kFltMax;
        uint32_t medium_event = ~0u;
        if (!tracker.vacuum()) {// :275-311
            const float u_sel = lcg(state), ul0 = lcg(state), ul1 = lcg(state);
            Interaction it_medium{};// Interaction{ray->origin()}: pg = ng = origin, default frame, zero offset factor
            it_medium.pg = o;
            it_medium.ng = o;
            it_medium.shading = Frame{v3(1.f, 0.f, 0.f), v3(0.f, 1.f, 0.f), v3(0.f, 0.f, 1.f)};
            it_medium.shape.intersection_offset = 0.f;
            const LightSample ls = sample_light_from(sc, it_medium, v3(0.f), u_sel, ul0, ul1);// p_shading of Interaction{origin} is the world origin
            const DeviceTransmittance T = general_transmittance<ALPHA>(sc, rng, tracker, ls.ray_o_tmin, ls.ray_d_tmax, shadow_rays, tracker_overflow);
            if (T.pdf > 0.f) {
                const float w = 1.f / (pdf_bsdf + T.pdf + ls.eval.pdf);
                Li = Li + w * beta * T.f * ls.eval.L;
            }
            const lrk_medium m = sc.media[tracker.current_tag()];
            eta = m.eta;
            V3 mf, no, nd;
            float mpdf;
            homogeneous_medium_sample(v3(m.sigma_a[0], m.sigma_a[1], m.sigma_a[2]), v3(m.sigma_s[0], m.sigma_s[1], m.sigma_s[2]), m.g, o, d, t_max, rng,
                                      medium_event, mf, mpdf, no, nd);
            ro = make_float4(no.x, no.y, no.z, 0.f);
            rd = make_float4(nd.x, nd.y, nd.z, kFltMax);
            o = no;
            d = nd;
            const float w = mpdf > 0.f ? 1.f / mpdf : 0.f;
            beta = beta * (mf * w);
            pdf_bsdf = mpdf;
        }
        if (medium_event == ~0u || medium_event == 3u) {
            if (!valid) {// :315-321
                if (sc.env_present) {
                    LightEval e = environment_evaluate(sc, d);
                    e.pdf *= sc.env_prob;
                    Li = Li + beta * e.L * balance_heuristic(pdf_bsdf, e.pdf);
                }
                break;
            }
            if (sc.light_count != 0u && it.shape.has_light()) {
                const LightEval e = evaluate_hit(sc, it, o);
                Li = Li + beta * e.L * balance_heuristic(pdf_bsdf, e.pdf);
            }
            if (!it.shape.has_surface()) break;
            const float u_sel = lcg(state), ul0 = lcg(state), ul1 = lcg(state);
            const float u_lobe = lcg(state), ub0 = lcg(state), ub1 = lcg(state);
            const LightSample ls = sample_light(sc, it, u_sel, ul0, ul1);
            const DeviceTransmittance T = general_transmittance<ALPHA>(sc, rng, tracker, ls.ray_o_tmin, ls.ray_d_tmax, shadow_rays, tracker_overflow);
            const uint32_t medium_tag = it.shape.medium_tag;// 0 for a shape without a medium (geometry.cpp:134)
            uint32_t medium_priority = LRK_MEDIUM_VACUUM_PRIORITY;
            float eta_next = 1.f;
            if (has_medium) {
                medium_priority = sc.media[medium_tag].priority;
                eta_next = sc.media[medium_tag].eta;
            }
            const V3 wo = -d;
            const uint32_t kind = __ldg(sc.inst_kind + hit.x);
            const lrk_surface *surf = sc.surfaces + it.shape.surface_tag;
            const Frame shading = closure_frame<true>(sc, surf, it, wo);
            const uint32_t surface_event_skip = surface_event_of(shading, wo, d);
            uint32_t surface_event;
            // true_hit gets the medium TAG where it expects a priority (:387, medium_tracker.cpp:19-21)
            if (!tracker.true_hit(medium_tag)) {
                surface_event = surface_event_skip;
                const V3 po = p_robust(it, d);
                ro = make_float4(po.x, po.y, po.z, 0.f);
                rd = make_float4(d.x, d.y, d.z, kFltMax);
                pdf_bsdf = 1e16f;
            } else {
                const GeneralSurfaceSample ss = general_surface_shade(sc, kind, surf, it, shading, wo, ls, u_lobe, ub0, ub1);
                if (ls.eval.pdf > 0.0f) {
                    const float w = 1.f / (ls.eval.pdf + ss.light.pdf + T.pdf);
                    Li = Li + w * beta * ss.light.f * ls.eval.L * T.f;
                }
                surface_event = ss.event;
                const float w = ss.pdf > 0.f ? 1.f / ss.pdf : 0.f;
                pdf_bsdf = ss.pdf;
                const V3 po = p_robust(it, ss.wi);
                ro = make_float4(po.x, po.y, po.z, 0.f);
                rd = make_float4(ss.wi.x, ss.wi.y, ss.wi.z, kFltMax);
                beta = beta * (w * ss.f);
                if (has_medium) {// :436-446
                    if (surface_event == LRK_EVENT_ENTER) eta_scale = sqr(eta_next / eta);
                    else if (surface_event == LRK_EVENT_EXIT) eta_scale = sqr(eta / eta_next);
                }
            }
            if (has_medium) {// :449-458
                if (surface_event == LRK_EVENT_ENTER) tracker.enter(medium_priority, medium_tag);
                else if (surface_event == LRK_EVENT_EXIT) tracker.exit(medium_priority, medium_tag);
            }
        }
        if (isnan(beta.x) || isnan(beta.y) || isnan(beta.z)) beta = v3(0.f);
        if (beta.x <= 0.f && beta.y <= 0.f && beta.z <= 0.f) break;
        const float q = fmaxf(max3(beta) * eta_scale, .05f);
        if (depth + 1u >= sc.rr_depth) {
            if (q < sc.rr_threshold && u_rr >= q) break;
            beta = beta * (q < sc.rr_threshold ? 1.0f / q : 1.f);
        }
    }
    tracker_overflow = tracker_overflow || tracker.overflow;
    return Li;
}

#ifdef __CUDACC__
constexpr int kGeneralBlock = 128;

template<bool ALPHA>
__global__ void __launch_bounds__(kGeneralBlock) volume_general_kernel(DeviceScene scp, PathBuffers pb, const uint32_t *__restrict__ pixel_list,
                                                                       uint32_t pixel_offset, uint32_t npix, uint32_t spp_begin, uint32_t n) {
    const DeviceScene &sc = *scp.self;// every callee takes the scene by reference: use the device-resident copy (scene.cuh)
    const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t closest_rays = 0u, shadow_rays = 0u;
    if (id < n) {
        const uint32_t pixel = __ldg(pixel_list + pixel_offset + id % npix);
        bool tracker_overflow = false;
        const V3 Li = volume_general_li<ALPHA>(sc, pixel & 0xffffu, pixel >> 16u, spp_begin + id / npix, closest_rays, shadow_rays, tracker_overflow);
        pb.li[id] = make_float4(Li.x, Li.y, Li.z, 0.f);
        if (tracker_overflow) atomicOr(sc.traversal_overflow, 2u);
    }
    // ray totals of the pass (the wavefront kernels derive them from their queue sizes)
    for (int off = 16; off > 0; off >>= 1) {
        closest_rays += __shfl_xor_sync(0xffffffffu, closest_rays, off);
        shadow_rays += __shfl_xor_sync(0xffffffffu, shadow_rays, off);
    }
    if ((threadIdx.x & 31u) == 0u) {
        atomicAdd(pb.stats, static_cast<unsigned long long>(closest_rays));
        atomicAdd(pb.stats + 1, static_cast<unsigned long long>(shadow_rays));
    }
    if (id == 0u) {
        for (uint32_t k = 0; k < kCountSlots * kMaxDepthSlots; k++) pb.counts[k] = 0u;// accumulate_kernel adds the queue sizes: none here
    }
}

#endif// __CUDACC__

}// namespace lrk
