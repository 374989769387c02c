// The closure kernels of the wavefront integrators: shade_kernel<KIND> (surface integrator: emitter MIS, light sample + shadow
// record, closure evaluate / sample, Russian roulette, compaction) and the volume integrator's medium / surface steps.
// Included by shade.cu ONLY.  shade.cu is compiled twice, with different arithmetic (see its header); LRK_SHADE_VARIANT names the
// namespace the kernels of each compilation live in, so that the two sets of __global__ functions stay distinct symbols.
#pragma once
#ifndef LRK_SHADE_VARIANT
#error "shade_kernels.cuh is compiled through shade.cu with -DLRK_SHADE_VARIANT=fast|strict"
#endif
#include "pathcommon.cuh"
#include "pathstate.cuh"
#include "samplers.cuh"

namespace lrk {
namespace LRK_SHADE_VARIANT {

// The numbers one bounce consumes, drawn from a table-driven sampler (row f2) for the path with generation slot `id`: pixel and
// sample index follow from the slot (PathBuffers::pass_*), `word` is the dimension counter the path carries.  Out of line, so
// that the Independent sampler's path through shade_kernel is the code it was before the table-driven samplers existed.
struct BounceDraws {
    float u_sel, ul0, ul1, u_lobe, ub0, ub1, u_rr;
    uint32_t state;
};
__device__ __noinline__ inline BounceDraws draw_bounce_from_tables(SamplerRef sc, const uint32_t *pixel_list, uint32_t pixel_offset, uint32_t npix,
                                                            uint32_t spp_begin, uint32_t id, uint32_t word, bool draw_rr) {
    const uint32_t pixel = __ldg(pixel_list + pixel_offset + id % npix);
    PathSampler smp;
    smp.resume(sc, word, pixel & 0xffffu, pixel >> 16u, spp_begin + id / npix);
    BounceDraws d;
    d.u_sel = smp.next1d(sc);
    const float2 ul = smp.next2d(sc);
    d.ul0 = ul.x;
    d.ul1 = ul.y;
    d.u_lobe = smp.next1d(sc);
    const float2 ub = smp.next2d(sc);
    d.ub0 = ub.x;
    d.ub1 = ub.y;
    d.u_rr = draw_rr ? smp.next1d(sc) : 0.f;
    d.state = smp.state;
    return d;
}

// The light sampling of the resampling shade kernels, chosen at run time from light_tree_of(sc): one instantiation per TEXTURED
// serves every (selection, point) pair, out of line so that the kernels hold one call site each.  `sc`: *DeviceScene::self.
template<bool TEXTURED>
__device__ __noinline__ LightSample sample_light_configured(const DeviceScene &sc, const Interaction &it, float u_sel, float u0, float u1) {
    if (sc.light_count == 0u && sc.env_prob == 0.f) {
        LightSample ls;
        ls.eval.L = v3(0.f);
        ls.eval.pdf = 0.f;
        ls.ray_o_tmin = make_float4(0.f, 0.f, 0.f, 0.f);
        ls.ray_d_tmax = make_float4(0.f, 0.f, 1.f, 0.f);
        return ls;
    }
    const DeviceLightTree &lt = light_tree_of(sc);
    if (lt.select == kLightSelectTree)
        return lt.point == kLightPointSolidAngle ? sample_light<TEXTURED, kLightSelectTree, kLightPointSolidAngle>(sc, it, u_sel, u0, u1)
                                                 : sample_light<TEXTURED, kLightSelectTree, kLightPointArea>(sc, it, u_sel, u0, u1);
    return lt.point == kLightPointSolidAngle ? sample_light<TEXTURED, kLightSelectUniform, kLightPointSolidAngle>(sc, it, u_sel, u0, u1)
                                             : sample_light<TEXTURED, kLightSelectUniform, kLightPointArea>(sc, it, u_sel, u0, u1);
}
template<bool TEXTURED>
__device__ __noinline__ LightEval evaluate_hit_configured(const DeviceScene &sc, const Interaction &it, V3 p_from, uint32_t inst) {
    const DeviceLightTree &lt = light_tree_of(sc);
    if (lt.select == kLightSelectTree)
        return lt.point == kLightPointSolidAngle ? evaluate_hit<TEXTURED, kLightSelectTree, kLightPointSolidAngle>(sc, it, p_from, inst)
                                                 : evaluate_hit<TEXTURED, kLightSelectTree, kLightPointArea>(sc, it, p_from, inst);
    return lt.point == kLightPointSolidAngle ? evaluate_hit<TEXTURED, kLightSelectUniform, kLightPointSolidAngle>(sc, it, p_from, inst)
                                             : evaluate_hit<TEXTURED, kLightSelectUniform, kLightPointArea>(sc, it, p_from, inst);
}

// Sorted-by-material dispatch, step 2: one shade kernel per closure kind, each over its own hit bucket.  SEL: the light selection
// of next-event estimation (kLightSelectTree with the option "light_tree"); PT: its point sampling (kLightPointSolidAngle with the
// option "light_solid_angle").  RESAMPLE: resampled next-event estimation (option "light_candidates" >= 2, every kind but
// emitter-only): the light sampling and the candidate count come from light_tree_of(sc) at run time instead of SEL and PT.
template<uint32_t KIND, bool TEXTURED = false, uint32_t SEL = kLightSelectUniform, uint32_t PT = kLightPointArea, bool RESAMPLE = false>
__global__ void __launch_bounds__(kShadeBlock, LRK_SHADE_MIN_BLOCKS) shade_kernel(DeviceScene sc, PathBuffers pb, uint32_t depth) {
    static_assert(!RESAMPLE || (KIND != kHitEmitter && SEL == kLightSelectUniform && PT == kLightPointArea), "one resampling kernel per kind");
    // the compaction is written out here rather than through block_append, which raises registers or spills of most instantiations
    __shared__ uint32_t s_warp_next[kShadeBlock / 32], s_warp_shadow[kShadeBlock / 32];
    __shared__ uint32_t s_base_next, s_base_shadow;
    const uint32_t n = *bucket_count(pb.counts, KIND, depth);// size of this kind's hit bucket
    const int in = depth & 1u, out = in ^ 1;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5u;
    for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
        const uint32_t j = base + threadIdx.x;
        bool push_next = false, push_shadow = false;
        float4 nro, nrd, nbeta, sro, srd, scon;
        uint2 nid;
        if (j < n) {
            const uint32_t i = pb.hit_index[KIND][j];
            const uint4 hit = pb.hit[i];
            {
                float4 ro = pb.ray_o[in][i], rd = pb.ray_d[in][i];
                float4 bp = pb.beta_pdf[in][i];
                uint2 ir = pb.id_rng[in][i];
                V3 beta = v3(bp.x, bp.y, bp.z);
                float pdf_bsdf = bp.w;
                uint32_t state = ir.y;
                V3 wo = -v3(rd.x, rd.y, rd.z);
                float bu = __uint_as_float(hit.z), bv = __uint_as_float(hit.w);
                Interaction it = make_interaction(sc, hit.x, hit.y, v3(1.f - bu - bv, bu, bv));
                it.back_facing = dot(wo, it.ng) < 0.0f;
                // emitter hit with MIS: mega_path.cpp:80-87, uniform.cpp:50-65
                if (sc.light_count != 0u && it.shape.has_light()) {
                    LightEval e;
                    if constexpr (RESAMPLE) e = evaluate_hit_configured<TEXTURED>(*sc.self, it, v3(ro.x, ro.y, ro.z), hit.x);
                    else e = evaluate_hit<TEXTURED, SEL, PT>(sc, it, v3(ro.x, ro.y, ro.z), hit.x);
                    V3 add = beta * e.L * balance_heuristic(pdf_bsdf, e.pdf);
                    float4 li = pb.li[ir.x];
                    li.x += add.x;
                    li.y += add.y;
                    li.z += add.z;
                    pb.li[ir.x] = li;
                }
                if (KIND != kHitEmitter) {// an emitter-only hit (no surface): the path ends here (mega_path.cpp:89)
                    // draw order is normative: mega_path.cpp:91-98
                    float u_sel, ul0, ul1, u_lobe, ub0, ub1, u_rr = 0.f;
                    if (sc.sampler_type == LRK_SAMPLER_INDEPENDENT) {// the headline path: an LCG word in a register
                        u_sel = lcg(state);
                        ul0 = lcg(state);
                        ul1 = lcg(state);
                        u_lobe = lcg(state);
                        ub0 = lcg(state);
                        ub1 = lcg(state);
                        if (depth + 1u >= sc.rr_depth) u_rr = lcg(state);
                    } else {// table-driven samplers: all of the bounce's numbers from one out-of-line call
                        BounceDraws dr = draw_bounce_from_tables(sampler_ref(sc), pb.pass_pixel_list, pb.pass_pixel_offset, pb.pass_npix, pb.pass_spp_begin,
                                                                 ir.x, state, depth + 1u >= sc.rr_depth);
                        u_sel = dr.u_sel; ul0 = dr.ul0; ul1 = dr.ul1; u_lobe = dr.u_lobe; ub0 = dr.ub0; ub1 = dr.ub1; u_rr = dr.u_rr;
                        state = dr.state;
                    }
                    LightSample ls;// with RESAMPLE: the kept candidate's shadow ray only
                    ls.eval.L = v3(0.f);
                    ls.eval.pdf = 0.f;
                    ls.ray_o_tmin = make_float4(0.f, 0.f, 0.f, 0.f);
                    ls.ray_d_tmax = make_float4(0.f, 0.f, 1.f, 0.f);
                    if constexpr (!RESAMPLE)
                        if (sc.light_count != 0u || sc.env_prob != 0.f) ls = sample_light<TEXTURED, SEL, PT>(sc, it, u_sel, ul0, ul1);
                    const lrk_surface *surf = sc.surfaces + it.shape.surface_tag;
                    V3 contrib, wi, f;
                    float pdf;
                    const float eta_scale = with_hit_closure<KIND, TEXTURED>(sc, surf, it, wo, [&] { return closure_frame<TEXTURED>(sc, surf, it, wo); },
                                                                           [&](auto &cl, const Frame &fr) {
                        if constexpr (RESAMPLE) {
                            const auto draw_light = [&](float us, float u0, float u1) { return sample_light_configured<TEXTURED>(*sc.self, it, us, u0, u1); };
                            shade_surface_resampled(cl, it, fr, wo, draw_light, light_tree_of(sc).candidates, depth, u_sel, ul0, ul1, beta, u_lobe, ub0, ub1,
                                                    contrib, ls.ray_o_tmin, ls.ray_d_tmax, wi, f, pdf);
                        } else {
                            shade_surface<false>(cl, it, fr, wo, ls, beta, u_lobe, ub0, ub1, contrib, wi, f, pdf);
                        }
                    });
                    if (contrib.x != 0.f || contrib.y != 0.f || contrib.z != 0.f) {
                        // a zero (or NaN-free zero) contribution needs no shadow ray; NaNs must reach the film filter
                        push_shadow = true;
                        sro = ls.ray_o_tmin;
                        srd = ls.ray_d_tmax;
                        scon = make_float4(contrib.x, contrib.y, contrib.z, __uint_as_float(ir.x));
                    }
                    // continue the path: mega_path.cpp:128-151
                    V3 po = p_robust(it, wi);
                    float w = pdf > 0.f ? 1.f / pdf : 0.f;
                    beta = beta * (w * f);
                    if (isnan(beta.x) || isnan(beta.y) || isnan(beta.z)) beta = v3(0.f);
                    bool alive = !(beta.x <= 0.f && beta.y <= 0.f && beta.z <= 0.f);
                    if (alive) {
                        float q = fmaxf(max3(beta) * eta_scale, .05f);
                        if (depth + 1u >= sc.rr_depth) {
                            if (q < sc.rr_threshold && u_rr >= q) alive = false;
                            beta = beta * (q < sc.rr_threshold ? 1.0f / q : 1.f);
                        }
                    }
                    if (alive && depth + 1u < sc.max_depth) {
                        push_next = true;
                        nro = make_float4(po.x, po.y, po.z, 0.f);
                        nrd = make_float4(wi.x, wi.y, wi.z, kFltMax);
                        nbeta = make_float4(beta.x, beta.y, beta.z, pdf);
                        nid = make_uint2(ir.x, state);
                    }
                }
            }
        }
        // block-aggregated compaction: ballots inside the warp, one atomic per queue per block iteration
        uint32_t m_next = __ballot_sync(0xffffffffu, push_next);
        uint32_t m_shadow = __ballot_sync(0xffffffffu, push_shadow);
        if (lane == 0u) {
            s_warp_next[warp] = __popc(m_next);
            s_warp_shadow[warp] = __popc(m_shadow);
        }
        __syncthreads();
        if (threadIdx.x == 0u) {
            uint32_t tn = 0u, ts = 0u;
            for (int w = 0; w < kShadeBlock / 32; w++) {
                uint32_t a = s_warp_next[w], b = s_warp_shadow[w];
                s_warp_next[w] = tn;
                s_warp_shadow[w] = ts;
                tn += a;
                ts += b;
            }
            s_base_next = tn ? atomicAdd(path_count(pb.counts, depth + 1u), tn) : 0u;
            s_base_shadow = ts ? atomicAdd(shadow_count(pb.counts, depth), ts) : 0u;
        }
        __syncthreads();
        const uint32_t lt = (1u << lane) - 1u;
        if (push_next) {
            uint32_t slot = s_base_next + s_warp_next[warp] + __popc(m_next & lt);
            pb.ray_o[out][slot] = nro;
            pb.ray_d[out][slot] = nrd;
            pb.beta_pdf[out][slot] = nbeta;
            pb.id_rng[out][slot] = nid;
        }
        if (push_shadow) {
            uint32_t slot = s_base_shadow + s_warp_shadow[warp] + __popc(m_shadow & lt);
            pb.sray_o[slot] = sro;
            pb.sray_d[slot] = srd;
            pb.scontrib[slot] = scon;
        }
        __syncthreads();
    }
}

// What a path carries into the next depth of the volume integrator (the queues of the next wave).
struct VolumeNext {
    bool push;
    float4 ro, rd, beta, s1o, s1d;
    uint2 id;
    ulonglong2 pcg;
    float u_rr;
};

// End of one loop iteration of mega_vpt_naive.cpp:439-452 (NaN guard, Russian roulette) and, for the survivors, the draws at
// the top of the next iteration (:256-273): u_rr, then the in-medium light sample whose shadow ray the next wave traces.
__device__ __forceinline__ void volume_continue(const DeviceScene &sc, uint32_t depth, bool alive, V3 beta, float pdf_bsdf, float u_rr,
                                                V3 next_o, V3 next_d, uint32_t path_id, uint32_t state, const PCG32 &rng, VolumeNext &nx) {
    nx.push = false;
    nx.u_rr = 0.f;
    if (alive) {
        if (isnan(beta.x) || isnan(beta.y) || isnan(beta.z)) beta = v3(0.f);
        alive = !(beta.x <= 0.f && beta.y <= 0.f && beta.z <= 0.f);
        if (alive) {
            float q = fmaxf(max3(beta) * 1.f, .05f);
            if (depth + 1u >= sc.rr_depth) {
                if (q < sc.rr_threshold && u_rr >= q) alive = false;
                beta = beta * (q < sc.rr_threshold ? 1.0f / q : 1.f);
            }
        }
    }
    if (alive && depth + 1u < sc.max_depth) {
        nx.push = true;
        if (depth + 2u >= sc.rr_depth) nx.u_rr = lcg(state);
        float u_sel = lcg(state), ul0 = lcg(state), ul1 = lcg(state);
        medium_light_shadow_ray(sc, next_o, u_sel, ul0, ul1, nx.s1o, nx.s1d);
        nx.ro = make_float4(next_o.x, next_o.y, next_o.z, 0.f);
        nx.rd = make_float4(next_d.x, next_d.y, next_d.z, kFltMax);
        nx.beta = make_float4(beta.x, beta.y, beta.z, pdf_bsdf);
        nx.id = make_uint2(path_id, state);
        nx.pcg = make_ulonglong2(rng.state, rng.inc);
    }
}

__device__ __forceinline__ void volume_store_next(const PathBuffers &pb, int out, uint32_t slot, const VolumeNext &nx) {
    pb.ray_o[out][slot] = nx.ro;
    pb.ray_d[out][slot] = nx.rd;
    pb.beta_pdf[out][slot] = nx.beta;
    pb.id_rng[out][slot] = nx.id;
    pb.pcg[out][slot] = nx.pcg;
    pb.u_rr[out][slot] = nx.u_rr;
    pb.s1ray_o[slot] = nx.s1o;
    pb.s1ray_d[slot] = nx.s1d;
    pb.occl2[out][slot] = 0u;
}

// Volume wave, step 1 (every path of the depth): advance the PCG32 stream by the occlusion results, sample the medium
// along the ray (homogeneous.cpp:48-118).  Absorption / scattering events finish here; paths that reach their surface hit
// (event 3) write their updated throughput, pdf, PCG state and the MOVED ray origin back in place and are appended to the
// hit bucket of their closure kind - the same material sort as the surface integrator - for volume_surface_kernel.
__global__ void __launch_bounds__(kBlock) volume_medium_kernel(DeviceScene sc, PathBuffers pb, uint32_t depth) {
    const uint32_t n = *path_count(pb.counts, depth);
    const int in = depth & 1u, out = in ^ 1;
    const V3 sigma_a = v3(sc.sigma_a[0], sc.sigma_a[1], sc.sigma_a[2]), sigma_s = v3(sc.sigma_s[0], sc.sigma_s[1], sc.sigma_s[2]);
    for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        uint32_t list = ~0u;// which list this item is appended to, if any
        VolumeNext nx;
        nx.push = false;
        if (i < n) {
            const uint4 hit = pb.hit[i];
            float4 ro = pb.ray_o[in][i], rd = pb.ray_d[in][i];
            float4 bp = pb.beta_pdf[in][i];
            uint2 ir = pb.id_rng[in][i];
            ulonglong2 pc = pb.pcg[in][i];
            PCG32 rng{pc.x, pc.y};
            // transmittance rays that hit a surface consumed three draws each: previous bounce's surface NEE, then this
            // bounce's in-medium direct light (their contribution is f = Tr * bsdf(-d, d) = 0 for opaque closures)
            if (pb.occl2[in][i] != 0u) { rng.uniform_uint(); rng.uniform_uint(); rng.uniform_uint(); }
            if (pb.occl1[i] != 0u) { rng.uniform_uint(); rng.uniform_uint(); rng.uniform_uint(); }
            V3 beta = v3(bp.x, bp.y, bp.z);
            V3 o = v3(ro.x, ro.y, ro.z), d = v3(rd.x, rd.y, rd.z);
            const bool valid = hit.x != ~0u;
            const float bu = __uint_as_float(hit.z), bv = __uint_as_float(hit.w);
            float t_max = kFltMax;
            if (valid) t_max = length(hit_position(sc, hit.x, hit.y, v3(1.f - bu - bv, bu, bv)) - o);
            uint32_t event;
            V3 mf, no, nd;
            float mpdf;
            homogeneous_medium_sample(sigma_a, sigma_s, sc.medium_g, o, d, t_max, rng, event, mf, mpdf, no, nd);
            {
                float w = mpdf > 0.f ? 1.f / mpdf : 0.f;
                beta = beta * (mf * w);
            }
            if (event == 3u) {
                if (valid) {// surface event: handed to volume_surface_kernel<kind>
                    list = 1u + __ldg(sc.inst_kind + hit.x);
                    pb.ray_o[in][i] = make_float4(no.x, no.y, no.z, ro.w);
                    pb.beta_pdf[in][i] = make_float4(beta.x, beta.y, beta.z, mpdf);
                    pb.pcg[in][i] = make_ulonglong2(rng.state, rng.inc);
                }
            } else {
                volume_continue(sc, depth, true, beta, mpdf, pb.u_rr[in][i], no, nd, ir.x, ir.y, rng, nx);
                if (nx.push) list = 0u;
            }
        }
        // list 0: the next wave, list 1 + k: hit bucket k
        block_append<kBlock, 1u + kHitKinds>(list != ~0u ? 1u << list : 0u,
                                             [&](uint32_t l) { return l == 0u ? path_count(pb.counts, depth + 1u) : bucket_count(pb.counts, l - 1u, depth); },
                                             [&](uint32_t l, uint32_t slot) {
                                                 if (l == 0u) volume_store_next(pb, out, slot, nx);
                                                 else pb.hit_index[l - 1u][slot] = i;
                                             });
    }
}

// Volume wave, step 2 (surface events of one closure kind): emitter hit seen from the moved origin, surface NEE +
// closure sample (mega_vpt_naive.cpp:300-437), then the common end of the iteration.
template<uint32_t KIND, bool TEXTURED = false>
__global__ void __launch_bounds__(kBlock, 2) volume_surface_kernel(DeviceScene sc, PathBuffers pb, uint32_t depth) {
    const uint32_t n = *bucket_count(pb.counts, KIND, depth);
    const int in = depth & 1u, out = in ^ 1;
    for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
        const uint32_t j = base + threadIdx.x;
        bool push_shadow = false;
        float4 sro, srd, scon;
        VolumeNext nx;
        nx.push = false;
        if (j < n) {
            const uint32_t i = pb.hit_index[KIND][j];
            const uint4 hit = pb.hit[i];
            float4 ro = pb.ray_o[in][i], rd = pb.ray_d[in][i];// ro = the origin moved onto the surface by the medium step
            float4 bp = pb.beta_pdf[in][i];
            uint2 ir = pb.id_rng[in][i];
            ulonglong2 pc = pb.pcg[in][i];
            PCG32 rng{pc.x, pc.y};
            V3 beta = v3(bp.x, bp.y, bp.z);
            float pdf_bsdf = bp.w;
            uint32_t state = ir.y;
            V3 no = v3(ro.x, ro.y, ro.z), d = v3(rd.x, rd.y, rd.z);
            const float bu = __uint_as_float(hit.z), bv = __uint_as_float(hit.w);
            Interaction it = make_interaction(sc, hit.x, hit.y, v3(1.f - bu - bv, bu, bv));
            it.back_facing = dot(-d, it.ng) < 0.0f;
            if (it.shape.has_light()) {// evaluate_hit from the MOVED ray origin (mega_vpt_naive.cpp:308,319)
                LightEval e = evaluate_hit<TEXTURED>(sc, it, no);
                V3 add = beta * e.L * balance_heuristic(pdf_bsdf, e.pdf);
                float4 li = pb.li[ir.x];
                li.x += add.x;
                li.y += add.y;
                li.z += add.z;
                pb.li[ir.x] = li;
            }
            if (KIND != kHitEmitter) {
                float u_sel = lcg(state);
                float ul0 = lcg(state), ul1 = lcg(state);
                float u_lobe = lcg(state);
                float ub0 = lcg(state), ub1 = lcg(state);
                LightSample ls = sample_light<TEXTURED>(sc, it, u_sel, ul0, ul1);
                const lrk_surface *surf = sc.surfaces + it.shape.surface_tag;
                V3 wo = -d;
                V3 contrib = v3(0.f), wi, f;
                float pdf;
                // true_hit(medium_tag = 0) <=> 0 <= priority of the environment medium: always true (medium_tracker.cpp:19-21)
                with_hit_closure<KIND, TEXTURED>(sc, surf, it, wo, [&] { return closure_frame<TEXTURED>(sc, surf, it, wo); }, [&](auto &cl, const Frame &fr) {
                    shade_surface<true>(cl, it, fr, wo, ls, beta, u_lobe, ub0, ub1, contrib, wi, f, pdf);
                });
                push_shadow = true;// traced even with a zero contribution: its occlusion advances the PCG stream of the next bounce
                sro = ls.ray_o_tmin;
                srd = ls.ray_d_tmax;
                scon = make_float4(contrib.x, contrib.y, contrib.z, __uint_as_float(ir.x));
                V3 next_o = p_robust(it, wi);
                float w = pdf > 0.f ? 1.f / pdf : 0.f;
                beta = beta * (w * f);
                volume_continue(sc, depth, true, beta, pdf, pb.u_rr[in][i], next_o, wi, ir.x, state, rng, nx);
                if (!nx.push && scon.x == 0.f && scon.y == 0.f && scon.z == 0.f) push_shadow = false;// nothing depends on it
            }
        }
        // list 0: the next wave, list 1: the surface NEE shadow records (list 0's slot is stored first: the record points at it)
        uint32_t next_slot = ~0u;
        block_append<kBlock, 2u>((nx.push ? 1u : 0u) | (push_shadow ? 2u : 0u),
                                 [&](uint32_t l) { return l == 0u ? path_count(pb.counts, depth + 1u) : shadow_count(pb.counts, depth); },
                                 [&](uint32_t l, uint32_t slot) {
                                     if (l == 0u) {
                                         next_slot = slot;
                                         volume_store_next(pb, out, slot, nx);
                                     } else {
                                         pb.sray_o[slot] = sro;
                                         pb.sray_d[slot] = srd;
                                         pb.scontrib[slot] = scon;
                                         pb.s2_target[slot] = next_slot;
                                     }
                                 });
    }
}

}// namespace LRK_SHADE_VARIANT
}// namespace lrk
