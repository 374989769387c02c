// Per-path device functions shared by the wavefront kernels (kernels.cuh) and the per-thread volume kernel (volume_general.cuh):
// camera ray generation, closure set-up and the light / sampled-direction evaluation of a surface hit, PCG32, the homogeneous
// medium's distance sampling.  No CUDA built-ins: tests/host_device compiles this file for the host.
#pragma once
#include <type_traits>
#include <utility>

#include "hit_kinds.h"
#include "shading.cuh"

namespace lrk {

// ---- Camera: src/base/filter.cpp:50-64, src/base/camera.cpp:212-224, src/cameras/pinhole.cpp:60-67 ----
__device__ __forceinline__ void sample_alias_filter(const lrk_camera *cam, float u_in, uint32_t &index, float &uu) {
    constexpr uint32_t n = LRK_FILTER_LUT_SIZE - 1u;
    float u = u_in * static_cast<float>(n);
    uint32_t i = min(max(static_cast<uint32_t>(u), 0u), n - 1u);
    float u_remapped = u - floorf(u);
    float prob = cam->filter_alias_probs[i];
    bool keep = u_remapped < prob;
    index = keep ? i : cam->filter_alias_indices[i];
    uu = keep ? u_remapped / prob : (u_remapped - prob) / (1.0f - prob);
}

// Camera ray for pixel (px, py) from the two filter numbers: Filter::Instance::sample + Camera::generate_ray + pinhole
__device__ __forceinline__ void camera_ray(const lrk_camera *cam, uint32_t px, uint32_t py, float ux, float uy, float4 &ro, float4 &rd,
                                           float &weight_out) {
    uint32_t iy, ix;
    float fy, fx;
    sample_alias_filter(cam, ux, iy, fy);
    sample_alias_filter(cam, uy, ix, fx);
    float pdf = cam->filter_pdf[iy] * cam->filter_pdf[ix];
    float f = lerp(cam->filter_lut[ix], cam->filter_lut[ix + 1u], fx) * lerp(cam->filter_lut[iy], cam->filter_lut[iy + 1u], fy);
    float ppx = static_cast<float>(ix) + fx, ppy = static_cast<float>(iy) + fy;
    constexpr float inv_size = 1.0f / static_cast<float>(LRK_FILTER_LUT_SIZE);
    float ox = (ppx * inv_size * 2.0f - 1.0f) * cam->filter_radius + cam->filter_shift[0];
    float oy = (ppy * inv_size * 2.0f - 1.0f) * cam->filter_radius + cam->filter_shift[1];
    float weight = 1.f * (f / pdf);
    float pixel_x = static_cast<float>(px) + .5f + ox;
    float pixel_y = static_cast<float>(py) + .5f + oy;
    float rx = static_cast<float>(cam->resolution[0]), ry = static_cast<float>(cam->resolution[1]);
    float kk = cam->tan_half_fov / ry;
    float p_x = (pixel_x * 2.0f - rx) * kk;
    float p_y = (pixel_y * 2.0f - ry) * kk;
    V3 direction = normalize(v3(p_x, -p_y, -1.f));
    const float *m = cam->camera_to_world;
    V3 c0 = v3(m[0], m[4], m[8]), c1 = v3(m[1], m[5], m[9]), c2 = v3(m[2], m[6], m[10]), c3 = v3(m[3], m[7], m[11]);
    V3 o = 0.f * c0 + 0.f * c1 + 0.f * c2 + 1.f * c3;
    V3 d = normalize(direction.x * c0 + direction.y * c1 + direction.z * c2);
    ro = make_float4(o.x, o.y, o.z, 0.f);
    rd = make_float4(d.x, d.y, d.z, kFltMax);
    weight_out = weight;
}

// ---- shade ----------------------------------------------------------------------------------------------
// Closure of the hit's surface node: constants straight from the node, image-textured parameters evaluated at the hit's uv.
// TEXTURED = false is the instantiation for scenes without image-textured parameters / normal maps: the constants-only code.
template<bool TEXTURED, typename Closure>
__device__ __forceinline__ void init_closure(const DeviceScene &sc, Closure &cl, const lrk_surface *node, const Interaction &it) {
    if (TEXTURED && (node->flags & LRK_SURFACE_HAS_TEXTURES)) {
        lrk_surface s = *node;
        resolve_surface_textures(sc, s, it.u, it.v);
        cl.init(s);
    } else {
        cl.init(*node);
    }
}

// The frame the closure works in: the interaction's shading frame, or the normal-mapped one (surface.h:236-253).
template<bool TEXTURED>
__device__ __forceinline__ Frame closure_frame(const DeviceScene &sc, const lrk_surface *node, const Interaction &it, V3 wo) {
    if (TEXTURED && (node->flags & LRK_SURFACE_HAS_NORMAL_MAP)) return normal_mapped_frame(sc, node, it, wo);
    return it.shading;
}

// The closure of hit bucket KIND (hit_kinds.h) at a hit seen from wo: calls f(closure, frame) with the frame the closure works in,
// frame_of() (closure_frame, or the caller's copy of it), and returns the closure's eta scale for Russian roulette
// (mega_path.cpp:113,133-138).  Layered's init needs the frame, so Layered alone takes the frame before init.  Emitter-only hits
// have no closure: f is not called.
template<uint32_t KIND> struct hit_closure { using type = MicrofacetFamilyClosure<KIND - 1u>; };// Mirror .. Metal: kind = type + 1
template<> struct hit_closure<kHitMatte> { using type = MatteClosure; };
template<> struct hit_closure<kHitDisney> { using type = DisneyClosure; };
template<> struct hit_closure<kHitMix> { using type = MixClosure; };
template<> struct hit_closure<kHitDisneyTrans> { using type = DisneyTransClosure; };
template<> struct hit_closure<kHitDisneyThin> { using type = DisneyThinClosure; };

template<uint32_t KIND, bool TEXTURED, typename FrameOf, typename F>
__device__ __forceinline__ float with_hit_closure(const DeviceScene &sc, const lrk_surface *surf, const Interaction &it, const V3 &wo, FrameOf &&frame_of,
                                                 F &&f) {
    if constexpr (KIND == kHitEmitter) {
        return 1.f;
    } else if constexpr (KIND == kHitLayered) {
        LayeredClosure cl;
        const Frame fr = frame_of();
        cl.init(*surf, sc.surfaces, it, fr, wo);
        f(cl, fr);
        return cl.rr_eta_scale;
    } else {
        typename hit_closure<KIND>::type cl;
        if constexpr (KIND == kHitMix) cl.init(*surf, sc.surfaces);
        else init_closure<TEXTURED>(sc, cl, surf, it);
        f(cl, frame_of());
        if constexpr (KIND == kHitDisneyTrans) return (surf->lobes & LRK_DISNEY_LOBE_SPEC_TRANS) ? cl.rr_eta_scale : 1.f;// disney.cpp:531-533
        else if constexpr (KIND == kHitMatte || KIND == kHitDisney || KIND == kHitDisneyThin) return 1.f;// closure->eta() is empty
        else return cl.rr_eta_scale;
    }
}

// Evaluates the closure for the light sample's direction (NEE term) and for the direction the closure itself samples.
// Both evaluations run through ONE copy of the closure code (a two-trip loop that is deliberately not unrolled): the Disney
// closure is several thousand SASS instructions and two inlined copies thrash the instruction cache.
// VOLUME selects the direct-light weight of the volume integrator: 1 / (pdf_light + pdf_bsdf + pdf_transmittance) with
// pdf_transmittance = 0 for an unoccluded ray (mega_vpt_naive.cpp:403-407) instead of the balance heuristic (mega_path.cpp:108-113).
// f / pdf of the closure's own sample: evaluate_local at the sampled direction for every closure (matte.cpp:118-134,
// disney.cpp:583-586, ...) except Mix, whose sample is not its evaluate (mix.cpp:158-180) and which provides evaluate_sampled.
// The choice is made at compile time so that the other closures keep ONE call site of evaluate_local in the two-trip loop.
template<typename Closure, typename = void>
struct has_evaluate_sampled : std::false_type {};
template<typename Closure>
struct has_evaluate_sampled<Closure, std::void_t<decltype(std::declval<const Closure &>().evaluate_sampled(V3{}, V3{}))>> : std::true_type {};

// Closures that work on world-space directions and return the sample's f / pdf themselves (Layered: its random walks are seeded
// from the bits of the world-space vectors): evaluate_world(wi), sample_world(u_lobe, u0, u1) -> sampled_wi, sampled.
template<typename Closure, typename = void>
struct has_world_api : std::false_type {};
template<typename Closure>
struct has_world_api<Closure, std::void_t<decltype(std::declval<Closure &>().sample_world(0.f, 0.f, 0.f))>> : std::true_type {};

template<typename Closure>
__device__ __forceinline__ void shade_surface_eval(Closure &cl, const Interaction &it, const Frame &shading, V3 wo, const LightSample &ls,
                                                   float u_lobe, float ub0, float ub1, SurfEval &e_light, V3 &wi_world, V3 &f_over, float &pdf_bsdf) {
    V3 wo_local = shading.world_to_local(wo);
    cl.prepare(wo_local);
    V3 wi_sampled_local;
    bool run_sampled;
    if constexpr (has_world_api<Closure>::value) {
        run_sampled = cl.sample_world(u_lobe, ub0, ub1);
        wi_world = cl.sampled_wi;
        wi_sampled_local = shading.world_to_local(wi_world);
    } else {
        run_sampled = cl.sample_direction(wo_local, u_lobe, ub0, ub1, wi_sampled_local);
        wi_world = shading.local_to_world(wi_sampled_local);
    }
    const bool run_light = ls.eval.pdf > 0.0f;
    V3 wi_w = v3(ls.ray_d_tmax.x, ls.ray_d_tmax.y, ls.ray_d_tmax.z);
    V3 wi_l = shading.world_to_local(wi_w);
    bool run = run_light;
    e_light.f = f_over = v3(0.f);
    e_light.pdf = pdf_bsdf = 0.f;
#pragma unroll 1
    for (int k = 0; k < 2; k++) {
        SurfEval e;
        e.f = v3(0.f);
        e.pdf = 0.f;
        if (run) {
            if constexpr (has_world_api<Closure>::value) {
                if (k == 0) {
                    e = cl.evaluate_world(wi_w);
                } else {
                    e.f = cl.sampled.f;
                    e.pdf = cl.sampled.pdf;
                }
            } else if constexpr (has_evaluate_sampled<Closure>::value) {
                e = k == 0 ? cl.evaluate_local(wo_local, wi_l) : cl.evaluate_sampled(wo_local, wi_l);
            } else {
                e = cl.evaluate_local(wo_local, wi_l);
            }
            if (!validate_surface_sides(it.ng, shading.n, wo, wi_w)) {
                e.f = v3(0.f);
                e.pdf = 0.f;
            }
        }
        if (k == 0) {
            e_light = e;
            wi_w = wi_world;
            wi_l = wi_sampled_local;
            run = run_sampled;
        } else {
            f_over = e.f;
            pdf_bsdf = e.pdf;
        }
    }
}

template<bool VOLUME, typename Closure>
__device__ __forceinline__ void shade_surface(Closure &cl, const Interaction &it, const Frame &shading, V3 wo, const LightSample &ls, V3 beta,
                                              float u_lobe, float ub0, float ub1, V3 &contrib, V3 &wi_world, V3 &f_over, float &pdf_bsdf) {
    SurfEval e_light;
    shade_surface_eval(cl, it, shading, wo, ls, u_lobe, ub0, ub1, e_light, wi_world, f_over, pdf_bsdf);
    const bool run_light = ls.eval.pdf > 0.0f;
    contrib = v3(0.f);
    if (run_light) {
        if (VOLUME) {
            float w = 1.f / (ls.eval.pdf + e_light.pdf + 0.f);
            contrib = w * beta * e_light.f * ls.eval.L * v3(1.f);
        } else {
            float w = balance_heuristic(ls.eval.pdf, e_light.pdf) / ls.eval.pdf;
            contrib = w * beta * e_light.f * ls.eval.L;
        }
    }
}

struct PCG32 {// src/util/rng.cpp:142-174
    unsigned long long state, inc;
    __device__ __forceinline__ uint32_t uniform_uint() {
        unsigned long long oldstate = state;
        state = oldstate * 0x5851f42d4c957f2dull + inc;
        uint32_t xorshifted = static_cast<uint32_t>(((oldstate >> 18u) ^ oldstate) >> 27u);
        uint32_t rot = static_cast<uint32_t>(oldstate >> 59u);
        return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31u));
    }
    __device__ __forceinline__ void set_sequence(unsigned long long init_seq) {
        state = 0ull;
        inc = (init_seq << 1u) | 1ull;
        uniform_uint();
        state = state + 0x853c49e6748fea9bull;
        uniform_uint();
    }
    __device__ __forceinline__ float uniform_float() { return fminf(kOneMinusEpsilon, static_cast<float>(uniform_uint()) * 0x1p-32f); }
};

__device__ __forceinline__ float comp3(V3 a, uint32_t i) { return i == 0u ? a.x : i == 1u ? a.y : a.z; }
__device__ __forceinline__ V3 exp3(V3 a) { return {expf(a.x), expf(a.y), expf(a.z)}; }

// HomogeneousMediumClosure::sample (src/media/homogeneous.cpp:48-118) with HenyeyGreenstein::sample_p (henyey_greenstein.cpp:28-48):
// event 0 absorb, 1 scatter, 3 hit surface (src/base/medium.h:31-36); f and pdf of the event, the ray that continues the path
__device__ __forceinline__ void homogeneous_medium_sample(V3 sigma_a, V3 sigma_s, float g, V3 o, V3 d, float t_max, PCG32 &rng, uint32_t &event,
                                                          V3 &mf, float &mpdf, V3 &no, V3 &nd) {
    const V3 sigma_t = sigma_a + sigma_s;
    V3 pch;
    pch.x = rng.uniform_float();
    pch.y = rng.uniform_float();
    pch.z = rng.uniform_float();
    float psum = pch.x + pch.y + pch.z;
    pch = v3(pch.x / psum, pch.y / psum, pch.z / psum);
    float u_rescaled = rng.uniform_float() * (pch.x + pch.y + pch.z);
    uint32_t channel = ~0u;
    float accum = 0.f;
#pragma unroll
    for (uint32_t c = 0; c < 3u; c++) {
        accum += comp3(pch, c);
        if (channel == ~0u && u_rescaled <= accum) channel = c;
    }
    float u = rng.uniform_float();
    float st = channel < 3u ? comp3(sigma_t, channel) : __int_as_float(0x7fc00000);
    float t = -logf(fmaxf(1.f - u, 1.17549435e-38f)) / st;
    no = o;
    nd = d;
    if (t > t_max) {
        event = 3u;
        t = t_max;
        V3 Tr = exp3(-sigma_t * t);
        no = o + d * t;
        mf = Tr;
        mpdf = (pch * Tr).x + (pch * Tr).y + (pch * Tr).z;
    } else {
        float p_absorb = comp3(sigma_a, channel) / st, p_scatter = comp3(sigma_s, channel) / st;
        float ur = rng.uniform_float() * (p_absorb + p_scatter);
        if (ur <= p_absorb) {
            event = 0u;
            mf = v3(0.f);
            V3 pp = pch * sigma_t;
            mpdf = pp.x + pp.y + pp.z;
        } else {
            event = 1u;
            V3 Tr = exp3(-sigma_t * t);
            float u0 = rng.uniform_float(), u1 = rng.uniform_float();
            float cosTheta = fabsf(g) < 1e-3f ? 1.f - 2.f * u0
                                              : -1.f / (2.f * g) * (1.f + sqr(g) - sqr((1.f - sqr(g)) / (1.f + g - 2.f * g * u0)));
            float sinTheta = sqrtf(fmaxf(0.f, 1.f - sqr(cosTheta)));
            float phi = 2.f * kPi * u1;
            float sphi, cphi;
            sincosf(phi, &sphi, &cphi);
            no = o + d * t;
            nd = v3(sinTheta * cphi, cosTheta, sinTheta * sphi);
            mf = Tr * sigma_s;
            V3 pp = pch * (sigma_t * Tr);
            mpdf = pp.x + pp.y + pp.z;
        }
    }
}

// shadow ray from a point in the medium towards a sampled light point: LightSampler::sample with
// Interaction{ray->origin()} (mega_vpt_naive.cpp:270-273): zero offset factor, so the origin is the point itself
__device__ __forceinline__ void medium_light_shadow_ray(const DeviceScene &sc, V3 p_from, float u_sel, float u0, float u1,
                                                        float4 &ro, float4 &rd) {
    float n = static_cast<float>(sc.light_count);
    uint32_t tag = static_cast<uint32_t>(clampf(u_sel * n, 0.f, n - 1.f));
    const lrk_light_handle handle = sc.light_handles[tag];
    ShapeHandle light_inst = decode_handle(__ldg(sc.inst_handles + handle.instance_id));
    const lrk_mesh mesh = sc.meshes[light_inst.mesh];
    float u = u0 * static_cast<float>(light_inst.tri_count);
    uint32_t i = min(max(static_cast<uint32_t>(u), 0u), light_inst.tri_count - 1u);
    float u_remapped = u - floorf(u);
    lrk_alias_entry entry = sc.alias[mesh.triangle_offset + i];
    bool keep = u_remapped < entry.prob;
    uint32_t triangle_id = keep ? i : entry.alias;
    float ux = keep ? u_remapped / entry.prob : (u_remapped - entry.prob) / (1.0f - entry.prob);
    V3 uvw = sample_uniform_triangle(ux, u1);
    V3 Lv = hit_position(sc, handle.instance_id, triangle_id, uvw) - p_from;
    float d = length(Lv);
    V3 dir = Lv * (1.f / d);
    ro = make_float4(p_from.x, p_from.y, p_from.z, 0.f);
    rd = make_float4(dir.x, dir.y, dir.z, d * .9999f);
}

}// namespace lrk
