// Resampled next-event estimation of the option "light_candidates" (DESIGN.md §4 (Resampled light sampling)): at a surface vertex,
// M candidates are drawn from the light sampling the other options configure, each is weighted by its unshadowed contribution, and
// one of them is kept for the shadow ray (resampled importance sampling, Talbot et al. 2005).  This header holds the parts that do
// not touch the scene: the candidates' numbers, the weight rule, the reservoir and the kept candidate's weight.
//
// No CUDA built-ins: the shade kernels (pathcommon.cuh) and tests/host_device compile the same expressions.  The hash and the LCG
// are the library's own (vecmath.cuh), so the host harness compiles this header with the CUDA headers on its include path.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "vecmath.cuh"

namespace lrk {

constexpr uint32_t kLightCandidatesMax = 32u;// "light_candidates" takes 0 .. 32; 0 and 1 are one light sample without resampling

// ---- the candidates' numbers ------------------------------------------------------------------------------------------------------
// Candidate 0 takes the bounce's own (u_sel, ul0, ul1).  Candidates 1 .. M - 1 take theirs, and the reservoir's number, from the
// library's LCG seeded with a hash of those three numbers and the depth: the sampler's own draws per bounce do not change, so a
// sample's radiance still depends on (pixel, sample index) alone.
__device__ __forceinline__ uint32_t resampling_float_bits(float x) {
    uint32_t b;
    memcpy(&b, &x, sizeof(b));
    return b;
}
__device__ __forceinline__ uint32_t light_candidates_seed(float u_sel, float ul0, float ul1, uint32_t depth) {
    return xxhash32_uint4(resampling_float_bits(u_sel), resampling_float_bits(ul0), resampling_float_bits(ul1), depth);
}
// The numbers of the next candidate (i >= 1), in this order: its selection number, its two point numbers, its reservoir number.
__device__ __forceinline__ void light_candidate_numbers(uint32_t &state, float &u_sel, float &u0, float &u1, float &u_reservoir) {
    u_sel = lcg(state);
    u0 = lcg(state);
    u1 = lcg(state);
    u_reservoir = lcg(state);
}

// ---- the target and the weight ----------------------------------------------------------------------------------------------------
// p_hat = Y(c), the luminance of the candidate's unshadowed contribution c = f * L * balance(p, b) with the weights of the adaptive
// mode's display luminance
__device__ __forceinline__ float resampling_target(float r, float g, float b) { return 0.2126f * r + 0.7152f * g + 0.0722f * b; }

// w = p_hat / p for a source pdf p > 0 and a finite p_hat > 0; 0 otherwise.  A candidate of weight 0 still counts in M.
__device__ __forceinline__ float resampling_weight(float p_hat, float p) {
    return p > 0.f && p_hat > 0.f && p_hat <= kFltMax ? p_hat / p : 0.f;
}

// ---- the reservoir ----------------------------------------------------------------------------------------------------------------
// Candidates arrive in order 0, 1, ...; candidate i >= 1 replaces the kept one with probability w_i / W, W the sum of the weights so
// far, with its reservoir number u.  A weight that is not finite and positive counts as 0: such a candidate is never kept.
struct LightReservoir {
    float w_sum;
    uint32_t chosen;
};
__device__ __forceinline__ LightReservoir light_reservoir_empty() { return {0.f, 0u}; }
// Adds candidate i of weight w; true when it is now the kept candidate (for candidate 0: when its weight is positive).
__device__ __forceinline__ bool light_reservoir_add(LightReservoir &r, uint32_t i, float w, float u) {
    if (!(w > 0.f && w <= kFltMax)) w = 0.f;
    r.w_sum += w;
    if (w == 0.f) return false;
    if (i != 0u && !(u < w / r.w_sum)) return false;
    r.chosen = i;
    return true;
}

// The weight of the kept candidate's contribution c_y: W / (M * p_hat_y); 0 when every weight was 0 (no shadow ray).
__device__ __forceinline__ float light_reservoir_weight(const LightReservoir &r, uint32_t m, float p_hat_chosen) {
    return r.w_sum > 0.f ? r.w_sum / (static_cast<float>(m) * p_hat_chosen) : 0.f;
}

}// namespace lrk
