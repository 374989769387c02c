// The denoiser's kernels (lrk_denoise, lrk_download_gbuffer in lrk.cu; the arithmetic is in denoise.h).  One thread per film pixel:
// guides from the G-buffer sums, the demodulated input, five à-trous steps ping-ponging (I.rgb, var), the remodulated output.
#pragma once
#include "denoise.h"
#include "pathstate.cuh"

namespace lrk {

// albedo_cov, normal_depth and v = adaptive_variance(S1, S2, film weight) of every pixel; zero_empty: v = 0 for pixels without
// samples (the download's convention) instead of the +inf of fewer than two samples.
__global__ void __launch_bounds__(kBlock) denoise_guides_kernel(const float4 *__restrict__ film, const float2 *__restrict__ moments,
                                                                const float4 *__restrict__ gb_albedo, const float4 *__restrict__ gb_normal,
                                                                const float *__restrict__ gb_hits, DenoiseVec4 *__restrict__ albedo_cov,
                                                                DenoiseVec4 *__restrict__ normal_depth, float *__restrict__ variance, uint32_t n,
                                                                bool zero_empty) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 a = gb_albedo[i], nt = gb_normal[i];
    DenoiseVec4 ac, nd;
    denoise_guides(DenoiseVec4{a.x, a.y, a.z, a.w}, DenoiseVec4{nt.x, nt.y, nt.z, nt.w}, gb_hits[i], ac, nd);
    albedo_cov[i] = ac;
    normal_depth[i] = nd;
    const float2 m = moments[i];
    variance[i] = zero_empty && a.w == 0.f ? 0.f : adaptive_variance(m.x, m.y, film[i].w);
}

// The filter's input from the film normalised as convert_film_kernel normalises it.
__global__ void __launch_bounds__(kBlock) denoise_input_kernel(DeviceScene sc, const float4 *__restrict__ film, const DenoiseVec4 *__restrict__ albedo_cov,
                                                               const float *__restrict__ variance, DenoiseVec4 *__restrict__ out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 c = film[i];
    const float inv = 1.f / fmaxf(c.w, 1.f);
    out[i] = denoise_input((inv * sc.film_scale[0]) * c.x, (inv * sc.film_scale[1]) * c.y, (inv * sc.film_scale[2]) * c.z, albedo_cov[i], variance[i]);
}

__global__ void __launch_bounds__(kBlock) denoise_atrous_kernel(const DenoiseVec4 *__restrict__ in, const DenoiseVec4 *__restrict__ albedo_cov,
                                                                const DenoiseVec4 *__restrict__ normal_depth, DenoiseVec4 *__restrict__ out, uint32_t w,
                                                                uint32_t h, int step) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w * h) return;
    out[i] = denoise_pixel(in, albedo_cov, normal_depth, static_cast<int>(w), static_cast<int>(h), static_cast<int>(i % w), static_cast<int>(i / w), step);
}

__global__ void __launch_bounds__(kBlock) denoise_output_kernel(const DenoiseVec4 *__restrict__ in, const DenoiseVec4 *__restrict__ albedo_cov,
                                                                DenoiseVec4 *__restrict__ out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = denoise_output(in[i], albedo_cov[i]);
}

}// namespace lrk
