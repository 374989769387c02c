// The pixel error of the adaptive mode (lrk_render_adaptive, DESIGN.md §4 (Adaptive sampling)).  Plain C++ without CUDA built-ins: the sm_90a
// test kernel (adaptive.cuh) and tests/host_device compile the same expressions, in IEEE fp32 and in this operation order
// (lrk.cu is built with -fmad=false, the host test with -ffp-contract=off), so a numpy restatement matches them bit for bit.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define LRK_ADAPTIVE_FN __host__ __device__ __forceinline__
#else
#define LRK_ADAPTIVE_FN inline
#endif

namespace lrk {

// Variance of the pixel's mean display luminance from n = the film weight (samples the film kept) and the moments
// s1 = sum Y, s2 = sum Y^2 of those samples.  Fewer than two samples give no estimate: +inf.
LRK_ADAPTIVE_FN float adaptive_variance(float s1, float s2, float n) {
    if (!(n >= 2.f)) return INFINITY;
    const float m = s1 / n;
    return fmaxf(s2 / n - m * m, 0.f) / (n - 1.f);
}

// Relative standard error of the pixel's mean: sqrt(v) / max(m, 0.01).  +inf with fewer than two samples.
LRK_ADAPTIVE_FN float adaptive_error(float s1, float s2, float n) {
    if (!(n >= 2.f)) return INFINITY;
    const float m = s1 / n;
    const float v = fmaxf(s2 / n - m * m, 0.f) / (n - 1.f);
    return sqrtf(v) / fmaxf(m, 0.01f);
}

}// namespace lrk
