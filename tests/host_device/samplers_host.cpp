// samplers_host.cpp — the DEVICE samplers (luisarender_b200/csrc/device/samplers.cuh: PathSampler's index derivation, the scrambled
// ZSobol index, permutation_element and the draws of every table-driven sampler) compiled for the host, so that
// tests/test_sampler_ranges_cpu.py can compare them bit for bit with the oracle's Sampler at the frame sizes and sample indices
// of the benchmark configurations without a GPU.  TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cmath>
#include <cstdint>
#include <cstring>

#include <cuda_runtime.h>

template<typename T>
static inline T __ldg(const T *p) { return *p; }
static inline uint32_t __brev(uint32_t v) {
    v = ((v >> 1u) & 0x55555555u) | ((v & 0x55555555u) << 1u);
    v = ((v >> 2u) & 0x33333333u) | ((v & 0x33333333u) << 2u);
    v = ((v >> 4u) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4u);
    v = ((v >> 8u) & 0x00ff00ffu) | ((v & 0x00ff00ffu) << 8u);
    return (v >> 16u) | (v << 16u);
}
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

#include "../../luisarender_b200/csrc/device/samplers.cuh"

// the layout of oracle_sampler_state (oracle/oracle.h): derived index, scrambled ZSobol index per dimension, and the pixel 2D
// followed by 1D, 2D, 1D, 2D per bounce, drawn as the shade kernels draw them
extern "C" int sh_state(const lrk_sampler *rec, uint32_t seed, const uint32_t *points, uint64_t n, const uint32_t *dims, uint32_t dim_count,
                        uint32_t bounces, uint64_t *index_out, uint64_t *zsobol_out, float *draws_out) {
    for (uint64_t i = 0; i < n; i++)
        if (rec->type == LRK_SAMPLER_PMJ02BN && points[3u * i + 2u] >= rec->spp) return -2;
    const lrk::SamplerRef ref{rec->type, seed, rec};
    const uint32_t per_point = 2u + 6u * bounces;
    for (uint64_t i = 0; i < n; i++) {
        lrk::PathSampler s;
        s.start(ref, points[3u * i], points[3u * i + 1u], points[3u * i + 2u]);
        index_out[i] = rec->type == LRK_SAMPLER_SOBOL || rec->type == LRK_SAMPLER_ZSOBOL ? s.index : 0u;
        for (uint32_t j = 0; j < dim_count; j++)
            zsobol_out[i * dim_count + j] = rec->type == LRK_SAMPLER_ZSOBOL ? lrk::PathSampler::zsobol_sample_index(*rec, s.index, dims[j]) : 0u;
        float *u = draws_out + i * per_point;
        const float2 p = s.pixel2d(ref);
        u[0] = p.x, u[1] = p.y;
        for (uint32_t b = 0; b < bounces; b++, u += 6) {
            u[2] = s.next1d(ref);
            const float2 l = s.next2d(ref);
            u[3] = l.x, u[4] = l.y;
            u[5] = s.next1d(ref);
            const float2 d = s.next2d(ref);
            u[6] = d.x, u[7] = d.y;
        }
    }
    return 0;
}

// rows (i, l, w, p) -> permutation_element(i, l, w, p)
extern "C" void sh_permutation_element(const uint32_t *in, uint64_t n, uint32_t *out) {
    for (uint64_t k = 0; k < n; k++) out[k] = lrk::permutation_element(in[4u * k], in[4u * k + 1u], in[4u * k + 2u], in[4u * k + 3u]);
}
