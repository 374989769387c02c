// The adaptive mode's kernels (lrk_render_adaptive in lrk.cu, DESIGN.md §4 (Adaptive sampling)).
//
// A round renders the active pixel list, which is always a concatenation of whole 8x4 pixel blocks of build_pixel_list's order:
// block b covers list[start[b] .. start[b + 1]) (at most 32 pixels, fewer at tile edges).  After the round, one warp per block
// takes the maximum pixel error (adaptive.h) over the block's pixels; a block whose maximum is below the threshold stops, and
// its pixels' sample counts are recorded.  The surviving blocks are then compacted, in order, into the next round's list:
// adaptive_test_kernel writes one packed {pixels, 1} word per surviving block, an exclusive scan of those words
// (cub::DeviceScan) gives every survivor its new block index and pixel offset, and adaptive_compact_kernel moves it there.
#pragma once
#include "adaptive.h"
#include "pathstate.cuh"

namespace lrk {

constexpr int kAdaptiveBlock = 256;// 8 warps: 8 pixel blocks per thread block

// keep[b] = 0 when block b stops (its pixels' counts are set to `count`), else (pixels << 32) | 1; keep[nblocks] = 0, so that the
// exclusive scan of keep[0 .. nblocks] ends with the totals.  last: the round reached max_spp, every block stops.
__global__ void __launch_bounds__(kAdaptiveBlock) adaptive_test_kernel(uint32_t width, const float4 *__restrict__ film, const float2 *__restrict__ moments,
                                                                       const uint32_t *__restrict__ list, const uint32_t *__restrict__ start,
                                                                       uint32_t nblocks, float threshold, uint32_t count, bool last,
                                                                       uint32_t *__restrict__ counts, unsigned long long *__restrict__ keep) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5u, lane = threadIdx.x & 31u;
    if (b > nblocks) return;// whole warps
    if (b == nblocks) {
        if (lane == 0u) keep[b] = 0ull;
        return;
    }
    const uint32_t first = start[b], n = start[b + 1u] - first;
    float e = 0.f;
    size_t pid = 0u;
    if (lane < n) {
        const uint32_t pixel = list[first + lane];
        pid = static_cast<size_t>(pixel >> 16u) * width + (pixel & 0xffffu);
        const float2 m = moments[pid];
        e = adaptive_error(m.x, m.y, film[pid].w);
    }
#pragma unroll
    for (uint32_t o = 16u; o > 0u; o >>= 1u) e = fmaxf(e, __shfl_xor_sync(0xffffffffu, e, o));
    const bool stop = last || e < threshold;
    if (stop && lane < n) counts[pid] = count;
    if (lane == 0u) keep[b] = stop ? 0ull : (static_cast<unsigned long long>(n) << 32u) | 1ull;
}

// offsets = exclusive scan of keep[0 .. nblocks]: surviving block b becomes block (uint32_t)offsets[b] of the next list, its
// pixels start at offsets[b] >> 32 there; start_out gets the new block starts and the closing sentinel.
__global__ void __launch_bounds__(kAdaptiveBlock) adaptive_compact_kernel(const uint32_t *__restrict__ list, const uint32_t *__restrict__ start,
                                                                          uint32_t nblocks, const unsigned long long *__restrict__ keep,
                                                                          const unsigned long long *__restrict__ offsets,
                                                                          uint32_t *__restrict__ list_out, uint32_t *__restrict__ start_out) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5u, lane = threadIdx.x & 31u;
    if (b == 0u && lane == 0u) {
        const unsigned long long total = offsets[nblocks];
        start_out[static_cast<uint32_t>(total)] = static_cast<uint32_t>(total >> 32u);
    }
    if (b >= nblocks) return;
    const unsigned long long k = keep[b];
    if (k == 0ull) return;
    const unsigned long long o = offsets[b];
    const uint32_t n = static_cast<uint32_t>(k >> 32u), to = static_cast<uint32_t>(o >> 32u);
    if (lane < n) list_out[to + lane] = list[start[b] + lane];
    if (lane == 0u) start_out[static_cast<uint32_t>(o)] = to;
}

// lrk_download_film_variance: v of adaptive.h for every pixel with a sample count, 0 elsewhere
__global__ void __launch_bounds__(kBlock) adaptive_variance_kernel(const float4 *__restrict__ film, const float2 *__restrict__ moments,
                                                                   const uint32_t *__restrict__ counts, float *__restrict__ out, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float2 m = moments[i];
    out[i] = counts[i] != 0u ? adaptive_variance(m.x, m.y, film[i].w) : 0.f;
}

}// namespace lrk
