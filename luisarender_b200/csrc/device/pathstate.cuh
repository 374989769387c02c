// The path state of the wavefront kernels: queue layout and launch constants shared by the two translation units of the device
// library - lrk.cu (ray generation, traversal, classification, film; IEEE arithmetic, bit-exact with the oracle) and shade.cu
// (the closure kernels; compiled with the arithmetic the reference's own CUDA backend uses, see shade.cu).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "hit_kinds.h"
#include "scene.cuh"

namespace lrk {


constexpr int kBlock = 256;
#ifndef LRK_TRACE_MIN_BLOCKS
#define LRK_TRACE_MIN_BLOCKS 4// blocks of kTraceBlock threads per SM the traversal kernels are compiled for (register budget)
#endif
#ifndef LRK_SHADOW_MIN_BLOCKS
// the any-hit kernel has its own bound: a fifth resident block (at a few spilled bytes) helps it, the closest-hit kernel keeps four
// (the sweep behind these bounds was made on an earlier GPU and has not been repeated on the H100)
#define LRK_SHADOW_MIN_BLOCKS 5
#endif
#ifndef LRK_SHADE_BLOCK
#define LRK_SHADE_BLOCK 256
#endif
#ifndef LRK_SHADE_MIN_BLOCKS
#define LRK_SHADE_MIN_BLOCKS 2
#endif
constexpr int kShadeBlock = LRK_SHADE_BLOCK;// threads per block of the surface shade kernels (register-bound: see DESIGN.md)
constexpr uint32_t kCountSlots = 16u;   // rows of counters in PathBuffers::counts: 4 queue / cursor rows + one per hit bucket
constexpr uint32_t kMaxDepthSlots = 64u;// counters per row: one per depth

struct PathBuffers {
    float4 *ray_o[2];
    float4 *ray_d[2];
    float4 *beta_pdf[2];
    uint2 *id_rng[2];
    uint4 *hit;// {inst, prim, bary} per ray of the current queue (inst == ~0u: escaped)
    uint32_t *hit_index[kHitKinds];// per hit kind (hit_kinds.h): indices (into the current ray queue) of the rays that hit such a surface
    float4 *sray_o;
    float4 *sray_d;
    float4 *scontrib;// rgb + path id bits
    float4 *li;
    uint32_t *counts;
    uint32_t capacity;
    // the pass being rendered: generation slot id -> (pixel, sample index) for the table-driven samplers (samplers.cuh)
    const uint32_t *pass_pixel_list;
    uint32_t pass_pixel_offset, pass_npix, pass_spp_begin;
    // volume path integrator only (config C4)
    ulonglong2 *pcg[2]; // per-path PCG32 {state, inc}
    float *u_rr[2];     // Russian-roulette number of the coming bounce (drawn at the top of the loop, mega_vpt_naive.cpp:256-257)
    float4 *s1ray_o;    // in-medium direct-light shadow ray of the coming bounce (from the ray origin)
    float4 *s1ray_d;
    uint32_t *occl1;    // ... and whether it hit a surface (advances the PCG32 stream by three draws)
    uint32_t *occl2[2]; // same for the surface NEE shadow ray of the previous bounce
    uint32_t *s2_target;// queue slot (next bounce) that receives occl2 for each shadow record, ~0u if the path ended
    // cost probe of lrk_balance_shards: live rays per pixel tile, counted by classify_hits_kernel (nullptr outside the probe)
    uint32_t *tile_cost;
    uint32_t tile_cost_size, tile_cost_tiles_x;
    unsigned long long *stats;// [0] closest rays, [1] shadow rays, [2..4] closest nodes/tris/xforms, [5..7] shadow nodes/tris/xforms
};

// The rows of PathBuffers::counts, kMaxDepthSlots counters each (one per depth), all zeroed by the ray generation kernels at the start
// of a pass.  Free functions of the pointer rather than members: a member call on a kernel's PathBuffers parameter takes its address,
// which changes the shade kernels' code.
__host__ __device__ __forceinline__ uint32_t *path_count(uint32_t *counts, uint32_t depth) { return counts + depth; }// path-queue size
__host__ __device__ __forceinline__ uint32_t *shadow_count(uint32_t *counts, uint32_t depth) { return counts + kMaxDepthSlots + depth; }// shadow-queue size
__host__ __device__ __forceinline__ uint32_t *closest_cursor(uint32_t *counts, uint32_t depth) { return counts + 2u * kMaxDepthSlots + depth; }// closest-hit fetch cursor
__host__ __device__ __forceinline__ uint32_t *shadow_cursor(uint32_t *counts, uint32_t depth) { return counts + 3u * kMaxDepthSlots + depth; }// shadow fetch cursor
// fetch cursor of the volume integrator's in-medium shadow rays: the upper half of the shadow-cursor row (its depths stay below 32)
__host__ __device__ __forceinline__ uint32_t *medium_shadow_cursor(uint32_t *counts, uint32_t depth) { return counts + 3u * kMaxDepthSlots + 32u + depth; }
__host__ __device__ __forceinline__ uint32_t *bucket_count(uint32_t *counts, uint32_t kind, uint32_t depth) {// size of hit bucket `kind`
    return counts + ((4u + kind) * kMaxDepthSlots + depth);
}
static_assert(4u + kHitKinds <= kCountSlots, "PathBuffers::counts has one row of counters per hit bucket behind the four queue rows");

#ifdef __CUDACC__
// Block-aggregated append: every thread of the block calls it with the set of lists it appends one item to (bit l: list l < LISTS),
// and store(l, slot) is called for each of them with the item's slot in list l.  Ballots inside the warp, a scan of the warp counts in
// shared memory, one atomicAdd on counter(l) per list with items; the order inside a block is the thread order.  The last barrier
// lets the next call reuse the shared counts.
template<int BLOCK, uint32_t LISTS, typename Counter, typename Store>
__device__ __forceinline__ void block_append(uint32_t lists, Counter &&counter, Store &&store) {
    __shared__ uint32_t s_warp[LISTS][BLOCK / 32], s_base[LISTS];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5u;
    uint32_t masks[LISTS];
#pragma unroll
    for (uint32_t l = 0; l < LISTS; l++) {
        masks[l] = __ballot_sync(0xffffffffu, (lists >> l) & 1u);
        if (lane == 0u) s_warp[l][warp] = __popc(masks[l]);
    }
    __syncthreads();
    if (threadIdx.x < LISTS) {
        const uint32_t l = threadIdx.x;
        uint32_t total = 0u;
        for (int w = 0; w < BLOCK / 32; w++) {
            const uint32_t c = s_warp[l][w];
            s_warp[l][w] = total;
            total += c;
        }
        s_base[l] = total ? atomicAdd(counter(l), total) : 0u;
    }
    __syncthreads();
    const uint32_t lane_lt = (1u << lane) - 1u;
#pragma unroll
    for (uint32_t l = 0; l < LISTS; l++)
        if ((lists >> l) & 1u) store(l, s_base[l] + s_warp[l][warp] + __popc(masks[l] & lane_lt));
    __syncthreads();
}
#endif

}// namespace lrk
