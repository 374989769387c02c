// C-ABI implementation of include/lrk.h: context, scene upload, the pass scheduler and film I/O.
// Host-side scheduling replaces the reference's pass/bounce loop (src/integrators/wave_path.cpp:506-561):
// no host synchronisation inside a pass, queue sizes stay on the device.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "kernels.cuh"
#include "shade_launch.h"
#include "bvh_build.cuh"
#include "comm.cuh"
#include "adaptive.cuh"
#include "gbuffer.cuh"
#include "denoise.cuh"
#include <cub/device/device_scan.cuh>

using namespace lrk;

namespace {

// Owner of one device allocation of the context, sized exactly to the largest request so far.  reserve() keeps the allocation when
// it is large enough; otherwise it frees it before allocating the new size, so that growing a buffer never holds both (the path
// state of one pass is tens of GB).
class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(DeviceBuffer &&o) noexcept : ptr_{o.ptr_}, bytes_{o.bytes_} {
        o.ptr_ = nullptr;
        o.bytes_ = 0u;
    }
    ~DeviceBuffer() { release(); }
    cudaError_t reserve(size_t bytes) {
        if (ptr_ != nullptr && bytes_ >= bytes) return cudaSuccess;
        release();
        const cudaError_t e = cudaMalloc(&ptr_, bytes);
        if (e != cudaSuccess) ptr_ = nullptr;
        else bytes_ = bytes;
        return e;
    }
    void release() {
        if (ptr_ != nullptr) cudaFree(ptr_);
        ptr_ = nullptr;
        bytes_ = 0u;
    }
    template<typename T = void>
    T *get() const { return static_cast<T *>(ptr_); }
    size_t bytes() const { return bytes_; }

private:
    void *ptr_{nullptr};
    size_t bytes_{0u};
};

struct DeviceArrays {
    DeviceBuffer vertices, triangles, alias, pdf, meshes, inst_handles, inst_kind, inst_o2w, inst_xform, bvh_nodes, traversal_overflow, sobol, vdc, vdc_inv, pmj, blue_noise, pmj_pixels, zsobol_hash, sampler, build_scratch, mesh_bounds, inst_mesh, visible_ids, scene_copy, media, textures, texels, env_alias, env_pdf,
        tri_verts, surfaces, lights, light_handles, camera, lt_nodes, lt_light_inst, lt_trail, lt_inst_light, lt_bottom_nodes, lt_inst_bottom,
        lt_bottom_trail;
};

enum KernelCategory { CAT_TRACE_CLOSEST = 0, CAT_TRACE_SHADOW = 1, CAT_SHADE = 2, CAT_OTHER = 3, CAT_COUNT = 4 };

struct TimedLaunch {
    int cat;
    cudaEvent_t start, stop;
};

}// namespace

struct lrk_ctx {
    int device{0};
    int sm_count{0};
    cudaStream_t stream{};
    std::string error;
    bool has_scene{false};
    DeviceArrays arrays;
    DeviceScene scene{};
    uint32_t spp_hint{0};
    // sharding
    uint32_t rank{0}, world{1}, tile_size{32};
    DeviceBuffer d_pixel_list;
    uint32_t npix_owned{0};
    uint32_t pixel_list_key[6]{0, 0, 0, 0, 0, 0};// width, height, rank, world, tile size, owner-table version of the cached list
    uint32_t tile_owner_version{0};// bumped whenever tile_owner changes
    uint32_t *probe_cost{nullptr};// device counters of a running lrk_balance_shards probe
    std::vector<uint32_t> tile_owner;// lrk_balance_shards: owner of every tile (empty: the static lrk_tile_owner map)
    bool textured{false};// some surface has image-textured parameters or a normal map: the shade kernels' TEXTURED variants run
    bool any_non_opaque{false};// some instance carries LRK_SHAPE_MAYBE_NON_OPAQUE: traversal runs its alpha-testing variants
    size_t film_pixels{0};
    // path state
    uint64_t max_paths{0}, capacity{0};
    PathBuffers pb{};
    std::vector<DeviceBuffer> path_allocs;// one allocation per array of pb
    DeviceBuffer d_film, d_film_out;
    DeviceBuffer d_query_cursor;
    // options
    bool count_traversal{false}, time_kernels{false};
    bool device_bvh{false};// option device_bvh: build the hierarchy on the GPU (bvh_build.cuh) instead of uploading the host's
    double bvh_build_ms{0.0};
    const void *sampler_table_src[3]{nullptr, nullptr, nullptr};// host addresses of the static sampler tables already on the device
    bool pin_host{false};// option pin_host_buffers: page-lock the caller's scene arrays / film buffers on first sight (see pin_range)
    std::unordered_map<const void *, size_t> pinned;
    // multi-GPU film reduce (comm.cuh)
    ncclComm_t comm{nullptr};
    uint32_t comm_rank{0}, comm_world{1};
    cudaEvent_t ev_reduce_begin{}, ev_reduce_end{};
    uint32_t h_overflow{0u};// host copy of DeviceScene::traversal_overflow, fetched with every render / trace call
    // stats
    lrk_stats stats{};
    cudaEvent_t ev_begin{}, ev_end{};
    std::vector<TimedLaunch> timed;
    std::vector<cudaEvent_t> event_pool;
    int grid_trace{0}, grid_shade[2][kHitKinds]{}, grid_shadow{0}, grid_classify{0};// grid_shade[variant]: 0 = fast, 1 = strict arithmetic
    uint32_t used_kinds{1u};     // bit k: an instance of the scene has hit kind k (bit 0 always: emitter-only hits of an image emission)
    uint32_t allocated_kinds{0u};// bit k: hit_index[k] is allocated
    bool volume{false};
    bool strict_math{false};// option strict_math: every closure kernel from shade.cu's IEEE-arithmetic compilation
    bool volume_general{false};// the volume integrator's per-thread kernel (volume_general.cuh) instead of the wavefront one
    int grid_vgeneral{0};
    uint64_t volume_capacity{0};
    int grid_vshade[2][3]{}, grid_vmedium[2]{0, 0}, grid_vshadow{0};
    // adaptive mode (lrk_render_adaptive); the device buffers are allocated on its first call
    std::vector<uint32_t> block_start;// offsets of the 8x4 pixel blocks in the pixel list, closed by npix_owned (build_pixel_list)
    float2 *pass_moments{nullptr};// set while lrk_render_adaptive runs: the film accumulation also adds the luminance moments here
    DeviceBuffer d_moments;
    DeviceBuffer d_sample_counts;
    DeviceBuffer d_active[2];// ping-pong active pixel lists of the rounds after the first
    DeviceBuffer d_block_start[3];// [0]: block_start; [1], [2]: the ping-pong lists' blocks
    DeviceBuffer d_keep;// keep words and their exclusive scan (adaptive.cuh), 2 x (blocks + 1)
    DeviceBuffer d_scan_temp;
    bool adaptive_valid{false};// the film is the result of an adaptive render: sample counts and variance can be downloaded
    // G-buffer mode (option "gbuffer"): the option's value is latched into gbuffer_film at every film clear, and a G-buffer film's
    // renders add the first-hit sums (gbuffer.cuh) and the luminance moments (d_moments) until the next clear
    bool gbuffer_option{false}, gbuffer_film{false};
    DeviceBuffer d_gb_albedo, d_gb_normal, d_gb_hits;// per pixel (sum albedo, S), (sum n, sum t), H
    DeviceBuffer d_dn_albedo_cov, d_dn_normal_depth, d_dn_variance, d_dn_ping[2];// lrk_denoise / lrk_download_gbuffer scratch
    // next-event light sampling: light_requested holds the options "light_tree", "light_tree_triangles" and "light_solid_angle";
    // lrk_upload_scene latches it into light_active, which selects the shade kernels' instantiations (upload_light_sampling)
    LightSampling light_requested, light_active;

    ~lrk_ctx();
};

namespace {

int fail(lrk_ctx *ctx, int code, const std::string &msg) {
    if (ctx) ctx->error = msg;
    return code;
}

#define LRK_CUDA(call)                                                                                        \
    do {                                                                                                      \
        cudaError_t err__ = (call);                                                                           \
        if (err__ != cudaSuccess) {                                                                           \
            return fail(ctx, LRK_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(err__));            \
        }                                                                                                     \
    } while (0)

// Option `pin_host_buffers`: the caller promises that the host arrays it passes (scene arrays, film destinations) stay allocated
// until lrk_destroy or until the option is switched off; they are then page-locked once (cudaHostRegister) so that every
// later upload / download of the same buffer is a full-speed asynchronous DMA instead of a staged pageable copy.  This is
// the per-frame path of an animation or of bench.py's end-to-end leg, where the same buffers cross the bus every step.
void pin_range(lrk_ctx *ctx, const void *p, size_t bytes) {
    if (!ctx->pin_host || p == nullptr || bytes < (256u << 10)) return;
    auto it = ctx->pinned.find(p);
    if (it != ctx->pinned.end()) {
        if (it->second >= bytes) return;
        cudaHostUnregister(const_cast<void *>(p));
        ctx->pinned.erase(it);
    }
    if (cudaHostRegister(const_cast<void *>(p), bytes, cudaHostRegisterDefault) == cudaSuccess) ctx->pinned[p] = bytes;
    else cudaGetLastError();// not fatal (e.g. the range overlaps an earlier registration): the copy falls back to pageable
}

void unpin_all(lrk_ctx *ctx) {
    for (auto &kv : ctx->pinned) cudaHostUnregister(const_cast<void *>(kv.first));
    ctx->pinned.clear();
    cudaGetLastError();
}

// Host -> device copy of one scene array.  The allocation is kept across uploads when it is large enough, so
// re-uploading a scene of the same shape (the end-to-end path of bench.py, animation frames) costs only the copy.
template<typename T>
int upload(lrk_ctx *ctx, DeviceBuffer &dst, const T *src, size_t count) {
    LRK_CUDA(dst.reserve(std::max<size_t>(count * sizeof(T), 16u)));
    if (count) {
        pin_range(ctx, src, count * sizeof(T));
        LRK_CUDA(cudaMemcpyAsync(dst.get(), src, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    }
    return LRK_OK;
}

int alloc_paths(lrk_ctx *ctx, uint64_t capacity) {
    const uint32_t kinds = ctx->used_kinds | 7u;// buckets 0..2 always, the others only for scenes that use them
    if (ctx->capacity >= capacity && (!ctx->volume || ctx->volume_capacity >= capacity) && (ctx->allocated_kinds & kinds) == kinds) return LRK_OK;
    // all of the old path state is freed before any of the new one is allocated
    ctx->path_allocs.clear();
    ctx->pb = PathBuffers{};// no dangling pointers: lrk_film_clear / lrk_get_stats look at pb.stats
    ctx->capacity = 0;
    ctx->volume_capacity = 0;
    ctx->allocated_kinds = 0u;
    auto alloc = [&](auto *&p, size_t count) {
        ctx->path_allocs.emplace_back();
        const cudaError_t e = ctx->path_allocs.back().reserve(count * sizeof(*p));
        p = ctx->path_allocs.back().get<std::remove_reference_t<decltype(*p)>>();
        return e;
    };
    auto &pb = ctx->pb;
    for (int k = 0; k < 2; k++) {
        LRK_CUDA(alloc(pb.ray_o[k], capacity));
        LRK_CUDA(alloc(pb.ray_d[k], capacity));
        LRK_CUDA(alloc(pb.beta_pdf[k], capacity));
        LRK_CUDA(alloc(pb.id_rng[k], capacity));
    }
    LRK_CUDA(alloc(pb.hit, capacity));
    for (int k = 0; k < static_cast<int>(kHitKinds); k++)
        if (kinds & (1u << k)) LRK_CUDA(alloc(pb.hit_index[k], capacity));
    ctx->allocated_kinds = kinds;
    LRK_CUDA(alloc(pb.sray_o, capacity));
    LRK_CUDA(alloc(pb.sray_d, capacity));
    LRK_CUDA(alloc(pb.scontrib, capacity));
    LRK_CUDA(alloc(pb.li, capacity));
    LRK_CUDA(alloc(pb.counts, kCountSlots * kMaxDepthSlots));
    pb.capacity = static_cast<uint32_t>(capacity);
    LRK_CUDA(alloc(pb.stats, 8u));
    LRK_CUDA(cudaMemsetAsync(pb.stats, 0, 8u * sizeof(unsigned long long), ctx->stream));
    ctx->capacity = capacity;
    if (ctx->volume) {
        for (int k = 0; k < 2; k++) {
            LRK_CUDA(alloc(pb.pcg[k], capacity));
            LRK_CUDA(alloc(pb.u_rr[k], capacity));
            LRK_CUDA(alloc(pb.occl2[k], capacity));
        }
        LRK_CUDA(alloc(pb.s1ray_o, capacity));
        LRK_CUDA(alloc(pb.s1ray_d, capacity));
        LRK_CUDA(alloc(pb.occl1, capacity));
        LRK_CUDA(alloc(pb.s2_target, capacity));
        ctx->volume_capacity = capacity;
    }
    return LRK_OK;
}

// Pixel order of a shard: tiles in row-major tile order (lrk_tile_owner(tile_id, world) == rank), inside a tile 8x4
// pixel blocks so that a warp's 32 consecutive paths cover a compact screen region.
int build_pixel_list(lrk_ctx *ctx) {
    const uint32_t W = ctx->scene.width, H = ctx->scene.height, ts = ctx->tile_size;
    const uint32_t key[6]{W, H, ctx->rank, ctx->world, ts, ctx->tile_owner.empty() ? 0u : ctx->tile_owner_version};
    if (ctx->d_pixel_list.get() != nullptr && std::memcmp(key, ctx->pixel_list_key, sizeof(key)) == 0) return LRK_OK;
    std::memcpy(ctx->pixel_list_key, key, sizeof(key));
    const uint32_t tiles_x = (W + ts - 1u) / ts, tiles_y = (H + ts - 1u) / ts;
    std::vector<uint32_t> list;
    list.reserve(static_cast<size_t>(W) * H / ctx->world + 1024u);
    ctx->block_start.clear();
    for (uint32_t ty = 0; ty < tiles_y; ty++) {
        for (uint32_t tx = 0; tx < tiles_x; tx++) {
            uint32_t tile_id = ty * tiles_x + tx;
            const uint32_t owner = ctx->tile_owner.empty() ? lrk_tile_owner(tile_id, ctx->world) : ctx->tile_owner[tile_id];
            if (owner != ctx->rank) continue;
            uint32_t x0 = tx * ts, y0 = ty * ts;
            uint32_t x1 = std::min(W, x0 + ts), y1 = std::min(H, y0 + ts);
            for (uint32_t by = y0; by < y1; by += 4u)
                for (uint32_t bx = x0; bx < x1; bx += 8u) {
                    ctx->block_start.push_back(static_cast<uint32_t>(list.size()));
                    for (uint32_t y = by; y < std::min(y1, by + 4u); y++)
                        for (uint32_t x = bx; x < std::min(x1, bx + 8u); x++) list.push_back(x | (y << 16u));
                }
        }
    }
    ctx->block_start.push_back(static_cast<uint32_t>(list.size()));
    ctx->npix_owned = static_cast<uint32_t>(list.size());
    LRK_CUDA(ctx->d_pixel_list.reserve(std::max<size_t>(list.size(), 4u) * sizeof(uint32_t)));
    LRK_CUDA(cudaMemcpyAsync(ctx->d_pixel_list.get(), list.data(), list.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    return LRK_OK;
}

cudaEvent_t take_event(lrk_ctx *ctx) {
    if (!ctx->event_pool.empty()) {
        auto e = ctx->event_pool.back();
        ctx->event_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}

struct ScopedTimer {
    lrk_ctx *ctx;
    TimedLaunch t{};
    bool on;
    ScopedTimer(lrk_ctx *c, int cat) : ctx{c}, on{c->time_kernels} {
        if (on) {
            t.cat = cat;
            t.start = take_event(ctx);
            t.stop = take_event(ctx);
            cudaEventRecord(t.start, ctx->stream);
        }
    }
    ~ScopedTimer() {
        if (on) {
            cudaEventRecord(t.stop, ctx->stream);
            ctx->timed.push_back(t);
        }
    }
};

int blocks_for(lrk_ctx *ctx, uint64_t n, int persistent_grid) {
    uint64_t need = (n + kBlock - 1u) / kBlock;
    return static_cast<int>(std::max<uint64_t>(1u, std::min<uint64_t>(need, static_cast<uint64_t>(persistent_grid))));
}

// Every traversal kernel family is launched from one place, which also picks its instantiation: traversal counters (option
// count_traversal) or any-hit queries x the stochastic alpha test (scenes with non-opaque surfaces).  The kernels are named directly
// rather than through a generic lambda, so that they are instantiated in source order and the cubin's function order stays put.
void launch_query(lrk_ctx *ctx, int g, bool any_hit, const float4 *d_rays, uint4 *d_hits, uint32_t n) {
    const auto kernel = ctx->any_non_opaque ? (any_hit ? trace_query_kernel<true, true> : trace_query_kernel<false, true>)
                                            : (any_hit ? trace_query_kernel<true, false> : trace_query_kernel<false, false>);
    kernel<<<g, kTraceBlock, 0, ctx->stream>>>(ctx->scene, d_rays, d_hits, n, ctx->d_query_cursor.get<uint32_t>());
}

// stats.kernel_launches counts the kernels of lrk_render and lrk_render_adaptive (a cub call counts as one): each launch there adds
// itself where it is issued.

// The film accumulation of a pass; with the adaptive mode's moments while lrk_render_adaptive runs.
void launch_accumulate(lrk_ctx *ctx, const uint32_t *pixel_list, uint32_t pixel_offset, uint32_t npix, uint32_t spp) {
    ScopedTimer t{ctx, CAT_OTHER};
    const auto kernel = ctx->pass_moments != nullptr ? accumulate_kernel<true> : accumulate_kernel<false>;
    kernel<<<(npix + kBlock - 1u) / kBlock, kBlock, 0, ctx->stream>>>(ctx->scene, ctx->pb.li, ctx->d_film.get<float4>(), pixel_list, pixel_offset, npix, spp,
                                                                    ctx->pb.counts, ctx->pb.stats, ctx->pass_moments);
    ctx->stats.kernel_launches++;
}

// The G-buffer sums of a pass (G-buffer films only): after depth 0's closest-hit trace, while pb.hit and ray_o / ray_d[0] still hold
// the camera samples' hits and rays.
void launch_gbuffer(lrk_ctx *ctx, const uint32_t *pixel_list, uint32_t pixel_offset, uint32_t npix, uint32_t spp) {
    ScopedTimer t{ctx, CAT_OTHER};
    const auto &pb = ctx->pb;
    gbuffer_kernel<<<(npix + kBlock - 1u) / kBlock, kBlock, 0, ctx->stream>>>(ctx->scene, pb.ray_o[0], pb.ray_d[0], pb.hit, pixel_list, pixel_offset, npix, spp,
                                                                            ctx->d_gb_albedo.get<float4>(), ctx->d_gb_normal.get<float4>(),
                                                                            ctx->d_gb_hits.get<float>());
    ctx->stats.kernel_launches++;
}

// Closest-hit traversal of the path queue of `depth`.  The volume pass launches it with alpha = false: the volume integrator rejects
// non-opaque surfaces at upload.
void launch_trace_closest(lrk_ctx *ctx, bool alpha, uint64_t n, uint32_t depth) {
    ScopedTimer t{ctx, CAT_TRACE_CLOSEST};
    const auto &pb = ctx->pb;
    const bool count = ctx->count_traversal;
    const auto kernel = alpha ? (count ? trace_closest_kernel<true, true> : trace_closest_kernel<false, true>)
                              : (count ? trace_closest_kernel<true, false> : trace_closest_kernel<false, false>);
    const int in = depth & 1u;
    kernel<<<blocks_for(ctx, n, ctx->grid_trace), kTraceBlock, 0, ctx->stream>>>(ctx->scene, pb.ray_o[in], pb.ray_d[in], pb.hit, path_count(pb.counts, depth),
                                                                                 closest_cursor(pb.counts, depth), pb.stats);
    ctx->stats.kernel_launches++;
}

// One pass: sample indices [spp_begin, spp_begin + spp) of the pixels pixel_list[pixel_offset .. pixel_offset + npix).
int render_pass(lrk_ctx *ctx, const uint32_t *pixel_list, uint32_t pixel_offset, uint32_t npix, uint32_t spp_begin, uint32_t spp) {
    const uint64_t n = static_cast<uint64_t>(npix) * spp;
    auto &pb = ctx->pb;
    pb.pass_pixel_list = pixel_list;
    pb.pass_pixel_offset = pixel_offset;
    pb.pass_npix = npix;
    pb.pass_spp_begin = spp_begin;
    pb.tile_cost = ctx->probe_cost;// lrk_balance_shards' cost probe (nullptr otherwise); survives a reallocation of the path state
    pb.tile_cost_size = ctx->tile_size;
    pb.tile_cost_tiles_x = (ctx->scene.width + ctx->tile_size - 1u) / ctx->tile_size;
    const auto &sc = ctx->scene;
    {
        ScopedTimer t{ctx, CAT_OTHER};
        generate_rays_kernel<<<static_cast<unsigned>((n + kBlock - 1u) / kBlock), kBlock, 0, ctx->stream>>>(
            sc, pb, pixel_list, pixel_offset, npix, spp_begin, static_cast<uint32_t>(n));
        ctx->stats.kernel_launches++;
    }
    // upper bound of the live queue at depth d is n; launch persistent-size grids and let kernels read *count
    for (uint32_t depth = 0; depth < sc.max_depth; depth++) {
        launch_trace_closest(ctx, ctx->any_non_opaque, n, depth);
        if (depth == 0u && ctx->gbuffer_film) launch_gbuffer(ctx, pixel_list, pixel_offset, npix, spp);
        {
            ScopedTimer t{ctx, CAT_SHADE};
            if (sc.env_present) {
                shade_miss_kernel<<<blocks_for(ctx, n, ctx->grid_classify), kBlock, 0, ctx->stream>>>(sc, pb, depth);
                ctx->stats.kernel_launches++;
            }
            classify_hits_kernel<<<blocks_for(ctx, n, ctx->grid_classify), kBlock, 0, ctx->stream>>>(sc, pb, depth);
            ctx->stats.kernel_launches++;
            // one kernel per closure kind over its own hit bucket (shade.cu); TEXTURED variants only for scenes with image-textured
            // parameters / normal maps
            for (uint32_t kind = 0; kind < kHitKinds; kind++) {
                if (!(ctx->used_kinds & (1u << kind))) continue;
                const bool strict = ctx->strict_math || hit_kind_always_strict(kind);
                const int blocks = blocks_for(ctx, n, ctx->grid_shade[strict ? 1 : 0][kind]);
                if (strict) strict::launch_shade(kind, ctx->textured, ctx->light_active, blocks, ctx->stream, sc, pb, depth);
                else fast::launch_shade(kind, ctx->textured, ctx->light_active, blocks, ctx->stream, sc, pb, depth);
                ctx->stats.kernel_launches++;
            }
        }
        {
            ScopedTimer t{ctx, CAT_TRACE_SHADOW};
            const bool count = ctx->count_traversal;
            const auto kernel = ctx->any_non_opaque ? (count ? trace_shadow_kernel<true, true> : trace_shadow_kernel<false, true>)
                                                    : (count ? trace_shadow_kernel<true, false> : trace_shadow_kernel<false, false>);
            kernel<<<blocks_for(ctx, n, ctx->grid_shadow), kTraceBlock, 0, ctx->stream>>>(sc, pb, shadow_count(pb.counts, depth), shadow_cursor(pb.counts, depth));
            ctx->stats.kernel_launches++;
        }
    }
    launch_accumulate(ctx, pixel_list, pixel_offset, npix, spp);
    ctx->stats.passes++;
    LRK_CUDA(cudaGetLastError());
    return LRK_OK;
}

// One pass of the volume path integrator (config C4); schedule described in kernels.cuh.
// the general volume path: one thread per camera sample (volume_general.cuh), then the common film accumulation
int render_pass_volume_general(lrk_ctx *ctx, const uint32_t *pixel_list, uint32_t pixel_offset, uint32_t npix, uint32_t spp_begin, uint32_t spp) {
    const uint64_t n = static_cast<uint64_t>(npix) * spp;
    auto &pb = ctx->pb;
    const auto &sc = ctx->scene;
    {
        ScopedTimer t{ctx, CAT_SHADE};
        const unsigned blocks = static_cast<unsigned>((n + kGeneralBlock - 1u) / kGeneralBlock);
        const auto kernel = ctx->any_non_opaque ? volume_general_kernel<true> : volume_general_kernel<false>;
        kernel<<<blocks, kGeneralBlock, 0, ctx->stream>>>(sc, pb, pixel_list, pixel_offset, npix, spp_begin, static_cast<uint32_t>(n));
        ctx->stats.kernel_launches++;
    }
    launch_accumulate(ctx, pixel_list, pixel_offset, npix, spp);
    ctx->stats.passes++;
    LRK_CUDA(cudaGetLastError());
    return LRK_OK;
}

int render_pass_volume(lrk_ctx *ctx, const uint32_t *pixel_list, uint32_t pixel_offset, uint32_t npix, uint32_t spp_begin, uint32_t spp) {
    if (ctx->volume_general) return render_pass_volume_general(ctx, pixel_list, pixel_offset, npix, spp_begin, spp);
    const uint64_t n = static_cast<uint64_t>(npix) * spp;
    auto &pb = ctx->pb;
    const auto &sc = ctx->scene;
    {
        ScopedTimer t{ctx, CAT_OTHER};
        generate_rays_volume_kernel<<<static_cast<unsigned>((n + kBlock - 1u) / kBlock), kBlock, 0, ctx->stream>>>(
            sc, pb, pixel_list, pixel_offset, npix, spp_begin, static_cast<uint32_t>(n));
        ctx->stats.kernel_launches++;
    }
    for (uint32_t depth = 0; depth < sc.max_depth; depth++) {
        const int out = (depth & 1u) ^ 1;
        {
            ScopedTimer t{ctx, CAT_TRACE_SHADOW};
            // the in-medium shadow rays share the depth's path-queue size
            const auto kernel = ctx->count_traversal ? trace_medium_shadow_kernel<true> : trace_medium_shadow_kernel<false>;
            kernel<<<blocks_for(ctx, n, ctx->grid_vshadow), kTraceBlock, 0, ctx->stream>>>(sc, pb, path_count(pb.counts, depth), medium_shadow_cursor(pb.counts, depth));
            ctx->stats.kernel_launches++;
        }
        launch_trace_closest(ctx, false, n, depth);
        {
            ScopedTimer t{ctx, CAT_SHADE};
            const int v = ctx->strict_math ? 1 : 0;
            if (v) strict::launch_volume_medium(blocks_for(ctx, n, ctx->grid_vmedium[v]), ctx->stream, sc, pb, depth);
            else fast::launch_volume_medium(blocks_for(ctx, n, ctx->grid_vmedium[v]), ctx->stream, sc, pb, depth);
            ctx->stats.kernel_launches++;
            for (uint32_t kind = 0; kind <= kHitDisney; kind++) {
                if (!(ctx->used_kinds & (1u << kind))) continue;
                const int blocks = blocks_for(ctx, n, ctx->grid_vshade[v][kind]);
                if (v) strict::launch_volume_surface(kind, ctx->textured, blocks, ctx->stream, sc, pb, depth);
                else fast::launch_volume_surface(kind, ctx->textured, blocks, ctx->stream, sc, pb, depth);
                ctx->stats.kernel_launches++;
            }
        }
        {
            ScopedTimer t{ctx, CAT_TRACE_SHADOW};
            const auto kernel = ctx->count_traversal ? trace_volume_nee_kernel<true> : trace_volume_nee_kernel<false>;
            kernel<<<blocks_for(ctx, n, ctx->grid_vshadow), kTraceBlock, 0, ctx->stream>>>(sc, pb, shadow_count(pb.counts, depth), shadow_cursor(pb.counts, depth),
                                                                                         pb.occl2[out]);
            ctx->stats.kernel_launches++;
        }
    }
    launch_accumulate(ctx, pixel_list, pixel_offset, npix, spp);
    ctx->stats.passes++;
    LRK_CUDA(cudaGetLastError());
    return LRK_OK;
}

// Hierarchy build on the device (bvh_build.cuh): fills a.bvh_nodes / a.tri_verts from the uploaded geometry, returns the root of
// every mesh's BLAS and of the TLAS.  One round of kernels per unique mesh, one for the instances.
int build_bvh_on_device(lrk_ctx *ctx, const lrk_scene_desc *s, std::vector<uint32_t> &mesh_root, uint32_t &tlas_root) {
    auto &a = ctx->arrays;
    std::vector<uint32_t> visible, inst_mesh(s->instance_count);
    for (uint32_t i = 0; i < s->instance_count; i++) {
        inst_mesh[i] = s->instances[i].mesh;
        if (s->instances[i].visible) visible.push_back(i);
    }
    // node layout: per mesh max(n - 1, 1) nodes, then the TLAS
    mesh_root.resize(s->mesh_count);
    uint64_t nodes = 0u, max_n = std::max<uint64_t>(visible.size(), 2u);
    for (uint32_t m = 0; m < s->mesh_count; m++) {
        mesh_root[m] = static_cast<uint32_t>(nodes);
        const uint64_t n = s->meshes[m].triangle_count;
        if (n == 0u) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: mesh without triangles");
        nodes += std::max<uint64_t>(n - 1u, 1u);
        max_n = std::max(max_n, n);
    }
    tlas_root = static_cast<uint32_t>(nodes);
    nodes += std::max<uint64_t>(visible.size(), 2u) - 1u;
    if (nodes >= 0x7fffffffull || s->triangle_count >= (1ull << 28)) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: scene too large for the BVH encoding");
    int rc;
    LRK_CUDA(a.bvh_nodes.reserve(nodes * 64u));
    LRK_CUDA(a.tri_verts.reserve(std::max<uint64_t>(s->triangle_count, 1u) * 48u));
    LRK_CUDA(a.mesh_bounds.reserve(std::max<uint64_t>(s->mesh_count, 1u) * sizeof(BuildBox)));
    if ((rc = upload(ctx, a.inst_mesh, inst_mesh.data(), inst_mesh.size()))) return rc;
    if ((rc = upload(ctx, a.visible_ids, visible.data(), visible.size()))) return rc;
    // scratch: boxes, node boxes, keys / values (double buffered), radix nodes, leaf parents, visit counters, whole-set bounds, cub
    size_t cub_bytes = 0u;
    cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, static_cast<const uint32_t *>(nullptr), static_cast<uint32_t *>(nullptr),
                                    static_cast<const uint32_t *>(nullptr), static_cast<uint32_t *>(nullptr), static_cast<int>(max_n), 0, 30, ctx->stream);
    const size_t n8 = (max_n + 7u) & ~size_t{7u};
    const size_t off_boxes = 0u, off_node_boxes = off_boxes + n8 * sizeof(BuildBox), off_keys = off_node_boxes + n8 * sizeof(BuildBox),
                 off_keys2 = off_keys + n8 * 4u, off_vals = off_keys2 + n8 * 4u, off_vals2 = off_vals + n8 * 4u, off_radix = off_vals2 + n8 * 4u,
                 off_leaf_parent = off_radix + n8 * sizeof(RadixNode), off_visits = off_leaf_parent + n8 * 4u, off_whole = off_visits + n8 * 4u,
                 off_cub = off_whole + 64u, total = off_cub + cub_bytes;
    LRK_CUDA(a.build_scratch.reserve(total));
    auto base = a.build_scratch.get<char>();
    auto boxes = reinterpret_cast<BuildBox *>(base + off_boxes), node_boxes = reinterpret_cast<BuildBox *>(base + off_node_boxes);
    auto keys = reinterpret_cast<uint32_t *>(base + off_keys), keys2 = reinterpret_cast<uint32_t *>(base + off_keys2);
    auto vals = reinterpret_cast<uint32_t *>(base + off_vals), vals2 = reinterpret_cast<uint32_t *>(base + off_vals2);
    auto radix = reinterpret_cast<RadixNode *>(base + off_radix);
    auto leaf_parent = reinterpret_cast<uint32_t *>(base + off_leaf_parent), visits = reinterpret_cast<uint32_t *>(base + off_visits);
    auto whole = reinterpret_cast<uint32_t *>(base + off_whole);
    auto out_nodes = a.bvh_nodes.get<float4>();
    auto stream = ctx->stream;
    static const uint32_t whole_init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
    auto blocks = [](uint64_t n) { return static_cast<unsigned>((n + 255u) / 256u); };
    // common tail: sort, radix tree, fit, emit
    auto hierarchy = [&](uint32_t n, bool tlas, uint32_t node_base, uint32_t slot_base) -> int {
        if (n == 1u) {
            if (tlas) build_single_kernel<true><<<1, 1, 0, stream>>>(boxes, whole, a.visible_ids.get<const uint32_t>(), node_base, slot_base, out_nodes);
            else build_single_kernel<false><<<1, 1, 0, stream>>>(boxes, whole, nullptr, node_base, slot_base, out_nodes);
            LRK_CUDA(cudaMemsetAsync(vals2, 0, 4u, stream));// sorted order of one primitive
            return LRK_OK;
        }
        build_morton_kernel<<<blocks(n), 256, 0, stream>>>(boxes, n, whole, keys, vals);
        size_t bytes = cub_bytes;
        LRK_CUDA(cub::DeviceRadixSort::SortPairs(base + off_cub, bytes, keys, keys2, vals, vals2, static_cast<int>(n), 0, 30, stream));
        LRK_CUDA(cudaMemsetAsync(visits, 0, static_cast<size_t>(n) * 4u, stream));
        build_radix_tree_kernel<<<blocks(n - 1u), 256, 0, stream>>>(keys2, static_cast<int>(n), radix, leaf_parent);
        build_fit_kernel<<<blocks(n), 256, 0, stream>>>(radix, leaf_parent, vals2, boxes, static_cast<int>(n), node_boxes, visits);
        if (tlas) build_emit_kernel<true><<<blocks(n - 1u), 256, 0, stream>>>(radix, vals2, boxes, node_boxes, static_cast<int>(n), whole,
                                                                               a.visible_ids.get<const uint32_t>(), node_base, slot_base, out_nodes);
        else build_emit_kernel<false><<<blocks(n - 1u), 256, 0, stream>>>(radix, vals2, boxes, node_boxes, static_cast<int>(n), whole, nullptr, node_base,
                                                                          slot_base, out_nodes);
        LRK_CUDA(cudaGetLastError());
        return LRK_OK;
    };
    uint32_t slot_base = 0u;
    for (uint32_t m = 0; m < s->mesh_count; m++) {
        const auto &mesh = s->meshes[m];
        const uint32_t n = mesh.triangle_count;
        auto verts = a.vertices.get<const lrk_vertex>() + mesh.vertex_offset;
        auto tris = a.triangles.get<const lrk_triangle>() + mesh.triangle_offset;
        LRK_CUDA(cudaMemcpyAsync(whole, whole_init, sizeof(whole_init), cudaMemcpyHostToDevice, stream));
        build_triangle_bounds_kernel<<<blocks(n), 256, 0, stream>>>(verts, tris, n, boxes, whole);
        build_store_mesh_bounds_kernel<<<1, 1, 0, stream>>>(whole, a.mesh_bounds.get<BuildBox>(), m);
        if ((rc = hierarchy(n, false, mesh_root[m], slot_base))) return rc;
        build_tri_verts_kernel<<<blocks(n), 256, 0, stream>>>(verts, tris, vals2, n, a.tri_verts.get<float4>() + static_cast<size_t>(slot_base) * 3u);
        slot_base += n;
    }
    const uint32_t nv = static_cast<uint32_t>(visible.size());
    if (nv == 0u) {// nothing to hit: a root with two empty children
        const float inf = std::numeric_limits<float>::infinity();
        lrk_bvh_node root{};
        for (int k = 0; k < 3; k++) { root.lo0[k] = root.lo1[k] = inf; root.hi0[k] = root.hi1[k] = -inf; }
        root.ref0 = root.ref1 = root.parent = LRK_BVH_EMPTY;
        LRK_CUDA(cudaMemcpyAsync(out_nodes + static_cast<size_t>(tlas_root) * 4u, &root, sizeof(root), cudaMemcpyHostToDevice, stream));
    } else {
        LRK_CUDA(cudaMemcpyAsync(whole, whole_init, sizeof(whole_init), cudaMemcpyHostToDevice, stream));
        build_instance_bounds_kernel<<<blocks(nv), 256, 0, stream>>>(a.inst_o2w.get<const float4>(), a.inst_mesh.get<const uint32_t>(),
                                                                    a.visible_ids.get<const uint32_t>(), nv, a.mesh_bounds.get<const BuildBox>(), boxes, whole);
        if ((rc = hierarchy(nv, true, tlas_root, 0u))) return rc;
    }
    LRK_CUDA(cudaStreamSynchronize(stream));// host vectors (visible, inst_mesh) and the static init block are done with
    LRK_CUDA(cudaGetLastError());
    return LRK_OK;
}

// The triangles of `mesh`, 9 doubles each: in world space through the row-major 3x4 object-to-world matrix m, or in object space
// when m is null.
void gather_triangles(const lrk_scene_desc *s, const lrk_mesh &mesh, const float *m, std::vector<double> &tris) {
    tris.clear();
    for (uint32_t t = 0; t < mesh.triangle_count; t++) {
        const lrk_triangle &tri = s->triangles[mesh.triangle_offset + t];
        for (uint32_t v : {tri.i0, tri.i1, tri.i2}) {
            const float *p = s->vertices[mesh.vertex_offset + v].p;
            for (int r = 0; r < 3; r++)
                tris.push_back(m == nullptr ? static_cast<double>(p[r])
                                            : static_cast<double>(m[4 * r]) * p[0] + static_cast<double>(m[4 * r + 1]) * p[1] +
                                                  static_cast<double>(m[4 * r + 2]) * p[2] + m[4 * r + 3]);
        }
    }
}

// The light tree of the option "light_tree" (light_tree.h) over every instance that carries a light - not only the first light_count
// handles - from the scene's own arrays: world-space triangles, the emission (the mean of max(texel, 0) of an image emission) and the
// sidedness.  tree_inst: per tree light its instance; inst_light: per instance its tree light, kLightTreeNone for instances without
// a light or without power.
int build_light_tree(lrk_ctx *ctx, const lrk_scene_desc *s, LightTreeBuild &tree, std::vector<uint32_t> &tree_inst, std::vector<uint32_t> &inst_light) {
    std::vector<LightTreeEmitter> emitters;
    inst_light.assign(s->instance_count, kLightTreeNone);
    std::vector<double> tris;
    for (uint32_t i = 0; i < s->instance_count; i++) {
        const auto &inst = s->instances[i];
        if (!(inst.handle[0] & LRK_SHAPE_HAS_LIGHT)) continue;
        const uint32_t tag = inst.handle[1] & 4095u;
        if (tag >= s->light_count) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: light tag out of range");
        const lrk_light &light = s->lights[tag];
        double rgb[3] = {light.emission[0], light.emission[1], light.emission[2]};
        if (light.emission_tex != 0u) {
            const lrk_texture &t = s->textures[light.emission_tex - 1u];
            const size_t texels = static_cast<size_t>(t.width) * t.height;
            double sum[3] = {0.0, 0.0, 0.0};
            for (size_t k = 0; k < texels; k++)
                for (int c = 0; c < 3; c++) sum[c] += std::max(static_cast<double>(s->texels[(t.texel_offset + k) * 4u + c]), 0.0);
            for (int c = 0; c < 3; c++) rgb[c] = sum[c] / static_cast<double>(texels);
        }
        for (double &c : rgb) c = std::max(c, 0.0);
        const double lum = 0.2126 * rgb[0] + 0.7152 * rgb[1] + 0.0722 * rgb[2];
        gather_triangles(s, s->meshes[inst.mesh], inst.object_to_world, tris);
        inst_light[i] = static_cast<uint32_t>(emitters.size());
        tree_inst.push_back(i);
        emitters.push_back(light_tree_emitter(tris, lum * light.scale, light.two_sided != 0u));
    }
    tree = light_tree_build(emitters);
    for (uint32_t i = 0; i < s->instance_count; i++)
        if (inst_light[i] != kLightTreeNone && !(emitters[inst_light[i]].phi > 0.0)) inst_light[i] = kLightTreeNone;
    return LRK_OK;
}

// The bottom trees of the option "light_tree_triangles" (light_tree_build_triangles): one per distinct (mesh, side) pair among the
// instances of the top tree, shared by all of them.  nodes: the trees one after the other; inst_bottom: per instance {root, first
// trail} (2 words), root kLightTreeNone for none; trail: per tree, one trail per triangle of its mesh.
void build_bottom_light_trees(const lrk_scene_desc *s, const std::vector<uint32_t> &inst_light, std::vector<LightTreeNode> &nodes,
                              std::vector<uint32_t> &inst_bottom, std::vector<unsigned long long> &trail) {
    inst_bottom.assign(2u * s->instance_count, 0u);
    std::map<std::pair<uint32_t, uint32_t>, std::pair<uint32_t, uint32_t>> built;// (mesh, side) -> (root, first trail)
    std::vector<double> tris;
    for (uint32_t i = 0; i < s->instance_count; i++) {
        inst_bottom[2u * i] = kLightTreeNone;
        if (inst_light[i] == kLightTreeNone) continue;
        const auto &inst = s->instances[i];
        const float *m = inst.object_to_world;// row-major 3x4
        const double det = static_cast<double>(m[0]) * (static_cast<double>(m[5]) * m[10] - static_cast<double>(m[6]) * m[9]) -
                           static_cast<double>(m[1]) * (static_cast<double>(m[4]) * m[10] - static_cast<double>(m[6]) * m[8]) +
                           static_cast<double>(m[2]) * (static_cast<double>(m[4]) * m[9] - static_cast<double>(m[5]) * m[8]);
        const LightTreeSide side = s->lights[inst.handle[1] & 4095u].two_sided ? kLightTreeTwoSided : det < 0.0 ? kLightTreeMirrored : kLightTreeOneSided;
        auto it = built.find({inst.mesh, side});
        if (it == built.end()) {
            gather_triangles(s, s->meshes[inst.mesh], nullptr, tris);
            const LightTreeBuild b = light_tree_build_triangles(tris, side);
            const uint32_t root = b.nodes.empty() ? kLightTreeNone : static_cast<uint32_t>(nodes.size());
            it = built.emplace(std::make_pair(inst.mesh, static_cast<uint32_t>(side)), std::make_pair(root, static_cast<uint32_t>(trail.size()))).first;
            nodes.insert(nodes.end(), b.nodes.begin(), b.nodes.end());
            trail.insert(trail.end(), b.trail.begin(), b.trail.end());
        }
        inst_bottom[2u * i] = it->second.first;
        inst_bottom[2u * i + 1u] = it->second.second;
    }
}

// The field of LightSampling the option `name` sets, or null for another option
bool LightSampling::*light_sampling_option(const std::string &name) {
    if (name == "light_tree") return &LightSampling::tree;
    if (name == "light_tree_triangles") return &LightSampling::triangles;
    if (name == "light_solid_angle") return &LightSampling::solid_angle;
    return nullptr;
}

// lrk_upload_scene's refusals of the requested light sampling
int check_light_sampling(lrk_ctx *ctx, const lrk_scene_desc *s) {
    const LightSampling &want = ctx->light_requested;
    const bool volume = s->integrator.type == LRK_INTEGRATOR_VOLUME_PATH;
    if (want.tree && volume)
        return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: the light tree (option light_tree) serves the surface integrator only; the volume "
                                              "integrator selects its lights uniformly");
    if (want.triangles && !want.tree)
        return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: the triangle-level light trees (option light_tree_triangles) are the bottom "
                                                   "level of the light tree: set the option light_tree too");
    if (want.solid_angle && volume)
        return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: solid-angle light sampling (option light_solid_angle) serves the surface integrator "
                                              "only; the volume integrator evaluates its light pdfs from the world origin");
    if (want.candidates >= 2u && volume)
        return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: resampled next-event estimation (option light_candidates >= 2) serves the surface "
                                              "integrator only; the volume integrator traces every light sample it draws, since the "
                                              "occlusion of each advances its random stream");
    return LRK_OK;
}

// lrk_upload_scene's part for the requested light sampling, once the scene record is in a.scene_copy: builds and uploads the light
// tree and its bottom trees where requested, writes the record the kernels find them through (scene.cuh: null arrays for what is
// off) after the scene record, and latches the request into ctx->light_active.
int upload_light_sampling(lrk_ctx *ctx, const lrk_scene_desc *s) {
    const LightSampling want = ctx->light_requested;
    auto &a = ctx->arrays;
    int rc;
    DeviceLightTree rec{};
    LightTreeBuild tree;
    std::vector<uint32_t> tree_inst, inst_light;
    if (want.tree) {
        if ((rc = build_light_tree(ctx, s, tree, tree_inst, inst_light))) return rc;
        if ((rc = upload(ctx, a.lt_nodes, tree.nodes.data(), tree.nodes.size()))) return rc;
        if ((rc = upload(ctx, a.lt_light_inst, tree_inst.data(), tree_inst.size()))) return rc;
        if ((rc = upload(ctx, a.lt_trail, tree.trail.data(), tree.trail.size()))) return rc;
        if ((rc = upload(ctx, a.lt_inst_light, inst_light.data(), inst_light.size()))) return rc;
        rec.nodes = tree.nodes.empty() ? nullptr : a.lt_nodes.get<const LightTreeNode>();
        rec.light_inst = a.lt_light_inst.get<const uint32_t>();
        rec.trail = a.lt_trail.get<const unsigned long long>();
        rec.inst_light = a.lt_inst_light.get<const uint32_t>();
    }
    std::vector<LightTreeNode> bottom_nodes;
    std::vector<uint32_t> inst_bottom;
    std::vector<unsigned long long> bottom_trail;
    if (want.triangles) {
        build_bottom_light_trees(s, inst_light, bottom_nodes, inst_bottom, bottom_trail);
        if ((rc = upload(ctx, a.lt_bottom_nodes, bottom_nodes.data(), bottom_nodes.size()))) return rc;
        if ((rc = upload(ctx, a.lt_inst_bottom, inst_bottom.data(), inst_bottom.size()))) return rc;
        if ((rc = upload(ctx, a.lt_bottom_trail, bottom_trail.data(), bottom_trail.size()))) return rc;
        if (!bottom_nodes.empty()) {
            rec.bottom_nodes = a.lt_bottom_nodes.get<const LightTreeNode>();
            rec.inst_bottom = a.lt_inst_bottom.get<const uint2>();
            rec.bottom_trail = a.lt_bottom_trail.get<const unsigned long long>();
        }
    }
    rec.select = want.tree ? kLightSelectTree : kLightSelectUniform;
    rec.point = want.solid_angle ? kLightPointSolidAngle : kLightPointArea;
    rec.candidates = want.candidates;
    LRK_CUDA(cudaMemcpyAsync(a.scene_copy.get<char>() + sizeof(DeviceScene), &rec, sizeof(DeviceLightTree), cudaMemcpyHostToDevice, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));// the host arrays and `rec` are locals
    ctx->light_active = want;
    return LRK_OK;
}

}// namespace

// The one teardown of a context, run with its device current and its stream idle (lrk_destroy, or a failed lrk_create).  The device
// buffers release themselves after this body.
lrk_ctx::~lrk_ctx() {
    unpin_all(this);
    for (auto &t : timed) {
        cudaEventDestroy(t.start);
        cudaEventDestroy(t.stop);
    }
    for (auto e : event_pool) cudaEventDestroy(e);
    if (comm != nullptr) {
        lrk::nccl_api().comm_destroy(comm);
        cudaEventDestroy(ev_reduce_begin);
        cudaEventDestroy(ev_reduce_end);
    }
    if (ev_begin != nullptr) cudaEventDestroy(ev_begin);
    if (ev_end != nullptr) cudaEventDestroy(ev_end);
    if (stream != nullptr) cudaStreamDestroy(stream);
}

extern "C" {

int lrk_abi_version(void) { return static_cast<int>(LRK_ABI_VERSION); }

int lrk_create(const lrk_device_cfg *cfg, lrk_ctx **out) {
    if (!out) return LRK_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return LRK_ERR_NO_DEVICE;
    int dev = cfg ? cfg->device_index : -1;
    if (dev < 0) {
        if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
    }
    if (dev >= count || cudaSetDevice(dev) != cudaSuccess) return LRK_ERR_NO_DEVICE;
    auto ctx = std::make_unique<lrk_ctx>();// a failed creation releases what it made in ~lrk_ctx
    ctx->device = dev;
    cudaDeviceProp prop{};
    cudaGetDeviceProperties(&prop, dev);
    ctx->sm_count = prop.multiProcessorCount;
    ctx->max_paths = cfg && cfg->max_paths_per_pass ? cfg->max_paths_per_pass : (136ull << 20);
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) return LRK_ERR_CUDA;
    cudaEventCreate(&ctx->ev_begin);
    cudaEventCreate(&ctx->ev_end);
    if (ctx->d_query_cursor.reserve(64u * sizeof(uint32_t)) != cudaSuccess) return LRK_ERR_OUT_OF_MEMORY;
    auto grid_for = [&](const void *fn, int block = kBlock) {
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, block, 0);
        return std::max(1, per_sm) * ctx->sm_count;
    };
    ctx->grid_trace = grid_for(reinterpret_cast<const void *>(trace_closest_kernel<false, false>), kTraceBlock);
    ctx->grid_shadow = grid_for(reinterpret_cast<const void *>(trace_shadow_kernel<false, false>), kTraceBlock);
    for (uint32_t kind = 0; kind < kHitKinds; kind++) {
        if (!hit_kind_always_strict(kind)) ctx->grid_shade[0][kind] = fast::shade_grid(kind, ctx->sm_count);
        ctx->grid_shade[1][kind] = strict::shade_grid(kind, ctx->sm_count);
    }
    ctx->grid_classify = grid_for(reinterpret_cast<const void *>(classify_hits_kernel));
    ctx->grid_vmedium[0] = fast::volume_medium_grid(ctx->sm_count);
    ctx->grid_vmedium[1] = strict::volume_medium_grid(ctx->sm_count);
    for (uint32_t kind = 0; kind < 3u; kind++) {
        ctx->grid_vshade[0][kind] = fast::volume_surface_grid(kind, ctx->sm_count);
        ctx->grid_vshade[1][kind] = strict::volume_surface_grid(kind, ctx->sm_count);
    }
    ctx->grid_vshadow = grid_for(reinterpret_cast<const void *>(trace_volume_nee_kernel<false>), kTraceBlock);
    *out = ctx.release();
    return LRK_OK;
}

void lrk_destroy(lrk_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    delete ctx;
}

const char *lrk_last_error(const lrk_ctx *ctx) { return ctx ? ctx->error.c_str() : "null context"; }

int lrk_upload_scene(lrk_ctx *ctx, const lrk_scene_desc *s) {
    if (!ctx || !s) return LRK_ERR_INVALID_ARGUMENT;
    if (s->abi_version != LRK_ABI_VERSION) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: ABI version mismatch");
    // The volume integrator has two implementations.  The wavefront kernels (kernels.cuh) cover config C4's shape: ONE homogeneous
    // environment medium around opaque Matte / Disney closures, nothing else.  Everything beyond that - media bound to shapes,
    // transmissive surfaces, no environment medium, an environment light - runs the per-thread kernel of volume_general.cuh.
    bool volume_general = false;
    if (s->integrator.type == LRK_INTEGRATOR_VOLUME_PATH) {
        if (s->medium_count > 256u || (s->medium_count != 0u && s->media == nullptr))
            return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: invalid media table");
        if (s->environment_medium_tag != LRK_MEDIUM_INVALID_TAG && s->environment_medium_tag >= s->medium_count)
            return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: environment medium tag outside the media table");
        for (uint32_t m = 0; m < s->medium_count; m++) {
            if (s->media[m].present != LRK_MEDIUM_HOMOGENEOUS && s->media[m].present != LRK_MEDIUM_VACUUM)
                return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: unknown medium kind");
            if (s->media[m].present == LRK_MEDIUM_HOMOGENEOUS && s->media[m].eta != 1.f)
                return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: media with eta != 1 are not supported");
        }
        volume_general = !s->environment_medium.present || s->medium_count != 1u || s->environment.present;
        for (uint32_t i = 0; i < s->instance_count && !volume_general; i++)
            if (s->instances[i].handle[0] & LRK_SHAPE_HAS_MEDIUM) volume_general = true;
        for (uint32_t i = 0; i < s->surface_count && !volume_general; i++)
            if (s->surfaces[i].type > LRK_SURFACE_DISNEY || (s->surfaces[i].flags & (LRK_SURFACE_DISNEY_TRANSMISSIVE | LRK_SURFACE_DISNEY_THIN))) volume_general = true;
        for (uint32_t i = 0; i < s->instance_count; i++) {
            const uint32_t flags = s->instances[i].handle[0] & 1023u, tag = (s->instances[i].handle[1] >> 24u) & 255u;
            if ((flags & LRK_SHAPE_HAS_MEDIUM) && tag >= s->medium_count)
                return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: a shape's medium tag is outside the media table");
        }
        if (volume_general && s->sampler.type != LRK_SAMPLER_INDEPENDENT)
            return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: the volume path with shape media / transmissive surfaces takes the Independent sampler");
        if (s->integrator.max_depth > 31u) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: volume path depth > 31");
    } else if (s->integrator.type != LRK_INTEGRATOR_PATH) {
        return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: unknown integrator type");
    } else if (s->environment_medium.present) {
        return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: an environment medium needs the volume path integrator (MegaVPTNaive)");
    }
    if (s->integrator.max_depth > kMaxDepthSlots - 1u) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: max depth > 63");
    if (const int rc = check_light_sampling(ctx, s)) return rc;
    if (s->camera.resolution[0] > 65535u || s->camera.resolution[1] > 65535u)
        return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: film larger than 65535 pixels per side");
    if (s->light_count == 0u && !s->environment.present)// !pipeline().has_lighting(), wave_path.cpp:224-228
        return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "No lights in scene. Rendering aborted.");
    if (s->environment.present) {
        const auto &e = s->environment;
        if (e.emission_tex > s->texture_count || !(e.env_prob > 0.f && e.env_prob <= 1.f) ||
            (e.emission_tex != 0u && (e.map_width == 0u || e.map_height == 0u || e.alias == nullptr || e.pdf == nullptr)))
            return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: invalid environment record");
        if (s->light_count == 0u && e.env_prob != 1.f) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: env_prob must be 1 without area lights");
    }
    for (uint32_t i = 0; i < s->surface_count; i++) {
        if (s->surfaces[i].type >= LRK_SURFACE_TYPE_COUNT) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: unknown surface type");
        if (s->surfaces[i].type == LRK_SURFACE_MIX && (s->surfaces[i].flags & LRK_SURFACE_HAS_TEXTURES) && s->surfaces[i].tex[0] != 0u)
            return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: the ratio of a Mix is a constant");
        if ((s->surfaces[i].flags & LRK_SURFACE_RAW_PARAMS) && (s->surfaces[i].type < LRK_SURFACE_MIRROR || s->surfaces[i].type > LRK_SURFACE_METAL))
            return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: LRK_SURFACE_RAW_PARAMS is for Mirror / Glass / Plastic / Metal records");
        if (s->surfaces[i].type == LRK_SURFACE_LAYERED) {
            if (s->integrator.type == LRK_INTEGRATOR_VOLUME_PATH)
                return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: Layered surfaces are not supported by the volume path integrator");
            if ((s->surfaces[i].lobes >> 16u) == 0u) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: a Layered surface needs samples >= 1");
        }
        if (s->surfaces[i].type == LRK_SURFACE_MIX || s->surfaces[i].type == LRK_SURFACE_LAYERED) {
            for (uint32_t child : {s->surfaces[i].mix_a, s->surfaces[i].mix_b}) {
                if (child >= s->surface_count || s->surfaces[child].type >= LRK_SURFACE_MIX || s->surfaces[child].type == LRK_SURFACE_DISNEY ||
                    (s->surfaces[child].flags & (LRK_SURFACE_HAS_TEXTURES | LRK_SURFACE_HAS_NORMAL_MAP | LRK_SURFACE_MAYBE_NON_OPAQUE)))
                    return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: a Mix / Layered surface combines two constant Matte / Mirror / Glass / Plastic / Metal records");
            }
        }
        for (uint32_t k = 0; k < 16u; k++)
            if (s->surfaces[i].tex[k] > s->texture_count) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: texture id out of range");
        if (s->surfaces[i].opacity_tex > s->texture_count || s->surfaces[i].normal_tex > s->texture_count)
            return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: texture id out of range");
        if ((s->surfaces[i].flags & LRK_SURFACE_MAYBE_NON_OPAQUE) && s->integrator.type == LRK_INTEGRATOR_VOLUME_PATH)
            return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: non-opaque surfaces are not supported by the volume path integrator");
    }
    if (s->sampler.type > LRK_SAMPLER_ZSOBOL) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: unknown sampler type");
    if (s->sampler.type != LRK_SAMPLER_INDEPENDENT) {
        const auto &q = s->sampler;
        if (s->integrator.type == LRK_INTEGRATOR_VOLUME_PATH)
            return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_upload_scene: the volume path integrator supports the Independent sampler only");
        const bool ok = q.spp != 0u && q.sobol_matrices != nullptr &&
                        (q.type != LRK_SAMPLER_PMJ02BN || (q.pmj_samples && q.blue_noise && q.pmj_pixel_samples && q.tile != 0u && q.spp <= 65536u &&
                                                           q.pmj_pixel_sample_count == static_cast<uint64_t>(q.tile) * q.tile * q.spp)) &&
                        (q.type != LRK_SAMPLER_SOBOL || (q.vdc && q.vdc_inv && q.scale != 0u && q.scale <= 0xffffu)) &&
                        (q.type != LRK_SAMPLER_ZSOBOL || (q.zsobol_hash != nullptr && q.num_base4_digits <= 32u));
        if (!ok) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: incomplete sampler record");
    }
    ctx->textured = false;
    for (uint32_t i = 0; i < s->surface_count; i++)
        if (s->surfaces[i].flags & (LRK_SURFACE_HAS_TEXTURES | LRK_SURFACE_HAS_NORMAL_MAP)) ctx->textured = true;
    for (uint32_t i = 0; i < s->light_count; i++)
        if (s->lights[i].emission_tex != 0u) ctx->textured = true;// image emission: looked up by the TEXTURED kernel variants only
    for (uint32_t i = 0; i < s->texture_count; i++) {
        const auto &t = s->textures[i];
        if (t.width == 0u || t.height == 0u || t.texel_offset + static_cast<uint64_t>(t.width) * t.height > s->texel_count ||
            t.address > LRK_TEX_ADDRESS_ZERO || t.filter > LRK_TEX_FILTER_LINEAR || t.encoding > LRK_TEX_ENCODING_GAMMA)
            return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: invalid image texture record");
    }
    for (uint32_t i = 0; i < s->light_count; i++)
        if (s->lights[i].emission_tex > s->texture_count) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: a light's emission texture id is out of range");
    LRK_CUDA(cudaSetDevice(ctx->device));
    auto &a = ctx->arrays;
    int rc;
    if ((rc = upload(ctx, a.vertices, s->vertices, s->vertex_count))) return rc;
    if ((rc = upload(ctx, a.triangles, s->triangles, s->triangle_count))) return rc;
    if ((rc = upload(ctx, a.alias, s->alias, s->triangle_count))) return rc;
    if ((rc = upload(ctx, a.pdf, s->pdf, s->triangle_count))) return rc;
    if ((rc = upload(ctx, a.meshes, s->meshes, s->mesh_count))) return rc;
    if (!ctx->device_bvh)
        if ((rc = upload(ctx, a.bvh_nodes, s->bvh_nodes, s->bvh_node_count))) return rc;
    {
        static const uint32_t zero = 0u;
        if ((rc = upload(ctx, a.traversal_overflow, &zero, 1u))) return rc;
    }
    if (!ctx->device_bvh)
        if ((rc = upload(ctx, a.tri_verts, s->tri_verts, s->tri_slot_count * 12u))) return rc;
    if ((rc = upload(ctx, a.surfaces, s->surfaces, s->surface_count))) return rc;
    if ((rc = upload(ctx, a.textures, s->textures, s->texture_count))) return rc;
    {
        const auto &e = s->environment;
        const bool mapped = e.present && e.emission_tex != 0u;
        const size_t cells = mapped ? static_cast<size_t>(e.map_width) * e.map_height : 0u;
        if ((rc = upload(ctx, a.env_alias, e.alias, mapped ? cells + e.map_height : 0u))) return rc;
        if ((rc = upload(ctx, a.env_pdf, e.pdf, cells))) return rc;
    }
    if ((rc = upload(ctx, a.texels, s->texels, s->texel_count * 4u))) return rc;
    if ((rc = upload(ctx, a.lights, s->lights, s->light_count))) return rc;
    if ((rc = upload(ctx, a.light_handles, s->light_handles, s->light_count))) return rc;
    if ((rc = upload(ctx, a.camera, &s->camera, 1))) return rc;
    if (s->sampler.type != LRK_SAMPLER_INDEPENDENT) {
        // the static tables (213 KB / 2.6 MB / 1.5 MB) cross the bus once per context: same host address = same table
        const auto &q = s->sampler;
        if (ctx->sampler_table_src[0] != q.sobol_matrices) {
            if ((rc = upload(ctx, a.sobol, q.sobol_matrices, 1024u * 52u))) return rc;
            ctx->sampler_table_src[0] = q.sobol_matrices;
        }
        if (q.type == LRK_SAMPLER_PMJ02BN) {
            if (ctx->sampler_table_src[1] != q.pmj_samples) {
                if ((rc = upload(ctx, a.pmj, q.pmj_samples, 5u * 65536u * 2u))) return rc;
                ctx->sampler_table_src[1] = q.pmj_samples;
            }
            if (ctx->sampler_table_src[2] != q.blue_noise) {
                if ((rc = upload(ctx, a.blue_noise, q.blue_noise, 48u * 128u * 128u))) return rc;
                ctx->sampler_table_src[2] = q.blue_noise;
            }
            if ((rc = upload(ctx, a.pmj_pixels, q.pmj_pixel_samples, q.pmj_pixel_sample_count * 2u))) return rc;
        }
        if (q.type == LRK_SAMPLER_SOBOL) {
            if ((rc = upload(ctx, a.vdc, q.vdc, 52u))) return rc;
            if ((rc = upload(ctx, a.vdc_inv, q.vdc_inv, 52u))) return rc;
        }
        if (q.type == LRK_SAMPLER_ZSOBOL)
            if ((rc = upload(ctx, a.zsobol_hash, q.zsobol_hash, 2048u))) return rc;
    }
    std::vector<uint32_t> handles(static_cast<size_t>(s->instance_count) * 4u), kinds(s->instance_count);
    ctx->used_kinds = 1u;
    ctx->any_non_opaque = false;
    std::vector<float> o2w(static_cast<size_t>(s->instance_count) * 12u), xform(static_cast<size_t>(s->instance_count) * 16u);
    for (uint32_t i = 0; i < s->instance_count; i++) {
        const auto &inst = s->instances[i];
        std::memcpy(&handles[i * 4u], inst.handle, 16);
        {// closure kind of the instance: the bucket key of the material sort
            const uint32_t flags = inst.handle[0] & 1023u, surface_tag = (inst.handle[1] >> 12u) & 4095u;
            uint32_t kind = kHitEmitter;
            if (flags & LRK_SHAPE_HAS_SURFACE) {
                if (surface_tag >= s->surface_count) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: surface tag out of range");
                kind = hit_kind_of(s->surfaces[surface_tag]);
            }
            kinds[i] = kind;
            ctx->used_kinds |= 1u << kind;
            if ((flags & LRK_SHAPE_MAYBE_NON_OPAQUE) && (flags & LRK_SHAPE_HAS_SURFACE)) ctx->any_non_opaque = true;
        }
        if (inst.mesh >= s->mesh_count) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: mesh index out of range");
        std::memcpy(&o2w[i * 12u], inst.object_to_world, 48);
        std::memcpy(&xform[i * 16u], inst.world_to_object, 48);
        xform[i * 16u + 12u] = xform[i * 16u + 13u] = xform[i * 16u + 14u] = xform[i * 16u + 15u] = 0.f;
    }
    if ((rc = upload(ctx, a.inst_handles, handles.data(), handles.size()))) return rc;
    if ((rc = upload(ctx, a.inst_kind, kinds.data(), kinds.size()))) return rc;
    if ((rc = upload(ctx, a.inst_o2w, o2w.data(), o2w.size()))) return rc;
    // the hierarchy: the host's (the parity path: the oracle walks the same nodes) or one built here on the device
    std::vector<uint32_t> mesh_root(s->mesh_count);
    uint32_t tlas_root = s->tlas_root;
    if (ctx->device_bvh) {
        const auto t0 = std::chrono::steady_clock::now();
        if ((rc = build_bvh_on_device(ctx, s, mesh_root, tlas_root))) return rc;
        ctx->bvh_build_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    } else {
        for (uint32_t m = 0; m < s->mesh_count; m++) mesh_root[m] = s->meshes[m].bvh_root;
    }
    for (uint32_t i = 0; i < s->instance_count; i++) std::memcpy(&xform[i * 16u + 12u], &mesh_root[s->instances[i].mesh], 4);
    if ((rc = upload(ctx, a.inst_xform, xform.data(), xform.size()))) return rc;
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));

    auto &sc = ctx->scene;
    sc.vertices = a.vertices.get<const lrk_vertex>();
    sc.triangles = a.triangles.get<const lrk_triangle>();
    sc.alias = a.alias.get<const lrk_alias_entry>();
    sc.pdf = a.pdf.get<const float>();
    sc.meshes = a.meshes.get<const lrk_mesh>();
    sc.inst_handles = a.inst_handles.get<const uint4>();
    sc.inst_kind = a.inst_kind.get<const uint32_t>();
    sc.inst_o2w = a.inst_o2w.get<const float4>();
    sc.inst_xform = a.inst_xform.get<const float4>();
    sc.bvh_nodes = a.bvh_nodes.get<const float4>();
    sc.traversal_overflow = a.traversal_overflow.get<uint32_t>();
    sc.tri_verts = a.tri_verts.get<const float4>();
    sc.surfaces = a.surfaces.get<const lrk_surface>();
    sc.textures = a.textures.get<const lrk_texture>();
    sc.env_alias = a.env_alias.get<const lrk_alias_entry>();
    sc.env_pdf = a.env_pdf.get<const float>();
    sc.env_present = s->environment.present ? 1u : 0u;
    sc.env_emission_tex = s->environment.present ? s->environment.emission_tex : 0u;
    sc.env_map_width = s->environment.map_width;
    sc.env_map_height = s->environment.map_height;
    sc.env_scale = s->environment.scale;
    sc.env_prob = s->environment.present ? s->environment.env_prob : 0.f;
    for (int k = 0; k < 3; k++) sc.env_emission[k] = s->environment.emission[k];
    for (int k = 0; k < 9; k++) sc.env_to_world[k] = s->environment.to_world[k];
    sc.texels = a.texels.get<const float4>();
    sc.lights = a.lights.get<const lrk_light>();
    sc.light_handles = a.light_handles.get<const lrk_light_handle>();
    sc.camera = a.camera.get<const lrk_camera>();
    sc.tlas_root = tlas_root;
    sc.light_count = s->light_count;
    sc.instance_count = s->instance_count;
    sc.surface_count = s->surface_count;
    sc.max_depth = s->integrator.max_depth;
    sc.rr_depth = s->integrator.rr_depth;
    sc.rr_threshold = s->integrator.rr_threshold;
    sc.sampler_seed = s->integrator.sampler_seed;
    {// the sampler record in device memory, its table pointers replaced by the device copies
        lrk_sampler rec = s->sampler;
        rec.sobol_matrices = a.sobol.get<const uint32_t>();
        rec.vdc = a.vdc.get<const uint64_t>();
        rec.vdc_inv = a.vdc_inv.get<const uint64_t>();
        rec.pmj_samples = a.pmj.get<const uint32_t>();
        rec.blue_noise = a.blue_noise.get<const uint16_t>();
        rec.pmj_pixel_samples = a.pmj_pixels.get<const float>();
        rec.zsobol_hash = a.zsobol_hash.get<const uint32_t>();
        if ((rc = upload(ctx, a.sampler, &rec, 1))) return rc;
        LRK_CUDA(cudaStreamSynchronize(ctx->stream));// `rec` is a stack object
        sc.sampler_type = rec.type;
        sc.sampler = a.sampler.get<const lrk_sampler>();
    }
    sc.film_clamp = s->film.clamp;
    for (int i = 0; i < 3; i++) sc.film_scale[i] = s->film.scale[i];
    sc.width = s->camera.resolution[0];
    sc.height = s->camera.resolution[1];
    ctx->spp_hint = s->camera.spp;
    if (sc.refill_below == 0u) sc.refill_below = static_cast<uint32_t>(kRefillBelow);
    if (sc.inner_min == 0u) sc.inner_min = static_cast<uint32_t>(kInnerMin);
    ctx->volume = s->integrator.type == LRK_INTEGRATOR_VOLUME_PATH;
    for (int i = 0; i < 3; i++) {
        sc.sigma_a[i] = s->environment_medium.sigma_a[i];
        sc.sigma_s[i] = s->environment_medium.sigma_s[i];
    }
    sc.medium_g = s->environment_medium.g;
    sc.medium_priority = s->environment_medium.priority;
    ctx->volume_general = volume_general;
    if ((rc = upload(ctx, a.media, s->media, s->medium_count))) return rc;
    sc.media = a.media.get<const lrk_medium>();
    sc.medium_count = s->medium_count;
    sc.env_medium_tag = s->environment_medium_tag;

    const size_t npix = static_cast<size_t>(sc.width) * sc.height;
    ctx->film_pixels = 0;
    LRK_CUDA(ctx->d_film.reserve(npix * sizeof(float4)));
    LRK_CUDA(ctx->d_film_out.reserve(npix * sizeof(float4)));
    ctx->film_pixels = npix;
    {// the scene record itself in device memory, for the out-of-line device functions (DeviceScene::self), and the light tree's after it
        LRK_CUDA(a.scene_copy.reserve(sizeof(DeviceScene) + sizeof(DeviceLightTree)));
        sc.self = a.scene_copy.get<const DeviceScene>();
        LRK_CUDA(cudaMemcpyAsync(a.scene_copy.get(), &sc, sizeof(DeviceScene), cudaMemcpyHostToDevice, ctx->stream));
        if ((rc = upload_light_sampling(ctx, s))) return rc;
    }
    ctx->has_scene = true;
    // a balanced assignment stays a valid partition for any scene of the same film size (a frame loop re-uploads per frame and
    // keeps the table of the frame it probed); another film size drops it
    {
        const uint32_t ts = ctx->tile_size, tiles = ((sc.width + ts - 1u) / ts) * ((sc.height + ts - 1u) / ts);
        if (ctx->tile_owner.size() != tiles) ctx->tile_owner.clear();
    }
    if ((rc = build_pixel_list(ctx))) return rc;
    return lrk_film_clear(ctx);
}

int lrk_assign_tiles(const uint32_t *cost, uint32_t tile_count, uint32_t world, uint32_t *owner) {
    if (!cost || !owner || world == 0u) return LRK_ERR_INVALID_ARGUMENT;
    std::vector<uint32_t> order(tile_count);
    for (uint32_t t = 0; t < tile_count; t++) order[t] = t;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return cost[a] > cost[b]; });// ties keep the lower tile id first
    std::vector<uint64_t> load(world, 0u);
    for (uint32_t t : order) {
        uint32_t best = 0u;
        for (uint32_t r = 1u; r < world; r++) if (load[r] < load[best]) best = r;
        owner[t] = best;
        load[best] += cost[t];
    }
    return LRK_OK;
}

int lrk_balance_shards(lrk_ctx *ctx, uint32_t rank, uint32_t world, uint32_t tile_size, uint32_t probe_spp) {
    if (!ctx || world == 0u || rank >= world || tile_size == 0u || probe_spp == 0u)
        return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_balance_shards: invalid arguments");
    if (!ctx->has_scene) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_balance_shards: no scene");
    if (ctx->volume) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_balance_shards: the cost probe runs the surface integrator's kernels");
    LRK_CUDA(cudaSetDevice(ctx->device));
    // the probe: the whole frame on this context
    ctx->tile_owner.clear();
    int rc = lrk_set_shard(ctx, 0u, 1u, tile_size);
    if (rc) return rc;
    const uint32_t tiles_x = (ctx->scene.width + tile_size - 1u) / tile_size, tiles_y = (ctx->scene.height + tile_size - 1u) / tile_size;
    const uint32_t tile_count = tiles_x * tiles_y;
    DeviceBuffer d_cost;
    LRK_CUDA(d_cost.reserve(static_cast<size_t>(tile_count) * sizeof(uint32_t)));
    cudaMemsetAsync(d_cost.get(), 0, static_cast<size_t>(tile_count) * sizeof(uint32_t), ctx->stream);
    ctx->probe_cost = d_cost.get<uint32_t>();
    rc = lrk_render(ctx, 0u, probe_spp);
    ctx->probe_cost = nullptr;
    std::vector<uint32_t> cost(tile_count);
    if (rc == LRK_OK && cudaMemcpy(cost.data(), d_cost.get(), static_cast<size_t>(tile_count) * sizeof(uint32_t), cudaMemcpyDeviceToHost) != cudaSuccess) rc = LRK_ERR_CUDA;
    if (rc) return rc;
    std::vector<uint32_t> owner(tile_count);
    lrk_assign_tiles(cost.data(), tile_count, world, owner.data());
    ctx->tile_owner = std::move(owner);
    ctx->tile_owner_version++;
    ctx->rank = rank;
    ctx->world = world;
    ctx->tile_size = tile_size;
    if ((rc = build_pixel_list(ctx))) return rc;
    return lrk_film_clear(ctx);
}

int lrk_set_shard(lrk_ctx *ctx, uint32_t rank, uint32_t world, uint32_t tile_size) {
    if (!ctx || world == 0u || rank >= world || tile_size == 0u) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_set_shard: invalid shard");
    ctx->tile_owner.clear();
    ctx->rank = rank;
    ctx->world = world;
    ctx->tile_size = tile_size;
    if (ctx->has_scene) {
        LRK_CUDA(cudaSetDevice(ctx->device));
        return build_pixel_list(ctx);
    }
    return LRK_OK;
}

int lrk_set_option(lrk_ctx *ctx, const char *name, int64_t value) {
    if (!ctx || !name) return LRK_ERR_INVALID_ARGUMENT;
    std::string n{name};
    if (n == "count_traversal") ctx->count_traversal = value != 0;
    else if (n == "time_kernels") ctx->time_kernels = value != 0;
    else if (n == "device_bvh") ctx->device_bvh = value != 0;
    else if (n == "strict_math") ctx->strict_math = value != 0;
    else if (n == "gbuffer") ctx->gbuffer_option = value != 0;// takes effect at the next film clear
    else if (bool LightSampling::*field = light_sampling_option(n)) {// takes effect at the next lrk_upload_scene
        if (value != 0 && value != 1) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_set_option: " + n + " is 0 or 1");
        ctx->light_requested.*field = value != 0;
    } else if (n == "light_candidates") {// takes effect at the next lrk_upload_scene
        if (value < 0 || value > static_cast<int64_t>(kLightCandidatesMax))
            return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_set_option: light_candidates is 0 to 32 (0 and 1: one light sample, no resampling)");
        ctx->light_requested.candidates = static_cast<uint32_t>(value);
    }
    else if (n == "pin_host_buffers") {
        ctx->pin_host = value != 0;
        if (!ctx->pin_host) unpin_all(ctx);
    } else if (n == "max_paths_per_pass") ctx->max_paths = value > 0 ? static_cast<uint64_t>(value) : ctx->max_paths;
    else if (n == "refill_below" || n == "inner_min") {
        (n == "refill_below" ? ctx->scene.refill_below : ctx->scene.inner_min) = static_cast<uint32_t>(std::min<int64_t>(std::max<int64_t>(value, 1), 32));
        if (ctx->has_scene && ctx->arrays.scene_copy.get() != nullptr) {// keep DeviceScene::self in step
            LRK_CUDA(cudaMemcpyAsync(ctx->arrays.scene_copy.get(), &ctx->scene, sizeof(DeviceScene), cudaMemcpyHostToDevice, ctx->stream));
            LRK_CUDA(cudaStreamSynchronize(ctx->stream));
        }
    }
    else return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_set_option: unknown option '" + n + "'");
    return LRK_OK;
}

int lrk_film_clear(lrk_ctx *ctx) {
    if (!ctx || !ctx->has_scene) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_film_clear: no scene");
    LRK_CUDA(cudaSetDevice(ctx->device));
    const size_t npix = static_cast<size_t>(ctx->scene.width) * ctx->scene.height;
    LRK_CUDA(cudaMemsetAsync(ctx->d_film.get(), 0, npix * sizeof(float4), ctx->stream));
    if (ctx->pb.stats) LRK_CUDA(cudaMemsetAsync(ctx->pb.stats, 0, 8u * sizeof(unsigned long long), ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->stats = lrk_stats{};
    ctx->adaptive_valid = false;
    ctx->gbuffer_film = false;
    if (ctx->gbuffer_option) {
        LRK_CUDA(ctx->d_gb_albedo.reserve(npix * sizeof(float4)));
        LRK_CUDA(ctx->d_gb_normal.reserve(npix * sizeof(float4)));
        LRK_CUDA(ctx->d_gb_hits.reserve(npix * sizeof(float)));
        LRK_CUDA(ctx->d_moments.reserve(npix * sizeof(float2)));
        LRK_CUDA(cudaMemsetAsync(ctx->d_gb_albedo.get(), 0, npix * sizeof(float4), ctx->stream));
        LRK_CUDA(cudaMemsetAsync(ctx->d_gb_normal.get(), 0, npix * sizeof(float4), ctx->stream));
        LRK_CUDA(cudaMemsetAsync(ctx->d_gb_hits.get(), 0, npix * sizeof(float), ctx->stream));
        LRK_CUDA(cudaMemsetAsync(ctx->d_moments.get(), 0, npix * sizeof(float2), ctx->stream));
        LRK_CUDA(cudaStreamSynchronize(ctx->stream));
        ctx->gbuffer_film = true;
    }
    return LRK_OK;
}

// The film accumulation adds the luminance moments to d_moments while one of these is alive (adaptive renders, G-buffer films).
struct PassMoments {
    lrk_ctx *ctx;
    explicit PassMoments(lrk_ctx *c, bool on) : ctx{c} { ctx->pass_moments = on ? ctx->d_moments.get<float2>() : nullptr; }
    ~PassMoments() { ctx->pass_moments = nullptr; }
};

// The G-buffer is written after depth 0's trace by the surface integrator's passes only.
static int check_gbuffer_supported(lrk_ctx *ctx, bool gbuffer, const char *what) {
    if (gbuffer && ctx->volume) return fail(ctx, LRK_ERR_UNSUPPORTED, std::string(what) + ": the G-buffer mode does not support the volume integrator");
    if (gbuffer && ctx->scene.max_depth == 0u) return fail(ctx, LRK_ERR_UNSUPPORTED, std::string(what) + ": the G-buffer mode needs max_depth >= 1");
    return LRK_OK;
}

// Pass sizing of a render over npix pixels: chunks of whole pixels, one sample each, when the pixels alone exceed
// max_paths_per_pass; else all the pixels with as many samples per pixel as fit.
struct PassShape {
    uint32_t chunk_pix, spp_per_pass;
};

static PassShape pass_shape(const lrk_ctx *ctx, uint32_t npix, uint32_t total_spp) {
    const uint64_t max_paths = std::max<uint64_t>(ctx->max_paths, 1024u);
    PassShape sh{npix, 1u};
    if (npix > max_paths) sh.chunk_pix = static_cast<uint32_t>(max_paths);
    else sh.spp_per_pass = static_cast<uint32_t>(std::min<uint64_t>(total_spp, max_paths / npix));
    return sh;
}

// Sample indices [spp_begin, spp_end) of the pixels list[0 .. npix), in passes of the given shape (path state already allocated).
static int render_passes(lrk_ctx *ctx, const uint32_t *list, uint32_t npix, uint32_t spp_begin, uint32_t spp_end, PassShape sh) {
    const uint32_t total_spp = spp_end - spp_begin;
    for (uint32_t s = 0; s < total_spp; s += sh.spp_per_pass) {
        uint32_t spp = std::min(sh.spp_per_pass, total_spp - s);
        for (uint32_t p = 0; p < npix; p += sh.chunk_pix) {
            uint32_t np = std::min(sh.chunk_pix, npix - p);
            int rc = ctx->volume ? render_pass_volume(ctx, list, p, np, spp_begin + s, spp) : render_pass(ctx, list, p, np, spp_begin + s, spp);
            if (rc) return rc;
        }
    }
    return LRK_OK;
}

// The end of a render timed from ctx->ev_begin: waits for the stream, reports the kernels' overflow flags, and adds the device
// time, the kernel-category times and the samples to the stats.
static int finish_render(lrk_ctx *ctx, const std::string &what, uint64_t samples) {
    LRK_CUDA(cudaEventRecord(ctx->ev_end, ctx->stream));
    LRK_CUDA(cudaMemcpyAsync(&ctx->h_overflow, ctx->scene.traversal_overflow, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    LRK_CUDA(cudaGetLastError());
    if (ctx->h_overflow & 2u) return fail(ctx, LRK_ERR_UNSUPPORTED, what + ": a path was inside more than 8 media at once (medium tracker overflow)");
    if (ctx->h_overflow != 0u) return fail(ctx, LRK_ERR_UNSUPPORTED, what + ": traversal stack overflow (BVH deeper than the kernels support)");
    float ms = 0.f;
    LRK_CUDA(cudaEventElapsedTime(&ms, ctx->ev_begin, ctx->ev_end));
    ctx->stats.render_ms += ms;
    ctx->stats.samples += samples;
    for (auto &t : ctx->timed) {
        float kms = 0.f;
        cudaEventElapsedTime(&kms, t.start, t.stop);
        double *dst = t.cat == CAT_TRACE_CLOSEST ? &ctx->stats.trace_closest_ms :
                      t.cat == CAT_TRACE_SHADOW  ? &ctx->stats.trace_shadow_ms :
                      t.cat == CAT_SHADE         ? &ctx->stats.shade_ms :
                                                   &ctx->stats.other_ms;
        *dst += kms;
        ctx->event_pool.push_back(t.start);
        ctx->event_pool.push_back(t.stop);
    }
    ctx->timed.clear();
    return LRK_OK;
}

int lrk_render(lrk_ctx *ctx, uint32_t spp_begin, uint32_t spp_end) {
    if (!ctx || !ctx->has_scene) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_render: no scene");
    if (spp_end < spp_begin) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_render: spp_end < spp_begin");
    LRK_CUDA(cudaSetDevice(ctx->device));
    const uint32_t npix = ctx->npix_owned;
    if (npix == 0u || spp_end == spp_begin) return LRK_OK;
    int rc = check_gbuffer_supported(ctx, ctx->gbuffer_film, "lrk_render");
    if (rc) return rc;
    ctx->adaptive_valid = false;// the film no longer holds what the sample counts describe
    const PassShape sh = pass_shape(ctx, npix, spp_end - spp_begin);
    if ((rc = alloc_paths(ctx, static_cast<uint64_t>(sh.chunk_pix) * sh.spp_per_pass))) return rc;
    PassMoments moments{ctx, ctx->gbuffer_film};
    LRK_CUDA(cudaEventRecord(ctx->ev_begin, ctx->stream));
    if ((rc = render_passes(ctx, ctx->d_pixel_list.get<uint32_t>(), npix, spp_begin, spp_end, sh))) return rc;
    return finish_render(ctx, "lrk_render", static_cast<uint64_t>(npix) * (spp_end - spp_begin));
}

// Buffers of the adaptive mode, grown to the film / pixel list / block count of this context; clears the moments and counts.
static int alloc_adaptive(lrk_ctx *ctx) {
    const size_t pixels = ctx->film_pixels, list = std::max<size_t>(ctx->npix_owned, 1u), blocks = ctx->block_start.size();
    LRK_CUDA(ctx->d_moments.reserve(pixels * sizeof(float2)));
    LRK_CUDA(ctx->d_sample_counts.reserve(pixels * sizeof(uint32_t)));
    for (auto &b : ctx->d_active) LRK_CUDA(b.reserve(list * sizeof(uint32_t)));
    for (auto &b : ctx->d_block_start) LRK_CUDA(b.reserve(blocks * sizeof(uint32_t)));
    LRK_CUDA(ctx->d_keep.reserve(blocks * 2u * sizeof(unsigned long long)));
    size_t temp = 0u;
    auto keep = ctx->d_keep.get<unsigned long long>();
    cub::DeviceScan::ExclusiveSum(nullptr, temp, keep, keep + blocks, static_cast<int>(blocks), ctx->stream);
    LRK_CUDA(ctx->d_scan_temp.reserve(temp));
    LRK_CUDA(cudaMemsetAsync(ctx->d_moments.get(), 0, pixels * sizeof(float2), ctx->stream));
    LRK_CUDA(cudaMemsetAsync(ctx->d_sample_counts.get(), 0, pixels * sizeof(uint32_t), ctx->stream));
    LRK_CUDA(cudaMemcpyAsync(ctx->d_block_start[0].get(), ctx->block_start.data(), blocks * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));// block_start is pageable host memory
    return LRK_OK;
}

// Schedule and rule: include/lrk.h and DESIGN.md §4 (Adaptive sampling).  Every round renders [c, next) for the active list (pass sizing of
// lrk_render, applied to the active pixel count), then adaptive_test_kernel stops the blocks below the threshold and the rest are
// compacted into the next list; one 8-byte read-back per round tells the host how many pixels and blocks are left.
int lrk_render_adaptive(lrk_ctx *ctx, const lrk_adaptive *p) {
    if (!ctx || !ctx->has_scene) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_render_adaptive: no scene");
    if (!p || p->min_spp < 2u || p->max_spp < p->min_spp || !(p->threshold >= 0.f) || !std::isfinite(p->threshold))
        return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_render_adaptive: needs 2 <= min_spp <= max_spp and a finite threshold >= 0");
    int rc = check_gbuffer_supported(ctx, ctx->gbuffer_option, "lrk_render_adaptive");
    if (rc) return rc;
    if ((rc = lrk_film_clear(ctx))) return rc;
    if (rc) return rc;
    if ((rc = alloc_adaptive(ctx))) return rc;
    const uint32_t npix = ctx->npix_owned;
    if (npix == 0u) {
        ctx->adaptive_valid = true;
        return LRK_OK;
    }
    PassMoments moments{ctx, true};
    const uint32_t *list = ctx->d_pixel_list.get<uint32_t>();
    const uint32_t *blocks = ctx->d_block_start[0].get<uint32_t>();
    uint32_t active = npix, nblocks = static_cast<uint32_t>(ctx->block_start.size() - 1u), c = 0u, next = p->min_spp;
    unsigned long long *keep = ctx->d_keep.get<unsigned long long>(), *offsets = keep + ctx->block_start.size();
    uint64_t samples = 0u;
    bool timing = false;
    for (uint32_t round = 0u;; round++) {
        const PassShape sh = pass_shape(ctx, active, next - c);
        if ((rc = alloc_paths(ctx, static_cast<uint64_t>(sh.chunk_pix) * sh.spp_per_pass))) return rc;
        if (!timing) {
            LRK_CUDA(cudaEventRecord(ctx->ev_begin, ctx->stream));
            timing = true;
        }
        if ((rc = render_passes(ctx, list, active, c, next, sh))) return rc;
        samples += static_cast<uint64_t>(active) * (next - c);
        c = next;
        const bool last = c >= p->max_spp;
        const unsigned grid = static_cast<unsigned>((static_cast<uint64_t>(nblocks + 1u) * 32u + kAdaptiveBlock - 1u) / kAdaptiveBlock);
        adaptive_test_kernel<<<grid, kAdaptiveBlock, 0, ctx->stream>>>(ctx->scene.width, ctx->d_film.get<float4>(), ctx->d_moments.get<float2>(), list, blocks,
                                                                        nblocks, p->threshold, c, last, ctx->d_sample_counts.get<uint32_t>(), keep);
        ctx->stats.kernel_launches++;
        if (last) break;
        size_t temp = ctx->d_scan_temp.bytes();
        LRK_CUDA(cub::DeviceScan::ExclusiveSum(ctx->d_scan_temp.get(), temp, keep, offsets, static_cast<int>(nblocks + 1u), ctx->stream));
        ctx->stats.kernel_launches++;
        uint32_t *list_out = ctx->d_active[round & 1u].get<uint32_t>(), *blocks_out = ctx->d_block_start[1u + (round & 1u)].get<uint32_t>();
        adaptive_compact_kernel<<<grid, kAdaptiveBlock, 0, ctx->stream>>>(list, blocks, nblocks, keep, offsets, list_out, blocks_out);
        ctx->stats.kernel_launches++;
        LRK_CUDA(cudaGetLastError());
        unsigned long long total = 0ull;
        LRK_CUDA(cudaMemcpyAsync(&total, offsets + nblocks, sizeof(total), cudaMemcpyDeviceToHost, ctx->stream));
        LRK_CUDA(cudaStreamSynchronize(ctx->stream));
        active = static_cast<uint32_t>(total >> 32u);
        nblocks = static_cast<uint32_t>(total);
        if (active == 0u) break;
        list = list_out;
        blocks = blocks_out;
        next = static_cast<uint32_t>(std::min<uint64_t>(2ull * c, p->max_spp));
    }
    LRK_CUDA(cudaGetLastError());
    if ((rc = finish_render(ctx, "lrk_render_adaptive", samples))) return rc;
    ctx->adaptive_valid = true;
    return LRK_OK;
}

int lrk_download_sample_counts(lrk_ctx *ctx, uint32_t *counts) {
    if (!ctx || !ctx->has_scene || !counts) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_download_sample_counts: no scene / null buffer");
    if (!ctx->adaptive_valid) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_download_sample_counts: no adaptive render since the last film clear");
    LRK_CUDA(cudaSetDevice(ctx->device));
    LRK_CUDA(cudaMemcpyAsync(counts, ctx->d_sample_counts.get(), ctx->film_pixels * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    return LRK_OK;
}

int lrk_download_film_variance(lrk_ctx *ctx, float *v) {
    if (!ctx || !ctx->has_scene || !v) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_download_film_variance: no scene / null buffer");
    if (!ctx->adaptive_valid) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_download_film_variance: no adaptive render since the last film clear");
    LRK_CUDA(cudaSetDevice(ctx->device));
    const uint32_t n = static_cast<uint32_t>(ctx->film_pixels);
    float *out = ctx->d_film_out.get<float>();// the staging buffer of lrk_download_film
    adaptive_variance_kernel<<<(n + kBlock - 1u) / kBlock, kBlock, 0, ctx->stream>>>(ctx->d_film.get<float4>(), ctx->d_moments.get<float2>(),
                                                                                    ctx->d_sample_counts.get<uint32_t>(), out, n);
    LRK_CUDA(cudaGetLastError());
    LRK_CUDA(cudaMemcpyAsync(v, out, static_cast<size_t>(n) * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    return LRK_OK;
}

// The guides of lrk_download_gbuffer / lrk_denoise into the denoiser's scratch buffers.
static int gbuffer_guides(lrk_ctx *ctx, const char *what, bool zero_empty) {
    if (!ctx->gbuffer_film) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, std::string(what) + ": the film is not a G-buffer film (set the option \"gbuffer\" before the film clear)");
    const size_t n = ctx->film_pixels;
    LRK_CUDA(ctx->d_dn_albedo_cov.reserve(n * sizeof(float4)));
    LRK_CUDA(ctx->d_dn_normal_depth.reserve(n * sizeof(float4)));
    LRK_CUDA(ctx->d_dn_variance.reserve(n * sizeof(float)));
    denoise_guides_kernel<<<static_cast<unsigned>((n + kBlock - 1u) / kBlock), kBlock, 0, ctx->stream>>>(
        ctx->d_film.get<float4>(), ctx->d_moments.get<float2>(), ctx->d_gb_albedo.get<float4>(), ctx->d_gb_normal.get<float4>(), ctx->d_gb_hits.get<float>(),
        ctx->d_dn_albedo_cov.get<DenoiseVec4>(), ctx->d_dn_normal_depth.get<DenoiseVec4>(), ctx->d_dn_variance.get<float>(), static_cast<uint32_t>(n), zero_empty);
    LRK_CUDA(cudaGetLastError());
    return LRK_OK;
}

int lrk_download_gbuffer(lrk_ctx *ctx, float *albedo_cov, float *normal_depth, float *variance) {
    if (!ctx || !ctx->has_scene || !albedo_cov || !normal_depth || !variance)
        return fail(ctx, LRK_ERR_NO_SCENE, "lrk_download_gbuffer: no scene / null buffer");
    LRK_CUDA(cudaSetDevice(ctx->device));
    int rc = gbuffer_guides(ctx, "lrk_download_gbuffer", true);
    if (rc) return rc;
    const size_t n = ctx->film_pixels;
    LRK_CUDA(cudaMemcpyAsync(albedo_cov, ctx->d_dn_albedo_cov.get(), n * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaMemcpyAsync(normal_depth, ctx->d_dn_normal_depth.get(), n * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaMemcpyAsync(variance, ctx->d_dn_variance.get(), n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    return LRK_OK;
}

// Filter and schedule: denoise.h.  The film is read, never written; the output goes through lrk_download_film's staging buffer.
int lrk_denoise(lrk_ctx *ctx, float *rgba) {
    if (!ctx || !ctx->has_scene || !rgba) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_denoise: no scene / null buffer");
    LRK_CUDA(cudaSetDevice(ctx->device));
    if (!ctx->gbuffer_film) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_denoise: the film is not a G-buffer film (set the option \"gbuffer\" before the film clear)");
    if (ctx->world > 1u) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_denoise: a sharded context holds only its own tiles' G-buffer");
    int rc = gbuffer_guides(ctx, "lrk_denoise", false);
    if (rc) return rc;
    const uint32_t w = ctx->scene.width, h = ctx->scene.height, n = w * h;
    const unsigned grid = (n + kBlock - 1u) / kBlock;
    for (auto &b : ctx->d_dn_ping) LRK_CUDA(b.reserve(static_cast<size_t>(n) * sizeof(float4)));
    const auto *ac = ctx->d_dn_albedo_cov.get<const DenoiseVec4>(), *nd = ctx->d_dn_normal_depth.get<const DenoiseVec4>();
    DenoiseVec4 *ping[2] = {ctx->d_dn_ping[0].get<DenoiseVec4>(), ctx->d_dn_ping[1].get<DenoiseVec4>()};
    denoise_input_kernel<<<grid, kBlock, 0, ctx->stream>>>(ctx->scene, ctx->d_film.get<float4>(), ac, ctx->d_dn_variance.get<float>(), ping[0], n);
    for (int it = 0; it < kDenoiseIterations; it++)
        denoise_atrous_kernel<<<grid, kBlock, 0, ctx->stream>>>(ping[it & 1], ac, nd, ping[(it & 1) ^ 1], w, h, 1 << it);
    denoise_output_kernel<<<grid, kBlock, 0, ctx->stream>>>(ping[kDenoiseIterations & 1], ac, ctx->d_film_out.get<DenoiseVec4>(), n);
    LRK_CUDA(cudaGetLastError());
    pin_range(ctx, rgba, static_cast<size_t>(n) * sizeof(float4));
    LRK_CUDA(cudaMemcpyAsync(rgba, ctx->d_film_out.get(), static_cast<size_t>(n) * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    return LRK_OK;
}

static int convert_and_copy(lrk_ctx *ctx, const float4 *raw, float *rgba) {
    const uint32_t npix = ctx->scene.width * ctx->scene.height;
    convert_film_kernel<<<(npix + kBlock - 1u) / kBlock, kBlock, 0, ctx->stream>>>(ctx->scene, raw, ctx->d_film_out.get<float4>(), npix);
    LRK_CUDA(cudaGetLastError());
    pin_range(ctx, rgba, static_cast<size_t>(npix) * sizeof(float4));
    LRK_CUDA(cudaMemcpyAsync(rgba, ctx->d_film_out.get(),static_cast<size_t>(npix) * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    return LRK_OK;
}

int lrk_download_film(lrk_ctx *ctx, float *rgba) {
    if (!ctx || !ctx->has_scene || !rgba) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_download_film: no scene / null buffer");
    LRK_CUDA(cudaSetDevice(ctx->device));
    return convert_and_copy(ctx, ctx->d_film.get<float4>(), rgba);
}

int lrk_download_film_raw(lrk_ctx *ctx, float *rgba) {
    if (!ctx || !ctx->has_scene || !rgba) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_download_film_raw: no scene / null buffer");
    LRK_CUDA(cudaSetDevice(ctx->device));
    const size_t npix = static_cast<size_t>(ctx->scene.width) * ctx->scene.height;
    pin_range(ctx, rgba, npix * sizeof(float4));
    LRK_CUDA(cudaMemcpyAsync(rgba, ctx->d_film.get(), npix * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    return LRK_OK;
}

int lrk_film_device_ptr(lrk_ctx *ctx, void **ptr, uint64_t *bytes) {
    if (!ctx || !ctx->has_scene || !ptr || !bytes) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_film_device_ptr: no scene");
    *ptr = ctx->d_film.get();
    *bytes = static_cast<uint64_t>(ctx->scene.width) * ctx->scene.height * sizeof(float4);
    return LRK_OK;
}

int lrk_film_normalize_to_host(lrk_ctx *ctx, const void *device_raw, float *rgba) {
    if (!ctx || !ctx->has_scene || !device_raw || !rgba) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_film_normalize_to_host: bad argument");
    LRK_CUDA(cudaSetDevice(ctx->device));
    return convert_and_copy(ctx, static_cast<const float4 *>(device_raw), rgba);
}

int lrk_trace(lrk_ctx *ctx, const lrk_ray *rays, uint64_t n, int any_hit, lrk_hit *hits) {
    if (!ctx || !ctx->has_scene) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_trace: no scene");
    if (n == 0u) return LRK_OK;
    if (!rays || !hits || n > 0xffffffffull) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_trace: bad argument");
    LRK_CUDA(cudaSetDevice(ctx->device));
    DeviceBuffer d_rays, d_hits;
    LRK_CUDA(d_rays.reserve(n * sizeof(lrk_ray)));
    if (d_hits.reserve(n * sizeof(lrk_hit)) != cudaSuccess) return fail(ctx, LRK_ERR_OUT_OF_MEMORY, "lrk_trace: out of device memory");
    cudaMemcpyAsync(d_rays.get(), rays, n * sizeof(lrk_ray), cudaMemcpyHostToDevice, ctx->stream);
    int g = blocks_for(ctx, n, ctx->grid_trace);
    cudaMemsetAsync(ctx->d_query_cursor.get(), 0, sizeof(uint32_t), ctx->stream);
    launch_query(ctx, g, any_hit != 0, d_rays.get<float4>(), d_hits.get<uint4>(), static_cast<uint32_t>(n));
    cudaMemcpyAsync(hits, d_hits.get(), n * sizeof(lrk_hit), cudaMemcpyDeviceToHost, ctx->stream);
    cudaMemcpyAsync(&ctx->h_overflow, ctx->scene.traversal_overflow, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, LRK_ERR_CUDA, std::string("lrk_trace: ") + cudaGetErrorString(e));
    if (ctx->h_overflow != 0u) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_trace: traversal stack overflow (BVH deeper than the kernels support)");
    return LRK_OK;
}

int lrk_trace_device(lrk_ctx *ctx, const void *d_rays, uint64_t n, int any_hit, void *d_hits, uint32_t repeat, float *avg_ms) {
    if (!ctx || !ctx->has_scene) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_trace_device: no scene");
    if (!d_rays || !d_hits || n == 0u || n > 0xffffffffull || repeat == 0u) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_trace_device: bad argument");
    LRK_CUDA(cudaSetDevice(ctx->device));
    int g = blocks_for(ctx, n, ctx->grid_trace);
    LRK_CUDA(cudaEventRecord(ctx->ev_begin, ctx->stream));
    for (uint32_t r = 0; r < repeat; r++) {
        LRK_CUDA(cudaMemsetAsync(ctx->d_query_cursor.get(), 0, sizeof(uint32_t), ctx->stream));
        launch_query(ctx, g, any_hit != 0, static_cast<const float4 *>(d_rays), static_cast<uint4 *>(d_hits), static_cast<uint32_t>(n));
    }
    LRK_CUDA(cudaEventRecord(ctx->ev_end, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    LRK_CUDA(cudaGetLastError());
    float ms = 0.f;
    LRK_CUDA(cudaEventElapsedTime(&ms, ctx->ev_begin, ctx->ev_end));
    if (avg_ms) *avg_ms = ms / static_cast<float>(repeat);
    return LRK_OK;
}

int lrk_comm_unique_id(uint8_t *id) {
    if (id == nullptr) return LRK_ERR_INVALID_ARGUMENT;
    static_assert(sizeof(ncclUniqueId) == LRK_COMM_ID_BYTES, "LRK_COMM_ID_BYTES must be NCCL's unique id size");
    auto &api = lrk::nccl_api();
    if (!api.error.empty()) return LRK_ERR_UNSUPPORTED;
    ncclUniqueId uid;
    if (api.get_unique_id(&uid) != ncclSuccess) return LRK_ERR_CUDA;
    std::memcpy(id, &uid, sizeof(uid));
    return LRK_OK;
}

int lrk_comm_init(lrk_ctx *ctx, const uint8_t *id, uint32_t rank, uint32_t world) {
    if (!ctx || !id || world == 0u || rank >= world) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_comm_init: bad arguments");
    auto &api = lrk::nccl_api();
    if (!api.error.empty()) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_comm_init: " + api.error);
    LRK_CUDA(cudaSetDevice(ctx->device));
    if (ctx->comm != nullptr) {
        api.comm_destroy(ctx->comm);
        ctx->comm = nullptr;
    } else {
        LRK_CUDA(cudaEventCreate(&ctx->ev_reduce_begin));
        LRK_CUDA(cudaEventCreate(&ctx->ev_reduce_end));
    }
    ncclUniqueId uid;
    std::memcpy(&uid, id, sizeof(uid));
    ncclResult_t r = api.comm_init_rank(&ctx->comm, static_cast<int>(world), uid, static_cast<int>(rank));
    if (r != ncclSuccess) {
        ctx->comm = nullptr;
        cudaEventDestroy(ctx->ev_reduce_begin);
        cudaEventDestroy(ctx->ev_reduce_end);
        return fail(ctx, LRK_ERR_CUDA, std::string("lrk_comm_init: ncclCommInitRank: ") + api.error_string(r));
    }
    ctx->comm_rank = rank;
    ctx->comm_world = world;
    return LRK_OK;
}

int lrk_reduce_film(lrk_ctx *ctx, uint32_t root) {
    if (!ctx || !ctx->has_scene) return fail(ctx, LRK_ERR_NO_SCENE, "lrk_reduce_film: no scene");
    if (ctx->comm == nullptr) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_reduce_film: lrk_comm_init was not called");
    if (root >= ctx->comm_world) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_reduce_film: root outside the communicator");
    LRK_CUDA(cudaSetDevice(ctx->device));
    auto &api = lrk::nccl_api();
    const size_t count = static_cast<size_t>(ctx->scene.width) * ctx->scene.height * 4u;
    LRK_CUDA(cudaEventRecord(ctx->ev_reduce_begin, ctx->stream));
    ncclResult_t r = api.reduce(ctx->d_film.get(), ctx->d_film.get(), count, ncclFloat, ncclSum, static_cast<int>(root), ctx->comm, ctx->stream);
    if (r != ncclSuccess) return fail(ctx, LRK_ERR_CUDA, std::string("lrk_reduce_film: ncclReduce: ") + api.error_string(r));
    LRK_CUDA(cudaEventRecord(ctx->ev_reduce_end, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    float ms = 0.f;
    LRK_CUDA(cudaEventElapsedTime(&ms, ctx->ev_reduce_begin, ctx->ev_reduce_end));
    ctx->stats.reduce_ms += ms;
    return LRK_OK;
}

int lrk_get_stats(lrk_ctx *ctx, lrk_stats *stats) {
    if (!ctx || !stats) return LRK_ERR_INVALID_ARGUMENT;
    LRK_CUDA(cudaSetDevice(ctx->device));
    if (ctx->pb.stats) {
        unsigned long long h[8]{};
        LRK_CUDA(cudaMemcpy(h, ctx->pb.stats, sizeof(h), cudaMemcpyDeviceToHost));
        ctx->stats.closest_rays = h[0];
        ctx->stats.shadow_rays = h[1];
        ctx->stats.closest_nodes = h[2];
        ctx->stats.closest_tris = h[3];
        ctx->stats.closest_xforms = h[4];
        ctx->stats.shadow_nodes = h[5];
        ctx->stats.shadow_tris = h[6];
        ctx->stats.shadow_xforms = h[7];
    }
    *stats = ctx->stats;
    return LRK_OK;
}

void *lrk_stream(lrk_ctx *ctx) { return ctx ? static_cast<void *>(ctx->stream) : nullptr; }

}// extern "C"
