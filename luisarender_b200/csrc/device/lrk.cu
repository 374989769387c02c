// C-ABI implementation of include/lrk.h: context, scene upload, the pass scheduler and film I/O.
// Host-side scheduling replaces the reference's pass/bounce loop (src/integrators/wave_path.cpp:506-561):
// no host synchronisation inside a pass, queue sizes stay on the device.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstddef>
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
#include "affine_inverse.h"
#include "alias_table.h"
#include "scene_check.h"
#include <cub/device/device_scan.cuh>

using namespace lrk;

static_assert(kMaxDepth + 1u == kMaxDepthSlots, "check_scene_desc refuses the depths that have no counter slot");

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
    void swap(DeviceBuffer &o) noexcept {
        std::swap(ptr_, o.ptr_);
        std::swap(bytes_, o.bytes_);
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
        lt_bottom_trail, update_staging, mesh_staging, mesh_refit, refit_starts, refit_scratch, refit_visits, node_runs;
};

// CAT_NONE: counted in stats.kernel_launches, never timed
enum KernelCategory { CAT_NONE = -1, CAT_TRACE_CLOSEST = 0, CAT_TRACE_SHADOW = 1, CAT_SHADE = 2, CAT_OTHER = 3 };

struct TimedLaunch {
    int cat;
    cudaEvent_t start, stop;
};

// The persistent grid of every kernel that a pass launches over a path queue (blocks_for caps the launch there): resident blocks per
// SM x SM count, measured by measure_grids at lrk_create so that no occupancy query runs inside a timed render.  Each grid is
// measured on the kernel's untextured, uniform/area, non-counting, non-alpha instantiation and launches all of its instantiations.
// [v]: 0 = fast, 1 = strict arithmetic (shade.cu).
struct Grids {
    int closest, query, shadow, classify, miss, shade[2][kHitKinds];
    int medium_shadow, volume_medium[2], volume_surface[2][3], volume_nee;
};

// The host state of the uploaded scene that the scene updates (lrk_update_*, lrk_replace_meshes) read and keep, set whole by
// lrk_upload_scene.  Every update rebuilds the instance level of the hierarchy on the device from the per-instance meshes and the
// visible instances.  Mesh updates and replacements keep the current mesh table and, per mesh, whether an instance with a light
// uses it; derived on a mesh's first update and kept until the next upload or replacement: its refit's start nodes (the reachable
// inner nodes of its hierarchy without inner children) at refit_start[m] in a.refit_starts, and an emissive mesh's triangles.
struct SceneUpdateState {
    std::vector<uint32_t> inst_mesh_host, visible_host;// per instance its mesh; the visible instances in order
    uint32_t mesh_count{0};
    uint64_t bvh_node_count{0};// of the current hierarchy, whose last max(visible, 2) - 1 nodes are the instance level
    bool tlas_inputs{false};// a.inst_mesh, a.visible_ids and a.mesh_bounds hold the scene's (device_bvh, or since the first update)
    std::vector<lrk_mesh> meshes_host;
    std::vector<uint8_t> mesh_emissive;
    std::vector<uint32_t> refit_starts_host;
    std::vector<std::pair<uint32_t, uint32_t>> refit_start;// (first, count); count 0: not derived yet
    std::map<uint32_t, std::vector<lrk_triangle>> emissive_triangles;
    LightTreeSource light_source;// while light_active.tree
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
    uint32_t sampler_spp{0};// lrk_sampler::spp of the uploaded scene: the table-driven samplers take the sample indices [0, spp)
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
    Grids grids{};
    uint32_t used_kinds{1u};     // bit k: an instance of the scene has hit kind k (bit 0 always: emitter-only hits of an image emission)
    uint32_t allocated_kinds{0u};// bit k: hit_index[k] is allocated
    bool volume{false};
    bool strict_math{false};// option strict_math: every closure kernel from shade.cu's IEEE-arithmetic compilation
    bool volume_general{false};// the volume integrator's per-thread kernel (volume_general.cuh) instead of the wavefront one
    uint64_t volume_capacity{0};
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
    // next-event light sampling: light_requested holds the options "light_tree", "light_tree_triangles", "light_solid_angle",
    // "light_candidates" and "light_receiver"; lrk_upload_scene latches it into light_active, which selects the shade kernels'
    // instantiations (upload_light_sampling)
    LightSampling light_requested, light_active;
    uint32_t *receiver_words{nullptr};// in path_allocs while light_active.receiver (alloc_paths)
    SceneUpdateState update;

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

// The receiver words' pointer in the record after the scene (DeviceLightTree::receiver): the path array while the option
// "light_receiver" is active, else null.
int write_receiver_record(lrk_ctx *ctx) {
    if (ctx->arrays.scene_copy.get() == nullptr) return LRK_OK;
    uint32_t *words = ctx->light_active.receiver ? ctx->receiver_words : nullptr;
    LRK_CUDA(cudaMemcpyAsync(ctx->arrays.scene_copy.get<char>() + sizeof(DeviceScene) + offsetof(DeviceLightTree, receiver), &words, sizeof(words),
                             cudaMemcpyHostToDevice, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));// `words` is a local
    return LRK_OK;
}

int alloc_paths(lrk_ctx *ctx, uint64_t capacity) {
    const uint32_t kinds = ctx->used_kinds | 7u;// buckets 0..2 always, the others only for scenes that use them
    if (ctx->capacity >= capacity && (!ctx->volume || ctx->volume_capacity >= capacity) && (ctx->allocated_kinds & kinds) == kinds &&
        (!ctx->light_active.receiver || ctx->receiver_words != nullptr))
        return LRK_OK;
    // all of the old path state is freed before any of the new one is allocated
    ctx->path_allocs.clear();
    ctx->pb = PathBuffers{};// no dangling pointers: lrk_film_clear / lrk_get_stats look at pb.stats
    ctx->receiver_words = nullptr;
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
    if (ctx->light_active.receiver) {// only while the option is active; the kernels find them through the scene's record
        LRK_CUDA(alloc(ctx->receiver_words, capacity));
        return write_receiver_record(ctx);
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

// A stage of a pass: launches its kernels on ctx->stream and counts each in stats.kernel_launches (stats.kernel_launches counts the
// kernels of lrk_render and lrk_render_adaptive: a cub call there counts itself as one).  With the option time_kernels a stage with
// a category is one timed interval, the gaps between its kernels included.  A stage of one launch can be a temporary:
// Stage(ctx, CAT_OTHER).launch(...) records its end after the launch.
class Stage {
public:
    Stage(lrk_ctx *ctx, int cat) : ctx_{ctx}, on_{cat != CAT_NONE && ctx->time_kernels} {
        if (on_) {
            t_.cat = cat;
            t_.start = take_event(ctx_);
            t_.stop = take_event(ctx_);
            cudaEventRecord(t_.start, ctx_->stream);
        }
    }
    ~Stage() {
        if (on_) {
            cudaEventRecord(t_.stop, ctx_->stream);
            ctx_->timed.push_back(t_);
        }
    }
    template<typename... Params, typename... Args>
    void launch(void (*kernel)(Params...), unsigned blocks, int block, Args &&...args) {
        kernel<<<blocks, block, 0, ctx_->stream>>>(std::forward<Args>(args)...);
        ctx_->stats.kernel_launches++;
    }

private:
    lrk_ctx *ctx_;
    bool on_;
    TimedLaunch t_{};
};

int blocks_for(lrk_ctx *ctx, uint64_t n, int grid) {
    uint64_t need = (n + kBlock - 1u) / kBlock;
    return static_cast<int>(std::max<uint64_t>(1u, std::min<uint64_t>(need, static_cast<uint64_t>(grid))));
}

// The instantiation of every kernel template that lrk.cu launches, picked from the context's flags: any-hit queries, traversal
// counters (option count_traversal), the stochastic alpha test (scenes with non-opaque surfaces) and the film accumulation's
// luminance moments (adaptive renders, G-buffer films).  The kernels are named directly rather than through a generic lambda, so
// that they are instantiated in source order and the cubin's function order stays put.
auto query_kernel(const lrk_ctx *ctx, bool any_hit) {
    return ctx->any_non_opaque ? (any_hit ? trace_query_kernel<true, true> : trace_query_kernel<false, true>)
                               : (any_hit ? trace_query_kernel<true, false> : trace_query_kernel<false, false>);
}
auto accumulation_kernel(const lrk_ctx *ctx) { return ctx->pass_moments != nullptr ? accumulate_kernel<true> : accumulate_kernel<false>; }
auto closest_kernel(const lrk_ctx *ctx, bool alpha) {
    return alpha ? (ctx->count_traversal ? trace_closest_kernel<true, true> : trace_closest_kernel<false, true>)
                 : (ctx->count_traversal ? trace_closest_kernel<true, false> : trace_closest_kernel<false, false>);
}
auto shadow_kernel(const lrk_ctx *ctx) {
    return ctx->any_non_opaque ? (ctx->count_traversal ? trace_shadow_kernel<true, true> : trace_shadow_kernel<false, true>)
                               : (ctx->count_traversal ? trace_shadow_kernel<true, false> : trace_shadow_kernel<false, false>);
}
auto general_kernel(const lrk_ctx *ctx) { return ctx->any_non_opaque ? volume_general_kernel<true> : volume_general_kernel<false>; }
auto medium_shadow_kernel(const lrk_ctx *ctx) { return ctx->count_traversal ? trace_medium_shadow_kernel<true> : trace_medium_shadow_kernel<false>; }
auto volume_nee_kernel(const lrk_ctx *ctx) { return ctx->count_traversal ? trace_volume_nee_kernel<true> : trace_volume_nee_kernel<false>; }

// lrk_trace / lrk_trace_device: not a render's kernel, so not counted
void launch_query(lrk_ctx *ctx, bool any_hit, const float4 *d_rays, uint4 *d_hits, uint32_t n) {
    query_kernel(ctx, any_hit)<<<blocks_for(ctx, n, ctx->grids.query), kTraceBlock, 0, ctx->stream>>>(ctx->scene, d_rays, d_hits, n,
                                                                                                      ctx->d_query_cursor.get<uint32_t>());
}

// Closest-hit traversal of the path queue of `depth`.  The volume pass launches it with alpha = false: the volume integrator rejects
// non-opaque surfaces at upload.
void launch_trace_closest(lrk_ctx *ctx, bool alpha, uint64_t n, uint32_t depth) {
    const auto &pb = ctx->pb;
    const int in = depth & 1u;
    Stage(ctx, CAT_TRACE_CLOSEST).launch(closest_kernel(ctx, alpha), blocks_for(ctx, n, ctx->grids.closest), kTraceBlock, ctx->scene, pb.ray_o[in],
                                         pb.ray_d[in], pb.hit, path_count(pb.counts, depth), closest_cursor(pb.counts, depth), pb.stats);
}

// The end of every pass: the film accumulation, with the adaptive mode's moments while lrk_render_adaptive runs.
int finish_pass(lrk_ctx *ctx, const uint32_t *pixel_list, uint32_t pixel_offset, uint32_t npix, uint32_t spp) {
    Stage(ctx, CAT_OTHER).launch(accumulation_kernel(ctx), (npix + kBlock - 1u) / kBlock, kBlock, ctx->scene, ctx->pb.li, ctx->d_film.get<float4>(),
                                 pixel_list, pixel_offset, npix, spp, ctx->pb.counts, ctx->pb.stats, ctx->pass_moments);
    ctx->stats.passes++;
    LRK_CUDA(cudaGetLastError());
    return LRK_OK;
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
    const auto &grids = ctx->grids;
    Stage(ctx, CAT_OTHER).launch(generate_rays_kernel, static_cast<unsigned>((n + kBlock - 1u) / kBlock), kBlock, sc, pb, pixel_list, pixel_offset,
                                 npix, spp_begin, static_cast<uint32_t>(n));
    // upper bound of the live queue at depth d is n; launch persistent-size grids and let kernels read *count
    for (uint32_t depth = 0; depth < sc.max_depth; depth++) {
        launch_trace_closest(ctx, ctx->any_non_opaque, n, depth);
        // the G-buffer sums (G-buffer films only): pb.hit and ray_o / ray_d[0] still hold the camera samples' hits and rays
        if (depth == 0u && ctx->gbuffer_film)
            Stage(ctx, CAT_OTHER).launch(gbuffer_kernel, (npix + kBlock - 1u) / kBlock, kBlock, sc, pb.ray_o[0], pb.ray_d[0], pb.hit, pixel_list,
                                         pixel_offset, npix, spp, ctx->d_gb_albedo.get<float4>(), ctx->d_gb_normal.get<float4>(),
                                         ctx->d_gb_hits.get<float>());
        {
            Stage shade{ctx, CAT_SHADE};
            if (sc.env_present) shade.launch(shade_miss_kernel, blocks_for(ctx, n, grids.miss), kBlock, sc, pb, depth);
            shade.launch(classify_hits_kernel, blocks_for(ctx, n, grids.classify), kBlock, sc, pb, depth);
            // one kernel per closure kind over its own hit bucket (shade.cu); TEXTURED variants only for scenes with image-textured
            // parameters / normal maps
            for (uint32_t kind = 0; kind < kHitKinds; kind++) {
                if (!(ctx->used_kinds & (1u << kind))) continue;
                const bool strict = ctx->strict_math || hit_kind_always_strict(kind);
                const ShadeKernel kernel = strict ? strict::shade_kernel_for(kind, ctx->textured, ctx->light_active)
                                                  : fast::shade_kernel_for(kind, ctx->textured, ctx->light_active);
                shade.launch(kernel, blocks_for(ctx, n, grids.shade[strict][kind]), kShadeBlock, sc, pb, depth);
            }
        }
        Stage(ctx, CAT_TRACE_SHADOW).launch(shadow_kernel(ctx), blocks_for(ctx, n, grids.shadow), kTraceBlock, sc, pb, shadow_count(pb.counts, depth),
                                            shadow_cursor(pb.counts, depth));
    }
    return finish_pass(ctx, pixel_list, pixel_offset, npix, spp);
}

// One pass of the volume path integrator.  Media bound to shapes and the other scenes beyond config C4 (SceneCheck::volume_general):
// one thread per camera sample (volume_general.cuh).  Config C4: the wavefront schedule described in kernels.cuh.
int render_pass_volume(lrk_ctx *ctx, const uint32_t *pixel_list, uint32_t pixel_offset, uint32_t npix, uint32_t spp_begin, uint32_t spp) {
    const uint64_t n = static_cast<uint64_t>(npix) * spp;
    auto &pb = ctx->pb;
    const auto &sc = ctx->scene;
    const auto &grids = ctx->grids;
    if (ctx->volume_general) {
        Stage(ctx, CAT_SHADE).launch(general_kernel(ctx), static_cast<unsigned>((n + kGeneralBlock - 1u) / kGeneralBlock), kGeneralBlock, sc, pb,
                                     pixel_list, pixel_offset, npix, spp_begin, static_cast<uint32_t>(n));
        return finish_pass(ctx, pixel_list, pixel_offset, npix, spp);
    }
    Stage(ctx, CAT_OTHER).launch(generate_rays_volume_kernel, static_cast<unsigned>((n + kBlock - 1u) / kBlock), kBlock, sc, pb, pixel_list,
                                 pixel_offset, npix, spp_begin, static_cast<uint32_t>(n));
    for (uint32_t depth = 0; depth < sc.max_depth; depth++) {
        const int out = (depth & 1u) ^ 1;
        // the in-medium shadow rays share the depth's path-queue size
        Stage(ctx, CAT_TRACE_SHADOW).launch(medium_shadow_kernel(ctx), blocks_for(ctx, n, grids.medium_shadow), kTraceBlock, sc, pb,
                                            path_count(pb.counts, depth), medium_shadow_cursor(pb.counts, depth));
        launch_trace_closest(ctx, false, n, depth);
        {
            Stage shade{ctx, CAT_SHADE};
            const int v = ctx->strict_math ? 1 : 0;
            const ShadeKernel medium = v ? strict::volume_medium_kernel_for() : fast::volume_medium_kernel_for();
            shade.launch(medium, blocks_for(ctx, n, grids.volume_medium[v]), kBlock, sc, pb, depth);
            for (uint32_t kind = 0; kind <= kHitDisney; kind++) {
                if (!(ctx->used_kinds & (1u << kind))) continue;
                const ShadeKernel kernel = v ? strict::volume_surface_kernel_for(kind, ctx->textured)
                                             : fast::volume_surface_kernel_for(kind, ctx->textured);
                shade.launch(kernel, blocks_for(ctx, n, grids.volume_surface[v][kind]), kBlock, sc, pb, depth);
            }
        }
        Stage(ctx, CAT_TRACE_SHADOW).launch(volume_nee_kernel(ctx), blocks_for(ctx, n, grids.volume_nee), kTraceBlock, sc, pb,
                                            shadow_count(pb.counts, depth), shadow_cursor(pb.counts, depth), pb.occl2[out]);
    }
    return finish_pass(ctx, pixel_list, pixel_offset, npix, spp);
}

// Scratch of the device hierarchy build (bvh_build.cuh) for sets of at most max_n primitives, carved out of a.build_scratch: boxes,
// node boxes, keys / values (double buffered), radix nodes, leaf parents, visit counters, whole-set bounds, cub's temporary storage.
struct BuildScratch {
    BuildBox *boxes, *node_boxes;
    uint32_t *keys, *keys2, *vals, *vals2;
    RadixNode *radix;
    uint32_t *leaf_parent, *visits, *whole;
    void *cub;
    size_t cub_bytes;
};

int reserve_build_scratch(lrk_ctx *ctx, uint64_t max_n, BuildScratch &b) {
    size_t cub_bytes = 0u;
    cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, static_cast<const uint32_t *>(nullptr), static_cast<uint32_t *>(nullptr),
                                    static_cast<const uint32_t *>(nullptr), static_cast<uint32_t *>(nullptr), static_cast<int>(max_n), 0, 30, ctx->stream);
    const size_t n8 = (max_n + 7u) & ~size_t{7u};
    const size_t off_boxes = 0u, off_node_boxes = off_boxes + n8 * sizeof(BuildBox), off_keys = off_node_boxes + n8 * sizeof(BuildBox),
                 off_keys2 = off_keys + n8 * 4u, off_vals = off_keys2 + n8 * 4u, off_vals2 = off_vals + n8 * 4u, off_radix = off_vals2 + n8 * 4u,
                 off_leaf_parent = off_radix + n8 * sizeof(RadixNode), off_visits = off_leaf_parent + n8 * 4u, off_whole = off_visits + n8 * 4u,
                 off_cub = off_whole + 64u, total = off_cub + cub_bytes;
    LRK_CUDA(ctx->arrays.build_scratch.reserve(total));
    auto base = ctx->arrays.build_scratch.get<char>();
    b.boxes = reinterpret_cast<BuildBox *>(base + off_boxes);
    b.node_boxes = reinterpret_cast<BuildBox *>(base + off_node_boxes);
    b.keys = reinterpret_cast<uint32_t *>(base + off_keys);
    b.keys2 = reinterpret_cast<uint32_t *>(base + off_keys2);
    b.vals = reinterpret_cast<uint32_t *>(base + off_vals);
    b.vals2 = reinterpret_cast<uint32_t *>(base + off_vals2);
    b.radix = reinterpret_cast<RadixNode *>(base + off_radix);
    b.leaf_parent = reinterpret_cast<uint32_t *>(base + off_leaf_parent);
    b.visits = reinterpret_cast<uint32_t *>(base + off_visits);
    b.whole = reinterpret_cast<uint32_t *>(base + off_whole);
    b.cub = base + off_cub;
    b.cub_bytes = cub_bytes;
    return LRK_OK;
}

const uint32_t kWholeInit[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};// empty whole-set bounds (bvh_build.cuh: grow_whole)

unsigned build_blocks(uint64_t n) { return static_cast<unsigned>((n + 255u) / 256u); }

// The common tail of every hierarchy over the n boxes in b.boxes (whole-set bounds in b.whole): sort, radix tree, fit, emit.
int build_hierarchy(lrk_ctx *ctx, const BuildScratch &b, uint32_t n, bool tlas, uint32_t node_base, uint32_t slot_base) {
    auto &a = ctx->arrays;
    auto out_nodes = a.bvh_nodes.get<float4>();
    auto stream = ctx->stream;
    if (n == 1u) {
        if (tlas) build_single_kernel<true><<<1, 1, 0, stream>>>(b.boxes, b.whole, a.visible_ids.get<const uint32_t>(), node_base, slot_base, out_nodes);
        else build_single_kernel<false><<<1, 1, 0, stream>>>(b.boxes, b.whole, nullptr, node_base, slot_base, out_nodes);
        LRK_CUDA(cudaMemsetAsync(b.vals2, 0, 4u, stream));// sorted order of one primitive
        return LRK_OK;
    }
    build_morton_kernel<<<build_blocks(n), 256, 0, stream>>>(b.boxes, n, b.whole, b.keys, b.vals);
    size_t bytes = b.cub_bytes;
    LRK_CUDA(cub::DeviceRadixSort::SortPairs(b.cub, bytes, b.keys, b.keys2, b.vals, b.vals2, static_cast<int>(n), 0, 30, stream));
    LRK_CUDA(cudaMemsetAsync(b.visits, 0, static_cast<size_t>(n) * 4u, stream));
    build_radix_tree_kernel<<<build_blocks(n - 1u), 256, 0, stream>>>(b.keys2, static_cast<int>(n), b.radix, b.leaf_parent);
    build_fit_kernel<<<build_blocks(n), 256, 0, stream>>>(b.radix, b.leaf_parent, b.vals2, b.boxes, static_cast<int>(n), b.node_boxes, b.visits);
    if (tlas) build_emit_kernel<true><<<build_blocks(n - 1u), 256, 0, stream>>>(b.radix, b.vals2, b.boxes, b.node_boxes, static_cast<int>(n), b.whole,
                                                                                 a.visible_ids.get<const uint32_t>(), node_base, slot_base, out_nodes);
    else build_emit_kernel<false><<<build_blocks(n - 1u), 256, 0, stream>>>(b.radix, b.vals2, b.boxes, b.node_boxes, static_cast<int>(n), b.whole, nullptr,
                                                                            node_base, slot_base, out_nodes);
    LRK_CUDA(cudaGetLastError());
    return LRK_OK;
}

// The instance level over the nv visible instances (a.visible_ids) from their object-to-world rows (a.inst_o2w) and their meshes'
// object-space bounds (a.inst_mesh, a.mesh_bounds): max(nv, 2) - 1 nodes from tlas_root on, the root first.
int build_instance_level(lrk_ctx *ctx, const BuildScratch &b, uint32_t nv, uint32_t tlas_root) {
    auto &a = ctx->arrays;
    auto stream = ctx->stream;
    if (nv == 0u) {// nothing to hit: a root with two empty children
        const float inf = std::numeric_limits<float>::infinity();
        lrk_bvh_node root{};
        for (int k = 0; k < 3; k++) { root.lo0[k] = root.lo1[k] = inf; root.hi0[k] = root.hi1[k] = -inf; }
        root.ref0 = root.ref1 = root.parent = LRK_BVH_EMPTY;
        LRK_CUDA(cudaMemcpyAsync(a.bvh_nodes.get<float4>() + static_cast<size_t>(tlas_root) * 4u, &root, sizeof(root), cudaMemcpyHostToDevice, stream));
        LRK_CUDA(cudaStreamSynchronize(stream));// `root` is a local
        return LRK_OK;
    }
    LRK_CUDA(cudaMemcpyAsync(b.whole, kWholeInit, sizeof(kWholeInit), cudaMemcpyHostToDevice, stream));
    build_instance_bounds_kernel<<<build_blocks(nv), 256, 0, stream>>>(a.inst_o2w.get<const float4>(), a.inst_mesh.get<const uint32_t>(),
                                                                       a.visible_ids.get<const uint32_t>(), nv, a.mesh_bounds.get<const BuildBox>(), b.boxes, b.whole);
    return build_hierarchy(ctx, b, nv, true, tlas_root, 0u);
}

// The hierarchy of mesh `m` (its records `mesh` in a.vertices / a.triangles): its bounds into a.mesh_bounds[m], its BLAS from node
// `root` on and its triangle records from slot `slot_base` on.  b holds scratch for at least mesh.triangle_count primitives.
int build_mesh_hierarchy(lrk_ctx *ctx, const BuildScratch &b, uint32_t m, const lrk_mesh &mesh, uint32_t root, uint32_t slot_base) {
    auto &a = ctx->arrays;
    auto stream = ctx->stream;
    const uint32_t n = mesh.triangle_count;
    auto verts = a.vertices.get<const lrk_vertex>() + mesh.vertex_offset;
    auto tris = a.triangles.get<const lrk_triangle>() + mesh.triangle_offset;
    LRK_CUDA(cudaMemcpyAsync(b.whole, kWholeInit, sizeof(kWholeInit), cudaMemcpyHostToDevice, stream));
    build_triangle_bounds_kernel<<<build_blocks(n), 256, 0, stream>>>(verts, tris, n, b.boxes, b.whole);
    build_store_mesh_bounds_kernel<<<1, 1, 0, stream>>>(b.whole, a.mesh_bounds.get<BuildBox>(), m);
    if (const int rc = build_hierarchy(ctx, b, n, false, root, slot_base)) return rc;
    build_tri_verts_kernel<<<build_blocks(n), 256, 0, stream>>>(verts, tris, b.vals2, n, a.tri_verts.get<float4>() + static_cast<size_t>(slot_base) * 3u);
    return LRK_OK;
}

// Hierarchy build on the device (bvh_build.cuh): fills a.bvh_nodes / a.tri_verts from the uploaded geometry in the node layout
// that check_scene_desc derived (per mesh max(n - 1, 1) nodes from its root, then the TLAS).  One round of kernels per unique mesh,
// one for the instances.
int build_bvh_on_device(lrk_ctx *ctx, const lrk_scene_desc *s, const SceneCheck &layout) {
    auto &a = ctx->arrays;
    const std::vector<uint32_t> &visible = ctx->update.visible_host, &inst_mesh = ctx->update.inst_mesh_host;
    int rc;
    LRK_CUDA(a.bvh_nodes.reserve(layout.node_count * 64u));
    LRK_CUDA(a.tri_verts.reserve(std::max<uint64_t>(s->triangle_count, 1u) * 48u));
    LRK_CUDA(a.mesh_bounds.reserve(std::max<uint64_t>(s->mesh_count, 1u) * sizeof(BuildBox)));
    if ((rc = upload(ctx, a.inst_mesh, inst_mesh.data(), inst_mesh.size()))) return rc;
    if ((rc = upload(ctx, a.visible_ids, visible.data(), visible.size()))) return rc;
    BuildScratch b;
    if ((rc = reserve_build_scratch(ctx, std::max<uint64_t>({visible.size(), 2u, layout.largest_mesh}), b))) return rc;
    uint32_t slot_base = 0u;
    for (uint32_t m = 0; m < s->mesh_count; m++) {
        if ((rc = build_mesh_hierarchy(ctx, b, m, s->meshes[m], layout.mesh_root[m], slot_base))) return rc;
        slot_base += s->meshes[m].triangle_count;
    }
    if ((rc = build_instance_level(ctx, b, static_cast<uint32_t>(visible.size()), layout.tlas_root))) return rc;
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));// the static init block is done with
    LRK_CUDA(cudaGetLastError());
    ctx->update.tlas_inputs = true;
    return LRK_OK;
}

// One entry of lrk_update_instances' staging buffer: the instance and its new object-to-world rows.
struct InstanceUpdate {
    uint32_t id;
    float o2w[12];
};

// The instance records of an update: object-to-world rows and rows 0-2 of inst_xform (world-to-object, through the flattening's
// own inverse, affine_inverse.h); row 3, the BLAS root, stays.  The host has refused singular rows.
__global__ void __launch_bounds__(256) update_instances_kernel(const InstanceUpdate *__restrict__ updates, uint32_t count, float4 *__restrict__ inst_o2w,
                                                               float4 *__restrict__ inst_xform) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const InstanceUpdate u = updates[k];
    float w2o[12];
    inverse_affine_rows(u.o2w, w2o);
    for (uint32_t r = 0; r < 3u; r++) {
        inst_o2w[u.id * 3u + r] = make_float4(u.o2w[4u * r], u.o2w[4u * r + 1u], u.o2w[4u * r + 2u], u.o2w[4u * r + 3u]);
        inst_xform[u.id * 4u + r] = make_float4(w2o[4u * r], w2o[4u * r + 1u], w2o[4u * r + 2u], w2o[4u * r + 3u]);
    }
}

// Object-space bounds of every mesh of a host-built hierarchy, for the instance-level rebuild: the union of its BLAS root's two
// child boxes, which contain the mesh (padded like every box of that hierarchy; an empty child is +inf / -inf).
__global__ void __launch_bounds__(256) blas_root_bounds_kernel(const lrk_mesh *__restrict__ meshes, const float4 *__restrict__ nodes, uint32_t mesh_count,
                                                               BuildBox *__restrict__ mesh_bounds) {
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= mesh_count) return;
    const float4 *n = nodes + static_cast<size_t>(meshes[m].bvh_root) * 4u;
    const float4 a = n[0], b = n[1], c = n[2];// lo0, hi0, lo1, hi1 (lrk_bvh_node)
    BuildBox box;
    box.lo[0] = fminf(a.x, b.z), box.lo[1] = fminf(a.y, b.w), box.lo[2] = fminf(a.z, c.x);
    box.hi[0] = fmaxf(a.w, c.y), box.hi[1] = fmaxf(b.x, c.z), box.hi[2] = fmaxf(b.y, c.w);
    mesh_bounds[m] = box;
}

// One entry of lrk_update_meshes' table, one per updated mesh in call order.  The call's vertices, triangle slots and refit start
// nodes are numbered consecutively over the entries: entry k owns those from its *_begin to the next entry's.
struct MeshRefit {
    uint32_t mesh, vertex_offset, triangle_offset, slot_offset;// the mesh and its records (lrk_mesh)
    uint32_t vertex_begin, slot_begin, start_begin;// its first staged vertex, call slot and call start node
    uint32_t start_first;// its start nodes in a.refit_starts
};

// The entry (MeshRefit, NodeRun) that owns item i of the call: the last entry whose `Begin` is <= i (entry 0 begins at 0)
template<auto Begin, typename Entry>
__device__ __forceinline__ uint32_t owning_entry(const Entry *__restrict__ entries, uint32_t count, uint32_t i) {
    uint32_t lo = 0u, hi = count;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) / 2u;
        if (entries[mid].*Begin <= i) lo = mid;
        else hi = mid;
    }
    return lo;
}

// The staged vertices of every updated mesh into its vertex range
__global__ void __launch_bounds__(256) update_vertices_kernel(const MeshRefit *__restrict__ entries, uint32_t count, const lrk_vertex *__restrict__ staged,
                                                              uint32_t n, lrk_vertex *__restrict__ vertices) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const MeshRefit e = entries[owning_entry<&MeshRefit::vertex_begin>(entries, count, i)];
    vertices[e.vertex_offset + (i - e.vertex_begin)] = staged[i];
}

// The triangle records of every slot of the updated meshes, in their uploaded BVH order (v0.w keeps the primitive id), from the new
// vertices as build_tri_verts_kernel writes them; the slot's triangle box goes to slot_boxes[call slot] and grows the mesh's bounds
// (6 keys per entry, grow_whole)
__global__ void __launch_bounds__(256) refit_triangles_kernel(const MeshRefit *__restrict__ entries, uint32_t count, uint32_t n,
                                                              const lrk_vertex *__restrict__ vertices, const lrk_triangle *__restrict__ triangles,
                                                              float4 *__restrict__ tri_verts, BuildBox *__restrict__ slot_boxes, uint32_t *whole) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t k = owning_entry<&MeshRefit::slot_begin>(entries, count, i);
    const MeshRefit e = entries[k];
    float4 *dst = tri_verts + static_cast<size_t>(e.slot_offset + (i - e.slot_begin)) * 3u;
    const uint32_t prim = __float_as_uint(dst[0].w);
    const lrk_triangle t = triangles[e.triangle_offset + prim];
    const lrk_vertex *v = vertices + e.vertex_offset;
    const float *p0 = v[t.i0].p, *p1 = v[t.i1].p, *p2 = v[t.i2].p;
    dst[0] = make_float4(p0[0], p0[1], p0[2], __uint_as_float(prim));
    dst[1] = make_float4(p1[0], p1[1], p1[2], 0.f);
    dst[2] = make_float4(p2[0], p2[1], p2[2], 0.f);
    const BuildBox b = refit_triangle_box(p0, p1, p2);
    slot_boxes[i] = b;
    grow_whole(whole + 6u * k, b);
}

__device__ __forceinline__ bool refit_inner(uint32_t ref) { return (ref & LRK_BVH_LEAF) == 0u; }// LRK_BVH_EMPTY has the leaf bit

// A box another thread of this launch wrote: through L2, never a stale L1 line
__device__ __forceinline__ BuildBox refit_load_box(const BuildBox *b) {
    const float *f = b->lo;
    BuildBox r;
    for (int a = 0; a < 3; a++) { r.lo[a] = __ldcg(f + a); r.hi[a] = __ldcg(f + 3 + a); }
    return r;
}

// The bottom-up refit of the updated meshes' hierarchies (bvh_refit.h), with build_fit_kernel's arrival counters: one thread per
// start node (a reachable inner node without inner children) walks towards the root; a node with two inner children is computed
// by the second thread to arrive.  Every node keeps its references and parent and gets new padded child boxes; its unpadded
// box goes to node_boxes[node] for its parent.  Only nodes reachable from a mesh's root are read or written: a device-built
// hierarchy's range also holds Karras nodes of collapsed subtrees that were never written.  The thread that computes a counter's
// node resets the counter, so `visits` is all zero again when the launch ends.  At the root, the mesh's bounds for the instance
// level: the union of the root's stored boxes, as blas_root_bounds_kernel derives them.
__global__ void __launch_bounds__(256) refit_nodes_kernel(const MeshRefit *__restrict__ entries, uint32_t count, uint32_t n,
                                                          const uint32_t *__restrict__ starts, const uint32_t *__restrict__ whole,
                                                          const BuildBox *__restrict__ slot_boxes, BuildBox *node_boxes, uint32_t *visits, float4 *nodes,
                                                          BuildBox *__restrict__ mesh_bounds) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t k = owning_entry<&MeshRefit::start_begin>(entries, count, i);
    const MeshRefit e = entries[k];
    BuildBox bounds;
    for (int a = 0; a < 3; a++) { bounds.lo[a] = key_float(whole[6u * k + a]); bounds.hi[a] = key_float(whole[6u * k + 3u + a]); }
    const float pad = refit_pad(refit_extent(bounds));
    uint32_t node = starts[e.start_first + (i - e.start_begin)];
    for (;;) {
        float4 *dst = nodes + static_cast<size_t>(node) * 4u;
        const float4 r = dst[3];
        const uint32_t ref[2] = {__float_as_uint(r.x), __float_as_uint(r.y)}, parent = __float_as_uint(r.z);
        BuildBox box[2];
        for (int c = 0; c < 2; c++) {
            if (ref[c] == LRK_BVH_EMPTY) box[c] = refit_empty_box();
            else if (ref[c] & LRK_BVH_LEAF) box[c] = refit_leaf_box(slot_boxes + e.slot_begin + ((ref[c] & 0x0fffffffu) - e.slot_offset), ((ref[c] >> 28u) & 7u) + 1u);
            else box[c] = refit_load_box(node_boxes + ref[c]);
        }
        node_boxes[node] = refit_union(box[0], box[1]);
        const BuildBox s0 = refit_padded(box[0], pad), s1 = refit_padded(box[1], pad);
        float f[12];
        refit_node_boxes(s0, s1, f);
        dst[0] = make_float4(f[0], f[1], f[2], f[3]);
        dst[1] = make_float4(f[4], f[5], f[6], f[7]);
        dst[2] = make_float4(f[8], f[9], f[10], f[11]);
        if (parent == LRK_BVH_EMPTY) {
            mesh_bounds[e.mesh] = refit_union(s0, s1);
            return;
        }
        __threadfence();// the box written above is visible before the arrival is counted
        const float4 pr = nodes[static_cast<size_t>(parent) * 4u + 3u];
        const uint32_t inner = (refit_inner(__float_as_uint(pr.x)) ? 1u : 0u) + (refit_inner(__float_as_uint(pr.y)) ? 1u : 0u);
        if (atomicAdd(visits + parent, 1u) + 1u < inner) return;
        visits[parent] = 0u;
        __threadfence();
        node = parent;
    }
}

// One run of lrk_replace_meshes' node move: the node ranges of consecutive unchanged meshes, which move together from old_first to
// new_first while their triangle slots move by slot_delta.  The call's moved nodes are numbered consecutively over the runs: run k
// owns those from its `begin` to the next run's.
struct NodeRun {
    uint32_t old_first, new_first, slot_delta, begin;
};

// Every node of the runs from the old bvh_nodes into the new, its references moved (bvh_refit.h: relayout_node_refs) and its boxes
// as they are.  A device-built range also holds Karras nodes that nothing references; they are moved like the others and never read.
__global__ void __launch_bounds__(256) relayout_nodes_kernel(const NodeRun *__restrict__ runs, uint32_t count, uint32_t n, const float4 *__restrict__ old_nodes,
                                                             float4 *__restrict__ new_nodes) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const NodeRun r = runs[owning_entry<&NodeRun::begin>(runs, count, i)];
    const float4 *src = old_nodes + static_cast<size_t>(r.old_first + (i - r.begin)) * 4u;
    float4 *dst = new_nodes + static_cast<size_t>(r.new_first + (i - r.begin)) * 4u;
    const float4 w = src[3];
    uint32_t refs[3] = {__float_as_uint(w.x), __float_as_uint(w.y), __float_as_uint(w.z)};
    relayout_node_refs(refs, r.new_first - r.old_first, r.slot_delta);
    dst[0] = src[0];
    dst[1] = src[1];
    dst[2] = src[2];
    dst[3] = make_float4(__uint_as_float(refs[0]), __uint_as_float(refs[1]), __uint_as_float(refs[2]), w.w);
}

// The instance records that follow their meshes to a new layout (lrk_replace_meshes), from the new mesh table: the BLAS root in
// row 3 of inst_xform, as lrk_upload_scene stores it, and the triangle count in handle[2], from which the uniform light sampler
// picks a triangle.  An instance's mesh is its handle's buffer_base / 4, as the shade kernels decode it.
__global__ void __launch_bounds__(256) rebase_instances_kernel(const lrk_mesh *__restrict__ meshes, uint32_t n, uint4 *__restrict__ inst_handles,
                                                               float4 *__restrict__ inst_xform) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const lrk_mesh m = meshes[(inst_handles[i].x >> 10u) >> 2u];
    inst_handles[i].z = m.triangle_count;
    inst_xform[i * 4u + 3u] = make_float4(__uint_as_float(m.bvh_root), 0.f, 0.f, 0.f);
}

// The triangles of an emissive mesh (LightTreeSource::mesh_points), 9 doubles each: in world space through the row-major 3x4
// object-to-world matrix m, or in object space when m is null.
void gather_triangles(const std::vector<float> &points, const float *m, std::vector<double> &tris) {
    tris.clear();
    for (size_t k = 0; k < points.size(); k += 3u) {
        const float *p = &points[k];
        for (int r = 0; r < 3; r++)
            tris.push_back(m == nullptr ? static_cast<double>(p[r])
                                        : static_cast<double>(m[4 * r]) * p[0] + static_cast<double>(m[4 * r + 1]) * p[1] +
                                              static_cast<double>(m[4 * r + 2]) * p[2] + m[4 * r + 3]);
    }
}

// The light tree of the option "light_tree" (light_tree.h) over the emitters of `src`: world-space triangles, power and sidedness.
// tree_inst: per tree light its instance; inst_light: per instance its tree light, kLightTreeNone for instances without a light or
// without power.
void build_light_tree(const LightTreeSource &src, LightTreeBuild &tree, std::vector<uint32_t> &tree_inst, std::vector<uint32_t> &inst_light) {
    std::vector<LightTreeEmitter> emitters;
    inst_light.assign(src.instance_count, kLightTreeNone);
    std::vector<double> tris;
    for (size_t e = 0; e < src.inst.size(); e++) {
        gather_triangles(src.mesh_points.at(src.mesh[e]), &src.o2w[12u * e], tris);
        inst_light[src.inst[e]] = static_cast<uint32_t>(emitters.size());
        tree_inst.push_back(src.inst[e]);
        emitters.push_back(light_tree_emitter(tris, src.power[e], src.two_sided[e] != 0u));
    }
    tree = light_tree_build(emitters);
    for (uint32_t i = 0; i < src.instance_count; i++)
        if (inst_light[i] != kLightTreeNone && !(emitters[inst_light[i]].phi > 0.0)) inst_light[i] = kLightTreeNone;
}

// The bottom trees of the option "light_tree_triangles" (light_tree_build_triangles): one per distinct (mesh, side) pair among the
// instances of the top tree, shared by all of them.  nodes: the trees one after the other; inst_bottom: per instance {root, first
// trail} (2 words), root kLightTreeNone for none; trail: per tree, one trail per triangle of its mesh.
void build_bottom_light_trees(const LightTreeSource &src, const std::vector<uint32_t> &inst_light, std::vector<LightTreeNode> &nodes,
                              std::vector<uint32_t> &inst_bottom, std::vector<unsigned long long> &trail) {
    inst_bottom.assign(2u * src.instance_count, 0u);
    for (uint32_t i = 0; i < src.instance_count; i++) inst_bottom[2u * i] = kLightTreeNone;
    std::map<std::pair<uint32_t, uint32_t>, std::pair<uint32_t, uint32_t>> built;// (mesh, side) -> (root, first trail)
    std::vector<double> tris;
    for (size_t e = 0; e < src.inst.size(); e++) {
        const uint32_t i = src.inst[e];
        if (inst_light[i] == kLightTreeNone) continue;
        const float *m = &src.o2w[12u * e];// row-major 3x4
        const double det = static_cast<double>(m[0]) * (static_cast<double>(m[5]) * m[10] - static_cast<double>(m[6]) * m[9]) -
                           static_cast<double>(m[1]) * (static_cast<double>(m[4]) * m[10] - static_cast<double>(m[6]) * m[8]) +
                           static_cast<double>(m[2]) * (static_cast<double>(m[4]) * m[9] - static_cast<double>(m[5]) * m[8]);
        const LightTreeSide side = src.two_sided[e] ? kLightTreeTwoSided : det < 0.0 ? kLightTreeMirrored : kLightTreeOneSided;
        auto it = built.find({src.mesh[e], side});
        if (it == built.end()) {
            gather_triangles(src.mesh_points.at(src.mesh[e]), nullptr, tris);
            const LightTreeBuild b = light_tree_build_triangles(tris, side);
            const uint32_t root = b.nodes.empty() ? kLightTreeNone : static_cast<uint32_t>(nodes.size());
            it = built.emplace(std::make_pair(src.mesh[e], static_cast<uint32_t>(side)), std::make_pair(root, static_cast<uint32_t>(trail.size()))).first;
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
    if (name == "light_receiver") return &LightSampling::receiver;
    return nullptr;
}

// The light sampling `want` of the uploaded scene, once the scene record is in a.scene_copy (lrk_upload_scene: the requested one,
// the scene updates: the active one): builds and uploads the light tree and its bottom trees from ctx->update.light_source where
// requested, writes the record the kernels find them through (scene.cuh: null arrays for what is off) after the scene record,
// and latches `want` into ctx->light_active.
int upload_light_sampling(lrk_ctx *ctx, const LightSampling want) {
    auto &a = ctx->arrays;
    int rc;
    DeviceLightTree rec{};
    LightTreeBuild tree;
    std::vector<uint32_t> tree_inst, inst_light;
    if (want.tree) {
        build_light_tree(ctx->update.light_source, tree, tree_inst, inst_light);
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
        build_bottom_light_trees(ctx->update.light_source, inst_light, bottom_nodes, inst_bottom, bottom_trail);
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
    if (want.receiver) {// null until alloc_paths allocates them (it then writes them here)
        rec.receiver = ctx->receiver_words;
    }
    LRK_CUDA(cudaMemcpyAsync(a.scene_copy.get<char>() + sizeof(DeviceScene), &rec, sizeof(DeviceLightTree), cudaMemcpyHostToDevice, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));// the host arrays and `rec` are locals
    ctx->light_active = want;
    return LRK_OK;
}

// Scene updates rebuild the instance level in place: the host's SAH build with one instance per leaf and the device's LBVH both
// emit max(visible, 2) - 1 nodes, behind every mesh's BLAS.  Checked before an update changes anything.
int check_instance_level(lrk_ctx *ctx, const char *call) {
    const uint32_t visible = static_cast<uint32_t>(ctx->update.visible_host.size());
    if (static_cast<uint64_t>(ctx->scene.tlas_root) + std::max(visible, 2u) - 1u != ctx->update.bvh_node_count)
        return fail(ctx, LRK_ERR_UNSUPPORTED, std::string(call) + ": the uploaded hierarchy's instance level is not its last max(visible instances, 2) - 1 "
                                                                 "nodes, so it cannot be rebuilt in place");
    return LRK_OK;
}

// The common end of every scene update, once the instances' rows or the meshes' geometry and hierarchies are new: the first
// update's instance-level inputs (a host-built hierarchy: the per-instance meshes, the visible ids and the meshes' bounds from
// their BLAS roots), the instance level, the light sampling when an emitter changed, and the film clear.
int finish_scene_update(lrk_ctx *ctx, bool lights_changed) {
    auto &a = ctx->arrays;
    auto stream = ctx->stream;
    int rc;
    if (!ctx->update.tlas_inputs) {
        LRK_CUDA(a.inst_mesh.reserve(std::max<size_t>(ctx->update.inst_mesh_host.size() * sizeof(uint32_t), 16u)));
        LRK_CUDA(a.visible_ids.reserve(std::max<size_t>(ctx->update.visible_host.size() * sizeof(uint32_t), 16u)));
        LRK_CUDA(a.mesh_bounds.reserve(std::max<size_t>(ctx->update.mesh_count, 1u) * sizeof(BuildBox)));
        LRK_CUDA(cudaMemcpyAsync(a.inst_mesh.get(), ctx->update.inst_mesh_host.data(), ctx->update.inst_mesh_host.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
        LRK_CUDA(cudaMemcpyAsync(a.visible_ids.get(), ctx->update.visible_host.data(), ctx->update.visible_host.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
        blas_root_bounds_kernel<<<build_blocks(ctx->update.mesh_count), 256, 0, stream>>>(a.meshes.get<const lrk_mesh>(), a.bvh_nodes.get<const float4>(), ctx->update.mesh_count,
                                                                                  a.mesh_bounds.get<BuildBox>());
        LRK_CUDA(cudaGetLastError());
        ctx->update.tlas_inputs = true;
    }
    const uint32_t visible = static_cast<uint32_t>(ctx->update.visible_host.size());
    BuildScratch b;
    if ((rc = reserve_build_scratch(ctx, std::max(visible, 2u), b))) return rc;
    if ((rc = build_instance_level(ctx, b, visible, ctx->scene.tlas_root))) return rc;
    if (lights_changed && (rc = upload_light_sampling(ctx, ctx->light_active))) return rc;
    LRK_CUDA(cudaStreamSynchronize(stream));// the callers' staged locals; the caller may free its arrays
    LRK_CUDA(cudaGetLastError());
    return lrk_film_clear(ctx);
}

// What a mesh's first update derives from the uploaded hierarchy (one download of the mesh's node range; the caller's bvh_nodes
// may be gone): the refit's start nodes, i.e. the inner nodes reachable from its root that have no inner child.  The range ends
// at the next mesh's root or at the instance level: both builders lay the meshes' hierarchies out one after the other.
int derive_refit_starts(lrk_ctx *ctx, uint32_t mesh) {
    const uint32_t root = ctx->update.meshes_host[mesh].bvh_root;
    uint32_t end = ctx->scene.tlas_root;
    for (const auto &m : ctx->update.meshes_host)
        if (m.bvh_root > root && m.bvh_root < end) end = m.bvh_root;
    std::vector<lrk_bvh_node> nodes(end - root);
    LRK_CUDA(cudaMemcpyAsync(nodes.data(), ctx->arrays.bvh_nodes.get<const lrk_bvh_node>() + root, nodes.size() * sizeof(lrk_bvh_node), cudaMemcpyDeviceToHost,
                             ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    const uint32_t first = static_cast<uint32_t>(ctx->update.refit_starts_host.size());
    std::vector<uint32_t> stack{root};
    size_t walked = 0u;
    while (!stack.empty()) {
        const uint32_t n = stack.back();
        stack.pop_back();
        if (++walked > nodes.size()) return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_update_meshes: the hierarchy of mesh " + std::to_string(mesh) + " is not a tree");
        const lrk_bvh_node &nd = nodes[n - root];
        uint32_t inner = 0u;
        for (const uint32_t ref : {nd.ref0, nd.ref1}) {
            if (ref & LRK_BVH_LEAF) continue;// a leaf, or LRK_BVH_EMPTY
            if (ref < root || ref >= end)
                return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_update_meshes: the hierarchy of mesh " + std::to_string(mesh) + " leaves its node range");
            stack.push_back(ref);
            inner++;
        }
        if (inner == 0u) ctx->update.refit_starts_host.push_back(n);
    }
    ctx->update.refit_start[mesh] = {first, static_cast<uint32_t>(ctx->update.refit_starts_host.size()) - first};
    return LRK_OK;
}

// refit_starts_host to a.refit_starts: a pageable copy, not through upload(), which may page-lock the context's own vector
int send_refit_starts(lrk_ctx *ctx) {
    const auto &starts = ctx->update.refit_starts_host;
    if (starts.empty()) return LRK_OK;
    LRK_CUDA(ctx->arrays.refit_starts.reserve(starts.size() * sizeof(uint32_t)));
    LRK_CUDA(cudaMemcpyAsync(ctx->arrays.refit_starts.get(), starts.data(), starts.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    return LRK_OK;
}

// The opening of every scene update `call`: a context with a scene, and no null array among those the call reads
int open_scene_update(lrk_ctx *ctx, const char *call, bool null_array) {
    if (!ctx) return LRK_ERR_INVALID_ARGUMENT;
    if (!ctx->has_scene) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, std::string(call) + ": no scene");
    if (null_array) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, std::string(call) + ": null array");
    return LRK_OK;
}

// Id k of a scene update `call`: a `noun` (instance, mesh) below entry.size() and named once (entry[id] is ~0u until it is k)
int claim_update_id(lrk_ctx *ctx, const char *call, const char *noun, uint32_t id, uint32_t k, std::vector<uint32_t> &entry) {
    if (id >= entry.size() || entry[id] != ~0u)
        return fail(ctx, LRK_ERR_INVALID_ARGUMENT, std::string(call) + ": " + noun + " id " + std::to_string(id) + (id < entry.size() ? " repeated" : " out of range"));
    entry[id] = k;
    return LRK_OK;
}

// The n vertices a `call` gives mesh `id`, with finite positions
int check_finite_positions(lrk_ctx *ctx, const char *call, uint32_t id, const lrk_vertex *v, uint64_t n) {
    for (uint64_t i = 0; i < n; i++)
        for (int j = 0; j < 3; j++)
            if (!std::isfinite(v[i].p[j])) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, std::string(call) + ": non-finite position in mesh " + std::to_string(id));
    return LRK_OK;
}

// The light data of emissive mesh `id` from its new geometry (n triangles over vertices v): its area alias table, built on the host
// as the flattening builds it into `table` / `pdf_table` (sent asynchronously: alive until finish_scene_update synchronises) and
// sent to `alias` / `pdf`, and with the light tree its points in the tree's source, which sets lights_changed.
int refresh_emissive_mesh(lrk_ctx *ctx, uint32_t id, const lrk_vertex *v, const lrk_triangle *tris, uint32_t n, lrk_alias_entry *alias, float *pdf,
                          std::vector<lrk_alias_entry> &table, std::vector<float> &pdf_table, bool &lights_changed) {
    mesh_area_alias_table(v, tris, n, table, pdf_table);
    LRK_CUDA(cudaMemcpyAsync(alias, table.data(), table.size() * sizeof(lrk_alias_entry), cudaMemcpyHostToDevice, ctx->stream));
    LRK_CUDA(cudaMemcpyAsync(pdf, pdf_table.data(), pdf_table.size() * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->light_active.tree) return LRK_OK;
    const auto it = ctx->update.light_source.mesh_points.find(id);
    if (it == ctx->update.light_source.mesh_points.end()) return LRK_OK;
    auto &points = it->second;
    points.clear();
    for (uint32_t t = 0; t < n; t++)
        for (uint32_t i : {tris[t].i0, tris[t].i1, tris[t].i2}) points.insert(points.end(), v[i].p, v[i].p + 3);
    lights_changed = true;
    return LRK_OK;
}

// The scene record's geometry: its pointers to the geometry arrays, which lrk_upload_scene fills and lrk_replace_meshes
// reallocates, and the instance level's root
void point_scene_at_geometry(lrk_ctx *ctx, uint32_t tlas_root) {
    const auto &a = ctx->arrays;
    auto &sc = ctx->scene;
    sc.vertices = a.vertices.get<const lrk_vertex>();
    sc.triangles = a.triangles.get<const lrk_triangle>();
    sc.alias = a.alias.get<const lrk_alias_entry>();
    sc.pdf = a.pdf.get<const float>();
    sc.meshes = a.meshes.get<const lrk_mesh>();
    sc.bvh_nodes = a.bvh_nodes.get<const float4>();
    sc.tri_verts = a.tri_verts.get<const float4>();
    sc.tlas_root = tlas_root;
}

// The scene record's copy in device memory (DeviceScene::self), for the out-of-line device functions; the light-tree record behind
// it (upload_light_sampling) stays.  Asynchronous: the caller synchronises before ctx->scene changes again.
int write_scene_record(lrk_ctx *ctx) {
    LRK_CUDA(cudaMemcpyAsync(ctx->arrays.scene_copy.get(), &ctx->scene, sizeof(DeviceScene), cudaMemcpyHostToDevice, ctx->stream));
    return LRK_OK;
}

// The blocks of one persistent grid: as many as are resident at once, (blocks per SM at full occupancy) x SM count.
template<typename... Params>
int persistent_grid(void (*kernel)(Params...), int block, int sm_count) {
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0);
    return std::max(1, per_sm) * sm_count;
}

// The grid table (Grids).  Three kernels borrow another kernel's grid instead of being measured themselves.
Grids measure_grids(int sm_count) {
    Grids g{};
    g.closest = persistent_grid(trace_closest_kernel<false, false>, kTraceBlock, sm_count);
    g.query = g.closest;// lrk_trace's queries: the same trace_queue walk at the same block size
    g.shadow = persistent_grid(trace_shadow_kernel<false, false>, kTraceBlock, sm_count);
    for (uint32_t kind = 0; kind < kHitKinds; kind++) {// the fast variant has no kernel for the kinds that are always strict
        if (!hit_kind_always_strict(kind)) g.shade[0][kind] = persistent_grid(fast::shade_kernel_for(kind, false, LightSampling{}), kShadeBlock, sm_count);
        g.shade[1][kind] = persistent_grid(strict::shade_kernel_for(kind, false, LightSampling{}), kShadeBlock, sm_count);
    }
    g.classify = persistent_grid(classify_hits_kernel, kBlock, sm_count);
    g.miss = g.classify;// the escaped rays: a loop over the same depth's queue at the same block size, launched just before classification
    g.volume_medium[0] = persistent_grid(fast::volume_medium_kernel_for(), kBlock, sm_count);
    g.volume_medium[1] = persistent_grid(strict::volume_medium_kernel_for(), kBlock, sm_count);
    for (uint32_t kind = 0; kind < 3u; kind++) {
        g.volume_surface[0][kind] = persistent_grid(fast::volume_surface_kernel_for(kind, false), kBlock, sm_count);
        g.volume_surface[1][kind] = persistent_grid(strict::volume_surface_kernel_for(kind, false), kBlock, sm_count);
    }
    g.volume_nee = persistent_grid(trace_volume_nee_kernel<false>, kTraceBlock, sm_count);
    g.medium_shadow = g.volume_nee;// the in-medium shadow rays: the same any-hit trace_queue walk as the surface NEE rays
    return g;
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
    ctx->grids = measure_grids(ctx->sm_count);
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
    SceneCheck checked = check_scene_desc(*s, ctx->light_requested, ctx->device_bvh);
    if (checked.status != LRK_OK) return fail(ctx, checked.status, checked.error);
    LRK_CUDA(cudaSetDevice(ctx->device));
    // from here on the context has no scene until the scene record and its device copy are complete: a CUDA failure on the way
    // leaves no record that points at half-written arrays
    ctx->has_scene = false;
    ctx->textured = checked.textured;
    ctx->used_kinds = checked.used_kinds;
    ctx->any_non_opaque = checked.any_non_opaque;
    ctx->volume = checked.volume;
    ctx->volume_general = checked.volume_general;
    {
        SceneUpdateState u;
        u.inst_mesh_host = std::move(checked.inst_mesh);
        u.visible_host = std::move(checked.visible);
        u.mesh_count = s->mesh_count;
        u.bvh_node_count = checked.node_count;
        u.meshes_host.assign(s->meshes, s->meshes + s->mesh_count);
        for (uint32_t m = 0; m < s->mesh_count; m++) u.meshes_host[m].bvh_root = checked.mesh_root[m];// the device builder's roots with device_bvh
        u.mesh_emissive = std::move(checked.mesh_emissive);
        u.refit_start.assign(s->mesh_count, {0u, 0u});
        u.light_source = std::move(checked.light_source);
        ctx->update = std::move(u);
    }
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
    std::vector<uint32_t> handles(static_cast<size_t>(s->instance_count) * 4u);
    std::vector<float> o2w(static_cast<size_t>(s->instance_count) * 12u), xform(static_cast<size_t>(s->instance_count) * 16u);
    for (uint32_t i = 0; i < s->instance_count; i++) {
        const auto &inst = s->instances[i];
        std::memcpy(&handles[i * 4u], inst.handle, 16);
        std::memcpy(&o2w[i * 12u], inst.object_to_world, 48);
        std::memcpy(&xform[i * 16u], inst.world_to_object, 48);
        xform[i * 16u + 12u] = xform[i * 16u + 13u] = xform[i * 16u + 14u] = xform[i * 16u + 15u] = 0.f;
    }
    if ((rc = upload(ctx, a.inst_handles, handles.data(), handles.size()))) return rc;
    if ((rc = upload(ctx, a.inst_kind, checked.inst_kind.data(), checked.inst_kind.size()))) return rc;
    if ((rc = upload(ctx, a.inst_o2w, o2w.data(), o2w.size()))) return rc;
    // the hierarchy: the host's (the parity path: the oracle walks the same nodes) or one built here on the device
    if (ctx->device_bvh) {
        const auto t0 = std::chrono::steady_clock::now();
        if ((rc = build_bvh_on_device(ctx, s, checked))) return rc;
        ctx->bvh_build_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    for (uint32_t i = 0; i < s->instance_count; i++) std::memcpy(&xform[i * 16u + 12u], &checked.mesh_root[s->instances[i].mesh], 4);
    if ((rc = upload(ctx, a.inst_xform, xform.data(), xform.size()))) return rc;
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));

    auto &sc = ctx->scene;
    point_scene_at_geometry(ctx, checked.tlas_root);
    sc.inst_handles = a.inst_handles.get<const uint4>();
    sc.inst_kind = a.inst_kind.get<const uint32_t>();
    sc.inst_o2w = a.inst_o2w.get<const float4>();
    sc.inst_xform = a.inst_xform.get<const float4>();
    sc.traversal_overflow = a.traversal_overflow.get<uint32_t>();
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
    ctx->sampler_spp = s->sampler.spp;
    if (sc.refill_below == 0u) sc.refill_below = static_cast<uint32_t>(kRefillBelow);
    if (sc.inner_min == 0u) sc.inner_min = static_cast<uint32_t>(kInnerMin);
    for (int i = 0; i < 3; i++) {
        sc.sigma_a[i] = s->environment_medium.sigma_a[i];
        sc.sigma_s[i] = s->environment_medium.sigma_s[i];
    }
    sc.medium_g = s->environment_medium.g;
    sc.medium_priority = s->environment_medium.priority;
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
        if ((rc = write_scene_record(ctx))) return rc;
        if ((rc = upload_light_sampling(ctx, ctx->light_requested))) return rc;
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

int lrk_update_instances(lrk_ctx *ctx, const uint32_t *ids, uint32_t count, const float *object_to_world) {
    if (const int rc = open_scene_update(ctx, "lrk_update_instances", count != 0u && (!ids || !object_to_world))) return rc;
    // everything is checked before anything changes
    std::vector<InstanceUpdate> updates(count);
    std::vector<uint32_t> entry(ctx->scene.instance_count, ~0u);
    for (uint32_t k = 0; k < count; k++) {
        const uint32_t id = ids[k];
        if (const int rc = claim_update_id(ctx, "lrk_update_instances", "instance", id, k, entry)) return rc;
        const float *m = object_to_world + 12u * static_cast<size_t>(k);
        for (int j = 0; j < 12; j++)
            if (!std::isfinite(m[j])) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_update_instances: non-finite transform of instance " + std::to_string(id));
        float w2o[12];
        if (!inverse_affine_rows(m, w2o)) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_update_instances: singular transform of instance " + std::to_string(id));
        updates[k].id = id;
        std::memcpy(updates[k].o2w, m, sizeof(updates[k].o2w));
    }
    if (const int rc = check_instance_level(ctx, "lrk_update_instances")) return rc;
    LRK_CUDA(cudaSetDevice(ctx->device));
    auto &a = ctx->arrays;
    auto stream = ctx->stream;
    bool emitter_moved = false;
    if (ctx->light_active.tree) {
        auto &src = ctx->update.light_source;
        for (const auto &u : updates) {
            const auto it = std::lower_bound(src.inst.begin(), src.inst.end(), u.id);
            if (it == src.inst.end() || *it != u.id) continue;
            std::memcpy(&src.o2w[12u * static_cast<size_t>(it - src.inst.begin())], u.o2w, sizeof(u.o2w));
            emitter_moved = true;
        }
    }
    if (count != 0u) {// a pageable copy of a local: not through upload(), which may page-lock what it copies from
        LRK_CUDA(a.update_staging.reserve(updates.size() * sizeof(InstanceUpdate)));
        LRK_CUDA(cudaMemcpyAsync(a.update_staging.get(), updates.data(), updates.size() * sizeof(InstanceUpdate), cudaMemcpyHostToDevice, stream));
        update_instances_kernel<<<build_blocks(count), 256, 0, stream>>>(a.update_staging.get<const InstanceUpdate>(), count, a.inst_o2w.get<float4>(),
                                                                        a.inst_xform.get<float4>());
        LRK_CUDA(cudaGetLastError());
    }
    return finish_scene_update(ctx, emitter_moved);
}

int lrk_update_meshes(lrk_ctx *ctx, const uint32_t *ids, uint32_t count, const lrk_vertex *vertices, uint64_t vertex_count) {
    if (const int rc = open_scene_update(ctx, "lrk_update_meshes", count != 0u && (!ids || !vertices))) return rc;
    // everything is checked before anything changes
    std::vector<MeshRefit> entries(count);
    std::vector<uint32_t> entry(ctx->update.mesh_count, ~0u);
    uint64_t total = 0u, slots = 0u;
    for (uint32_t k = 0; k < count; k++) {
        const uint32_t id = ids[k];
        if (const int rc = claim_update_id(ctx, "lrk_update_meshes", "mesh", id, k, entry)) return rc;
        const lrk_mesh &m = ctx->update.meshes_host[id];
        entries[k] = MeshRefit{id, m.vertex_offset, m.triangle_offset, m.tri_slot_offset, static_cast<uint32_t>(total), static_cast<uint32_t>(slots), 0u, 0u};
        total += m.vertex_count;
        slots += m.triangle_count;
    }
    if (vertex_count != total)
        return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_update_meshes: vertex_count is " + std::to_string(vertex_count) + ", the meshes have " +
                                                       std::to_string(total) + " vertices");
    for (uint32_t k = 0; k < count; k++)
        if (const int rc = check_finite_positions(ctx, "lrk_update_meshes", ids[k], vertices + entries[k].vertex_begin, ctx->update.meshes_host[ids[k]].vertex_count))
            return rc;
    if (const int rc = check_instance_level(ctx, "lrk_update_meshes")) return rc;
    LRK_CUDA(cudaSetDevice(ctx->device));
    auto &a = ctx->arrays;
    auto stream = ctx->stream;
    int rc;
    // a mesh's first update derives its refit's start nodes and, for an emissive mesh, downloads its triangles: nothing changes yet
    bool new_starts = false;
    for (const auto &e : entries) {
        if (ctx->update.refit_start[e.mesh].second == 0u) {
            if ((rc = derive_refit_starts(ctx, e.mesh))) return rc;
            new_starts = true;
        }
        if (ctx->update.mesh_emissive[e.mesh] && ctx->update.emissive_triangles.count(e.mesh) == 0u) {
            const lrk_mesh &m = ctx->update.meshes_host[e.mesh];
            std::vector<lrk_triangle> tris(m.triangle_count);
            LRK_CUDA(cudaMemcpyAsync(tris.data(), a.triangles.get<const lrk_triangle>() + m.triangle_offset, tris.size() * sizeof(lrk_triangle),
                                     cudaMemcpyDeviceToHost, stream));
            LRK_CUDA(cudaStreamSynchronize(stream));
            ctx->update.emissive_triangles.emplace(e.mesh, std::move(tris));
        }
    }
    if (new_starts && (rc = send_refit_starts(ctx))) return rc;
    bool lights_changed = false;
    std::vector<std::vector<lrk_alias_entry>> tables(count);// sent asynchronously: alive until finish_scene_update synchronises
    std::vector<std::vector<float>> pdfs(count);
    if (count != 0u) {
        uint32_t starts = 0u;
        for (auto &e : entries) {
            e.start_begin = starts;
            e.start_first = ctx->update.refit_start[e.mesh].first;
            starts += ctx->update.refit_start[e.mesh].second;
        }
        std::vector<uint32_t> whole(6u * static_cast<size_t>(count));
        for (uint32_t k = 0; k < count; k++) std::memcpy(&whole[6u * k], kWholeInit, sizeof(kWholeInit));
        // scratch: per entry the bounds keys, per call slot its triangle box, per node of the meshes' hierarchies its unpadded box
        const size_t whole_bytes = (whole.size() * sizeof(uint32_t) + 15u) & ~size_t{15u}, slot_bytes = slots * sizeof(BuildBox),
                     node_bytes = static_cast<size_t>(ctx->scene.tlas_root) * sizeof(BuildBox);
        LRK_CUDA(a.refit_scratch.reserve(whole_bytes + slot_bytes + node_bytes));
        auto *d_whole = a.refit_scratch.get<uint32_t>();
        auto *slot_boxes = reinterpret_cast<BuildBox *>(a.refit_scratch.get<char>() + whole_bytes);
        auto *node_boxes = reinterpret_cast<BuildBox *>(a.refit_scratch.get<char>() + whole_bytes + slot_bytes);
        const size_t visit_bytes = std::max<size_t>(static_cast<size_t>(ctx->scene.tlas_root) * sizeof(uint32_t), 16u);
        if (a.refit_visits.bytes() < visit_bytes) {// zero once: every refit leaves its counters at zero
            LRK_CUDA(a.refit_visits.reserve(visit_bytes));
            LRK_CUDA(cudaMemsetAsync(a.refit_visits.get(), 0, visit_bytes, stream));
        }
        LRK_CUDA(a.mesh_staging.reserve(vertex_count * sizeof(lrk_vertex)));
        LRK_CUDA(a.mesh_refit.reserve(entries.size() * sizeof(MeshRefit)));
        LRK_CUDA(cudaMemcpyAsync(a.mesh_staging.get(), vertices, vertex_count * sizeof(lrk_vertex), cudaMemcpyHostToDevice, stream));
        LRK_CUDA(cudaMemcpyAsync(a.mesh_refit.get(), entries.data(), entries.size() * sizeof(MeshRefit), cudaMemcpyHostToDevice, stream));
        LRK_CUDA(cudaMemcpyAsync(d_whole, whole.data(), whole.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
        const auto *d_entries = a.mesh_refit.get<const MeshRefit>();
        update_vertices_kernel<<<build_blocks(vertex_count), 256, 0, stream>>>(d_entries, count, a.mesh_staging.get<const lrk_vertex>(),
                                                                               static_cast<uint32_t>(vertex_count), a.vertices.get<lrk_vertex>());
        refit_triangles_kernel<<<build_blocks(slots), 256, 0, stream>>>(d_entries, count, static_cast<uint32_t>(slots), a.vertices.get<const lrk_vertex>(),
                                                                        a.triangles.get<const lrk_triangle>(), a.tri_verts.get<float4>(), slot_boxes, d_whole);
        LRK_CUDA(a.mesh_bounds.reserve(std::max<size_t>(ctx->update.mesh_count, 1u) * sizeof(BuildBox)));
        refit_nodes_kernel<<<build_blocks(starts), 256, 0, stream>>>(d_entries, count, starts, a.refit_starts.get<const uint32_t>(), d_whole, slot_boxes,
                                                                     node_boxes, a.refit_visits.get<uint32_t>(), a.bvh_nodes.get<float4>(),
                                                                     a.mesh_bounds.get<BuildBox>());
        LRK_CUDA(cudaGetLastError());
        // the emissive meshes' area alias tables, and their triangles in the light tree's source
        for (uint32_t k = 0; k < count; k++) {
            const MeshRefit &e = entries[k];
            if (!ctx->update.mesh_emissive[e.mesh]) continue;
            const auto &tris = ctx->update.emissive_triangles.at(e.mesh);
            if ((rc = refresh_emissive_mesh(ctx, e.mesh, vertices + e.vertex_begin, tris.data(), static_cast<uint32_t>(tris.size()),
                                            a.alias.get<lrk_alias_entry>() + e.triangle_offset, a.pdf.get<float>() + e.triangle_offset, tables[k], pdfs[k], lights_changed)))
                return rc;
        }
    }
    return finish_scene_update(ctx, lights_changed);
}

int lrk_replace_meshes(lrk_ctx *ctx, const uint32_t *ids, uint32_t count, const uint32_t *vertex_counts, const lrk_vertex *vertices,
                       const uint32_t *triangle_counts, const lrk_triangle *triangles) {
    if (const int rc = open_scene_update(ctx, "lrk_replace_meshes", count != 0u && (!ids || !vertex_counts || !vertices || !triangle_counts || !triangles)))
        return rc;
    // everything is checked before anything changes
    const uint32_t mesh_count = ctx->update.mesh_count;
    std::vector<uint32_t> entry(mesh_count, ~0u);// per mesh the index k of its id, ~0u for an unchanged mesh
    std::vector<uint64_t> vertex_begin(count + 1u, 0u), triangle_begin(count + 1u, 0u);// where id k's records start in the caller's arrays
    for (uint32_t k = 0; k < count; k++) {
        const uint32_t id = ids[k];
        if (const int rc = claim_update_id(ctx, "lrk_replace_meshes", "mesh", id, k, entry)) return rc;
        if (vertex_counts[k] == 0u || triangle_counts[k] == 0u)
            return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_replace_meshes: mesh id " + std::to_string(id) + " gets no vertices or no triangles");
        vertex_begin[k + 1u] = vertex_begin[k] + vertex_counts[k];
        triangle_begin[k + 1u] = triangle_begin[k] + triangle_counts[k];
    }
    for (uint32_t k = 0; k < count; k++) {
        if (const int rc = check_finite_positions(ctx, "lrk_replace_meshes", ids[k], vertices + vertex_begin[k], vertex_counts[k])) return rc;
        for (uint64_t t = triangle_begin[k]; t < triangle_begin[k + 1u]; t++)
            if (std::max({triangles[t].i0, triangles[t].i1, triangles[t].i2}) >= vertex_counts[k])
                return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_replace_meshes: triangle index out of range in mesh " + std::to_string(ids[k]) + " (" +
                                                               std::to_string(vertex_counts[k]) + " vertices)");
    }
    if (const int rc = check_instance_level(ctx, "lrk_replace_meshes")) return rc;
    // the new layout, in mesh order: an unchanged mesh keeps the size of its node range (from its root to the next root, or to the
    // instance level), a replaced one gets the device builder's max(n - 1, 1) nodes; the instance level goes last
    const uint32_t old_tlas = ctx->scene.tlas_root;
    std::vector<uint32_t> roots(mesh_count);
    for (uint32_t m = 0; m < mesh_count; m++) roots[m] = ctx->update.meshes_host[m].bvh_root;
    std::sort(roots.begin(), roots.end());
    std::vector<lrk_mesh> layout(ctx->update.meshes_host);
    std::vector<uint32_t> node_count(mesh_count);
    uint64_t vertex_total = 0u, triangle_total = 0u, node_total = 0u, max_n = 0u;
    for (uint32_t m = 0; m < mesh_count; m++) {
        lrk_mesh &r = layout[m];
        if (entry[m] == ~0u) {
            const auto next = std::upper_bound(roots.begin(), roots.end(), r.bvh_root);
            node_count[m] = (next == roots.end() ? old_tlas : *next) - r.bvh_root;
        } else {
            r.vertex_count = vertex_counts[entry[m]];
            r.triangle_count = triangle_counts[entry[m]];
            node_count[m] = std::max(r.triangle_count, 2u) - 1u;
            max_n = std::max<uint64_t>(max_n, r.triangle_count);
        }
        r.vertex_offset = static_cast<uint32_t>(vertex_total);
        r.triangle_offset = r.tri_slot_offset = static_cast<uint32_t>(triangle_total);
        r.bvh_root = static_cast<uint32_t>(node_total);
        vertex_total += r.vertex_count;
        triangle_total += r.triangle_count;
        node_total += node_count[m];
        if (!fits_bvh_encoding(node_total, triangle_total, vertex_total))
            return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_replace_meshes: scene too large for the BVH encoding");
    }
    const uint32_t visible = static_cast<uint32_t>(ctx->update.visible_host.size());
    const uint32_t tlas_root = static_cast<uint32_t>(node_total);
    node_total += std::max(visible, 2u) - 1u;
    if (!fits_bvh_encoding(node_total, triangle_total, vertex_total))
        return fail(ctx, LRK_ERR_UNSUPPORTED, "lrk_replace_meshes: scene too large for the BVH encoding");
    // the unchanged meshes' records move in runs: consecutive meshes whose old ranges follow each other in every array
    struct Run {
        uint32_t last, old_v, new_v, vertices, old_t, new_t, old_s, triangles, old_n, new_n, nodes;
    };
    std::vector<Run> runs;
    for (uint32_t m = 0; m < mesh_count; m++) {
        if (entry[m] != ~0u) continue;
        const lrk_mesh &o = ctx->update.meshes_host[m], &r = layout[m];
        if (!runs.empty()) {
            Run &p = runs.back();
            if (p.last + 1u == m && p.old_v + p.vertices == o.vertex_offset && p.old_t + p.triangles == o.triangle_offset &&
                p.old_s + p.triangles == o.tri_slot_offset && p.old_n + p.nodes == o.bvh_root) {
                p.last = m;
                p.vertices += o.vertex_count;
                p.triangles += o.triangle_count;
                p.nodes += node_count[m];
                continue;
            }
        }
        runs.push_back(Run{m, o.vertex_offset, r.vertex_offset, o.vertex_count, o.triangle_offset, r.triangle_offset, o.tri_slot_offset, o.triangle_count,
                           o.bvh_root, r.bvh_root, node_count[m]});
    }
    std::vector<NodeRun> node_runs;
    uint32_t moved_nodes = 0u;
    for (const Run &p : runs) {
        if (p.nodes == 0u) continue;
        node_runs.push_back(NodeRun{p.old_n, p.new_n, p.new_t - p.old_s, moved_nodes});
        moved_nodes += p.nodes;
    }
    // every allocation before anything changes: a refusal for memory leaves the scene as it was
    LRK_CUDA(cudaSetDevice(ctx->device));
    auto &a = ctx->arrays;
    auto stream = ctx->stream;
    DeviceBuffer nv, nt, nalias, npdf, ntv, nnodes, nmeshes;
    {
        const std::pair<DeviceBuffer *, uint64_t> sizes[] = {{&nv, vertex_total * sizeof(lrk_vertex)}, {&nt, triangle_total * sizeof(lrk_triangle)},
                                                             {&nalias, triangle_total * sizeof(lrk_alias_entry)}, {&npdf, triangle_total * sizeof(float)},
                                                             {&ntv, triangle_total * 48u}, {&nnodes, node_total * sizeof(lrk_bvh_node)},
                                                             {&nmeshes, mesh_count * sizeof(lrk_mesh)}};
        for (const auto &s : sizes) {
            const cudaError_t e = s.first->reserve(std::max<uint64_t>(s.second, 16u));
            if (e == cudaErrorMemoryAllocation) {
                cudaGetLastError();
                return fail(ctx, LRK_ERR_OUT_OF_MEMORY, "lrk_replace_meshes: out of device memory for the new geometry arrays (" +
                                                            std::to_string(s.second) + " bytes); the scene is unchanged");
            }
            LRK_CUDA(e);
        }
    }
    BuildScratch b;
    int rc;
    if ((rc = reserve_build_scratch(ctx, std::max<uint64_t>(max_n, std::max(visible, 2u)), b))) return rc;// the instance level's too
    LRK_CUDA(a.mesh_bounds.reserve(std::max<size_t>(mesh_count, 1u) * sizeof(BuildBox)));
    LRK_CUDA(a.node_runs.reserve(std::max<size_t>(node_runs.size() * sizeof(NodeRun), 16u)));
    // the unchanged meshes: one copy per run and array, and their nodes in one launch
    auto copy = [&](const DeviceBuffer &to, uint64_t to_off, const DeviceBuffer &from, uint64_t from_off, uint64_t bytes) {
        return bytes ? cudaMemcpyAsync(to.get<char>() + to_off, from.get<const char>() + from_off, bytes, cudaMemcpyDeviceToDevice, stream) : cudaSuccess;
    };
    for (const Run &p : runs) {
        LRK_CUDA(copy(nv, uint64_t{p.new_v} * sizeof(lrk_vertex), a.vertices, uint64_t{p.old_v} * sizeof(lrk_vertex), uint64_t{p.vertices} * sizeof(lrk_vertex)));
        LRK_CUDA(copy(nt, uint64_t{p.new_t} * sizeof(lrk_triangle), a.triangles, uint64_t{p.old_t} * sizeof(lrk_triangle), uint64_t{p.triangles} * sizeof(lrk_triangle)));
        LRK_CUDA(copy(nalias, uint64_t{p.new_t} * sizeof(lrk_alias_entry), a.alias, uint64_t{p.old_t} * sizeof(lrk_alias_entry),
                      uint64_t{p.triangles} * sizeof(lrk_alias_entry)));
        LRK_CUDA(copy(npdf, uint64_t{p.new_t} * sizeof(float), a.pdf, uint64_t{p.old_t} * sizeof(float), uint64_t{p.triangles} * sizeof(float)));
        LRK_CUDA(copy(ntv, uint64_t{p.new_t} * 48u, a.tri_verts, uint64_t{p.old_s} * 48u, uint64_t{p.triangles} * 48u));
    }
    if (moved_nodes != 0u) {
        LRK_CUDA(cudaMemcpyAsync(a.node_runs.get(), node_runs.data(), node_runs.size() * sizeof(NodeRun), cudaMemcpyHostToDevice, stream));
        relayout_nodes_kernel<<<build_blocks(moved_nodes), 256, 0, stream>>>(a.node_runs.get<const NodeRun>(), static_cast<uint32_t>(node_runs.size()), moved_nodes,
                                                                             a.bvh_nodes.get<const float4>(), nnodes.get<float4>());
        LRK_CUDA(cudaGetLastError());
    }
    // the replaced meshes' records, the emissive ones' light data from the caller's arrays (the other replaced meshes' area tables
    // are never read), and the new mesh table
    bool lights_changed = false;
    std::vector<std::vector<lrk_alias_entry>> tables(count);
    std::vector<std::vector<float>> pdfs(count);
    for (uint32_t k = 0; k < count; k++) {
        const uint32_t id = ids[k];
        const lrk_mesh &r = layout[id];
        const lrk_triangle *tris = triangles + triangle_begin[k];
        LRK_CUDA(cudaMemcpyAsync(nv.get<lrk_vertex>() + r.vertex_offset, vertices + vertex_begin[k], uint64_t{r.vertex_count} * sizeof(lrk_vertex), cudaMemcpyHostToDevice, stream));
        LRK_CUDA(cudaMemcpyAsync(nt.get<lrk_triangle>() + r.triangle_offset, tris, uint64_t{r.triangle_count} * sizeof(lrk_triangle), cudaMemcpyHostToDevice, stream));
        if (ctx->update.mesh_emissive[id]) {
            if ((rc = refresh_emissive_mesh(ctx, id, vertices + vertex_begin[k], tris, r.triangle_count, nalias.get<lrk_alias_entry>() + r.triangle_offset,
                                            npdf.get<float>() + r.triangle_offset, tables[k], pdfs[k], lights_changed)))
                return rc;
            ctx->update.emissive_triangles[id].assign(tris, tris + r.triangle_count);
        } else {
            LRK_CUDA(cudaMemsetAsync(nalias.get<lrk_alias_entry>() + r.triangle_offset, 0, uint64_t{r.triangle_count} * sizeof(lrk_alias_entry), stream));
            LRK_CUDA(cudaMemsetAsync(npdf.get<float>() + r.triangle_offset, 0, uint64_t{r.triangle_count} * sizeof(float), stream));
        }
    }
    LRK_CUDA(cudaMemcpyAsync(nmeshes.get(), layout.data(), layout.size() * sizeof(lrk_mesh), cudaMemcpyHostToDevice, stream));
    // the new arrays become the scene's; the old ones are freed when this call returns, after finish_scene_update synchronises
    a.vertices.swap(nv);
    a.triangles.swap(nt);
    a.alias.swap(nalias);
    a.pdf.swap(npdf);
    a.tri_verts.swap(ntv);
    a.bvh_nodes.swap(nnodes);
    a.meshes.swap(nmeshes);
    for (uint32_t k = 0; k < count; k++) {
        const lrk_mesh &r = layout[ids[k]];
        if ((rc = build_mesh_hierarchy(ctx, b, ids[k], r, r.bvh_root, r.tri_slot_offset))) return rc;
    }
    if (ctx->scene.instance_count != 0u) {
        rebase_instances_kernel<<<build_blocks(ctx->scene.instance_count), 256, 0, stream>>>(a.meshes.get<const lrk_mesh>(), ctx->scene.instance_count,
                                                                                              a.inst_handles.get<uint4>(), a.inst_xform.get<float4>());
        LRK_CUDA(cudaGetLastError());
    }
    // the host's copy of the layout: the refit starts of moved meshes move with their nodes, those of replaced meshes are derived again
    std::vector<uint32_t> starts;
    for (uint32_t m = 0; m < mesh_count; m++) {
        auto &range = ctx->update.refit_start[m];
        if (entry[m] != ~0u || range.second == 0u) {
            range = {0u, 0u};
            continue;
        }
        const uint32_t first = static_cast<uint32_t>(starts.size()), delta = layout[m].bvh_root - ctx->update.meshes_host[m].bvh_root;
        for (uint32_t j = 0; j < range.second; j++) starts.push_back(ctx->update.refit_starts_host[range.first + j] + delta);
        range.first = first;
    }
    ctx->update.refit_starts_host.swap(starts);
    if ((rc = send_refit_starts(ctx))) return rc;// never larger than the buffer it had
    ctx->update.meshes_host.swap(layout);
    ctx->update.bvh_node_count = node_total;
    point_scene_at_geometry(ctx, tlas_root);
    if ((rc = write_scene_record(ctx))) return rc;
    return finish_scene_update(ctx, lights_changed);
}

// The table-driven samplers are defined for the sample indices [0, lrk_sampler::spp) that the uploaded record was derived for: past
// them PMJ02BN reads another tile position's pixel samples (past the end of its table for the last one) and ZSobol's index runs into
// the Morton bits of the next pixel.  Independent takes any index.
static int check_sample_range(lrk_ctx *ctx, uint32_t spp_end, const char *what) {
    static const char *const names[] = {"Independent", "PMJ02BN", "Sobol", "PaddedSobol", "ZSobol"};
    if (ctx->scene.sampler_type == LRK_SAMPLER_INDEPENDENT || spp_end <= ctx->sampler_spp) return LRK_OK;
    return fail(ctx, LRK_ERR_INVALID_ARGUMENT, std::string(what) + ": sample index " + std::to_string(spp_end - 1u) + " is outside the " +
                names[ctx->scene.sampler_type] + " sampler's spp " + std::to_string(ctx->sampler_spp) +
                " (a larger spp needs lrk_upload_scene)");
}

int lrk_update_camera(lrk_ctx *ctx, const lrk_camera *camera) {
    if (!ctx) return LRK_ERR_INVALID_ARGUMENT;
    if (!camera) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_update_camera: null camera");
    if (!ctx->has_scene) return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_update_camera: no scene");
    if (camera->resolution[0] != ctx->scene.width || camera->resolution[1] != ctx->scene.height)
        return fail(ctx, LRK_ERR_INVALID_ARGUMENT, "lrk_update_camera: the film size differs from the uploaded camera's (a new film size needs lrk_upload_scene)");
    LRK_CUDA(cudaSetDevice(ctx->device));
    LRK_CUDA(cudaMemcpyAsync(ctx->arrays.camera.get(), camera, sizeof(lrk_camera), cudaMemcpyHostToDevice, ctx->stream));
    LRK_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->spp_hint = camera->spp;
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
    if (int rc = check_sample_range(ctx, probe_spp, "lrk_balance_shards")) return rc;
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
            if (const int rc = write_scene_record(ctx)) return rc;
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
    if (int rc = check_sample_range(ctx, spp_end, "lrk_render")) return rc;
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
    int rc = check_sample_range(ctx, p->max_spp, "lrk_render_adaptive");
    if (rc) return rc;
    rc = check_gbuffer_supported(ctx, ctx->gbuffer_option, "lrk_render_adaptive");
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
        Stage stage{ctx, CAT_NONE};
        stage.launch(adaptive_test_kernel, grid, kAdaptiveBlock, ctx->scene.width, ctx->d_film.get<float4>(), ctx->d_moments.get<float2>(), list, blocks,
                     nblocks, p->threshold, c, last, ctx->d_sample_counts.get<uint32_t>(), keep);
        if (last) break;
        size_t temp = ctx->d_scan_temp.bytes();
        LRK_CUDA(cub::DeviceScan::ExclusiveSum(ctx->d_scan_temp.get(), temp, keep, offsets, static_cast<int>(nblocks + 1u), ctx->stream));
        ctx->stats.kernel_launches++;
        uint32_t *list_out = ctx->d_active[round & 1u].get<uint32_t>(), *blocks_out = ctx->d_block_start[1u + (round & 1u)].get<uint32_t>();
        stage.launch(adaptive_compact_kernel, grid, kAdaptiveBlock, list, blocks, nblocks, keep, offsets, list_out, blocks_out);
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
    cudaMemsetAsync(ctx->d_query_cursor.get(), 0, sizeof(uint32_t), ctx->stream);
    launch_query(ctx, any_hit != 0, d_rays.get<float4>(), d_hits.get<uint4>(), static_cast<uint32_t>(n));
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
    LRK_CUDA(cudaEventRecord(ctx->ev_begin, ctx->stream));
    for (uint32_t r = 0; r < repeat; r++) {
        LRK_CUDA(cudaMemsetAsync(ctx->d_query_cursor.get(), 0, sizeof(uint32_t), ctx->stream));
        launch_query(ctx, any_hit != 0, static_cast<const float4 *>(d_rays), static_cast<uint4 *>(d_hits), static_cast<uint32_t>(n));
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
