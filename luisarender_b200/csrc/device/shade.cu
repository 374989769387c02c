// shade.cu - the closure kernels of the device library, as their own translation unit, compiled TWICE.
//
// lrk.cu (ray generation, BVH traversal, hit classification, film) is compiled with IEEE arithmetic and no FMA contraction: its
// results are compared with the oracle bit for bit.  The kernels in THIS file evaluate closures, lights and media - thousands of
// fp32 operations per path vertex whose exact rounding no interface depends on.
//   -DLRK_SHADE_VARIANT=fast   --use_fast_math: the arithmetic the reference's own CUDA backend uses for every kernel (it passes
//                              -use_fast_math to NVRTC by default: src/compute/src/backends/cuda/cuda_device.cpp:697-698,
//                              ShaderOption::enable_fast_math{true} in src/compute/include/luisa/runtime/rhi/resource.h:109).
//                              The default for the emitter / Matte / Disney buckets and the volume integrator's steps (bench.py
//                              reports the same workload under strict_math next to it: arithmetic.strict_math).
//   -DLRK_SHADE_VARIANT=strict -fmad=false, IEEE div / sqrt: bit-compatible with lrk.cu and the oracle.  Always used for the
//                              Mirror / Glass / Plastic / Metal / Mix buckets (near-specular lobes amplify a 1e-6 error in the half
//                              vector into percents of the lobe value), for the Layered and thin Disney buckets, and for everything with lrk_set_option("strict_math", 1) -
//                              the configuration the tight parity tests run (films equal the oracle's to rel-L2 ~ 1e-7).
// The closures' source is the same in both, and is checked against the reference's closures bit for bit when compiled for the host
// (tests/test_device_closures_on_host.py).  build.py compiles the two objects; cross products and the uv determinant are written so
// that contraction cannot turn their exact zeros into rounding residue (vecmath.cuh: mul_exact).
#include "shade_launch.h"
#include "shade_kernels.cuh"

namespace lrk {
namespace LRK_SHADE_VARIANT {

namespace {

// LRK_SHADE_VARIANT as a compile-time value
#define LRK_SHADE_IS_FAST_fast true
#define LRK_SHADE_IS_FAST_strict false
#define LRK_SHADE_IS_FAST_OF(v) LRK_SHADE_IS_FAST_##v
#define LRK_SHADE_IS_FAST(v) LRK_SHADE_IS_FAST_OF(v)
constexpr bool kFastVariant = LRK_SHADE_IS_FAST(LRK_SHADE_VARIANT);

template<typename Kernel>
int grid_of(Kernel kernel, int block, int sm_count) {
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0);
    return (per_sm > 0 ? per_sm : 1) * sm_count;
}

// calls f(std::bool_constant<b>{}): the run-time flag as a compile-time one
template<typename F>
void with_flag(bool b, F &&f) {
    if (b) f(std::true_type{});
    else f(std::false_type{});
}

// calls f(kernel) with the shade kernel instantiation of (kind, textured, light selection, light point sampling), or with the
// kind's resampling instantiation (RESAMPLE; none for emitter-only hits).  The fast variant has none for the kinds that always run
// in strict arithmetic (hit_kind_always_strict): render_pass never launches them there.
template<uint32_t SEL, uint32_t PT, bool RESAMPLE = false, bool RECEIVER = false, typename F>
void with_shade_kernel(uint32_t kind, bool textured, F &&f) {
    with_hit_kind(kind, [&](auto k) {
        constexpr uint32_t K = decltype(k)::value;
        if constexpr (!(kFastVariant && hit_kind_always_strict(K)) && !(RESAMPLE && K == kHitEmitter))
            textured ? f(shade_kernel<K, true, SEL, PT, RESAMPLE, RECEIVER>) : f(shade_kernel<K, false, SEL, PT, RESAMPLE, RECEIVER>);
    });
}
// the volume integrator's surface step exists for the kinds of config C4's closures: emitter-only, Matte and Disney
template<typename F>
void with_volume_surface_kernel(uint32_t kind, bool textured, F &&f) {
    with_hit_kind(kind, [&](auto k) {
        constexpr uint32_t K = decltype(k)::value;
        if constexpr (K <= kHitDisney) textured ? f(volume_surface_kernel<K, true>) : f(volume_surface_kernel<K, false>);
    });
}

}// namespace

int shade_grid(uint32_t kind, int sm_count) {
    int g = 1;
    with_shade_kernel<kLightSelectUniform, kLightPointArea>(kind, false, [&](auto kernel) { g = grid_of(kernel, kShadeBlock, sm_count); });
    return g;
}

int volume_medium_grid(int sm_count) { return grid_of(volume_medium_kernel, kBlock, sm_count); }

int volume_surface_grid(uint32_t kind, int sm_count) {
    int g = 1;
    with_volume_surface_kernel(kind, false, [&](auto kernel) { g = grid_of(kernel, kBlock, sm_count); });
    return g;
}

// The light sampling as the kernels' <SEL, PT, RESAMPLE, RECEIVER>.  The triangle-level trees need no instantiation of their own: the
// kernels find them through light_tree_of(sc).bottom_nodes.  Resampling (candidates >= 2) has one instantiation per kind, which reads
// the selection, the point sampling and the candidate count from light_tree_of(sc); emitter-only hits sample no light and keep
// theirs.  The receiver refines the tree, the solid-angle sampler and the resampling only: uniform area sampling keeps its kernel.
void launch_shade(uint32_t kind, bool textured, const LightSampling &light, int blocks, cudaStream_t stream, const DeviceScene &sc,
                  const PathBuffers &pb, uint32_t depth) {
    const bool resample = light.candidates >= 2u && kind != kHitEmitter;
    const bool tree = light.tree && !resample, solid_angle = light.solid_angle && !resample;
    const bool receiver = light.receiver && (resample || tree || solid_angle);
    with_flag(resample, [&](auto r) { with_flag(tree, [&](auto t) { with_flag(solid_angle, [&](auto s) { with_flag(receiver, [&](auto v) {
        constexpr bool RESAMPLE = decltype(r)::value, TREE = decltype(t)::value, SOLID_ANGLE = decltype(s)::value, RECEIVER = decltype(v)::value;
        if constexpr (!(RESAMPLE && (TREE || SOLID_ANGLE)) && (!RECEIVER || RESAMPLE || TREE || SOLID_ANGLE))// the flags' combinations above
            with_shade_kernel<TREE ? kLightSelectTree : kLightSelectUniform, SOLID_ANGLE ? kLightPointSolidAngle : kLightPointArea, RESAMPLE, RECEIVER>(
                    kind, textured, [&](auto kernel) { kernel<<<blocks, kShadeBlock, 0, stream>>>(sc, pb, depth); });
    }); }); }); });
}

void launch_volume_medium(int blocks, cudaStream_t stream, const DeviceScene &sc, const PathBuffers &pb, uint32_t depth) {
    volume_medium_kernel<<<blocks, kBlock, 0, stream>>>(sc, pb, depth);
}

void launch_volume_surface(uint32_t kind, bool textured, int blocks, cudaStream_t stream, const DeviceScene &sc, const PathBuffers &pb, uint32_t depth) {
    with_volume_surface_kernel(kind, textured, [&](auto kernel) { kernel<<<blocks, kBlock, 0, stream>>>(sc, pb, depth); });
}

}// namespace LRK_SHADE_VARIANT
}// namespace lrk
