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

// calls f(std::bool_constant<b>{}): the run-time flag as a compile-time one
template<typename F>
void with_flag(bool b, F &&f) {
    if (b) f(std::true_type{});
    else f(std::false_type{});
}

// The shade kernel instantiation of (kind, textured, light selection, light point sampling), or the kind's resampling instantiation
// (RESAMPLE; none for emitter-only hits).  The fast variant has none for the kinds that always run in strict arithmetic
// (hit_kind_always_strict): render_pass never launches them there.
template<uint32_t SEL, uint32_t PT, bool RESAMPLE = false, bool RECEIVER = false>
ShadeKernel shade_kernel_of(uint32_t kind, bool textured) {
    ShadeKernel kernel = nullptr;
    with_hit_kind(kind, [&](auto k) {
        constexpr uint32_t K = decltype(k)::value;
        if constexpr (!(kFastVariant && hit_kind_always_strict(K)) && !(RESAMPLE && K == kHitEmitter))
            kernel = textured ? shade_kernel<K, true, SEL, PT, RESAMPLE, RECEIVER> : shade_kernel<K, false, SEL, PT, RESAMPLE, RECEIVER>;
    });
    return kernel;
}

// Defined below the volume steps' lookups: the kernels are instantiated in source order, and the cubin keeps its function order.
ShadeKernel light_option_kernel(uint32_t kind, bool textured, bool resample, bool tree, bool solid_angle, bool receiver);

}// namespace

// The light sampling as the kernels' <SEL, PT, RESAMPLE, RECEIVER>.  The triangle-level trees need no instantiation of their own: the
// kernels find them through light_tree_of(sc).bottom_nodes.  Resampling (candidates >= 2) has one instantiation per kind, which reads
// the selection, the point sampling and the candidate count from light_tree_of(sc); emitter-only hits sample no light and keep
// theirs.  The receiver refines the tree, the solid-angle sampler and the resampling only: uniform area sampling keeps its kernel.
ShadeKernel shade_kernel_for(uint32_t kind, bool textured, const LightSampling &light) {
    const bool resample = light.candidates >= 2u && kind != kHitEmitter;
    const bool tree = light.tree && !resample, solid_angle = light.solid_angle && !resample;
    if (!resample && !tree && !solid_angle) return shade_kernel_of<kLightSelectUniform, kLightPointArea>(kind, textured);
    return light_option_kernel(kind, textured, resample, tree, solid_angle, light.receiver);
}

ShadeKernel volume_medium_kernel_for() { return volume_medium_kernel; }

// the volume integrator's surface step exists for the kinds of config C4's closures: emitter-only, Matte and Disney
ShadeKernel volume_surface_kernel_for(uint32_t kind, bool textured) {
    ShadeKernel kernel = nullptr;
    with_hit_kind(kind, [&](auto k) {
        constexpr uint32_t K = decltype(k)::value;
        if constexpr (K <= kHitDisney) kernel = textured ? volume_surface_kernel<K, true> : volume_surface_kernel<K, false>;
    });
    return kernel;
}

namespace {

// shade_kernel_for's flags when resample, tree or solid_angle is set
ShadeKernel light_option_kernel(uint32_t kind, bool textured, bool resample, bool tree, bool solid_angle, bool receiver) {
    ShadeKernel kernel = nullptr;
    with_flag(resample, [&](auto r) { with_flag(tree, [&](auto t) { with_flag(solid_angle, [&](auto s) { with_flag(receiver, [&](auto v) {
        constexpr bool RESAMPLE = decltype(r)::value, TREE = decltype(t)::value, SOLID_ANGLE = decltype(s)::value, RECEIVER = decltype(v)::value;
        if constexpr (!(RESAMPLE && (TREE || SOLID_ANGLE)) && (!RECEIVER || RESAMPLE || TREE || SOLID_ANGLE))// the combinations shade_kernel_for passes
            kernel = shade_kernel_of<TREE ? kLightSelectTree : kLightSelectUniform, SOLID_ANGLE ? kLightPointSolidAngle : kLightPointArea, RESAMPLE,
                                     RECEIVER>(kind, textured);
    }); }); }); });
    return kernel;
}

}// namespace

}// namespace LRK_SHADE_VARIANT
}// namespace lrk
