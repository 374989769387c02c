// The hit buckets of the material sort, also called closure kinds: every instance's surface maps to one kind, classify_hits_kernel
// partitions the hits of a depth by kind, and each kind has its own shade kernel.  Plain C++ without CUDA built-ins: the kernels,
// lrk_upload_scene and tests/host_device compile the same table.
#pragma once
#include <stdint.h>

#include <type_traits>

#include "../../../include/lrk.h"

#ifdef __CUDACC__
#define LRK_HIT_KINDS_FN __host__ __device__ __forceinline__
#else
#define LRK_HIT_KINDS_FN inline
#endif

namespace lrk {

constexpr uint32_t kHitEmitter = 0u;     // the instance has no surface: only its emission is looked at
constexpr uint32_t kHitMatte = 1u;
constexpr uint32_t kHitDisney = 2u;
constexpr uint32_t kHitMirror = 3u;      // kinds 3..6: MicrofacetFamilyClosure<surface type>
constexpr uint32_t kHitGlass = 4u;
constexpr uint32_t kHitPlastic = 5u;
constexpr uint32_t kHitMetal = 6u;
constexpr uint32_t kHitMix = 7u;
constexpr uint32_t kHitDisneyTrans = 8u; // "disney_trans": Disney records with LRK_SURFACE_DISNEY_TRANSMISSIVE
constexpr uint32_t kHitLayered = 9u;
constexpr uint32_t kHitDisneyThin = 10u; // "disney_thin": Disney records with LRK_SURFACE_DISNEY_THIN
constexpr uint32_t kHitKinds = 11u;

// Kind of an instance whose surface is `s` (lrk_upload_scene checks the surface tag and type first).
LRK_HIT_KINDS_FN uint32_t hit_kind_of(const lrk_surface &s) {
    if (s.type == LRK_SURFACE_DISNEY && (s.flags & LRK_SURFACE_DISNEY_THIN)) return kHitDisneyThin;
    if (s.type == LRK_SURFACE_DISNEY && (s.flags & LRK_SURFACE_DISNEY_TRANSMISSIVE)) return kHitDisneyTrans;
    if (s.type == LRK_SURFACE_LAYERED) return kHitLayered;
    return s.type + 1u;// Matte .. Mix
}

// Kinds whose shade kernel runs in IEEE arithmetic even without the option strict_math: the near-specular closures (Mirror, Glass,
// Plastic, Metal and Mix of them), whose lobes amplify a 1e-6 error in the half vector into percents of the lobe value, and Layered
// and thin Disney.  constexpr: the fast variant of shade.cu does not compile these kinds' kernels.
LRK_HIT_KINDS_FN constexpr bool hit_kind_always_strict(uint32_t kind) { return (kind >= kHitMirror && kind <= kHitMix) || kind >= kHitLayered; }

// Calls f(std::integral_constant<uint32_t, kind>{}): the run-time kind as a compile-time one.  Host and device code call it with
// their own kind of f.
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template<typename F>
LRK_HIT_KINDS_FN void with_hit_kind(uint32_t kind, F &&f) {
    switch (kind) {
        case 0u: f(std::integral_constant<uint32_t, 0u>{}); break;
        case 1u: f(std::integral_constant<uint32_t, 1u>{}); break;
        case 2u: f(std::integral_constant<uint32_t, 2u>{}); break;
        case 3u: f(std::integral_constant<uint32_t, 3u>{}); break;
        case 4u: f(std::integral_constant<uint32_t, 4u>{}); break;
        case 5u: f(std::integral_constant<uint32_t, 5u>{}); break;
        case 6u: f(std::integral_constant<uint32_t, 6u>{}); break;
        case 7u: f(std::integral_constant<uint32_t, 7u>{}); break;
        case 8u: f(std::integral_constant<uint32_t, 8u>{}); break;
        case 9u: f(std::integral_constant<uint32_t, 9u>{}); break;
        case 10u: f(std::integral_constant<uint32_t, 10u>{}); break;
        default: break;
    }
}
static_assert(kHitKinds == 11u, "with_hit_kind has one case per kind");

}// namespace lrk
