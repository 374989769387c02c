// The closure kernels of shade.cu (shade_kernels.cuh) for lrk.cu, which sizes and launches them like its own kernels.
// shade.cu is compiled twice: namespace `fast` (nvcc fast math, the arithmetic of the reference's CUDA backend) and namespace
// `strict` (IEEE arithmetic, no FMA contraction: what lrk.cu and the oracle use).  lrk.cu picks per launch (option strict_math).
#pragma once
#include "pathstate.cuh"
#include "scene_check.h"// LightSampling

namespace lrk {

// every kernel of shade.cu takes the scene, the path state and the depth whose queue it works on
using ShadeKernel = void (*)(DeviceScene, PathBuffers, uint32_t);

#define LRK_DECLARE_SHADE_VARIANT(NS)                                                                                                        \
    namespace NS {                                                                                                                           \
    /* the surface shade kernel of hit bucket `kind` (0 .. kHitKinds - 1) for that light sampling; `textured`: the instantiation that */    \
    /* evaluates image-textured parameters / normal maps.  Null for a kind that always runs in strict arithmetic in namespace fast. */    \
    ShadeKernel shade_kernel_for(uint32_t kind, bool textured, const LightSampling &light);                                                  \
    /* the volume integrator's medium step, and its surface step of bucket `kind` (0 .. 2) */                                              \
    ShadeKernel volume_medium_kernel_for();                                                                                                  \
    ShadeKernel volume_surface_kernel_for(uint32_t kind, bool textured);                                                                     \
    }

LRK_DECLARE_SHADE_VARIANT(fast)
LRK_DECLARE_SHADE_VARIANT(strict)
#undef LRK_DECLARE_SHADE_VARIANT

}// namespace lrk
