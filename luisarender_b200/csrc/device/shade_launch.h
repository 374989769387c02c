// Host-side entry points of shade.cu - the translation unit that holds the closure kernels (shade_kernels.cuh) - for lrk.cu.
// shade.cu is compiled twice: namespace `fast` (nvcc fast math, the arithmetic of the reference's CUDA backend) and namespace
// `strict` (IEEE arithmetic, no FMA contraction: what lrk.cu and the oracle use).  lrk.cu picks per launch (option strict_math).
#pragma once
#include <cuda_runtime.h>

#include "pathstate.cuh"
#include "scene_check.h"// LightSampling

namespace lrk {

#define LRK_DECLARE_SHADE_VARIANT(NS)                                                                                                        \
    namespace NS {                                                                                                                           \
    /* blocks of one persistent grid (occupancy x SM count): surface shade kernel of hit bucket `kind` (0 .. kHitKinds - 1), the     */      \
    /* volume integrator's medium step, its surface step of bucket `kind` (0 .. 2)                                                    */      \
    int shade_grid(uint32_t kind, int sm_count);                                                                                             \
    int volume_medium_grid(int sm_count);                                                                                                    \
    int volume_surface_grid(uint32_t kind, int sm_count);                                                                                    \
    /* `textured`: the instantiation that evaluates image-textured parameters / normal maps; `light`: the one of that light sampling */   \
    void launch_shade(uint32_t kind, bool textured, const LightSampling &light, int blocks, cudaStream_t stream, const DeviceScene &sc,       \
                      const PathBuffers &pb, uint32_t depth);                                                                                \
    void launch_volume_medium(int blocks, cudaStream_t stream, const DeviceScene &sc, const PathBuffers &pb, uint32_t depth);                \
    void launch_volume_surface(uint32_t kind, bool textured, int blocks, cudaStream_t stream, const DeviceScene &sc, const PathBuffers &pb,  \
                               uint32_t depth);                                                                                              \
    }

LRK_DECLARE_SHADE_VARIANT(fast)
LRK_DECLARE_SHADE_VARIANT(strict)
#undef LRK_DECLARE_SHADE_VARIANT

}// namespace lrk
