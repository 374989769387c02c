// Box arithmetic of the mesh hierarchies: the boxes the device builder (bvh_build.cuh) fits and the refit of a deformed mesh's
// hierarchy (lrk_update_meshes) keeps, with the padding of the host builder (bvh.cpp).  A refit keeps every node, reference and
// slot of the uploaded hierarchy and recomputes its boxes bottom-up from the deformed triangles: a leaf child's box is the union
// of its slots' triangle boxes, an inner child's the union of its own children's unpadded boxes, and every stored box is padded
// once by 5e-7 x the deformed mesh's extent.  Closest hits do not depend on the boxes as long as they contain their triangles, so
// a refit hierarchy finds what a fresh build over the deformed mesh finds.
//
// Plain C++ without CUDA built-ins: tests/host_device compiles it for the host too.
#pragma once
#include <cmath>
#include <cstdint>

#ifdef __CUDACC__
#define LRK_REFIT_FN __host__ __device__ __forceinline__
#else
#define LRK_REFIT_FN inline
#endif

namespace lrk {

struct BuildBox {
    float lo[3], hi[3];
};

// The empty box: +inf / -inf, the box of an unused child (LRK_BVH_EMPTY)
LRK_REFIT_FN BuildBox refit_empty_box() {
    BuildBox b;
    for (int a = 0; a < 3; a++) { b.lo[a] = INFINITY; b.hi[a] = -INFINITY; }
    return b;
}

// The box of one triangle, as the builders compute it (bvh_build.cuh: build_triangle_bounds_kernel; bvh.cpp through Aabb::grow)
LRK_REFIT_FN BuildBox refit_triangle_box(const float p0[3], const float p1[3], const float p2[3]) {
    BuildBox b;
    for (int a = 0; a < 3; a++) {
        b.lo[a] = fminf(fminf(p0[a], p1[a]), p2[a]);
        b.hi[a] = fmaxf(fmaxf(p0[a], p1[a]), p2[a]);
    }
    return b;
}

LRK_REFIT_FN BuildBox refit_union(const BuildBox &x, const BuildBox &y) {
    BuildBox u;
    for (int a = 0; a < 3; a++) { u.lo[a] = fminf(x.lo[a], y.lo[a]); u.hi[a] = fmaxf(x.hi[a], y.hi[a]); }
    return u;
}

// The box of a leaf: the union of its `count` (<= LRK_BVH_MAX_LEAF_TRIS) consecutive slots' triangle boxes
LRK_REFIT_FN BuildBox refit_leaf_box(const BuildBox *slot_boxes, uint32_t count) {
    BuildBox b = slot_boxes[0];
    for (uint32_t k = 1; k < count; k++) b = refit_union(b, slot_boxes[k]);
    return b;
}

// The extent the padding scales with: the largest of |lo|, |hi| and hi - lo over the axes of the whole mesh's bounds, as bvh.cpp
// and build_emit_kernel compute it
LRK_REFIT_FN float refit_extent(const BuildBox &whole) {
    float extent = 0.f;
    for (int a = 0; a < 3; a++) extent = fmaxf(extent, fmaxf(fmaxf(fabsf(whole.lo[a]), fabsf(whole.hi[a])), whole.hi[a] - whole.lo[a]));
    return extent;
}

// The padding of every stored box of a mesh hierarchy (bvh.cpp explains its size: it must stay below the spawned-ray offset)
LRK_REFIT_FN float refit_pad(float extent) { return 5e-7f * extent; }

// One child's box as a node stores it: padded by `pad`; an empty box stays +inf / -inf
LRK_REFIT_FN BuildBox refit_padded(const BuildBox &b, float pad) {
    BuildBox p;
    for (int a = 0; a < 3; a++) { p.lo[a] = b.lo[a] - pad; p.hi[a] = b.hi[a] + pad; }
    return p;
}

// The first 12 floats of an lrk_bvh_node (lo0, hi0, lo1, hi1) from its children's stored boxes
LRK_REFIT_FN void refit_node_boxes(const BuildBox &c0, const BuildBox &c1, float out[12]) {
    for (int a = 0; a < 3; a++) {
        out[a] = c0.lo[a];
        out[3 + a] = c0.hi[a];
        out[6 + a] = c1.lo[a];
        out[9 + a] = c1.hi[a];
    }
}

}// namespace lrk
