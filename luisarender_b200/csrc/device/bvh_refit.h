// Box arithmetic of the mesh hierarchies: the boxes the device builder (bvh_build.cuh) fits and the refit of a deformed mesh's
// hierarchy (lrk_update_meshes) keeps, with the padding of the host builder (bvh.cpp).  A refit keeps every node, reference and
// slot of the uploaded hierarchy and recomputes its boxes bottom-up from the deformed triangles: a leaf child's box is the union
// of its slots' triangle boxes, an inner child's the union of its own children's unpadded boxes, and every stored box is padded
// once by 5e-7 x the deformed mesh's extent.  Closest hits do not depend on the boxes as long as they contain their triangles, so
// a refit hierarchy finds what a fresh build over the deformed mesh finds.
//
// The reference arithmetic of a hierarchy that moves to another place in bvh_nodes when lrk_replace_meshes lays the meshes out
// again is here too (relayout_node_refs).
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

// The references of one node of a mesh hierarchy that lrk_replace_meshes moves to a new place in bvh_nodes: words[0..2] are the
// node's ref0, ref1 and parent (lrk_bvh_node).  The whole hierarchy moves by node_delta nodes and its triangle slots by
// slot_delta (both modulo 2^32, so a move towards the front is a wrapped negative delta): an inner reference and the parent gain
// node_delta, a leaf keeps its count bits 28..31 and its first slot gains slot_delta.  An unused child and a root's parent are
// LRK_BVH_EMPTY (0xffffffff), which has the leaf bit: it is tested first and stays.  Boxes do not move.
LRK_REFIT_FN void relayout_node_refs(uint32_t words[3], uint32_t node_delta, uint32_t slot_delta) {
    for (int c = 0; c < 2; c++) {
        const uint32_t ref = words[c];
        if (ref == 0xffffffffu) continue;
        words[c] = (ref & 0x80000000u) ? (ref & 0xf0000000u) | ((ref + slot_delta) & 0x0fffffffu) : ref + node_delta;
    }
    if (words[2] != 0xffffffffu) words[2] += node_delta;
}

}// namespace lrk
