// Device-side BVH build (SURVEY.md §8 row f4): replaces, for scenes that ask for it (lrk_set_option("device_bvh", 1)), the host's
// binned-SAH build with an LBVH built on the GPU from the uploaded vertex / triangle / instance arrays.  The reference delegates
// acceleration-structure builds to OptiX / Embree (Geometry::build, src/base/geometry.cpp:12-27 -> Accel::build,
// src/compute/src/backends/cuda/cuda_accel.cpp:38-135); there is no reference arithmetic to follow, and results do not depend
// on the hierarchy: every box contains its triangles (padded like the host's, bvh.cpp), the triangle test and its tie rule
// are the traversal's, so hits - and films - are bit-identical to those with the host-built hierarchy (tests/test_gpu_parity.py).
//
// Per unique mesh, then once for the instances (TLAS):
//   1. bounds + centroids of the primitives, bounds of the whole set (float atomics on order-preserving integer keys);
//   2. 30-bit Morton codes of the centroids, radix sort of (code, primitive) pairs (cub::DeviceRadixSort - a library sort);
//   3. Karras' parallel radix-tree construction (one thread per internal node, ties between equal codes broken by index);
//   4. bottom-up bounds (each leaf walks up, the second child to arrive at a node computes it);
//   5. emission in the traversal's format: 64-byte two-child nodes; subtrees of at most LRK_BVH_MAX_LEAF_TRIS primitives become
//      leaves (a Karras node covers a contiguous range of the sorted order, so a leaf is a slot range) and the triangle
//      records (three float4 per BVH-ordered slot) are written in sorted order.
// Node i of a hierarchy is Karras' internal node i (no compaction: nodes inside collapsed subtrees stay unused), the root is 0.
#pragma once
#include <cub/device/device_radix_sort.cuh>

#include "bvh_refit.h"
#include "scene.cuh"

namespace lrk {

// order-preserving float <-> uint mapping for atomicMin / atomicMax
__device__ __forceinline__ uint32_t float_key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// whole[0..2] = min keys, whole[3..5] = max keys (initialised to 0xffffffff / 0)
__device__ __forceinline__ void grow_whole(uint32_t *whole, const BuildBox &b) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
        atomicMin(whole + a, float_key(b.lo[a]));
        atomicMax(whole + 3 + a, float_key(b.hi[a]));
    }
}

__global__ void __launch_bounds__(256) build_triangle_bounds_kernel(const lrk_vertex *__restrict__ vertices, const lrk_triangle *__restrict__ triangles,
                                                                    uint32_t n, BuildBox *__restrict__ boxes, uint32_t *whole) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const lrk_triangle t = triangles[i];
    const float *p[3] = {vertices[t.i0].p, vertices[t.i1].p, vertices[t.i2].p};
    BuildBox b;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        b.lo[a] = fminf(fminf(p[0][a], p[1][a]), p[2][a]);
        b.hi[a] = fmaxf(fmaxf(p[0][a], p[1][a]), p[2][a]);
    }
    boxes[i] = b;
    grow_whole(whole, b);
}

// world-space box of a visible instance: the eight corners of its BLAS' bounds through object_to_world, padded by a few ulps
// (object-space intersection rounds differently from this world-space box: flatten.cpp does the same with the vertices)
__global__ void __launch_bounds__(256) build_instance_bounds_kernel(const float4 *__restrict__ inst_o2w, const uint32_t *__restrict__ inst_mesh,
                                                                    const uint32_t *__restrict__ visible_ids, uint32_t n,
                                                                    const BuildBox *__restrict__ mesh_bounds, BuildBox *__restrict__ boxes, uint32_t *whole) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint32_t inst = visible_ids[k];
    const BuildBox mb = mesh_bounds[inst_mesh[inst]];
    const float4 r0 = inst_o2w[inst * 3u + 0u], r1 = inst_o2w[inst * 3u + 1u], r2 = inst_o2w[inst * 3u + 2u];
    BuildBox b;
    for (int a = 0; a < 3; a++) { b.lo[a] = __uint_as_float(0x7f800000u); b.hi[a] = -__uint_as_float(0x7f800000u); }
    for (int c = 0; c < 8; c++) {
        const float x = (c & 1) ? mb.hi[0] : mb.lo[0], y = (c & 2) ? mb.hi[1] : mb.lo[1], z = (c & 4) ? mb.hi[2] : mb.lo[2];
        const float w[3] = {r0.x * x + r0.y * y + r0.z * z + r0.w, r1.x * x + r1.y * y + r1.z * z + r1.w, r2.x * x + r2.y * y + r2.z * z + r2.w};
        for (int a = 0; a < 3; a++) { b.lo[a] = fminf(b.lo[a], w[a]); b.hi[a] = fmaxf(b.hi[a], w[a]); }
    }
    for (int a = 0; a < 3; a++) {
        const float e = 4e-6f * fmaxf(fabsf(b.lo[a]), fabsf(b.hi[a])) + 1e-30f;
        b.lo[a] -= e;
        b.hi[a] += e;
    }
    boxes[k] = b;
    grow_whole(whole, b);
}

__device__ __forceinline__ uint32_t expand_bits10(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

__global__ void __launch_bounds__(256) build_morton_kernel(const BuildBox *__restrict__ boxes, uint32_t n, const uint32_t *__restrict__ whole,
                                                           uint32_t *__restrict__ keys, uint32_t *__restrict__ values) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const BuildBox b = boxes[i];
    uint32_t code = 0u;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float lo = key_float(whole[a]), hi = key_float(whole[3 + a]);
        const float extent = hi - lo;
        const float c = 0.5f * (b.lo[a] + b.hi[a]);
        const float t = extent > 0.f ? (c - lo) / extent : 0.f;
        const uint32_t q = static_cast<uint32_t>(fminf(fmaxf(t * 1024.f, 0.f), 1023.f));
        code |= expand_bits10(q) << (2 - a);
    }
    keys[i] = code;
    values[i] = i;
}

// Karras 2012, "Maximizing parallelism in the construction of BVHs, octrees, and k-d trees": internal node i of n - 1, leaves
// are the sorted primitives.  child < 0x80000000: internal node, else leaf (sorted position) | 0x80000000.
struct RadixNode {
    uint32_t left, right;// child references
    uint32_t first, last;// range of sorted positions this node covers
    uint32_t parent;
};

__device__ __forceinline__ int radix_delta(const uint32_t *keys, int n, int i, int j) {
    if (j < 0 || j >= n) return -1;
    const uint32_t a = keys[i], b = keys[j];
    if (a == b) return 32 + __clz(static_cast<uint32_t>(i) ^ static_cast<uint32_t>(j));
    return __clz(a ^ b);
}

__global__ void __launch_bounds__(256) build_radix_tree_kernel(const uint32_t *__restrict__ keys, int n, RadixNode *__restrict__ nodes,
                                                               uint32_t *__restrict__ leaf_parent) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const int d = (radix_delta(keys, n, i, i + 1) - radix_delta(keys, n, i, i - 1)) >= 0 ? 1 : -1;
    const int delta_min = radix_delta(keys, n, i, i - d);
    int lmax = 2;
    while (radix_delta(keys, n, i, i + lmax * d) > delta_min) lmax *= 2;
    int l = 0;
    for (int t = lmax / 2; t >= 1; t /= 2)
        if (radix_delta(keys, n, i, i + (l + t) * d) > delta_min) l += t;
    const int j = i + l * d;
    const int delta_node = radix_delta(keys, n, i, j);
    int s = 0;
    for (int t = (l + 1) / 2;; t = (t + 1) / 2) {
        if (radix_delta(keys, n, i, i + (s + t) * d) > delta_node) s += t;
        if (t == 1) break;
    }
    const int gamma = i + s * d + min(d, 0);
    const bool left_leaf = min(i, j) == gamma, right_leaf = max(i, j) == gamma + 1;
    nodes[i].left = left_leaf ? (static_cast<uint32_t>(gamma) | 0x80000000u) : static_cast<uint32_t>(gamma);
    nodes[i].right = right_leaf ? (static_cast<uint32_t>(gamma + 1) | 0x80000000u) : static_cast<uint32_t>(gamma + 1);
    nodes[i].first = static_cast<uint32_t>(min(i, j));
    nodes[i].last = static_cast<uint32_t>(max(i, j));
    if (i == 0) nodes[0].parent = 0xffffffffu;// every other node's parent field is written by its parent's thread
    if (left_leaf) leaf_parent[gamma] = static_cast<uint32_t>(i);
    else nodes[gamma].parent = static_cast<uint32_t>(i);
    if (right_leaf) leaf_parent[gamma + 1] = static_cast<uint32_t>(i);
    else nodes[gamma + 1].parent = static_cast<uint32_t>(i);
}

// bounds of the internal nodes, bottom-up: every leaf walks towards the root; the first thread to reach a node stops, the second
// one (whose fence guarantees that both children are visible) computes it
__global__ void __launch_bounds__(256) build_fit_kernel(const RadixNode *__restrict__ nodes, const uint32_t *__restrict__ leaf_parent,
                                                        const uint32_t *__restrict__ sorted, const BuildBox *__restrict__ prim_boxes, int n,
                                                        BuildBox *__restrict__ node_boxes, uint32_t *__restrict__ visits) {
    const int leaf = blockIdx.x * blockDim.x + threadIdx.x;
    if (leaf >= n) return;
    uint32_t node = leaf_parent[leaf];
    while (node != 0xffffffffu) {
        __threadfence();// the box written in the previous trip is visible before the arrival is counted
        if (atomicAdd(visits + node, 1u) == 0u) return;
        __threadfence();
        const RadixNode nd = nodes[node];
        auto box_of = [&](uint32_t ref) { return (ref & 0x80000000u) ? prim_boxes[sorted[ref & 0x7fffffffu]] : node_boxes[ref]; };
        const BuildBox a = box_of(nd.left), b = box_of(nd.right);
        BuildBox u;
        for (int k = 0; k < 3; k++) { u.lo[k] = fminf(a.lo[k], b.lo[k]); u.hi[k] = fmaxf(a.hi[k], b.hi[k]); }
        node_boxes[node] = u;
        node = nd.parent;
    }
}

// Emission of hierarchy nodes in the traversal's layout.  TLAS: leaves are single instances (leaf ref = LEAF | instance id);
// BLAS: a subtree of at most LRK_BVH_MAX_LEAF_TRIS primitives is a leaf = LEAF | (count - 1) << 28 | first slot.
template<bool TLAS>
__global__ void __launch_bounds__(256) build_emit_kernel(const RadixNode *__restrict__ nodes, const uint32_t *__restrict__ sorted,
                                                         const BuildBox *__restrict__ prim_boxes, const BuildBox *__restrict__ node_boxes, int n,
                                                         const uint32_t *__restrict__ whole, const uint32_t *__restrict__ leaf_ids, uint32_t node_base,
                                                         uint32_t slot_base, float4 *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const RadixNode nd = nodes[i];
    if (!TLAS && nd.last - nd.first + 1u <= LRK_BVH_MAX_LEAF_TRIS && i != 0) return;// inside a collapsed subtree: never referenced
    // the padding of the host builder (bvh.cpp): 5e-7 x the hierarchy's extent
    float extent = 0.f;
    for (int a = 0; a < 3; a++) {
        const float lo = key_float(whole[a]), hi = key_float(whole[3 + a]);
        extent = fmaxf(extent, fmaxf(fmaxf(fabsf(lo), fabsf(hi)), hi - lo));
    }
    const float pad = 5e-7f * extent;
    float lo[2][3], hi[2][3];
    uint32_t ref[2];
    for (int c = 0; c < 2; c++) {
        const uint32_t r = c == 0 ? nd.left : nd.right;
        BuildBox b;
        if (r & 0x80000000u) {
            const uint32_t pos = r & 0x7fffffffu;
            b = prim_boxes[sorted[pos]];
            ref[c] = TLAS ? (LRK_BVH_LEAF | leaf_ids[sorted[pos]]) : (LRK_BVH_LEAF | (slot_base + pos));
        } else {
            b = node_boxes[r];
            const RadixNode ch = nodes[r];
            const uint32_t count = ch.last - ch.first + 1u;
            if (!TLAS && count <= LRK_BVH_MAX_LEAF_TRIS) ref[c] = LRK_BVH_LEAF | ((count - 1u) << 28u) | (slot_base + ch.first);
            else ref[c] = node_base + r;
        }
        for (int a = 0; a < 3; a++) { lo[c][a] = b.lo[a] - pad; hi[c][a] = b.hi[a] + pad; }
    }
    if (!TLAS && i == 0 && nd.last - nd.first + 1u <= LRK_BVH_MAX_LEAF_TRIS) {// the whole mesh is one leaf: root {leaf, empty}
        const BuildBox b = node_boxes[0];
        for (int a = 0; a < 3; a++) { lo[0][a] = b.lo[a] - pad; hi[0][a] = b.hi[a] + pad; }
        ref[0] = LRK_BVH_LEAF | ((nd.last - nd.first) << 28u) | (slot_base + nd.first);
        const float inf = __uint_as_float(0x7f800000u);
        for (int a = 0; a < 3; a++) { lo[1][a] = inf; hi[1][a] = -inf; }
        ref[1] = LRK_BVH_EMPTY;
    }
    float4 *dst = out + static_cast<size_t>(node_base + static_cast<uint32_t>(i)) * 4u;
    dst[0] = make_float4(lo[0][0], lo[0][1], lo[0][2], hi[0][0]);
    dst[1] = make_float4(hi[0][1], hi[0][2], lo[1][0], lo[1][1]);
    dst[2] = make_float4(lo[1][2], hi[1][0], hi[1][1], hi[1][2]);
    dst[3] = make_float4(__uint_as_float(ref[0]), __uint_as_float(ref[1]),
                         __uint_as_float(nd.parent == 0xffffffffu ? LRK_BVH_EMPTY : node_base + nd.parent), 0.f);
}

// a hierarchy over ONE primitive: root {leaf, empty}
template<bool TLAS>
__global__ void build_single_kernel(const BuildBox *__restrict__ prim_boxes, const uint32_t *__restrict__ whole, const uint32_t *__restrict__ leaf_ids,
                                    uint32_t node_base, uint32_t slot_base, float4 *__restrict__ out) {
    float extent = 0.f;
    for (int a = 0; a < 3; a++) {
        const float lo = key_float(whole[a]), hi = key_float(whole[3 + a]);
        extent = fmaxf(extent, fmaxf(fmaxf(fabsf(lo), fabsf(hi)), hi - lo));
    }
    const float pad = 5e-7f * extent;
    const BuildBox b = prim_boxes[0];
    const float inf = __uint_as_float(0x7f800000u);
    float4 *dst = out + static_cast<size_t>(node_base) * 4u;
    dst[0] = make_float4(b.lo[0] - pad, b.lo[1] - pad, b.lo[2] - pad, b.hi[0] + pad);
    dst[1] = make_float4(b.hi[1] + pad, b.hi[2] + pad, inf, inf);
    dst[2] = make_float4(inf, -inf, -inf, -inf);
    dst[3] = make_float4(__uint_as_float(TLAS ? (LRK_BVH_LEAF | leaf_ids[0]) : (LRK_BVH_LEAF | slot_base)), __uint_as_float(LRK_BVH_EMPTY),
                         __uint_as_float(LRK_BVH_EMPTY), 0.f);
}

// triangle records in BVH order: three float4 per slot, v0.w = the primitive id
__global__ void __launch_bounds__(256) build_tri_verts_kernel(const lrk_vertex *__restrict__ vertices, const lrk_triangle *__restrict__ triangles,
                                                              const uint32_t *__restrict__ sorted, uint32_t n, float4 *__restrict__ tri_verts) {
    const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= n) return;
    const uint32_t prim = sorted[pos];
    const lrk_triangle t = triangles[prim];
    const float *p0 = vertices[t.i0].p, *p1 = vertices[t.i1].p, *p2 = vertices[t.i2].p;
    float4 *dst = tri_verts + static_cast<size_t>(pos) * 3u;
    dst[0] = make_float4(p0[0], p0[1], p0[2], __uint_as_float(prim));
    dst[1] = make_float4(p1[0], p1[1], p1[2], 0.f);
    dst[2] = make_float4(p2[0], p2[1], p2[2], 0.f);
}

__global__ void build_store_mesh_bounds_kernel(const uint32_t *__restrict__ whole, BuildBox *__restrict__ mesh_bounds, uint32_t mesh) {
    BuildBox b;
    for (int a = 0; a < 3; a++) { b.lo[a] = key_float(whole[a]); b.hi[a] = key_float(whole[3 + a]); }
    mesh_bounds[mesh] = b;
}

}// namespace lrk
