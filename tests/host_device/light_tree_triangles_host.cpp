// light_tree_triangles_host.cpp — the bottom level of the light tree (option "light_tree_triangles": light_tree_build_triangles and
// the object-space walks of luisarender_b200/csrc/device/light_tree.h) compiled for the host, so that
// tests/test_light_tree_triangles_cpu.py can check the build, the sampling and the pmf without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../luisarender_b200/csrc/device/light_tree.h"

namespace {

// probability that the descent from node i (reached with probability `reach`) meets two importances of 0
double dead_mass(const std::vector<lrk::LightTreeNode> &nodes, uint32_t i, const float *q, double reach) {
    const uint32_t index = nodes[i].index;
    if (index & lrk::kLightTreeLeaf) return 0.0;
    const float il = lrk::light_tree_importance(nodes[index], q[0], q[1], q[2]);
    const float ir = lrk::light_tree_importance(nodes[index + 1u], q[0], q[1], q[2]);
    const float total = il + ir;
    if (!(total > 0.f)) return reach;
    return dead_mass(nodes, index, q, reach * (il / total)) + dead_mass(nodes, index + 1u, q, reach * (ir / total));
}

void to_object(const float *w2o, const float *p, float *q) { lrk::light_tree_object_point(w2o, p[0], p[1], p[2], q[0], q[1], q[2]); }

}// namespace

// the bottom tree of n object-space triangles (9 doubles each) for side 0 (one-sided), 1 (mirrored) or 2 (two-sided)
extern "C" void *ltt_build(int64_t n, const double *tris, int side) {
    std::vector<double> t(tris, tris + 9 * n);
    return new lrk::LightTreeBuild(lrk::light_tree_build_triangles(t, static_cast<lrk::LightTreeSide>(side)));
}

extern "C" void ltt_free(void *h) { delete static_cast<lrk::LightTreeBuild *>(h); }

extern "C" int64_t ltt_node_count(void *h) { return static_cast<int64_t>(static_cast<lrk::LightTreeBuild *>(h)->nodes.size()); }

// nodes as 48-byte records, then one trail per triangle
extern "C" void ltt_copy(void *h, void *nodes, uint64_t *trails) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    std::memcpy(nodes, b.nodes.data(), b.nodes.size() * sizeof(lrk::LightTreeNode));
    for (size_t e = 0; e < b.trail.size(); e++) trails[e] = b.trail[e];
}

// pmf of triangle `prim` at n world points (3 floats each) seen through the world-to-object rows w2o (12 floats): what an emitter
// hit evaluates
extern "C" void ltt_pmf(void *h, int64_t n, const float *pts, const float *w2o, int prim, float *out) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        out[i] = 0.f;
        if (b.nodes.empty()) continue;
        float q[3];
        to_object(w2o, pts + 3 * i, q);
        out[i] = lrk::light_tree_triangle_pmf_at(b.nodes.data(), q[0], q[1], q[2], b.trail[prim], static_cast<uint32_t>(prim));
    }
}

// one sample per (point, u): the triangle (kLightTreeNone for none) and the pmf it returns
extern "C" void ltt_sample(void *h, int64_t n, const float *pts, const float *w2o, const float *u, uint32_t *tri, float *pmf) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        tri[i] = lrk::kLightTreeNone;
        pmf[i] = 0.f;
        if (b.nodes.empty()) continue;
        float q[3];
        to_object(w2o, pts + 3 * i, q);
        tri[i] = lrk::light_tree_walk<true>(b.nodes.data(), q[0], q[1], q[2], u[i], 0ull, pmf[i]);
    }
}

// the u a sampling descent leaves at its leaf (world points taken as they are), with the leaf
extern "C" void ltt_sample_u_left(void *h, int64_t n, const float *pts, const float *u, uint32_t *tri, float *u_left) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        float pmf;
        u_left[i] = -1.f;
        tri[i] = lrk::light_tree_walk<true>(b.nodes.data(), pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], u[i], 0ull, pmf, &u_left[i]);
    }
}

extern "C" void ltt_dead_mass(void *h, int64_t n, const float *pts, const float *w2o, double *out) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        float q[3];
        to_object(w2o, pts + 3 * i, q);
        out[i] = b.nodes.empty() ? 1.0 : dead_mass(b.nodes, 0u, q, 1.0);
    }
}
