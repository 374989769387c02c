// light_tree_host.cpp — the light tree (luisarender_b200/csrc/device/light_tree.h, the header the shade kernels and lrk_upload_scene
// include) compiled for the host, so that tests/test_light_tree_cpu.py (the instance-level trees: lt_*) and
// tests/test_light_tree_triangles_cpu.py (the bottom level of the option "light_tree_triangles": ltt_*) can check the builds, the
// sampling and the pmfs without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../luisarender_b200/csrc/device/light_tree.h"

namespace {

struct Tree {
    lrk::LightTreeBuild build;
    std::vector<uint8_t> in_tree;// per emitter: phi > 0
};

// probability that the descent from node i (reached with probability `reach`) meets two importances of 0
double dead_mass(const std::vector<lrk::LightTreeNode> &nodes, uint32_t i, const float *p, double reach) {
    const uint32_t index = nodes[i].index;
    if (index & lrk::kLightTreeLeaf) return 0.0;
    const float il = lrk::light_tree_importance(nodes[index], p[0], p[1], p[2]);
    const float ir = lrk::light_tree_importance(nodes[index + 1u], p[0], p[1], p[2]);
    const float total = il + ir;
    if (!(total > 0.f)) return reach;
    return dead_mass(nodes, index, p, reach * (il / total)) + dead_mass(nodes, index + 1u, p, reach * (ir / total));
}

void to_object(const float *w2o, const float *p, float *q) { lrk::light_tree_object_point(w2o, p[0], p[1], p[2], q[0], q[1], q[2]); }

}// namespace

// n emitters; emitter e has tri_counts[e] world-space triangles (9 doubles each, consecutive in `tris`)
extern "C" void *lt_build(int n, const int *tri_counts, const double *tris, const double *power_density, const int *two_sided) {
    std::vector<lrk::LightTreeEmitter> emitters;
    size_t offset = 0u;
    for (int e = 0; e < n; e++) {
        std::vector<double> t(tris + offset, tris + offset + 9u * static_cast<size_t>(tri_counts[e]));
        offset += 9u * static_cast<size_t>(tri_counts[e]);
        emitters.push_back(lrk::light_tree_emitter(t, power_density[e], two_sided[e] != 0));
    }
    auto *tree = new Tree;
    tree->build = lrk::light_tree_build(emitters);
    for (const auto &e : emitters) tree->in_tree.push_back(e.phi > 0.0 ? 1u : 0u);
    return tree;
}

extern "C" void lt_free(void *h) { delete static_cast<Tree *>(h); }

extern "C" int64_t lt_node_count(void *h) { return static_cast<int64_t>(static_cast<Tree *>(h)->build.nodes.size()); }

// nodes as 48-byte records, then one trail per emitter
extern "C" void lt_copy(void *h, void *nodes, uint64_t *trails) {
    const Tree &t = *static_cast<Tree *>(h);
    std::memcpy(nodes, t.build.nodes.data(), t.build.nodes.size() * sizeof(lrk::LightTreeNode));
    for (size_t e = 0; e < t.build.trail.size(); e++) trails[e] = t.build.trail[e];
}

// pmf(p, emitter) at n points (3 floats each): what an emitter hit evaluates
extern "C" void lt_pmf(void *h, int64_t n, const float *pts, int emitter, float *out) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) {
        out[i] = 0.f;
        if (t.build.nodes.empty() || !t.in_tree[emitter]) continue;
        lrk::light_tree_walk<false>(t.build.nodes.data(), pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], 0.f, t.build.trail[emitter], out[i]);
    }
}

// one sample per (point, u): the emitter (kLightTreeNone for none) and the pmf it returns
extern "C" void lt_sample(void *h, int64_t n, const float *pts, const float *u, uint32_t *light, float *pmf) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) {
        light[i] = lrk::kLightTreeNone;
        pmf[i] = 0.f;
        if (t.build.nodes.empty()) continue;
        light[i] = lrk::light_tree_walk<true>(t.build.nodes.data(), pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], u[i], 0ull, pmf[i]);
    }
}

extern "C" void lt_dead_mass(void *h, int64_t n, const float *pts, double *out) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) out[i] = t.build.nodes.empty() ? 1.0 : dead_mass(t.build.nodes, 0u, pts + 3 * i, 1.0);
}

// importance of node `node` at n points
extern "C" void lt_importance(void *h, int64_t n, const float *pts, int node, float *out) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) out[i] = lrk::light_tree_importance(t.build.nodes[node], pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
}

// ---- the bottom level (option "light_tree_triangles") ----

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
