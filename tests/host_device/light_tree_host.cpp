// light_tree_host.cpp — the light tree (luisarender_b200/csrc/device/light_tree.h, the header the shade kernels and lrk_upload_scene
// include) compiled for the host, so that tests/test_light_tree_cpu.py can check the build, the sampling and the pmf without a GPU.
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
double dead_mass(const Tree &t, uint32_t i, const float *p, double reach) {
    const uint32_t index = t.build.nodes[i].index;
    if (index & lrk::kLightTreeLeaf) return 0.0;
    const float il = lrk::light_tree_importance(t.build.nodes[index], p[0], p[1], p[2]);
    const float ir = lrk::light_tree_importance(t.build.nodes[index + 1u], p[0], p[1], p[2]);
    const float total = il + ir;
    if (!(total > 0.f)) return reach;
    return dead_mass(t, index, p, reach * (il / total)) + dead_mass(t, index + 1u, p, reach * (ir / total));
}

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
    for (int64_t i = 0; i < n; i++) out[i] = t.build.nodes.empty() ? 1.0 : dead_mass(t, 0u, pts + 3 * i, 1.0);
}

// importance of node `node` at n points
extern "C" void lt_importance(void *h, int64_t n, const float *pts, int node, float *out) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) out[i] = lrk::light_tree_importance(t.build.nodes[node], pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
}
