// light_tree_host.cpp — the light tree (luisarender_b200/csrc/device/light_tree.h, the header the shade kernels and lrk_upload_scene
// include) and the receiver word (receiver.h, option "light_receiver") compiled for the host, so that the light-sampling tests
// (tests/light_sampling_checks.py) can check the instance-level trees (lt_*), the bottom level of the option "light_tree_triangles"
// (ltt_*) and the word's encoding (lr_*) without a GPU.
//
// The pmf, sample and dead-mass queries take one receiver word per point; a null word array is the word 0, no receiver, with which
// every query computes what it computes without the option.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../luisarender_b200/csrc/device/light_tree.h"
#include "../../luisarender_b200/csrc/device/receiver.h"

namespace {

struct Tree {
    lrk::LightTreeBuild build;
    std::vector<uint8_t> in_tree;// per emitter: phi > 0
};

// probability that the descent from node i (reached with probability `reach`) meets two importances of 0
double dead_mass(const std::vector<lrk::LightTreeNode> &nodes, uint32_t i, const float *p, const lrk::Receiver &r, double reach) {
    const uint32_t index = nodes[i].index;
    if (index & lrk::kLightTreeLeaf) return 0.0;
    const float il = lrk::light_tree_importance(nodes[index], p[0], p[1], p[2], r);
    const float ir = lrk::light_tree_importance(nodes[index + 1u], p[0], p[1], p[2], r);
    const float total = il + ir;
    if (!(total > 0.f)) return reach;
    return dead_mass(nodes, index, p, r, reach * (il / total)) + dead_mass(nodes, index + 1u, p, r, reach * (ir / total));
}

lrk::Receiver receiver(const uint32_t *words, int64_t i) { return lrk::receiver_decode(words ? words[i] : 0u); }

// the bottom level's point and receiver: world point i through the world-to-object rows w2o (12 floats), its receiver through the
// transpose of the object-to-world linear part o2w (9 floats, row-major; not read for the word 0)
lrk::Receiver to_object(const float *w2o, const float *o2w, const float *pts, const uint32_t *words, int64_t i, float *q) {
    lrk::light_tree_object_point(w2o, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], q[0], q[1], q[2]);
    return lrk::receiver_to_object(o2w, receiver(words, i));
}

}// namespace

// ---- the receiver word ----

extern "C" void lr_encode(int64_t n, const float *normals, const int *one_sided, uint32_t *words) {
    for (int64_t i = 0; i < n; i++) words[i] = lrk::receiver_encode(normals[3 * i], normals[3 * i + 1], normals[3 * i + 2], one_sided[i] != 0);
}

extern "C" void lr_decode(int64_t n, const uint32_t *words, float *normals, uint32_t *kinds) {
    for (int64_t i = 0; i < n; i++) {
        const lrk::Receiver r = lrk::receiver_decode(words[i]);
        normals[3 * i] = r.x, normals[3 * i + 1] = r.y, normals[3 * i + 2] = r.z;
        kinds[i] = r.kind;
    }
}

// ---- the instance level ----

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

// pmf(p, word, emitter) at n points (3 floats each): what an emitter hit evaluates
extern "C" void lt_pmf(void *h, int64_t n, const float *pts, const uint32_t *words, int emitter, float *out) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) {
        out[i] = 0.f;
        if (t.build.nodes.empty() || !t.in_tree[emitter]) continue;
        lrk::light_tree_walk<false>(t.build.nodes.data(), pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], 0.f, t.build.trail[emitter], out[i], nullptr,
                                    receiver(words, i));
    }
}

// one sample per (point, word, u): the emitter (kLightTreeNone for none) and the pmf it returns
extern "C" void lt_sample(void *h, int64_t n, const float *pts, const uint32_t *words, const float *u, uint32_t *light, float *pmf) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) {
        light[i] = lrk::kLightTreeNone;
        pmf[i] = 0.f;
        if (t.build.nodes.empty()) continue;
        light[i] = lrk::light_tree_walk<true>(t.build.nodes.data(), pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], u[i], 0ull, pmf[i], nullptr,
                                              receiver(words, i));
    }
}

extern "C" void lt_dead_mass(void *h, int64_t n, const float *pts, const uint32_t *words, double *out) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) out[i] = t.build.nodes.empty() ? 1.0 : dead_mass(t.build.nodes, 0u, pts + 3 * i, receiver(words, i), 1.0);
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

// pmf of triangle `prim` at n (world point, word) pairs: what an emitter hit evaluates
extern "C" void ltt_pmf(void *h, int64_t n, const float *pts, const uint32_t *words, const float *w2o, const float *o2w, int prim, float *out) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        out[i] = 0.f;
        if (b.nodes.empty()) continue;
        float q[3];
        const lrk::Receiver r = to_object(w2o, o2w, pts, words, i, q);
        out[i] = lrk::light_tree_triangle_pmf_at(b.nodes.data(), q[0], q[1], q[2], b.trail[prim], static_cast<uint32_t>(prim), r);
    }
}

// one sample per (world point, word, u): the triangle (kLightTreeNone for none) and the pmf it returns
extern "C" void ltt_sample(void *h, int64_t n, const float *pts, const uint32_t *words, const float *w2o, const float *o2w, const float *u,
                           uint32_t *tri, float *pmf) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        tri[i] = lrk::kLightTreeNone;
        pmf[i] = 0.f;
        if (b.nodes.empty()) continue;
        float q[3];
        const lrk::Receiver r = to_object(w2o, o2w, pts, words, i, q);
        tri[i] = lrk::light_tree_walk<true>(b.nodes.data(), q[0], q[1], q[2], u[i], 0ull, pmf[i], nullptr, r);
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

extern "C" void ltt_dead_mass(void *h, int64_t n, const float *pts, const uint32_t *words, const float *w2o, const float *o2w, double *out) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        float q[3];
        const lrk::Receiver r = to_object(w2o, o2w, pts, words, i, q);
        out[i] = b.nodes.empty() ? 1.0 : dead_mass(b.nodes, 0u, q, r, 1.0);
    }
}
