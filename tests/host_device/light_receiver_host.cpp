// light_receiver_host.cpp — the receiver word and its two uses (option "light_receiver": luisarender_b200/csrc/device/receiver.h, the
// receiver term of light_tree.h and the warp of spherical_triangle.h, the headers the shade kernels include) compiled for the host, so
// that tests/test_light_receiver_cpu.py can check the encoding, the tree's pmfs and culls and the warped sampler without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>
#include <vector>

#include "../../luisarender_b200/csrc/device/light_tree.h"
#include "../../luisarender_b200/csrc/device/receiver.h"
#include "../../luisarender_b200/csrc/device/spherical_triangle.h"

namespace {

struct Tree {
    lrk::LightTreeBuild build;
    std::vector<uint8_t> in_tree;
};

double dead_mass(const std::vector<lrk::LightTreeNode> &nodes, uint32_t i, const float *p, const lrk::Receiver &r, double reach) {
    const uint32_t index = nodes[i].index;
    if (index & lrk::kLightTreeLeaf) return 0.0;
    const float il = lrk::light_tree_importance(nodes[index], p[0], p[1], p[2], r);
    const float ir = lrk::light_tree_importance(nodes[index + 1u], p[0], p[1], p[2], r);
    const float total = il + ir;
    if (!(total > 0.f)) return reach;
    return dead_mass(nodes, index, p, r, reach * (il / total)) + dead_mass(nodes, index + 1u, p, r, reach * (ir / total));
}

lrk::SphVec vec(const float *a) { return {a[0], a[1], a[2]}; }

}// namespace

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

// as lt_build of light_tree_host.cpp
extern "C" void *lr_build(int n, const int *tri_counts, const double *tris, const double *power_density, const int *two_sided) {
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

extern "C" void lr_free(void *h) { delete static_cast<Tree *>(h); }

// pmf(p, word, emitter) at n (point, word) pairs: what an emitter hit evaluates
extern "C" void lr_pmf(void *h, int64_t n, const float *pts, const uint32_t *words, int emitter, float *out) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) {
        out[i] = 0.f;
        if (t.build.nodes.empty() || !t.in_tree[emitter]) continue;
        lrk::light_tree_walk<false>(t.build.nodes.data(), pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], 0.f, t.build.trail[emitter], out[i], nullptr,
                                    lrk::receiver_decode(words[i]));
    }
}

extern "C" void lr_sample(void *h, int64_t n, const float *pts, const uint32_t *words, const float *u, uint32_t *light, float *pmf) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++) {
        light[i] = lrk::kLightTreeNone;
        pmf[i] = 0.f;
        if (t.build.nodes.empty()) continue;
        light[i] = lrk::light_tree_walk<true>(t.build.nodes.data(), pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], u[i], 0ull, pmf[i], nullptr,
                                              lrk::receiver_decode(words[i]));
    }
}

extern "C" void lr_dead_mass(void *h, int64_t n, const float *pts, const uint32_t *words, double *out) {
    const Tree &t = *static_cast<Tree *>(h);
    for (int64_t i = 0; i < n; i++)
        out[i] = t.build.nodes.empty() ? 1.0 : dead_mass(t.build.nodes, 0u, pts + 3 * i, lrk::receiver_decode(words[i]), 1.0);
}

// ---- the bottom level: world points through w2o (12 floats), receivers through the transpose of o2w (9 floats, row-major) ----

extern "C" void *lrt_build(int64_t n, const double *tris, int side) {
    std::vector<double> t(tris, tris + 9 * n);
    return new lrk::LightTreeBuild(lrk::light_tree_build_triangles(t, static_cast<lrk::LightTreeSide>(side)));
}

extern "C" void lrt_free(void *h) { delete static_cast<lrk::LightTreeBuild *>(h); }

extern "C" void lrt_pmf(void *h, int64_t n, const float *pts, const uint32_t *words, const float *w2o, const float *o2w, int prim, float *out) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        out[i] = 0.f;
        if (b.nodes.empty()) continue;
        float q[3];
        lrk::light_tree_object_point(w2o, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], q[0], q[1], q[2]);
        out[i] = lrk::light_tree_triangle_pmf_at(b.nodes.data(), q[0], q[1], q[2], b.trail[prim], static_cast<uint32_t>(prim),
                                                 lrk::receiver_to_object(o2w, lrk::receiver_decode(words[i])));
    }
}

extern "C" void lrt_sample(void *h, int64_t n, const float *pts, const uint32_t *words, const float *w2o, const float *o2w, const float *u,
                           uint32_t *tri, float *pmf) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        tri[i] = lrk::kLightTreeNone;
        pmf[i] = 0.f;
        if (b.nodes.empty()) continue;
        float q[3];
        lrk::light_tree_object_point(w2o, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], q[0], q[1], q[2]);
        tri[i] = lrk::light_tree_walk<true>(b.nodes.data(), q[0], q[1], q[2], u[i], 0ull, pmf[i], nullptr,
                                            lrk::receiver_to_object(o2w, lrk::receiver_decode(words[i])));
    }
}

extern "C" void lrt_dead_mass(void *h, int64_t n, const float *pts, const uint32_t *words, const float *w2o, const float *o2w, double *out) {
    const auto &b = *static_cast<lrk::LightTreeBuild *>(h);
    for (int64_t i = 0; i < n; i++) {
        float q[3];
        lrk::light_tree_object_point(w2o, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], q[0], q[1], q[2]);
        out[i] = b.nodes.empty() ? 1.0 : dead_mass(b.nodes, 0u, q, lrk::receiver_to_object(o2w, lrk::receiver_decode(words[i])), 1.0);
    }
}

// ---- the warp ----

// n samples: point p (3), receiver normal (3), triangle (9), (u0, u1) -> the unit direction, the point's barycentrics, the warp's pdf
// factor evaluated at the point made (spherical_warp_pdf), the solid angle
extern "C" void lr_warp_sample(int64_t n, const float *p, const float *nr, const float *v, const float *u, float *dir, float *bary, float *factor,
                               float *omega_out, int warp) {
    for (int64_t i = 0; i < n; i++) {
        const lrk::SphVec P = vec(p + 3 * i), N = vec(nr + 3 * i), A = vec(v + 9 * i), B = vec(v + 9 * i + 3), Cc = vec(v + 9 * i + 6);
        const float omega = lrk::solid_angle(P, A, B, Cc);
        float u0 = u[2 * i], u1 = u[2 * i + 1];
        if (warp) lrk::sample_bilinear(lrk::spherical_warp_weights(P, N, A, B, Cc), u0, u1);
        const lrk::SphVec w = lrk::sample_spherical_direction(P, A, B, Cc, omega, u0, u1);
        const lrk::SphVec b = lrk::spherical_barycentrics(P, A, B, Cc, w);
        const lrk::SphVec x = {b.x * A.x + b.y * B.x + b.z * Cc.x, b.x * A.y + b.y * B.y + b.z * Cc.y, b.x * A.z + b.y * B.z + b.z * Cc.z};
        dir[3 * i] = w.x, dir[3 * i + 1] = w.y, dir[3 * i + 2] = w.z;
        bary[3 * i] = b.x, bary[3 * i + 1] = b.y, bary[3 * i + 2] = b.z;
        factor[i] = warp ? lrk::spherical_warp_pdf(P, N, A, B, Cc, omega, x) : 1.f;
        omega_out[i] = omega;
    }
}

// (u0, u1) of unit directions w (unwarped: the inverse of sample_spherical_direction)
extern "C" void lr_invert(int64_t n, const float *p, const float *v, const float *w, float *u) {
    for (int64_t i = 0; i < n; i++) {
        const lrk::SphVec P = vec(p + 3 * i), A = vec(v + 9 * i), B = vec(v + 9 * i + 3), Cc = vec(v + 9 * i + 6);
        lrk::invert_spherical_triangle_sample(P, A, B, Cc, lrk::solid_angle(P, A, B, Cc), vec(w + 3 * i), u[2 * i], u[2 * i + 1]);
    }
}
