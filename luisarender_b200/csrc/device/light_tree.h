// The light tree of the option "light_tree" (DESIGN.md §4 (Light tree)): a binary tree over the scene's emitters whose nodes carry
// bounds, power and a normal cone (Conty & Kulla 2018, pbrt-v4's BVHLightSampler).  Next-event estimation descends it, choosing at
// every inner node one child with probability proportional to its importance for the shading point; the pmf of an emitter is the
// product of those choices along its root-to-leaf bit trail.
//
// Plain C++ without CUDA built-ins: the shade kernels (shading.cuh), lrk_upload_scene (the build, host only) and tests/host_device
// compile the same expressions.  One function, light_tree_walk, both samples and evaluates the pmf, so that the pmf a sample returns
// is the pmf evaluated at an emitter hit bit for bit (within one compilation).
#pragma once
#include <math.h>
#include <stdint.h>

#include "receiver.h"

#ifdef __CUDACC__
#define LRK_LIGHT_TREE_FN __host__ __device__ __forceinline__
#else
#define LRK_LIGHT_TREE_FN inline
#endif

namespace lrk {

constexpr uint32_t kLightTreeLeaf = 0x80000000u;// LightTreeNode::index: a leaf holding light (index & ~kLightTreeLeaf)
constexpr uint32_t kLightTreeNone = 0xffffffffu;// no light: the descent met two importances of 0, or an emitter outside the tree
constexpr float kLightTreeMinCos = 1e-3f;       // cosine floor of a node that is not culled (its padded cone may reach cos < 0)

// 48 B.  Inner nodes: children at index and index + 1.  Cone cosines quantized to 16 bits each, rounded towards a wider cone.
struct alignas(16) LightTreeNode {
    float lo[3], hi[3];// world-space bounds
    float phi;         // power: sum of lum(L) * scale * area * (two-sided ? 2 : 1) of its emitters
    float axis[3];     // normal cone axis (unit)
    uint32_t cos_q;    // cos theta_o | cos theta_e << 16, each as floor(32767 * (c + 1) / 2) - 1
    uint32_t index;    // first child, or kLightTreeLeaf | light
};
static_assert(sizeof(LightTreeNode) == 48, "light tree node is 48 B");

LRK_LIGHT_TREE_FN float light_tree_dequantize_cos(uint32_t q) { return 2.f * (static_cast<float>(q & 0xffffu) * (1.f / 32767.f)) - 1.f; }

// The receiver term's cull pad (option "light_receiver"): a one-sided receiver culls a node only when its bounding sphere lies behind
// the receiver's plane by more than this angle, seen from p.  It covers the octahedral rounding of the normal (below 2e-4 rad,
// receiver.h) and an evaluation point that is not the sampling point: an emitter hit evaluates the pmf from the offset ray origin,
// a light sample from the surface point, which lie within 1 % of the distance to the node of each other.
constexpr float kLightTreeReceiverPadSin = 0.01f;// sin of the pad

// pbrt-v4's LightBounds::Importance.  Conservative: 0 only when no point of the node's bounds emits towards p (or, for a one-sided
// receiver, lies in front of it).  p inside the bounding sphere of the bounds skips the orientation and receiver tests; the cone
// angles are padded at the build.  The receiver term cos theta'_i = cos(max(theta_i - theta_b, 0)), theta_i the angle between the
// receiver's normal and the direction to the node's centre: |cos theta_i| for a two-sided receiver, as pbrt-v4; none (the
// expressions without it) for kReceiverNone.
LRK_LIGHT_TREE_FN float light_tree_importance(const LightTreeNode &n, float px, float py, float pz, const Receiver &rcv = Receiver{0.f, 0.f, 0.f, kReceiverNone}) {
    const float ex = n.hi[0] - n.lo[0], ey = n.hi[1] - n.lo[1], ez = n.hi[2] - n.lo[2];
    const float dx = px - 0.5f * (n.lo[0] + n.hi[0]), dy = py - 0.5f * (n.lo[1] + n.hi[1]), dz = pz - 0.5f * (n.lo[2] + n.hi[2]);
    const float dist2 = dx * dx + dy * dy + dz * dz;
    const float diag2 = ex * ex + ey * ey + ez * ez;
    const float r2 = 0.2501f * diag2;// bounding sphere radius^2, padded
    float cos_p = 1.f;
    const float cos_o = light_tree_dequantize_cos(n.cos_q);
    if (dist2 > r2 && cos_o > -1.f) {
        const float inv_d = 1.f / sqrtf(dist2);
        const float cos_w = fminf(fmaxf((n.axis[0] * dx + n.axis[1] * dy + n.axis[2] * dz) * inv_d, -1.f), 1.f);
        const float sin_w = sqrtf(fmaxf(1.f - cos_w * cos_w, 0.f));
        const float sin_o = sqrtf(fmaxf(1.f - cos_o * cos_o, 0.f));
        const float sin2_b = r2 / dist2;
        const float cos_b = sqrtf(fmaxf(1.f - sin2_b, 0.f)), sin_b = sqrtf(sin2_b);
        // theta_x = max(theta_w - theta_o, 0), theta_p = max(theta_x - theta_b, 0)
        const float cos_x = cos_w > cos_o ? 1.f : cos_w * cos_o + sin_w * sin_o;
        const float sin_x = cos_w > cos_o ? 0.f : sin_w * cos_o - cos_w * sin_o;
        cos_p = cos_x > cos_b ? 1.f : cos_x * cos_b + sin_x * sin_b;
        if (cos_p <= light_tree_dequantize_cos(n.cos_q >> 16u)) return 0.f;
    }
    const float d2 = fmaxf(dist2, 0.5f * sqrtf(diag2));
    if (rcv.kind == kReceiverNone) return n.phi * fmaxf(cos_p, kLightTreeMinCos) / d2;
    float cos_r = 1.f;
    if (dist2 > r2) {
        const float inv_d = 1.f / sqrtf(dist2);
        const float sin2_b = r2 / dist2;
        const float cos_b = sqrtf(fmaxf(1.f - sin2_b, 0.f)), sin_b = sqrtf(sin2_b);
        float cos_i = fminf(fmaxf(-(rcv.x * dx + rcv.y * dy + rcv.z * dz) * inv_d, -1.f), 1.f);
        if (rcv.kind == kReceiverTwoSided) cos_i = fabsf(cos_i);
        const float sin_i = sqrtf(fmaxf(1.f - cos_i * cos_i, 0.f));
        cos_r = cos_i > cos_b ? 1.f : cos_i * cos_b + sin_i * sin_b;
        if (cos_r < -kLightTreeReceiverPadSin) return 0.f;// one-sided only: cos_i >= 0 for a two-sided receiver
    }
    return n.phi * fmaxf(cos_p, kLightTreeMinCos) * fmaxf(cos_r, kLightTreeMinCos) / d2;
}

// The descent from the root.  SAMPLE: chooses with u in [0, 1) and returns the light; otherwise follows `trail` (bit d = 1: the
// second child at depth d) and returns the leaf's light.  pmf: the probability of that choice, 0 with kLightTreeNone.  u_left: where
// not null, receives u as the sampling descent left it at the leaf, remapped to [0, 1) by every choice on the way.  rcv: the receiver
// of light_tree_importance (option "light_receiver"), the same for the sample and the evaluation of one point.
template<bool SAMPLE>
LRK_LIGHT_TREE_FN uint32_t light_tree_walk(const LightTreeNode *nodes, float px, float py, float pz, float u, unsigned long long trail, float &pmf,
                                           float *u_left = nullptr, const Receiver &rcv = Receiver{0.f, 0.f, 0.f, kReceiverNone}) {
    pmf = 1.f;
    uint32_t i = 0u;
    for (;;) {
        const uint32_t index = nodes[i].index;
        if (index & kLightTreeLeaf) {
            if (u_left != nullptr) *u_left = u;
            return index & ~kLightTreeLeaf;
        }
        const float il = light_tree_importance(nodes[index], px, py, pz, rcv), ir = light_tree_importance(nodes[index + 1u], px, py, pz, rcv);
        const float total = il + ir;
        if (!(total > 0.f)) {
            pmf = 0.f;
            return kLightTreeNone;
        }
        const float pl = il / total, pr = ir / total;
        bool second;
        if (SAMPLE) {
            second = !(u < pl);
            u = fminf(second ? (u - pl) / pr : u / pl, 0x1.fffffep-1f);
        } else {
            second = (trail & 1ull) != 0ull;
            trail >>= 1u;
        }
        pmf *= second ? pr : pl;
        i = index + (second ? 1u : 0u);
    }
}

// The bottom level of the option "light_tree_triangles": one tree per emissive mesh over its triangles, in the mesh's object space.
// The shading point enters it mapped by the instance's world-to-object rows w2o (row-major 3x4) with the expressions traversal uses
// (traverse.cuh); facing is invariant under that map, so the orientation cull stays conservative for any invertible transform.  A
// receiver enters it through receiver_to_object (receiver.h), which keeps the side of its plane for the same reason.
LRK_LIGHT_TREE_FN void light_tree_object_point(const float *w2o, float px, float py, float pz, float &qx, float &qy, float &qz) {
    qx = fmaf(w2o[0], px, fmaf(w2o[1], py, fmaf(w2o[2], pz, w2o[3])));
    qy = fmaf(w2o[4], px, fmaf(w2o[5], py, fmaf(w2o[6], pz, w2o[7])));
    qz = fmaf(w2o[8], px, fmaf(w2o[9], py, fmaf(w2o[10], pz, w2o[11])));
}

// pmf of triangle `prim` of a bottom tree at object-space point q, following its trail.  A triangle the build left out (no area)
// has trail 0, which leads to another triangle's leaf: pmf 0.
LRK_LIGHT_TREE_FN float light_tree_triangle_pmf_at(const LightTreeNode *nodes, float qx, float qy, float qz, unsigned long long trail, uint32_t prim,
                                                   const Receiver &rcv = Receiver{0.f, 0.f, 0.f, kReceiverNone}) {
    float pmf;
    return light_tree_walk<false>(nodes, qx, qy, qz, 0.f, trail, pmf, nullptr, rcv) == prim ? pmf : 0.f;
}

}// namespace lrk

// ---- the build (host code: lrk_upload_scene, tests/host_device) ------------------------------------------------------------------
#include <algorithm>
#include <cmath>
#include <vector>

namespace lrk {

// One emitter's bounds in double precision, before padding and rounding to a node.
struct LightTreeEmitter {
    double lo[3]{0.0, 0.0, 0.0}, hi[3]{0.0, 0.0, 0.0};
    double phi{0.0};
    double axis[3]{0.0, 0.0, 1.0};
    double cos_o{-1.0};// -1: the whole sphere
};

struct LightTreeBuild {
    std::vector<LightTreeNode> nodes;     // empty when no emitter has power
    std::vector<unsigned long long> trail;// per emitter: its root-to-leaf bit trail (0 for emitters left out, phi = 0)
};

namespace light_tree_detail {

constexpr double kPi = 3.14159265358979323846;
constexpr double kConePad = 1e-3;// radians added to theta_o
constexpr double kEmitPad = 1e-2;// radians added to theta_e = pi / 2 (a diffuse emitter)

inline double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// DirectionCone::Union (pbrt-v4 util/vecmath.cpp) on (axis, cos theta)
inline void cone_union(const double *wa, double ca, const double *wb, double cb, double *w, double &c) {
    if (ca <= -1.0 || cb <= -1.0) {
        w[0] = 0.0, w[1] = 0.0, w[2] = 1.0, c = -1.0;
        return;
    }
    const double ta = std::acos(std::min(std::max(ca, -1.0), 1.0)), tb = std::acos(std::min(std::max(cb, -1.0), 1.0));
    const double td = std::acos(std::min(std::max(dot3(wa, wb), -1.0), 1.0));
    if (std::min(td + tb, kPi) <= ta) { std::copy(wa, wa + 3, w); c = ca; return; }
    if (std::min(td + ta, kPi) <= tb) { std::copy(wb, wb + 3, w); c = cb; return; }
    const double to = 0.5 * (ta + td + tb);
    double r[3] = {wa[1] * wb[2] - wa[2] * wb[1], wa[2] * wb[0] - wa[0] * wb[2], wa[0] * wb[1] - wa[1] * wb[0]};
    const double rl = std::sqrt(dot3(r, r));
    if (to >= kPi || rl == 0.0) {
        w[0] = 0.0, w[1] = 0.0, w[2] = 1.0, c = -1.0;
        return;
    }
    for (double &x : r) x /= rl;
    // rotate wa by theta_r = to - ta about r (Rodrigues)
    const double tr = to - ta, s = std::sin(tr), k = std::cos(tr), rd = dot3(r, wa);
    const double cr[3] = {r[1] * wa[2] - r[2] * wa[1], r[2] * wa[0] - r[0] * wa[2], r[0] * wa[1] - r[1] * wa[0]};
    for (int j = 0; j < 3; j++) w[j] = wa[j] * k + cr[j] * s + r[j] * rd * (1.0 - k);
    const double wl = std::sqrt(dot3(w, w));
    for (int j = 0; j < 3; j++) w[j] /= wl;
    c = std::cos(to);
}

inline void merge(LightTreeEmitter &acc, const LightTreeEmitter &e, bool first) {
    if (first) {
        acc = e;
        return;
    }
    for (int j = 0; j < 3; j++) {
        acc.lo[j] = std::min(acc.lo[j], e.lo[j]);
        acc.hi[j] = std::max(acc.hi[j], e.hi[j]);
    }
    acc.phi += e.phi;
    double w[3], c;
    cone_union(acc.axis, acc.cos_o, e.axis, e.cos_o, w, c);
    std::copy(w, w + 3, acc.axis);
    acc.cos_o = c;
}

// pbrt-v4's EvaluateCost: phi * M_omega * K_r * surface area, theta_e = pi / 2
inline double cost(const LightTreeEmitter &b, double kr) {
    const double to = std::acos(std::min(std::max(b.cos_o, -1.0), 1.0)), tw = std::min(to + 0.5 * kPi, kPi);
    const double so = std::sqrt(std::max(1.0 - b.cos_o * b.cos_o, 0.0));
    const double m = 2.0 * kPi * (1.0 - b.cos_o) + 0.5 * kPi * (2.0 * tw * so - std::cos(to - 2.0 * tw) - 2.0 * to * so + b.cos_o);
    const double e[3] = {b.hi[0] - b.lo[0], b.hi[1] - b.lo[1], b.hi[2] - b.lo[2]};
    const double area = 2.0 * (e[0] * e[1] + e[1] * e[2] + e[2] * e[0]);
    return b.phi * m * kr * area;
}

inline uint32_t quantize_cos(double c) {
    const double q = std::floor(32767.0 * (std::min(std::max(c, -1.0), 1.0) + 1.0) * 0.5) - 1.0;
    return static_cast<uint32_t>(std::max(q, 0.0));
}

inline float round_down(double x) {
    const double pad = 1e-5 * std::fabs(x) + 1e-30;
    float f = static_cast<float>(x - pad);
    if (static_cast<double>(f) > x - pad) f = std::nextafter(f, -INFINITY);
    return f;
}
inline float round_up(double x) {
    const double pad = 1e-5 * std::fabs(x) + 1e-30;
    float f = static_cast<float>(x + pad);
    if (static_cast<double>(f) < x + pad) f = std::nextafter(f, INFINITY);
    return f;
}

inline LightTreeNode to_node(const LightTreeEmitter &b, uint32_t index) {
    LightTreeNode n{};
    const double ext = std::max({b.hi[0] - b.lo[0], b.hi[1] - b.lo[1], b.hi[2] - b.lo[2]});
    for (int j = 0; j < 3; j++) {
        n.lo[j] = round_down(b.lo[j] - 1e-6 * ext);
        n.hi[j] = round_up(b.hi[j] + 1e-6 * ext);
        n.axis[j] = static_cast<float>(b.axis[j]);
    }
    n.phi = static_cast<float>(b.phi);
    const double to = b.cos_o <= -1.0 ? kPi : std::acos(std::min(b.cos_o, 1.0)) + kConePad;
    const uint32_t qo = to >= kPi ? 0u : quantize_cos(std::cos(to)), qe = quantize_cos(std::cos(0.5 * kPi + kEmitPad));
    n.cos_q = qo | (qe << 16u);
    n.index = index;
    return n;
}

struct Builder {
    const std::vector<LightTreeEmitter> &e;
    LightTreeBuild &out;

    static int ceil_log2(size_t n) {
        int d = 0;
        while ((size_t{1} << d) < n) d++;
        return d;
    }

    // lights[begin, end) under node `node` at `depth` with trail prefix `trail`
    void build(std::vector<uint32_t> &lights, size_t begin, size_t end, uint32_t node, int depth, unsigned long long trail) {
        LightTreeEmitter b;
        for (size_t i = begin; i < end; i++) merge(b, e[lights[i]], i == begin);
        if (end - begin == 1u) {
            out.nodes[node] = to_node(b, kLightTreeLeaf | lights[begin]);
            out.trail[lights[begin]] = trail;
            return;
        }
        size_t mid = begin + (end - begin) / 2u;
        if (depth + ceil_log2(end - begin) < 62) mid = split(lights, begin, end, b);
        const uint32_t child = static_cast<uint32_t>(out.nodes.size());
        out.nodes.resize(out.nodes.size() + 2u);
        out.nodes[node] = to_node(b, child);
        build(lights, begin, mid, child, depth + 1, trail);
        build(lights, mid, end, child + 1u, depth + 1, trail | (1ull << depth));
    }

    // SAOH over 12 buckets per axis of the emitters' centroids; the median of the current order when no axis separates them
    size_t split(std::vector<uint32_t> &lights, size_t begin, size_t end, const LightTreeEmitter &b) {
        constexpr int kBuckets = 12;
        double cmin[3], cmax[3];
        for (int j = 0; j < 3; j++) cmin[j] = INFINITY, cmax[j] = -INFINITY;
        auto centroid = [&](uint32_t l, int j) { return 0.5 * (e[l].lo[j] + e[l].hi[j]); };
        for (size_t i = begin; i < end; i++)
            for (int j = 0; j < 3; j++) {
                cmin[j] = std::min(cmin[j], centroid(lights[i], j));
                cmax[j] = std::max(cmax[j], centroid(lights[i], j));
            }
        const double ext[3] = {b.hi[0] - b.lo[0], b.hi[1] - b.lo[1], b.hi[2] - b.lo[2]};
        const double ext_max = std::max({ext[0], ext[1], ext[2]});
        auto bucket_of = [&](uint32_t l, int j) {
            const int k = static_cast<int>(kBuckets * (centroid(l, j) - cmin[j]) / (cmax[j] - cmin[j]));
            return std::min(std::max(k, 0), kBuckets - 1);
        };
        double best = INFINITY;
        int best_dim = -1, best_bucket = -1;
        for (int j = 0; j < 3; j++) {
            if (!(cmax[j] > cmin[j])) continue;
            LightTreeEmitter bucket[kBuckets];
            bool used[kBuckets] = {};
            for (size_t i = begin; i < end; i++) {
                const int k = bucket_of(lights[i], j);
                merge(bucket[k], e[lights[i]], !used[k]);
                used[k] = true;
            }
            const double kr = ext[j] > 0.0 ? ext_max / ext[j] : 1.0;
            for (int s = 0; s < kBuckets - 1; s++) {
                LightTreeEmitter l, r;
                bool hl = false, hr = false;
                for (int k = 0; k <= s; k++)
                    if (used[k]) merge(l, bucket[k], !hl), hl = true;
                for (int k = s + 1; k < kBuckets; k++)
                    if (used[k]) merge(r, bucket[k], !hr), hr = true;
                if (!hl || !hr) continue;
                const double c = cost(l, kr) + cost(r, kr);
                if (c < best) best = c, best_dim = j, best_bucket = s;
            }
        }
        if (best_dim < 0) return begin + (end - begin) / 2u;
        auto it = std::stable_partition(lights.begin() + static_cast<std::ptrdiff_t>(begin), lights.begin() + static_cast<std::ptrdiff_t>(end),
                                        [&](uint32_t l) { return bucket_of(l, best_dim) <= best_bucket; });
        return static_cast<size_t>(it - lights.begin());
    }
};

}// namespace light_tree_detail

// The bounds of one emitter from its world-space triangles (9 doubles each).  `power_density` = lum(L) * scale: phi is that times
// the area, doubled for a two-sided emitter, whose cone is the whole sphere; a one-sided emitter's cone bounds the geometric
// normals cross(p1 - p0, p2 - p0) of its triangles, the side it emits to.
inline LightTreeEmitter light_tree_emitter(const std::vector<double> &tris, double power_density, bool two_sided) {
    LightTreeEmitter out;
    for (int j = 0; j < 3; j++) out.lo[j] = INFINITY, out.hi[j] = -INFINITY;
    std::vector<double> normals;
    double area = 0.0, sum[3] = {0.0, 0.0, 0.0};
    for (size_t t = 0; t + 9u <= tris.size(); t += 9u) {
        const double *p = tris.data() + t;
        for (int v = 0; v < 3; v++)
            for (int j = 0; j < 3; j++) {
                out.lo[j] = std::min(out.lo[j], p[3 * v + j]);
                out.hi[j] = std::max(out.hi[j], p[3 * v + j]);
            }
        const double a[3] = {p[3] - p[0], p[4] - p[1], p[5] - p[2]}, b[3] = {p[6] - p[0], p[7] - p[1], p[8] - p[2]};
        const double c[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
        const double len = std::sqrt(light_tree_detail::dot3(c, c));
        if (len == 0.0) continue;// a degenerate triangle is never sampled and cannot be hit
        area += 0.5 * len;
        for (int j = 0; j < 3; j++) {
            normals.push_back(c[j] / len);
            sum[j] += c[j] / len;
        }
    }
    out.phi = area > 0.0 ? std::fabs(power_density) * area * (two_sided ? 2.0 : 1.0) : 0.0;
    if (normals.empty()) {
        for (int j = 0; j < 3; j++) out.lo[j] = out.hi[j] = 0.0;
        out.phi = 0.0;
        return out;
    }
    const double sl = std::sqrt(light_tree_detail::dot3(sum, sum));
    if (two_sided || sl < 1e-9 * static_cast<double>(normals.size())) return out;// cos_o = -1
    for (int j = 0; j < 3; j++) out.axis[j] = sum[j] / sl;
    double cmin = 1.0;
    for (size_t i = 0; i < normals.size(); i += 3u) cmin = std::min(cmin, light_tree_detail::dot3(out.axis, normals.data() + i));
    out.cos_o = cmin;
    return out;
}

// The tree over every emitter with phi > 0.  Deterministic: one thread, the emitters' order breaks every tie.
inline LightTreeBuild light_tree_build(const std::vector<LightTreeEmitter> &emitters) {
    LightTreeBuild out;
    out.trail.assign(emitters.size(), 0ull);
    std::vector<uint32_t> lights;
    for (uint32_t l = 0; l < emitters.size(); l++)
        if (emitters[l].phi > 0.0) lights.push_back(l);
    if (lights.empty()) return out;
    out.nodes.reserve(2u * lights.size() - 1u);
    out.nodes.resize(1u);
    light_tree_detail::Builder{emitters, out}.build(lights, 0u, lights.size(), 0u, 0, 0ull);
    return out;
}

// The sides a bottom tree is built for: the triangles emit along cross(p1 - p0, p2 - p0) in object space; an instance whose
// transform has a negative determinant emits along the negated normal (make_interaction takes ng from world-space edges); a
// two-sided light emits along both.
enum LightTreeSide : uint32_t { kLightTreeOneSided = 0u, kLightTreeMirrored = 1u, kLightTreeTwoSided = 2u };

// The bottom tree of one emissive mesh: one emitter per object-space triangle (9 doubles each), phi = its area, its cone the
// triangle's normal on the side it emits to (the whole sphere when two-sided).  Degenerate triangles get phi = 0 and stay out.
inline LightTreeBuild light_tree_build_triangles(const std::vector<double> &tris, LightTreeSide side) {
    std::vector<LightTreeEmitter> emitters;
    emitters.reserve(tris.size() / 9u);
    std::vector<double> one(9u);
    for (size_t t = 0; t + 9u <= tris.size(); t += 9u) {
        std::copy(tris.begin() + static_cast<std::ptrdiff_t>(t), tris.begin() + static_cast<std::ptrdiff_t>(t + 9u), one.begin());
        LightTreeEmitter e = light_tree_emitter(one, 1.0, side == kLightTreeTwoSided);
        if (side == kLightTreeTwoSided) e.phi *= 0.5;
        if (side == kLightTreeMirrored)
            for (double &a : e.axis) a = -a;
        emitters.push_back(e);
    }
    return light_tree_build(emitters);
}

}// namespace lrk
