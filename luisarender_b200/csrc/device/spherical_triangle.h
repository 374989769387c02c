// Solid-angle sampling of a triangle for the option "light_solid_angle" (DESIGN.md §4 (Solid-angle light sampling)): next-event
// estimation picks the point of an emissive triangle uniformly over the spherical triangle it subtends at the shading point (Arvo
// 1995, as pbrt-v4's SampleSphericalTriangle formulates it) instead of uniformly by area, where the solid angle is neither tiny
// nor close to a hemisphere.  The pdf of such a point is then pdf[tri] / Ω, constant over the triangle.
//
// Plain C++ without CUDA built-ins: the shade kernels (shading.cuh) and tests/host_device compile the same expressions.  The pdf is
// never returned by the sampler: a sample and an emitter hit both take it from solid_angle() and use_spherical(), so that for the
// same point the two agree bit for bit (within one compilation).
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define LRK_SPHERICAL_FN __host__ __device__ __forceinline__
#else
#define LRK_SPHERICAL_FN inline
#endif

namespace lrk {

struct SphVec {
    float x, y, z;
};

namespace spherical_detail {
constexpr float kSphericalPi = 3.14159265358979323846f;
LRK_SPHERICAL_FN SphVec sub(SphVec a, SphVec b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
LRK_SPHERICAL_FN SphVec add(SphVec a, SphVec b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
LRK_SPHERICAL_FN SphVec scale(SphVec a, float s) { return {a.x * s, a.y * s, a.z * s}; }
LRK_SPHERICAL_FN float dot(SphVec a, SphVec b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
LRK_SPHERICAL_FN SphVec cross(SphVec a, SphVec b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
LRK_SPHERICAL_FN float length(SphVec a) { return sqrtf(dot(a, a)); }
LRK_SPHERICAL_FN SphVec normalize(SphVec a) { return scale(a, 1.f / sqrtf(dot(a, a))); }
LRK_SPHERICAL_FN float safe_asin(float x) { return asinf(fminf(fmaxf(x, -1.f), 1.f)); }
LRK_SPHERICAL_FN float safe_sqrt(float x) { return sqrtf(fmaxf(x, 0.f)); }
// pbrt-v4's AngleBetween of two unit vectors: accurate near 0 and near pi, where acos(dot) is not
LRK_SPHERICAL_FN float angle_between(SphVec a, SphVec b) {
    return dot(a, b) < 0.f ? kSphericalPi - 2.f * safe_asin(0.5f * length(add(a, b))) : 2.f * safe_asin(0.5f * length(sub(b, a)));
}
// the unit vector of a orthogonal to the unit vector b (Gram-Schmidt)
LRK_SPHERICAL_FN SphVec orthogonal_part(SphVec a, SphVec b) { return normalize(sub(a, scale(b, dot(a, b)))); }
}// namespace spherical_detail

// Solid angle of triangle (v0, v1, v2) seen from p: Van Oosterom & Strackee's tan(Ω / 2) = |a·(b×c)| / (1 + a·b + b·c + c·a) for the
// unit vectors a, b, c from p to the vertices, with both sides multiplied by |v0 - p| |v1 - p| |v2 - p|.  The triple product is
// taken as (v0 - p)·((v1 - v0)×(v2 - v0)), which equals it and keeps its relative precision when the triangle is far away.
// In [0, 2π]; 0 for p on a vertex or in the plane of the triangle outside it.
LRK_SPHERICAL_FN float solid_angle(SphVec p, SphVec v0, SphVec v1, SphVec v2) {
    using namespace spherical_detail;
    const SphVec d0 = sub(v0, p), d1 = sub(v1, p), d2 = sub(v2, p);
    const float l0 = length(d0), l1 = length(d1), l2 = length(d2);
    const float num = fabsf(dot(d0, cross(sub(v1, v0), sub(v2, v0))));
    const float den = l0 * l1 * l2 + dot(d0, d1) * l2 + dot(d1, d2) * l0 + dot(d2, d0) * l1;
    return 2.f * atan2f(num, den);
}

// The one rule: sample the spherical triangle when its solid angle is in pbrt-v4's bounds, by area otherwise (below, the spherical
// construction loses precision in fp32 and area sampling is already near uniform in solid angle; above, the triangle covers
// nearly a hemisphere and the construction degenerates).  False for NaN.
LRK_SPHERICAL_FN bool use_spherical(float omega) { return omega >= 3e-4f && omega <= 6.22f; }

// A direction sampled uniformly in the spherical triangle of (v0, v1, v2) seen from p, as a unit vector.  `omega`: solid_angle(p,
// v0, v1, v2), for which use_spherical holds; u0 picks the area of the sub-triangle (u0 * omega) whose far vertex c' lies on the arc
// from a to c, u1 the point on the arc from b to c'.  The arguments of sinf / cosf stay in [-π, π], where the fast-math
// approximations of the shade kernels' fast variant are accurate to 2^-21 absolute.  The direction to v1 where the construction
// fails (p on the line of an edge).
LRK_SPHERICAL_FN SphVec sample_spherical_direction(SphVec p, SphVec v0, SphVec v1, SphVec v2, float omega, float u0, float u1) {
    using namespace spherical_detail;
    const SphVec a = normalize(sub(v0, p)), b = normalize(sub(v1, p)), c = normalize(sub(v2, p));
    const SphVec n_ab = cross(a, b), n_ca = cross(c, a);
    const float lab = dot(n_ab, n_ab), lca = dot(n_ca, n_ca);
    if (lab == 0.f || lca == 0.f) return b;
    // the interior angle at a, between the planes (a, b) and (a, c)
    const float alpha = angle_between(scale(n_ab, 1.f / sqrtf(lab)), scale(n_ca, -1.f / sqrtf(lca)));
    // pbrt-v4's A' = pi + u0 * (alpha + beta + gamma - pi), here pi + u0 * omega with u0 * omega in [0, 6.22] taken into [-pi, pi]
    const float area = u0 * omega;
    const float t = area > kSphericalPi ? area - 2.f * kSphericalPi : area;
    const float sin_ap = -sinf(t), cos_ap = -cosf(t);
    const float cos_alpha = cosf(alpha), sin_alpha = sinf(alpha);
    const float sin_phi = sin_ap * cos_alpha - cos_ap * sin_alpha;
    const float cos_phi = cos_ap * cos_alpha + sin_ap * sin_alpha;
    const float k1 = cos_phi + cos_alpha;
    const float k2 = sin_phi - sin_alpha * dot(a, b);
    float cos_bp = (k2 + (k2 * cos_phi - k1 * sin_phi) * cos_alpha) / ((k2 * sin_phi + k1 * cos_phi) * sin_alpha);
    cos_bp = fminf(fmaxf(cos_bp, -1.f), 1.f);// NaN clamps to -1
    const float sin_bp = safe_sqrt(1.f - cos_bp * cos_bp);
    const SphVec cp = add(scale(a, cos_bp), scale(orthogonal_part(c, a), sin_bp));
    const float cos_theta = 1.f - u1 * (1.f - dot(cp, b));
    const float sin_theta = safe_sqrt(1.f - cos_theta * cos_theta);
    return add(scale(b, cos_theta), scale(orthogonal_part(cp, b), sin_theta));
}

// Barycentrics (of v0, v1, v2) of the point where the ray p + s w meets the triangle's plane (Moller-Trumbore), clamped to [0, 1]
// and renormalised when they sum to more than 1, as pbrt-v4 does (NaN clamps to 0).  The centroid for w parallel to the plane.
LRK_SPHERICAL_FN SphVec spherical_barycentrics(SphVec p, SphVec v0, SphVec v1, SphVec v2, SphVec w) {
    using namespace spherical_detail;
    const SphVec e1 = sub(v1, v0), e2 = sub(v2, v0);
    const SphVec s1 = cross(w, e2);
    const float divisor = dot(s1, e1);
    if (!(divisor != 0.f)) return {1.f / 3.f, 1.f / 3.f, 1.f / 3.f};
    const float inv = 1.f / divisor;
    const SphVec s = sub(p, v0);
    float b1 = fminf(fmaxf(dot(s, s1) * inv, 0.f), 1.f);
    float b2 = fminf(fmaxf(dot(w, cross(s, e1)) * inv, 0.f), 1.f);
    const float sum = b1 + b2;
    if (sum > 1.f) {
        b1 /= sum;
        b2 /= sum;
    }
    return {fmaxf(1.f - b1 - b2, 0.f), b1, b2};
}

// pbrt-v4's SampleSphericalTriangle without its pdf: the barycentrics of a point sampled uniformly in solid angle
LRK_SPHERICAL_FN SphVec sample_spherical_triangle(SphVec p, SphVec v0, SphVec v1, SphVec v2, float omega, float u0, float u1) {
    return spherical_barycentrics(p, v0, v1, v2, sample_spherical_direction(p, v0, v1, v2, omega, u0, u1));
}

// ---- the receiver-cosine warp of the option "light_receiver" (DESIGN.md §4 (Receiver-aware light sampling)) -------------------------
// pbrt-v4's Triangle::Sample with a receiver normal n: (u0, u1) is first warped by a bilinear density whose corner weights are
// max(0.01, |n . w_k|) for the unit directions w_k to the vertices the corners map to (u1 = 0: v1; (0, 1): v0; (1, 1): v2), so that the
// points follow the receiver's cosine roughly.  The pdf of a point is pdf[tri] / omega * spherical_warp_pdf(...) at the (u0, u1)
// that pbrt-v4's InvertSphericalTriangleSample recovers from the point: the one function a sample and an emitter hit both call.

struct SphWarp {
    float w[4];// corner weights of (0, 0), (1, 0), (0, 1), (1, 1)
};

LRK_SPHERICAL_FN SphWarp spherical_warp_weights(SphVec p, SphVec n, SphVec v0, SphVec v1, SphVec v2) {
    using namespace spherical_detail;
    const float wa = fmaxf(0.01f, fabsf(dot(n, normalize(sub(v0, p)))));
    const float wb = fmaxf(0.01f, fabsf(dot(n, normalize(sub(v1, p)))));
    const float wc = fmaxf(0.01f, fabsf(dot(n, normalize(sub(v2, p)))));
    return {{wb, wb, wa, wc}};
}

namespace spherical_detail {
LRK_SPHERICAL_FN float lerp_t(float t, float a, float b) { return (1.f - t) * a + t * b; }
// pbrt-v4's SampleLinear: x in [0, 1) with density proportional to lerp(x, a, b)
LRK_SPHERICAL_FN float sample_linear(float u, float a, float b) {
    if (u == 0.f && a == 0.f) return 0.f;
    const float x = u * (a + b) / (a + sqrtf(lerp_t(u, a * a, b * b)));
    return fminf(x, 0x1.fffffep-1f);
}
}// namespace spherical_detail

// pbrt-v4's SampleBilinear and BilinearPDF
LRK_SPHERICAL_FN void sample_bilinear(const SphWarp &w, float &u0, float &u1) {
    using namespace spherical_detail;
    const float y = sample_linear(u1, w.w[0] + w.w[1], w.w[2] + w.w[3]);
    const float x = sample_linear(u0, lerp_t(y, w.w[0], w.w[2]), lerp_t(y, w.w[1], w.w[3]));
    u0 = x;
    u1 = y;
}
LRK_SPHERICAL_FN float bilinear_pdf(const SphWarp &w, float x, float y) {
    if (x < 0.f || x > 1.f || y < 0.f || y > 1.f) return 0.f;
    const float sum = w.w[0] + w.w[1] + w.w[2] + w.w[3];
    if (sum == 0.f) return 1.f;
    return 4.f * ((1.f - x) * (1.f - y) * w.w[0] + x * (1.f - y) * w.w[1] + (1.f - x) * y * w.w[2] + x * y * w.w[3]) / sum;
}

// pbrt-v4's InvertSphericalTriangleSample: the (u0, u1) for which sample_spherical_direction returns the unit direction w, with the
// area of the triangle taken as omega (what the sampler uses).  (0.5, 0.5) where the construction degenerates, as pbrt-v4.
LRK_SPHERICAL_FN void invert_spherical_triangle_sample(SphVec p, SphVec v0, SphVec v1, SphVec v2, float omega, SphVec w, float &u0, float &u1) {
    using namespace spherical_detail;
    const SphVec a = normalize(sub(v0, p)), b = normalize(sub(v1, p)), c = normalize(sub(v2, p));
    SphVec n_ab = cross(a, b), n_ca = cross(c, a);
    const float lab = dot(n_ab, n_ab), lca = dot(n_ca, n_ca);
    u0 = 0.5f;
    u1 = 0.5f;
    if (lab == 0.f || lca == 0.f) return;
    n_ab = scale(n_ab, 1.f / sqrtf(lab));
    n_ca = scale(n_ca, 1.f / sqrtf(lca));
    const float alpha = angle_between(n_ab, scale(n_ca, -1.f));
    SphVec cp = cross(cross(b, w), n_ca);
    const float lcp = dot(cp, cp);
    if (lcp == 0.f) return;
    cp = scale(cp, 1.f / sqrtf(lcp));
    if (dot(cp, add(a, c)) < 0.f) cp = scale(cp, -1.f);
    float x;
    if (dot(a, cp) > 0.99999847691f) {// 0.1 degrees
        x = 0.f;
    } else {
        SphVec n_cpb = cross(cp, b), n_acp = cross(a, cp);
        const float l1 = dot(n_cpb, n_cpb), l2 = dot(n_acp, n_acp);
        if (l1 == 0.f || l2 == 0.f) return;
        n_cpb = scale(n_cpb, 1.f / sqrtf(l1));
        n_acp = scale(n_acp, 1.f / sqrtf(l2));
        const float ap = alpha + angle_between(n_ab, n_cpb) + angle_between(n_acp, scale(n_cpb, -1.f)) - kSphericalPi;
        x = ap / omega;
    }
    const float y = (1.f - dot(w, b)) / (1.f - dot(cp, b));
    u0 = fminf(fmaxf(x, 0.f), 1.f);
    u1 = fminf(fmaxf(y, 0.f), 1.f);
}

// The warp's factor of the pdf of point x of the triangle seen from p with the receiver normal n (unit): BilinearPDF at the inverted
// sample of the direction to x.  The caller multiplies pdf[tri] / omega by it; omega as use_spherical requires.
LRK_SPHERICAL_FN float spherical_warp_pdf(SphVec p, SphVec n, SphVec v0, SphVec v1, SphVec v2, float omega, SphVec x) {
    using namespace spherical_detail;
    float u0, u1;
    invert_spherical_triangle_sample(p, v0, v1, v2, omega, normalize(sub(x, p)), u0, u1);
    return bilinear_pdf(spherical_warp_weights(p, n, v0, v1, v2), u0, u1);
}

}// namespace lrk
