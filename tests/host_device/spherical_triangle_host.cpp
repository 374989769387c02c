// spherical_triangle_host.cpp — the solid-angle triangle sampler (luisarender_b200/csrc/device/spherical_triangle.h, the header the
// shade kernels include) compiled for the host, so that tests/test_light_solid_angle_cpu.py can check it without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cmath>
#include <cstdint>

#include "../../luisarender_b200/csrc/device/spherical_triangle.h"

namespace {

using lrk::SphVec;

SphVec at(const float *a, int64_t i) { return {a[3 * i], a[3 * i + 1], a[3 * i + 2]}; }

// the shade kernels' light-point pdf in solid angle for a triangle of alias probability 1 (shading.cuh: light_point_pdf on top of
// diffuse_light_evaluate): 1 / omega where the rule picks the spherical sampler, the area pdf d^2 / (A cos) otherwise
float point_pdf(SphVec p, SphVec v0, SphVec v1, SphVec v2, SphVec x, int32_t *spherical) {
    using namespace lrk::spherical_detail;
    const float omega = lrk::solid_angle(p, v0, v1, v2);
    *spherical = lrk::use_spherical(omega);
    if (*spherical) return 1.f / omega;
    const SphVec c = cross(sub(v1, v0), sub(v2, v0));
    const float area = length(c) * .5f;
    const SphVec ng = normalize(c), diff = sub(x, p);
    const float cos_wo = fabsf(dot(normalize(sub(p, x)), ng));
    return cos_wo < 1e-6f ? 0.f : dot(diff, diff) * (1.f / area) * (1.0f / cos_wo);
}

// shading.cuh's sample_uniform_triangle
SphVec uniform_triangle(float ux, float uy) {
    float a, b;
    if (ux < uy) { a = 0.5f * ux; b = -0.5f * ux + uy; }
    else { a = -0.5f * uy + ux; b = 0.5f * uy; }
    return {a, b, 1.0f - a - b};
}

SphVec point_of(SphVec v0, SphVec v1, SphVec v2, SphVec b) {
    return {b.x * v0.x + b.y * v1.x + b.z * v2.x, b.x * v0.y + b.y * v1.y + b.z * v2.y, b.x * v0.z + b.y * v1.z + b.z * v2.z};
}

}// namespace

// n (point, triangle) pairs: p 3 floats each, v 9 floats each
extern "C" void st_solid_angle(int64_t n, const float *p, const float *v, float *out) {
    for (int64_t i = 0; i < n; i++) out[i] = lrk::solid_angle(at(p, i), at(v, 3 * i), at(v, 3 * i + 1), at(v, 3 * i + 2));
}

extern "C" void st_use_spherical(int64_t n, const float *omega, int32_t *out) {
    for (int64_t i = 0; i < n; i++) out[i] = lrk::use_spherical(omega[i]);
}

// one light-point sample per pair, as the shade kernels draw it: the rule picks the spherical sampler or the area sampler; the
// barycentrics, the point, the sampled direction (0 for the area sampler), the pdf and the rule's choice
extern "C" void st_sample(int64_t n, const float *p, const float *v, const float *u, float *bary, float *point, float *dir, float *pdf,
                          int32_t *spherical) {
    for (int64_t i = 0; i < n; i++) {
        const SphVec pi = at(p, i), v0 = at(v, 3 * i), v1 = at(v, 3 * i + 1), v2 = at(v, 3 * i + 2);
        const float omega = lrk::solid_angle(pi, v0, v1, v2);
        SphVec b, w{0.f, 0.f, 0.f};
        if (lrk::use_spherical(omega)) {
            w = lrk::sample_spherical_direction(pi, v0, v1, v2, omega, u[2 * i], u[2 * i + 1]);
            b = lrk::spherical_barycentrics(pi, v0, v1, v2, w);
            const SphVec whole = lrk::sample_spherical_triangle(pi, v0, v1, v2, omega, u[2 * i], u[2 * i + 1]);
            if (whole.x != b.x || whole.y != b.y || whole.z != b.z) b = {NAN, NAN, NAN};// the two steps are the whole sampler
        } else {
            b = uniform_triangle(u[2 * i], u[2 * i + 1]);
        }
        const SphVec x = point_of(v0, v1, v2, b);
        bary[3 * i] = b.x, bary[3 * i + 1] = b.y, bary[3 * i + 2] = b.z;
        point[3 * i] = x.x, point[3 * i + 1] = x.y, point[3 * i + 2] = x.z;
        dir[3 * i] = w.x, dir[3 * i + 1] = w.y, dir[3 * i + 2] = w.z;
        pdf[i] = point_pdf(pi, v0, v1, v2, x, spherical + i);
    }
}

// the pdf an emitter hit at point x evaluates, and the rule's choice there
extern "C" void st_pdf(int64_t n, const float *p, const float *v, const float *x, float *pdf, int32_t *spherical) {
    for (int64_t i = 0; i < n; i++) pdf[i] = point_pdf(at(p, i), at(v, 3 * i), at(v, 3 * i + 1), at(v, 3 * i + 2), at(x, i), spherical + i);
}
