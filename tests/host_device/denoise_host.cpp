// denoise_host.cpp — the denoiser's arithmetic (luisarender_b200/csrc/device/denoise.h, the header the sm_90a kernels include)
// compiled for the host and run in the kernels' schedule, so that tests/test_denoise_cpu.py can hold it against a numpy
// restatement without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>
#include <utility>
#include <vector>

#include "../../luisarender_b200/csrc/device/denoise.h"

using lrk::DenoiseVec4;

static DenoiseVec4 at(const float *p, int64_t i) { return DenoiseVec4{p[4 * i], p[4 * i + 1], p[4 * i + 2], p[4 * i + 3]}; }
static void put(float *p, int64_t i, DenoiseVec4 v) {
    p[4 * i] = v.x;
    p[4 * i + 1] = v.y;
    p[4 * i + 2] = v.z;
    p[4 * i + 3] = v.w;
}

extern "C" int denoise_guides_host(int64_t n, const float *albedo, const float *normal, const float *hits, float *albedo_cov, float *normal_depth) {
    for (int64_t i = 0; i < n; i++) {
        DenoiseVec4 ac, nd;
        lrk::denoise_guides(at(albedo, i), at(normal, i), hits[i], ac, nd);
        put(albedo_cov, i, ac);
        put(normal_depth, i, nd);
    }
    return 0;
}

extern "C" int denoise_normal_weight_host(int64_t n, const float *np, const float *cov_p, const float *nq, const float *cov_q, float *w) {
    for (int64_t i = 0; i < n; i++) w[i] = lrk::denoise_normal_weight(at(np, i), cov_p[i], at(nq, i), cov_q[i]);
    return 0;
}

// color: W*H float4 (the normalised film), albedo_cov / normal_depth: W*H float4, variance: W*H float -> out: W*H float4
extern "C" int denoise_host(int w, int h, const float *color, const float *albedo_cov, const float *normal_depth, const float *variance, float *out) {
    const int64_t n = static_cast<int64_t>(w) * h;
    std::vector<DenoiseVec4> ac(n), nd(n), a(n), b(n);
    for (int64_t i = 0; i < n; i++) {
        ac[i] = at(albedo_cov, i);
        nd[i] = at(normal_depth, i);
        a[i] = lrk::denoise_input(color[4 * i], color[4 * i + 1], color[4 * i + 2], ac[i], variance[i]);
    }
    for (int it = 0; it < lrk::kDenoiseIterations; it++) {
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) b[static_cast<int64_t>(y) * w + x] = lrk::denoise_pixel(a.data(), ac.data(), nd.data(), w, h, x, y, 1 << it);
        std::swap(a, b);
    }
    for (int64_t i = 0; i < n; i++) put(out, i, lrk::denoise_output(a[i], ac[i]));
    return 0;
}
