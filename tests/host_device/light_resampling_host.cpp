// light_resampling_host.cpp — the resampling of next-event estimation (luisarender_b200/csrc/device/light_resampling.h, the header
// the shade kernels include) compiled for the host, so that tests/test_light_resampling_cpu.py can check it without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>

#include "../../luisarender_b200/csrc/device/light_resampling.h"

namespace {

// the kernels' balance heuristic (shading.cuh)
float balance(float f_pdf, float g_pdf) {
    const float sum = f_pdf + g_pdf;
    return sum == 0.0f ? 0.0f : f_pdf / sum;
}

}// namespace

// n draws over one weight set w[0 .. k): the reservoir's choice per draw (-1: no sample), u[d * k + i] the number of candidate i
extern "C" void lr_choose(int64_t n, int32_t k, const float *w, const float *u, int32_t *out) {
    for (int64_t d = 0; d < n; d++) {
        lrk::LightReservoir r = lrk::light_reservoir_empty();
        for (int32_t i = 0; i < k; i++) lrk::light_reservoir_add(r, static_cast<uint32_t>(i), w[i], u[d * k + i]);
        out[d] = r.w_sum > 0.f ? static_cast<int32_t>(r.chosen) : -1;
    }
}

// the numbers of m candidates for n bounces (u_sel, ul0, ul1 in triple[3 n]) at `depth`: out[(j * m + i) * 4 + ...] = (u_sel, u0, u1,
// u_reservoir) of candidate i, u_reservoir 0 for candidate 0
extern "C" void lr_candidates(int64_t n, const float *triple, uint32_t depth, int32_t m, float *out) {
    for (int64_t j = 0; j < n; j++) {
        const float *t = triple + 3 * j;
        uint32_t state = lrk::light_candidates_seed(t[0], t[1], t[2], depth);
        float *o = out + j * m * 4;
        o[0] = t[0], o[1] = t[1], o[2] = t[2], o[3] = 0.f;
        for (int32_t i = 1; i < m; i++) lrk::light_candidate_numbers(state, o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
    }
}

// The resampled estimate of sum_l c_l * balance(p_l, b_l) on a discrete problem of k lights: source pmf p, rgb contributions c[3 k],
// MIS partner pdfs b.  Candidates pick their light by inverse cdf from their selection number; bounce j's numbers are u[3 j ...].
// out[3 j ...]: the rgb estimate, beta = 1.
extern "C" void lr_estimate(int64_t n, int32_t k, const float *p, const float *c, const float *b, int32_t m, const float *u, float *out) {
    for (int64_t j = 0; j < n; j++) {
        const float *t = u + 3 * j;
        uint32_t state = lrk::light_candidates_seed(t[0], t[1], t[2], 1u);
        lrk::LightReservoir r = lrk::light_reservoir_empty();
        float kept[3] = {0.f, 0.f, 0.f}, p_hat_kept = 0.f;
        for (int32_t i = 0; i < m; i++) {
            float us = t[0], u0 = t[1], u1 = t[2], ur = 0.f;
            if (i != 0) lrk::light_candidate_numbers(state, us, u0, u1, ur);
            int32_t l = 0;
            float cdf = p[0];
            while (l < k - 1 && !(us < cdf)) cdf += p[++l];
            const float mis = balance(p[l], b[l]);
            const float cc[3] = {c[3 * l] * mis, c[3 * l + 1] * mis, c[3 * l + 2] * mis};
            const float p_hat = lrk::resampling_target(cc[0], cc[1], cc[2]);
            if (lrk::light_reservoir_add(r, static_cast<uint32_t>(i), lrk::resampling_weight(p_hat, p[l]), ur)) {
                kept[0] = cc[0], kept[1] = cc[1], kept[2] = cc[2];
                p_hat_kept = p_hat;
            }
        }
        const float w = lrk::light_reservoir_weight(r, static_cast<uint32_t>(m), p_hat_kept);
        for (int q = 0; q < 3; q++) out[3 * j + q] = w > 0.f ? kept[q] * w : 0.f;
    }
}

// M = 1: the contribution c * W / (1 * p_hat) of one candidate of rgb contribution c[3 j ...] and source pdf p[j]
extern "C" void lr_single(int64_t n, const float *c, const float *p, float *out) {
    for (int64_t j = 0; j < n; j++) {
        const float *cc = c + 3 * j;
        const float p_hat = lrk::resampling_target(cc[0], cc[1], cc[2]);
        lrk::LightReservoir r = lrk::light_reservoir_empty();
        lrk::light_reservoir_add(r, 0u, lrk::resampling_weight(p_hat, p[j]), 0.f);
        const float w = lrk::light_reservoir_weight(r, 1u, p_hat);
        for (int q = 0; q < 3; q++) out[3 * j + q] = cc[q] * w;
    }
}
