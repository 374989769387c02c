// The denoiser's per-pixel arithmetic (lrk_denoise, DESIGN.md §4 (G-buffer and denoiser)): the guides of a pixel from its
// G-buffer sums, the demodulated input, one à-trous step and the remodulated output.  Plain C++ without CUDA built-ins: the
// sm_90a kernels (denoise.cuh) and tests/host_device compile the same expressions in IEEE fp32 and in this operation order
// (lrk.cu is built with -fmad=false, the host test with -ffp-contract=off), so a numpy restatement can follow them.
//
// The filter is the spatial part of SVGF (Schied et al. 2017): an edge-avoiding à-trous wavelet (Dammertz et al. 2010) over
// albedo-demodulated colour, its luminance edge-stopping scaled by the filtered standard deviation of the pixel's noise.
#pragma once
#include <math.h>

#include "adaptive.h"

namespace lrk {

struct alignas(16) DenoiseVec4 {
    float x, y, z, w;
};

// Edge-stopping parameters.  sigma_n = 128 is applied as seven squarings of the normals' cosine (exact in fp32).
constexpr float kDenoiseSigmaL = 4.f;
constexpr float kDenoiseSigmaZ = 0.05f;
constexpr int kDenoiseNormalSquarings = 7;
constexpr int kDenoiseIterations = 5;// steps 1, 2, 4, 8, 16
constexpr float kDenoiseAlbedoBias = 0.01f;// D = A + 0.01: demodulation never divides by a black albedo

LRK_ADAPTIVE_FN float denoise_lum(float r, float g, float b) { return 0.2126f * r + 0.7152f * g + 0.0722f * b; }

// The guides of one pixel from its G-buffer sums (albedo = (sum albedo, S samples), normal = (sum n, sum t), hits = H):
// albedo_cov = (A = sum albedo / S, H / S), normal_depth = (normalize(sum n) or 0, sum t / H or 0).  All 0 without samples.
LRK_ADAPTIVE_FN void denoise_guides(DenoiseVec4 albedo, DenoiseVec4 normal, float hits, DenoiseVec4 &albedo_cov, DenoiseVec4 &normal_depth) {
    albedo_cov = DenoiseVec4{0.f, 0.f, 0.f, 0.f};
    normal_depth = DenoiseVec4{0.f, 0.f, 0.f, 0.f};
    const float s = albedo.w;
    if (s == 0.f) return;
    albedo_cov = DenoiseVec4{albedo.x / s, albedo.y / s, albedo.z / s, hits / s};
    const float nn = normal.x * normal.x + normal.y * normal.y + normal.z * normal.z;
    if (nn != 0.f) {
        const float inv = 1.0f / sqrtf(nn);
        normal_depth.x = normal.x * inv;
        normal_depth.y = normal.y * inv;
        normal_depth.z = normal.z * inv;
    }
    if (hits > 0.f) normal_depth.w = normal.w / hits;
}

// The filter's input: I = C / D and its variance v / lum(D)^2, D = A + 0.01 (C: the normalised film, v: adaptive_variance).
LRK_ADAPTIVE_FN DenoiseVec4 denoise_input(float cr, float cg, float cb, DenoiseVec4 albedo_cov, float v) {
    const float dr = albedo_cov.x + kDenoiseAlbedoBias, dg = albedo_cov.y + kDenoiseAlbedoBias, db = albedo_cov.z + kDenoiseAlbedoBias;
    const float ld = denoise_lum(dr, dg, db);
    return DenoiseVec4{cr / dr, cg / dg, cb / db, v / (ld * ld)};
}

// The output: D * I, alpha 1.
LRK_ADAPTIVE_FN DenoiseVec4 denoise_output(DenoiseVec4 i, DenoiseVec4 albedo_cov) {
    return DenoiseVec4{(albedo_cov.x + kDenoiseAlbedoBias) * i.x, (albedo_cov.y + kDenoiseAlbedoBias) * i.y, (albedo_cov.z + kDenoiseAlbedoBias) * i.z, 1.f};
}

// w_n = max(0, N_p . N_q)^128; 1 between two pixels without hits, 0 between a pixel with hits and one without.
LRK_ADAPTIVE_FN float denoise_normal_weight(DenoiseVec4 np, float cov_p, DenoiseVec4 nq, float cov_q) {
    const bool hp = cov_p != 0.f, hq = cov_q != 0.f;
    if (!hp && !hq) return 1.f;
    if (hp != hq) return 0.f;
    float c = fmaxf(0.f, np.x * nq.x + np.y * nq.y + np.z * nq.z);
    for (int k = 0; k < kDenoiseNormalSquarings; k++) c = c * c;
    return c;
}

// w = w_l * w_n * w_z of a tap q of pixel p at step `step`; g_p is the pixel's filtered standard deviation.
LRK_ADAPTIVE_FN float denoise_tap_weight(float lum_p, float lum_q, float g_p, DenoiseVec4 np, float cov_p, DenoiseVec4 nq, float cov_q, int step) {
    const float wl = expf(-fabsf(lum_p - lum_q) / (kDenoiseSigmaL * g_p + 1e-6f));
    const float wn = denoise_normal_weight(np, cov_p, nq, cov_q);
    const float wz = expf(-fabsf(np.w - nq.w) / (kDenoiseSigmaZ * static_cast<float>(step) * fmaxf(np.w, nq.w) + 1e-6f));
    return wl * wn * wz;
}

// One à-trous step at pixel (x, y) of a w x h image: in = (I.rgb, var), albedo_cov / normal_depth = the guides.  Taps outside the
// image are skipped.  A tap whose weight h * w is 0 adds nothing, and neither does a variance term whose (h * w)^2 is 0, so that
// an infinite variance (fewer than two samples) never meets a zero weight.
LRK_ADAPTIVE_FN DenoiseVec4 denoise_pixel(const DenoiseVec4 *in, const DenoiseVec4 *albedo_cov, const DenoiseVec4 *normal_depth, int w, int h,
                                          int x, int y, int step) {
    const float b3[3] = {0.25f, 0.5f, 0.25f};
    const float k5[5] = {1.f / 16.f, 1.f / 4.f, 3.f / 8.f, 1.f / 4.f, 1.f / 16.f};
    const int p = y * w + x;
    float g = 0.f;// 3x3 binomial of the variance around p
    for (int dy = -1; dy <= 1; dy++) {
        const int qy = y + dy;
        if (qy < 0 || qy >= h) continue;
        for (int dx = -1; dx <= 1; dx++) {
            const int qx = x + dx;
            if (qx < 0 || qx >= w) continue;
            g += (b3[dy + 1] * b3[dx + 1]) * in[qy * w + qx].w;
        }
    }
    g = sqrtf(g);
    const DenoiseVec4 ip = in[p], np = normal_depth[p];
    const float cov_p = albedo_cov[p].w, lum_p = denoise_lum(ip.x, ip.y, ip.z);
    float sw = 0.f, sr = 0.f, sg = 0.f, sb = 0.f, sv = 0.f;
    for (int dy = -2; dy <= 2; dy++) {
        const int qy = y + step * dy;
        if (qy < 0 || qy >= h) continue;
        for (int dx = -2; dx <= 2; dx++) {
            const int qx = x + step * dx;
            if (qx < 0 || qx >= w) continue;
            const int q = qy * w + qx;
            const DenoiseVec4 iq = in[q];
            const float wt = (dx == 0 && dy == 0) ? 1.f
                                                  : denoise_tap_weight(lum_p, denoise_lum(iq.x, iq.y, iq.z), g, np, cov_p, normal_depth[q], albedo_cov[q].w, step);
            const float hw = (k5[dy + 2] * k5[dx + 2]) * wt;
            if (hw == 0.f) continue;
            sw += hw;
            sr += hw * iq.x;
            sg += hw * iq.y;
            sb += hw * iq.z;
            const float hw2 = hw * hw;
            if (hw2 != 0.f) sv += hw2 * iq.w;
        }
    }
    return DenoiseVec4{sr / sw, sg / sw, sb / sw, sv / (sw * sw)};
}

}// namespace lrk
