// CPU oracle — TEST INFRASTRUCTURE ONLY (see oracle.h).  Scalar fp32 restatement of the reference's
// per-sample path-tracing estimator; every function cites the reference file:line it follows
// (paths relative to /root/reference).  Compiled with -ffp-contract=off so that a*b+c never fuses
// unless fmaf() is written explicitly (only in the BVH traversal, which has no reference arithmetic:
// the reference delegates traversal to Embree / OptiX, SURVEY.md §8c).
//
// PARITY UNPINNED: the reference holds no golden vectors for this path and cannot be built here.
#include "oracle.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <thread>
#include <vector>

namespace {

// ------------------------------------------------------------------------------------------------
// small vector algebra (component-wise, evaluation order = LuisaCompute's device math,
// src/compute/src/backends/cuda/cuda_builtin/cuda_device_math.h)
// ------------------------------------------------------------------------------------------------
struct V3 {
    float x, y, z;
};
inline V3 v3(float x, float y, float z) { return {x, y, z}; }
inline V3 v3(float s) { return {s, s, s}; }
inline V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
inline V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 operator*(V3 a, V3 b) { return {a.x * b.x, a.y * b.y, a.z * b.z}; }
inline V3 operator*(V3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
inline V3 operator*(float s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
inline V3 operator+(V3 a, float s) { return {a.x + s, a.y + s, a.z + s}; }
inline V3 operator-(V3 a) { return {-a.x, -a.y, -a.z}; }
inline float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }// :lc_dot
inline V3 cross(V3 a, V3 b) { return {a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y}; }
inline float length(V3 a) { return std::sqrt(dot(a, a)); }
// the CUDA backend uses v * rsqrt(dot) (cuda_device_math.h:3509), the CPU backend a true sqrt; the
// oracle and the sm_90a kernels both use the IEEE form v * (1 / sqrt(dot)).
inline V3 normalize(V3 a) { return a * (1.0f / std::sqrt(dot(a, a))); }
inline float sqr(float x) { return x * x; }
inline float saturate(float x) { return std::fmin(std::fmax(x, 0.f), 1.f); }// lc_clamp = min(max(v,lo),hi)
inline float clampf(float x, float lo, float hi) { return std::fmin(std::fmax(x, lo), hi); }
inline float lerp(float a, float b, float t) { return t * (b - a) + a; }// cuda_device_math.h:3353
// The builtin pow of the reference's backends (src/compute/src/backends/cuda/cuda_builtin/cuda_device_math.h:21-36): an exponent
// that is a whole number at run time selects square-and-multiply (exactly rounded products) instead of powf - 1 ulp apart
// from glibc's powf for a few arguments, e.g. a gamma-2.0 texture decode (found by the 320x240 textured reference render).
inline float builtin_pow(float x, float y) {
    const int n = static_cast<int>(y);
    if (static_cast<float>(n) != y) return std::pow(x, y);
    float acc = 1.0f, base = x;
    for (unsigned bits = n < 0 ? 0u - static_cast<unsigned>(n) : static_cast<unsigned>(n); bits != 0u; bits >>= 1) {
        if (bits & 1u) acc *= base;
        base *= base;
    }
    return n < 0 ? 1.0f / acc : acc;
}
inline V3 lerp(V3 a, V3 b, float t) { return t * (b - a) + a; }// src/util/spec.h:272
inline float sign(float x) { return std::copysign(1.0f, x); }// src/compute/include/luisa/dsl/builtin.h:1542-1543
inline V3 reflect(V3 v, V3 n) { return v - 2.0f * dot(v, n) * n; }// cuda_device_math.h:3680-3682
inline V3 face_forward(V3 v, V3 n) { return dot(v, n) < 0.f ? -v : v; }// src/util/scattering.cpp:79-81
inline float max3(V3 a) { return std::fmax(std::fmax(std::fmax(0.f, a.x), a.y), a.z); }// SampledSpectrum::max, src/util/spec.h:125-129

constexpr float kPi = 3.14159265358979323846264338327950288f;
constexpr float kPiOverTwo = 1.57079632679489661923132169163975144f;
constexpr float kPiOverFour = 0.785398163397448309615660845819875721f;
constexpr float kInvPi = 0.318309886183790671537767526745028724f;
constexpr float kOneMinusEpsilon = 0x1.fffffep-1f;

// ------------------------------------------------------------------------------------------------
// RNG: src/util/rng.cpp:53-68 (xxhash32 of a uint4), :128-140 (lcg), src/samplers/independent.cpp:57-82
// ------------------------------------------------------------------------------------------------
inline uint32_t rotl(uint32_t x, uint32_t r) { return (x << r) | (x >> (32u - r)); }

uint32_t xxhash32_uint4(uint32_t px, uint32_t py, uint32_t pz, uint32_t pw) {
    constexpr uint32_t PRIME32_2 = 2246822519u, PRIME32_3 = 3266489917u;
    constexpr uint32_t PRIME32_4 = 668265263u, PRIME32_5 = 374761393u;
    uint32_t h32 = pw + PRIME32_5 + px * PRIME32_3;
    h32 = PRIME32_4 * rotl(h32, 17u);
    h32 += py * PRIME32_3;
    h32 = PRIME32_4 * rotl(h32, 17u);
    h32 += pz * PRIME32_3;
    h32 = PRIME32_4 * rotl(h32, 17u);
    h32 = PRIME32_2 * (h32 ^ (h32 >> 15u));
    h32 = PRIME32_3 * (h32 ^ (h32 >> 13u));
    return h32 ^ (h32 >> 16u);
}

// The reference draws several random numbers inside ONE C++ argument list in a few places (homogeneous.cpp:91,
// layered.cpp: sample(w, lcg(seed), make_float2(lcg(seed), lcg(seed)), mode)); the DSL records in C++ evaluation order, which the
// language leaves unspecified: clang / MSVC go left to right (the oracle's default, and the CUDA kernels'), GCC right to left -
// what the reference built under oracle/ref does.  oracle_set_hg_args_right_to_left(1) mirrors the GCC build for the comparisons.
std::atomic<bool> g_hg_args_right_to_left{false};

inline uint32_t xxhash32_uint3(uint32_t px, uint32_t py, uint32_t pz) {// src/util/rng.cpp:38-51
    constexpr uint32_t PRIME32_2 = 2246822519u, PRIME32_3 = 3266489917u, PRIME32_4 = 668265263u, PRIME32_5 = 374761393u;
    uint32_t h32 = pz + PRIME32_5 + px * PRIME32_3;
    h32 = PRIME32_4 * rotl(h32, 17u);
    h32 += py * PRIME32_3;
    h32 = PRIME32_4 * rotl(h32, 17u);
    h32 = PRIME32_2 * (h32 ^ (h32 >> 15u));
    h32 = PRIME32_3 * (h32 ^ (h32 >> 13u));
    return h32 ^ (h32 >> 16u);
}

inline float lcg(uint32_t &state) {
    state = 1664525u * state + 1013904223u;
    return std::fmin(kOneMinusEpsilon, static_cast<float>(state) * 0x1p-32f);
}

inline uint32_t xxhash32_uint2(uint32_t px, uint32_t py) {// src/util/rng.cpp (xxhash32(uint2))
    constexpr uint32_t PRIME32_2 = 2246822519u, PRIME32_3 = 3266489917u, PRIME32_4 = 668265263u, PRIME32_5 = 374761393u;
    uint32_t h32 = py + PRIME32_5 + px * PRIME32_3;
    h32 = PRIME32_4 * rotl(h32, 17u);
    h32 = PRIME32_2 * (h32 ^ (h32 >> 15u));
    h32 = PRIME32_3 * (h32 ^ (h32 >> 13u));
    return h32 ^ (h32 >> 16u);
}

inline uint32_t reverse_bits32(uint32_t v) {
    v = ((v >> 1u) & 0x55555555u) | ((v & 0x55555555u) << 1u);
    v = ((v >> 2u) & 0x33333333u) | ((v & 0x33333333u) << 2u);
    v = ((v >> 4u) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4u);
    v = ((v >> 8u) & 0x00ff00ffu) | ((v & 0x00ff00ffu) << 8u);
    return (v >> 16u) | (v << 16u);
}

// The samplers (SURVEY.md §8 rows a1 / f2): src/base/sampler.h:42-48 implemented by src/samplers/independent.cpp:57-82,
// pmj02bn.cpp:46-207, sobol.cpp:38-166, padded_sobol.cpp:34-146, zsobol.cpp:40-177.  One struct, switched by lrk_sampler::type.
struct Sampler {
    const lrk_sampler *cfg{nullptr};
    uint32_t seed{0u};
    uint32_t state{0u};      // INDEPENDENT: LCG state
    uint32_t px{0u}, py{0u}, sample_index{0u}, dimension{0u};
    uint64_t sobol_index{0u};// SOBOL: index of the sample in the global sequence; ZSOBOL: Morton index

    static uint32_t permutation_element(uint32_t i, uint32_t l, uint32_t w, uint32_t p) {// pmj02bn.cpp:60-86, padded_sobol.cpp:57-90
        do {
            i ^= p;
            i *= 0xe170893du;
            i ^= p >> 16u;
            i ^= (i & w) >> 4u;
            i ^= p >> 8u;
            i *= 0x0929eb3fu;
            i ^= p >> 23u;
            i ^= (i & w) >> 1u;
            i *= 1u | p >> 27u;
            i *= 0x6935fa69u;
            i ^= (i & w) >> 11u;
            i *= 0x74dcb303u;
            i ^= (i & w) >> 2u;
            i *= 0x9e501cc3u;
            i ^= (i & w) >> 2u;
            i *= 0xc860a3dfu;
            i &= w;
            i ^= i >> 5u;
        } while (i >= l);
        return (i + p) % l;
    }
    static uint32_t fast_owen_scramble(uint32_t seed, uint32_t v) {// sobol.cpp:40-48
        v = reverse_bits32(v);
        v ^= v * 0x3d20adeau;
        v += seed;
        v *= (seed >> 16u) | 1u;
        v ^= v * 0x05526c56u;
        v ^= v * 0x53a22864u;
        return reverse_bits32(v);
    }
    uint32_t sobol_bits(uint64_t a, uint32_t dim) const {// sobol.cpp:52-62: the generator matrix of `dim` applied to the index
        uint32_t v = 0u;
        for (uint32_t i = dim * 52u; a != 0u; a >>= 1u, i++)
            if (a & 1u) v ^= cfg->sobol_matrices[i];
        return v;
    }
    float blue_noise(uint32_t tex_index, uint32_t x, uint32_t y) const {// pmj02bn.cpp:46-51: p.yx % 128, SHORT1 storage = u16 / 65535
        const uint32_t u = y % 128u, v = x % 128u, wv = tex_index % 48u;
        return static_cast<float>(cfg->blue_noise[(static_cast<size_t>(wv) * 128u + v) * 128u + u]) / 65535.f;
    }
    void pmj_sample(uint32_t set_id, uint32_t sample_id, float &x, float &y) const {// pmj02bn.cpp:53-58
        const uint32_t *e = cfg->pmj_samples + (static_cast<size_t>(set_id % 5u) * 65536u + sample_id) * 2u;
        x = static_cast<float>(e[0]) * 0x1p-32f;
        y = static_cast<float>(e[1]) * 0x1p-32f;
    }
    static uint64_t mix_bits(uint64_t v) {// zsobol.cpp:112-119 (the last xor uses the HIGH word: v.hi() >> 1)
        v ^= v >> 31u;
        v *= 0x7fb5d329728ea185ull;
        v ^= v >> 27u;
        v *= 0x81dadef4bc2dd44dull;
        v ^= (v >> 32u) >> 1u;
        return v;
    }
    uint64_t zsobol_sample_index() const {// zsobol.cpp:104-140
        static const uint8_t permutations[24][4] = {
            {0, 1, 2, 3}, {0, 1, 3, 2}, {0, 2, 1, 3}, {0, 2, 3, 1}, {0, 3, 2, 1}, {0, 3, 1, 2}, {1, 0, 2, 3}, {1, 0, 3, 2},
            {1, 2, 0, 3}, {1, 2, 3, 0}, {1, 3, 2, 0}, {1, 3, 0, 2}, {2, 1, 0, 3}, {2, 1, 3, 0}, {2, 0, 1, 3}, {2, 0, 3, 1},
            {2, 3, 0, 1}, {2, 3, 1, 0}, {3, 1, 2, 0}, {3, 1, 0, 2}, {3, 2, 1, 0}, {3, 2, 0, 1}, {3, 0, 2, 1}, {3, 0, 1, 2}};
        uint64_t sample = 0u;
        const bool pow2_samples = (cfg->log2_spp & 1u) != 0u;
        const int last_digit = pow2_samples ? 1 : 0;
        const uint64_t morton = sobol_index;
        for (int i = static_cast<int>(cfg->num_base4_digits) - 1; i >= last_digit; i--) {
            const uint32_t digit_shift = 2u * static_cast<uint32_t>(i) - (pow2_samples ? 1u : 0u);
            const uint32_t digit = static_cast<uint32_t>(morton >> digit_shift) & 3u;
            const uint64_t higher = morton >> (digit_shift + 2u);
            const uint32_t p = static_cast<uint32_t>((mix_bits(higher ^ (static_cast<uint64_t>(dimension * 0x55555555u))) >> 24u) % 24u);
            sample |= static_cast<uint64_t>(permutations[p][digit]) << digit_shift;
        }
        if (pow2_samples) {
            const uint64_t digit = (morton & 1u) ^ (mix_bits((morton >> 1u) ^ static_cast<uint64_t>(dimension * 0x55555555u)) & 1u);
            sample |= digit;
        }
        return sample;
    }
    static uint64_t left_shift2(uint64_t x) {// zsobol.cpp:144-152
        x = (x ^ (x << 16u)) & 0x0000ffff0000ffffull;
        x = (x ^ (x << 8u)) & 0x00ff00ff00ff00ffull;
        x = (x ^ (x << 4u)) & 0x0f0f0f0f0f0f0f0full;
        x = (x ^ (x << 2u)) & 0x3333333333333333ull;
        x = (x ^ (x << 1u)) & 0x5555555555555555ull;
        return x;
    }

    void start(const lrk_scene_desc &sc, uint32_t x, uint32_t y, uint32_t index) {
        cfg = &sc.sampler;
        seed = sc.integrator.sampler_seed;
        px = x;
        py = y;
        sample_index = index;
        switch (cfg->type) {
            case LRK_SAMPLER_PMJ02BN: dimension = 2u; break;
            case LRK_SAMPLER_SOBOL: {// sobol.cpp:64-96,132-137: the index whose first two dimensions fall into this pixel
                dimension = 2u;
                const uint32_t scale = cfg->scale;
                uint32_t m = 0u;
                while ((1u << m) < scale) m++;
                if (m == 0u) { sobol_index = index; break; }
                uint64_t idx = static_cast<uint64_t>(index) << (2u * m);
                uint64_t delta = 0u;
                uint32_t frame = index;
                for (uint32_t c = 0u; frame != 0u; frame >>= 1u, c++)
                    if (frame & 1u) delta ^= cfg->vdc[c];
                uint64_t b = delta ^ ((static_cast<uint64_t>(x) << m) | y);
                for (uint32_t d = 0u; b != 0u; b >>= 1u, d++)
                    if (b & 1u) idx ^= cfg->vdc_inv[d];
                sobol_index = idx;
                break;
            }
            case LRK_SAMPLER_PADDED_SOBOL: dimension = 0u; break;
            case LRK_SAMPLER_ZSOBOL:
                dimension = 0u;
                sobol_index = (((left_shift2(y) << 1u) | left_shift2(x)) << cfg->log2_spp) | index;
                break;
            default: state = xxhash32_uint4(x, y, seed, index); break;
        }
    }
    float generate_1d() {
        switch (cfg->type) {
            case LRK_SAMPLER_PMJ02BN: {// pmj02bn.cpp:179-191
                const uint32_t hash = xxhash32_uint4(px, py, dimension, seed);
                const uint32_t index = permutation_element(sample_index, cfg->spp, cfg->w, hash);
                const float delta = blue_noise(dimension, px, py);
                const float u = (static_cast<float>(index) + delta) * (1.f / static_cast<float>(cfg->spp));
                dimension += 1u;
                return std::fmin(std::fmax(u, 0.f), kOneMinusEpsilon);
            }
            case LRK_SAMPLER_SOBOL: {// sobol.cpp:148-154
                if (dimension >= 1024u) dimension = 2u;
                const uint32_t hash = xxhash32_uint2(dimension, seed);
                const float u = static_cast<float>(fast_owen_scramble(hash, sobol_bits(sobol_index, dimension))) * 0x1p-32f;
                dimension += 1u;
                return std::fmin(std::fmax(u, 0.f), kOneMinusEpsilon);
            }
            case LRK_SAMPLER_PADDED_SOBOL: {// padded_sobol.cpp:124-133
                const uint32_t hash = xxhash32_uint4(px, py, sample_index ^ seed, dimension);
                uint32_t w = cfg->spp - 1u;
                w |= w >> 1u; w |= w >> 2u; w |= w >> 4u; w |= w >> 8u; w |= w >> 16u;
                const uint32_t index = permutation_element(sample_index, cfg->spp, w, hash);
                const float u = std::fmin(static_cast<float>(fast_owen_scramble(hash, sobol_bits(index, 0u))) * 0x1p-32f, kOneMinusEpsilon);
                dimension += 1u;
                return u;
            }
            case LRK_SAMPLER_ZSOBOL: {// zsobol.cpp:164-169
                const uint64_t si = zsobol_sample_index();
                const uint32_t hash = cfg->zsobol_hash[dimension * 2u];
                dimension = (dimension + 1u) % 1024u;
                return std::fmin(static_cast<float>(fast_owen_scramble(hash, sobol_bits(si, 0u))) * 0x1p-32f, kOneMinusEpsilon);
            }
            default: return lcg(state);
        }
    }
    void generate_2d(float &ux, float &uy) {
        switch (cfg->type) {
            case LRK_SAMPLER_PMJ02BN: {// pmj02bn.cpp:192-207
                uint32_t index = sample_index;
                const uint32_t pmj_instance = dimension / 2u;
                if (pmj_instance >= 5u) {
                    const uint32_t hash = xxhash32_uint4(px, py, dimension, seed);
                    index = permutation_element(sample_index, cfg->spp, cfg->w, hash);
                }
                float sx, sy;
                pmj_sample(pmj_instance, index, sx, sy);
                const float u0 = sx + blue_noise(dimension, px, py), u1 = sy + blue_noise(dimension + 1u, px, py);
                ux = u0 - std::floor(u0);
                uy = u1 - std::floor(u1);
                dimension += 2u;
                return;
            }
            case LRK_SAMPLER_SOBOL: {// sobol.cpp:155-163
                if (dimension + 1u >= 1024u) dimension = 2u;
                const uint32_t hx = xxhash32_uint2(dimension, seed), hy = xxhash32_uint2(dimension + 1u, seed);
                const float x = static_cast<float>(fast_owen_scramble(hx, sobol_bits(sobol_index, dimension))) * 0x1p-32f;
                const float y = static_cast<float>(fast_owen_scramble(hy, sobol_bits(sobol_index, dimension + 1u))) * 0x1p-32f;
                dimension += 2u;
                ux = std::fmin(std::fmax(x, 0.f), kOneMinusEpsilon);
                uy = std::fmin(std::fmax(y, 0.f), kOneMinusEpsilon);
                return;
            }
            case LRK_SAMPLER_PADDED_SOBOL: {// padded_sobol.cpp:134-146
                const uint32_t hx = xxhash32_uint4(px, py, sample_index ^ seed, dimension);
                const uint32_t hy = xxhash32_uint4(px, py, sample_index ^ seed, dimension + 1u);
                uint32_t w = cfg->spp - 1u;
                w |= w >> 1u; w |= w >> 2u; w |= w >> 4u; w |= w >> 8u; w |= w >> 16u;
                const uint32_t index = permutation_element(sample_index, cfg->spp, w, hx);
                ux = std::fmin(static_cast<float>(fast_owen_scramble(hx, sobol_bits(index, 0u))) * 0x1p-32f, kOneMinusEpsilon);
                uy = std::fmin(static_cast<float>(fast_owen_scramble(hy, sobol_bits(index, 1u))) * 0x1p-32f, kOneMinusEpsilon);
                dimension += 2u;
                return;
            }
            case LRK_SAMPLER_ZSOBOL: {// zsobol.cpp:170-177
                const uint64_t si = zsobol_sample_index();
                const uint32_t hx = cfg->zsobol_hash[dimension * 2u], hy = cfg->zsobol_hash[dimension * 2u + 1u];
                dimension = (dimension + 2u) % 1024u;
                ux = std::fmin(static_cast<float>(fast_owen_scramble(hx, sobol_bits(si, 0u))) * 0x1p-32f, kOneMinusEpsilon);
                uy = std::fmin(static_cast<float>(fast_owen_scramble(hy, sobol_bits(si, 1u))) * 0x1p-32f, kOneMinusEpsilon);
                return;
            }
            default:
                ux = lcg(state);
                uy = lcg(state);
                return;
        }
    }
    void generate_pixel_2d(float &ux, float &uy) {// sampler.h:48: generate_2d unless the sampler stratifies the pixel itself
        switch (cfg->type) {
            case LRK_SAMPLER_PMJ02BN: {// pmj02bn.cpp:209-213
                const uint32_t tx = px % cfg->tile, ty = py % cfg->tile;
                const size_t offset = static_cast<size_t>(tx + ty * cfg->tile) * cfg->spp + sample_index;
                ux = cfg->pmj_pixel_samples[offset * 2u];
                uy = cfg->pmj_pixel_samples[offset * 2u + 1u];
                return;
            }
            case LRK_SAMPLER_SOBOL: {// sobol.cpp:164-170: the unscrambled first two dimensions, relative to the pixel
                const float x = static_cast<float>(sobol_bits(sobol_index, 0u)) * 0x1p-32f;
                const float y = static_cast<float>(sobol_bits(sobol_index, 1u)) * 0x1p-32f;
                const float s = static_cast<float>(cfg->scale);
                ux = std::fmin(std::fmax(x * s - static_cast<float>(px), 0.f), kOneMinusEpsilon);
                uy = std::fmin(std::fmax(y * s - static_cast<float>(py), 0.f), kOneMinusEpsilon);
                return;
            }
            default: generate_2d(ux, uy); return;
        }
    }
};

// ------------------------------------------------------------------------------------------------
// warps: src/util/sampling.cpp:13-31 (concentric disk, cosine hemisphere), :89-98 (triangle),
// src/util/sampling.h:38-70 (alias table), sampling.cpp:133-155 (balance heuristic)
// ------------------------------------------------------------------------------------------------
inline void sample_uniform_disk_concentric(float ux, float uy, float &dx, float &dy) {
    float x = ux * 2.0f - 1.0f, y = uy * 2.0f - 1.0f;
    bool p = std::fabs(x) > std::fabs(y);
    float r = p ? x : y;
    float theta = p ? kPiOverFour * (y / x) : kPiOverTwo - kPiOverFour * (x / y);
    dx = r * std::cos(theta);
    dy = r * std::sin(theta);
}
inline V3 sample_cosine_hemisphere(float ux, float uy) {
    float dx, dy;
    sample_uniform_disk_concentric(ux, uy, dx, dy);
    float z = std::sqrt(std::fmax(1.0f - dx * dx - dy * dy, 0.0f));
    return {dx, dy, z};
}
inline V3 sample_uniform_triangle(float ux, float uy) {
    float a, b;
    if (ux < uy) { a = 0.5f * ux; b = -0.5f * ux + uy; }
    else { a = -0.5f * uy + ux; b = 0.5f * uy; }
    return {a, b, 1.0f - a - b};
}
inline V3 sample_uniform_sphere(float u0, float u1) {// sampling.cpp:99-108
    float z = 1.0f - 2.0f * u0;
    float r = std::sqrt(std::fmax(1.0f - z * z, 0.0f));
    float phi = 2.0f * kPi * u1;
    return {r * std::cos(phi), r * std::sin(phi), z};
}
inline float balance_heuristic(float f_pdf, float g_pdf) {
    float sum_f = 1.0f * f_pdf;// nf = 1
    float sum = sum_f + 1.0f * g_pdf;
    return sum == 0.0f ? 0.0f : sum_f / sum;
}
template<typename ProbAt, typename AliasAt>
inline void sample_alias_table(ProbAt prob_at, AliasAt alias_at, uint32_t n, float u_in, uint32_t &index, float &uu) {
    float u = u_in * static_cast<float>(n);
    // cast<uint>(u) then clamp to [0, n-1]
    uint32_t i = static_cast<uint32_t>(u);
    i = std::min(std::max(i, 0u), n - 1u);
    float u_remapped = u - std::floor(u);// fract
    float prob = prob_at(i);
    bool keep = u_remapped < prob;
    index = keep ? i : alias_at(i);
    uu = keep ? u_remapped / prob : (u_remapped - prob) / (1.0f - prob);
}

// ------------------------------------------------------------------------------------------------
// Frame: src/util/frame.cpp:21-42
// ------------------------------------------------------------------------------------------------
struct Frame {
    V3 s, t, n;
    static Frame make(V3 n) {
        float sgn = sign(n.z);
        float a = -1.f / (sgn + n.z);
        float b = n.x * n.y * a;
        V3 s = v3(1.f + sgn * sqr(n.x) * a, sgn * b, -sgn * n.x);
        V3 t = v3(b, sgn + sqr(n.y) * a, -n.y);
        return {normalize(s), normalize(t), n};
    }
    static Frame make(V3 n, V3 s) {
        V3 ss = normalize(s - n * dot(n, s));
        V3 tt = normalize(cross(n, ss));
        return {ss, tt, n};
    }
    V3 local_to_world(V3 d) const { return normalize(d.x * s + d.y * t + d.z * n); }
    V3 world_to_local(V3 d) const { return normalize(v3(dot(d, s), dot(d, t), dot(d, n))); }
};

// local-frame trigonometry: src/util/frame.h:50-71
inline float cos_theta(V3 w) { return w.z; }
inline float cos2_theta(V3 w) { return sqr(w.z); }
inline float abs_cos_theta(V3 w) { return std::fabs(w.z); }
inline float sin2_theta(V3 w) { return saturate(1.0f - cos2_theta(w)); }
inline float sin_theta(V3 w) { return std::sqrt(sin2_theta(w)); }
inline float tan_theta(V3 w) { return sin_theta(w) / cos_theta(w); }
inline float tan2_theta(V3 w) { return sin2_theta(w) / cos2_theta(w); }
inline float cos_phi(V3 w) {
    float s = sin_theta(w);
    return s == 0.0f ? 1.0f : clampf(w.x / s, -1.0f, 1.0f);
}
inline float sin_phi(V3 w) {
    float s = sin_theta(w);
    return s == 0.0f ? 0.0f : clampf(w.y / s, -1.0f, 1.0f);
}
inline float cos2_phi(V3 w) { return sqr(cos_phi(w)); }
inline float sin2_phi(V3 w) { return sqr(sin_phi(w)); }
inline bool same_hemisphere(V3 w, V3 wp) { return w.z * wp.z > 0.0f; }
inline float abs_dot(V3 a, V3 b) { return std::fabs(dot(a, b)); }

// ------------------------------------------------------------------------------------------------
// Shape::Handle::decode: src/base/shape.cpp:72-93
// ------------------------------------------------------------------------------------------------
struct ShapeHandle {
    uint32_t buffer_base, flags, surface_tag, light_tag, medium_tag, tri_count;
    float shadow_terminator, intersection_offset;
    bool has_vertex_normal() const { return flags & LRK_SHAPE_HAS_VERTEX_NORMAL; }
    bool has_vertex_uv() const { return flags & LRK_SHAPE_HAS_VERTEX_UV; }
    bool has_surface() const { return flags & LRK_SHAPE_HAS_SURFACE; }
    bool has_light() const { return flags & LRK_SHAPE_HAS_LIGHT; }
    bool has_medium() const { return flags & LRK_SHAPE_HAS_MEDIUM; }
};
ShapeHandle decode_handle(const uint32_t c[4]) {
    ShapeHandle h;
    h.buffer_base = c[0] >> 10u;
    h.flags = c[0] & 1023u;
    h.surface_tag = (c[1] >> 12u) & 4095u;
    h.light_tag = c[1] & 4095u;
    h.medium_tag = (c[1] >> 24u) & 255u;
    h.tri_count = c[2];
    auto fixed = [](uint32_t x) { return static_cast<float>(x & 0xffffu) * (1.0f / 65536.f); };
    h.shadow_terminator = fixed(c[3] >> 16u);
    float off = fixed(c[3] & 0xffffu);
    h.intersection_offset = clampf(off * 255.f + 1.f, 1.f, 256.f);
    return h;
}

// ------------------------------------------------------------------------------------------------
// Interaction and hit reconstruction: src/base/geometry.cpp:281-389, src/base/interaction.{h,cpp}
// ------------------------------------------------------------------------------------------------
struct Interaction {
    ShapeHandle shape{};
    V3 pg{}, ng{}, ps{};
    float u{}, v{};
    Frame shading{};
    uint32_t inst{~0u}, prim{~0u};
    float prim_area{};
    bool back_facing{};
    bool valid() const { return inst != ~0u; }
};

// src/compute/src/dsl/rtx/ray.cpp:16-23 — integer-ULP offset along n
V3 offset_ray_origin(V3 p, V3 n) {
    constexpr float origin = 1.0f / 32.0f;
    constexpr float float_scale = 1.0f / 65536.0f;
    constexpr float int_scale = 256.0f;
    auto one = [&](float pc, float nc) {
        int32_t of_i = static_cast<int32_t>(int_scale * nc);
        int32_t bits;
        std::memcpy(&bits, &pc, 4);
        bits += pc < 0.0f ? -of_i : of_i;
        float p_i;
        std::memcpy(&p_i, &bits, 4);
        return std::fabs(pc) < origin ? pc + float_scale * nc : p_i;
    };
    return {one(p.x, n.x), one(p.y, n.y), one(p.z, n.z)};
}

// src/base/interaction.cpp:13-30
V3 p_robust(const Interaction &it, V3 w) {
    bool front = dot(it.shading.n, w) > 0.f;
    V3 n = front ? it.ng : -it.ng;
    return offset_ray_origin(it.pg, it.shape.intersection_offset * n);
}
lrk_ray make_ray(V3 o, V3 d, float tmin, float tmax) { return {{o.x, o.y, o.z}, tmin, {d.x, d.y, d.z}, tmax}; }
lrk_ray spawn_ray(const Interaction &it, V3 wi) {
    return make_ray(p_robust(it, wi), wi, 0.f, std::numeric_limits<float>::max());
}
lrk_ray spawn_ray_to(const Interaction &it, V3 p) {
    V3 p_from = p_robust(it, p - it.pg);
    V3 L = p - p_from;
    float d = length(L);
    return make_ray(p_from, L * (1.f / d), 0.f, d * .9999f);
}

struct Mat34 {// row-major 3x4; columns c0..c2 are the 3x3 part, c3 the translation
    const float *m;
    V3 col(int j) const { return {m[j], m[4 + j], m[8 + j]}; }
};
// float3x3 * float3 = v.x*m[0] + v.y*m[1] + v.z*m[2] (cuda_device_math.h:2746)
inline V3 mul3(const Mat34 &m, V3 v) { return v.x * m.col(0) + v.y * m.col(1) + v.z * m.col(2); }

inline V3 vertex_p(const lrk_vertex &v) { return {v.p[0], v.p[1], v.p[2]}; }
inline V3 vertex_n(const lrk_vertex &v) { return {v.n[0], v.n[1], v.n[2]}; }

// Geometry::shading_point, src/base/geometry.cpp:345-389, then the Interaction constructor
// (src/base/interaction.h:97-101): shading frame = Frame::make(ns, dpdu)
Interaction make_interaction(const lrk_scene_desc &sc, uint32_t inst_id, uint32_t prim_id, V3 bary, bool use_wo, V3 wo,
                             V3 p_from_for_back_facing) {
    Interaction it;
    const auto &inst = sc.instances[inst_id];
    it.shape = decode_handle(inst.handle);
    const auto &mesh = sc.meshes[it.shape.buffer_base >> 2u];
    const auto &tri = sc.triangles[mesh.triangle_offset + prim_id];
    const auto &v0 = sc.vertices[mesh.vertex_offset + tri.i0];
    const auto &v1 = sc.vertices[mesh.vertex_offset + tri.i1];
    const auto &v2 = sc.vertices[mesh.vertex_offset + tri.i2];
    Mat34 m{inst.object_to_world};
    V3 t = m.col(3);
    V3 p0 = vertex_p(v0), p1 = vertex_p(v1), p2 = vertex_p(v2);
    V3 ns_local = bary.x * vertex_n(v0) + bary.y * vertex_n(v1) + bary.z * vertex_n(v2);
    float duv0x = v1.uv[0] - v0.uv[0], duv0y = v1.uv[1] - v0.uv[1];
    float duv1x = v2.uv[0] - v0.uv[0], duv1y = v2.uv[1] - v0.uv[1];
    float det = duv0x * duv1y - duv0y * duv1x;
    float inv_det = 1.f / det;
    V3 dp0 = p1 - p0, dp1 = p2 - p0;
    V3 dpdu_local = (dp0 * duv1y - dp1 * duv0y) * inv_det;
    V3 p = mul3(m, bary.x * p0 + bary.y * p1 + bary.z * p2) + t;
    V3 c = cross(mul3(m, dp0), mul3(m, dp1));
    float area = length(c) * .5f;
    V3 ng = normalize(c);
    Frame fallback = Frame::make(ng);
    V3 dpdu = det == 0.f ? fallback.s : mul3(m, dpdu_local);
    // mn = transpose(inverse(m)), GLM-style inverse (cuda_device_math.h:3615-3630)
    V3 m0 = m.col(0), m1 = m.col(1), m2 = m.col(2);
    float one_over_det = 1.0f / (m0.x * (m1.y * m2.z - m2.y * m1.z) - m1.x * (m0.y * m2.z - m2.y * m0.z) +
                                 m2.x * (m0.y * m1.z - m1.y * m0.z));
    V3 i0 = v3((m1.y * m2.z - m2.y * m1.z) * one_over_det, (m2.y * m0.z - m0.y * m2.z) * one_over_det,
               (m0.y * m1.z - m1.y * m0.z) * one_over_det);
    V3 i1 = v3((m2.x * m1.z - m1.x * m2.z) * one_over_det, (m0.x * m2.z - m2.x * m0.z) * one_over_det,
               (m1.x * m0.z - m0.x * m1.z) * one_over_det);
    V3 i2 = v3((m1.x * m2.y - m2.x * m1.y) * one_over_det, (m2.x * m0.y - m0.x * m2.y) * one_over_det,
               (m0.x * m1.y - m1.x * m0.y) * one_over_det);
    // transpose: columns of mn are the rows of the inverse
    V3 mn0 = v3(i0.x, i1.x, i2.x), mn1 = v3(i0.y, i1.y, i2.y), mn2 = v3(i0.z, i1.z, i2.z);
    V3 ns = it.shape.has_vertex_normal() ? normalize(ns_local.x * mn0 + ns_local.y * mn1 + ns_local.z * mn2) : ng;
    if (it.shape.has_vertex_uv()) {
        it.u = bary.x * v0.uv[0] + bary.y * v1.uv[0] + bary.z * v2.uv[0];
        it.v = bary.x * v0.uv[1] + bary.y * v1.uv[1] + bary.z * v2.uv[1];
    } else {
        it.u = bary.y;
        it.v = bary.z;
    }
    it.pg = p;
    it.ps = p;
    it.ng = ng;
    it.prim_area = area;
    it.shading = Frame::make(face_forward(ns, ng), dpdu);
    it.inst = inst_id;
    it.prim = prim_id;
    // geometry.cpp:290 (hit): dot(wo, ng) < 0 ; uniform.cpp:121 (sampled light point): dot(ng, p_from - p) < 0
    it.back_facing = use_wo ? dot(wo, ng) < 0.0f : dot(ng, p_from_for_back_facing - p) < 0.f;
    return it;
}

Interaction interaction_from_hit(const lrk_scene_desc &sc, const lrk_ray &ray, const lrk_hit &hit) {
    if (hit.inst == ~0u) return {};
    V3 bary = v3(1.f - hit.bary[0] - hit.bary[1], hit.bary[0], hit.bary[1]);
    V3 wo = -v3(ray.d[0], ray.d[1], ray.d[2]);
    return make_interaction(sc, hit.inst, hit.prim, bary, true, wo, v3(0.f));
}

// ------------------------------------------------------------------------------------------------
// BVH traversal.  No reference arithmetic exists for this (Embree / OptiX); these rules are OURS and the
// sm_90a kernel follows exactly the same ones (luisarender_b200/csrc/device/traverse.cuh):
//   * slab test in the fused form t = fma(plane, inv_d, -o*inv_d), |d| clamped to >= 1e-30 before 1/d,
//     child hit <=> max(tnear, tmin) <= min(tfar, t_best);
//   * both children hit -> visit the one with the smaller entry distance first (ties: child 0);
//   * Moeller-Trumbore in object space with explicit fma dot/cross, accept tmin < t < t_best (t == t_best: the lower (inst, prim) wins),
//     u >= 0, v >= 0, u + v <= 1, det != 0;
//   * instances: ray transformed with world_to_object (fma chains), direction NOT renormalised (t is shared).
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kSentinelDone = 0xfffffffdu;
constexpr uint32_t kSentinelExit = 0xfffffffeu;

struct TraceCounters {
    uint64_t nodes{0}, tris{0}, xforms{0};
};

inline float fdot(V3 a, V3 b) { return std::fmaf(a.x, b.x, std::fmaf(a.y, b.y, a.z * b.z)); }
inline V3 fcross(V3 a, V3 b) {
    return {std::fmaf(a.y, b.z, -(a.z * b.y)), std::fmaf(a.z, b.x, -(a.x * b.z)), std::fmaf(a.x, b.y, -(a.y * b.x))};
}
inline float safe_rcp(float d) {
    float a = std::fabs(d) < 1e-30f ? std::copysign(1e-30f, d) : d;
    return 1.0f / a;
}

struct RaySetup {
    V3 o, d, inv, ood;
    void set(V3 oo, V3 dd) {
        o = oo;
        d = dd;
        inv = v3(safe_rcp(dd.x), safe_rcp(dd.y), safe_rcp(dd.z));
        ood = v3(oo.x * inv.x, oo.y * inv.y, oo.z * inv.z);
    }
};

// exit distance (t_best included) scaled by 1 + 2^-20 before the comparison: the rounding of the slab distances is relative to the
// distance from the origin, which the boxes' pad does not cover (derivation at kSlabExitScale in traverse.cuh)
constexpr float kSlabExitScale = 0x1.00001p+0f;

inline bool slab(const float lo[3], const float hi[3], const RaySetup &r, float tmin, float tbest, float &tnear) {
    float t0x = std::fmaf(lo[0], r.inv.x, -r.ood.x), t1x = std::fmaf(hi[0], r.inv.x, -r.ood.x);
    float t0y = std::fmaf(lo[1], r.inv.y, -r.ood.y), t1y = std::fmaf(hi[1], r.inv.y, -r.ood.y);
    float t0z = std::fmaf(lo[2], r.inv.z, -r.ood.z), t1z = std::fmaf(hi[2], r.inv.z, -r.ood.z);
    float tn = std::fmax(std::fmax(std::fmin(t0x, t1x), std::fmin(t0y, t1y)), std::fmax(std::fmin(t0z, t1z), tmin));
    float tf = std::fmin(std::fmin(std::fmax(t0x, t1x), std::fmax(t0y, t1y)), std::fmin(std::fmax(t0z, t1z), tbest)) * kSlabExitScale;
    tnear = tn;
    return tn <= tf;
}

// Geometry::_alpha_skip, src/base/geometry.cpp:165-192 (defined with the texture code below)
bool alpha_skip(const lrk_scene_desc &sc, uint32_t inst_id, uint32_t prim_id, float bu, float bv);

lrk_hit trace_brute(const lrk_scene_desc &sc, const lrk_ray &ray, bool any_hit);
std::atomic<bool> g_trace_brute_force{false};// diagnostic: every ray through the brute-force loop (oracle_set_trace_brute_force)
lrk_hit trace_bvh(const lrk_scene_desc &sc, const lrk_ray &ray, bool any_hit, TraceCounters *cnt) {
    if (g_trace_brute_force.load(std::memory_order_relaxed)) return trace_brute(sc, ray, any_hit);
    lrk_hit best{~0u, ~0u, {0.f, 0.f}};
    float tbest = ray.tmax;
    const float tmin = ray.tmin;
    RaySetup world, cur;
    world.set(v3(ray.o[0], ray.o[1], ray.o[2]), v3(ray.d[0], ray.d[1], ray.d[2]));
    cur = world;
    uint32_t stack[512];// one entry per level: the host builder caps a hierarchy's depth at 48 + log2(n) (bvh.cpp), TLAS + BLAS stay far below
    int sp = 0;
    stack[sp++] = kSentinelDone;
    uint32_t node = sc.tlas_root;
    bool in_blas = false;
    uint32_t cur_inst = ~0u;
    for (;;) {
        while (!(node & LRK_BVH_LEAF)) {
            const auto &n = sc.bvh_nodes[node];
            if (cnt) cnt->nodes++;
            float tn0, tn1;
            bool h0 = slab(n.lo0, n.hi0, cur, tmin, tbest, tn0);
            bool h1 = slab(n.lo1, n.hi1, cur, tmin, tbest, tn1);
            if (h0 && h1) {
                bool first0 = tn0 <= tn1;
                stack[sp++] = first0 ? n.ref1 : n.ref0;
                node = first0 ? n.ref0 : n.ref1;
            } else if (h0) {
                node = n.ref0;
            } else if (h1) {
                node = n.ref1;
            } else {
                node = stack[--sp];
            }
        }
        if (node == kSentinelDone) break;
        if (node == kSentinelExit) {
            cur = world;
            in_blas = false;
            node = stack[--sp];
            continue;
        }
        if (node == LRK_BVH_EMPTY) {
            node = stack[--sp];
            continue;
        }
        if (in_blas) {
            uint32_t first = node & 0x0fffffffu;
            uint32_t count = ((node >> 28u) & 7u) + 1u;
            for (uint32_t k = 0; k < count; k++) {
                const float *tv = sc.tri_verts + static_cast<size_t>(first + k) * 12u;
                if (cnt) cnt->tris++;
                V3 p0 = v3(tv[0], tv[1], tv[2]), p1 = v3(tv[4], tv[5], tv[6]), p2 = v3(tv[8], tv[9], tv[10]);
                V3 e1 = p1 - p0, e2 = p2 - p0;
                V3 pvec = fcross(cur.d, e2);
                float det = fdot(e1, pvec);
                if (!(det != 0.0f)) continue;
                float inv_det = 1.0f / det;
                V3 tvec = cur.o - p0;
                float u = fdot(tvec, pvec) * inv_det;
                if (!(u >= 0.0f && u <= 1.0f)) continue;
                V3 qvec = fcross(tvec, e1);
                float v = fdot(cur.d, qvec) * inv_det;
                if (!(v >= 0.0f && u + v <= 1.0f)) continue;
                float t = fdot(e2, qvec) * inv_det;
                uint32_t prim;
                std::memcpy(&prim, &tv[3], 4);
                // exact ties in t (coincident faces of two shapes) go to the lower (instance, primitive), which is what the
                // brute-force loop below - and oracle/ref's backend - yield: the result does not depend on the visiting order
                const bool tie = t == tbest && best.inst != ~0u && (cur_inst < best.inst || (cur_inst == best.inst && prim < best.prim));
                if (!(t > tmin && (t < tbest || tie))) continue;
                if (alpha_skip(sc, cur_inst, prim, u, v)) continue;// candidate not committed (geometry.cpp:248-279)
                tbest = t;
                best = {cur_inst, prim, {u, v}};
                if (any_hit) return best;
            }
            node = stack[--sp];
        } else {
            cur_inst = node & 0x7fffffffu;
            if (cnt) cnt->xforms++;
            const auto &inst = sc.instances[cur_inst];
            const float *w = inst.world_to_object;
            V3 o = world.o, d = world.d;
            V3 oo = v3(std::fmaf(w[0], o.x, std::fmaf(w[1], o.y, std::fmaf(w[2], o.z, w[3]))),
                       std::fmaf(w[4], o.x, std::fmaf(w[5], o.y, std::fmaf(w[6], o.z, w[7]))),
                       std::fmaf(w[8], o.x, std::fmaf(w[9], o.y, std::fmaf(w[10], o.z, w[11]))));
            V3 dd = v3(std::fmaf(w[0], d.x, std::fmaf(w[1], d.y, w[2] * d.z)),
                       std::fmaf(w[4], d.x, std::fmaf(w[5], d.y, w[6] * d.z)),
                       std::fmaf(w[8], d.x, std::fmaf(w[9], d.y, w[10] * d.z)));
            cur.set(oo, dd);
            stack[sp++] = kSentinelExit;
            in_blas = true;
            node = sc.meshes[inst.mesh].bvh_root;
        }
    }
    return best;
}

lrk_hit trace_brute(const lrk_scene_desc &sc, const lrk_ray &ray, bool any_hit) {
    lrk_hit best{~0u, ~0u, {0.f, 0.f}};
    float tbest = ray.tmax;
    V3 o = v3(ray.o[0], ray.o[1], ray.o[2]), d = v3(ray.d[0], ray.d[1], ray.d[2]);
    for (uint32_t i = 0; i < sc.instance_count; i++) {
        const auto &inst = sc.instances[i];
        if (!inst.visible) continue;
        const float *w = inst.world_to_object;
        V3 oo = v3(std::fmaf(w[0], o.x, std::fmaf(w[1], o.y, std::fmaf(w[2], o.z, w[3]))),
                   std::fmaf(w[4], o.x, std::fmaf(w[5], o.y, std::fmaf(w[6], o.z, w[7]))),
                   std::fmaf(w[8], o.x, std::fmaf(w[9], o.y, std::fmaf(w[10], o.z, w[11]))));
        V3 dd = v3(std::fmaf(w[0], d.x, std::fmaf(w[1], d.y, w[2] * d.z)),
                   std::fmaf(w[4], d.x, std::fmaf(w[5], d.y, w[6] * d.z)),
                   std::fmaf(w[8], d.x, std::fmaf(w[9], d.y, w[10] * d.z)));
        const auto &mesh = sc.meshes[inst.mesh];
        for (uint32_t k = 0; k < mesh.triangle_count; k++) {
            const auto &tri = sc.triangles[mesh.triangle_offset + k];
            V3 p0 = vertex_p(sc.vertices[mesh.vertex_offset + tri.i0]);
            V3 p1 = vertex_p(sc.vertices[mesh.vertex_offset + tri.i1]);
            V3 p2 = vertex_p(sc.vertices[mesh.vertex_offset + tri.i2]);
            V3 e1 = p1 - p0, e2 = p2 - p0;
            V3 pvec = fcross(dd, e2);
            float det = fdot(e1, pvec);
            if (!(det != 0.0f)) continue;
            float inv_det = 1.0f / det;
            V3 tvec = oo - p0;
            float u = fdot(tvec, pvec) * inv_det;
            if (!(u >= 0.0f && u <= 1.0f)) continue;
            V3 qvec = fcross(tvec, e1);
            float v = fdot(dd, qvec) * inv_det;
            if (!(v >= 0.0f && u + v <= 1.0f)) continue;
            float t = fdot(e2, qvec) * inv_det;
            if (!(t > ray.tmin && t < tbest)) continue;
            if (alpha_skip(sc, i, k, u, v)) continue;
            tbest = t;
            best = {i, k, {u, v}};
            if (any_hit) return best;
        }
    }
    return best;
}

// ------------------------------------------------------------------------------------------------
// Camera: src/base/filter.cpp:50-64, src/base/camera.cpp:212-224, src/cameras/pinhole.cpp:60-67
// ------------------------------------------------------------------------------------------------
void sample_filter(const lrk_camera &cam, float ux, float uy, float &ox, float &oy, float &weight) {
    constexpr uint32_t n = LRK_FILTER_LUT_SIZE - 1u;
    uint32_t iy, ix;
    float fy, fx;
    auto prob = [&](uint32_t i) { return cam.filter_alias_probs[i]; };
    auto alias = [&](uint32_t i) { return cam.filter_alias_indices[i]; };
    sample_alias_table(prob, alias, n, ux, iy, fy);
    sample_alias_table(prob, alias, n, uy, ix, fx);
    float pdf = cam.filter_pdf[iy] * cam.filter_pdf[ix];
    float f = lerp(cam.filter_lut[ix], cam.filter_lut[ix + 1u], fx) * lerp(cam.filter_lut[iy], cam.filter_lut[iy + 1u], fy);
    float px = static_cast<float>(ix) + fx, py = static_cast<float>(iy) + fy;
    constexpr float inv_size = 1.0f / static_cast<float>(LRK_FILTER_LUT_SIZE);
    ox = (px * inv_size * 2.0f - 1.0f) * cam.filter_radius + cam.filter_shift[0];
    oy = (py * inv_size * 2.0f - 1.0f) * cam.filter_radius + cam.filter_shift[1];
    weight = f / pdf;
}

lrk_ray generate_camera_ray(const lrk_camera &cam, uint32_t px, uint32_t py, float ux, float uy, float &weight) {
    float ox, oy, fw;
    sample_filter(cam, ux, uy, ox, oy, fw);
    float pixel_x = static_cast<float>(px) + .5f + ox;
    float pixel_y = static_cast<float>(py) + .5f + oy;
    float rx = static_cast<float>(cam.resolution[0]), ry = static_cast<float>(cam.resolution[1]);
    float k = cam.tan_half_fov / ry;
    float p_x = (pixel_x * 2.0f - rx) * k;
    float p_y = (pixel_y * 2.0f - ry) * k;
    V3 direction = normalize(v3(p_x, -p_y, -1.f));
    weight = 1.f * fw;
    Mat34 c2w{cam.camera_to_world};
    // c2w * (0,0,0,1) = 0*c0 + 0*c1 + 0*c2 + 1*c3 (cuda_device_math.h:2754)
    V3 o = 0.f * c2w.col(0) + 0.f * c2w.col(1) + 0.f * c2w.col(2) + 1.f * c2w.col(3);
    V3 d = normalize(mul3(c2w, direction));
    return make_ray(o, d, 0.f, std::numeric_limits<float>::max());
}

// ------------------------------------------------------------------------------------------------
// Lights: src/lights/diffuse.cpp:67-88, src/lightsamplers/uniform.cpp:50-65,78-137,
// src/base/light_sampler.cpp:57-78,116-119
// ------------------------------------------------------------------------------------------------
struct LightEval {
    V3 L{0.f, 0.f, 0.f};
    float pdf{0.f};
};

// image emission: max(texel.xyz, 0) at the interaction's uv (Texture::Instance::evaluate_illuminant_spectrum, texture.cpp:47-57 -
// no extend_color_to_rgb on the non-static path; decode_illuminant, srgb.cpp:48-54).  Defined with the texture code below.
V3 light_emission(const lrk_scene_desc &sc, const lrk_light &light, float u, float v);
LightEval diffuse_light_evaluate(const lrk_scene_desc &sc, const Interaction &it_light, V3 p_from) {
    const auto &light = sc.lights[it_light.shape.light_tag];
    const auto &mesh = sc.meshes[it_light.shape.buffer_base >> 2u];
    float pdf_triangle = sc.pdf[mesh.triangle_offset + it_light.prim];
    float pdf_area = pdf_triangle / it_light.prim_area;
    float cos_wo = abs_dot(normalize(p_from - it_light.pg), it_light.ng);
    V3 L = light_emission(sc, light, it_light.u, it_light.v) * light.scale;
    V3 diff = it_light.pg - p_from;
    float pdf = dot(diff, diff) * pdf_area * (1.0f / cos_wo);
    bool invalid = std::fabs(cos_wo) < 1e-6f || (!light.two_sided && it_light.back_facing);
    LightEval e;
    e.L = invalid ? v3(0.f) : L;
    e.pdf = invalid ? 0.0f : pdf;
    return e;
}

inline float env_prob(const lrk_scene_desc &sc) { return sc.environment.present ? sc.environment.env_prob : 0.f; }
LightEval evaluate_hit(const lrk_scene_desc &sc, const Interaction &it, V3 p_from) {
    LightEval e = diffuse_light_evaluate(sc, it, p_from);
    float n = static_cast<float>(sc.light_count);
    e.pdf *= (1.f - env_prob(sc)) / n;// uniform.cpp:63
    return e;
}
// the environment (defined with the texture code below): src/environments/spherical.cpp:83-137
struct EnvSample {
    LightEval eval;
    V3 wi{};
};
LightEval environment_evaluate(const lrk_scene_desc &sc, V3 wi);
EnvSample environment_sample(const lrk_scene_desc &sc, float u0, float u1);

struct LightSample {
    LightEval eval;
    lrk_ray shadow_ray{};
};

LightSample sample_light(const lrk_scene_desc &sc, const Interaction &it_from, float u_sel, float u0, float u1) {
    LightSample s;
    const float ep = env_prob(sc);
    if (sc.light_count == 0u && ep == 0.f) return s;// !has_lighting (light_sampler.cpp:58)
    float n = static_cast<float>(sc.light_count);
    // UniformLightSamplerInstance::select, uniform.cpp:78-90
    bool is_env = ep == 1.f;
    uint32_t tag = 0u;
    float sel_prob = 1.f;
    if (ep == 0.f) {
        tag = static_cast<uint32_t>(clampf(u_sel * n, 0.f, n - 1.f));
        sel_prob = 1.f / n;
    } else if (ep != 1.f) {
        float uu = (u_sel - ep) / (1.f - ep);
        tag = static_cast<uint32_t>(clampf(uu * n, 0.f, n - 1.f));
        is_env = u_sel < ep;
        sel_prob = is_env ? ep : (1.f - ep) / n;
    }
    if (is_env) {// sample_environment + Sample::from_environment, light_sampler.cpp:84-90,120-123
        EnvSample es = environment_sample(sc, u0, u1);
        s.eval = es.eval;
        s.eval.pdf *= sel_prob;
        s.shadow_ray = spawn_ray(it_from, es.wi);
        return s;
    }
    const auto &handle = sc.light_handles[tag];
    ShapeHandle light_inst = decode_handle(sc.instances[handle.instance_id].handle);
    const auto &mesh = sc.meshes[light_inst.buffer_base >> 2u];
    uint32_t triangle_id;
    float ux;
    sample_alias_table([&](uint32_t i) { return sc.alias[mesh.triangle_offset + i].prob; },
                       [&](uint32_t i) { return sc.alias[mesh.triangle_offset + i].alias; },
                       light_inst.tri_count, u0, triangle_id, ux);
    V3 uvw = sample_uniform_triangle(ux, u1);
    Interaction it_light = make_interaction(sc, handle.instance_id, triangle_id, uvw, false, v3(0.f), it_from.pg);
    // the light sampler builds this interaction itself with the full shading attributes (uniform.cpp:108-123: shading_point, so
    // the uv is the sampled point's) and asks the light's closure to evaluate() it; DiffuseLightClosure::sample is not on this path
    s.eval = diffuse_light_evaluate(sc, it_light, it_from.ps);
    s.eval.pdf *= sel_prob;
    s.shadow_ray = spawn_ray_to(it_from, it_light.pg);
    return s;
}

// ------------------------------------------------------------------------------------------------
// Surfaces.  Validation wrapper: src/base/surface.cpp:35-68.
// ------------------------------------------------------------------------------------------------
struct SurfEval {
    V3 f{0.f, 0.f, 0.f};
    float pdf{0.f};
};
struct SurfSample {
    SurfEval eval;
    V3 wi{0.f, 0.f, 1.f};
    uint32_t event{0u};// Surface::event_*, src/base/surface.h:37-40
};

inline bool validate_surface_sides(V3 ng, V3 ns, V3 wo, V3 wi) {
    float flip = sign(dot(ng, ns));
    return sign(flip * dot(wo, ns)) == sign(dot(wo, ng)) && sign(flip * dot(wi, ns)) == sign(dot(wi, ng));
}

// --- Matte / Oren-Nayar: src/surfaces/matte.cpp:78-134, src/util/scattering.cpp:247-264,370-400
struct OrenNayar {
    V3 r;
    float a, b;
    OrenNayar(V3 R, float sigma) : r{R} {
        float sigma2 = sqr(sigma * (kPi / 180.0f));// DSL radians(): x * (pi/180), builtin.h:1523-1525
        a = 1.f - (sigma2 / (2.f * sigma2 + 0.66f));
        b = 0.45f * sigma2 / (sigma2 + 0.09f);
    }
    V3 evaluate(V3 wo, V3 wi) const {
        float s = same_hemisphere(wo, wi) ? kInvPi : 0.f;
        float sinThetaI = sin_theta(wi), sinThetaO = sin_theta(wo);
        float sinPhiI = sin_phi(wi), cosPhiI = cos_phi(wi);
        float sinPhiO = sin_phi(wo), cosPhiO = cos_phi(wo);
        float dCos = cosPhiI * cosPhiO + sinPhiI * sinPhiO;
        float maxCos = (sinThetaI > 1e-4f && sinThetaO > 1e-4f) ? std::fmax(0.f, dCos) : 0.f;
        float absCosThetaI = abs_cos_theta(wi), absCosThetaO = abs_cos_theta(wo);
        float sinAlpha = absCosThetaI > absCosThetaO ? sinThetaO : sinThetaI;
        float tanBeta = absCosThetaI > absCosThetaO ? sinThetaI / absCosThetaI : sinThetaO / absCosThetaO;
        float scale = a + b * maxCos * sinAlpha * tanBeta;
        return s * scale * r;
    }
};
inline float lambert_pdf(V3 wo, V3 wi) { return same_hemisphere(wo, wi) ? abs_cos_theta(wi) * kInvPi : 0.f; }

SurfEval matte_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi) {
    OrenNayar refl{v3(s.p[0], s.p[1], s.p[2]), s.p[3]};
    V3 wo_local = it.shading.world_to_local(wo);
    V3 wi_local = it.shading.world_to_local(wi);
    SurfEval e;
    e.f = refl.evaluate(wo_local, wi_local) * abs_cos_theta(wi_local);
    e.pdf = lambert_pdf(wo_local, wi_local);
    return e;
}
SurfSample matte_sample(const lrk_surface &s, const Interaction &it, V3 wo, float, float u0, float u1) {
    OrenNayar refl{v3(s.p[0], s.p[1], s.p[2]), s.p[3]};
    V3 wo_local = it.shading.world_to_local(wo);
    V3 wi_local = sample_cosine_hemisphere(u0, u1);
    wi_local.z *= sign(cos_theta(wo_local));
    float pdf = lambert_pdf(wo_local, wi_local);// valid == true
    V3 f = refl.evaluate(wo_local, wi_local);
    SurfSample out;
    out.wi = it.shading.local_to_world(wi_local);
    out.eval.f = f * abs_cos_theta(wi_local);
    out.eval.pdf = pdf;
    return out;
}

// --- microfacet machinery: src/util/scattering.cpp:30-52,117-237,286-320
float fresnel_dielectric(float cosThetaI_in, float etaI_in, float etaT_in) {
    float cosThetaI = clampf(cosThetaI_in, -1.f, 1.f);
    bool entering = cosThetaI > 0.f;
    float etaI = entering ? etaI_in : etaT_in;
    float etaT = entering ? etaT_in : etaI_in;
    cosThetaI = std::fabs(cosThetaI);
    float sinThetaI = std::sqrt(std::fmax(0.f, 1.f - sqr(cosThetaI)));
    float sinThetaT = etaI / etaT * sinThetaI;
    float cosThetaT = std::sqrt(std::fmax(0.f, 1.f - sqr(sinThetaT)));
    float Rparl = (etaT * cosThetaI - etaI * cosThetaT) / (etaT * cosThetaI + etaI * cosThetaT);
    float Rperp = (etaI * cosThetaI - etaT * cosThetaT) / (etaI * cosThetaI + etaT * cosThetaT);
    float fr = (Rparl * Rparl + Rperp * Rperp) * .5f;
    return sinThetaT < 1.f ? fr : 1.f;
}

struct TrowbridgeReitz {
    float ax, ay;
    TrowbridgeReitz(float x, float y) : ax{std::fmax(x, 1e-4f)}, ay{std::fmax(y, 1e-4f)} {}// scattering.cpp:131-132
    float D(V3 wh) const {
        float tan2Theta = tan2_theta(wh);
        float cos4Theta = sqr(cos2_theta(wh));
        float e = tan2Theta * (sqr(cos_phi(wh) / ax) + sqr(sin_phi(wh) / ay));
        float d = 1.0f / (kPi * ax * ay * cos4Theta * sqr(1.f + e));
        return std::isinf(tan2Theta) ? 0.f : d;
    }
    float Lambda(V3 w) const {
        float tanTheta = std::fabs(tan_theta(w));
        float alpha2 = cos2_phi(w) * sqr(ax) + sin2_phi(w) * sqr(ay);
        float alpha2Tan2Theta = alpha2 * sqr(tanTheta);
        float L = (-1.f + std::sqrt(1.f + alpha2Tan2Theta)) * .5f;
        return std::isinf(tanTheta) ? 0.f : L;
    }
    float G1(V3 w) const { return 1.0f / (1.0f + Lambda(w)); }
    float G(V3 wo, V3 wi) const { return 1.0f / (1.0f + Lambda(wo) + Lambda(wi)); }
    float pdf(V3 wo, V3 wh) const { return D(wh) * G1(wo) * abs_dot(wo, wh) / abs_cos_theta(wo); }
    static void sample11(float cosTheta, float U1, float U2, float &slope_x, float &slope_y) {
        if (cosTheta <= .9999f) {
            float sinTheta = std::sqrt(std::fmax(0.f, 1.f - sqr(cosTheta)));
            float tanTheta = sinTheta / cosTheta;
            float a = 1.f / tanTheta;
            float G1 = 2.f / (1.f + std::sqrt(1.f + 1.f / sqr(a)));
            float A = 2.f * U1 / G1 - 1.f;
            float tmp = std::fmin(1.f / (sqr(A) - 1.f), 1e10f);
            float B = tanTheta;
            float D = std::sqrt(std::fmax(sqr(B * tmp) - (sqr(A) - sqr(B)) * tmp, 0.f));
            float slope_x_1 = B * tmp - D;
            float slope_x_2 = B * tmp + D;
            slope_x = (A < 0.f || slope_x_2 * tanTheta > 1.f) ? slope_x_1 : slope_x_2;
            float S = U2 > .5f ? 1.f : -1.f;
            float V = U2 > .5f ? 2.f * (U2 - .5f) : 2.f * (.5f - U2);
            float z = (V * (V * (V * 0.27385f - 0.73369f) + 0.46341f)) /
                      (V * (V * (V * 0.093073f + 0.309420f) - 1.000000f) + 0.597999f);
            slope_y = S * z * std::sqrt(1.f + sqr(slope_x));
        } else {
            float r = std::sqrt(U1 / (1.f - U1));
            float phi = (2.f * kPi) * U2;
            slope_x = r * std::cos(phi);
            slope_y = r * std::sin(phi);
        }
    }
    V3 sample_wh(V3 wo, float u0, float u1) const {
        float s = sign(cos_theta(wo));
        V3 wi = s * wo;
        V3 wiStretched = normalize(v3(ax * wi.x, ay * wi.y, wi.z));
        float sx, sy;
        sample11(cos_theta(wiStretched), u0, u1, sx, sy);
        float cp = cos_phi(wiStretched), sp = sin_phi(wiStretched);
        float rx = cp * sx - sp * sy;
        float ry = sp * sx + cp * sy;
        rx = ax * rx;
        ry = ay * ry;
        V3 wh = normalize(v3(-rx, -ry, 1.f));
        return s * wh;
    }
};

// --- BxDF library shared by the Mirror / Glass / Metal / Plastic closures and pinned against the reference's own code
//     (oracle/ref, tests/test_ref_pins.py): src/util/scattering.cpp:14-125 (refract, Fresnel terms, spherical helpers),
//     :238-345 (BxDF base, Lambertian, microfacet reflection / transmission), :402-447 (FresnelBlend);
//     src/util/sampling.cpp:99-175
inline bool refract(V3 wi, V3 n, float eta, V3 &wt) {// scattering.cpp:14-28
    float cosThetaI = dot(n, wi);
    float sin2ThetaI = std::fmax(0.0f, 1.f - sqr(cosThetaI));
    float sin2ThetaT = sqr(eta) * sin2ThetaI;
    float cosThetaT = std::sqrt(1.f - sin2ThetaT);
    wt = (eta * cosThetaI - cosThetaT) * n - eta * wi;
    return sin2ThetaT < 1.0f;
}
inline V3 spherical_direction(float sinTheta, float cosTheta, float phi) {// :81-83
    return {sinTheta * std::cos(phi), sinTheta * std::sin(phi), cosTheta};
}
inline float spherical_theta(V3 v) { return std::acos(clampf(v.z, -1.f, 1.f)); }// :89-91
inline float spherical_phi(V3 v) {// :93-96
    float p = std::atan2(v.y, v.x);
    return p < 0.f ? p + 2.f * kPi : p;
}
inline V3 exp3(V3 a) { return {std::exp(a.x), std::exp(a.y), std::exp(a.z)}; }
inline V3 vdiv(V3 a, V3 b) { return {a.x / b.x, a.y / b.y, a.z / b.z}; }
inline V3 vsqrt(V3 a) { return {std::sqrt(a.x), std::sqrt(a.y), std::sqrt(a.z)}; }
inline V3 operator-(float s, V3 a) { return {s - a.x, s - a.y, s - a.z}; }
inline V3 operator-(V3 a, float s) { return {a.x - s, a.y - s, a.z - s}; }
inline V3 operator/(V3 a, float s) { return {a.x / s, a.y / s, a.z / s}; }
V3 fresnel_conductor(float cosThetaI, float etai, V3 etat, V3 k) {// :56-75
    cosThetaI = clampf(cosThetaI, -1.f, 1.f);
    V3 eta = etat / etai;
    V3 etak = k / etai;
    float cosThetaI2 = cosThetaI * cosThetaI;
    float sinThetaI2 = 1.f - cosThetaI2;
    V3 eta2 = eta * eta;
    V3 etak2 = etak * etak;
    V3 t0 = eta2 - etak2 - sinThetaI2;
    V3 a2plusb2 = vsqrt(t0 * t0 + 4.f * eta2 * etak2);
    V3 t1 = a2plusb2 + cosThetaI2;
    V3 a = vsqrt(.5f * (a2plusb2 + t0));
    V3 t2 = 2.f * cosThetaI * a;
    V3 Rs = vdiv(t1 - t2, t1 + t2);
    V3 t3 = cosThetaI2 * a2plusb2 + sinThetaI2 * sinThetaI2;
    V3 t4 = t2 * sinThetaI2;
    V3 Rp = vdiv(Rs * (t3 - t4), t3 + t4);// Rs * (t3 - t4) / (t3 + t4): left to right
    return .5f * (Rp + Rs);
}
inline float fresnel_dielectric_integral(float eta) {// :98-108; polynomial() = Horner from the last coefficient, spec.h:45-51
    float r;
    if (eta == 1.f) {
        r = 0.f;
    } else if (eta < 1.f) {
        r = eta * (eta * (eta * -0.90663979f + 2.23559031f) + -2.09069066f) + 0.75985009f;
    } else {
        float x = 1.f / eta;
        r = x * (x * -1.18995376f + 0.21762732f) + 0.97945724f;
    }
    return saturate(r);
}

// the Fresnel term of a MicrofacetReflection: dielectric (glass, plastic coat), conductor (metal), Schlick (mirror.cpp:67-79)
struct FresnelTerm {
    enum Kind { DIELECTRIC, CONDUCTOR, SCHLICK } kind{DIELECTRIC};
    float eta_i{1.f}, eta_t{1.5f};
    V3 eta{}, k{}, r0{};
    V3 evaluate(float cosI) const {
        switch (kind) {
            case DIELECTRIC: return v3(fresnel_dielectric(cosI, eta_i, eta_t));// :243-245
            case CONDUCTOR: return fresnel_conductor(std::fabs(cosI), eta_i, eta, k);// :239-241
            default: {
                float m = saturate(1.f - cosI);
                float weight = sqr(sqr(m)) * m;
                return (1.f - weight) * r0 + weight;
            }
        }
    }
    static FresnelTerm dielectric(float ei, float et) { FresnelTerm f; f.kind = DIELECTRIC; f.eta_i = ei; f.eta_t = et; return f; }
    static FresnelTerm conductor(float ei, V3 eta, V3 k) { FresnelTerm f; f.kind = CONDUCTOR; f.eta_i = ei; f.eta = eta; f.k = k; return f; }
    static FresnelTerm schlick(V3 r0) { FresnelTerm f; f.kind = SCHLICK; f.r0 = r0; return f; }
};

struct BxDFSample {
    V3 wi{0.f, 0.f, 0.f};
    bool valid{false};
};
inline BxDFSample lambert_sample_wi(V3 wo, float u0, float u1) {// BxDF::sample_wi :260-264
    V3 wi = sample_cosine_hemisphere(u0, u1);
    wi.z *= sign(cos_theta(wo));
    return {wi, true};
}
inline V3 lambert_evaluate(V3 r, V3 wo, V3 wi) { return r * (same_hemisphere(wo, wi) ? kInvPi : 0.f); }// :266-269

struct MicrofacetReflection {// :290-329
    V3 r;
    TrowbridgeReitz d;
    FresnelTerm fr;
    V3 evaluate(V3 wo, V3 wi) const {
        V3 wh = wi + wo;
        V3 f = v3(0.f);
        if (same_hemisphere(wo, wi) && any_nonzero_v(wh)) {
            wh = normalize(wh);
            V3 F = fr.evaluate(dot(wi, face_forward(wh, v3(0.f, 0.f, 1.f))));
            float D = d.D(wh);
            float G = d.G(wo, wi);
            float cos_o = cos_theta(wo), cos_i = cos_theta(wi);
            f = r * F * std::fabs(0.25f * D * G / (cos_i * cos_o));
        }
        return f;
    }
    BxDFSample sample_wi(V3 wo, float u0, float u1) const {
        V3 wh = d.sample_wh(wo, u0, u1);
        V3 wi = reflect(-wo, wh);
        return {wi, same_hemisphere(wo, wi)};
    }
    float pdf(V3 wo, V3 wi) const {
        float p = 0.f;
        V3 wh = wi + wo;
        if (same_hemisphere(wo, wi) && any_nonzero_v(wh)) {
            wh = normalize(wh);
            p = d.pdf(wo, wh) / (4.f * dot(wo, wh));
        }
        return p;
    }
    static bool any_nonzero_v(V3 w) { return w.x != 0.f || w.y != 0.f || w.z != 0.f; }
};

struct MicrofacetTransmission {// :331-380
    V3 t;
    TrowbridgeReitz d;
    float eta_a, eta_b;
    bool importance{false};// TransportMode::IMPORTANCE: f *= eta^2 (:340-342); only the Layered surface asks for it
    V3 evaluate(V3 wo, V3 wi) const {
        float cosThetaO = cos_theta(wo), cosThetaI = cos_theta(wi);
        float eta = cosThetaO > 0.f ? eta_b / eta_a : eta_a / eta_b;
        V3 wh = normalize(wo + wi * eta);
        wh = sign(cos_theta(wh)) * wh;
        V3 f = v3(0.f);
        if (!same_hemisphere(wo, wi) && cosThetaO != 0.f && cosThetaI != 0.f && dot(wo, wh) * dot(wi, wh) < 0.f) {
            float G = d.G(wo, wi);
            float sqrtDenom = dot(wo, wh) + eta * dot(wi, wh);
            float F = fresnel_dielectric(dot(wo, wh), eta_a, eta_b);
            float D = d.D(wh);
            f = (1.f - F) * t * D * G * dot(wi, wh) * dot(wo, wh) / (cosThetaI * cosThetaO * sqr(sqrtDenom));
            if (importance) f = f * sqr(eta);
        }
        return f;
    }
    BxDFSample sample_wi(V3 wo, float u0, float u1) const {
        float eta = cos_theta(wo) > 0.f ? eta_a / eta_b : eta_b / eta_a;
        V3 wh = d.sample_wh(wo, u0, u1);
        V3 wi = v3(0.f);
        bool refr = refract(wo, wh, eta, wi);
        return {wi, refr && !same_hemisphere(wo, wi)};
    }
    float pdf(V3 wo, V3 wi) const {
        float p = 0.f;
        bool entering = cos_theta(wo) > 0.f;
        float eta = entering ? eta_b / eta_a : eta_a / eta_b;
        V3 wh = normalize(wo + wi * eta);
        if (!same_hemisphere(wo, wi) && dot(wo, wh) * dot(wi, wh) < 0.f) {
            float sqrtDenom = dot(wo, wh) + eta * dot(wi, wh);
            float dwh_dwi = sqr(eta / sqrtDenom) * abs_dot(wi, wh);
            p = d.pdf(wo, wh) * dwh_dwi;
        }
        return p;
    }
};

struct FresnelBlend {// :402-447
    V3 rd, rs;
    float rd_ratio;
    TrowbridgeReitz d;
    FresnelBlend(V3 Rd, V3 Rs, TrowbridgeReitz dist, float ratio = .5f) : rd{Rd}, rs{Rs}, rd_ratio{clampf(ratio, .05f, .95f)}, d{dist} {}
    static float pow5(float v) { return sqr(sqr(v)) * v; }
    V3 schlick(float cosTheta) const { return rs + pow5(1.f - cosTheta) * (1.f - rs); }
    V3 evaluate(V3 wo, V3 wi) const {
        V3 wh = wi + wo;
        bool valid = same_hemisphere(wo, wi) && MicrofacetReflection::any_nonzero_v(wh);
        wh = normalize(wh);
        float D = d.D(wh);
        float absCosThetaI = abs_cos_theta(wi), absCosThetaO = abs_cos_theta(wo);
        V3 diffuse = (28.f / (23.f * kPi)) * rd * (1.f - rs) * (1.f - pow5(1.f - .5f * absCosThetaI)) * (1.f - pow5(1.f - .5f * absCosThetaO));
        V3 specular = D / (4.f * abs_dot(wi, wh) * std::fmax(absCosThetaI, absCosThetaO)) * schlick(dot(wi, wh));
        return valid ? diffuse + specular : v3(0.f);
    }
    BxDFSample sample_wi(V3 wo, float u0, float u1) const {
        V3 wi;
        if (u0 < rd_ratio) {
            u0 = u0 / rd_ratio;
            wi = sample_cosine_hemisphere(u0, u1);
            wi.z *= sign(cos_theta(wo));
        } else {
            u0 = (u0 - rd_ratio) / (1.f - rd_ratio);
            V3 wh = d.sample_wh(wo, u0, u1);
            wi = reflect(-wo, wh);
        }
        return {wi, same_hemisphere(wo, wi)};
    }
    float pdf(V3 wo, V3 wi) const {
        V3 wh = normalize(wo + wi);
        float pdf_wh = d.pdf(wo, wh);
        float p = lerp(pdf_wh / (4.f * dot(wo, wh)), abs_cos_theta(wi) * kInvPi, rd_ratio);
        return same_hemisphere(wo, wi) ? p : 0.f;
    }
};

// --- Disney: src/surfaces/disney.cpp:95-303 (lobes), :376-478 (closure set-up), :481-587 (evaluate / sample)
inline float SchlickWeight(float cosTheta) {
    float m = saturate(1.f - cosTheta);
    return sqr(sqr(m)) * m;
}
inline float FrSchlick(float R0, float cosTheta) { return lerp(R0, 1.f, SchlickWeight(cosTheta)); }
inline float SchlickR0FromEta(float eta) { return sqr((eta - 1.f) / (eta + 1.f)); }
inline float GTR1(float cosTheta, float alpha) {
    float alpha2 = sqr(alpha);
    float denom = kPi * std::log(alpha2) * (1.f + (alpha2 - 1.f) * sqr(cosTheta));
    return (alpha2 - 1.f) / denom;
}
inline float smithG_GGX(float cosTheta, float alpha) {
    float alpha2 = sqr(alpha);
    float cosTheta2 = sqr(cosTheta);
    return 1.f / (cosTheta + std::sqrt(alpha2 + cosTheta2 - alpha2 * cosTheta2));
}
inline bool any_nonzero(V3 w) { return w.x != 0.f || w.y != 0.f || w.z != 0.f; }

struct DisneyClosure {
    // context
    V3 color;
    float color_lum, metallic, eta_t, roughness, specular_tint, anisotropic, sheen, sheen_tint, clearcoat,
        clearcoat_gloss, specular_trans, flatness;
    uint32_t lobes;
    // derived
    bool has_diffuse{false}, has_fake_ss{false}, has_sheen{false}, has_clearcoat{false};
    V3 Cdiff{}, Css{}, Csheen{}, Cspec0{};
    float fresnel_eta{}, gloss{};
    TrowbridgeReitz distrib{1.f, 1.f};
    // techniques: diffuse-like, specular, clearcoat and - transmissive closure ("disney_trans", disney.cpp:376-383,452-464) only -
    // specular transmission; the thin closure ("disney_thin", disney.cpp:590-845) has specular transmission through a rescaled
    // distribution and a fifth technique, Lambertian diffuse transmission
    float w[5]{0.f, 0.f, 0.f, 0.f, 0.f};
    bool enabled[5]{false, false, false, false, false};
    bool transmissive{false};
    bool thin{false};
    bool has_spec_trans{false};
    bool has_diff_trans{false};
    V3 Cdt{};
    float diffuse_trans{0.f};
    MicrofacetTransmission spec_trans{v3(0.f), TrowbridgeReitz{1.f, 1.f}, 1.f, 1.f};
    int techniques() const { return thin ? 5 : transmissive ? 4 : 3; }

    explicit DisneyClosure(const lrk_surface &s) {
        thin = (s.flags & LRK_SURFACE_DISNEY_THIN) != 0u;
        transmissive = !thin && (s.flags & LRK_SURFACE_DISNEY_TRANSMISSIVE) != 0u;
        diffuse_trans = thin ? s.p[15] : 0.f;
        color = v3(s.p[0], s.p[1], s.p[2]);
        color_lum = s.p[3]; metallic = s.p[4]; eta_t = s.p[5]; roughness = s.p[6]; specular_tint = s.p[7];
        anisotropic = s.p[8]; sheen = s.p[9]; sheen_tint = s.p[10]; clearcoat = s.p[11]; clearcoat_gloss = s.p[12];
        specular_trans = s.p[13]; flatness = s.p[14];
        lobes = s.lobes;
        const float eta_i = 1.f;
        float diffuse_weight = (1.f - metallic) * (1.f - specular_trans);
        float tint_weight = color_lum > 0.f ? 1.f / color_lum : 1.f;
        V3 tc = color * tint_weight;
        V3 tint = v3(saturate(tc.x), saturate(tc.y), saturate(tc.z));
        float tint_lum = color_lum * tint_weight;
        // thin closure (disney.cpp:620-622,633,643,651): the diffuse-like lobes keep the reflected share of the diffuse weight, and
        // fake subsurface / sheen are scaled by (1 - diffuse_trans) once more
        const float diff_refl_weight = thin ? diffuse_weight * (1.f - diffuse_trans) : diffuse_weight;
        const float diff_trans_weight = diffuse_weight * diffuse_trans;
        float diffuse_like_sampling_weight = diff_refl_weight * color_lum;
        if ((lobes & LRK_DISNEY_LOBE_DIFFUSE) || (lobes & LRK_DISNEY_LOBE_RETRO)) {
            float Cdiff_weight = diff_refl_weight * (1.f - flatness);
            Cdiff = color * Cdiff_weight;
            has_diffuse = true;
            enabled[0] = true;
        }
        if (lobes & LRK_DISNEY_LOBE_FAKE_SS) {
            float Css_weight = thin ? diff_refl_weight * flatness * (1.f - diffuse_trans) : diffuse_weight * flatness;
            Css = Css_weight * color;
            has_fake_ss = true;
            enabled[0] = true;
        }
        if (lobes & LRK_DISNEY_LOBE_SHEEN) {
            float Csheen_weight = thin ? diff_refl_weight * sheen * (1.f - diffuse_trans) : diffuse_weight * sheen;
            Csheen = Csheen_weight * lerp(v3(1.f), tint, sheen_tint);
            has_sheen = true;
            float sheen_lum = Csheen_weight * lerp(1.f, tint_lum, sheen_tint);
            diffuse_like_sampling_weight += sheen_lum * .1f;
            if (!thin) enabled[0] = true;// the thin closure's sheen block does not enable the technique (disney.cpp:650-657)
        }
        w[0] = saturate(diffuse_like_sampling_weight);
        float eta = eta_t / eta_i;
        float SchlickR0 = SchlickR0FromEta(eta);
        Cspec0 = lerp(lerp(v3(1.f), tint, specular_tint) * SchlickR0, color, metallic);
        fresnel_eta = eta;
        float aspect = std::sqrt(1.f - anisotropic * .9f);
        distrib = TrowbridgeReitz{std::fmax(0.001f, roughness / aspect), std::fmax(0.001f, roughness * aspect)};
        float Cspec0_lum = lerp(lerp(1.f, tint_lum, specular_tint) * SchlickR0, color_lum, metallic);
        w[1] = saturate(Cspec0_lum);
        enabled[1] = true;
        if (lobes & LRK_DISNEY_LOBE_CLEARCOAT) {
            gloss = lerp(.1f, .001f, clearcoat_gloss);
            has_clearcoat = true;
            w[2] = saturate(clearcoat * FrSchlick(.04f, 1.f));
            enabled[2] = true;
        }
        if (transmissive && (lobes & LRK_DISNEY_LOBE_SPEC_TRANS)) {// disney.cpp:452-464
            float Cst_weight = (1.f - metallic) * specular_trans;
            V3 Cst = Cst_weight * v3(std::sqrt(color.x), std::sqrt(color.y), std::sqrt(color.z));
            spec_trans = MicrofacetTransmission{Cst, distrib, eta_i, eta_t};
            has_spec_trans = true;
            float Cst_lum = Cst_weight * std::sqrt(color_lum);
            w[3] = saturate(Cst_lum);
            enabled[3] = true;
        }
        if (thin && (lobes & LRK_DISNEY_LOBE_SPEC_TRANS)) {// disney.cpp:686-701: a rescaled distribution, the colour itself (no sqrt)
            float rscaled = (.65f * eta - .35f) * roughness;
            TrowbridgeReitz thin_distrib{std::fmax(.001f, rscaled / aspect), std::fmax(.001f, rscaled * aspect)};
            float Cst_weight = (1.f - metallic) * specular_trans;
            V3 Cst = Cst_weight * color;
            spec_trans = MicrofacetTransmission{Cst, thin_distrib, eta_i, eta_t};
            has_spec_trans = true;
            float Cst_lum = Cst_weight * color_lum;
            w[3] = saturate(Cst_lum);
            enabled[3] = true;
        }
        if (thin && (lobes & LRK_DISNEY_LOBE_DIFF_TRANS)) {// disney.cpp:703-710
            Cdt = diff_trans_weight * color;
            float Cdt_lum = diff_trans_weight * color_lum;
            has_diff_trans = true;
            w[4] = saturate(Cdt_lum);
            enabled[4] = true;
        }
        float sum_weights = 0.f;
        for (int i = 0; i < techniques(); i++) if (enabled[i]) sum_weights += w[i];
        float inv_sum_weights = sum_weights == 0.f ? 0.f : 1.f / sum_weights;
        for (int i = 0; i < techniques(); i++) if (enabled[i]) w[i] *= inv_sum_weights;
    }

    V3 disney_fresnel(float cosI_in) const {// DisneyFresnel::evaluate, two_sided = !is_transmissive (disney.cpp:287-292,425)
        float cosI = (transmissive || thin) ? cosI_in : std::fabs(cosI_in);// the thin closure's term is one-sided too (disney.cpp:666)
        float fr = fresnel_dielectric(cosI, 1.f, fresnel_eta);
        V3 f0 = v3(FrSchlick(Cspec0.x, cosI), FrSchlick(Cspec0.y, cosI), FrSchlick(Cspec0.z, cosI));
        return lerp(v3(fr), f0, metallic);
    }
    V3 specular_evaluate(V3 wo, V3 wi) const {// MicrofacetReflection::evaluate, R = 1
        V3 wh = wi + wo;
        V3 f = v3(0.f);
        if (same_hemisphere(wo, wi) && any_nonzero(wh)) {
            wh = normalize(wh);
            V3 F = disney_fresnel(dot(wi, face_forward(wh, v3(0.f, 0.f, 1.f))));
            float D = distrib.D(wh);
            float G = distrib.G(wo, wi);
            float cos_o = cos_theta(wo), cos_i = cos_theta(wi);
            f = v3(1.f) * F * std::fabs(0.25f * D * G / (cos_i * cos_o));
        }
        return f;
    }
    float specular_pdf(V3 wo, V3 wi) const {
        float p = 0.f;
        V3 wh = wi + wo;
        if (same_hemisphere(wo, wi) && any_nonzero(wh)) {
            wh = normalize(wh);
            p = distrib.pdf(wo, wh) / (4.f * dot(wo, wh));
        }
        return p;
    }
    float clearcoat_evaluate(V3 wo, V3 wi) const {
        V3 wh = wi + wo;
        bool valid = any_nonzero(wh);
        wh = normalize(wh);
        float Dr = GTR1(abs_cos_theta(wh), gloss);
        float Fr = FrSchlick(.04f, dot(wo, wh));
        float Gr = smithG_GGX(abs_cos_theta(wo), .25f) * smithG_GGX(abs_cos_theta(wi), .25f);
        return valid ? clearcoat * Gr * Fr * Dr * .25f : 0.f;
    }
    float clearcoat_pdf(V3 wo, V3 wi) const {
        V3 wh = wi + wo;
        bool valid = same_hemisphere(wo, wi) && any_nonzero(wh);
        wh = normalize(wh);
        float Dr = GTR1(abs_cos_theta(wh), gloss);
        return valid ? Dr * abs_cos_theta(wh) / (4.f * dot(wo, wh)) : 0.f;
    }
    V3 clearcoat_sample_wi(V3 wo, float u0, float u1, bool &valid) const {
        float alpha2 = gloss * gloss;
        float cosTheta = std::sqrt(std::fmax(0.f, (1.f - builtin_pow(alpha2, 1.f - u0)) / (1.f - alpha2)));
        float sinTheta = std::sqrt(std::fmax(0.f, 1.f - cosTheta * cosTheta));
        float phi = 2.f * kPi * u1;
        V3 wh = v3(sinTheta * std::cos(phi), sinTheta * std::sin(phi), cosTheta);
        wh = same_hemisphere(wo, wh) ? wh : -wh;
        V3 wi = reflect(-wo, wh);
        valid = same_hemisphere(wo, wi);
        return wi;
    }

    SurfEval evaluate_local(V3 wo, V3 wi) const {
        V3 f = v3(0.f);
        float pdf = 0.f;
        if (same_hemisphere(wo, wi)) {
            if (has_diffuse) {
                if (w[0] > 0.f) {
                    {// DisneyDiffuse
                        float Fo = SchlickWeight(abs_cos_theta(wo)), Fi = SchlickWeight(abs_cos_theta(wi));
                        f = f + Cdiff * (kInvPi * (1.f - Fo * .5f) * (1.f - Fi * .5f));
                    }
                    {// DisneyRetro
                        V3 wh = wi + wo;
                        bool valid = any_nonzero(wh);
                        wh = normalize(wh);
                        float cosThetaD = dot(wi, wh);
                        float Fo = SchlickWeight(abs_cos_theta(wo)), Fi = SchlickWeight(abs_cos_theta(wi));
                        float Rr = 2.f * roughness * cosThetaD * cosThetaD;
                        f = f + Cdiff * (valid ? kInvPi * Rr * (Fo + Fi + Fo * Fi * (Rr - 1.f)) : 0.f);
                    }
                    if (has_fake_ss) {
                        V3 wh = wi + wo;
                        bool valid = any_nonzero(wh);
                        wh = normalize(wh);
                        float cosThetaD = dot(wi, wh);
                        float Fss90 = cosThetaD * cosThetaD * roughness;
                        float Fo = SchlickWeight(abs_cos_theta(wo)), Fi = SchlickWeight(abs_cos_theta(wi));
                        float Fss = lerp(1.0f, Fss90, Fo) * lerp(1.0f, Fss90, Fi);
                        float ss = 1.25f * (Fss * (1.f / (abs_cos_theta(wo) + abs_cos_theta(wi)) - .5f) + .5f);
                        f = f + Css * (valid ? kInvPi * ss : 0.f);
                    }
                    if (has_sheen) {
                        V3 wh = wi + wo;
                        bool valid = any_nonzero(wh);
                        wh = normalize(wh);
                        float cosThetaD = dot(wi, wh);
                        f = f + Csheen * (valid ? SchlickWeight(cosThetaD) : 0.f);
                    }
                    pdf += w[0] * lambert_pdf(wo, wi);
                }
            }
            if (w[1] > 0.f) {
                f = f + specular_evaluate(wo, wi);
                pdf += w[1] * specular_pdf(wo, wi);
            }
            if (has_clearcoat) {
                if (w[2] > 0.f) {
                    f = f + clearcoat_evaluate(wo, wi);
                    pdf += w[2] * clearcoat_pdf(wo, wi);
                }
            }
        } else {// transmission, disney.cpp:514-522 (transmissive), :755-774 (thin)
            if (has_spec_trans) {
                if (w[3] > 0.f) {
                    f = f + spec_trans.evaluate(wo, wi);
                    pdf += w[3] * spec_trans.pdf(wo, wi);
                }
            }
            if (has_diff_trans) {
                if (w[4] > 0.f) {// LambertianTransmission, scattering.cpp:271-284 (wo and wi are in opposite hemispheres here)
                    f = f + Cdt * kInvPi;
                    pdf += w[4] * (abs_cos_theta(wi) * kInvPi);
                }
            }
        }
        SurfEval e;
        e.f = f * abs_cos_theta(wi);
        e.pdf = pdf;
        return e;
    }
};

SurfEval disney_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi) {
    DisneyClosure c{s};
    return c.evaluate_local(it.shading.world_to_local(wo), it.shading.world_to_local(wi));
}
SurfSample disney_sample(const lrk_surface &s, const Interaction &it, V3 wo, float u_lobe, float u0, float u1) {
    DisneyClosure c{s};
    uint32_t tech = 0u;
    float sum_weights = 0.f;
    for (uint32_t i = 0; i < static_cast<uint32_t>(c.techniques()); i++) {
        if (c.enabled[i]) {
            tech = u_lobe > sum_weights ? i : tech;
            sum_weights += c.w[i];
        }
    }
    V3 wo_local = it.shading.world_to_local(wo);
    V3 wi_local = v3(0.f);
    bool valid = false;
    uint32_t event = LRK_EVENT_REFLECT;
    if (tech == 0u) {
        if (c.has_diffuse) {// BxDF::sample_wi, scattering.cpp:274-278
            wi_local = sample_cosine_hemisphere(u0, u1);
            wi_local.z *= sign(cos_theta(wo_local));
            valid = true;
        }
    } else if (tech == 1u) {// MicrofacetReflection::sample_wi
        V3 wh = c.distrib.sample_wh(wo_local, u0, u1);
        wi_local = reflect(-wo_local, wh);
        valid = same_hemisphere(wo_local, wi_local);
    } else if (tech == 2u) {
        if (c.has_clearcoat) wi_local = c.clearcoat_sample_wi(wo_local, u0, u1, valid);
    } else if (tech == 3u) {
        if (c.has_spec_trans) {// disney.cpp:571-576; the thin closure's event is "through" (:820-825): the ray stays in its medium
            BxDFSample bs = c.spec_trans.sample_wi(wo_local, u0, u1);
            wi_local = bs.wi;
            valid = bs.valid;
            event = c.thin ? LRK_EVENT_THROUGH : cos_theta(wo_local) > 0.f ? LRK_EVENT_ENTER : LRK_EVENT_EXIT;
        }
    } else if (c.has_diff_trans) {// LambertianTransmission::sample_wi, scattering.cpp:276-280 (disney.cpp:827-832)
        wi_local = sample_cosine_hemisphere(u0, u1);
        wi_local.z *= -sign(cos_theta(wo_local));
        valid = true;
        event = LRK_EVENT_THROUGH;
    }
    SurfSample out;
    out.wi = it.shading.local_to_world(wi_local);
    if (valid) out.eval = c.evaluate_local(wo_local, wi_local);
    out.event = event;
    return out;
}

// --- Mirror / Glass / Plastic / Metal (SURVEY.md §8 row f3).  lrk_surface.p holds each closure's Context as
//     populate_closure computes it for constant textures (include/lrk.h); pinned against the reference's closures through
//     Surface::Closure::{evaluate,sample} (oracle/ref/pin_<name>.cpp, tests/test_ref_pins.py).
inline SurfSample finish_sample(const Interaction &it, V3 wi_local, V3 f, float pdf, uint32_t event) {
    SurfSample out;
    out.wi = it.shading.local_to_world(wi_local);
    out.eval.f = f * abs_cos_theta(wi_local);
    out.eval.pdf = pdf;
    out.event = event;
    return out;
}
template<typename B>
inline void bxdf_sample(const B &bxdf, V3 wo, float u0, float u1, V3 &wi, V3 &f, float &pdf) {// BxDF::sample, scattering.cpp:247-254
    BxDFSample s = bxdf.sample_wi(wo, u0, u1);
    wi = s.wi;
    pdf = s.valid ? bxdf.pdf(wo, wi) : 0.f;
    f = s.valid ? bxdf.evaluate(wo, wi) : v3(0.f);
}

// mirror.cpp:81-131: MicrofacetReflection with a Schlick Fresnel term around the reflectance colour
inline MicrofacetReflection mirror_lobe(const lrk_surface &s) {
    V3 refl = v3(s.p[0], s.p[1], s.p[2]);
    return {refl, TrowbridgeReitz{s.p[3], s.p[4]}, FresnelTerm::schlick(refl)};
}
SurfEval mirror_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi) {
    MicrofacetReflection refl = mirror_lobe(s);
    V3 wo_local = it.shading.world_to_local(wo), wi_local = it.shading.world_to_local(wi);
    SurfEval e;
    e.f = refl.evaluate(wo_local, wi_local) * abs_cos_theta(wi_local);
    e.pdf = refl.pdf(wo_local, wi_local);
    return e;
}
SurfSample mirror_sample(const lrk_surface &s, const Interaction &it, V3 wo, float, float u0, float u1) {
    MicrofacetReflection refl = mirror_lobe(s);
    V3 wo_local = it.shading.world_to_local(wo), wi_local = v3(0.f, 0.f, 1.f), f;
    float pdf = 0.f;
    bxdf_sample(refl, wo_local, u0, u1, wi_local, f, pdf);
    return finish_sample(it, wi_local, f, pdf, LRK_EVENT_REFLECT);
}

// metal.cpp:205-266: conductor Fresnel from (n, k), result tinted by the `Kd` reflectance
inline MicrofacetReflection metal_lobe(const lrk_surface &s) {
    return {v3(1.f), TrowbridgeReitz{s.p[9], s.p[10]}, FresnelTerm::conductor(1.f, v3(s.p[0], s.p[1], s.p[2]), v3(s.p[3], s.p[4], s.p[5]))};
}
SurfEval metal_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi) {
    MicrofacetReflection lobe = metal_lobe(s);
    V3 wo_local = it.shading.world_to_local(wo), wi_local = it.shading.world_to_local(wi);
    V3 f = lobe.evaluate(wo_local, wi_local);
    f = f * v3(s.p[6], s.p[7], s.p[8]);
    SurfEval e;
    e.f = f * abs_cos_theta(wi_local);
    e.pdf = lobe.pdf(wo_local, wi_local);
    return e;
}
SurfSample metal_sample(const lrk_surface &s, const Interaction &it, V3 wo, float, float u0, float u1) {
    MicrofacetReflection lobe = metal_lobe(s);
    V3 wo_local = it.shading.world_to_local(wo), wi_local = v3(0.f, 0.f, 1.f), f;
    float pdf = 0.f;
    bxdf_sample(lobe, wo_local, u0, u1, wi_local, f, pdf);
    f = f * v3(s.p[6], s.p[7], s.p[8]);
    return finish_sample(it, wi_local, f, pdf, LRK_EVENT_REFLECT);
}

// glass.cpp:129-222: reflection / transmission lobes chosen by Kr_ratio-weighted Fresnel
struct GlassLobes {
    MicrofacetReflection refl;
    MicrofacetTransmission trans;
    float eta_t, kr_ratio;
    explicit GlassLobes(const lrk_surface &s, bool importance = false)
        : refl{v3(s.p[0], s.p[1], s.p[2]), TrowbridgeReitz{s.p[7], s.p[8]}, FresnelTerm::dielectric(1.f, s.p[6])},
          trans{v3(s.p[3], s.p[4], s.p[5]), TrowbridgeReitz{s.p[7], s.p[8]}, 1.f, s.p[6], importance}, eta_t{s.p[6]}, kr_ratio{s.p[9]} {}
    float refl_prob(V3 wo_local) const {// :162-167
        float F = fresnel_dielectric(cos_theta(wo_local), 1.f, eta_t);
        float r = kr_ratio * F;
        float t = (1.f - kr_ratio) * (1.f - F);
        return r == 0.f ? 0.f : r / (r + t);
    }
};
SurfEval glass_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi, bool importance = false) {
    GlassLobes g{s, importance};
    V3 wo_local = it.shading.world_to_local(wo), wi_local = it.shading.world_to_local(wi);
    float ratio = g.refl_prob(wo_local);
    V3 f;
    float pdf;
    if (same_hemisphere(wo_local, wi_local)) {
        f = g.refl.evaluate(wo_local, wi_local);
        pdf = g.refl.pdf(wo_local, wi_local) * ratio;
    } else {
        f = g.trans.evaluate(wo_local, wi_local);
        pdf = g.trans.pdf(wo_local, wi_local) * (1.f - ratio);
    }
    SurfEval e;
    e.f = f * abs_cos_theta(wi_local);
    e.pdf = pdf;
    return e;
}
SurfSample glass_sample(const lrk_surface &s, const Interaction &it, V3 wo, float u_lobe, float u0, float u1, bool importance = false) {
    GlassLobes g{s, importance};
    V3 wo_local = it.shading.world_to_local(wo), wi_local = v3(0.f, 0.f, 1.f), f;
    float pdf = 0.f;
    uint32_t event = LRK_EVENT_REFLECT;
    float ratio = g.refl_prob(wo_local);
    if (u_lobe < ratio) {
        bxdf_sample(g.refl, wo_local, u0, u1, wi_local, f, pdf);
        pdf *= ratio;
    } else {
        bxdf_sample(g.trans, wo_local, u0, u1, wi_local, f, pdf);
        pdf *= (1.f - ratio);
        event = cos_theta(wo_local) > 0.f ? LRK_EVENT_ENTER : LRK_EVENT_EXIT;
    }
    return finish_sample(it, wi_local, f, pdf, event);
}

// plastic.cpp:116-214: dielectric coat over a Lambertian substrate with absorption (Tungsten's rough plastic)
struct PlasticLobes {
    V3 kd, sigma_a;
    float kd_weight, eta;
    MicrofacetReflection coat;
    explicit PlasticLobes(const lrk_surface &s)
        : kd{v3(s.p[0], s.p[1], s.p[2])}, sigma_a{v3(s.p[4], s.p[5], s.p[6])}, kd_weight{s.p[3]}, eta{s.p[7]},
          coat{v3(1.f), TrowbridgeReitz{s.p[8], s.p[9]}, FresnelTerm::dielectric(1.f, s.p[7])} {}
    static float substrate_weight(float Fo, float kd_w) {// :125-128
        float w = kd_w * (1.0f - Fo);
        return w == 0.f ? 0.f : w / (w + Fo);
    }
    V3 diffuse(V3 wo_local, V3 wi_local, float Fo) const {// :155-159
        float Fi = fresnel_dielectric(abs_cos_theta(wi_local), 1.f, eta);
        V3 a = exp3(-(1.f / abs_cos_theta(wi_local) + 1.f / abs_cos_theta(wo_local)) * sigma_a);
        return (1.f - Fi) * (1.f - Fo) * sqr(1.f / eta) * a * lambert_evaluate(kd, wo_local, wi_local);
    }
};
SurfEval plastic_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi) {
    PlasticLobes p{s};
    V3 wo_local = it.shading.world_to_local(wo);
    V3 sgn = cos_theta(wo_local) < 0.f ? v3(1.f, 1.f, -1.f) : v3(1.f, 1.f, 1.f);
    wo_local = wo_local * sgn;
    V3 wi_local = it.shading.world_to_local(wi) * sgn;
    SurfEval e;
    V3 f_coat = p.coat.evaluate(wo_local, wi_local);
    float pdf_coat = p.coat.pdf(wo_local, wi_local);
    float Fo = fresnel_dielectric(abs_cos_theta(wo_local), 1.f, p.eta);
    V3 f_diffuse = p.diffuse(wo_local, wi_local, Fo);
    float pdf_diffuse = lambert_pdf(wo_local, wi_local);
    float sw = PlasticLobes::substrate_weight(Fo, p.kd_weight);
    e.f = (f_coat + f_diffuse) * abs_cos_theta(wi_local);
    e.pdf = lerp(pdf_coat, pdf_diffuse, sw);
    return e;
}
SurfSample plastic_sample(const lrk_surface &s, const Interaction &it, V3 wo, float u_lobe, float u0, float u1) {
    PlasticLobes p{s};
    V3 wo_local = it.shading.world_to_local(wo);
    V3 sgn = cos_theta(wo_local) < 0.f ? v3(1.f, 1.f, -1.f) : v3(1.f, 1.f, 1.f);
    wo_local = wo_local * sgn;
    float Fo = fresnel_dielectric(abs_cos_theta(wo_local), 1.f, p.eta);
    float sw = PlasticLobes::substrate_weight(Fo, p.kd_weight);
    BxDFSample ws = u_lobe < sw ? lambert_sample_wi(wo_local, u0, u1) : p.coat.sample_wi(wo_local, u0, u1);
    SurfSample out;
    out.wi = v3(0.f, 0.f, 1.f);
    out.event = LRK_EVENT_REFLECT;
    if (ws.valid) {
        V3 wi_local = ws.wi;
        out.wi = it.shading.local_to_world(ws.wi * sgn);
        V3 f_coat = p.coat.evaluate(wo_local, wi_local);
        float pdf_coat = p.coat.pdf(wo_local, wi_local);
        V3 f_diffuse = p.diffuse(wo_local, wi_local, Fo);
        float pdf_diffuse = lambert_pdf(wo_local, wi_local);
        out.eval.f = (f_coat + f_diffuse) * abs_cos_theta(wi_local);
        out.eval.pdf = lerp(pdf_coat, pdf_diffuse, sw);
    }
    return out;
}

// `records` = lrk_scene_desc::surfaces (the two mixed surfaces of a Mix node are records of the same array); nullptr where a
// closure is evaluated on its own (unit tests: no Mix)
// `importance`: TransportMode::IMPORTANCE (the Layered surface samples its exit interface in the reverse mode); RADIANCE everywhere else
SurfEval surface_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi, const lrk_surface *records = nullptr, bool importance = false);
SurfSample surface_sample(const lrk_surface &s, const Interaction &it, V3 wo, float u_lobe, float u0, float u1, const lrk_surface *records = nullptr,
                          bool importance = false);

// Mix: src/surfaces/mix.cpp:82-193.  _mix(a, b, ratio) = lerp(a, b, 1 - ratio) on f and pdf.
inline SurfEval mix_eval(const SurfEval &a, const SurfEval &b, float ratio) {
    float t = 1.f - ratio;
    SurfEval e;
    e.f = lerp(a.f, b.f, t);
    e.pdf = lerp(a.pdf, b.pdf, t);
    return e;
}
SurfEval mix_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi, const lrk_surface *records) {
    SurfEval eval_a = surface_evaluate(records[s.mix_a], it, wo, wi, records);
    SurfEval eval_b = surface_evaluate(records[s.mix_b], it, wo, wi, records);
    return mix_eval(eval_a, eval_b, s.p[0]);
}
SurfSample mix_sample(const lrk_surface &s, const Interaction &it, V3 wo, float u_lobe, float u0, float u1, const lrk_surface *records) {
    const float ratio = s.p[0];
    const lrk_surface &a = records[s.mix_a], &b = records[s.mix_b];
    SurfSample out;
    if (u_lobe < ratio) {// sample a
        SurfSample sample_a = surface_sample(a, it, wo, u_lobe / ratio, u0, u1, records);
        SurfEval eval_b = surface_evaluate(b, it, wo, sample_a.wi, records);
        out.eval = mix_eval(sample_a.eval, eval_b, ratio);
        out.wi = sample_a.wi;
        out.event = sample_a.event;
    } else {// "sample b" — the reference samples `a` again and evaluates `b` in a's place (mix.cpp:170-176); kept as is
        SurfSample sample_b = surface_sample(a, it, wo, (u_lobe - ratio) / (1.f - ratio), u0, u1, records);
        SurfEval eval_a = surface_evaluate(b, it, wo, sample_b.wi, records);
        out.eval = mix_eval(eval_a, sample_b.eval, ratio);
        out.wi = sample_b.wi;
        out.event = sample_b.event;
    }
    return out;
}
// ------------------------------------------------------------------------------------------------
// Layered: src/surfaces/layered.cpp (pbrt-v4's LayeredBxDF as the reference restates it): two interfaces (`top`, `bottom`: records
// mix_a / mix_b) around a homogeneous slab (thickness p[0], Henyey-Greenstein g p[1], albedo p[2..4]); evaluate() is a stochastic
// random walk with its own LCG stream seeded from the hit position and wi (:277), sample() from the sample numbers and wo (:427).
// lobes = max_depth | samples << 16.  Both children are bound to the SAME interaction (:500-502), so to_local / to_world of the
// reference's TopOrBottom are the Layered closure's own frame.
// ------------------------------------------------------------------------------------------------
inline bool is_zero3(V3 a) { return a.x == 0.f && a.y == 0.f && a.z == 0.f; }
inline uint32_t float_bits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
inline float power_heuristic(float f_pdf, float g_pdf) {// src/util/sampling.cpp:142-151 with nf = ng = 1
    float f = 1.f * f_pdf, g = 1.f * g_pdf;
    float ff = f * f, gg = g * g, sum = ff + gg;
    return std::isinf(ff) ? 1.f : (sum == 0.f ? 0.f : ff / sum);
}
struct LayeredPhase {// HGPhaseFunction, layered.cpp:14-61
    float g;
    static float hg(float cosTheta, float g) {
        float denom = 1.f + sqr(g) + 2.f * g * cosTheta;
        return kInvPi / 4.0f * (1.f - sqr(g)) / (denom * std::sqrt(denom));
    }
    float p(V3 wo, V3 wi) const { return hg(dot(wo, wi), g); }
    struct Sample {
        float p;
        V3 wi;
        float pdf;
    };
    Sample sample_p(V3 wo, float ux, float uy) const {
        float cosTheta = std::fabs(g) < 1e-3f ? 1.f - 2.f * ux : -1.f / (2.f * g) * (1.f + sqr(g) - sqr((1.f - sqr(g)) / (1.f + g - 2.f * g * ux)));
        float sinTheta = std::sqrt(1.f - sqr(cosTheta));
        float phi = 2.f * kPi * uy;
        Frame wFrame = Frame::make(wo);
        V3 wi = wFrame.local_to_world(spherical_direction(sinTheta, cosTheta, phi));
        float pdf = hg(cosTheta, g);
        return {pdf, wi, pdf};
    }
};
struct LayeredCtx {
    const lrk_surface *top, *bottom, *records;
    float thickness, g;
    V3 albedo;
    uint32_t max_depth, samples;
    LayeredCtx(const lrk_surface &s, const lrk_surface *rec)
        : top{rec + s.mix_a}, bottom{rec + s.mix_b}, records{rec}, thickness{s.p[0]}, g{s.p[1]}, albedo{v3(s.p[2], s.p[3], s.p[4])},
          max_depth{s.lobes & 0xffffu}, samples{s.lobes >> 16u} {}
    static float Tr(float dz, V3 w) { return std::fabs(dz) <= std::numeric_limits<float>::min() ? 1.f : std::exp(-std::fabs(dz / w.z)); }
};
// lcg draws of `f(x, lcg(seed), make_float2(lcg(seed), lcg(seed)))` and of `make_float2(lcg(seed), lcg(seed))` in the compiler's order
inline void layered_draw3(uint32_t &seed, float &uc, float &u0, float &u1) {
    if (g_hg_args_right_to_left.load(std::memory_order_relaxed)) { u1 = lcg(seed); u0 = lcg(seed); uc = lcg(seed); }
    else { uc = lcg(seed); u0 = lcg(seed); u1 = lcg(seed); }
}
inline void layered_draw2(uint32_t &seed, float &u0, float &u1) {
    if (g_hg_args_right_to_left.load(std::memory_order_relaxed)) { u1 = lcg(seed); u0 = lcg(seed); }
    else { u0 = lcg(seed); u1 = lcg(seed); }
}

SurfEval layered_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi, const lrk_surface *records, bool mode) {// :251-404
    const LayeredCtx ctx{s, records};
    auto eval = [&](const lrk_surface *c, V3 a, V3 b, bool m) { return surface_evaluate(*c, it, a, b, records, m); };
    auto sample = [&](const lrk_surface *c, V3 a, float uc, float u0, float u1, bool m) { return surface_sample(*c, it, a, uc, u0, u1, records, m); };
    const V3 wi_local = it.shading.world_to_local(wi), wo_local = it.shading.world_to_local(wo);
    const bool entered_top = wo_local.z > 0.f;
    const bool exit_is_bottom = same_hemisphere(wo_local, wi_local) != entered_top;// same_hemisphere ^ entered_top
    const lrk_surface *enter_interface = entered_top ? ctx.top : ctx.bottom;
    const lrk_surface *exit_interface = exit_is_bottom ? ctx.bottom : ctx.top;
    const lrk_surface *nonexit_interface = exit_is_bottom ? ctx.top : ctx.bottom;
    const float exitZ = exit_is_bottom ? 0.f : ctx.thickness;
    const float n_samples = static_cast<float>(ctx.samples);
    V3 f = same_hemisphere(wi_local, wo_local) ? n_samples * eval(enter_interface, wo, wi, mode).f : v3(0.f);
    uint32_t seed = xxhash32_uint4(float_bits(it.pg.x), float_bits(it.pg.y), float_bits(it.pg.z),
                                   xxhash32_uint3(float_bits(wi.x), float_bits(wi.y), float_bits(wi.z)));
    float pdf_sum = same_hemisphere(wi_local, wo_local)
                        ? (entered_top ? n_samples * eval(ctx.top, wo, wi, mode).pdf : n_samples * eval(ctx.bottom, wo, wi, mode).pdf)
                        : 0.f;
    const LayeredPhase phase{ctx.g};
    for (uint32_t i = 0; i < ctx.samples; i++) {
        float uc, u0, u1;
        layered_draw3(seed, uc, u0, u1);
        const SurfSample wos = sample(enter_interface, wo, uc, u0, u1, mode);
        if (is_zero3(wos.eval.f) || wos.eval.pdf <= 0.f) continue;
        layered_draw3(seed, uc, u0, u1);
        const SurfSample wis = sample(exit_interface, wi, uc, u0, u1, !mode);
        const V3 wis_wi_local = it.shading.world_to_local(wis.wi);
        if (is_zero3(wis.eval.f) || wis.eval.pdf <= 0.f) continue;
        V3 beta = wos.eval.f / wos.eval.pdf;
        float z = entered_top ? ctx.thickness : 0.f;
        V3 w = wos.wi;
        V3 w_local = it.shading.world_to_local(w);
        for (uint32_t depth = 0; depth < ctx.max_depth; depth++) {
            if (depth > 3u && max3(beta) < 0.25f) {
                float q = std::fmax(0.f, 1.f - max3(beta));
                if (lcg(seed) < q) break;
                beta = beta / (1.f - q);
            }
            if (is_zero3(ctx.albedo)) {
                z = z == ctx.thickness ? 0.f : ctx.thickness;
                beta = beta * LayeredCtx::Tr(ctx.thickness, w_local);
            } else {
                const float sigma_t = 1.f;
                float dz = -std::log(1.f - lcg(seed)) / (sigma_t / std::fabs(w_local.z));
                float zp = w_local.z > 0.f ? z + dz : z - dz;
                if (z == zp) continue;
                if (zp > 0.f && zp < ctx.thickness) {
                    float wt = power_heuristic(wis.eval.pdf, eval(nonexit_interface, -w, -wis.wi, mode).pdf);
                    f = f + beta * ctx.albedo * phase.p(-w_local, -wis_wi_local) * wt * LayeredCtx::Tr(zp - exitZ, wis_wi_local) * wis.eval.f / wis.eval.pdf;
                    float ux, uy;
                    layered_draw2(seed, ux, uy);
                    LayeredPhase::Sample ps = phase.sample_p(-w_local, ux, uy);
                    if (ps.pdf <= 0.f || ps.wi.z == 0.f) continue;
                    beta = beta * (ctx.albedo * ps.p / ps.pdf);
                    w_local = ps.wi;
                    w = it.shading.local_to_world(w_local);
                    z = zp;
                    if ((z < exitZ && w_local.z > 0.f) || (z > exitZ && w_local.z < 0.f)) {
                        V3 fExit = eval(exit_interface, -w, wi, mode).f;
                        if (!is_zero3(fExit)) {
                            float exitPDF = eval(exit_interface, -w, wi, mode).pdf;
                            float wt2 = power_heuristic(ps.pdf, exitPDF);
                            f = f + beta * LayeredCtx::Tr(zp - exitZ, w_local) * fExit * wt2;
                        }
                    }
                    continue;
                }
                z = clampf(zp, 0.f, ctx.thickness);
            }
            if (z == exitZ) {
                float uc2 = lcg(seed), ua, ub;
                layered_draw2(seed, ua, ub);
                SurfSample bs = sample(exit_interface, -w, uc2, ua, ub, mode);
                if (is_zero3(bs.eval.f) || bs.eval.pdf <= 0.f) break;
                beta = beta * (bs.eval.f / bs.eval.pdf);
                w = bs.wi;
                w_local = it.shading.world_to_local(w);
            } else {
                SurfEval wns = eval(nonexit_interface, -w, -wis.wi, mode);
                float wt = power_heuristic(wis.eval.pdf, wns.pdf);
                f = f + beta * wns.f * wt * LayeredCtx::Tr(ctx.thickness, wis_wi_local) * wis.eval.f / wis.eval.pdf;
                float uc2 = lcg(seed), ua, ub;
                layered_draw2(seed, ua, ub);
                SurfSample bs = sample(nonexit_interface, -w, uc2, ua, ub, mode);
                if (is_zero3(bs.eval.f) || bs.eval.pdf <= 0.f) break;
                beta = beta * (bs.eval.f / bs.eval.pdf);
                w = bs.wi;
                w_local = it.shading.world_to_local(w);
                SurfEval wes = eval(exit_interface, -w, wi, mode);
                V3 fExit = wes.f;
                if (!is_zero3(fExit)) {
                    float wt2 = power_heuristic(bs.eval.pdf, wes.pdf);
                    f = f + beta * LayeredCtx::Tr(ctx.thickness, it.shading.world_to_local(bs.wi)) * fExit * wt2;
                }
            }
        }
    }
    for (uint32_t k = 0; k < ctx.samples; k++) {// pdf: :361-400
        if (same_hemisphere(wo_local, wi_local)) {
            const lrk_surface *r_interface = entered_top ? ctx.bottom : ctx.top;
            const lrk_surface *t_interface = entered_top ? ctx.top : ctx.bottom;
            float uc, u0, u1;
            layered_draw3(seed, uc, u0, u1);
            SurfSample wos = sample(t_interface, wo, uc, u0, u1, mode);
            layered_draw3(seed, uc, u0, u1);
            SurfSample wis = sample(t_interface, wi, uc, u0, u1, !mode);
            if (!is_zero3(wos.eval.f) && wos.eval.pdf > 0.f && !is_zero3(wis.eval.f) && wis.eval.pdf > 0.f) {
                layered_draw3(seed, uc, u0, u1);
                SurfSample rs = sample(r_interface, -wos.wi, uc, u0, u1, mode);
                if (!is_zero3(rs.eval.f) && rs.eval.pdf > 0.f) {
                    float r_pdf = eval(r_interface, -wos.wi, -wis.wi, mode).pdf;
                    float wt = power_heuristic(wis.eval.pdf, r_pdf);
                    pdf_sum += wt * r_pdf;
                    float t_pdf = eval(t_interface, -rs.wi, wi, mode).pdf;
                    wt = power_heuristic(rs.eval.pdf, t_pdf);
                    pdf_sum += wt * t_pdf;
                }
            }
        } else {
            const lrk_surface *ti_interface = entered_top ? ctx.bottom : ctx.top;
            const lrk_surface *to_interface = entered_top ? ctx.top : ctx.bottom;
            float uc, u0, u1;
            layered_draw3(seed, uc, u0, u1);
            SurfSample wos = sample(to_interface, wo, uc, u0, u1, mode);
            layered_draw3(seed, uc, u0, u1);
            SurfSample wis = sample(ti_interface, wi, uc, u0, u1, !mode);
            if (is_zero3(wos.eval.f) || wos.eval.pdf <= 0.f || is_zero3(wis.eval.f) || wis.eval.pdf <= 0.f) continue;
            pdf_sum += .5f * (eval(to_interface, wo, -wis.wi, mode).pdf + eval(ti_interface, -wos.wi, wi, mode).pdf);
        }
    }
    SurfEval e;
    e.f = f / n_samples;
    e.pdf = lerp(1.f / (4.f * kPi), pdf_sum / n_samples, 0.9f);
    return e;
}

SurfSample layered_sample(const lrk_surface &s, const Interaction &it, V3 wo, float u_lobe, float u0, float u1, const lrk_surface *records, bool mode) {// :405-472
    const LayeredCtx ctx{s, records};
    auto sample = [&](const lrk_surface *c, V3 a, float uc, float ua, float ub, bool m) { return surface_sample(*c, it, a, uc, ua, ub, records, m); };
    const V3 wo_local = it.shading.world_to_local(wo);
    const bool entered_top = wo_local.z > 0.f;
    SurfSample bs = sample(entered_top ? ctx.top : ctx.bottom, wo, u_lobe, u0, u1, mode);
    SurfSample out;// Surface::Sample::zero: f = 0, pdf = 0, wi = (0, 0, 1), event_reflect
    out.wi = v3(0.f, 0.f, 1.f);
    out.event = LRK_EVENT_REFLECT;
    if (!is_zero3(bs.eval.f) && bs.eval.pdf != 0.f) {
        V3 wi_local = it.shading.world_to_local(bs.wi);
        if (same_hemisphere(wi_local, wo_local)) {
            out = bs;
        } else {
            V3 w = bs.wi;
            V3 w_local = it.shading.world_to_local(bs.wi);
            uint32_t seed = xxhash32_uint4(float_bits(u0), float_bits(u1), float_bits(u_lobe), xxhash32_uint3(float_bits(wo.x), float_bits(wo.y), float_bits(wo.z)));
            V3 f = bs.eval.f;
            float pdf = bs.eval.pdf;
            float z = entered_top ? ctx.thickness : 0.f;
            const LayeredPhase phase{ctx.g};
            for (uint32_t depth = 0; depth < ctx.max_depth; depth++) {
                float rr_beta = max3(f) / pdf;
                if (depth > 3u && rr_beta < 0.25f) {
                    float q = std::fmax(0.f, 1.f - rr_beta);
                    if (lcg(seed) < q) break;
                    pdf *= 1.f - q;
                }
                if (w_local.z == 0.f) break;
                if (!is_zero3(ctx.albedo)) {
                    const float sigma_t = 1.f;
                    float dz = -std::log(1.f - lcg(seed)) / (sigma_t / std::fabs(w_local.z));
                    float zp = w_local.z > 0.f ? z + dz : z - dz;
                    if (z == zp) break;
                    if (0.f < zp && zp < ctx.thickness) {
                        float ux, uy;
                        layered_draw2(seed, ux, uy);
                        LayeredPhase::Sample ps = phase.sample_p(-w_local, ux, uy);
                        if (ps.pdf <= 0.f) break;
                        f = f * (ctx.albedo * ps.p);
                        pdf *= ps.pdf;
                        w = ps.wi;// sic: the phase function's LOCAL direction is taken as the world direction (:449-450)
                        w_local = it.shading.world_to_local(w);
                        z = zp;
                        continue;
                    }
                    z = clampf(zp, 0.f, ctx.thickness);
                } else {
                    z = z == ctx.thickness ? 0.f : ctx.thickness;
                    f = f * LayeredCtx::Tr(ctx.thickness, w_local);
                }
                const lrk_surface *interface = z == 0.f ? ctx.bottom : ctx.top;
                float uc = lcg(seed), ua, ub;
                layered_draw2(seed, ua, ub);
                SurfSample is = sample(interface, -w, uc, ua, ub, mode);
                if (is_zero3(is.eval.f) || is.eval.pdf <= 0.f) break;
                f = f * is.eval.f;
                pdf *= is.eval.pdf;
                w = is.wi;
                w_local = it.shading.world_to_local(w);
                if ((is.event & 3u) != 0u) {// Surface::event_transmit = enter | exit
                    out.eval.f = f;
                    out.eval.pdf = pdf;
                    out.wi = w;
                    out.event = same_hemisphere(w_local, wo_local) ? LRK_EVENT_REFLECT : (w_local.z > 0.f ? LRK_EVENT_EXIT : LRK_EVENT_ENTER);
                    break;
                }
            }
        }
    }
    return out;
}

// Surface::Closure::eta() for the Russian-roulette eta scale (mega_path.cpp:133): Glass has one, a Mix lerps / forwards them
// (mix.cpp:133-141); 0 = nullopt
float surface_eta(const lrk_surface &s, const lrk_surface *records) {
    if (s.type == LRK_SURFACE_GLASS) return s.p[6];
    // DisneyClosureImpl::eta(): eta_t when the specular-transmission lobe exists (disney.cpp:531-533)
    if (s.type == LRK_SURFACE_DISNEY && (s.flags & LRK_SURFACE_DISNEY_TRANSMISSIVE) && (s.lobes & LRK_DISNEY_LOBE_SPEC_TRANS)) return s.p[5];
    if (s.type == LRK_SURFACE_MIX) {
        float ea = surface_eta(records[s.mix_a], records), eb = surface_eta(records[s.mix_b], records);
        if (ea == 0.f) return eb;
        if (eb == 0.f) return ea;
        return lerp(eb, ea, s.p[0]);
    }
    if (s.type == LRK_SURFACE_LAYERED) return surface_eta(records[s.mix_b], records);// _bottom->eta(), layered.cpp:248
    return 0.f;
}

SurfEval surface_evaluate(const lrk_surface &s, const Interaction &it, V3 wo, V3 wi, const lrk_surface *records, bool importance) {
    SurfEval e;
    switch (s.type) {
        case LRK_SURFACE_MATTE: e = matte_evaluate(s, it, wo, wi); break;
        case LRK_SURFACE_DISNEY: e = disney_evaluate(s, it, wo, wi); break;
        case LRK_SURFACE_MIRROR: e = mirror_evaluate(s, it, wo, wi); break;
        case LRK_SURFACE_GLASS: e = glass_evaluate(s, it, wo, wi, importance); break;
        case LRK_SURFACE_PLASTIC: e = plastic_evaluate(s, it, wo, wi); break;
        case LRK_SURFACE_MIX: e = mix_evaluate(s, it, wo, wi, records); break;
        case LRK_SURFACE_LAYERED: e = layered_evaluate(s, it, wo, wi, records, importance); break;
        default: e = metal_evaluate(s, it, wo, wi); break;
    }
    if (!validate_surface_sides(it.ng, it.shading.n, wo, wi)) {
        e.f = v3(0.f);
        e.pdf = 0.f;
    }
    return e;
}
SurfSample surface_sample(const lrk_surface &s, const Interaction &it, V3 wo, float u_lobe, float u0, float u1, const lrk_surface *records,
                          bool importance) {
    SurfSample r;
    switch (s.type) {
        case LRK_SURFACE_MATTE: r = matte_sample(s, it, wo, u_lobe, u0, u1); break;
        case LRK_SURFACE_DISNEY: r = disney_sample(s, it, wo, u_lobe, u0, u1); break;
        case LRK_SURFACE_MIRROR: r = mirror_sample(s, it, wo, u_lobe, u0, u1); break;
        case LRK_SURFACE_GLASS: r = glass_sample(s, it, wo, u_lobe, u0, u1, importance); break;
        case LRK_SURFACE_PLASTIC: r = plastic_sample(s, it, wo, u_lobe, u0, u1); break;
        case LRK_SURFACE_MIX: r = mix_sample(s, it, wo, u_lobe, u0, u1, records); break;
        case LRK_SURFACE_LAYERED: r = layered_sample(s, it, wo, u_lobe, u0, u1, records, importance); break;
        default: r = metal_sample(s, it, wo, u_lobe, u0, u1); break;
    }
    if (!validate_surface_sides(it.ng, it.shading.n, wo, r.wi)) {
        r.eval.f = v3(0.f);
        r.eval.pdf = 0.f;
    }
    return r;
}

// ------------------------------------------------------------------------------------------------
// Image textures (SURVEY.md §8 row f1): ImageTextureInstance::evaluate, src/textures/image.cpp:132-166, sampled
// with the reference's software sampler, src/compute/src/rust/luisa_compute_backend_impl/src/cpu/codegen/
// cpu_texture.h:418-464 (coordinates / bilinear), :489-493 (point), :63 (unorm conversion, done by the host loader).
// ------------------------------------------------------------------------------------------------
struct F4 {
    float x, y, z, w;
};
inline float tex_fract(float x) { return x - std::floor(x); }// device_math.h:3429
inline float tex_coord_point(uint32_t address, float uv, float s) {
    constexpr float one_minus_epsilon = 0x1.fffffep-1f;// cpu_texture.h:12
    switch (address) {
        case LRK_TEX_ADDRESS_EDGE: return std::fmin(std::fmax(uv, 0.0f), one_minus_epsilon) * s;
        case LRK_TEX_ADDRESS_REPEAT: return tex_fract(uv) * s;
        case LRK_TEX_ADDRESS_MIRROR: {
            uv = std::fmod(std::fabs(uv), 2.0f);
            uv = uv < 1.f ? uv : 2.f - uv;
            return std::fmin(uv, one_minus_epsilon) * s;
        }
        default: return (uv < 0.f || uv >= 1.f) ? 65536.f : uv * s;// ZERO: lands outside, reads 0
    }
}
inline F4 tex_read(const lrk_scene_desc &sc, const lrk_texture &t, uint32_t x, uint32_t y) {
    if (!(x < t.width && y < t.height)) return {0.f, 0.f, 0.f, 0.f};// cpu_texture.h:369-372
    const float *p = sc.texels + 4u * (t.texel_offset + static_cast<uint64_t>(y) * t.width + x);
    return {p[0], p[1], p[2], p[3]};
}
inline F4 lerp4(F4 a, F4 b, float t) { return {lerp(a.x, b.x, t), lerp(a.y, b.y, t), lerp(a.z, b.z, t), lerp(a.w, b.w, t)}; }
F4 texture_sample(const lrk_scene_desc &sc, const lrk_texture &t, float u, float v) {
    const float sx = static_cast<float>(t.width), sy = static_cast<float>(t.height);
    if (t.filter == LRK_TEX_FILTER_POINT) {
        float cx = tex_coord_point(t.address, u, sx), cy = tex_coord_point(t.address, v, sy);
        return tex_read(sc, t, static_cast<uint32_t>(cx), static_cast<uint32_t>(cy));
    }
    const float inv_sx = 1.f / sx, inv_sy = 1.f / sy;
    float ax = tex_coord_point(t.address, u - .5f * inv_sx, sx), bx = tex_coord_point(t.address, u + .5f * inv_sx, sx);
    float ay = tex_coord_point(t.address, v - .5f * inv_sy, sy), by = tex_coord_point(t.address, v + .5f * inv_sy, sy);
    float x_min = std::fmin(ax, bx), x_max = std::fmax(ax, bx), y_min = std::fmin(ay, by), y_max = std::fmax(ay, by);
    float tx = tex_fract(x_max), ty = tex_fract(y_max);
    uint32_t x0 = static_cast<uint32_t>(x_min), y0 = static_cast<uint32_t>(y_min);
    uint32_t x1 = static_cast<uint32_t>(x_max), y1 = static_cast<uint32_t>(y_max);
    F4 v00 = tex_read(sc, t, x0, y0), v01 = tex_read(sc, t, x1, y0), v10 = tex_read(sc, t, x0, y1), v11 = tex_read(sc, t, x1, y1);
    return lerp4(lerp4(v00, v01, tx), lerp4(v10, v11, tx), ty);
}
inline float tex_decode(const lrk_texture &t, float x) {// image.cpp:143-158
    if (t.encoding == LRK_TEX_ENCODING_SRGB) {
        float lin = x <= 0.04045f ? x * (1.0f / 12.92f) : builtin_pow((x + 0.055f) * (1.0f / 1.055f), 2.4f);
        return t.scale * lin;
    }
    if (t.encoding == LRK_TEX_ENCODING_GAMMA) return t.scale * builtin_pow(x, t.gamma);
    return t.scale * x;
}
F4 texture_evaluate(const lrk_scene_desc &sc, uint32_t tex_id, float u, float v) {
    const lrk_texture &t = sc.textures[tex_id];
    F4 s = texture_sample(sc, t, u * t.uv_scale[0] + t.uv_offset[0], v * t.uv_scale[1] + t.uv_offset[1]);
    return {tex_decode(t, s.x), tex_decode(t, s.y), tex_decode(t, s.z), tex_decode(t, s.w)};
}
// ------------------------------------------------------------------------------------------------
// Spherical environment: src/environments/spherical.cpp:42-137 (uv mapping, evaluate, sample); tables built by the host.
// ------------------------------------------------------------------------------------------------
V3 light_emission(const lrk_scene_desc &sc, const lrk_light &light, float u, float v) {
    if (light.emission_tex == 0u) return v3(light.emission[0], light.emission[1], light.emission[2]);
    F4 t = texture_evaluate(sc, light.emission_tex - 1u, u, v);
    return v3(std::fmax(t.x, 0.f), std::fmax(t.y, 0.f), std::fmax(t.z, 0.f));
}
inline V3 env_mul(const float m[9], V3 v, bool transposed) {// float3x3 * float3 = v.x*col0 + v.y*col1 + v.z*col2
    if (!transposed) return v.x * v3(m[0], m[3], m[6]) + v.y * v3(m[1], m[4], m[7]) + v.z * v3(m[2], m[5], m[8]);
    return v.x * v3(m[0], m[1], m[2]) + v.y * v3(m[3], m[4], m[5]) + v.z * v3(m[6], m[7], m[8]);
}
inline V3 env_radiance(const lrk_scene_desc &sc, float u, float v) {// _evaluate (:70-75) + decode_illuminant (srgb.cpp:48-54)
    const lrk_environment &e = sc.environment;
    V3 rgb = v3(e.emission[0], e.emission[1], e.emission[2]);
    if (e.emission_tex != 0u) {
        F4 t = texture_evaluate(sc, e.emission_tex - 1u, u, v);
        rgb = v3(std::fmax(t.x, 0.f), std::fmax(t.y, 0.f), std::fmax(t.z, 0.f));
    }
    return rgb * e.scale;
}
inline float env_directional_pdf(float p, float theta) {// :77-81
    float s = std::sin(theta);
    float inv_s = s > 0.f ? 1.f / s : 0.f;
    return p * inv_s * (.5f * kInvPi * kInvPi);
}
LightEval environment_evaluate(const lrk_scene_desc &sc, V3 wi) {
    const lrk_environment &e = sc.environment;
    V3 w = normalize(env_mul(e.to_world, wi, true));
    float theta = std::acos(w.y), phi = std::atan2(w.x, w.z);// direction_to_uv, :53-59
    float u = 1.f - 0.5f * kInvPi * phi, v = theta * kInvPi;
    u = u - std::floor(u);
    v = v - std::floor(v);
    LightEval out;
    out.L = env_radiance(sc, u, v);
    if (e.emission_tex == 0u) {
        out.pdf = kInvPi * 0.25f;// uniform_sphere_pdf
    } else {
        float sx = static_cast<float>(e.map_width), sy = static_cast<float>(e.map_height);
        uint32_t ix = static_cast<uint32_t>(clampf(u * sx, 0.f, sx - 1.f)), iy = static_cast<uint32_t>(clampf(v * sy, 0.f, sy - 1.f));
        out.pdf = env_directional_pdf(e.pdf[static_cast<size_t>(iy) * e.map_width + ix], theta);
    }
    return out;
}
EnvSample environment_sample(const lrk_scene_desc &sc, float u0, float u1) {
    const lrk_environment &e = sc.environment;
    EnvSample s;
    V3 w;
    if (e.emission_tex == 0u) {
        w = sample_uniform_sphere(u0, u1);
        float theta = std::acos(w.y), ph = std::atan2(w.x, w.z);
        float u = 1.f - 0.5f * kInvPi * ph, v = theta * kInvPi;
        s.eval.L = env_radiance(sc, u - std::floor(u), v - std::floor(v));
        s.eval.pdf = kInvPi * 0.25f;
    } else {
        const uint32_t W = e.map_width, H = e.map_height;
        uint32_t iy, ix;
        float uy, ux;
        sample_alias_table([&](uint32_t i) { return e.alias[i].prob; }, [&](uint32_t i) { return e.alias[i].alias; }, H, u1, iy, uy);
        const size_t offset = static_cast<size_t>(H) + static_cast<size_t>(iy) * W;
        sample_alias_table([&](uint32_t i) { return e.alias[offset + i].prob; }, [&](uint32_t i) { return e.alias[offset + i].alias; }, W, u0, ix, ux);
        float u = (static_cast<float>(ix) + ux) / static_cast<float>(W), v = (static_cast<float>(iy) + uy) / static_cast<float>(H);
        float p = e.pdf[static_cast<size_t>(iy) * W + ix];
        float phi = 2.f * kPi * (1.f - u), theta = kPi * v;// uv_to_direction, :42-51
        float y = std::cos(theta), sin_theta = std::sin(theta);
        w = normalize(v3(std::sin(phi) * sin_theta, y, std::cos(phi) * sin_theta));
        s.eval.L = env_radiance(sc, u, v);
        s.eval.pdf = env_directional_pdf(p, theta);
    }
    s.wi = normalize(env_mul(e.to_world, w, false));
    return s;
}

bool alpha_skip(const lrk_scene_desc &sc, uint32_t inst_id, uint32_t prim_id, float bu, float bv) {
    const auto &inst = sc.instances[inst_id];
    ShapeHandle shape = decode_handle(inst.handle);
    if (!((shape.flags & LRK_SHAPE_MAYBE_NON_OPAQUE) && shape.has_surface())) return false;
    const lrk_surface &surf = sc.surfaces[shape.surface_tag];
    if (!(surf.flags & LRK_SURFACE_MAYBE_NON_OPAQUE)) return false;// evaluate_opacity -> nullopt (surface.h:186)
    uint32_t ub, vb;
    std::memcpy(&ub, &bu, 4);
    std::memcpy(&vb, &bv, 4);
    const float u = static_cast<float>(xxhash32_uint4(inst_id, prim_id, ub, vb)) * 0x1p-32f;
    float alpha = surf.opacity;
    if (surf.opacity_tex != 0u) {
        const lrk_mesh &mesh = sc.meshes[shape.buffer_base / 4u];// buffer_base = mesh index * 4 (shape.cpp:46-70)
        const lrk_triangle &tri = sc.triangles[mesh.triangle_offset + prim_id];
        const lrk_vertex &a = sc.vertices[mesh.vertex_offset + tri.i0], &b = sc.vertices[mesh.vertex_offset + tri.i1],
                         &c = sc.vertices[mesh.vertex_offset + tri.i2];
        const float b0 = 1.f - bu - bv;
        float tu = b0 * a.uv[0] + bu * b.uv[0] + bv * c.uv[0], tv = b0 * a.uv[1] + bu * b.uv[1] + bv * c.uv[1];// geometry.cpp:372
        alpha = texture_evaluate(sc, surf.opacity_tex - 1u, tu, tv).x;
    }
    return u > alpha;
}

// clamp_shading_normal, src/util/frame.cpp:49-54
V3 clamp_shading_normal(V3 ns, V3 ng, V3 w) {
    V3 w_refl = reflect(-w, ns);
    V3 w_refl_clip = dot(w_refl, ng) * dot(w, ng) > 0.f ? w_refl : normalize(w_refl - ng * dot(w_refl, ng));
    return normalize(w_refl_clip + w);
}
// NormalMapWrapper::populate_closure, src/base/surface.h:236-253: the interaction the closure is bound to
Interaction closure_interaction(const lrk_scene_desc &sc, const lrk_surface &node, const Interaction &it, V3 wo) {
    if (!(node.flags & LRK_SURFACE_HAS_NORMAL_MAP)) return it;
    V3 rgb = v3(node.normal_value[0], node.normal_value[1], node.normal_value[2]);
    if (node.normal_tex != 0u) {
        F4 t = texture_evaluate(sc, node.normal_tex - 1u, it.u, it.v);
        rgb = v3(t.x, t.y, t.z);
    }
    V3 nl = 2.f * rgb + (-1.f);
    if (node.normal_strength != 1.f) nl = nl * v3(node.normal_strength, node.normal_strength, 1.f);
    V3 normal = it.shading.local_to_world(nl);
    Interaction mapped = it;
    mapped.shading = Frame::make(clamp_shading_normal(normal, it.ng, wo), it.shading.s);
    return mapped;
}

// Surface parameters at a hit (MatteInstance::populate_closure src/surfaces/matte.cpp:117-131,
// DisneySurfaceInstance::populate_closure src/surfaces/disney.cpp:932-956; colours through
// Texture::Instance::evaluate_albedo_spectrum src/base/texture.cpp:20-31 and the sRGB spectrum src/spectra/srgb.cpp:34-40,70-72)
// Mirror / Glass / Plastic / Metal with image-textured parameters (LRK_SURFACE_RAW_PARAMS, include/lrk.h): evaluate the textured
// raw parameters at the hit and derive the closure context as the surfaces' populate_closure do (mirror.cpp:142-162,
// glass.cpp:236-279, plastic.cpp:252-291, metal.cpp:273-310)
lrk_surface resolve_raw_surface(const lrk_scene_desc &sc, lrk_surface s, const Interaction &it) {
    auto colour = [&](uint32_t slot) {// evaluate_albedo_spectrum with the sRGB spectrum: saturate(extend_color_to_rgb(v))
        if (s.tex[slot] == 0u) return;
        F4 val = texture_evaluate(sc, s.tex[slot] - 1u, it.u, it.v);
        const uint32_t ch = sc.textures[s.tex[slot] - 1u].channels;
        V3 rgb = ch == 1u ? v3(val.x, val.x, val.x) : ch == 2u ? v3(val.x, val.y, 1.f) : v3(val.x, val.y, val.z);
        s.p[slot] = saturate(rgb.x);
        s.p[slot + 1u] = saturate(rgb.y);
        s.p[slot + 2u] = saturate(rgb.z);
    };
    auto alpha = [&](uint32_t slot) {// one channel feeds both axes; roughness_to_alpha = max(r^2, 1e-4) (scattering.cpp:129-135)
        if (s.tex[slot] == 0u) return;
        F4 r = texture_evaluate(sc, s.tex[slot] - 1u, it.u, it.v);
        const bool one = sc.textures[s.tex[slot] - 1u].channels == 1u;
        float ax = r.x, ay = one ? r.x : r.y;
        if (s.flags & LRK_SURFACE_REMAP_ROUGHNESS) {
            ax = std::fmax(ax * ax, 1e-4f);
            ay = std::fmax(ay * ay, 1e-4f);
        }
        s.p[slot] = ax;
        s.p[slot + 1u] = ay;
    };
    auto lum = [](const float *c) { return 0.212671f * c[0] + 0.715160f * c[1] + 0.072169f * c[2]; };// src/util/colorspace.h:21-25
    switch (s.type) {
        case LRK_SURFACE_MIRROR:
            colour(0u);
            alpha(3u);
            break;
        case LRK_SURFACE_GLASS: {
            colour(0u);
            colour(3u);
            alpha(7u);
            const float kr_lum = lum(&s.p[0]), kt_lum = lum(&s.p[3]);
            s.p[9] = kr_lum == 0.f ? 0.f : kr_lum / (kr_lum + kt_lum);
            break;
        }
        case LRK_SURFACE_PLASTIC: {
            colour(0u);
            colour(4u);
            alpha(8u);
            if (s.tex[10] != 0u) s.p[10] = texture_evaluate(sc, s.tex[10] - 1u, it.u, it.v).x;
            const float kd_lum = lum(&s.p[0]), sa_lum = lum(&s.p[4]);
            const float average_transmittance = std::exp(-2.f * sa_lum * s.p[10]);
            const float fdr = fresnel_dielectric_integral(s.p[7]);
            for (int c = 0; c < 3; c++) s.p[c] = s.p[c] / (1.f - s.p[c] * fdr);
            s.p[3] = kd_lum * average_transmittance;
            break;
        }
        default:// METAL
            colour(6u);
            alpha(9u);
            break;
    }
    return s;
}

lrk_surface resolve_surface(const lrk_scene_desc &sc, const lrk_surface &node, const Interaction &it) {
    lrk_surface s = node;
    if (!(s.flags & LRK_SURFACE_HAS_TEXTURES)) return s;
    if (s.flags & LRK_SURFACE_RAW_PARAMS) return resolve_raw_surface(sc, s, it);
    if (s.tex[0] != 0u) {
        F4 val = texture_evaluate(sc, s.tex[0] - 1u, it.u, it.v);
        const uint32_t ch = sc.textures[s.tex[0] - 1u].channels;
        V3 rgb = ch == 1u ? v3(val.x, val.x, val.x) : ch == 2u ? v3(val.x, val.y, 1.f) : v3(val.x, val.y, val.z);// texture.cpp:14-18
        rgb = v3(saturate(rgb.x), saturate(rgb.y), saturate(rgb.z));
        s.p[0] = rgb.x;
        s.p[1] = rgb.y;
        s.p[2] = rgb.z;
        if (s.type == LRK_SURFACE_DISNEY) s.p[3] = 0.212671f * rgb.x + 0.715160f * rgb.y + 0.072169f * rgb.z;
    }
    if (s.type == LRK_SURFACE_MATTE) {
        if (s.tex[3] != 0u) s.p[3] = saturate(texture_evaluate(sc, s.tex[3] - 1u, it.u, it.v).x) * 90.f;
    } else {
        for (uint32_t k = 4u; k < 16u; k++) {
            if (s.tex[k] == 0u) continue;
            float x = texture_evaluate(sc, s.tex[k] - 1u, it.u, it.v).x;
            if (k == 6u && (s.flags & LRK_SURFACE_REMAP_ROUGHNESS)) x = std::fmax(x * x, 1e-4f);// scattering.cpp:137-139
            s.p[k] = x;
        }
    }
    return s;
}

// ------------------------------------------------------------------------------------------------
// The estimator: src/integrators/mega_path.cpp:49-156 (identical, up to kernel boundaries, to
// src/integrators/wave_path.cpp:254-469).  Draw order is normative (SURVEY.md App. A).
// ------------------------------------------------------------------------------------------------
V3 path_li(const lrk_scene_desc &sc, uint32_t px, uint32_t py, uint32_t sample_index, oracle_counters *cnt) {
    Sampler sampler;
    sampler.start(sc, px, py, sample_index);
    float uf0, uf1;
    sampler.generate_pixel_2d(uf0, uf1);
    float camera_weight;
    lrk_ray ray = generate_camera_ray(sc.camera, px, py, uf0, uf1, camera_weight);
    V3 beta = v3(camera_weight);
    V3 Li = v3(0.f);
    float pdf_bsdf = 1e16f;
    TraceCounters tc;
    for (uint32_t depth = 0; depth < sc.integrator.max_depth; depth++) {
        V3 wo = -v3(ray.d[0], ray.d[1], ray.d[2]);
        lrk_hit hit = trace_bvh(sc, ray, false, &tc);
        if (cnt) cnt->closest_rays++;
        Interaction it = interaction_from_hit(sc, ray, hit);
        if (!it.valid()) {// miss: mega_path.cpp:68-75, uniform.cpp:67-76
            if (sc.environment.present) {
                LightEval e = environment_evaluate(sc, v3(ray.d[0], ray.d[1], ray.d[2]));
                e.pdf *= env_prob(sc);
                Li = Li + beta * e.L * balance_heuristic(pdf_bsdf, e.pdf);
            }
            break;
        }
        if (sc.light_count != 0u && it.shape.has_light()) {
            LightEval e = evaluate_hit(sc, it, v3(ray.o[0], ray.o[1], ray.o[2]));
            Li = Li + beta * e.L * balance_heuristic(pdf_bsdf, e.pdf);
        }
        if (!it.shape.has_surface()) break;
        if (cnt) cnt->path_vertices++;
        float u_light_selection = sampler.generate_1d();
        float ul0, ul1;
        sampler.generate_2d(ul0, ul1);
        float u_lobe = sampler.generate_1d();
        float ub0, ub1;
        sampler.generate_2d(ub0, ub1);
        float u_rr = 0.f;
        if (depth + 1u >= sc.integrator.rr_depth) u_rr = sampler.generate_1d();
        LightSample ls = sample_light(sc, it, u_light_selection, ul0, ul1);
        // the shadow ray is traced unconditionally (mega_path.cpp:108)
        bool occluded = trace_bvh(sc, ls.shadow_ray, true, &tc).inst != ~0u;
        if (cnt) cnt->shadow_rays++;
        const lrk_surface surface = resolve_surface(sc, sc.surfaces[it.shape.surface_tag], it);
        const Interaction cit = closure_interaction(sc, surface, it, wo);// the closure's (normal-mapped) view of the hit
        if (ls.eval.pdf > 0.0f && !occluded) {
            V3 wi = v3(ls.shadow_ray.d[0], ls.shadow_ray.d[1], ls.shadow_ray.d[2]);
            SurfEval ev = surface_evaluate(surface, cit, wo, wi, sc.surfaces);
            float w = balance_heuristic(ls.eval.pdf, ev.pdf) / ls.eval.pdf;
            Li = Li + w * beta * ev.f * ls.eval.L;
        }
        SurfSample ss = surface_sample(surface, cit, wo, u_lobe, ub0, ub1, sc.surfaces);
        ray = spawn_ray(it, ss.wi);
        pdf_bsdf = ss.eval.pdf;
        float w = ss.eval.pdf > 0.f ? 1.f / ss.eval.pdf : 0.f;
        beta = beta * (w * ss.eval.f);
        float eta_scale = 1.f;// mega_path.cpp:113,133-138
        if (float eta = surface_eta(surface, sc.surfaces); eta != 0.f) {// closure->eta().value_or(1.f)
            if (ss.event == LRK_EVENT_ENTER) eta_scale = sqr(eta);
            else if (ss.event == LRK_EVENT_EXIT) eta_scale = sqr(1.f / eta);
        }
        // zero_if_any_nan: src/util/spec.cpp:404-407
        if (std::isnan(beta.x) || std::isnan(beta.y) || std::isnan(beta.z)) beta = v3(0.f);
        if (beta.x <= 0.f && beta.y <= 0.f && beta.z <= 0.f) break;
        float q = std::fmax(max3(beta) * eta_scale, .05f);
        if (depth + 1u >= sc.integrator.rr_depth) {
            if (q < sc.integrator.rr_threshold && u_rr >= q) break;
            beta = beta * (q < sc.integrator.rr_threshold ? 1.0f / q : 1.f);
        }
    }
    if (cnt) {
        cnt->samples++;
        cnt->nodes_visited += tc.nodes;
        cnt->tris_tested += tc.tris;
        cnt->xforms += tc.xforms;
    }
    return Li;
}

// ------------------------------------------------------------------------------------------------
// Volumetric estimator (config C4): src/integrators/mega_vpt_naive.cpp:170-485 with
// VPT_NAIVE_ENABLE_DIRECT_LIGHTING defined (:16) and VPT_NAIVE_ENABLE_MEDIUM_STACK_INIT not (:15).
// Scope: homogeneous and vacuum media with eta = 1 (the closures are built with eta_i = 1), as the environment medium and on
// shapes; the medium tracker, the surface events and the transmittance walk through transmissive surfaces are restated in full.
// The reference's quirks are kept on purpose (they define its output):
//   * `_transmittance` (:96-168) only accumulates medium transmittance up to a surface it HITS; an unoccluded
//     shadow ray returns f = 1, pdf = 0 — light reaches surfaces unattenuated, and the in-medium direct light
//     (guarded by pdf > 0, :279) only ever adds f = Tr * bsdf(-d, d) = 0 for opaque closures;
//   * each surface hit by a transmittance ray draws three numbers from the path's PCG32 stream
//     (homogeneous.cpp:119-125), which shifts all later medium decisions — so the shadow rays must be traced;
//   * Henyey-Greenstein returns its sampled direction in a fixed y-up frame, not around wo
//     (henyey_greenstein.cpp:30-43); the phase value is not part of f/pdf (homogeneous.cpp:88-96);
//   * after a "hit surface" medium event the ray origin has moved to the surface, and that moved origin is
//     what `evaluate_hit` gets (mega_vpt_naive.cpp:308,319).
// ------------------------------------------------------------------------------------------------
struct PCG32 {// src/util/rng.cpp:142-174, constants src/util/rng.h:36-38
    uint64_t state, inc;
    static constexpr uint64_t default_state = 0x853c49e6748fea9bull;
    static constexpr uint64_t mult = 0x5851f42d4c957f2dull;
    uint32_t uniform_uint() {
        uint64_t oldstate = state;
        state = oldstate * mult + inc;
        uint32_t xorshifted = static_cast<uint32_t>(((oldstate >> 18u) ^ oldstate) >> 27u);
        uint32_t rot = static_cast<uint32_t>(oldstate >> 59u);
        return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31u));
    }
    void set_sequence(uint64_t init_seq) {
        state = 0u;
        inc = (init_seq << 1u) | 1u;
        uniform_uint();
        state = state + default_state;
        uniform_uint();
    }
    float uniform_float() { return std::fmin(kOneMinusEpsilon, static_cast<float>(uniform_uint()) * 0x1p-32f); }
};

struct MediumSample {
    V3 f{0.f, 0.f, 0.f};
    float pdf{0.f};
    V3 o{}, d{};
    uint32_t event{~0u};// 0 absorb, 1 scatter, 3 hit surface, ~0 invalid (src/base/medium.h:31-36)
};
inline float sum3(V3 a) { return a.x + a.y + a.z; }
inline float comp(V3 a, uint32_t i) { return i == 0u ? a.x : i == 1u ? a.y : a.z; }

// HomogeneousMediumClosure::sample, src/media/homogeneous.cpp:48-118
MediumSample homogeneous_sample(const lrk_medium &m, V3 o, V3 d, float t_max, PCG32 &rng) {
    V3 sigma_a = v3(m.sigma_a[0], m.sigma_a[1], m.sigma_a[2]), sigma_s = v3(m.sigma_s[0], m.sigma_s[1], m.sigma_s[2]);
    V3 sigma_t = sigma_a + sigma_s;
    MediumSample s;
    V3 pdf_channels;
    pdf_channels.x = rng.uniform_float();
    pdf_channels.y = rng.uniform_float();
    pdf_channels.z = rng.uniform_float();
    float psum = sum3(pdf_channels);
    pdf_channels = v3(pdf_channels.x / psum, pdf_channels.y / psum, pdf_channels.z / psum);
    // sample_discrete(spectrum, u): src/util/sampling.cpp:177-190
    float u_rescaled = rng.uniform_float() * sum3(pdf_channels);
    uint32_t channel = ~0u;
    float accum = 0.f;
    for (uint32_t i = 0; i < 3u; i++) {
        accum += comp(pdf_channels, i);
        if (u_rescaled <= accum) { channel = i; break; }
    }
    float u = rng.uniform_float();
    float st = channel < 3u ? comp(sigma_t, channel) : std::numeric_limits<float>::quiet_NaN();
    float t = -std::log(std::fmax(1.f - u, std::numeric_limits<float>::min())) / st;
    if (t > t_max) {
        s.event = 3u;
        t = t_max;
        V3 Tr = exp3(-sigma_t * t);
        s.o = o + d * t;
        s.d = d;
        s.f = Tr;
        s.pdf = sum3(pdf_channels * Tr);
    } else {
        float p_absorb = comp(sigma_a, channel) / st, p_scatter = comp(sigma_s, channel) / st;
        float ur = rng.uniform_float() * (p_absorb + p_scatter);// sample_discrete(float2, u): sampling.cpp:157-161
        if (ur <= p_absorb) {
            s.event = 0u;
            s.o = o;
            s.d = d;
            s.f = v3(0.f);
            s.pdf = sum3(pdf_channels * sigma_t);
        } else {
            s.event = 1u;
            V3 Tr = exp3(-sigma_t * t);
            // HenyeyGreenstein::sample_p(wo = -d, u), src/phasefunctions/henyey_greenstein.cpp:28-48
            // make_float2(rng.uniform_float(), rng.uniform_float()) (homogeneous.cpp:91): the ORDER of the two draws is the C++
            // compiler's argument evaluation order - unspecified by the language.  clang and MSVC (what the reference's
            // supported toolchains are: BUILD.md) evaluate left to right: u.x is drawn first; GCC evaluates right to left.
            // The oracle follows clang/MSVC; oracle_set_hg_args_right_to_left(1) mirrors a GCC build of the reference (the only
            // one that can be built here, oracle/ref) so that tests/test_ref_render.py can compare like with like.
            float u0, u1;
            if (g_hg_args_right_to_left.load(std::memory_order_relaxed)) { u1 = rng.uniform_float(); u0 = rng.uniform_float(); }
            else { u0 = rng.uniform_float(); u1 = rng.uniform_float(); }
            float g = m.g;
            float cosTheta = std::fabs(g) < 1e-3f ? 1.f - 2.f * u0
                                                  : -1.f / (2.f * g) * (1.f + sqr(g) - sqr((1.f - sqr(g)) / (1.f + g - 2.f * g * u0)));
            float sinTheta = std::sqrt(std::fmax(0.f, 1.f - sqr(cosTheta)));
            float phi = 2.f * kPi * u1;
            V3 wi = v3(sinTheta * std::cos(phi), cosTheta, sinTheta * std::sin(phi));
            s.o = o + d * t;
            s.d = wi;
            s.f = Tr * sigma_s;
            s.pdf = sum3(pdf_channels * (sigma_t * Tr));
        }
    }
    return s;
}

// MediumTracker (src/util/medium_tracker.{h,cpp}): the media a path is inside of, sorted by priority (lowest value first;
// equal priorities keep their order of entry).  Restated with its quirks: `size` also counts entries that were never stored
// (VACUUM_PRIORITY never sorts in front of anything), exit() scans capacity - 1 slots and clears slot `size` after removing.
struct MediumTracker {
    static constexpr uint32_t capacity = 32u;
    uint32_t priority[capacity], tag[capacity];
    uint32_t size{0u};
    MediumTracker() {
        for (uint32_t i = 0; i < capacity; i++) {
            priority[i] = LRK_MEDIUM_VACUUM_PRIORITY;
            tag[i] = LRK_MEDIUM_INVALID_TAG;
        }
    }
    bool vacuum() const { return priority[0] == LRK_MEDIUM_VACUUM_PRIORITY; }
    bool true_hit(uint32_t p) const { return p <= priority[0]; }
    uint32_t current_tag() const { return vacuum() ? LRK_MEDIUM_INVALID_TAG : tag[0]; }
    void enter(uint32_t p, uint32_t t) {
        if (size == capacity) return;// the reference logs "Medium stack overflow" and carries on
        size += 1u;
        uint32_t x = p, v = t;
        for (uint32_t i = 0; i < capacity; i++) {
            const uint32_t pi = priority[i], ti = tag[i];
            const bool swap = pi > x;
            priority[i] = swap ? x : pi;
            tag[i] = swap ? v : ti;
            x = swap ? pi : x;
            v = swap ? ti : v;
        }
    }
    void exit(uint32_t p, uint32_t t) {
        uint32_t removed = 0u;
        for (uint32_t i = 0; i < capacity - 1u; i++) {
            const bool should_remove = priority[i] == p && tag[i] == t && removed == 0u;
            removed += should_remove ? 1u : 0u;
            priority[i] = priority[i + removed];
            tag[i] = tag[i + removed];
        }
        if (removed != 0u) {
            size -= 1u;
            priority[size] = LRK_MEDIUM_VACUUM_PRIORITY;
            tag[size] = LRK_MEDIUM_INVALID_TAG;
        }// else: "trying to exit nonexistent" is logged, nothing changes
    }
};

// _event (mega_vpt_naive.cpp:68-94): which side of the surface wo and wi are on, in the closure's shading frame
uint32_t volume_surface_event(const lrk_scene_desc &sc, const Interaction &it, V3 wo, V3 wi) {
    Frame shading = it.shading;
    if (it.shape.has_surface()) {
        const lrk_surface surface = resolve_surface(sc, sc.surfaces[it.shape.surface_tag], it);
        shading = closure_interaction(sc, surface, it, wo).shading;
    }
    const V3 wo_local = shading.world_to_local(wo), wi_local = shading.world_to_local(wi);
    return wo_local.z * wi_local.z > 0.f ? LRK_EVENT_REFLECT : wi_local.z > 0.f ? LRK_EVENT_EXIT : LRK_EVENT_ENTER;
}

// _transmittance (mega_vpt_naive.cpp:96-168).  The tracker is taken BY VALUE, as the reference does: what the shadow ray enters
// and leaves does not change the path's own tracker.  Draws three numbers from rng for every surface reached inside a medium.
struct Transmittance {
    V3 f{1.f, 1.f, 1.f};
    float pdf{0.f};
};
Transmittance volume_transmittance(const lrk_scene_desc &sc, PCG32 &rng, MediumTracker tracker, lrk_ray origin_ray, TraceCounters *tc,
                                   oracle_counters *cnt) {
    float t_max = origin_ray.tmax;
    V3 dir = v3(origin_ray.d[0], origin_ray.d[1], origin_ray.d[2]);
    lrk_ray ray = origin_ray;
    V3 light_p = v3(origin_ray.o[0], origin_ray.o[1], origin_ray.o[2]) + dir * t_max;
    Transmittance T;
    while (T.f.x > 0.f || T.f.y > 0.f || T.f.z > 0.f) {
        lrk_hit hit = trace_bvh(sc, ray, false, tc);
        if (cnt) cnt->shadow_rays++;
        Interaction it = interaction_from_hit(sc, ray, hit);
        if (!it.valid()) break;
        float t2surface = length(it.pg - v3(ray.o[0], ray.o[1], ray.o[2]));
        V3 wo = -dir, wi = dir;
        const uint32_t surface_event = volume_surface_event(sc, it, wo, wi);
        if (!tracker.vacuum()) {// HomogeneousMediumClosure::transmittance, homogeneous.cpp:119-133
            const lrk_medium &m = sc.media[tracker.current_tag()];
            V3 sigma_t = v3(m.sigma_a[0] + m.sigma_s[0], m.sigma_a[1] + m.sigma_s[1], m.sigma_a[2] + m.sigma_s[2]);
            V3 pc;
            pc.x = rng.uniform_float();
            pc.y = rng.uniform_float();
            pc.z = rng.uniform_float();
            float ps = sum3(pc);
            pc = v3(pc.x / ps, pc.y / ps, pc.z / ps);
            V3 Tr = exp3(-sigma_t * t2surface);
            T.f = T.f * Tr;
            T.pdf += sum3(pc * Tr);
        }
        if (it.shape.has_medium()) {// :134-146 (a reflect event enters, like the reference's $else)
            const uint32_t tag = it.shape.medium_tag, priority = sc.media[tag].priority;
            if (surface_event == LRK_EVENT_EXIT) tracker.exit(priority, tag);
            else tracker.enter(priority, tag);
        }
        if (it.shape.has_surface()) {// :149-160: the closure is built with eta_i = 1 and evaluated straight through
            const lrk_surface surface = resolve_surface(sc, sc.surfaces[it.shape.surface_tag], it);
            SurfEval ev = surface_evaluate(surface, closure_interaction(sc, surface, it, wo), wo, wi);
            T.f = T.f * ev.f;
            T.pdf += ev.pdf;
        }
        ray = spawn_ray_to(it, light_p);
    }
    return T;
}

V3 volume_path_li(const lrk_scene_desc &sc, uint32_t px, uint32_t py, uint32_t sample_index, oracle_counters *cnt) {
    Sampler sampler;
    sampler.start(sc, px, py, sample_index);
    float uf0, uf1;
    sampler.generate_pixel_2d(uf0, uf1);
    float camera_weight;
    lrk_ray ray = generate_camera_ray(sc.camera, px, py, uf0, uf1, camera_weight);
    V3 beta = v3(camera_weight);
    V3 Li = v3(0.f);
    // PCG32 rng(U64(as<UInt2>(sampler()->generate_2d()))): x = high word, y = low word (src/util/u64.h:48,58-59)
    float s0, s1;
    sampler.generate_2d(s0, s1);
    uint32_t hi, lo;
    std::memcpy(&hi, &s0, 4);
    std::memcpy(&lo, &s1, 4);
    PCG32 rng;
    rng.set_sequence((static_cast<uint64_t>(hi) << 32u) | lo);
    // the path starts inside the environment medium (:184-190); VPT_NAIVE_ENABLE_MEDIUM_STACK_INIT is off (:15)
    MediumTracker tracker;
    if (sc.environment_medium_tag != LRK_MEDIUM_INVALID_TAG)
        tracker.enter(sc.media[sc.environment_medium_tag].priority, sc.environment_medium_tag);
    float pdf_bsdf = 1e16f;
    float eta_scale = 1.f;
    TraceCounters tc;
    for (uint32_t depth = 0; depth < sc.integrator.max_depth; depth++) {
        float eta = 1.f;
        float u_rr = 0.f;
        if (depth + 1u >= sc.integrator.rr_depth) u_rr = sampler.generate_1d();
        lrk_hit hit = trace_bvh(sc, ray, false, &tc);
        if (cnt) cnt->closest_rays++;
        Interaction it = interaction_from_hit(sc, ray, hit);
        const bool has_medium = it.valid() && it.shape.has_medium();
        V3 ro = v3(ray.o[0], ray.o[1], ray.o[2]), rd = v3(ray.d[0], ray.d[1], ray.d[2]);
        float t_max = it.valid() ? length(it.pg - ro) : std::numeric_limits<float>::max();
        MediumSample ms;
        if (!tracker.vacuum()) {// :275-311: direct light at the ray origin, then distance sampling in the current medium
            float u_sel = sampler.generate_1d();
            float ul0, ul1;
            sampler.generate_2d(ul0, ul1);
            Interaction it_medium;// Interaction{ray->origin()}: pg = ng = origin, default frame, zero offset factor
            it_medium.pg = ro;
            it_medium.ng = ro;
            it_medium.ps = v3(0.f);
            it_medium.shading = Frame{v3(1.f, 0.f, 0.f), v3(0.f, 1.f, 0.f), v3(0.f, 0.f, 1.f)};
            it_medium.shape.intersection_offset = 0.f;
            LightSample ls = sample_light(sc, it_medium, u_sel, ul0, ul1);
            Transmittance T = volume_transmittance(sc, rng, tracker, ls.shadow_ray, &tc, cnt);
            if (T.pdf > 0.f) {
                float w = 1.f / (pdf_bsdf + T.pdf + ls.eval.pdf);
                Li = Li + w * beta * T.f * ls.eval.L;
            }
            const lrk_medium &medium = sc.media[tracker.current_tag()];
            eta = medium.eta;
            ms = homogeneous_sample(medium, ro, rd, t_max, rng);
            ray = make_ray(ms.o, ms.d, 0.f, std::numeric_limits<float>::max());
            float w = ms.pdf > 0.f ? 1.f / ms.pdf : 0.f;
            beta = beta * (ms.f * w);
            pdf_bsdf = ms.pdf;
        }
        if (ms.event == ~0u || ms.event == 3u) {
            if (!it.valid()) {// :315-321
                if (sc.environment.present) {
                    LightEval e = environment_evaluate(sc, v3(ray.d[0], ray.d[1], ray.d[2]));// uniform.cpp:67-76
                    e.pdf *= env_prob(sc);
                    Li = Li + beta * e.L * balance_heuristic(pdf_bsdf, e.pdf);
                }
                break;
            }
            if (sc.light_count != 0u && it.shape.has_light()) {
                LightEval e = evaluate_hit(sc, it, v3(ray.o[0], ray.o[1], ray.o[2]));
                Li = Li + beta * e.L * balance_heuristic(pdf_bsdf, e.pdf);
            }
            if (!it.shape.has_surface()) break;
            if (cnt) cnt->path_vertices++;
            float u_light_selection = sampler.generate_1d();
            float ul0, ul1;
            sampler.generate_2d(ul0, ul1);
            float u_lobe = sampler.generate_1d();
            float ub0, ub1;
            sampler.generate_2d(ub0, ub1);
            LightSample ls = sample_light(sc, it, u_light_selection, ul0, ul1);
            Transmittance T = volume_transmittance(sc, rng, tracker, ls.shadow_ray, &tc, cnt);
            const uint32_t medium_tag = it.shape.medium_tag;// 0 for a shape without a medium (geometry.cpp:134)
            uint32_t medium_priority = LRK_MEDIUM_VACUUM_PRIORITY;
            float eta_next = 1.f;
            if (has_medium) {
                medium_priority = sc.media[medium_tag].priority;
                eta_next = sc.media[medium_tag].eta;
            }
            const V3 dir = v3(ray.d[0], ray.d[1], ray.d[2]);
            const uint32_t surface_event_skip = volume_surface_event(sc, it, -dir, dir);
            V3 wo = -dir;
            const lrk_surface surface = resolve_surface(sc, sc.surfaces[it.shape.surface_tag], it);
            const Interaction cit = closure_interaction(sc, surface, it, wo);
            uint32_t surface_event;
            // true_hit is given the medium TAG where it expects a priority (:387, medium_tracker.cpp:19-21): `tag <= priority of
            // the current medium`.  A shape without a medium has tag 0 and is always a true hit.
            if (!tracker.true_hit(medium_tag)) {
                surface_event = surface_event_skip;
                ray = spawn_ray(it, dir);
                pdf_bsdf = 1e16f;
            } else {
                if (ls.eval.pdf > 0.0f) {
                    V3 wi = v3(ls.shadow_ray.d[0], ls.shadow_ray.d[1], ls.shadow_ray.d[2]);
                    SurfEval ev = surface_evaluate(surface, cit, wo, wi);
                    float w = 1.f / (ls.eval.pdf + ev.pdf + T.pdf);
                    Li = Li + w * beta * ev.f * ls.eval.L * T.f;
                }
                SurfSample ss = surface_sample(surface, cit, wo, u_lobe, ub0, ub1);
                surface_event = ss.event;
                float w = ss.eval.pdf > 0.f ? 1.f / ss.eval.pdf : 0.f;
                pdf_bsdf = ss.eval.pdf;
                ray = spawn_ray(it, ss.wi);
                beta = beta * (w * ss.eval.f);
                if (has_medium) {// :436-446
                    if (surface_event == LRK_EVENT_ENTER) eta_scale = sqr(eta_next / eta);
                    else if (surface_event == LRK_EVENT_EXIT) eta_scale = sqr(eta / eta_next);
                }
            }
            if (has_medium) {// :449-458
                if (surface_event == LRK_EVENT_ENTER) tracker.enter(medium_priority, medium_tag);
                else if (surface_event == LRK_EVENT_EXIT) tracker.exit(medium_priority, medium_tag);
            }
        }
        if (std::isnan(beta.x) || std::isnan(beta.y) || std::isnan(beta.z)) beta = v3(0.f);
        if (beta.x <= 0.f && beta.y <= 0.f && beta.z <= 0.f) break;
        float q = std::fmax(max3(beta) * eta_scale, .05f);
        if (depth + 1u >= sc.integrator.rr_depth) {
            if (q < sc.integrator.rr_threshold && u_rr >= q) break;
            beta = beta * (q < sc.integrator.rr_threshold ? 1.0f / q : 1.f);
        }
    }
    if (cnt) {
        cnt->samples++;
        cnt->nodes_visited += tc.nodes;
        cnt->tris_tested += tc.tris;
        cnt->xforms += tc.xforms;
    }
    return Li;
}

inline V3 sample_li(const lrk_scene_desc &sc, uint32_t px, uint32_t py, uint32_t s, oracle_counters *cnt) {
    return sc.integrator.type == LRK_INTEGRATOR_VOLUME_PATH ? volume_path_li(sc, px, py, s, cnt) : path_li(sc, px, py, s, cnt);
}

// Film accumulation of one sample: src/films/color.cpp:107-130 (effective_spp = 1)
inline void film_accumulate(float *px4, V3 rgb, float film_clamp) {
    bool bad = std::isnan(rgb.x) || std::isnan(rgb.y) || std::isnan(rgb.z) || std::isinf(rgb.x) || std::isinf(rgb.y) || std::isinf(rgb.z);
    if (bad) return;
    float threshold = film_clamp * std::fmax(1.f, 1.f);
    float strength = std::fmax(std::fmax(std::fmax(std::fabs(rgb.x), std::fabs(rgb.y)), std::fabs(rgb.z)), 0.f);
    V3 c = rgb * (threshold / std::fmax(strength, threshold));
    if (c.x != 0.f || c.y != 0.f || c.z != 0.f) {
        px4[0] += c.x;
        px4[1] += c.y;
        px4[2] += c.z;
    }
    px4[3] += 1.f;
}

}// namespace

// ================================================================================================
static double g_last_render_stats[4] = {0.0, 0.0, 0.0, 0.0};// threads used, thread utilisation, work items, wall seconds

extern "C" {

// {threads, busy fraction of those threads, work items, seconds} of the last oracle_render call (bench.py reports them)
void oracle_last_render_stats(double out[4]) {
    for (int i = 0; i < 4; i++) out[i] = g_last_render_stats[i];
}

int oracle_render(const lrk_scene_desc *scene, uint32_t spp_begin, uint32_t spp_end, uint32_t threads, uint32_t rank,
                  uint32_t world, uint32_t tile_size, float *film_raw, oracle_counters *counters) {
    if (!scene || !film_raw || scene->abi_version != LRK_ABI_VERSION) return -1;
    if (scene->integrator.type == LRK_INTEGRATOR_VOLUME_PATH) {
        // supported volume scope: homogeneous / vacuum media with eta = 1 (see volume_path_li)
        for (uint32_t m = 0; m < scene->medium_count; m++)
            if (scene->media[m].present == LRK_MEDIUM_HOMOGENEOUS && scene->media[m].eta != 1.f) return -5;
    } else if (scene->integrator.type != LRK_INTEGRATOR_PATH || scene->environment_medium.present) {
        return -5;
    }
    // the table-driven samplers are defined for the sample indices [0, spp) that Sampler::Instance::reset prepared them for
    if (scene->sampler.type != LRK_SAMPLER_INDEPENDENT && spp_end > scene->sampler.spp) return -2;
    const uint32_t W = scene->camera.resolution[0], H = scene->camera.resolution[1];
    if (threads == 0u) threads = std::max(1u, std::thread::hardware_concurrency());
    // Work items: the 8x8-pixel blocks this shard OWNS, listed up front and handed out through one atomic cursor.  (Round 1
    // walked every 16x16 block of the whole frame and skipped foreign pixels inside: a 1/76 shard then had ~100 productive
    // items for 128 threads and the timed CPU arm starved - VERDICT r01 "what's weak" #1.)
    const uint32_t ts = 8u;
    const uint32_t tiles_x = (W + ts - 1u) / ts, tiles_y = (H + ts - 1u) / ts;
    auto owned = [&](uint32_t x, uint32_t y) {
        if (tile_size == 0u || world <= 1u) return true;
        uint32_t shard_tiles_x = (W + tile_size - 1u) / tile_size;
        uint32_t tile_id = (y / tile_size) * shard_tiles_x + (x / tile_size);
        return lrk_tile_owner(tile_id, world) == rank;
    };
    std::vector<uint32_t> items;
    for (uint32_t t = 0; t < tiles_x * tiles_y; t++) {
        const uint32_t tx = t % tiles_x, ty = t / tiles_x;
        bool any = false;
        for (uint32_t y = ty * ts; y < std::min(H, (ty + 1u) * ts) && !any; y++)
            for (uint32_t x = tx * ts; x < std::min(W, (tx + 1u) * ts) && !any; x++) any = owned(x, y);
        if (any) items.push_back(t);
    }
    threads = std::max(1u, std::min<uint32_t>(threads, static_cast<uint32_t>(std::max<size_t>(items.size(), 1u))));
    std::atomic<uint32_t> next{0u};
    std::vector<oracle_counters> local(threads);
    std::vector<double> busy(threads, 0.0);
    const auto t_begin = std::chrono::steady_clock::now();
    auto worker = [&](uint32_t tid) {
        oracle_counters c{};
        const auto t0 = std::chrono::steady_clock::now();
        for (;;) {
            uint32_t k = next.fetch_add(1u);
            if (k >= items.size()) break;
            uint32_t t = items[k];
            uint32_t tx = t % tiles_x, ty = t / tiles_x;
            for (uint32_t y = ty * ts; y < std::min(H, (ty + 1u) * ts); y++) {
                for (uint32_t x = tx * ts; x < std::min(W, (tx + 1u) * ts); x++) {
                    if (!owned(x, y)) continue;
                    float *px4 = film_raw + (static_cast<size_t>(y) * W + x) * 4u;
                    for (uint32_t s = spp_begin; s < spp_end; s++) {
                        V3 li = sample_li(*scene, x, y, s, &c);
                        film_accumulate(px4, li * 1.0f, scene->film.clamp);// shutter weight 1
                    }
                }
            }
        }
        busy[tid] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        local[tid] = c;
    };
    std::vector<std::thread> pool;
    for (uint32_t i = 1; i < threads; i++) pool.emplace_back(worker, i);
    worker(0u);
    for (auto &t : pool) t.join();
    {// how well the host threads were fed: sum of the workers' busy time / (threads x wall time of the parallel region)
        const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
        double sum = 0.0;
        for (double b : busy) sum += b;
        g_last_render_stats[0] = static_cast<double>(threads);
        g_last_render_stats[1] = wall > 0.0 ? sum / (wall * threads) : 0.0;
        g_last_render_stats[2] = static_cast<double>(items.size());
        g_last_render_stats[3] = wall;
    }
    if (counters) {
        for (auto &c : local) {
            counters->samples += c.samples;
            counters->closest_rays += c.closest_rays;
            counters->shadow_rays += c.shadow_rays;
            counters->nodes_visited += c.nodes_visited;
            counters->tris_tested += c.tris_tested;
            counters->xforms += c.xforms;
            counters->path_vertices += c.path_vertices;
        }
    }
    return 0;
}

void oracle_convert_film(const lrk_scene_desc *scene, const float *film_raw, float *rgba) {
    const size_t n = static_cast<size_t>(scene->camera.resolution[0]) * scene->camera.resolution[1];
    for (size_t i = 0; i < n; i++) {
        float nrm = std::fmax(film_raw[i * 4 + 3], 1.f);
        float inv = 1.f / nrm;
        for (int c = 0; c < 3; c++) rgba[i * 4 + c] = (inv * scene->film.scale[c]) * film_raw[i * 4 + c];
        rgba[i * 4 + 3] = 1.f;
    }
}

void oracle_li(const lrk_scene_desc *scene, uint32_t px, uint32_t py, uint32_t sample_index, float rgb[3]) {
    V3 li = sample_li(*scene, px, py, sample_index, nullptr);
    rgb[0] = li.x; rgb[1] = li.y; rgb[2] = li.z;
}

int oracle_trace(const lrk_scene_desc *scene, const lrk_ray *rays, uint64_t n, int any_hit, lrk_hit *hits,
                 oracle_counters *counters) {
    if (!scene || !rays || !hits) return -1;
    TraceCounters tc;
    for (uint64_t i = 0; i < n; i++) {
        lrk_hit h = trace_bvh(*scene, rays[i], any_hit != 0, &tc);
        if (any_hit) h = {h.inst != ~0u ? 1u : 0u, 0u, {0.f, 0.f}};
        hits[i] = h;
    }
    if (counters) {
        counters->nodes_visited += tc.nodes;
        counters->tris_tested += tc.tris;
        counters->xforms += tc.xforms;
        (any_hit ? counters->shadow_rays : counters->closest_rays) += n;
    }
    return 0;
}

int oracle_trace_brute(const lrk_scene_desc *scene, const lrk_ray *rays, uint64_t n, int any_hit, lrk_hit *hits) {
    if (!scene || !rays || !hits) return -1;
    for (uint64_t i = 0; i < n; i++) {
        lrk_hit h = trace_brute(*scene, rays[i], any_hit != 0);
        if (any_hit) h = {h.inst != ~0u ? 1u : 0u, 0u, {0.f, 0.f}};
        hits[i] = h;
    }
    return 0;
}

uint32_t oracle_xxhash32_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return xxhash32_uint4(x, y, z, w); }
float oracle_lcg(uint32_t *state) { return lcg(*state); }

void oracle_sample_filter(const lrk_scene_desc *scene, const float u[2], float offset[2], float *weight) {
    sample_filter(scene->camera, u[0], u[1], offset[0], offset[1], *weight);
}

void oracle_generate_ray(const lrk_scene_desc *scene, uint32_t px, uint32_t py, uint32_t sample_index, lrk_ray *ray,
                         float weight[3], uint32_t *rng_state) {
    Sampler s;
    s.start(*scene, px, py, sample_index);
    float u0, u1;
    s.generate_pixel_2d(u0, u1);
    float w;
    *ray = generate_camera_ray(scene->camera, px, py, u0, u1, w);
    weight[0] = weight[1] = weight[2] = w;
    if (rng_state) *rng_state = s.state;
}

int oracle_sampler_state(const lrk_scene_desc *scene, const uint32_t *points, uint64_t n, const uint32_t *dims, uint32_t dim_count,
                         uint32_t bounces, uint64_t *index_out, uint64_t *zsobol_out, float *draws_out) {
    if (!scene || !points || !index_out || !zsobol_out || !draws_out || (dim_count != 0u && !dims)) return -1;
    const lrk_sampler &cfg = scene->sampler;
    for (uint64_t i = 0; i < n; i++)// PMJ02BN's pixel samples exist for [0, spp) only
        if (cfg.type == LRK_SAMPLER_PMJ02BN && points[3u * i + 2u] >= cfg.spp) return -2;
    const uint32_t per_point = 2u + 6u * bounces;
    for (uint64_t i = 0; i < n; i++) {
        Sampler s;
        s.start(*scene, points[3u * i], points[3u * i + 1u], points[3u * i + 2u]);
        index_out[i] = cfg.type == LRK_SAMPLER_SOBOL || cfg.type == LRK_SAMPLER_ZSOBOL ? s.sobol_index : 0u;
        for (uint32_t j = 0; j < dim_count; j++) {
            uint64_t v = 0u;
            if (cfg.type == LRK_SAMPLER_ZSOBOL) {
                Sampler d = s;
                d.dimension = dims[j];
                v = d.zsobol_sample_index();
            }
            zsobol_out[i * dim_count + j] = v;
        }
        float *u = draws_out + i * per_point;
        s.generate_pixel_2d(u[0], u[1]);
        for (uint32_t b = 0; b < bounces; b++, u += 6) {// path_li: light selection, light point, lobe, BSDF direction
            u[2] = s.generate_1d();
            s.generate_2d(u[3], u[4]);
            u[5] = s.generate_1d();
            s.generate_2d(u[6], u[7]);
        }
    }
    return 0;
}

void oracle_offset_ray_origin(const float p[3], const float n[3], float out[3]) {
    V3 r = offset_ray_origin(v3(p[0], p[1], p[2]), v3(n[0], n[1], n[2]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}

void oracle_decode_handle(const uint32_t handle[4], uint32_t out_u32[6], float out_f32[2]) {
    ShapeHandle h = decode_handle(handle);
    out_u32[0] = h.buffer_base; out_u32[1] = h.flags; out_u32[2] = h.surface_tag; out_u32[3] = h.light_tag;
    out_u32[4] = h.medium_tag; out_u32[5] = h.tri_count;
    out_f32[0] = h.shadow_terminator; out_f32[1] = h.intersection_offset;
}

void oracle_sample_cosine_hemisphere(const float u[2], float w[3]) {
    V3 r = sample_cosine_hemisphere(u[0], u[1]);
    w[0] = r.x; w[1] = r.y; w[2] = r.z;
}
void oracle_sample_uniform_triangle(const float u[2], float uvw[3]) {
    V3 r = sample_uniform_triangle(u[0], u[1]);
    uvw[0] = r.x; uvw[1] = r.y; uvw[2] = r.z;
}

static Interaction synthetic_interaction(const float ng[3], const float ns[3], const float dpdu[3]) {
    Interaction it;
    it.ng = v3(ng[0], ng[1], ng[2]);
    it.shading = Frame::make(face_forward(v3(ns[0], ns[1], ns[2]), it.ng), v3(dpdu[0], dpdu[1], dpdu[2]));
    it.inst = 0u;
    it.prim = 0u;
    it.shape.intersection_offset = 1.f;
    return it;
}

void oracle_surface_evaluate(const lrk_surface *surface, const float ng[3], const float ns[3], const float dpdu[3],
                             const float wo[3], const float wi[3], float f[3], float *pdf) {
    Interaction it = synthetic_interaction(ng, ns, dpdu);
    SurfEval e = surface_evaluate(*surface, it, v3(wo[0], wo[1], wo[2]), v3(wi[0], wi[1], wi[2]));
    f[0] = e.f.x; f[1] = e.f.y; f[2] = e.f.z;
    *pdf = e.pdf;
}

void oracle_surface_sample(const lrk_surface *surface, const float ng[3], const float ns[3], const float dpdu[3],
                           const float wo[3], float u_lobe, const float u[2], float wi[3], float f[3], float *pdf) {
    Interaction it = synthetic_interaction(ng, ns, dpdu);
    SurfSample s = surface_sample(*surface, it, v3(wo[0], wo[1], wo[2]), u_lobe, u[0], u[1]);
    wi[0] = s.wi.x; wi[1] = s.wi.y; wi[2] = s.wi.z;
    f[0] = s.eval.f.x; f[1] = s.eval.f.y; f[2] = s.eval.f.z;
    *pdf = s.eval.pdf;
}

void oracle_interaction(const lrk_scene_desc *scene, const lrk_ray *ray, const lrk_hit *hit, float out[19]) {
    Interaction it = interaction_from_hit(*scene, *ray, *hit);
    const float vals[19]{it.pg.x, it.pg.y, it.pg.z, it.ng.x, it.ng.y, it.ng.z, it.shading.n.x, it.shading.n.y, it.shading.n.z,
                         it.shading.s.x, it.shading.s.y, it.shading.s.z, it.shading.t.x, it.shading.t.y, it.shading.t.z,
                         it.u, it.v, it.prim_area, it.back_facing ? 1.f : 0.f};
    std::memcpy(out, vals, sizeof(vals));
}

void oracle_sample_light(const lrk_scene_desc *scene, const lrk_ray *ray, const lrk_hit *hit, float u_sel,
                         const float u_light[2], float out[12]) {
    Interaction it = interaction_from_hit(*scene, *ray, *hit);
    LightSample s = sample_light(*scene, it, u_sel, u_light[0], u_light[1]);
    const float vals[12]{s.eval.L.x, s.eval.L.y, s.eval.L.z, s.eval.pdf, s.shadow_ray.o[0], s.shadow_ray.o[1], s.shadow_ray.o[2],
                         s.shadow_ray.tmin, s.shadow_ray.d[0], s.shadow_ray.d[1], s.shadow_ray.d[2], s.shadow_ray.tmax};
    std::memcpy(out, vals, sizeof(vals));
}

void oracle_environment_sample(const lrk_scene_desc *scene, const float u[2], float out[7]) {
    EnvSample s = environment_sample(*scene, u[0], u[1]);
    const float vals[7]{s.eval.L.x, s.eval.L.y, s.eval.L.z, s.eval.pdf, s.wi.x, s.wi.y, s.wi.z};
    std::memcpy(out, vals, sizeof(vals));
}

void oracle_environment_evaluate(const lrk_scene_desc *scene, const float wi[3], float out[4]) {
    LightEval e = environment_evaluate(*scene, v3(wi[0], wi[1], wi[2]));
    out[0] = e.L.x, out[1] = e.L.y, out[2] = e.L.z, out[3] = e.pdf;
}

void oracle_texture_evaluate(const lrk_scene_desc *scene, uint32_t texture_id, const float uv[2], float out[4]) {
    F4 v = texture_evaluate(*scene, texture_id, uv[0], uv[1]);
    out[0] = v.x, out[1] = v.y, out[2] = v.z, out[3] = v.w;
}

void oracle_resolve_surface(const lrk_scene_desc *scene, uint32_t surface_tag, const float uv[2], lrk_surface *out) {
    Interaction it;
    it.u = uv[0];
    it.v = uv[1];
    *out = resolve_surface(*scene, scene->surfaces[surface_tag], it);
}

}// extern "C"

// ------------------------------------------------------------------------------------------------
// oracle_unit: one named numerical unit on packed 32-bit words (floats as bit patterns), the same names, argument order
// and result packing as the reference pins in oracle/ref/pins.cpp, so tests/test_ref_pins.py can compare them 1:1.
// ------------------------------------------------------------------------------------------------
namespace {
struct Words {
    const uint32_t *in;
    uint32_t *out;
    float f() { float v; std::memcpy(&v, in++, 4); return v; }
    uint32_t u() { return *in++; }
    V3 v() { float x = f(), y = f(), z = f(); return {x, y, z}; }
    void put(float v) { std::memcpy(out++, &v, 4); }
    void put(uint32_t v) { *out++ = v; }
    void put(V3 v) { put(v.x); put(v.y); put(v.z); }
    void put(bool b) { put(b ? 1.0f : 0.0f); }
};
template<typename B>
void put_bxdf_sample(Words &w, const B &bxdf, V3 wo, float u0, float u1) {// BxDF::sample, scattering.cpp:247-254
    BxDFSample s = bxdf.sample_wi(wo, u0, u1);
    w.put(s.wi);
    w.put(s.valid ? bxdf.pdf(wo, s.wi) : 0.f);
    w.put(s.valid ? bxdf.evaluate(wo, s.wi) : v3(0.f));
}
struct LambertBxDF {
    V3 r;
    BxDFSample sample_wi(V3 wo, float u0, float u1) const { return lambert_sample_wi(wo, u0, u1); }
    float pdf(V3 wo, V3 wi) const { return lambert_pdf(wo, wi); }
    V3 evaluate(V3 wo, V3 wi) const { return lambert_evaluate(r, wo, wi); }
};
}// namespace

extern "C" void oracle_set_trace_brute_force(int enabled) { g_trace_brute_force.store(enabled != 0); }
extern "C" void oracle_set_hg_args_right_to_left(int enabled) { g_hg_args_right_to_left.store(enabled != 0); }

// the Layered surface on the records of a flattened scene: same row layout as tests/host_device/closures_host.cpp device_layered_unit
extern "C" int oracle_layered_unit(const lrk_surface *records, uint32_t index, const float *in, float *out, int count) {
    for (int i = 0; i < count; i++, in += 16, out += 12) {
        Interaction it{};
        it.pg = v3(in[0], in[1], in[2]);
        it.ng = normalize(v3(in[3], in[4], in[5]));
        it.shading = Frame::make(it.ng);
        const V3 wo = normalize(v3(in[6], in[7], in[8])), wi = normalize(v3(in[9], in[10], in[11]));
        const SurfEval e = surface_evaluate(records[index], it, wo, wi, records);
        const SurfSample s = surface_sample(records[index], it, wo, in[12], in[13], in[14], records);
        out[0] = e.f.x; out[1] = e.f.y; out[2] = e.f.z; out[3] = e.pdf;
        out[4] = s.wi.x; out[5] = s.wi.y; out[6] = s.wi.z;
        out[7] = s.eval.f.x; out[8] = s.eval.f.y; out[9] = s.eval.f.z; out[10] = s.eval.pdf;
        out[11] = static_cast<float>(s.event);
    }
    return 0;
}

extern "C" int oracle_unit(const char *name_c, const uint32_t *in, uint32_t *out, int count, const void *buffer, uint64_t buffer_count) {
    const std::string name{name_c};
    Words w{in, out};
    for (int n = 0; n < count; n++) {
        if (name == "xxhash32_4") { uint32_t a = w.u(), b = w.u(), c = w.u(), d = w.u(); w.put(xxhash32_uint4(a, b, c, d)); }
        else if (name == "permutation_element") { uint32_t i = w.u(), l = w.u(), m = w.u(), p = w.u(); w.put(Sampler::permutation_element(i, l, m, p)); }
        else if (name == "uniform_uint_to_float") { w.put(std::fmin(kOneMinusEpsilon, static_cast<float>(w.u()) * 0x1p-32f)); }
        else if (name == "lcg") { uint32_t st = w.u(); float u = lcg(st); w.put(u); w.put(st); }
        else if (name == "pcg32_seq") {
            uint32_t hi = w.u(), lo = w.u();
            PCG32 rng{};
            rng.set_sequence((static_cast<uint64_t>(hi) << 32u) | lo);
            for (int i = 0; i < 4; i++) { w.put(rng.uniform_uint()); }
            w.put(rng.uniform_float());
            w.put(rng.uniform_float());
            w.put(static_cast<uint32_t>(rng.state >> 32u)); w.put(static_cast<uint32_t>(rng.state));
            w.put(static_cast<uint32_t>(rng.inc >> 32u)); w.put(static_cast<uint32_t>(rng.inc));
        }
        else if (name == "sample_uniform_triangle") { float a = w.f(), b = w.f(); w.put(sample_uniform_triangle(a, b)); }
        else if (name == "sample_uniform_disk_concentric") { float a = w.f(), b = w.f(), x, y; sample_uniform_disk_concentric(a, b, x, y); w.put(x); w.put(y); }
        else if (name == "sample_cosine_hemisphere") { float a = w.f(), b = w.f(); w.put(sample_cosine_hemisphere(a, b)); }
        else if (name == "cosine_hemisphere_pdf") { w.put(w.f() * kInvPi); }
        else if (name == "sample_uniform_sphere") { float a = w.f(), b = w.f(); w.put(sample_uniform_sphere(a, b)); }
        else if (name == "balance_heuristic") { float a = w.f(), b = w.f(); w.put(balance_heuristic(a, b)); }
        else if (name == "sample_alias_table") {
            auto table = static_cast<const lrk_alias_entry *>(buffer);
            uint32_t cnt = w.u(), index; float u = w.f(), uu;
            if (cnt > buffer_count) { return -2; }
            sample_alias_table([&](uint32_t i) { return table[i].prob; }, [&](uint32_t i) { return table[i].alias; }, cnt, u, index, uu);
            w.put(index); w.put(uu);
        }
        else if (name == "frame_make_n") { Frame f = Frame::make(w.v()); w.put(f.s); w.put(f.t); w.put(f.n); }
        else if (name == "frame_make_ns") { V3 nn = w.v(), ss = w.v(); Frame f = Frame::make(nn, ss); w.put(f.s); w.put(f.t); w.put(f.n); }
        else if (name == "frame_local_to_world") { V3 s = w.v(), t = w.v(), nn = w.v(), d = w.v(); w.put(Frame{s, t, nn}.local_to_world(d)); }
        else if (name == "frame_world_to_local") { V3 s = w.v(), t = w.v(), nn = w.v(), d = w.v(); w.put(Frame{s, t, nn}.world_to_local(d)); }
        else if (name == "clamp_shading_normal") { V3 ns = w.v(), ng = w.v(), d = w.v(); w.put(clamp_shading_normal(ns, ng, d)); }
        else if (name == "refract") { V3 wi = w.v(), nn = w.v(); float eta = w.f(); V3 wt; bool ok = refract(wi, nn, eta, wt); w.put(ok); w.put(wt); }
        else if (name == "face_forward") { V3 a = w.v(), b = w.v(); w.put(face_forward(a, b)); }
        else if (name == "spherical_direction") { float a = w.f(), b = w.f(), c = w.f(); w.put(spherical_direction(a, b, c)); }
        else if (name == "spherical_theta") { w.put(spherical_theta(w.v())); }
        else if (name == "spherical_phi") { w.put(spherical_phi(w.v())); }
        else if (name == "tr_roughness_to_alpha") { w.put(std::fmax(sqr(w.f()), 1e-4f)); }
        else if (name == "tr_D") { float ax = w.f(), ay = w.f(); w.put(TrowbridgeReitz{ax, ay}.D(w.v())); }
        else if (name == "tr_Lambda") { float ax = w.f(), ay = w.f(); w.put(TrowbridgeReitz{ax, ay}.Lambda(w.v())); }
        else if (name == "tr_G1") { float ax = w.f(), ay = w.f(); w.put(TrowbridgeReitz{ax, ay}.G1(w.v())); }
        else if (name == "tr_G") { float ax = w.f(), ay = w.f(); V3 a = w.v(), b = w.v(); w.put(TrowbridgeReitz{ax, ay}.G(a, b)); }
        else if (name == "tr_sample_wh") { float ax = w.f(), ay = w.f(); V3 wo = w.v(); float a = w.f(), b = w.f(); w.put(TrowbridgeReitz{ax, ay}.sample_wh(wo, a, b)); }
        else if (name == "tr_pdf") { float ax = w.f(), ay = w.f(); V3 a = w.v(), b = w.v(); w.put(TrowbridgeReitz{ax, ay}.pdf(a, b)); }
        else if (name == "fresnel_dielectric") { float a = w.f(), b = w.f(), c = w.f(); w.put(fresnel_dielectric(a, b, c)); }
        else if (name == "fresnel_conductor") { float a = w.f(), b = w.f(); V3 e = w.v(), k = w.v(); w.put(fresnel_conductor(a, b, e, k)); }
        else if (name == "fresnel_dielectric_integral") { w.put(fresnel_dielectric_integral(w.f())); }
        else if (name == "lambert_reflection_evaluate") { V3 r = w.v(), wo = w.v(), wi = w.v(); w.put(lambert_evaluate(r, wo, wi)); }
        else if (name == "lambert_reflection_sample") { V3 r = w.v(), wo = w.v(); float a = w.f(), b = w.f(); put_bxdf_sample(w, LambertBxDF{r}, wo, a, b); }
        else if (name == "lambert_reflection_pdf") { w.v(); V3 wo = w.v(), wi = w.v(); w.put(lambert_pdf(wo, wi)); }
        else if (name == "oren_nayar_evaluate") { V3 r = w.v(); float sg = w.f(); V3 wo = w.v(), wi = w.v(); w.put(OrenNayar{r, sg}.evaluate(wo, wi)); }
        else if (name == "microfacet_reflection_dielectric_evaluate" || name == "microfacet_reflection_dielectric_pdf" ||
                 name == "microfacet_reflection_dielectric_sample") {
            V3 r = w.v(); float ax = w.f(), ay = w.f(), ei = w.f(), et = w.f(); V3 wo = w.v();
            MicrofacetReflection bxdf{r, TrowbridgeReitz{ax, ay}, FresnelTerm::dielectric(ei, et)};
            if (name.back() == 'e' && name[name.size() - 2] == 't') { w.put(bxdf.evaluate(wo, w.v())); }
            else if (name.back() == 'f') { w.put(bxdf.pdf(wo, w.v())); }
            else { float a = w.f(), b = w.f(); put_bxdf_sample(w, bxdf, wo, a, b); }
        }
        else if (name == "microfacet_reflection_conductor_evaluate" || name == "microfacet_reflection_conductor_sample") {
            V3 r = w.v(); float ax = w.f(), ay = w.f(); V3 eta = w.v(), k = w.v(), wo = w.v();
            MicrofacetReflection bxdf{r, TrowbridgeReitz{ax, ay}, FresnelTerm::conductor(1.f, eta, k)};
            if (name.back() == 'e' && name[name.size() - 2] == 't') { w.put(bxdf.evaluate(wo, w.v())); }
            else { float a = w.f(), b = w.f(); put_bxdf_sample(w, bxdf, wo, a, b); }
        }
        else if (name == "microfacet_transmission_evaluate" || name == "microfacet_transmission_pdf" || name == "microfacet_transmission_sample") {
            V3 t = w.v(); float ax = w.f(), ay = w.f(), ea = w.f(), eb = w.f(); V3 wo = w.v();
            MicrofacetTransmission bxdf{t, TrowbridgeReitz{ax, ay}, ea, eb};
            if (name.back() == 'e' && name[name.size() - 2] == 't') { w.put(bxdf.evaluate(wo, w.v())); }
            else if (name.back() == 'f') { w.put(bxdf.pdf(wo, w.v())); }
            else { float a = w.f(), b = w.f(); put_bxdf_sample(w, bxdf, wo, a, b); }
        }
        else if (name == "fresnel_blend_evaluate" || name == "fresnel_blend_pdf" || name == "fresnel_blend_sample") {
            V3 rd = w.v(), rs = w.v(); float ax = w.f(), ay = w.f(), ratio = w.f(); V3 wo = w.v();
            FresnelBlend bxdf{rd, rs, TrowbridgeReitz{ax, ay}, ratio};
            if (name.back() == 'e' && name[name.size() - 2] == 't') { w.put(bxdf.evaluate(wo, w.v())); }
            else if (name.back() == 'f') { w.put(bxdf.pdf(wo, w.v())); }
            else { float a = w.f(), b = w.f(); put_bxdf_sample(w, bxdf, wo, a, b); }
        }
        else if (name.rfind("_evaluate") != std::string::npos || name.rfind("_sample") != std::string::npos) {
            // closure pins (oracle/ref/pin_<surface>.cpp): context words in lrk_surface.p order, then ng, ns, tangent, wo, ...
            lrk_surface sf{};
            auto take = [&](int count, int at = 0) { for (int i = 0; i < count; i++) sf.p[at + i] = w.f(); };
            bool is_eval = name.find("_evaluate") != std::string::npos;
            if (name.rfind("matte_", 0) == 0) { sf.type = LRK_SURFACE_MATTE; take(4); }
            else if (name.rfind("disney_", 0) == 0 || name.rfind("disneytrans_", 0) == 0 || name.rfind("disneythin_", 0) == 0) {
                const bool thin = name.rfind("disneythin_", 0) == 0;
                sf.type = LRK_SURFACE_DISNEY; take(thin ? 16 : 15);
                sf.lobes = static_cast<uint32_t>(std::stoul(name.substr(name.rfind('_') + 1)));
                if (name.rfind("disneytrans_", 0) == 0) sf.flags |= LRK_SURFACE_DISNEY_TRANSMISSIVE;// closure class "disney_trans"
                if (thin) sf.flags |= LRK_SURFACE_DISNEY_THIN;                                       // closure class "disney_thin"
            }
            else if (name.rfind("mirror_", 0) == 0) { sf.type = LRK_SURFACE_MIRROR; take(5); }
            else if (name.rfind("glass_", 0) == 0) { sf.type = LRK_SURFACE_GLASS; take(10); }
            else if (name.rfind("plastic_", 0) == 0) { sf.type = LRK_SURFACE_PLASTIC; take(10); }
            else if (name.rfind("metal_", 0) == 0) { sf.type = LRK_SURFACE_METAL; take(11); }
            else { return -1; }
            V3 ng = w.v(), ns = w.v(), tg = w.v(), wo = w.v();
            Interaction it;
            it.ng = ng;
            it.shading = Frame::make(ns, tg);
            if (is_eval) {
                SurfEval e = surface_evaluate(sf, it, wo, w.v());
                w.put(e.f); w.put(e.pdf);
            } else {
                float ul = w.f(), u0 = w.f(), u1 = w.f();
                SurfSample r = surface_sample(sf, it, wo, ul, u0, u1);
                w.put(r.wi); w.put(r.eval.f); w.put(r.eval.pdf); w.put(r.event);
            }
        }
        else { return -1; }
    }
    return 0;
}
