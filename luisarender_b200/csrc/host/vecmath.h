// Minimal host-side vector/matrix types for scene flattening (fp32, like the reference's
// host math in src/compute/include/luisa/core/mathematics.h; matrices are column-major there,
// we keep column vectors m.c[col] to make the transcription of transform products obvious).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace lrh {

struct float2 { float x{}, y{}; };
struct float3 {
    float x{}, y{}, z{};
    float &operator[](int i) { return (&x)[i]; }
    float operator[](int i) const { return (&x)[i]; }
};
struct float4 {
    float x{}, y{}, z{}, w{};
    float &operator[](int i) { return (&x)[i]; }
    float operator[](int i) const { return (&x)[i]; }
};

inline float3 operator+(float3 a, float3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
inline float3 operator-(float3 a, float3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline float3 operator*(float3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
inline float3 operator*(float s, float3 a) { return {a.x * s, a.y * s, a.z * s}; }
inline float3 operator-(float3 a) { return {-a.x, -a.y, -a.z}; }
inline float3 &operator+=(float3 &a, float3 b) { a = a + b; return a; }
inline float dot(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline float3 cross(float3 a, float3 b) {
    return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
inline float length(float3 a) { return std::sqrt(dot(a, a)); }
inline float3 normalize(float3 a) { return a * (1.0f / length(a)); }
inline float3 min3(float3 a, float3 b) { return {std::fmin(a.x, b.x), std::fmin(a.y, b.y), std::fmin(a.z, b.z)}; }
inline float3 max3(float3 a, float3 b) { return {std::fmax(a.x, b.x), std::fmax(a.y, b.y), std::fmax(a.z, b.z)}; }

// 4x4 with column vectors (m.c[j] is column j), so (A*B).c[j] = A * B.c[j].
struct float4x4 {
    float4 c[4];
    static float4x4 identity() {
        float4x4 m;
        m.c[0] = {1, 0, 0, 0}; m.c[1] = {0, 1, 0, 0}; m.c[2] = {0, 0, 1, 0}; m.c[3] = {0, 0, 0, 1};
        return m;
    }
    bool is_identity() const {
        auto id = identity();
        return std::memcmp(this, &id, sizeof(id)) == 0 ||
               (c[0].x == 1 && c[0].y == 0 && c[0].z == 0 && c[0].w == 0 &&
                c[1].x == 0 && c[1].y == 1 && c[1].z == 0 && c[1].w == 0 &&
                c[2].x == 0 && c[2].y == 0 && c[2].z == 1 && c[2].w == 0 &&
                c[3].x == 0 && c[3].y == 0 && c[3].z == 0 && c[3].w == 1);
    }
};

inline float4 mul(const float4x4 &m, float4 v) {
    return {m.c[0].x * v.x + m.c[1].x * v.y + m.c[2].x * v.z + m.c[3].x * v.w,
            m.c[0].y * v.x + m.c[1].y * v.y + m.c[2].y * v.z + m.c[3].y * v.w,
            m.c[0].z * v.x + m.c[1].z * v.y + m.c[2].z * v.z + m.c[3].z * v.w,
            m.c[0].w * v.x + m.c[1].w * v.y + m.c[2].w * v.z + m.c[3].w * v.w};
}
inline float4x4 operator*(const float4x4 &a, const float4x4 &b) {
    float4x4 r;
    for (int j = 0; j < 4; j++) r.c[j] = mul(a, b.c[j]);
    return r;
}
inline float3 transform_point(const float4x4 &m, float3 p) {
    auto v = mul(m, {p.x, p.y, p.z, 1.f});
    return {v.x, v.y, v.z};
}

// row-major 3x4 (what the C-ABI carries)
inline void to_rows_3x4(const float4x4 &m, float out[12]) {
    for (int r = 0; r < 3; r++)
        for (int col = 0; col < 4; col++) out[r * 4 + col] = m.c[col][r];
}

constexpr float kPi = 3.14159265358979323846264338327950288f;
// host-side radians(): src/compute/include/luisa/core/mathematics.h:70 (left-to-right: (deg*pi)/180)
inline float radians(float deg) { return deg * kPi / 180.0f; }

}// namespace lrh
