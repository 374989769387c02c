// The receiver word of the option "light_receiver" (DESIGN.md §4 (Receiver-aware light sampling)): one 32-bit word per path that
// holds the geometric normal of the vertex that sampled a light, face-forwarded to the side the outgoing direction leaves from, as
// an octahedral encoding, plus a one-sided bit.  The shade kernels encode it where they sample a light, use the decoded word there and
// store the word with the continuing path, so that the emitter hit of the next depth evaluates the light pdf from the same bits.
//
// Plain C++ without CUDA built-ins: the shade kernels (shading.cuh, shade_kernels.cuh) and tests/host_device compile the same
// expressions.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define LRK_RECEIVER_FN __host__ __device__ __forceinline__
#else
#define LRK_RECEIVER_FN inline
#endif

namespace lrk {

// bits 0..14: u, 15..29: v (octahedral coordinates in [-1, 1], 32767 steps); bit 30: one-sided; bit 31: a receiver is present.
// The word 0 is no receiver (the camera vertex, or the option off): every consumer then computes what it computed without it.
constexpr uint32_t kReceiverPresent = 0x80000000u;
constexpr uint32_t kReceiverOneSided = 0x40000000u;
constexpr float kReceiverSteps = 32767.f;

// Kind of a decoded receiver.  One-sided: the closure at the vertex returns f = 0 and pdf = 0 for every direction on the other side
// of the normal, so lights wholly behind its plane can be culled; two-sided: the |cos| term, which never culls.
enum ReceiverKind : uint32_t { kReceiverNone = 0u, kReceiverTwoSided = 1u, kReceiverOneSidedKind = 2u };

struct Receiver {
    float x, y, z;// unit normal (0 for kReceiverNone)
    uint32_t kind;
};

LRK_RECEIVER_FN float receiver_sign(float a) { return a >= 0.f ? 1.f : -1.f; }

LRK_RECEIVER_FN uint32_t receiver_quantize(float a) {
    const float q = floorf((fminf(fmaxf(a, -1.f), 1.f) * 0.5f + 0.5f) * kReceiverSteps + 0.5f);
    return static_cast<uint32_t>(q);
}

// The word of the (not necessarily unit, nonzero) normal n.  A zero or NaN normal gives the two-sided word of +z's octant: such a
// vertex gets no cull and a bounded warp.
LRK_RECEIVER_FN uint32_t receiver_encode(float nx, float ny, float nz, bool one_sided) {
    const float s = fabsf(nx) + fabsf(ny) + fabsf(nz);
    if (!(s > 0.f)) return kReceiverPresent | receiver_quantize(0.f) | (receiver_quantize(0.f) << 15u);
    float u = nx / s, v = ny / s;
    if (nz < 0.f) {
        const float ou = (1.f - fabsf(v)) * receiver_sign(u), ov = (1.f - fabsf(u)) * receiver_sign(v);
        u = ou;
        v = ov;
    }
    return kReceiverPresent | (one_sided ? kReceiverOneSided : 0u) | receiver_quantize(u) | (receiver_quantize(v) << 15u);
}

LRK_RECEIVER_FN Receiver receiver_decode(uint32_t word) {
    Receiver r{0.f, 0.f, 0.f, kReceiverNone};
    if (!(word & kReceiverPresent)) return r;
    float u = static_cast<float>(word & 0x7fffu) * (2.f / kReceiverSteps) - 1.f;
    float v = static_cast<float>((word >> 15u) & 0x7fffu) * (2.f / kReceiverSteps) - 1.f;
    const float z = 1.f - fabsf(u) - fabsf(v);
    if (z < 0.f) {
        const float ou = (1.f - fabsf(v)) * receiver_sign(u), ov = (1.f - fabsf(u)) * receiver_sign(v);
        u = ou;
        v = ov;
    }
    const float inv = 1.f / sqrtf(u * u + v * v + z * z);
    r.x = u * inv;
    r.y = v * inv;
    r.z = z * inv;
    r.kind = (word & kReceiverOneSided) ? kReceiverOneSidedKind : kReceiverTwoSided;
    return r;
}

// The receiver in an instance's object space: the normal times the transpose of the object-to-world linear part m (row-major 3x3),
// normalised.  n.(M x) = (M^T n).x: the side of the receiver's plane a point lies on is the same in both spaces, for any invertible
// (also mirrored or non-uniform) transform.
LRK_RECEIVER_FN Receiver receiver_to_object(const float *m, Receiver r) {
    if (r.kind == kReceiverNone) return r;
    const float x = m[0] * r.x + m[3] * r.y + m[6] * r.z;
    const float y = m[1] * r.x + m[4] * r.y + m[7] * r.z;
    const float z = m[2] * r.x + m[5] * r.y + m[8] * r.z;
    const float inv = 1.f / sqrtf(x * x + y * y + z * z);
    return {x * inv, y * inv, z * inv, r.kind};
}

}// namespace lrk
