// The world-to-object rows of an instance from its object-to-world rows: the host's scene flattening (flatten.cpp) and the
// device library's instance updates (lrk_update_instances) compile these same expressions, so that an update writes the rows
// a fresh flattening of the moved scene would carry, bit for bit.  Both compile them without contraction into FMAs (the host
// with -ffp-contract=off, lrk.cu with -fmad=false), and the IEEE double operations then round identically.
//
// Plain C++ without CUDA built-ins: tests/host_device compiles it for the host too.
#pragma once

#ifdef __CUDACC__
#define LRK_AFFINE_FN __host__ __device__ __forceinline__
#else
#define LRK_AFFINE_FN inline
#endif

namespace lrk {

// Inverse of the affine transform with row-major 3x4 rows m (linear part m[4r + c], translation m[4r + 3]) in double precision,
// as row-major 3x4 floats.  False, with `out` untouched, when the linear part is singular (determinant exactly 0).
LRK_AFFINE_FN bool inverse_affine_rows(const float m[12], float out[12]) {
    double a[3][3], t[3];
    for (int r = 0; r < 3; r++) {
        for (int col = 0; col < 3; col++) a[r][col] = m[r * 4 + col];
        t[r] = m[r * 4 + 3];
    }
    double det = a[0][0] * (a[1][1] * a[2][2] - a[1][2] * a[2][1]) -
                 a[0][1] * (a[1][0] * a[2][2] - a[1][2] * a[2][0]) +
                 a[0][2] * (a[1][0] * a[2][1] - a[1][1] * a[2][0]);
    if (det == 0.0) return false;
    double id = 1.0 / det, inv[3][3];
    inv[0][0] = (a[1][1] * a[2][2] - a[1][2] * a[2][1]) * id;
    inv[0][1] = (a[0][2] * a[2][1] - a[0][1] * a[2][2]) * id;
    inv[0][2] = (a[0][1] * a[1][2] - a[0][2] * a[1][1]) * id;
    inv[1][0] = (a[1][2] * a[2][0] - a[1][0] * a[2][2]) * id;
    inv[1][1] = (a[0][0] * a[2][2] - a[0][2] * a[2][0]) * id;
    inv[1][2] = (a[0][2] * a[1][0] - a[0][0] * a[1][2]) * id;
    inv[2][0] = (a[1][0] * a[2][1] - a[1][1] * a[2][0]) * id;
    inv[2][1] = (a[0][1] * a[2][0] - a[0][0] * a[2][1]) * id;
    inv[2][2] = (a[0][0] * a[1][1] - a[0][1] * a[1][0]) * id;
    for (int r = 0; r < 3; r++) {
        for (int col = 0; col < 3; col++) out[r * 4 + col] = static_cast<float>(inv[r][col]);
        out[r * 4 + 3] = static_cast<float>(-(inv[r][0] * t[0] + inv[r][1] * t[1] + inv[r][2] * t[2]));
    }
    return true;
}

}// namespace lrk
