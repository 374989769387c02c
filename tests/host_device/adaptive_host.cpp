// adaptive_host.cpp — the adaptive mode's pixel error (luisarender_b200/csrc/device/adaptive.h, the header the sm_90a test kernel
// includes) compiled for the host, so that tests/test_adaptive_cpu.py can hold it against a numpy restatement without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>

#include "../../luisarender_b200/csrc/device/adaptive.h"

extern "C" int adaptive_error_host(const float *s1, const float *s2, const float *n, float *e, float *v, int64_t count) {
    for (int64_t i = 0; i < count; i++) {
        e[i] = lrk::adaptive_error(s1[i], s2[i], n[i]);
        v[i] = lrk::adaptive_variance(s1[i], s2[i], n[i]);
    }
    return 0;
}
