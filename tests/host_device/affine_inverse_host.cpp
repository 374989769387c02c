// affine_inverse_host.cpp — the instances' world-to-object inverse (luisarender_b200/csrc/device/affine_inverse.h, the header the
// host's flattening and the device library's instance updates include) compiled for the host, so that
// tests/test_scene_update_cpu.py can check it against the rows of flattened scenes without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include "../../luisarender_b200/csrc/device/affine_inverse.h"

extern "C" int affine_inverse_rows(const float *o2w, float *w2o, int count) {
    int singular = 0;
    for (int i = 0; i < count; i++)
        if (!lrk::inverse_affine_rows(o2w + 12 * i, w2o + 12 * i)) singular++;
    return singular;
}
