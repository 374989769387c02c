// hit_kinds_host.cpp — luisarender_b200/csrc/device/hit_kinds.h compiled for the host (tests/test_hit_kinds_cpu.py).
#include <cstdint>

#include "../../luisarender_b200/csrc/device/hit_kinds.h"

extern "C" {
// kinds[i] = hit_kind_of(surfaces[i])
void hit_kinds_of_surfaces(const lrk_surface *surfaces, uint32_t count, uint32_t *kinds) {
    for (uint32_t i = 0; i < count; i++) kinds[i] = lrk::hit_kind_of(surfaces[i]);
}
// bit k: hit_kind_always_strict(k); also checks that with_hit_kind hands every kind back as itself
uint32_t hit_kinds_always_strict_mask() {
    uint32_t mask = 0u;
    for (uint32_t k = 0; k < lrk::kHitKinds; k++)
        lrk::with_hit_kind(k, [&](auto c) {
            if (decltype(c)::value == k && lrk::hit_kind_always_strict(decltype(c)::value)) mask |= 1u << k;
        });
    return mask;
}
uint32_t hit_kinds_count() { return lrk::kHitKinds; }
}
