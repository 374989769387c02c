// The per-mesh area alias tables that pick emissive triangles: the host's scene flattening (flatten.cpp) and the device library's
// mesh updates (lrk_update_meshes) compile these same expressions, so that an update writes the tables a fresh flattening of the
// deformed scene would carry, bit for bit.  Both compile them for the host without contraction into FMAs (the host library with
// -ffp-contract=off, lrk.cu's host code with -Xcompiler -ffp-contract=off).
//
// Plain C++: tests/host_device compiles it for the host too.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../../include/lrk.h"

namespace lrk {

// The area weight of a triangle: |length(cross(p1 - p0, p2 - p0))| in float, evaluated in the order of the host's vecmath.h.
inline float triangle_area_weight(const float p0[3], const float p1[3], const float p2[3]) {
    const float a[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
    const float b[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
    const float c[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
    return std::abs(std::sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]));
}

// Alias table construction, restating src/util/sampling.cpp:38-87 (sum in double, table in float,
// LIFO over/under work lists, leftovers forced to probability 1).
inline void create_alias_table(const float *values, size_t n, std::vector<lrk_alias_entry> &table, std::vector<float> &pdf) {
    double sum = 0.0;
    for (size_t i = 0; i < n; i++) sum += std::abs(values[i]);
    pdf.resize(n);
    if (sum == 0.0) {
        for (size_t i = 0; i < n; i++) pdf[i] = static_cast<float>(1.0 / static_cast<double>(n));
    } else {
        auto inv_sum = 1.0 / sum;
        for (size_t i = 0; i < n; i++) pdf[i] = static_cast<float>(std::abs(values[i]) * inv_sum);
    }
    auto ratio = static_cast<double>(n) / sum;
    std::vector<uint32_t> over, under;
    table.resize(n);
    for (uint32_t i = 0; i < n; i++) {
        auto p = static_cast<float>(values[i] * ratio);
        table[i] = {p, i};
        (p > 1.0f ? over : under).push_back(i);
    }
    while (!over.empty() && !under.empty()) {
        auto o = over.back();
        auto u = under.back();
        over.pop_back();
        under.pop_back();
        table[o].prob -= 1.0f - table[u].prob;
        table[u].alias = o;
        if (table[o].prob > 1.0f) over.push_back(o);
        else if (table[o].prob < 1.0f) under.push_back(o);
    }
    for (auto i : over) table[i] = {1.0f, i};
    for (auto i : under) table[i] = {1.0f, i};
}

// The area alias table of one mesh: its triangles' area weights over its own vertex records.
inline void mesh_area_alias_table(const lrk_vertex *vertices, const lrk_triangle *triangles, size_t triangle_count,
                                  std::vector<lrk_alias_entry> &table, std::vector<float> &pdf) {
    std::vector<float> areas(triangle_count);
    for (size_t i = 0; i < triangle_count; i++)
        areas[i] = triangle_area_weight(vertices[triangles[i].i0].p, vertices[triangles[i].i1].p, vertices[triangles[i].i2].p);
    create_alias_table(areas.data(), areas.size(), table, pdf);
}

}// namespace lrk
