// bvh_refit_host.cpp — the refit arithmetic of lrk_update_meshes and the node move of lrk_replace_meshes
// (luisarender_b200/csrc/device/bvh_refit.h) and the shared area alias tables (luisarender_b200/csrc/device/alias_table.h) compiled
// for the host, so that tests/test_mesh_update_cpu.py and tests/test_mesh_replace_cpu.py can refit flattened hierarchies to
// deformed vertices, move them to a new layout and rebuild alias tables without a GPU.  The refit's walk here is a recursive one
// over the reachable nodes; the device kernel visits the same nodes bottom-up and computes every box with the same functions.
// The device's relayout_nodes_kernel moves every node of a run with the same function as relayout_nodes here.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/lrk.h"
#include "../../luisarender_b200/csrc/device/alias_table.h"
#include "../../luisarender_b200/csrc/device/bvh_refit.h"

namespace {

struct Refit {
    lrk_bvh_node *nodes;
    uint32_t begin, end;// the mesh's node range
    const float *tri_verts;// 12 floats per slot, the deformed positions
    float pad;
    int error{0};

    lrk::BuildBox slot_box(uint32_t slot) const {
        const float *r = tri_verts + 12u * static_cast<size_t>(slot);
        return lrk::refit_triangle_box(r, r + 4, r + 8);
    }
    // the unpadded box of the subtree `ref`; writes the padded child boxes of every inner node on the way
    lrk::BuildBox fit(uint32_t ref) {
        if (ref == LRK_BVH_EMPTY) return lrk::refit_empty_box();
        if (ref & LRK_BVH_LEAF) {
            const uint32_t first = ref & 0x0fffffffu, count = ((ref >> 28u) & 7u) + 1u;
            lrk::BuildBox boxes[LRK_BVH_MAX_LEAF_TRIS];
            for (uint32_t k = 0; k < count; k++) boxes[k] = slot_box(first + k);
            return lrk::refit_leaf_box(boxes, count);
        }
        if (ref < begin || ref >= end) {
            error = 1;
            return lrk::refit_empty_box();
        }
        lrk_bvh_node &n = nodes[ref];
        const lrk::BuildBox b0 = fit(n.ref0), b1 = fit(n.ref1);
        float f[12];
        lrk::refit_node_boxes(lrk::refit_padded(b0, pad), lrk::refit_padded(b1, pad), f);
        std::memcpy(n.lo0, f, 3 * sizeof(float));
        std::memcpy(n.hi0, f + 3, 3 * sizeof(float));
        std::memcpy(n.lo1, f + 6, 3 * sizeof(float));
        std::memcpy(n.hi1, f + 9, 3 * sizeof(float));
        return lrk::refit_union(b0, b1);
    }
};

}// namespace

// Refits the hierarchy of one mesh (nodes[root .. end), its slots [slot_offset, +slot_count) of tri_verts) in place; returns the
// pad it used through *pad_out, and 0 (or 1 when a reference leaves the node range).
extern "C" int refit_mesh(lrk_bvh_node *nodes, uint32_t root, uint32_t end, const float *tri_verts, uint32_t slot_offset, uint32_t slot_count, float *pad_out) {
    Refit r{nodes, root, end, tri_verts, 0.f};
    lrk::BuildBox whole = r.slot_box(slot_offset);
    for (uint32_t s = 1; s < slot_count; s++) whole = lrk::refit_union(whole, r.slot_box(slot_offset + s));
    r.pad = lrk::refit_pad(lrk::refit_extent(whole));
    *pad_out = r.pad;
    r.fit(root);
    return r.error;
}

// The area alias table of one mesh from its vertices (lrk_vertex records) and triangles
extern "C" void mesh_alias_table(const lrk_vertex *vertices, const lrk_triangle *triangles, uint32_t triangle_count, lrk_alias_entry *table_out, float *pdf_out) {
    std::vector<lrk_alias_entry> table;
    std::vector<float> pdf;
    lrk::mesh_area_alias_table(vertices, triangles, triangle_count, table, pdf);
    std::memcpy(table_out, table.data(), table.size() * sizeof(lrk_alias_entry));
    std::memcpy(pdf_out, pdf.data(), pdf.size() * sizeof(float));
}

// dst[i] = src[i] moved by node_delta nodes and slot_delta triangle slots (both modulo 2^32), for i < count
extern "C" void relayout_nodes(const lrk_bvh_node *src, lrk_bvh_node *dst, uint32_t count, uint32_t node_delta, uint32_t slot_delta) {
    for (uint32_t i = 0; i < count; i++) {
        lrk_bvh_node n = src[i];
        uint32_t words[3] = {n.ref0, n.ref1, n.parent};
        lrk::relayout_node_refs(words, node_delta, slot_delta);
        n.ref0 = words[0];
        n.ref1 = words[1];
        n.parent = words[2];
        dst[i] = n;
    }
}
