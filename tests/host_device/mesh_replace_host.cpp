// mesh_replace_host.cpp — the node move of lrk_replace_meshes (relayout_node_refs, luisarender_b200/csrc/device/bvh_refit.h) compiled
// for the host, so that tests/test_mesh_replace_cpu.py can move flattened hierarchies to a new layout without a GPU.  The device's
// relayout_nodes_kernel moves every node of a run with the same function.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>

#include "../../include/lrk.h"
#include "../../luisarender_b200/csrc/device/bvh_refit.h"

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
