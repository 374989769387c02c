// scene_check_host.cpp — the check of a scene description that lrk_upload_scene makes before it changes anything
// (luisarender_b200/csrc/device/scene_check.h) compiled for the host, so that tests/test_scene_check_cpu.py can check descriptions
// and read what the upload would commit without a GPU.
// TEST INFRASTRUCTURE: nothing here is part of the product.
#include <cstdint>
#include <cstring>

#include "../../luisarender_b200/csrc/device/scene_check.h"

namespace {

template<typename T>
size_t copy_out(const std::vector<T> &v, void *out) {
    if (out != nullptr && !v.empty()) std::memcpy(out, v.data(), v.size() * sizeof(T));
    return v.size();
}

}// namespace

extern "C" {

// The check under the light options (bit 0 light_tree, 1 light_tree_triangles, 2 light_solid_angle, 3 light_receiver), the option
// light_candidates and the option device_bvh; free with scene_check_free
void *scene_check_run(const lrk_scene_desc *s, uint32_t light_bits, uint32_t candidates, int device_bvh) {
    lrk::LightSampling light;
    light.tree = (light_bits & 1u) != 0u;
    light.triangles = (light_bits & 2u) != 0u;
    light.solid_angle = (light_bits & 4u) != 0u;
    light.receiver = (light_bits & 8u) != 0u;
    light.candidates = candidates;
    return new lrk::SceneCheck(lrk::check_scene_desc(*s, light, device_bvh != 0));
}

void scene_check_free(void *h) { delete static_cast<lrk::SceneCheck *>(h); }

int scene_check_status(const void *h) { return static_cast<const lrk::SceneCheck *>(h)->status; }

const char *scene_check_error(const void *h) { return static_cast<const lrk::SceneCheck *>(h)->error.c_str(); }

// volume, volume_general, textured, any_non_opaque, used_kinds, tlas_root, node_count, largest_mesh
void scene_check_scalars(const void *h, uint64_t out[8]) {
    const auto &r = *static_cast<const lrk::SceneCheck *>(h);
    const uint64_t v[8] = {r.volume, r.volume_general, r.textured, r.any_non_opaque, r.used_kinds, r.tlas_root, r.node_count, r.largest_mesh};
    std::memcpy(out, v, sizeof(v));
}

// The array `name` into `out` (when not null); returns its length.  uint32: inst_kind, inst_mesh, visible, mesh_root,
// light_inst, light_mesh; uint8: mesh_emissive, light_two_sided; float: light_o2w; double: light_power; ~0 for another name.
size_t scene_check_array(const void *h, const char *name, void *out) {
    const auto &r = *static_cast<const lrk::SceneCheck *>(h);
    const std::string n{name};
    if (n == "inst_kind") return copy_out(r.inst_kind, out);
    if (n == "inst_mesh") return copy_out(r.inst_mesh, out);
    if (n == "visible") return copy_out(r.visible, out);
    if (n == "mesh_root") return copy_out(r.mesh_root, out);
    if (n == "mesh_emissive") return copy_out(r.mesh_emissive, out);
    if (n == "light_inst") return copy_out(r.light_source.inst, out);
    if (n == "light_mesh") return copy_out(r.light_source.mesh, out);
    if (n == "light_o2w") return copy_out(r.light_source.o2w, out);
    if (n == "light_power") return copy_out(r.light_source.power, out);
    if (n == "light_two_sided") return copy_out(r.light_source.two_sided, out);
    return ~size_t{0};
}

// The light source's instance count, and the meshes that have points, into `meshes` (when not null); returns their number
size_t scene_check_light_meshes(const void *h, uint32_t *instance_count, uint32_t *meshes) {
    const auto &src = static_cast<const lrk::SceneCheck *>(h)->light_source;
    *instance_count = src.instance_count;
    size_t k = 0;
    for (const auto &kv : src.mesh_points) {
        if (meshes != nullptr) meshes[k] = kv.first;
        k++;
    }
    return k;
}

// The points of emissive mesh `mesh` (9 floats per triangle) into `out` (when not null); returns their number of floats
size_t scene_check_mesh_points(const void *h, uint32_t mesh, float *out) {
    const auto &points = static_cast<const lrk::SceneCheck *>(h)->light_source.mesh_points;
    const auto it = points.find(mesh);
    return it == points.end() ? 0u : copy_out(it->second, out);
}
}
