// The check of a scene description that lrk_upload_scene makes before it changes anything, and the values it derives from the
// description on the host.  The check reads the description and the options the upload reads, and nothing else: a refused upload
// leaves the context as it was, and an accepted one commits from the values returned here.
//
// Plain C++ without CUDA built-ins: lrk.cu and tests/host_device compile the same code.
#pragma once
#include <algorithm>
#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "../../../include/lrk.h"
#include "hit_kinds.h"

namespace lrk {

// How next-event estimation picks a light and a point on it: the options "light_tree", "light_tree_triangles" (the light tree's
// bottom level: set with tree only), "light_solid_angle", "light_candidates" (M: 0 .. 32, resampling from M candidates for
// M >= 2) and "light_receiver" (the receiver's normal in the tree and the solid-angle sampler: set with tree or solid angle only; no
// instantiation of its own).  Not part of the ABI.
struct LightSampling {
    bool tree{false}, triangles{false}, solid_angle{false}, receiver{false};
    uint32_t candidates{0u};
};

// What the light tree of the option "light_tree" and its bottom trees are built from, copied from the scene description by
// lrk_upload_scene so that every scene update rebuilds them with the same code: per instance that carries a light (in instance
// order) its mesh, object-to-world rows, power (luminance of the emission x the light's scale) and sidedness, and per such mesh
// the object-space positions of its triangles' vertices (9 floats per triangle).
struct LightTreeSource {
    uint32_t instance_count{0};
    std::vector<uint32_t> inst, mesh;
    std::vector<float> o2w;
    std::vector<double> power;
    std::vector<uint8_t> two_sided;
    std::map<uint32_t, std::vector<float>> mesh_points;
};

constexpr uint32_t kMaxDepth = 63u;// the path state counts per depth in 64 slots (pathstate.cuh: kMaxDepthSlots)

// The hierarchy's references hold node indices below 2^31 - 1 and triangle slots below 2^28 (lrk.h: LRK_BVH_LEAF), and the mesh
// records 32-bit vertex offsets
inline bool fits_bvh_encoding(uint64_t nodes, uint64_t triangles, uint64_t vertices = 0u) {
    return nodes < 0x7fffffffull && triangles < (1ull << 28) && vertices <= 0xffffffffull;
}

// The outcome of check_scene_desc: a refusal (status != LRK_OK, with its message) or what the upload derives from the description
struct SceneCheck {
    int status{LRK_OK};
    std::string error;
    bool volume{false};
    bool volume_general{false};// the volume integrator's per-thread kernel (volume_general.cuh) instead of the wavefront one
    bool textured{false};      // some surface has image-textured parameters or a normal map, or some light an image emission
    bool any_non_opaque{false};// some instance with a surface carries LRK_SHAPE_MAYBE_NON_OPAQUE
    uint32_t used_kinds{1u};   // bit k: an instance has hit kind k (bit 0 always: emitter-only hits of an image emission)
    std::vector<uint32_t> inst_kind, inst_mesh;// per instance
    std::vector<uint32_t> visible;             // the visible instances in order
    std::vector<uint8_t> mesh_emissive;        // per mesh: an instance with a light uses it
    LightTreeSource light_source;              // with the option "light_tree"
    // the hierarchy's node layout: the description's, or with the option "device_bvh" the device builder's (per mesh
    // max(n - 1, 1) nodes in mesh order, then the instance level)
    std::vector<uint32_t> mesh_root;
    uint32_t tlas_root{0u};
    uint64_t node_count{0u};
    uint64_t largest_mesh{0u};// triangles of the largest mesh (device_bvh only)
};

namespace scene_check_detail {

inline SceneCheck refuse(int status, const char *message) {
    SceneCheck r;
    r.status = status;
    r.error = message;
    return r;
}

// The light tree's input from the scene's own arrays: every instance that carries a light - not only the first light_count
// handles -, the emission (the mean of max(texel, 0) of an image emission), the sidedness and the emissive meshes' triangles.
// check_scene_desc has checked the light tags, the mesh indices and the emission texture ids.
inline void capture_light_source(const lrk_scene_desc &s, LightTreeSource &src) {
    src = LightTreeSource{};
    src.instance_count = s.instance_count;
    for (uint32_t i = 0; i < s.instance_count; i++) {
        const auto &inst = s.instances[i];
        if (!(inst.handle[0] & LRK_SHAPE_HAS_LIGHT)) continue;
        const lrk_light &light = s.lights[inst.handle[1] & 4095u];
        double rgb[3] = {light.emission[0], light.emission[1], light.emission[2]};
        if (light.emission_tex != 0u) {
            const lrk_texture &t = s.textures[light.emission_tex - 1u];
            const size_t texels = static_cast<size_t>(t.width) * t.height;
            double sum[3] = {0.0, 0.0, 0.0};
            for (size_t k = 0; k < texels; k++)
                for (int c = 0; c < 3; c++) sum[c] += std::max(static_cast<double>(s.texels[(t.texel_offset + k) * 4u + c]), 0.0);
            for (int c = 0; c < 3; c++) rgb[c] = sum[c] / static_cast<double>(texels);
        }
        for (double &c : rgb) c = std::max(c, 0.0);
        const double lum = 0.2126 * rgb[0] + 0.7152 * rgb[1] + 0.0722 * rgb[2];
        src.inst.push_back(i);
        src.mesh.push_back(inst.mesh);
        src.o2w.insert(src.o2w.end(), inst.object_to_world, inst.object_to_world + 12);
        src.power.push_back(lum * light.scale);
        src.two_sided.push_back(light.two_sided != 0u ? 1u : 0u);
        auto &points = src.mesh_points[inst.mesh];
        if (!points.empty()) continue;
        const lrk_mesh &mesh = s.meshes[inst.mesh];
        for (uint32_t t = 0; t < mesh.triangle_count; t++) {
            const lrk_triangle &tri = s.triangles[mesh.triangle_offset + t];
            for (uint32_t v : {tri.i0, tri.i1, tri.i2}) points.insert(points.end(), s.vertices[mesh.vertex_offset + v].p, s.vertices[mesh.vertex_offset + v].p + 3);
        }
    }
}

}// namespace scene_check_detail

// Every check lrk_upload_scene makes of the description `s` under the requested light sampling and the option "device_bvh", in
// the order the upload has always made them, and with a pass the values the upload commits.  Reads only the description.
inline SceneCheck check_scene_desc(const lrk_scene_desc &s, const LightSampling &light, bool device_bvh) {
    using scene_check_detail::refuse;
    if (s.abi_version != LRK_ABI_VERSION) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: ABI version mismatch");
    SceneCheck r;
    // The volume integrator has two implementations.  The wavefront kernels (kernels.cuh) cover config C4's shape: ONE homogeneous
    // environment medium around opaque Matte / Disney closures, nothing else.  Everything beyond that - media bound to shapes,
    // transmissive surfaces, no environment medium, an environment light - runs the per-thread kernel of volume_general.cuh.
    r.volume = s.integrator.type == LRK_INTEGRATOR_VOLUME_PATH;
    if (r.volume) {
        if (s.medium_count > 256u || (s.medium_count != 0u && s.media == nullptr)) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: invalid media table");
        if (s.environment_medium_tag != LRK_MEDIUM_INVALID_TAG && s.environment_medium_tag >= s.medium_count)
            return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: environment medium tag outside the media table");
        for (uint32_t m = 0; m < s.medium_count; m++) {
            if (s.media[m].present != LRK_MEDIUM_HOMOGENEOUS && s.media[m].present != LRK_MEDIUM_VACUUM)
                return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: unknown medium kind");
            if (s.media[m].present == LRK_MEDIUM_HOMOGENEOUS && s.media[m].eta != 1.f)
                return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: media with eta != 1 are not supported");
        }
        bool general = !s.environment_medium.present || s.medium_count != 1u || s.environment.present;
        for (uint32_t i = 0; i < s.instance_count && !general; i++)
            if (s.instances[i].handle[0] & LRK_SHAPE_HAS_MEDIUM) general = true;
        for (uint32_t i = 0; i < s.surface_count && !general; i++)
            if (s.surfaces[i].type > LRK_SURFACE_DISNEY || (s.surfaces[i].flags & (LRK_SURFACE_DISNEY_TRANSMISSIVE | LRK_SURFACE_DISNEY_THIN))) general = true;
        for (uint32_t i = 0; i < s.instance_count; i++) {
            const uint32_t flags = s.instances[i].handle[0] & 1023u, tag = (s.instances[i].handle[1] >> 24u) & 255u;
            if ((flags & LRK_SHAPE_HAS_MEDIUM) && tag >= s.medium_count)
                return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: a shape's medium tag is outside the media table");
        }
        if (general && s.sampler.type != LRK_SAMPLER_INDEPENDENT)
            return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: the volume path with shape media / transmissive surfaces takes the Independent sampler");
        if (s.integrator.max_depth > 31u) return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: volume path depth > 31");
        r.volume_general = general;
    } else if (s.integrator.type != LRK_INTEGRATOR_PATH) {
        return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: unknown integrator type");
    } else if (s.environment_medium.present) {
        return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: an environment medium needs the volume path integrator (MegaVPTNaive)");
    }
    if (s.integrator.max_depth > kMaxDepth) return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: max depth > 63");
    if (light.tree && r.volume)
        return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: the light tree (option light_tree) serves the surface integrator only; the volume "
                                           "integrator selects its lights uniformly");
    if (light.triangles && !light.tree)
        return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: the triangle-level light trees (option light_tree_triangles) are the bottom "
                                                "level of the light tree: set the option light_tree too");
    if (light.solid_angle && r.volume)
        return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: solid-angle light sampling (option light_solid_angle) serves the surface integrator "
                                           "only; the volume integrator evaluates its light pdfs from the world origin");
    if (light.candidates >= 2u && r.volume)
        return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: resampled next-event estimation (option light_candidates >= 2) serves the surface "
                                           "integrator only; the volume integrator traces every light sample it draws, since the "
                                           "occlusion of each advances its random stream");
    if (light.receiver && r.volume)
        return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: receiver-aware light sampling (option light_receiver) serves the surface integrator "
                                           "only; the volume integrator selects its lights uniformly by area");
    if (light.receiver && !light.tree && !light.solid_angle)
        return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: receiver-aware light sampling (option light_receiver) refines the light tree "
                                                "and solid-angle sampling: set the option light_tree or light_solid_angle too");
    if (s.camera.resolution[0] > 65535u || s.camera.resolution[1] > 65535u)
        return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: film larger than 65535 pixels per side");
    if (s.light_count == 0u && !s.environment.present)// !pipeline().has_lighting(), wave_path.cpp:224-228
        return refuse(LRK_ERR_INVALID_ARGUMENT, "No lights in scene. Rendering aborted.");
    if (s.environment.present) {
        const auto &e = s.environment;
        if (e.emission_tex > s.texture_count || !(e.env_prob > 0.f && e.env_prob <= 1.f) ||
            (e.emission_tex != 0u && (e.map_width == 0u || e.map_height == 0u || e.alias == nullptr || e.pdf == nullptr)))
            return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: invalid environment record");
        if (s.light_count == 0u && e.env_prob != 1.f) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: env_prob must be 1 without area lights");
    }
    for (uint32_t i = 0; i < s.surface_count; i++) {
        const lrk_surface &sf = s.surfaces[i];
        if (sf.type >= LRK_SURFACE_TYPE_COUNT) return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: unknown surface type");
        if (sf.type == LRK_SURFACE_MIX && (sf.flags & LRK_SURFACE_HAS_TEXTURES) && sf.tex[0] != 0u)
            return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: the ratio of a Mix is a constant");
        if ((sf.flags & LRK_SURFACE_RAW_PARAMS) && (sf.type < LRK_SURFACE_MIRROR || sf.type > LRK_SURFACE_METAL))
            return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: LRK_SURFACE_RAW_PARAMS is for Mirror / Glass / Plastic / Metal records");
        if (sf.type == LRK_SURFACE_LAYERED) {
            if (r.volume) return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: Layered surfaces are not supported by the volume path integrator");
            if ((sf.lobes >> 16u) == 0u) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: a Layered surface needs samples >= 1");
        }
        if (sf.type == LRK_SURFACE_MIX || sf.type == LRK_SURFACE_LAYERED) {
            for (uint32_t child : {sf.mix_a, sf.mix_b}) {
                if (child >= s.surface_count || s.surfaces[child].type >= LRK_SURFACE_MIX || s.surfaces[child].type == LRK_SURFACE_DISNEY ||
                    (s.surfaces[child].flags & (LRK_SURFACE_HAS_TEXTURES | LRK_SURFACE_HAS_NORMAL_MAP | LRK_SURFACE_MAYBE_NON_OPAQUE)))
                    return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: a Mix / Layered surface combines two constant Matte / Mirror / Glass / Plastic / Metal records");
            }
        }
        for (uint32_t k = 0; k < 16u; k++)
            if (sf.tex[k] > s.texture_count) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: texture id out of range");
        if (sf.opacity_tex > s.texture_count || sf.normal_tex > s.texture_count) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: texture id out of range");
        if ((sf.flags & LRK_SURFACE_MAYBE_NON_OPAQUE) && r.volume)
            return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: non-opaque surfaces are not supported by the volume path integrator");
    }
    if (s.sampler.type > LRK_SAMPLER_ZSOBOL) return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: unknown sampler type");
    if (s.sampler.type != LRK_SAMPLER_INDEPENDENT) {
        const auto &q = s.sampler;
        if (r.volume) return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: the volume path integrator supports the Independent sampler only");
        const bool ok = q.spp != 0u && q.sobol_matrices != nullptr &&
                        (q.type != LRK_SAMPLER_PMJ02BN || (q.pmj_samples && q.blue_noise && q.pmj_pixel_samples && q.tile != 0u && q.spp <= 65536u &&
                                                           q.pmj_pixel_sample_count == static_cast<uint64_t>(q.tile) * q.tile * q.spp)) &&
                        (q.type != LRK_SAMPLER_SOBOL || (q.vdc && q.vdc_inv && q.scale != 0u && q.scale <= 0xffffu)) &&
                        (q.type != LRK_SAMPLER_ZSOBOL || (q.zsobol_hash != nullptr && q.num_base4_digits <= 32u));
        if (!ok) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: incomplete sampler record");
    }
    for (uint32_t i = 0; i < s.surface_count; i++)
        if (s.surfaces[i].flags & (LRK_SURFACE_HAS_TEXTURES | LRK_SURFACE_HAS_NORMAL_MAP)) r.textured = true;
    for (uint32_t i = 0; i < s.light_count; i++)
        if (s.lights[i].emission_tex != 0u) r.textured = true;// image emission: looked up by the TEXTURED kernel variants only
    for (uint32_t i = 0; i < s.texture_count; i++) {
        const auto &t = s.textures[i];
        if (t.width == 0u || t.height == 0u || t.texel_offset + static_cast<uint64_t>(t.width) * t.height > s.texel_count || t.address > LRK_TEX_ADDRESS_ZERO ||
            t.filter > LRK_TEX_FILTER_LINEAR || t.encoding > LRK_TEX_ENCODING_GAMMA)
            return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: invalid image texture record");
    }
    for (uint32_t i = 0; i < s.light_count; i++)
        if (s.lights[i].emission_tex > s.texture_count) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: a light's emission texture id is out of range");
    r.inst_kind.resize(s.instance_count);
    r.inst_mesh.resize(s.instance_count);
    r.mesh_emissive.assign(s.mesh_count, 0u);
    for (uint32_t i = 0; i < s.instance_count; i++) {
        const auto &inst = s.instances[i];
        r.inst_mesh[i] = inst.mesh;
        if (inst.visible) r.visible.push_back(i);
        // closure kind of the instance: the bucket key of the material sort
        const uint32_t flags = inst.handle[0] & 1023u, surface_tag = (inst.handle[1] >> 12u) & 4095u;
        uint32_t kind = kHitEmitter;
        if (flags & LRK_SHAPE_HAS_SURFACE) {
            if (surface_tag >= s.surface_count) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: surface tag out of range");
            kind = hit_kind_of(s.surfaces[surface_tag]);
        }
        r.inst_kind[i] = kind;
        r.used_kinds |= 1u << kind;
        if ((flags & LRK_SHAPE_MAYBE_NON_OPAQUE) && (flags & LRK_SHAPE_HAS_SURFACE)) r.any_non_opaque = true;
        if (inst.mesh >= s.mesh_count) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: mesh index out of range");
        if (inst.handle[0] & LRK_SHAPE_HAS_LIGHT) r.mesh_emissive[inst.mesh] = 1u;
    }
    r.mesh_root.resize(s.mesh_count);
    if (device_bvh) {
        uint64_t nodes = 0u;
        for (uint32_t m = 0; m < s.mesh_count; m++) {
            r.mesh_root[m] = static_cast<uint32_t>(nodes);
            const uint64_t n = s.meshes[m].triangle_count;
            if (n == 0u) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: mesh without triangles");
            nodes += std::max<uint64_t>(n - 1u, 1u);
            r.largest_mesh = std::max(r.largest_mesh, n);
        }
        r.tlas_root = static_cast<uint32_t>(nodes);
        r.node_count = nodes + std::max<uint64_t>(r.visible.size(), 2u) - 1u;
        if (!fits_bvh_encoding(r.node_count, s.triangle_count)) return refuse(LRK_ERR_UNSUPPORTED, "lrk_upload_scene: scene too large for the BVH encoding");
    } else {
        for (uint32_t m = 0; m < s.mesh_count; m++) r.mesh_root[m] = s.meshes[m].bvh_root;
        r.tlas_root = s.tlas_root;
        r.node_count = s.bvh_node_count;
    }
    // the shade kernels index the lights with an emitter's light tag and the instances with a light handle's instance
    for (uint32_t i = 0; i < s.instance_count; i++)
        if ((s.instances[i].handle[0] & LRK_SHAPE_HAS_LIGHT) && (s.instances[i].handle[1] & 4095u) >= s.light_count)
            return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: light tag out of range");
    for (uint32_t k = 0; k < s.light_count; k++)
        if (s.light_handles[k].instance_id >= s.instance_count) return refuse(LRK_ERR_INVALID_ARGUMENT, "lrk_upload_scene: light handle instance id out of range");
    if (light.tree) scene_check_detail::capture_light_source(s, r.light_source);
    return r;
}

}// namespace lrk
