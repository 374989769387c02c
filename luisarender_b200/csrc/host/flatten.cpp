#include "flatten.h"

#include "envmap.h"

#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <map>
#include <unordered_map>

#include "../device/affine_inverse.h"
#include "bvh.h"

namespace lrh {

lrk_scene_desc FlatScene::desc(uint32_t camera_index) const {
    if (camera_index >= cameras.size()) throw Error("Camera index out of range.");
    lrk_scene_desc d{};
    d.abi_version = LRK_ABI_VERSION;
    d.vertices = vertices.data();
    d.vertex_count = vertices.size();
    d.triangles = triangles.data();
    d.alias = alias.data();
    d.pdf = pdf.data();
    d.triangle_count = triangles.size();
    d.meshes = meshes.data();
    d.mesh_count = static_cast<uint32_t>(meshes.size());
    d.instances = instances.data();
    d.instance_count = static_cast<uint32_t>(instances.size());
    d.bvh_nodes = bvh_nodes.data();
    d.bvh_node_count = bvh_nodes.size();
    d.tlas_root = tlas_root;
    d.tri_verts = tri_verts.data();
    d.tri_slot_count = tri_verts.size() / 12u;
    d.surfaces = surfaces.data();
    d.surface_count = static_cast<uint32_t>(surfaces.size());
    d.textures = textures.empty() ? nullptr : textures.data();
    d.texture_count = static_cast<uint32_t>(textures.size());
    d.texels = texels.empty() ? nullptr : texels.data();
    d.texel_count = texels.size() / 4u;
    d.lights = lights.data();
    d.light_count = static_cast<uint32_t>(lights.size());
    d.light_handles = light_handles.data();
    d.camera = cameras[camera_index].camera;
    d.film = cameras[camera_index].film;
    d.integrator = integrator;
    d.environment_medium = environment_medium;
    d.media = media.empty() ? nullptr : media.data();
    d.medium_count = static_cast<uint32_t>(media.size());
    d.environment_medium_tag = environment_medium_tag;
    d.environment = environment;
    d.environment.alias = env_alias.empty() ? nullptr : env_alias.data();
    d.environment.pdf = env_pdf.empty() ? nullptr : env_pdf.data();
    const auto &cam = cameras[camera_index];
    d.sampler = cam.sampler;
    if (d.sampler.type != LRK_SAMPLER_INDEPENDENT) {
        const auto &t = sampler_tables();
        d.sampler.sobol_matrices = t.sobol_matrices.data();
        d.sampler.pmj_samples = t.pmj_samples.data();
        d.sampler.blue_noise = t.blue_noise.data();
        d.sampler.vdc = cam.vdc.empty() ? nullptr : cam.vdc.data();
        d.sampler.vdc_inv = cam.vdc_inv.empty() ? nullptr : cam.vdc_inv.data();
        d.sampler.pmj_pixel_samples = cam.pmj_pixel_samples.empty() ? nullptr : cam.pmj_pixel_samples.data();
        d.sampler.pmj_pixel_sample_count = cam.pmj_pixel_samples.size() / 2u;
        d.sampler.zsobol_hash = cam.zsobol_hash.empty() ? nullptr : cam.zsobol_hash.data();
    }
    return d;
}

// ---- quasi-Monte-Carlo sampler tables (row f2) --------------------------------------------------------------------------------
// luisarender_b200/data/sampler_tables.bin (tools/extract_sampler_tables.py): Sobol' generator matrices, van-der-Corput matrices,
// pmj02bn sets, blue-noise textures - the data of pbrt-v4's samplers that the reference's samplers are built on.  Located next
// to this library (<lib dir>/../data/) or through LRH_DATA_DIR; loaded once, on first use.
std::filesystem::path data_directory() {
    if (auto env = std::getenv("LRH_DATA_DIR")) return env;
    Dl_info info{};
    if (dladdr(reinterpret_cast<const void *>(&data_directory), &info) == 0 || info.dli_fname == nullptr)
        throw Error("Cannot locate the host library to find its data directory (set LRH_DATA_DIR).");
    return std::filesystem::path{info.dli_fname}.parent_path().parent_path() / "data";
}

const MetalIor &metal_ior_table(const std::string &name) {
    static const std::map<std::string, MetalIor> tables = [] {
        auto path = data_directory() / "metal_ior.bin";
        std::ifstream f{path, std::ios::binary};
        if (!f) throw Error("Cannot open the metal IOR tables '" + path.string() + "' (tools/extract_metal_ior.py writes them).");
        char magic[4];
        uint32_t header[3]{};
        f.read(magic, 4);
        f.read(reinterpret_cast<char *>(header), 12);
        if (!f || std::memcmp(magic, "LRMI", 4) != 0 || header[0] != 1u || header[2] != 95u) throw Error("'" + path.string() + "' is not a metal IOR table file.");
        std::map<std::string, MetalIor> out;
        for (uint32_t m = 0; m < header[1]; m++) {
            char nm[9]{};
            MetalIor ior;
            ior.n.resize(header[2]);
            ior.k.resize(header[2]);
            f.read(nm, 8);
            f.read(reinterpret_cast<char *>(ior.n.data()), header[2] * 4u);
            f.read(reinterpret_cast<char *>(ior.k.data()), header[2] * 4u);
            if (!f) throw Error("'" + path.string() + "' is truncated.");
            out.emplace(nm, std::move(ior));
        }
        return out;
    }();
    auto it = tables.find(name);
    if (it == tables.end()) throw Error("No IOR table for metal '" + name + "'.");
    return it->second;
}

const SamplerTables &sampler_tables() {
    static const SamplerTables tables = [] {
        auto dir = data_directory();
        auto path = dir / "sampler_tables.bin";
        std::ifstream f{path, std::ios::binary};
        if (!f) throw Error("Cannot open the sampler tables '" + path.string() + "' (tools/extract_sampler_tables.py writes them).");
        char magic[4];
        uint32_t version = 0u;
        f.read(magic, 4);
        f.read(reinterpret_cast<char *>(&version), 4);
        if (!f || std::memcmp(magic, "LRST", 4) != 0 || version != 1u) throw Error("'" + path.string() + "' is not a sampler table file.");
        SamplerTables t;
        for (int section = 0; section < 5; section++) {
            uint32_t tag = 0u, elem = 0u;
            uint64_t count = 0u;
            f.read(reinterpret_cast<char *>(&tag), 4);
            f.read(reinterpret_cast<char *>(&elem), 4);
            f.read(reinterpret_cast<char *>(&count), 8);
            auto read_into = [&](auto &vec, uint32_t want_elem, uint64_t want_count) {
                if (elem != want_elem || count != want_count) throw Error("Unexpected section in '" + path.string() + "'.");
                vec.resize(count);
                f.read(reinterpret_cast<char *>(vec.data()), static_cast<std::streamsize>(count * elem));
            };
            switch (tag) {
                case 1u: read_into(t.sobol_matrices, 4u, 1024u * 52u); break;
                case 2u: read_into(t.vdc, 8u, 25u * 52u); break;
                case 3u: read_into(t.vdc_inv, 8u, 26u * 52u); break;
                case 4u: read_into(t.pmj_samples, 4u, 5u * 65536u * 2u); break;
                case 5u: read_into(t.blue_noise, 2u, 48u * 128u * 128u); break;
                default: throw Error("Unknown section in '" + path.string() + "'.");
            }
            if (!f) throw Error("'" + path.string() + "' is truncated.");
        }
        return t;
    }();
    return tables;
}

namespace {

// XXH3_64bits_withSeed for an 8-byte input: what luisa::hash_value(uint64_t) computes (src/compute/src/core/stl/hash.cpp:10-12,
// seed = hash64_default_seed = 2^61 - 1, hash_fwd.h:10) - ZSobol's per-dimension hashes (zsobol.cpp:71-79).  Published
// algorithm (xxHash, XXH3_len_4to8_64b + XXH3_rrmxmx); the secret words are bytes 8..23 of its default secret.
uint64_t xxh3_64_of_u64(uint64_t value, uint64_t seed) {
    auto rotl64 = [](uint64_t x, int r) { return (x << r) | (x >> (64 - r)); };
    auto swap32 = [](uint32_t x) { return (x << 24) | ((x << 8) & 0x00ff0000u) | ((x >> 8) & 0x0000ff00u) | (x >> 24); };
    constexpr uint64_t secret8 = 0x1cad21f72c81017cull, secret16 = 0xdb979083e96dd4deull;// little-endian reads of the secret
    seed ^= static_cast<uint64_t>(swap32(static_cast<uint32_t>(seed))) << 32;
    const uint32_t input1 = static_cast<uint32_t>(value), input2 = static_cast<uint32_t>(value >> 32);
    const uint64_t bitflip = (secret8 ^ secret16) - seed;
    const uint64_t input64 = input2 + (static_cast<uint64_t>(input1) << 32);
    uint64_t h = input64 ^ bitflip;
    h ^= rotl64(h, 49) ^ rotl64(h, 24);
    h *= 0x9FB21C651E98DF25ull;
    h ^= (h >> 35) + 8u;
    h *= 0x9FB21C651E98DF25ull;
    return h ^ (h >> 28);
}

uint32_t next_pow2_u32(uint32_t x) {
    uint32_t p = 1u;
    while (p < x) p <<= 1u;
    return p;
}

// Sampler::Instance::reset(resolution, state_count, spp) of the node's sampler, for one camera
void flatten_sampler(const Sampler *node, FlatCamera &cam) {
    auto &s = cam.sampler;
    s = lrk_sampler{};
    s.type = node ? node->type : LRK_SAMPLER_INDEPENDENT;
    s.spp = cam.camera.spp;
    const uint32_t w = cam.camera.resolution[0], h = cam.camera.resolution[1], spp = cam.camera.spp;
    if (s.type == LRK_SAMPLER_INDEPENDENT) return;
    if (spp == 0u) throw Error("The camera's spp must be positive for a table-driven sampler.");
    const auto &t = sampler_tables();
    auto log2u = [](uint32_t x) { uint32_t l = 0u; while ((2u << l) <= x) l++; return l; };// bit_width(x) - 1
    switch (s.type) {
        case LRK_SAMPLER_PMJ02BN: {// pmj02bn.cpp:103-162
            auto log4 = [&](uint32_t x) { return log2u(x) / 2u; };
            auto is_pow4 = [&](uint32_t x) { return x == (1u << (2u * log4(x))); };
            auto next_pow4 = [&](uint32_t x) { return is_pow4(x) ? x : 1u << (2u * (log4(x) + 1u)); };
            if (spp > 65536u) throw Error("PMJ02BNSampler only supports up to 65536 samples per pixel (" + std::to_string(spp) + " requested).");
            uint32_t mask = spp - 1u;
            mask |= mask >> 1u; mask |= mask >> 2u; mask |= mask >> 4u; mask |= mask >> 8u; mask |= mask >> 16u;
            s.w = mask;
            s.tile = 1u << (log4(65536u) - log4(next_pow4(spp)));
            const size_t count = static_cast<size_t>(s.tile) * s.tile * spp;
            cam.pmj_pixel_samples.assign(count * 2u, 0.f);
            std::vector<uint32_t> stored(static_cast<size_t>(s.tile) * s.tile, 0u);
            for (uint32_t i = 0u; i < 65536u; i++) {
                // pmj02bn_sample(0, i): the doubles are narrowed to float BEFORE the scaling (make_float2(static_cast<float>(...)))
                const float sx = static_cast<float>(t.pmj_samples[static_cast<size_t>(i) * 2u] * 0x1p-32);
                const float sy = static_cast<float>(t.pmj_samples[static_cast<size_t>(i) * 2u + 1u] * 0x1p-32);
                const float px = sx * static_cast<float>(s.tile), py = sy * static_cast<float>(s.tile);
                const uint32_t pixel_offset = static_cast<uint32_t>(py) * s.tile + static_cast<uint32_t>(px);
                if (stored[pixel_offset] == spp) {
                    if (is_pow4(spp)) throw Error("Invalid pmj02bn pixel sorting state.");
                    continue;
                }
                const size_t at = static_cast<size_t>(pixel_offset) * spp + stored[pixel_offset];
                cam.pmj_pixel_samples[at * 2u] = px - std::floor(px);
                cam.pmj_pixel_samples[at * 2u + 1u] = py - std::floor(py);
                stored[pixel_offset]++;
            }
            for (auto c : stored)
                if (c != spp) throw Error("Invalid pmj02bn pixel sorting state.");
            break;
        }
        case LRK_SAMPLER_SOBOL: {// sobol.cpp:112-131
            s.scale = next_pow2_u32(std::max(w, h));
            if (s.scale > 0xffffu) throw Error("Sobol sampler scale is too large.");
            const uint32_t m = log2u(s.scale);
            cam.vdc.assign(52u, 0u);
            cam.vdc_inv.assign(52u, 0u);
            if (m >= 1u) {
                for (uint32_t i = 0u; i < 52u; i++) {
                    cam.vdc[i] = t.vdc[static_cast<size_t>(m - 1u) * 52u + i];
                    cam.vdc_inv[i] = t.vdc_inv[static_cast<size_t>(m - 1u) * 52u + i];
                }
            }
            break;
        }
        case LRK_SAMPLER_PADDED_SOBOL: break;// spp only (padded_sobol.cpp:99-111)
        case LRK_SAMPLER_ZSOBOL: {// zsobol.cpp:69-103
            auto log2_ceil = [&](uint32_t x) { return log2u(next_pow2_u32(x)); };// bit_width(next_pow2(x)) - 1
            s.log2_spp = log2_ceil(spp);
            const uint32_t log4_spp = (s.log2_spp + 1u) / 2u;
            s.num_base4_digits = log2_ceil(std::max(w, h)) + log4_spp;
            cam.zsobol_hash.resize(2048u);
            for (uint32_t i = 0u; i < 1024u; i++) {
                const uint64_t hsh = xxh3_64_of_u64((static_cast<uint64_t>(node->seed) << 32u) | i, (1ull << 61u) - 1ull);
                cam.zsobol_hash[i * 2u] = static_cast<uint32_t>(hsh & 0xffffffffull);
                cam.zsobol_hash[i * 2u + 1u] = static_cast<uint32_t>(hsh >> 32u);
            }
            break;
        }
        default: throw Error("Unknown sampler type.");
    }
}

uint64_t fnv1a(const void *data, size_t bytes, uint64_t h = 1469598103934665603ull) {
    auto p = static_cast<const unsigned char *>(data);
    for (size_t i = 0; i < bytes; i++) {
        h ^= p[i];
        h *= 1099511628211ull;
    }
    return h;
}

// Shape::Handle::encode, src/base/shape.cpp:46-70
void encode_handle(uint32_t out[4], uint32_t buffer_base, uint32_t flags, uint32_t surface_tag, uint32_t light_tag,
                   uint32_t medium_tag, uint32_t tri_count, float shadow_terminator, float intersection_offset) {
    if (buffer_base > (1u << 22u) - 1u) throw Error("Invalid geometry buffer base.");
    if (surface_tag > 4095u) throw Error("Invalid surface tag (more than 4096 surfaces).");
    if (light_tag > 4095u) throw Error("Invalid light tag (more than 4096 lights).");
    if (medium_tag > 255u) throw Error("Invalid medium tag (more than 256 media).");
    auto fixed = [](float x) {
        x = std::min(std::max(x, 0.f), 1.f);
        constexpr float scale = 1.f / 65536.f;
        return static_cast<uint32_t>(std::min(std::max(std::round(x / scale), 0.f), 65535.f));
    };
    out[0] = (buffer_base << 10u) | flags;
    out[1] = (surface_tag << 12u) | light_tag | (medium_tag << 24u);
    out[2] = tri_count;
    out[3] = (fixed(shadow_terminator) << 16u) | fixed(intersection_offset);
}

struct Flattener {
    const Scene &scene;
    FlatScene &out;
    std::unordered_map<const Shape *, uint32_t> shape_mesh;
    std::multimap<uint64_t, uint32_t> mesh_by_hash;
    std::unordered_map<const Surface *, uint32_t> surface_tags;
    std::unordered_map<const Light *, uint32_t> light_tags;
    std::unordered_map<const Medium *, uint32_t> medium_tags;
    std::vector<const Surface *> surface_nodes;
    std::vector<const Light *> light_nodes;
    std::vector<float4x4> xform_stack;
    std::vector<Aabb> mesh_bounds;

    uint32_t register_mesh(const Shape *shape) {
        if (auto it = shape_mesh.find(shape); it != shape_mesh.end()) return it->second;
        auto &v = shape->vertices();
        auto &t = shape->triangles();
        if (v.empty() || t.empty()) throw Error("Empty mesh.");
        auto h = fnv1a(v.data(), v.size() * sizeof(lrk_vertex));
        h = fnv1a(t.data(), t.size() * sizeof(lrk_triangle), h);
        auto range = mesh_by_hash.equal_range(h);
        for (auto it = range.first; it != range.second; ++it) {
            auto &m = out.meshes[it->second];
            if (m.vertex_count == v.size() && m.triangle_count == t.size() &&
                std::memcmp(&out.vertices[m.vertex_offset], v.data(), v.size() * sizeof(lrk_vertex)) == 0 &&
                std::memcmp(&out.triangles[m.triangle_offset], t.data(), t.size() * sizeof(lrk_triangle)) == 0) {
                shape_mesh.emplace(shape, it->second);
                return it->second;
            }
        }
        lrk_mesh m{};
        m.vertex_offset = static_cast<uint32_t>(out.vertices.size());
        m.vertex_count = static_cast<uint32_t>(v.size());
        m.triangle_offset = static_cast<uint32_t>(out.triangles.size());
        m.triangle_count = static_cast<uint32_t>(t.size());
        out.vertices.insert(out.vertices.end(), v.begin(), v.end());
        out.triangles.insert(out.triangles.end(), t.begin(), t.end());
        // per-mesh area alias table (src/base/geometry.cpp:71-80)
        std::vector<float> areas(t.size());
        std::vector<Aabb> tri_bounds(t.size());
        Aabb mb;
        auto pos = [&](uint32_t i) { return float3{v[i].p[0], v[i].p[1], v[i].p[2]}; };
        for (size_t i = 0; i < t.size(); i++) {
            if (t[i].i0 >= v.size() || t[i].i1 >= v.size() || t[i].i2 >= v.size()) throw Error("Triangle index out of range.");
            auto p0 = pos(t[i].i0), p1 = pos(t[i].i1), p2 = pos(t[i].i2);
            areas[i] = lrk::triangle_area_weight(v[t[i].i0].p, v[t[i].i1].p, v[t[i].i2].p);
            tri_bounds[i].grow(p0); tri_bounds[i].grow(p1); tri_bounds[i].grow(p2);
            mb.grow(tri_bounds[i]);
        }
        std::vector<lrk_alias_entry> table;
        std::vector<float> pdf;
        create_alias_table(areas.data(), areas.size(), table, pdf);
        out.alias.insert(out.alias.end(), table.begin(), table.end());
        out.pdf.insert(out.pdf.end(), pdf.begin(), pdf.end());
        // BLAS
        auto bvh = build_bvh(tri_bounds.data(), static_cast<uint32_t>(t.size()), LRK_BVH_MAX_LEAF_TRIS, false);
        auto node_base = static_cast<uint32_t>(out.bvh_nodes.size());
        auto slot_base = static_cast<uint32_t>(out.tri_verts.size() / 12u);
        if (static_cast<uint64_t>(slot_base) + t.size() >= (1ull << 28)) throw Error("Too many triangles for the BVH leaf encoding.");
        m.bvh_root = node_base;
        m.tri_slot_offset = slot_base;
        auto rebase = [&](uint32_t ref) {
            if (ref == LRK_BVH_EMPTY) return ref;
            if (ref & LRK_BVH_LEAF) return (ref & 0xf0000000u) | ((ref & 0x0fffffffu) + slot_base);
            return ref + node_base;
        };
        for (auto n : bvh.nodes) {
            n.ref0 = rebase(n.ref0);
            n.ref1 = rebase(n.ref1);
            n.parent = n.parent == LRK_BVH_EMPTY ? LRK_BVH_EMPTY : n.parent + node_base;
            out.bvh_nodes.push_back(n);
        }
        out.tri_verts.reserve(out.tri_verts.size() + t.size() * 12u);
        for (auto prim : bvh.prim_order) {
            auto p0 = pos(t[prim].i0), p1 = pos(t[prim].i1), p2 = pos(t[prim].i2);
            float id_bits;
            std::memcpy(&id_bits, &prim, 4);
            float rec[12]{p0.x, p0.y, p0.z, id_bits, p1.x, p1.y, p1.z, 0.f, p2.x, p2.y, p2.z, 0.f};
            out.tri_verts.insert(out.tri_verts.end(), rec, rec + 12);
        }
        auto index = static_cast<uint32_t>(out.meshes.size());
        out.meshes.push_back(m);
        mesh_bounds.push_back(mb);
        mesh_by_hash.emplace(h, index);
        shape_mesh.emplace(shape, index);
        return index;
    }

    uint32_t register_surface(const Surface *s) {
        if (auto it = surface_tags.find(s); it != surface_tags.end()) return it->second;
        auto tag = static_cast<uint32_t>(surface_nodes.size());
        surface_nodes.push_back(s);
        surface_tags.emplace(s, tag);
        return tag;
    }
    // Pipeline::register_medium (src/base/pipeline.cpp:36-42): one record per medium node, in first-use order
    uint32_t register_medium(const Medium *m) {
        if (auto it = medium_tags.find(m); it != medium_tags.end()) return it->second;
        auto tag = static_cast<uint32_t>(out.media.size());
        lrk_medium rec{};
        rec.present = m->is_vacuum() ? LRK_MEDIUM_VACUUM : LRK_MEDIUM_HOMOGENEOUS;
        rec.priority = m->is_vacuum() ? LRK_MEDIUM_VACUUM_PRIORITY : m->priority;
        rec.eta = m->eta;
        rec.g = m->phase ? m->phase->g : 0.f;
        for (int i = 0; i < 3; i++) {
            rec.sigma_a[i] = m->sigma_a[i];
            rec.sigma_s[i] = m->sigma_s[i];
            rec.le[i] = m->le[i];
        }
        out.media.push_back(rec);
        medium_tags.emplace(m, tag);
        return tag;
    }
    uint32_t register_light(const Light *l) {
        if (auto it = light_tags.find(l); it != light_tags.end()) return it->second;
        auto tag = static_cast<uint32_t>(light_nodes.size());
        light_nodes.push_back(l);
        light_tags.emplace(l, tag);
        return tag;
    }

    // TransformTree::Node::matrix (src/base/transform.cpp:18-24): innermost first, parents applied on the left
    float4x4 chain_matrix(const Transform *leaf) const {
        std::vector<float4x4> chain = xform_stack;
        if (leaf != nullptr && !leaf->is_identity()) chain.push_back(leaf->matrix());
        if (chain.empty()) return float4x4::identity();
        auto m = chain.back();
        for (auto i = chain.size() - 1u; i-- > 0u;) m = chain[i] * m;
        return m;
    }

    // Geometry::_process_shape (src/base/geometry.cpp:29-163)
    void process(const Shape *shape, const Surface *ov_surface, const Light *ov_light, const Medium *ov_medium, bool ov_visible) {
        auto surface = ov_surface == nullptr ? shape->surface : ov_surface;
        auto light = ov_light == nullptr ? shape->light : ov_light;
        auto medium = ov_medium == nullptr ? shape->medium : ov_medium;
        auto visible = ov_visible && shape->visible;
        if (shape->is_mesh()) {
            auto mesh_index = register_mesh(shape);
            auto &mesh = out.meshes[mesh_index];
            auto instance_id = static_cast<uint32_t>(out.instances.size());
            auto o2w = chain_matrix(shape->transform);
            auto &v = shape->vertices();
            for (auto &vert : v) {
                auto p = transform_point(o2w, {vert.p[0], vert.p[1], vert.p[2]});
                for (int a = 0; a < 3; a++) {
                    out.world_max[a] = std::max(out.world_max[a], p[a]);
                    out.world_min[a] = std::min(out.world_min[a], p[a]);
                }
            }
            uint32_t surface_tag = 0u, light_tag = 0u, medium_tag = 0u;
            auto properties = shape->vertex_properties();
            if (surface != nullptr && !surface->is_null()) {
                surface_tag = register_surface(surface);
                properties |= LRK_SHAPE_HAS_SURFACE;
                if (surface->maybe_non_opaque()) properties |= LRK_SHAPE_MAYBE_NON_OPAQUE;// geometry.cpp:123-126
            }
            if (light != nullptr && !light->is_null()) {
                light_tag = register_light(light);
                properties |= LRK_SHAPE_HAS_LIGHT;
            }
            if (medium != nullptr && !medium->is_null()) {// geometry.cpp:139-142
                medium_tag = register_medium(medium);
                properties |= LRK_SHAPE_HAS_MEDIUM;
            }
            auto fixed16 = [](float x) {
                return static_cast<float>(static_cast<uint16_t>(std::min(std::max(std::round(x * 65535.f), 0.f), 65535.f))) / 65535.f;
            };
            auto has_normal = (shape->vertex_properties() & LRK_SHAPE_HAS_VERTEX_NORMAL) != 0u;
            lrk_instance inst{};
            encode_handle(inst.handle, mesh_index * 4u, properties, surface_tag, light_tag, medium_tag, mesh.triangle_count,
                          fixed16(has_normal ? shape->shadow_terminator : 0.f), fixed16(shape->intersection_offset));
            to_rows_3x4(o2w, inst.object_to_world);
            if (!lrk::inverse_affine_rows(inst.object_to_world, inst.world_to_object))
                throw Error("Singular instance transform. [" + shape->desc()->location() + "]");
            inst.mesh = mesh_index;
            inst.visible = visible ? 1u : 0u;
            out.instances.push_back(inst);
            if (properties & LRK_SHAPE_HAS_LIGHT) out.light_handles.push_back({instance_id, light_tag});
            out.total_instanced_triangles += mesh.triangle_count;
        } else {
            bool pushed = shape->transform != nullptr && !shape->transform->is_identity();
            if (pushed) xform_stack.push_back(shape->transform->matrix());
            for (auto child : shape->children()) process(child, surface, light, medium, visible);
            if (pushed) xform_stack.pop_back();
        }
    }

    void build_tlas() {
        std::vector<Aabb> bounds;
        std::vector<uint32_t> ids;
        for (uint32_t i = 0; i < out.instances.size(); i++) {
            auto &inst = out.instances[i];
            if (!inst.visible) continue;// invisible instances are skipped by all rays (src/base/geometry.cpp:130-131)
            auto &mesh = out.meshes[inst.mesh];
            Aabb b;
            const float *m = inst.object_to_world;
            for (uint32_t k = 0; k < mesh.vertex_count; k++) {
                auto &v = out.vertices[mesh.vertex_offset + k];
                float3 p{m[0] * v.p[0] + m[1] * v.p[1] + m[2] * v.p[2] + m[3],
                         m[4] * v.p[0] + m[5] * v.p[1] + m[6] * v.p[2] + m[7],
                         m[8] * v.p[0] + m[9] * v.p[1] + m[10] * v.p[2] + m[11]};
                b.grow(p);
            }
            // pad by a few ulps: object-space intersection rounds differently from this world-space box
            for (int a = 0; a < 3; a++) {
                auto e = 4e-7f * std::max(std::abs(b.lo[a]), std::abs(b.hi[a])) + 1e-30f;
                b.lo[a] -= e;
                b.hi[a] += e;
            }
            bounds.push_back(b);
            ids.push_back(i);
        }
        auto bvh = build_bvh(bounds.data(), static_cast<uint32_t>(bounds.size()), 1u, true);
        auto node_base = static_cast<uint32_t>(out.bvh_nodes.size());
        out.tlas_root = node_base;
        auto rebase = [&](uint32_t ref) {
            if (ref == LRK_BVH_EMPTY) return ref;
            if (ref & LRK_BVH_LEAF) return LRK_BVH_LEAF | ids[ref & 0x7fffffffu];
            return ref + node_base;
        };
        for (auto n : bvh.nodes) {
            n.ref0 = rebase(n.ref0);
            n.ref1 = rebase(n.ref1);
            n.parent = n.parent == LRK_BVH_EMPTY ? LRK_BVH_EMPTY : n.parent + node_base;
            out.bvh_nodes.push_back(n);
        }
    }
};

FlatCamera flatten_camera(const Camera *cam) {
    FlatCamera fc{};
    auto &c = fc.camera;
    to_rows_3x4(cam->camera_to_world, c.camera_to_world);
    c.resolution[0] = cam->film->resolution[0];
    c.resolution[1] = cam->film->resolution[1];
    c.tan_half_fov = cam->tan_half_fov();
    c.filter_radius = cam->filter->radius;
    c.filter_shift[0] = cam->filter->shift[0];
    c.filter_shift[1] = cam->filter->shift[1];
    c.spp = cam->spp;
    // Filter::Instance::Instance, src/base/filter.cpp:24-48
    constexpr uint32_t n = LRK_FILTER_LUT_SIZE - 1u;
    constexpr float inv_n = 1.0f / static_cast<float>(n);
    float abs_f[n];
    auto filter = cam->filter;
    c.filter_lut[0] = filter->evaluate(-filter->radius);
    auto integral = 0.0f;
    for (uint32_t i = 0; i < n; i++) {
        auto x = static_cast<float>(i + 1u) * inv_n * 2.0f - 1.0f;
        c.filter_lut[i + 1u] = filter->evaluate(x * filter->radius);
        auto f_mid = 0.5f * (c.filter_lut[i] + c.filter_lut[i + 1u]);
        integral += f_mid;
        abs_f[i] = std::abs(f_mid);
    }
    auto inv_integral = 1.0f / integral;
    for (auto &f : c.filter_lut) f *= inv_integral;
    std::vector<lrk_alias_entry> table;
    std::vector<float> pdf;
    create_alias_table(abs_f, n, table, pdf);
    for (uint32_t i = 0; i < n; i++) {
        c.filter_pdf[i] = pdf[i];
        c.filter_alias_probs[i] = table[i].prob;
        c.filter_alias_indices[i] = table[i].alias;
    }
    for (int i = 0; i < 3; i++) fc.film.scale[i] = cam->film->scale[i];
    fc.film.clamp = cam->film->clamp;
    fc.file = cam->file;
    return fc;
}

}// namespace

std::unique_ptr<FlatScene> flatten_scene(const Scene &scene) {
    auto out = std::make_unique<FlatScene>();
    for (int a = 0; a < 3; a++) {
        out->world_max[a] = -std::numeric_limits<float>::max();
        out->world_min[a] = std::numeric_limits<float>::max();
    }
    auto t0 = std::chrono::steady_clock::now();
    Flattener f{scene, *out};
    for (auto shape : scene.shapes()) f.process(shape, nullptr, nullptr, nullptr, true);
    if (out->instances.empty()) throw Error("The scene has no geometry.");
    f.build_tlas();
    out->bvh_build_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();

    // surfaces; Disney lobes are OR-ed over all disney nodes of one closure class - opaque "disney", transmissive "disney_trans",
    // thin "disney_thin" (one shared closure per class, src/surfaces/disney.cpp:869,925-930,994)
    uint32_t disney_lobes[3] = {0u, 0u, 0u};
    auto disney_class = [](const lrk_surface &s) { return (s.flags & LRK_SURFACE_DISNEY_THIN) ? 2 : (s.flags & LRK_SURFACE_DISNEY_TRANSMISSIVE) ? 1 : 0; };
    TextureTable texture_table;
    for (auto s : f.surface_nodes) {
        out->surfaces.push_back(s->flatten(texture_table));
        if (out->surfaces.back().type == LRK_SURFACE_DISNEY) disney_lobes[disney_class(out->surfaces.back())] |= out->surfaces.back().lobes;
    }
    // Mix nodes: their two surfaces become extra records behind the tagged ones (never referenced by an instance handle)
    for (size_t tag = 0, tagged = f.surface_nodes.size(); tag < tagged; tag++) {
        auto [a, b] = f.surface_nodes[tag]->mix_children();
        if (a == nullptr) continue;
        const bool layered = out->surfaces[tag].type == LRK_SURFACE_LAYERED;
        for (auto child : {a, b}) {
            auto rec = child->flatten(texture_table);
            if (rec.type == LRK_SURFACE_DISNEY || (rec.flags & LRK_SURFACE_HAS_TEXTURES))
                throw Error(std::string{layered ? "Layered" : "Mix"} + ": only constant Matte / Mirror / Glass / Plastic / Metal surfaces can be " +
                            (layered ? "layered." : "mixed."));
            (child == a ? out->surfaces[tag].mix_a : out->surfaces[tag].mix_b) = static_cast<uint32_t>(out->surfaces.size());
            out->surfaces.push_back(rec);
        }
        if (layered) {
            // the bottom closure is built with eta_i = top->eta().value_or(1) (layered.cpp:500-502); every closure here takes eta_i = 1,
            // so under a Glass top only interfaces that never look at eta_i are accepted
            const auto &top = out->surfaces[out->surfaces[tag].mix_a], &bottom = out->surfaces[out->surfaces[tag].mix_b];
            if (top.type == LRK_SURFACE_GLASS && top.p[6] != 1.f && bottom.type != LRK_SURFACE_MATTE && bottom.type != LRK_SURFACE_MIRROR)
                throw Error("Layered: under a Glass top (eta != 1) the bottom interface must be Matte or Mirror.");
            continue;
        }
        // MixSurfaceClosure::eta() (mix.cpp:133-141) for the Russian-roulette eta scale: Glass children have one
        auto eta_of = [&](uint32_t i) { return out->surfaces[i].type == LRK_SURFACE_GLASS ? out->surfaces[i].p[6] : 0.f; };
        float ea = eta_of(out->surfaces[tag].mix_a), eb = eta_of(out->surfaces[tag].mix_b), ratio = out->surfaces[tag].p[0];
        out->surfaces[tag].p[1] = ea == 0.f ? eb : eb == 0.f ? ea : ratio * (ea - eb) + eb;// lerp(eta_b, eta_a, ratio)
    }
    for (auto &s : out->surfaces)
        if (s.type == LRK_SURFACE_DISNEY) s.lobes = disney_lobes[disney_class(s)];
    // the environment light (SURVEY.md §8 rows a12 / f3): src/environments/spherical.cpp, src/lightsamplers/uniform.cpp:40-47
    if (auto env = scene.environment(); env != nullptr && !env->is_null() && !env->is_black()) {
        auto &e = out->environment;
        e.present = 1u;
        e.scale = env->scale;
        e.emission_tex = texture_table.slot(env->emission);
        if (e.emission_tex == 0u) {
            auto c = env->emission->value();
            auto n = env->emission->channels();
            float rgb[3] = {c.x, n == 1u ? c.x : c.y, n == 1u ? c.x : (n == 2u ? 1.f : c.z)};// extend_color_to_rgb
            for (int k = 0; k < 3; k++) e.emission[k] = std::max(rgb[k], 0.f);                  // encode/decode_illuminant
        }
        auto m = env->transform != nullptr ? env->transform->matrix() : float4x4::identity();// make_float3x3(transform), environment.cpp:18-20
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++) e.to_world[r * 3 + c] = m.c[c][r];// columns c[], row-major output
        auto w = scene.integrator()->light_sampler ? scene.integrator()->light_sampler->environment_weight : .5f;
        e.env_prob = f.light_nodes.empty() ? 1.f : std::min(std::max(w, 0.01f), 0.99f);
        if (e.emission_tex != 0u) {
            const auto &rec = texture_table.records[e.emission_tex - 1u];
            build_environment_map(rec, texture_table.texels.data() + rec.texel_offset * 4u, env->compensate_mis, out->env_alias, out->env_pdf);
            e.map_width = kEnvMapWidth;
            e.map_height = kEnvMapHeight;
        }
    }
    for (auto l : f.light_nodes) out->lights.push_back(l->flatten(texture_table));
    out->textures = std::move(texture_table.records);
    out->texels = std::move(texture_table.texels);

    for (auto cam : scene.cameras()) out->cameras.push_back(flatten_camera(cam));
    if (out->cameras.empty()) throw Error("The scene has no camera.");

    auto integ = scene.integrator();
    for (auto &cam : out->cameras) flatten_sampler(integ->sampler, cam);
    out->integrator.type = integ->kind;
    out->integrator.max_depth = integ->max_depth;
    out->integrator.rr_depth = integ->rr_depth;
    out->integrator.rr_threshold = integ->rr_threshold;
    out->integrator.samples_per_pass = integ->samples_per_pass;
    out->integrator.sampler_seed = integ->sampler->seed;

    // the environment medium is registered after the shapes' media (src/base/pipeline.cpp:72-79); a vacuum one never enters a
    // path's medium tracker (its priority is VACUUM_PRIORITY, medium_tracker.cpp:29-41) and counts as none
    if (auto m = scene.environment_medium(); m != nullptr && !m->is_null() && !m->is_vacuum()) {
        out->environment_medium_tag = f.register_medium(m);
        out->environment_medium = out->media[out->environment_medium_tag];
    }
    return out;
}

}// namespace lrh
