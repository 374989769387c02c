// Host scene graph: the node categories and implementations marked in scope by SURVEY.md §2.1,
// instantiated from a SceneDesc through a plugin registry keyed "<tag>-<impl>" exactly like the
// reference's dlopen name "luisa-render-<tag>-<impl>" (src/base/scene.cpp:64-75), with the same
// create/destroy C signature as LUISA_RENDER_MAKE_SCENE_NODE_PLUGIN (src/base/scene_node.h:58-67).
// Unknown node implementations are a hard error naming the plugin (reference: dlopen failure abort).
#pragma once
#include <utility>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../../include/lrk.h"
#include "../device/alias_table.h"
#include "sdl.h"
#include "vecmath.h"

namespace lrh {

class Scene;

class SceneNode {
public:
    SceneNode(const Scene *scene, const NodeDesc *desc, Tag tag) : _scene{scene}, _desc{desc}, _tag{tag} {}
    virtual ~SceneNode() = default;
    Tag tag() const { return _tag; }
    const NodeDesc *desc() const { return _desc; }
    const std::string &impl_type() const { return _desc->impl_type(); }
    const Scene *scene() const { return _scene; }

private:
    const Scene *_scene;
    const NodeDesc *_desc;
    Tag _tag;
};

// plugin ABI (same shape as the reference's `create` / `destroy` exports)
using NodeCreator = SceneNode *(Scene *, const NodeDesc *);
using NodeDeleter = void(SceneNode *);
struct Plugin {
    NodeCreator *create;
    NodeDeleter *destroy;
};
// key = "<tag>-<impl>", lower case, e.g. "shape-inlinemesh"
void register_plugin(const std::string &key, Plugin plugin);
const Plugin *find_plugin(const std::string &key);
std::vector<std::string> registered_plugins();

// ---- node categories -------------------------------------------------------------------------

struct Texture : SceneNode {
    using SceneNode::SceneNode;
    virtual bool is_black() const = 0;
    virtual bool is_constant() const = 0;
    virtual uint32_t channels() const = 0;
    virtual float4 value() const = 0;// constant value (scale applied); image textures: not meaningful
    // image textures (src/textures/image.cpp) append their record + texels to the flattened scene
    virtual bool is_image() const { return false; }
    virtual void emit(lrk_texture &, std::vector<float> &) const { throw Error("Texture::emit: not an image texture."); }
};

// The image textures a flattened scene references: one lrk_texture record + texels per distinct Texture node.
struct TextureTable {
    std::vector<lrk_texture> records;
    std::vector<float> texels;// RGBA
    std::unordered_map<const Texture *, uint32_t> slots;
    // value for lrk_surface::tex[k]: 0 for constants / null, index + 1 for image textures
    uint32_t slot(const Texture *t) {
        if (t == nullptr || !t->is_image()) return 0u;
        if (auto it = slots.find(t); it != slots.end()) return it->second;
        lrk_texture rec{};
        rec.texel_offset = texels.size() / 4u;
        t->emit(rec, texels);
        records.push_back(rec);
        auto id = static_cast<uint32_t>(records.size());
        slots.emplace(t, id);
        return id;
    }
};

struct Transform : SceneNode {
    using SceneNode::SceneNode;
    virtual float4x4 matrix() const = 0;
    virtual bool is_identity() const { return matrix().is_identity(); }
};

struct Spectrum : SceneNode {
    using SceneNode::SceneNode;
};

struct Filter : SceneNode {
    Filter(const Scene *s, const NodeDesc *d);
    float radius;
    float shift[2];
    virtual float evaluate(float x) const = 0;
};

struct Film : SceneNode {
    using SceneNode::SceneNode;
    uint32_t resolution[2]{};
    float scale[3]{1, 1, 1};
    float clamp{256.f};
};

struct Sampler : SceneNode {
    Sampler(const Scene *s, const NodeDesc *d);
    uint32_t seed;
    uint32_t type{LRK_SAMPLER_INDEPENDENT};// LRK_SAMPLER_*: src/samplers/{independent,pmj02bn,sobol,padded_sobol,zsobol}.cpp
};

struct LightSampler : SceneNode {
    using SceneNode::SceneNode;
    float environment_weight{.5f};
};

struct Integrator : SceneNode {
    Integrator(Scene *s, const NodeDesc *d);
    const Sampler *sampler{};
    const LightSampler *light_sampler{};
    uint32_t kind{LRK_INTEGRATOR_PATH};
    uint32_t max_depth{10}, rr_depth{0}, samples_per_pass{16};
    float rr_threshold{.95f};
};

struct PhaseFunction : SceneNode {
    using SceneNode::SceneNode;
    float g{0.f};
};

struct Medium : SceneNode {
    using SceneNode::SceneNode;
    virtual bool is_null() const { return false; }
    virtual bool is_vacuum() const { return false; }
    uint32_t priority{0};
    float eta{1.f};
    float sigma_a[3]{}, sigma_s[3]{}, le[3]{};
    const PhaseFunction *phase{};
};

struct Surface : SceneNode {
    // every surface node is NormalMapWrapper<OpacitySurfaceWrapper<Base>> (src/base/surface.h:160-275, e.g. matte.cpp:136)
    Surface(Scene *scene, const NodeDesc *desc, Tag tag);
    virtual bool is_null() const { return false; }
    virtual lrk_surface flatten(TextureTable &textures) const = 0;
    // Mix (src/surfaces/mix.cpp): the two mixed surface nodes, flattened to extra records behind the tagged ones
    virtual std::pair<const Surface *, const Surface *> mix_children() const { return {nullptr, nullptr}; }
    // OpacitySurfaceWrapper::Instance::maybe_non_opaque (surface.h:177-181)
    bool maybe_non_opaque() const;
    const Texture *opacity{};
    const Texture *normal_map{};
    float normal_map_strength{1.f};

protected:
    void flatten_wrappers(lrk_surface &out, TextureTable &textures) const;
};

struct Environment : SceneNode {
    // src/base/environment.cpp:11-13 ; the Spherical plugin: src/environments/spherical.cpp:16-33
    Environment(Scene *scene, const NodeDesc *desc);
    virtual bool is_null() const { return false; }
    virtual bool is_black() const = 0;
    const Transform *transform{};
    const Texture *emission{};
    float scale{1.f};
    bool compensate_mis{true};
};

struct Light : SceneNode {
    using SceneNode::SceneNode;
    virtual bool is_null() const { return false; }
    virtual lrk_light flatten(TextureTable &textures) const = 0;
};

struct Camera : SceneNode {
    Camera(Scene *s, const NodeDesc *d);
    const Film *film{};
    const Filter *filter{};
    const Transform *transform{};
    float4x4 camera_to_world{float4x4::identity()};
    uint32_t spp{1024};
    std::filesystem::path file;
    virtual float tan_half_fov() const = 0;
};

struct Shape : SceneNode {
    Shape(Scene *s, const NodeDesc *d);
    const Surface *surface{};
    const Light *light{};
    const Medium *medium{};
    const Transform *transform{};
    bool visible{true};
    float shadow_terminator{0.f};
    float intersection_offset{0.f};
    virtual bool is_mesh() const { return false; }
    virtual uint32_t vertex_properties() const { return 0u; }
    virtual const std::vector<lrk_vertex> &vertices() const;
    virtual const std::vector<lrk_triangle> &triangles() const;
    virtual std::vector<const Shape *> children() const { return {}; }
};

// ---- the scene ---------------------------------------------------------------------------------

class Scene {
public:
    static std::unique_ptr<Scene> create(const SceneDesc *desc);
    ~Scene();

    SceneNode *load_node(Tag tag, const NodeDesc *desc);
    template<typename T>
    T *load(Tag tag, const NodeDesc *desc) {
        auto n = load_node(tag, desc);
        if (!n) return nullptr;
        auto t = dynamic_cast<T *>(n);
        if (!t) throw Error("Scene node '" + desc->identifier() + "' has an unexpected category.");
        return t;
    }
    Texture *load_texture(const NodeDesc *d) { return load<Texture>(Tag::TEXTURE, d); }
    Transform *load_transform(const NodeDesc *d) { return load<Transform>(Tag::TRANSFORM, d); }
    Surface *load_surface(const NodeDesc *d) { return load<Surface>(Tag::SURFACE, d); }
    Light *load_light(const NodeDesc *d) { return load<Light>(Tag::LIGHT, d); }
    Medium *load_medium(const NodeDesc *d) { return load<Medium>(Tag::MEDIUM, d); }
    Shape *load_shape(const NodeDesc *d) { return load<Shape>(Tag::SHAPE, d); }
    Film *load_film(const NodeDesc *d) { return load<Film>(Tag::FILM, d); }
    Filter *load_filter(const NodeDesc *d) { return load<Filter>(Tag::FILTER, d); }
    Sampler *load_sampler(const NodeDesc *d) { return load<Sampler>(Tag::SAMPLER, d); }
    LightSampler *load_light_sampler(const NodeDesc *d) { return load<LightSampler>(Tag::LIGHT_SAMPLER, d); }
    PhaseFunction *load_phase_function(const NodeDesc *d) { return load<PhaseFunction>(Tag::PHASE_FUNCTION, d); }

    // shared defaults like SceneNodeDesc::shared_default_* (src/sdl/scene_node_desc.cpp:44-63)
    const NodeDesc *shared_default(Tag tag, const std::string &impl);

    const Integrator *integrator() const { return _integrator; }
    const Spectrum *spectrum() const { return _spectrum; }
    const Medium *environment_medium() const { return _environment_medium; }
    const Environment *environment() const { return _environment; }
    const std::vector<const Camera *> &cameras() const { return _cameras; }
    const std::vector<const Shape *> &shapes() const { return _shapes; }
    float shadow_terminator_factor() const { return _shadow_terminator; }
    float intersection_offset_factor() const { return _intersection_offset; }

private:
    Scene() = default;
    struct Handle {
        SceneNode *node;
        NodeDeleter *destroy;
    };
    std::vector<Handle> _internal_nodes;
    std::unordered_map<std::string, Handle> _nodes;
    std::vector<std::unique_ptr<NodeDesc>> _default_descs;
    std::unordered_map<std::string, const NodeDesc *> _default_lookup;
    std::recursive_mutex _mutex;
    const Integrator *_integrator{};
    const Spectrum *_spectrum{};
    const Medium *_environment_medium{};
    const Environment *_environment{};
    std::vector<const Camera *> _cameras;
    std::vector<const Shape *> _shapes;
    float _shadow_terminator{0.f};
    float _intersection_offset{0.f};
};

// ---- helpers shared with flatten ---------------------------------------------------------------

// alias table exactly as src/util/sampling.cpp:38-87 (shared with the device library's mesh updates)
using lrk::create_alias_table;

// icosphere by Loop subdivision, then projection to the unit sphere (src/shapes/sphere.cpp:60-101)
void make_sphere(uint32_t subdivision, std::vector<lrk_vertex> &vertices, std::vector<lrk_triangle> &triangles);
void loop_subdivide_mesh(const std::vector<lrk_vertex> &base_v, const std::vector<lrk_triangle> &base_t, uint32_t level,
                         std::vector<lrk_vertex> &vertices, std::vector<lrk_triangle> &triangles);

}// namespace lrh
