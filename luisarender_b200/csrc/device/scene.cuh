// Device-resident scene: the flattened POD arrays of include/lrk.h re-laid for 16-byte loads.
#pragma once
#include <cstdint>

#include "../../../include/lrk.h"
#include "light_tree.h"
#include "vecmath.cuh"

namespace lrk {

// One traversal instance record, 64 B = 4 x float4 (counted as N_xform in the roofline model):
//   rows 0..2 : world_to_object 3x4, row 3 : {as_float(blas_root), 0, 0, 0}
// One shading instance record: handle (uint4, 16 B) + object_to_world 3x4 (3 x float4, 48 B).
struct DeviceScene {
    // A copy of this very record in device memory (lrk_upload_scene).  Out-of-line device functions take the scene by reference;
    // handing them the kernel PARAMETER would make the compiler copy all of it into every thread's local memory (416 bytes of
    // stack and ~200 instructions per thread in the shade kernels before this pointer existed) - they get *self instead.
    const DeviceScene *self;
    const lrk_vertex *vertices;
    const lrk_triangle *triangles;
    const lrk_alias_entry *alias;
    const float *pdf;
    const lrk_mesh *meshes;
    const uint4 *inst_handles;
    const uint32_t *inst_kind;// per instance: its hit kind (hit_kinds.h), the bucket key of the material sort
    const float4 *inst_o2w;
    const float4 *inst_xform;
    const float4 *bvh_nodes;// 4 x float4 per node: {lo0.xyz,hi0.x} {hi0.yz,lo1.xy} {lo1.z,hi1.xyz} {ref0,ref1,parent,-}
    uint32_t *traversal_overflow;// set by a traversal kernel whose stack ran out (hierarchy deeper than the kernels support)
    const float4 *tri_verts;// 3 x float4 per BVH-ordered triangle slot, v0.w = prim id bits
    const lrk_surface *surfaces;
    const lrk_texture *textures;// image textures referenced by lrk_surface::tex
    const float4 *texels;       // RGBA float texels of all textures
    // environment light (spherical.cpp): importance map tables + parameters; env_prob = 0 <=> no environment
    const lrk_alias_entry *env_alias;
    const float *env_pdf;
    uint32_t env_present, env_emission_tex, env_map_width, env_map_height;
    float env_emission[3], env_scale, env_prob;
    float env_to_world[9];
    const lrk_light *lights;
    const lrk_light_handle *light_handles;
    const lrk_camera *camera;
    uint32_t tlas_root;
    uint32_t light_count;
    uint32_t instance_count;
    uint32_t surface_count;
    // integrator
    uint32_t max_depth;
    uint32_t rr_depth;
    float rr_threshold;
    uint32_t sampler_seed;
    uint32_t sampler_type;     // LRK_SAMPLER_*: uniform over a launch
    const lrk_sampler *sampler;// the record in device memory, its table pointers DEVICE copies (a kernel PARAMETER whose address is
                               // taken would be copied to every thread's local memory)
    // film
    float film_clamp;
    float film_scale[3];
    uint32_t width, height;
    // traversal warp scheduling (tunable, results do not depend on them)
    uint32_t refill_below;// refill idle lanes when fewer than this many lanes hold a live ray
    uint32_t inner_min;   // leave the inner-node phase when fewer lanes than this have inner work and leaves are waiting
    // homogeneous environment medium (volume path integrator only)
    float sigma_a[3], sigma_s[3];
    float medium_g;
    uint32_t medium_priority;
    // every medium of the scene, indexed by the shape handles' medium tags (general volume path, volume_general.cuh)
    const lrk_medium *media;
    uint32_t medium_count;
    uint32_t env_medium_tag;// LRK_MEDIUM_INVALID_TAG: none
};

// The light tree's arrays (option "light_tree", light_tree.h), in device memory right after the record DeviceScene::self points
// to: kept out of the kernel parameter, so that the parameter layout - and the code - of every kernel stays what it is without the
// tree.  All null unless the option was on at lrk_upload_scene (nodes also when no emitter has power).
struct DeviceLightTree {
    const LightTreeNode *nodes;
    const uint32_t *light_inst;        // per tree light: its instance
    const unsigned long long *trail;   // per tree light: its root-to-leaf bit trail
    const uint32_t *inst_light;        // per instance: its tree light, kLightTreeNone for none
    // The bottom level (option "light_tree_triangles"): a tree over the triangles of each emissive (mesh, side) pair, in object
    // space.  All null unless the option was on at lrk_upload_scene; then the triangle's probability is part of the selection pmf.
    const LightTreeNode *bottom_nodes;         // every bottom tree, each a slice whose child indices are relative to its root
    const uint2 *inst_bottom;                  // per instance: {root of its bottom tree in bottom_nodes, first of its trails}, root
                                               // kLightTreeNone for none
    const unsigned long long *bottom_trail;    // per triangle of a bottom tree: its trail
    // The light sampling as the resampling shade kernels read it at run time (option "light_candidates" >= 2; the other kernels
    // have it as template values): LightSelect, LightPoint (shading.cuh) and the candidate count M.
    uint32_t select, point, candidates;
    // The receiver words (option "light_receiver", receiver.h): one per path, indexed by its generation slot (id_rng.x); null unless
    // the option was on at lrk_upload_scene.  The shade kernels of the tree and solid-angle light samplings and the resampling ones
    // read the word of the previous vertex at the emitter hit, then overwrite it with their own where they sample a light.
    uint32_t *receiver;
};
__device__ __forceinline__ const DeviceLightTree &light_tree_of(const DeviceScene &sc) {
    return *reinterpret_cast<const DeviceLightTree *>(sc.self + 1);
}

}// namespace lrk
