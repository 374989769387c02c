// Device-side hit reconstruction, light sampling and closures for the sm_90a shade kernel.
// Hand-written restatement of the reference's DSL-staged functions (they only exist as AST
// recorders there); each block cites the reference file:line it follows (paths relative to the
// reference tree).  Expression order follows the reference so that the CPU oracle (oracle/oracle.cpp)
// and this file evaluate the same fp32 expressions.
#pragma once
#include "scene.cuh"
#include "spherical_triangle.h"

namespace lrk {

// ---- warps / sampling: src/util/sampling.cpp:13-31,89-98,133-155 ; src/util/sampling.h:38-70 ------
__device__ __forceinline__ void sample_uniform_disk_concentric(float ux, float uy, float &dx, float &dy) {
    float x = ux * 2.0f - 1.0f, y = uy * 2.0f - 1.0f;
    bool p = fabsf(x) > fabsf(y);
    float r = p ? x : y;
    float theta = p ? kPiOverFour * (y / x) : kPiOverTwo - kPiOverFour * (x / y);
    float s, c;
    sincosf(theta, &s, &c);
    dx = r * c;
    dy = r * s;
}
__device__ __forceinline__ V3 sample_cosine_hemisphere(float ux, float uy) {
    float dx, dy;
    sample_uniform_disk_concentric(ux, uy, dx, dy);
    float z = sqrtf(fmaxf(1.0f - dx * dx - dy * dy, 0.0f));
    return {dx, dy, z};
}
__device__ __forceinline__ V3 sample_uniform_triangle(float ux, float uy) {
    float a, b;
    if (ux < uy) { a = 0.5f * ux; b = -0.5f * ux + uy; }
    else { a = -0.5f * uy + ux; b = 0.5f * uy; }
    return {a, b, 1.0f - a - b};
}
__device__ __forceinline__ float balance_heuristic(float f_pdf, float g_pdf) {
    float sum_f = 1.0f * f_pdf;
    float sum = sum_f + 1.0f * g_pdf;
    return sum == 0.0f ? 0.0f : sum_f / sum;
}

// ---- Frame: src/util/frame.cpp:21-42 ; local trigonometry: src/util/frame.h:50-71 -------------------
struct Frame {
    V3 s, t, n;
    __device__ __forceinline__ static Frame make(V3 n) {
        float sgn = sign(n.z);
        float a = -1.f / (sgn + n.z);
        float b = n.x * n.y * a;
        V3 s = v3(1.f + sgn * sqr(n.x) * a, sgn * b, -sgn * n.x);
        V3 t = v3(b, sgn + sqr(n.y) * a, -n.y);
        return {normalize(s), normalize(t), n};
    }
    __device__ __forceinline__ static Frame make(V3 n, V3 s) {
        V3 ss = normalize(s - n * dot(n, s));
        V3 tt = normalize(cross(n, ss));
        return {ss, tt, n};
    }
    __device__ __forceinline__ V3 local_to_world(V3 d) const { return normalize(d.x * s + d.y * t + d.z * n); }
    __device__ __forceinline__ V3 world_to_local(V3 d) const { return normalize(v3(dot(d, s), dot(d, t), dot(d, n))); }
};
__device__ __forceinline__ float cos_theta(V3 w) { return w.z; }
__device__ __forceinline__ float cos2_theta(V3 w) { return sqr(w.z); }
__device__ __forceinline__ float abs_cos_theta(V3 w) { return fabsf(w.z); }
__device__ __forceinline__ float sin2_theta(V3 w) { return saturate(1.0f - cos2_theta(w)); }
__device__ __forceinline__ float sin_theta(V3 w) { return sqrtf(sin2_theta(w)); }
__device__ __forceinline__ float tan_theta(V3 w) { return sin_theta(w) / cos_theta(w); }
__device__ __forceinline__ float tan2_theta(V3 w) { return sin2_theta(w) / cos2_theta(w); }
__device__ __forceinline__ float cos_phi(V3 w) {
    float s = sin_theta(w);
    return s == 0.0f ? 1.0f : clampf(w.x / s, -1.0f, 1.0f);
}
__device__ __forceinline__ float sin_phi(V3 w) {
    float s = sin_theta(w);
    return s == 0.0f ? 0.0f : clampf(w.y / s, -1.0f, 1.0f);
}
__device__ __forceinline__ float cos2_phi(V3 w) { return sqr(cos_phi(w)); }
__device__ __forceinline__ float sin2_phi(V3 w) { return sqr(sin_phi(w)); }
__device__ __forceinline__ bool same_hemisphere(V3 w, V3 wp) { return w.z * wp.z > 0.0f; }
__device__ __forceinline__ float abs_dot(V3 a, V3 b) { return fabsf(dot(a, b)); }

// ---- Shape::Handle::decode: src/base/shape.cpp:72-93 ----------------------------------------------
struct ShapeHandle {
    uint32_t mesh, flags, surface_tag, light_tag, medium_tag, tri_count;
    float intersection_offset;
    __device__ __forceinline__ bool has_vertex_normal() const { return flags & LRK_SHAPE_HAS_VERTEX_NORMAL; }
    __device__ __forceinline__ bool has_vertex_uv() const { return flags & LRK_SHAPE_HAS_VERTEX_UV; }
    __device__ __forceinline__ bool has_surface() const { return flags & LRK_SHAPE_HAS_SURFACE; }
    __device__ __forceinline__ bool has_light() const { return flags & LRK_SHAPE_HAS_LIGHT; }
    __device__ __forceinline__ bool has_medium() const { return flags & LRK_SHAPE_HAS_MEDIUM; }
};
__device__ __forceinline__ ShapeHandle decode_handle(uint4 c) {
    ShapeHandle h;
    h.mesh = (c.x >> 10u) >> 2u;// buffer_base = 4 * mesh index (include/lrk.h)
    h.flags = c.x & 1023u;
    h.surface_tag = (c.y >> 12u) & 4095u;
    h.light_tag = c.y & 4095u;
    h.medium_tag = (c.y >> 24u) & 255u;
    h.tri_count = c.z;
    float off = static_cast<float>(c.w & 0xffffu) * (1.0f / 65536.f);
    h.intersection_offset = clampf(off * 255.f + 1.f, 1.f, 256.f);
    return h;
}

// ---- Interaction: src/base/interaction.{h,cpp}, src/base/geometry.cpp:281-389 ----------------------
struct Interaction {
    ShapeHandle shape;
    V3 pg, ng;
    float u, v;// interpolated vertex uv (geometry.cpp:372)
    Frame shading;
    uint32_t prim;
    float prim_area;
    bool back_facing;
};

// src/compute/src/dsl/rtx/ray.cpp:16-23
__device__ __forceinline__ float offset_component(float pc, float nc) {
    constexpr float origin = 1.0f / 32.0f;
    constexpr float float_scale = 1.0f / 65536.0f;
    constexpr float int_scale = 256.0f;
    int32_t of_i = static_cast<int32_t>(int_scale * nc);
    int32_t bits = __float_as_int(pc) + (pc < 0.0f ? -of_i : of_i);
    return fabsf(pc) < origin ? pc + float_scale * nc : __int_as_float(bits);
}
__device__ __forceinline__ V3 offset_ray_origin(V3 p, V3 n) {
    return {offset_component(p.x, n.x), offset_component(p.y, n.y), offset_component(p.z, n.z)};
}
// src/base/interaction.cpp:13-30
__device__ __forceinline__ V3 p_robust(const Interaction &it, V3 w) {
    bool front = dot(it.shading.n, w) > 0.f;
    V3 n = front ? it.ng : -it.ng;
    return offset_ray_origin(it.pg, it.shape.intersection_offset * n);
}

struct Mat34 {// three float4 rows
    float4 r0, r1, r2;
    __device__ __forceinline__ V3 col(int j) const {
        return j == 0 ? v3(r0.x, r1.x, r2.x) : j == 1 ? v3(r0.y, r1.y, r2.y) : j == 2 ? v3(r0.z, r1.z, r2.z) : v3(r0.w, r1.w, r2.w);
    }
};
// float3x3 * float3 = v.x*m[0] + v.y*m[1] + v.z*m[2] (cuda_device_math.h:2746)
__device__ __forceinline__ V3 mul3(const Mat34 &m, V3 v) { return v.x * m.col(0) + v.y * m.col(1) + v.z * m.col(2); }

__device__ __forceinline__ Mat34 load_o2w(const DeviceScene &sc, uint32_t inst) {
    const float4 *p = sc.inst_o2w + static_cast<size_t>(inst) * 3u;
    return {__ldg(p), __ldg(p + 1), __ldg(p + 2)};
}

// Geometry::shading_point (src/base/geometry.cpp:345-389) + Interaction ctor (src/base/interaction.h:97-101).
// `back_facing` is filled by the caller (geometry.cpp:290 for hits, uniform.cpp:121 for sampled light points).
__device__ __forceinline__ Interaction make_interaction(const DeviceScene &sc, uint32_t inst_id, uint32_t prim_id, V3 bary) {
    Interaction it;
    it.shape = decode_handle(__ldg(sc.inst_handles + inst_id));
    const lrk_mesh mesh = sc.meshes[it.shape.mesh];
    const lrk_triangle tri = sc.triangles[mesh.triangle_offset + prim_id];
    const float4 *vb = reinterpret_cast<const float4 *>(sc.vertices + mesh.vertex_offset);
    float4 a0 = __ldg(vb + tri.i0 * 2u), a1 = __ldg(vb + tri.i0 * 2u + 1u);
    float4 b0 = __ldg(vb + tri.i1 * 2u), b1 = __ldg(vb + tri.i1 * 2u + 1u);
    float4 c0 = __ldg(vb + tri.i2 * 2u), c1 = __ldg(vb + tri.i2 * 2u + 1u);
    // Vertex = {px,py,pz,nx | ny,nz,u,v}
    V3 p0 = v3(a0.x, a0.y, a0.z), p1 = v3(b0.x, b0.y, b0.z), p2 = v3(c0.x, c0.y, c0.z);
    V3 n0 = v3(a0.w, a1.x, a1.y), n1 = v3(b0.w, b1.x, b1.y), n2 = v3(c0.w, c1.x, c1.y);
    Mat34 m = load_o2w(sc, inst_id);
    V3 t = m.col(3);
    V3 ns_local = bary.x * n0 + bary.y * n1 + bary.z * n2;
    float duv0x = b1.z - a1.z, duv0y = b1.w - a1.w;
    float duv1x = c1.z - a1.z, duv1y = c1.w - a1.w;
    float det = mul_exact(duv0x, duv1y) - mul_exact(duv0y, duv1x);// exactly 0 for degenerate uv: selects the fallback frame below
    float inv_det = 1.f / det;
    V3 dp0 = p1 - p0, dp1 = p2 - p0;
    V3 dpdu_local = (dp0 * duv1y - dp1 * duv0y) * inv_det;
    V3 p = mul3(m, bary.x * p0 + bary.y * p1 + bary.z * p2) + t;
    it.u = bary.x * a1.z + bary.y * b1.z + bary.z * c1.z;
    it.v = bary.x * a1.w + bary.y * b1.w + bary.z * c1.w;
    V3 c = cross(mul3(m, dp0), mul3(m, dp1));
    float area = length(c) * .5f;
    V3 ng = normalize(c);
    Frame fallback = Frame::make(ng);
    V3 dpdu = det == 0.f ? fallback.s : mul3(m, dpdu_local);
    V3 ns = ng;
    if (it.shape.has_vertex_normal()) {
        // mn = transpose(inverse(m)), GLM-style inverse (cuda_device_math.h:3615-3630)
        V3 m0 = m.col(0), m1 = m.col(1), m2 = m.col(2);
        float one_over_det = 1.0f / (m0.x * (m1.y * m2.z - m2.y * m1.z) - m1.x * (m0.y * m2.z - m2.y * m0.z) +
                                     m2.x * (m0.y * m1.z - m1.y * m0.z));
        V3 i0 = v3((m1.y * m2.z - m2.y * m1.z) * one_over_det, (m2.y * m0.z - m0.y * m2.z) * one_over_det,
                   (m0.y * m1.z - m1.y * m0.z) * one_over_det);
        V3 i1 = v3((m2.x * m1.z - m1.x * m2.z) * one_over_det, (m0.x * m2.z - m2.x * m0.z) * one_over_det,
                   (m1.x * m0.z - m0.x * m1.z) * one_over_det);
        V3 i2 = v3((m1.x * m2.y - m2.x * m1.y) * one_over_det, (m2.x * m0.y - m0.x * m2.y) * one_over_det,
                   (m0.x * m1.y - m1.x * m0.y) * one_over_det);
        V3 mn0 = v3(i0.x, i1.x, i2.x), mn1 = v3(i0.y, i1.y, i2.y), mn2 = v3(i0.z, i1.z, i2.z);
        ns = normalize(ns_local.x * mn0 + ns_local.y * mn1 + ns_local.z * mn2);
    }
    it.pg = p;
    it.ng = ng;
    it.prim_area = area;
    it.shading = Frame::make(face_forward(ns, ng), dpdu);
    it.prim = prim_id;
    it.back_facing = false;
    return it;
}

// World-space position of a hit only — the same expression as make_interaction's `pg`, for callers that need nothing else
// (distance to the surface in the volume integrator, sampled light points seen from inside a medium).
__device__ __forceinline__ V3 hit_position(const DeviceScene &sc, uint32_t inst_id, uint32_t prim_id, V3 bary) {
    ShapeHandle shape = decode_handle(__ldg(sc.inst_handles + inst_id));
    const lrk_mesh mesh = sc.meshes[shape.mesh];
    const lrk_triangle tri = sc.triangles[mesh.triangle_offset + prim_id];
    const float4 *vb = reinterpret_cast<const float4 *>(sc.vertices + mesh.vertex_offset);
    float4 a0 = __ldg(vb + tri.i0 * 2u), b0 = __ldg(vb + tri.i1 * 2u), c0 = __ldg(vb + tri.i2 * 2u);
    V3 p0 = v3(a0.x, a0.y, a0.z), p1 = v3(b0.x, b0.y, b0.z), p2 = v3(c0.x, c0.y, c0.z);
    Mat34 m = load_o2w(sc, inst_id);
    return mul3(m, bary.x * p0 + bary.y * p1 + bary.z * p2) + m.col(3);
}

// ---- lights: src/lights/diffuse.cpp:67-88 ; src/lightsamplers/uniform.cpp:50-65,78-137 ------------------
struct LightEval {
    V3 L;
    float pdf;
};

// image emission: max(texel.xyz, 0) at the interaction's uv (texture.cpp:47-57, srgb.cpp:48-54).  TEX: only the TEXTURED kernel
// variants contain the lookup (lrk_upload_scene selects them when a light has an emission texture); the others keep the constant
__device__ __noinline__ inline V3 light_emission_texel(const DeviceScene &sc, uint32_t emission_tex, float u, float v);
// triangle_selected: the light selection chose the triangle itself (the bottom light trees), so its probability is in the selection
// pmf and the point's pdf is 1 / area of the triangle
template<bool TEX = true>
__device__ __forceinline__ LightEval diffuse_light_evaluate(const DeviceScene &sc, const Interaction &it_light, V3 p_from, bool triangle_selected = false) {
    const lrk_light light = sc.lights[it_light.shape.light_tag];
    const lrk_mesh mesh = sc.meshes[it_light.shape.mesh];
    float pdf_triangle = triangle_selected ? 1.f : __ldg(sc.pdf + mesh.triangle_offset + it_light.prim);
    float pdf_area = pdf_triangle / it_light.prim_area;
    float cos_wo = abs_dot(normalize(p_from - it_light.pg), it_light.ng);
    V3 L = v3(light.emission[0], light.emission[1], light.emission[2]);
    if (TEX && light.emission_tex != 0u) L = light_emission_texel(sc, light.emission_tex, it_light.u, it_light.v);
    L = L * light.scale;
    V3 diff = it_light.pg - p_from;
    float pdf = dot(diff, diff) * pdf_area * (1.0f / cos_wo);
    bool invalid = fabsf(cos_wo) < 1e-6f || (!light.two_sided && it_light.back_facing);
    LightEval e;
    e.L = invalid ? v3(0.f) : L;
    e.pdf = invalid ? 0.0f : pdf;
    return e;
}

// Light selection of next-event estimation: the reference's uniform sampler over the light NODES (uniform.cpp), or the light tree
// of the option "light_tree" over the emissive instances (light_tree.h)
enum LightSelect : uint32_t { kLightSelectUniform = 0u, kLightSelectTree = 1u };

// The descents of the light tree, out of line so that the shade kernels' register allocation does not grow with them.
__device__ __noinline__ inline uint32_t light_tree_sample(const LightTreeNode *nodes, V3 p, float u, float &pmf, float &u_left) {
    return light_tree_walk<true>(nodes, p.x, p.y, p.z, u, 0ull, pmf, &u_left);
}
__device__ __noinline__ inline float light_tree_pmf(const LightTreeNode *nodes, const uint32_t *inst_light, const unsigned long long *trail, V3 p,
                                                    uint32_t inst) {
    const uint32_t l = __ldg(inst_light + inst);
    if (l == kLightTreeNone) return 0.f;// an emitter without power
    float pmf;
    light_tree_walk<false>(nodes, p.x, p.y, p.z, 0.f, __ldg(trail + l), pmf);
    return pmf;
}

// The bottom level (option "light_tree_triangles", light_tree_of(sc).bottom_nodes not null): the walk of instance inst's tree over
// its mesh's triangles at p mapped to object space.  Sampling continues with the u the top walk left; both return pmf 0 and the
// sample kLightTreeNone for an instance without a tree or a point no triangle faces.
__device__ __forceinline__ V3 light_tree_to_object(const DeviceScene &sc, uint32_t inst, V3 p) {
    const float4 *x = sc.inst_xform + static_cast<size_t>(inst) * 4u;
    const float4 m0 = __ldg(x + 0), m1 = __ldg(x + 1), m2 = __ldg(x + 2);
    const float w2o[12] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w, m2.x, m2.y, m2.z, m2.w};
    V3 q;
    light_tree_object_point(w2o, p.x, p.y, p.z, q.x, q.y, q.z);
    return q;
}
__device__ __noinline__ inline uint32_t light_tree_sample_triangle(const DeviceScene &sc, uint32_t inst, V3 p, float u, float &pmf) {
    const DeviceLightTree &lt = light_tree_of(sc);
    const uint32_t root = __ldg(lt.inst_bottom + inst).x;
    pmf = 0.f;
    if (root == kLightTreeNone) return kLightTreeNone;
    const V3 q = light_tree_to_object(sc, inst, p);
    return light_tree_walk<true>(lt.bottom_nodes + root, q.x, q.y, q.z, u, 0ull, pmf);
}
__device__ __noinline__ inline float light_tree_triangle_pmf(const DeviceScene &sc, uint32_t inst, uint32_t prim, V3 p) {
    const DeviceLightTree &lt = light_tree_of(sc);
    const uint2 b = __ldg(lt.inst_bottom + inst);
    if (b.x == kLightTreeNone) return 0.f;
    const V3 q = light_tree_to_object(sc, inst, p);
    return light_tree_triangle_pmf_at(lt.bottom_nodes + b.x, q.x, q.y, q.z, __ldg(lt.bottom_trail + b.y + prim), prim);
}

// Point sampling of next-event estimation: the reference's area sampling of the chosen triangle, or, with the option
// "light_solid_angle", uniform sampling of the spherical triangle it subtends where use_spherical allows (spherical_triangle.h)
enum LightPoint : uint32_t { kLightPointArea = 0u, kLightPointSolidAngle = 1u };

// The solid-angle code, out of line like the tree's descents.  Both read the triangle's world-space vertices as make_interaction
// transforms them; a sample and an emitter hit take omega from the one function, so their pdfs agree bit for bit for one point.
__device__ __forceinline__ void light_triangle_world(const DeviceScene &sc, uint32_t inst, uint32_t prim, SphVec &v0, SphVec &v1, SphVec &v2) {
    const ShapeHandle shape = decode_handle(__ldg(sc.inst_handles + inst));
    const lrk_mesh mesh = sc.meshes[shape.mesh];
    const lrk_triangle tri = sc.triangles[mesh.triangle_offset + prim];
    const float4 *vb = reinterpret_cast<const float4 *>(sc.vertices + mesh.vertex_offset);
    const float4 a0 = __ldg(vb + tri.i0 * 2u), b0 = __ldg(vb + tri.i1 * 2u), c0 = __ldg(vb + tri.i2 * 2u);
    const Mat34 m = load_o2w(sc, inst);
    const V3 t = m.col(3);
    const V3 w0 = mul3(m, v3(a0.x, a0.y, a0.z)) + t, w1 = mul3(m, v3(b0.x, b0.y, b0.z)) + t, w2 = mul3(m, v3(c0.x, c0.y, c0.z)) + t;
    v0 = {w0.x, w0.y, w0.z};
    v1 = {w1.x, w1.y, w1.z};
    v2 = {w2.x, w2.y, w2.z};
}
__device__ __noinline__ inline float light_triangle_solid_angle(const DeviceScene &sc, uint32_t inst, uint32_t prim, V3 p) {
    SphVec v0, v1, v2;
    light_triangle_world(sc, inst, prim, v0, v1, v2);
    return solid_angle({p.x, p.y, p.z}, v0, v1, v2);
}
__device__ __noinline__ inline V3 light_triangle_sample_spherical(const DeviceScene &sc, uint32_t inst, uint32_t prim, V3 p, float omega, float u0,
                                                                  float u1) {
    SphVec v0, v1, v2;
    light_triangle_world(sc, inst, prim, v0, v1, v2);
    const SphVec b = sample_spherical_triangle({p.x, p.y, p.z}, v0, v1, v2, omega, u0, u1);
    return v3(b.x, b.y, b.z);
}
// The pdf of a light point of triangle it_light.prim seen from a point where its solid angle is omega: pdf[tri] / omega where the
// spherical sampler serves the triangle there, else area_pdf, the reference's area pdf in solid angle (diffuse_light_evaluate;
// 0 for a point that emits nothing there, which stays 0; triangle_selected as in diffuse_light_evaluate: 1 / omega)
__device__ __forceinline__ float light_point_pdf(const DeviceScene &sc, const Interaction &it_light, float area_pdf, float omega,
                                                 bool triangle_selected = false) {
    if (area_pdf == 0.f || !use_spherical(omega)) return area_pdf;
    return (triangle_selected ? 1.f : __ldg(sc.pdf + sc.meshes[it_light.shape.mesh].triangle_offset + it_light.prim)) / omega;
}

// `inst`: the instance hit (used by the light tree and the solid-angle sampler only)
template<bool TEX = true, uint32_t SEL = kLightSelectUniform, uint32_t PT = kLightPointArea>
__device__ __forceinline__ LightEval evaluate_hit(const DeviceScene &sc, const Interaction &it, V3 p_from, uint32_t inst = 0u) {
    // with the bottom light trees the selection pmf holds the triangle's probability (the top pmf times the bottom pmf)
    const bool tri_sel = SEL == kLightSelectTree && light_tree_of(sc).bottom_nodes != nullptr;
    LightEval e = diffuse_light_evaluate<TEX>(sc, it, p_from, tri_sel);
    if (PT == kLightPointSolidAngle && e.pdf != 0.f)
        e.pdf = light_point_pdf(sc, it, e.pdf, light_triangle_solid_angle(*sc.self, inst, it.prim, p_from), tri_sel);
    if (SEL == kLightSelectTree) {
        const DeviceLightTree &lt = light_tree_of(sc);
        float pmf = light_tree_pmf(lt.nodes, lt.inst_light, lt.trail, p_from, inst);
        if (tri_sel && pmf != 0.f) pmf *= light_tree_triangle_pmf(*sc.self, inst, it.prim, p_from);
        e.pdf *= (1.f - sc.env_prob) * pmf;
        return e;
    }
    float n = static_cast<float>(sc.light_count);
    e.pdf *= (1.f - sc.env_prob) / n;// uniform.cpp:63 (env_prob = 0 without an environment)
    return e;
}

// the environment light (defined after the texture code): src/environments/spherical.cpp:83-137
__device__ inline LightEval environment_evaluate(const DeviceScene &sc, V3 wi);
__device__ inline LightEval environment_sample(const DeviceScene &sc, float u0, float u1, V3 &wi);

struct LightSample {
    LightEval eval;
    float4 ray_o_tmin, ray_d_tmax;
};

// `p_shading`: it_from.p_shading(), the point the light's emission and pdf are evaluated from (diffuse.cpp:62-86) - the hit point
// for a surface interaction, but the WORLD ORIGIN for the volume integrator's Interaction{ray->origin()}, whose shading point is
// never set (mega_vpt_naive.cpp:283-285; the reference's renders carry that, so this library does too)
template<bool TEX = true, uint32_t SEL = kLightSelectUniform, uint32_t PT = kLightPointArea>
__device__ __forceinline__ LightSample sample_light_from(const DeviceScene &sc, const Interaction &it_from, V3 p_shading, float u_sel, float u0, float u1) {
    LightSample s;
    float n = static_cast<float>(sc.light_count);
    // UniformLightSamplerInstance::select, uniform.cpp:78-90
    const float ep = sc.env_prob;
    bool is_env = ep == 1.f;
    uint32_t tag = 0u;
    float sel_prob = 1.f;
    bool tri_sel = false;// the bottom light trees chose the triangle: tree_tri
    uint32_t tree_tri = 0u;
    if (SEL == kLightSelectTree) {// the environment keeps its probability; the tree divides the rest
        float uu = u_sel;
        if (ep != 0.f && ep != 1.f) {
            uu = (u_sel - ep) / (1.f - ep);
            is_env = u_sel < ep;
        }
        if (is_env) {
            sel_prob = ep;
        } else {
            const DeviceLightTree &lt = light_tree_of(sc);
            const LightTreeNode *nodes = lt.nodes;
            float pmf = 0.f, u_left = 0.f;
            uint32_t l = nodes != nullptr ? light_tree_sample(nodes, it_from.pg, uu, pmf, u_left) : kLightTreeNone;
            if (l != kLightTreeNone) tag = __ldg(lt.light_inst + l);// the instance itself
            tri_sel = lt.bottom_nodes != nullptr;
            if (tri_sel && l != kLightTreeNone) {// one selection number for the whole descent: the top walk's u continues
                float tri_pmf;
                tree_tri = light_tree_sample_triangle(*sc.self, tag, it_from.pg, u_left, tri_pmf);
                if (tree_tri == kLightTreeNone) l = kLightTreeNone;
                pmf *= tri_pmf;
            }
            if (l == kLightTreeNone) {// no emitter can reach the point: nothing to trace
                s.eval.L = v3(0.f);
                s.eval.pdf = 0.f;
                s.ray_o_tmin = make_float4(0.f, 0.f, 0.f, 0.f);
                s.ray_d_tmax = make_float4(0.f, 0.f, 1.f, 0.f);
                return s;
            }
            sel_prob = ep == 0.f ? pmf : (1.f - ep) * pmf;
        }
    } else if (ep == 0.f) {
        tag = static_cast<uint32_t>(clampf(u_sel * n, 0.f, n - 1.f));
        sel_prob = 1.f / n;
    } else if (ep != 1.f) {
        float uu = (u_sel - ep) / (1.f - ep);
        tag = static_cast<uint32_t>(clampf(uu * n, 0.f, n - 1.f));
        is_env = u_sel < ep;
        sel_prob = is_env ? ep : (1.f - ep) / n;
    }
    if (is_env) {// sample_environment + Sample::from_environment (light_sampler.cpp:84-90,120-123): a ray to infinity
        V3 wi;
        s.eval = environment_sample(*sc.self, u0, u1, wi);
        s.eval.pdf *= sel_prob;
        V3 o = p_robust(it_from, wi);
        s.ray_o_tmin = make_float4(o.x, o.y, o.z, 0.f);
        s.ray_d_tmax = make_float4(wi.x, wi.y, wi.z, kFltMax);
        return s;
    }
    lrk_light_handle handle;
    if (SEL == kLightSelectTree) handle.instance_id = tag;
    else handle = sc.light_handles[tag];
    ShapeHandle light_inst = decode_handle(__ldg(sc.inst_handles + handle.instance_id));
    const lrk_mesh mesh = sc.meshes[light_inst.mesh];
    uint32_t triangle_id;
    float ux;
    if (SEL == kLightSelectTree && tri_sel) {
        triangle_id = tree_tri;
        ux = u0;
    } else {// sample_alias_table: src/util/sampling.h:38-50
        float u = u0 * static_cast<float>(light_inst.tri_count);
        uint32_t i = min(max(static_cast<uint32_t>(u), 0u), light_inst.tri_count - 1u);
        float u_remapped = u - floorf(u);
        lrk_alias_entry entry = sc.alias[mesh.triangle_offset + i];
        bool keep = u_remapped < entry.prob;
        triangle_id = keep ? i : entry.alias;
        ux = keep ? u_remapped / entry.prob : (u_remapped - entry.prob) / (1.0f - entry.prob);
    }
    V3 uvw;
    float omega = 0.f;
    if (PT == kLightPointSolidAngle) {// the same two numbers drive either sampler
        omega = light_triangle_solid_angle(*sc.self, handle.instance_id, triangle_id, p_shading);
        uvw = use_spherical(omega) ? light_triangle_sample_spherical(*sc.self, handle.instance_id, triangle_id, p_shading, omega, ux, u1)
                                   : sample_uniform_triangle(ux, u1);
    } else {
        uvw = sample_uniform_triangle(ux, u1);
    }
    Interaction it_light = make_interaction(sc, handle.instance_id, triangle_id, uvw);
    it_light.back_facing = dot(it_light.ng, it_from.pg - it_light.pg) < 0.f;
    s.eval = diffuse_light_evaluate<TEX>(sc, it_light, p_shading, tri_sel);
    if (PT == kLightPointSolidAngle) s.eval.pdf = light_point_pdf(sc, it_light, s.eval.pdf, omega, tri_sel);
    s.eval.pdf *= sel_prob;
    // Interaction::spawn_ray_to, src/base/interaction.cpp:25-30
    V3 p_from = p_robust(it_from, it_light.pg - it_from.pg);
    V3 Lv = it_light.pg - p_from;
    float d = length(Lv);
    V3 dir = Lv * (1.f / d);
    s.ray_o_tmin = make_float4(p_from.x, p_from.y, p_from.z, 0.f);
    s.ray_d_tmax = make_float4(dir.x, dir.y, dir.z, d * .9999f);
    return s;
}

template<bool TEX = true, uint32_t SEL = kLightSelectUniform, uint32_t PT = kLightPointArea>
__device__ __forceinline__ LightSample sample_light(const DeviceScene &sc, const Interaction &it_from, float u_sel, float u0, float u1) {
    return sample_light_from<TEX, SEL, PT>(sc, it_from, it_from.pg, u_sel, u0, u1);
}

// ---- image textures: src/textures/image.cpp:132-166, sampled like the reference's software sampler
// (src/compute/src/rust/luisa_compute_backend_impl/src/cpu/codegen/cpu_texture.h:418-464,489-493) --------------------
__device__ __forceinline__ float tex_fract(float x) { return x - floorf(x); }
__device__ __forceinline__ float tex_coord_point(uint32_t address, float uv, float s) {
    switch (address) {
        case LRK_TEX_ADDRESS_EDGE: return clampf(uv, 0.0f, kOneMinusEpsilon) * s;
        case LRK_TEX_ADDRESS_REPEAT: return tex_fract(uv) * s;
        case LRK_TEX_ADDRESS_MIRROR: {
            uv = fmodf(fabsf(uv), 2.0f);
            uv = uv < 1.f ? uv : 2.f - uv;
            return fminf(uv, kOneMinusEpsilon) * s;
        }
        default: return (uv < 0.f || uv >= 1.f) ? 65536.f : uv * s;// ZERO
    }
}
__device__ __forceinline__ float4 tex_read(const DeviceScene &sc, const lrk_texture &t, uint32_t x, uint32_t y) {
    if (!(x < t.width & y < t.height)) return make_float4(0.f, 0.f, 0.f, 0.f);
    return __ldg(sc.texels + t.texel_offset + static_cast<size_t>(y) * t.width + x);
}
__device__ __forceinline__ float4 lerp4(float4 a, float4 b, float t) {
    return make_float4(lerp(a.x, b.x, t), lerp(a.y, b.y, t), lerp(a.z, b.z, t), lerp(a.w, b.w, t));
}
__device__ __forceinline__ float4 texture_sample(const DeviceScene &sc, const lrk_texture &t, float u, float v) {
    const float sx = static_cast<float>(t.width), sy = static_cast<float>(t.height);
    if (t.filter == LRK_TEX_FILTER_POINT) {
        float cx = tex_coord_point(t.address, u, sx), cy = tex_coord_point(t.address, v, sy);
        return tex_read(sc, t, static_cast<uint32_t>(cx), static_cast<uint32_t>(cy));
    }
    const float inv_sx = 1.f / sx, inv_sy = 1.f / sy;
    float ax = tex_coord_point(t.address, u - .5f * inv_sx, sx), bx = tex_coord_point(t.address, u + .5f * inv_sx, sx);
    float ay = tex_coord_point(t.address, v - .5f * inv_sy, sy), by = tex_coord_point(t.address, v + .5f * inv_sy, sy);
    float x_min = fminf(ax, bx), x_max = fmaxf(ax, bx), y_min = fminf(ay, by), y_max = fmaxf(ay, by);
    float tx = tex_fract(x_max), ty = tex_fract(y_max);
    uint32_t x0 = static_cast<uint32_t>(x_min), y0 = static_cast<uint32_t>(y_min);
    uint32_t x1 = static_cast<uint32_t>(x_max), y1 = static_cast<uint32_t>(y_max);
    float4 v00 = tex_read(sc, t, x0, y0), v01 = tex_read(sc, t, x1, y0), v10 = tex_read(sc, t, x0, y1), v11 = tex_read(sc, t, x1, y1);
    return lerp4(lerp4(v00, v01, tx), lerp4(v10, v11, tx), ty);
}
// ImageTextureInstance::evaluate: uv transform, sample, decode (image.cpp:136-166)
__device__ __forceinline__ float tex_decode(const lrk_texture &t, float x) {
    if (t.encoding == LRK_TEX_ENCODING_SRGB) {
        float lin = x <= 0.04045f ? x * (1.0f / 12.92f) : builtin_pow((x + 0.055f) * (1.0f / 1.055f), 2.4f);
        return t.scale * lin;
    }
    if (t.encoding == LRK_TEX_ENCODING_GAMMA) return t.scale * builtin_pow(x, t.gamma);
    return t.scale * x;
}
// Not inlined on purpose: up to a dozen call sites per closure, executed only for textured materials.
__device__ __noinline__ inline float4 texture_evaluate(const DeviceScene &sc, uint32_t tex_id, float u, float v) {
    const lrk_texture t = sc.textures[tex_id];
    float4 s = texture_sample(sc, t, u * t.uv_scale[0] + t.uv_offset[0], v * t.uv_scale[1] + t.uv_offset[1]);
    return make_float4(tex_decode(t, s.x), tex_decode(t, s.y), tex_decode(t, s.z), tex_decode(t, s.w));
}
__device__ __noinline__ inline V3 light_emission_texel(const DeviceScene &sc, uint32_t emission_tex, float u, float v) {
    const float4 t = texture_evaluate(sc, emission_tex - 1u, u, v);
    return v3(fmaxf(t.x, 0.f), fmaxf(t.y, 0.f), fmaxf(t.z, 0.f));
}
// Surface parameters at a hit: the node's constants with the image-textured slots evaluated at the hit's uv
// (MatteInstance::populate_closure matte.cpp:117-131, DisneySurfaceInstance::populate_closure disney.cpp:932-956;
// colours through Texture::Instance::evaluate_albedo_spectrum texture.cpp:20-31 + srgb.cpp:34-40,70-72).
// fresnel_dielectric_integral (src/util/scattering.cpp:98-108): the fitted polynomials, Horner from the last coefficient
__device__ __forceinline__ float fresnel_dielectric_integral(float eta) {
    float r;
    if (eta == 1.f) {
        r = 0.f;
    } else if (eta < 1.f) {
        r = eta * (eta * (eta * -0.90663979f + 2.23559031f) + -2.09069066f) + 0.75985009f;
    } else {
        float x = 1.f / eta;
        r = x * (x * -1.18995376f + 0.21762732f) + 0.97945724f;
    }
    return saturate(r);
}

// Mirror / Glass / Plastic / Metal with image-textured parameters (LRK_SURFACE_RAW_PARAMS, include/lrk.h): evaluates the textured
// raw parameters at the hit and derives the closure context as the surfaces' populate_closure do (mirror.cpp:142-162,
// glass.cpp:236-279, plastic.cpp:252-291, metal.cpp:273-310).  Out of line: these kernels are not the headline's.
__device__ __noinline__ inline void resolve_raw_surface(const DeviceScene &sc, lrk_surface &s, float u, float v) {
    auto colour = [&](uint32_t slot) {// evaluate_albedo_spectrum with the sRGB spectrum: saturate(extend_color_to_rgb(v))
        if (s.tex[slot] == 0u) return;
        const float4 val = texture_evaluate(sc, s.tex[slot] - 1u, u, v);
        const uint32_t ch = sc.textures[s.tex[slot] - 1u].channels;
        const V3 rgb = ch == 1u ? v3(val.x, val.x, val.x) : ch == 2u ? v3(val.x, val.y, 1.f) : v3(val.x, val.y, val.z);
        s.p[slot] = saturate(rgb.x);
        s.p[slot + 1u] = saturate(rgb.y);
        s.p[slot + 2u] = saturate(rgb.z);
    };
    auto alpha = [&](uint32_t slot) {// one channel feeds both axes; roughness_to_alpha = max(r^2, 1e-4) (scattering.cpp:129-135)
        if (s.tex[slot] == 0u) return;
        const float4 r = texture_evaluate(sc, s.tex[slot] - 1u, u, v);
        const bool one = sc.textures[s.tex[slot] - 1u].channels == 1u;
        float ax = r.x, ay = one ? r.x : r.y;
        if (s.flags & LRK_SURFACE_REMAP_ROUGHNESS) {
            ax = fmaxf(ax * ax, 1e-4f);
            ay = fmaxf(ay * ay, 1e-4f);
        }
        s.p[slot] = ax;
        s.p[slot + 1u] = ay;
    };
    auto lum = [](const float *c) { return 0.212671f * c[0] + 0.715160f * c[1] + 0.072169f * c[2]; };// src/util/colorspace.h:21-25
    switch (s.type) {
        case LRK_SURFACE_MIRROR:
            colour(0u);
            alpha(3u);
            break;
        case LRK_SURFACE_GLASS: {
            colour(0u);
            colour(3u);
            alpha(7u);
            const float kr_lum = lum(&s.p[0]), kt_lum = lum(&s.p[3]);
            s.p[9] = kr_lum == 0.f ? 0.f : kr_lum / (kr_lum + kt_lum);
            break;
        }
        case LRK_SURFACE_PLASTIC: {
            colour(0u);
            colour(4u);
            alpha(8u);
            if (s.tex[10] != 0u) s.p[10] = texture_evaluate(sc, s.tex[10] - 1u, u, v).x;
            const float kd_lum = lum(&s.p[0]), sa_lum = lum(&s.p[4]);
            const float average_transmittance = expf(-2.f * sa_lum * s.p[10]);
            const float fdr = fresnel_dielectric_integral(s.p[7]);
            for (int c = 0; c < 3; c++) s.p[c] = s.p[c] / (1.f - s.p[c] * fdr);
            s.p[3] = kd_lum * average_transmittance;
            break;
        }
        default:// METAL
            colour(6u);
            alpha(9u);
            break;
    }
}

__device__ __forceinline__ void resolve_surface_textures(const DeviceScene &sc, lrk_surface &s, float u, float v) {
    if (s.flags & LRK_SURFACE_RAW_PARAMS) {
        resolve_raw_surface(*sc.self, s, u, v);
        return;
    }
    if (s.tex[0] != 0u) {
        float4 val = texture_evaluate(*sc.self, s.tex[0] - 1u, u, v);
        const uint32_t ch = sc.textures[s.tex[0] - 1u].channels;
        V3 rgb = ch == 1u ? v3(val.x, val.x, val.x) : ch == 2u ? v3(val.x, val.y, 1.f) : v3(val.x, val.y, val.z);
        rgb = v3(saturate(rgb.x), saturate(rgb.y), saturate(rgb.z));// encode_srgb_albedo's clamp, decode_albedo's saturate
        s.p[0] = rgb.x;
        s.p[1] = rgb.y;
        s.p[2] = rgb.z;
        if (s.type == LRK_SURFACE_DISNEY) s.p[3] = 0.212671f * rgb.x + 0.715160f * rgb.y + 0.072169f * rgb.z;
    }
    if (s.type == LRK_SURFACE_MATTE) {
        if (s.tex[3] != 0u) s.p[3] = saturate(texture_evaluate(*sc.self, s.tex[3] - 1u, u, v).x) * 90.f;
    } else {
#pragma unroll
        for (uint32_t k = 4u; k < 16u; k++) {
            if (s.tex[k] != 0u) {
                float x = texture_evaluate(*sc.self, s.tex[k] - 1u, u, v).x;
                if (k == 6u && (s.flags & LRK_SURFACE_REMAP_ROUGHNESS)) x = fmaxf(x * x, 1e-4f);// roughness_to_alpha
                s.p[k] = x;
            }
        }
    }
}

// ---- Spherical environment: src/environments/spherical.cpp:42-137 (uv mapping, evaluate, sample); tables built by the host ----
__device__ __forceinline__ V3 env_mul(const float *m, V3 v, bool transposed) {// float3x3 * float3 = v.x*col0 + v.y*col1 + v.z*col2
    if (!transposed) return v.x * v3(m[0], m[3], m[6]) + v.y * v3(m[1], m[4], m[7]) + v.z * v3(m[2], m[5], m[8]);
    return v.x * v3(m[0], m[1], m[2]) + v.y * v3(m[3], m[4], m[5]) + v.z * v3(m[6], m[7], m[8]);
}
__device__ __forceinline__ V3 env_radiance(const DeviceScene &sc, float u, float v) {// _evaluate (:70-75) + decode_illuminant
    V3 rgb = v3(sc.env_emission[0], sc.env_emission[1], sc.env_emission[2]);
    if (sc.env_emission_tex != 0u) {
        float4 t = texture_evaluate(*sc.self, sc.env_emission_tex - 1u, u, v);
        rgb = v3(fmaxf(t.x, 0.f), fmaxf(t.y, 0.f), fmaxf(t.z, 0.f));
    }
    return rgb * sc.env_scale;
}
__device__ __forceinline__ float env_directional_pdf(float p, float theta) {// :77-81
    float s = sinf(theta);
    float inv_s = s > 0.f ? 1.f / s : 0.f;
    return p * inv_s * (.5f * kInvPi * kInvPi);
}
__device__ __noinline__ inline LightEval environment_evaluate(const DeviceScene &sc, V3 wi) {
    V3 w = normalize(env_mul(sc.env_to_world, wi, true));
    float theta = acosf(w.y), phi = atan2f(w.x, w.z);// direction_to_uv, :53-59
    float u = 1.f - 0.5f * kInvPi * phi, v = theta * kInvPi;
    u = u - floorf(u);
    v = v - floorf(v);
    LightEval out;
    out.L = env_radiance(sc, u, v);
    if (sc.env_emission_tex == 0u) {
        out.pdf = kInvPi * 0.25f;// uniform_sphere_pdf
    } else {
        float sx = static_cast<float>(sc.env_map_width), sy = static_cast<float>(sc.env_map_height);
        uint32_t ix = static_cast<uint32_t>(clampf(u * sx, 0.f, sx - 1.f)), iy = static_cast<uint32_t>(clampf(v * sy, 0.f, sy - 1.f));
        out.pdf = env_directional_pdf(__ldg(sc.env_pdf + static_cast<size_t>(iy) * sc.env_map_width + ix), theta);
    }
    return out;
}
__device__ __forceinline__ void sample_alias(const lrk_alias_entry *table, uint32_t n, float u_in, uint32_t &index, float &uu) {
    float u = u_in * static_cast<float>(n);// sample_alias_table, src/util/sampling.h:38-50
    uint32_t i = min(max(static_cast<uint32_t>(u), 0u), n - 1u);
    float u_remapped = u - floorf(u);
    lrk_alias_entry entry = table[i];
    bool keep = u_remapped < entry.prob;
    index = keep ? i : entry.alias;
    uu = keep ? u_remapped / entry.prob : (u_remapped - entry.prob) / (1.0f - entry.prob);
}
__device__ __noinline__ inline LightEval environment_sample(const DeviceScene &sc, float u0, float u1, V3 &wi) {
    LightEval e;
    V3 w;
    if (sc.env_emission_tex == 0u) {
        float z = 1.0f - 2.0f * u0;// sample_uniform_sphere, sampling.cpp:100-108
        float r = sqrtf(fmaxf(1.0f - z * z, 0.0f));
        float phi = 2.0f * kPi * u1;
        float sp, cp;
        sincosf(phi, &sp, &cp);
        w = v3(r * cp, r * sp, z);
        float theta = acosf(w.y), ph = atan2f(w.x, w.z);
        float u = 1.f - 0.5f * kInvPi * ph, v = theta * kInvPi;
        e.L = env_radiance(sc, u - floorf(u), v - floorf(v));
        e.pdf = kInvPi * 0.25f;
    } else {
        const uint32_t W = sc.env_map_width, H = sc.env_map_height;
        uint32_t iy, ix;
        float uy, ux;
        sample_alias(sc.env_alias, H, u1, iy, uy);
        sample_alias(sc.env_alias + static_cast<size_t>(H) + static_cast<size_t>(iy) * W, W, u0, ix, ux);
        float u = (static_cast<float>(ix) + ux) / static_cast<float>(W), v = (static_cast<float>(iy) + uy) / static_cast<float>(H);
        float p = __ldg(sc.env_pdf + static_cast<size_t>(iy) * W + ix);
        float phi = 2.f * kPi * (1.f - u), theta = kPi * v;// uv_to_direction, :42-51
        float sphi, cphi, sth, cth;
        sincosf(phi, &sphi, &cphi);
        sincosf(theta, &sth, &cth);
        w = normalize(v3(sphi * sth, cth, cphi * sth));
        e.L = env_radiance(sc, u, v);
        e.pdf = env_directional_pdf(p, theta);
    }
    wi = normalize(env_mul(sc.env_to_world, w, false));
    return e;
}

// Geometry::_alpha_skip (src/base/geometry.cpp:165-192): whether a traversal candidate (instance, primitive, barycentrics of
// the triangle test) is stochastically transparent.  The random number is a hash of the hit, so the decision is the same
// in every traversal that meets this candidate.
__device__ __noinline__ inline bool alpha_skip(const DeviceScene &sc, uint32_t inst_id, uint32_t prim_id, float bu, float bv) {
    const ShapeHandle shape = decode_handle(__ldg(sc.inst_handles + inst_id));
    if (!((shape.flags & LRK_SHAPE_MAYBE_NON_OPAQUE) && shape.has_surface())) return false;
    const lrk_surface *surf = sc.surfaces + shape.surface_tag;
    if (!(surf->flags & LRK_SURFACE_MAYBE_NON_OPAQUE)) return false;// evaluate_opacity -> nullopt (surface.h:186)
    const float u = static_cast<float>(xxhash32_uint4(inst_id, prim_id, __float_as_uint(bu), __float_as_uint(bv))) * 0x1p-32f;
    float alpha = surf->opacity;
    if (surf->opacity_tex != 0u) {
        const lrk_mesh mesh = sc.meshes[shape.mesh];
        const lrk_triangle tri = sc.triangles[mesh.triangle_offset + prim_id];
        const float4 *vb = reinterpret_cast<const float4 *>(sc.vertices + mesh.vertex_offset);
        float4 a1 = __ldg(vb + tri.i0 * 2u + 1u), b1 = __ldg(vb + tri.i1 * 2u + 1u), c1 = __ldg(vb + tri.i2 * 2u + 1u);
        const float b0 = 1.f - bu - bv;
        float tu = b0 * a1.z + bu * b1.z + bv * c1.z, tv = b0 * a1.w + bu * b1.w + bv * c1.w;// geometry.cpp:372
        alpha = texture_evaluate(*sc.self, surf->opacity_tex - 1u, tu, tv).x;
    }
    return u > alpha;
}

// clamp_shading_normal, src/util/frame.cpp:49-54
__device__ __forceinline__ V3 clamp_shading_normal(V3 ns, V3 ng, V3 w) {
    V3 w_refl = reflect(-w, ns);
    V3 w_refl_clip = dot(w_refl, ng) * dot(w, ng) > 0.f ? w_refl : normalize(w_refl - ng * dot(w_refl, ng));
    return normalize(w_refl_clip + w);
}
// NormalMapWrapper::populate_closure, src/base/surface.h:236-253: the shading frame the closure sees
__device__ __forceinline__ Frame normal_mapped_frame(const DeviceScene &sc, const lrk_surface *surf, const Interaction &it, V3 wo) {
    V3 rgb = v3(surf->normal_value[0], surf->normal_value[1], surf->normal_value[2]);
    if (surf->normal_tex != 0u) {
        float4 t = texture_evaluate(*sc.self, surf->normal_tex - 1u, it.u, it.v);
        rgb = v3(t.x, t.y, t.z);
    }
    V3 nl = 2.f * rgb + (-1.f);
    if (surf->normal_strength != 1.f) nl = nl * v3(surf->normal_strength, surf->normal_strength, 1.f);
    V3 normal = it.shading.local_to_world(nl);
    return Frame::make(clamp_shading_normal(normal, it.ng, wo), it.shading.s);
}

// ---- surfaces ------------------------------------------------------------------------------------------
struct SurfEval {
    V3 f;
    float pdf;
};

// src/base/surface.cpp:35-43
__device__ __forceinline__ bool validate_surface_sides(V3 ng, V3 ns, V3 wo, V3 wi) {
    float flip = sign(dot(ng, ns));
    return sign(flip * dot(wo, ns)) == sign(dot(wo, ng)) && sign(flip * dot(wi, ns)) == sign(dot(wi, ng));
}
__device__ __forceinline__ float lambert_pdf(V3 wo, V3 wi) { return same_hemisphere(wo, wi) ? abs_cos_theta(wi) * kInvPi : 0.f; }

// Matte / Oren-Nayar: src/surfaces/matte.cpp:78-134, src/util/scattering.cpp:247-264,370-400
struct MatteClosure {
    V3 r;
    float a, b;
    __device__ __forceinline__ void init(const lrk_surface &s) {
        r = v3(s.p[0], s.p[1], s.p[2]);
        float sigma2 = sqr(s.p[3] * (kPi / 180.0f));
        a = 1.f - (sigma2 / (2.f * sigma2 + 0.66f));
        b = 0.45f * sigma2 / (sigma2 + 0.09f);
    }
    __device__ __forceinline__ void prepare(V3) {}
    __device__ __forceinline__ V3 oren_nayar(V3 wo, V3 wi) const {
        float s = same_hemisphere(wo, wi) ? kInvPi : 0.f;
        float sinThetaI = sin_theta(wi), sinThetaO = sin_theta(wo);
        float sinPhiI = sin_phi(wi), cosPhiI = cos_phi(wi);
        float sinPhiO = sin_phi(wo), cosPhiO = cos_phi(wo);
        float dCos = cosPhiI * cosPhiO + sinPhiI * sinPhiO;
        float maxCos = (sinThetaI > 1e-4f && sinThetaO > 1e-4f) ? fmaxf(0.f, dCos) : 0.f;
        float absCosThetaI = abs_cos_theta(wi), absCosThetaO = abs_cos_theta(wo);
        float sinAlpha = absCosThetaI > absCosThetaO ? sinThetaO : sinThetaI;
        float tanBeta = absCosThetaI > absCosThetaO ? sinThetaI / absCosThetaI : sinThetaO / absCosThetaO;
        float scale = a + b * maxCos * sinAlpha * tanBeta;
        return s * scale * r;
    }
    __device__ __forceinline__ SurfEval evaluate_local(V3 wo, V3 wi) const {
        SurfEval e;
        e.f = oren_nayar(wo, wi) * abs_cos_theta(wi);
        e.pdf = lambert_pdf(wo, wi);
        return e;
    }
    // matte.cpp:118-134: cosine-hemisphere direction on wo's side; the sample's f and pdf are evaluate_local at that direction
    __device__ __forceinline__ bool sample_direction(V3 wo, float, float u0, float u1, V3 &wi) const {
        wi = sample_cosine_hemisphere(u0, u1);
        wi.z *= sign(cos_theta(wo));
        return true;
    }
};

// microfacet machinery: src/util/scattering.cpp:30-52,117-237
__device__ __forceinline__ float fresnel_dielectric(float cosThetaI_in, float etaI_in, float etaT_in) {
    float cosThetaI = clampf(cosThetaI_in, -1.f, 1.f);
    bool entering = cosThetaI > 0.f;
    float etaI = entering ? etaI_in : etaT_in;
    float etaT = entering ? etaT_in : etaI_in;
    cosThetaI = fabsf(cosThetaI);
    float sinThetaI = sqrtf(fmaxf(0.f, 1.f - sqr(cosThetaI)));
    float sinThetaT = etaI / etaT * sinThetaI;
    float cosThetaT = sqrtf(fmaxf(0.f, 1.f - sqr(sinThetaT)));
    float Rparl = (etaT * cosThetaI - etaI * cosThetaT) / (etaT * cosThetaI + etaI * cosThetaT);
    float Rperp = (etaI * cosThetaI - etaT * cosThetaT) / (etaI * cosThetaI + etaT * cosThetaT);
    float fr = (Rparl * Rparl + Rperp * Rperp) * .5f;
    return sinThetaT < 1.f ? fr : 1.f;
}

struct TrowbridgeReitz {
    float ax, ay;
    __device__ __forceinline__ float D(V3 wh) const {
        float tan2Theta = tan2_theta(wh);
        float cos4Theta = sqr(cos2_theta(wh));
        float e = tan2Theta * (sqr(cos_phi(wh) / ax) + sqr(sin_phi(wh) / ay));
        float d = 1.0f / (kPi * ax * ay * cos4Theta * sqr(1.f + e));
        return isinf(tan2Theta) ? 0.f : d;
    }
    __device__ __forceinline__ float Lambda(V3 w) const {
        float tanTheta = fabsf(tan_theta(w));
        float alpha2 = cos2_phi(w) * sqr(ax) + sin2_phi(w) * sqr(ay);
        float alpha2Tan2Theta = alpha2 * sqr(tanTheta);
        float L = (-1.f + sqrtf(1.f + alpha2Tan2Theta)) * .5f;
        return isinf(tanTheta) ? 0.f : L;
    }
    __device__ __forceinline__ float G1(V3 w) const { return 1.0f / (1.0f + Lambda(w)); }
    __device__ __forceinline__ float G(V3 wo, V3 wi) const { return 1.0f / (1.0f + Lambda(wo) + Lambda(wi)); }
    __device__ __forceinline__ float pdf(V3 wo, V3 wh) const { return D(wh) * G1(wo) * abs_dot(wo, wh) / abs_cos_theta(wo); }
    __device__ __forceinline__ static void sample11(float cosTheta, float U1, float U2, float &slope_x, float &slope_y) {
        if (cosTheta <= .9999f) {
            float sinTheta = sqrtf(fmaxf(0.f, 1.f - sqr(cosTheta)));
            float tanTheta = sinTheta / cosTheta;
            float a = 1.f / tanTheta;
            float G1 = 2.f / (1.f + sqrtf(1.f + 1.f / sqr(a)));
            float A = 2.f * U1 / G1 - 1.f;
            float tmp = fminf(1.f / (sqr(A) - 1.f), 1e10f);
            float B = tanTheta;
            float D = sqrtf(fmaxf(sqr(B * tmp) - (sqr(A) - sqr(B)) * tmp, 0.f));
            float slope_x_1 = B * tmp - D;
            float slope_x_2 = B * tmp + D;
            slope_x = (A < 0.f || slope_x_2 * tanTheta > 1.f) ? slope_x_1 : slope_x_2;
            float S = U2 > .5f ? 1.f : -1.f;
            float V = U2 > .5f ? 2.f * (U2 - .5f) : 2.f * (.5f - U2);
            float z = (V * (V * (V * 0.27385f - 0.73369f) + 0.46341f)) /
                      (V * (V * (V * 0.093073f + 0.309420f) - 1.000000f) + 0.597999f);
            slope_y = S * z * sqrtf(1.f + sqr(slope_x));
        } else {
            float r = sqrtf(U1 / (1.f - U1));
            float phi = (2.f * kPi) * U2;
            float s, c;
            sincosf(phi, &s, &c);
            slope_x = r * c;
            slope_y = r * s;
        }
    }
    __device__ __forceinline__ V3 sample_wh(V3 wo, float u0, float u1) const {
        float s = sign(cos_theta(wo));
        V3 wi = s * wo;
        V3 wiStretched = normalize(v3(ax * wi.x, ay * wi.y, wi.z));
        float sx, sy;
        sample11(cos_theta(wiStretched), u0, u1, sx, sy);
        float cp = cos_phi(wiStretched), sp = sin_phi(wiStretched);
        float rx = cp * sx - sp * sy;
        float ry = sp * sx + cp * sy;
        rx = ax * rx;
        ry = ay * ry;
        V3 wh = normalize(v3(-rx, -ry, 1.f));
        return s * wh;
    }
};

// Disney: src/surfaces/disney.cpp:95-303 (lobes), :376-478 (closure set-up), :481-587 (evaluate / sample)
__device__ __forceinline__ float SchlickWeight(float cosTheta) {
    float m = saturate(1.f - cosTheta);
    return sqr(sqr(m)) * m;
}
__device__ __forceinline__ float FrSchlick(float R0, float cosTheta) { return lerp(R0, 1.f, SchlickWeight(cosTheta)); }
__device__ __forceinline__ float GTR1(float cosTheta, float alpha) {
    float alpha2 = sqr(alpha);
    float denom = kPi * logf(alpha2) * (1.f + (alpha2 - 1.f) * sqr(cosTheta));
    return (alpha2 - 1.f) / denom;
}
__device__ __forceinline__ float smithG_GGX(float cosTheta, float alpha) {
    float alpha2 = sqr(alpha);
    float cosTheta2 = sqr(cosTheta);
    return 1.f / (cosTheta + sqrtf(alpha2 + cosTheta2 - alpha2 * cosTheta2));
}

// MicrofacetTransmission (src/util/scattering.cpp:326-373) with eta_a = 1, as free functions over (t, distribution, eta_b):
// the Glass closure below and the transmissive Disney closure share them.
__device__ __forceinline__ bool refract(V3 wi, V3 n, float eta, V3 &wt);
__device__ __forceinline__ V3 microfacet_transmission_evaluate(V3 t, const TrowbridgeReitz &d, float eta, V3 wo, V3 wi) {
    float cosThetaO = cos_theta(wo), cosThetaI = cos_theta(wi);
    float e = cosThetaO > 0.f ? eta / 1.f : 1.f / eta;
    V3 wh = normalize(wo + wi * e);
    wh = sign(cos_theta(wh)) * wh;
    V3 f = v3(0.f);
    if (!same_hemisphere(wo, wi) && cosThetaO != 0.f && cosThetaI != 0.f && dot(wo, wh) * dot(wi, wh) < 0.f) {
        float G = d.G(wo, wi);
        float sqrtDenom = dot(wo, wh) + e * dot(wi, wh);
        float F = fresnel_dielectric(dot(wo, wh), 1.f, eta);
        float D = d.D(wh);
        V3 num = (1.f - F) * t * D * G * dot(wi, wh) * dot(wo, wh);
        float den = cosThetaI * cosThetaO * sqr(sqrtDenom);
        f = v3(num.x / den, num.y / den, num.z / den);
    }
    return f;
}
__device__ __forceinline__ float microfacet_transmission_pdf(const TrowbridgeReitz &d, float eta, V3 wo, V3 wi) {
    float p = 0.f;
    float e = cos_theta(wo) > 0.f ? eta / 1.f : 1.f / eta;
    V3 wh = normalize(wo + wi * e);
    if (!same_hemisphere(wo, wi) && dot(wo, wh) * dot(wi, wh) < 0.f) {
        float sqrtDenom = dot(wo, wh) + e * dot(wi, wh);
        float dwh_dwi = sqr(e / sqrtDenom) * abs_dot(wi, wh);
        p = d.pdf(wo, wh) * dwh_dwi;
    }
    return p;
}

// TRANS: the closure class "disney_trans" of a transmissive node (LRK_SURFACE_DISNEY_TRANSMISSIVE, src/surfaces/disney.cpp:376-383,
// 425,452-464,514-522,571-576): a fourth technique with a MicrofacetTransmission lobe, a one-sided Fresnel term, eta() = eta_t.
// THIN: the closure class "disney_thin" (LRK_SURFACE_DISNEY_THIN, ThinDisneyClosureImpl disney.cpp:590-845): the diffuse-like lobes
// keep (1 - diffuse_trans) of the diffuse weight, the transmission lobe runs through a rescaled distribution with the colour itself,
// a fifth technique is Lambertian diffuse transmission; both transmissions are "through" events (no medium change, no eta).
enum DisneyMode : int { kDisneyOpaque = 0, kDisneyTransmissive = 1, kDisneyThin = 2 };
template<int MODE>
struct DisneyClosureT {
    static constexpr bool TRANS = MODE == kDisneyTransmissive;
    static constexpr bool THIN = MODE == kDisneyThin;
    V3 Cdiff, Css, Csheen, Cspec0;
    float metallic, roughness, clearcoat, fresnel_eta, gloss;
    TrowbridgeReitz distrib;
    float w0, w1, w2;
    bool has_diffuse, has_fake_ss, has_sheen, has_clearcoat;
    // transmissive and thin closures only
    V3 Cst;
    float w3, eta_t_;
    bool has_spec_trans;
    // thin closure only
    TrowbridgeReitz thin_distrib;
    V3 Cdt;
    float w4;
    bool has_diff_trans;
    float rr_eta_scale;// eta scale of the sampled event for Russian roulette (mega_path.cpp:133-138)
    uint32_t event;    // Surface::event_* of the sampled direction (what the volume integrator's medium tracker follows)

    __device__ __forceinline__ void init(const lrk_surface &s) {
        rr_eta_scale = 1.f;
        event = LRK_EVENT_REFLECT;
        Cst = v3(0.f);
        w3 = 0.f;
        has_spec_trans = false;
        Cdt = v3(0.f);
        w4 = 0.f;
        has_diff_trans = false;
        eta_t_ = s.p[5];
        V3 color = v3(s.p[0], s.p[1], s.p[2]);
        float color_lum = s.p[3];
        metallic = s.p[4];
        float eta_t = s.p[5];
        roughness = s.p[6];
        float specular_tint = s.p[7], anisotropic = s.p[8], sheen = s.p[9], sheen_tint = s.p[10];
        clearcoat = s.p[11];
        float clearcoat_gloss = s.p[12], specular_trans = s.p[13], flatness = s.p[14];
        uint32_t lobes = s.lobes;
        has_diffuse = has_fake_ss = has_sheen = has_clearcoat = false;
        Cdiff = Css = Csheen = v3(0.f);
        w0 = w1 = w2 = 0.f;
        gloss = 0.f;
        bool en0 = false, en2 = false;
        float diffuse_weight = (1.f - metallic) * (1.f - specular_trans);
        float tint_weight = color_lum > 0.f ? 1.f / color_lum : 1.f;
        V3 tc = color * tint_weight;
        V3 tint = v3(saturate(tc.x), saturate(tc.y), saturate(tc.z));
        float tint_lum = color_lum * tint_weight;
        const float diffuse_trans = THIN ? s.p[15] : 0.f;
        const float diff_refl_weight = THIN ? diffuse_weight * (1.f - diffuse_trans) : diffuse_weight;// disney.cpp:620-622
        float diffuse_like_sampling_weight = diff_refl_weight * color_lum;
        if ((lobes & LRK_DISNEY_LOBE_DIFFUSE) || (lobes & LRK_DISNEY_LOBE_RETRO)) {
            float Cdiff_weight = diff_refl_weight * (1.f - flatness);
            Cdiff = color * Cdiff_weight;
            has_diffuse = true;
            en0 = true;
        }
        if (lobes & LRK_DISNEY_LOBE_FAKE_SS) {
            float Css_weight = THIN ? diff_refl_weight * flatness * (1.f - diffuse_trans) : diffuse_weight * flatness;// :643
            Css = Css_weight * color;
            has_fake_ss = true;
            en0 = true;
        }
        if (lobes & LRK_DISNEY_LOBE_SHEEN) {
            float Csheen_weight = THIN ? diff_refl_weight * sheen * (1.f - diffuse_trans) : diffuse_weight * sheen;// :651
            Csheen = Csheen_weight * lerp(v3(1.f), tint, sheen_tint);
            has_sheen = true;
            float sheen_lum = Csheen_weight * lerp(1.f, tint_lum, sheen_tint);
            diffuse_like_sampling_weight += sheen_lum * .1f;
            if (!THIN) en0 = true;// the thin closure's sheen block does not enable the technique (:650-657)
        }
        w0 = saturate(diffuse_like_sampling_weight);
        float eta = eta_t / 1.f;
        float SchlickR0 = sqr((eta - 1.f) / (eta + 1.f));
        Cspec0 = lerp(lerp(v3(1.f), tint, specular_tint) * SchlickR0, color, metallic);
        fresnel_eta = eta;
        float aspect = sqrtf(1.f - anisotropic * .9f);
        distrib.ax = fmaxf(fmaxf(0.001f, roughness / aspect), 1e-4f);
        distrib.ay = fmaxf(fmaxf(0.001f, roughness * aspect), 1e-4f);
        float Cspec0_lum = lerp(lerp(1.f, tint_lum, specular_tint) * SchlickR0, color_lum, metallic);
        w1 = saturate(Cspec0_lum);
        if (lobes & LRK_DISNEY_LOBE_CLEARCOAT) {
            gloss = lerp(.1f, .001f, clearcoat_gloss);
            has_clearcoat = true;
            w2 = saturate(clearcoat * FrSchlick(.04f, 1.f));
            en2 = true;
        }
        if (TRANS && (lobes & LRK_DISNEY_LOBE_SPEC_TRANS)) {
            float Cst_weight = (1.f - metallic) * specular_trans;
            Cst = Cst_weight * v3(sqrtf(color.x), sqrtf(color.y), sqrtf(color.z));
            has_spec_trans = true;
            float Cst_lum = Cst_weight * sqrtf(color_lum);
            w3 = saturate(Cst_lum);
        }
        if (THIN && (lobes & LRK_DISNEY_LOBE_SPEC_TRANS)) {// disney.cpp:686-701
            float rscaled = (.65f * eta - .35f) * roughness;
            thin_distrib.ax = fmaxf(fmaxf(.001f, rscaled / aspect), 1e-4f);
            thin_distrib.ay = fmaxf(fmaxf(.001f, rscaled * aspect), 1e-4f);
            float Cst_weight = (1.f - metallic) * specular_trans;
            Cst = Cst_weight * color;
            has_spec_trans = true;
            float Cst_lum = Cst_weight * color_lum;
            w3 = saturate(Cst_lum);
        }
        if (THIN && (lobes & LRK_DISNEY_LOBE_DIFF_TRANS)) {// disney.cpp:703-710
            float diff_trans_weight = diffuse_weight * diffuse_trans;
            Cdt = diff_trans_weight * color;
            float Cdt_lum = diff_trans_weight * color_lum;
            has_diff_trans = true;
            w4 = saturate(Cdt_lum);
        }
        float sum_weights = 0.f;
        if (en0) sum_weights += w0;
        sum_weights += w1;
        if (en2) sum_weights += w2;
        if ((TRANS || THIN) && has_spec_trans) sum_weights += w3;
        if (THIN && has_diff_trans) sum_weights += w4;
        float inv_sum_weights = sum_weights == 0.f ? 0.f : 1.f / sum_weights;
        if (en0) w0 *= inv_sum_weights;
        w1 *= inv_sum_weights;
        if (en2) w2 *= inv_sum_weights;
        if ((TRANS || THIN) && has_spec_trans) w3 *= inv_sum_weights;
        if (THIN && has_diff_trans) w4 *= inv_sum_weights;
        enabled0 = en0;
        enabled2 = en2;
    }
    bool enabled0, enabled2;
    // values that depend on wo (or on constants) only, shared by the light-direction and the sampled-direction
    // evaluations of one shading point; every one is the same expression the per-lobe formulas contain
    // (disney.cpp:95-303), hoisted — not re-associated — so results stay bit-identical to the oracle.
    float lambda_o, g1_o, schlick_o, ggx_o, gtr1_a2m1, gtr1_pi_log_a2;

    __device__ __forceinline__ void prepare(V3 wo) {
        lambda_o = distrib.Lambda(wo);
        g1_o = 1.0f / (1.0f + lambda_o);
        schlick_o = SchlickWeight(abs_cos_theta(wo));
        ggx_o = smithG_GGX(abs_cos_theta(wo), .25f);
        float alpha2 = sqr(gloss);
        gtr1_a2m1 = alpha2 - 1.f;
        gtr1_pi_log_a2 = kPi * logf(alpha2);
    }
    __device__ __forceinline__ V3 disney_fresnel(float cosI_in) const {
        float cosI = (TRANS || THIN) ? cosI_in : fabsf(cosI_in);// DisneyFresnel: two_sided = !is_transmissive, false when thin (disney.cpp:287-292,425,666)
        float fr = fresnel_dielectric(cosI, 1.f, fresnel_eta);
        V3 f0 = v3(FrSchlick(Cspec0.x, cosI), FrSchlick(Cspec0.y, cosI), FrSchlick(Cspec0.z, cosI));
        return lerp(v3(fr), f0, metallic);
    }
    __device__ __forceinline__ SurfEval evaluate_local(V3 wo, V3 wi) const {
        V3 f = v3(0.f);
        float pdf = 0.f;
        if (same_hemisphere(wo, wi)) {
            // the half vector every lobe uses (DisneyRetro/FakeSS/Sheen :118-190, MicrofacetReflection scattering.cpp:286-320,
            // DisneyClearcoat :215-260)
            V3 whs = wi + wo;
            bool valid = any_nonzero(whs);
            V3 wh = normalize(whs);
            float cosThetaD = dot(wi, wh);
            float wo_dot_wh = dot(wo, wh);
            if (has_diffuse) {
                if (w0 > 0.f) {
                    float Fo = schlick_o, Fi = SchlickWeight(abs_cos_theta(wi));
                    f = f + Cdiff * (kInvPi * (1.f - Fo * .5f) * (1.f - Fi * .5f));
                    {// DisneyRetro
                        float Rr = 2.f * roughness * cosThetaD * cosThetaD;
                        f = f + Cdiff * (valid ? kInvPi * Rr * (Fo + Fi + Fo * Fi * (Rr - 1.f)) : 0.f);
                    }
                    if (has_fake_ss) {
                        float Fss90 = cosThetaD * cosThetaD * roughness;
                        float Fss = lerp(1.0f, Fss90, Fo) * lerp(1.0f, Fss90, Fi);
                        float ss = 1.25f * (Fss * (1.f / (abs_cos_theta(wo) + abs_cos_theta(wi)) - .5f) + .5f);
                        f = f + Css * (valid ? kInvPi * ss : 0.f);
                    }
                    if (has_sheen) f = f + Csheen * (valid ? SchlickWeight(cosThetaD) : 0.f);
                    pdf += w0 * lambert_pdf(wo, wi);
                }
            }
            if (w1 > 0.f) {
                V3 fs = v3(0.f);
                float ps = 0.f;
                if (valid) {
                    // dot(wi, face_forward(wh, +z)) = +-dot(wi, wh); the opaque closure's Fresnel term takes its absolute value
                    V3 F = disney_fresnel((TRANS || THIN) ? (cos_theta(wh) < 0.f ? -cosThetaD : cosThetaD) : cosThetaD);
                    float D = distrib.D(wh);
                    float G = 1.0f / (1.0f + lambda_o + distrib.Lambda(wi));
                    float cos_o = cos_theta(wo), cos_i = cos_theta(wi);
                    fs = v3(1.f) * F * fabsf(0.25f * D * G / (cos_i * cos_o));
                    ps = (D * g1_o * fabsf(wo_dot_wh) / abs_cos_theta(wo)) / (4.f * wo_dot_wh);
                }
                f = f + fs;
                pdf += w1 * ps;
            }
            if (has_clearcoat) {
                if (w2 > 0.f) {
                    float cos_h = abs_cos_theta(wh);
                    float Dr = gtr1_a2m1 / (gtr1_pi_log_a2 * (1.f + gtr1_a2m1 * sqr(cos_h)));
                    float Fr = FrSchlick(.04f, wo_dot_wh);
                    float Gr = ggx_o * smithG_GGX(abs_cos_theta(wi), .25f);
                    f = f + (valid ? clearcoat * Gr * Fr * Dr * .25f : 0.f);
                    pdf += w2 * (valid ? Dr * cos_h / (4.f * wo_dot_wh) : 0.f);
                }
            }
        } else if (TRANS && has_spec_trans) {// transmission, disney.cpp:514-522
            if (w3 > 0.f) {
                f = f + microfacet_transmission_evaluate(Cst, distrib, eta_t_, wo, wi);
                pdf += w3 * microfacet_transmission_pdf(distrib, eta_t_, wo, wi);
            }
        } else if (THIN) {// disney.cpp:755-774
            if (has_spec_trans) {
                if (w3 > 0.f) {
                    f = f + microfacet_transmission_evaluate(Cst, thin_distrib, eta_t_, wo, wi);
                    pdf += w3 * microfacet_transmission_pdf(thin_distrib, eta_t_, wo, wi);
                }
            }
            if (has_diff_trans) {
                if (w4 > 0.f) {// LambertianTransmission (scattering.cpp:271-284): wo and wi lie in opposite hemispheres here
                    f = f + Cdt * kInvPi;
                    pdf += w4 * (abs_cos_theta(wi) * kInvPi);
                }
            }
        }
        SurfEval e;
        e.f = f * abs_cos_theta(wi);
        e.pdf = pdf;
        return e;
    }
    __device__ __forceinline__ bool sample_direction(V3 wo, float u_lobe, float u0, float u1, V3 &wi) {
        // technique selection: src/surfaces/disney.cpp:544-551 (strict '>' against the running sum)
        uint32_t tech = 0u;
        float sum_weights = 0.f;
        if (enabled0) {
            tech = u_lobe > sum_weights ? 0u : tech;
            sum_weights += w0;
        }
        tech = u_lobe > sum_weights ? 1u : tech;
        sum_weights += w1;
        if (enabled2) {
            tech = u_lobe > sum_weights ? 2u : tech;
            sum_weights += w2;
        }
        if ((TRANS || THIN) && has_spec_trans) {
            tech = u_lobe > sum_weights ? 3u : tech;
            sum_weights += w3;
        }
        if (THIN && has_diff_trans) {
            tech = u_lobe > sum_weights ? 4u : tech;
            sum_weights += w4;
        }
        wi = v3(0.f);
        bool valid = false;
        rr_eta_scale = 1.f;
        event = LRK_EVENT_REFLECT;
        if (TRANS && tech == 3u) {// MicrofacetTransmission::sample_wi (scattering.cpp:352-358), event enter / exit (disney.cpp:571-576)
            float e = cos_theta(wo) > 0.f ? 1.f / eta_t_ : eta_t_ / 1.f;
            V3 wh = distrib.sample_wh(wo, u0, u1);
            bool refr = refract(wo, wh, e, wi);
            valid = refr && !same_hemisphere(wo, wi);
            rr_eta_scale = cos_theta(wo) > 0.f ? sqr(eta_t_) : sqr(1.f / eta_t_);
            event = cos_theta(wo) > 0.f ? LRK_EVENT_ENTER : LRK_EVENT_EXIT;
        } else if (THIN && tech == 3u) {// the same lobe through the rescaled distribution; a "through" event (disney.cpp:820-825)
            float e = cos_theta(wo) > 0.f ? 1.f / eta_t_ : eta_t_ / 1.f;
            V3 wh = thin_distrib.sample_wh(wo, u0, u1);
            bool refr = refract(wo, wh, e, wi);
            valid = refr && !same_hemisphere(wo, wi);
            event = LRK_EVENT_THROUGH;
        } else if (THIN && tech == 4u) {// LambertianTransmission::sample_wi (scattering.cpp:276-280, disney.cpp:827-832)
            wi = sample_cosine_hemisphere(u0, u1);
            wi.z *= -sign(cos_theta(wo));
            valid = true;
            event = LRK_EVENT_THROUGH;
        } else if (tech == 0u) {
            if (has_diffuse) {
                wi = sample_cosine_hemisphere(u0, u1);
                wi.z *= sign(cos_theta(wo));
                valid = true;
            }
        } else if (tech == 1u) {
            V3 wh = distrib.sample_wh(wo, u0, u1);
            wi = reflect(-wo, wh);
            valid = same_hemisphere(wo, wi);
        } else {
            if (has_clearcoat) {
                float alpha2 = gloss * gloss;
                // builtin_pow(alpha2, 1 - u0) with the exponent in (0, 1]: the whole-number case is u0 == 0 only, x^1 = x
                // (the general builtin_pow here made the Disney kernel measurably slower)
                const float e = 1.f - u0;
                const float p = e == 1.f ? alpha2 : powf(alpha2, e);
                float cosTheta = sqrtf(fmaxf(0.f, (1.f - p) / (1.f - alpha2)));
                float sinTheta = sqrtf(fmaxf(0.f, 1.f - cosTheta * cosTheta));
                float phi = 2.f * kPi * u1;
                float s, c;
                sincosf(phi, &s, &c);
                V3 wh = v3(sinTheta * c, sinTheta * s, cosTheta);
                wh = same_hemisphere(wo, wh) ? wh : -wh;
                wi = reflect(-wo, wh);
                valid = same_hemisphere(wo, wi);
            }
        }
        return valid;// f and pdf of the sample are evaluate_local(wo, wi) (disney.cpp:583-586)
    }
};
using DisneyClosure = DisneyClosureT<kDisneyOpaque>;
using DisneyTransClosure = DisneyClosureT<kDisneyTransmissive>;
using DisneyThinClosure = DisneyClosureT<kDisneyThin>;

// Mirror / Glass / Plastic / Metal (SURVEY.md §8 row f3): src/surfaces/{mirror,glass,plastic,metal}.cpp over the BxDFs of
// src/util/scattering.cpp:14-125,238-345.  One closure type for the four nodes (hit bucket 3): they are rare next to the
// Matte / Disney buckets and share the microfacet code.  lrk_surface.p holds each node's closure Context (include/lrk.h).
// The expressions are the oracle's (oracle/oracle.cpp: MicrofacetReflection, MicrofacetTransmission, PlasticLobes, ...),
// which are pinned bit for bit against the reference's closures (tests/test_ref_pins.py, tests/test_ref_render.py).
__device__ __forceinline__ bool refract(V3 wi, V3 n, float eta, V3 &wt) {// scattering.cpp:14-28
    float cosThetaI = dot(n, wi);
    float sin2ThetaI = fmaxf(0.0f, 1.f - sqr(cosThetaI));
    float sin2ThetaT = sqr(eta) * sin2ThetaI;
    float cosThetaT = sqrtf(1.f - sin2ThetaT);
    wt = (eta * cosThetaI - cosThetaT) * n - eta * wi;
    return sin2ThetaT < 1.0f;
}
__device__ __forceinline__ V3 vdiv(V3 a, V3 b) { return v3(a.x / b.x, a.y / b.y, a.z / b.z); }
__device__ __forceinline__ V3 vsqrt(V3 a) { return v3(sqrtf(a.x), sqrtf(a.y), sqrtf(a.z)); }
__device__ __forceinline__ V3 vsub(V3 a, float s) { return v3(a.x - s, a.y - s, a.z - s); }
__device__ __forceinline__ V3 vrsub(float s, V3 a) { return v3(s - a.x, s - a.y, s - a.z); }
__device__ __forceinline__ V3 fresnel_conductor(float cosThetaI, float etai, V3 etat, V3 k) {// scattering.cpp:56-75
    cosThetaI = clampf(cosThetaI, -1.f, 1.f);
    V3 eta = v3(etat.x / etai, etat.y / etai, etat.z / etai);
    V3 etak = v3(k.x / etai, k.y / etai, k.z / etai);
    float cosThetaI2 = cosThetaI * cosThetaI;
    float sinThetaI2 = 1.f - cosThetaI2;
    V3 eta2 = eta * eta;
    V3 etak2 = etak * etak;
    V3 t0 = vsub(eta2 - etak2, sinThetaI2);
    V3 a2plusb2 = vsqrt(t0 * t0 + 4.f * eta2 * etak2);
    V3 t1 = a2plusb2 + cosThetaI2;
    V3 a = vsqrt(.5f * (a2plusb2 + t0));
    V3 t2 = (2.f * cosThetaI) * a;
    V3 Rs = vdiv(t1 - t2, t1 + t2);
    V3 t3 = cosThetaI2 * a2plusb2 + sinThetaI2 * sinThetaI2;
    V3 t4 = t2 * sinThetaI2;
    V3 Rp = vdiv(Rs * (t3 - t4), t3 + t4);
    return .5f * (Rp + Rs);
}

// TYPE (LRK_SURFACE_MIRROR .. LRK_SURFACE_METAL) is a template parameter: each node type gets its own hit bucket and shade
// kernel instantiation (sorted-by-material dispatch), so a warp runs ONE closure's code - the first version switched on a
// run-time type inside one kernel and was instruction-fetch bound.
template<uint32_t TYPE>
struct MicrofacetFamilyClosure {
    static constexpr uint32_t type = TYPE;
    V3 c0, c1, c2;     // MIRROR: refl | GLASS: Kr, Kt | PLASTIC: Kd', sigma_a | METAL: n, k, tint
    float eta, w0;     // GLASS: eta_t, Kr_ratio | PLASTIC: eta, Kd_weight
    TrowbridgeReitz d;
    float flip;        // PLASTIC: sign applied to the z components (plastic.cpp:143-147)
    float rr_eta_scale;// eta scale of the sampled event for Russian roulette (mega_path.cpp:133-138)
    uint32_t event;    // Surface::event_* of the sampled direction
    bool importance;   // TransportMode::IMPORTANCE: the transmission lobe is scaled by eta^2 (scattering.cpp:340-342); Layered only
    __device__ __forceinline__ void init(const lrk_surface &s) {
        rr_eta_scale = 1.f;
        event = LRK_EVENT_REFLECT;
        importance = false;
        flip = 1.f;
        eta = 1.5f;
        w0 = 0.f;
        c0 = v3(s.p[0], s.p[1], s.p[2]);
        c1 = c2 = v3(0.f);
        float ax = 0.f, ay = 0.f;
        if (type == LRK_SURFACE_MIRROR) {
            ax = s.p[3]; ay = s.p[4];
        } else if (type == LRK_SURFACE_GLASS) {
            c1 = v3(s.p[3], s.p[4], s.p[5]);
            eta = s.p[6]; ax = s.p[7]; ay = s.p[8]; w0 = s.p[9];
        } else if (type == LRK_SURFACE_PLASTIC) {
            w0 = s.p[3];
            c1 = v3(s.p[4], s.p[5], s.p[6]);
            eta = s.p[7]; ax = s.p[8]; ay = s.p[9];
        } else {
            c1 = v3(s.p[3], s.p[4], s.p[5]);
            c2 = v3(s.p[6], s.p[7], s.p[8]);
            ax = s.p[9]; ay = s.p[10];
        }
        d.ax = fmaxf(ax, 1e-4f);// MicrofacetDistribution ctor, scattering.cpp:124-125
        d.ay = fmaxf(ay, 1e-4f);
    }
    __device__ __forceinline__ void prepare(V3 wo_local) { flip = (type == LRK_SURFACE_PLASTIC && cos_theta(wo_local) < 0.f) ? -1.f : 1.f; }

    // Fresnel term of the reflection lobe: Schlick around the colour (mirror.cpp:67-79), dielectric, conductor
    __device__ __forceinline__ V3 fresnel(float cosI) const {
        if (type == LRK_SURFACE_MIRROR) {
            float m = saturate(1.f - cosI);
            float weight = sqr(sqr(m)) * m;
            return (1.f - weight) * c0 + weight;
        }
        if (type == LRK_SURFACE_METAL) return fresnel_conductor(fabsf(cosI), 1.f, c0, c1);
        return v3(fresnel_dielectric(cosI, 1.f, eta));
    }
    __device__ __forceinline__ V3 reflection_evaluate(V3 r, V3 wo, V3 wi) const {// MicrofacetReflection::evaluate :290-308
        V3 wh = wi + wo;
        V3 f = v3(0.f);
        if (same_hemisphere(wo, wi) && any_nonzero(wh)) {
            wh = normalize(wh);
            V3 F = fresnel(dot(wi, face_forward(wh, v3(0.f, 0.f, 1.f))));
            float D = d.D(wh);
            float G = d.G(wo, wi);
            float cos_o = cos_theta(wo), cos_i = cos_theta(wi);
            f = r * F * fabsf(0.25f * D * G / (cos_i * cos_o));
        }
        return f;
    }
    __device__ __forceinline__ float reflection_pdf(V3 wo, V3 wi) const {// :316-324
        float p = 0.f;
        V3 wh = wi + wo;
        if (same_hemisphere(wo, wi) && any_nonzero(wh)) {
            wh = normalize(wh);
            p = d.pdf(wo, wh) / (4.f * dot(wo, wh));
        }
        return p;
    }
    __device__ __forceinline__ V3 transmission_evaluate(V3 wo, V3 wi) const {// MicrofacetTransmission::evaluate :326-350, eta_a = 1
        float cosThetaO = cos_theta(wo), cosThetaI = cos_theta(wi);
        float e = cosThetaO > 0.f ? eta / 1.f : 1.f / eta;
        V3 wh = normalize(wo + wi * e);
        wh = sign(cos_theta(wh)) * wh;
        V3 f = v3(0.f);
        if (!same_hemisphere(wo, wi) && cosThetaO != 0.f && cosThetaI != 0.f && dot(wo, wh) * dot(wi, wh) < 0.f) {
            float G = d.G(wo, wi);
            float sqrtDenom = dot(wo, wh) + e * dot(wi, wh);
            float F = fresnel_dielectric(dot(wo, wh), 1.f, eta);
            float D = d.D(wh);
            V3 num = (1.f - F) * c1 * D * G * dot(wi, wh) * dot(wo, wh);
            float den = cosThetaI * cosThetaO * sqr(sqrtDenom);
            f = v3(num.x / den, num.y / den, num.z / den);
            if (importance) f = f * sqr(e);
        }
        return f;
    }
    __device__ __forceinline__ float transmission_pdf(V3 wo, V3 wi) const {// :360-373
        float p = 0.f;
        float e = cos_theta(wo) > 0.f ? eta / 1.f : 1.f / eta;
        V3 wh = normalize(wo + wi * e);
        if (!same_hemisphere(wo, wi) && dot(wo, wh) * dot(wi, wh) < 0.f) {
            float sqrtDenom = dot(wo, wh) + e * dot(wi, wh);
            float dwh_dwi = sqr(e / sqrtDenom) * abs_dot(wi, wh);
            p = d.pdf(wo, wh) * dwh_dwi;
        }
        return p;
    }
    __device__ __forceinline__ float glass_refl_prob(V3 wo) const {// glass.cpp:162-167
        float F = fresnel_dielectric(cos_theta(wo), 1.f, eta);
        float r = w0 * F;
        float t = (1.f - w0) * (1.f - F);
        return r == 0.f ? 0.f : r / (r + t);
    }
    __device__ __forceinline__ static float substrate_weight(float Fo, float kd_w) {// plastic.cpp:125-128
        float w = kd_w * (1.0f - Fo);
        return w == 0.f ? 0.f : w / (w + Fo);
    }

    __device__ __forceinline__ SurfEval evaluate_local(V3 wo, V3 wi) const {
        SurfEval e;
        if (type == LRK_SURFACE_MIRROR) {
            e.f = reflection_evaluate(c0, wo, wi) * abs_cos_theta(wi);
            e.pdf = reflection_pdf(wo, wi);
        } else if (type == LRK_SURFACE_METAL) {
            V3 f = reflection_evaluate(v3(1.f), wo, wi);
            f = f * c2;
            e.f = f * abs_cos_theta(wi);
            e.pdf = reflection_pdf(wo, wi);
        } else if (type == LRK_SURFACE_GLASS) {// glass.cpp:169-191
            float ratio = glass_refl_prob(wo);
            V3 f;
            float pdf;
            if (same_hemisphere(wo, wi)) {
                f = reflection_evaluate(c0, wo, wi);
                pdf = reflection_pdf(wo, wi) * ratio;
            } else {
                f = transmission_evaluate(wo, wi);
                pdf = transmission_pdf(wo, wi) * (1.f - ratio);
            }
            e.f = f * abs_cos_theta(wi);
            e.pdf = pdf;
        } else {// plastic.cpp:138-165
            V3 wo_l = v3(wo.x, wo.y, wo.z * flip), wi_l = v3(wi.x, wi.y, wi.z * flip);
            V3 f_coat = reflection_evaluate(v3(1.f), wo_l, wi_l);
            float pdf_coat = reflection_pdf(wo_l, wi_l);
            float Fi = fresnel_dielectric(abs_cos_theta(wi_l), 1.f, eta);
            float Fo = fresnel_dielectric(abs_cos_theta(wo_l), 1.f, eta);
            float ex = -(1.f / abs_cos_theta(wi_l) + 1.f / abs_cos_theta(wo_l));
            V3 a = v3(expf(ex * c1.x), expf(ex * c1.y), expf(ex * c1.z));
            V3 lam = c0 * (same_hemisphere(wo_l, wi_l) ? kInvPi : 0.f);
            V3 f_diffuse = (1.f - Fi) * (1.f - Fo) * sqr(1.f / eta) * a * lam;
            float pdf_diffuse = lambert_pdf(wo_l, wi_l);
            float sw = substrate_weight(Fo, w0);
            e.f = (f_coat + f_diffuse) * abs_cos_theta(wi_l);
            e.pdf = lerp(pdf_coat, pdf_diffuse, sw);
        }
        return e;
    }

    __device__ __forceinline__ bool sample_direction(V3 wo, float u_lobe, float u0, float u1, V3 &wi) {
        rr_eta_scale = 1.f;
        event = LRK_EVENT_REFLECT;
        if (type == LRK_SURFACE_MIRROR || type == LRK_SURFACE_METAL) {
            V3 wh = d.sample_wh(wo, u0, u1);
            wi = reflect(-wo, wh);
            return same_hemisphere(wo, wi);
        }
        if (type == LRK_SURFACE_GLASS) {// glass.cpp:193-221
            float ratio = glass_refl_prob(wo);
            if (u_lobe < ratio) {
                V3 wh = d.sample_wh(wo, u0, u1);
                wi = reflect(-wo, wh);
                return same_hemisphere(wo, wi);
            }
            float e = cos_theta(wo) > 0.f ? 1.f / eta : eta / 1.f;
            V3 wh = d.sample_wh(wo, u0, u1);
            wi = v3(0.f);
            bool refr = refract(wo, wh, e, wi);
            rr_eta_scale = cos_theta(wo) > 0.f ? sqr(eta) : sqr(1.f / eta);// event_enter / event_exit
            event = cos_theta(wo) > 0.f ? LRK_EVENT_ENTER : LRK_EVENT_EXIT;
            return refr && !same_hemisphere(wo, wi);
        }
        // plastic.cpp:168-214: sampled above the flipped surface, returned in the original frame
        V3 wo_l = v3(wo.x, wo.y, wo.z * flip);
        float Fo = fresnel_dielectric(abs_cos_theta(wo_l), 1.f, eta);
        float sw = substrate_weight(Fo, w0);
        V3 w;
        bool valid;
        if (u_lobe < sw) {
            w = sample_cosine_hemisphere(u0, u1);
            w.z *= sign(cos_theta(wo_l));
            valid = true;
        } else {
            V3 wh = d.sample_wh(wo_l, u0, u1);
            w = reflect(-wo_l, wh);
            valid = same_hemisphere(wo_l, w);
        }
        wi = valid ? v3(w.x, w.y, w.z * flip) : v3(0.f, 0.f, 1.f);
        return valid;
    }
};

// Mix (src/surfaces/mix.cpp:82-193): two constant, non-Disney surface records blended by a ratio; hit bucket 7.
// The children are evaluated through out-of-line dispatchers (ONE copy of each closure's code in the kernel, called two or
// three times per shaded hit): a Mix is rare, and inlining every closure several times is what made the first row-f3 kernel
// instruction-fetch bound.  Expressions and quirks are the oracle's mix_evaluate / mix_sample, bit-identical to the reference
// render (tests/test_ref_render.py::materials_mix).
template<typename Closure>
__device__ __forceinline__ SurfEval child_evaluate(const lrk_surface *s, V3 wo, V3 wi) {
    Closure c;
    c.init(*s);
    c.prepare(wo);
    return c.evaluate_local(wo, wi);
}
// `importance`: TransportMode::IMPORTANCE, which only the Glass transmission lobe looks at (the Layered surface asks for it)
__device__ __noinline__ inline SurfEval any_evaluate_local(const lrk_surface *s, V3 wo, V3 wi, bool importance = false) {
    switch (s->type) {
        case LRK_SURFACE_MATTE: return child_evaluate<MatteClosure>(s, wo, wi);
        case LRK_SURFACE_MIRROR: return child_evaluate<MicrofacetFamilyClosure<LRK_SURFACE_MIRROR>>(s, wo, wi);
        case LRK_SURFACE_GLASS: {
            MicrofacetFamilyClosure<LRK_SURFACE_GLASS> c;
            c.init(*s);
            c.importance = importance;
            c.prepare(wo);
            return c.evaluate_local(wo, wi);
        }
        case LRK_SURFACE_PLASTIC: return child_evaluate<MicrofacetFamilyClosure<LRK_SURFACE_PLASTIC>>(s, wo, wi);
        default: return child_evaluate<MicrofacetFamilyClosure<LRK_SURFACE_METAL>>(s, wo, wi);
    }
}
// returns the sample's validity; `transmitted`: the sampled event is a refraction (Surface::event_enter / event_exit)
__device__ __noinline__ inline bool any_sample_direction(const lrk_surface *s, V3 wo, float u_lobe, float u0, float u1, V3 &wi, bool &transmitted) {
    transmitted = false;
    switch (s->type) {
        case LRK_SURFACE_MATTE: { MatteClosure c; c.init(*s); c.prepare(wo); return c.sample_direction(wo, u_lobe, u0, u1, wi); }
        case LRK_SURFACE_MIRROR: { MicrofacetFamilyClosure<LRK_SURFACE_MIRROR> c; c.init(*s); c.prepare(wo); return c.sample_direction(wo, u_lobe, u0, u1, wi); }
        case LRK_SURFACE_GLASS: {
            MicrofacetFamilyClosure<LRK_SURFACE_GLASS> c;
            c.init(*s);
            c.prepare(wo);
            bool valid = c.sample_direction(wo, u_lobe, u0, u1, wi);
            transmitted = !(u_lobe < c.glass_refl_prob(wo));
            return valid;
        }
        case LRK_SURFACE_PLASTIC: { MicrofacetFamilyClosure<LRK_SURFACE_PLASTIC> c; c.init(*s); c.prepare(wo); return c.sample_direction(wo, u_lobe, u0, u1, wi); }
        default: { MicrofacetFamilyClosure<LRK_SURFACE_METAL> c; c.init(*s); c.prepare(wo); return c.sample_direction(wo, u_lobe, u0, u1, wi); }
    }
}

struct MixClosure {
    const lrk_surface *a, *b;
    float ratio, eta;  // eta: MixSurfaceClosure::eta() (mix.cpp:133-141), 0 = none; computed by the host into p[1]
    float rr_eta_scale;
    uint32_t event;
    bool first_branch, child_valid;
    __device__ __forceinline__ void init(const lrk_surface &s, const lrk_surface *records) {
        a = records + s.mix_a;
        b = records + s.mix_b;
        ratio = s.p[0];
        eta = s.p[1];
        rr_eta_scale = 1.f;
        event = LRK_EVENT_REFLECT;
        first_branch = true;
        child_valid = false;
    }
    __device__ __forceinline__ void prepare(V3) {}
    __device__ __forceinline__ static SurfEval mix(const SurfEval &x, const SurfEval &y, float ratio) {// _mix: lerp(x, y, 1 - ratio)
        float t = 1.f - ratio;
        SurfEval e;
        e.f = lerp(x.f, y.f, t);
        e.pdf = lerp(x.pdf, y.pdf, t);
        return e;
    }
    __device__ __forceinline__ SurfEval evaluate_local(V3 wo, V3 wi) const {
        SurfEval ea = any_evaluate_local(a, wo, wi);
        SurfEval eb = any_evaluate_local(b, wo, wi);
        return mix(ea, eb, ratio);
    }
    // mix.cpp:158-180: both branches sample child `a` (the second one with the rescaled lobe number)
    __device__ __forceinline__ bool sample_direction(V3 wo, float u_lobe, float u0, float u1, V3 &wi) {
        first_branch = u_lobe < ratio;
        float ul = first_branch ? u_lobe / ratio : (u_lobe - ratio) / (1.f - ratio);
        bool transmitted;
        child_valid = any_sample_direction(a, wo, ul, u0, u1, wi, transmitted);
        rr_eta_scale = 1.f;
        if (transmitted && eta != 0.f) rr_eta_scale = cos_theta(wo) > 0.f ? sqr(eta) : sqr(1.f / eta);
        event = transmitted ? (cos_theta(wo) > 0.f ? LRK_EVENT_ENTER : LRK_EVENT_EXIT) : LRK_EVENT_REFLECT;// sample_a.event (mix.cpp:158-180)
        return true;// the other child is evaluated at wi whether or not a's sample is valid
    }
    // f and pdf of the sample: first branch mix(a's sample, b(wi)); second branch mix(b(wi), a's sample) — sic
    __device__ __forceinline__ SurfEval evaluate_sampled(V3 wo, V3 wi) const {
        SurfEval sa;
        sa.f = v3(0.f);
        sa.pdf = 0.f;
        if (child_valid) sa = any_evaluate_local(a, wo, wi);
        SurfEval ob = any_evaluate_local(b, wo, wi);
        return first_branch ? mix(sa, ob, ratio) : mix(ob, sa, ratio);
    }
};


// ---- Layered (src/surfaces/layered.cpp; pbrt-v4's LayeredBxDF as the reference restates it): hit bucket 9 ---------------------------
// Two interfaces - constant, non-Disney surface records `top` (mix_a) and `bottom` (mix_b) - around a homogeneous slab (thickness
// p[0], Henyey-Greenstein g p[1], albedo p[2..4]; lobes = max_depth | samples << 16).  evaluate() is a stochastic random walk with
// its own LCG stream seeded from the BITS of the hit position and of the world-space wi, sample() from the sample numbers and wo:
// the closure therefore works on world-space directions (LayeredHit carries the frame, the geometric normal and the position) and
// hands the kernel its sampled direction and f / pdf directly.  The interfaces are evaluated through the out-of-line dispatchers
// of the Mix closure, with the reference's per-call side validation (surface.cpp:35-68).  The code below is the oracle's
// layered_evaluate / layered_sample (bit-identical to the reference's renders, tests/test_ref_render.py::materials_layered*) with
// the device's types; where the reference draws several numbers inside one argument list the draws go left to right (clang's
// order, see oracle.cpp).
struct LayeredHit {
    Frame shading;
    V3 ng, pg;
};
struct LayeredSampleEval {
    V3 f;
    float pdf;
};
struct LayeredSample {
    LayeredSampleEval eval;
    V3 wi;
    uint32_t event;
};
__device__ __forceinline__ bool is_zero3(V3 a) { return a.x == 0.f && a.y == 0.f && a.z == 0.f; }
__device__ __forceinline__ V3 spherical_direction(float sinTheta, float cosTheta, float phi) {// src/util/scattering.h:81-83
    return v3(sinTheta * cosf(phi), sinTheta * sinf(phi), cosTheta);
}
// Surface::Closure::evaluate of an interface: the closure in the shared frame + validate_surface_sides
__device__ __forceinline__ SurfEval layered_child_evaluate(const lrk_surface *c, const LayeredHit &it, V3 wo, V3 wi, bool importance) {
    SurfEval e = any_evaluate_local(c, it.shading.world_to_local(wo), it.shading.world_to_local(wi), importance);
    if (!validate_surface_sides(it.ng, it.shading.n, wo, wi)) {
        e.f = v3(0.f);
        e.pdf = 0.f;
    }
    return e;
}
// Surface::Closure::sample of an interface: direction from the closure's sampler, f and pdf from its evaluate at that direction
__device__ __forceinline__ LayeredSample layered_child_sample(const lrk_surface *c, const LayeredHit &it, V3 wo, float u_lobe, float u0, float u1, bool importance) {
    const V3 wo_local = it.shading.world_to_local(wo);
    V3 wi_local;
    bool transmitted;
    const bool valid = any_sample_direction(c, wo_local, u_lobe, u0, u1, wi_local, transmitted);
    LayeredSample out;
    out.eval.f = v3(0.f);
    out.eval.pdf = 0.f;
    if (valid) {
        const SurfEval e = any_evaluate_local(c, wo_local, wi_local, importance);
        out.eval.f = e.f;
        out.eval.pdf = e.pdf;
    }
    out.wi = it.shading.local_to_world(wi_local);
    out.event = transmitted ? (cos_theta(wo_local) > 0.f ? LRK_EVENT_ENTER : LRK_EVENT_EXIT) : LRK_EVENT_REFLECT;
    if (!validate_surface_sides(it.ng, it.shading.n, wo, out.wi)) {
        out.eval.f = v3(0.f);
        out.eval.pdf = 0.f;
    }
    return out;
}
__device__ __forceinline__ float power_heuristic(float f_pdf, float g_pdf) {// src/util/sampling.cpp:142-151 with nf = ng = 1
    float f = 1.f * f_pdf, g = 1.f * g_pdf;
    float ff = f * f, gg = g * g, sum = ff + gg;
    return isinf(ff) ? 1.f : (sum == 0.f ? 0.f : ff / sum);
}
struct LayeredPhase {// HGPhaseFunction, layered.cpp:14-61
    float g;
    __device__ __forceinline__ static float hg(float cosTheta, float g) {
        float denom = 1.f + sqr(g) + 2.f * g * cosTheta;
        return kInvPi / 4.0f * (1.f - sqr(g)) / (denom * sqrtf(denom));
    }
    __device__ __forceinline__ float p(V3 wo, V3 wi) const { return hg(dot(wo, wi), g); }
    struct Sample {
        float p;
        V3 wi;
        float pdf;
    };
    __device__ __forceinline__ Sample sample_p(V3 wo, float ux, float uy) const {
        float cosTheta = fabsf(g) < 1e-3f ? 1.f - 2.f * ux : -1.f / (2.f * g) * (1.f + sqr(g) - sqr((1.f - sqr(g)) / (1.f + g - 2.f * g * ux)));
        float sinTheta = sqrtf(1.f - sqr(cosTheta));
        float phi = 2.f * kPi * uy;
        Frame wFrame = Frame::make(wo);
        V3 wi = wFrame.local_to_world(spherical_direction(sinTheta, cosTheta, phi));
        float pdf = hg(cosTheta, g);
        return {pdf, wi, pdf};
    }
};
struct LayeredCtx {
    const lrk_surface *top, *bottom, *records;
    float thickness, g;
    V3 albedo;
    uint32_t max_depth, samples;
    __device__ __forceinline__ LayeredCtx(const lrk_surface &s, const lrk_surface *rec)
        : top{rec + s.mix_a}, bottom{rec + s.mix_b}, records{rec}, thickness{s.p[0]}, g{s.p[1]}, albedo{v3(s.p[2], s.p[3], s.p[4])},
          max_depth{s.lobes & 0xffffu}, samples{s.lobes >> 16u} {}
    __device__ __forceinline__ static float Tr(float dz, V3 w) { return fabsf(dz) <= 1.17549435e-38f ? 1.f : expf(-fabsf(dz / w.z)); }
};

__device__ __noinline__ inline SurfEval layered_evaluate(const lrk_surface &s, const LayeredHit &it, V3 wo, V3 wi, const lrk_surface *records, bool mode) {// layered.cpp:251-404
    const LayeredCtx ctx{s, records};
    auto eval = [&](const lrk_surface *c, V3 a, V3 b, bool m) { return layered_child_evaluate(c, it, a, b, m); };
    auto sample = [&](const lrk_surface *c, V3 a, float uc, float u0, float u1, bool m) { return layered_child_sample(c, it, a, uc, u0, u1, m); };
    const V3 wi_local = it.shading.world_to_local(wi), wo_local = it.shading.world_to_local(wo);
    const bool entered_top = wo_local.z > 0.f;
    const bool exit_is_bottom = same_hemisphere(wo_local, wi_local) != entered_top;// same_hemisphere ^ entered_top
    const lrk_surface *enter_interface = entered_top ? ctx.top : ctx.bottom;
    const lrk_surface *exit_interface = exit_is_bottom ? ctx.bottom : ctx.top;
    const lrk_surface *nonexit_interface = exit_is_bottom ? ctx.top : ctx.bottom;
    const float exitZ = exit_is_bottom ? 0.f : ctx.thickness;
    const float n_samples = static_cast<float>(ctx.samples);
    V3 f = same_hemisphere(wi_local, wo_local) ? n_samples * eval(enter_interface, wo, wi, mode).f : v3(0.f);
    uint32_t seed = xxhash32_uint4(__float_as_uint(it.pg.x), __float_as_uint(it.pg.y), __float_as_uint(it.pg.z),
                                   xxhash32_uint3(__float_as_uint(wi.x), __float_as_uint(wi.y), __float_as_uint(wi.z)));
    float pdf_sum = same_hemisphere(wi_local, wo_local)
                        ? (entered_top ? n_samples * eval(ctx.top, wo, wi, mode).pdf : n_samples * eval(ctx.bottom, wo, wi, mode).pdf)
                        : 0.f;
    const LayeredPhase phase{ctx.g};
    for (uint32_t i = 0; i < ctx.samples; i++) {
        float uc, u0, u1;
        uc = lcg(seed); u0 = lcg(seed); u1 = lcg(seed);
        const LayeredSample wos = sample(enter_interface, wo, uc, u0, u1, mode);
        if (is_zero3(wos.eval.f) || wos.eval.pdf <= 0.f) continue;
        uc = lcg(seed); u0 = lcg(seed); u1 = lcg(seed);
        const LayeredSample wis = sample(exit_interface, wi, uc, u0, u1, !mode);
        const V3 wis_wi_local = it.shading.world_to_local(wis.wi);
        if (is_zero3(wis.eval.f) || wis.eval.pdf <= 0.f) continue;
        V3 beta = wos.eval.f / wos.eval.pdf;
        float z = entered_top ? ctx.thickness : 0.f;
        V3 w = wos.wi;
        V3 w_local = it.shading.world_to_local(w);
        for (uint32_t depth = 0; depth < ctx.max_depth; depth++) {
            if (depth > 3u && max3(beta) < 0.25f) {
                float q = fmaxf(0.f, 1.f - max3(beta));
                if (lcg(seed) < q) break;
                beta = beta / (1.f - q);
            }
            if (is_zero3(ctx.albedo)) {
                z = z == ctx.thickness ? 0.f : ctx.thickness;
                beta = beta * LayeredCtx::Tr(ctx.thickness, w_local);
            } else {
                const float sigma_t = 1.f;
                float dz = -logf(1.f - lcg(seed)) / (sigma_t / fabsf(w_local.z));
                float zp = w_local.z > 0.f ? z + dz : z - dz;
                if (z == zp) continue;
                if (zp > 0.f && zp < ctx.thickness) {
                    float wt = power_heuristic(wis.eval.pdf, eval(nonexit_interface, -w, -wis.wi, mode).pdf);
                    f = f + beta * ctx.albedo * phase.p(-w_local, -wis_wi_local) * wt * LayeredCtx::Tr(zp - exitZ, wis_wi_local) * wis.eval.f / wis.eval.pdf;
                    float ux, uy;
                    ux = lcg(seed); uy = lcg(seed);
                    LayeredPhase::Sample ps = phase.sample_p(-w_local, ux, uy);
                    if (ps.pdf <= 0.f || ps.wi.z == 0.f) continue;
                    beta = beta * (ctx.albedo * ps.p / ps.pdf);
                    w_local = ps.wi;
                    w = it.shading.local_to_world(w_local);
                    z = zp;
                    if ((z < exitZ && w_local.z > 0.f) || (z > exitZ && w_local.z < 0.f)) {
                        V3 fExit = eval(exit_interface, -w, wi, mode).f;
                        if (!is_zero3(fExit)) {
                            float exitPDF = eval(exit_interface, -w, wi, mode).pdf;
                            float wt2 = power_heuristic(ps.pdf, exitPDF);
                            f = f + beta * LayeredCtx::Tr(zp - exitZ, w_local) * fExit * wt2;
                        }
                    }
                    continue;
                }
                z = clampf(zp, 0.f, ctx.thickness);
            }
            if (z == exitZ) {
                float uc2 = lcg(seed), ua, ub;
                ua = lcg(seed); ub = lcg(seed);
                LayeredSample bs = sample(exit_interface, -w, uc2, ua, ub, mode);
                if (is_zero3(bs.eval.f) || bs.eval.pdf <= 0.f) break;
                beta = beta * (bs.eval.f / bs.eval.pdf);
                w = bs.wi;
                w_local = it.shading.world_to_local(w);
            } else {
                SurfEval wns = eval(nonexit_interface, -w, -wis.wi, mode);
                float wt = power_heuristic(wis.eval.pdf, wns.pdf);
                f = f + beta * wns.f * wt * LayeredCtx::Tr(ctx.thickness, wis_wi_local) * wis.eval.f / wis.eval.pdf;
                float uc2 = lcg(seed), ua, ub;
                ua = lcg(seed); ub = lcg(seed);
                LayeredSample bs = sample(nonexit_interface, -w, uc2, ua, ub, mode);
                if (is_zero3(bs.eval.f) || bs.eval.pdf <= 0.f) break;
                beta = beta * (bs.eval.f / bs.eval.pdf);
                w = bs.wi;
                w_local = it.shading.world_to_local(w);
                SurfEval wes = eval(exit_interface, -w, wi, mode);
                V3 fExit = wes.f;
                if (!is_zero3(fExit)) {
                    float wt2 = power_heuristic(bs.eval.pdf, wes.pdf);
                    f = f + beta * LayeredCtx::Tr(ctx.thickness, it.shading.world_to_local(bs.wi)) * fExit * wt2;
                }
            }
        }
    }
    for (uint32_t k = 0; k < ctx.samples; k++) {// pdf: :361-400
        if (same_hemisphere(wo_local, wi_local)) {
            const lrk_surface *r_interface = entered_top ? ctx.bottom : ctx.top;
            const lrk_surface *t_interface = entered_top ? ctx.top : ctx.bottom;
            float uc, u0, u1;
            uc = lcg(seed); u0 = lcg(seed); u1 = lcg(seed);
            LayeredSample wos = sample(t_interface, wo, uc, u0, u1, mode);
            uc = lcg(seed); u0 = lcg(seed); u1 = lcg(seed);
            LayeredSample wis = sample(t_interface, wi, uc, u0, u1, !mode);
            if (!is_zero3(wos.eval.f) && wos.eval.pdf > 0.f && !is_zero3(wis.eval.f) && wis.eval.pdf > 0.f) {
                uc = lcg(seed); u0 = lcg(seed); u1 = lcg(seed);
                LayeredSample rs = sample(r_interface, -wos.wi, uc, u0, u1, mode);
                if (!is_zero3(rs.eval.f) && rs.eval.pdf > 0.f) {
                    float r_pdf = eval(r_interface, -wos.wi, -wis.wi, mode).pdf;
                    float wt = power_heuristic(wis.eval.pdf, r_pdf);
                    pdf_sum += wt * r_pdf;
                    float t_pdf = eval(t_interface, -rs.wi, wi, mode).pdf;
                    wt = power_heuristic(rs.eval.pdf, t_pdf);
                    pdf_sum += wt * t_pdf;
                }
            }
        } else {
            const lrk_surface *ti_interface = entered_top ? ctx.bottom : ctx.top;
            const lrk_surface *to_interface = entered_top ? ctx.top : ctx.bottom;
            float uc, u0, u1;
            uc = lcg(seed); u0 = lcg(seed); u1 = lcg(seed);
            LayeredSample wos = sample(to_interface, wo, uc, u0, u1, mode);
            uc = lcg(seed); u0 = lcg(seed); u1 = lcg(seed);
            LayeredSample wis = sample(ti_interface, wi, uc, u0, u1, !mode);
            if (is_zero3(wos.eval.f) || wos.eval.pdf <= 0.f || is_zero3(wis.eval.f) || wis.eval.pdf <= 0.f) continue;
            pdf_sum += .5f * (eval(to_interface, wo, -wis.wi, mode).pdf + eval(ti_interface, -wos.wi, wi, mode).pdf);
        }
    }
    SurfEval e;
    e.f = f / n_samples;
    e.pdf = lerp(1.f / (4.f * kPi), pdf_sum / n_samples, 0.9f);
    return e;
}

__device__ __noinline__ inline LayeredSample layered_sample(const lrk_surface &s, const LayeredHit &it, V3 wo, float u_lobe, float u0, float u1, const lrk_surface *records, bool mode) {// layered.cpp:405-472
    const LayeredCtx ctx{s, records};
    auto sample = [&](const lrk_surface *c, V3 a, float uc, float ua, float ub, bool m) { return layered_child_sample(c, it, a, uc, ua, ub, m); };
    const V3 wo_local = it.shading.world_to_local(wo);
    const bool entered_top = wo_local.z > 0.f;
    LayeredSample bs = sample(entered_top ? ctx.top : ctx.bottom, wo, u_lobe, u0, u1, mode);
    LayeredSample out;// Surface::Sample::zero: f = 0, pdf = 0, wi = (0, 0, 1), event_reflect
    out.eval.f = v3(0.f);
    out.eval.pdf = 0.f;
    out.wi = v3(0.f, 0.f, 1.f);
    out.event = LRK_EVENT_REFLECT;
    if (!is_zero3(bs.eval.f) && bs.eval.pdf != 0.f) {
        V3 wi_local = it.shading.world_to_local(bs.wi);
        if (same_hemisphere(wi_local, wo_local)) {
            out = bs;
        } else {
            V3 w = bs.wi;
            V3 w_local = it.shading.world_to_local(bs.wi);
            uint32_t seed = xxhash32_uint4(__float_as_uint(u0), __float_as_uint(u1), __float_as_uint(u_lobe), xxhash32_uint3(__float_as_uint(wo.x), __float_as_uint(wo.y), __float_as_uint(wo.z)));
            V3 f = bs.eval.f;
            float pdf = bs.eval.pdf;
            float z = entered_top ? ctx.thickness : 0.f;
            const LayeredPhase phase{ctx.g};
            for (uint32_t depth = 0; depth < ctx.max_depth; depth++) {
                float rr_beta = max3(f) / pdf;
                if (depth > 3u && rr_beta < 0.25f) {
                    float q = fmaxf(0.f, 1.f - rr_beta);
                    if (lcg(seed) < q) break;
                    pdf *= 1.f - q;
                }
                if (w_local.z == 0.f) break;
                if (!is_zero3(ctx.albedo)) {
                    const float sigma_t = 1.f;
                    float dz = -logf(1.f - lcg(seed)) / (sigma_t / fabsf(w_local.z));
                    float zp = w_local.z > 0.f ? z + dz : z - dz;
                    if (z == zp) break;
                    if (0.f < zp && zp < ctx.thickness) {
                        float ux, uy;
                        ux = lcg(seed); uy = lcg(seed);
                        LayeredPhase::Sample ps = phase.sample_p(-w_local, ux, uy);
                        if (ps.pdf <= 0.f) break;
                        f = f * (ctx.albedo * ps.p);
                        pdf *= ps.pdf;
                        w = ps.wi;// sic: the phase function's LOCAL direction is taken as the world direction (:449-450)
                        w_local = it.shading.world_to_local(w);
                        z = zp;
                        continue;
                    }
                    z = clampf(zp, 0.f, ctx.thickness);
                } else {
                    z = z == ctx.thickness ? 0.f : ctx.thickness;
                    f = f * LayeredCtx::Tr(ctx.thickness, w_local);
                }
                const lrk_surface *interface = z == 0.f ? ctx.bottom : ctx.top;
                float uc = lcg(seed), ua, ub;
                ua = lcg(seed); ub = lcg(seed);
                LayeredSample is = sample(interface, -w, uc, ua, ub, mode);
                if (is_zero3(is.eval.f) || is.eval.pdf <= 0.f) break;
                f = f * is.eval.f;
                pdf *= is.eval.pdf;
                w = is.wi;
                w_local = it.shading.world_to_local(w);
                if ((is.event & 3u) != 0u) {// Surface::event_transmit = enter | exit
                    out.eval.f = f;
                    out.eval.pdf = pdf;
                    out.wi = w;
                    out.event = same_hemisphere(w_local, wo_local) ? LRK_EVENT_REFLECT : (w_local.z > 0.f ? LRK_EVENT_EXIT : LRK_EVENT_ENTER);
                    break;
                }
            }
        }
    }
    return out;
}


struct LayeredClosure {
    const lrk_surface *node, *records;
    LayeredHit hit;
    V3 wo_world, sampled_wi;
    LayeredSampleEval sampled;
    float rr_eta_scale;
    uint32_t event;
    __device__ __forceinline__ void init(const lrk_surface &s, const lrk_surface *rec, const Interaction &it, const Frame &shading, V3 wo) {
        node = &s;
        records = rec;
        hit.shading = shading;
        hit.ng = it.ng;
        hit.pg = it.pg;
        wo_world = wo;
        rr_eta_scale = 1.f;
        event = LRK_EVENT_REFLECT;
    }
    __device__ __forceinline__ void prepare(V3) {}
    // evaluate(wo, wi) for a WORLD-space wi (the light sample's direction)
    __device__ __forceinline__ SurfEval evaluate_world(V3 wi) const {
        SurfEval e = layered_evaluate(*node, hit, wo_world, wi, records, false);
        if (!validate_surface_sides(hit.ng, hit.shading.n, wo_world, wi)) {
            e.f = v3(0.f);
            e.pdf = 0.f;
        }
        return e;
    }
    // sample(wo, u_lobe, u): the walk's direction, f and pdf; eta() = the bottom interface's (layered.cpp:248)
    __device__ __forceinline__ bool sample_world(float u_lobe, float u0, float u1) {
        const LayeredSample s = layered_sample(*node, hit, wo_world, u_lobe, u0, u1, records, false);
        sampled = s.eval;
        sampled_wi = s.wi;
        event = s.event;
        if (!validate_surface_sides(hit.ng, hit.shading.n, wo_world, s.wi)) {
            sampled.f = v3(0.f);
            sampled.pdf = 0.f;
        }
        const lrk_surface *bottom = records + node->mix_b;
        const float eta = bottom->type == LRK_SURFACE_GLASS ? bottom->p[6] : 0.f;
        rr_eta_scale = 1.f;
        if (eta != 0.f) rr_eta_scale = event == LRK_EVENT_ENTER ? sqr(eta) : event == LRK_EVENT_EXIT ? sqr(1.f / eta) : 1.f;
        return true;
    }
};

}// namespace lrk
