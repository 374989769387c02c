// Host geometry helpers: the procedural sphere (the alias tables are in ../device/alias_table.h).
#include <algorithm>
#include <cmath>
#include <map>

#include "scene.h"

namespace lrh {

// ---------------------------------------------------------------- Loop subdivision (index based)
//
// The reference's Sphere is the icosahedron of src/shapes/sphere.cpp:15-50 refined by pbrt-style Loop
// subdivision (src/util/loop_subdiv.cpp:131-377), pushed to the limit surface and projected onto the
// unit sphere (sphere.cpp:88-97).  What must be preserved for scene parity is the vertex order (even
// vertices keep their index, odd vertices are appended in face/edge visiting order), the triangle order
// (4 children per face, child 3 is the centre), each vertex's start face (it fixes the one-ring summation
// order) and the fp32 evaluation order of the stencils.  This is a restatement over index arrays instead
// of the reference's pointer graph; only closed meshes are needed (boundary rules are still provided).

namespace {

constexpr int32_t kNone = -1;
inline int next3(int e) { return (e + 1) % 3; }
inline int prev3(int e) { return (e + 2) % 3; }

struct SVertex {
    float3 p;
    int32_t start_face{kNone};
    int32_t child{kNone};
    bool regular{false};
    bool boundary{false};
};
struct SFace {
    int32_t v[3]{kNone, kNone, kNone};
    int32_t f[3]{kNone, kNone, kNone};
    int32_t children[4]{kNone, kNone, kNone, kNone};
};

struct Level {
    std::vector<SVertex> verts;
    std::vector<SFace> faces;

    int vnum(int32_t face, int32_t vert) const {
        for (int i = 0; i < 3; i++) if (faces[face].v[i] == vert) return i;
        throw Error("Loop subdivision: vertex not on face.");
    }
    int32_t next_face(int32_t face, int32_t vert) const { return faces[face].f[vnum(face, vert)]; }
    int32_t prev_face(int32_t face, int32_t vert) const { return faces[face].f[prev3(vnum(face, vert))]; }
    int32_t next_vert(int32_t face, int32_t vert) const { return faces[face].v[next3(vnum(face, vert))]; }
    int32_t prev_vert(int32_t face, int32_t vert) const { return faces[face].v[prev3(vnum(face, vert))]; }
    int32_t other_vert(int32_t face, int32_t v0, int32_t v1) const {
        for (auto x : faces[face].v) if (x != v0 && x != v1) return x;
        throw Error("Loop subdivision: degenerate face.");
    }
    uint32_t valence(int32_t vi) const {
        auto &v = verts[vi];
        auto f = v.start_face;
        if (!v.boundary) {
            uint32_t nf = 1u;
            while ((f = next_face(f, vi)) != v.start_face) ++nf;
            return nf;
        }
        uint32_t nf = 1u;
        while ((f = next_face(f, vi)) != kNone) ++nf;
        f = v.start_face;
        while ((f = prev_face(f, vi)) != kNone) ++nf;
        return nf + 1u;
    }
    void one_ring(int32_t vi, std::vector<float3> &ring) const {
        ring.clear();
        auto &v = verts[vi];
        if (!v.boundary) {
            auto face = v.start_face;
            do {
                ring.push_back(verts[next_vert(face, vi)].p);
                face = next_face(face, vi);
            } while (face != v.start_face);
        } else {
            auto face = v.start_face;
            int32_t f2;
            while ((f2 = next_face(face, vi)) != kNone) face = f2;
            ring.push_back(verts[next_vert(face, vi)].p);
            do {
                ring.push_back(verts[prev_vert(face, vi)].p);
                face = prev_face(face, vi);
            } while (face != kNone);
        }
    }
    float3 weight_one_ring(int32_t vi, float beta, std::vector<float3> &ring) const {
        auto val = valence(vi);
        one_ring(vi, ring);
        auto p = (1.f - static_cast<float>(val) * beta) * verts[vi].p;
        for (uint32_t i = 0; i < val; i++) p += beta * ring[i];
        return p;
    }
    float3 weight_boundary(int32_t vi, float beta, std::vector<float3> &ring) const {
        auto val = valence(vi);
        one_ring(vi, ring);
        return (1.f - 2.f * beta) * verts[vi].p + beta * ring[0] + beta * ring[val - 1];
    }
};

inline float loop_beta(uint32_t valence) { return 3.f / (valence == 3u ? 16.f : 8.f * static_cast<float>(valence)); }
inline float loop_gamma(uint32_t valence) { return 1.f / (static_cast<float>(valence) + 3.f / (8.f * loop_beta(valence))); }

using EdgeKey = std::pair<int32_t, int32_t>;
inline EdgeKey edge_key(int32_t a, int32_t b) { return {std::min(a, b), std::max(a, b)}; }

void loop_subdivide_positions(const std::vector<float3> &base_p, const std::vector<lrk_triangle> &base_t, uint32_t level,
                              std::vector<float3> &out_p, std::vector<lrk_triangle> &out_t, std::vector<float3> *out_n = nullptr) {
    if (level == 0u) {
        out_p = base_p;
        out_t = base_t;
        return;
    }
    Level cur;
    cur.verts.resize(base_p.size());
    for (size_t i = 0; i < base_p.size(); i++) cur.verts[i].p = base_p[i];
    cur.faces.resize(base_t.size());
    for (size_t i = 0; i < base_t.size(); i++) {
        uint32_t t[3]{base_t[i].i0, base_t[i].i1, base_t[i].i2};
        for (int j = 0; j < 3; j++) {
            cur.faces[i].v[j] = static_cast<int32_t>(t[j]);
            cur.verts[t[j]].start_face = static_cast<int32_t>(i);
        }
    }
    {// neighbour links through shared edges
        std::map<EdgeKey, std::pair<int32_t, int>> open;
        for (size_t i = 0; i < cur.faces.size(); i++) {
            for (int e = 0; e < 3; e++) {
                auto key = edge_key(cur.faces[i].v[e], cur.faces[i].v[next3(e)]);
                if (auto it = open.find(key); it == open.end()) {
                    open.emplace(key, std::make_pair(static_cast<int32_t>(i), e));
                } else {
                    cur.faces[it->second.first].f[it->second.second] = static_cast<int32_t>(i);
                    cur.faces[i].f[e] = it->second.first;
                    open.erase(it);
                }
            }
        }
    }
    for (size_t i = 0; i < cur.verts.size(); i++) {
        auto &v = cur.verts[i];
        auto f = v.start_face;
        do {
            f = cur.next_face(f, static_cast<int32_t>(i));
        } while (f != kNone && f != v.start_face);
        v.boundary = (f == kNone);
        auto val = cur.valence(static_cast<int32_t>(i));
        v.regular = (!v.boundary && val == 6u) || (v.boundary && val == 4u);
    }

    std::vector<float3> ring;
    for (uint32_t l = 0; l < level; l++) {
        Level nxt;
        nxt.verts.reserve(cur.verts.size() + cur.faces.size() * 3 / 2 + 8);
        nxt.verts.resize(cur.verts.size());
        for (size_t i = 0; i < cur.verts.size(); i++) {
            cur.verts[i].child = static_cast<int32_t>(i);
            nxt.verts[i].regular = cur.verts[i].regular;
            nxt.verts[i].boundary = cur.verts[i].boundary;
        }
        nxt.faces.resize(cur.faces.size() * 4);
        for (size_t i = 0; i < cur.faces.size(); i++)
            for (int k = 0; k < 4; k++) cur.faces[i].children[k] = static_cast<int32_t>(i * 4 + k);

        // even vertices
        for (size_t i = 0; i < cur.verts.size(); i++) {
            auto vi = static_cast<int32_t>(i);
            if (!cur.verts[i].boundary) {
                auto b = cur.verts[i].regular ? 1.f / 16.f : loop_beta(cur.valence(vi));
                nxt.verts[i].p = cur.weight_one_ring(vi, b, ring);
            } else {
                nxt.verts[i].p = cur.weight_boundary(vi, 1.f / 8.f, ring);
            }
        }
        // odd vertices, appended in face/edge visiting order
        std::map<EdgeKey, int32_t> edge_verts;
        for (size_t i = 0; i < cur.faces.size(); i++) {
            auto &face = cur.faces[i];
            for (int k = 0; k < 3; k++) {
                auto a = face.v[k], b = face.v[next3(k)];
                auto key = edge_key(a, b);
                if (edge_verts.count(key)) continue;
                SVertex nv;
                nv.regular = true;
                nv.boundary = (face.f[k] == kNone);
                nv.start_face = face.children[3];
                if (nv.boundary) {
                    nv.p = .5f * cur.verts[key.first].p + .5f * cur.verts[key.second].p;
                } else {
                    nv.p = 3.f / 8.f * cur.verts[key.first].p + 3.f / 8.f * cur.verts[key.second].p +
                           1.f / 8.f * cur.verts[cur.other_vert(static_cast<int32_t>(i), a, b)].p +
                           1.f / 8.f * cur.verts[cur.other_vert(face.f[k], a, b)].p;
                }
                edge_verts.emplace(key, static_cast<int32_t>(nxt.verts.size()));
                nxt.verts.push_back(nv);
            }
        }
        // even vertex start faces
        for (size_t i = 0; i < cur.verts.size(); i++) {
            auto sf = cur.verts[i].start_face;
            nxt.verts[i].start_face = cur.faces[sf].children[cur.vnum(sf, static_cast<int32_t>(i))];
        }
        // face neighbour links
        for (size_t i = 0; i < cur.faces.size(); i++) {
            auto &face = cur.faces[i];
            for (int j = 0; j < 3; j++) {
                nxt.faces[face.children[3]].f[j] = face.children[next3(j)];
                nxt.faces[face.children[j]].f[next3(j)] = face.children[3];
                auto f2 = face.f[j];
                nxt.faces[face.children[j]].f[j] = f2 != kNone ? cur.faces[f2].children[cur.vnum(f2, face.v[j])] : kNone;
                f2 = face.f[prev3(j)];
                nxt.faces[face.children[j]].f[prev3(j)] = f2 != kNone ? cur.faces[f2].children[cur.vnum(f2, face.v[j])] : kNone;
            }
        }
        // face vertex links
        for (size_t i = 0; i < cur.faces.size(); i++) {
            auto &face = cur.faces[i];
            for (int j = 0; j < 3; j++) {
                nxt.faces[face.children[j]].v[j] = cur.verts[face.v[j]].child;
                auto vert = edge_verts.at(edge_key(face.v[j], face.v[next3(j)]));
                nxt.faces[face.children[j]].v[next3(j)] = vert;
                nxt.faces[face.children[next3(j)]].v[j] = vert;
                nxt.faces[face.children[3]].v[j] = vert;
            }
        }
        cur = std::move(nxt);
    }
    // limit surface
    out_p.resize(cur.verts.size());
    for (size_t i = 0; i < cur.verts.size(); i++) {
        auto vi = static_cast<int32_t>(i);
        out_p[i] = cur.verts[i].boundary ? cur.weight_boundary(vi, 1.f / 5.f, ring)
                                         : cur.weight_one_ring(vi, loop_gamma(cur.valence(vi)), ring);
    }
    if (out_n != nullptr) {
        // limit-surface normals from the one-ring tangents of the LIMIT positions (src/util/loop_subdiv.cpp:320-358)
        constexpr float pi = 3.14159265358979323846264338327950288f;
        for (size_t i = 0; i < cur.verts.size(); i++) cur.verts[i].p = out_p[i];
        out_n->resize(cur.verts.size());
        for (size_t i = 0; i < cur.verts.size(); i++) {
            auto vi = static_cast<int32_t>(i);
            auto val = cur.valence(vi);
            cur.one_ring(vi, ring);
            float3 S{0.f, 0.f, 0.f}, T{0.f, 0.f, 0.f};
            if (!cur.verts[i].boundary) {
                for (uint32_t j = 0; j < val; j++) {
                    S += std::cos(2.f * pi * static_cast<float>(j) / static_cast<float>(val)) * ring[j];
                    T += std::sin(2.f * pi * static_cast<float>(j) / static_cast<float>(val)) * ring[j];
                }
            } else {
                S = ring[val - 1u] - ring[0];
                if (val == 2u) {
                    T = ring[0] + ring[1] - 2.f * cur.verts[i].p;
                } else if (val == 3u) {
                    T = ring[1] - cur.verts[i].p;
                } else if (val == 4u) {
                    T = -1.f * ring[0] + 2.f * ring[1] + 2.f * ring[2] - 1.f * ring[3] - 2.f * cur.verts[i].p;
                } else {
                    auto theta = pi / static_cast<float>(val - 1u);
                    T = std::sin(theta) * (ring[0] + ring[val - 1u]);
                    for (uint32_t k = 1u; k < val - 1u; k++) {
                        auto wt = (2.f * std::cos(theta) - 2.f) * std::sin(static_cast<float>(k) * theta);
                        T += wt * ring[k];
                    }
                    T = -T;
                }
            }
            (*out_n)[i] = normalize(cross(T, S));
        }
    }
    out_t.resize(cur.faces.size());
    for (size_t i = 0; i < cur.faces.size(); i++) {
        out_t[i] = {static_cast<uint32_t>(cur.faces[i].v[0]), static_cast<uint32_t>(cur.faces[i].v[1]),
                    static_cast<uint32_t>(cur.faces[i].v[2])};
    }
}

}// namespace

void loop_subdivide_mesh(const std::vector<lrk_vertex> &base_v, const std::vector<lrk_triangle> &base_t, uint32_t level,
                         std::vector<lrk_vertex> &vertices, std::vector<lrk_triangle> &triangles) {
    // loop_subdivide, src/util/loop_subdiv.cpp:131-377: limit positions, limit normals, uv = 0 ("FIXME: uv" there)
    std::vector<float3> bp(base_v.size()), p, n;
    for (size_t i = 0; i < base_v.size(); i++) bp[i] = {base_v[i].p[0], base_v[i].p[1], base_v[i].p[2]};
    loop_subdivide_positions(bp, base_t, level, p, triangles, &n);
    vertices.resize(p.size());
    for (size_t i = 0; i < p.size(); i++) vertices[i] = {{p[i].x, p[i].y, p[i].z}, {n[i].x, n[i].y, n[i].z}, {0.f, 0.f}};
}

void make_sphere(uint32_t subdivision, std::vector<lrk_vertex> &vertices, std::vector<lrk_triangle> &triangles) {
    // src/shapes/sphere.cpp:15-50
    static const float3 base_vertices[12]{
        {0.f, -0.525731f, 0.850651f}, {0.850651f, 0.f, 0.525731f}, {0.850651f, 0.f, -0.525731f},
        {-0.850651f, 0.f, -0.525731f}, {-0.850651f, 0.f, 0.525731f}, {-0.525731f, 0.850651f, 0.f},
        {0.525731f, 0.850651f, 0.f}, {0.525731f, -0.850651f, 0.f}, {-0.525731f, -0.850651f, 0.f},
        {0.f, -0.525731f, -0.850651f}, {0.f, 0.525731f, -0.850651f}, {0.f, 0.525731f, 0.850651f}};
    static const lrk_triangle base_triangles[20]{
        {1u, 2u, 6u}, {1u, 7u, 2u}, {3u, 4u, 5u}, {4u, 3u, 8u}, {6u, 5u, 11u}, {5u, 6u, 10u}, {9u, 10u, 2u},
        {10u, 9u, 3u}, {7u, 8u, 9u}, {8u, 7u, 0u}, {11u, 0u, 1u}, {0u, 11u, 4u}, {6u, 2u, 10u}, {1u, 6u, 11u},
        {3u, 5u, 10u}, {5u, 4u, 11u}, {2u, 7u, 9u}, {7u, 1u, 0u}, {3u, 9u, 8u}, {4u, 8u, 0u}};
    std::vector<float3> bp(12);
    for (int i = 0; i < 12; i++) bp[i] = normalize(base_vertices[i]);
    std::vector<lrk_triangle> bt(base_triangles, base_triangles + 20);
    std::vector<float3> p;
    loop_subdivide_positions(bp, bt, std::min(subdivision, 8u), p, triangles);
    vertices.resize(p.size());
    constexpr float inv_pi = 0.318309886183790671537767526745028724f;
    for (size_t i = 0; i < p.size(); i++) {
        // every level (0 included) re-projects and recomputes p = n and uv from the un-normalised position
        // (sphere.cpp:90-95)
        auto w = p[i];
        auto n = normalize(w);
        auto theta = std::acos(w.y);
        auto phi = std::atan2(w.x, w.z);
        auto fu = .5f * inv_pi * phi, fv = theta * inv_pi;
        auto u = fu - std::floor(fu);
        auto v = fv - std::floor(fv);
        vertices[i] = {{n.x, n.y, n.z}, {n.x, n.y, n.z}, {u, v}};
    }
}

}// namespace lrh
