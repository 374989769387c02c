"""The edge-case catalogue of the hierarchy tests (tests/test_hierarchy_edges.py, tests/test_update_hierarchy_edges*.py): scenes
built to break the claim that closest hits do not depend on the hierarchy (DESIGN.md §4) - leaf-sized meshes, exact ties, flat and
graded geometry, extreme sizes and offsets, awkward instance transforms, many and invisible instances -, the ray set of a scene
(rays aimed at vertices and edges from near and from very far), the float64 reference of the brute-force loop, and the rays whose
hit the float32 triangle test places outside the triangle's own padded box (exempt from bit-exactness: no box test can keep them)."""
from __future__ import annotations

from pathlib import Path

import numpy as np

from luisarender_b200 import scenes
from luisarender_b200.api import Scene
from oracle import binding as O

REPO = Path(__file__).resolve().parents[1]
MISS = 0xFFFFFFFF
FMAX = np.finfo(np.float32).max
FAR_FACTORS = (3, 30, 100, 1000)
FAR_RAYS = 20_000  # per distance factor and scene: the BVH-vs-brute-force comparison is cheap, missed hits are rare events
F64_RAYS = 3_000   # rays per scene that also go through the float64 reference


# ---- scene catalogue --------------------------------------------------------------------------------------------------------

def _affine(linear=np.eye(3), translate=(0.0, 0.0, 0.0)):
    return np.concatenate([np.asarray(linear, np.float64), np.asarray(translate, np.float64)[:, None]], axis=1)


def _random_tris(rng, n, center=(0.0, 0.0, 0.0), radius=0.5):
    p = rng.normal(size=(n * 3, 3))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    return p * radius + np.asarray(center), np.arange(n * 3).reshape(n, 3)


def _fan(n, radius=0.5):
    a = np.linspace(0.0, 2.0 * np.pi, n, endpoint=False)
    ring = np.stack([radius * np.cos(a), 0.1 * np.sin(3 * a), radius * np.sin(a)], axis=1)
    p = np.concatenate([[[0.0, 0.0, 0.0]], ring])
    return p, np.array([[0, 1 + k, 1 + (k + 1) % n] for k in range(n)])


def _grid(n=6, size=1.0):
    xs = np.linspace(-size / 2, size / 2, n + 1)
    p = np.array([[x, 0.0, z] for z in xs for x in xs])
    idx = []
    for j in range(n):
        for i in range(n):
            a, b, c, d = j * (n + 1) + i, j * (n + 1) + i + 1, (j + 1) * (n + 1) + i, (j + 1) * (n + 1) + i + 1
            idx += [[a, b, d], [a, d, c]]
    return p, np.array(idx)


def _graded(kmax=40):
    """Self-similar triangles of size 2^-k at x = 2^-k: a hierarchy as deep as the number of triangles."""
    base = np.array([[1.0, 0.0, 0.0], [1.5, 1.0, 0.2], [1.2, 0.3, 1.0]])
    p = np.concatenate([base * 2.0 ** -k for k in range(kmax + 1)])
    return p, np.arange(len(p)).reshape(-1, 3)


def _rotation(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(angle) * k + (1 - np.cos(angle)) * k @ k


def catalogue():
    """name -> (meshes [(positions, indices)], instances [(mesh, 3x4 object_to_world, visible)])."""
    rng = np.random.default_rng(2024)
    I = _affine()
    cat = {}
    for n in (1, 2, 3, 4, 5, 8, 9, 33):
        cat[f"tris_{n}"] = ([_random_tris(rng, n)], [(0, I, True)])
    tri = np.array([[-0.4, -0.3, 0.1], [0.5, -0.2, -0.1], [0.0, 0.45, 0.05]])
    cat["copies_12"] = ([(np.tile(tri, (12, 1)), np.arange(36).reshape(12, 3))], [(0, I, True)])
    cat["fan_8"] = ([_fan(8)], [(0, I, True)])
    cat["fan_64"] = ([_fan(64)], [(0, I, True)])
    blob = _random_tris(rng, 40)
    cat["same_transform_twice"] = ([blob], [(0, _affine(_rotation((1, 2, 3), 0.7), (0.1, 0.2, 0.3)), True)] * 2)
    cat["flat_grid"] = ([_grid()], [(0, I, True)])
    cat["graded"] = ([_graded()], [(0, I, True)])
    cat["size_1e-4"] = ([_random_tris(rng, 30, radius=1e-4)], [(0, I, True)])
    cat["size_1e4"] = ([_random_tris(rng, 30, radius=1e4)], [(0, I, True)])
    cat["offset_1e4"] = ([_random_tris(rng, 30, center=(1e4, -3e3, 5e3))], [(0, I, True)])
    far = (3000.0, -2000.0, 5000.0)
    cat["cancelling_instance"] = ([_random_tris(rng, 60, center=far)], [(0, _affine(translate=-np.asarray(far)), True)])
    cat["scaled_instance"] = ([_random_tris(rng, 60)], [(0, _affine(0.05 * np.eye(3)), True)])
    skew = _rotation((0.3, -1.0, 0.5), 1.1) @ np.diag([-1.0, 0.25, 3.0])  # rotation, mirroring, non-uniform scale
    cat["rotated_mirrored_instance"] = ([_random_tris(rng, 60)], [(0, _affine(skew, (0.2, -0.1, 0.4)), True)])
    small = _random_tris(rng, 4, radius=0.05)
    cat["one_instance"] = ([small], [(0, _affine(translate=(0.3, 0.1, -0.2)), True)])
    cat["two_instances"] = ([small], [(0, _affine(translate=(0.3, 0.1, -0.2)), True), (0, _affine(translate=(-0.3, 0.0, 0.1)), True)])
    grid = np.stack(np.meshgrid(*[np.linspace(-1.0, 1.0, 10)] * 3, indexing="ij"), axis=-1).reshape(-1, 3)
    cat["instances_1000"] = ([small], [(0, _affine(_rotation(rng.normal(size=3), rng.uniform(0, 6)), t), True) for t in grid])
    # invisible instances between and in front of visible ones: rays along z cross both kinds
    cat["invisible_interleaved"] = ([blob], [(0, _affine(0.3 * np.eye(3), (0.15 * (k % 5), 0.0, 0.4 * k - 2.0)), k % 2 == 1) for k in range(10)])
    # world-to-object rounding of distant rays: a flat mesh under the mirrored, skewed transform above, and the 1000 rotated
    # instances of a mesh that sits far from its own origin
    [(p, idx)], [(_, xf, _)] = cat["rotated_mirrored_instance"]
    cat["flat_mirrored_instance"] = ([(p * [1.0, 0.0, 1.0], idx)], [(0, xf, True)])
    far_small = (small[0] + [1e4, -3e3, 5e3], small[1])
    cat["far_mesh_instances_1000"] = ([far_small], cat["instances_1000"][1])
    # a mesh far from its origin brought back by a rotation: o2w = [R | -R far]
    rot = _rotation((1.0, -0.5, 0.25), 2.0)
    cat["rotated_cancelling_instance"] = ([cat["cancelling_instance"][0][0]], [(0, _affine(rot, -rot @ np.asarray(far)), True)])
    return cat


CATALOGUE = catalogue()
# ray-set seeds of the scenes whose default seed (position in the catalogue + 1) draws no ray that the instance level's box test
# loses: these draw one (from 1000 and from 100 scene sizes away), which outside_instance_box must exempt
SEEDS = {"flat_mirrored_instance": 3, "far_mesh_instances_1000": 1}


def _world_triangles(meshes, instances):
    """float64 world-space triangles [(inst, prim, p0, p1, p2)] of the visible instances (the ray generator's view)."""
    out = []
    for i, (m, xf, vis) in enumerate(instances):
        if vis:
            p, idx = meshes[m]
            w = p @ xf[:, :3].T + xf[:, 3]
            out.append(w[idx])
    return np.concatenate(out)


def scene_text(meshes, instances, frame=None):
    """The scene's text: the meshes and instances, a lamp above them and a camera that sees them.  The lamp and the camera are
    placed around the world triangles of `frame` ((meshes, instances), default the scene itself): frames of one update chain pass
    the union of the chain's scenes, so that they differ only in what the update changes."""
    f = scenes._fmt
    tris = _world_triangles(meshes, instances) if frame is None else _world_triangles(*frame)
    lo, hi = tris.reshape(-1, 3).min(axis=0), tris.reshape(-1, 3).max(axis=0)
    c, r = (lo + hi) / 2, float((hi - lo).max())
    ly, s = hi[1] + 0.05 * r, 0.05 * r
    lamp = [c[0] - s, ly, c[2] - s, c[0] + s, ly, c[2] - s, c[0] + s, ly, c[2] + s, c[0] - s, ly, c[2] + s]
    eye = c + r * np.array([0.4, 0.9, 2.2])
    front = (c - eye) / np.linalg.norm(c - eye)
    lines = ['Surface white : Matte { Kd : Constant { v { 0.6, 0.5, 0.4 } } }',
             'Light lamp_light : Diffuse { emission : Constant { v { 8.0, 8.0, 8.0 } } }']
    for k, (p, idx) in enumerate(meshes):
        lines.append(f"Shape m{k} : InlineMesh {{ positions {{ {', '.join(f(v) for v in p.ravel())} }} "
                     f"indices {{ {', '.join(str(int(v)) for v in idx.ravel())} }} }}")
    for k, (m, xf, vis) in enumerate(instances):
        mat = np.concatenate([xf, [[0.0, 0.0, 0.0, 1.0]]]).ravel()
        lines.append(f"Shape i{k} : Instance {{ shape {{ @m{m} }} surface {{ @white }} visible {{ {'true' if vis else 'false'} }} "
                     f"transform : Matrix {{ m {{ {', '.join(f(v) for v in mat)} }} }} }}")
    lines.append(f"Shape lamp : InlineMesh {{ positions {{ {', '.join(f(v) for v in lamp)} }} indices {{ 0, 1, 2, 0, 2, 3 }} "
                 "light { @lamp_light } }")
    shapes = ", ".join([f"@i{k}" for k in range(len(instances))] + ["@lamp"])
    lines.append(f"Camera camera : Pinhole {{ position {{ {', '.join(f(v) for v in eye)} }} front {{ {', '.join(f(v) for v in front)} }} "
                 "up { 0.0, 1.0, 0.0 } fov { 45.0 } spp { 4 } film : Color { resolution { 24, 24 } } filter : Box { radius { 0.5 } } "
                 'file { "edges.exr" } }')
    lines.append("render { integrator : WavePath { depth { 3 } sampler : Independent { seed { 7 } } } cameras { @camera } "
                 f"shapes {{ {shapes} }} }}")
    return "\n".join(lines)


# ---- rays ---------------------------------------------------------------------------------------------------------------------

def desc_triangles(d):
    """float64 world-space triangles of the flattened scene, with their (instance, primitive) - what the oracle intersects - and the
    size of their object-space coordinates in world units (what the float32 test's rounding is relative to)."""
    tris, ids, mags = [], [], []
    for i in range(d.instance_count):
        inst = d.instances[i]
        if not inst.visible:
            continue
        mesh = d.meshes[inst.mesh]
        m = np.array(inst.object_to_world, np.float64).reshape(3, 4)
        v = np.array([d.vertices[mesh.vertex_offset + k].p[:] for k in range(mesh.vertex_count)], np.float64)
        t = np.array([[d.triangles[mesh.triangle_offset + k].i0, d.triangles[mesh.triangle_offset + k].i1,
                       d.triangles[mesh.triangle_offset + k].i2] for k in range(mesh.triangle_count)])
        tris.append((v @ m[:, :3].T + m[:, 3])[t])
        ids.append(np.stack([np.full(len(t), i), np.arange(len(t))], axis=1))
        mags.append(np.abs(v[t]).max(axis=(1, 2)) * np.linalg.norm(m[:, :3], 2))
    return np.concatenate(tris), np.concatenate(ids).astype(np.uint32), np.concatenate(mags)


def _pack(o, d, tmax=FMAX, tmin=0.0):
    rays = np.zeros((len(o), 8), np.float32)
    rays[:, :3], rays[:, 3], rays[:, 4:7], rays[:, 7] = o, tmin, d, tmax
    return rays


def _unit(v):
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _aimed(rng, targets, dist):
    d = _unit(rng.normal(size=targets.shape))
    return _pack(targets - d * dist[:, None] if np.ndim(dist) else targets - d * dist, d)


def make_rays(d, tris, ids, seed, aim=None):
    """The ray set of one scene (fixed seed): [base rays (checked against float64 too) ..., far rays].  The rays are sized by and
    aimed at the triangles `aim` (a mask over tris; default all of them)."""
    rng = np.random.default_rng(seed)
    target = tris if aim is None else tris[aim]
    pts = target.reshape(-1, 3)
    lo, hi = pts.min(axis=0), pts.max(axis=0)
    c, r = (lo + hi) / 2, float((hi - lo).max())
    pick = lambda a, n: a[rng.integers(0, len(a), n)]  # noqa: E731
    cent = target.mean(axis=1)
    mids = np.concatenate([(target[:, 0] + target[:, 1]) / 2, (target[:, 1] + target[:, 2]) / 2, (target[:, 2] + target[:, 0]) / 2])
    feats = np.concatenate([pts, mids])
    jitter = lambda p: p + rng.normal(size=p.shape) * 1e-4 * r  # noqa: E731
    parts = []
    # one ray per triangle (at most 400) at its centroid, from around the scene
    parts.append(_aimed(rng, pick(cent, min(len(cent), 400)), rng.uniform(0.5, 2.0, min(len(cent), 400)) * r))
    # vertices and edge midpoints, jittered: silhouettes, shared edges and corners
    parts.append(_aimed(rng, jitter(pick(feats, 800)), rng.uniform(0.5, 2.0, 800) * r))
    # random rays through the scene's box (as in test_gpu_parity._random_rays), a third of them short
    o = rng.uniform(lo - 0.5 * r, hi + 0.5 * r, size=(600, 3))
    rand = _pack(o, _unit(rng.uniform(lo, hi, size=(600, 3)) - o))
    rand[::3, 7] = rng.uniform(0.05, 1.0, size=len(rand[::3])) * r
    parts.append(rand)
    # axis-aligned directions and negative-zero components through vertices and edge midpoints (on the flat grid: rays in its
    # plane, along its grid lines)
    ax = _aimed(rng, jitter(pick(feats, 300)), 1.5 * r)
    ax[:100, 4:7] = np.eye(3)[rng.integers(0, 3, 100)] * rng.choice([-1.0, 1.0], size=(100, 1))
    ax[100:, 4 + rng.integers(0, 3)] = -0.0
    ax[:, :3] = pick(feats, 300) - ax[:, 4:7] * (1.5 * r)
    parts.append(ax)
    base = np.concatenate(parts)
    # rays that start on surfaces: points on the hit triangles (rounded to float32, so on either side), random directions
    ref, _ = O.trace(d, base, brute=True)
    hit = np.flatnonzero(ref["inst"] != MISS)[:600]
    key = {(int(a), int(b)): k for k, (a, b) in enumerate(ids)}
    bary = ref["bary"][hit].astype(np.float64)
    tri = tris[[key[(int(a), int(b))] for a, b in zip(ref["inst"][hit], ref["prim"][hit])]]
    p = (1 - bary.sum(axis=1))[:, None] * tri[:, 0] + bary[:, :1] * tri[:, 1] + bary[:, 1:] * tri[:, 2]
    dirs = _unit(rng.normal(size=p.shape))
    dirs[::5, 1] = -0.0
    bounce = _pack(p, dirs)
    bounce[1::4, 7] = 1e-3 * r
    base = np.concatenate([base, bounce])
    # distant origins aimed at vertices and edge midpoints (with a tiny jitter: silhouettes)
    far = [_aimed(rng, pick(feats, FAR_RAYS) + rng.normal(size=(FAR_RAYS, 3)) * 1e-5 * r, k * r) for k in FAR_FACTORS]
    return base, far


# ---- float64 reference ----------------------------------------------------------------------------------------------------------

def f64_check(rays, tris, ids, mags, brute, scale):
    """Independent float64 Moeller-Trumbore over every visible triangle.  Where the answer is unambiguous - the nearest hit is more
    than 1e-4 relative ahead of every other candidate and of the ray's ends, and at least 1e-5 inside its triangle (more for distant
    origins, large object-space coordinates and grazing rays) - the brute force must hit the same (instance, primitive) at the same
    point (1e-5 of the distance); a ray that passes every triangle by more than 1e-3 in the barycentrics must miss.  Returns the
    number of rays with an unambiguous answer."""
    p0, e1, e2 = tris[:, 0], tris[:, 1] - tris[:, 0], tris[:, 2] - tris[:, 0]
    size = np.sqrt(np.linalg.norm(np.cross(e1, e2), axis=1))
    kept = 0
    for s in range(0, len(rays), 128):
        with np.errstate(divide="ignore", invalid="ignore"):
            kept += _f64_chunk(rays[s:s + 128], brute[s:s + 128], s, tris, ids, mags, scale, p0, e1, e2, size)
    return kept


def _f64_chunk(rays, b, first, tris, ids, mags, scale, p0, e1, e2, size):
    o, dd = rays[:, :3].astype(np.float64), rays[:, 4:7].astype(np.float64)
    tmin, tmax = rays[:, 3].astype(np.float64), rays[:, 7].astype(np.float64)
    pvec = np.cross(dd[:, None, :], e2[None])
    det = np.einsum("tk,rtk->rt", e1, pvec)
    tvec = o[:, None, :] - p0[None]
    u = np.einsum("rtk,rtk->rt", tvec, pvec) / det
    q = np.cross(tvec, e1[None])
    v = np.einsum("rk,rtk->rt", dd, q) / det
    t = np.einsum("tk,rtk->rt", e2, q) / det
    inside = np.minimum(np.minimum(u, v), 1.0 - u - v)
    # candidates include those just outside the ray's ends: a ray that starts on a surface meets it again near t = 0, on either
    # side of tmin (by up to 1e-4 x the scene size for grazing rays and large object-space coordinates)
    in_range = (t > tmin[:, None] - 1e-3 * scale) & (t < tmax[:, None] * (1 + 1e-4)) & np.isfinite(t)
    # 1e-5 of the barycentrics, more from far away, for large object-space coordinates and for grazing rays: the float32 test's
    # barycentrics err by ~1e-7 x (distance or coordinate size) / (triangle size x |cos| of the angle to the normal)
    dn = np.linalg.norm(dd, axis=1)[:, None]
    reach = np.nan_to_num(np.abs(t), posinf=0.0) * dn + mags[None]
    cos = np.abs(det) / (dn * size[None] ** 2)
    margin = 1e-5 * np.maximum(1.0, np.nan_to_num(reach / size[None] / cos / 10.0, nan=np.inf))
    cand_t = np.where(in_range & (inside >= -margin), t, np.inf)
    order = np.argsort(cand_t, axis=1)[:, :2]
    rows = np.arange(len(rays))
    best = order[:, 0]
    t1, t2 = cand_t[rows, best], cand_t[rows, order[:, 1]] if cand_t.shape[1] > 1 else np.full(len(rays), np.inf)
    # a clear miss: no triangle within 1e-3 of its edges anywhere on the line before tmax (rays that start on a surface and
    # rays from far away are decided by the float32 rounding of their own triangle)
    miss = ~((t < tmax[:, None]) & (inside >= -np.maximum(1e-3, 10 * margin))).any(axis=1)
    assert (b["inst"][miss] == MISS).all(), f"brute force hit where float64 finds no candidate: rays {(first + np.flatnonzero(miss & (b['inst'] != MISS)))[:5]}"
    tol = 1e-4 * np.abs(t1) + 1e-5 * scale + 1e-6 * mags[best] / dn[:, 0]  # t rounds with the object-space coordinates too
    clear = np.isfinite(t1) & (inside[rows, best] >= margin[rows, best]) & (t2 - t1 > tol) & (t1 - tmin > tol) & (tmax - t1 > tol)
    k = np.flatnonzero(clear)
    wrong = k[(b["inst"][k] != ids[best[k], 0]) | (b["prim"][k] != ids[best[k], 1])]
    assert not len(wrong), f"brute force disagrees with float64 on unambiguous hits: rays {(first + wrong)[:5].tolist()}, " \
        f"brute {b[wrong[:3]].tolist()}, float64 {ids[best[wrong[:3]]].tolist()} at t {t1[wrong[:3]].tolist()}"
    # the hit point: 1e-5 of the distance, or what the barycentric margin allows
    tb, bu = best[k], b["bary"][k].astype(np.float64)
    ph = (1 - bu.sum(axis=1))[:, None] * tris[tb, 0] + bu[:, :1] * tris[tb, 1] + bu[:, 1:] * tris[tb, 2]
    gap = np.linalg.norm(ph - (o[k] + t1[k, None] * dd[k]), axis=1)
    assert (gap <= 1e-5 * t1[k] * dn[k, 0] + 4 * margin[k, tb] * size[tb]).all(), "brute-force hit point disagrees with float64"
    return int(miss.sum()) + len(k)


# ---- hits the triangle test takes outside its own box ----------------------------------------------------------------------------

def _fma(a, b, c):
    """fmaf on float32 arrays: the product of two float32 is exact in float64."""
    return (a.astype(np.float64) * b + c).astype(np.float32)


def _fdot(a, b):
    return _fma(a[:, 0], b[:, 0], _fma(a[:, 1], b[:, 1], a[:, 2] * b[:, 2]))


def _fcross(a, b):
    return np.stack([_fma(a[:, 1], b[:, 2], -(a[:, 2] * b[:, 1])), _fma(a[:, 2], b[:, 0], -(a[:, 0] * b[:, 2])),
                     _fma(a[:, 0], b[:, 1], -(a[:, 1] * b[:, 0]))], axis=1)


def outside_own_box(d, rays, hits):
    """Rays whose hit the float32 triangle test places outside the hit triangle's own padded box.

    The Moeller-Trumbore test rounds too, by an amount that grows with the distance from the ray origin to the triangle and with how
    grazing the ray is: rays from far away that pass a silhouette edge by a few 1e-7 of their length, or that graze a fan of
    triangles through a shared vertex, can be accepted at a point that lies outside every box holding the triangle.  Whether such a
    hit is found then depends on the hierarchy - no box test can be made to contain it - so these rays are the ones exempt from
    the bit-exact comparison with the brute force.  This restates the test's arithmetic (object-space ray by fma, edges, t) and
    flags the rays that miss the triangle's bounds, padded like bvh.cpp pads a leaf box, in exact arithmetic, and the rays whose t
    lies outside the exact entry and exit distances of those bounds by more than the box test's own margin (kSlabExitScale)."""
    out = np.zeros(len(rays), bool)
    hit = np.flatnonzero(hits["inst"] != MISS)
    if not len(hit):
        return out
    inst, oo, od, p, t = _triangle_test(d, rays, hits, hit)
    verts = np.array([v.p[:] for v in d.vertices[:d.vertex_count]], np.float32)
    pad = np.zeros(d.instance_count, np.float32)
    for i in range(d.instance_count):
        m = d.meshes[d.instances[i].mesh]
        v = verts[m.vertex_offset:m.vertex_offset + m.vertex_count]
        pad[i] = np.float32(5e-7) * np.float32(max(np.abs(v).max(), (v.max(axis=0) - v.min(axis=0)).max()))
    lo = (p.min(axis=1) - pad[inst][:, None]).astype(np.float64)
    hi = (p.max(axis=1) + pad[inst][:, None]).astype(np.float64)
    out[hit] = _outside(oo, od, lo, hi, t)
    return out


def outside_instance_box(d, rays, hits):
    """Rays whose hit, at the t the float32 triangle test computes, lies on the world ray outside the hit instance's box in the
    instance level.

    The triangle test runs on the object-space ray, which the world-to-object transform rounds by an amount relative to the
    origin's distance (and to the transform's condition): from far away the object-space ray is moved sideways against the world
    ray that the instance level's box test sees, so a hit inside the triangle's own padded box can lie outside the instance's world
    box, by more than any pad below the spawned-ray offset.  Whether such a hit is found depends on the instance level.  This
    takes the instance's box as the description's instance level stores it (a host-built box: the device-built boxes hold it) and
    flags, in exact arithmetic, the rays whose t lies outside that box's entry and exit distances along the world ray by more than
    the box test's own margin, as outside_own_box does with the triangle's box."""
    out = np.zeros(len(rays), bool)
    hit = np.flatnonzero(hits["inst"] != MISS)
    if not len(hit):
        return out
    inst, _, _, _, t = _triangle_test(d, rays, hits, hit)
    boxes = np.full((d.instance_count, 2, 3), np.nan)
    for n in range(d.tlas_root, d.bvh_node_count):
        node = d.bvh_nodes[n]
        for ref, lo, hi in ((node.ref0, node.lo0, node.hi0), (node.ref1, node.lo1, node.hi1)):
            if ref != MISS and ref & 0x80000000:
                boxes[ref & 0x7FFFFFFF] = [lo[:], hi[:]]
    b = boxes[inst]
    out[hit] = _outside(rays[hit, :3], rays[hit, 4:7], b[:, 0], b[:, 1], t)
    return out


def _triangle_test(d, rays, hits, hit):
    """The hit instances of the rays `hit` and the float32 triangle test's object-space ray, triangle and t of their hits."""
    inst = hits["inst"][hit].astype(np.int64)
    w = np.array([d.instances[i].world_to_object[:] for i in range(d.instance_count)], np.float32).reshape(-1, 3, 4)[inst]
    o, dd = rays[hit, :3], rays[hit, 4:7]
    oo = np.stack([_fma(w[:, a, 0], o[:, 0], _fma(w[:, a, 1], o[:, 1], _fma(w[:, a, 2], o[:, 2], w[:, a, 3]))) for a in range(3)], axis=1)
    od = np.stack([_fma(w[:, a, 0], dd[:, 0], _fma(w[:, a, 1], dd[:, 1], w[:, a, 2] * dd[:, 2])) for a in range(3)], axis=1)
    verts = np.array([v.p[:] for v in d.vertices[:d.vertex_count]], np.float32)
    tris = np.array([(t.i0, t.i1, t.i2) for t in d.triangles[:d.triangle_count]], np.int64)
    meshes = [d.meshes[d.instances[i].mesh] for i in range(d.instance_count)]
    first = np.array([m.triangle_offset for m in meshes])[inst] + hits["prim"][hit]
    voff = np.array([m.vertex_offset for m in meshes])[inst]
    p = verts[tris[first] + voff[:, None]]
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    pvec = _fcross(od, e2)
    with np.errstate(divide="ignore"):
        inv_det = np.float32(1.0) / _fdot(e1, pvec)
    t = _fdot(e2, _fcross(oo - p[:, 0], e1)) * inv_det
    return inst, oo, od, p, t


def _outside(o, dd, lo, hi, t):
    """In exact arithmetic: the ray o + t dd misses the box [lo, hi], or t lies outside its entry and exit distances by more than
    the box test's margin (kSlabExitScale, 2^-20 relative)."""
    o64, d64 = o.astype(np.float64), dd.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        t0, t1 = (lo - o64) / d64, (hi - o64) / d64
    inside = (o64 >= lo) & (o64 <= hi)  # axes the ray is parallel to: all or nothing
    near = np.where(d64 == 0, np.where(inside, -np.inf, np.inf), np.minimum(t0, t1)).max(axis=1)
    far = np.where(d64 == 0, np.where(inside, np.inf, -np.inf), np.maximum(t0, t1)).min(axis=1)
    t = t.astype(np.float64)
    return (near > far) | (t < near - 2.0 ** -20 * np.abs(near)) | (t > far + 2.0 ** -20 * np.abs(far))


def assert_few_exempt(c, what):
    """The exemption stays the exception: under 2 % of c's near rays and under 8 % of all its rays."""
    near = c.loose[:len(c.base)].mean()
    assert near < 0.02 and c.loose.mean() < 0.08, f"{what}: {near:.2%} of the near rays and {c.loose.mean():.2%} of all are exempt"


def differ(got, ref):
    return ((got["inst"] != ref["inst"]) | (got["prim"] != ref["prim"])
            | (got["bary"].view(np.uint32) != ref["bary"].view(np.uint32)).any(axis=1))


def assert_equal_hits(got, ref, loose, what):
    """Bit-identical hit records, except on the `loose` rays (outside_own_box, outside_instance_box)."""
    bad = np.flatnonzero(differ(got, ref) & ~loose)
    lost = int(((got["inst"] == MISS) & (ref["inst"] != MISS))[bad].sum())
    assert not len(bad), f"{what}: {len(bad)} of {len(got)} rays differ from the brute force ({lost} lost a hit), first: {bad[:5].tolist()}"


class Case:
    """One scene of the catalogue (or any (meshes, instances)) with its ray set (seed), the brute force's closest and any hits of
    every ray and the rays exempt from bit-exactness (`loose`): those whose hit lies outside its triangle's own box (`own`) or its
    instance's box (`instance`).

    A frame of an update chain (`frame` given: its lamp is placed around the whole chain) aims its rays at its own instances only,
    sized by their extent: the lamp's place, and the other frames' sizes, must not set the scale of a frame's vertex and edge
    rays.  A catalogue scene's lamp sits just above the scene and is aimed at with it."""

    def __init__(self, meshes, instances, seed, frame=None):
        self.scene = Scene.from_source(scene_text(meshes, instances, frame), REPO)
        self.desc = self.scene.desc()
        self.tris, self.ids, self.mags = desc_triangles(self.desc)
        aim = None if frame is None else self.ids[:, 0] != self.desc.instance_count - 1  # the lamp is the last instance
        self.base, self.far = make_rays(self.desc, self.tris, self.ids, seed=seed, aim=aim)
        self.rays = np.concatenate([self.base] + self.far)
        self.brute, _ = O.trace(self.desc, self.rays, brute=True)
        self.occ_brute, _ = O.trace(self.desc, self.rays, any_hit=True, brute=True)
        self.own = outside_own_box(self.desc, self.rays, self.brute)
        self.instance = outside_instance_box(self.desc, self.rays, self.brute)
        self.loose = self.own | self.instance


# ---- update transitions -----------------------------------------------------------------------------------------------------------

def _moved(name, moves):
    """The catalogue scene `name` with the instances {k: object_to_world} of `moves` moved."""
    meshes, instances = CATALOGUE[name]
    return meshes, [(m, moves.get(k, xf), vis) for k, (m, xf, vis) in enumerate(instances)]


def _deformed(name, fn):
    """The catalogue scene `name` with its (only) mesh's positions replaced by fn(positions), its triangles kept."""
    (p, idx), = CATALOGUE[name][0]
    return [(fn(p.copy()), idx)], CATALOGUE[name][1]


def _replaced(meshes, instances, k, mesh):
    return [mesh if j == k else m for j, m in enumerate(meshes)], instances


def _shuffled(p):
    return p[np.random.default_rng(5).permutation(len(p))]


def _collapsed(p):
    """Every triangle onto the first one (the scene's indices are 0, 1, 2, 3, ...): exact ties everywhere."""
    return np.tile(p[:3], (len(p) // 3, 1))


def _transitions():
    """name -> (step, frames): a chain of scenes (meshes, instances) that starts and ends at the same frame, each frame reached
    from the one before it by `step` - "update" (lrk_update_instances), "deform" (lrk_update_meshes, same triangles) or
    "replace" (lrk_replace_meshes)."""
    skew = _rotation((0.3, -1.0, 0.5), 1.1) @ np.diag([-1.0, 0.25, 3.0])
    at = lambda linear, t=(0.3, 0.1, -0.2): _affine(linear, t)  # noqa: E731
    two = CATALOGUE["two_instances"][1]
    perm = np.random.default_rng(11).permutation(len(CATALOGUE["instances_1000"][1]))
    moves = {
        "mirrored": _moved("two_instances", {0: at(skew)}),
        "scale_1e-3": _moved("two_instances", {0: at(1e-3 * np.eye(3))}),
        "scale_1e3": _moved("two_instances", {0: at(1e3 * np.eye(3))}),
        "translate_1e4": _moved("two_instances", {0: _affine(translate=(1e4, -3e3, 5e3))}),
        "onto_another": _moved("two_instances", {1: two[0][1]}),  # exact ties: both instances on one transform
        "reordered_1000": _moved("instances_1000", {k: CATALOGUE["instances_1000"][1][j][1] for k, j in enumerate(perm)}),
    }
    out = {f"move_{k}": ("update", [CATALOGUE[base], b, CATALOGUE[base]])
           for k, b in moves.items() for base in ["instances_1000" if k == "reordered_1000" else "two_instances"]}
    out["move_rotated_cancelling"] = ("update", [CATALOGUE["cancelling_instance"], CATALOGUE["rotated_cancelling_instance"],
                                                 CATALOGUE["cancelling_instance"]])
    deforms = {
        "flatten": ("rotated_mirrored_instance", lambda p: p * [1.0, 0.0, 1.0]),
        "scale_1e4": ("fan_64", lambda p: p * 1e4),
        "scale_1e-4": ("scaled_instance", lambda p: p * 1e-4),
        "offset_1e4": ("instances_1000", lambda p: p + [1e4, -3e3, 5e3]),
        "shuffled": ("same_transform_twice", _shuffled),
        "collapsed": ("graded", _collapsed),
    }
    for k, (base, fn) in deforms.items():
        out[f"deform_{k}"] = ("deform", [CATALOGUE[base], _deformed(base, fn), CATALOGUE[base]])
    # three meshes side by side, each replaced in turn (first, middle, last) by a catalogue mesh and back: the unchanged meshes'
    # hierarchies move towards the front and back again, or the other way round
    trio = ([CATALOGUE["same_transform_twice"][0][0], CATALOGUE["fan_8"][0][0], CATALOGUE["flat_grid"][0][0]],
            [(k, _affine(translate=(1.2 * (k - 1), 0.0, 0.0)), True) for k in range(3)])
    for j, name in enumerate(["tris_1", "tris_2", "tris_3", "tris_4", "tris_5", "tris_8", "tris_9", "tris_33", "copies_12",
                              "fan_64", "graded"]):
        out[f"replace_{j % 3}_{name}"] = ("replace", [trio, _replaced(*trio, j % 3, CATALOGUE[name][0][0]), trio])
    return out


TRANSITIONS = _transitions()
# the least share of a chain frame's rays that hit, where it is not 0.2: frames whose own geometry is sparse, so that rays jittered
# by 1e-5 of the frame's size pass most of it from far away (two instances 0.1 wide and 1e4 apart; 1000 clusters 0.1 wide spread
# over 2.4e4 - the catalogue's far_mesh_instances_1000)
SPARSE_FRAMES = {("move_translate_1e4", 1): 0.02, ("deform_offset_1e4", 1): 0.01}


def union(frames):
    """One (meshes, instances) holding every frame's meshes and instances: what scene_text places a chain's lamp and camera by."""
    meshes, instances = [], []
    for ms, insts in frames:
        instances += [(len(meshes) + m, xf, vis) for m, xf, vis in insts]
        meshes += list(ms)
    return meshes, instances


_CHAIN_CASES: dict[tuple[str, int], Case] = {}


def chain_case(name, k) -> Case:
    """Frame k of the transition `name`, its lamp and camera placed around the whole chain, with its ray set (one per frame)."""
    if (name, k) not in _CHAIN_CASES:
        frames = TRANSITIONS[name][1]
        first = next(j for j, f in enumerate(frames) if f is frames[k])  # a frame the chain returns to shares its first case
        if (name, first) not in _CHAIN_CASES:
            _CHAIN_CASES[(name, first)] = Case(*frames[first], seed=1000 + list(TRANSITIONS).index(name) * 8 + first,
                                               frame=union(frames))
        _CHAIN_CASES[(name, k)] = _CHAIN_CASES[(name, first)]
    return _CHAIN_CASES[(name, k)]
