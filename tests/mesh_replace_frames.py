"""Frames for the mesh-replacement tests (lrk_replace_meshes, DESIGN.md §4 (Mesh replacement)), shared by
tests/test_mesh_replace_cpu.py and tests/test_mesh_replace.py: frame chains whose meshes change their vertex and triangle counts
while every other part of the scene stays, and the helper that reads the replaced meshes out of two flattened descriptions."""
from __future__ import annotations

import re

import numpy as np

import mesh_update_frames as M
from luisarender_b200 import _ffi as F
from luisarender_b200 import scenes


def triangles(d):
    return M.array(d.triangles, d.triangle_count, F.Triangle, np.uint32, 3)


def replaced_meshes(a, b):
    """The mesh ids whose vertex or triangle records differ between the descriptions a and b (same mesh count), and B's vertex
    [n, 8] and local triangle [m, 3] arrays of each."""
    assert a.mesh_count == b.mesh_count
    va, vb, ta, tb = M.vertices(a), M.vertices(b), triangles(a), triangles(b)
    ma, mb = M.meshes(a), M.meshes(b)
    ids, verts, tris = [], [], []
    for k in range(b.mesh_count):
        (vo_a, vc_a, to_a, tc_a), (vo, vc, to, tc) = ma[k][:4], mb[k][:4]
        if vc == vc_a and tc == tc_a and np.array_equal(va[vo_a:vo_a + vc].view(np.uint32), vb[vo:vo + vc].view(np.uint32)) and \
                np.array_equal(ta[to_a:to_a + tc], tb[to:to + tc]):
            continue
        ids.append(k)
        verts.append(vb[vo:vo + vc].copy())
        tris.append(tb[to:to + tc].copy())
    return ids, verts, tris


def replace_inline(text, shape, positions, indices, uvs=None):
    """The scene text with the InlineMesh `shape`'s positions, indices (and uvs, when given) replaced; its other fields stay."""
    pattern = rf"(Shape {shape} : InlineMesh \{{\n)(.*?)(\n  (?:surface|light) )"
    found = re.findall(pattern, text, flags=re.S)
    assert len(found) == 1

    def numbers(values):
        return ", ".join(repr(float(x)) if isinstance(x, (float, np.floating)) else str(int(x)) for x in np.asarray(values).reshape(-1))

    body = [f"  positions {{ {numbers(np.asarray(positions, np.float64))} }}"]
    if uvs is not None:
        body.append(f"  uvs {{ {numbers(np.asarray(uvs, np.float64))} }}")
    body.append(f"  indices {{ {numbers(np.asarray(indices, np.int64))} }}")
    return re.sub(pattern, lambda m: m.group(1) + "\n".join(body) + m.group(3), text, flags=re.S)


# the footprint of the Cornell box's tall box, counter-clockwise seen from above, and its height
_TALL_FOOT = np.array([[-0.53, 0.09], [0.04, -0.09], [-0.14, -0.67], [-0.71, -0.49]])
_TALL_HEIGHT = 1.2


def bevelled_box(foot=_TALL_FOOT, height=_TALL_HEIGHT, chamfer=0.06, bevel=0.05):
    """A box on the floor over the quad `foot` with its vertical edges chamfered and its top edge bevelled: an octagonal prism to
    height - bevel, a ring that leans in by `bevel` to the top, and the top (no bottom, as the box it replaces): 38 triangles."""
    ring = []
    for i in range(4):
        p, prev, nxt = foot[i], foot[i - 1], foot[(i + 1) % 4]
        ring.append(p + chamfer * (prev - p) / np.linalg.norm(prev - p))
        ring.append(p + chamfer * (nxt - p) / np.linalg.norm(nxt - p))
    ring = np.array(ring)
    centre = ring.mean(axis=0)
    inner = ring + bevel * (centre - ring) / np.linalg.norm(centre - ring, axis=1, keepdims=True)
    pos = [[x, 0.0, z] for x, z in ring] + [[x, height - bevel, z] for x, z in ring] + [[x, height, z] for x, z in inner]
    tris = []
    for i in range(8):
        j = (i + 1) % 8
        tris += [[i, j, 8 + j], [i, 8 + j, 8 + i]]  # side
        tris += [[8 + i, 8 + j, 16 + j], [8 + i, 16 + j, 16 + i]]  # bevel
    tris += [[16, 16 + k + 1, 16 + k] for k in range(1, 7)]  # top fan
    return np.array(pos), np.array(tris)


def grid(corners, nx, ny):
    """A grid of nx x ny quads over the bilinear patch of the four corners (in the order 00, 10, 11, 01), with uvs over [0, 1]^2."""
    c = np.asarray(corners, np.float64)
    u, v = np.meshgrid(np.linspace(0.0, 1.0, nx + 1), np.linspace(0.0, 1.0, ny + 1))
    u, v = u.reshape(-1, 1), v.reshape(-1, 1)
    pos = (1 - u) * (1 - v) * c[0] + u * (1 - v) * c[1] + u * v * c[2] + (1 - u) * v * c[3]
    tris = []
    for j in range(ny):
        for i in range(nx):
            a = j * (nx + 1) + i
            tris += [[a, a + 1, a + nx + 2], [a, a + nx + 2, a + nx + 1]]
    return pos, np.array(tris), np.hstack([u, v])


def cornell(replaced):
    text = scenes.cornell_box(resolution=(48, 48), spp=4)
    if not replaced:
        return text
    return replace_inline(text, "tall_box", *bevelled_box())


def cornell_ends(replaced):
    """The Cornell box with its first mesh (the floor) and its last (the emissive light) each split into a finer grid."""
    text = scenes.cornell_box(resolution=(48, 48), spp=4)
    if not replaced:
        return text
    floor, _, _ = grid([[-1.01, 0.0, 0.99], [1.0, 0.0, 0.99], [1.0, 0.0, -1.04], [-0.99, 0.0, -1.04]], 5, 4)
    light, _, _ = grid([[-0.24, 1.98, 0.16], [-0.24, 1.98, -0.22], [0.23, 1.98, -0.22], [0.23, 1.98, 0.16]], 3, 2)
    text = replace_inline(text, "floor", floor, grid(np.zeros((4, 3)), 5, 4)[1])
    return replace_inline(text, "light", light, grid(np.zeros((4, 3)), 3, 2)[1])


def textured_room(replaced):
    text = scenes.textured_room(resolution=(48, 32), spp=4, wrappers=True)
    if not replaced:
        return text
    pos, tris, uvs = grid([[0.2, 0.0, 1.0], [1.6, 0.0, 0.6], [1.6, 1.3, 0.6], [0.2, 1.3, 1.0]], 8, 6)
    pos[:, 2] += 0.08 * np.sin(np.pi * uvs[:, 1:2] * 2.0)[:, 0]  # a gently folded screen, so that the new triangles are not coplanar
    return replace_inline(text, "screen", pos, tris, uvs)


def media_box(replaced):
    text = scenes.media_box(resolution=(32, 32))
    if not replaced:
        return text
    return replace_inline(text, "tall_box", *bevelled_box())


def sheet(segments, **kw):
    return scenes.wavy_sheet(resolution=(48, 32), spp=4, segments=segments, time=0.3, **kw)


def globe(subdivision):
    return scenes.emissive_globe(resolution=(48, 48), spp=8, subdivision=subdivision)


# frame chains whose meshes change their vertex and triangle counts; every frame after the first is reached from the one before it
# by lrk_replace_meshes
FRAMES = {
    "cornell_tall_box": lambda: [cornell(False), cornell(True), cornell(False)],
    "wavy_sheet": lambda: [sheet((16, 10)), sheet((24, 16)), sheet((8, 5))],
    "textured_room_screen": lambda: [textured_room(False), textured_room(True)],
    "media_box": lambda: [media_box(False), media_box(True)],
    "cornell_first_and_last": lambda: [cornell_ends(False), cornell_ends(True), cornell_ends(False)],
}

EMISSIVE_FRAMES = {
    "emissive_globe": lambda: [globe(3), globe(4), globe(2)],
}
