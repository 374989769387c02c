"""Frames for the scene-update tests (DESIGN.md §4: Scene updates, Mesh deformation, Mesh replacement), shared by
tests/test_scene_update*.py, tests/test_mesh_update*.py and tests/test_mesh_replace*.py: one dict of frame chains per kind of
update, in which every frame after the first is reached from the one before it by that update, and the helpers that read meshes
out of flattened descriptions."""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

import numpy as np

from luisarender_b200 import _ffi as F
from luisarender_b200 import scenes
from luisarender_b200.api import Scene

REPO = Path(__file__).resolve().parents[1]


def scene(text):
    return Scene.from_source(text, REPO)


def array(ptr, count, cls, dtype=np.float32, width=None):
    """count records of the ctypes type cls at ptr as a numpy array of `dtype` (a copy), reshaped to [count, width]."""
    raw = C.string_at(C.cast(ptr, C.c_void_p), count * C.sizeof(cls)) if count else b""
    a = np.frombuffer(raw, dtype=dtype).copy()
    return a.reshape(count, -1) if width is None else a.reshape(count, width)


def vertices(d):
    return array(d.vertices, d.vertex_count, F.Vertex, width=8)


def triangles(d):
    return array(d.triangles, d.triangle_count, F.Triangle, np.uint32, 3)


def meshes(d):
    return array(d.meshes, d.mesh_count, F.Mesh, np.uint32, 8)


def rows(d):
    """Every instance's object-to-world rows [n, 3, 4]."""
    return np.array([list(d.instances[i].object_to_world) for i in range(d.instance_count)], np.float32).reshape(-1, 3, 4)


def deformed_meshes(a, b):
    """The mesh ids whose vertex records differ between the descriptions a and b (same mesh layout), and B's records of each."""
    va, vb, m = vertices(a), vertices(b), meshes(b)
    ids, parts = [], []
    for k, (off, cnt) in enumerate(m[:, :2]):
        if not np.array_equal(va[off:off + cnt].view(np.uint32), vb[off:off + cnt].view(np.uint32)):
            ids.append(k)
            parts.append(vb[off:off + cnt])
    return ids, parts


def replaced_meshes(a, b):
    """The mesh ids whose vertex or triangle records differ between the descriptions a and b (same mesh count), and B's vertex
    [n, 8] and local triangle [m, 3] arrays of each."""
    assert a.mesh_count == b.mesh_count
    va, vb, ta, tb = vertices(a), vertices(b), triangles(a), triangles(b)
    ma, mb = meshes(a), meshes(b)
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


def move(text, shape, srt):
    """The scene text with `transform : SRT { srt }` added to the definition of the shape `shape`."""
    pattern = rf"(Shape {shape} : \w+ \{{)"
    assert len(re.findall(pattern, text)) == 1
    return re.sub(pattern, rf"\1 transform : SRT {{ {srt} }}", text)


def deform_inline(text, shape, fn):
    """The scene text with the positions of the InlineMesh `shape` replaced by fn(positions [n, 3] float64)."""
    pattern = rf"(Shape {shape} : InlineMesh \{{\s*positions \{{)([^}}]*)(\}})"
    found = re.findall(pattern, text)
    assert len(found) == 1
    def repl(m):
        p = np.array([float(x) for x in m.group(2).split(",")], np.float64).reshape(-1, 3)
        q = fn(p)
        return m.group(1) + " " + ", ".join(repr(float(x)) for x in q.reshape(-1)) + " " + m.group(3)
    return re.sub(pattern, repl, text)


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


def _shear(p):  # the tall box leans by 0.25 over its height and its top grows
    q = p.copy()
    q[:, 0] += 0.25 * p[:, 1] / 1.2
    q[:, 2] -= 0.1 * p[:, 1] / 1.2
    q[:, 1] *= 1.0 + 0.08 * (p[:, 1] > 0.0)
    return q


def _bend(p):  # the screen's top edge folds forwards
    q = p.copy()
    q[2:, 2] += 0.35
    q[3, 0] -= 0.1
    return q


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


def cornell():
    return scenes.cornell_box(resolution=(48, 48), spp=4)


def cornell_ends():
    """The Cornell box with its first mesh (the floor) and its last (the emissive light) each split into a finer grid."""
    floor, _, _ = grid([[-1.01, 0.0, 0.99], [1.0, 0.0, 0.99], [1.0, 0.0, -1.04], [-0.99, 0.0, -1.04]], 5, 4)
    light, _, _ = grid([[-0.24, 1.98, 0.16], [-0.24, 1.98, -0.22], [0.23, 1.98, -0.22], [0.23, 1.98, 0.16]], 3, 2)
    text = replace_inline(cornell(), "floor", floor, grid(np.zeros((4, 3)), 5, 4)[1])
    return replace_inline(text, "light", light, grid(np.zeros((4, 3)), 3, 2)[1])


def spheres(time):
    return scenes.instanced_spheres(resolution=(64, 36), spp=4, big_subdivision=4, small_subdivision=2, small_count=12, time=time)


def flatten_stress(moved):
    text = scenes.flatten_stress()
    if moved:  # a nested Instance's SRT, a Stack member (an emitter) and a Group's Matrix
        for old, new in (("translate { 2.2, 0.0, -1.6 }", "translate { 2.5, 0.2, -1.1 }"), ("translate { 0.0, 2.6, 0.0 }", "translate { 0.3, 2.4, 0.2 }"),
                         ("0.8, 0.0, 0.0, -1.5,", "0.7, 0.1, 0.0, -1.2,")):
            assert text.count(old) == 1
            text = text.replace(old, new)
    return text


def globe(spp=8, subdivision=3, **kw):
    return scenes.emissive_globe(resolution=(48, 48), spp=spp, subdivision=subdivision, **kw)


def transformed_globe(kind):
    """emissive_globe frames over one Sphere mesh: "uniform" (SRT), "stretched" (Matrix) and "mirrored" (the stretched frame's
    Matrix replaced by one of negative determinant)."""
    if kind != "mirrored":
        return globe(spp=4, transform=kind)
    m = "transform : Matrix { m { -0.25, 0.0, 0.0, 0.1, 0.0, 0.25, 0.0, 1.1, 0.0, 0.0, 0.25, -0.35, 0.0, 0.0, 0.0, 1.0 } }"
    text, n = re.subn(r"transform : Matrix \{ m \{[^}]*\} \}", m, globe(spp=4, transform="stretched"))
    assert n == 1
    return text


def textured_room():
    return scenes.textured_room(resolution=(48, 32), spp=4, wrappers=True)


def moved_textured_room():
    """The textured room with wrappers: the OBJ cube turned and moved, the alpha-tested screen moved."""
    old = "rotate { 0.0, 1.0, 0.0, 30.0 } translate { -0.6, 0.4, -0.3 }"
    text = textured_room()
    assert text.count(old) == 1
    return move(text.replace(old, "rotate { 0.0, 1.0, 0.0, 50.0 } translate { -0.4, 0.5, -0.1 }"), "screen", "translate { -0.1, 0.0, 0.2 }")


def replaced_textured_room():
    pos, tris, uvs = grid([[0.2, 0.0, 1.0], [1.6, 0.0, 0.6], [1.6, 1.3, 0.6], [0.2, 1.3, 1.0]], 8, 6)
    pos[:, 2] += 0.08 * np.sin(np.pi * uvs[:, 1:2] * 2.0)[:, 0]  # a gently folded screen, so that the new triangles are not coplanar
    return replace_inline(textured_room(), "screen", pos, tris, uvs)


def media_box():
    return scenes.media_box(resolution=(32, 32))


def sheet(time=0.3, segments=(16, 10), shift=0.0, **kw):
    """The wavy sheet at `time`, its instance raised by `shift`."""
    text = scenes.wavy_sheet(resolution=(48, 32), spp=4, segments=segments, time=time, **kw)
    return text.replace("translate { -0.2, 1.15, -0.35 }", f"translate {{ -0.2, {1.15 + shift!r}, -0.35 }}")


# frame chains whose instances (or camera) move: lrk_update_instances
INSTANCE_FRAMES = {
    "cornell_tall_box": lambda: [cornell(), move(cornell(), "tall_box", "rotate { 0.0, 1.0, 0.0, 15.0 } translate { 0.2, 0.0, 0.25 }")],
    "spheres_chain": lambda: [spheres(0.0), spheres(0.5), spheres(1.0)],
    "flatten_stress": lambda: [flatten_stress(False), flatten_stress(True)],
    "textured_room": lambda: [textured_room(), moved_textured_room()],
    "media_box": lambda: [media_box(), move(media_box(), "tall_box", "translate { 0.15, 0.0, 0.2 }")],
}

# frame chains whose meshes deform, keeping their layout and triangles: lrk_update_meshes
DEFORM_FRAMES = {
    "cornell_tall_box": lambda: [cornell(), deform_inline(cornell(), "tall_box", _shear)],
    "wavy_sheet": lambda: [sheet(0.0), sheet(0.4), sheet(0.9, amplitude=0.08)],
    "textured_room_screen": lambda: [textured_room(), deform_inline(textured_room(), "screen", _bend)],
    "media_box": lambda: [media_box(), deform_inline(media_box(), "tall_box", _shear)],
}

DEFORM_EMISSIVE_FRAMES = {
    "emissive_sheet": lambda: [sheet(0.0, emissive=True), sheet(0.6, emissive=True)],
    "wobbling_globe": lambda: [globe(wobble=0.0), globe(wobble=0.15), globe(wobble=-0.1)],
}

# frame chains whose meshes change their vertex and triangle counts while every other part of the scene stays:
# lrk_replace_meshes
REPLACE_FRAMES = {
    "cornell_tall_box": lambda: [cornell(), replace_inline(cornell(), "tall_box", *bevelled_box()), cornell()],
    "wavy_sheet": lambda: [sheet(segments=(16, 10)), sheet(segments=(24, 16)), sheet(segments=(8, 5))],
    "textured_room_screen": lambda: [textured_room(), replaced_textured_room()],
    "media_box": lambda: [media_box(), replace_inline(media_box(), "tall_box", *bevelled_box())],
    "cornell_first_and_last": lambda: [cornell(), cornell_ends(), cornell()],
}

REPLACE_EMISSIVE_FRAMES = {
    "emissive_globe": lambda: [globe(subdivision=3), globe(subdivision=4), globe(subdivision=2)],
}
