"""Deformed frames for the mesh-update tests (lrk_update_meshes, DESIGN.md §4 (Mesh deformation)), shared by
tests/test_mesh_update_cpu.py and tests/test_mesh_update.py: frame pairs and chains whose meshes keep their layout and triangles while
their vertex positions move, and the helpers that read meshes out of flattened descriptions."""
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


def meshes(d):
    return array(d.meshes, d.mesh_count, F.Mesh, np.uint32, 8)


def deformed_meshes(a, b):
    """The mesh ids whose vertex records differ between the descriptions a and b (same mesh layout), and B's records of each."""
    va, vb, m = vertices(a), vertices(b), meshes(b)
    ids, parts = [], []
    for k, (off, cnt) in enumerate(m[:, :2]):
        if not np.array_equal(va[off:off + cnt].view(np.uint32), vb[off:off + cnt].view(np.uint32)):
            ids.append(k)
            parts.append(vb[off:off + cnt])
    return ids, parts


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


def cornell(deformed):
    text = scenes.cornell_box(resolution=(48, 48), spp=4)
    return deform_inline(text, "tall_box", _shear) if deformed else text


def textured_room(deformed):
    text = scenes.textured_room(resolution=(48, 32), spp=4, wrappers=True)
    return deform_inline(text, "screen", _bend) if deformed else text


def media_box(deformed):
    text = scenes.media_box(resolution=(32, 32))
    return deform_inline(text, "tall_box", _shear) if deformed else text


def sheet(time, **kw):
    return scenes.wavy_sheet(resolution=(48, 32), spp=4, segments=(16, 10), time=time, **kw)


def globe(wobble):
    return scenes.emissive_globe(resolution=(48, 48), spp=8, subdivision=3, wobble=wobble)


# frame chains whose meshes deform; every frame after the first is reached from the one before it by lrk_update_meshes
FRAMES = {
    "cornell_tall_box": lambda: [cornell(False), cornell(True)],
    "wavy_sheet": lambda: [sheet(0.0), sheet(0.4), sheet(0.9, amplitude=0.08)],
    "textured_room_screen": lambda: [textured_room(False), textured_room(True)],
    "media_box": lambda: [media_box(False), media_box(True)],
}

EMISSIVE_FRAMES = {
    "emissive_sheet": lambda: [sheet(0.0, emissive=True), sheet(0.6, emissive=True)],
    "wobbling_globe": lambda: [globe(0.0), globe(0.15), globe(-0.1)],
}
