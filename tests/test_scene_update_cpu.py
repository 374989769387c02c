"""Scene updates without a GPU: the animated instanced-spheres frames and the world-to-object inverse that the flattening and
lrk_update_instances share (luisarender_b200/csrc/device/affine_inverse.h)."""
from __future__ import annotations

import ctypes as C
import hashlib
from pathlib import Path

import numpy as np
import pytest

from host_harness import DEVICE, load
from luisarender_b200 import _ffi as F
from luisarender_b200 import scenes
from luisarender_b200.api import Scene

REPO = Path(__file__).resolve().parents[1]
SMALL = dict(resolution=(64, 36), spp=4, big_subdivision=4, small_subdivision=2, small_count=12)

# sha256 of the scene texts before instanced_spheres had a `time`: the still scene must stay byte for byte what every fixture,
# golden render and benchmark of it was made from
STILL_TEXTS = {
    "c3": ({}, "40a924c93e784387d77e3ef13ff6a3432639e2e8925a7a9639b04da30a689314"),
    "small": (SMALL, "4ccc5fbc6c7fa481c0518bf887f6c01ab66a04794a9fa01ac4ba0e1f7f6cda25"),
    "medium": ({"medium": True}, "9ec77cd79185841d69806156d83f753aaf6f734f058277f89355a9cc44a2d6c5"),
}


@pytest.mark.parametrize("name", list(STILL_TEXTS))
def test_time_zero_is_the_still_scene(name):
    kw, digest = STILL_TEXTS[name]
    assert hashlib.sha256(scenes.instanced_spheres(**kw, time=0.0).encode()).hexdigest() == digest
    assert scenes.instanced_spheres(**kw) == scenes.instanced_spheres(**kw, time=0.0)
    assert hashlib.sha256(scenes.many_lights().encode()).hexdigest() == "c9e29d18d42cbf1983243463605818e8135833b059572dfc9111b70e90ced8b4"


def _bytes(ptr, count, cls):
    return C.string_at(C.cast(ptr, C.c_void_p), count * C.sizeof(cls)) if count else b""


def _instances(d):
    return [d.instances[i] for i in range(d.instance_count)]


@pytest.mark.parametrize("make", [lambda t: scenes.instanced_spheres(**SMALL, time=t),
                                  lambda t: scenes.many_lights(resolution=(48, 32), spp=4, count=12, big_subdivision=3, small_subdivision=2, time=t)],
                         ids=["spheres", "many_lights"])
def test_frames_differ_only_in_the_instance_transforms(make):
    frames = [Scene.from_source(make(t), REPO) for t in (0.0, 0.5, 2.0)]
    d0 = frames[0].desc()
    for f in frames[1:]:
        d = f.desc()
        for ptr, count, cls in (("vertices", "vertex_count", F.Vertex), ("triangles", "triangle_count", F.Triangle),
                                ("alias", "triangle_count", F.AliasEntry), ("pdf", "triangle_count", C.c_float), ("meshes", "mesh_count", F.Mesh),
                                ("surfaces", "surface_count", F.Surface), ("lights", "light_count", F.Light),
                                ("light_handles", "light_count", F.LightHandle), ("tri_verts", "tri_slot_count", C.c_float * 12)):
            assert getattr(d, count) == getattr(d0, count)
            assert _bytes(getattr(d, ptr), getattr(d, count), cls) == _bytes(getattr(d0, ptr), getattr(d0, count), cls), ptr
        # the meshes' hierarchies come first and are the same; the instance level behind them has the same size
        assert d.tlas_root == d0.tlas_root and d.bvh_node_count == d0.bvh_node_count
        assert _bytes(d.bvh_nodes, d.tlas_root, F.BvhNode) == _bytes(d0.bvh_nodes, d0.tlas_root, F.BvhNode)
        assert bytes(d.camera) == bytes(d0.camera)
        moved = 0
        for a, b in zip(_instances(d0), _instances(d)):
            assert list(a.handle) == list(b.handle) and a.mesh == b.mesh and a.visible == b.visible
            rows_a, rows_b = np.array(a.object_to_world).reshape(3, 4), np.array(b.object_to_world).reshape(3, 4)
            assert np.array_equal(rows_a[:, :3], rows_b[:, :3])  # only the translation moves
            moved += not np.array_equal(rows_a, rows_b)
        assert moved == d.instance_count - 3  # every instance but the ground and the two quad lights


@pytest.fixture(scope="module")
def inverse():
    lib = load("affine_inverse_host", [DEVICE / "affine_inverse.h"], ["-O2", "-march=x86-64-v3", "-ffp-contract=off"])
    lib.affine_inverse_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    return lib


@pytest.mark.parametrize("text", [lambda: scenes.flatten_stress(),
                                  *[(lambda k=k: scenes.emissive_globe(resolution=(16, 16), subdivision=2, transform=k)) for k in ("uniform", "stretched", "mirrored")],
                                  *[(lambda t=t: scenes.instanced_spheres(**SMALL, time=t)) for t in (0.0, 0.37, 1.5, -4.0)]],
                         ids=["flatten_stress", "globe_uniform", "globe_stretched", "globe_mirrored", "spheres_t0", "spheres_t0.37", "spheres_t1.5",
                              "spheres_t-4"])
def test_shared_inverse_reproduces_the_flattened_rows(text, inverse):
    d = Scene.from_source(text(), REPO).desc()
    o2w = np.array([list(i.object_to_world) for i in _instances(d)], np.float32)
    w2o = np.array([list(i.world_to_object) for i in _instances(d)], np.float32)
    out = np.full_like(w2o, np.nan)
    assert inverse.affine_inverse_rows(o2w.ctypes.data, out.ctypes.data, len(o2w)) == 0
    assert np.array_equal(out.view(np.uint32), w2o.view(np.uint32))


def test_shared_inverse_refuses_singular_rows(inverse):
    rows = np.array([[1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 5], [1, 2, 3, 0, 2, 4, 6, 0, 0, 0, 1, 0], [2, 0, 0, 1, 0, 2, 0, 1, 0, 0, 2, 1]], np.float32)
    out = np.zeros_like(rows)
    assert inverse.affine_inverse_rows(rows.ctypes.data, out.ctypes.data, 3) == 2
    assert np.array_equal(out[2], np.array([0.5, 0, 0, -0.5, 0, 0.5, 0, -0.5, 0, 0, 0.5, -0.5], np.float32))
