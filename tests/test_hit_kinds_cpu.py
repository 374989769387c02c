"""The hit kinds of the material sort without a GPU: csrc/device/hit_kinds.h, the table lrk_upload_scene and the kernels share,
compiled for the host.  Its surface -> kind mapping is checked against a restatement over every surface of the scene library and of
the reference-render scenes, and the set of kinds that always run in IEEE arithmetic is pinned."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import host_harness
from luisarender_b200 import _ffi as F
from luisarender_b200 import scenes
from luisarender_b200.api import Scene

REPO = Path(__file__).resolve().parents[1]
SURFACE_DISNEY, SURFACE_LAYERED = 1, 7
SURFACE_DISNEY_TRANSMISSIVE, SURFACE_DISNEY_THIN = 16, 64


@pytest.fixture(scope="module")
def lib():
    h = host_harness.load("hit_kinds_host", [host_harness.DEVICE / "hit_kinds.h", REPO / "include" / "lrk.h"], ["-O2"])
    h.hit_kinds_of_surfaces.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    h.hit_kinds_always_strict_mask.restype = C.c_uint32
    h.hit_kinds_count.restype = C.c_uint32
    return h


def expected_kind(s) -> int:
    """Matte 1, Disney 2, Mirror 3, Glass 4, Plastic 5, Metal 6, Mix 7, transmissive Disney 8, Layered 9, thin Disney 10."""
    if s.type == SURFACE_DISNEY and s.flags & SURFACE_DISNEY_THIN:
        return 10
    if s.type == SURFACE_DISNEY and s.flags & SURFACE_DISNEY_TRANSMISSIVE:
        return 8
    if s.type == SURFACE_LAYERED:
        return 9
    return s.type + 1


def _library_sources():
    yield "cornell_box", scenes.cornell_box()
    yield "materials_box", scenes.materials_box()
    yield "layered_box", scenes.layered_box()
    yield "textured_materials", scenes.textured_materials()
    yield "media_box", scenes.media_box()
    yield "textured_room", scenes.textured_room()
    yield "environment_scene", scenes.environment_scene()
    z = np.load(REPO / "tests" / "golden" / "ref_renders.npz")
    for key in z.files:
        if key.endswith("/scene"):
            yield key, bytes(z[key]).decode()


def test_hit_kind_of_matches_the_restatement_on_every_library_surface(lib):
    assert F.SURFACE_DISNEY_TRANSMISSIVE == SURFACE_DISNEY_TRANSMISSIVE
    seen = set()
    for name, src in _library_sources():
        d = Scene.from_source(src, REPO).desc()
        n = d.surface_count
        kinds = np.zeros(n, np.uint32)
        lib.hit_kinds_of_surfaces(C.cast(d.surfaces, C.c_void_p), n, kinds.ctypes.data)
        want = [expected_kind(d.surfaces[i]) for i in range(n)]
        assert kinds.tolist() == want, name
        seen.update(want)
    assert seen == set(range(1, 11)), sorted(seen)  # every kind with a surface occurs somewhere


def test_thin_takes_precedence_over_transmissive(lib):
    """A Disney record with both flags is a thin Disney surface; no library scene has one."""
    surfaces = (F.Surface * 4)()
    for s, flags in zip(surfaces, [SURFACE_DISNEY_TRANSMISSIVE | SURFACE_DISNEY_THIN, SURFACE_DISNEY_TRANSMISSIVE, SURFACE_DISNEY_THIN, 0]):
        s.type, s.flags = SURFACE_DISNEY, flags
    kinds = np.zeros(4, np.uint32)
    lib.hit_kinds_of_surfaces(C.cast(surfaces, C.c_void_p), 4, kinds.ctypes.data)
    assert kinds.tolist() == [10, 8, 10, 2] == [expected_kind(s) for s in surfaces]


def test_always_strict_kinds(lib):
    """Mirror, Glass, Plastic, Metal, Mix, Layered and thin Disney run in IEEE arithmetic whatever the option strict_math says."""
    assert lib.hit_kinds_count() == 11
    mask = lib.hit_kinds_always_strict_mask()
    assert {k for k in range(32) if mask >> k & 1} == {3, 4, 5, 6, 7, 9, 10}
