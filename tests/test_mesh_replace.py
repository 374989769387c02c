"""Mesh replacement (lrk_replace_meshes, DESIGN.md §4 (Mesh replacement)) on the GPU, in both arithmetic modes: a context that
uploaded frame A and replaced meshes with B's vertices and triangles renders, traces, writes G-buffers and renders adaptively what a
context that uploaded B does, bit for bit; refused replacements change nothing."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import scene_update_checks as U
import scene_update_frames as S
from luisarender_b200 import _ffi as F
from scene_update_checks import make  # noqa: F401  (the context fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
@pytest.mark.parametrize("name", list(S.REPLACE_FRAMES))
def test_mesh_replace_equals_fresh_upload(name, device_bvh, make):
    frames = [S.scene(t) for t in S.REPLACE_FRAMES[name]()]
    U.check_frames(make, frames, U.replace_to, 4, {"device_bvh": device_bvh})


LIGHT_OPTIONS = [{}, {"light_tree": True, "light_tree_triangles": True},
                 {"light_tree": True, "light_tree_triangles": True, "light_solid_angle": True},
                 {"light_tree": True, "light_tree_triangles": True, "light_receiver": True}]


@pytest.mark.parametrize("options", LIGHT_OPTIONS, ids=["uniform", "tree_triangles", "solid_angle", "receiver"])
@pytest.mark.parametrize("name", list(S.REPLACE_EMISSIVE_FRAMES))
def test_replaced_emitters_rebuild_alias_tables_and_light_trees(name, options, make):
    frames = [S.scene(t) for t in S.REPLACE_EMISSIVE_FRAMES[name]()]
    U.check_frames(make, frames, U.replace_to, 8, options, trace=options == {})


def _sheet(segments, time, shift=0.0, amplitude=0.08):
    return S.scene(S.sheet(time, segments, shift, amplitude=amplitude))


def test_replace_update_and_instance_moves_compose(make):
    """Replace, refit the replaced mesh (lrk_update_meshes after lrk_replace_meshes), move instances, replace and refit again:
    every step equals a fresh upload of its frame."""
    steps = [(None, ((16, 10), 0.0, 0.0)), (U.replace_to, ((24, 16), 0.0, 0.0)), (U.deform_to, ((24, 16), 0.5, 0.0)),
             (U.update_to, ((24, 16), 0.5, 0.2)), (U.replace_to, ((8, 5), 0.5, 0.2)), (U.deform_to, ((8, 5), 1.1, 0.2))]
    frames = [_sheet(*args) for _, args in steps]
    r = make()
    r.upload(frames[0].desc())
    for (step, _), prev, cur in zip(steps[1:], frames, frames[1:]):
        step(r, prev.desc(), cur.desc())
        U.check_against_fresh(make, r, cur, 4, {})


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
def test_replace_with_the_uploaded_arrays_keeps_the_film(device_bvh, make):
    s = _sheet((16, 10), 0.3)
    d = s.desc()
    r = make(device_bvh=device_bvh)
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    v, t, m = S.vertices(d), S.triangles(d), S.meshes(d)
    ids = np.arange(d.mesh_count)[::-1]
    r.replace_meshes(ids, [v[m[k, 0]:m[k, 0] + m[k, 1]] for k in ids], [t[m[k, 2]:m[k, 2] + m[k, 3]] for k in ids])
    assert not r.film(raw=True).any()  # the call clears the film
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)


def test_refit_then_rebuild_of_a_large_deformation(make):
    """The amplitude-0.3 sheet deformed by a refit, then given a fresh hierarchy by replacing it with its own arrays."""
    a, b = _sheet((24, 16), 0.0, amplitude=0.3), _sheet((24, 16), 0.6, amplitude=0.3)
    r = make()
    r.upload(a.desc())
    U.deform_to(r, a.desc(), b.desc())
    U.check_against_fresh(make, r, b, 4, {})
    d = b.desc()
    k = S.deformed_meshes(a.desc(), d)[0]
    m = S.meshes(d)
    r.replace_meshes(k, [S.vertices(d)[m[j, 0]:m[j, 0] + m[j, 1]] for j in k], [S.triangles(d)[m[j, 2]:m[j, 2] + m[j, 3]] for j in k])
    U.check_against_fresh(make, r, b, 4, {})


def test_gbuffer_adaptive_and_shards_after_a_mesh_replace(make):
    U.check_gbuffer_adaptive_and_shards(make, _sheet((16, 10), 0.3), _sheet((24, 16), 0.3), U.replace_to)


def test_refused_mesh_replacements_change_nothing(make):
    a, b = _sheet((16, 10), 0.3), _sheet((24, 16), 0.3)
    d = a.desc()
    ids, verts, tris = S.replaced_meshes(d, b.desc())
    k, v, t = ids[0], verts[0], tris[0]
    empty = make()
    with pytest.raises(RuntimeError, match=r"\(-1\).*no scene"):
        empty.replace_meshes([k], [v], [t])
    r = make()
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    nan = v.copy()
    nan[3, 1] = np.inf
    past = t.copy()
    past[5, 2] = len(v)
    U.check_refusals(r, film, [(lambda: r.replace_meshes([d.mesh_count], [v], [t]), "out of range"),
                               (lambda: r.replace_meshes([k, k], [v, v], [t, t]), "repeated"),
                               (lambda: r.replace_meshes([k], [v[:0]], [t[:0]]), "no vertices or no triangles"),
                               (lambda: r.replace_meshes([k], [v], [t[:0]]), "no vertices or no triangles"),
                               (lambda: r.replace_meshes([k], [v], [past]), "triangle index out of range"),
                               (lambda: r.replace_meshes([k], [nan], [t]), "non-finite")])
    # a hierarchy whose instance level is not its last max(visible, 2) - 1 nodes (one unused node behind it) cannot be laid out again
    nodes = S.array(d.bvh_nodes, d.bvh_node_count, F.BvhNode, np.uint32, 16)
    padded = np.ascontiguousarray(np.concatenate([nodes, np.zeros((1, 16), np.uint32)]))
    h = F.SceneDesc()
    C.memmove(C.byref(h), C.byref(d), C.sizeof(F.SceneDesc))
    h.bvh_nodes = padded.ctypes.data_as(C.POINTER(F.BvhNode))
    h.bvh_node_count = len(padded)
    u = make()
    u.upload(h)
    u.render(0, 4)
    assert np.array_equal(u.film(raw=True), film)
    with pytest.raises(RuntimeError, match=r"\(-5\).*instance level"):
        u.replace_meshes([k], [v], [t])
    assert np.array_equal(u.film(raw=True), film)
