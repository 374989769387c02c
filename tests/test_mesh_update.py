"""Mesh updates (lrk_update_meshes, DESIGN.md §4 (Mesh deformation)) on the GPU, in both arithmetic modes: a context that uploaded
frame A and was updated to B's vertices renders, traces, writes G-buffers and renders adaptively what a context that uploaded B
does, bit for bit; refused updates change nothing."""
from __future__ import annotations

import numpy as np
import pytest

import scene_update_checks as U
import scene_update_frames as S
from scene_update_checks import make  # noqa: F401  (the context fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
@pytest.mark.parametrize("name", list(S.DEFORM_FRAMES))
def test_mesh_update_equals_fresh_upload(name, device_bvh, make):
    frames = [S.scene(t) for t in S.DEFORM_FRAMES[name]()]
    U.check_frames(make, frames, U.deform_to, 4, {"device_bvh": device_bvh})


LIGHT_OPTIONS = [{}, {"light_tree": True, "light_tree_triangles": True},
                 {"light_tree": True, "light_tree_triangles": True, "light_solid_angle": True},
                 {"light_tree": True, "light_tree_triangles": True, "light_receiver": True}]


@pytest.mark.parametrize("options", LIGHT_OPTIONS, ids=["uniform", "tree_triangles", "solid_angle", "receiver"])
@pytest.mark.parametrize("name", list(S.DEFORM_EMISSIVE_FRAMES))
def test_deforming_emitters_rebuild_alias_tables_and_light_trees(name, options, make):
    frames = [S.scene(t) for t in S.DEFORM_EMISSIVE_FRAMES[name]()]
    U.check_frames(make, frames, U.deform_to, 8, options, trace=options == {})


def test_instance_and_mesh_updates_compose(make):
    """A chain that moves instances and deforms meshes in turn: every step equals a fresh upload of its frame."""
    frames = [S.scene(S.sheet(t, shift=shift)) for t, shift in ((0.0, 0.0), (0.5, 0.0), (0.5, 0.2), (1.1, 0.2), (1.1, -0.1))]
    r = make()
    r.upload(frames[0].desc())
    for k, (prev, cur) in enumerate(zip(frames, frames[1:])):
        (U.deform_to if k % 2 == 0 else U.update_to)(r, prev.desc(), cur.desc())
        film, _ = U.fresh(make, cur, 4, {})
        r.render(0, 4)
        assert np.array_equal(r.film(raw=True), film)


def test_update_to_the_uploaded_vertices_keeps_the_film(make):
    s = S.scene(S.sheet(0.3))
    d = s.desc()
    r = make()
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    v, m = S.vertices(d), S.meshes(d)
    r.update_meshes(np.arange(d.mesh_count), [v[o:o + c] for o, c in m[:, :2]])
    assert not r.film(raw=True).any()  # the update clears the film
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)


def test_gbuffer_adaptive_and_shards_after_a_mesh_update(make):
    U.check_gbuffer_adaptive_and_shards(make, S.scene(S.sheet(0.0)), S.scene(S.sheet(0.7)), U.deform_to)


def test_refused_mesh_updates_change_nothing(make):
    d = S.scene(S.sheet(0.0)).desc()
    deformed = S.scene(S.sheet(0.5)).desc()
    ids, parts = S.deformed_meshes(d, deformed)
    k = ids[0]
    empty = make()
    with pytest.raises(RuntimeError, match=r"\(-1\).*no scene"):
        empty.update_meshes([k], parts[:1])
    r = make()
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    nan = parts[0].copy()
    nan[3, 1] = np.inf
    U.check_refusals(r, film, [(lambda: r.update_meshes([d.mesh_count], parts[:1]), "out of range"),
                               (lambda: r.update_meshes([k, k], [parts[0], parts[0]]), "repeated"),
                               (lambda: r.update_meshes([k], [parts[0][:-1]]), "vertex_count"),
                               (lambda: r.update_meshes([k], [nan]), "non-finite")])
