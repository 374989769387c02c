"""Mesh updates (lrk_update_meshes, DESIGN.md §4 (Mesh deformation)) on the GPU, in both arithmetic modes: a context that uploaded
frame A and was updated to B's vertices renders, traces, writes G-buffers and renders adaptively what a context that uploaded B
does, bit for bit; refused updates change nothing."""
from __future__ import annotations

import numpy as np
import pytest

import mesh_update_frames as M
from oracle import binding as O
from test_scene_update import _random_rays, _update_to, make  # noqa: F401  (make: test_scene_update's context fixture)

pytestmark = pytest.mark.gpu


def _deform_to(r, a_desc, b_desc):
    ids, parts = M.deformed_meshes(a_desc, b_desc)
    assert ids
    r.update_meshes(ids, parts)


def _fresh(make, scene, spp, options):
    r = make(**options)
    r.upload(scene.desc())
    r.render(0, spp)
    return r.film(raw=True).copy(), r.stats()["kernel_launches"]


def _check_frames(make, frames, spp, options, trace=True):
    """Upload frames[0], then deform through frames[1:], each time against a fresh upload of that frame: raw film, launches, and
    (trace=True) closest hits and occlusion of random rays against the oracle's trace of the frame's description."""
    r = make(**options)
    r.upload(frames[0].desc())
    r.render(0, spp)
    for prev, cur in zip(frames, frames[1:]):
        _deform_to(r, prev.desc(), cur.desc())
        film, launches = _fresh(make, cur, spp, options)
        r.render(0, spp)
        assert np.array_equal(r.film(raw=True), film)
        assert r.stats()["kernel_launches"] == launches
        if trace:
            d = cur.desc()
            rays = _random_rays(cur, 100_000, seed=3)
            ref, _ = O.trace(d, rays)
            got = r.trace(rays)
            assert np.array_equal(got["inst"], ref["inst"]) and np.array_equal(got["prim"], ref["prim"])
            assert np.array_equal(got["bary"].view(np.uint32), ref["bary"].view(np.uint32))
            assert (ref["inst"] != 0xFFFFFFFF).mean() > 0.05
            occ_ref, _ = O.trace(d, rays, any_hit=True)
            assert np.array_equal(r.trace(rays, any_hit=True)["inst"], occ_ref["inst"])
    return r


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
@pytest.mark.parametrize("name", list(M.FRAMES))
def test_mesh_update_equals_fresh_upload(name, device_bvh, make):
    frames = [M.scene(t) for t in M.FRAMES[name]()]
    _check_frames(make, frames, 4, {"device_bvh": device_bvh})


LIGHT_OPTIONS = [{}, {"light_tree": True, "light_tree_triangles": True},
                 {"light_tree": True, "light_tree_triangles": True, "light_solid_angle": True},
                 {"light_tree": True, "light_tree_triangles": True, "light_receiver": True}]


@pytest.mark.parametrize("options", LIGHT_OPTIONS, ids=["uniform", "tree_triangles", "solid_angle", "receiver"])
@pytest.mark.parametrize("name", list(M.EMISSIVE_FRAMES))
def test_deforming_emitters_rebuild_alias_tables_and_light_trees(name, options, make):
    frames = [M.scene(t) for t in M.EMISSIVE_FRAMES[name]()]
    _check_frames(make, frames, 8, options, trace=options == {})


def test_instance_and_mesh_updates_compose(make):
    """A chain that moves instances and deforms meshes in turn: every step equals a fresh upload of its frame."""
    def moved(time, shift):
        text = M.sheet(time)
        return text.replace("translate { -0.2, 1.15, -0.35 }", f"translate {{ -0.2, {1.15 + shift!r}, -0.35 }}")
    frames = [M.scene(t) for t in (moved(0.0, 0.0), moved(0.5, 0.0), moved(0.5, 0.2), moved(1.1, 0.2), moved(1.1, -0.1))]
    r = make()
    r.upload(frames[0].desc())
    for k, (prev, cur) in enumerate(zip(frames, frames[1:])):
        if k % 2 == 0:
            _deform_to(r, prev.desc(), cur.desc())
        else:
            _update_to(r, prev.desc(), cur.desc())
        film, launches = _fresh(make, cur, 4, {})
        r.render(0, 4)
        assert np.array_equal(r.film(raw=True), film)


def test_update_to_the_uploaded_vertices_keeps_the_film(make):
    s = M.scene(M.sheet(0.3))
    d = s.desc()
    r = make()
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    v, m = M.vertices(d), M.meshes(d)
    r.update_meshes(np.arange(d.mesh_count), [v[o:o + c] for o, c in m[:, :2]])
    assert not r.film(raw=True).any()  # the update clears the film
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)


def test_gbuffer_adaptive_and_shards_after_a_mesh_update(make):
    a, b = M.scene(M.sheet(0.0)), M.scene(M.sheet(0.7))
    fresh = make(gbuffer=True)
    fresh.upload(b.desc())
    fresh.render(0, 4)
    film, guides = fresh.film(raw=True).copy(), fresh.gbuffer()
    r = make(gbuffer=True)
    r.upload(a.desc())
    r.render(0, 4)
    _deform_to(r, a.desc(), b.desc())
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)
    for got, want in zip(r.gbuffer(), guides):
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    r.set_option("gbuffer", 0)
    r.render_adaptive(0.0, 2, 4)  # threshold 0: every pixel gets max_spp, as lrk_render(0, 4)
    assert np.array_equal(r.film(raw=True), film)
    total = np.zeros_like(film)
    for rank in range(3):
        s = make()
        s.upload(a.desc())
        s.balance_shards(rank, 3, tile_size=16, probe_spp=1)
        _deform_to(s, a.desc(), b.desc())
        s.render(0, 4)
        total += s.film(raw=True)
    assert np.array_equal(total, film)


def test_refused_mesh_updates_change_nothing(make):
    d = M.scene(M.sheet(0.0)).desc()
    deformed = M.scene(M.sheet(0.5)).desc()
    ids, parts = M.deformed_meshes(d, deformed)
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
    refusals = [(lambda: r.update_meshes([d.mesh_count], parts[:1]), "out of range"),
                (lambda: r.update_meshes([k, k], [parts[0], parts[0]]), "repeated"),
                (lambda: r.update_meshes([k], [parts[0][:-1]]), "vertex_count"),
                (lambda: r.update_meshes([k], [nan]), "non-finite")]
    for call, what in refusals:
        with pytest.raises(RuntimeError, match=rf"\(-1\).*{what}"):
            call()
        assert np.array_equal(r.film(raw=True), film)  # not even cleared
    r.clear()
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)  # the scene is the uploaded one
