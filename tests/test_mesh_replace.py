"""Mesh replacement (lrk_replace_meshes, DESIGN.md §4 (Mesh replacement)) on the GPU, in both arithmetic modes: a context that
uploaded frame A and replaced meshes with B's vertices and triangles renders, traces, writes G-buffers and renders adaptively what a
context that uploaded B does, bit for bit; refused replacements change nothing."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import mesh_replace_frames as R
import mesh_update_frames as M
from luisarender_b200 import _ffi as F
from luisarender_b200 import scenes
from oracle import binding as O
from test_mesh_update import LIGHT_OPTIONS, _deform_to, _fresh
from test_scene_update import _random_rays, _update_to, make  # noqa: F401  (make: test_scene_update's context fixture)

pytestmark = pytest.mark.gpu


def _replace_to(r, a_desc, b_desc):
    """Replace the meshes that differ between a_desc and b_desc with B's, passing the ids in descending order."""
    ids, verts, tris = R.replaced_meshes(a_desc, b_desc)
    assert ids
    r.replace_meshes(ids[::-1], verts[::-1], tris[::-1])


def _check_against_fresh(make, r, scene, spp, options, trace=True):
    """r renders (and, with trace=True, traces closest hits and occlusion of random rays) what a fresh upload of `scene` does,
    and what the oracle traces on its description."""
    film, launches = _fresh(make, scene, spp, options)
    r.render(0, spp)
    assert np.array_equal(r.film(raw=True), film)
    assert r.stats()["kernel_launches"] == launches
    if trace:
        d = scene.desc()
        rays = _random_rays(scene, 100_000, seed=3)
        ref, _ = O.trace(d, rays)
        got = r.trace(rays)
        assert np.array_equal(got["inst"], ref["inst"]) and np.array_equal(got["prim"], ref["prim"])
        assert np.array_equal(got["bary"].view(np.uint32), ref["bary"].view(np.uint32))
        assert (ref["inst"] != 0xFFFFFFFF).mean() > 0.05
        occ_ref, _ = O.trace(d, rays, any_hit=True)
        assert np.array_equal(r.trace(rays, any_hit=True)["inst"], occ_ref["inst"])


def _check_frames(make, frames, spp, options, trace=True):
    r = make(**options)
    r.upload(frames[0].desc())
    r.render(0, spp)
    for prev, cur in zip(frames, frames[1:]):
        _replace_to(r, prev.desc(), cur.desc())
        _check_against_fresh(make, r, cur, spp, options, trace)


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
@pytest.mark.parametrize("name", list(R.FRAMES))
def test_mesh_replace_equals_fresh_upload(name, device_bvh, make):
    frames = [M.scene(t) for t in R.FRAMES[name]()]
    _check_frames(make, frames, 4, {"device_bvh": device_bvh})


@pytest.mark.parametrize("options", LIGHT_OPTIONS, ids=["uniform", "tree_triangles", "solid_angle", "receiver"])
@pytest.mark.parametrize("name", list(R.EMISSIVE_FRAMES))
def test_replaced_emitters_rebuild_alias_tables_and_light_trees(name, options, make):
    frames = [M.scene(t) for t in R.EMISSIVE_FRAMES[name]()]
    _check_frames(make, frames, 8, options, trace=options == {})


def _sheet(segments, time, shift=0.0, amplitude=0.08):
    text = scenes.wavy_sheet(resolution=(48, 32), spp=4, segments=segments, time=time, amplitude=amplitude)
    return M.scene(text.replace("translate { -0.2, 1.15, -0.35 }", f"translate {{ -0.2, {1.15 + shift!r}, -0.35 }}"))


def test_replace_update_and_instance_moves_compose(make):
    """Replace, refit the replaced mesh (lrk_update_meshes after lrk_replace_meshes), move instances, replace and refit again:
    every step equals a fresh upload of its frame."""
    steps = [(None, ((16, 10), 0.0, 0.0)), (_replace_to, ((24, 16), 0.0, 0.0)), (_deform_to, ((24, 16), 0.5, 0.0)),
             (_update_to, ((24, 16), 0.5, 0.2)), (_replace_to, ((8, 5), 0.5, 0.2)), (_deform_to, ((8, 5), 1.1, 0.2))]
    frames = [_sheet(*args) for _, args in steps]
    r = make()
    r.upload(frames[0].desc())
    for (step, _), prev, cur in zip(steps[1:], frames, frames[1:]):
        step(r, prev.desc(), cur.desc())
        _check_against_fresh(make, r, cur, 4, {})


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
def test_replace_with_the_uploaded_arrays_keeps_the_film(device_bvh, make):
    s = _sheet((16, 10), 0.3)
    d = s.desc()
    r = make(device_bvh=device_bvh)
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    v, t, m = M.vertices(d), R.triangles(d), M.meshes(d)
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
    _deform_to(r, a.desc(), b.desc())
    _check_against_fresh(make, r, b, 4, {})
    d = b.desc()
    k = M.deformed_meshes(a.desc(), d)[0]
    m = M.meshes(d)
    r.replace_meshes(k, [M.vertices(d)[m[j, 0]:m[j, 0] + m[j, 1]] for j in k], [R.triangles(d)[m[j, 2]:m[j, 2] + m[j, 3]] for j in k])
    _check_against_fresh(make, r, b, 4, {})


def test_gbuffer_adaptive_and_shards_after_a_mesh_replace(make):
    a, b = _sheet((16, 10), 0.3), _sheet((24, 16), 0.3)
    fresh = make(gbuffer=True)
    fresh.upload(b.desc())
    fresh.render(0, 4)
    film, guides = fresh.film(raw=True).copy(), fresh.gbuffer()
    r = make(gbuffer=True)
    r.upload(a.desc())
    r.render(0, 4)
    _replace_to(r, a.desc(), b.desc())
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
        _replace_to(s, a.desc(), b.desc())
        s.render(0, 4)
        total += s.film(raw=True)
    assert np.array_equal(total, film)


def test_refused_mesh_replacements_change_nothing(make):
    a, b = _sheet((16, 10), 0.3), _sheet((24, 16), 0.3)
    d = a.desc()
    ids, verts, tris = R.replaced_meshes(d, b.desc())
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
    refusals = [(lambda: r.replace_meshes([d.mesh_count], [v], [t]), "out of range"),
                (lambda: r.replace_meshes([k, k], [v, v], [t, t]), "repeated"),
                (lambda: r.replace_meshes([k], [v[:0]], [t[:0]]), "no vertices or no triangles"),
                (lambda: r.replace_meshes([k], [v], [t[:0]]), "no vertices or no triangles"),
                (lambda: r.replace_meshes([k], [v], [past]), "triangle index out of range"),
                (lambda: r.replace_meshes([k], [nan], [t]), "non-finite")]
    for call, what in refusals:
        with pytest.raises(RuntimeError, match=rf"\(-1\).*{what}"):
            call()
        assert np.array_equal(r.film(raw=True), film)  # not even cleared
    r.clear()
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)  # the scene is the uploaded one
    # a hierarchy whose instance level is not its last max(visible, 2) - 1 nodes (one unused node behind it) cannot be laid out again
    nodes = M.array(d.bvh_nodes, d.bvh_node_count, F.BvhNode, np.uint32, 16)
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
