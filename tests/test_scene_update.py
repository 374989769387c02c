"""Scene updates (lrk_update_instances / lrk_update_camera, DESIGN.md §4 (Scene updates)) on the GPU, in both arithmetic modes: a
context that uploaded scene A and was updated to B's transforms (or camera) renders, traces, writes G-buffers and renders
adaptively what a context that uploaded B does, bit for bit; refused updates change nothing."""
from __future__ import annotations

import numpy as np
import pytest

import scene_update_checks as U
import scene_update_frames as S
from luisarender_b200 import scenes
from scene_update_checks import make  # noqa: F401  (the context fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
@pytest.mark.parametrize("name", list(S.INSTANCE_FRAMES))
def test_update_equals_fresh_upload(name, device_bvh, make):
    frames = [S.scene(t) for t in S.INSTANCE_FRAMES[name]()]
    U.check_frames(make, frames, U.update_to, 4, {"device_bvh": device_bvh})


LIGHT_OPTIONS = [{"light_tree": True, "light_tree_triangles": True}, {"light_tree": True, "light_tree_triangles": True, "light_solid_angle": True},
                 {"light_tree": True, "light_tree_triangles": True, "light_receiver": True}]


@pytest.mark.parametrize("options", LIGHT_OPTIONS, ids=["tree_triangles", "solid_angle", "receiver"])
def test_moving_emitters_rebuild_the_light_tree(options, make):
    """The globe moves, is stretched and mirrored (its bottom tree changes side); the many-light frame's emitters move."""
    globe = [S.scene(S.transformed_globe(k)) for k in ("uniform", "stretched", "mirrored")]
    U.check_frames(make, globe, U.update_to, 8, options)
    many = [S.scene(scenes.many_lights(resolution=(48, 32), spp=4, count=12, big_subdivision=3, small_subdivision=2, time=t)) for t in (0.0, 0.7)]
    U.check_frames(make, many, U.update_to, 4, {"light_tree": True}, trace=False)


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
def test_camera_update_equals_fresh_upload(device_bvh, make):
    a = S.scene(S.cornell())
    b = S.scene(S.cornell().replace("position { -0.01, 0.995, 5.0 }", "position { 0.3, 1.2, 4.4 }"))
    r = make(device_bvh=device_bvh)
    r.upload(a.desc())
    r.render(0, 4)
    r.update_camera(b.desc().camera)
    U.check_against_fresh(make, r, b, 4, {"device_bvh": device_bvh}, trace=False)


def test_update_to_the_uploaded_transforms_keeps_the_film(spheres_small, make):
    d = spheres_small.desc()
    r = make()
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    r.update_instances(np.arange(d.instance_count), S.rows(d))
    assert not r.film(raw=True).any()  # the update clears the film
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)


def test_gbuffer_adaptive_and_shards_after_an_update(make):
    U.check_gbuffer_adaptive_and_shards(make, S.scene(S.spheres(0.0)), S.scene(S.spheres(0.8)), U.update_to)


def test_refused_updates_change_nothing(cornell_small, make):
    d = cornell_small.desc()
    rows = S.rows(d)
    empty = make()
    with pytest.raises(RuntimeError, match=r"\(-1\).*no scene"):
        empty.update_instances([0], rows[:1])
    with pytest.raises(RuntimeError, match=r"\(-1\).*no scene"):
        empty.update_camera(d.camera)
    r = make()
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    moved = rows[:2].copy()
    moved[:, :, 3] += 0.5
    nan, singular = moved.copy(), moved.copy()
    nan[1, 0, 3] = np.nan
    singular[1, :, 0] = 0.0
    other = S.scene(S.cornell().replace("resolution { 48, 48 }", "resolution { 40, 48 }")).desc().camera
    U.check_refusals(r, film, [(lambda: r.update_instances([0, d.instance_count], moved), "out of range"),
                               (lambda: r.update_instances([1, 1], moved), "repeated"),
                               (lambda: r.update_instances([0, 1], nan), "non-finite"),
                               (lambda: r.update_instances([0, 1], singular), "singular"),
                               (lambda: r.update_camera(other), "film size")])
