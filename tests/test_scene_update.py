"""Scene updates (lrk_update_instances / lrk_update_camera, DESIGN.md §4 (Scene updates)) on the GPU, in both arithmetic modes: a
context that uploaded scene A and was updated to B's transforms (or camera) renders, traces, writes G-buffers and renders
adaptively what a context that uploaded B does, bit for bit; refused updates change nothing."""
from __future__ import annotations

import re
from pathlib import Path

import numpy as np
import pytest

from luisarender_b200 import scenes
from luisarender_b200.api import Renderer, Scene
from oracle import binding as O

pytestmark = pytest.mark.gpu
REPO = Path(__file__).resolve().parents[1]


@pytest.fixture
def make(gpu_renderer):
    """Fresh contexts in gpu_renderer's arithmetic mode, with the given Renderer options (and "device_bvh"), closed afterwards."""
    made = []

    def new(device_bvh=False, gbuffer=False, **options):
        r = Renderer(device_index=0, **options)
        r.set_option("strict_math", 0 if gpu_renderer.fast else 1)
        r.set_option("device_bvh", int(device_bvh))
        r.set_option("gbuffer", int(gbuffer))
        made.append(r)
        return r

    yield new
    for r in made:
        r.close()


def _scene(text):
    return Scene.from_source(text, REPO)


def _rows(desc):
    return np.array([list(desc.instances[i].object_to_world) for i in range(desc.instance_count)], np.float32).reshape(-1, 3, 4)


def _update_to(r, a_desc, b_desc):
    """Update the context r (holding a_desc's transforms) to b_desc's: the instances whose rows differ."""
    a, b = _rows(a_desc), _rows(b_desc)
    ids = np.flatnonzero((a.view(np.uint32) != b.view(np.uint32)).any(axis=(1, 2)))
    assert len(ids) > 0
    r.update_instances(ids, b[ids])


def _random_rays(scene, n, seed):
    rng = np.random.default_rng(seed)
    info = scene.info()
    lo, hi = np.array(info["world_min"]), np.array(info["world_max"])
    o = rng.uniform(lo - 0.5, hi + 0.5, size=(n, 3))
    d = rng.uniform(lo, hi, size=(n, 3)) - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.zeros((n, 8), np.float32)
    rays[:, :3], rays[:, 4:7], rays[:, 7] = o, d, np.finfo(np.float32).max
    rays[::3, 7] = rng.uniform(0.5, 6.0, size=len(rays[::3]))
    return rays


def _fresh(make, scene, spp, options):
    r = make(**options)
    r.upload(scene.desc())
    r.render(0, spp)
    return r, r.film(raw=True).copy(), r.stats()["kernel_launches"]


def _check_frames(make, frames, spp, options, trace=True):
    """Upload frames[0], then update through frames[1:], each time against a fresh upload of that frame: raw film, launches, and
    (trace=True) closest hits and occlusion of random rays against the oracle's trace of the frame's description."""
    r = make(**options)
    r.upload(frames[0].desc())
    r.render(0, spp)
    for prev, cur in zip(frames, frames[1:]):
        _update_to(r, prev.desc(), cur.desc())
        _, film, launches = _fresh(make, cur, spp, options)
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


def _move(text, shape, srt):
    """The scene text with `transform : SRT { srt }` added to the definition of the shape `shape`."""
    pattern = rf"(Shape {shape} : \w+ \{{)"
    assert len(re.findall(pattern, text)) == 1
    return re.sub(pattern, rf"\1 transform : SRT {{ {srt} }}", text)


def _cornell(**kw):
    return scenes.cornell_box(resolution=(48, 48), spp=4, **kw)


def _spheres(time):
    return scenes.instanced_spheres(resolution=(64, 36), spp=4, big_subdivision=4, small_subdivision=2, small_count=12, time=time)


def _flatten_stress(moved):
    text = scenes.flatten_stress()
    if moved:  # a nested Instance's SRT, a Stack member (an emitter) and a Group's Matrix
        for old, new in (("translate { 2.2, 0.0, -1.6 }", "translate { 2.5, 0.2, -1.1 }"), ("translate { 0.0, 2.6, 0.0 }", "translate { 0.3, 2.4, 0.2 }"),
                         ("0.8, 0.0, 0.0, -1.5,", "0.7, 0.1, 0.0, -1.2,")):
            assert text.count(old) == 1
            text = text.replace(old, new)
    return text


def _globe(kind):
    """emissive_globe frames over one Sphere mesh: "uniform" (SRT), "stretched" (Matrix) and "mirrored" (the stretched frame's
    Matrix replaced by one of negative determinant)."""
    if kind != "mirrored":
        return scenes.emissive_globe(resolution=(48, 48), spp=4, subdivision=3, transform=kind)
    text = scenes.emissive_globe(resolution=(48, 48), spp=4, subdivision=3, transform="stretched")
    m = "transform : Matrix { m { -0.25, 0.0, 0.0, 0.1, 0.0, 0.25, 0.0, 1.1, 0.0, 0.0, 0.25, -0.35, 0.0, 0.0, 0.0, 1.0 } }"
    text, n = re.subn(r"transform : Matrix \{ m \{[^}]*\} \}", m, text)
    assert n == 1
    return text


def _textured_room(moved):
    """The textured room with wrappers: the OBJ cube turned and moved, the alpha-tested screen moved."""
    text = scenes.textured_room(resolution=(48, 32), spp=4, wrappers=True)
    if moved:
        old = "rotate { 0.0, 1.0, 0.0, 30.0 } translate { -0.6, 0.4, -0.3 }"
        assert text.count(old) == 1
        text = _move(text.replace(old, "rotate { 0.0, 1.0, 0.0, 50.0 } translate { -0.4, 0.5, -0.1 }"), "screen", "translate { -0.1, 0.0, 0.2 }")
    return text


FRAMES = {
    "cornell_tall_box": lambda: [_cornell(), _move(_cornell(), "tall_box", "rotate { 0.0, 1.0, 0.0, 15.0 } translate { 0.2, 0.0, 0.25 }")],
    "spheres_chain": lambda: [_spheres(0.0), _spheres(0.5), _spheres(1.0)],
    "flatten_stress": lambda: [_flatten_stress(False), _flatten_stress(True)],
    "textured_room": lambda: [_textured_room(False), _textured_room(True)],
    "media_box": lambda: [scenes.media_box(resolution=(32, 32)), _move(scenes.media_box(resolution=(32, 32)), "tall_box", "translate { 0.15, 0.0, 0.2 }")],
}


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
@pytest.mark.parametrize("name", list(FRAMES))
def test_update_equals_fresh_upload(name, device_bvh, make):
    frames = [_scene(t) for t in FRAMES[name]()]
    _check_frames(make, frames, 4, {"device_bvh": device_bvh})


LIGHT_OPTIONS = [{"light_tree": True, "light_tree_triangles": True}, {"light_tree": True, "light_tree_triangles": True, "light_solid_angle": True},
                 {"light_tree": True, "light_tree_triangles": True, "light_receiver": True}]


@pytest.mark.parametrize("options", LIGHT_OPTIONS, ids=["tree_triangles", "solid_angle", "receiver"])
def test_moving_emitters_rebuild_the_light_tree(options, make):
    """The globe moves, is stretched and mirrored (its bottom tree changes side); the many-light frame's emitters move."""
    globe = [_scene(_globe(k)) for k in ("uniform", "stretched", "mirrored")]
    _check_frames(make, globe, 8, options)
    many = [_scene(scenes.many_lights(resolution=(48, 32), spp=4, count=12, big_subdivision=3, small_subdivision=2, time=t)) for t in (0.0, 0.7)]
    _check_frames(make, many, 4, {"light_tree": True}, trace=False)


@pytest.mark.parametrize("device_bvh", [False, True], ids=["host_bvh", "device_bvh"])
def test_camera_update_equals_fresh_upload(device_bvh, make):
    a = _scene(_cornell())
    b = _scene(_cornell().replace("position { -0.01, 0.995, 5.0 }", "position { 0.3, 1.2, 4.4 }"))
    r = make(device_bvh=device_bvh)
    r.upload(a.desc())
    r.render(0, 4)
    r.update_camera(b.desc().camera)
    _, film, launches = _fresh(make, b, 4, {"device_bvh": device_bvh})
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)
    assert r.stats()["kernel_launches"] == launches


def test_update_to_the_uploaded_transforms_keeps_the_film(spheres_small, make):
    d = spheres_small.desc()
    r = make()
    r.upload(d)
    r.render(0, 4)
    film = r.film(raw=True).copy()
    r.update_instances(np.arange(d.instance_count), _rows(d))
    assert not r.film(raw=True).any()  # the update clears the film
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)


def test_gbuffer_adaptive_and_shards_after_an_update(make):
    a, b = _scene(_spheres(0.0)), _scene(_spheres(0.8))
    fresh = make(gbuffer=True)
    fresh.upload(b.desc())
    fresh.render(0, 4)
    film, guides = fresh.film(raw=True).copy(), fresh.gbuffer()
    r = make(gbuffer=True)
    r.upload(a.desc())
    r.render(0, 4)
    _update_to(r, a.desc(), b.desc())
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
        _update_to(s, a.desc(), b.desc())
        s.render(0, 4)
        total += s.film(raw=True)
    assert np.array_equal(total, film)


def test_refused_updates_change_nothing(cornell_small, make):
    d = cornell_small.desc()
    rows = _rows(d)
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
    other = _scene(_cornell().replace("resolution { 48, 48 }", "resolution { 40, 48 }")).desc().camera
    refusals = [(lambda: r.update_instances([0, d.instance_count], moved), "out of range"),
                (lambda: r.update_instances([1, 1], moved), "repeated"),
                (lambda: r.update_instances([0, 1], nan), "non-finite"),
                (lambda: r.update_instances([0, 1], singular), "singular"),
                (lambda: r.update_camera(other), "film size")]
    for call, what in refusals:
        with pytest.raises(RuntimeError, match=rf"\(-1\).*{what}"):
            call()
        assert np.array_equal(r.film(raw=True), film)  # not even cleared
    r.clear()
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)  # the scene is the uploaded one
