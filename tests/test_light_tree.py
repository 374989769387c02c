"""The light tree on the GPU (option "light_tree"; include/lrk.h, csrc/device/light_tree.h).

Off, the option must change nothing; on, a scene with one light must render bit for bit as without it, the many-light frame must
render the same image as the uniform sampler within its noise (and with less of it), shapes that share a Light node must all be
sampled, and scheduling, sharding, the G-buffer mode and the adaptive mode must compose with it unchanged.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

from light_sampling_checks import SUB_SPP, SUBRENDERS, Z_MAX, bits, r, reference, rel_mse, render, sub_renders, z_scores  # noqa: F401

REPO = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu
RES = (128, 72)
UNIFORM, TREE = {"light_tree": 0}, {"light_tree": 1}


def _scene(src):
    from luisarender_b200.api import Scene

    return Scene.from_source(src, REPO)


@pytest.fixture(scope="module")
def many_small():
    from luisarender_b200 import scenes

    return _scene(scenes.many_lights(resolution=RES, spp=16, count=48, big_subdivision=3, small_subdivision=2))


@pytest.fixture(scope="module")
def many_equal():
    """The many-light frame with every sphere of the same emission, one Light node each ..."""
    from luisarender_b200 import scenes

    return _scene(scenes.many_lights(resolution=RES, spp=16, count=48, spread=False, big_subdivision=3, small_subdivision=2))


@pytest.fixture(scope="module")
def many_shared():
    """... and the same spheres sharing one node."""
    from luisarender_b200 import scenes

    return _scene(scenes.many_lights(resolution=RES, spp=16, count=48, shared_node=True, big_subdivision=3, small_subdivision=2))


@pytest.fixture(scope="module")
def environment_one_light():
    from luisarender_b200 import scenes

    return _scene(scenes.environment_scene(resolution=(48, 30), spp=4, area_light=True))


@pytest.fixture(scope="module")
def medium_small():
    from luisarender_b200 import scenes

    return _scene(scenes.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3, small_subdivision=2,
                                           small_count=12))


# ---- 1. off changes nothing -------------------------------------------------------------------------------------------------------
def test_option_off_equals_a_context_that_never_set_it(spheres_small, r):
    from luisarender_b200.api import Renderer

    fresh = Renderer(device_index=0)
    try:
        fresh.set_option("strict_math", 0 if r.fast else 1)
        fresh.upload(spheres_small.desc())
        fresh.render(0, 4)
        want, want_launches = fresh.film(raw=True), fresh.stats()["kernel_launches"]
    finally:
        fresh.close()
    got = render(r, spheres_small.desc(), 0, 4, UNIFORM)
    assert np.array_equal(bits(got), bits(want))
    assert r.stats()["kernel_launches"] == want_launches


# ---- 2. one light: the tree's pmf is exactly 1 -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cornell_small", "textured_wrappers_small", "environment_one_light"])
def test_one_light_scenes_render_bit_identically(request, name, r):
    d = request.getfixturevalue(name).desc()
    assert sum(1 for i in range(d.instance_count) if d.instances[i].handle[0] & 8) == 1  # one emissive instance
    off = render(r, d, 0, 8, UNIFORM)
    on = render(r, d, 0, 8, TREE)
    assert np.array_equal(bits(on), bits(off))


# ---- 3. unbiased: the same image as the uniform sampler ---------------------------------------------------------------------------
def test_many_lights_tree_agrees_with_uniform(many_small, r):
    d = many_small.desc()
    uniform = sub_renders(r, d, UNIFORM, 0, SUBRENDERS, SUB_SPP)
    tree = sub_renders(r, d, TREE, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)  # disjoint sample indices
    z = z_scores(tree, uniform)
    assert np.abs(z).max() < Z_MAX, z


def test_shared_light_node_is_sampled_whole(many_equal, many_shared, r):
    """With the tree, spheres that share one Light node light the frame as spheres with a node each do under the uniform sampler;
    the uniform sampler draws only the first of the shared ones, and its MIS weights drop part of the others' light."""
    own = sub_renders(r, many_equal.desc(), UNIFORM, 0, SUBRENDERS, SUB_SPP)
    shared_tree = sub_renders(r, many_shared.desc(), TREE, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)
    z = z_scores(shared_tree, own)
    assert np.abs(z).max() < Z_MAX, z
    shared_uniform = sub_renders(r, many_shared.desc(), UNIFORM, 2 * SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)
    assert z_scores(shared_uniform, own)[0] < -Z_MAX  # the whole image is darker beyond its noise


# ---- 4. less noise ----------------------------------------------------------------------------------------------------------------
def test_many_lights_tree_halves_the_error(many_small, r):
    """16 spp against a 1024-spp reference of disjoint sample indices: relative MSE of the tree at most 0.5x that of the uniform
    sampler, averaged over 8 independent 16-spp renders each."""
    d = many_small.desc()
    ref = reference(r, d, TREE)
    uniform, tree = rel_mse(r, d, UNIFORM, ref, 0), rel_mse(r, d, TREE, ref, 4096)
    assert tree <= 0.5 * uniform, (tree, uniform, tree / uniform)


# ---- 5. scheduling and the other modes --------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(many_small, r):
    d = many_small.desc()
    whole = render(r, d, 0, 8, TREE)
    r.clear()
    r.render(0, 3)
    r.render(3, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(whole))
    r.set_option("max_paths_per_pass", 1024)
    r.clear()
    r.render(0, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(whole))
    r.set_option("max_paths_per_pass", 136 << 20)
    total = np.zeros_like(whole)
    for rank in range(3):
        r.upload(d)
        r.balance_shards(rank, 3, 32, 1)  # the cost probe runs the tree's kernels too
        r.render(0, 8)
        part = r.film(raw=True)
        assert not np.any((total != 0) & (part != 0))  # every pixel has one owner
        total += part
    assert np.array_equal(bits(total), bits(whole))


def test_gbuffer_and_adaptive_compose(many_small, r):
    d = many_small.desc()
    r.set_option("gbuffer", 1)
    off = render(r, d, 0, 4, UNIFORM)
    gb_off = r.gbuffer()
    on = render(r, d, 0, 4, TREE)
    gb_on = r.gbuffer()
    assert not np.array_equal(bits(on), bits(off))  # the tree changes the film ...
    for a, b in zip(gb_on[:2], gb_off[:2]):  # ... not the first hits
        assert np.array_equal(bits(a), bits(b))
    r.set_option("gbuffer", 0)
    uniform = render(r, d, 0, 8, TREE)
    r.render_adaptive(0.0, 4, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(uniform))


# ---- 6. errors --------------------------------------------------------------------------------------------------------------------
def test_volume_integrator_is_refused_at_upload(medium_small, r):
    d = medium_small.desc()
    before = render(r, d, 0, 2, UNIFORM)
    r.set_option("light_tree", 1)
    with pytest.raises(RuntimeError, match=r"lrk_upload_scene failed \(-5\): .*light tree"):
        r.upload(d)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        r.set_option("light_tree", 2)
    assert np.array_equal(bits(render(r, d, 0, 2, UNIFORM)), bits(before))
