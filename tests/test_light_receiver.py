"""Receiver-aware light sampling on the GPU (option "light_receiver"; include/lrk.h, csrc/device/receiver.h, the receiver term of
light_tree.h and the warp of spherical_triangle.h).

Off, the option must change nothing; on, every frame must render the same image as without it within its noise, the irradiance
frame must match Lambert's formula, the near-light and many-light frames are measured for noise, and scheduling, sharding, the
G-buffer mode and the adaptive mode must compose with it unchanged.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

from light_sampling_checks import SUB_SPP, SUBRENDERS, Z_MAX, bits, block_means, reference, rel_mse, render, sub_renders, z_scores
from test_light_solid_angle import analytic_irradiance_film

REPO = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu
OFF, ON = {"light_receiver": 0}, {"light_receiver": 1}
TREE, SOLID, TRIANGLES = {"light_tree": 1}, {"light_solid_angle": 1}, {"light_tree": 1, "light_tree_triangles": 1}


@pytest.fixture
def r(gpu_renderer):
    """gpu_renderer, with every light-sampling option this file touches back at its default afterwards."""
    yield gpu_renderer
    for name, value in (("light_receiver", 0), ("light_candidates", 0), ("light_tree_triangles", 0), ("light_tree", 0),
                        ("light_solid_angle", 0), ("gbuffer", 0), ("max_paths_per_pass", 136 << 20)):
        gpu_renderer.set_option(name, value)
    gpu_renderer.set_shard(0, 1, 32)


def _scene(src):
    from luisarender_b200.api import Scene

    return Scene.from_source(src, REPO)


def _frame(name):
    from luisarender_b200 import scenes

    if name == "cornell":
        return _scene(scenes.cornell_box(resolution=(64, 64), spp=16))
    if name == "textured_lamp":
        return _scene(scenes.textured_room(resolution=(96, 64), spp=8, textured_light=True))
    if name == "environment_area":
        return _scene(scenes.environment_scene(resolution=(64, 48), spp=4, area_light=True))
    if name == "flatten":
        return _scene(scenes.flatten_stress(resolution=(64, 48), spp=4))
    if name == "mix":
        return _scene(scenes.materials_box(mix=True))
    if name == "layered":
        return _scene(scenes.layered_box())
    if name == "many":
        return _scene(scenes.many_lights(resolution=(128, 72), spp=16, count=48, big_subdivision=3, small_subdivision=2))
    if name.startswith("globe_"):
        return _scene(scenes.emissive_globe(resolution=(64, 64), spp=16, subdivision=3, transform=name[6:]))
    if name == "near":
        return _scene(scenes.near_light(resolution=(96, 96), spp=16))
    if name == "irradiance":
        return _scene(scenes.near_light(resolution=(64, 64), spp=16, irradiance=True))
    if name == "medium":
        return _scene(scenes.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3, small_subdivision=2,
                                               small_count=12))
    raise KeyError(name)


@pytest.fixture(scope="module")
def frames():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _frame(name)
        return cache[name]

    return get


# ---- 1. off changes nothing -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("base", [TREE, SOLID], ids=["tree", "solid_angle"])
def test_option_off_equals_a_context_that_never_set_it(frames, r, base):
    from luisarender_b200.api import Renderer

    d = frames("many").desc()
    fresh = Renderer(device_index=0)
    try:
        fresh.set_option("strict_math", 0 if r.fast else 1)
        for k, v in base.items():
            fresh.set_option(k, v)
        fresh.upload(d)
        fresh.render(0, 4)
        want, want_launches = fresh.film(raw=True), fresh.stats()["kernel_launches"]
    finally:
        fresh.close()
    render(r, d, 0, 4, {**base, **ON})  # leaves the receiver words behind in this context
    got = render(r, d, 0, 4, {**base, **OFF})
    assert np.array_equal(bits(got), bits(want))
    assert r.stats()["kernel_launches"] == want_launches


# ---- 2. unbiased: the same image as without the option ----------------------------------------------------------------------------
CASES = [("cornell", SOLID), ("cornell", {**TREE, **SOLID}), ("textured_lamp", SOLID), ("environment_area", {**TREE, **SOLID}), ("flatten", SOLID),
         ("mix", SOLID), ("layered", SOLID), ("many", TREE), ("many", TRIANGLES), ("many", SOLID), ("globe_uniform", TRIANGLES),
         ("globe_stretched", TRIANGLES), ("globe_mirrored", TRIANGLES), ("cornell", {**SOLID, "light_candidates": 4})]


@pytest.mark.parametrize("name,base", CASES, ids=[f"{n}-{'+'.join(sorted(b))}" for n, b in CASES])
def test_receiver_agrees_without_it(frames, r, name, base):
    d = frames(name).desc()
    # the same sample indices give another film: the option changes the sampling on this frame
    assert not np.array_equal(bits(render(r, d, 0, 2, {**base, **OFF})), bits(render(r, d, 0, 2, {**base, **ON})))
    off = sub_renders(r, d, {**base, **OFF}, 0, SUBRENDERS, SUB_SPP)
    on = sub_renders(r, d, {**base, **ON}, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)  # disjoint sample indices
    z = z_scores(on, off)
    assert np.abs(z).max() < Z_MAX, z


def test_one_emitter_tree_is_unchanged(frames, r):
    """The Cornell box has one emissive instance: the tree picks it with probability 1 at any receiver, so the option leaves the
    tree-only film bit for bit as it was."""
    d = frames("cornell").desc()
    assert np.array_equal(bits(render(r, d, 0, 4, {**TREE, **OFF})), bits(render(r, d, 0, 4, {**TREE, **ON})))


# ---- 3. the irradiance frame against Lambert's formula ----------------------------------------------------------------------------
def test_irradiance_frame_matches_lambert(frames, r):
    d = frames("irradiance").desc()
    films = sub_renders(r, d, {**SOLID, **ON}, 0, SUBRENDERS, SUB_SPP)
    want = analytic_irradiance_film(d)
    m = block_means(films)
    w = block_means(np.repeat(want[None, :, :, None], 3, axis=3))[0]
    se = m.std(axis=0, ddof=1) / np.sqrt(len(m))
    assert (se > 0).all()
    z = (m.mean(axis=0) - w) / se
    assert np.abs(z).max() < Z_MAX, z


# ---- 4. noise at equal spp ---------------------------------------------------------------------------------------------------------
# The 16-spp relative MSE with the option over that without it, each averaged over 8 renders.  Measured on an H100 80GB HBM3 at a
# 700 W power limit: near_light (solid angle) 0.9565 in both arithmetic modes, the many-light frame (tree) 0.9584 strict and 0.9576
# fast (DESIGN.md §5).  The renders are seeded, so the bound's margin is for changes of the code around the samplers, not for chance.
ERROR_RATIO = 0.98


@pytest.mark.parametrize("name,base", [("near", SOLID), ("many", TREE)], ids=["near_light-solid_angle", "many_lights-tree"])
def test_error_at_16_spp(frames, r, name, base):
    d = frames(name).desc()
    ref = reference(r, d, {**base, **ON})
    off, on = rel_mse(r, d, {**base, **OFF}, ref, 0), rel_mse(r, d, {**base, **ON}, ref, 4096)
    print(f"{name} 16 spp rel. MSE: off {off:.4e}, on {on:.4e}, ratio {on / off:.4f} (fast={r.fast})")
    assert on <= ERROR_RATIO * off, (on, off, on / off)


# ---- 5. scheduling and the other modes --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("base", [SOLID, TRIANGLES], ids=["solid_angle", "tree_triangles"])
def test_scheduling_and_sharding_change_no_bit(frames, r, base):
    d = frames("many").desc()
    opts = {**base, **ON}
    whole = render(r, d, 0, 8, opts)
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
        r.balance_shards(rank, 3, 32, 1)
        r.render(0, 8)
        part = r.film(raw=True)
        assert not np.any((total != 0) & (part != 0))
        total += part
    assert np.array_equal(bits(total), bits(whole))


def test_gbuffer_and_adaptive_compose(frames, r):
    d = frames("near").desc()
    r.set_option("gbuffer", 1)
    off = render(r, d, 0, 4, {**SOLID, **OFF})
    gb_off = r.gbuffer()
    on = render(r, d, 0, 4, {**SOLID, **ON})
    gb_on = r.gbuffer()
    assert not np.array_equal(bits(on), bits(off))
    for a, b in zip(gb_on[:2], gb_off[:2]):
        assert np.array_equal(bits(a), bits(b))
    r.set_option("gbuffer", 0)
    uniform = render(r, d, 0, 8, {**SOLID, **ON})
    r.render_adaptive(0.0, 4, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(uniform))


# ---- 6. errors --------------------------------------------------------------------------------------------------------------------
def test_refusals_keep_the_previous_film(frames, r):
    d = frames("cornell").desc()
    before = render(r, d, 0, 2, SOLID)
    r.set_option("light_solid_angle", 0)
    r.set_option("light_receiver", 1)
    with pytest.raises(RuntimeError, match=r"lrk_upload_scene failed \(-1\): .*light_receiver"):
        r.upload(d)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        r.set_option("light_receiver", 2)
    assert np.array_equal(bits(r.film(raw=True)), bits(before))
    m = frames("medium").desc()
    with pytest.raises(RuntimeError, match=r"lrk_upload_scene failed \(-5\)"):
        r.upload(m)
    r.set_option("light_receiver", 0)
    assert np.array_equal(bits(render(r, d, 0, 2, SOLID)), bits(before))
