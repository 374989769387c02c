"""The triangle-level light trees on the GPU (option "light_tree_triangles"; include/lrk.h, csrc/device/light_tree.h).

Off, the option must change nothing; on, scenes whose emitters are single triangles must render bit for bit as without it, every
frame must render the same image as the uniform sampler within its noise, the emissive globe and the many-light frame must have
less noise than with the instance-level tree, and scheduling, sharding, the G-buffer mode and the adaptive mode must compose with
it unchanged.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

from light_sampling_checks import SUB_SPP, SUBRENDERS, Z_MAX, bits, r, reference, rel_mse, render, sub_renders, z_scores  # noqa: F401

REPO = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu


def _scene(src):
    from luisarender_b200.api import Scene

    return Scene.from_source(src, REPO)


@pytest.fixture(scope="module")
def frames():
    """Frame name -> scene, built on first use."""
    from luisarender_b200 import scenes

    makers = {
        "cornell": lambda: scenes.cornell_box(resolution=(64, 64), spp=16),
        "textured_lamp": lambda: scenes.textured_room(resolution=(96, 64), spp=8, textured_light=True),
        "environment_area": lambda: scenes.environment_scene(resolution=(64, 48), spp=4, area_light=True),
        "flatten": lambda: scenes.flatten_stress(resolution=(64, 48), spp=4),
        "many": lambda: scenes.many_lights(resolution=(128, 72), spp=16, count=48, big_subdivision=3, small_subdivision=2),
        "globe_uniform": lambda: scenes.emissive_globe(resolution=(96, 96), spp=16, subdivision=4, transform="uniform"),
        "globe_stretched": lambda: scenes.emissive_globe(resolution=(96, 96), spp=16, subdivision=4, transform="stretched"),
        "globe_mirrored": lambda: scenes.emissive_globe(resolution=(96, 96), spp=16, subdivision=4, transform="mirrored"),
        "irradiance": lambda: scenes.near_light(resolution=(64, 64), spp=16, irradiance=True),
        "medium": lambda: scenes.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3, small_subdivision=2,
                                                   small_count=12),
    }
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _scene(makers[name]())
        return cache[name]

    return get


MODES = {"uniform": {"light_tree": 0, "light_tree_triangles": 0}, "tree": {"light_tree": 1, "light_tree_triangles": 0},
         "triangles": {"light_tree": 1, "light_tree_triangles": 1}}


# ---- 1. off changes nothing; single-triangle emitters render bit for bit ----------------------------------------------------------
def test_option_off_equals_a_context_that_never_set_it(frames, r):
    from luisarender_b200.api import Renderer

    d = frames("many").desc()
    fresh = Renderer(device_index=0, light_tree=True)
    try:
        fresh.set_option("strict_math", 0 if r.fast else 1)
        fresh.upload(d)
        fresh.render(0, 4)
        want, want_launches = fresh.film(raw=True), fresh.stats()["kernel_launches"]
    finally:
        fresh.close()
    render(r, d, 0, 4, MODES["triangles"])  # leaves the bottom trees behind in this context
    got = render(r, d, 0, 4, MODES["tree"])
    assert np.array_equal(bits(got), bits(want))
    assert r.stats()["kernel_launches"] == want_launches


@pytest.mark.parametrize("solid_angle", [0, 1])
def test_single_triangle_emitters_render_bit_identically(frames, r, solid_angle):
    d = frames("irradiance").desc()
    r.set_option("light_solid_angle", solid_angle)
    off = render(r, d, 0, 8, MODES["tree"])
    on = render(r, d, 0, 8, MODES["triangles"])
    assert np.array_equal(bits(on), bits(off))


# ---- 2. unbiased: the same image as the uniform sampler ---------------------------------------------------------------------------
@pytest.mark.parametrize("name, solid_angle", [("cornell", 0), ("textured_lamp", 0), ("environment_area", 0), ("flatten", 0), ("many", 0),
                                               ("globe_uniform", 0), ("globe_stretched", 0), ("globe_mirrored", 0), ("many", 1),
                                               ("globe_uniform", 1)])
def test_triangle_tree_agrees_with_uniform(frames, r, name, solid_angle):
    d = frames(name).desc()
    r.set_option("light_solid_angle", solid_angle)
    uniform = sub_renders(r, d, MODES["uniform"], 0, SUBRENDERS, SUB_SPP)
    tris = sub_renders(r, d, MODES["triangles"], SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)  # disjoint sample indices
    assert uniform.mean() > 0
    z = z_scores(tris, uniform)
    assert np.abs(z).max() < Z_MAX, z


def test_globe_transforms_light_the_room_alike(frames, r):
    """The mirrored globe is the uniform one's sphere (wound inwards, then mirrored in x, so that it faces outwards): it lights the
    room alike.  The mirror swaps which side of the globe faces the red and the green wall, so only the image means are compared."""
    a = sub_renders(r, frames("globe_uniform").desc(), MODES["triangles"], 0, 16, SUB_SPP).mean(axis=(1, 2, 3))
    b = sub_renders(r, frames("globe_mirrored").desc(), MODES["triangles"], 16 * SUB_SPP, 16, SUB_SPP).mean(axis=(1, 2, 3))
    se = np.sqrt(a.var(ddof=1) / len(a) + b.var(ddof=1) / len(b))
    assert a.mean() > 0 and abs(a.mean() - b.mean()) < 0.05 * a.mean() + Z_MAX * se


# ---- 3. less noise ----------------------------------------------------------------------------------------------------------------
# The 16-spp relative MSE of the triangle-level trees over that of the instance-level tree, each averaged over 8 renders, against a
# 1024-spp reference of disjoint sample indices.  Measured on an H100 in both arithmetic modes: 0.610 on the globe, 0.884-0.885 on
# the many-light frame (DESIGN.md §4).  The renders are seeded, so the margins are for changes of the code around the sampler, not
# for chance.
ERROR_RATIO_BOUND = {"globe_uniform": 0.7, "many": 0.95}


@pytest.mark.parametrize("name", sorted(ERROR_RATIO_BOUND))
def test_error_is_lower_than_the_instance_tree(frames, r, name):
    d = frames(name).desc()
    ref = reference(r, d, MODES["triangles"])
    tree, tris = rel_mse(r, d, MODES["tree"], ref, 0), rel_mse(r, d, MODES["triangles"], ref, 4096)
    print(f"{name} 16 spp rel. MSE: instance tree {tree:.4e}, triangle trees {tris:.4e}, ratio {tris / tree:.4f} (fast={r.fast})")
    assert tris <= ERROR_RATIO_BOUND[name] * tree, (tris, tree, tris / tree)


# ---- 4. scheduling and the other modes --------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(frames, r):
    d = frames("many").desc()
    whole = render(r, d, 0, 8, MODES["triangles"])
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
        r.balance_shards(rank, 3, 32, 1)  # the cost probe runs the option's kernels too
        r.render(0, 8)
        part = r.film(raw=True)
        assert not np.any((total != 0) & (part != 0))  # every pixel has one owner
        total += part
    assert np.array_equal(bits(total), bits(whole))


def test_gbuffer_and_adaptive_compose(frames, r):
    d = frames("globe_stretched").desc()
    r.set_option("gbuffer", 1)
    off = render(r, d, 0, 4, MODES["tree"])
    gb_off = r.gbuffer()
    on = render(r, d, 0, 4, MODES["triangles"])
    gb_on = r.gbuffer()
    assert not np.array_equal(bits(on), bits(off))  # the option changes the film ...
    for a, b in zip(gb_on[:2], gb_off[:2]):  # ... not the first-hit guides
        assert np.array_equal(bits(a), bits(b))
    r.set_option("gbuffer", 0)
    want = render(r, d, 0, 8, MODES["triangles"])
    r.render_adaptive(0.0, 4, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(want))


# ---- 5. errors --------------------------------------------------------------------------------------------------------------------
def test_refusals(frames, r):
    d = frames("medium").desc()
    before = render(r, d, 0, 2, MODES["uniform"])
    r.set_option("light_tree", 1)
    r.set_option("light_tree_triangles", 1)
    with pytest.raises(RuntimeError, match=r"lrk_upload_scene failed \(-5\)"):
        r.upload(d)
    r.set_option("light_tree", 0)
    with pytest.raises(RuntimeError, match=r"lrk_upload_scene failed \(-1\): .*set the option light_tree too"):
        r.upload(frames("cornell").desc())
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        r.set_option("light_tree_triangles", 2)
    assert np.array_equal(bits(render(r, d, 0, 2, MODES["uniform"])), bits(before))
