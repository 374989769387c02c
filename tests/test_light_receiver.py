"""Receiver-aware light sampling on the GPU (option "light_receiver"; include/lrk.h, csrc/device/receiver.h, the receiver term of
light_tree.h and the warp of spherical_triangle.h).

Off, the option must change nothing; on, every frame must render the same image as without it within its noise, the irradiance
frame must match Lambert's formula, the near-light and many-light frames are measured for noise, and scheduling, sharding, the
G-buffer mode and the adaptive mode must compose with it unchanged.  The checks every light-sampling option passes are in
light_sampling_checks.py.
"""
from __future__ import annotations

import numpy as np
import pytest

from light_sampling_checks import (bits, check_agrees_without_it, check_error_ratio, check_gbuffer_and_adaptive,  # noqa: F401
                                   check_irradiance_frame_matches_lambert, check_off_equals_a_fresh_context, check_refusals,
                                   check_scheduling_and_sharding, frames, r, render)

pytestmark = pytest.mark.gpu
OFF, ON = {"light_receiver": 0}, {"light_receiver": 1}
TREE, SOLID, TRIANGLES = {"light_tree": 1}, {"light_solid_angle": 1}, {"light_tree": 1, "light_tree_triangles": 1}


# ---- 1. off changes nothing -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("base", [TREE, SOLID], ids=["tree", "solid_angle"])
def test_option_off_equals_a_context_that_never_set_it(frames, r, base):
    # the option renders first, leaving the receiver words behind in this context
    check_off_equals_a_fresh_context(r, frames("many").desc(), {name: True for name in base}, {**base, **ON}, [{**base, **OFF}])


# ---- 2. unbiased: the same image as without the option ----------------------------------------------------------------------------
CASES = [("cornell", SOLID), ("cornell", {**TREE, **SOLID}), ("textured_lamp", SOLID), ("environment_area", {**TREE, **SOLID}), ("flatten", SOLID),
         ("mix", SOLID), ("layered", SOLID), ("many", TREE), ("many", TRIANGLES), ("many", SOLID), ("small_globe_uniform", TRIANGLES),
         ("small_globe_stretched", TRIANGLES), ("small_globe_mirrored", TRIANGLES), ("cornell", {**SOLID, "light_candidates": 4})]


# ids name a globe by its transform alone
@pytest.mark.parametrize("name,base", CASES, ids=[f"{n.replace('small_', '')}-{'+'.join(sorted(b))}" for n, b in CASES])
def test_receiver_agrees_without_it(frames, r, name, base):
    check_agrees_without_it(r, frames(name).desc(), {**base, **OFF}, {**base, **ON}, changes_the_film=True)


def test_one_emitter_tree_is_unchanged(frames, r):
    """The Cornell box has one emissive instance: the tree picks it with probability 1 at any receiver, so the option leaves the
    tree-only film bit for bit as it was."""
    d = frames("cornell").desc()
    assert np.array_equal(bits(render(r, d, 0, 4, {**TREE, **OFF})), bits(render(r, d, 0, 4, {**TREE, **ON})))


# ---- 3. the irradiance frame against Lambert's formula ----------------------------------------------------------------------------
def test_irradiance_frame_matches_lambert(frames, r):
    check_irradiance_frame_matches_lambert(r, frames("irradiance").desc(), {**SOLID, **ON})


# ---- 4. noise at equal spp ---------------------------------------------------------------------------------------------------------
# The 16-spp relative MSE with the option over that without it, each averaged over 8 renders.  Measured on an H100 80GB HBM3 at a
# 700 W power limit: near_light (solid angle) 0.9565 in both arithmetic modes, the many-light frame (tree) 0.9584 strict and 0.9576
# fast (DESIGN.md §5).  The renders are seeded, so the bound's margin is for changes of the code around the samplers, not for chance.
ERROR_RATIO = 0.98


@pytest.mark.parametrize("name,base", [("near", SOLID), ("many", TREE)], ids=["near_light-solid_angle", "many_lights-tree"])
def test_error_at_16_spp(frames, r, name, base):
    check_error_ratio(r, frames(name).desc(), {**base, **OFF}, {**base, **ON}, ERROR_RATIO, name)


# ---- 5. scheduling and the other modes --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("base", [SOLID, TRIANGLES], ids=["solid_angle", "tree_triangles"])
def test_scheduling_and_sharding_change_no_bit(frames, r, base):
    check_scheduling_and_sharding(r, frames("many").desc(), {**base, **ON})


def test_gbuffer_and_adaptive_compose(frames, r):
    check_gbuffer_and_adaptive(r, frames("near").desc(), {**SOLID, **OFF}, {**SOLID, **ON})


# ---- 6. errors --------------------------------------------------------------------------------------------------------------------
def test_refusals_keep_the_previous_film(frames, r):
    check_refusals(r, frames, frames("cornell").desc(), {**SOLID, **OFF},
                   [{"light_solid_angle": 0, **ON}, ("upload", "cornell", r"lrk_upload_scene failed \(-1\): .*light_receiver"),
                    ("set", "light_receiver", 2), "film", ("upload", "medium", r"lrk_upload_scene failed \(-5\)")])
