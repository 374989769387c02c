"""The light tree on the GPU (option "light_tree"; include/lrk.h, csrc/device/light_tree.h).

Off, the option must change nothing; on, a scene with one light must render bit for bit as without it, the many-light frame must
render the same image as the uniform sampler within its noise (and with less of it), shapes that share a Light node must all be
sampled, and scheduling, sharding, the G-buffer mode and the adaptive mode must compose with it unchanged.  The checks every
light-sampling option passes are in light_sampling_checks.py.
"""
from __future__ import annotations

import numpy as np
import pytest

from light_sampling_checks import (SUB_SPP, SUBRENDERS, Z_MAX, bits, check_agrees_without_it, check_error_ratio,  # noqa: F401
                                   check_gbuffer_and_adaptive, check_off_equals_a_fresh_context, check_refusals,
                                   check_scheduling_and_sharding, frames, r, render, sub_renders, z_scores)

pytestmark = pytest.mark.gpu
UNIFORM, TREE = {"light_tree": 0}, {"light_tree": 1}


# ---- 1. off changes nothing -------------------------------------------------------------------------------------------------------
def test_option_off_equals_a_context_that_never_set_it(frames, r):
    check_off_equals_a_fresh_context(r, frames("spheres_small").desc(), {}, None, [UNIFORM])


# ---- 2. one light: the tree's pmf is exactly 1 -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cornell_small", "textured_wrappers_small", "environment_one_light"])
def test_one_light_scenes_render_bit_identically(frames, name, r):
    d = frames(name).desc()
    assert sum(1 for i in range(d.instance_count) if d.instances[i].handle[0] & 8) == 1  # one emissive instance
    off = render(r, d, 0, 8, UNIFORM)
    on = render(r, d, 0, 8, TREE)
    assert np.array_equal(bits(on), bits(off))


# ---- 3. unbiased: the same image as the uniform sampler ---------------------------------------------------------------------------
def test_many_lights_tree_agrees_with_uniform(frames, r):
    check_agrees_without_it(r, frames("many").desc(), UNIFORM, TREE)


def test_shared_light_node_is_sampled_whole(frames, r):
    """With the tree, spheres that share one Light node light the frame as spheres with a node each do under the uniform sampler;
    the uniform sampler draws only the first of the shared ones, and its MIS weights drop part of the others' light."""
    own = sub_renders(r, frames("many_equal").desc(), UNIFORM, 0, SUBRENDERS, SUB_SPP)
    shared_tree = sub_renders(r, frames("many_shared").desc(), TREE, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)
    z = z_scores(shared_tree, own)
    assert np.abs(z).max() < Z_MAX, z
    shared_uniform = sub_renders(r, frames("many_shared").desc(), UNIFORM, 2 * SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)
    assert z_scores(shared_uniform, own)[0] < -Z_MAX  # the whole image is darker beyond its noise


# ---- 4. less noise ----------------------------------------------------------------------------------------------------------------
def test_many_lights_tree_halves_the_error(frames, r):
    """16 spp against a 1024-spp reference of disjoint sample indices: relative MSE of the tree at most 0.5x that of the uniform
    sampler, averaged over 8 independent 16-spp renders each.  Measured on an H100 80GB HBM3 at a 700 W power limit: 0.3543 in the
    strict and 0.3544 in the fast arithmetic mode."""
    check_error_ratio(r, frames("many").desc(), UNIFORM, TREE, 0.5, "many")


# ---- 5. scheduling and the other modes --------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(frames, r):
    check_scheduling_and_sharding(r, frames("many").desc(), TREE)


def test_gbuffer_and_adaptive_compose(frames, r):
    check_gbuffer_and_adaptive(r, frames("many").desc(), UNIFORM, TREE)


# ---- 6. errors --------------------------------------------------------------------------------------------------------------------
def test_volume_integrator_is_refused_at_upload(frames, r):
    check_refusals(r, frames, frames("medium").desc(), UNIFORM,
                   [TREE, ("upload", "medium", r"lrk_upload_scene failed \(-5\): .*light tree"), ("set", "light_tree", 2)])
