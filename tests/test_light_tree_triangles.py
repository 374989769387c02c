"""The triangle-level light trees on the GPU (option "light_tree_triangles"; include/lrk.h, csrc/device/light_tree.h).

Off, the option must change nothing; on, scenes whose emitters are single triangles must render bit for bit as without it, every
frame must render the same image as the uniform sampler within its noise, the emissive globe and the many-light frame must have
less noise than with the instance-level tree, and scheduling, sharding, the G-buffer mode and the adaptive mode must compose with
it unchanged.  The checks every light-sampling option passes are in light_sampling_checks.py.
"""
from __future__ import annotations

import numpy as np
import pytest

from light_sampling_checks import (SUB_SPP, Z_MAX, bits, check_agrees_without_it, check_error_ratio,  # noqa: F401
                                   check_gbuffer_and_adaptive, check_off_equals_a_fresh_context, check_refusals,
                                   check_scheduling_and_sharding, frames, r, render, sub_renders)

pytestmark = pytest.mark.gpu
MODES = {"uniform": {"light_tree": 0, "light_tree_triangles": 0}, "tree": {"light_tree": 1, "light_tree_triangles": 0},
         "triangles": {"light_tree": 1, "light_tree_triangles": 1}}


# ---- 1. off changes nothing; single-triangle emitters render bit for bit ----------------------------------------------------------
def test_option_off_equals_a_context_that_never_set_it(frames, r):
    # the triangle trees render first, leaving the bottom trees behind in this context
    check_off_equals_a_fresh_context(r, frames("many").desc(), {"light_tree": True}, MODES["triangles"], [MODES["tree"]])


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
    r.set_option("light_solid_angle", solid_angle)
    check_agrees_without_it(r, frames(name).desc(), MODES["uniform"], MODES["triangles"])


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
    check_error_ratio(r, frames(name).desc(), MODES["tree"], MODES["triangles"], ERROR_RATIO_BOUND[name], name)


# ---- 4. scheduling and the other modes --------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(frames, r):
    check_scheduling_and_sharding(r, frames("many").desc(), MODES["triangles"])


def test_gbuffer_and_adaptive_compose(frames, r):
    check_gbuffer_and_adaptive(r, frames("globe_stretched").desc(), MODES["tree"], MODES["triangles"])


# ---- 5. errors --------------------------------------------------------------------------------------------------------------------
def test_refusals(frames, r):
    check_refusals(r, frames, frames("medium").desc(), MODES["uniform"],
                   [MODES["triangles"], ("upload", "medium", r"lrk_upload_scene failed \(-5\)"), {"light_tree": 0},
                    ("upload", "cornell", r"lrk_upload_scene failed \(-1\): .*set the option light_tree too"),
                    ("set", "light_tree_triangles", 2)])
