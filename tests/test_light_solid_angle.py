"""Solid-angle light sampling on the GPU (option "light_solid_angle"; include/lrk.h, csrc/device/spherical_triangle.h).

Off, the option must change nothing; on, every frame must render the same image as area sampling within its noise, the irradiance
frame must match Lambert's formula, the near-light frame must have less noise, and scheduling, sharding, the G-buffer mode and
the adaptive mode must compose with it unchanged.  The checks every light-sampling option passes are in light_sampling_checks.py.
"""
from __future__ import annotations

import pytest

from light_sampling_checks import (check_agrees_without_it, check_error_ratio, check_gbuffer_and_adaptive,  # noqa: F401
                                   check_irradiance_frame_matches_lambert, check_off_equals_a_fresh_context, check_refusals,
                                   check_scheduling_and_sharding, frames, r)

pytestmark = pytest.mark.gpu
AREA, SOLID_ANGLE = {"light_solid_angle": 0}, {"light_solid_angle": 1}


# ---- 1. off changes nothing -------------------------------------------------------------------------------------------------------
def test_option_off_equals_a_context_that_never_set_it(frames, r):
    # the option renders first, leaving its kernels behind in this context
    check_off_equals_a_fresh_context(r, frames("cornell").desc(), {}, SOLID_ANGLE, [AREA])


# ---- 2. unbiased: the same image as area sampling ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cornell", "textured_lamp", "environment_area", "flatten", "many"])
def test_solid_angle_agrees_with_area_sampling(frames, name, r):
    if name == "many":
        r.set_option("light_tree", 1)  # both choices of next-event estimation at once
    check_agrees_without_it(r, frames(name).desc(), AREA, SOLID_ANGLE)


# ---- 3. the irradiance frame against Lambert's formula ----------------------------------------------------------------------------
@pytest.mark.parametrize("solid_angle", [False, True])
def test_irradiance_frame_matches_lambert(frames, r, solid_angle):
    check_irradiance_frame_matches_lambert(r, frames("irradiance").desc(), {"light_solid_angle": solid_angle})


# ---- 4. less noise where the light is large and close -----------------------------------------------------------------------------
# The 16-spp relative MSE of the option over that of area sampling on the 96x96 near-light frame, each averaged over 8 renders.
# Measured on an H100: 0.707 in both arithmetic modes (DESIGN.md §5).  The renders are seeded, so the bound's margin is for changes
# of the code around the sampler, not for chance.
NEAR_LIGHT_ERROR_RATIO = 0.8


def test_near_light_error_is_lower(frames, r):
    check_error_ratio(r, frames("near").desc(), AREA, SOLID_ANGLE, NEAR_LIGHT_ERROR_RATIO, "near_light")


# ---- 5. scheduling and the other modes --------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(frames, r):
    check_scheduling_and_sharding(r, frames("near").desc(), SOLID_ANGLE)


def test_gbuffer_and_adaptive_compose(frames, r):
    check_gbuffer_and_adaptive(r, frames("near").desc(), AREA, SOLID_ANGLE)


# ---- 6. errors --------------------------------------------------------------------------------------------------------------------
def test_volume_integrator_and_bad_values_are_refused(frames, r):
    check_refusals(r, frames, frames("medium").desc(), AREA,
                   [SOLID_ANGLE, ("upload", "medium", r"lrk_upload_scene failed \(-5\): .*solid-angle"), ("set", "light_solid_angle", 2)])
