"""Resampled next-event estimation on the GPU (option "light_candidates"; include/lrk.h, csrc/device/light_resampling.h).

Values 0 and 1 must change nothing; M >= 2 must render the same image as one light sample within its noise on every kind of frame
and light sampling, match Lambert's formula on the irradiance frame, lower the noise of the glossy-desk frame, and compose with
scheduling, sharding, the G-buffer mode and the adaptive mode unchanged.  The checks every light-sampling option passes are in
light_sampling_checks.py.
"""
from __future__ import annotations

import pytest

from light_sampling_checks import (check_agrees_without_it, check_error_ratio, check_gbuffer_and_adaptive,  # noqa: F401
                                   check_irradiance_frame_matches_lambert, check_off_equals_a_fresh_context, check_refusals,
                                   check_scheduling_and_sharding, frames, r)

pytestmark = pytest.mark.gpu
SINGLE = {"light_candidates": 0}


def candidates(m):
    return {"light_candidates": m}


# ---- 1. values 0 and 1 change nothing ---------------------------------------------------------------------------------------------
def test_values_zero_and_one_equal_a_context_that_never_set_the_option(frames, r):
    # M = 4 renders first, leaving the resampling kernels behind in this context
    check_off_equals_a_fresh_context(r, frames("cornell").desc(), {}, candidates(4), [candidates(0), candidates(1)])


# ---- 2. unbiased: the same image as one light sample ------------------------------------------------------------------------------
CASES = [  # (id, frame, other light-sampling options, M)
    ("cornell", "cornell", {}, 4),
    ("textured_lamp", "textured_lamp", {}, 4),
    ("environment_area", "environment_area", {}, 4),
    ("flatten", "flatten", {}, 4),
    ("many_tree", "many", {"light_tree": 1}, 4),
    ("many_tree_triangles", "many", {"light_tree": 1, "light_tree_triangles": 1}, 4),
    ("many_solid_angle", "many", {"light_solid_angle": 1}, 4),
    ("materials_mix", "mix_64x48", {}, 4),
    ("layered", "layered_64x48", {}, 4),
    ("padded_sobol", "sobol_cornell", {}, 4),
    ("cornell_m32", "cornell", {}, 32),
]


@pytest.mark.parametrize("frame, options, m", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_resampling_agrees_with_one_light_sample(frames, r, frame, options, m):
    check_agrees_without_it(r, frames(frame).desc(), {**options, **SINGLE}, {**options, **candidates(m)})


# ---- 3. the irradiance frame against Lambert's formula ----------------------------------------------------------------------------
def test_irradiance_frame_matches_lambert(frames, r):
    check_irradiance_frame_matches_lambert(r, frames("irradiance").desc(), candidates(8))


# ---- 4. less noise where the closure decides which light samples matter -----------------------------------------------------------
# The 16-spp relative MSE at M = 8 over that at M = 1 on the 96x96 glossy-desk frame, each averaged over 8 renders.  Measured on an
# NVIDIA H100 80GB HBM3 (700 W power limit): 0.9556 in the fast and 0.9561 in the strict arithmetic mode (DESIGN.md §5).  The renders
# are seeded, so the bound's margin is for changes of the code around the estimator, not for chance.
GLOSSY_DESK_ERROR_RATIO = 0.98


def test_glossy_desk_error_is_lower(frames, r):
    check_error_ratio(r, frames("glossy_desk").desc(), SINGLE, candidates(8), GLOSSY_DESK_ERROR_RATIO, "glossy_desk")


# ---- 5. scheduling and sharding ---------------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(frames, r):
    check_scheduling_and_sharding(r, frames("glossy_desk").desc(), candidates(4))


# ---- 6. the other modes -----------------------------------------------------------------------------------------------------------
def test_gbuffer_and_adaptive_compose(frames, r):
    check_gbuffer_and_adaptive(r, frames("glossy_desk").desc(), SINGLE, candidates(4))


# ---- 7. errors --------------------------------------------------------------------------------------------------------------------
def test_volume_integrator_and_bad_values_are_refused(frames, r):
    check_refusals(r, frames, frames("medium").desc(), SINGLE,
                   [candidates(2), ("upload", "medium", r"lrk_upload_scene failed \(-5\): .*light_candidates"),
                    ("set", "light_candidates", -1), ("set", "light_candidates", 33)])
