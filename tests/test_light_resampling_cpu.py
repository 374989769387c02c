"""Resampled next-event estimation (option "light_candidates") without a GPU: csrc/device/light_resampling.h, the header the shade
kernels include, compiled for the host - the reservoir's choice, the candidates' numbers, the estimator's mean and variance on a
synthetic discrete problem, and the single-candidate weight.  Also the option's surface in Python and on the command
line, and the glossy-desk scene generator."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
from scipy import stats

import host_harness
from light_sampling_checks import check_cli_flag, check_python_option

f32 = np.float32


@pytest.fixture(scope="module")
def lib():
    deps = [host_harness.DEVICE / "light_resampling.h", host_harness.DEVICE / "vecmath.cuh"]
    h = host_harness.load("light_resampling_host", deps, ["-O2", "-ffp-contract=off", host_harness.cuda_include_flag()])
    h.lr_choose.argtypes = [C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    h.lr_candidates.argtypes = [C.c_int64, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p]
    h.lr_estimate.argtypes = [C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    h.lr_single.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    return h


def choose(lib, w, draws, seed):
    w = np.ascontiguousarray(w, f32)
    u = np.ascontiguousarray(np.random.default_rng(seed).random((draws, len(w))), f32)
    out = np.zeros(draws, np.int32)
    lib.lr_choose(draws, len(w), w.ctypes.data, u.ctypes.data, out.ctypes.data)
    return out


def candidates(lib, triples, m, depth=3):
    triples = np.ascontiguousarray(triples, f32)
    out = np.zeros((len(triples), m, 4), f32)
    lib.lr_candidates(len(triples), triples.ctypes.data, depth, m, out.ctypes.data)
    return out


def estimate(lib, p, c, b, m, u):
    p, c, b, u = (np.ascontiguousarray(a, f32) for a in (p, c, b, u))
    out = np.zeros((len(u), 3), f32)
    lib.lr_estimate(len(u), len(p), p.ctypes.data, c.ctypes.data, b.ctypes.data, m, u.ctypes.data, out.ctypes.data)
    return out.astype(np.float64)


# ---- the reservoir ----------------------------------------------------------------------------------------------------------------
WEIGHT_SETS = {
    "equal": [1.0, 1.0, 1.0, 1.0],
    "dominant": [1000.0, 1.0, 2.0, 0.5],
    "zeros": [0.0, 2.0, 0.0, 1.0, 0.0],
    "non_finite": [1.0, np.nan, 2.0, np.inf, 0.5, -np.inf, -1.0],
    "dominant_last": [0.1, 0.2, 0.3, 50.0],
}


@pytest.mark.parametrize("name", sorted(WEIGHT_SETS))
def test_reservoir_choice_follows_the_weights(lib, name):
    """Chi-square of 10^6 choices against w_i / W, with weights that are not finite and positive counted as 0; fails at p < 1e-4."""
    w = np.array(WEIGHT_SETS[name], np.float64)
    valid = np.isfinite(w) & (w > 0)
    draws = 1_000_000
    got = choose(lib, w, draws, seed=sorted(WEIGHT_SETS).index(name))
    assert (got >= 0).all()
    counts = np.bincount(got, minlength=len(w))
    assert (counts[~valid] == 0).all()
    expected = np.where(valid, w, 0.0) / np.where(valid, w, 0.0).sum() * draws
    keep = expected > 0
    assert stats.chisquare(counts[keep], expected[keep]).pvalue > 1e-4


def test_all_zero_weights_give_no_sample(lib):
    assert (choose(lib, [0.0, 0.0, np.nan, 0.0], 1000, seed=9) == -1).all()
    assert (choose(lib, [0.0], 10, seed=9) == -1).all()


# ---- the candidates' numbers ------------------------------------------------------------------------------------------------------
def test_candidate_zero_is_the_bounce_numbers_and_the_stream_is_deterministic(lib):
    t = np.random.default_rng(1).random((10_000, 3)).astype(f32)
    a, b = candidates(lib, t, 8), candidates(lib, t, 8)
    assert np.array_equal(a[:, 0, :3].view(np.uint32), t.view(np.uint32))
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert (a >= 0).all() and (a < 1).all()
    # the depth is part of the seed
    assert not np.array_equal(candidates(lib, t, 8, depth=4)[:, 1:], a[:, 1:])


def test_candidate_numbers_are_uniform(lib):
    """Chi-square over 64 bins of each of the four numbers of candidates 1 and 7 for 10^6 seeds; fails at p < 1e-4."""
    t = np.random.default_rng(2).random((1_000_000, 3)).astype(f32)
    nums = candidates(lib, t, 8)
    for i in (1, 7):
        for q in range(4):
            counts = np.bincount(np.minimum((nums[:, i, q] * 64).astype(int), 63), minlength=64)
            assert stats.chisquare(counts).pvalue > 1e-4, (i, q)
    # and the numbers of one candidate are not correlated with each other or with the bounce's
    assert abs(np.corrcoef(nums[:, 1, 0], nums[:, 1, 1])[0, 1]) < 5e-3
    assert abs(np.corrcoef(nums[:, 0, 0], nums[:, 1, 0])[0, 1]) < 5e-3


# ---- the estimator ----------------------------------------------------------------------------------------------------------------
# six lights: source pmf p (not proportional to the contribution), rgb contributions c (one light contributes nothing), MIS partner
# pdfs b (the closure's pdf of the light's direction)
P = np.array([0.05, 0.3, 0.1, 0.25, 0.2, 0.1])
CONTRIB = np.array([[4.0, 0.5, 0.2], [0.1, 0.1, 0.1], [0.0, 0.0, 0.0], [1.0, 2.0, 3.0], [0.3, 0.9, 0.1], [6.0, 6.0, 0.5]])
B = np.array([0.0, 0.5, 2.0, 0.1, 0.0, 3.0])


@pytest.mark.parametrize("m", [1, 2, 4, 8, 32])
def test_estimator_is_unbiased(lib, m):
    """The mean of 4 x 10^5 estimates equals sum_l c_l p_l / (p_l + b_l) per channel within 4 sigma."""
    n = 400_000
    u = np.random.default_rng(10 + m).random((n, 3))
    est = estimate(lib, P, CONTRIB, B, m, u)
    p, c, b = (np.asarray(a, f32).astype(np.float64) for a in (P, CONTRIB, B))
    want = (c * (p / (p + b))[:, None]).sum(axis=0)
    se = est.std(axis=0, ddof=1) / np.sqrt(n)
    assert (np.abs(est.mean(axis=0) - want) <= 4.0 * se + 1e-6 * want).all(), (est.mean(axis=0), want, se)


def test_variance_falls_as_one_over_m_for_a_proportional_target(lib):
    """Grey contributions and no MIS partner make the target exactly proportional to c: the estimate at M = 8 is then the mean of 8
    independent importance-sampling estimates, so its variance is 1/8 of that at M = 1.  Margin: 10 % for the spread of the two
    variance estimates over 4 x 10^5 draws (their relative standard error is about 1 % here)."""
    n = 400_000
    grey = np.repeat(np.array([4.0, 0.1, 0.0, 2.0, 0.6, 6.0])[:, None], 3, axis=1)
    zero = np.zeros(len(P))
    v1 = estimate(lib, P, grey, zero, 1, np.random.default_rng(20).random((n, 3)))[:, 0].var()
    v8 = estimate(lib, P, grey, zero, 8, np.random.default_rng(21).random((n, 3)))[:, 0].var()
    print(f"variance M=1 {v1:.5g}, M=8 {v8:.5g}, ratio {v8 / v1:.4f}")
    assert v8 <= v1 / 8 * 1.1


def test_single_candidate_weight_is_c_over_p(lib):
    """M = 1: c * W / (1 * p_hat) = c * (p_hat / p) / p_hat equals c / p to within 2 ulp per channel."""
    rng = np.random.default_rng(30)
    n = 200_000
    c = (rng.random((n, 3)) * 10.0 ** rng.uniform(-3, 3, (n, 1))).astype(f32)
    p = (10.0 ** rng.uniform(-4, 4, n)).astype(f32)
    out = np.zeros((n, 3), f32)
    lib.lr_single(n, c.ctypes.data, p.ctypes.data, out.ctypes.data)
    want = c / p[:, None]
    assert (np.abs(out - want) <= 2 * np.spacing(want)).all()


# ---- the option's surface ---------------------------------------------------------------------------------------------------------
def test_python_option_accepts_counts_and_rejects_other_values():
    check_python_option("light_candidates")


def test_cli_lists_and_parses_light_candidates(tmp_path):
    check_cli_flag("light_candidates", tmp_path)


# ---- the scene generator ----------------------------------------------------------------------------------------------------------
def test_glossy_desk_scene_generator():
    from luisarender_b200 import scenes

    plain = scenes.near_light(resolution=(32, 18))
    glossy = scenes.near_light(resolution=(32, 18), glossy_desk=True)
    assert "Surface desk : Matte" in plain and "Disney" not in plain
    assert "Surface desk : Disney" in glossy and "roughness : Constant { v { 0.15 } }" in glossy and "metallic : Constant { v { 0.6 } }" in glossy
    assert glossy.replace(next(line for line in glossy.splitlines() if line.startswith("Surface desk")),
                          next(line for line in plain.splitlines() if line.startswith("Surface desk"))) == plain
