"""The light tree (option "light_tree") without a GPU: csrc/device/light_tree.h, the header the shade kernels and lrk_upload_scene
include, compiled for the host and checked on synthetic light sets of 1, 2, 7 and 1000 emitters that mix one-sided, two-sided,
coincident and zero-power lights, at points inside and outside their bounds.  Also the option's surface in Python and on the
command line, and the many-light scene generator."""
from __future__ import annotations

import numpy as np
import pytest
from scipy import stats

from light_sampling_checks import NONE, LightSet, check_cli_flag, check_python_option, f32, lib  # noqa: F401 (lib: the harness's fixture)


SETS = [1, 2, 7, 1000]


@pytest.mark.parametrize("n", SETS)
def test_pmf_sums_to_one(lib, n):
    """Over 10^4 points, the pmfs of all emitters and the probability of a descent that finds no emitter (both children of 0
    importance, which happens only where neither can emit towards the point) sum to 1."""
    ls = LightSet(n, seed=n)
    tree = ls.build(lib)
    p = ls.points(10_000, seed=1)
    total = np.zeros(len(p), np.float64)
    for e in range(n):
        total += tree.pmf(p, e)
    dead = tree.dead_mass(p)
    assert np.abs(total + dead - 1.0).max() <= 1e-5
    assert (total <= 1.0 + 1e-5).all()


@pytest.mark.parametrize("n", SETS)
def test_sampled_pmf_is_the_evaluated_pmf(lib, n):
    ls = LightSet(n, seed=n)
    tree = ls.build(lib)
    p = ls.points(10_000, seed=2)
    light, pmf = tree.sample(p, np.random.default_rng(3).random(len(p)))
    chosen = light != NONE
    assert chosen.mean() > 0.5
    assert (pmf[~chosen] == 0).all() and (pmf[chosen] > 0).all()
    for e in np.unique(light[chosen]):
        sel = light == e
        assert np.array_equal(tree.pmf(p[sel], int(e)).view(np.uint32), pmf[sel].view(np.uint32))


@pytest.mark.parametrize("n", SETS)
def test_every_emitter_that_can_illuminate_has_a_positive_pmf(lib, n):
    ls = LightSet(n, seed=n)
    tree = ls.build(lib)
    p = ls.points(2_000 if n == 1000 else 10_000, seed=4)
    rng = np.random.default_rng(5)
    reached = 0
    for e in range(n):
        pmf = tree.pmf(p, e)
        lit = ls.can_illuminate(e, p, rng)
        assert (pmf[lit] > 0).all(), (e, int((pmf[lit] == 0).sum()))
        if ls.power[e] == 0.0:
            assert (pmf == 0).all()
        reached += lit.sum()
    assert reached > 0


@pytest.mark.parametrize("n, seed", [(7, 11), (1000, 12)])
def test_sampled_frequencies_follow_the_pmf(lib, n, seed):
    """Chi-square of 10^6 draws at one point inside and one outside the bounds.  Cells with an expected count below 5 are pooled;
    the test fails at p < 1e-4, one false alarm in 10^4 seeds."""
    ls = LightSet(n, seed=n)
    tree = ls.build(lib)
    rng = np.random.default_rng(seed)
    for p0 in ls.points(2, seed=seed):
        draws = 1_000_000
        p = np.ascontiguousarray(np.repeat(p0[None], draws, axis=0), f32)
        light, _ = tree.sample(p, rng.random(draws))
        want = np.array([tree.pmf(p[:1], e)[0] for e in range(n)], np.float64)
        counts = np.bincount(light[light != NONE].astype(np.int64), minlength=n)[:n].astype(np.float64)
        expected = want * draws
        assert counts[want == 0].sum() == 0
        big = expected >= 5
        obs = np.append(counts[big], counts[~big].sum() + (light == NONE).sum())
        exp = np.append(expected[big], draws - expected[big].sum())
        keep = exp > 0
        assert stats.chisquare(obs[keep], exp[keep] * obs[keep].sum() / exp[keep].sum()).pvalue > 1e-4


@pytest.mark.parametrize("n", SETS)
def test_build_is_deterministic(lib, n):
    a = LightSet(n, seed=n).build(lib).bytes()
    b = LightSet(n, seed=n).build(lib).bytes()
    assert a == b
    powered = sum(1 for w in LightSet(n, seed=n).power if w > 0)
    assert len(a) == (2 * powered - 1) * 48 + 8 * n  # one 48-byte node per leaf and per inner node


def test_single_light_pmf_is_exactly_one(lib):
    ls = LightSet(1, seed=1)
    tree = ls.build(lib)
    p = ls.points(10_000, seed=6)
    assert (tree.pmf(p, 0) == f32(1.0)).all()
    light, pmf = tree.sample(p, np.random.default_rng(7).random(len(p)))
    assert (light == 0).all() and (pmf == f32(1.0)).all()


def test_python_option_rejects_unknown_values():
    check_python_option("light_tree")


def test_cli_lists_and_parses_light_tree(tmp_path):
    check_cli_flag("light_tree", tmp_path)


def test_many_light_scene_generator():
    from luisarender_b200 import scenes

    own = scenes.many_lights(resolution=(32, 18), count=12)
    shared = scenes.many_lights(resolution=(32, 18), count=12, shared_node=True)
    assert own.count("Light sphere_light_") == 12 and own.count("light { @sphere_light_") == 12
    assert shared.count("Light sphere_light ") == 1 and shared.count("light { @sphere_light }") == 12
    assert "sphere_light" not in scenes.instanced_spheres()
