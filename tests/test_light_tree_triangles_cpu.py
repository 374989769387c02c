"""The triangle-level light trees (option "light_tree_triangles") without a GPU: the bottom trees of csrc/device/light_tree.h, built
in object space over a level-3 icosphere (one-sided, mirrored and two-sided), a quad, a single triangle, a soup with degenerate
triangles and a 20 480-triangle icosphere, and queried at world points mapped through identity, non-uniform and mirrored 3x4
transforms with the expressions the shade kernels use.  Also the top-level trees' bytes against the parent's, the option's surface
in Python and on the command line, and the emissive globe's generator."""
from __future__ import annotations

import hashlib

import numpy as np
import pytest
from scipy import stats

from light_sampling_checks import (MIRRORED, NONE, ONE_SIDED, TWO_SIDED, Bottom, LightSet, check_cli_flag, check_python_option,  # noqa: F401
                                   f32, icosphere, lib, quad, single, soup)


def cases():
    return [("ico3", icosphere(3), ONE_SIDED, "identity"), ("ico3", icosphere(3), ONE_SIDED, "stretched"),
            ("ico3", icosphere(3)[:, ::-1], MIRRORED, "mirrored"), ("ico3", icosphere(3), TWO_SIDED, "stretched"),
            ("quad", quad(), ONE_SIDED, "identity"), ("single", single(), ONE_SIDED, "stretched"),
            ("soup", soup(), ONE_SIDED, "identity"), ("soup", soup(), MIRRORED, "mirrored")]


CASES = cases()
IDS = [f"{c[0]}-{['one', 'mirrored', 'two'][c[2]]}-{c[3]}" for c in CASES]


@pytest.fixture(scope="module")
def big(lib):
    return Bottom(lib, icosphere(5), ONE_SIDED, "stretched")


def all_pmfs(b, p):
    return b.pmfs(p).T.astype(np.float64)  # [points, triangles]


# ---- 1. the pmf is a distribution, and sampling returns it bit for bit ------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_pmf_sums_to_one(lib, case):
    b = Bottom(lib, *case[1:])
    p = b.points(2_000, seed=1)
    total = all_pmfs(b, p).sum(axis=1)
    assert np.abs(total + b.dead_mass(p) - 1.0).max() <= 1e-5


def test_pmf_sums_to_one_on_a_large_mesh(big):
    p = big.points(64, seed=1)
    total = all_pmfs(big, p).sum(axis=1)
    assert np.abs(total + big.dead_mass(p) - 1.0).max() <= 1e-5


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_sampled_pmf_is_the_evaluated_pmf(lib, case):
    b = Bottom(lib, *case[1:])
    p = b.points(20_000, seed=2)
    tri, pmf = b.sample(p, np.random.default_rng(3).random(len(p)))
    chosen = tri != NONE
    assert chosen.mean() > 0.3
    assert (pmf[~chosen] == 0).all() and (pmf[chosen] > 0).all()
    for k in np.unique(tri[chosen]):
        sel = tri == k
        assert np.array_equal(b.pmf(p[sel], int(k)).view(np.uint32), pmf[sel].view(np.uint32))


def test_sampled_pmf_is_the_evaluated_pmf_on_a_large_mesh(big):
    p = big.points(20_000, seed=2)
    tri, pmf = big.sample(p, np.random.default_rng(3).random(len(p)))
    chosen = tri != NONE
    assert chosen.mean() > 0.3
    for i in np.flatnonzero(chosen)[:4000]:
        assert big.pmf(p[i:i + 1], int(tri[i]))[0].view(np.uint32) == pmf[i].view(np.uint32)


# ---- 2. conservative: every triangle that faces the point can be drawn ------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_every_facing_triangle_has_a_positive_pmf(lib, case):
    b = Bottom(lib, *case[1:])
    p = b.points(2_000, seed=4)
    pmf = all_pmfs(b, p)
    facing = b.facing(p)
    assert facing.any()
    assert (pmf[facing] > 0).all(), int((pmf[facing] == 0).sum())
    assert (b.dead_mass(p)[facing.any(axis=1)] < 1.0).all()  # P(no light) is 1 only where no triangle faces the point
    assert (pmf[:, ~b.facing(p, margin=-1.0).any(axis=0)] == 0).all()  # degenerate triangles are never drawn


def test_every_facing_triangle_has_a_positive_pmf_on_a_large_mesh(big):
    p = big.points(48, seed=4)
    pmf = all_pmfs(big, p)
    facing = big.facing(p)
    assert facing.any() and (pmf[facing] > 0).all()
    assert (big.dead_mass(p)[facing.any(axis=1)] < 1.0).all()


def test_orientation_favours_the_facing_side_of_a_sphere(lib):
    """Outside a one-sided sphere the tree puts on the triangles that face the point at least 1.5x the probability area sampling puts
    there (the fraction (1 - r/d) / 2 of the area, less than a half): the waste of shadow rays the option removes."""
    for side, kind, mesh in ((ONE_SIDED, "identity", icosphere(3)), (MIRRORED, "mirrored", icosphere(3)[:, ::-1])):
        b = Bottom(lib, mesh, side, kind)  # the mirrored instance of a sphere wound inwards faces outwards, as emissive_globe's
        c = b.world.reshape(-1, 3).mean(0)
        p = np.ascontiguousarray((c + np.array([[0.0, -1.6, 0.0], [2.5, 0.3, 0.0], [0.0, 0.0, -4.0]])), f32)
        pmf = all_pmfs(b, p)
        facing = b.facing(p, margin=0.0)
        w = b.world
        area = 0.5 * np.linalg.norm(np.cross(w[:, 1] - w[:, 0], w[:, 2] - w[:, 0]), axis=1)
        by_area = (facing * area).sum(axis=1) / area.sum()
        assert (by_area < 0.5).all()
        assert ((pmf * facing).sum(axis=1) >= 1.5 * by_area).all(), ((pmf * facing).sum(axis=1), by_area)


# ---- 3. the draws follow the pmf ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind, seed", [("identity", 11), ("stretched", 12)])
def test_sampled_frequencies_follow_the_pmf(lib, kind, seed):
    """Chi-square of 10^6 draws at one point inside and one outside the bounds; cells with an expected count below 5 pooled; fails at
    p < 1e-4."""
    b = Bottom(lib, icosphere(3), ONE_SIDED, kind)
    rng = np.random.default_rng(seed)
    c = b.world.reshape(-1, 3).mean(0)
    for p0 in np.array([c + (0.8, 0.8, 0.2), c + (0.0, -2.5, 0.5)], f32):  # inside the bounds (outside the sphere), and outside
        draws = 1_000_000
        p = np.ascontiguousarray(np.repeat(p0[None], draws, axis=0), f32)
        tri, _ = b.sample(p, rng.random(draws))
        want = all_pmfs(b, p[:1])[0]
        counts = np.bincount(tri[tri != NONE].astype(np.int64), minlength=b.n)[:b.n].astype(np.float64)
        assert counts[want == 0].sum() == 0
        expected = want * draws
        big_ = expected >= 5
        obs = np.append(counts[big_], counts[~big_].sum() + (tri == NONE).sum())
        exp = np.append(expected[big_], draws - expected[big_].sum())
        keep = exp > 0
        assert stats.chisquare(obs[keep], exp[keep] * obs[keep].sum() / exp[keep].sum()).pvalue > 1e-4


def test_top_walk_leaves_a_uniform_number(lib):
    """The u the sampling descent leaves at its leaf - the number the bottom walk continues with - is uniform on [0, 1) given the
    leaf, so one selection number serves both levels."""
    b = Bottom(lib, icosphere(2), ONE_SIDED, "identity")
    p = np.ascontiguousarray(np.repeat(np.array([[0.3, -2.0, 0.4]], f32), 400_000, axis=0))
    u = np.ascontiguousarray(np.random.default_rng(13).random(len(p)), f32)
    tri, u_left = np.zeros(len(p), np.uint32), np.zeros(len(p), f32)
    lib.ltt_sample_u_left(b.h, len(p), p.ctypes.data, u.ctypes.data, tri.ctypes.data, u_left.ctypes.data)
    u_left = u_left[tri != NONE]
    tri = tri[tri != NONE]
    assert len(tri) > 0.5 * len(p) and ((u_left >= 0) & (u_left < 1)).all()
    counts = np.bincount(tri.astype(np.int64))
    for k in np.argsort(counts)[-5:]:
        assert stats.kstest(u_left[tri == k], "uniform").pvalue > 1e-4


# ---- 4. the build ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_build_is_deterministic(lib, case):
    a = Bottom(lib, *case[1:]).bytes()
    assert a == Bottom(lib, *case[1:]).bytes()
    b = Bottom(lib, *case[1:])
    powered = int(b.facing(b.points(2, 0), margin=-np.inf).any(axis=0).sum()) if case[2] != TWO_SIDED else b.n
    assert len(a) == (2 * powered - 1) * 48 + 8 * b.n  # one 48-byte node per leaf and per inner node, one trail per triangle


def test_large_build_is_deterministic(lib, big):
    assert big.bytes() == Bottom(lib, icosphere(5), ONE_SIDED, "stretched").bytes()


def test_single_triangle_pmf_is_exactly_one(lib):
    b = Bottom(lib, single(), ONE_SIDED, "stretched")
    p = b.points(10_000, seed=6)
    facing = b.facing(p, margin=0.0)[:, 0]
    pmf = b.pmf(p, 0)
    assert (pmf == f32(1.0)).all()  # the root is the leaf: no choice, even where the triangle faces away
    tri, spmf = b.sample(p, np.random.default_rng(7).random(len(p)))
    assert (tri == 0).all() and (spmf == f32(1.0)).all() and facing.any() and not facing.all()


def test_mirrored_cones_are_the_negated_one_sided_ones(lib):
    one = Bottom(lib, icosphere(3), ONE_SIDED, "identity")
    mir = Bottom(lib, icosphere(3), MIRRORED, "mirrored")
    (na, ta), (nb, tb) = one.nodes_and_trails(), mir.nodes_and_trails()
    assert np.array_equal(ta, tb)
    ra, rb = na.view(f32).reshape(-1, 12), nb.view(f32).reshape(-1, 12)
    assert np.array_equal(ra[:, :7].view(np.uint32), rb[:, :7].view(np.uint32))  # bounds and power
    assert np.array_equal(ra[:, 7:10], -rb[:, 7:10])  # the axes, negated
    assert np.array_equal(ra[:, 10:].view(np.uint32), rb[:, 10:].view(np.uint32))  # cone cosines and indices
    two = Bottom(lib, icosphere(3), TWO_SIDED, "identity")
    rt = two.nodes_and_trails()[0].view(np.uint32).reshape(-1, 12)
    assert ((rt[:, 10] & 0xFFFF) == 0).all()  # the whole sphere
    leaf_phi = lambda r: {int(x[11]) & 0x7FFFFFFF: int(x[6]) for x in r if int(x[11]) & 0x80000000}
    assert leaf_phi(rt) == leaf_phi(ra.view(np.uint32))  # power = object-space area, not doubled


# ---- 5. the instance-level trees keep their bytes -------------------------------------------------------------------------------
# SHA-256 of the nodes and trails of LightSet(n, seed=n), taken at the commit before the triangle-level trees
PARENT_TOP_TREE_SHA256 = {
    1: "c1db4f2f46bd727f2872d1741e2a1e4f841f00e4754ccdce09be1869d1e88339",
    2: "eee2820fb4a1e8201741ebf6f54c7c49ce97a8393cdb54c2757a769564c343ce",
    7: "64bb2ff2736decbb0eabdfd262428b35ae66060e862c6ab7cc36f8afa64965c3",
    1000: "bab0993e8ac8bfca45cede6c7b438a1d8d7dd6eb63136a153a146e65cc5b7d62",
}


@pytest.mark.parametrize("n", sorted(PARENT_TOP_TREE_SHA256))
def test_instance_level_trees_keep_their_bytes(lib, n):
    assert hashlib.sha256(LightSet(n, seed=n).build(lib).bytes()).hexdigest() == PARENT_TOP_TREE_SHA256[n]


# ---- 6. the option's surface ------------------------------------------------------------------------------------------------------
def test_python_option_rejects_bad_values():
    check_python_option("light_tree_triangles")


def test_cli_lists_and_parses_light_tree_triangles(tmp_path):
    check_cli_flag("light_tree_triangles", tmp_path)


# ---- 7. the scene generator -------------------------------------------------------------------------------------------------------
def test_emissive_globe_generator():
    from luisarender_b200 import scenes

    for t in ("uniform", "stretched", "mirrored"):
        s = scenes.emissive_globe(resolution=(16, 16), spp=1, subdivision=2, transform=t)
        assert s.count("light { @globe_light }") == 1 and "two_sided { false }" in s
        assert ("transform : Matrix" in s) == (t != "uniform")
    with pytest.raises(ValueError):
        scenes.emissive_globe(transform="sheared")
    m = scenes.emissive_globe(subdivision=1, transform="mirrored")
    vals = [float(x) for x in m.split("transform : Matrix { m { ")[1].split(" }")[0].split(",")]
    assert np.linalg.det(np.array(vals).reshape(4, 4)[:3, :3]) < 0
