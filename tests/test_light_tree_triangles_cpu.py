"""The triangle-level light trees (option "light_tree_triangles") without a GPU: the bottom trees of csrc/device/light_tree.h, built
in object space over a level-3 icosphere (one-sided, mirrored and two-sided), a quad, a single triangle, a soup with degenerate
triangles and a 20 480-triangle icosphere, and queried at world points mapped through identity, non-uniform and mirrored 3x4
transforms with the expressions the shade kernels use.  Also the top-level trees' bytes against the parent's, and the option's
surface in Python and on the command line."""
from __future__ import annotations

import hashlib

import numpy as np
import pytest
from scipy import stats

from light_sampling_checks import check_cli_lists_and_parses_flag, check_python_option_rejects_bad_values
from luisarender_b200.scenes import _icosphere
from test_light_tree_cpu import LightSet, lib  # noqa: F401 (lib: the fixture of light_tree.h's harness)

NONE = 0xFFFFFFFF
ONE_SIDED, MIRRORED, TWO_SIDED = 0, 1, 2
f32 = np.float32


# ---- meshes (object space, [n, 3, 3]) and transforms (object-to-world 3x4) -------------------------------------------------------
def icosphere(level):
    v, f = _icosphere(level)
    return v[f]


def quad():
    v = np.array([(-1.0, 0.0, -1.0), (1.0, 0.0, -1.0), (1.0, 0.0, 1.0), (-1.0, 0.0, 1.0)])
    return np.array([[v[0], v[2], v[1]], [v[0], v[3], v[2]]])  # normal +y


def single():
    return np.array([[(0.1, 0.2, 0.0), (1.3, -0.1, 0.2), (0.4, 0.9, -0.3)]])


def soup():
    """Random triangles, every fourth degenerate (two coincident vertices or three collinear ones)."""
    rng = np.random.default_rng(5)
    t = rng.uniform(-1.0, 1.0, (40, 3, 3))
    t[::8, 1] = t[::8, 0]
    t[4::8, 2] = 0.5 * (t[4::8, 0] + t[4::8, 1])
    return t


def xform(kind):
    if kind == "identity":
        return np.hstack([np.eye(3), np.zeros((3, 1))])
    if kind == "stretched":  # rotation times non-uniform scale
        a, b = np.radians(35.0), np.radians(20.0)
        rz = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
        ry = np.array([[np.cos(b), 0.0, np.sin(b)], [0.0, 1.0, 0.0], [-np.sin(b), 0.0, np.cos(b)]])
        return np.hstack([ry @ rz @ np.diag([1.3, 0.4, 0.8]), [[0.3], [1.1], [-0.4]]])
    if kind == "mirrored":  # negative determinant
        return np.hstack([np.diag([-0.7, 1.1, 0.9]) @ np.array([[0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]) @ np.diag([1, 1, -1]),
                          [[-0.2], [0.5], [0.1]]])
    raise ValueError(kind)


def world_to_object(o2w):
    """The 12 floats of the instance's world-to-object rows, as lrk_upload_scene stores them (rows of the inverse, in float)."""
    m = np.vstack([o2w, [0.0, 0.0, 0.0, 1.0]])
    return np.ascontiguousarray(np.linalg.inv(m)[:3].reshape(-1), f32)


class Bottom:
    def __init__(self, lib, tris, side, kind):
        self.lib, self.tris, self.side, self.kind = lib, np.asarray(tris, np.float64), side, kind
        flat = np.ascontiguousarray(self.tris.reshape(-1), np.float64)
        self.h = lib.ltt_build(len(self.tris), flat.ctypes.data, side)
        self.o2w = xform(kind)
        self.w2o = world_to_object(self.o2w)
        self.world = self.tris @ self.o2w[:, :3].T + self.o2w[:, 3]
        self.n = len(self.tris)

    def __del__(self):
        self.lib.ltt_free(self.h)

    def pmf(self, p, prim):
        out = np.zeros(len(p), f32)
        self.lib.ltt_pmf(self.h, len(p), p.ctypes.data, self.w2o.ctypes.data, prim, out.ctypes.data)
        return out

    def sample(self, p, u):
        tri, pmf = np.zeros(len(p), np.uint32), np.zeros(len(p), f32)
        u = np.ascontiguousarray(u, f32)
        self.lib.ltt_sample(self.h, len(p), p.ctypes.data, self.w2o.ctypes.data, u.ctypes.data, tri.ctypes.data, pmf.ctypes.data)
        return tri, pmf

    def dead_mass(self, p):
        out = np.zeros(len(p), np.float64)
        self.lib.ltt_dead_mass(self.h, len(p), p.ctypes.data, self.w2o.ctypes.data, out.ctypes.data)
        return out

    def nodes_and_trails(self):
        nodes = np.zeros(self.lib.ltt_node_count(self.h) * 48, np.uint8)
        trails = np.zeros(self.n, np.uint64)
        self.lib.ltt_copy(self.h, nodes.ctypes.data, trails.ctypes.data)
        return nodes, trails

    def bytes(self):
        nodes, trails = self.nodes_and_trails()
        return nodes.tobytes() + trails.tobytes()

    def points(self, count, seed):
        """World points: half inside the mesh's world bounds, half in a box three times their size around them."""
        rng = np.random.default_rng(seed)
        lo, hi = self.world.reshape(-1, 3).min(0), self.world.reshape(-1, 3).max(0)
        c, e = 0.5 * (lo + hi), 0.5 * (hi - lo) + 1e-3
        inside = rng.uniform(lo, hi, (count // 2, 3))
        outside = rng.uniform(c - 3 * e, c + 3 * e, (count - count // 2, 3))
        return np.ascontiguousarray(np.concatenate([inside, outside]), f32)

    def facing(self, p, margin=1e-3):
        """[points, triangles]: the world point lies in front of the triangle's emitting side by more than `margin` (relative to the
        mesh's size), judged at the triangle's three vertices and centroid; always for two-sided, never for a degenerate triangle.
        World-space normals are cross(p1 - p0, p2 - p0) of the world vertices, as the shade kernels take them."""
        w = self.world
        n = np.cross(w[:, 1] - w[:, 0], w[:, 2] - w[:, 0])
        nl = np.linalg.norm(n, axis=1)
        ok = nl > 1e-12 * max(1.0, float(np.abs(w).max())) ** 2
        if self.side == TWO_SIDED:
            return np.repeat(ok[None], len(p), axis=0)
        n = n / np.where(ok, nl, 1.0)[:, None]
        size = float(np.ptp(w.reshape(-1, 3), axis=0).max())
        pts = np.concatenate([w, w.mean(axis=1, keepdims=True)], axis=1)  # [tri, 4, 3]
        d = np.einsum("tc,ptkc->ptk", n, p.astype(np.float64)[:, None, None, :] - pts[None])
        return (d > margin * size).any(axis=2) & ok[None]


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
    return np.stack([b.pmf(p, k) for k in range(b.n)], axis=1).astype(np.float64)  # [points, triangles]


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
# SHA-256 of the nodes and trails of test_light_tree_cpu.LightSet(n, seed=n), taken at the commit before the triangle-level trees
PARENT_TOP_TREE_SHA256 = {
    1: "c1db4f2f46bd727f2872d1741e2a1e4f841f00e4754ccdce09be1869d1e88339",
    2: "eee2820fb4a1e8201741ebf6f54c7c49ce97a8393cdb54c2757a769564c343ce",
    7: "64bb2ff2736decbb0eabdfd262428b35ae66060e862c6ab7cc36f8afa64965c3",
    1000: "bab0993e8ac8bfca45cede6c7b438a1d8d7dd6eb63136a153a146e65cc5b7d62",
}


@pytest.mark.parametrize("n", sorted(PARENT_TOP_TREE_SHA256))
def test_instance_level_trees_keep_their_bytes(lib, n):
    assert hashlib.sha256(LightSet(n, seed=n).build(lib).bytes()).hexdigest() == PARENT_TOP_TREE_SHA256[n]


# ---- 6. the option's surface ----------------------------------------------------------------------------------------------------
def test_python_option_rejects_bad_values():
    from luisarender_b200.api import Renderer

    check_python_option_rejects_bad_values("light_tree_triangles", light_tree=True)
    with pytest.raises(ValueError, match="light_tree=True"):
        Renderer(light_tree_triangles=True)


def test_cli_lists_and_parses_light_tree_triangles(tmp_path):
    check_cli_lists_and_parses_flag("--light-tree-triangles", tmp_path)


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
