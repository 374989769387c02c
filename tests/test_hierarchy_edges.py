"""Closest hits do not depend on the hierarchy (DESIGN.md §4): boxes contain their triangles, and the triangle test and its tie
rule are shared, so any hierarchy walked in any order returns what a loop over every triangle returns.  This module checks that
claim on scenes built to break it: leaf-sized meshes, exact ties, flat and graded geometry, extreme sizes and offsets, awkward
instance transforms, many and invisible instances - and on rays aimed at vertices and edges from near and from very far.

CPU: the oracle's BVH walk against its brute-force loop (bit for bit), and the brute force against an independent float64
Moeller-Trumbore wherever the float64 answer is unambiguous.  GPU: lrk_trace with the host-built and the device-built (LBVH)
hierarchy against the same brute force, under every warp-scheduling setting and queue length, and the films of both hierarchies.
The only rays exempt from bit-exactness are those whose hit the triangle test itself places outside the triangle's padded box
(outside_own_box) or, along the world ray, outside its instance's box (outside_instance_box): no box test can keep them, and they
are counted and bounded.  The catalogue, the rays and the float64 reference are in hierarchy_edge_cases.py.
"""
from __future__ import annotations

import numpy as np
import pytest

from hierarchy_edge_cases import (CATALOGUE, F64_RAYS, FAR_FACTORS, MISS, SEEDS, Case as _Case, assert_equal_hits as _assert_equal_hits,
                                  differ as _differ, f64_check)
from oracle import binding as O

# ---- fixtures -------------------------------------------------------------------------------------------------------------------

NAMES = list(CATALOGUE)
# the 1000 clusters of far_mesh_instances_1000 are 0.1 wide and 2.4e4 apart: rays jittered by 1e-5 of the scene pass most of them
MIN_HITS = {"far_mesh_instances_1000": 0.002}
_CASES: dict[str, _Case] = {}


def case(name) -> _Case:
    if name not in _CASES:
        _CASES[name] = _Case(*CATALOGUE[name], seed=SEEDS.get(name, NAMES.index(name) + 1))
    return _CASES[name]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_bvh_equals_brute_force(name):
    c = case(name)
    got, cnt = O.trace(c.desc, c.rays)
    _assert_equal_hits(got, c.brute, c.loose, "oracle BVH")
    occ, _ = O.trace(c.desc, c.rays, any_hit=True)
    assert not (occ["inst"] != c.occ_brute["inst"])[~c.loose].any()
    assert np.array_equal(c.occ_brute["inst"] == 1, c.brute["inst"] != MISS)
    assert (c.brute["inst"] != MISS).mean() > MIN_HITS.get(name, 0.2) and cnt["nodes_visited"] > 0
    near = slice(0, len(c.base))
    print(f"{name}: {len(c.rays)} rays, {int(c.loose.sum())} exempt ({int(c.loose[near].sum())} of the {len(c.base)} near ones), "
          f"{int(_differ(got, c.brute).sum())} of those differ")
    # the exemption stays the exception: silhouette and shared-vertex rays from far away, grazing rays through shared vertices
    assert c.loose[near].mean() < 0.02 and c.loose.mean() < 0.08


@pytest.mark.parametrize("name", NAMES)
def test_oracle_bvh_equals_brute_force_from_far_away(name):
    """Origins 3, 30, 100 and 1000 scene sizes away, aimed at vertices and edges: the slab test's rounding grows with the
    distance to the box, not with the box's size, and must not cull a box that holds the nearest hit."""
    c = case(name)
    begin = len(c.base)
    for k, rays in zip(FAR_FACTORS, c.far):
        sl = slice(begin, begin + len(rays))
        begin += len(rays)
        got, _ = O.trace(c.desc, rays)
        assert (c.brute["inst"][sl] != MISS).mean() > MIN_HITS.get(name, 0.2)  # aimed at silhouettes: many pass by
        _assert_equal_hits(got, c.brute[sl], c.loose[sl], f"origins {k}x the scene size away")


@pytest.mark.parametrize("name", list(SEEDS))
def test_seeded_scenes_draw_a_hit_the_instance_level_loses(name):
    """The reproductions of outside_instance_box stay reproductions: their rays include one whose hit the oracle's walk of the
    host-built hierarchy does not return and that only outside_instance_box exempts (its hit is inside its triangle's own box)."""
    c = case(name)
    got, _ = O.trace(c.desc, c.rays)
    lost = _differ(got, c.brute) & c.instance & ~c.own
    assert lost.any() and not (_differ(got, c.brute) & ~c.loose).any()


@pytest.mark.parametrize("name", NAMES)
def test_brute_force_matches_float64_reference(name):
    c = case(name)
    idx = np.linspace(0, len(c.base) - 1, min(F64_RAYS, len(c.base))).astype(int)
    far_idx = len(c.base) + np.arange(0, len(c.rays) - len(c.base), (len(c.rays) - len(c.base)) // 400)
    sel = np.concatenate([idx, far_idx])
    pts = c.tris.reshape(-1, 3)
    kept = f64_check(c.rays[sel], c.tris, c.ids, c.mags, c.brute[sel], float((pts.max(axis=0) - pts.min(axis=0)).max()))
    print(f"{name}: {kept} of {len(sel)} rays have an unambiguous float64 answer")
    # copies of one triangle, and two instances with one transform, tie on every hit: only their misses are unambiguous
    assert kept >= (0.05 if name in ("same_transform_twice", "copies_12") else 0.2) * len(sel), \
        f"only {kept} of {len(sel)} rays were checked against float64"


def test_invisible_instances_are_never_hit():
    c = case("invisible_interleaved")
    hit = c.brute["inst"] != MISS
    lamp = c.desc.instance_count - 1
    visible = {i for i in range(c.desc.instance_count) if c.desc.instances[i].visible}
    assert set(np.unique(c.brute["inst"][hit]).tolist()) <= visible
    assert {i for i in range(lamp) if not c.desc.instances[i].visible} == set(range(0, lamp, 2))
    got, _ = O.trace(c.desc, c.rays)
    assert set(np.unique(got["inst"][got["inst"] != MISS]).tolist()) <= visible


# ---- GPU: both hierarchies, every schedule and queue length, films -------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_traversal_equals_brute_force(name, gpu_renderer):
    c = case(name)
    r = gpu_renderer
    try:
        for device_bvh in (0, 1):
            r.set_option("device_bvh", device_bvh)
            r.upload(c.desc)
            what = "device LBVH" if device_bvh else "host BVH"
            full = r.trace(c.rays)  # every call raises on a traversal stack overflow
            # the exempt rays may go either way here too: the kernels' box test takes 1/d from rcp.approx, the oracle's divides
            _assert_equal_hits(full, c.brute, c.loose, what)
            occ = r.trace(c.rays, any_hit=True)
            assert not (occ["inst"] != c.occ_brute["inst"])[~c.loose].any(), what
            # warp scheduling changes no bit
            for refill in (1, 16, 32):
                for inner in (1, 8, 32):
                    r.set_option("refill_below", refill)
                    r.set_option("inner_min", inner)
                    got = r.trace(c.rays)
                    bad = np.flatnonzero(_differ(got, full))
                    assert not len(bad), f"{what}, refill_below {refill}, inner_min {inner}: rays {bad[:5].tolist()} differ"
                    assert np.array_equal(r.trace(c.base, any_hit=True)["inst"], occ["inst"][:len(c.base)])
            r.set_option("refill_below", 16)
            r.set_option("inner_min", 8)
            # queues shorter than a warp, and ending just past a warp or a block
            for n in (0, 1, 31, 32, 33, 255, 257, 4097):
                assert not _differ(r.trace(c.rays[:n]), full[:n]).any(), f"{what}, {n} rays"
    finally:
        r.set_option("refill_below", 16)
        r.set_option("inner_min", 8)
        r.set_option("device_bvh", 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_films_of_host_and_device_hierarchies_are_identical(name, gpu_renderer):
    c = case(name)
    r = gpu_renderer
    try:
        films = []
        for device_bvh in (0, 1):
            r.set_option("device_bvh", device_bvh)
            r.upload(c.desc)
            r.clear()
            r.render(0, 3)  # raises on a traversal stack overflow
            films.append(r.film(raw=True).copy())
        assert (films[0][..., 3] == 3).all() and (films[0][..., :3].max() > 0 or name in MIN_HITS)  # the sparse scene is black
        assert np.array_equal(films[0], films[1])
    finally:
        r.set_option("device_bvh", 0)
