"""Scene updates on the edge-case catalogue without a GPU (DESIGN.md §4): the hierarchies that lrk_update_meshes and
lrk_replace_meshes leave, rebuilt on the host with the library's own arithmetic (bvh_refit.h through tests/host_device), find what
a loop over every triangle of the frame they reach finds, on that frame's whole edge ray set (hierarchy_edge_cases.make_rays),
closest and any hit, bit for bit except on the rays exempt as in test_hierarchy_edges.py.  A deformed mesh keeps the topology
built for its old vertices with refit boxes; a replaced mesh gets the next frame's own host-built hierarchy (the device LBVH
does not compile for the host) and the unchanged meshes' hierarchies move (relayout_node_refs)."""
from __future__ import annotations

import numpy as np
import pytest

import hierarchy_edge_cases as H
import scene_update_checks as U
import scene_update_frames as S
from oracle import binding as O
from scene_update_checks import refit_host  # noqa: F401  (the host-compiled bvh_refit.h)

STEPS = {step: [n for n, (s, _) in H.TRANSITIONS.items() if s == step] for step in ("update", "deform", "replace")}


def check_against_brute_force(h, c, what):
    """The oracle's walk of the description h traces c's rays (closest and any hit) as the brute force over c's frame."""
    got, _ = O.trace(h, c.rays)
    H.assert_equal_hits(got, c.brute, c.loose, what)
    occ, _ = O.trace(h, c.rays, any_hit=True)
    bad = np.flatnonzero((occ["inst"] != c.occ_brute["inst"]) & ~c.loose)
    assert not len(bad), f"{what}: any hit differs from the brute force on rays {bad[:5].tolist()}"


@pytest.mark.parametrize("name", list(H.TRANSITIONS))
def test_chain_frames_aim_at_their_own_geometry(name):
    """Every frame of a chain (the first, which the chain returns to, included): its rays hit its own instances, not the chain's
    lamp, and few of them are exempt."""
    for k in (0, 1):
        c = H.chain_case(name, k)
        hit = c.brute["inst"] != H.MISS
        lamp = c.brute["inst"] == c.desc.instance_count - 1
        assert (hit & ~lamp).mean() > H.SPARSE_FRAMES.get((name, k), 0.2), f"frame {k}: {hit.mean():.2%} of the rays hit"
        assert lamp.mean() < 0.02, f"frame {k}: {lamp.mean():.2%} of the rays hit the lamp"
        H.assert_few_exempt(c, f"{name}, frame {k}")


@pytest.mark.parametrize("name", list(H.TRANSITIONS))
def test_transition_changes_only_what_its_step_changes(name):
    step, frames = H.TRANSITIONS[name]
    assert frames[0] is frames[-1] and len(frames) == 3  # every chain returns to its first frame
    a, b = H.chain_case(name, 0).desc, H.chain_case(name, 1).desc
    assert bytes(a.camera) == bytes(b.camera)  # the lamp and the camera are the chain's
    same_rows = np.array_equal(S.rows(a).view(np.uint32), S.rows(b).view(np.uint32))
    same_vertices = np.array_equal(S.vertices(a).view(np.uint32), S.vertices(b).view(np.uint32))
    same_triangles = np.array_equal(S.triangles(a), S.triangles(b))
    if step == "update":
        assert not same_rows and same_vertices and same_triangles
    elif step == "deform":
        assert same_rows and not same_vertices and same_triangles and S.deformed_meshes(a, b)[0]
    else:
        assert same_rows and len(S.replaced_meshes(a, b)[0]) == 1


@pytest.mark.parametrize("name", STEPS["update"])
def test_moved_frame_upload_traces_like_brute_force(name):
    """The frame an instance move reaches, uploaded: the host-built instance level over its moved instances."""
    c = H.chain_case(name, 1)
    check_against_brute_force(c.desc, c, f"{name}: upload of the moved frame")


@pytest.mark.parametrize("name", STEPS["deform"])
def test_refit_hierarchy_traces_like_brute_force(name, refit_host):
    a, b = H.chain_case(name, 0), H.chain_case(name, 1)
    h, keep, pads, *_ = U.refit_frame(a.desc, b.desc, refit_host)
    assert pads  # a mesh was refit
    check_against_brute_force(h, b, f"{name}: refit hierarchy")
    check_against_brute_force(b.desc, b, f"{name}: upload of the deformed frame")
    del keep


@pytest.mark.parametrize("name", STEPS["replace"])
def test_relaid_hierarchy_traces_like_brute_force(name, refit_host):
    """Both steps of the chain: the unchanged meshes' hierarchies move one way, then back."""
    for k in (1, 2):
        a, b = H.chain_case(name, k - 1), H.chain_case(name, k)
        h, keep, _, ids = U.relaid_frame(a.desc, b.desc, refit_host)
        assert len(ids) == 1
        check_against_brute_force(h, b, f"{name}: relaid hierarchy of step {k}")
        del keep
