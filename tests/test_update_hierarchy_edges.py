"""Scene updates on the edge-case catalogue on the GPU (DESIGN.md §4): a context taken through each chain of
hierarchy_edge_cases.TRANSITIONS by lrk_update_instances, lrk_update_meshes or lrk_replace_meshes traces every frame's edge ray set
as the oracle's loop over every triangle of that frame does, closest and any hit, bit for bit except on the rays exempt as in
test_hierarchy_edges.py - with the host-built and the device-built hierarchy, in both arithmetic modes.  Back at its first frame
the context traces what it traced before the chain (bit for bit but on the exempt rays), and after the first step it renders the film, with the kernel launch
count, of a fresh upload of that frame.  Warp scheduling and queue lengths are test_hierarchy_edges.py's."""
from __future__ import annotations

import numpy as np
import pytest

import hierarchy_edge_cases as H
import scene_update_checks as U
from scene_update_checks import make  # noqa: F401  (fresh contexts in gpu_renderer's arithmetic mode)

STEP = {"update": U.update_to, "deform": U.deform_to, "replace": U.replace_to}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(H.TRANSITIONS))
def test_updated_context_traces_like_brute_force(name, make):
    step, frames = H.TRANSITIONS[name]
    cases = [H.chain_case(name, k) for k in range(len(frames))]
    for k, c in enumerate(cases):
        H.assert_few_exempt(c, f"{name}, frame {k}")
    for device_bvh in (0, 1):
        r = make(device_bvh=device_bvh)
        r.upload(cases[0].desc)
        r.render(0, 4)
        first, first_occ = r.trace(cases[0].rays), r.trace(cases[0].rays, any_hit=True)
        H.assert_equal_hits(first, cases[0].brute, cases[0].loose, f"{name}, {'device' if device_bvh else 'host'} hierarchy, upload")
        for k in range(1, len(frames)):
            what = f"{name}, {'device' if device_bvh else 'host'} hierarchy, frame {k}"
            STEP[step](r, cases[k - 1].desc, cases[k].desc)
            c = cases[k]
            got = r.trace(c.rays)  # raises on a traversal stack overflow
            H.assert_equal_hits(got, c.brute, c.loose, what)
            occ = r.trace(c.rays, any_hit=True)
            bad = np.flatnonzero((occ["inst"] != c.occ_brute["inst"]) & ~c.loose)
            assert not len(bad), f"{what}: any hit differs from the brute force on rays {bad[:5].tolist()}"
            if k == 1:
                U.check_against_fresh(make, r, c.scene, 4, {"device_bvh": device_bvh}, trace=False)
        # back at the first frame: what the context traced before the chain, bit for bit except on the exempt rays (whose hits
        # depend on the boxes, and a refit, moved or rebuilt hierarchy has other boxes than the upload's)
        keep = ~cases[0].loose
        assert not (H.differ(got, first) & keep).any() and np.array_equal(occ["inst"][keep], first_occ["inst"][keep]), \
            f"{name}: the chain's end"
