"""What the tests of scene updates share (test_scene_update*.py, test_mesh_update*.py, test_mesh_replace*.py): the steps that take
a context from one frame to the next, the checks that compare an updated context with a fresh upload of the frame, and, for the
CPU tests, the host-compiled hierarchy arithmetic, the splice of a frame's instance level behind other mesh hierarchies and a
stand-in for the device library."""
from __future__ import annotations

import ctypes as C
import types

import numpy as np
import pytest

import scene_update_frames as S
from host_harness import DEVICE, REPO, load
from luisarender_b200 import _ffi as F
from luisarender_b200.api import Renderer
from oracle import binding as O


@pytest.fixture
def make(gpu_renderer):
    """Fresh contexts in gpu_renderer's arithmetic mode, with the given Renderer options (and "device_bvh"), closed afterwards."""
    made = []

    def new(device_bvh=False, gbuffer=False, **options):
        r = Renderer(device_index=0, **options)
        r.set_option("strict_math", 0 if gpu_renderer.fast else 1)
        r.set_option("device_bvh", int(device_bvh))
        r.set_option("gbuffer", int(gbuffer))
        made.append(r)
        return r

    yield new
    for r in made:
        r.close()


def random_rays(scene, n, seed):
    rng = np.random.default_rng(seed)
    info = scene.info()
    lo, hi = np.array(info["world_min"]), np.array(info["world_max"])
    o = rng.uniform(lo - 0.5, hi + 0.5, size=(n, 3))
    d = rng.uniform(lo, hi, size=(n, 3)) - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.zeros((n, 8), np.float32)
    rays[:, :3], rays[:, 4:7], rays[:, 7] = o, d, np.finfo(np.float32).max
    rays[::3, 7] = rng.uniform(0.5, 6.0, size=len(rays[::3]))
    return rays


def update_to(r, a_desc, b_desc):
    """Update the context r (holding a_desc's transforms) to b_desc's: the instances whose rows differ."""
    a, b = S.rows(a_desc), S.rows(b_desc)
    ids = np.flatnonzero((a.view(np.uint32) != b.view(np.uint32)).any(axis=(1, 2)))
    assert len(ids) > 0
    r.update_instances(ids, b[ids])


def deform_to(r, a_desc, b_desc):
    ids, parts = S.deformed_meshes(a_desc, b_desc)
    assert ids
    r.update_meshes(ids, parts)


def replace_to(r, a_desc, b_desc):
    """Replace the meshes that differ between a_desc and b_desc with B's, passing the ids in descending order."""
    ids, verts, tris = S.replaced_meshes(a_desc, b_desc)
    assert ids
    r.replace_meshes(ids[::-1], verts[::-1], tris[::-1])


def fresh(make, scene, spp, options):
    """The raw film and kernel launches of a fresh upload of `scene` rendered at spp."""
    r = make(**options)
    r.upload(scene.desc())
    r.render(0, spp)
    return r.film(raw=True).copy(), r.stats()["kernel_launches"]


def check_against_fresh(make, r, scene, spp, options, trace=True):
    """r renders (and, with trace=True, traces closest hits and occlusion of random rays) what a fresh upload of `scene` does,
    and what the oracle traces on its description."""
    film, launches = fresh(make, scene, spp, options)
    r.render(0, spp)
    assert np.array_equal(r.film(raw=True), film)
    assert r.stats()["kernel_launches"] == launches
    if trace:
        d = scene.desc()
        rays = random_rays(scene, 100_000, seed=3)
        ref, _ = O.trace(d, rays)
        got = r.trace(rays)
        assert np.array_equal(got["inst"], ref["inst"]) and np.array_equal(got["prim"], ref["prim"])
        assert np.array_equal(got["bary"].view(np.uint32), ref["bary"].view(np.uint32))
        assert (ref["inst"] != 0xFFFFFFFF).mean() > 0.05
        occ_ref, _ = O.trace(d, rays, any_hit=True)
        assert np.array_equal(r.trace(rays, any_hit=True)["inst"], occ_ref["inst"])


def check_frames(make, frames, step, spp, options, trace=True):
    """Upload frames[0], then go through frames[1:] by `step` (update_to, deform_to, replace_to), each time against a fresh upload
    of that frame (check_against_fresh)."""
    r = make(**options)
    r.upload(frames[0].desc())
    r.render(0, spp)
    for prev, cur in zip(frames, frames[1:]):
        step(r, prev.desc(), cur.desc())
        check_against_fresh(make, r, cur, spp, options, trace)


def check_gbuffer_adaptive_and_shards(make, a, b, step):
    """A context that uploaded frame a and was taken to frame b by `step` writes b's G-buffer guides, renders adaptively at
    threshold 0 what lrk_render does, and renders b in three balanced shards that add up to b's film."""
    ref = make(gbuffer=True)
    ref.upload(b.desc())
    ref.render(0, 4)
    film, guides = ref.film(raw=True).copy(), ref.gbuffer()
    r = make(gbuffer=True)
    r.upload(a.desc())
    r.render(0, 4)
    step(r, a.desc(), b.desc())
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)
    for got, want in zip(r.gbuffer(), guides):
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    r.set_option("gbuffer", 0)
    r.render_adaptive(0.0, 2, 4)  # threshold 0: every pixel gets max_spp, as lrk_render(0, 4)
    assert np.array_equal(r.film(raw=True), film)
    total = np.zeros_like(film)
    for rank in range(3):
        s = make()
        s.upload(a.desc())
        s.balance_shards(rank, 3, tile_size=16, probe_spp=1)
        step(s, a.desc(), b.desc())
        s.render(0, 4)
        total += s.film(raw=True)
    assert np.array_equal(total, film)


def check_refusals(r, film, refusals):
    """Every (call, pattern) of `refusals` raises an invalid-argument error that matches pattern and leaves r's film (`film`, a
    render at 4 spp) and scene as they were."""
    for call, what in refusals:
        with pytest.raises(RuntimeError, match=rf"\(-1\).*{what}"):
            call()
        assert np.array_equal(r.film(raw=True), film)  # not even cleared
    r.clear()
    r.render(0, 4)
    assert np.array_equal(r.film(raw=True), film)  # the scene is the uploaded one


@pytest.fixture(scope="module")
def refit_host():
    """tests/host_device/bvh_refit_host.cpp: the refit, the node move and the area alias tables of the device library on the host."""
    lib = load("bvh_refit_host", [DEVICE / "bvh_refit.h", DEVICE / "alias_table.h", REPO / "include" / "lrk.h"],
               ["-O2", "-march=x86-64-v3", "-ffp-contract=off"])
    lib.refit_mesh.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_float)]
    lib.mesh_alias_table.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.relayout_nodes.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    return lib


def node_ranges(d):
    """Per mesh its hierarchy's node range (first, end): from its root to the next mesh's root, or to the instance level."""
    roots = S.meshes(d)[:, 4].astype(np.int64)
    return [(int(r), int(roots[roots > r].min()) if (roots > r).any() else int(d.tlas_root)) for r in roots]


def with_hierarchies(b, blas, mesh_table):
    """Frame b's description with the mesh hierarchies `blas` (nodes [n, 16] uint32) and the mesh table `mesh_table` in place of
    its own, and b's instance level moved behind them.  Returns the description and the arrays it points into."""
    tlas = S.array(b.bvh_nodes, b.bvh_node_count, F.BvhNode, np.uint32, 16)[b.tlas_root:].copy()
    for col in (12, 13, 14):  # inner references and parents move with the level
        inner = (tlas[:, col] & np.uint32(0x80000000)) == 0
        tlas[inner, col] = (tlas[inner, col].astype(np.int64) + (len(blas) - int(b.tlas_root))).astype(np.uint32)
    nodes = np.ascontiguousarray(np.concatenate([blas, tlas]))
    h = F.SceneDesc()
    C.memmove(C.byref(h), C.byref(b), C.sizeof(F.SceneDesc))
    keep = [nodes, np.ascontiguousarray(mesh_table)]
    h.bvh_nodes = nodes.ctypes.data_as(C.POINTER(F.BvhNode))
    h.bvh_node_count = len(nodes)
    h.tlas_root = len(blas)
    h.meshes = keep[1].ctypes.data_as(C.POINTER(F.Mesh))
    return h, keep


def refit_frame(a, b, lib):
    """A description that renders frame b with frame a's mesh hierarchies refit to b's vertices (what lrk_update_meshes leaves on
    the device): a's refit BLAS nodes and mesh table, a's slot order with b's positions, b's vertices and instances, and b's
    instance level appended behind a's meshes.  Returns the description, the arrays it points into and the refit meshes' pads."""
    nodes_a = S.array(a.bvh_nodes, a.bvh_node_count, F.BvhNode, np.uint32, 16)
    blas = np.ascontiguousarray(nodes_a[:a.tlas_root])
    # a's slot order, b's positions: every slot's primitive re-read through b's triangles and vertices
    tv = S.array(a.tri_verts, a.tri_slot_count, C.c_float * 12).copy()
    vb, tris = S.vertices(b), S.triangles(b)
    m = S.meshes(a)
    for vo, vc, to, tc, _root, so, *_ in m:
        prim = tv[so:so + tc, 3].view(np.uint32)
        t = tris[to + prim]
        for c in range(3):
            tv[so:so + tc, 4 * c:4 * c + 3] = vb[vo + t[:, c], :3]
    ids, _ = S.deformed_meshes(a, b)
    pads = {}
    for k in ids:
        root, end = node_ranges(a)[k]
        pad = C.c_float()
        assert lib.refit_mesh(blas.ctypes.data, root, end, tv.ctypes.data, int(m[k][5]), int(m[k][3]), C.byref(pad)) == 0
        pads[k] = pad.value
    h, keep = with_hierarchies(b, blas, m)
    h.tri_verts = tv.ctypes.data_as(C.POINTER(C.c_float))
    return h, keep + [tv], pads, blas, tv, ids


def move_nodes(lib, nodes, node_delta, slot_delta):
    out = np.zeros_like(nodes)
    lib.relayout_nodes(nodes.ctypes.data, out.ctypes.data, len(nodes), node_delta % 2**32, slot_delta % 2**32)
    return out


def relaid_frame(a, b, lib):
    """The hierarchy lrk_replace_meshes leaves for frame a replaced by frame b's meshes, built on the host: in mesh order, every
    unchanged mesh's node range of a moved to its new place, every replaced mesh's range of max(n - 1, 1) nodes starting with b's
    own hierarchy of it (moved), and b's instance level behind them.  Returns the description (b's with these nodes and roots),
    the arrays it points into, and the new ranges."""
    ids, _, _ = S.replaced_meshes(a, b)
    nodes_a = S.array(a.bvh_nodes, a.bvh_node_count, F.BvhNode, np.uint32, 16)
    nodes_b = S.array(b.bvh_nodes, b.bvh_node_count, F.BvhNode, np.uint32, 16)
    ma, mb = S.meshes(a), S.meshes(b).copy()
    ra, rb = node_ranges(a), node_ranges(b)
    parts, ranges, base = [], [], 0
    for k in range(b.mesh_count):
        if k in ids:
            first, end = rb[k]
            size = max(int(mb[k, 3]) - 1, 1)
            assert end - first <= size  # the host's hierarchy never has more nodes than the device builder's
            part = np.zeros((size, 16), np.uint32)
            part[:end - first] = move_nodes(lib, nodes_b[first:end], base - first, 0)
        else:
            first, end = ra[k]
            part = move_nodes(lib, nodes_a[first:end], base - first, int(mb[k, 5]) - int(ma[k, 5]))
            # the same mesh's hierarchy in b (the host build is deterministic), moved from b's place to the new one
            assert np.array_equal(part, move_nodes(lib, nodes_b[rb[k][0]:rb[k][1]], base - rb[k][0], 0))
        mb[k, 4] = base
        ranges.append((base, base + len(part)))
        parts.append(part)
        base += len(part)
    h, keep = with_hierarchies(b, np.concatenate(parts), mb)
    return h, keep, ranges, ids


def recording_renderer(call, record=lambda *args: args):
    """A Renderer over a stand-in for the device library whose function `call` appends record(*its arguments) to the returned
    list and succeeds; record runs while the call's arrays are alive."""
    calls = []
    r = Renderer.__new__(Renderer)
    r._lib, r._ctx = types.SimpleNamespace(**{call: lambda *args: calls.append(record(*args)) or 0}), None
    r._check = lambda rc, what: None
    return r, calls
