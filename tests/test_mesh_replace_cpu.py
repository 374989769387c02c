"""Mesh replacement without a GPU: consecutive frames of the replacement chains differ only where lrk_replace_meshes' definition
says, the node move of bvh_refit.h (relayout_node_refs) turns the first frame's hierarchies of the unchanged meshes into ones that,
with the next frame's own hierarchies spliced in for the replaced meshes, the oracle traces exactly as the next frame, and
Renderer.replace_meshes refuses malformed arrays before the library is reached."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import scene_update_checks as U
import scene_update_frames as S
from luisarender_b200 import _ffi as F
from oracle import binding as O
from scene_update_checks import refit_host  # noqa: F401  (the host-compiled bvh_refit.h)

ALL_FRAMES = {**S.REPLACE_FRAMES, **S.REPLACE_EMISSIVE_FRAMES}


def _pairs(name):
    frames = [S.scene(t) for t in ALL_FRAMES[name]()]
    return [(a, b) for a, b in zip(frames, frames[1:])]


def _slices(d):
    """Per mesh its vertex, triangle, alias, pdf and tri_verts records as bytes."""
    arrays = (S.vertices(d), S.triangles(d), S.array(d.alias, d.triangle_count, F.AliasEntry, np.uint32),
              S.array(d.pdf, d.triangle_count, C.c_float, np.uint32, 1), S.array(d.tri_verts, d.tri_slot_count, C.c_float * 12, np.uint32))
    out = []
    for vo, vc, to, tc, _root, so, *_ in S.meshes(d):
        v, t, alias, pdf, tv = arrays
        out.append((v[vo:vo + vc].tobytes(), t[to:to + tc].tobytes(), alias[to:to + tc].tobytes(), pdf[to:to + tc].tobytes(), tv[so:so + tc].tobytes()))
    return out


@pytest.mark.parametrize("name", list(ALL_FRAMES))
def test_frames_differ_only_in_the_replaced_meshes(name):
    for fa, fb in _pairs(name):
        a, b = fa.desc(), fb.desc()
        ids, verts, tris = S.replaced_meshes(a, b)
        assert ids
        for ptr, count, cls in (("surfaces", "surface_count", F.Surface), ("lights", "light_count", F.Light), ("light_handles", "light_count", F.LightHandle)):
            assert getattr(b, count) == getattr(a, count)
            assert S.array(getattr(b, ptr), getattr(b, count), cls, np.uint8).tobytes() == S.array(getattr(a, ptr), getattr(a, count), cls, np.uint8).tobytes()
        assert bytes(b.camera) == bytes(a.camera) and b.instance_count == a.instance_count and b.mesh_count == a.mesh_count
        ma, mb = S.meshes(a), S.meshes(b)
        # the layout: prefix sums over the new counts, in mesh order
        for col, count in ((0, 1), (2, 3), (5, 3)):
            assert np.array_equal(mb[:, col], np.concatenate([[0], np.cumsum(mb[:-1, count])]))
        for k in range(b.mesh_count):
            if k in ids:
                j = ids.index(k)
                assert (mb[k, 1], mb[k, 3]) == (len(verts[j]), len(tris[j]))
            else:
                assert (mb[k, 1], mb[k, 3]) == (ma[k, 1], ma[k, 3])
        sa, sb = _slices(a), _slices(b)
        emissive = {b.instances[i].mesh for i in range(b.instance_count) if b.instances[i].handle[0] & F.SHAPE_HAS_LIGHT}
        for k in range(b.mesh_count):
            if k not in ids:
                assert sb[k] == sa[k]  # an unchanged mesh's records move as they are
        assert set(ids) & emissive or name not in S.REPLACE_EMISSIVE_FRAMES
        # the instances: only handle[2] of the replaced meshes' instances, their new triangle count
        for i in range(b.instance_count):
            x, y = F.Instance.from_buffer_copy(bytes(a.instances[i])), b.instances[i]
            assert y.handle[2] == mb[y.mesh, 3]
            assert (y.handle[2] != x.handle[2]) == (y.mesh in ids and ma[y.mesh, 3] != mb[y.mesh, 3])
            x.handle[2] = y.handle[2]
            assert bytes(x) == bytes(y)


def test_relayout_rules(refit_host):
    leaf = lambda count, slot: 0x80000000 | ((count - 1) << 28) | slot
    node = np.zeros((3, 16), np.uint32)
    node[:, :12] = np.arange(36).reshape(3, 12)
    node[:, 12:15] = [[5, leaf(3, 40), 0xFFFFFFFF], [0xFFFFFFFF, leaf(4, 0x0FFFFFF0), 9], [leaf(1, 7), 12, 2]]
    node[:, 15] = 77
    for nd, sd in ((7, 3), (-4, -7), (0, 0x10)):
        out = U.move_nodes(refit_host, node, nd, sd)
        assert np.array_equal(out[:, :12], node[:, :12]) and np.array_equal(out[:, 15], node[:, 15])  # boxes stay
        for got, ref in zip(out[:, 12:14].reshape(-1), node[:, 12:14].reshape(-1)):
            if ref == 0xFFFFFFFF:
                assert got == ref  # an unused child stays
            elif ref & 0x80000000:  # a leaf: its count bits stay, its slot moves
                assert got >> 28 == ref >> 28 and got & 0x0FFFFFFF == (int(ref & 0x0FFFFFFF) + sd) % 2**28
            else:
                assert got == (int(ref) + nd) % 2**32
        parents = node[:, 14].astype(np.int64)
        assert np.array_equal(out[:, 14], np.where(parents == 0xFFFFFFFF, parents, (parents + nd) % 2**32))  # a root's parent stays


@pytest.mark.parametrize("name", list(ALL_FRAMES))
def test_relaid_hierarchies_trace_like_the_replaced_frame(name, refit_host):
    for fa, fb in _pairs(name):
        a, b = fa.desc(), fb.desc()
        h, keep, ranges, ids = U.relaid_frame(a, b, refit_host)
        rays = U.random_rays(fb, 100_000, seed=5)
        for any_hit in (False, True):
            want, _ = O.trace(b, rays, any_hit=any_hit)
            got, _ = O.trace(h, rays, any_hit=any_hit)
            assert np.array_equal(got["inst"], want["inst"])
            if not any_hit:
                assert np.array_equal(got["prim"], want["prim"]) and np.array_equal(got["bary"].view(np.uint32), want["bary"].view(np.uint32))
                assert (want["inst"] != 0xFFFFFFFF).mean() > 0.05
        del keep


def _read_call(ctx, ids, count, vertex_counts, vertices, triangle_counts, triangles):
    """What reached lrk_replace_meshes, read while the call's arrays are alive."""
    u32 = lambda ptr, n: list((C.c_uint32 * n).from_address(ptr))
    vc, tc = u32(vertex_counts, count), u32(triangle_counts, count)
    return u32(ids, count), vc, tc, list((C.c_float * (8 * sum(vc))).from_address(vertices)), u32(triangles, 3 * sum(tc))


def test_replace_meshes_argument_shapes():
    r, calls = U.recording_renderer("lrk_replace_meshes", _read_call)
    v, t = np.zeros((4, 8), np.float32), np.array([[0, 1, 2], [0, 2, 3]])
    refusals = [(lambda: r.replace_meshes([0, 1], [v], [t]), "vertices must have one array per id"),
                (lambda: r.replace_meshes([0], [v], [t, t]), "triangles must have one array per id"),
                (lambda: r.replace_meshes([0], [np.zeros((4, 7), np.float32)], [t]), r"\[vertex_count, 8\] float32"),
                (lambda: r.replace_meshes([0], [v.astype(np.float64)], [t]), r"\[vertex_count, 8\] float32"),
                (lambda: r.replace_meshes([0], [v], [t.astype(np.float32)]), r"\[triangle_count, 3\] integers"),
                (lambda: r.replace_meshes([0], [v], [t.reshape(-1)]), r"\[triangle_count, 3\] integers"),
                (lambda: r.replace_meshes([0], [v], [np.zeros((2, 4), np.int32)]), r"\[triangle_count, 3\] integers"),
                (lambda: r.replace_meshes([0], [v], [-t]), r"outside \[0, 2\^32\)")]
    for call, what in refusals:
        with pytest.raises(ValueError, match=what):
            call()
    assert calls == []  # refused before the library is reached
    records = (F.Vertex * 3)()
    records[1].p[0] = 2.5
    r.replace_meshes(np.array([3, 1]), [v, np.ctypeslib.as_array(records)], [t.astype(np.int64), np.array([[0, 1, 2]], np.uint16)])
    (ids, vc, tc, verts, tris), = calls
    assert ids == [3, 1] and vc == [4, 3] and tc == [2, 1]
    assert tris == [0, 1, 2, 0, 2, 3, 0, 1, 2]
    assert verts[8 * 5] == 2.5 and sum(verts) == 2.5
