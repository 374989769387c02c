"""Mesh updates without a GPU: the deformed frames differ from their first frame only where lrk_update_meshes' definition says, the
shared area alias tables (luisarender_b200/csrc/device/alias_table.h) rebuild a deformed frame's tables bit for bit, and the refit
arithmetic (luisarender_b200/csrc/device/bvh_refit.h) turns the first frame's hierarchies into ones that the oracle traces exactly
as the deformed frame's own."""
from __future__ import annotations

import ctypes as C
import hashlib

import numpy as np
import pytest

import scene_update_checks as U
import scene_update_frames as S
from luisarender_b200 import _ffi as F
from luisarender_b200 import scenes
from oracle import binding as O
from scene_update_checks import refit_host  # noqa: F401  (the host-compiled bvh_refit.h)

ALL_FRAMES = {**S.DEFORM_FRAMES, **S.DEFORM_EMISSIVE_FRAMES}


def test_default_globe_text_is_unchanged():
    # sha256 of emissive_globe's text before it had `wobble`: the undeformed globe stays what its tests and benchmarks were made from
    assert hashlib.sha256(scenes.emissive_globe().encode()).hexdigest() == "5fbb0d1a6d8f02a83d5b8ec36a38609622c8b335cb51054608f186c93dc2914d"
    for kind in ("uniform", "stretched", "mirrored"):
        assert scenes.emissive_globe(resolution=(16, 16), subdivision=2, transform=kind) == \
            scenes.emissive_globe(resolution=(16, 16), subdivision=2, transform=kind, wobble=None)


def _emissive_meshes(d):
    return {d.instances[i].mesh for i in range(d.instance_count) if d.instances[i].handle[0] & F.SHAPE_HAS_LIGHT}


@pytest.mark.parametrize("name", list(ALL_FRAMES))
def test_frames_differ_only_in_the_deformed_vertices(name):
    frames = [S.scene(t) for t in ALL_FRAMES[name]()]
    d0 = frames[0].desc()
    m0 = S.meshes(d0)
    for f in frames[1:]:
        d = f.desc()
        for ptr, count, cls in (("triangles", "triangle_count", F.Triangle), ("surfaces", "surface_count", F.Surface),
                                ("lights", "light_count", F.Light), ("light_handles", "light_count", F.LightHandle)):
            assert getattr(d, count) == getattr(d0, count)
            assert S.array(getattr(d, ptr), getattr(d, count), cls, np.uint8).tobytes() == \
                S.array(getattr(d0, ptr), getattr(d0, count), cls, np.uint8).tobytes(), ptr
        assert d.vertex_count == d0.vertex_count and d.tri_slot_count == d0.tri_slot_count
        m = S.meshes(d)
        assert np.array_equal(np.delete(m, 4, axis=1), np.delete(m0, 4, axis=1))  # the layout; the hierarchy's roots may move
        assert bytes(d.camera) == bytes(d0.camera)
        for i in range(d.instance_count):
            a, b = d0.instances[i], d.instances[i]
            assert bytes(a) == bytes(b)
        ids, _ = S.deformed_meshes(d0, d)
        assert ids
        alias0, alias = S.array(d0.alias, d0.triangle_count, F.AliasEntry, np.uint32), S.array(d.alias, d.triangle_count, F.AliasEntry, np.uint32)
        pdf0, pdf = S.array(d0.pdf, d0.triangle_count, C.c_float, np.uint32, 1), S.array(d.pdf, d.triangle_count, C.c_float, np.uint32, 1)
        tv0, tv = S.array(d0.tri_verts, d0.tri_slot_count, C.c_float * 12), S.array(d.tri_verts, d.tri_slot_count, C.c_float * 12)
        for k, row in enumerate(m):
            t0, tn, s0 = row[2], row[3], row[5]
            same_tris = slice(t0, t0 + tn)
            if k not in ids:  # untouched meshes keep everything
                assert np.array_equal(alias[same_tris], alias0[same_tris]) and np.array_equal(pdf[same_tris], pdf0[same_tris])
                assert np.array_equal(tv[s0:s0 + tn].view(np.uint32), tv0[s0:s0 + tn].view(np.uint32))
            else:
                pos = np.delete(tv[s0:s0 + tn], [3, 7, 11], axis=1)
                pos0 = np.delete(tv0[s0:s0 + tn], [3, 7, 11], axis=1)
                assert not np.array_equal(np.sort(pos, axis=0), np.sort(pos0, axis=0))
        if name in S.DEFORM_EMISSIVE_FRAMES:
            assert set(ids) <= _emissive_meshes(d)


@pytest.mark.parametrize("name", list(S.DEFORM_EMISSIVE_FRAMES))
def test_shared_alias_tables_reproduce_the_flattened_ones(name, refit_host):
    for f in [S.scene(t) for t in S.DEFORM_EMISSIVE_FRAMES[name]()]:
        d = f.desc()
        v, tris = S.vertices(d), S.triangles(d)
        alias = S.array(d.alias, d.triangle_count, F.AliasEntry, np.uint32)
        pdf = S.array(d.pdf, d.triangle_count, C.c_float, np.uint32, 1)
        for k in _emissive_meshes(d):
            vo, vc, to, tc = S.meshes(d)[k][:4]
            v_k, t_k = np.ascontiguousarray(v[vo:vo + vc]), np.ascontiguousarray(tris[to:to + tc])
            table, p = np.zeros((tc, 2), np.uint32), np.zeros(tc, np.uint32)
            refit_host.mesh_alias_table(v_k.ctypes.data, t_k.ctypes.data, int(tc), table.ctypes.data, p.ctypes.data)
            assert np.array_equal(table, alias[to:to + tc]) and np.array_equal(p, pdf[to:to + tc, 0])


def _check_refit_boxes(a, blas, tv, ids, pads):
    """Every reachable leaf child's stored box is its slots' triangle box padded by exactly 5e-7 x the deformed mesh's extent."""
    m = S.meshes(a)
    for k in ids:
        so, tc = int(m[k][5]), int(m[k][3])
        pos = tv[so:so + tc].reshape(-1, 3, 4)[:, :, :3]
        lo, hi = pos.reshape(-1, 3).min(axis=0), pos.reshape(-1, 3).max(axis=0)
        extent = np.float32(max(max(abs(float(lo[i])), abs(float(hi[i])), float(np.float32(hi[i] - lo[i]))) for i in range(3)))
        assert pads[k] == np.float32(np.float32(5e-7) * extent)
        pad = np.float32(pads[k])
        stack, seen = [int(m[k][4])], 0
        while stack:
            n = blas[stack.pop()]
            seen += 1
            f = n[:12].view(np.float32)
            for c, ref in enumerate((n[12], n[13])):
                if ref == 0xFFFFFFFF:
                    continue
                if ref & 0x80000000:
                    first, count = int(ref & 0x0FFFFFFF), int((ref >> 28) & 7) + 1
                    p = tv[first:first + count].reshape(-1, 3, 4)[:, :, :3].reshape(-1, 3)
                    assert np.array_equal(f[6 * c:6 * c + 3], (p.min(axis=0) - pad).astype(np.float32))
                    assert np.array_equal(f[6 * c + 3:6 * c + 6], (p.max(axis=0) + pad).astype(np.float32))
                else:
                    stack.append(int(ref))
        assert seen >= 1


@pytest.mark.parametrize("name", list(ALL_FRAMES))
def test_refit_hierarchies_trace_like_the_deformed_frame(name, refit_host):
    frames = [S.scene(t) for t in ALL_FRAMES[name]()]
    a = frames[0].desc()
    for f in frames[1:]:
        b = f.desc()
        h, keep, pads, blas, tv, ids = U.refit_frame(a, b, refit_host)
        _check_refit_boxes(a, blas, tv, ids, pads)
        rays = U.random_rays(f, 100_000, seed=5)
        for any_hit in (False, True):
            want, _ = O.trace(b, rays, any_hit=any_hit)
            got, _ = O.trace(h, rays, any_hit=any_hit)
            assert np.array_equal(got["inst"], want["inst"])
            if not any_hit:
                assert np.array_equal(got["prim"], want["prim"]) and np.array_equal(got["bary"].view(np.uint32), want["bary"].view(np.uint32))
                assert (want["inst"] != 0xFFFFFFFF).mean() > 0.05
        del keep


def test_update_meshes_argument_shapes():
    r, calls = U.recording_renderer("lrk_update_meshes")
    v = np.zeros((4, 8), np.float32)
    with pytest.raises(ValueError, match="one array per id"):
        r.update_meshes([0, 1], [v])
    with pytest.raises(ValueError, match=r"\[vertex_count, 8\] float32"):
        r.update_meshes([0], [np.zeros((4, 7), np.float32)])
    with pytest.raises(ValueError, match=r"\[vertex_count, 8\] float32"):
        r.update_meshes([0], [np.zeros((4, 8), np.float64)])
    assert calls == []  # refused before the library is reached
    records = (F.Vertex * 3)()
    records[1].p[0] = 2.5
    r.update_meshes(np.array([3, 1]), [v, np.ctypeslib.as_array(records)])
    (ctx, ids_ptr, count, verts_ptr, total), = calls
    assert count == 2 and total == 7
