"""Mesh replacement against re-uploads in a frame loop of a mesh whose topology changes, and refit against rebuild, on cuda:0.
Prints one JSON line.

    python tools/bench_mesh_replace.py [--frames 8] [--segments 800:980] [--refit-segments 1000] [--out DIR]

Workload: scenes.wavy_sheet at 1920x1080 with a sheet read through `Mesh { file }` from binary PLY frames written under DIR
(removed afterwards), as tools/bench_mesh_update.py does.
  * topology: the sheet's segment count changes every frame, linearly over --segments (800:980: 1.28 M to 1.92 M triangles).
    Two contexts, two arms per frame: re-upload (Scene.from_source: PLY parse + flatten with the host SAH builds, then
    lrk_upload_scene) and replace (lrk_replace_meshes of the sheet's mesh with the same frame's vertices and triangles).
  * refit_vs_rebuild: the amplitude-0.3 sheet of --refit-segments x --refit-segments quads over K frames of the travelling wave,
    uploaded once.  Two contexts: refit (lrk_update_meshes: the first frame's hierarchy refit to every frame) and rebuild
    (lrk_replace_meshes with the frame's own triangles: a fresh device LBVH every frame).
Host milliseconds per call are wall-clock around calls that synchronise before they return; render_ms is lrk_stats::render_ms
(CUDA events inside the library) at 1 and 16 spp; medians over the frames.  pixels_differing_* counts the pixels whose raw films
differ between the two arms over all frames: zero, except for hits the triangle test places outside their triangle's padded box,
the one hierarchy dependence of the traversal (DESIGN.md §4 (Mesh deformation)).  The card's name and power limit are read in the
same run, since the times depend on them.
"""
from __future__ import annotations

import argparse
import json
import shutil
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

from bench_mesh_update import frame_text, write_ply  # noqa: E402
from bench_scene_update import gpu_card  # noqa: E402


def _mesh_arrays(d, mesh):
    """The vertex [n, 8] float32 and local triangle [m, 3] uint32 records of `mesh` in the description d."""
    m = d.meshes[mesh]
    v = np.ctypeslib.as_array(d.vertices, (d.vertex_count,))
    t = np.ctypeslib.as_array(d.triangles, (d.triangle_count,))
    verts = np.frombuffer(v[m.vertex_offset:m.vertex_offset + m.vertex_count].tobytes(), np.float32).reshape(-1, 8).copy()
    tris = np.frombuffer(t[m.triangle_offset:m.triangle_offset + m.triangle_count].tobytes(), np.uint32).reshape(-1, 3).copy()
    return verts, tris


def _render_both(arms, spps, rows, differ):
    for spp in spps:
        films = []
        for arm, r in arms:
            r.clear()
            r.render(0, spp)
            rows[f"render_{arm}_{spp}spp_ms"].append(r.stats()["render_ms"])
            films.append(r.film(raw=True).copy())
        differ[spp] += int((films[0].view(np.uint32) != films[1].view(np.uint32)).any(axis=-1).sum())


def _summary(rows, differ, **head):
    res = dict(head)
    res.update({k: round(float(np.median(v)), 3) for k, v in rows.items()})
    res.update({f"pixels_differing_{spp}spp": n for spp, n in differ.items()})
    return res


def topology(out: Path, frames: int, seg_range, spps) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer, Scene

    segments = [int(round(seg_range[0] + (seg_range[1] - seg_range[0]) * k / max(frames - 1, 1))) for k in range(frames)]
    for k, s in enumerate(segments):
        write_ply(out / f"topology_{k}.ply", *scenes.wavy_sheet_grid((s, s), 0.08, 0.1 * k))
    fresh, rep = Renderer(device_index=0), Renderer(device_index=0)
    rows = {"parse_flatten_ms": [], "upload_ms": [], "replace_ms": []}
    for spp in spps:
        rows[f"render_reupload_{spp}spp_ms"], rows[f"render_replace_{spp}spp_ms"] = [], []
    differ = {spp: 0 for spp in spps}
    for k in range(frames):
        t0 = time.perf_counter()
        s = Scene.from_source(frame_text(f"topology_{k}.ply", False), out)
        d = s.desc()
        t1 = time.perf_counter()
        fresh.upload(d)
        t2 = time.perf_counter()
        mesh = d.instances[d.instance_count - 1].mesh  # the sheet: the mesh of the sheet's instances
        if k == 0:
            rep.upload(d)
        else:
            verts, tris = _mesh_arrays(d, mesh)
            t3 = time.perf_counter()
            rep.replace_meshes([mesh], [verts], [tris])
            rows["replace_ms"].append((time.perf_counter() - t3) * 1e3)
        rows["parse_flatten_ms"].append((t1 - t0) * 1e3)
        rows["upload_ms"].append((t2 - t1) * 1e3)
        _render_both((("reupload", fresh), ("replace", rep)), spps, rows, differ)
        print(f"[topology] frame {k}: {2 * segments[k] ** 2} triangles, parse + flatten {rows['parse_flatten_ms'][-1]:.0f} ms, "
              f"upload {rows['upload_ms'][-1]:.1f} ms" + (f", replace {rows['replace_ms'][-1]:.1f} ms" if k else ""), file=sys.stderr, flush=True)
    fresh.close()
    rep.close()
    return _summary(rows, differ, case="topology", frames=frames, triangles=[2 * s * s for s in segments])


def refit_vs_rebuild(out: Path, frames: int, segments: int, spps) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer, Scene

    amplitude = 0.3
    write_ply(out / "refit_0.ply", *scenes.wavy_sheet_grid((segments, segments), amplitude, 0.0))
    first = Scene.from_source(frame_text("refit_0.ply", False), out)
    d = first.desc()
    mesh = d.instances[d.instance_count - 1].mesh
    verts, tris = _mesh_arrays(d, mesh)
    # the mesh loader renumbers the PLY's vertices in first-use order and keeps the triangle order: per loaded vertex its PLY index
    source = np.empty(len(verts), np.int64)
    source[tris.reshape(-1)] = scenes.wavy_sheet_grid((segments, segments), amplitude, 0.0)[3].reshape(-1)
    refit, rebuild = Renderer(device_index=0), Renderer(device_index=0)
    refit.upload(d)
    rebuild.upload(d)
    rows = {"update_meshes_ms": [], "replace_meshes_ms": []}
    for spp in spps:
        rows[f"render_refit_{spp}spp_ms"], rows[f"render_rebuild_{spp}spp_ms"] = [], []
    differ = {spp: 0 for spp in spps}
    for k in range(1, frames + 1):
        p, n, _, _ = scenes.wavy_sheet_grid((segments, segments), amplitude, 0.8 * k / frames)
        v = verts.copy()  # the uvs stay
        n = n[source].astype(np.float32)
        v[:, :3], v[:, 3:6] = p[source], n / np.linalg.norm(n, axis=1, keepdims=True)  # unit normals, as the mesh loader makes them
        t0 = time.perf_counter()
        refit.update_meshes([mesh], [v])
        t1 = time.perf_counter()
        rebuild.replace_meshes([mesh], [v], [tris])
        t2 = time.perf_counter()
        rows["update_meshes_ms"].append((t1 - t0) * 1e3)
        rows["replace_meshes_ms"].append((t2 - t1) * 1e3)
        _render_both((("refit", refit), ("rebuild", rebuild)), spps, rows, differ)
        print(f"[refit_vs_rebuild] frame {k}: update {rows['update_meshes_ms'][-1]:.1f} ms, replace {rows['replace_meshes_ms'][-1]:.1f} ms",
              file=sys.stderr, flush=True)
    refit.close()
    rebuild.close()
    return _summary(rows, differ, case="refit_vs_rebuild", frames=frames, amplitude=amplitude, triangles=2 * segments * segments)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--segments", default="800:980", help="first:last segment count of the topology frames")
    ap.add_argument("--refit-segments", type=int, default=1000)
    ap.add_argument("--spp", default="1,16")
    ap.add_argument("--out", help="directory for the PLY frames (default: a temporary directory, removed afterwards)")
    args = ap.parse_args()
    out = Path(args.out) if args.out else Path(tempfile.mkdtemp(prefix="bench_mesh_replace_"))
    out.mkdir(parents=True, exist_ok=True)
    spps = [int(x) for x in args.spp.split(",")]
    seg_range = [int(x) for x in args.segments.split(":")]
    card = gpu_card(0)
    try:
        results = [topology(out, args.frames, seg_range, spps), refit_vs_rebuild(out, args.frames, args.refit_segments, spps)]
    finally:
        for f in out.glob("*.ply"):
            f.unlink()
        if not args.out:
            shutil.rmtree(out, ignore_errors=True)
    print(json.dumps({"bench": "mesh_replace", "gpu": card, "cases": results}), flush=True)


if __name__ == "__main__":
    main()
