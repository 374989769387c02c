"""Mesh updates against re-uploads in a frame loop of a deforming mesh on cuda:0.  Prints one JSON line.

    python tools/bench_mesh_update.py [--frames 8] [--segments 1000] [--amplitudes 0.02,0.3] [--out DIR]

Workload: scenes.wavy_sheet with a sheet of segments x segments quads (1000: 2 M triangles, 1 M vertices), read through
`Mesh { file }` from binary PLY frames written under DIR (removed afterwards), at 1920x1080, over K frames of the travelling wave;
at a small and a large amplitude, and the emissive variant (the sheet is the light: alias tables rebuilt on the host) at the small one.  Two contexts, two
arms per frame:
  * re-upload: Scene.from_source (PLY parse + flatten, host SAH builds) + desc + lrk_upload_scene + lrk_render;
  * update:    lrk_update_meshes of the sheet's mesh with the same frame's vertices + lrk_render.
Host milliseconds per phase are wall-clock around calls that synchronise before they return; render_ms is lrk_stats::render_ms
(CUDA events inside the library) at 1 and 16 spp.  The pixels whose raw films differ between the two arms are counted over all
frames (pixels_differing_*): zero, except for hits the triangle test places outside their triangle's padded box, the one
hierarchy dependence of the traversal (traverse.cuh: safe_rcp; DESIGN.md §4 (Mesh deformation)).  The render times of the two
arms compare the refit of the first frame's hierarchy with a fresh SAH build of each frame.  The card's name and power limit are
read in the same run, since the times depend on them.
"""
from __future__ import annotations

import argparse
import json
import re
import shutil
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

from bench_scene_update import gpu_card  # noqa: E402


def write_ply(path: Path, p, n, uv, tris):
    v = np.concatenate([p, n, uv], axis=1).astype("<f4")
    f = np.empty(len(tris), dtype=[("k", "u1"), ("i", "<i4", (3,))])
    f["k"], f["i"] = 3, tris
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(v)}\nproperty float x\nproperty float y\nproperty float z\n"
              "property float nx\nproperty float ny\nproperty float nz\nproperty float u\nproperty float v\n"
              f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode())
        fh.write(v.tobytes())
        fh.write(f.tobytes())


def frame_text(ply: str, emissive: bool) -> str:
    from luisarender_b200 import scenes

    text = scenes.wavy_sheet(resolution=(1920, 1080), spp=16, segments=(1, 1), emissive=emissive)
    text, count = re.subn(r"Shape sheet_mesh : InlineMesh \{[^\n]*\}", f'Shape sheet_mesh : Mesh {{ file {{ "{ply}" }} }}', text)
    assert count == 1
    return text


def run(out: Path, frames: int, segments: int, amplitude: float, emissive: bool, spps) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer, Scene

    tag = f"a{amplitude}_{'emissive' if emissive else 'matte'}"
    times = [0.8 * k / frames for k in range(frames)]
    for k, t in enumerate(times):
        write_ply(out / f"{tag}_{k}.ply", *scenes.wavy_sheet_grid((segments, segments), amplitude, t))
    fresh, upd = Renderer(device_index=0), Renderer(device_index=0)
    rows = {"parse_flatten_ms": [], "upload_ms": [], "update_ms": []}
    for spp in spps:
        rows[f"render_reupload_{spp}spp_ms"], rows[f"render_update_{spp}spp_ms"] = [], []
    first = Scene.from_source(frame_text(f"{tag}_0.ply", emissive), out)
    upd.upload(first.desc())
    differ = {spp: 0 for spp in spps}
    mesh = None
    for k in range(frames):
        t0 = time.perf_counter()
        s = Scene.from_source(frame_text(f"{tag}_{k}.ply", emissive), out)
        d = s.desc()
        t1 = time.perf_counter()
        fresh.upload(d)
        t2 = time.perf_counter()
        if mesh is None:  # the sheet: the mesh of the sheet's instances
            mesh = d.instances[d.instance_count - 1].mesh
            m = d.meshes[mesh]
        v = np.frombuffer((np.ctypeslib.as_array(d.vertices, (d.vertex_count,))).tobytes(), np.float32).reshape(-1, 8)
        part = np.ascontiguousarray(v[m.vertex_offset:m.vertex_offset + m.vertex_count])
        t3 = time.perf_counter()
        upd.update_meshes([mesh], [part])
        t4 = time.perf_counter()
        rows["parse_flatten_ms"].append((t1 - t0) * 1e3)
        rows["upload_ms"].append((t2 - t1) * 1e3)
        rows["update_ms"].append((t4 - t3) * 1e3)
        for spp in spps:
            films = []
            for arm, r in (("reupload", fresh), ("update", upd)):
                r.clear()
                r.render(0, spp)
                rows[f"render_{arm}_{spp}spp_ms"].append(r.stats()["render_ms"])
                films.append(r.film(raw=True).copy())
            differ[spp] += int((films[0].view(np.uint32) != films[1].view(np.uint32)).any(axis=-1).sum())
        print(f"[{tag}] frame {k}: parse + flatten {rows['parse_flatten_ms'][-1]:.0f} ms, update {rows['update_ms'][-1]:.2f} ms",
              file=sys.stderr, flush=True)
    fresh.close()
    upd.close()
    res = {"amplitude": amplitude, "emissive": emissive, "triangles": int(2 * segments * segments), "frames": frames}
    res.update({k: round(float(np.median(v)), 3) for k, v in rows.items()})
    res.update({f"pixels_differing_{spp}spp": n for spp, n in differ.items()})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--segments", type=int, default=1000)
    ap.add_argument("--spp", default="1,16")
    ap.add_argument("--amplitudes", default="0.02,0.3", help="the Matte sheet's wave heights; the emissive sheet runs at the first")
    ap.add_argument("--out", help="directory for the PLY frames (default: a temporary directory, removed afterwards)")
    args = ap.parse_args()
    out = Path(args.out) if args.out else Path(tempfile.mkdtemp(prefix="bench_mesh_update_"))
    out.mkdir(parents=True, exist_ok=True)
    spps = [int(x) for x in args.spp.split(",")]
    card = gpu_card(0)
    amplitudes = [float(a) for a in args.amplitudes.split(",")]
    cases = [(a, False) for a in amplitudes] + [(amplitudes[0], True)]
    try:
        results = [run(out, args.frames, args.segments, a, e, spps) for a, e in cases]
    finally:
        for f in out.glob("*.ply"):
            f.unlink()
        if not args.out:
            shutil.rmtree(out, ignore_errors=True)
    print(json.dumps({"bench": "mesh_update", "gpu": card, "cases": results}), flush=True)


if __name__ == "__main__":
    main()
