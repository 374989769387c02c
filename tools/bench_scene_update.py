"""Scene updates against re-uploads in frame loops on cuda:0.  Prints one JSON line per case.

    python tools/bench_scene_update.py [--case instances|deform|replace] [--frames 8] [--spp 1,16]
        [--deform-segments 1000] [--amplitudes 0.02,0.3] [--replace-segments 800:980] [--refit-segments 1000] [--out DIR]

Every case runs two contexts side by side, one that re-uploads every frame and one that updates; without --case all three run,
in this order:
  * instances (lrk_update_instances): config C3 (1920x1080, 1.39M instanced triangles) with its 64 spheres moving
    (scenes.instanced_spheres(time=k / 8)), K frames at each spp.  Two arms per frame:
      re-upload: Scene.from_source (parse + flatten, host BLAS and TLAS builds) + desc + lrk_upload_scene + lrk_render;
      update:    lrk_update_instances of every moved instance (rows taken from the same frame's description) + lrk_render.
    Each frame's two raw films must be bit-identical.  The render times of the two arms compare the device-built instance level
    of the update (LBVH) with the host's SAH instance level.  Scaling: the update of 10^3 and 10^4 small spheres, all moved, and
    the update of none of them (the instance-level rebuild and the film clear alone).
  * deform (lrk_update_meshes): scenes.wavy_sheet with a sheet of --deform-segments squared quads (1000: 2 M triangles, 1 M
    vertices) at 1920x1080, over K frames of the travelling wave; at a small and a large amplitude, and the emissive variant (the
    sheet is the light: alias tables rebuilt on the host) at the small one.  Two arms per frame:
      re-upload: Scene.from_source (PLY parse + flatten, host SAH builds) + desc + lrk_upload_scene + lrk_render;
      update:    lrk_update_meshes of the sheet's mesh with the same frame's vertices + lrk_render.
    The render times of the two arms compare the refit of the first frame's hierarchy with a fresh SAH build of each frame.
  * replace (lrk_replace_meshes):
      topology: the sheet's segment count changes every frame, linearly over --replace-segments (800:980: 1.28 M to 1.92 M
        triangles).  Two arms per frame: re-upload (Scene.from_source: PLY parse + flatten with the host SAH builds, then
        lrk_upload_scene) and replace (lrk_replace_meshes of the sheet's mesh with the same frame's vertices and triangles).
      refit_vs_rebuild: the amplitude-0.3 sheet of --refit-segments squared quads over K frames of the travelling wave, uploaded
        once.  Two contexts: refit (lrk_update_meshes: the first frame's hierarchy refit to every frame) and rebuild
        (lrk_replace_meshes with the frame's own triangles: a fresh device LBVH every frame).
The deform and replace cases read the sheet through `Mesh { file }` from binary PLY frames written under DIR (removed afterwards).
Host milliseconds per phase are wall-clock around calls that synchronise before they return; render_ms is lrk_stats::render_ms
(CUDA events inside the library); medians over the frames.  pixels_differing_* counts the pixels whose raw films differ between
the two arms over all frames: zero, except for hits the triangle test places outside their triangle's padded box, the one
hierarchy dependence of the traversal (traverse.cuh: safe_rcp; DESIGN.md §4 (Mesh deformation)).  The card's name and power
limit are read in the same run, since the times depend on them.
"""
from __future__ import annotations

import argparse
import json
import re
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
CASES = ("instances", "deform", "replace")


def gpu_card(index: int) -> dict:
    import torch

    card = {"name": torch.cuda.get_device_name(index), "power_limit": None}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        card = {"name": q[0].strip(), "power_limit": q[1].strip()}
    except (OSError, IndexError, subprocess.SubprocessError):
        pass
    return card


def rows(desc) -> np.ndarray:
    return np.array([list(desc.instances[i].object_to_world) for i in range(desc.instance_count)], np.float32).reshape(-1, 3, 4)


def ms_since(t0: float) -> float:
    return (time.perf_counter() - t0) * 1e3


def medians(per: dict) -> dict:
    return {k: round(float(np.median(v)), 3) for k, v in per.items()}


def summary(per, differ, **head) -> dict:
    res = dict(head)
    res.update(medians(per))
    res.update({f"pixels_differing_{spp}spp": n for spp, n in differ.items()})
    return res


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


def render_both(arms, spps, per, differ):
    """Both arms' renders of the current frame at every spp: their render_ms into per, their differing pixels into differ."""
    for spp in spps:
        films = []
        for arm, r in arms:
            r.clear()
            r.render(0, spp)
            per[f"render_{arm}_{spp}spp_ms"].append(r.stats()["render_ms"])
            films.append(r.film(raw=True).copy())
        differ[spp] += int((films[0].view(np.uint32) != films[1].view(np.uint32)).any(axis=-1).sum())


def two_arm_rows(host, arms, spps) -> dict:
    """The per-frame lists of a two-arm loop: the host phases, then each arm's render_ms at every spp."""
    per = {k: [] for k in host}
    for spp in spps:
        for arm in arms:
            per[f"render_{arm}_{spp}spp_ms"] = []
    return per


def frame_loop(frames: int, spp: int) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer, Scene

    src = [scenes.instanced_spheres(resolution=(1920, 1080), spp=spp, time=k / 8.0) for k in range(frames + 1)]
    fresh, upd = Renderer(device_index=0), Renderer(device_index=0)
    first = Scene.from_source(src[0], REPO)
    upd.upload(first.desc())
    upd.render(0, spp)  # warm-up of the kernels
    fresh.upload(first.desc())
    fresh.render(0, spp)
    prev = rows(first.desc())
    per = {k: [] for k in ("parse_flatten_ms", "upload_ms", "reupload_render_ms", "update_ms", "update_render_ms")}
    identical = True
    for k in range(1, frames + 1):
        t0 = time.perf_counter()
        scene = Scene.from_source(src[k], REPO)
        desc = scene.desc()
        per["parse_flatten_ms"].append(ms_since(t0))
        t0 = time.perf_counter()
        fresh.upload(desc)
        per["upload_ms"].append(ms_since(t0))
        fresh.render(0, spp)
        per["reupload_render_ms"].append(fresh.stats()["render_ms"])
        cur = rows(desc)
        ids = np.flatnonzero((cur.view(np.uint32) != prev.view(np.uint32)).any(axis=(1, 2)))
        t0 = time.perf_counter()
        upd.update_instances(ids, cur[ids])
        per["update_ms"].append(ms_since(t0))
        upd.render(0, spp)
        per["update_render_ms"].append(upd.stats()["render_ms"])
        identical &= bool(np.array_equal(fresh.film(raw=True), upd.film(raw=True)))
        prev = cur
        scene.close()
    fresh.close()
    upd.close()
    out = medians(per)
    out.update({"spp": spp, "frames": frames, "moved_instances": int(len(ids)), "films_bit_identical": identical})
    return out


def scaling(count: int, repeats: int = 5) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer, Scene

    a = Scene.from_source(scenes.instanced_spheres(resolution=(480, 270), spp=1, big_count=4, small_count=count, small_subdivision=1), REPO)
    b = Scene.from_source(scenes.instanced_spheres(resolution=(480, 270), spp=1, big_count=4, small_count=count, small_subdivision=1, time=0.5), REPO)
    r = Renderer(device_index=0)
    r.upload(a.desc())
    ra, rb = rows(a.desc()), rows(b.desc())
    ids = np.arange(len(ra))
    r.update_instances(ids, rb)  # the first update also derives the meshes' bounds from the host hierarchy
    all_ms, none_ms = [], []
    for k in range(repeats):
        t0 = time.perf_counter()
        r.update_instances(ids, ra if k % 2 == 0 else rb)
        all_ms.append(ms_since(t0))
        t0 = time.perf_counter()
        r.update_instances([], np.zeros((0, 3, 4), np.float32))
        none_ms.append(ms_since(t0))
    r.close()
    return {"instances": int(len(ra)), "update_all_ms": round(float(np.median(all_ms)), 3), "rebuild_only_ms": round(float(np.median(none_ms)), 3)}


def deform(out: Path, frames: int, segments: int, amplitude: float, emissive: bool, spps) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer, Scene

    tag = f"a{amplitude}_{'emissive' if emissive else 'matte'}"
    times = [0.8 * k / frames for k in range(frames)]
    for k, t in enumerate(times):
        write_ply(out / f"{tag}_{k}.ply", *scenes.wavy_sheet_grid((segments, segments), amplitude, t))
    fresh, upd = Renderer(device_index=0), Renderer(device_index=0)
    per = two_arm_rows(("parse_flatten_ms", "upload_ms", "update_ms"), ("reupload", "update"), spps)
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
        per["parse_flatten_ms"].append((t1 - t0) * 1e3)
        per["upload_ms"].append((t2 - t1) * 1e3)
        per["update_ms"].append((t4 - t3) * 1e3)
        render_both((("reupload", fresh), ("update", upd)), spps, per, differ)
        print(f"[{tag}] frame {k}: parse + flatten {per['parse_flatten_ms'][-1]:.0f} ms, update {per['update_ms'][-1]:.2f} ms",
              file=sys.stderr, flush=True)
    fresh.close()
    upd.close()
    return summary(per, differ, amplitude=amplitude, emissive=emissive, triangles=int(2 * segments * segments), frames=frames)


def _mesh_arrays(d, mesh):
    """The vertex [n, 8] float32 and local triangle [m, 3] uint32 records of `mesh` in the description d."""
    m = d.meshes[mesh]
    v = np.ctypeslib.as_array(d.vertices, (d.vertex_count,))
    t = np.ctypeslib.as_array(d.triangles, (d.triangle_count,))
    verts = np.frombuffer(v[m.vertex_offset:m.vertex_offset + m.vertex_count].tobytes(), np.float32).reshape(-1, 8).copy()
    tris = np.frombuffer(t[m.triangle_offset:m.triangle_offset + m.triangle_count].tobytes(), np.uint32).reshape(-1, 3).copy()
    return verts, tris


def topology(out: Path, frames: int, seg_range, spps) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer, Scene

    segments = [int(round(seg_range[0] + (seg_range[1] - seg_range[0]) * k / max(frames - 1, 1))) for k in range(frames)]
    for k, s in enumerate(segments):
        write_ply(out / f"topology_{k}.ply", *scenes.wavy_sheet_grid((s, s), 0.08, 0.1 * k))
    fresh, rep = Renderer(device_index=0), Renderer(device_index=0)
    per = two_arm_rows(("parse_flatten_ms", "upload_ms", "replace_ms"), ("reupload", "replace"), spps)
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
            per["replace_ms"].append(ms_since(t3))
        per["parse_flatten_ms"].append((t1 - t0) * 1e3)
        per["upload_ms"].append((t2 - t1) * 1e3)
        render_both((("reupload", fresh), ("replace", rep)), spps, per, differ)
        print(f"[topology] frame {k}: {2 * segments[k] ** 2} triangles, parse + flatten {per['parse_flatten_ms'][-1]:.0f} ms, "
              f"upload {per['upload_ms'][-1]:.1f} ms" + (f", replace {per['replace_ms'][-1]:.1f} ms" if k else ""), file=sys.stderr, flush=True)
    fresh.close()
    rep.close()
    return summary(per, differ, case="topology", frames=frames, triangles=[2 * s * s for s in segments])


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
    per = two_arm_rows(("update_meshes_ms", "replace_meshes_ms"), ("refit", "rebuild"), spps)
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
        per["update_meshes_ms"].append((t1 - t0) * 1e3)
        per["replace_meshes_ms"].append((t2 - t1) * 1e3)
        render_both((("refit", refit), ("rebuild", rebuild)), spps, per, differ)
        print(f"[refit_vs_rebuild] frame {k}: update {per['update_meshes_ms'][-1]:.1f} ms, replace {per['replace_meshes_ms'][-1]:.1f} ms",
              file=sys.stderr, flush=True)
    refit.close()
    rebuild.close()
    return summary(per, differ, case="refit_vs_rebuild", frames=frames, amplitude=amplitude, triangles=2 * segments * segments)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--case", choices=CASES, help="one case (default: all three)")
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--spp", default="1,16")
    ap.add_argument("--deform-segments", type=int, default=1000, help="deform: the sheet's segments per side")
    ap.add_argument("--amplitudes", default="0.02,0.3", help="deform: the Matte sheet's wave heights; the emissive sheet runs at the first")
    ap.add_argument("--replace-segments", default="800:980", help="replace: first:last segment count of the topology frames")
    ap.add_argument("--refit-segments", type=int, default=1000, help="replace: the refit_vs_rebuild sheet's segments per side")
    ap.add_argument("--out", help="directory for the PLY frames (default: a temporary directory, removed afterwards)")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_scene_update.py measures on a CUDA device; none is available")
    spps = [int(x) for x in args.spp.split(",")]
    card = gpu_card(0)
    for case in [args.case] if args.case else CASES:
        if case == "instances":
            print(json.dumps({"bench": "scene_update", "card": card, "frame_loop": [frame_loop(args.frames, spp) for spp in spps],
                              "scaling": [scaling(n) for n in (1000, 10000)]}), flush=True)
            continue
        out = Path(args.out) if args.out else Path(tempfile.mkdtemp(prefix="bench_scene_update_"))
        out.mkdir(parents=True, exist_ok=True)
        try:
            if case == "deform":
                amplitudes = [float(a) for a in args.amplitudes.split(",")]
                results = [deform(out, args.frames, args.deform_segments, a, e, spps) for a, e in [(a, False) for a in amplitudes] + [(amplitudes[0], True)]]
            else:
                seg_range = [int(x) for x in args.replace_segments.split(":")]
                results = [topology(out, args.frames, seg_range, spps), refit_vs_rebuild(out, args.frames, args.refit_segments, spps)]
        finally:
            for f in out.glob("*.ply"):
                f.unlink()
            if not args.out:
                shutil.rmtree(out, ignore_errors=True)
        print(json.dumps({"bench": "mesh_update" if case == "deform" else "mesh_replace", "gpu": card, "cases": results}), flush=True)


if __name__ == "__main__":
    main()
