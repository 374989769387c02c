"""Scene updates against re-uploads in a frame loop on cuda:0.  Prints one JSON line.

    python tools/bench_scene_update.py [--frames 8] [--spp 1,16]

Frame loop: config C3 (1920x1080, 1.39M instanced triangles) with its 64 spheres moving (scenes.instanced_spheres(time=k / 8)),
K frames at each spp.  Two contexts, two arms per frame:
  * re-upload: Scene.from_source (parse + flatten, host BLAS and TLAS builds) + desc + lrk_upload_scene + lrk_render;
  * update:    lrk_update_instances of every moved instance (rows taken from the same frame's description) + lrk_render.
Host milliseconds per phase are wall-clock around calls that synchronise before they return; render_ms is lrk_stats::render_ms
(CUDA events inside the library).  Each frame's two raw films must be bit-identical.  The render times of the two arms compare the
device-built instance level of the update (LBVH) with the host's SAH instance level.
Scaling: the update of 10^3 and 10^4 small spheres, all moved, and the update of none of them (the instance-level rebuild and the
film clear alone).  The card's name and power limit are read in the same run, since the times depend on them.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))


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
    out = {k: round(float(np.median(v)), 3) for k, v in per.items()}
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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--spp", default="1,16")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_scene_update.py measures on a CUDA device; none is available")
    line = {"bench": "scene_update", "card": gpu_card(0),
            "frame_loop": [frame_loop(args.frames, int(s)) for s in args.spp.split(",")],
            "scaling": [scaling(n) for n in (1000, 10000)]}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
