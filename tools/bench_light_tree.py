"""The light tree (option "light_tree") against the uniform light sampler on cuda:0.  Prints one JSON line.

    python tools/bench_light_tree.py [--spp 64] [--reference-spp 4096]

  * The many-light frame (scenes.many_lights: C3 with 48 emissive spheres, 1920x1080): a 4096-spp reference of sample indices
    [SPP, SPP + 4096) rendered with the tree, then alternately, twice each, the uniform and the tree render of [0, SPP).  Device time
    and rel_mse = sum((x - ref)^2) / sum(ref^2) over the normalised rgb.  equal_time_error_ratio = (rel_mse * ms) of the tree over
    that of the uniform sampler: the error ratio at equal device time, since the error of an unbiased render falls as 1 / samples.
  * C3 (two quad lights, 1920x1080 @1024) with the option off and on, alternately, twice each: what the tree costs where it has
    nothing to choose from.
Device times are lrk_stats::render_ms (CUDA events inside the library).  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

from bench_adaptive import gpu_card, rel_mse  # noqa: E402


def render(r, desc, tree: bool, spp_begin: int, spp_end: int):
    r.set_option("light_tree", int(tree))
    r.upload(desc)
    r.render(spp_begin, spp_end)
    return r.stats()["render_ms"], r.film().copy()


def many_lights(r, spp: int, ref_spp: int) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Scene

    d = Scene.from_source(scenes.many_lights(resolution=(1920, 1080), spp=spp), REPO).desc()
    _, ref = render(r, d, True, spp, spp + ref_spp)
    runs = {"uniform": [], "tree": []}
    err = {}
    for _ in range(2):
        for name in ("uniform", "tree"):
            ms, img = render(r, d, name == "tree", 0, spp)
            runs[name].append(round(ms, 3))
            err[name] = rel_mse(img, ref)
    ms = {k: min(v) for k, v in runs.items()}
    return {"resolution": [1920, 1080], "spp": spp, "reference_spp": ref_spp, "emitters": int(sum(1 for i in range(d.instance_count)
                                                                                                     if d.instances[i].handle[0] & 8)),
            "device_ms": ms, "runs_ms": runs, "rel_mse": err,
            "error_ratio": round(err["tree"] / err["uniform"], 4), "time_ratio": round(ms["tree"] / ms["uniform"], 4),
            "equal_time_error_ratio": round(err["tree"] * ms["tree"] / (err["uniform"] * ms["uniform"]), 4)}


def c3_overhead(r) -> dict:
    from luisarender_b200 import scenes
    from luisarender_b200.api import Scene

    d = Scene.from_source(scenes.instanced_spheres(resolution=(1920, 1080), spp=1024, seed=1), REPO).desc()
    render(r, d, True, 0, 64)  # warm-up of the tree's kernels
    runs = {"off": [], "on": []}
    for _ in range(2):
        for name in ("off", "on"):
            ms, _ = render(r, d, name == "on", 0, 1024)
            runs[name].append(round(ms, 3))
    ms = {k: min(v) for k, v in runs.items()}
    return {"spp": 1024, "device_ms": ms, "runs_ms": runs, "overhead": round(ms["on"] / ms["off"] - 1.0, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spp", type=int, default=64)
    ap.add_argument("--reference-spp", type=int, default=4096)
    args = ap.parse_args()
    if args.spp < 1 or args.reference_spp < 1:
        ap.error("--spp and --reference-spp take counts >= 1")
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_light_tree.py: no CUDA device (the radiance path has no CPU fallback)")
    from luisarender_b200.api import Renderer

    r = Renderer(device_index=0)
    out = {"gpu": gpu_card(0), "many_lights": many_lights(r, args.spp, args.reference_spp), "c3": c3_overhead(r)}
    r.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
