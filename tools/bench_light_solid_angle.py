"""Solid-angle light sampling (option "light_solid_angle") against area sampling on cuda:0.  Prints one JSON line.

    python tools/bench_light_solid_angle.py [--spp 64] [--reference-spp 4096]

Frames: C2's Cornell box (1024x1024: its ceiling light seen from the upper walls and the top of the tall box), C3 (1920x1080: two
quad lights), scenes.near_light (1024x1024: a desk 0.3 under a panel light) and the many-light frame (scenes.many_lights,
1920x1080) with the light tree on in both settings.  Per frame: a reference of `--reference-spp` samples of the indices
[SPP, SPP + reference) rendered with the option on, then alternately, twice each, the renders of [0, SPP) with the option off and
on.  Device time (lrk_stats::render_ms, CUDA events inside the library, the minimum of the two runs) and rel_mse = sum((x - ref)^2)
/ sum(ref^2) over the normalised rgb.  error_ratio: on over off at equal spp; equal_time_error_ratio = (rel_mse * ms) on over off,
since the error of an unbiased render falls as 1 / samples.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

from bench_adaptive import gpu_card, rel_mse  # noqa: E402


def render(r, desc, solid_angle: bool, spp_begin: int, spp_end: int):
    r.set_option("light_solid_angle", int(solid_angle))
    r.upload(desc)
    r.render(spp_begin, spp_end)
    return r.stats()["render_ms"], r.film().copy()


def frame(r, src: str, spp: int, ref_spp: int, light_tree: bool = False) -> dict:
    from luisarender_b200.api import Scene

    d = Scene.from_source(src, REPO).desc()
    r.set_option("light_tree", int(light_tree))
    _, ref = render(r, d, True, spp, spp + ref_spp)
    runs = {"off": [], "on": []}
    err = {}
    for _ in range(2):
        for name in ("off", "on"):
            ms, img = render(r, d, name == "on", 0, spp)
            runs[name].append(round(ms, 3))
            err[name] = rel_mse(img, ref)
    r.set_option("light_tree", 0)
    ms = {k: min(v) for k, v in runs.items()}
    return {"resolution": [d.camera.resolution[0], d.camera.resolution[1]], "spp": spp, "reference_spp": ref_spp, "light_tree": light_tree,
            "device_ms": ms, "runs_ms": runs, "rel_mse": err,
            "error_ratio": round(err["on"] / err["off"], 4), "time_ratio": round(ms["on"] / ms["off"], 4),
            "equal_time_error_ratio": round(err["on"] * ms["on"] / (err["off"] * ms["off"]), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spp", type=int, default=64)
    ap.add_argument("--reference-spp", type=int, default=4096)
    args = ap.parse_args()
    if args.spp < 1 or args.reference_spp < 1:
        ap.error("--spp and --reference-spp take counts >= 1")
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_light_solid_angle.py: no CUDA device (the radiance path has no CPU fallback)")
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer

    spp, ref = args.spp, args.reference_spp
    r = Renderer(device_index=0)
    out = {"gpu": gpu_card(0),
           "c2_cornell": frame(r, scenes.cornell_box(resolution=(1024, 1024), spp=spp), spp, ref),
           "c3": frame(r, scenes.instanced_spheres(resolution=(1920, 1080), spp=spp, seed=1), spp, ref),
           "near_light": frame(r, scenes.near_light(resolution=(1024, 1024), spp=spp), spp, ref),
           "many_lights_tree": frame(r, scenes.many_lights(resolution=(1920, 1080), spp=spp), spp, ref, light_tree=True)}
    r.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
