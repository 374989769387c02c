"""The triangle-level light trees (option "light_tree_triangles") against the instance-level light tree on cuda:0.  Prints one JSON
line.

    python tools/bench_light_tree_triangles.py [--spp 64] [--reference-spp 4096]

  * Four frames: the many-light frame (scenes.many_lights, 1920x1080: 48 emissive level-3 spheres and two quads), the emissive
    globe (scenes.emissive_globe, 1024x1024, one level-5 sphere), C3 (1920x1080 @1024 by its own count: two quad lights, nothing to
    choose) and near_light (1024x1024, one quad).  Per frame a reference of sample indices [SPP, SPP + REF) rendered with the
    triangle-level trees, then alternately, twice each, the uniform sampler ("uniform"), the instance-level tree ("tree") and the
    triangle-level trees ("triangles") over [0, SPP).  rel_mse = sum((x - ref)^2) / sum(ref^2) over the normalised rgb;
    equal_time_error_ratio = (rel_mse * ms) of "triangles" over that of "tree", the error ratio at equal device time.
  * The host time of lrk_upload_scene with the option off and on (light_tree on in both), for the many-light frame and for the
    globe at subdivision 7 (327 680 emissive triangles): the bottom trees are built there.
Device times are lrk_stats::render_ms (CUDA events inside the library).  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

from bench_adaptive import gpu_card, rel_mse  # noqa: E402

MODES = {"uniform": (0, 0), "tree": (1, 0), "triangles": (1, 1)}


def render(r, desc, mode: str, spp_begin: int, spp_end: int):
    tree, tris = MODES[mode]
    r.set_option("light_tree", tree)
    r.set_option("light_tree_triangles", tris)
    r.upload(desc)
    r.render(spp_begin, spp_end)
    return r.stats()["render_ms"], r.film().copy()


def frame(r, desc, spp: int, ref_spp: int) -> dict:
    _, ref = render(r, desc, "triangles", spp, spp + ref_spp)
    runs = {m: [] for m in MODES}
    err = {}
    for _ in range(2):
        for m in MODES:
            ms, img = render(r, desc, m, 0, spp)
            runs[m].append(round(ms, 3))
            err[m] = rel_mse(img, ref)
    ms = {k: min(v) for k, v in runs.items()}
    return {"resolution": [desc.camera.resolution[0], desc.camera.resolution[1]], "spp": spp, "reference_spp": ref_spp,
            "device_ms": ms, "runs_ms": runs, "rel_mse": err,
            "error_ratio": round(err["triangles"] / err["tree"], 4), "time_ratio": round(ms["triangles"] / ms["tree"], 4),
            "equal_time_error_ratio": round(err["triangles"] * ms["triangles"] / (err["tree"] * ms["tree"]), 4)}


def upload_ms(r, desc) -> dict:
    out = {}
    r.set_option("light_tree", 1)
    for _ in range(2):
        for name, tris in (("off", 0), ("on", 1)):
            r.set_option("light_tree_triangles", tris)
            t0 = time.perf_counter()
            r.upload(desc)
            out.setdefault(name, []).append(round(1e3 * (time.perf_counter() - t0), 1))
    return {k: min(v) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spp", type=int, default=64)
    ap.add_argument("--reference-spp", type=int, default=4096)
    args = ap.parse_args()
    if args.spp < 1 or args.reference_spp < 1:
        ap.error("--spp and --reference-spp take counts >= 1")
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_light_tree_triangles.py: no CUDA device (the radiance path has no CPU fallback)")
    from luisarender_b200 import scenes
    from luisarender_b200.api import Renderer, Scene

    def desc(src):
        return Scene.from_source(src, REPO).desc()

    r = Renderer(device_index=0)
    many = desc(scenes.many_lights(resolution=(1920, 1080), spp=args.spp))
    out = {"gpu": gpu_card(0),
           "many_lights": frame(r, many, args.spp, args.reference_spp),
           "emissive_globe": frame(r, desc(scenes.emissive_globe(resolution=(1024, 1024), spp=args.spp)), args.spp, args.reference_spp),
           "c3": frame(r, desc(scenes.instanced_spheres(resolution=(1920, 1080), spp=1024, seed=1)), args.spp, args.reference_spp),
           "near_light": frame(r, desc(scenes.near_light(resolution=(1024, 1024), spp=args.spp)), args.spp, args.reference_spp),
           "upload_ms": {"many_lights": upload_ms(r, many),
                         "globe_subdivision_7": upload_ms(r, desc(scenes.emissive_globe(resolution=(64, 64), spp=1, subdivision=7)))}}
    r.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
