"""Next-event light sampling options against what they replace, on cuda:0.  Prints one JSON line.

    python tools/bench_light_sampling.py --compare {tree,solid_angle,triangles,candidates,receiver} [--spp 64] [--reference-spp 4096]

A frame's comparison: a reference of `--reference-spp` samples of the indices [SPP, SPP + reference) rendered with the setting under
test, then alternately, twice each, the renders of [0, SPP) under every setting of the comparison.  Device time (lrk_stats::
render_ms, CUDA events inside the library, the minimum of the two runs) and rel_mse = sum((x - ref)^2) / sum(ref^2) over the
normalised rgb.  error_ratio: the setting under test over the baseline at equal spp; equal_time_error_ratio = (rel_mse * ms) of the
one over that of the other, since the error of an unbiased render falls as 1 / samples.

  * tree (option "light_tree" against the uniform sampler): the many-light frame (scenes.many_lights: C3 with 48 emissive spheres,
    1920x1080), and C3 (two quad lights, 1920x1080 @1024) with the option off and on, alternately, twice each: what the tree costs
    where it has nothing to choose from.
  * solid_angle (option "light_solid_angle" against area sampling): C2's Cornell box (1024x1024: its ceiling light seen from the
    upper walls and the top of the tall box), C3 (1920x1080: two quad lights), scenes.near_light (1024x1024: a desk 0.3 under a
    panel light) and the many-light frame (1920x1080) with the light tree on in both settings.
  * triangles (option "light_tree_triangles" against the instance-level tree; the uniform sampler rendered too): the many-light
    frame, the emissive globe (scenes.emissive_globe, 1024x1024, one level-5 sphere), C3 (1920x1080 @1024 by its own count) and
    near_light (1024x1024, one quad).  Also the host time of lrk_upload_scene with the option off and on (light_tree on in both),
    for the many-light frame and for the globe at subdivision 7 (327 680 emissive triangles): the bottom trees are built there.
  * candidates (option "light_candidates" M = 2, 4, 8 against M = 1, one light sample; the reference at M = 8): C3 (1920x1080: Disney
    spheres, two quads), C2's Cornell box (1024x1024), near_light (1024x1024), near_light with its glossy Disney desk (1024x1024:
    the frame where the closure decides which light samples matter) and the many-light frame (1920x1080) with the light tree on
    in every setting.
  * receiver (option "light_receiver" on against off, with the light sampling it refines the same in both): near_light (1024x1024)
    and C2's Cornell box (1024x1024) with solid-angle points; the many-light frame (1920x1080) with the tree, and with the tree and
    its triangle level; the emissive globe (1024x1024) with the triangle level; C3 (1920x1080) with the tree, where there is
    little to gain.
The card's name and power limit are read in the same run.
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


def render(r, desc, options: dict, spp_begin: int, spp_end: int):
    for name, value in options.items():
        r.set_option(name, value)
    r.upload(desc)
    r.render(spp_begin, spp_end)
    return r.stats()["render_ms"], r.film().copy()


def alternate(r, desc, settings: dict, spp: int, ref=None):
    """Renders of [0, spp) under each setting in turn, twice over: the device times per setting, and its rel_mse against `ref`."""
    runs, err = {name: [] for name in settings}, {}
    for _ in range(2):
        for name, options in settings.items():
            ms, img = render(r, desc, options, 0, spp)
            runs[name].append(round(ms, 3))
            if ref is not None:
                err[name] = rel_mse(img, ref)
    return runs, err


def frame(r, desc, settings: dict, base: str, spp: int, ref_spp: int, **extra) -> dict:
    """The comparison of the last of `settings` - the one under test, which also renders the reference - with `base`."""
    test = list(settings)[-1]
    _, ref = render(r, desc, settings[test], spp, spp + ref_spp)
    runs, err = alternate(r, desc, settings, spp, ref)
    ms = {k: min(v) for k, v in runs.items()}
    return {"resolution": [desc.camera.resolution[0], desc.camera.resolution[1]], "spp": spp, "reference_spp": ref_spp, **extra,
            "device_ms": ms, "runs_ms": runs, "rel_mse": err,
            "error_ratio": round(err[test] / err[base], 4), "time_ratio": round(ms[test] / ms[base], 4),
            "equal_time_error_ratio": round(err[test] * ms[test] / (err[base] * ms[base]), 4)}


def compare_tree(r, desc, spp: int, ref_spp: int) -> dict:
    from luisarender_b200 import scenes

    many = desc(scenes.many_lights(resolution=(1920, 1080), spp=spp))
    emitters = int(sum(1 for i in range(many.instance_count) if many.instances[i].handle[0] & 8))
    out = {"many_lights": frame(r, many, {"uniform": {"light_tree": 0}, "tree": {"light_tree": 1}}, "uniform", spp, ref_spp,
                                emitters=emitters)}
    c3 = desc(scenes.instanced_spheres(resolution=(1920, 1080), spp=1024, seed=1))
    render(r, c3, {"light_tree": 1}, 0, 64)  # warm-up of the tree's kernels
    runs, _ = alternate(r, c3, {"off": {"light_tree": 0}, "on": {"light_tree": 1}}, 1024)
    ms = {k: min(v) for k, v in runs.items()}
    out["c3"] = {"spp": 1024, "device_ms": ms, "runs_ms": runs, "overhead": round(ms["on"] / ms["off"] - 1.0, 4)}
    return out


def compare_solid_angle(r, desc, spp: int, ref_spp: int) -> dict:
    from luisarender_b200 import scenes

    def solid_angle_frame(src, light_tree=False):
        settings = {"off": {"light_tree": int(light_tree), "light_solid_angle": 0}, "on": {"light_tree": int(light_tree), "light_solid_angle": 1}}
        return frame(r, desc(src), settings, "off", spp, ref_spp, light_tree=light_tree)

    return {"c2_cornell": solid_angle_frame(scenes.cornell_box(resolution=(1024, 1024), spp=spp)),
            "c3": solid_angle_frame(scenes.instanced_spheres(resolution=(1920, 1080), spp=spp, seed=1)),
            "near_light": solid_angle_frame(scenes.near_light(resolution=(1024, 1024), spp=spp)),
            "many_lights_tree": solid_angle_frame(scenes.many_lights(resolution=(1920, 1080), spp=spp), light_tree=True)}


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


def compare_triangles(r, desc, spp: int, ref_spp: int) -> dict:
    from luisarender_b200 import scenes

    settings = {"uniform": {"light_tree": 0, "light_tree_triangles": 0}, "tree": {"light_tree": 1, "light_tree_triangles": 0},
                "triangles": {"light_tree": 1, "light_tree_triangles": 1}}
    many = desc(scenes.many_lights(resolution=(1920, 1080), spp=spp))
    return {"many_lights": frame(r, many, settings, "tree", spp, ref_spp),
            "emissive_globe": frame(r, desc(scenes.emissive_globe(resolution=(1024, 1024), spp=spp)), settings, "tree", spp, ref_spp),
            "c3": frame(r, desc(scenes.instanced_spheres(resolution=(1920, 1080), spp=1024, seed=1)), settings, "tree", spp, ref_spp),
            "near_light": frame(r, desc(scenes.near_light(resolution=(1024, 1024), spp=spp)), settings, "tree", spp, ref_spp),
            "upload_ms": {"many_lights": upload_ms(r, many),
                          "globe_subdivision_7": upload_ms(r, desc(scenes.emissive_globe(resolution=(64, 64), spp=1, subdivision=7)))}}


def compare_candidates(r, desc, spp: int, ref_spp: int) -> dict:
    from luisarender_b200 import scenes

    def candidates_frame(src, light_tree=False):
        settings = {f"m{m}": {"light_tree": int(light_tree), "light_candidates": m} for m in (1, 2, 4, 8)}
        return frame(r, desc(src), settings, "m1", spp, ref_spp, light_tree=light_tree)

    return {"c3": candidates_frame(scenes.instanced_spheres(resolution=(1920, 1080), spp=spp, seed=1)),
            "c2_cornell": candidates_frame(scenes.cornell_box(resolution=(1024, 1024), spp=spp)),
            "near_light": candidates_frame(scenes.near_light(resolution=(1024, 1024), spp=spp)),
            "glossy_desk": candidates_frame(scenes.near_light(resolution=(1024, 1024), spp=spp, glossy_desk=True)),
            "many_lights_tree": candidates_frame(scenes.many_lights(resolution=(1920, 1080), spp=spp), light_tree=True)}


def compare_receiver(r, desc, spp: int, ref_spp: int) -> dict:
    from luisarender_b200 import scenes

    def receiver_frame(src, **base):
        base = {"light_tree": 0, "light_tree_triangles": 0, "light_solid_angle": 0, "light_candidates": 0, **base}
        settings = {"off": {**base, "light_receiver": 0}, "on": {**base, "light_receiver": 1}}
        return frame(r, desc(src), settings, "off", spp, ref_spp, **{k: v for k, v in base.items() if v})

    many = scenes.many_lights(resolution=(1920, 1080), spp=spp)
    return {"near_light_solid_angle": receiver_frame(scenes.near_light(resolution=(1024, 1024), spp=spp), light_solid_angle=1),
            "c2_cornell_solid_angle": receiver_frame(scenes.cornell_box(resolution=(1024, 1024), spp=spp), light_solid_angle=1),
            "many_lights_tree": receiver_frame(many, light_tree=1),
            "many_lights_triangles": receiver_frame(many, light_tree=1, light_tree_triangles=1),
            "emissive_globe_triangles": receiver_frame(scenes.emissive_globe(resolution=(1024, 1024), spp=spp), light_tree=1,
                                                       light_tree_triangles=1),
            "c3_tree": receiver_frame(scenes.instanced_spheres(resolution=(1920, 1080), spp=spp, seed=1), light_tree=1)}


COMPARE = {"tree": compare_tree, "solid_angle": compare_solid_angle, "triangles": compare_triangles, "candidates": compare_candidates,
           "receiver": compare_receiver}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compare", required=True, choices=sorted(COMPARE))
    ap.add_argument("--spp", type=int, default=64)
    ap.add_argument("--reference-spp", type=int, default=4096)
    args = ap.parse_args()
    if args.spp < 1 or args.reference_spp < 1:
        ap.error("--spp and --reference-spp take counts >= 1")
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_light_sampling.py: no CUDA device (the radiance path has no CPU fallback)")
    from luisarender_b200.api import Renderer, Scene

    def desc(src):
        return Scene.from_source(src, REPO).desc()

    r = Renderer(device_index=0)
    out = {"gpu": gpu_card(0), **COMPARE[args.compare](r, desc, args.spp, args.reference_spp)}
    r.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
