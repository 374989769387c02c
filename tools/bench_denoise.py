"""The G-buffer mode and the denoiser on cuda:0: what the mode costs, what lrk_denoise costs, and what it buys.  Prints one JSON line.

    python tools/bench_denoise.py [--frames C3,C2]

Frames: C3 (1.39M-tri instanced, Disney + NEE, 1920x1080) and C2's Cornell box (1024x1024).  Per frame:
  * a uniform 4096-spp reference of sample indices [1024, 5120), independent of the samples under test;
  * the cost of the mode: lrk_render of 64 spp with the option off and on, alternated, twice each (lrk_stats::render_ms, CUDA
    events inside the library);
  * the time of lrk_denoise: a host clock around the synchronised call, which includes the copy of the image to the host;
  * rel_mse = sum((x - ref)^2) / sum(ref^2) over the normalised rgb of the raw and the denoised films at 16, 64 and 256 spp, and of
    the raw film at the doublings up to 1024 spp;
  * equal quality: the spp at which the raw film reaches the denoised 16 / 64 spp error, interpolated log-log between the raw
    levels that bracket it (null beyond 1024).
The card's name and power limit are read in the same run, since the times depend on them.
"""
from __future__ import annotations

import argparse
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))

REF_BEGIN, REF_SPP, COST_SPP = 1024, 4096, 64
DENOISED_SPP = [16, 64, 256]
RAW_SPP = [16, 32, 64, 128, 256, 512, 1024]


def frames():
    from luisarender_b200 import scenes

    return {"C3": lambda: scenes.instanced_spheres(resolution=(1920, 1080), spp=1024, seed=1),
            "C2": lambda: scenes.cornell_box(resolution=(1024, 1024), spp=REF_SPP)}


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


def rel_mse(img, ref) -> float:
    a, b = img[..., :3].astype(np.float64), ref[..., :3].astype(np.float64)
    return float(((a - b) ** 2).sum() / (b ** 2).sum())


def equal_quality_spp(raw: dict, target: float):
    levels = sorted(raw)
    for lo, hi in zip(levels, levels[1:]):
        if raw[lo] >= target >= raw[hi]:
            t = (math.log(raw[lo]) - math.log(target)) / (math.log(raw[lo]) - math.log(raw[hi]))
            return round(math.exp(math.log(lo) + t * (math.log(hi) - math.log(lo))), 1)
    return levels[0] if target >= raw[levels[0]] else None


def measure(r, src: str) -> dict:
    from luisarender_b200.api import Scene

    d = Scene.from_source(src, REPO).desc()
    w, h = d.camera.resolution[0], d.camera.resolution[1]
    r.set_option("gbuffer", 0)
    r.upload(d)
    r.render(REF_BEGIN, REF_BEGIN + REF_SPP)
    ref = r.film().copy()
    runs = {"off": [], "on": []}
    for _ in range(2):
        for mode in ("off", "on"):
            r.set_option("gbuffer", 1 if mode == "on" else 0)
            r.clear()
            r.render(0, COST_SPP)
            runs[mode].append(r.stats()["render_ms"])
    r.set_option("gbuffer", 1)
    raw, denoised, denoise_ms = {}, {}, []
    r.clear()
    done = 0
    for spp in RAW_SPP:
        r.render(done, spp)
        done = spp
        raw[spp] = rel_mse(r.film(), ref)
        if spp in DENOISED_SPP:
            r.denoise()  # untimed: scratch buffers
            for _ in range(3):
                t0 = time.perf_counter()
                img = r.denoise()
                denoise_ms.append((time.perf_counter() - t0) * 1e3)
            denoised[spp] = rel_mse(img, ref)
    r.set_option("gbuffer", 0)
    off, on = min(runs["off"]), min(runs["on"])
    return {
        "resolution": [w, h],
        "mode_cost": {"spp": COST_SPP, "off_ms": [round(x, 3) for x in runs["off"]], "on_ms": [round(x, 3) for x in runs["on"]],
                      "overhead": round(on / off - 1.0, 4)},
        "denoise_ms": {"min": round(min(denoise_ms), 3), "median": round(float(np.median(denoise_ms)), 3)},
        "rel_mse_raw": {str(k): v for k, v in raw.items()},
        "rel_mse_denoised": {str(k): v for k, v in denoised.items()},
        "raw_spp_of_equal_quality": {str(k): equal_quality_spp(raw, denoised[k]) for k in (16, 64)},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="C3,C2")
    args = ap.parse_args()
    table = frames()
    names = args.frames.split(",")
    unknown = [n for n in names if n not in table]
    if unknown:
        ap.error(f"unknown frames {unknown}: choose from {sorted(table)}")
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_denoise.py: no CUDA device (the radiance path has no CPU fallback)")
    from luisarender_b200.api import Renderer

    r = Renderer(device_index=0)
    out = {"reference_spp": REF_SPP, "gpu": gpu_card(0), "frames": {n: measure(r, table[n]()) for n in names}}
    r.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
