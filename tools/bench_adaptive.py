"""Adaptive sampling against uniform sampling on cuda:0: time to a given image quality.  Prints one JSON line.

    python tools/bench_adaptive.py [--threshold 0.01] [--frames C3,C2]

Frames: C3 (1.39M-tri instanced, Disney + NEE, 1920x1080) and C2's Cornell box (1024x1024).  Per frame:
  * a uniform 4096-spp reference of sample indices [1024, 5120), independent of the samples under test;
  * alternately, twice each, the uniform 1024-spp render (lrk_render) and the adaptive render with threshold 0 (the same samples:
    the film must be bit-identical, and the time difference is what the rounds cost);
  * the adaptive render at THRESHOLD (64 to 1024 spp), after one untimed run.
Device times are lrk_stats::render_ms (CUDA events inside the library); rel_mse = sum((x - ref)^2) / sum(ref^2) over the normalised
rgb.  The card's name and power limit are read in the same run, since the times depend on them.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))

MIN_SPP, MAX_SPP, REF_SPP = 64, 1024, 4096


def frames():
    from luisarender_b200 import scenes

    return {"C3": lambda: scenes.instanced_spheres(resolution=(1920, 1080), spp=MAX_SPP, seed=1),
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


def measure(r, src: str, threshold: float) -> dict:
    from luisarender_b200.api import Scene

    d = Scene.from_source(src, REPO).desc()
    w, h = d.camera.resolution[0], d.camera.resolution[1]
    r.upload(d)
    r.render(MAX_SPP, MAX_SPP + REF_SPP)
    ref = r.film().copy()
    uniform_ms, zero_ms, zero_same = [], [], True
    for _ in range(2):
        r.clear()
        r.render(0, MAX_SPP)
        uniform_ms.append(r.stats()["render_ms"])
        uniform_raw = r.film(raw=True).copy()
        uniform = r.film().copy()
        r.render_adaptive(0.0, MIN_SPP, MAX_SPP)
        zero_ms.append(r.stats()["render_ms"])
        zero_same &= bool(np.array_equal(r.film(raw=True).view(np.uint32), uniform_raw.view(np.uint32)))
    r.render_adaptive(threshold, MIN_SPP, MAX_SPP)  # untimed: buffers
    r.render_adaptive(threshold, MIN_SPP, MAX_SPP)
    st = r.stats()
    img = r.film()
    levels, pixels = np.unique(r.sample_counts(), return_counts=True)
    uniform_samples = w * h * MAX_SPP
    return {
        "resolution": [w, h],
        "uniform": {"spp": MAX_SPP, "device_ms": round(min(uniform_ms), 3), "samples": uniform_samples, "rel_mse": rel_mse(uniform, ref)},
        "adaptive": {"device_ms": round(st["render_ms"], 3), "samples": int(st["samples"]), "rel_mse": rel_mse(img, ref),
                     "pixels_per_count": {str(int(k)): int(v) for k, v in zip(levels, pixels)}},
        "time_ratio": round(st["render_ms"] / min(uniform_ms), 4),
        "sample_ratio": round(st["samples"] / uniform_samples, 4),
        "threshold0": {"device_ms": round(min(zero_ms), 3), "overhead": round(min(zero_ms) / min(uniform_ms) - 1.0, 4),
                       "bit_identical_to_uniform": zero_same,
                       "runs_ms": {"uniform": [round(x, 3) for x in uniform_ms], "threshold0": [round(x, 3) for x in zero_ms]}},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threshold", type=float, default=0.01)
    ap.add_argument("--frames", default="C3,C2")
    args = ap.parse_args()
    if not (np.isfinite(args.threshold) and args.threshold >= 0.0):
        ap.error("--threshold takes a finite value >= 0")
    table = frames()
    names = args.frames.split(",")
    unknown = [n for n in names if n not in table]
    if unknown:
        ap.error(f"unknown frames {unknown}: choose from {sorted(table)}")
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_adaptive.py: no CUDA device (the radiance path has no CPU fallback)")
    from luisarender_b200.api import Renderer

    r = Renderer(device_index=0)
    out = {"threshold": args.threshold, "min_spp": MIN_SPP, "max_spp": MAX_SPP, "reference_spp": REF_SPP, "gpu": gpu_card(0),
           "frames": {n: measure(r, table[n](), args.threshold) for n in names}}
    r.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
