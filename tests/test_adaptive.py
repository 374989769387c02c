"""Adaptive sampling on the GPU (lrk_render_adaptive, include/lrk.h).

Every pixel of an adaptive render must hold exactly the samples [0, n) of a uniform render of n samples per pixel, bit for bit,
so that the parity of uniform renders with the oracle carries over.  Scenes: the two small surface scenes, a C4-shaped scene in
a homogeneous environment medium (wavefront volume kernels) and shape media (the per-thread volume kernel); all of it in both
arithmetic modes (gpu_renderer).
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

REPO = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu

MIN_SPP, MAX_SPP = 4, 64
LEVELS = [4, 8, 16, 32, 64]
TILE = 32  # lrk_set_shard's default tile size; a multiple of the 8x4 block, so blocks sit on the global 8x4 grid


@pytest.fixture(scope="module")
def medium_small():
    from luisarender_b200 import scenes
    from luisarender_b200.api import Scene

    return Scene.from_source(scenes.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3,
                                                      small_subdivision=2, small_count=12), REPO)


@pytest.fixture(scope="module")
def shape_media_small():
    from luisarender_b200 import scenes
    from luisarender_b200.api import Scene

    return Scene.from_source(scenes.media_box(resolution=(40, 40), spp=4), REPO)


SCENES = ["cornell_small", "spheres_small", "medium_small", "shape_media_small"]


@pytest.fixture(params=SCENES)
def scene(request):
    return request.getfixturevalue(request.param)


def block_ids(h: int, w: int) -> np.ndarray:
    y, x = np.mgrid[0:h, 0:w]
    return (y // 4) * ((w + 7) // 8) + x // 8


def adaptive(r, threshold, min_spp=MIN_SPP, max_spp=MAX_SPP):
    r.render_adaptive(threshold, min_spp, max_spp)
    return r.film(raw=True).copy(), r.sample_counts(), r.film_variance(), r.stats()["samples"]


def block_errors(film, var, scale, blocks):
    """e of include/lrk.h per pixel, with m from the raw film (the device sums the luminance of every sample, which rounds
    differently: hence the tolerance of the decision-rule check), and its maximum per 8x4 block."""
    f = np.float32
    n = film[..., 3]
    y = (f(0.2126) * (film[..., 0] * f(scale[0])) + f(0.7152) * (film[..., 1] * f(scale[1])) + f(0.0722) * (film[..., 2] * f(scale[2])))
    m = y.astype(f) / n
    e = (np.sqrt(var) / np.maximum(m, f(0.01))).astype(np.float64)
    return np.array([e[blocks == b].max() for b in range(blocks.max() + 1)])


def test_threshold_zero_equals_uniform(scene, gpu_renderer):
    r = gpu_renderer
    r.upload(scene.desc())
    r.render(0, 16)
    uniform = r.film(raw=True).copy()
    film, counts, _, samples = adaptive(r, 0.0, 4, 16)
    assert np.array_equal(film.view(np.uint32), uniform.view(np.uint32))
    assert (counts == 16).all() and samples == counts.size * 16


def test_invariant_decision_rule_and_blocks(scene, gpu_renderer):
    r = gpu_renderer
    d = scene.desc()
    r.upload(d)
    h, w = d.camera.resolution[1], d.camera.resolution[0]
    blocks = block_ids(h, w)
    # the buffers every block has at every level: a threshold-0 render stopped at that level
    level = {k: adaptive(r, 0.0, MIN_SPP, k) for k in LEVELS}
    for k, (film, counts, var, _) in level.items():
        assert (counts == k).all() and (film[..., 3] <= k).all()
    errors = {k: block_errors(level[k][0], level[k][2], list(d.film.scale), blocks) for k in LEVELS}

    def expected(threshold):
        out = np.full(blocks.max() + 1, MAX_SPP)
        done = np.zeros_like(out, bool)
        for k in LEVELS:
            stop = ~done & (errors[k] < threshold)
            out[stop] = k
            done |= stop
        return out

    # a threshold, away from every block error, that leaves at least three count levels
    all_e = np.concatenate([errors[k] for k in LEVELS])
    all_e = np.unique(all_e[np.isfinite(all_e)])
    threshold = None
    for q in (0.5, 0.4, 0.6, 0.3, 0.7, 0.2, 0.8):
        i = int(q * (len(all_e) - 1))
        t = float(np.float32((all_e[i] + all_e[min(i + 1, len(all_e) - 1)]) / 2))
        if len(np.unique(expected(t))) >= 3 and (np.abs(all_e - t) > 1e-4 * t).all():
            threshold = t
            break
    assert threshold is not None, "no threshold gives three count levels"

    film, counts, var, samples = adaptive(r, threshold)
    got_levels = np.unique(counts)
    assert len(got_levels) >= 3 and set(got_levels) <= set(LEVELS), got_levels
    assert samples == int(counts.astype(np.int64).sum())
    # blocks: one count per 8x4 block
    for b in range(blocks.max() + 1):
        assert len(np.unique(counts[blocks == b])) == 1, b
    # invariant: a pixel with n samples holds the film and the variance of a uniform n-sample render, bit for bit
    for k in got_levels:
        sel = counts == k
        assert np.array_equal(film[sel].view(np.uint32), level[k][0][sel].view(np.uint32)), k
        assert np.array_equal(var[sel].view(np.uint32), level[k][2][sel].view(np.uint32)), k
    # decision rule, recomputed from the level buffers
    want = expected(threshold)
    got = np.array([counts[blocks == b][0] for b in range(blocks.max() + 1)])
    near = np.zeros_like(want, bool)
    for k in LEVELS:
        near |= np.abs(errors[k] - threshold) <= 1e-5 * threshold
    print(f"threshold {threshold:.6g}: levels {got_levels.tolist()}, {int(near.sum())} blocks within 1e-5 of it")
    assert near.sum() == 0
    assert np.array_equal(got, want), int((got != want).sum())


def test_scheduling_does_not_change_a_bit(scene, gpu_renderer):
    from luisarender_b200.api import Renderer

    r = gpu_renderer
    d = scene.desc()
    r.upload(d)
    threshold = 0.05
    ref = adaptive(r, threshold)
    again = adaptive(r, threshold)
    for a, b in zip(ref[:3], again[:3]):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    # tiny passes
    small = Renderer(device_index=0, max_paths_per_pass=1024)
    small.set_option("strict_math", 0 if r.fast else 1)
    small.upload(d)
    got = adaptive(small, threshold)
    assert small.stats()["passes"] > r.stats()["passes"]
    small.close()
    for a, b in zip(ref[:3], got[:3]):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    # three shards on one GPU: summed films and counts equal the single-context render
    films, counts = [], []
    for rank in range(3):
        r.set_shard(rank, 3, TILE)
        f, c, _, _ = adaptive(r, threshold)
        films.append(f)
        counts.append(c)
        assert (f[c == 0] == 0).all()  # nothing outside the shard
    r.set_shard(0, 1, TILE)
    owned = np.stack([c > 0 for c in counts]).sum(axis=0)
    assert (owned == 1).all()
    assert np.array_equal((films[0] + films[1] + films[2]).view(np.uint32), ref[0].view(np.uint32))
    assert np.array_equal(counts[0] + counts[1] + counts[2], ref[1])


def test_invalid_parameters_and_early_downloads(cornell_small, gpu_renderer):
    r = gpu_renderer
    r.upload(cornell_small.desc())
    for threshold, lo, hi in [(0.1, 1, 16), (0.1, 0, 16), (0.1, 8, 4), (-0.1, 4, 16), (float("nan"), 4, 16), (float("inf"), 4, 16)]:
        with pytest.raises(RuntimeError, match=r"lrk_render_adaptive failed \(-1\)"):
            r.render_adaptive(threshold, lo, hi)
    for download in (r.sample_counts, r.film_variance):
        with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
            download()  # nothing adaptive since the upload
    r.render_adaptive(0.1, 4, 8)
    r.sample_counts()
    r.film_variance()
    r.render(8, 9)  # the film no longer matches the counts
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        r.sample_counts()
    r.render_adaptive(0.1, 4, 8)
    r.clear()
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        r.film_variance()
