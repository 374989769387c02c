"""The table-driven samplers on the GPU at the frame sizes and sample counts of the benchmark configurations (-m gpu).

Every other GPU test of PMJ02BN, Sobol, PaddedSobol and ZSobol renders small frames at a few samples per pixel; the frames the
project is measured on run code those never reach: Sobol indices past 2^32 from sample 256 of a 3840x2160 frame on, 40-bit ZSobol
Morton indices, PMJ02BN's pixel tile of one pixel at 65536 spp.  Here each sampler renders the first samples, the last samples
below spp and, at 3840x2160, the samples around the 2^32 crossing of those frames on one shard that holds the frame's last tile
row and column (partial tiles at 1080 and 2160 rows), against the oracle on the same shard.  A render past the sampler's spp is
refused (include/lrk.h, lrk_render); tests/test_sampler_ranges_cpu.py pins the same arithmetic without a GPU."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

from luisarender_b200 import _ffi as F
from luisarender_b200 import scenes
from luisarender_b200.api import Renderer, Scene
from luisarender_b200.distributed import owned_pixel_mask
from oracle import binding as O
from oracle_shards import TILE, shard, with_depth

pytestmark = pytest.mark.gpu
REPO = Path(__file__).resolve().parents[1]
TABLE_SAMPLERS = ("PMJ02BN", "Sobol", "PaddedSobol", "ZSobol")
DEFAULT_PATHS_PER_PASS = 136 << 20  # the default of lrk_create
REDUCED = dict(big_subdivision=3, small_subdivision=2)
FRAMES = {
    "c2_cornell_1024x1024_4096": lambda: scenes.cornell_box(resolution=(1024, 1024), spp=4096),
    "c3_1920x1080_1024": lambda: scenes.instanced_spheres(resolution=(1920, 1080), spp=1024, **REDUCED),
    "c5_3840x2160_65536": lambda: scenes.instanced_spheres(resolution=(3840, 2160), spp=65536, **REDUCED),
    # an odd log2 spp, not a power of 4, at PMJ02BN's one-pixel tile
    "3840x2160_32768": lambda: scenes.instanced_spheres(resolution=(3840, 2160), spp=32768, **REDUCED),
    # an spp that is not a power of 2
    "cornell_1024x1024_1000": lambda: scenes.cornell_box(resolution=(1024, 1024), spp=1000),
    "c3_full_1920x1080_1024": lambda: scenes.instanced_spheres(resolution=(1920, 1080), spp=1024),
}

_scenes: dict = {}
_oracle: dict = {}


def scene(frame: str, sampler: str) -> Scene:
    if (frame, sampler) not in _scenes:
        src = FRAMES[frame]()
        if sampler != "Independent":
            assert "sampler : Independent" in src
            src = src.replace("sampler : Independent", f"sampler : {sampler}")
        _scenes[(frame, sampler)] = Scene.from_source(src, REPO)
    return _scenes[(frame, sampler)]


def oracle(frame, sampler, d, depth, begin, end):
    """O.render on the shard, once per module: both arithmetic modes compare against the same film."""
    key = (frame, sampler, depth, begin, end)
    if key not in _oracle:
        rank, world = shard(d)
        _oracle[key] = O.render(d, begin, end, rank=rank, world=world, tile_size=TILE)
    return _oracle[key]


def gpu_render(r, begin, end):
    r.clear()
    r.render(begin, end)
    return r.film(raw=True), r.stats()


def ranges(spp: int, width: int):
    out = [(0, 2), (spp - 2, spp)]
    if width == 3840:
        out.append((255, 257))  # Sobol: the global index s << 24 passes 2^32 at s = 256
    return out


@pytest.mark.parametrize("sampler", TABLE_SAMPLERS)
@pytest.mark.parametrize("frame", list(FRAMES))
def test_range_ends_match_oracle(frame, sampler, gpu_renderer):
    """Depth 1 (camera ray, emitter hit, one NEE ray): the sampler's numbers, traversal and the light point are exact integer or
    IEEE arithmetic, so weights and ray counts are exact and strict mode matches the oracle to rel-L2 1e-5 with no pixel off by
    1e-4; fast mode to the suite's fast-math tolerance.  Full depth on the last samples: the off-pixel shares of
    test_render_matches_oracle, stated like its fast-math branch for both modes.  At 2 spp on a shard of ~32 tiles one path that
    takes another branch after a 1-ulp libm difference (strict: 1 - 11 of ~32 k pixels, 0 - 1 of ~100 k closest rays on the
    H100) and then finds a light moves the shard's rel-L2 to 2e-3 - 6e-3, so the rel-L2 is stated for the pixels outside that
    share.  Then the sample range is additive bit for bit, also in passes of 1024 paths that start in the middle of the range."""
    fast = gpu_renderer.fast
    d = scene(frame, sampler).desc()
    spp, w, h = d.camera.spp, d.camera.resolution[0], d.camera.resolution[1]
    assert d.sampler.spp == spp
    rank, world = shard(d)
    mask = owned_pixel_mask(w, h, rank, world, TILE)
    assert mask[-1, -1] and mask[-1].any() and mask[:, -1].any() and mask.sum() >= 16 * TILE * TILE

    def compare(g, c, label):
        gm, cm = g[mask][:, :3], c[mask][:, :3]
        rel = float(np.linalg.norm(gm - cm) / np.linalg.norm(cm))
        err = np.abs(gm - cm).max(axis=-1)
        off = float((err > 1e-4 * np.maximum(np.abs(cm).max(axis=-1), 1.0)).mean())
        print(f"{frame} {sampler} {'fast' if fast else 'strict'} {label}: rel_l2 {rel:.3e} off {off:.3e}")
        return rel, off, err, gm, cm

    d1 = with_depth(d, 1)
    gpu_renderer.upload(d1)
    gpu_renderer.set_shard(rank, world, TILE)
    for begin, end in ranges(spp, w):
        g, st = gpu_render(gpu_renderer, begin, end)
        c, cnt = oracle(frame, sampler, d1, 1, begin, end)
        assert np.array_equal(g[..., 3], c[..., 3]) and (c[mask][:, 3] == end - begin).all()
        assert not g[~mask].any()
        assert st["closest_rays"] == cnt["closest_rays"] == int(mask.sum()) * (end - begin)
        rel, off, err, gm, cm = compare(g, c, f"depth1_{begin}_{end}")
        if fast:
            assert off <= 1e-2, off
            keep = err <= np.quantile(err, 0.99)
            assert np.linalg.norm((gm - cm)[keep]) / np.linalg.norm(cm[keep]) <= 1e-4
            assert gm.mean() == pytest.approx(cm.mean(), rel=5e-3)
        else:
            assert rel <= 1e-5 and off == 0.0, (begin, end, rel, off)

    gpu_renderer.upload(d)
    gpu_renderer.set_shard(rank, world, TILE)
    g, st = gpu_render(gpu_renderer, spp - 2, spp)
    c, cnt = oracle(frame, sampler, d, d.integrator.max_depth, spp - 2, spp)
    assert np.array_equal(g[..., 3], c[..., 3]) and not g[~mask].any()
    rel, off, err, gm, cm = compare(g, c, "full_depth_last")
    share = 1e-2 if fast else 5e-3
    assert off <= share, off
    keep = err <= np.quantile(err, 1.0 - share)
    assert np.linalg.norm((gm - cm)[keep]) / np.linalg.norm(cm[keep]) <= (1e-4 if fast else 1e-5)
    assert gm.mean() == pytest.approx(cm.mean(), rel=5e-3)
    assert st["closest_rays"] == pytest.approx(cnt["closest_rays"], rel=2e-3 if fast else 1e-4)

    # additivity: [spp - 4, spp - 2) + [spp - 2, spp) == [spp - 4, spp), also in passes of 1024 paths
    gpu_renderer.clear()
    gpu_renderer.render(spp - 4, spp)
    whole = gpu_renderer.film(raw=True)
    gpu_renderer.clear()
    gpu_renderer.render(spp - 4, spp - 2)
    gpu_renderer.render(spp - 2, spp)
    assert np.array_equal(gpu_renderer.film(raw=True), whole)
    gpu_renderer.clear()
    gpu_renderer.set_option("max_paths_per_pass", 1024)
    try:
        gpu_renderer.render(spp - 4, spp - 2)
        gpu_renderer.render(spp - 2, spp)
    finally:
        gpu_renderer.set_option("max_paths_per_pass", DEFAULT_PATHS_PER_PASS)
    assert np.array_equal(gpu_renderer.film(raw=True), whole)


def _small(sampler: str, spp: int = 8) -> Scene:
    src = scenes.cornell_box(resolution=(64, 48), spp=spp)
    return Scene.from_source(src.replace("sampler : Independent", f"sampler : {sampler}"), REPO)


@pytest.mark.parametrize("sampler", TABLE_SAMPLERS)
def test_sample_range_past_spp_is_refused(sampler, gpu_renderer):
    """render, render_adaptive and balance_shards past the uploaded sampler's spp raise (-1) naming the sampler and its spp, and
    leave film, stats and shard as they were; a camera update with a larger spp keeps the uploaded sampler record."""
    spp = 8
    d = _small(sampler, spp).desc()
    r = gpu_renderer
    r.upload(d)
    r.set_shard(1, 3, 16)
    r.render(0, 2)
    film, stats = r.film(raw=True), r.stats()
    refused = rf"failed \(-1\): .*{sampler} sampler's spp {spp}\b"
    for call in (lambda: r.render(spp, spp + 1), lambda: r.render(0, spp + 1),
                 lambda: r.render_adaptive(0.01, 2, spp + 1), lambda: r.balance_shards(0, 2, 16, spp + 1)):
        with pytest.raises(RuntimeError, match=refused):
            call()
        assert np.array_equal(r.film(raw=True), film) and r.stats() == stats
    r.render(spp, spp)  # an empty range at the end stays valid
    assert np.array_equal(r.film(raw=True), film)
    r.clear()
    r.render(0, spp)
    got = r.film(raw=True)
    fresh = Renderer(device_index=0)
    try:
        fresh.set_option("strict_math", 0 if r.fast else 1)
        fresh.upload(d)
        fresh.set_shard(1, 3, 16)
        fresh.render(0, spp)
        assert np.array_equal(got, fresh.film(raw=True))
    finally:
        fresh.close()
    camera = F.Camera.from_buffer_copy(d.camera)
    camera.spp = 2 * spp
    r.update_camera(camera)
    with pytest.raises(RuntimeError, match=refused):
        r.render(0, 2 * spp)
    assert not r.film(raw=True).any()


def test_independent_takes_any_range(gpu_renderer):
    spp = 8
    d = _small("Independent", spp).desc()
    gpu_renderer.upload(d)
    gpu_renderer.set_shard(0, 1)
    gpu_renderer.render(spp, spp + 4)
    assert (gpu_renderer.film(raw=True)[..., 3] == 4).all()
