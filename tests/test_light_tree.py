"""The light tree on the GPU (option "light_tree"; include/lrk.h, csrc/device/light_tree.h).

Off, the option must change nothing; on, a scene with one light must render bit for bit as without it, the many-light frame must
render the same image as the uniform sampler within its noise (and with less of it), shapes that share a Light node must all be
sampled, and scheduling, sharding, the G-buffer mode and the adaptive mode must compose with it unchanged.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

REPO = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu
f32 = np.float32
RES = (128, 72)
BLOCK = 16


def _scene(src):
    from luisarender_b200.api import Scene

    return Scene.from_source(src, REPO)


@pytest.fixture(scope="module")
def many_small():
    from luisarender_b200 import scenes

    return _scene(scenes.many_lights(resolution=RES, spp=16, count=48, big_subdivision=3, small_subdivision=2))


@pytest.fixture(scope="module")
def many_equal():
    """The many-light frame with every sphere of the same emission, one Light node each ..."""
    from luisarender_b200 import scenes

    return _scene(scenes.many_lights(resolution=RES, spp=16, count=48, spread=False, big_subdivision=3, small_subdivision=2))


@pytest.fixture(scope="module")
def many_shared():
    """... and the same spheres sharing one node."""
    from luisarender_b200 import scenes

    return _scene(scenes.many_lights(resolution=RES, spp=16, count=48, shared_node=True, big_subdivision=3, small_subdivision=2))


@pytest.fixture(scope="module")
def environment_one_light():
    from luisarender_b200 import scenes

    return _scene(scenes.environment_scene(resolution=(48, 30), spp=4, area_light=True))


@pytest.fixture(scope="module")
def medium_small():
    from luisarender_b200 import scenes

    return _scene(scenes.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3, small_subdivision=2,
                                           small_count=12))


@pytest.fixture
def r(gpu_renderer):
    """gpu_renderer, with the options this file touches back at their defaults afterwards (the renderer is shared by the session)."""
    yield gpu_renderer
    for name, value in (("light_tree", 0), ("gbuffer", 0), ("max_paths_per_pass", 136 << 20)):
        gpu_renderer.set_option(name, value)
    gpu_renderer.set_shard(0, 1, 32)


def render(r, desc, spp_begin, spp_end, tree, raw=True):
    r.set_option("light_tree", int(tree))
    r.upload(desc)
    r.render(spp_begin, spp_end)
    return r.film(raw=raw).copy()


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def sub_renders(r, desc, tree, first, count, spp):
    """`count` independent renders of `spp` samples each from sample index `first` on, as normalised films [count, H, W, 3]."""
    return np.stack([render(r, desc, first + k * spp, first + (k + 1) * spp, tree, raw=False)[..., :3] for k in range(count)]).astype(np.float64)


def block_means(films):
    n, h, w, _ = films.shape
    hb, wb = h // BLOCK, w // BLOCK
    b = films[:, :hb * BLOCK, :wb * BLOCK].reshape(n, hb, BLOCK, wb, BLOCK, 3).mean(axis=(2, 4, 5)).reshape(n, -1)
    return np.concatenate([films.mean(axis=(1, 2, 3))[:, None], b], axis=1)  # column 0: the whole image


def z_scores(a, b):
    """(mean a - mean b) / its standard error, per block, from the spread of the independent sub-renders.  A block without noise in
    either (the black background) gives 0 if the means agree, else inf."""
    ma, mb = block_means(a), block_means(b)
    se = np.sqrt(ma.var(axis=0, ddof=1) / len(ma) + mb.var(axis=0, ddof=1) / len(mb))
    diff = ma.mean(axis=0) - mb.mean(axis=0)
    return np.where(se > 0, diff / np.where(se > 0, se, 1.0), np.where(diff == 0, 0.0, np.inf))


# Unbiasedness checks compare 1 + 32 block means (the image and its 16 x 16 blocks) of 32 + 32 sub-renders at 4 sigma: for a normal
# estimate each comparison fails with probability 6e-5, with sigma estimated from the sub-renders (t, 62 dof) 1.7e-4, so a frame
# fails by chance about 0.6 % of the time (the renders are seeded, so a given seed passes or fails for good).
SUBRENDERS, SUB_SPP, Z_MAX = 32, 16, 4.0


# ---- 1. off changes nothing -------------------------------------------------------------------------------------------------------
def test_option_off_equals_a_context_that_never_set_it(spheres_small, r):
    from luisarender_b200.api import Renderer

    fresh = Renderer(device_index=0)
    try:
        fresh.set_option("strict_math", 0 if r.fast else 1)
        fresh.upload(spheres_small.desc())
        fresh.render(0, 4)
        want, want_launches = fresh.film(raw=True), fresh.stats()["kernel_launches"]
    finally:
        fresh.close()
    got = render(r, spheres_small.desc(), 0, 4, tree=False)
    assert np.array_equal(bits(got), bits(want))
    assert r.stats()["kernel_launches"] == want_launches


# ---- 2. one light: the tree's pmf is exactly 1 -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cornell_small", "textured_wrappers_small", "environment_one_light"])
def test_one_light_scenes_render_bit_identically(request, name, r):
    d = request.getfixturevalue(name).desc()
    assert sum(1 for i in range(d.instance_count) if d.instances[i].handle[0] & 8) == 1  # one emissive instance
    off = render(r, d, 0, 8, tree=False)
    on = render(r, d, 0, 8, tree=True)
    assert np.array_equal(bits(on), bits(off))


# ---- 3. unbiased: the same image as the uniform sampler ---------------------------------------------------------------------------
def test_many_lights_tree_agrees_with_uniform(many_small, r):
    d = many_small.desc()
    uniform = sub_renders(r, d, False, 0, SUBRENDERS, SUB_SPP)
    tree = sub_renders(r, d, True, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)  # disjoint sample indices
    z = z_scores(tree, uniform)
    assert np.abs(z).max() < Z_MAX, z


def test_shared_light_node_is_sampled_whole(many_equal, many_shared, r):
    """With the tree, spheres that share one Light node light the frame as spheres with a node each do under the uniform sampler;
    the uniform sampler draws only the first of the shared ones, and its MIS weights drop part of the others' light."""
    own = sub_renders(r, many_equal.desc(), False, 0, SUBRENDERS, SUB_SPP)
    shared_tree = sub_renders(r, many_shared.desc(), True, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)
    z = z_scores(shared_tree, own)
    assert np.abs(z).max() < Z_MAX, z
    shared_uniform = sub_renders(r, many_shared.desc(), False, 2 * SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)
    assert z_scores(shared_uniform, own)[0] < -Z_MAX  # the whole image is darker beyond its noise


# ---- 4. less noise ----------------------------------------------------------------------------------------------------------------
def test_many_lights_tree_halves_the_error(many_small, r):
    """16 spp against a 1024-spp reference of disjoint sample indices: relative MSE of the tree at most 0.5x that of the uniform
    sampler, averaged over 8 independent 16-spp renders each."""
    d = many_small.desc()
    ref = render(r, d, 1 << 20, (1 << 20) + 1024, True, raw=False)[..., :3].astype(np.float64)

    def rel_mse(tree, first):
        errs = [((render(r, d, first + 16 * k, first + 16 * (k + 1), tree, raw=False)[..., :3] - ref) ** 2 / (ref ** 2 + 1e-2)).mean()
                for k in range(8)]
        return float(np.mean(errs))

    uniform, tree = rel_mse(False, 0), rel_mse(True, 4096)
    assert tree <= 0.5 * uniform, (tree, uniform, tree / uniform)


# ---- 5. scheduling and the other modes --------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(many_small, r):
    d = many_small.desc()
    whole = render(r, d, 0, 8, tree=True)
    r.clear()
    r.render(0, 3)
    r.render(3, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(whole))
    r.set_option("max_paths_per_pass", 1024)
    r.clear()
    r.render(0, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(whole))
    r.set_option("max_paths_per_pass", 136 << 20)
    total = np.zeros_like(whole)
    for rank in range(3):
        r.upload(d)
        r.balance_shards(rank, 3, 32, 1)  # the cost probe runs the tree's kernels too
        r.render(0, 8)
        part = r.film(raw=True)
        assert not np.any((total != 0) & (part != 0))  # every pixel has one owner
        total += part
    assert np.array_equal(bits(total), bits(whole))


def test_gbuffer_and_adaptive_compose(many_small, r):
    d = many_small.desc()
    r.set_option("gbuffer", 1)
    off = render(r, d, 0, 4, tree=False)
    gb_off = r.gbuffer()
    on = render(r, d, 0, 4, tree=True)
    gb_on = r.gbuffer()
    assert not np.array_equal(bits(on), bits(off))  # the tree changes the film ...
    for a, b in zip(gb_on[:2], gb_off[:2]):  # ... not the first hits
        assert np.array_equal(bits(a), bits(b))
    r.set_option("gbuffer", 0)
    uniform = render(r, d, 0, 8, tree=True)
    r.render_adaptive(0.0, 4, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(uniform))


# ---- 6. errors --------------------------------------------------------------------------------------------------------------------
def test_volume_integrator_is_refused_at_upload(medium_small, r):
    d = medium_small.desc()
    before = render(r, d, 0, 2, tree=False)
    r.set_option("light_tree", 1)
    with pytest.raises(RuntimeError, match=r"lrk_upload_scene failed \(-5\): .*light tree"):
        r.upload(d)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        r.set_option("light_tree", 2)
    assert np.array_equal(bits(render(r, d, 0, 2, tree=False)), bits(before))
