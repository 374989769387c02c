"""GPU parity tests (-m gpu): the sm_90a kernels, called through the C-ABI of libb200pt.so, against the CPU
oracle on the same seeded inputs, plus size-independent properties at the BASELINE.json sizes.

Tolerances (stated per SURVEY.md §8c): integer outputs (hit instance / primitive, ray counts) exact; fp32
per-function outputs 1e-5 relative; images: rel-L2 <= 1e-3 and <= 0.5 % of pixels outside 1e-4 relative
(ULP-level libm differences may flip a discrete decision on a handful of paths)."""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import pytest

from luisarender_b200 import scenes
from luisarender_b200.api import Scene
from oracle import binding as O

pytestmark = pytest.mark.gpu
REPO = Path(__file__).resolve().parents[1]
GOLD = json.loads((Path(__file__).resolve().parent / "golden" / "oracle_kat.json").read_text())


def _random_rays(scene, n, seed):
    rng = np.random.default_rng(seed)
    info = scene.info()
    lo, hi = np.array(info["world_min"]), np.array(info["world_max"])
    o = rng.uniform(lo - 0.5, hi + 0.5, size=(n, 3))
    t = rng.uniform(lo, hi, size=(n, 3))
    d = t - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rays = np.zeros((n, 8), np.float32)
    rays[:, :3], rays[:, 4:7], rays[:, 7] = o, d, np.finfo(np.float32).max
    # a share of short rays exercises tmax handling like the 0.9999*d shadow rays (interaction.cpp:29)
    rays[::3, 7] = rng.uniform(0.5, 6.0, size=len(rays[::3]))
    return rays


@pytest.mark.parametrize("fixture", ["cornell_small", "spheres_small", "textured_wrappers_small"])
def test_trace_matches_oracle_bit_exactly(fixture, request, gpu_renderer):
    scene = request.getfixturevalue(fixture)
    d = scene.desc()
    gpu_renderer.upload(d)
    rays = _random_rays(scene, 200_000, seed=11)
    ref, _ = O.trace(d, rays)
    got = gpu_renderer.trace(rays)
    assert np.array_equal(got["inst"], ref["inst"])
    assert np.array_equal(got["prim"], ref["prim"])
    assert np.array_equal(got["bary"].view(np.uint32), ref["bary"].view(np.uint32))  # same fma chains -> same bits
    assert (ref["inst"] != 0xFFFFFFFF).mean() > 0.1
    occ_ref, _ = O.trace(d, rays, any_hit=True)
    occ = gpu_renderer.trace(rays, any_hit=True)
    assert np.array_equal(occ["inst"], occ_ref["inst"])


def test_trace_edge_cases(cornell_small, gpu_renderer):
    d = cornell_small.desc()
    gpu_renderer.upload(d)
    fmax = np.finfo(np.float32).max
    rays = np.array([
        [0, 1, 0, 0, 0, 0, -1, fmax],        # axis-aligned direction (zero components -> clamped reciprocal)
        [0, 1, 0, 0, 0, -1, 0, fmax],
        [0, 1, 0, 0, 1, 0, 0, 0.5],          # tmax shorter than the wall distance: miss
        [0, 1, 0, 0, 1, 0, 0, 2.0],
        [0, 1, 10, 0, 0, 0, 1, fmax],        # pointing away from everything
        [0, 1, 0, 0, 0, 0, -1, 0.0],         # empty interval
        [-0.005, 1.98, -0.03, 0, 0, 1, 0, fmax],  # starts on the light quad, leaves upward to the ceiling
    ], dtype=np.float32)
    ref, _ = O.trace(d, rays)
    got = gpu_renderer.trace(rays)
    assert np.array_equal(got["inst"], ref["inst"]) and np.array_equal(got["prim"], ref["prim"])
    assert got["inst"][2] == 0xFFFFFFFF and got["inst"][3] == 3 and got["inst"][4] == 0xFFFFFFFF and got["inst"][5] == 0xFFFFFFFF
    assert gpu_renderer.trace(np.zeros((0, 8), np.float32)).shape == (0,)


def _image_parity(gpu_raw, cpu_raw):
    rel = float(np.linalg.norm(gpu_raw[..., :3] - cpu_raw[..., :3]) / np.linalg.norm(cpu_raw[..., :3]))
    scale = np.maximum(np.abs(cpu_raw[..., :3]).max(axis=-1), 1.0)
    off = float((np.abs(gpu_raw[..., :3] - cpu_raw[..., :3]).max(axis=-1) > 1e-4 * scale).mean())
    return rel, off


@pytest.mark.parametrize("name", ["cornell", "cornell_disney", "spheres", "spheres_medium", "textured", "textured_wrappers", "environment"])
def test_render_matches_oracle(name, gpu_renderer):
    import importlib.util
    spec = importlib.util.spec_from_file_location("generate_golden", Path(__file__).resolve().parent / "golden" / "generate_golden.py")
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    scene = Scene.from_source(gen.golden_scenes()[name], REPO)
    d = scene.desc()
    spp = d.camera.spp
    gpu_renderer.upload(d)
    gpu_renderer.render(0, spp)
    gpu_raw = gpu_renderer.film(raw=True)
    st = gpu_renderer.stats()
    cpu_raw, cnt = O.render(d, 0, spp)
    assert np.array_equal(gpu_raw[..., 3], cpu_raw[..., 3])  # weights: exact
    rel, off = _image_parity(gpu_raw, cpu_raw)
    fast = gpu_renderer.fast
    if name == "spheres_medium":
        # The reference's volume estimator evaluates an emitter hit from a ray origin that was moved ONTO the hit point
        # (mega_vpt_naive.cpp:308,319): cos_wo is the direction of a rounding-noise vector, so whether such a hit counts
        # (|cos_wo| < 1e-6 -> invalid, diffuse.cpp:82) is decided by the last bit of the scattered direction.  libm's and
        # CUDA's sin/cos differ by an ulp now and then, so a few paths per thousand flip by exactly the light's radiance.
        # Parity here is: identical ray counts (checked below), <= 1 % of pixels differ, and the rest agree to 1e-3 rel-L2.
        assert off <= 1e-2, off
        err = np.abs(gpu_raw[..., :3] - cpu_raw[..., :3]).max(axis=-1)
        keep = err <= np.quantile(err, 0.99)
        assert np.linalg.norm((gpu_raw[..., :3] - cpu_raw[..., :3])[keep]) / np.linalg.norm(cpu_raw[..., :3][keep]) <= 1e-3
    elif name == "textured_wrappers":
        # The stochastic alpha test hashes the candidate's barycentric BITS (geometry.cpp:170), so a bounce direction that
        # differs by one ulp (CUDA vs glibc sin/cos in the cosine-hemisphere warp) flips the decision for the faces it crosses:
        # a few per cent of the paths that meet a non-opaque surface after their first bounce take another, equally valid,
        # branch.  Parity is therefore exact for everything up to the first bounce (test_alpha_first_bounce_is_exact) and
        # statistical afterwards: <= 4 % of the pixels differ, the rest agree to 1e-3 rel-L2, and the image means agree.
        # fast_math: the shadow rays' origins differ in the last bit too, so the decisions of the alpha tests THEY meet flip as well
        limit = 0.12 if fast else 4e-2
        assert off <= limit, off
        err = np.abs(gpu_raw[..., :3] - cpu_raw[..., :3]).max(axis=-1)
        keep = err <= np.quantile(err, 1.0 - limit)
        assert np.linalg.norm((gpu_raw[..., :3] - cpu_raw[..., :3])[keep]) / np.linalg.norm(cpu_raw[..., :3][keep]) <= 1e-3
        assert gpu_raw[..., :3].mean() == pytest.approx(cpu_raw[..., :3].mean(), rel=0.03)
    elif fast:
        # fast_math closures differ from the oracle's in the last bits; a discrete decision (light triangle, lobe, Russian roulette)
        # flips for about one path in 10^4, and at 4 - 8 spp one such path that ends on a light moves the rel-L2 of the whole
        # image by percents.  Stated tolerance: <= 1 % of the pixels off by more than 1e-4, the other 99 % agree to 1e-4 rel-L2,
        # image means to 0.5 %.
        assert off <= 1e-2, off
        err = np.abs(gpu_raw[..., :3] - cpu_raw[..., :3]).max(axis=-1)
        keep = err <= np.quantile(err, 0.99)
        assert np.linalg.norm((gpu_raw[..., :3] - cpu_raw[..., :3])[keep]) / np.linalg.norm(cpu_raw[..., :3][keep]) <= 1e-4
        assert gpu_raw[..., :3].mean() == pytest.approx(cpu_raw[..., :3].mean(), rel=5e-3)
    else:
        assert rel <= 1e-3, rel
        assert off <= 5e-3, off
    if name != "textured_wrappers":
        assert st["closest_rays"] == pytest.approx(cnt["closest_rays"], rel=2e-3 if fast else 0)  # same paths, ray for ray (strict)
    assert st["shadow_rays"] <= cnt["shadow_rays"]    # zero-contribution shadow rays are not traced on the GPU
    # and against the committed golden film row (generated by the oracle, tests/golden/generate_golden.py)
    gold = np.array(GOLD["scenes"][name]["film_row0"], np.float32).reshape(-1, 3)
    row_ok = np.isclose(gpu_raw[0, :, :3], gold, rtol=1e-3, atol=1e-4).all(axis=-1)
    assert row_ok.all() if name not in ("spheres_medium", "textured_wrappers") and not fast else row_ok.mean() >= (0.85 if fast else 0.9)
    if name != "textured_wrappers":
        assert st["closest_rays"] == pytest.approx(GOLD["scenes"][name]["counters"]["closest_rays"], rel=2e-3 if fast else 0)
    # normalised film = (sum / max(w,1)) * 2^exposure (color.cpp:87-93)
    assert np.allclose(gpu_renderer.film(), O.convert_film(d, gpu_raw), rtol=1e-6, atol=1e-7)


def test_constant_environment_furnace(gpu_renderer):
    """Constant white environment, no area light, a lone convex Matte sphere: radiance 0.8 on the sphere, 1 on the background
    (miss term + uniform-sphere NEE + MIS), and parity with the oracle on the same samples."""
    src = scenes.environment_scene(resolution=(40, 40), spp=64, emission=(1.0, 1.0, 1.0), area_light=False, depth=12)
    src = src.replace("shapes { @ball, @floor }", "shapes { @ball }").replace("position { 0.0, 1.2, 4.0 }", "position { 0.0, 0.7, 4.0 }").replace(
        "front { 0.0, -0.12, -1.0 }", "front { 0.0, 0.0, -1.0 }")
    d = Scene.from_source(src, REPO).desc()
    gpu_renderer.upload(d)
    gpu_renderer.render(0, 64)
    img = gpu_renderer.film()[..., :3]
    assert np.allclose(img[:3], 1.0, atol=1e-5) and img[17:23, 17:23].mean() == pytest.approx(0.8, rel=0.02)
    cpu_raw, cnt = O.render(d, 0, 64)
    rel, off = _image_parity(gpu_renderer.film(raw=True), cpu_raw)
    assert rel <= 1e-3 and off <= 5e-3, (rel, off)
    assert gpu_renderer.stats()["closest_rays"] == cnt["closest_rays"]


def test_alpha_first_bounce_is_exact(gpu_renderer):
    """Alpha-tested and half-transparent surfaces with depth 1 (camera ray, emitter hit, one NEE shadow ray): every ray is
    generated by exact arithmetic, so closest-hit AND any-hit traversal with the stochastic alpha test must reproduce the
    oracle exactly; so must the counters."""
    scene = Scene.from_source(scenes.textured_room(resolution=(64, 40), spp=8, wrappers=True, depth=1), REPO)
    d = scene.desc()
    gpu_renderer.upload(d)
    gpu_renderer.render(0, 8)
    gpu_raw = gpu_renderer.film(raw=True)
    st = gpu_renderer.stats()
    cpu_raw, cnt = O.render(d, 0, 8)
    rel, off = _image_parity(gpu_raw, cpu_raw)
    assert st["closest_rays"] == cnt["closest_rays"] and np.array_equal(gpu_raw[..., 3], cpu_raw[..., 3])
    if gpu_renderer.fast:
        # the shadow ray's origin and direction come out of the fast-math shade kernel: one ulp there changes the barycentric BITS
        # the alpha test of every surface it crosses is hashed from - only the statistics survive
        assert off <= 0.12 and gpu_raw[..., :3].mean() == pytest.approx(cpu_raw[..., :3].mean(), rel=0.03), (rel, off)
    else:
        assert rel <= 1e-5 and off == 0.0, (rel, off)


def test_render_is_deterministic_and_independent_of_scheduling(cornell_small, gpu_renderer):
    d = cornell_small.desc()
    gpu_renderer.upload(d)
    gpu_renderer.render(0, 8)
    a = gpu_renderer.film(raw=True)
    gpu_renderer.clear()
    gpu_renderer.render(0, 8)
    assert np.array_equal(a, gpu_renderer.film(raw=True))  # run-to-run bit-identical (no float atomics on the film)
    # sample-range additivity and pass-size independence: same per-pixel sample order -> same bits
    gpu_renderer.clear()
    gpu_renderer.render(0, 3)
    gpu_renderer.render(3, 8)
    assert np.array_equal(a, gpu_renderer.film(raw=True))
    gpu_renderer.clear()
    gpu_renderer.set_option("max_paths_per_pass", 1024)  # many small passes, pixel chunks smaller than the film
    gpu_renderer.render(0, 8)
    gpu_renderer.set_option("max_paths_per_pass", 8 << 20)
    assert np.array_equal(a, gpu_renderer.film(raw=True))
    # traversal counting does not change the result and counts the oracle's numbers
    gpu_renderer.clear()
    gpu_renderer.set_option("count_traversal", 1)
    gpu_renderer.render(0, 8)
    gpu_renderer.set_option("count_traversal", 0)
    assert np.array_equal(a, gpu_renderer.film(raw=True))
    st = gpu_renderer.stats()
    _, cnt = O.render(d, 0, 8)
    assert st["closest_rays"] == cnt["closest_rays"] and st["closest_nodes"] > 0 and st["closest_tris"] > 0
    assert st["closest_xforms"] + st["shadow_xforms"] <= cnt["xforms"]


SURFACE_DISNEY, SURFACE_LAYERED, SURFACE_DISNEY_THIN, INTEGRATOR_VOLUME_PATH = 1, 7, 64, 1  # include/lrk.h


def _hit_buckets(d):
    """The hit buckets 1..10 the instances of a scene description use: the closure kind lrk_upload_scene gives each instance."""
    from luisarender_b200 import _ffi as F
    used = set()
    for inst in d.instances[:d.instance_count]:
        if inst.handle[0] & F.SHAPE_HAS_SURFACE:
            s = d.surfaces[(inst.handle[1] >> 12) & 4095]
            kind = s.type + 1  # Matte 1, Disney 2, Mirror 3, Glass 4, Plastic 5, Metal 6, Mix 7
            if s.type == SURFACE_DISNEY and s.flags & F.SURFACE_DISNEY_TRANSMISSIVE:
                kind = 8
            if s.type == SURFACE_LAYERED:
                kind = 9
            if s.type == SURFACE_DISNEY and s.flags & SURFACE_DISNEY_THIN:
                kind = 10
            used.add(kind)
    return used


@pytest.mark.parametrize("name", ["environment", "layered", "disney_thin", "c4_medium"])
def test_kernel_launch_count_follows_the_scene(name, gpu_renderer):
    """stats()["kernel_launches"] restated from the scene.  Surface path, per pass: ray generation and film accumulation, and per depth
    closest hit, classification, bucket 0's shade kernel, the shadow rays, the miss kernel when an environment light is present, and
    one shade kernel per further hit bucket in use.  Volume path (C4), per depth: in-medium shadow rays, closest hit, the medium step,
    bucket 0's surface step, the surface NEE rays, and the surface steps of buckets 1 and 2 when used."""
    if name in ("disney_thin", "c4_medium"):  # the reference-render fixtures' scene texts (tests/test_ref_render.py)
        key = {"disney_thin": "spheres_disney_thin", "c4_medium": "config_c4_full_scene"}[name]
        src = bytes(np.load(REPO / "tests" / "golden" / "ref_renders.npz")[f"{key}/scene"]).decode()
    else:
        src = scenes.environment_scene() if name == "environment" else scenes.layered_box()
    scene = Scene.from_source(src, REPO)
    d = scene.desc()
    buckets, depth = _hit_buckets(d), d.integrator.max_depth
    volume = d.integrator.type == INTEGRATOR_VOLUME_PATH
    # each scene exercises what it is here for
    assert {"environment": d.environment.present, "layered": 9 in buckets, "disney_thin": 10 in buckets, "c4_medium": volume}[name]
    if volume:
        per_pass = 2 + depth * (5 + (1 in buckets) + (2 in buckets))
    else:
        per_pass = 2 + depth * (4 + bool(d.environment.present) + len(buckets))
    gpu_renderer.upload(d)
    gpu_renderer.render(0, d.camera.spp)
    st = gpu_renderer.stats()
    assert st["passes"] >= 1
    assert st["kernel_launches"] == st["passes"] * per_pass


def test_pixel_tile_sharding_is_bit_identical(spheres_small, gpu_renderer):
    d = spheres_small.desc()
    gpu_renderer.upload(d)
    gpu_renderer.render(0, 4)
    full = gpu_renderer.film(raw=True)
    total = np.zeros_like(full)
    for rank in range(3):
        gpu_renderer.set_shard(rank, 3, 16)
        gpu_renderer.clear()
        gpu_renderer.render(0, 4)
        part = gpu_renderer.film(raw=True)
        assert ((part[..., 3] == 0) | (part[..., 3] == 4)).all()
        total += part
    gpu_renderer.set_shard(0, 1, 32)
    assert np.array_equal(full, total)  # disjoint tiles: the film reduce only adds zeros (SURVEY.md §8e)
    cpu_part, _ = O.render(d, 0, 4, rank=1, world=3, tile_size=16)
    gpu_renderer.set_shard(1, 3, 16)
    gpu_renderer.clear()
    gpu_renderer.render(0, 4)
    assert np.array_equal(gpu_renderer.film(raw=True)[..., 3], cpu_part[..., 3])
    gpu_renderer.set_shard(0, 1, 32)


def test_error_paths(cornell_small, gpu_renderer):
    from luisarender_b200 import _ffi as F
    import ctypes as C
    d = cornell_small.desc()
    bad = F.SceneDesc.from_buffer_copy(bytes(d))
    bad.abi_version = 99
    with pytest.raises(RuntimeError, match="ABI version"):
        gpu_renderer.upload(bad)
    nolight = F.SceneDesc.from_buffer_copy(bytes(d))
    nolight.light_count = 0
    with pytest.raises(RuntimeError, match="No lights in scene"):  # wave_path.cpp:224-228
        gpu_renderer.upload(nolight)
    with pytest.raises(RuntimeError, match="unknown option"):
        gpu_renderer.set_option("no_such_option", 1)
    gpu_renderer.upload(d)
    with pytest.raises(RuntimeError):
        gpu_renderer.render(5, 2)
    assert C.sizeof(F.Stats) > 0


def test_full_size_properties_c2_cornell(gpu_renderer):
    """Config C2 geometry/resolution (1024x1024 Cornell) at a bounded spp: size-independent properties."""
    scene = Scene.from_source(scenes.cornell_box(resolution=(1024, 1024), spp=4096), REPO)
    d = scene.desc()
    gpu_renderer.upload(d)
    spp = 32
    gpu_renderer.render(0, spp)
    raw = gpu_renderer.film(raw=True)
    st = gpu_renderer.stats()
    assert (raw[..., 3] == spp).all() and np.isfinite(raw).all()
    assert st["samples"] == 1024 * 1024 * spp and st["closest_rays"] >= st["samples"] and st["shadow_rays"] <= st["closest_rays"]
    img = gpu_renderer.film()
    # energy agrees with the oracle's estimate of the same scene at low resolution (same estimator, different pixels)
    small = Scene.from_source(scenes.cornell_box(resolution=(96, 96), spp=64), REPO)
    cpu = O.convert_film(small.desc(), O.render(small.desc(), 0, 64)[0])
    assert img[..., :3].mean() == pytest.approx(cpu[..., :3].mean(), rel=0.02)
    # left wall is red, right wall is green (test_path_tracing.cpp:104-113)
    left, right = img[512, 40, :3], img[512, 1024 - 40, :3]
    assert left[0] > 2 * left[1] and right[1] > 2 * right[0]


def test_full_size_properties_c3_spheres(gpu_renderer):
    """Config C3 scene (1 387 526 instanced triangles, Disney + NEE, 1920x1080) at a bounded spp."""
    scene = Scene.from_source(scenes.instanced_spheres(resolution=(1920, 1080), spp=1024), REPO)
    info = scene.info()
    assert info["instanced_triangles"] == 4 * 327680 + 60 * 1280 + 2 + 4
    d = scene.desc()
    gpu_renderer.upload(d)
    gpu_renderer.render(0, 4)
    raw = gpu_renderer.film(raw=True)
    assert (raw[..., 3] == 4).all() and np.isfinite(raw).all() and raw[..., :3].min() >= 0
    # a crop of the full-size frame against the oracle on exactly the same pixels/samples (tile-sharded oracle run)
    rays = _random_rays(scene, 100_000, seed=5)
    ref, _ = O.trace(d, rays)
    got = gpu_renderer.trace(rays)
    assert np.array_equal(got["inst"], ref["inst"]) and np.array_equal(got["prim"], ref["prim"])
    cpu_part, _ = O.render(d, 0, 4, rank=7, world=64, tile_size=32)
    mask = cpu_part[..., 3] > 0
    assert mask.sum() > 20000
    g, c = raw[mask][:, :3], cpu_part[mask][:, :3]
    rel = np.linalg.norm(g - c) / np.linalg.norm(c)
    if gpu_renderer.fast:  # see test_render_matches_oracle: a handful of diverged paths dominate rel-L2 at 4 spp
        # depth-10 paths over 1.39 M triangles: measured 1.4 % of the pixels carry a path that took another branch somewhere
        err = np.abs(g - c).max(axis=-1)
        keep = err <= np.quantile(err, 0.975)
        assert (err > 1e-4 * np.maximum(np.abs(c).max(axis=-1), 1.0)).mean() <= 2.5e-2
        assert np.linalg.norm((g - c)[keep]) / np.linalg.norm(c[keep]) <= 1e-4
        assert g.mean() == pytest.approx(c.mean(), rel=2e-3)
    else:
        assert rel <= 1e-3, rel


def test_full_size_properties_c4_medium(gpu_renderer):
    """Config C4 (C3 scene + homogeneous medium, depth 8, 3840x2160) at a bounded spp: weights, finiteness, and a
    tile-sharded oracle run on exactly the same pixels/samples (criteria of the small medium case, see above)."""
    scene = Scene.from_source(scenes.instanced_spheres(resolution=(3840, 2160), spp=4096, medium=True, depth=8), REPO)
    d = scene.desc()
    gpu_renderer.upload(d)
    spp = 2
    gpu_renderer.render(0, spp)
    raw = gpu_renderer.film(raw=True)
    st = gpu_renderer.stats()
    # the volume estimator returns NaN for ~0.1 % of the samples: an emitter hit is evaluated from the ray origin MOVED to
    # the hit (mega_vpt_naive.cpp:308,319); when that point equals the hit point bit for bit, normalize(0) = NaN
    # (diffuse.cpp:78-82).  The film drops such samples, weight included (color.cpp:107-130).  Verified on the oracle:
    # every dropped sample of the small medium scene is such a hit.
    assert (raw[..., 3] <= spp).all() and (raw[..., 3] == spp).mean() >= 0.99
    assert np.isfinite(raw).all() and raw[..., :3].min() >= 0
    assert st["samples"] == 3840 * 2160 * spp and st["closest_rays"] >= st["samples"]
    cpu_part, _ = O.render(d, 0, spp, rank=11, world=256, tile_size=32)
    from luisarender_b200.distributed import owned_pixel_mask
    tiles = owned_pixel_mask(3840, 2160, 11, 256, 32)
    mask = cpu_part[..., 3] > 0
    assert mask.sum() > 20000 and not (mask & ~tiles).any()
    # dropped samples are the emitter hits whose moved ray origin lands EXACTLY on the hit point (normalize(0) = NaN in
    # diffuse.cpp:78-82) - the same last-bit decision as the chaotic cos_wo test above, so a few per 10^4 pixels differ
    assert (raw[tiles][:, 3] != cpu_part[tiles][:, 3]).mean() <= (4e-3 if gpu_renderer.fast else 1e-3)
    mask &= raw[..., 3] == cpu_part[..., 3]
    g, c = raw[mask][:, :3], cpu_part[mask][:, :3]
    err = np.abs(g - c).max(axis=-1)
    assert (err > 1e-4 * np.maximum(np.abs(c).max(axis=-1), 1.0)).mean() <= 1e-2
    keep = err <= np.quantile(err, 0.99)
    assert np.linalg.norm((g - c)[keep]) / np.linalg.norm(c[keep]) <= 1e-3


@pytest.mark.parametrize("fixture", ["cornell_small", "spheres_small", "textured_wrappers_small"])
def test_device_built_bvh_gives_bit_identical_hits_and_films(fixture, request, gpu_renderer):
    """Row f4: the LBVH built on the GPU (csrc/device/bvh_build.cuh, option device_bvh) instead of the host's binned-SAH hierarchy.
    Closest hits do not depend on the hierarchy (boxes contain their triangles, ties in t go to the lower (instance, primitive)),
    so hit records equal the oracle's bit for bit and the film equals the film rendered with the host's hierarchy exactly."""
    scene = request.getfixturevalue(fixture)
    d = scene.desc()
    rays = _random_rays(scene, 100_000, seed=5)
    ref, _ = O.trace(d, rays)
    occ_ref, _ = O.trace(d, rays, any_hit=True)
    gpu_renderer.upload(d)
    gpu_renderer.clear()
    gpu_renderer.render(0, 4)
    film_host = gpu_renderer.film(raw=True).copy()
    try:
        gpu_renderer.set_option("device_bvh", 1)
        gpu_renderer.upload(d)
        got = gpu_renderer.trace(rays)
        assert np.array_equal(got["inst"], ref["inst"]) and np.array_equal(got["prim"], ref["prim"])
        assert np.array_equal(got["bary"].view(np.uint32), ref["bary"].view(np.uint32))
        occ = gpu_renderer.trace(rays, any_hit=True)
        assert np.array_equal(occ["inst"], occ_ref["inst"])
        gpu_renderer.clear()
        gpu_renderer.render(0, 4)
        assert np.array_equal(gpu_renderer.film(raw=True), film_host)
    finally:
        gpu_renderer.set_option("device_bvh", 0)


def test_device_built_bvh_full_size_scene(gpu_renderer):
    """BASELINE config C3's 1.39 M-triangle scene: the device build (five meshes, one of 327 680 triangles, 67 instances) against
    the oracle on random rays, and a 2-spp 480x270 film against the host-hierarchy film."""
    scene = Scene.from_source(scenes.instanced_spheres(resolution=(480, 270), spp=2), REPO)
    d = scene.desc()
    rays = _random_rays(scene, 50_000, seed=8)
    ref, _ = O.trace(d, rays)
    gpu_renderer.upload(d)
    gpu_renderer.clear()
    gpu_renderer.render(0, 2)
    film_host = gpu_renderer.film(raw=True).copy()
    try:
        gpu_renderer.set_option("device_bvh", 1)
        gpu_renderer.upload(d)
        got = gpu_renderer.trace(rays)
        assert np.array_equal(got["inst"], ref["inst"]) and np.array_equal(got["prim"], ref["prim"])
        assert np.array_equal(got["bary"].view(np.uint32), ref["bary"].view(np.uint32))
        gpu_renderer.clear()
        gpu_renderer.render(0, 2)
        assert np.array_equal(gpu_renderer.film(raw=True), film_host)
    finally:
        gpu_renderer.set_option("device_bvh", 0)


@pytest.mark.parametrize("kw", [{}, {"environment_medium": True, "rr_depth": 2}, {"skip_quirk": True}],
                         ids=["shape_media", "nested_in_environment_medium", "true_hit_quirk"])
def test_volume_with_shape_media_matches_oracle(kw, gpu_renderer):
    """Row a22 beyond config C4: media bound to Glass shells (medium tracker, surface events, transmittance walks through
    transmissive surfaces) on the per-thread volume kernel, against the oracle - which is bit-identical to the reference on
    these scenes (tests/test_ref_render.py).  Refraction chains amplify ulp-level libm differences into other discrete decisions
    for a few paths (as in the Glass scenes of the surface integrator): <= 3 % of the pixels may differ, the rest agree to 1e-3."""
    from luisarender_b200 import scenes

    scene = Scene.from_source(scenes.media_box(resolution=(96, 96), spp=8, **kw), REPO)
    d = scene.desc()
    gpu_renderer.upload(d)
    gpu_renderer.clear()
    gpu_renderer.render(0, 8)
    gpu_raw = gpu_renderer.film(raw=True)
    st = gpu_renderer.stats()
    cpu_raw, cnt = O.render(d, 0, 8)
    # An emitter hit after a medium event is evaluated from a ray origin that was moved ONTO the hit point (mega_vpt_naive.cpp:
    # 308,319): the vector to it is rounding noise, or exactly zero - then cos_wo is NaN and the film drops the sample
    # (color.cpp:110-113).  CUDA's and glibc's exp / log round the moved origin differently now and then, so with a medium around
    # the light a few samples per ten thousand are kept on one side and dropped on the other; without one the weights are exact.
    w_same = gpu_raw[..., 3] == cpu_raw[..., 3]
    assert w_same.all() if not kw.get("environment_medium") else w_same.mean() >= 0.995
    rel, off = _image_parity(gpu_raw, cpu_raw)
    assert off <= 3e-2, (rel, off)
    err = np.abs(gpu_raw[..., :3] - cpu_raw[..., :3]).max(axis=-1)
    keep = err <= np.quantile(err, 0.97)
    assert np.linalg.norm((gpu_raw[..., :3] - cpu_raw[..., :3])[keep]) / np.linalg.norm(cpu_raw[..., :3][keep]) <= 1e-3
    assert gpu_raw[..., :3].mean() == pytest.approx(cpu_raw[..., :3].mean(), rel=0.02)
    assert st["closest_rays"] == pytest.approx(cnt["closest_rays"], rel=5e-3)
    assert st["shadow_rays"] == pytest.approx(cnt["shadow_rays"], rel=5e-3)


def test_volume_with_thin_and_transmissive_disney_matches_oracle(gpu_renderer):
    """The three Disney closure classes inside an environment medium on the per-thread volume kernel: thin surfaces report "through"
    events (the medium tracker and the eta scale stay put), transmissive ones enter / exit.  The scene is the fixture
    tests/golden/ref_renders.npz: spheres_medium_disney_thin, on which the oracle is bit-identical to the reference renderer and the
    device code, compiled for the host, bit-identical to the oracle (tests/test_device_volume_on_host.py).  Tolerances as in
    test_volume_with_shape_media_matches_oracle (refraction chains, the moved-origin emitter hits)."""
    import sys

    sys.path.insert(0, str(REPO / "tools"))
    import gen_ref_renders as G

    scene = Scene.from_source(G.cases()["spheres_medium_disney_thin"].replace("resolution { 32, 18 }", "resolution { 96, 54 }"), REPO)
    d = scene.desc()
    assert d.camera.resolution[0] == 96
    gpu_renderer.upload(d)
    gpu_renderer.clear()
    gpu_renderer.render(0, 4)
    gpu_raw = gpu_renderer.film(raw=True)
    st = gpu_renderer.stats()
    cpu_raw, cnt = O.render(d, 0, 4)
    assert (gpu_raw[..., 3] == cpu_raw[..., 3]).mean() >= 0.995
    rel, off = _image_parity(gpu_raw, cpu_raw)
    assert off <= 3e-2, (rel, off)
    err = np.abs(gpu_raw[..., :3] - cpu_raw[..., :3]).max(axis=-1)
    keep = err <= np.quantile(err, 0.97)
    assert np.linalg.norm((gpu_raw[..., :3] - cpu_raw[..., :3])[keep]) / np.linalg.norm(cpu_raw[..., :3][keep]) <= 1e-3
    assert gpu_raw[..., :3].mean() == pytest.approx(cpu_raw[..., :3].mean(), rel=0.02)
    assert st["closest_rays"] == pytest.approx(cnt["closest_rays"], rel=5e-3)
    assert st["shadow_rays"] == pytest.approx(cnt["shadow_rays"], rel=5e-3)
