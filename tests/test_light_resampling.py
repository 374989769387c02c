"""Resampled next-event estimation on the GPU (option "light_candidates"; include/lrk.h, csrc/device/light_resampling.h).

Values 0 and 1 must change nothing; M >= 2 must render the same image as one light sample within its noise on every kind of frame
and light sampling, match Lambert's formula on the irradiance frame, lower the noise of the glossy-desk frame, and compose with
scheduling, sharding, the G-buffer mode and the adaptive mode unchanged.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

from light_sampling_checks import (SUB_SPP, SUBRENDERS, Z_MAX, bits, block_means, r, reference, rel_mse, render,  # noqa: F401
                                   sub_renders, z_scores)

REPO = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu
SINGLE = {"light_candidates": 0}


def candidates(m):
    return {"light_candidates": m}


@pytest.fixture
def rc(r):
    """The shared light-sampling fixture r, with "light_candidates" back at 0 afterwards too."""
    yield r
    r.set_option("light_candidates", 0)


def _scene(src):
    from luisarender_b200.api import Scene

    return Scene.from_source(src, REPO)


@pytest.fixture(scope="module")
def frames():
    """Scene sources by name, parsed on first use."""
    from luisarender_b200 import scenes

    sources = {
        "cornell": lambda: scenes.cornell_box(resolution=(64, 64), spp=16),
        "textured_lamp": lambda: scenes.textured_room(resolution=(96, 64), spp=8, textured_light=True),
        "environment_area": lambda: scenes.environment_scene(resolution=(64, 48), spp=4, area_light=True),
        "flatten": lambda: scenes.flatten_stress(resolution=(64, 48), spp=4),
        "many": lambda: scenes.many_lights(resolution=(128, 72), spp=16, count=48, big_subdivision=3, small_subdivision=2),
        "materials": lambda: scenes.materials_box(resolution=(64, 48), spp=4, mix=True),
        "layered": lambda: scenes.layered_box(resolution=(64, 48), spp=4),
        "sobol_cornell": lambda: scenes.cornell_box(resolution=(64, 64), spp=1024).replace("sampler : Independent", "sampler : PaddedSobol"),
        "near": lambda: scenes.near_light(resolution=(96, 96), spp=16),
        "glossy_desk": lambda: scenes.near_light(resolution=(96, 96), spp=16, glossy_desk=True),
        "irradiance": lambda: scenes.near_light(resolution=(64, 64), spp=16, irradiance=True),
        "medium_small": lambda: scenes.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3,
                                                         small_subdivision=2, small_count=12),
    }
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _scene(sources[name]())
        return cache[name]

    return get


# ---- 1. values 0 and 1 change nothing ---------------------------------------------------------------------------------------------
def test_values_zero_and_one_equal_a_context_that_never_set_the_option(frames, rc):
    from luisarender_b200.api import Renderer

    d = frames("cornell").desc()
    fresh = Renderer(device_index=0)
    try:
        fresh.set_option("strict_math", 0 if rc.fast else 1)
        fresh.upload(d)
        fresh.render(0, 4)
        want, want_launches = fresh.film(raw=True), fresh.stats()["kernel_launches"]
    finally:
        fresh.close()
    render(rc, d, 0, 4, candidates(4))  # leaves the resampling kernels behind in this context
    for m in (0, 1):
        got = render(rc, d, 0, 4, candidates(m))
        assert np.array_equal(bits(got), bits(want)), m
        assert rc.stats()["kernel_launches"] == want_launches


# ---- 2. unbiased: the same image as one light sample ------------------------------------------------------------------------------
CASES = [  # (id, frame, other light-sampling options, M)
    ("cornell", "cornell", {}, 4),
    ("textured_lamp", "textured_lamp", {}, 4),
    ("environment_area", "environment_area", {}, 4),
    ("flatten", "flatten", {}, 4),
    ("many_tree", "many", {"light_tree": 1}, 4),
    ("many_tree_triangles", "many", {"light_tree": 1, "light_tree_triangles": 1}, 4),
    ("many_solid_angle", "many", {"light_solid_angle": 1}, 4),
    ("materials_mix", "materials", {}, 4),
    ("layered", "layered", {}, 4),
    ("padded_sobol", "sobol_cornell", {}, 4),
    ("cornell_m32", "cornell", {}, 32),
]


@pytest.mark.parametrize("frame, options, m", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_resampling_agrees_with_one_light_sample(frames, rc, frame, options, m):
    d = frames(frame).desc()
    single = sub_renders(rc, d, {**options, **SINGLE}, 0, SUBRENDERS, SUB_SPP)
    resampled = sub_renders(rc, d, {**options, **candidates(m)}, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)  # disjoint sample indices
    assert not np.array_equal(single.mean(axis=0), resampled.mean(axis=0))
    z = z_scores(resampled, single)
    assert np.abs(z).max() < Z_MAX, z


# ---- 3. the irradiance frame against Lambert's formula ----------------------------------------------------------------------------
def lambert_irradiance(x, tri):
    """Irradiance at plane points x [n, 3] (normal +y) from a triangle of unit radiance wholly above the plane: E = 1/2 sum_i
    theta_i (n . g_i), g_i the unit normal of the plane through x and edge i."""
    a = np.asarray(tri, np.float64)[None, :, :] - x[:, None, :]
    a /= np.linalg.norm(a, axis=2, keepdims=True)
    e = np.zeros(len(x))
    for i in range(3):
        g = np.cross(a[:, i], a[:, (i + 1) % 3])
        gl = np.linalg.norm(g, axis=1)
        theta = np.arctan2(gl, np.einsum("ij,ij->i", a[:, i], a[:, (i + 1) % 3]))
        e += theta * g[:, 1] / gl
    return 0.5 * np.abs(e)


def analytic_irradiance_film(desc, sub=4):
    """(albedo / pi) * L * E of near_light(irradiance=True) per pixel, averaged over sub x sub points of the pixel's box footprint:
    the pinhole looks straight down at the plane, to which its image plane is parallel."""
    from luisarender_b200 import scenes

    src = scenes.near_light(irradiance=True)
    tri = [(-0.9, 0.5, 0.8), (-0.7, 0.5, -1.0), (1.1, 0.5, 0.1)]
    assert all(", ".join(repr(float(c)) for c in v) in src for v in tri)
    cam = desc.camera
    rx, ry = cam.resolution[0], cam.resolution[1]
    m = np.array(cam.camera_to_world, np.float64).reshape(3, 4)
    k = cam.tan_half_fov / ry
    f = (np.arange(sub) + 0.5) / sub
    px = (np.arange(rx)[:, None] + f[None, :]).reshape(-1)
    py = (np.arange(ry)[:, None] + f[None, :]).reshape(-1)
    gx, gy = np.meshgrid(px, py)
    local = np.stack([(gx * 2 - rx) * k, -(gy * 2 - ry) * k, -np.ones_like(gx)], axis=-1)
    d = local @ m[:, :3].T
    o = m[:, 3]
    t = -o[1] / d[..., 1]
    x = o + t[..., None] * d
    e = lambert_irradiance(x.reshape(-1, 3), tri).reshape(ry, sub, rx, sub).mean(axis=(1, 3))
    return 0.5 / np.pi * 4.0 * e


def test_irradiance_frame_matches_lambert(frames, rc):
    d = frames("irradiance").desc()
    films = sub_renders(rc, d, candidates(8), 0, SUBRENDERS, SUB_SPP)
    want = analytic_irradiance_film(d)
    m = block_means(films)
    w = block_means(np.repeat(want[None, :, :, None], 3, axis=3))[0]
    se = m.std(axis=0, ddof=1) / np.sqrt(len(m))
    assert (se > 0).all()
    z = (m.mean(axis=0) - w) / se
    assert np.abs(z).max() < Z_MAX, z


# ---- 4. less noise where the closure decides which light samples matter -----------------------------------------------------------
# The 16-spp relative MSE at M = 8 over that at M = 1 on the 96x96 glossy-desk frame, each averaged over 8 renders.  Measured on an
# NVIDIA H100 80GB HBM3 (700 W power limit): 0.9556 in the fast and 0.9561 in the strict arithmetic mode (DESIGN.md §5).  The renders
# are seeded, so the bound's margin is for changes of the code around the estimator, not for chance.
GLOSSY_DESK_ERROR_RATIO = 0.98


def test_glossy_desk_error_is_lower(frames, rc):
    d = frames("glossy_desk").desc()
    ref = reference(rc, d, candidates(8))
    one, eight = rel_mse(rc, d, SINGLE, ref, 0), rel_mse(rc, d, candidates(8), ref, 4096)
    print(f"glossy_desk 16 spp rel. MSE: M=1 {one:.4e}, M=8 {eight:.4e}, ratio {eight / one:.4f} (fast={rc.fast})")
    assert eight <= GLOSSY_DESK_ERROR_RATIO * one, (eight, one, eight / one)


# ---- 5. scheduling and sharding ---------------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(frames, rc):
    d = frames("glossy_desk").desc()
    whole = render(rc, d, 0, 8, candidates(4))
    rc.clear()
    rc.render(0, 3)
    rc.render(3, 8)
    assert np.array_equal(bits(rc.film(raw=True)), bits(whole))
    rc.set_option("max_paths_per_pass", 1024)
    rc.clear()
    rc.render(0, 8)
    assert np.array_equal(bits(rc.film(raw=True)), bits(whole))
    rc.set_option("max_paths_per_pass", 136 << 20)
    total = np.zeros_like(whole)
    for rank in range(3):
        rc.upload(d)
        rc.balance_shards(rank, 3, 32, 1)  # the cost probe runs the resampling kernels too
        rc.render(0, 8)
        part = rc.film(raw=True)
        assert not np.any((total != 0) & (part != 0))  # every pixel has one owner
        total += part
    assert np.array_equal(bits(total), bits(whole))


# ---- 6. the other modes -----------------------------------------------------------------------------------------------------------
def test_gbuffer_and_adaptive_compose(frames, rc):
    d = frames("glossy_desk").desc()
    rc.set_option("gbuffer", 1)
    off = render(rc, d, 0, 4, SINGLE)
    gb_off = rc.gbuffer()
    on = render(rc, d, 0, 4, candidates(4))
    gb_on = rc.gbuffer()
    assert not np.array_equal(bits(on), bits(off))  # the option changes the film ...
    for a, b in zip(gb_on[:2], gb_off[:2]):  # ... not the first-hit guides (the third, the luminance variance, follows the film)
        assert np.array_equal(bits(a), bits(b))
    rc.set_option("gbuffer", 0)
    uniform = render(rc, d, 0, 8, candidates(4))
    rc.render_adaptive(0.0, 4, 8)
    assert np.array_equal(bits(rc.film(raw=True)), bits(uniform))


# ---- 7. errors --------------------------------------------------------------------------------------------------------------------
def test_volume_integrator_and_bad_values_are_refused(frames, rc):
    d = frames("medium_small").desc()
    before = render(rc, d, 0, 2, SINGLE)
    rc.set_option("light_candidates", 2)
    with pytest.raises(RuntimeError, match=r"lrk_upload_scene failed \(-5\): .*light_candidates"):
        rc.upload(d)
    for bad in (-1, 33):
        with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
            rc.set_option("light_candidates", bad)
    assert np.array_equal(bits(render(rc, d, 0, 2, SINGLE)), bits(before))
