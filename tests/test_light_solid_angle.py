"""Solid-angle light sampling on the GPU (option "light_solid_angle"; include/lrk.h, csrc/device/spherical_triangle.h).

Off, the option must change nothing; on, every frame must render the same image as area sampling within its noise, the irradiance
frame must match Lambert's formula, the near-light frame must have less noise, and scheduling, sharding, the G-buffer mode and
the adaptive mode must compose with it unchanged.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

from light_sampling_checks import (SUB_SPP, SUBRENDERS, Z_MAX, bits, block_means, r, reference, rel_mse, render,  # noqa: F401
                                   sub_renders, z_scores)

REPO = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu
AREA, SOLID_ANGLE = {"light_solid_angle": 0}, {"light_solid_angle": 1}


def _scene(src):
    from luisarender_b200.api import Scene

    return Scene.from_source(src, REPO)


@pytest.fixture(scope="module")
def cornell():
    from luisarender_b200 import scenes

    return _scene(scenes.cornell_box(resolution=(64, 64), spp=16))


@pytest.fixture(scope="module")
def textured_lamp():
    from luisarender_b200 import scenes

    return _scene(scenes.textured_room(resolution=(96, 64), spp=8, textured_light=True))


@pytest.fixture(scope="module")
def environment_area():
    from luisarender_b200 import scenes

    return _scene(scenes.environment_scene(resolution=(64, 48), spp=4, area_light=True))


@pytest.fixture(scope="module")
def flatten():
    from luisarender_b200 import scenes

    return _scene(scenes.flatten_stress(resolution=(64, 48), spp=4))


@pytest.fixture(scope="module")
def many():
    from luisarender_b200 import scenes

    return _scene(scenes.many_lights(resolution=(128, 72), spp=16, count=48, big_subdivision=3, small_subdivision=2))


@pytest.fixture(scope="module")
def near():
    from luisarender_b200 import scenes

    return _scene(scenes.near_light(resolution=(96, 96), spp=16))


@pytest.fixture(scope="module")
def irradiance():
    from luisarender_b200 import scenes

    return _scene(scenes.near_light(resolution=(64, 64), spp=16, irradiance=True))


@pytest.fixture(scope="module")
def medium_small():
    from luisarender_b200 import scenes

    return _scene(scenes.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3, small_subdivision=2,
                                           small_count=12))


# ---- 1. off changes nothing -------------------------------------------------------------------------------------------------------
def test_option_off_equals_a_context_that_never_set_it(cornell, r):
    from luisarender_b200.api import Renderer

    fresh = Renderer(device_index=0)
    try:
        fresh.set_option("strict_math", 0 if r.fast else 1)
        fresh.upload(cornell.desc())
        fresh.render(0, 4)
        want, want_launches = fresh.film(raw=True), fresh.stats()["kernel_launches"]
    finally:
        fresh.close()
    render(r, cornell.desc(), 0, 4, SOLID_ANGLE)  # leaves the option's kernels behind in this context
    got = render(r, cornell.desc(), 0, 4, AREA)
    assert np.array_equal(bits(got), bits(want))
    assert r.stats()["kernel_launches"] == want_launches


# ---- 2. unbiased: the same image as area sampling ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cornell", "textured_lamp", "environment_area", "flatten", "many"])
def test_solid_angle_agrees_with_area_sampling(request, name, r):
    d = request.getfixturevalue(name).desc()
    if name == "many":
        r.set_option("light_tree", 1)  # both choices of next-event estimation at once
    area = sub_renders(r, d, AREA, 0, SUBRENDERS, SUB_SPP)
    solid = sub_renders(r, d, SOLID_ANGLE, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)  # disjoint sample indices
    assert not np.array_equal(area.mean(axis=0), solid.mean(axis=0))
    z = z_scores(solid, area)
    assert np.abs(z).max() < Z_MAX, z


# ---- 3. the irradiance frame against Lambert's formula ----------------------------------------------------------------------------
def lambert_irradiance(x, tri):
    """Irradiance at plane points x [n, 3] (normal +y) from a triangle of unit radiance wholly above the plane."""
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
    """(albedo / pi) * L * E of the irradiance frame per pixel, averaged over sub x sub points of the pixel's box footprint: the
    pinhole of pathcommon.cuh's camera_ray looks straight down at the plane, to which its image plane is parallel."""
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
    gx, gy = np.meshgrid(px, py)  # [ry * sub, rx * sub]
    local = np.stack([(gx * 2 - rx) * k, -(gy * 2 - ry) * k, -np.ones_like(gx)], axis=-1)
    d = local @ m[:, :3].T
    o = m[:, 3]
    t = -o[1] / d[..., 1]
    x = o + t[..., None] * d
    e = lambert_irradiance(x.reshape(-1, 3), tri).reshape(ry, sub, rx, sub).mean(axis=(1, 3))
    return 0.5 / np.pi * 4.0 * e


@pytest.mark.parametrize("solid_angle", [False, True])
def test_irradiance_frame_matches_lambert(irradiance, r, solid_angle):
    d = irradiance.desc()
    films = sub_renders(r, d, {"light_solid_angle": solid_angle}, 0, SUBRENDERS, SUB_SPP)
    want = analytic_irradiance_film(d)
    m = block_means(films)
    w = block_means(np.repeat(want[None, :, :, None], 3, axis=3))[0]
    se = m.std(axis=0, ddof=1) / np.sqrt(len(m))
    assert (se > 0).all()
    z = (m.mean(axis=0) - w) / se
    assert np.abs(z).max() < Z_MAX, z


# ---- 4. less noise where the light is large and close -----------------------------------------------------------------------------
# The 16-spp relative MSE of the option over that of area sampling on the 96x96 near-light frame, each averaged over 8 renders.
# Measured on an H100: 0.707 in both arithmetic modes (DESIGN.md §5).  The renders are seeded, so the bound's margin is for changes
# of the code around the sampler, not for chance.
NEAR_LIGHT_ERROR_RATIO = 0.8


def test_near_light_error_is_lower(near, r):
    d = near.desc()
    ref = reference(r, d, SOLID_ANGLE)
    area, solid = rel_mse(r, d, AREA, ref, 0), rel_mse(r, d, SOLID_ANGLE, ref, 4096)
    print(f"near_light 16 spp rel. MSE: area {area:.4e}, solid angle {solid:.4e}, ratio {solid / area:.4f} (fast={r.fast})")
    assert solid <= NEAR_LIGHT_ERROR_RATIO * area, (solid, area, solid / area)


# ---- 5. scheduling and the other modes --------------------------------------------------------------------------------------------
def test_scheduling_and_sharding_change_no_bit(near, r):
    d = near.desc()
    whole = render(r, d, 0, 8, SOLID_ANGLE)
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
        r.balance_shards(rank, 3, 32, 1)  # the cost probe runs the option's kernels too
        r.render(0, 8)
        part = r.film(raw=True)
        assert not np.any((total != 0) & (part != 0))  # every pixel has one owner
        total += part
    assert np.array_equal(bits(total), bits(whole))


def test_gbuffer_and_adaptive_compose(near, r):
    d = near.desc()
    r.set_option("gbuffer", 1)
    off = render(r, d, 0, 4, AREA)
    gb_off = r.gbuffer()
    on = render(r, d, 0, 4, SOLID_ANGLE)
    gb_on = r.gbuffer()
    assert not np.array_equal(bits(on), bits(off))  # the option changes the film ...
    for a, b in zip(gb_on[:2], gb_off[:2]):  # ... not the first-hit guides (the third, the luminance variance, follows the film)
        assert np.array_equal(bits(a), bits(b))
    r.set_option("gbuffer", 0)
    uniform = render(r, d, 0, 8, SOLID_ANGLE)
    r.render_adaptive(0.0, 4, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(uniform))


# ---- 6. errors --------------------------------------------------------------------------------------------------------------------
def test_volume_integrator_and_bad_values_are_refused(medium_small, r):
    d = medium_small.desc()
    before = render(r, d, 0, 2, AREA)
    r.set_option("light_solid_angle", 1)
    with pytest.raises(RuntimeError, match=r"lrk_upload_scene failed \(-5\): .*solid-angle"):
        r.upload(d)
    with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
        r.set_option("light_solid_angle", 2)
    assert np.array_equal(bits(render(r, d, 0, 2, AREA)), bits(before))
