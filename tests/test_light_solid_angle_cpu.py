"""Solid-angle light sampling (option "light_solid_angle") without a GPU: csrc/device/spherical_triangle.h, the header the shade kernels
include, compiled for the host and checked on seeded random triangles and points - general, grazing, near a vertex, very close
(solid angle near 2 pi) and far (below the 3e-4 sr threshold, area sampling).  Also the option's surface in Python and on the
command line, and the near-light scene generators."""
from __future__ import annotations

import numpy as np
import pytest
from scipy import stats

from light_sampling_checks import (check_cli_flag, check_python_option, f32, lambert_irradiance, spherical,  # noqa: F401 (a fixture)
                                   unit)

EPS = float(np.finfo(f32).eps)


def omega64(p, v):
    """Van Oosterom & Strackee in float64 with unit vectors, as stated."""
    a = unit(np.asarray(v, np.float64) - np.asarray(p, np.float64)[:, None, :])
    num = np.abs(np.einsum("ij,ij->i", a[:, 0], np.cross(a[:, 1], a[:, 2])))
    den = 1.0 + (np.einsum("ij,ij->i", a[:, 0], a[:, 1]) + np.einsum("ij,ij->i", a[:, 1], a[:, 2]) + np.einsum("ij,ij->i", a[:, 2], a[:, 0]))
    return 2.0 * np.arctan2(num, den)


def triangles(rng, n):
    """Triangles in [-1, 1]^3 with every angle at least 15 degrees (slivers only add conditioning the cases below already cover)."""
    out = []
    while len(out) < n:
        v = rng.uniform(-1.0, 1.0, (4 * n, 3, 3))
        angles = []
        for i in range(3):
            a, b = v[:, (i + 1) % 3] - v[:, i], v[:, (i + 2) % 3] - v[:, i]
            angles.append(np.degrees(np.arccos(np.einsum("ij,ij->i", a, b) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1))))
        out.extend(v[(np.min(angles, axis=0) >= 15.0) & (np.linalg.norm(v[:, 1] - v[:, 0], axis=1) > 0.3)])
    return np.array(out[:n])


CASES = ["general", "grazing", "near_vertex", "very_close", "far"]


def case(name: str, n: int, seed: int):
    """(points, triangles) as float32 arrays [n, 3], [n, 3, 3]."""
    rng = np.random.default_rng(seed)
    v = triangles(rng, n)
    c = v.mean(axis=1)
    nrm = unit(np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]))
    side = np.where(rng.random(n) < 0.5, 1.0, -1.0)[:, None]
    if name == "general":  # 0.5 to 5 from the centroid, any direction
        p = c + unit(rng.normal(size=(n, 3))) * rng.uniform(0.5, 5.0, (n, 1))
    elif name == "grazing":  # 2 to 4 away in the plane, raised by 0.01 to 0.1 rad
        t = unit(np.cross(nrm, rng.normal(size=(n, 3))))
        el = rng.uniform(1e-2, 1e-1, (n, 1))
        p = c + rng.uniform(2.0, 4.0, (n, 1)) * (np.cos(el) * t + np.sin(el) * side * nrm)
    elif name == "near_vertex":  # 1e-3 from v0, at least 0.1 rad off the plane
        d = unit(rng.normal(size=(n, 3)))
        d = np.where(np.abs(np.einsum("ij,ij->i", d, nrm))[:, None] >= np.sin(0.1), d, unit(d + 0.5 * side * nrm))
        p = v[:, 0] + 1e-3 * d
    elif name == "very_close":  # 1e-3 to 1e-2 above an interior point: the solid angle approaches 2 pi
        b = rng.dirichlet([2.0, 2.0, 2.0], n)
        p = np.einsum("ij,ijk->ik", b, v) + side * rng.uniform(1e-3, 1e-2, (n, 1)) * nrm
    else:  # far: 1e3 to 1e4 away, below the spherical threshold
        p = c + unit(rng.normal(size=(n, 3))) * rng.uniform(1e3, 1e4, (n, 1))
    return np.ascontiguousarray(p, f32), np.ascontiguousarray(v, f32)


def solid_angle(spherical, p, v):
    out = np.zeros(len(p), f32)
    spherical.st_solid_angle(len(p), p.ctypes.data, v.ctypes.data, out.ctypes.data)
    return out


def sample(spherical, p, v, u):
    n = len(p)
    u = np.ascontiguousarray(u, f32)
    b, x, w = (np.zeros((n, 3), f32) for _ in range(3))
    pdf, sph = np.zeros(n, f32), np.zeros(n, np.int32)
    spherical.st_sample(n, p.ctypes.data, v.ctypes.data, u.ctypes.data, b.ctypes.data, x.ctypes.data, w.ctypes.data, pdf.ctypes.data, sph.ctypes.data)
    return b, x, w, pdf, sph.astype(bool)


def evaluated_pdf(spherical, p, v, x):
    pdf, sph = np.zeros(len(p), f32), np.zeros(len(p), np.int32)
    x = np.ascontiguousarray(x, f32)
    spherical.st_pdf(len(p), p.ctypes.data, v.ctypes.data, x.ctypes.data, pdf.ctypes.data, sph.ctypes.data)
    return pdf, sph.astype(bool)


# ---- the solid angle --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_solid_angle_matches_float64(spherical, name):
    """|omega - omega64| / omega64 <= 32 eps (1 + kappa), kappa = |v0 - p| |N| / |(v0 - p).N| the condition number of the triple
    product (1 / sin of p's elevation over the plane seen from v0).  Measured: at most a third of that bound."""
    p, v = case(name, 200_000, seed=CASES.index(name) + 1)
    got = solid_angle(spherical, p, v).astype(np.float64)
    want = omega64(p, v)
    P, V = p.astype(np.float64), v.astype(np.float64)
    n = np.cross(V[:, 1] - V[:, 0], V[:, 2] - V[:, 0])
    d0 = V[:, 0] - P
    kappa = np.linalg.norm(d0, axis=1) * np.linalg.norm(n, axis=1) / np.abs(np.einsum("ij,ij->i", d0, n))
    rel = np.abs(got - want) / want
    assert (rel <= 32 * EPS * (1.0 + kappa)).all(), rel.max()
    in_rule = (want >= 3e-4) & (want <= 6.22)
    if name == "far":
        assert not in_rule.any()
    else:
        assert in_rule.mean() > 0.5


def test_rule_bounds(spherical):
    omega = np.array([0.0, 2.9e-4, 3e-4, 1.0, 6.22, 6.2201, 2 * np.pi, np.nan], f32)
    out = np.zeros(len(omega), np.int32)
    spherical.st_use_spherical(len(omega), omega.ctypes.data, out.ctypes.data)
    assert out.tolist() == [0, 0, 1, 1, 1, 0, 0, 0]


# ---- the sampler ------------------------------------------------------------------------------------------------------------------
# angle between the sampled direction and the direction to the point it produces, times |cos| of the direction at the triangle
# (the intersection with the plane loses precision as 1 / cos).  Measured maxima over 2 x 10^5 samples: 2e-5 (general, grazing),
# 3e-4 (very close, where the construction nears a hemisphere), 7e-4 (near a vertex, 1e-3 away).
DIRECTION_BOUND = {"general": 1e-4, "grazing": 1e-4, "near_vertex": 2e-3, "very_close": 2e-3, "far": 0.0}


@pytest.mark.parametrize("name", CASES)
def test_samples_are_points_of_the_triangle_in_the_sampled_direction(spherical, name):
    p, v = case(name, 200_000, seed=10 + CASES.index(name))
    b, x, w, _, sph = sample(spherical, p, v, np.random.default_rng(20).random((len(p), 2)))
    assert not np.isnan(b).any()
    assert (b >= 0).all() and (b <= 1).all()
    assert np.abs(b.astype(np.float64).sum(axis=1) - 1.0).max() <= 2 * EPS
    if name == "far":
        assert not sph.any()
        return
    assert sph.mean() > 0.5
    P, V, X, W = (a[sph].astype(np.float64) for a in (p, v, x, w))
    W = unit(W)
    angle = np.arccos(np.clip(np.einsum("ij,ij->i", unit(X - P), W), -1.0, 1.0))
    cos_x = np.abs(np.einsum("ij,ij->i", W, unit(np.cross(V[:, 1] - V[:, 0], V[:, 2] - V[:, 0]))))
    assert (angle * cos_x).max() <= DIRECTION_BOUND[name], (angle * cos_x).max()


@pytest.mark.parametrize("name", CASES)
def test_sampled_pdf_is_the_evaluated_pdf(spherical, name):
    """The pdf a sample returns and the pdf an emitter hit at the same point evaluates, bit for bit, with the same rule."""
    p, v = case(name, 100_000, seed=30 + CASES.index(name))
    _, x, _, pdf, sph = sample(spherical, p, v, np.random.default_rng(31).random((len(p), 2)))
    ev_pdf, ev_sph = evaluated_pdf(spherical, p, v, x)
    assert np.array_equal(sph, ev_sph)
    assert np.array_equal(pdf.view(np.uint32), ev_pdf.view(np.uint32))
    omega = solid_angle(spherical, p, v)
    assert np.array_equal(pdf[sph], (f32(1.0) / omega[sph]))


def cells(v, n):
    """The n^2 triangles of the regular barycentric subdivision of triangle v (float64 [3, 3]), and a table from (i, j, upper) -
    the lower or upper triangle of grid square (i, j) - to the index of each."""
    def at(a, c):
        return v[0] + (a / n) * (v[1] - v[0]) + (c / n) * (v[2] - v[0])
    tris, index = [], np.full((n, n, 2), -1)
    for i in range(n):
        for j in range(n - i):
            index[i, j, 0] = len(tris)
            tris.append((at(i, j), at(i + 1, j), at(i, j + 1)))
            if i + j < n - 1:
                index[i, j, 1] = len(tris)
                tris.append((at(i + 1, j), at(i + 1, j + 1), at(i, j + 1)))
    return np.array(tris), index


def cell_of(b, n, index):
    s, t = b[:, 1].astype(np.float64) * n, b[:, 2].astype(np.float64) * n
    i = np.minimum(np.floor(s), n - 1).astype(int)
    j = np.minimum(np.floor(t), n - 1 - i).astype(int)  # a point on the far edge belongs to the last cell of its row
    upper = ((s - i) + (t - j) > 1.0) & (i + j < n - 1)
    return index[i, j, upper.astype(int)]


CHI_CASES = [  # (point, triangle): the spherical sampler at its two ends and between
    ("close", (0.1, 0.2, 0.05), ((-1.0, -1.0, 0.0), (1.2, -0.8, 0.0), (0.1, 1.1, 0.0))),
    ("moderate", (0.3, 0.2, 1.5), ((-1.0, -1.0, 0.0), (1.2, -0.8, 0.0), (0.1, 1.1, 0.0))),
    ("grazing", (3.0, 0.5, 0.15), ((-1.0, -1.0, 0.0), (1.2, -0.8, 0.0), (0.1, 1.1, 0.0))),
    ("near_vertex", (-0.999, -0.9995, 0.001), ((-1.0, -1.0, 0.0), (1.2, -0.8, 0.0), (0.1, 1.1, 0.0))),
    ("small", (0.0, 0.0, 60.0), ((-1.0, -1.0, 0.0), (1.2, -0.8, 0.0), (0.1, 1.1, 0.0))),
]


@pytest.mark.parametrize("name, p0, tri", CHI_CASES, ids=[c[0] for c in CHI_CASES])
def test_samples_are_uniform_in_solid_angle(spherical, name, p0, tri):
    """Chi-square of 10^6 draws over the 64 cells of the triangle's regular subdivision, expected counts in proportion to the cells'
    float64 solid angles; fails at p < 1e-4."""
    draws, n = 1_000_000, 8
    p = np.ascontiguousarray(np.repeat(np.array([p0], f32), draws, axis=0))
    v = np.ascontiguousarray(np.repeat(np.array([tri], f32), draws, axis=0))
    b, _, _, _, sph = sample(spherical, p, v, np.random.default_rng(40).random((draws, 2)))
    assert sph.all()
    sub, index = cells(np.array(tri, f32).astype(np.float64), n)
    expected = omega64(np.repeat(np.array([p0], f32).astype(np.float64), len(sub), axis=0), sub)
    expected = expected / expected.sum() * draws
    counts = np.bincount(cell_of(b, n, index), minlength=len(sub)).astype(np.float64)
    assert len(counts) == len(sub)
    big = expected >= 5
    obs = np.append(counts[big], counts[~big].sum())
    exp = np.append(expected[big], expected[~big].sum())
    keep = exp > 0
    assert stats.chisquare(obs[keep], exp[keep]).pvalue > 1e-4


IRRADIANCE_CASES = [  # receiver point and normal under a triangle: close and large, moderate, tilted, far (area sampling)
    ((0.1, 0.0, 0.0), (0.0, 0.0, 1.0), ((-1.0, -1.0, 0.3), (1.2, -0.8, 0.3), (0.1, 1.1, 0.3))),
    ((0.0, 0.0, 0.0), (0.0, 0.0, 1.0), ((-1.0, -1.0, 2.0), (1.2, -0.8, 2.0), (0.1, 1.1, 2.0))),
    ((0.5, 0.0, 0.0), (0.6, 0.0, 0.8), ((-1.0, -1.0, 1.0), (1.2, -0.8, 0.6), (0.1, 1.1, 1.5))),
    ((0.0, 0.0, 0.0), (0.0, 0.0, 1.0), ((-1.0, -1.0, 150.0), (1.2, -0.8, 150.0), (0.1, 1.1, 150.0))),
]


@pytest.mark.parametrize("p0, n0, tri", IRRADIANCE_CASES)
def test_irradiance_estimate_matches_lambert(spherical, p0, n0, tri):
    """The mean of L cos(theta) / pdf over 10^6 samples against Lambert's polygon irradiance, within 4 sigma."""
    draws = 1_000_000
    p = np.ascontiguousarray(np.repeat(np.array([p0], f32), draws, axis=0))
    v = np.ascontiguousarray(np.repeat(np.array([tri], f32), draws, axis=0))
    _, x, _, pdf, sph = sample(spherical, p, v, np.random.default_rng(50).random((draws, 2)))
    wi = unit(x.astype(np.float64) - np.array(p0, np.float64))
    f = np.maximum(wi @ np.array(n0, np.float64), 0.0) / pdf.astype(np.float64)
    want = lambert_irradiance(p0, n0, tri)
    se = f.std(ddof=1) / np.sqrt(draws)
    assert abs(f.mean() - want) <= 4.0 * se + 1e-6 * want, (f.mean(), want, se, sph.mean())


def test_spherical_sampling_is_quieter_close_to_a_large_light(spherical):
    p0, n0, tri = IRRADIANCE_CASES[0]
    draws = 100_000
    p = np.ascontiguousarray(np.repeat(np.array([p0], f32), draws, axis=0))
    v = np.ascontiguousarray(np.repeat(np.array([tri], f32), draws, axis=0))
    u = np.random.default_rng(51).random((draws, 2))
    _, x, _, pdf, sph = sample(spherical, p, v, u)
    assert sph.all()
    wi = unit(x.astype(np.float64) - np.array(p0, np.float64))
    solid = np.maximum(wi @ np.array(n0, np.float64), 0.0) / pdf
    # area sampling of the same triangle from the same point: the pdf d^2 / (A cos_l)
    b = np.empty((draws, 3))
    lo = u[:, 0] < u[:, 1]
    b[:, 0] = np.where(lo, 0.5 * u[:, 0], -0.5 * u[:, 1] + u[:, 0])
    b[:, 1] = np.where(lo, -0.5 * u[:, 0] + u[:, 1], 0.5 * u[:, 1])
    b[:, 2] = 1.0 - b[:, 0] - b[:, 1]
    V = np.array(tri, np.float64)
    xa = b @ V
    d = xa - np.array(p0)
    nl = np.cross(V[1] - V[0], V[2] - V[0])
    area = 0.5 * np.linalg.norm(nl)
    cos_l = np.abs(unit(d) @ (nl / np.linalg.norm(nl)))
    area_est = np.maximum(unit(d) @ np.array(n0), 0.0) * area * cos_l / (d * d).sum(axis=1)
    assert solid.var() < 0.5 * area_est.var()


# ---- the option's surface ---------------------------------------------------------------------------------------------------------
def test_python_option_rejects_unknown_values():
    check_python_option("light_solid_angle")


def test_cli_lists_and_parses_light_solid_angle(tmp_path):
    check_cli_flag("light_solid_angle", tmp_path)


# ---- the scene generators ---------------------------------------------------------------------------------------------------------
def test_near_light_scene_generators():
    from luisarender_b200 import scenes

    room = scenes.near_light(resolution=(32, 18))
    assert room.count("Light ") == 1 and "two_sided { false }" in room and "Matte" in room
    plane = scenes.near_light(resolution=(32, 18), irradiance=True)
    assert plane.count("Light ") == 1 and "depth { 2 }" in plane
