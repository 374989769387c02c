"""Receiver-aware light sampling (option "light_receiver") without a GPU: csrc/device/receiver.h (the receiver word), the receiver term
of light_tree.h and the receiver-cosine warp of spherical_triangle.h, compiled for the host and checked on seeded normals, the light
sets and meshes of light_sampling_checks.py and random triangles.  Also the one-sided bit of each closure kind and the option's
surface in Python and on the command line."""
from __future__ import annotations

import ctypes as C
import hashlib

import numpy as np
import pytest
from scipy import stats

import host_harness
from light_sampling_checks import (NONE, Bottom, LightSet, check_cli_flag, check_python_option, decode, encode, f32, icosphere,  # noqa: F401
                                   lambert_irradiance, lib, spherical, unit)

ONE_SIDED_KINDS = {1, 2, 3, 5, 6}  # Matte, Disney, Mirror, Plastic, Metal (hit_kinds.h)


# ---- the word ---------------------------------------------------------------------------------------------------------------------
def test_encoding_round_trip(lib):
    """Within 2e-4 rad of the normal (measured: 1.3e-4), the one-sided bit kept, the word never 0; the word 0 decodes to no receiver."""
    rng = np.random.default_rng(1)
    n = unit(rng.normal(size=(200_000, 3)))
    n[:6] = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]])
    side = rng.random(len(n)) < 0.5
    words = encode(lib, n * rng.uniform(0.1, 10.0, (len(n), 1)), side)  # the length does not matter
    assert (words != 0).all()
    d, kind = decode(lib, words)
    d = d.astype(np.float64)
    ang = np.arctan2(np.linalg.norm(np.cross(d, n), axis=1), np.einsum("ij,ij->i", d, n))
    assert ang.max() < 2e-4, ang.max()
    assert (kind == np.where(side, 2, 1)).all()
    d0, k0 = decode(lib, np.zeros(1, np.uint32))
    assert k0[0] == 0 and (d0 == 0).all()


# ---- the tree -----------------------------------------------------------------------------------------------------------------------
SETS = [(2, 11), (7, 12), (1000, 13)]


@pytest.mark.parametrize("n,seed", SETS)
def test_tree_pmfs_with_receivers(lib, n, seed):
    """For one-sided, two-sided and no receivers: sum of pmfs + P(no light) = 1, sampled pmf = evaluated pmf bit for bit, a
    two-sided receiver culls nothing the tree without a receiver keeps, and the word 0 gives the pmfs of the tree without a receiver."""
    ls = LightSet(n, seed)
    tree = ls.build(lib)
    m = 64 if n == 1000 else 400
    pts = ls.points(m, seed + 100)
    rng = np.random.default_rng(seed)
    normals = unit(rng.normal(size=(m, 3)))
    base = tree.pmfs(pts, np.zeros(m, np.uint32))
    for one_sided in (False, True):
        words = encode(lib, normals, one_sided)
        p = tree.pmfs(pts, words)
        assert np.abs(p.astype(np.float64).sum(0) + tree.dead_mass(pts, words) - 1.0).max() < 1e-5
        if not one_sided:
            assert ((base > 0) <= (p > 0)).all()
        for u in rng.random((8, m)):
            light, pmf = tree.sample(pts, u, words)
            ok = light != NONE
            assert (pmf[~ok] == 0).all()
            assert (pmf[ok].view(np.uint32) == p[light[ok], np.nonzero(ok)[0]].view(np.uint32)).all()
    # the word 0 is the tree without a receiver, which is what test_light_tree_cpu.py checks
    light, pmf = tree.sample(pts, rng.random(m), np.zeros(m, np.uint32))
    ok = light != NONE
    assert (pmf[ok].view(np.uint32) == base[light[ok], np.nonzero(ok)[0]].view(np.uint32)).all()


def test_tree_culls_only_lights_behind_a_one_sided_receiver(lib):
    """Small two-sided emitters around a receiver at the origin with normal +z: those wholly below its plane by more than the pad get
    pmf 0, those above it by a margin keep pmf > 0 (two-sided emitters: the cone never culls them)."""
    rng = np.random.default_rng(5)
    n = 300
    ls = LightSet(1, 0)
    ls.tris, ls.power, ls.two_sided = [], [], []
    centres = unit(rng.normal(size=(n, 3))) * rng.uniform(2.0, 6.0, (n, 1))
    for c in centres:
        s = 0.05
        ls.tris.append(np.array([[c + [-s, -s, 0], c + [s, -s, 0], c + [s, s, 0]], [c + [-s, -s, 0], c + [s, s, 0], c + [-s, s, 0]]]))
        ls.power.append(1.0)
        ls.two_sided.append(1)
    ls.n = n
    tree = ls.build(lib)
    pts = np.zeros((1, 3), f32)
    p = tree.pmfs(pts, encode(lib, [[0.0, 0.0, 1.0]], True))[:, 0]
    elev = np.arcsin(centres[:, 2] / np.linalg.norm(centres, axis=1))
    radius = 0.1 / np.linalg.norm(centres, axis=1)  # angular radius of each emitter's bounds, padded
    assert (p[elev > radius + 0.05] > 0).all()
    assert (p[elev < -0.2] == 0).all()
    assert (elev < -0.2).sum() > 50
    two = tree.pmfs(pts, encode(lib, [[0.0, 0.0, 1.0]], False))[:, 0]
    assert (two > 0).all()


# SHA-256 of the float32 pmfs [emitter, point] of LightSet(n, seed=n) at LightSet.points(64, n + 7), and of the bottom trees of the
# level-3 icosphere at 32 seeded points per transform, computed with the parent commit's light_tree.h (through light_tree_host.cpp):
# the queries without words (a null word array) must give these bytes, and the word 0 the same.
PARENT_TOP_PMF_SHA256 = {2: "255860b266726efb54cfcedd5005e73890959970698710666b3f3ead5a14dd2d",
                         7: "c41d047eb665814970fa5826533174017f71b898715a007410c63698243f5f77",
                         1000: "23bf362820d626ff9a5ef35d6d3c69c94b38df7cceb975df786d618784aa9c37"}
PARENT_BOTTOM_PMF_SHA256 = {"identity": "49d5574e5678e16b72914cd98eaf1460a6ab9135932b1cd3100b8aab5f6bae02",
                            "stretched": "13c936ad5f1ce505cd63ccee925b07a0ef2ebb010a6db6f1faa61025d8e95ad3",
                            "mirrored": "9ab3ea8e0aec4a76a28f1138a0a350f9c4fd1c3b47a841be83fc1ffe1d357688"}


@pytest.mark.parametrize("n", sorted(PARENT_TOP_PMF_SHA256))
def test_zero_word_gives_the_parents_pmfs(lib, n):
    ls = LightSet(n, n)
    tree = ls.build(lib)
    pts = ls.points(64, n + 7)
    out = tree.pmfs(pts)
    assert hashlib.sha256(out.tobytes()).hexdigest() == PARENT_TOP_PMF_SHA256[n]
    assert np.array_equal(tree.pmfs(pts, np.zeros(64, np.uint32)).view(np.uint32), out.view(np.uint32))


def test_tree_draws_follow_the_pmf_with_a_receiver(lib):
    """10^6 draws at one point with a one-sided receiver: chi-square of the emitter counts against the evaluated pmfs."""
    ls = LightSet(7, 12)
    tree = ls.build(lib)
    pts = np.repeat(ls.points(1, 3)[:1], 1_000_000, axis=0)
    words = np.repeat(encode(lib, [[0.3, -0.5, 0.8]], True), len(pts))
    p = tree.pmfs(pts[:1], words[:1])[:, 0].astype(np.float64)
    light, _ = tree.sample(pts, np.random.default_rng(9).random(len(pts)), words)
    counts = np.bincount(light[light != NONE], minlength=7)
    keep = p > 0
    assert counts[~keep].sum() == 0 and p.sum() > 0.5
    chi = stats.chisquare(counts[keep], p[keep] / p[keep].sum() * counts.sum())
    assert chi.pvalue > 1e-4, chi


@pytest.mark.parametrize("kind,side", [("identity", 0), ("stretched", 0), ("mirrored", 1), ("stretched", 2)])
def test_bottom_trees_with_receivers(lib, kind, side):
    """The level-3 icosphere through identity, non-uniform and mirrored transforms: the word 0 gives the parent's pmfs; with one- and
    two-sided receivers, sum of pmfs + P(no light) = 1, sampled = evaluated bit for bit, a two-sided receiver culls nothing, and a
    one-sided receiver keeps every triangle that has a vertex in front of its WORLD-space plane by a margin (which a wrong
    object-space map of the normal would cull) and culls some that lie wholly behind it."""
    b = Bottom(lib, icosphere(3) if side != 1 else icosphere(3)[:, ::-1], side, kind)
    rng = np.random.default_rng(3)
    lo, hi = b.world.reshape(-1, 3).min(0), b.world.reshape(-1, 3).max(0)
    pts = np.ascontiguousarray(rng.uniform(lo - 1, hi + 1, (32, 3)), f32)
    base = b.pmfs(pts, np.zeros(32, np.uint32))
    assert np.array_equal(b.pmfs(pts).view(np.uint32), base.view(np.uint32))
    if side != 2:
        assert hashlib.sha256(base.tobytes()).hexdigest() == PARENT_BOTTOM_PMF_SHA256[kind]
    normals = unit(rng.normal(size=(32, 3)))
    size = float(np.ptp(b.world.reshape(-1, 3), axis=0).max())
    culled = 0
    for one_sided in (False, True):
        words = encode(lib, normals, one_sided)
        p = b.pmfs(pts, words)
        assert np.abs(p.astype(np.float64).sum(0) + b.dead_mass(pts, words) - 1.0).max() < 1e-5
        for u in rng.random((4, 32)):
            tri, pmf = b.sample(pts, u, words)
            ok = tri != NONE
            assert (pmf[ok].view(np.uint32) == p[tri[ok], np.nonzero(ok)[0]].view(np.uint32)).all()
        if not one_sided:
            assert ((base > 0) <= (p > 0)).all()
            continue
        # [tri, point]: signed distance of each world vertex to the receiver's world plane
        d = np.einsum("pc,tkpc->tkp", normals, b.world[:, :, None, :] - pts.astype(np.float64)[None, None])
        front = (d > 0.05 * size).any(axis=1)
        assert (p[front & (base > 0)] > 0).all()
        behind = (d < -0.05 * size).all(axis=1)
        culled += int(((p == 0) & behind & (base > 0)).sum())
    assert culled > 0


# ---- the warp -----------------------------------------------------------------------------------------------------------------------
def warp_case(n, seed, close=False):
    rng = np.random.default_rng(seed)
    v = rng.uniform(-1.0, 1.0, (n, 3, 3))
    v[:, :, 2] = rng.uniform(0.5, 1.5, (n, 3)) if not close else 0.3
    p = np.zeros((n, 3))
    nr = unit(rng.normal(size=(n, 3)))
    nr[:, 2] = np.abs(nr[:, 2])
    return np.ascontiguousarray(p, f32), np.ascontiguousarray(nr, f32), np.ascontiguousarray(v, f32)


def warp_sample(spherical, p, nr, v, u, warp=True):
    n = len(p)
    u = np.ascontiguousarray(u, f32)
    d, b = np.zeros((n, 3), f32), np.zeros((n, 3), f32)
    fac, om = np.zeros(n, f32), np.zeros(n, f32)
    spherical.st_warp_sample(n, p.ctypes.data, nr.ctypes.data, v.ctypes.data, u.ctypes.data, d.ctypes.data, b.ctypes.data, fac.ctypes.data,
                             om.ctypes.data, int(warp))
    return d, b, fac, om


def invert(spherical, p, v, d):
    back = np.zeros((len(p), 2), f32)
    spherical.st_invert(len(p), p.ctypes.data, v.ctypes.data, np.ascontiguousarray(d).ctypes.data, back.ctypes.data)
    return back


def test_invert_returns_the_sample_numbers(spherical):
    """Inverting sample_spherical_direction's direction gives (u0, u1) back.  Where the spherical triangle is not small (omega >= 0.05
    sr): median error below 1e-5, 99 % below 1e-4, all below 3e-3 (measured 8e-7, 4e-5, 1.4e-3).  Small spherical triangles
    (3e-4 to 0.05 sr), where fp32 loses the angles, separately: 99 % below 5e-2."""
    p, _, v = warp_case(100_000, 3)
    rng = np.random.default_rng(4)
    u = rng.uniform(0.02, 0.98, (len(p), 2)).astype(f32)
    d, _, _, om = warp_sample(spherical, p, np.zeros_like(p), v, u, warp=False)
    err = np.abs(invert(spherical, p, v, d) - u).max(axis=1)
    good = (om >= 0.05) & (om <= 6.22)
    small = (om >= 3e-4) & (om < 0.05)
    assert good.sum() > 50_000
    assert np.median(err[good]) < 1e-5 and np.quantile(err[good], 0.99) < 1e-4 and err[good].max() < 3e-3, np.quantile(err[good], [0.5, 0.99, 1])
    if small.any():
        assert np.quantile(err[small], 0.99) < 5e-2


def irradiance_estimates(spherical, p, nr, v, u, warp):
    """L cos / pdf for L = 1 of a light sample on each triangle (pdf = factor / omega)."""
    d, _, fac, om = warp_sample(spherical, p, nr, v, u, warp)
    cos = np.einsum("ij,ij->i", d.astype(np.float64), nr.astype(np.float64))
    pdf = fac.astype(np.float64) / om
    return np.where(pdf > 0, np.maximum(cos, 0.0) / pdf, 0.0)


@pytest.mark.parametrize("close", [False, True])
def test_warped_estimator_matches_lambert(spherical, close):
    """One receiver and one triangle wholly above it: the mean of L cos / pdf over 10^6 warped draws equals Lambert's polygon
    irradiance within 4 sigma; for a large, close triangle its variance is below the unwarped estimator's."""
    p, nr, v = warp_case(1, 21 if close else 22, close)
    nr[0] = np.array([0.0, 0.0, 1.0], f32)  # the triangles lie above z = 0.5: wholly above the horizon
    if close:
        # large and close, one vertex above the receiver and two near its horizon: measured variance ratio 0.34
        v[0] = np.array([[0.1, 0.1, 0.3], [3, 0, 0.05], [0, 3, 0.05]], f32)
        nr[0] = np.array([0.0, 0.0, 1.0], f32)  # the triangle wholly above the horizon, where Lambert's formula holds
    n = 1_000_000
    P, N, V = np.repeat(p, n, 0), np.repeat(nr, n, 0), np.repeat(v, n, 0)
    u = np.random.default_rng(7).random((n, 2)).astype(f32)
    est = irradiance_estimates(spherical, P, N, V, u, True)
    want = lambert_irradiance(p, nr, v)[0]
    assert abs(est.mean() - want) < 4 * est.std() / np.sqrt(n) + 1e-6 * want, (est.mean(), want)
    if close:
        plain = irradiance_estimates(spherical, P, N, V, u, False)
        assert est.var() < 0.5 * plain.var(), (est.var(), plain.var())


def test_warped_draws_follow_their_density(spherical):
    """10^6 warped draws on one triangle, binned by their unwarped (u0, u1) on an 8 x 8 grid: chi-square against the bilinear
    density's cell masses (float64 integration of pbrt-v4's bilinear density)."""
    p, nr, v = warp_case(1, 31)
    n = 1_000_000
    P, N, V = np.repeat(p, n, 0), np.repeat(nr, n, 0), np.repeat(v, n, 0)
    u = np.random.default_rng(8).random((n, 2)).astype(f32)
    d, _, _, om = warp_sample(spherical, P, N, V, u, True)
    back = invert(spherical, P, V, d)
    a = unit(v[0].astype(np.float64) - p[0].astype(np.float64))
    w = np.maximum(0.01, np.abs(a @ nr[0].astype(np.float64)))
    w4 = np.array([w[1], w[1], w[0], w[2]])
    edges = np.linspace(0, 1, 9)
    x0, x1 = edges[:-1], edges[1:]
    # cell masses of 4 ((1-x)(1-y) w0 + x(1-y) w1 + (1-x) y w2 + x y w3) / sum w
    ix = lambda f: (f(x1) - f(x0))
    mx = [ix(lambda t: t - t * t / 2), ix(lambda t: t * t / 2)]  # integrals of (1 - x) and x
    mass = 4 * (np.outer(mx[0], mx[0]).T * w4[0] + np.outer(mx[1], mx[0]).T * w4[1] + np.outer(mx[0], mx[1]).T * w4[2]
                + np.outer(mx[1], mx[1]).T * w4[3]) / w4.sum()  # [y, x]
    h, _, _ = np.histogram2d(back[:, 1], back[:, 0], bins=[edges, edges])
    chi = stats.chisquare(h.ravel(), mass.ravel() / mass.sum() * n)
    assert chi.pvalue > 1e-4, chi


# ---- the one-sided bit --------------------------------------------------------------------------------------------------------------
# The closure pins of tests/golden/ref_pins.npz (parameters in the first columns, then ng, ns, tg, wo, wi) name each closure kind and
# supply real parameter sets; the geometry is drawn here.  Kinds with the one-sided bit (hit_kind_one_sided) must give f = 0 and
# pdf = 0 for every wi on the other side of ng from wo; the transmissive kinds, which keep the two-sided term, must not (else this
# test could not tell the two apart).
ONE_SIDED_PINS = ["matte_evaluate", "mirror_evaluate", "plastic_evaluate", "metal_evaluate", "disney_evaluate_35", "disney_evaluate_59",
                  "disney_evaluate_63", "disney_evaluate_32"]
TWO_SIDED_PINS = ["glass_evaluate", "disneytrans_evaluate_163", "disneytrans_evaluate_191", "disneythin_evaluate_227",
                  "disneythin_evaluate_255"]


@pytest.fixture(scope="module")
def closures():
    h = host_harness.load("closures_host", [host_harness.DEVICE / "shading.cuh", host_harness.DEVICE / "vecmath.cuh"],
                          ["-O1", "-w", "-ffp-contract=off", host_harness.cuda_include_flag(), "-Wl,-Bsymbolic"])
    h.device_closure_unit.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int]
    return h


def behind_pairs(name, n, seed):
    """n evaluate rows of closure pin `name`: its parameter rows cycled, a random ng, a shading normal within 60 degrees of it, wo on
    a random side and wi on the other side of ng."""
    golden = np.load(host_harness.REPO / "tests" / "golden" / "ref_pins.npz")
    params = golden[f"{name}/in"].view(f32)[:, :-15]
    rng = np.random.default_rng(seed)
    ng = unit(rng.normal(size=(n, 3)))
    ns = unit(ng + 0.5 * unit(rng.normal(size=(n, 3))) * rng.random((n, 1)))
    tg = unit(np.cross(ns, rng.normal(size=(n, 3))))
    wo = unit(rng.normal(size=(n, 3)))
    wi = unit(rng.normal(size=(n, 3)))
    so, si = np.einsum("ij,ij->i", wo, ng), np.einsum("ij,ij->i", wi, ng)
    wi = np.where((so * si > 0)[:, None], wi - 2 * si[:, None] * ng, wi)  # mirror wi through the plane onto the other side
    keep = (np.abs(so) > 1e-3) & (np.abs(np.einsum("ij,ij->i", wi, ng)) > 1e-3)
    rows = np.concatenate([params[np.arange(n) % len(params)], ng, ns, tg, wo, wi], axis=1)[keep]
    return np.ascontiguousarray(rows, f32)


def evaluate(closures, name, rows):
    out = np.zeros((len(rows), 4), f32)
    assert closures.device_closure_unit(name.encode(), rows.ctypes.data, out.ctypes.data, len(rows)) == 0
    return out


@pytest.mark.parametrize("name", ONE_SIDED_PINS)
def test_one_sided_kinds_vanish_behind_the_geometric_normal(closures, name):
    rows = behind_pairs(name, 100_000, ONE_SIDED_PINS.index(name) + 1)
    out = evaluate(closures, name, rows)
    assert len(rows) > 99_000
    assert (out == 0).all(), out[np.flatnonzero((out != 0).any(axis=1))[:3]]


@pytest.mark.parametrize("name", TWO_SIDED_PINS)
def test_transmissive_kinds_do_not(closures, name):
    rows = behind_pairs(name, 100_000, 50 + TWO_SIDED_PINS.index(name))
    out = evaluate(closures, name, rows)
    assert (out[:, 3] > 0).any()


def test_one_sided_table_is_the_checked_kinds():
    """hit_kind_one_sided (hit_kinds.h, what the shade kernels compile) sets the bit for exactly the kinds checked above."""
    import re

    text = (host_harness.DEVICE / "hit_kinds.h").read_text()
    body = re.search(r"hit_kind_one_sided\(uint32_t kind\) \{(.*?)\}", text, re.S).group(1)
    kinds = {name: int(v) for name, v in re.findall(r"constexpr uint32_t kHit(\w+) = (\d+)u;", text)}
    assert {kinds[nm] for nm in re.findall(r"kHit(\w+)", body)} == ONE_SIDED_KINDS == {kinds["Matte"], kinds["Disney"], kinds["Mirror"],
                                                                                         kinds["Plastic"], kinds["Metal"]}


# ---- Python and CLI ---------------------------------------------------------------------------------------------------------------
def test_python_option_rejects_bad_values():
    check_python_option("light_receiver")


def test_cli_lists_and_parses_flag(tmp_path):
    check_cli_flag("light_receiver", tmp_path)
