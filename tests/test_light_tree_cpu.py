"""The light tree (option "light_tree") without a GPU: csrc/device/light_tree.h, the header the shade kernels and lrk_upload_scene
include, compiled for the host and checked on synthetic light sets of 1, 2, 7 and 1000 emitters that mix one-sided, two-sided,
coincident and zero-power lights, at points inside and outside their bounds.  Also the option's surface in Python and on the
command line."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest
from scipy import stats

from luisarender_b200 import _ffi as F

REPO = Path(__file__).resolve().parents[1]
SRC = REPO / "tests" / "host_device" / "light_tree_host.cpp"
OUT = REPO / "tests" / "host_device" / "_build" / "liblight_tree_host.so"
HEADER = REPO / "luisarender_b200" / "csrc" / "device" / "light_tree.h"
NONE = 0xFFFFFFFF
f32 = np.float32


@pytest.fixture(scope="module")
def lib():
    if not OUT.exists() or OUT.stat().st_mtime < max(p.stat().st_mtime for p in [SRC, HEADER]):
        OUT.parent.mkdir(parents=True, exist_ok=True)
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-shared", str(SRC), "-o", str(OUT)], check=True)
    h = C.CDLL(str(OUT))
    h.lt_build.restype = C.c_void_p
    h.lt_build.argtypes = [C.c_int] + [C.c_void_p] * 4
    h.lt_free.argtypes = [C.c_void_p]
    h.lt_node_count.restype = C.c_int64
    h.lt_node_count.argtypes = [C.c_void_p]
    h.lt_copy.argtypes = [C.c_void_p] * 3
    h.lt_pmf.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]
    h.lt_sample.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 4
    h.lt_dead_mass.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    return h


class LightSet:
    """Emitters as world-space triangles: one-sided quads facing random directions, two-sided quads, small one-sided boxes (normals
    over the whole sphere), exact duplicates of earlier emitters and emitters of zero power."""

    def __init__(self, n: int, seed: int):
        rng = np.random.default_rng(seed)
        self.tris, self.power, self.two_sided = [], [], []
        for i in range(n):
            kind = rng.integers(0, 5) if i else 0
            if kind == 3 and i >= 1:  # coincident with an earlier emitter
                j = int(rng.integers(0, i))
                self.tris.append(self.tris[j].copy())
                self.power.append(self.power[j])
                self.two_sided.append(self.two_sided[j])
                continue
            c = rng.uniform(-5.0, 5.0, 3)
            size = rng.uniform(0.05, 1.0)
            if kind == 2:
                t = box(c, size)
            else:
                n_ = rng.normal(size=3)
                t = quad(c, n_ / np.linalg.norm(n_), size)
            self.tris.append(t)
            self.power.append(0.0 if kind == 4 else float(10.0 ** rng.uniform(-1.0, 1.0)))
            self.two_sided.append(int(kind == 1))
        self.n = n

    def build(self, lib):
        counts = np.array([len(t) for t in self.tris], np.int32)
        tris = np.ascontiguousarray(np.concatenate([t.reshape(-1) for t in self.tris]), np.float64)
        power = np.array(self.power, np.float64)
        two = np.array(self.two_sided, np.int32)
        return Tree(lib, lib.lt_build(self.n, counts.ctypes.data, tris.ctypes.data, power.ctypes.data, two.ctypes.data), self.n)

    def points(self, count: int, seed: int) -> np.ndarray:
        """Half of them inside an emitter's bounds, half around the whole set."""
        rng = np.random.default_rng(seed)
        inside = []
        for _ in range(count // 2):
            t = self.tris[rng.integers(0, self.n)].reshape(-1, 3)
            lo, hi = t.min(0), t.max(0)
            inside.append(rng.uniform(lo, hi))
        outside = rng.uniform(-8.0, 8.0, (count - count // 2, 3))
        return np.ascontiguousarray(np.concatenate([np.array(inside).reshape(-1, 3), outside]), f32)

    def can_illuminate(self, e: int, p: np.ndarray, rng, samples: int = 64) -> np.ndarray:
        """Whether some sampled point of emitter e emits towards each of the points p: facing its triangle's geometric normal, or
        two-sided; never with zero power."""
        if self.power[e] == 0.0:
            return np.zeros(len(p), bool)
        if self.two_sided[e]:
            return np.ones(len(p), bool)
        t = self.tris[e].reshape(-1, 3, 3)
        k = rng.integers(0, len(t), samples)
        b = rng.dirichlet([1, 1, 1], samples)
        x = np.einsum("sj,sjc->sc", b, t[k])
        nrm = np.cross(t[k, 1] - t[k, 0], t[k, 2] - t[k, 0])
        facing = np.einsum("sc,psc->ps", nrm, p.astype(np.float64)[:, None, :] - x[None]) > 1e-6 * np.linalg.norm(nrm, axis=1)
        return facing.any(axis=1)


def quad(c, n, size):
    a = np.cross(n, [1.0, 0.0, 0.0] if abs(n[0]) < 0.9 else [0.0, 1.0, 0.0])
    a /= np.linalg.norm(a)
    b = np.cross(n, a)  # (a, b, n) right-handed: the triangles' normal is +n
    v = [c + size * (sa * a + sb * b) for sa, sb in ((-1, -1), (1, -1), (1, 1), (-1, 1))]
    return np.array([[v[0], v[1], v[2]], [v[0], v[2], v[3]]], np.float64)


def box(c, size):
    faces = []
    for axis in range(3):
        for sign in (-1.0, 1.0):
            n = np.zeros(3)
            n[axis] = sign
            faces.append(quad(c + size * n, n, size))
    return np.concatenate(faces)


class Tree:
    def __init__(self, lib, handle, n):
        self.lib, self.h, self.n = lib, handle, n

    def __del__(self):
        self.lib.lt_free(self.h)

    def pmf(self, p, e):
        out = np.zeros(len(p), f32)
        self.lib.lt_pmf(self.h, len(p), p.ctypes.data, e, out.ctypes.data)
        return out

    def sample(self, p, u):
        light, pmf = np.zeros(len(p), np.uint32), np.zeros(len(p), f32)
        u = np.ascontiguousarray(u, f32)
        self.lib.lt_sample(self.h, len(p), p.ctypes.data, u.ctypes.data, light.ctypes.data, pmf.ctypes.data)
        return light, pmf

    def dead_mass(self, p):
        out = np.zeros(len(p), np.float64)
        self.lib.lt_dead_mass(self.h, len(p), p.ctypes.data, out.ctypes.data)
        return out

    def bytes(self):
        nodes = np.zeros(self.lib.lt_node_count(self.h) * 48, np.uint8)
        trails = np.zeros(self.n, np.uint64)
        self.lib.lt_copy(self.h, nodes.ctypes.data, trails.ctypes.data)
        return nodes.tobytes() + trails.tobytes()


SETS = [1, 2, 7, 1000]


@pytest.mark.parametrize("n", SETS)
def test_pmf_sums_to_one(lib, n):
    """Over 10^4 points, the pmfs of all emitters and the probability of a descent that finds no emitter (both children of 0
    importance, which happens only where neither can emit towards the point) sum to 1."""
    ls = LightSet(n, seed=n)
    tree = ls.build(lib)
    p = ls.points(10_000, seed=1)
    total = np.zeros(len(p), np.float64)
    for e in range(n):
        total += tree.pmf(p, e)
    dead = tree.dead_mass(p)
    assert np.abs(total + dead - 1.0).max() <= 1e-5
    assert (total <= 1.0 + 1e-5).all()


@pytest.mark.parametrize("n", SETS)
def test_sampled_pmf_is_the_evaluated_pmf(lib, n):
    ls = LightSet(n, seed=n)
    tree = ls.build(lib)
    p = ls.points(10_000, seed=2)
    light, pmf = tree.sample(p, np.random.default_rng(3).random(len(p)))
    chosen = light != NONE
    assert chosen.mean() > 0.5
    assert (pmf[~chosen] == 0).all() and (pmf[chosen] > 0).all()
    for e in np.unique(light[chosen]):
        sel = light == e
        assert np.array_equal(tree.pmf(p[sel], int(e)).view(np.uint32), pmf[sel].view(np.uint32))


@pytest.mark.parametrize("n", SETS)
def test_every_emitter_that_can_illuminate_has_a_positive_pmf(lib, n):
    ls = LightSet(n, seed=n)
    tree = ls.build(lib)
    p = ls.points(2_000 if n == 1000 else 10_000, seed=4)
    rng = np.random.default_rng(5)
    reached = 0
    for e in range(n):
        pmf = tree.pmf(p, e)
        lit = ls.can_illuminate(e, p, rng)
        assert (pmf[lit] > 0).all(), (e, int((pmf[lit] == 0).sum()))
        if ls.power[e] == 0.0:
            assert (pmf == 0).all()
        reached += lit.sum()
    assert reached > 0


@pytest.mark.parametrize("n, seed", [(7, 11), (1000, 12)])
def test_sampled_frequencies_follow_the_pmf(lib, n, seed):
    """Chi-square of 10^6 draws at one point inside and one outside the bounds.  Cells with an expected count below 5 are pooled;
    the test fails at p < 1e-4, one false alarm in 10^4 seeds."""
    ls = LightSet(n, seed=n)
    tree = ls.build(lib)
    rng = np.random.default_rng(seed)
    for p0 in ls.points(2, seed=seed):
        draws = 1_000_000
        p = np.ascontiguousarray(np.repeat(p0[None], draws, axis=0), f32)
        light, _ = tree.sample(p, rng.random(draws))
        want = np.array([tree.pmf(p[:1], e)[0] for e in range(n)], np.float64)
        counts = np.bincount(light[light != NONE].astype(np.int64), minlength=n)[:n].astype(np.float64)
        expected = want * draws
        assert counts[want == 0].sum() == 0
        big = expected >= 5
        obs = np.append(counts[big], counts[~big].sum() + (light == NONE).sum())
        exp = np.append(expected[big], draws - expected[big].sum())
        keep = exp > 0
        assert stats.chisquare(obs[keep], exp[keep] * obs[keep].sum() / exp[keep].sum()).pvalue > 1e-4


@pytest.mark.parametrize("n", SETS)
def test_build_is_deterministic(lib, n):
    a = LightSet(n, seed=n).build(lib).bytes()
    b = LightSet(n, seed=n).build(lib).bytes()
    assert a == b
    powered = sum(1 for w in LightSet(n, seed=n).power if w > 0)
    assert len(a) == (2 * powered - 1) * 48 + 8 * n  # one 48-byte node per leaf and per inner node


def test_single_light_pmf_is_exactly_one(lib):
    ls = LightSet(1, seed=1)
    tree = ls.build(lib)
    p = ls.points(10_000, seed=6)
    assert (tree.pmf(p, 0) == f32(1.0)).all()
    light, pmf = tree.sample(p, np.random.default_rng(7).random(len(p)))
    assert (light == 0).all() and (pmf == f32(1.0)).all()


def test_python_option_rejects_unknown_values():
    from luisarender_b200.api import Renderer

    for bad in (2, -1, "yes", 0.5):
        with pytest.raises(ValueError):
            Renderer(light_tree=bad)  # checked before a device is looked for


def test_cli_lists_and_parses_light_tree(tmp_path):
    cli = F.LIB_DIR / "luisa-render-cli"
    r = subprocess.run([str(cli), "--help"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "--light-tree" in r.stdout
    # the flag parses: the run gets as far as reading the scene, which does not exist
    r = subprocess.run([str(cli), "-b", "cuda", "--light-tree", str(tmp_path / "missing.luisa")], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "Unrecognized options" not in r.stderr and "[error]" in r.stderr


def test_many_light_scene_generator():
    from luisarender_b200 import scenes

    own = scenes.many_lights(resolution=(32, 18), count=12)
    shared = scenes.many_lights(resolution=(32, 18), count=12, shared_node=True)
    assert own.count("Light sphere_light_") == 12 and own.count("light { @sphere_light_") == 12
    assert shared.count("Light sphere_light ") == 1 and shared.count("light { @sphere_light }") == 12
    assert "sphere_light" not in scenes.instanced_spheres()
