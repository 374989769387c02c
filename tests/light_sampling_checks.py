"""What the tests of next-event light sampling share (test_light_*.py): for the CPU tests, the harnesses of light_tree.h and
receiver.h and of spherical_triangle.h, the light sets, meshes and transforms the trees are built from, Lambert's polygon irradiance
and the checks of each option's surface in Python and on the command line; for the GPU tests, the frames they render, the renderer
fixture, renders under a set of light-sampling options, the statistics that compare two such settings and the checks every option
passes, which each option's module calls with its own cases.

A setting is a dict of options, e.g. {"light_tree": 1}; options it leaves out keep their value on the renderer."""
from __future__ import annotations

import ctypes as C
import functools
import subprocess
from pathlib import Path

import numpy as np
import pytest

import host_harness

REPO = Path(__file__).resolve().parents[1]
BLOCK = 16
NONE = 0xFFFFFFFF
ONE_SIDED, MIRRORED, TWO_SIDED = 0, 1, 2
f32 = np.float32


# ---- the host harnesses of light_tree.h and receiver.h, and of spherical_triangle.h -----------------------------------------------
@pytest.fixture(scope="module")
def lib():
    """tests/host_device/light_tree_host.cpp: the instance-level trees (lt_*), the triangle-level ones (ltt_*) and the receiver word
    (lr_*)."""
    deps = [host_harness.DEVICE / "light_tree.h", host_harness.DEVICE / "receiver.h"]
    h = host_harness.load("light_tree_host", deps, ["-O2", "-ffp-contract=off"])
    h.lr_encode.argtypes = [C.c_int64] + [C.c_void_p] * 3
    h.lr_decode.argtypes = [C.c_int64] + [C.c_void_p] * 3
    h.lt_build.restype = C.c_void_p
    h.lt_build.argtypes = [C.c_int] + [C.c_void_p] * 4
    h.lt_pmf.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    h.lt_sample.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 5
    h.lt_dead_mass.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 3
    h.ltt_build.restype = C.c_void_p
    h.ltt_build.argtypes = [C.c_int64, C.c_void_p, C.c_int]
    h.ltt_pmf.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p]
    h.ltt_sample.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 7
    h.ltt_sample_u_left.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 4
    h.ltt_dead_mass.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 5
    for level in ("lt_", "ltt_"):
        getattr(h, level + "free").argtypes = [C.c_void_p]
        getattr(h, level + "node_count").restype = C.c_int64
        getattr(h, level + "node_count").argtypes = [C.c_void_p]
        getattr(h, level + "copy").argtypes = [C.c_void_p] * 3
    return h


@pytest.fixture(scope="module")
def spherical():
    """tests/host_device/spherical_triangle_host.cpp: the solid-angle sampler (st_*) and its receiver-cosine warp."""
    h = host_harness.load("spherical_triangle_host", [host_harness.DEVICE / "spherical_triangle.h"], ["-O2", "-ffp-contract=off"])
    h.st_solid_angle.argtypes = [C.c_int64] + [C.c_void_p] * 3
    h.st_use_spherical.argtypes = [C.c_int64] + [C.c_void_p] * 2
    h.st_sample.argtypes = [C.c_int64] + [C.c_void_p] * 8
    h.st_pdf.argtypes = [C.c_int64] + [C.c_void_p] * 5
    h.st_warp_sample.argtypes = [C.c_int64] + [C.c_void_p] * 8 + [C.c_int]
    h.st_invert.argtypes = [C.c_int64] + [C.c_void_p] * 4
    return h


def unit(x):
    return x / np.linalg.norm(x, axis=-1, keepdims=True)


def encode(lib, normals, one_sided):
    """The receiver words of `normals` [n, 3], one-sided where `one_sided` (a flag or one per normal)."""
    normals = np.ascontiguousarray(normals, f32)
    flags = np.ascontiguousarray(np.broadcast_to(np.asarray(one_sided, np.int32), (len(normals),)))
    words = np.zeros(len(normals), np.uint32)
    lib.lr_encode(len(normals), normals.ctypes.data, flags.ctypes.data, words.ctypes.data)
    return words


def decode(lib, words):
    """(unit normals [n, 3], kinds [n]: 0 none, 1 two-sided, 2 one-sided) of receiver words."""
    words = np.ascontiguousarray(words, np.uint32)
    n, k = np.zeros((len(words), 3), f32), np.zeros(len(words), np.uint32)
    lib.lr_decode(len(words), words.ctypes.data, n.ctypes.data, k.ctypes.data)
    return n, k


class Tree:
    """A light tree of the harness, queried at float32 points [n, 3] with optional receiver words [n] (None: the word 0, no
    receiver).  Indices k are emitters here and triangles in Bottom."""

    level = "lt_"

    def __init__(self, lib, handle, n):
        self.lib, self.h, self.n = lib, handle, n

    def __del__(self):
        getattr(self.lib, self.level + "free")(self.h)

    def _space(self):
        """The arguments between the words and the rest: none at the instance level, the transform's rows at the bottom level."""
        return ()

    def _call(self, query, p, words, *rest):
        words = None if words is None else np.ascontiguousarray(words, np.uint32)
        getattr(self.lib, self.level + query)(self.h, len(p), p.ctypes.data, None if words is None else words.ctypes.data, *self._space(),
                                              *rest)

    def pmf(self, p, k, words=None):
        out = np.zeros(len(p), f32)
        self._call("pmf", p, words, k, out.ctypes.data)
        return out

    def pmfs(self, p, words=None):
        """[index, point]: every emitter's (triangle's) pmf."""
        return np.stack([self.pmf(p, k, words) for k in range(self.n)])

    def sample(self, p, u, words=None):
        k, pmf = np.zeros(len(p), np.uint32), np.zeros(len(p), f32)
        u = np.ascontiguousarray(u, f32)
        self._call("sample", p, words, u.ctypes.data, k.ctypes.data, pmf.ctypes.data)
        return k, pmf

    def dead_mass(self, p, words=None):
        out = np.zeros(len(p), np.float64)
        self._call("dead_mass", p, words, out.ctypes.data)
        return out

    def nodes_and_trails(self):
        nodes = np.zeros(getattr(self.lib, self.level + "node_count")(self.h) * 48, np.uint8)
        trails = np.zeros(self.n, np.uint64)
        getattr(self.lib, self.level + "copy")(self.h, nodes.ctypes.data, trails.ctypes.data)
        return nodes, trails

    def bytes(self):
        nodes, trails = self.nodes_and_trails()
        return nodes.tobytes() + trails.tobytes()


class Bottom(Tree):
    """The bottom tree (option "light_tree_triangles") of object-space triangles [n, 3, 3] for one side, instanced through the
    transform xform(kind) and queried at world points."""

    level = "ltt_"

    def __init__(self, lib, tris, side, kind):
        self.tris, self.side, self.kind = np.asarray(tris, np.float64), side, kind
        flat = np.ascontiguousarray(self.tris.reshape(-1), np.float64)
        super().__init__(lib, lib.ltt_build(len(self.tris), flat.ctypes.data, side), len(self.tris))
        self.o2w = xform(kind)
        self.w2o = world_to_object(self.o2w)
        self.o2w_linear = np.ascontiguousarray(self.o2w[:, :3].reshape(-1), f32)  # what receiver_to_object takes
        self.world = self.tris @ self.o2w[:, :3].T + self.o2w[:, 3]

    def _space(self):
        return self.w2o.ctypes.data, self.o2w_linear.ctypes.data

    def points(self, count, seed):
        """World points: half inside the mesh's world bounds, half in a box three times their size around them."""
        rng = np.random.default_rng(seed)
        lo, hi = self.world.reshape(-1, 3).min(0), self.world.reshape(-1, 3).max(0)
        c, e = 0.5 * (lo + hi), 0.5 * (hi - lo) + 1e-3
        inside = rng.uniform(lo, hi, (count // 2, 3))
        outside = rng.uniform(c - 3 * e, c + 3 * e, (count - count // 2, 3))
        return np.ascontiguousarray(np.concatenate([inside, outside]), f32)

    def facing(self, p, margin=1e-3):
        """[points, triangles]: the world point lies in front of the triangle's emitting side by more than `margin` (relative to the
        mesh's size), judged at the triangle's three vertices and centroid; always for two-sided, never for a degenerate triangle.
        World-space normals are cross(p1 - p0, p2 - p0) of the world vertices, as the shade kernels take them."""
        w = self.world
        n = np.cross(w[:, 1] - w[:, 0], w[:, 2] - w[:, 0])
        nl = np.linalg.norm(n, axis=1)
        ok = nl > 1e-12 * max(1.0, float(np.abs(w).max())) ** 2
        if self.side == TWO_SIDED:
            return np.repeat(ok[None], len(p), axis=0)
        n = n / np.where(ok, nl, 1.0)[:, None]
        size = float(np.ptp(w.reshape(-1, 3), axis=0).max())
        pts = np.concatenate([w, w.mean(axis=1, keepdims=True)], axis=1)  # [tri, 4, 3]
        d = np.einsum("tc,ptkc->ptk", n, p.astype(np.float64)[:, None, None, :] - pts[None])
        return (d > margin * size).any(axis=2) & ok[None]


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
                t = self.box(c, size)
            else:
                n_ = rng.normal(size=3)
                t = self.quad(c, n_ / np.linalg.norm(n_), size)
            self.tris.append(t)
            self.power.append(0.0 if kind == 4 else float(10.0 ** rng.uniform(-1.0, 1.0)))
            self.two_sided.append(int(kind == 1))
        self.n = n

    @staticmethod
    def quad(c, n, size):
        a = np.cross(n, [1.0, 0.0, 0.0] if abs(n[0]) < 0.9 else [0.0, 1.0, 0.0])
        a /= np.linalg.norm(a)
        b = np.cross(n, a)  # (a, b, n) right-handed: the triangles' normal is +n
        v = [c + size * (sa * a + sb * b) for sa, sb in ((-1, -1), (1, -1), (1, 1), (-1, 1))]
        return np.array([[v[0], v[1], v[2]], [v[0], v[2], v[3]]], np.float64)

    @staticmethod
    def box(c, size):
        faces = []
        for axis in range(3):
            for sign in (-1.0, 1.0):
                n = np.zeros(3)
                n[axis] = sign
                faces.append(LightSet.quad(c + size * n, n, size))
        return np.concatenate(faces)

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


# ---- meshes (object space, [n, 3, 3]) and transforms (object-to-world 3x4) of the bottom trees ------------------------------------
def icosphere(level):
    from luisarender_b200.scenes import _icosphere

    v, f = _icosphere(level)
    return v[f]


def quad():
    v = np.array([(-1.0, 0.0, -1.0), (1.0, 0.0, -1.0), (1.0, 0.0, 1.0), (-1.0, 0.0, 1.0)])
    return np.array([[v[0], v[2], v[1]], [v[0], v[3], v[2]]])  # normal +y


def single():
    return np.array([[(0.1, 0.2, 0.0), (1.3, -0.1, 0.2), (0.4, 0.9, -0.3)]])


def soup():
    """Random triangles, every fourth degenerate (two coincident vertices or three collinear ones)."""
    rng = np.random.default_rng(5)
    t = rng.uniform(-1.0, 1.0, (40, 3, 3))
    t[::8, 1] = t[::8, 0]
    t[4::8, 2] = 0.5 * (t[4::8, 0] + t[4::8, 1])
    return t


def xform(kind):
    if kind == "identity":
        return np.hstack([np.eye(3), np.zeros((3, 1))])
    if kind == "stretched":  # rotation times non-uniform scale
        a, b = np.radians(35.0), np.radians(20.0)
        rz = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
        ry = np.array([[np.cos(b), 0.0, np.sin(b)], [0.0, 1.0, 0.0], [-np.sin(b), 0.0, np.cos(b)]])
        return np.hstack([ry @ rz @ np.diag([1.3, 0.4, 0.8]), [[0.3], [1.1], [-0.4]]])
    if kind == "mirrored":  # negative determinant
        return np.hstack([np.diag([-0.7, 1.1, 0.9]) @ np.array([[0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]) @ np.diag([1, 1, -1]),
                          [[-0.2], [0.5], [0.1]]])
    raise ValueError(kind)


def world_to_object(o2w):
    """The 12 floats of the instance's world-to-object rows, as lrk_upload_scene stores them (rows of the inverse, in float)."""
    m = np.vstack([o2w, [0.0, 0.0, 0.0, 1.0]])
    return np.ascontiguousarray(np.linalg.inv(m)[:3].reshape(-1), f32)


# ---- Lambert's polygon irradiance -------------------------------------------------------------------------------------------------
def lambert_irradiance(p, n, tri):
    """Irradiance at points p [..., 3] with normals n [..., 3] from triangles tri [..., 3, 3] of unit radiance wholly above their
    planes, in float64: E = 1/2 sum_i theta_i (n . g_i), g_i the unit normal of the plane through p and edge i, theta_i the edge's
    angle seen from p."""
    p, n, tri = (np.asarray(a, np.float64) for a in (p, n, tri))
    a = unit(tri - p[..., None, :])
    b = np.roll(a, -1, axis=-2)  # edge i runs from vertex i to vertex i + 1
    g = np.cross(a, b)
    gl = np.linalg.norm(g, axis=-1)
    theta = np.arctan2(gl, (a * b).sum(axis=-1))
    return 0.5 * np.abs((theta * (g * n[..., None, :]).sum(axis=-1) / gl).sum(axis=-1))


def analytic_irradiance_film(desc, sub=4):
    """(albedo / pi) * L * E of the irradiance frame (near_light(irradiance=True)) per pixel, averaged over sub x sub points of the
    pixel's box footprint: the pinhole of pathcommon.cuh's camera_ray looks straight down at the plane, to which its image plane is
    parallel."""
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
    e = lambert_irradiance(x.reshape(-1, 3), (0.0, 1.0, 0.0), tri).reshape(ry, sub, rx, sub).mean(axis=(1, 3))
    return 0.5 / np.pi * 4.0 * e


# ---- the frames of the GPU tests --------------------------------------------------------------------------------------------------
def _globes(prefix, resolution, subdivision):
    return {f"{prefix}_{t}": (lambda s, t=t: s.emissive_globe(resolution=resolution, spp=16, subdivision=subdivision, transform=t))
            for t in ("uniform", "stretched", "mirrored")}


# Frame name -> the scene source, from luisarender_b200.scenes.  The session scenes of conftest.py (spheres_small, cornell_small,
# textured_wrappers_small) are frames too, under their fixtures' names.
FRAMES = {
    "cornell": lambda s: s.cornell_box(resolution=(64, 64), spp=16),
    "sobol_cornell": lambda s: s.cornell_box(resolution=(64, 64), spp=1024).replace("sampler : Independent", "sampler : PaddedSobol"),
    "textured_lamp": lambda s: s.textured_room(resolution=(96, 64), spp=8, textured_light=True),
    "environment_area": lambda s: s.environment_scene(resolution=(64, 48), spp=4, area_light=True),
    "environment_one_light": lambda s: s.environment_scene(resolution=(48, 30), spp=4, area_light=True),
    "flatten": lambda s: s.flatten_stress(resolution=(64, 48), spp=4),
    "mix": lambda s: s.materials_box(mix=True),
    "mix_64x48": lambda s: s.materials_box(resolution=(64, 48), spp=4, mix=True),
    "layered": lambda s: s.layered_box(),
    "layered_64x48": lambda s: s.layered_box(resolution=(64, 48), spp=4),
    "many": lambda s: s.many_lights(resolution=(128, 72), spp=16, count=48, big_subdivision=3, small_subdivision=2),
    # the many-light frame with every sphere of the same emission, one Light node each, and the same spheres sharing one node
    "many_equal": lambda s: s.many_lights(resolution=(128, 72), spp=16, count=48, spread=False, big_subdivision=3, small_subdivision=2),
    "many_shared": lambda s: s.many_lights(resolution=(128, 72), spp=16, count=48, shared_node=True, big_subdivision=3, small_subdivision=2),
    **_globes("globe", (96, 96), 4),
    **_globes("small_globe", (64, 64), 3),
    "near": lambda s: s.near_light(resolution=(96, 96), spp=16),
    "glossy_desk": lambda s: s.near_light(resolution=(96, 96), spp=16, glossy_desk=True),
    "irradiance": lambda s: s.near_light(resolution=(64, 64), spp=16, irradiance=True),
    "medium": lambda s: s.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3, small_subdivision=2,
                                            small_count=12),
}


@functools.lru_cache(maxsize=None)
def frame(name):
    """The scene of frame `name`, parsed once per session."""
    from luisarender_b200 import scenes
    from luisarender_b200.api import Scene

    return Scene.from_source(FRAMES[name](scenes), REPO)


@pytest.fixture
def frames(request):
    """Frame name -> scene."""
    return lambda name: frame(name) if name in FRAMES else request.getfixturevalue(name)


# ---- renders and their statistics -------------------------------------------------------------------------------------------------
# Unbiasedness checks compare the means of the image and of its 16 x 16 blocks over 32 + 32 sub-renders at 4 sigma: for a normal
# estimate each comparison fails with probability 6e-5, with sigma estimated from the sub-renders (t, 62 dof) 1.7e-4, so the
# many-light frame (1 + 32 means) fails by chance about 0.6 % of the time (the renders are seeded, so a given seed passes or fails
# for good).
SUBRENDERS, SUB_SPP, Z_MAX = 32, 16, 4.0


@pytest.fixture
def r(gpu_renderer):
    """gpu_renderer, with every option these tests touch back at its default afterwards (the renderer is shared by the session)."""
    yield gpu_renderer
    for name, value in (("light_receiver", 0), ("light_candidates", 0), ("light_tree_triangles", 0), ("light_tree", 0),
                        ("light_solid_angle", 0), ("gbuffer", 0), ("max_paths_per_pass", 136 << 20)):
        gpu_renderer.set_option(name, value)
    gpu_renderer.set_shard(0, 1, 32)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def upload(r, desc, options):
    for name, value in options.items():
        r.set_option(name, int(value))
    r.upload(desc)


def render(r, desc, spp_begin, spp_end, options, raw=True):
    upload(r, desc, options)
    r.render(spp_begin, spp_end)
    return r.film(raw=raw).copy()


def sub_renders(r, desc, options, first, count, spp):
    """`count` independent renders of `spp` samples each from sample index `first` on, as normalised films [count, H, W, 3]: one
    upload, then a cleared film per render."""
    upload(r, desc, options)
    films = []
    for k in range(count):
        r.clear()
        r.render(first + k * spp, first + (k + 1) * spp)
        films.append(r.film(raw=False)[..., :3].copy())
    return np.stack(films).astype(np.float64)


def reference(r, desc, options):
    """The 1024-spp film of sample indices [2^20, 2^20 + 1024), disjoint from those of the renders it is compared with."""
    return sub_renders(r, desc, options, 1 << 20, 1, 1024)[0]


def rel_mse(r, desc, options, ref, first):
    """The relative MSE against `ref` of 16-spp renders, averaged over 8 of them from sample index `first` on."""
    films = sub_renders(r, desc, options, first, 8, 16)
    return float(np.mean([((f - ref) ** 2 / (ref ** 2 + 1e-2)).mean() for f in films]))


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


# ---- the checks every light-sampling option passes --------------------------------------------------------------------------------
def check_off_equals_a_fresh_context(r, desc, fresh_options, first, offs):
    """A fresh Renderer(**fresh_options) renders `desc` as the shared context does under each setting of `offs` (film and launch
    count), after the setting `first` (None: none) was rendered there and left its kernels and buffers behind."""
    from luisarender_b200.api import Renderer

    fresh = Renderer(device_index=0, **fresh_options)
    try:
        fresh.set_option("strict_math", 0 if r.fast else 1)
        fresh.upload(desc)
        fresh.render(0, 4)
        want, want_launches = fresh.film(raw=True), fresh.stats()["kernel_launches"]
    finally:
        fresh.close()
    if first is not None:
        render(r, desc, 0, 4, first)
    for off in offs:
        got = render(r, desc, 0, 4, off)
        assert np.array_equal(bits(got), bits(want)), off
        assert r.stats()["kernel_launches"] == want_launches


def check_agrees_without_it(r, desc, off, on, changes_the_film=False):
    """The setting `on` renders the image of `off` within the noise of 32 + 32 sub-renders of disjoint sample indices; with
    `changes_the_film`, the same sample indices must first give another film (the option changes the sampling on this frame)."""
    if changes_the_film:
        assert not np.array_equal(bits(render(r, desc, 0, 2, off)), bits(render(r, desc, 0, 2, on)))
    without = sub_renders(r, desc, off, 0, SUBRENDERS, SUB_SPP)
    with_ = sub_renders(r, desc, on, SUBRENDERS * SUB_SPP, SUBRENDERS, SUB_SPP)
    assert without.mean() > 0
    assert not np.array_equal(without.mean(axis=0), with_.mean(axis=0))
    z = z_scores(with_, without)
    assert np.abs(z).max() < Z_MAX, z


def check_irradiance_frame_matches_lambert(r, desc, options):
    """The block means of the irradiance frame equal analytic_irradiance_film within Z_MAX standard errors."""
    films = sub_renders(r, desc, options, 0, SUBRENDERS, SUB_SPP)
    want = analytic_irradiance_film(desc)
    m = block_means(films)
    w = block_means(np.repeat(want[None, :, :, None], 3, axis=3))[0]
    se = m.std(axis=0, ddof=1) / np.sqrt(len(m))
    assert (se > 0).all()
    z = (m.mean(axis=0) - w) / se
    assert np.abs(z).max() < Z_MAX, z


def check_error_ratio(r, desc, off, on, bound, label):
    """The 16-spp relative MSE under `on` is at most `bound` times that under `off`, each averaged over 8 renders, against a
    1024-spp reference of disjoint sample indices rendered under `on`."""
    ref = reference(r, desc, on)
    e_off, e_on = rel_mse(r, desc, off, ref, 0), rel_mse(r, desc, on, ref, 4096)
    print(f"{label} 16 spp rel. MSE: off {e_off:.4e}, on {e_on:.4e}, ratio {e_on / e_off:.4f} (fast={r.fast})")
    assert e_on <= bound * e_off, (e_on, e_off, e_on / e_off)


def check_scheduling_and_sharding(r, desc, options):
    """Two calls, 1024-path passes and three balanced shards give the film of one render, bit for bit."""
    whole = render(r, desc, 0, 8, options)
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
        r.upload(desc)
        r.balance_shards(rank, 3, 32, 1)  # the cost probe runs the option's kernels too
        r.render(0, 8)
        part = r.film(raw=True)
        assert not np.any((total != 0) & (part != 0))  # every pixel has one owner
        total += part
    assert np.array_equal(bits(total), bits(whole))


def check_gbuffer_and_adaptive(r, desc, off, on):
    """`on` changes the film of `off` but not the first-hit guides of the G-buffer, and adaptive threshold 0 equals lrk_render."""
    r.set_option("gbuffer", 1)
    film_off = render(r, desc, 0, 4, off)
    gb_off = r.gbuffer()
    film_on = render(r, desc, 0, 4, on)
    gb_on = r.gbuffer()
    assert not np.array_equal(bits(film_on), bits(film_off))  # the option changes the film ...
    for a, b in zip(gb_on[:2], gb_off[:2]):  # ... not the first-hit guides (the third, the luminance variance, follows the film)
        assert np.array_equal(bits(a), bits(b))
    r.set_option("gbuffer", 0)
    want = render(r, desc, 0, 8, on)
    r.render_adaptive(0.0, 4, 8)
    assert np.array_equal(bits(r.film(raw=True)), bits(want))


def check_refusals(r, frames, desc, base, steps):
    """Render `desc` under `base`, run `steps` and render again: the film must not change.  A step is a dict of options to set,
    ("upload", frame, message) for an upload that must be refused, ("set", option, value) for a value lrk_set_option must refuse
    ("failed (-1)"), or "film": the film is still the first one."""
    before = render(r, desc, 0, 2, base)
    for step in steps:
        if isinstance(step, dict):
            for name, value in step.items():
                r.set_option(name, value)
        elif step == "film":
            assert np.array_equal(bits(r.film(raw=True)), bits(before))
        elif step[0] == "upload":
            with pytest.raises(RuntimeError, match=step[2]):
                r.upload(frames(step[1]).desc())
        else:
            with pytest.raises(RuntimeError, match=r"failed \(-1\)"):
                r.set_option(step[1], step[2])
    assert np.array_equal(bits(render(r, desc, 0, 2, base)), bits(before))


# ---- each option's surface in Python and on the command line ----------------------------------------------------------------------
FLAG_VALUES_REFUSED = (2, -1, "yes", 0.5)  # what a False / True keyword refuses
# option -> (the other keywords its refused values are passed with, the values Renderer refuses before a device is looked for, the
# refusal of the option alone when it needs another, the CLI help's entry, CLI arguments that parse, CLI arguments refused, the
# refusal's message)
SURFACE = {
    "light_tree": ({}, FLAG_VALUES_REFUSED, None, "--light-tree", [["--light-tree"]], [], None),
    "light_solid_angle": ({}, FLAG_VALUES_REFUSED, None, "--light-solid-angle", [["--light-solid-angle"]], [], None),
    "light_tree_triangles": ({"light_tree": True}, FLAG_VALUES_REFUSED, "light_tree=True", "--light-tree-triangles",
                             [["--light-tree-triangles"]], [], None),
    "light_candidates": ({"device_index": -1}, (-1, 33, 2.0, 4.5, True, False, "4", None), None, "--light-candidates <n>",
                         [["--light-candidates", "0"], ["--light-candidates", "8"], ["--light-candidates=32"]],
                         [["--light-candidates=-1"], ["--light-candidates=33"], ["--light-candidates=4x"]],
                         "--light-candidates takes a count from 0 to 32"),
    "light_receiver": ({"light_tree": True}, FLAG_VALUES_REFUSED, "light_tree=True", "--light-receiver", [["--light-receiver"]], [],
                       None),
}


def check_python_option(option):
    """Renderer(**needs, option=bad) raises ValueError before a device is looked for; so does an option without the one it refines."""
    from luisarender_b200.api import Renderer

    needs, refused, prerequisite = SURFACE[option][:3]
    for value in refused:
        with pytest.raises(ValueError):
            Renderer(**needs, **{option: value})
    if prerequisite:
        with pytest.raises(ValueError, match=prerequisite):
            Renderer(**{option: True})


def check_cli_flag(option, tmp_path):
    """luisa-render-cli lists the option's flag, parses its arguments (the run gets as far as reading the scene, which does not
    exist) and refuses bad values before the scene is read."""
    from luisarender_b200 import _ffi as F

    help_entry, parse, refuse, message = SURFACE[option][3:]
    cli = F.LIB_DIR / "luisa-render-cli"
    missing = str(tmp_path / "missing.luisa")
    r = subprocess.run([str(cli), "--help"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and help_entry in r.stdout
    for args in parse:
        r = subprocess.run([str(cli), "-b", "cuda", *args, missing], capture_output=True, text=True, timeout=60)
        assert r.returncode != 0 and "Unrecognized options" not in r.stderr, r.stderr
        assert "[error]" in r.stderr and "missing.luisa" in r.stderr, r.stderr
    for args in refuse:
        r = subprocess.run([str(cli), "-b", "cuda", *args, missing], capture_output=True, text=True, timeout=60)
        assert r.returncode != 0 and message in r.stderr, r.stderr
