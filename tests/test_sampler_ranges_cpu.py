"""The table-driven samplers at the frame sizes and sample counts of the benchmark configurations (BASELINE.json): 1024^2 at 4096 spp,
1920x1080 at 1024 spp and 3840x2160 at up to 65536 spp, where the Sobol index passes 2^32, ZSobol's Morton index reaches 40 bits
and PMJ02BN's pixel tile shrinks to one pixel.  References for the index arithmetic are Python integers computed from the sampler
tables, so no 32- or 64-bit wrap can hide an error; the device header compiled for the host (tests/host_device/samplers_host.cpp)
is then compared bit for bit with the oracle at the same points.  No GPU needed."""
from __future__ import annotations

import ctypes as C
import struct

import numpy as np
import pytest

import host_harness
from luisarender_b200 import scenes
from luisarender_b200.api import Scene
from oracle import binding as O

REPO = host_harness.REPO
TABLE_SAMPLERS = ("PMJ02BN", "Sobol", "PaddedSobol", "ZSobol")
# the benchmark frames, one with an odd log2 spp that is not a power of 4 at PMJ02BN's limit, and one with an spp that is not a
# power of 2
FRAMES = [((1024, 1024), 4096), ((1920, 1080), 1024), ((3840, 2160), 65536), ((3840, 2160), 32768), ((1024, 1024), 1000)]
DIMS = (0, 1, 2, 3, 7, 100, 1023)
BOUNCES = 3


def _scene(sampler: str, resolution, spp: int):
    src = scenes.cornell_box(resolution=resolution, spp=spp)
    if sampler != "Independent":
        src = src.replace("sampler : Independent", f"sampler : {sampler}")
        assert f"sampler : {sampler}" in src
    return Scene.from_source(src, REPO)


_scenes: dict = {}


def desc(sampler: str, resolution, spp: int):
    key = (sampler, tuple(resolution), spp)
    if key not in _scenes:
        _scenes[key] = _scene(sampler, resolution, spp)
    return _scenes[key].desc()


def sobol_matrices() -> list[list[int]]:
    """Section 1 of luisarender_b200/data/sampler_tables.bin (tools/extract_sampler_tables.py): u32[1024][52]."""
    data = (REPO / "luisarender_b200" / "data" / "sampler_tables.bin").read_bytes()
    assert data[:4] == b"LRST" and struct.unpack_from("<I", data, 4)[0] == 1
    at = 8
    while at < len(data):
        tag, elem, count = struct.unpack_from("<IIQ", data, at)
        at += 16
        if tag == 1:
            assert elem == 4 and count == 1024 * 52
            m = np.frombuffer(data, dtype="<u4", count=count, offset=at).reshape(1024, 52)
            return [[int(v) for v in row] for row in m[:2]]
        at += elem * count
    raise AssertionError("no Sobol matrices in sampler_tables.bin")


def sobol(matrices, index: int, dim: int) -> int:
    v, col = 0, 0
    while index:
        if index & 1:
            v ^= matrices[dim][col]
        index >>= 1
        col += 1
    return v


def log2_ceil(x: int) -> int:
    return (x - 1).bit_length()


def interleave(px: int, py: int) -> int:
    return sum(((px >> b) & 1) << (2 * b) | ((py >> b) & 1) << (2 * b + 1) for b in range(32))


def deinterleave(m: int) -> tuple[int, int]:
    return sum(((m >> (2 * b)) & 1) << b for b in range(32)), sum(((m >> (2 * b + 1)) & 1) << b for b in range(32))


def pixels(w: int, h: int, n_random: int = 200, seed: int = 3):
    """Every corner, points on every edge next to the corners and in the middle, and n_random pixels inside."""
    out = {(0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1)}
    for x in (1, w // 2, w - 2):
        out |= {(x, 0), (x, h - 1)}
    for y in (1, h // 2, h - 2):
        out |= {(0, y), (w - 1, y)}
    rng = np.random.default_rng(seed)
    out |= {(int(x), int(y)) for x, y in zip(rng.integers(0, w, n_random), rng.integers(0, h, n_random))}
    return sorted(out)


def sample_indices(w: int, h: int, spp: int):
    """0, 1, the indices on both sides of the one from which the Sobol index s << 2m passes 2^32, and the last two below spp."""
    m = log2_ceil(max(w, h))
    cross = 1 << (32 - 2 * m)
    return sorted(s for s in {0, 1, cross - 1, cross, spp - 2, spp - 1} if 0 <= s < spp)


def points(w: int, h: int, spp: int) -> np.ndarray:
    return np.array([(x, y, s) for x, y in pixels(w, h) for s in sample_indices(w, h, spp)], dtype=np.uint32)


@pytest.fixture(scope="module")
def device_samplers():
    lib = host_harness.load("samplers_host", [host_harness.DEVICE / "samplers.cuh", host_harness.DEVICE / "vecmath.cuh"],
                            ["-O2", "-w", "-ffp-contract=off", host_harness.cuda_include_flag(), "-Wl,-Bsymbolic"])
    lib.sh_state.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                             C.c_void_p]
    lib.sh_permutation_element.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    lib.sh_permutation_element.restype = None

    def state(d, pts, dims=(), bounces=0):
        pts = np.ascontiguousarray(pts, dtype=np.uint32).reshape(-1, 3)
        dims = np.ascontiguousarray(dims, dtype=np.uint32)
        index = np.zeros(len(pts), dtype=np.uint64)
        zsobol = np.zeros((len(pts), dims.size), dtype=np.uint64)
        draws = np.zeros((len(pts), 2 + 6 * bounces), dtype=np.float32)
        rc = lib.sh_state(C.addressof(d.sampler), d.integrator.sampler_seed, pts.ctypes.data, len(pts), dims.ctypes.data, dims.size,
                          bounces, index.ctypes.data, zsobol.ctypes.data, draws.ctypes.data)
        assert rc == 0
        return index, zsobol, draws

    def permutation_element(rows):
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        out = np.zeros(len(rows), dtype=np.uint32)
        lib.sh_permutation_element(rows.ctypes.data, len(rows), out.ctypes.data)
        return out

    return state, permutation_element


@pytest.mark.parametrize("resolution", [(1024, 1024), (1920, 1080), (3840, 2160)])
def test_sobol_index_falls_in_its_pixel(resolution, device_samplers):
    """The Sobol global index of (pixel, s) is the index with s in its bits above 2m whose unscrambled first two dimensions fall
    into the pixel: exactly one such index exists, since those dimensions stratify each aligned block of 4^m indices into the
    scale x scale grid.  Up to s = 65535 at 3840x2160 (m = 12) the index reaches 2^40."""
    w, h = resolution
    d = desc("Sobol", resolution, 65536)
    scale = d.sampler.scale
    m = log2_ceil(scale)
    assert scale == 1 << m == 1 << log2_ceil(max(w, h))
    mats = sobol_matrices()
    pts = np.array([(x, y, s) for x, y in pixels(w, h) for s in sorted({0, 1, (1 << (32 - 2 * m)) - 1, 1 << (32 - 2 * m), 65535})],
                   dtype=np.uint32)
    index, _, _ = O.sampler_state(d, pts)
    dev_index, _, _ = device_samplers[0](d, pts)
    assert np.array_equal(index, dev_index)
    for (x, y, s), idx in zip(pts.tolist(), index.tolist()):
        assert idx >> (2 * m) == s, (x, y, s, idx)
        assert (sobol(mats, idx, 0) * scale) >> 32 == x, (x, y, s, idx)
        assert (sobol(mats, idx, 1) * scale) >> 32 == y, (x, y, s, idx)
    if m == 12:
        assert int(index.max()) >= 1 << 32


@pytest.mark.parametrize("spp", [65536, 32768])
def test_zsobol_morton_index_and_blocks(spp, device_samplers):
    """The ZSobol index of (pixel, s) is the bit interleave of (px, py) shifted by log2_spp, or'ed with s; and for every dimension
    the scrambled indices of a pixel's samples s < 2^log2_spp are exactly one aligned block of 2^log2_spp indices.  3840x2160 at an
    even (65536) and an odd (32768) log2 spp: 20 base-4 digits, Morton indices up to 40 bits."""
    w, h = 3840, 2160
    d = desc("ZSobol", (w, h), spp)
    L = d.sampler.log2_spp
    assert 1 << L == spp and d.sampler.num_base4_digits == log2_ceil(max(w, h)) + (L + 1) // 2
    pts = points(w, h, spp)
    index, _, _ = O.sampler_state(d, pts)
    assert np.array_equal(index, device_samplers[0](d, pts)[0])
    for (x, y, s), idx in zip(pts.tolist(), index.tolist()):
        assert idx == (interleave(x, y) << L) | s
    for x, y in [(0, 0), (w - 1, h - 1), (1234, 567)]:
        block = np.array([(x, y, s) for s in range(spp)], dtype=np.uint32)
        _, zs, _ = O.sampler_state(d, block, DIMS)
        assert np.array_equal(zs, device_samplers[0](d, block, DIMS)[1])
        for j in range(len(DIMS)):
            v = np.sort(zs[:, j])
            base = int(v[0])
            assert base % spp == 0 and np.array_equal(v - np.uint64(base), np.arange(spp, dtype=np.uint64)), (x, y, DIMS[j])


@pytest.mark.parametrize("odd_morton", [False, True])
def test_zsobol_index_past_spp_aliases_another_sample(odd_morton, device_samplers):
    """Why a render must stay below the sampler's spp: ZSobol's sample index s = 2^log2_spp carries into the Morton bits, so its
    index is sample 0 of the Morton-next pixel (even Morton code) or of the pixel itself (odd), and the films of neighbouring
    pixels would correlate."""
    w, h, spp = 3840, 2160, 65536
    d = desc("ZSobol", (w, h), spp)
    x, y = (1235, 567) if odd_morton else (1234, 567)
    morton = interleave(x, y)
    assert morton & 1 == odd_morton
    nx, ny = (x, y) if odd_morton else deinterleave(morton + 1)
    pts = np.array([(x, y, spp), (nx, ny, 0)], dtype=np.uint32)
    for state in (O.sampler_state, device_samplers[0]):
        index, zs, _ = state(d, pts, DIMS)
        assert index[0] == index[1] and np.array_equal(zs[0], zs[1])


LENGTHS = (1, 2, 3, 8, 1000, 4096, 65535, 65536)


def _mask_covering(x: int) -> int:
    return (1 << x.bit_length()) - 1


def test_permutation_element_is_a_bijection(device_samplers):
    """permutation_element(i, l, w, p) permutes [0, l) under the mask both PMJ02BN and PaddedSobol pass (the bit mask covering
    l - 1), at lengths that are and are not powers of 2 up to PMJ02BN's 65536; oracle and device header agree.  The final rotation
    (i + p) % l adds in 32 bits, as pbrt-v4 and the reference do (pmj02bn.cpp:60-86): for a hash p > 2^32 - l and an l that is not
    a power of 2 the sum wraps and two indices share a stratum.  That is kept for bit-identity with the reference and pinned here:
    the cycle walk before the rotation is a permutation of [0, l) for every hash."""
    rng = np.random.default_rng(11)
    hashes = [0, 0xFFFFFFFF, 0xFFFFFFFF - 999] + rng.integers(0, 1 << 32, 13, dtype=np.uint64).tolist()
    for l in LENGTHS:
        for p in hashes:
            rows = np.empty((l, 4), dtype=np.uint32)
            rows[:, 0] = np.arange(l, dtype=np.uint32)
            rows[:, 1] = l
            rows[:, 2] = _mask_covering(l - 1)
            rows[:, 3] = p
            got = O.unit("permutation_element", rows, 1)[:, 0]
            rotated = (np.arange(l, dtype=np.uint64) + np.uint64(p)) % np.uint64(1 << 32) % np.uint64(l)
            assert np.array_equal(np.sort(got), np.sort(rotated).astype(np.uint32)), (l, p)
            if p <= (1 << 32) - l:
                assert np.array_equal(np.sort(got), np.arange(l, dtype=np.uint32)), (l, p)
            assert np.array_equal(device_samplers[1](rows), got), (l, p)


@pytest.mark.parametrize("sampler", ("Independent",) + TABLE_SAMPLERS)
@pytest.mark.parametrize("frame", FRAMES, ids=lambda f: f"{f[0][0]}x{f[0][1]}_{f[1]}")
def test_device_sampler_equals_oracle(sampler, frame, device_samplers):
    """The device's PathSampler, compiled for the host, equals the oracle's Sampler bit for bit: derived index, scrambled ZSobol
    indices, the pixel 2D and three bounces' draws, at corner, edge and random pixels and at the first, last and 2^32-crossing
    sample indices of each benchmark frame."""
    (w, h), spp = frame
    d = desc(sampler, (w, h), spp)
    assert d.sampler.spp == spp
    pts = points(w, h, spp)
    want = O.sampler_state(d, pts, DIMS, BOUNCES)
    got = device_samplers[0](d, pts, DIMS, BOUNCES)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32))
    assert np.isfinite(want[2]).all() and (want[2] >= 0).all() and (want[2] < 1).all()


@pytest.mark.parametrize("sampler", TABLE_SAMPLERS)
def test_oracle_refuses_indices_past_spp(sampler):
    """oracle_render takes sample indices below the table-driven sampler's spp only, and leaves the film alone when it refuses."""
    spp = 4
    d = desc(sampler, (16, 12), spp)
    for begin, end in [(spp, spp + 1), (0, spp + 1), (spp - 1, spp + 4)]:
        film = np.zeros((12, 16, 4), dtype=np.float32)
        with pytest.raises(ValueError, match="spp"):
            O.render(d, begin, end, film_raw=film)
        assert not film.any()
    film, _ = O.render(d, spp, spp)
    assert not film.any()
    film, _ = O.render(d, spp - 1, spp)
    assert (film[..., 3] == 1).all()


def test_oracle_independent_takes_any_range():
    spp = 4
    d = desc("Independent", (16, 12), spp)
    film, _ = O.render(d, spp, spp + 4)
    assert (film[..., 3] == 4).all()
