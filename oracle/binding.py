"""ctypes binding of the CPU oracle (oracle/_build/liboracle.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs — never by the luisarender_b200 package.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

ORACLE_DIR = Path(__file__).resolve().parent
LIB_PATH = ORACLE_DIR / "_build" / "liboracle.so"


class Counters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in
                ("samples", "closest_rays", "shadow_rays", "nodes_visited", "tris_tested", "xforms", "path_vertices")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


_lib = None


def build() -> None:
    subprocess.run(["make", "-C", str(ORACLE_DIR)], check=True, capture_output=True)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            build()
        _lib = C.CDLL(str(LIB_PATH))
        f32p, vp = C.POINTER(C.c_float), C.c_void_p
        _lib.oracle_render.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, C.POINTER(Counters)]
        _lib.oracle_last_render_stats.argtypes = [C.POINTER(C.c_double)]
        _lib.oracle_last_render_stats.restype = None
        _lib.oracle_convert_film.argtypes = [vp, vp, vp]
        _lib.oracle_convert_film.restype = None
        _lib.oracle_li.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, f32p]
        _lib.oracle_li.restype = None
        _lib.oracle_trace.argtypes = [vp, vp, C.c_uint64, C.c_int, vp, C.POINTER(Counters)]
        _lib.oracle_trace_brute.argtypes = [vp, vp, C.c_uint64, C.c_int, vp]
        _lib.oracle_xxhash32_uint4.argtypes = [C.c_uint32] * 4
        _lib.oracle_xxhash32_uint4.restype = C.c_uint32
        _lib.oracle_lcg.argtypes = [C.POINTER(C.c_uint32)]
        _lib.oracle_lcg.restype = C.c_float
        _lib.oracle_sample_filter.argtypes = [vp, f32p, f32p, f32p]
        _lib.oracle_sample_filter.restype = None
        _lib.oracle_generate_ray.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, vp, f32p, C.POINTER(C.c_uint32)]
        _lib.oracle_generate_ray.restype = None
        _lib.oracle_offset_ray_origin.argtypes = [f32p, f32p, f32p]
        _lib.oracle_offset_ray_origin.restype = None
        _lib.oracle_decode_handle.argtypes = [C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), f32p]
        _lib.oracle_decode_handle.restype = None
        _lib.oracle_sample_cosine_hemisphere.argtypes = [f32p, f32p]
        _lib.oracle_sample_cosine_hemisphere.restype = None
        _lib.oracle_sample_uniform_triangle.argtypes = [f32p, f32p]
        _lib.oracle_sample_uniform_triangle.restype = None
        _lib.oracle_surface_evaluate.argtypes = [vp, f32p, f32p, f32p, f32p, f32p, f32p, f32p]
        _lib.oracle_surface_evaluate.restype = None
        _lib.oracle_surface_sample.argtypes = [vp, f32p, f32p, f32p, f32p, C.c_float, f32p, f32p, f32p, f32p]
        _lib.oracle_surface_sample.restype = None
        _lib.oracle_interaction.argtypes = [vp, vp, vp, f32p]
        _lib.oracle_interaction.restype = None
        _lib.oracle_sample_light.argtypes = [vp, vp, vp, C.c_float, f32p, f32p]
        _lib.oracle_sample_light.restype = None
        _lib.oracle_environment_sample.argtypes = [vp, f32p, f32p]
        _lib.oracle_environment_sample.restype = None
        _lib.oracle_environment_evaluate.argtypes = [vp, f32p, f32p]
        _lib.oracle_environment_evaluate.restype = None
        _lib.oracle_texture_evaluate.argtypes = [vp, C.c_uint32, f32p, f32p]
        _lib.oracle_texture_evaluate.restype = None
        _lib.oracle_resolve_surface.argtypes = [vp, C.c_uint32, f32p, vp]
        _lib.oracle_resolve_surface.restype = None
        _lib.oracle_sampler_state.argtypes = [vp, vp, C.c_uint64, vp, C.c_uint32, C.c_uint32, vp, vp, vp]
    return _lib


def _fp(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def render(desc, spp_begin: int, spp_end: int, threads: int = 0, rank: int = 0, world: int = 1, tile_size: int = 0,
           film_raw: np.ndarray | None = None):
    """Returns (film_raw [H,W,4] float32 sums, counters dict)."""
    w, h = desc.camera.resolution[0], desc.camera.resolution[1]
    if film_raw is None:
        film_raw = np.zeros((h, w, 4), dtype=np.float32)
    c = Counters()
    rc = lib().oracle_render(C.byref(desc), spp_begin, spp_end, threads, rank, world, tile_size,
                             film_raw.ctypes.data, C.byref(c))
    if rc == -2:
        raise ValueError(f"oracle_render: sample indices [{spp_begin}, {spp_end}) exceed the table-driven sampler's spp "
                         f"{desc.sampler.spp}")
    if rc != 0:
        raise RuntimeError(f"oracle_render failed: {rc}")
    return film_raw, c.as_dict()


def last_render_stats() -> dict:
    """How the last render() used the host: threads, their busy fraction, work items, seconds."""
    out = (C.c_double * 4)()
    lib().oracle_last_render_stats(out)
    return {"threads": int(out[0]), "threads_busy": round(float(out[1]), 4), "work_items": int(out[2]), "seconds": float(out[3])}


def convert_film(desc, film_raw: np.ndarray) -> np.ndarray:
    out = np.empty_like(film_raw)
    lib().oracle_convert_film(C.byref(desc), film_raw.ctypes.data, out.ctypes.data)
    return out


def li(desc, px: int, py: int, sample: int) -> np.ndarray:
    out = np.zeros(3, dtype=np.float32)
    lib().oracle_li(C.byref(desc), px, py, sample, _fp(out))
    return out


def sampler_state(desc, points, dims=(), bounces: int = 0):
    """oracle_sampler_state at points [n,3] (px, py, sample index).  Returns (derived index uint64[n], scrambled ZSobol index
    uint64[n, len(dims)] at the dimensions `dims`, draws float32[n, 2 + 6 * bounces]: the pixel 2D, then 1D, 2D, 1D, 2D per
    bounce)."""
    points = np.ascontiguousarray(points, dtype=np.uint32).reshape(-1, 3)
    dims = np.ascontiguousarray(dims, dtype=np.uint32)
    n = points.shape[0]
    index = np.zeros(n, dtype=np.uint64)
    zsobol = np.zeros((n, dims.size), dtype=np.uint64)
    draws = np.zeros((n, 2 + 6 * bounces), dtype=np.float32)
    rc = lib().oracle_sampler_state(C.byref(desc), points.ctypes.data, n, dims.ctypes.data, dims.size, bounces, index.ctypes.data,
                                    zsobol.ctypes.data, draws.ctypes.data)
    if rc != 0:
        raise ValueError(f"oracle_sampler_state failed: {rc}")
    return index, zsobol, draws


def trace(desc, rays: np.ndarray, any_hit: bool = False, brute: bool = False):
    """rays: [n,8] float32 (o, tmin, d, tmax). Returns (hits structured array, counters dict)."""
    rays = np.ascontiguousarray(rays, dtype=np.float32)
    n = rays.shape[0]
    hits = np.zeros(n, dtype=np.dtype([("inst", "<u4"), ("prim", "<u4"), ("bary", "<f4", (2,))]))
    c = Counters()
    if brute:
        rc = lib().oracle_trace_brute(C.byref(desc), rays.ctypes.data, n, int(any_hit), hits.ctypes.data)
    else:
        rc = lib().oracle_trace(C.byref(desc), rays.ctypes.data, n, int(any_hit), hits.ctypes.data, C.byref(c))
    if rc != 0:
        raise RuntimeError(f"oracle_trace failed: {rc}")
    return hits, c.as_dict()


def generate_ray(desc, px: int, py: int, sample: int):
    ray = np.zeros(8, dtype=np.float32)
    weight = np.zeros(3, dtype=np.float32)
    state = C.c_uint32()
    lib().oracle_generate_ray(C.byref(desc), px, py, sample, ray.ctypes.data, _fp(weight), C.byref(state))
    return ray, weight, state.value


def unit(name: str, inputs: np.ndarray, n_out: int, buffer: np.ndarray | None = None, buffer_count: int = 0) -> np.ndarray:
    """oracle_unit: one named numerical unit on packed 32-bit words (same packing as oracle/ref/pins.cpp)."""
    L = lib()
    L.oracle_unit.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_uint64]
    inputs = np.ascontiguousarray(inputs, dtype=np.uint32)
    out = np.zeros((inputs.shape[0], n_out), dtype=np.uint32)
    bptr = buffer.ctypes.data_as(C.c_void_p) if buffer is not None else None
    rc = L.oracle_unit(name.encode(), inputs.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), inputs.shape[0], bptr,
                       buffer_count)
    if rc != 0:
        raise KeyError(f"oracle_unit('{name}') failed with {rc}")
    return out
