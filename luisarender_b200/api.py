"""Thin Python wrappers over the two native libraries (tests / bench only; the reference is C++ and so
is the product: see csrc/host and csrc/device, and the luisa-render-cli executable).

``Scene``     wraps libluisa_render_host.so  (include/lrh.h): parse -> scene graph -> flattened POD scene.
``Renderer``  wraps libb200pt.so             (include/lrk.h): upload, render on the GPU, download film.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from . import _ffi as F


class Scene:
    def __init__(self, handle: C.c_void_p):
        self._h = handle
        self._lib = F.host_lib()
        self._descs: dict[int, F.SceneDesc] = {}

    @classmethod
    def from_source(cls, source: str, base_dir: str | Path | None = None, macros: dict[str, str] | None = None,
                    json: bool = False) -> "Scene":
        lib = F.host_lib()
        keys, vals, n = _macro_arrays(macros)
        h = C.c_void_p()
        rc = lib.lrh_scene_load_source(source.encode(), int(json), str(base_dir or Path.cwd()).encode(), keys, vals, n, C.byref(h))
        if rc != 0:
            raise RuntimeError(lib.lrh_last_error().decode())
        return cls(h)

    @classmethod
    def from_file(cls, path: str | Path, macros: dict[str, str] | None = None) -> "Scene":
        lib = F.host_lib()
        keys, vals, n = _macro_arrays(macros)
        h = C.c_void_p()
        rc = lib.lrh_scene_load(str(path).encode(), keys, vals, n, C.byref(h))
        if rc != 0:
            raise RuntimeError(lib.lrh_last_error().decode())
        return cls(h)

    def desc(self, camera: int = 0) -> F.SceneDesc:
        if camera not in self._descs:
            d = F.SceneDesc()
            if self._lib.lrh_scene_get_desc(self._h, camera, C.byref(d)) != 0:
                raise RuntimeError(self._lib.lrh_last_error().decode())
            d._owner = self  # the view points into memory owned by this Scene: keep it alive with the view
            self._descs[camera] = d
        return self._descs[camera]

    def info(self) -> dict:
        i = F.SceneInfo()
        self._lib.lrh_scene_get_info(self._h, C.byref(i))
        out = {n: getattr(i, n) for n, _ in i._fields_ if n not in ("reserved", "world_min", "world_max")}
        out["world_min"] = list(i.world_min)
        out["world_max"] = list(i.world_max)
        return out

    def camera_file(self, camera: int = 0) -> str:
        return self._lib.lrh_scene_camera_file(self._h, camera).decode()

    def close(self):
        if self._h:
            self._lib.lrh_scene_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _macro_arrays(macros):
    if not macros:
        return None, None, 0
    n = len(macros)
    keys = (C.c_char_p * n)(*[k.encode() for k in macros])
    vals = (C.c_char_p * n)(*[str(v).encode() for v in macros.values()])
    return keys, vals, n


def save_image(path: str | Path, rgba: np.ndarray) -> None:
    rgba = np.ascontiguousarray(rgba, dtype=np.float32)
    h, w = rgba.shape[0], rgba.shape[1]
    lib = F.host_lib()
    if lib.lrh_save_image(str(path).encode(), rgba.ctypes.data, w, h) != 0:
        raise RuntimeError(lib.lrh_last_error().decode())


class Renderer:
    """One GPU context. Fails loudly when libb200pt.so or a CUDA device is missing (no CPU fallback).

    ``light_tree=True`` sets the option "light_tree" (include/lrk.h): from the next upload on, next-event estimation picks its
    lights from a light tree by power, distance and orientation instead of uniformly (surface integrator only).
    ``light_solid_angle=True`` sets the option "light_solid_angle": from the next upload on, next-event estimation samples the
    point on the chosen emissive triangle uniformly in solid angle instead of by area (surface integrator only).
    ``light_tree_triangles=True`` (with ``light_tree=True``) sets the option "light_tree_triangles": the light tree also picks the
    triangle of the chosen emitter, from a tree over its mesh's triangles, instead of by area.
    ``light_candidates=M`` (an int from 0 to 32) sets the option "light_candidates": for M >= 2, from the next upload on,
    next-event estimation draws M candidates from the light sampling above and traces the shadow ray of one, chosen by its
    unshadowed contribution (resampled importance sampling; surface integrator only).  0 and 1 keep one light sample per vertex."""

    def __init__(self, device_index: int = -1, max_paths_per_pass: int = 0, light_tree: bool = False, light_solid_angle: bool = False,
                 light_tree_triangles: bool = False, light_candidates: int = 1):
        light_options = {"light_tree": light_tree, "light_solid_angle": light_solid_angle, "light_tree_triangles": light_tree_triangles}
        for name, value in light_options.items():
            if value not in (0, 1):
                raise ValueError(f"{name} is False or True, not {value!r}")
        if light_tree_triangles and not light_tree:
            raise ValueError("light_tree_triangles is the bottom level of the light tree: it needs light_tree=True")
        if type(light_candidates) is not int or not 0 <= light_candidates <= 32:
            raise ValueError(f"light_candidates is an int from 0 to 32, not {light_candidates!r}")
        self._lib = F.device_lib()
        cfg = F.DeviceCfg(device_index, 0, max_paths_per_pass)
        self._ctx = C.c_void_p()
        rc = self._lib.lrk_create(C.byref(cfg), C.byref(self._ctx))
        if rc != 0:
            raise RuntimeError(f"lrk_create failed ({rc}): no usable CUDA device")
        self._res = None
        for name, value in light_options.items():
            if value:
                self.set_option(name, 1)
        if light_candidates >= 2:
            self.set_option("light_candidates", light_candidates)

    def _check(self, rc: int, what: str):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self._lib.lrk_last_error(self._ctx).decode()}")

    def upload(self, desc: F.SceneDesc):
        self._check(self._lib.lrk_upload_scene(self._ctx, C.byref(desc)), "lrk_upload_scene")
        self._res = (desc.camera.resolution[0], desc.camera.resolution[1])

    def set_shard(self, rank: int, world: int, tile_size: int = 32):
        self._check(self._lib.lrk_set_shard(self._ctx, rank, world, tile_size), "lrk_set_shard")

    @staticmethod
    def comm_unique_id() -> bytes:
        """lrk_comm_unique_id: the 128 bytes one rank creates and every rank passes to comm_init."""
        buf = C.create_string_buffer(128)
        rc = F.device_lib().lrk_comm_unique_id(buf)
        if rc != 0:
            raise RuntimeError(f"lrk_comm_unique_id failed ({rc}): NCCL (libnccl.so.2) is not available")
        return buf.raw

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        """lrk_comm_init (collective): join the film-reduce communicator."""
        assert len(unique_id) == 128
        self._check(self._lib.lrk_comm_init(self._ctx, C.c_char_p(unique_id), rank, world), "lrk_comm_init")

    def reduce_film(self, root: int = 0):
        """lrk_reduce_film (collective): rank `root`'s raw film becomes the sum over ranks."""
        self._check(self._lib.lrk_reduce_film(self._ctx, root), "lrk_reduce_film")

    def balance_shards(self, rank: int, world: int, tile_size: int = 32, probe_spp: int = 1):
        """lrk_balance_shards: probe the frame's cost per tile and take rank `rank`'s share of a cost-balanced tile assignment."""
        self._check(self._lib.lrk_balance_shards(self._ctx, rank, world, tile_size, probe_spp), "lrk_balance_shards")

    def set_option(self, name: str, value: int):
        """lrk_set_option; e.g. ("light_tree", 1): light-tree selection of next-event lights from the next upload on."""
        self._check(self._lib.lrk_set_option(self._ctx, name.encode(), value), f"lrk_set_option({name})")

    def clear(self):
        self._check(self._lib.lrk_film_clear(self._ctx), "lrk_film_clear")

    def render(self, spp_begin: int, spp_end: int):
        self._check(self._lib.lrk_render(self._ctx, spp_begin, spp_end), "lrk_render")

    def render_adaptive(self, threshold: float, min_spp: int, max_spp: int):
        """lrk_render_adaptive: clear the film, then render every pixel until the 8x4 block around it has a relative standard error
        below `threshold` (rounds of min_spp, 2 min_spp, 4 min_spp, ... samples, at most max_spp; include/lrk.h)."""
        p = F.Adaptive(min_spp, max_spp, threshold, 0)
        self._check(self._lib.lrk_render_adaptive(self._ctx, C.byref(p)), "lrk_render_adaptive")

    def sample_counts(self) -> np.ndarray:
        """The samples every pixel got in the last adaptive render, [H, W] uint32 (0 outside this context's shard)."""
        w, h = self._res
        out = np.empty((h, w), dtype=np.uint32)
        self._check(self._lib.lrk_download_sample_counts(self._ctx, out.ctypes.data), "lrk_download_sample_counts")
        return out

    def film_variance(self) -> np.ndarray:
        """The variance of every pixel's mean luminance after the last adaptive render, [H, W] float32 (0 outside the shard)."""
        w, h = self._res
        out = np.empty((h, w), dtype=np.float32)
        self._check(self._lib.lrk_download_film_variance(self._ctx, out.ctypes.data), "lrk_download_film_variance")
        return out

    def gbuffer(self) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The guides of a G-buffer film (option "gbuffer" set before the film clear; include/lrk.h): albedo_cov [H, W, 4] (mean
        first-hit albedo, fraction of samples that hit), normal_depth [H, W, 4] (normalised sum of normals, mean hit distance) and
        variance [H, W] (variance of the pixel's mean luminance)."""
        w, h = self._res
        albedo_cov, normal_depth = np.empty((h, w, 4), dtype=np.float32), np.empty((h, w, 4), dtype=np.float32)
        variance = np.empty((h, w), dtype=np.float32)
        self._check(self._lib.lrk_download_gbuffer(self._ctx, albedo_cov.ctypes.data, normal_depth.ctypes.data, variance.ctypes.data),
                    "lrk_download_gbuffer")
        return albedo_cov, normal_depth, variance

    def denoise(self) -> np.ndarray:
        """The denoised film of a G-buffer film, [H, W, 4] float32 normalised like film(); the film itself is left as it is."""
        w, h = self._res
        out = np.empty((h, w, 4), dtype=np.float32)
        self._check(self._lib.lrk_denoise(self._ctx, out.ctypes.data), "lrk_denoise")
        return out

    def film(self, raw: bool = False, out: np.ndarray | None = None) -> np.ndarray:
        """The film as [H, W, 4] float32: normalised like the reference's convert_image, or the raw sums (raw=True).
        `out`: destination to reuse (with the option pin_host_buffers the library page-locks it once)."""
        w, h = self._res
        if out is None:
            out = np.empty((h, w, 4), dtype=np.float32)
        assert out.shape == (h, w, 4) and out.dtype == np.float32 and out.flags.c_contiguous
        fn = self._lib.lrk_download_film_raw if raw else self._lib.lrk_download_film
        self._check(fn(self._ctx, out.ctypes.data), "lrk_download_film")
        return out

    def film_device_ptr(self) -> tuple[int, int]:
        p, n = C.c_void_p(), C.c_uint64()
        self._check(self._lib.lrk_film_device_ptr(self._ctx, C.byref(p), C.byref(n)), "lrk_film_device_ptr")
        return p.value, n.value

    def normalize_to_host(self, device_raw_ptr: int) -> np.ndarray:
        w, h = self._res
        out = np.empty((h, w, 4), dtype=np.float32)
        self._check(self._lib.lrk_film_normalize_to_host(self._ctx, C.c_void_p(device_raw_ptr), out.ctypes.data),
                    "lrk_film_normalize_to_host")
        return out

    def trace(self, rays: np.ndarray, any_hit: bool = False) -> np.ndarray:
        rays = np.ascontiguousarray(rays, dtype=np.float32)
        n = rays.shape[0]
        hits = np.zeros(n, dtype=np.dtype([("inst", "<u4"), ("prim", "<u4"), ("bary", "<f4", (2,))]))
        self._check(self._lib.lrk_trace(self._ctx, rays.ctypes.data, n, int(any_hit), hits.ctypes.data), "lrk_trace")
        return hits

    def trace_device(self, d_rays: int, n: int, d_hits: int, any_hit: bool = False, repeat: int = 1) -> float:
        ms = C.c_float()
        self._check(self._lib.lrk_trace_device(self._ctx, C.c_void_p(d_rays), n, int(any_hit), C.c_void_p(d_hits), repeat, C.byref(ms)),
                    "lrk_trace_device")
        return ms.value

    def stats(self) -> dict:
        s = F.Stats()
        self._check(self._lib.lrk_get_stats(self._ctx, C.byref(s)), "lrk_get_stats")
        return {n: getattr(s, n) for n, _ in s._fields_}

    def stream(self) -> int:
        return self._lib.lrk_stream(self._ctx)

    def close(self):
        if self._ctx:
            self._lib.lrk_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
