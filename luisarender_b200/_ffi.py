"""ctypes mirror of include/lrk.h and include/lrh.h, and loaders for the in-tree shared libraries.

The product is the two native libraries; Python only binds them for tests and bench.py.  The loaders
fail loudly when a library is missing — there is no Python/CPU fallback for the radiance path.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
REPO_DIR = PKG_DIR.parent
LIB_DIR = PKG_DIR / "lib"

LRK_ABI_VERSION = 8
TEX_ADDRESS_EDGE, TEX_ADDRESS_REPEAT, TEX_ADDRESS_MIRROR, TEX_ADDRESS_ZERO = 0, 1, 2, 3
TEX_FILTER_POINT, TEX_FILTER_LINEAR = 0, 1
TEX_ENCODING_LINEAR, TEX_ENCODING_SRGB, TEX_ENCODING_GAMMA = 0, 1, 2
SURFACE_HAS_TEXTURES, SURFACE_REMAP_ROUGHNESS, SURFACE_MAYBE_NON_OPAQUE, SURFACE_HAS_NORMAL_MAP, SURFACE_DISNEY_TRANSMISSIVE = 1, 2, 4, 8, 16
SHAPE_HAS_VERTEX_NORMAL, SHAPE_HAS_VERTEX_UV, SHAPE_HAS_SURFACE, SHAPE_HAS_LIGHT, SHAPE_MAYBE_NON_OPAQUE = 1, 2, 4, 8, 32
LRK_FILTER_LUT_SIZE = 64

u32, u64, i32, i64, f32, f64 = C.c_uint32, C.c_uint64, C.c_int32, C.c_int64, C.c_float, C.c_double


class Vertex(C.Structure):
    _fields_ = [("p", f32 * 3), ("n", f32 * 3), ("uv", f32 * 2)]


class Triangle(C.Structure):
    _fields_ = [("i0", u32), ("i1", u32), ("i2", u32)]


class AliasEntry(C.Structure):
    _fields_ = [("prob", f32), ("alias", u32)]


class Ray(C.Structure):
    _fields_ = [("o", f32 * 3), ("tmin", f32), ("d", f32 * 3), ("tmax", f32)]


class Hit(C.Structure):
    _fields_ = [("inst", u32), ("prim", u32), ("bary", f32 * 2)]


class Mesh(C.Structure):
    _fields_ = [("vertex_offset", u32), ("vertex_count", u32), ("triangle_offset", u32), ("triangle_count", u32),
                ("bvh_root", u32), ("tri_slot_offset", u32), ("reserved", u32 * 2)]


class BvhNode(C.Structure):
    _fields_ = [("lo0", f32 * 3), ("hi0", f32 * 3), ("lo1", f32 * 3), ("hi1", f32 * 3),
                ("ref0", u32), ("ref1", u32), ("parent", u32), ("reserved", u32)]


class Instance(C.Structure):
    _fields_ = [("handle", u32 * 4), ("object_to_world", f32 * 12), ("world_to_object", f32 * 12),
                ("mesh", u32), ("visible", u32), ("reserved", u32 * 2)]


class Surface(C.Structure):
    _fields_ = [("type", u32), ("lobes", u32), ("flags", u32), ("mix_a", u32), ("p", f32 * 16), ("tex", u32 * 16),
                ("opacity_tex", u32), ("opacity", f32), ("normal_tex", u32), ("normal_strength", f32), ("normal_value", f32 * 3), ("mix_b", u32)]


class Texture(C.Structure):
    _fields_ = [("texel_offset", u64), ("width", u32), ("height", u32), ("channels", u32), ("address", u32), ("filter", u32),
                ("encoding", u32), ("scale", f32), ("gamma", f32), ("uv_scale", f32 * 2), ("uv_offset", f32 * 2), ("reserved", u32 * 2)]


class Light(C.Structure):
    _fields_ = [("emission", f32 * 3), ("scale", f32), ("two_sided", u32), ("emission_tex", u32), ("reserved", u32 * 2)]


class LightHandle(C.Structure):
    _fields_ = [("instance_id", u32), ("light_tag", u32)]


class Camera(C.Structure):
    _fields_ = [("camera_to_world", f32 * 12), ("resolution", u32 * 2), ("tan_half_fov", f32),
                ("filter_radius", f32), ("filter_shift", f32 * 2), ("spp", u32), ("reserved", u32),
                ("filter_lut", f32 * 64), ("filter_pdf", f32 * 64), ("filter_alias_probs", f32 * 64),
                ("filter_alias_indices", u32 * 64)]


class Film(C.Structure):
    _fields_ = [("scale", f32 * 3), ("clamp", f32)]


class Integrator(C.Structure):
    _fields_ = [("type", u32), ("max_depth", u32), ("rr_depth", u32), ("rr_threshold", f32),
                ("samples_per_pass", u32), ("sampler_seed", u32), ("reserved", u32 * 2)]


class Medium(C.Structure):
    _fields_ = [("present", u32), ("priority", u32), ("eta", f32), ("g", f32), ("sigma_a", f32 * 3),
                ("sigma_s", f32 * 3), ("le", f32 * 3), ("reserved", f32 * 3)]


class Environment(C.Structure):
    _fields_ = [("present", u32), ("emission_tex", u32), ("emission", f32 * 3), ("scale", f32), ("env_prob", f32), ("to_world", f32 * 9),
                ("map_width", u32), ("map_height", u32), ("reserved", u32), ("alias", C.POINTER(AliasEntry)), ("pdf", C.POINTER(f32))]


SAMPLER_INDEPENDENT, SAMPLER_PMJ02BN, SAMPLER_SOBOL, SAMPLER_PADDED_SOBOL, SAMPLER_ZSOBOL = 0, 1, 2, 3, 4


class Sampler(C.Structure):
    _fields_ = [("type", u32), ("spp", u32), ("w", u32), ("tile", u32), ("scale", u32), ("log2_spp", u32), ("num_base4_digits", u32),
                ("reserved", u32), ("sobol_matrices", C.POINTER(u32)), ("vdc", C.POINTER(u64)), ("vdc_inv", C.POINTER(u64)),
                ("pmj_samples", C.POINTER(u32)), ("blue_noise", C.POINTER(C.c_uint16)), ("pmj_pixel_samples", C.POINTER(f32)),
                ("pmj_pixel_sample_count", u64), ("zsobol_hash", C.POINTER(u32))]


class SceneDesc(C.Structure):
    _fields_ = [
        ("abi_version", u32), ("reserved0", u32),
        ("vertices", C.POINTER(Vertex)), ("vertex_count", u64),
        ("triangles", C.POINTER(Triangle)), ("alias", C.POINTER(AliasEntry)), ("pdf", C.POINTER(f32)),
        ("triangle_count", u64),
        ("meshes", C.POINTER(Mesh)), ("mesh_count", u32), ("instance_count", u32),
        ("instances", C.POINTER(Instance)),
        ("bvh_nodes", C.POINTER(BvhNode)), ("bvh_node_count", u64), ("tlas_root", u32), ("reserved1", u32),
        ("tri_verts", C.POINTER(f32)), ("tri_slot_count", u64),
        ("surfaces", C.POINTER(Surface)), ("surface_count", u32), ("light_count", u32),
        ("lights", C.POINTER(Light)), ("light_handles", C.POINTER(LightHandle)),
        ("textures", C.POINTER(Texture)), ("texture_count", u32), ("reserved2", u32), ("texels", C.POINTER(f32)), ("texel_count", u64),
        ("camera", Camera), ("film", Film), ("integrator", Integrator), ("environment_medium", Medium),
        ("environment", Environment), ("sampler", Sampler),
        ("media", C.POINTER(Medium)), ("medium_count", u32), ("environment_medium_tag", u32),
    ]


class DeviceCfg(C.Structure):
    _fields_ = [("device_index", i32), ("reserved", u32), ("max_paths_per_pass", u64)]


class Stats(C.Structure):
    _fields_ = [("render_ms", f64), ("samples", u64), ("closest_rays", u64), ("shadow_rays", u64),
                ("kernel_launches", u64), ("passes", u64), ("closest_nodes", u64), ("closest_tris", u64),
                ("closest_xforms", u64), ("shadow_nodes", u64), ("shadow_tris", u64), ("shadow_xforms", u64), ("trace_closest_ms", f64), ("trace_shadow_ms", f64), ("shade_ms", f64),
                ("other_ms", f64), ("reduce_ms", f64)]


class Adaptive(C.Structure):
    _fields_ = [("min_spp", u32), ("max_spp", u32), ("threshold", f32), ("reserved", u32)]


class SceneInfo(C.Structure):
    _fields_ = [("unique_triangles", u64), ("instanced_triangles", u64), ("vertices", u64), ("bvh_nodes", u64),
                ("meshes", u32), ("instances", u32), ("surfaces", u32), ("lights", u32), ("cameras", u32),
                ("reserved", u32), ("bvh_build_ms", f64), ("world_min", f32 * 3), ("world_max", f32 * 3)]


LRK_SYMBOLS = [
    "lrk_abi_version", "lrk_create", "lrk_destroy", "lrk_last_error", "lrk_upload_scene", "lrk_set_shard",
    "lrk_set_option", "lrk_film_clear", "lrk_render", "lrk_download_film", "lrk_download_film_raw",
    "lrk_film_device_ptr", "lrk_film_normalize_to_host", "lrk_trace", "lrk_trace_device", "lrk_get_stats",
    "lrk_stream", "lrk_comm_unique_id", "lrk_comm_init", "lrk_reduce_film", "lrk_balance_shards", "lrk_assign_tiles",
    "lrk_render_adaptive", "lrk_download_sample_counts", "lrk_download_film_variance", "lrk_download_gbuffer", "lrk_denoise",
]
LRH_SYMBOLS = [
    "lrh_last_error", "lrh_scene_load", "lrh_scene_load_source", "lrh_scene_destroy", "lrh_scene_get_info",
    "lrh_scene_get_desc", "lrh_scene_camera_file", "lrh_save_image", "lrh_plugin_count", "lrh_plugin_name",
    "lrh_create_alias_table", "lrh_load_image",
]

_libs: dict[str, C.CDLL] = {}


def _load(name: str) -> C.CDLL:
    if name not in _libs:
        path = LIB_DIR / name
        if not path.exists():
            raise RuntimeError(
                f"native library {path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                f"(there is no Python fallback)")
        _libs[name] = C.CDLL(str(path), mode=C.RTLD_GLOBAL if hasattr(C, "RTLD_GLOBAL") else os.RTLD_NOW)
    return _libs[name]


def host_lib() -> C.CDLL:
    lib = _load("libluisa_render_host.so")
    if not getattr(lib, "_lrh_typed", False):
        lib.lrh_last_error.restype = C.c_char_p
        lib.lrh_scene_load.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), u32, C.POINTER(C.c_void_p)]
        lib.lrh_scene_load_source.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), u32, C.POINTER(C.c_void_p)]
        lib.lrh_scene_destroy.argtypes = [C.c_void_p]
        lib.lrh_scene_destroy.restype = None
        lib.lrh_scene_get_info.argtypes = [C.c_void_p, C.POINTER(SceneInfo)]
        lib.lrh_scene_get_desc.argtypes = [C.c_void_p, u32, C.POINTER(SceneDesc)]
        lib.lrh_scene_camera_file.argtypes = [C.c_void_p, u32]
        lib.lrh_scene_camera_file.restype = C.c_char_p
        lib.lrh_save_image.argtypes = [C.c_char_p, C.c_void_p, u32, u32]
        lib.lrh_plugin_count.restype = u32
        lib.lrh_plugin_name.argtypes = [u32]
        lib.lrh_plugin_name.restype = C.c_char_p
        lib._lrh_typed = True
    return lib


def device_lib() -> C.CDLL:
    # LRK_DEVICE_LIB: another build of the same library (kernel experiments: tools/build_variants.sh), never a different backend
    lib = _load(os.environ.get("LRK_DEVICE_LIB", "libb200pt.so"))
    if not getattr(lib, "_lrk_typed", False):
        lib.lrk_create.argtypes = [C.POINTER(DeviceCfg), C.POINTER(C.c_void_p)]
        lib.lrk_destroy.argtypes = [C.c_void_p]
        lib.lrk_destroy.restype = None
        lib.lrk_last_error.argtypes = [C.c_void_p]
        lib.lrk_last_error.restype = C.c_char_p
        lib.lrk_upload_scene.argtypes = [C.c_void_p, C.POINTER(SceneDesc)]
        lib.lrk_set_shard.argtypes = [C.c_void_p, u32, u32, u32]
        lib.lrk_set_option.argtypes = [C.c_void_p, C.c_char_p, i64]
        lib.lrk_film_clear.argtypes = [C.c_void_p]
        lib.lrk_render.argtypes = [C.c_void_p, u32, u32]
        lib.lrk_download_film.argtypes = [C.c_void_p, C.c_void_p]
        lib.lrk_download_film_raw.argtypes = [C.c_void_p, C.c_void_p]
        lib.lrk_film_device_ptr.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(u64)]
        lib.lrk_film_normalize_to_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.lrk_trace.argtypes = [C.c_void_p, C.c_void_p, u64, C.c_int, C.c_void_p]
        lib.lrk_trace_device.argtypes = [C.c_void_p, C.c_void_p, u64, C.c_int, C.c_void_p, u32, C.POINTER(f32)]
        lib.lrk_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        lib.lrk_stream.argtypes = [C.c_void_p]
        lib.lrk_stream.restype = C.c_void_p
        lib.lrk_comm_unique_id.argtypes = [C.c_void_p]
        lib.lrk_comm_init.argtypes = [C.c_void_p, C.c_void_p, u32, u32]
        lib.lrk_reduce_film.argtypes = [C.c_void_p, u32]
        lib.lrk_balance_shards.argtypes = [C.c_void_p, u32, u32, u32, u32]
        lib.lrk_assign_tiles.argtypes = [C.c_void_p, u32, u32, C.c_void_p]
        lib.lrk_render_adaptive.argtypes = [C.c_void_p, C.POINTER(Adaptive)]
        lib.lrk_download_sample_counts.argtypes = [C.c_void_p, C.c_void_p]
        lib.lrk_download_film_variance.argtypes = [C.c_void_p, C.c_void_p]
        lib.lrk_download_gbuffer.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.lrk_denoise.argtypes = [C.c_void_p, C.c_void_p]
        lib._lrk_typed = True
    return lib
