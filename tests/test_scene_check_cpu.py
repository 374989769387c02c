"""The check of a scene description that lrk_upload_scene makes before it changes anything (csrc/device/scene_check.h), compiled for
the host.  Every description of the scene library passes it, and what it derives for the upload equals a restatement from the
description's fields; every refusal it can return is triggered by a corrupted copy of a library description, with its status code
and message."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import host_harness
from luisarender_b200 import _ffi as F
from luisarender_b200 import scenes
from luisarender_b200.api import Scene

REPO = Path(__file__).resolve().parents[1]
INVALID, UNSUPPORTED = -1, -5
SHAPE_HAS_MEDIUM = 16
SURFACE_DISNEY, SURFACE_MIX, SURFACE_LAYERED, SURFACE_RAW_PARAMS, SURFACE_DISNEY_THIN = 1, 6, 7, 32, 64
INTEGRATOR_VOLUME_PATH = 1
TREE, TRIANGLES, SOLID_ANGLE, RECEIVER = 1, 2, 4, 8
# the light options of a surface-integrator scene: none, the tree with its bottom level and receiver, solid angle with resampling
LIGHT_OPTIONS = [(0, 0), (TREE, 0), (TREE | TRIANGLES | RECEIVER, 0), (SOLID_ANGLE | RECEIVER, 4)]

LIBRARY = {
    "cornell_matte": lambda: scenes.cornell_box(resolution=(32, 32), spp=4),
    "cornell_disney": lambda: scenes.cornell_box(resolution=(32, 32), spp=4, surface="Disney"),
    "instanced_spheres": lambda: scenes.instanced_spheres(resolution=(32, 18), spp=4, big_subdivision=3, small_subdivision=1, small_count=12,
                                                          emissive=4),
    "spheres_medium": lambda: scenes.instanced_spheres(resolution=(32, 18), spp=4, big_subdivision=3, small_subdivision=1, small_count=12,
                                                       medium=True),
    "textured_room": lambda: scenes.textured_room(resolution=(32, 24), spp=4, wrappers=True, textured_light=True),
    "media_box": lambda: scenes.media_box(resolution=(32, 32), spp=4),
    "emissive_globe": lambda: scenes.emissive_globe(resolution=(32, 32), spp=4, subdivision=2),
    "wavy_sheet": lambda: scenes.wavy_sheet(emissive=True),
    "many_lights": lambda: scenes.many_lights(resolution=(32, 18), spp=4, count=6, big_subdivision=3, small_subdivision=1, small_count=12),
    "flatten_stress": lambda: scenes.flatten_stress(),
    "layered_box": lambda: scenes.layered_box(),
    "environment_scene": lambda: scenes.environment_scene(),
}


@pytest.fixture(scope="module")
def lib():
    deps = [host_harness.DEVICE / n for n in ("scene_check.h", "hit_kinds.h")] + [REPO / "include" / "lrk.h"]
    h = host_harness.load("scene_check_host", deps, ["-O2", "-ffp-contract=off"])
    h.scene_check_run.restype = C.c_void_p
    h.scene_check_run.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]
    h.scene_check_free.argtypes = [C.c_void_p]
    h.scene_check_status.argtypes = [C.c_void_p]
    h.scene_check_error.argtypes = [C.c_void_p]
    h.scene_check_error.restype = C.c_char_p
    h.scene_check_scalars.argtypes = [C.c_void_p, C.c_void_p]
    h.scene_check_array.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
    h.scene_check_array.restype = C.c_size_t
    h.scene_check_light_meshes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    h.scene_check_light_meshes.restype = C.c_size_t
    h.scene_check_mesh_points.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    h.scene_check_mesh_points.restype = C.c_size_t
    return h


@pytest.fixture(scope="module")
def kinds_lib():
    h = host_harness.load("hit_kinds_host", [host_harness.DEVICE / "hit_kinds.h", REPO / "include" / "lrk.h"], ["-O2"])
    h.hit_kinds_of_surfaces.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    return h


@pytest.fixture(scope="module")
def library():
    return {name: Scene.from_source(make(), REPO) for name, make in LIBRARY.items()}


def run(lib, desc, light_bits=0, candidates=0, device_bvh=False):
    """(status, message, result dict or None) of the check of `desc`"""
    h = lib.scene_check_run(C.addressof(desc), light_bits, candidates, int(device_bvh))
    try:
        status, message = lib.scene_check_status(h), lib.scene_check_error(h).decode()
        if status != 0:
            return status, message, None
        scalars = np.zeros(8, np.uint64)
        lib.scene_check_scalars(h, scalars.ctypes.data)
        r = dict(zip(["volume", "volume_general", "textured", "any_non_opaque", "used_kinds", "tlas_root", "node_count", "largest_mesh"],
                     (int(v) for v in scalars)))
        dtypes = {"inst_kind": np.uint32, "inst_mesh": np.uint32, "visible": np.uint32, "mesh_root": np.uint32, "mesh_emissive": np.uint8,
                  "light_inst": np.uint32, "light_mesh": np.uint32, "light_o2w": np.float32, "light_power": np.float64,
                  "light_two_sided": np.uint8}
        for name, dt in dtypes.items():
            out = np.zeros(lib.scene_check_array(h, name.encode(), None), dt)
            lib.scene_check_array(h, name.encode(), out.ctypes.data)
            r[name] = out
        count = C.c_uint32()
        meshes = np.zeros(lib.scene_check_light_meshes(h, C.byref(count), None), np.uint32)
        lib.scene_check_light_meshes(h, C.byref(count), meshes.ctypes.data)
        r["light_instance_count"] = count.value
        r["mesh_points"] = {}
        for m in meshes.tolist():
            pts = np.zeros(lib.scene_check_mesh_points(h, m, None), np.float32)
            lib.scene_check_mesh_points(h, m, pts.ctypes.data)
            r["mesh_points"][m] = pts
        return status, message, r
    finally:
        lib.scene_check_free(h)


def accepts(d, light_bits, candidates) -> bool:
    """The light options a description's integrator takes"""
    return d.integrator.type != INTEGRATOR_VOLUME_PATH or (light_bits == 0 and candidates < 2)


def restated(d, kinds_lib, light_bits, device_bvh):
    """What the upload derives from `d`, computed here from its fields"""
    insts = np.ctypeslib.as_array(d.instances, (d.instance_count,))
    meshes = np.ctypeslib.as_array(d.meshes, (d.mesh_count,))
    surfaces = [d.surfaces[i] for i in range(d.surface_count)]
    lights = [d.lights[k] for k in range(d.light_count)]
    flags, tags = insts["handle"][:, 0], insts["handle"][:, 1]
    surface_kind = np.zeros(max(d.surface_count, 1), np.uint32)
    kinds_lib.hit_kinds_of_surfaces(C.cast(d.surfaces, C.c_void_p), d.surface_count, surface_kind.ctypes.data)
    has_surface, has_light = (flags & F.SHAPE_HAS_SURFACE) != 0, (flags & F.SHAPE_HAS_LIGHT) != 0
    inst_kind = np.where(has_surface, surface_kind[np.where(has_surface, (tags >> 12) & 4095, 0)], 0)
    volume = d.integrator.type == INTEGRATOR_VOLUME_PATH
    general = volume and (not d.environment_medium.present or d.medium_count != 1 or bool(d.environment.present) or
                          bool((flags & SHAPE_HAS_MEDIUM).any()) or
                          any(s.type > SURFACE_DISNEY or s.flags & (F.SURFACE_DISNEY_TRANSMISSIVE | SURFACE_DISNEY_THIN) for s in surfaces))
    mesh_emissive = np.zeros(d.mesh_count, np.uint8)
    mesh_emissive[insts["mesh"][has_light]] = 1
    r = {
        "volume": int(volume), "volume_general": int(general),
        "textured": int(any(s.flags & (F.SURFACE_HAS_TEXTURES | F.SURFACE_HAS_NORMAL_MAP) for s in surfaces) or
                        any(light.emission_tex != 0 for light in lights)),
        "any_non_opaque": int(((flags & F.SHAPE_MAYBE_NON_OPAQUE != 0) & has_surface).any()),
        "used_kinds": 1 | int(np.bitwise_or.reduce(np.uint32(1) << inst_kind.astype(np.uint32), initial=0)),
        "inst_kind": inst_kind, "inst_mesh": insts["mesh"], "visible": np.flatnonzero(insts["visible"]), "mesh_emissive": mesh_emissive,
    }
    tris = meshes["triangle_count"].astype(np.int64)
    if device_bvh:
        sizes = np.maximum(tris - 1, 1)
        r["mesh_root"] = np.cumsum(sizes) - sizes
        r["tlas_root"] = int(sizes.sum())
        r["node_count"] = r["tlas_root"] + max(len(r["visible"]), 2) - 1
        r["largest_mesh"] = int(tris.max(initial=0))
    else:
        r["mesh_root"] = meshes["bvh_root"]
        r["tlas_root"], r["node_count"], r["largest_mesh"] = d.tlas_root, d.bvh_node_count, 0
    # the light tree's source
    emitters = np.flatnonzero(has_light) if light_bits & TREE else np.zeros(0, np.int64)
    power, points = [], {}
    vertices = np.ctypeslib.as_array(d.vertices, (d.vertex_count,))["p"]
    triangles = np.ctypeslib.as_array(d.triangles, (d.triangle_count,))
    for i in emitters:
        light = lights[tags[i] & 4095]
        rgb = np.array(light.emission[:], np.float64)
        if light.emission_tex:
            t = d.textures[light.emission_tex - 1]
            texels = np.ctypeslib.as_array(d.texels, (d.texel_count * 4,))[t.texel_offset * 4:(t.texel_offset + t.width * t.height) * 4]
            # summed in order, as the library sums them
            rgb = np.cumsum(np.maximum(texels.reshape(-1, 4)[:, :3].astype(np.float64), 0.0), axis=0)[-1] / (t.width * t.height)
        rgb = np.maximum(rgb, 0.0)
        power.append((0.2126 * rgb[0] + 0.7152 * rgb[1] + 0.0722 * rgb[2]) * np.float64(np.float32(light.scale)))
        m = meshes[insts["mesh"][i]]
        if int(insts["mesh"][i]) not in points:
            tri = triangles[m["triangle_offset"]:m["triangle_offset"] + m["triangle_count"]]
            idx = np.stack([tri["i0"], tri["i1"], tri["i2"]], axis=1).astype(np.int64) + m["vertex_offset"]
            points[int(insts["mesh"][i])] = vertices[idx].reshape(-1)
    r.update(light_inst=emitters, light_mesh=insts["mesh"][emitters], light_o2w=insts["object_to_world"][emitters].reshape(-1),
             light_power=power, light_two_sided=[int(lights[tags[i] & 4095].two_sided != 0) for i in emitters],
             light_instance_count=d.instance_count if light_bits & TREE else 0, mesh_points=points)
    return r


@pytest.mark.parametrize("device_bvh", [False, True])
@pytest.mark.parametrize("name", list(LIBRARY))
def test_library_descriptions_pass_and_derive_their_fields(name, device_bvh, lib, kinds_lib, library):
    d = library[name].desc()
    checked = 0
    for light_bits, candidates in LIGHT_OPTIONS:
        if not accepts(d, light_bits, candidates):
            continue
        status, message, got = run(lib, d, light_bits, candidates, device_bvh)
        assert status == 0, (name, light_bits, message)
        want = restated(d, kinds_lib, light_bits, device_bvh)
        for key, value in want.items():
            if key == "mesh_points":
                assert sorted(got[key]) == sorted(value), (name, key)
                for m, pts in value.items():
                    assert np.array_equal(got[key][m], pts), (name, key, m)
            elif key == "light_power":
                assert got[key].tolist() == [float(p) for p in value], (name, key)
            else:
                assert np.array_equal(np.asarray(got[key]), np.asarray(value)), (name, key, got[key], value)
        checked += 1
    assert checked == (1 if d.integrator.type == INTEGRATOR_VOLUME_PATH else len(LIGHT_OPTIONS))


def test_library_covers_what_the_check_derives(lib, library):
    """The library descriptions reach every derived value: both volume kernels, textures, non-opaque surfaces, emissive meshes in
    the light tree's source, image emission and invisible instances."""
    seen = set()
    for name, scene in library.items():
        d = scene.desc()
        _, _, r = run(lib, d, TREE if d.integrator.type != INTEGRATOR_VOLUME_PATH else 0)
        seen |= {k for k in ("volume", "volume_general", "textured", "any_non_opaque") if r[k]}
        if r["volume"] and not r["volume_general"]:
            seen.add("volume_wavefront")
        if len(r["light_inst"]) and len(r["mesh_points"]):
            seen.add("light_source")
        if len(r["visible"]) < d.instance_count:
            seen.add("invisible")
        if any(d.lights[k].emission_tex for k in range(d.light_count)):
            seen.add("image_emission")
    assert seen == {"volume", "volume_general", "volume_wavefront", "textured", "any_non_opaque", "light_source", "invisible", "image_emission"}


class Corrupt:
    """A copy of a description whose arrays can be changed without touching the original's"""

    def __init__(self, desc):
        self.d = F.SceneDesc.from_buffer_copy(bytes(desc))
        self._keep = []

    def array(self, field, ctype, count):
        arr = (ctype * max(count, 1))()
        if count:
            C.memmove(arr, getattr(self.d, field), C.sizeof(ctype) * count)
        self._keep.append(arr)
        setattr(self.d, field, C.cast(arr, C.POINTER(ctype)))
        return arr

    def instances(self):
        return self.array("instances", F.Instance, self.d.instance_count)

    def surfaces(self):
        return self.array("surfaces", F.Surface, self.d.surface_count)

    def meshes(self):
        return self.array("meshes", F.Mesh, self.d.mesh_count)


def _first(items, pred):
    return next(i for i, x in enumerate(items) if pred(x))


def _light_instance(c):
    insts = c.instances()
    return insts, _first(insts, lambda x: x.handle[0] & F.SHAPE_HAS_LIGHT)


def _set(obj, **fields):
    for k, v in fields.items():
        setattr(obj, k, v)


def _medium_tag(c):
    insts = c.instances()
    insts[0].handle[0] |= SHAPE_HAS_MEDIUM
    insts[0].handle[1] |= 255 << 24


def _surface_tag(c):
    insts = c.instances()
    i = _first(insts, lambda x: x.handle[0] & F.SHAPE_HAS_SURFACE)
    insts[i].handle[1] = (insts[i].handle[1] & ~(4095 << 12)) | (c.d.surface_count << 12)


def _mesh_index(c):
    c.instances()[0].mesh = c.d.mesh_count


def _light_tag(c):
    insts, i = _light_instance(c)
    insts[i].handle[1] = (insts[i].handle[1] & ~4095) | c.d.light_count


def _light_handle(c):
    handles = c.array("light_handles", F.LightHandle, c.d.light_count)
    handles[c.d.light_count - 1].instance_id = c.d.instance_count


def _huge_mesh(c):
    c.meshes()[0].triangle_count = 1 << 28
    c.d.triangle_count = (1 << 28) + c.d.triangle_count


# (base description, light options, device_bvh, corruption, status, message); in the order the check makes them
REFUSALS = [
    ("cornell_matte", 0, False, lambda c: _set(c.d, abi_version=99), INVALID, "lrk_upload_scene: ABI version mismatch"),
    ("media_box", 0, False, lambda c: _set(c.d, medium_count=257), INVALID, "lrk_upload_scene: invalid media table"),
    ("media_box", 0, False, lambda c: _set(c.d, environment_medium_tag=c.d.medium_count), INVALID,
     "lrk_upload_scene: environment medium tag outside the media table"),
    ("media_box", 0, False, lambda c: _set(c.array("media", F.Medium, c.d.medium_count)[0], present=7), UNSUPPORTED,
     "lrk_upload_scene: unknown medium kind"),
    ("media_box", 0, False, lambda c: _set(c.array("media", F.Medium, c.d.medium_count)[0], present=1, eta=1.5), UNSUPPORTED,
     "lrk_upload_scene: media with eta != 1 are not supported"),
    ("media_box", 0, False, _medium_tag, INVALID, "lrk_upload_scene: a shape's medium tag is outside the media table"),
    ("media_box", 0, False, lambda c: _set(c.d.sampler, type=F.SAMPLER_SOBOL), UNSUPPORTED,
     "lrk_upload_scene: the volume path with shape media / transmissive surfaces takes the Independent sampler"),
    ("media_box", 0, False, lambda c: _set(c.d.integrator, max_depth=32), UNSUPPORTED, "lrk_upload_scene: volume path depth > 31"),
    ("cornell_matte", 0, False, lambda c: _set(c.d.integrator, type=5), UNSUPPORTED, "lrk_upload_scene: unknown integrator type"),
    ("cornell_matte", 0, False, lambda c: _set(c.d.environment_medium, present=1), UNSUPPORTED,
     "lrk_upload_scene: an environment medium needs the volume path integrator (MegaVPTNaive)"),
    ("cornell_matte", 0, False, lambda c: _set(c.d.integrator, max_depth=64), UNSUPPORTED, "lrk_upload_scene: max depth > 63"),
    ("media_box", (TREE, 0), False, None, UNSUPPORTED, "lrk_upload_scene: the light tree (option light_tree) serves the surface integrator only; the volume integrator selects its "
     "lights uniformly"),
    ("cornell_matte", (TRIANGLES, 0), False, None, INVALID,
     "lrk_upload_scene: the triangle-level light trees (option light_tree_triangles) are the bottom level of the light tree: set the "
     "option light_tree too"),
    ("media_box", (SOLID_ANGLE, 0), False, None, UNSUPPORTED, "lrk_upload_scene: solid-angle light sampling (option light_solid_angle) serves the surface "
     "integrator only; the volume integrator evaluates its light pdfs from the world origin"),
    ("media_box", (0, 2), False, None, UNSUPPORTED, "lrk_upload_scene: resampled next-event estimation (option light_candidates >= 2) serves the "
     "surface integrator only; the volume integrator traces every light sample it draws, since the occlusion of each advances its random "
     "stream"),
    ("media_box", (RECEIVER, 0), False, None, UNSUPPORTED, "lrk_upload_scene: receiver-aware light sampling (option light_receiver) serves the "
     "surface integrator only; the volume integrator selects its lights uniformly by area"),
    ("cornell_matte", (RECEIVER, 0), False, None, INVALID, "lrk_upload_scene: receiver-aware light sampling (option light_receiver) refines the "
     "light tree and solid-angle sampling: set the option light_tree or light_solid_angle too"),
    ("cornell_matte", 0, False, lambda c: _set(c.d.camera, resolution=(C.c_uint32 * 2)(65536, 32)), UNSUPPORTED,
     "lrk_upload_scene: film larger than 65535 pixels per side"),
    ("cornell_matte", 0, False, lambda c: _set(c.d, light_count=0), INVALID, "No lights in scene. Rendering aborted."),
    ("environment_scene", 0, False, lambda c: _set(c.d.environment, env_prob=0.0), INVALID, "lrk_upload_scene: invalid environment record"),
    ("environment_scene", 0, False, lambda c: _set(c.d, light_count=0), INVALID, "lrk_upload_scene: env_prob must be 1 without area lights"),
    ("cornell_matte", 0, False, lambda c: _set(c.surfaces()[0], type=8), UNSUPPORTED, "lrk_upload_scene: unknown surface type"),
    ("cornell_matte", 0, False, lambda c: _set(c.surfaces()[0], type=SURFACE_MIX, flags=F.SURFACE_HAS_TEXTURES, tex=(C.c_uint32 * 16)(1)),
     UNSUPPORTED, "lrk_upload_scene: the ratio of a Mix is a constant"),
    ("cornell_matte", 0, False, lambda c: _set(c.surfaces()[0], flags=SURFACE_RAW_PARAMS), INVALID,
     "lrk_upload_scene: LRK_SURFACE_RAW_PARAMS is for Mirror / Glass / Plastic / Metal records"),
    ("media_box", 0, False, lambda c: _set(c.surfaces()[0], type=SURFACE_LAYERED), UNSUPPORTED,
     "lrk_upload_scene: Layered surfaces are not supported by the volume path integrator"),
    ("cornell_matte", 0, False, lambda c: _set(c.surfaces()[0], type=SURFACE_LAYERED, lobes=0), INVALID,
     "lrk_upload_scene: a Layered surface needs samples >= 1"),
    ("cornell_matte", 0, False, lambda c: _set(c.surfaces()[0], type=SURFACE_MIX, mix_a=c.d.surface_count), UNSUPPORTED,
     "lrk_upload_scene: a Mix / Layered surface combines two constant Matte / Mirror / Glass / Plastic / Metal records"),
    ("cornell_matte", 0, False, lambda c: _set(c.surfaces()[0], tex=(C.c_uint32 * 16)(0, 0, 0, 1)), INVALID,
     "lrk_upload_scene: texture id out of range"),
    ("textured_room", 0, False, lambda c: _set(c.surfaces()[0], normal_tex=c.d.texture_count + 1), INVALID,
     "lrk_upload_scene: texture id out of range"),
    ("media_box", 0, False, lambda c: _set(c.surfaces()[0], flags=F.SURFACE_MAYBE_NON_OPAQUE), UNSUPPORTED,
     "lrk_upload_scene: non-opaque surfaces are not supported by the volume path integrator"),
    ("cornell_matte", 0, False, lambda c: _set(c.d.sampler, type=5), UNSUPPORTED, "lrk_upload_scene: unknown sampler type"),
    ("spheres_medium", 0, False, lambda c: _set(c.d.sampler, type=F.SAMPLER_SOBOL), UNSUPPORTED,
     "lrk_upload_scene: the volume path integrator supports the Independent sampler only"),
    ("cornell_matte", 0, False, lambda c: _set(c.d.sampler, type=F.SAMPLER_SOBOL, spp=4), INVALID, "lrk_upload_scene: incomplete sampler record"),
    ("textured_room", 0, False, lambda c: _set(c.array("textures", F.Texture, c.d.texture_count)[0], width=0), INVALID,
     "lrk_upload_scene: invalid image texture record"),
    ("cornell_matte", 0, False, lambda c: _set(c.array("lights", F.Light, c.d.light_count)[0], emission_tex=c.d.texture_count + 1), INVALID,
     "lrk_upload_scene: a light's emission texture id is out of range"),
    ("cornell_matte", 0, False, _surface_tag, INVALID, "lrk_upload_scene: surface tag out of range"),
    ("cornell_matte", 0, False, _mesh_index, INVALID, "lrk_upload_scene: mesh index out of range"),
    ("cornell_matte", 0, True, lambda c: _set(c.meshes()[1], triangle_count=0), INVALID, "lrk_upload_scene: mesh without triangles"),
    ("cornell_matte", 0, True, _huge_mesh, UNSUPPORTED, "lrk_upload_scene: scene too large for the BVH encoding"),
    ("cornell_matte", 0, False, _light_tag, INVALID, "lrk_upload_scene: light tag out of range"),
    ("cornell_matte", (TREE, 0), True, _light_tag, INVALID, "lrk_upload_scene: light tag out of range"),
    ("cornell_matte", 0, False, _light_handle, INVALID, "lrk_upload_scene: light handle instance id out of range"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_every_refusal_has_its_code_and_message(case, lib, library):
    base, options, device_bvh, corrupt, status, message = REFUSALS[case]
    light_bits, candidates = options or (0, 0)
    c = Corrupt(library[base].desc())
    if corrupt is not None:
        corrupt(c)
        assert run(lib, library[base].desc(), light_bits, candidates, device_bvh)[0] == 0  # the corruption is what is refused
    assert run(lib, c.d, light_bits, candidates, device_bvh)[:2] == (status, message)
