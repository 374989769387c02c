"""The DEVICE code of the general volume integrator, compiled for the host, against the oracle.

tests/host_device/volume_host.cpp includes luisarender_b200/csrc/device/volume_general.cuh - the per-sample loop the sm_90a kernel
`volume_general_kernel` runs, with the medium tracker, the surface events, the transmittance walk, and underneath them the
closures, light sampling, hit reconstruction and the single-ray traversal - and is compiled with g++ (-ffp-contract=off, as nvcc's
-fmad=false).  Same expressions + same libm => the raw film must equal the oracle's BIT FOR BIT, and the oracle is bit-identical
to the unmodified reference renderer on these scenes (tests/test_ref_render.py: media_*).  What remains for the GPU test
(tests/test_gpu_parity.py::test_volume_with_shape_media_matches_oracle) is CUDA's libm and code generation.  No GPU needed.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import host_harness
from luisarender_b200 import scenes
from luisarender_b200.api import Scene
from oracle import binding as O

REPO = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def lib():
    deps = sorted(host_harness.DEVICE.glob("*.cuh")) + [REPO / "include" / "lrk.h"]
    handle = host_harness.load("volume_host", deps, ["-O1", "-w", "-ffp-contract=off", host_harness.cuda_include_flag(), "-Wl,-Bsymbolic"])
    handle.volume_general_host.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    return handle


def _golden_case(name):
    import sys

    sys.path.insert(0, str(REPO / "tools"))
    import gen_ref_renders as G

    return G.cases()[name]


CASES = {
    "shape_media": lambda: scenes.media_box(resolution=(40, 40), spp=3),
    "shape_media_deep_rr": lambda: scenes.media_box(resolution=(32, 32), spp=3, depth=16, rr_depth=3, rr_threshold=0.9),
    "nested_in_environment_medium": lambda: scenes.media_box(resolution=(40, 40), spp=3, environment_medium=True, rr_depth=2),
    "true_hit_quirk": lambda: scenes.media_box(resolution=(40, 40), spp=3, skip_quirk=True),
    # image-textured Mirror / Glass / Plastic / Metal parameters: closure contexts derived per hit (run through the volume integrator
    # with no medium at all: the tracker stays empty)
    "textured_materials": lambda: scenes.textured_materials(resolution=(48, 30), spp=3, depth=6, integrator="MegaVPTNaive"),
    # config C4's shape (one environment medium, opaque closures): the wavefront kernels' territory, but the general code must agree
    "environment_medium_only": lambda: scenes.instanced_spheres(resolution=(32, 18), spp=2, depth=6, medium=True, big_subdivision=2,
                                                                small_subdivision=1, small_count=12),
    # the three Disney closure classes - thin ("through" events: the tracker must not move), transmissive (enter / exit), opaque -
    # inside an environment medium: the scene of tests/golden/ref_renders.npz: spheres_medium_disney_thin
    "disney_thin_and_transmissive": lambda: _golden_case("spheres_medium_disney_thin"),
    # a thin Disney surface with image-textured colour and diffuse_trans (slot 15 of the per-hit parameter resolution)
    "textured_disney_thin": lambda: _golden_case("textured_disney_thin").replace("integrator : WavePath", "integrator : MegaVPTNaive"),
    # media bound to shapes behind Disney shells: a thin one (through events) and a transmissive one (enter / exit), in an environment medium
    "media_disney_shells": lambda: _golden_case("media_disney_shells"),
    # an image-lit environment seen from inside an environment medium (environment misses and environment NEE in the volume loop),
    # next to an area light, with a thin Disney ball
    "environment_medium_thin": lambda: _golden_case("environment_medium_thin"),
    # an area light with an image emission (texture lookups at emitter hits and at sampled light points), no medium at all
    "textured_light": lambda: scenes.textured_room(resolution=(40, 30), spp=3, mesh_files=False, textured_light=True, integrator="MegaVPTNaive"),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_volume_code_is_bit_identical_to_the_oracle(lib, name):
    scene = Scene.from_source(CASES[name](), REPO)
    d = scene.desc()
    w, h, spp = d.camera.resolution[0], d.camera.resolution[1], d.camera.spp
    film = np.zeros((h, w, 4), np.float32)
    rays = np.zeros(2, np.uint64)
    assert lib.volume_general_host(C.byref(d), 0, spp, film.ctypes.data, rays.ctypes.data) == 0  # no stack / tracker overflow
    want, cnt = O.render(d, 0, spp)
    assert want[..., :3].mean() > 0.02
    same = (film.view(np.uint32) == want.view(np.uint32)).all(axis=-1)
    assert same.all(), f"{name}: {int((~same).sum())} of {same.size} pixels differ; first {np.argwhere(~same)[0].tolist()}"
    assert int(rays[0]) == cnt["closest_rays"] and int(rays[1]) == cnt["shadow_rays"]
