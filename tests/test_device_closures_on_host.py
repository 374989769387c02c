"""The DEVICE closures, compiled for the host, against the reference's own closures.

tests/host_device/closures_host.cpp includes luisarender_b200/csrc/device/shading.cuh — the file the sm_90a shade kernels
are built from — and is compiled with g++ (-ffp-contract=off, as nvcc's -fmad=false).  The Matte, Disney and
Mirror / Glass / Plastic / Metal closures are then driven exactly the way shade_surface() (kernels.cuh) drives them and
compared with tests/golden/ref_pins.npz: outputs of the reference's closure classes through Surface::Closure::
{evaluate,sample}.  Same expressions + same libm => the results must agree to the last bits; what remains for the GPU tests
is CUDA's libm and code generation.  No GPU, no /root/reference needed.
"""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

import host_harness

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO / "tools"))
import gen_ref_pins as G  # noqa: E402

CLOSURE_PINS = sorted(n for n in G.PINS if n.split("_")[0] in ("matte", "disney", "disneytrans", "disneythin", "mirror", "glass", "plastic", "metal"))


@pytest.fixture(scope="module")
def lib():
    handle = host_harness.load("closures_host", [host_harness.DEVICE / "shading.cuh", host_harness.DEVICE / "vecmath.cuh"],
                               ["-O1", "-w", "-ffp-contract=off", host_harness.cuda_include_flag(), "-Wl,-Bsymbolic"])
    handle.device_closure_unit.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int]
    return handle


@pytest.mark.parametrize("name", CLOSURE_PINS)
def test_device_closure_matches_reference_closure(lib, name):
    golden = np.load(REPO / "tests" / "golden" / "ref_pins.npz")
    inp, want = golden[f"{name}/in"], golden[f"{name}/out"]
    got = np.zeros_like(want)
    assert lib.device_closure_unit(name.encode(), inp.ctypes.data, got.ctypes.data, inp.shape[0]) == 0
    a, b = got.view(np.float32).astype(np.float64), want.view(np.float32).astype(np.float64)
    if "_sample" in name:
        # columns: wi (3), f (3), pdf, event.  The device carries the event as rr_eta_scale.  An invalid sample (pdf = 0) has no
        # meaningful direction on either side, and its f is 0 on the device where the reference may carry 0 * NaN (a refracted
        # direction under total internal reflection): both end the path, since beta *= f * (pdf > 0 ? 1 / pdf : 0) is then
        # 0 or NaN and NaN throughputs are zeroed (mega_path.cpp:141).
        valid = b[:, 6] > 0.0
        a, b = a[:, :7], b[:, :7]
        a[~valid, :6] = b[~valid, :6]
    with np.errstate(invalid="ignore"):
        close = np.abs(a - b) <= 2e-5 * np.maximum(1.0, np.abs(b))
    close |= np.isnan(a) & np.isnan(b)
    close |= np.isinf(a) & np.isinf(b) & (np.sign(a) == np.sign(b))
    bad = ~close.all(axis=1)
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {len(bad)} cases differ; first: in={inp[np.flatnonzero(bad)[0]].view(np.float32)} "
                           f"device={got[np.flatnonzero(bad)[0]].view(np.float32)} reference={want[np.flatnonzero(bad)[0]].view(np.float32)}")


def test_device_layered_closure_matches_the_oracle(lib):
    """The Layered closure (stochastic random walks between two interfaces, seeded from the bits of the hit position and the
    directions) as the device code evaluates and samples it, against the oracle's restatement - which is bit-identical to the
    reference's renders (tests/test_ref_render.py::materials_layered*).  Three Layered nodes (scattering slab, attenuating slab,
    defaults), 4000 random (position, normal, wo, wi, u) rows each; same libm on both sides => identical bits."""
    from luisarender_b200 import scenes
    from luisarender_b200.api import Scene
    from oracle import binding as O

    d = Scene.from_source(scenes.layered_box(resolution=(16, 12), spp=1), REPO).desc()
    layered = [i for i in range(d.surface_count) if d.surfaces[i].type == 7]
    assert len(layered) == 3
    rng = np.random.default_rng(11)
    rows = np.zeros((4000, 16), np.float32)
    rows[:, 0:3] = rng.uniform(-2, 2, (4000, 3))
    rows[:, 3:12] = rng.normal(size=(4000, 9))
    rows[:, 12:15] = rng.uniform(0, 1, (4000, 3))
    lib.device_layered_unit.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int]
    olib = O.lib()
    olib.oracle_layered_unit.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int]
    for index in layered:
        got, want = np.zeros((4000, 12), np.float32), np.zeros((4000, 12), np.float32)
        assert lib.device_layered_unit(d.surfaces, index, rows.ctypes.data, got.ctypes.data, 4000) == 0
        assert olib.oracle_layered_unit(d.surfaces, index, rows.ctypes.data, want.ctypes.data, 4000) == 0
        assert (want[:, 3] > 0).mean() > 0.5 and (want[:, 10] > 0).mean() > 0.3  # the cases exercise both calls
        same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
        bad = ~same.all(axis=1)
        assert not bad.any(), f"surface {index}: {int(bad.sum())} of 4000 rows differ; first: device {got[np.flatnonzero(bad)[0]]} oracle {want[np.flatnonzero(bad)[0]]}"
