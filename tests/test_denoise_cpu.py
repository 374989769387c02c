"""The G-buffer mode and the denoiser without a GPU: the denoiser's arithmetic (csrc/device/denoise.h, compiled for the host) against
the numpy restatement in denoise_ref.py on a synthetic frame, the ABI 8 surface, and the command line's check of --denoise."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import denoise_ref as R
import host_harness
from luisarender_b200 import _ffi as F

REPO = Path(__file__).resolve().parents[1]
f32 = np.float32
W, H = 64, 48


@pytest.fixture(scope="module")
def lib():
    handle = host_harness.load("denoise_host", [host_harness.DEVICE / h for h in ("denoise.h", "adaptive.h")], ["-O2", "-ffp-contract=off"])
    handle.denoise_guides_host.argtypes = [C.c_int64] + [C.c_void_p] * 5
    handle.denoise_normal_weight_host.argtypes = [C.c_int64] + [C.c_void_p] * 5
    handle.denoise_host.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 5
    return handle


def synthetic_frame(seed=11):
    """A seeded 64x48 frame of G-buffer sums and a noisy film: three regions with their own albedo, normal and depth, a coverage
    hole (samples that hit nothing), partly covered pixels along its border, and one pixel with a single sample (infinite variance)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    region = np.where(x < 24, 0, np.where(y < 20, 1, 2))
    s = rng.integers(8, 33, (H, W)).astype(f32)
    s[30, 40] = 1.0
    base_albedo = np.array([[0.8, 0.2, 0.1], [0.1, 0.6, 0.9], [0.5, 0.5, 0.5]], f32)
    base_normal = np.array([[0.0, 0.0, 1.0], [0.6, 0.0, 0.8], [0.0, -1.0, 0.0]], f32)
    base_depth = np.array([2.0, 5.0, 3.5], f32)
    hit_frac = np.ones((H, W), f32)
    hit_frac[8:16, 40:56] = 0.0  # the hole
    hit_frac[7, 40:56] = hit_frac[16, 40:56] = 0.5
    hits = np.floor(s * hit_frac).astype(f32)
    jitter = lambda scale, shape: rng.normal(0.0, scale, shape).astype(f32)  # noqa: E731
    albedo = (base_albedo[region] + jitter(0.02, (H, W, 3))).clip(0, 1).astype(f32)
    normal = base_normal[region] + jitter(0.05, (H, W, 3))
    depth = (base_depth[region] + jitter(0.05, (H, W))).astype(f32)
    albedo_sum = np.concatenate([albedo * hits[..., None], s[..., None]], axis=-1).astype(f32)
    normal_sum = np.concatenate([normal * hits[..., None], (depth * hits)[..., None]], axis=-1).astype(f32)
    shade = (0.5 + 0.5 * np.sin(x / 7.0) * np.cos(y / 5.0)).astype(f32)
    colour = (albedo * shade[..., None] * hit_frac[..., None] + (1 - hit_frac[..., None]) * f32(0.3)).astype(f32)
    colour = (colour * rng.gamma(4.0, 0.25, (H, W, 1))).astype(f32)
    film = np.concatenate([colour, np.ones((H, W, 1), f32)], axis=-1).astype(f32)
    v = rng.lognormal(-6.0, 1.5, (H, W)).astype(f32)
    v[30, 40] = np.inf
    return albedo_sum, normal_sum, hits, film, v


def test_guides_match_numpy_bit_for_bit(lib):
    albedo_sum, normal_sum, hits, _, _ = synthetic_frame()
    albedo_sum[0, 0] = 0.0  # a pixel without samples: all guides 0
    normal_sum[0, 0] = hits[0, 0] = 0.0
    n = W * H
    ac, nd = np.zeros((H, W, 4), f32), np.zeros((H, W, 4), f32)
    lib.denoise_guides_host(n, albedo_sum.ctypes.data, normal_sum.ctypes.data, hits.ctypes.data, ac.ctypes.data, nd.ctypes.data)
    want_ac, want_nd = R.guides(albedo_sum, normal_sum, hits)
    assert np.array_equal(ac.view(np.uint32), want_ac.view(np.uint32))
    assert np.array_equal(nd.view(np.uint32), want_nd.view(np.uint32))
    assert (ac[0, 0] == 0).all() and (nd[0, 0] == 0).all() and (ac[8:16, 40:56, 3] == 0).all() and (nd[8:16, 40:56] == 0).all()


def test_normal_weight_is_bit_exact(lib):
    rng = np.random.default_rng(3)
    n = 200_000
    a = rng.normal(size=(n, 4)).astype(f32)
    b = (a + rng.normal(0.0, 0.1, (n, 4))).astype(f32)
    for v in (a, b):
        v[:, :3] /= np.linalg.norm(v[:, :3], axis=1, keepdims=True)
    cov_a = rng.choice(np.array([0.0, 0.25, 1.0], f32), n)
    cov_b = rng.choice(np.array([0.0, 0.5, 1.0], f32), n)
    a, b = np.ascontiguousarray(a, f32), np.ascontiguousarray(b, f32)
    w = np.zeros(n, f32)
    lib.denoise_normal_weight_host(n, a.ctypes.data, cov_a.ctypes.data, b.ctypes.data, cov_b.ctypes.data, w.ctypes.data)
    want = R.normal_weight(a, cov_a, b, cov_b)
    assert np.array_equal(w.view(np.uint32), want.view(np.uint32))
    assert (w[(cov_a == 0) & (cov_b == 0)] == 1).all() and (w[(cov_a == 0) != (cov_b == 0)] == 0).all()
    assert ((w > 0) & (w < 1)).sum() > n // 10


def test_filter_matches_numpy(lib):
    albedo_sum, normal_sum, hits, film, v = synthetic_frame()
    ac, nd = R.guides(albedo_sum, normal_sum, hits)
    ac, nd, film, v = (np.ascontiguousarray(a, f32) for a in (ac, nd, film, v))
    out = np.zeros((H, W, 4), f32)
    lib.denoise_host(W, H, film.ctypes.data, ac.ctypes.data, nd.ctypes.data, v.ctypes.data, out.ctypes.data)
    want = R.denoise(film, ac, nd, v)
    assert np.isfinite(out).all() and (out[..., 3] == 1).all()
    rel = np.abs(out[..., :3].astype(np.float64) - want[..., :3]) / np.maximum(np.abs(want[..., :3]).astype(np.float64), 1e-30)
    assert rel.max() <= 1e-6, float(rel.max())
    # the filter did something: smoother than its input inside a region, and the hole stays apart from the surfaces around it
    assert np.std(out[25:45, 30:60, 0]) < 0.7 * np.std(film[25:45, 30:60, 0])
    assert np.allclose(out[9:15, 42:54, :3], f32(0.3) * np.mean(film[9:15, 42:54, :3] / f32(0.3)), rtol=0.5)


def test_abi_8_surface(tmp_path):
    assert F.LRK_ABI_VERSION == 8
    assert {"lrk_download_gbuffer", "lrk_denoise"} <= set(F.LRK_SYMBOLS)
    lib = F.device_lib()
    assert lib.lrk_abi_version() == 8
    assert lib.lrk_download_gbuffer.argtypes == [C.c_void_p] * 4 and lib.lrk_denoise.argtypes == [C.c_void_p] * 2
    # the declarations compile against calls with the documented argument types
    src = tmp_path / "abi8.c"
    src.write_text("\n".join([
        f'#include "{REPO / "include" / "lrk.h"}"',
        "int (*gb)(lrk_ctx *, float *, float *, float *) = lrk_download_gbuffer;",
        "int (*dn)(lrk_ctx *, float *) = lrk_denoise;",
        "_Static_assert(LRK_ABI_VERSION == 8u, \"ABI 8\");",
        "int main(void) { return gb == 0 || dn == 0; }"]))
    subprocess.run(["gcc", "-Werror", "-c", str(src), "-o", str(tmp_path / "abi8.o")], check=True)
    # null context / buffers are rejected without a device
    assert lib.lrk_denoise(None, None) != 0 and lib.lrk_download_gbuffer(None, None, None, None) != 0


@pytest.mark.parametrize("args, env", [(["--denoise", "--gpus", "2"], {}), (["--gpus", "2", "--denoise"], {}), (["--denoise"], {"WORLD_SIZE": "2"})])
def test_cli_rejects_denoise_on_several_gpus_before_reading_the_scene(tmp_path, args, env):
    """The check runs before the scene is read or a device is created: the scene file named here does not even exist."""
    import os

    cli = F.LIB_DIR / "luisa-render-cli"
    r = subprocess.run([str(cli), "-b", "cuda", *args, str(tmp_path / "missing.luisa")], capture_output=True, text=True, timeout=60,
                       env={**os.environ, **env})
    assert r.returncode == 255, (r.returncode, r.stdout, r.stderr)
    assert "[error] --denoise" in r.stderr and "Parsed" not in r.stdout
