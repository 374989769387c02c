"""The adaptive mode without a GPU: the pixel error the device computes (csrc/device/adaptive.h, compiled for the host) against a
numpy fp32 restatement, the C layout of lrk_adaptive against its ctypes mirror, and the command line's checks of --adaptive."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

from luisarender_b200 import _ffi as F

REPO = Path(__file__).resolve().parents[1]
SRC = REPO / "tests" / "host_device" / "adaptive_host.cpp"
OUT = REPO / "tests" / "host_device" / "_build" / "libadaptive_host.so"
HEADER = REPO / "luisarender_b200" / "csrc" / "device" / "adaptive.h"


@pytest.fixture(scope="module")
def lib():
    if not OUT.exists() or OUT.stat().st_mtime < max(SRC.stat().st_mtime, HEADER.stat().st_mtime):
        OUT.parent.mkdir(parents=True, exist_ok=True)
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-shared", str(SRC), "-o", str(OUT)], check=True)
    handle = C.CDLL(str(OUT))
    handle.adaptive_error_host.argtypes = [C.c_void_p] * 5 + [C.c_int64]
    return handle


def error_and_variance(s1, s2, n):
    """The rule of include/lrk.h in numpy fp32, one rounded operation at a time."""
    f = np.float32
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        m = s1 / n
        v = np.maximum(s2 / n - m * m, f(0)) / (n - f(1))
        e = np.sqrt(v) / np.maximum(m, f(0.01))
    few = ~(n >= f(2))
    return np.where(few, f(np.inf), e).astype(f), np.where(few, f(np.inf), v).astype(f)


def test_pixel_error_matches_numpy_fp32_bit_for_bit(lib):
    rng = np.random.default_rng(7)
    count = 100_000
    n = rng.integers(2, 4097, count).astype(np.float32)
    n[: count // 10] = 2.0  # the smallest sample count that has an estimate
    n[-100:] = rng.choice(np.array([0.0, 1.0], np.float32), 100)  # no estimate: +inf
    mean = rng.lognormal(-1.0, 2.0, count).astype(np.float32)
    mean[count // 10: count // 5] = 0.0  # m = 0: a black pixel
    spread = rng.uniform(0.0, 3.0, count).astype(np.float32)
    s1 = (mean * n).astype(np.float32)
    s2 = (n * (mean * mean + spread * mean * mean)).astype(np.float32)
    low = slice(count // 5, count // 5 + count // 10)  # S2 / n < m^2 by a few ulps: rounding of a noiseless pixel
    s2[low] = (s1[low] * s1[low] / n[low] * np.float32(1 - 3e-7)).astype(np.float32)
    mid = slice(count // 2, count // 2 + 1000)  # m = 0 with S2 > 0 cannot come from a film, but the function is total
    s1[mid] = 0.0
    s1, s2 = np.ascontiguousarray(s1), np.ascontiguousarray(s2)
    e, v = np.zeros(count, np.float32), np.zeros(count, np.float32)
    assert lib.adaptive_error_host(s1.ctypes.data, s2.ctypes.data, n.ctypes.data, e.ctypes.data, v.ctypes.data, count) == 0
    want_e, want_v = error_and_variance(s1, s2, n)
    with np.errstate(divide="ignore", invalid="ignore"):
        assert (s2[low] / n[low] < (s1[low] / n[low]) ** 2).sum() > 1000  # the clamp at 0 is exercised
    assert np.isinf(want_e).sum() >= 100 and np.isfinite(want_e).sum() > 0.9 * count
    assert np.array_equal(e.view(np.uint32), want_e.view(np.uint32)), int((e.view(np.uint32) != want_e.view(np.uint32)).sum())
    assert np.array_equal(v.view(np.uint32), want_v.view(np.uint32)), int((v.view(np.uint32) != want_v.view(np.uint32)).sum())


def test_adaptive_struct_layout_matches_c(tmp_path):
    src = tmp_path / "sizes.c"
    src.write_text("\n".join([
        "#include <stdio.h>", "#include <stddef.h>", f'#include "{REPO / "include" / "lrk.h"}"', "int main(void){",
        'printf("%zu %zu %zu %zu\\n", sizeof(lrk_adaptive), offsetof(lrk_adaptive, max_spp), offsetof(lrk_adaptive, threshold), '
        'offsetof(lrk_adaptive, reserved));', "return 0;}"]))
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(F.Adaptive), F.Adaptive.max_spp.offset, F.Adaptive.threshold.offset, F.Adaptive.reserved.offset]


@pytest.mark.parametrize("args", [["--adaptive", "-1"], ["--adaptive", "nan"], ["--adaptive", "inf"], ["--adaptive", "0.01x"],
                                  ["--adaptive", "0.01", "--adaptive-min-spp", "1"], ["--adaptive-min-spp", "8"]])
def test_cli_rejects_bad_adaptive_options_before_reading_the_scene(tmp_path, args):
    """The checks run before the scene is read or a device is created: the scene file named here does not even exist."""
    cli = F.LIB_DIR / "luisa-render-cli"
    r = subprocess.run([str(cli), "-b", "cuda", *args, str(tmp_path / "missing.luisa")], capture_output=True, text=True, timeout=60)
    assert r.returncode == 255, (r.returncode, r.stdout, r.stderr)
    assert "[error] --adaptive" in r.stderr and "Parsed" not in r.stdout
