"""The host harnesses of tests/host_device: C++ files that include device headers, compiled with g++ for the tests that check those
headers without a GPU."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import pytest

REPO = Path(__file__).resolve().parents[1]
DEVICE = REPO / "luisarender_b200" / "csrc" / "device"
CUDA_INCLUDE = Path("/usr/local/cuda/include")


def cuda_include_flag() -> str:
    """g++'s -I for the CUDA headers that the .cuh files include; skips the calling test where they are missing."""
    if not (CUDA_INCLUDE / "cuda_runtime.h").exists():
        pytest.skip("CUDA headers not found")
    return f"-I{CUDA_INCLUDE}"


def load(name: str, deps, flags) -> C.CDLL:
    """tests/host_device/<name>.cpp as a shared library, rebuilt with `g++ -std=c++17 -fPIC -shared <flags>` when it is missing or
    older than the source or one of `deps`."""
    src = REPO / "tests" / "host_device" / f"{name}.cpp"
    out = REPO / "tests" / "host_device" / "_build" / f"lib{name}.so"
    if not out.exists() or out.stat().st_mtime < max(p.stat().st_mtime for p in [src, *deps]):
        out.parent.mkdir(parents=True, exist_ok=True)
        subprocess.run(["g++", "-std=c++17", "-fPIC", "-shared", *flags, str(src), "-o", str(out)], check=True)
    return C.CDLL(str(out))
