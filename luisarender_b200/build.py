"""In-tree build of the native libraries (no pip, no JIT cache: the .so files travel with the repo snapshot).

  lib/libluisa_render_host.so   host front-end  (g++, csrc/host/*.cpp)          include/lrh.h
  lib/libb200pt.so              device library  (nvcc sm_90a, csrc/device)     include/lrk.h
  lib/luisa-render-cli          command-line front-end (links both)
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import time
from pathlib import Path

PKG = Path(__file__).resolve().parent
REPO = PKG.parent
LIB = PKG / "lib"
HOST_SRC = ["sdl.cpp", "scene.cpp", "geomutil.cpp", "bvh.cpp", "flatten.cpp", "imageio.cpp", "imageload.cpp", "jpegload.cpp", "meshload.cpp", "envmap.cpp", "lrh.cpp"]
NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
# the strict shade.cu object takes about 12 minutes on 8 cores: the device build reports progress at this interval, so that a
# caller watching its output can tell a long compile from a hung one
PROGRESS_SECONDS = 60
# -fmad=false: expressions evaluate as written (see csrc/device/vecmath.cuh); FMAs are explicit fmaf().
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-fmad=false", "--shared", "-Xcompiler", "-fPIC"]
SHADE_MATH = ["--use_fast_math"]  # arithmetic of shade.cu (see its header)
HOST_FLAGS = ["-std=c++17", "-O2", "-fPIC", "-march=x86-64-v3", "-ffp-contract=off", "-Wall", "-Wextra",
              "-Wno-unused-parameter", "-Wno-missing-field-initializers"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def _newer(target: Path, sources) -> bool:
    if not target.exists():
        return False
    t = target.stat().st_mtime
    return all(Path(s).stat().st_mtime <= t for s in sources)


def _run(cmd, verbose):
    if verbose:
        print("+", " ".join(str(c) for c in cmd), flush=True)
    r = subprocess.run([str(c) for c in cmd], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError(f"build step failed: {' '.join(str(c) for c in cmd[:3])} ...")
    return r


def build_host(force=False, verbose=False) -> Path:
    out = LIB / "libluisa_render_host.so"
    src_dir = PKG / "csrc" / "host"
    deps = list(src_dir.glob("*.cpp")) + list(src_dir.glob("*.h")) + list((REPO / "include").glob("*.h"))
    deps.append(PKG / "csrc" / "device" / "affine_inverse.h")  # shared with the device library (flatten.cpp)
    deps.append(PKG / "csrc" / "device" / "alias_table.h")  # shared with the device library (flatten.cpp, geomutil users)
    if not force and _newer(out, deps):
        return out
    LIB.mkdir(exist_ok=True)
    _run(["g++", *HOST_FLAGS, "-shared", *[src_dir / s for s in HOST_SRC], "-o", out, "-lpthread", "-lz", "-ldl"], verbose)
    return out


def build_device(force=False, verbose=False, name="libb200pt.so", extra_flags=()) -> Path:
    """libb200pt.so = lrk.cu + shade.cu (twice).  lrk.cu (ray generation, traversal, classification, film, the host API) is compiled
    with IEEE arithmetic and no FMA contraction: bit-exact with the oracle.  shade.cu (the closure kernels) is compiled once with
    nvcc's fast-math arithmetic, as the reference's CUDA backend compiles all of its kernels, and once like lrk.cu (see the
    header of shade.cu; lrk_set_option("strict_math") selects at run time)."""
    out = LIB / name
    src_dir = PKG / "csrc" / "device"
    deps = list(src_dir.glob("*.cu")) + list(src_dir.glob("*.cuh")) + list(src_dir.glob("*.h")) + list((REPO / "include").glob("*.h"))
    if not force and _newer(out, deps):
        return out
    LIB.mkdir(exist_ok=True)
    obj = LIB / ("_obj_" + Path(name).stem)
    obj.mkdir(exist_ok=True)
    common = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", *extra_flags]
    shade_math = ["-fmad=false"] if os.environ.get("LRK_SHADE_STRICT") == "1" else SHADE_MATH
    if os.environ.get("LRK_SHADE_FLAGS"):  # experiments (tools/build_variants.sh)
        shade_math = os.environ["LRK_SHADE_FLAGS"].split()
    objects = [obj / "lrk.o", obj / "shade_fast.o", obj / "shade_strict.o"]
    # lrk.cu's host code rebuilds alias tables (alias_table.h) as the host library computes them: no FMA contraction there either
    steps = [([_nvcc(), *NVCC_ARCH, *common, "-fmad=false", "-Xcompiler", "-ffp-contract=off", "-c", src_dir / "lrk.cu", "-o", objects[0]], None),
             ([_nvcc(), *NVCC_ARCH, *common, *shade_math, "-DLRK_SHADE_VARIANT=fast", "-c", src_dir / "shade.cu", "-o", objects[1]], None),
             ([_nvcc(), *NVCC_ARCH, *common, "-fmad=false", "-DLRK_SHADE_VARIANT=strict", "-c", src_dir / "shade.cu", "-o", objects[2]], None)]
    procs = []
    start = time.monotonic()
    for cmd, _ in steps:  # the three objects compile side by side
        if verbose:
            print("+", " ".join(str(c) for c in cmd), flush=True)
        procs.append((cmd, subprocess.Popen([str(c) for c in cmd], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    print(f"[build] compiling {', '.join(o.name for o in objects)} for sm_90a", flush=True)
    for cmd, proc in procs:
        while True:
            try:
                text, _ = proc.communicate(timeout=PROGRESS_SECONDS)
                break
            except subprocess.TimeoutExpired:
                print(f"[build] still compiling {Path(cmd[-1]).name} ({time.monotonic() - start:.0f} s)", flush=True)
        print(f"[build] {Path(cmd[-1]).name} done ({time.monotonic() - start:.0f} s)", flush=True)
        if proc.returncode != 0:
            sys.stderr.write(text)
            raise RuntimeError(f"build step failed: {' '.join(str(c) for c in cmd[:3])} ...")
    _run([_nvcc(), *NVCC_ARCH, "--shared", *objects, "-o", out], verbose)
    return out


def build_cli(force=False, verbose=False) -> Path:
    out = LIB / "luisa-render-cli"
    src = PKG / "csrc" / "host" / "cli.cpp"
    if not src.exists():
        return out
    deps = [src, LIB / "libluisa_render_host.so", LIB / "libb200pt.so"]
    if not force and _newer(out, deps):
        return out
    _run(["g++", "-std=c++17", "-O2", src, "-o", out, f"-L{LIB}", "-lluisa_render_host", "-lb200pt",
          "-Wl,-rpath,$ORIGIN", "-lpthread"], verbose)
    return out


def build_all(force=False, verbose=False):
    return [build_host(force, verbose), build_device(force, verbose), build_cli(force, verbose)]


if __name__ == "__main__":
    for p in build_all(force="--force" in sys.argv, verbose=True):
        print(p)
