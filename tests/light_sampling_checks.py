"""What the tests of next-event light sampling share (test_light_tree*.py, test_light_solid_angle*.py): the checks of an option's
surface in Python and on the command line and, for the GPU tests, renders under a set of light-sampling options and the statistics
that compare two such settings.

A setting is a dict of options, e.g. {"light_tree": 1}; options it leaves out keep their value on the renderer."""
from __future__ import annotations

import subprocess

import numpy as np
import pytest

BLOCK = 16


def check_python_option_rejects_bad_values(option, **needs):
    """Renderer(**needs, option=bad) raises ValueError for values other than False / True, before a device is looked for."""
    from luisarender_b200.api import Renderer

    for bad in (2, -1, "yes", 0.5):
        with pytest.raises(ValueError):
            Renderer(**needs, **{option: bad})


def check_cli_lists_and_parses_flag(flag, tmp_path):
    from luisarender_b200 import _ffi as F

    cli = F.LIB_DIR / "luisa-render-cli"
    r = subprocess.run([str(cli), "--help"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and flag in r.stdout
    # the flag parses: the run gets as far as reading the scene, which does not exist
    r = subprocess.run([str(cli), "-b", "cuda", flag, str(tmp_path / "missing.luisa")], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "Unrecognized options" not in r.stderr and "[error]" in r.stderr

# Unbiasedness checks compare the means of the image and of its 16 x 16 blocks over 32 + 32 sub-renders at 4 sigma: for a normal
# estimate each comparison fails with probability 6e-5, with sigma estimated from the sub-renders (t, 62 dof) 1.7e-4, so the
# many-light frame (1 + 32 means) fails by chance about 0.6 % of the time (the renders are seeded, so a given seed passes or fails
# for good).
SUBRENDERS, SUB_SPP, Z_MAX = 32, 16, 4.0


@pytest.fixture
def r(gpu_renderer):
    """gpu_renderer, with the options these tests touch back at their defaults afterwards (the renderer is shared by the session)."""
    yield gpu_renderer
    for name, value in (("light_tree_triangles", 0), ("light_tree", 0), ("light_solid_angle", 0), ("gbuffer", 0),
                        ("max_paths_per_pass", 136 << 20)):
        gpu_renderer.set_option(name, value)
    gpu_renderer.set_shard(0, 1, 32)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def upload(r, desc, options):
    for name, value in options.items():
        r.set_option(name, int(value))
    r.upload(desc)


def render(r, desc, spp_begin, spp_end, options, raw=True):
    upload(r, desc, options)
    r.render(spp_begin, spp_end)
    return r.film(raw=raw).copy()


def sub_renders(r, desc, options, first, count, spp):
    """`count` independent renders of `spp` samples each from sample index `first` on, as normalised films [count, H, W, 3]: one
    upload, then a cleared film per render."""
    upload(r, desc, options)
    films = []
    for k in range(count):
        r.clear()
        r.render(first + k * spp, first + (k + 1) * spp)
        films.append(r.film(raw=False)[..., :3].copy())
    return np.stack(films).astype(np.float64)


def reference(r, desc, options):
    """The 1024-spp film of sample indices [2^20, 2^20 + 1024), disjoint from those of the renders it is compared with."""
    return sub_renders(r, desc, options, 1 << 20, 1, 1024)[0]


def rel_mse(r, desc, options, ref, first):
    """The relative MSE against `ref` of 16-spp renders, averaged over 8 of them from sample index `first` on."""
    films = sub_renders(r, desc, options, first, 8, 16)
    return float(np.mean([((f - ref) ** 2 / (ref ** 2 + 1e-2)).mean() for f in films]))


def block_means(films):
    n, h, w, _ = films.shape
    hb, wb = h // BLOCK, w // BLOCK
    b = films[:, :hb * BLOCK, :wb * BLOCK].reshape(n, hb, BLOCK, wb, BLOCK, 3).mean(axis=(2, 4, 5)).reshape(n, -1)
    return np.concatenate([films.mean(axis=(1, 2, 3))[:, None], b], axis=1)  # column 0: the whole image


def z_scores(a, b):
    """(mean a - mean b) / its standard error, per block, from the spread of the independent sub-renders.  A block without noise in
    either (the black background) gives 0 if the means agree, else inf."""
    ma, mb = block_means(a), block_means(b)
    se = np.sqrt(ma.var(axis=0, ddof=1) / len(ma) + mb.var(axis=0, ddof=1) / len(mb))
    diff = ma.mean(axis=0) - mb.mean(axis=0)
    return np.where(se > 0, diff / np.where(se > 0, se, 1.0), np.where(diff == 0, 0.0, np.inf))
