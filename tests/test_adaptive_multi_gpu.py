"""Adaptive sampling on two GPUs, one process each: every rank renders its tiles adaptively, lrk_reduce_film sums the films, and
the result - film and sample counts - is bit-identical to one GPU rendering the whole frame (blocks never cross tiles, so every
stopping decision has exactly one owner).  Skipped on a single-GPU machine, like tests/test_multi_gpu.py."""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

import pytest

REPO = Path(__file__).resolve().parents[1]

pytestmark = pytest.mark.gpu


def _gpus() -> int:
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


WORKER = r"""
import os, sys
import numpy as np
sys.path.insert(0, os.environ["LRB_REPO"])
import torch
from luisarender_b200 import scenes, distributed as D
from luisarender_b200.api import Renderer, Scene

rank, world, local = D.env_world()
torch.cuda.set_device(local)
dist = D.init_process_group("nccl")
scene = Scene.from_source(scenes.instanced_spheres(resolution=(640, 360), spp=64), os.environ["LRB_REPO"])
r = Renderer(device_index=local)
r.upload(scene.desc())
D.init_film_comm(r, rank, world)
r.set_shard(rank, world, D.TILE_SIZE)
r.render_adaptive(0.05, 4, 64)
counts = torch.from_numpy(r.sample_counts().astype(np.int64)).cuda()
dist.all_reduce(counts)
r.reduce_film(0)
if rank == 0:
    reduced = r.film(raw=True).copy()
    r.set_shard(0, 1, D.TILE_SIZE)
    r.render_adaptive(0.05, 4, 64)
    single = r.film(raw=True)
    assert len(np.unique(r.sample_counts())) >= 2
    assert np.array_equal(reduced.view(np.uint32), single.view(np.uint32)), float(np.abs(reduced - single).max())
    assert np.array_equal(counts.cpu().numpy(), r.sample_counts().astype(np.int64))
dist.barrier()
dist.destroy_process_group()
"""


def test_two_rank_adaptive_render_is_bit_identical_to_one_gpu(tmp_path):
    if _gpus() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, LRB_REPO=str(REPO))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29543", str(script)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
