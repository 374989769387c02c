"""What the GPU tests that compare a full-size frame with the oracle on a shard of its tiles share (test_sampler_ranges.py,
test_bench_shapes.py): the shard, and a copy of a scene description with another path depth."""
from __future__ import annotations

from luisarender_b200 import _ffi as F
from luisarender_b200.distributed import tile_owner

TILE = 32


def with_depth(d, depth: int):
    """A copy of the description with another max_depth (the arrays stay the scene's)."""
    c = F.SceneDesc.from_buffer_copy(d)
    c.integrator.max_depth = depth
    return c


def shard(d):
    """(rank, world): a shard of about 32 tiles that owns the frame's last tile, so it holds tiles of the last row and column."""
    w, h = d.camera.resolution[0], d.camera.resolution[1]
    tiles = ((w + TILE - 1) // TILE) * ((h + TILE - 1) // TILE)
    world = max(tiles // 32, 1)
    return int(tile_owner(tiles - 1, world)), world
