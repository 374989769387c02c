"""The option "time_kernels" (include/lrk.h): CUDA-event time per kernel category in stats().  Timing only observes: a render with it
gives the film and the launch count of the render without it, and every category that the scene's pass launches kernels in reports
time, the others none."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

from luisarender_b200 import scenes
from luisarender_b200.api import Scene

pytestmark = pytest.mark.gpu
REPO = Path(__file__).resolve().parents[1]

CATEGORIES = ("trace_closest_ms", "trace_shadow_ms", "shade_ms", "other_ms")
# scene and the categories its passes launch kernels in
SCENES = {
    "surface": (lambda: scenes.cornell_box(resolution=(48, 48), spp=8), CATEGORIES),
    "c4_medium": (lambda: scenes.instanced_spheres(resolution=(64, 36), spp=4, medium=True, depth=8, big_subdivision=3, small_subdivision=2,
                                                   small_count=12), CATEGORIES),
    "shape_media": (lambda: scenes.media_box(resolution=(40, 40), spp=4), ("shade_ms", "other_ms")),  # one kernel per sample, then the film
}


@pytest.mark.parametrize("name", list(SCENES))
def test_kernel_timing_leaves_the_render_alone(name, gpu_renderer):
    source, timed_categories = SCENES[name]
    scene = Scene.from_source(source(), REPO)
    d = scene.desc()
    gpu_renderer.upload(d)
    runs = {}
    try:
        for timing in (0, 1):
            gpu_renderer.set_option("time_kernels", timing)
            gpu_renderer.clear()
            gpu_renderer.render(0, d.camera.spp)
            runs[timing] = gpu_renderer.film(raw=True), gpu_renderer.stats()
    finally:
        gpu_renderer.set_option("time_kernels", 0)
    (film_off, off), (film_on, on) = runs[0], runs[1]
    assert np.array_equal(film_on, film_off)
    assert on["kernel_launches"] == off["kernel_launches"] > 0 and on["passes"] == off["passes"] >= 1
    for c in CATEGORIES:
        assert off[c] == 0.0, c
        assert (on[c] > 0.0) if c in timed_categories else (on[c] == 0.0), (c, on[c])
