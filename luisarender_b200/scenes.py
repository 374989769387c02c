"""Synthetic scene generators (SURVEY.md §8d "Synthetic inputs").

Both scenes are emitted as LuisaRender scene-description text (.luisa grammar,
/root/reference/src/sdl/scene_parser.cpp:72-451) so the *same file* would load in the reference.

* ``cornell_box``  — configs C1/C2: the 16 quads (32 triangles) of the Cornell box fixture embedded in
  the LuisaCompute path-tracing demo (src/compute/src/tests/common/cornell_box.h:17-145, minus the two
  never-visible "Bottom Face" quads), colours / camera / emission from
  src/compute/src/tests/test_path_tracing.cpp:104-113,159-160,192.
* ``instanced_spheres`` — configs C3-C5: one level-7 icosphere (327 680 triangles) instanced 4x
  (1 310 720 triangles) + 60 level-3 spheres + a ground quad, 8 Disney surfaces, 2 one-sided quad area
  lights; all random numbers from ``numpy.random.default_rng(seed)``.
"""
from __future__ import annotations

import numpy as np

# quads as (name, [4 vertices]); triangulated (0,1,2),(0,2,3)
_CORNELL_QUADS = {
    "floor": [[(-1.01, 0.00, 0.99), (1.00, 0.00, 0.99), (1.00, 0.00, -1.04), (-0.99, 0.00, -1.04)]],
    "ceiling": [[(-1.02, 1.99, 0.99), (-1.02, 1.99, -1.04), (1.00, 1.99, -1.04), (1.00, 1.99, 0.99)]],
    "back_wall": [[(-0.99, 0.00, -1.04), (1.00, 0.00, -1.04), (1.00, 1.99, -1.04), (-1.02, 1.99, -1.04)]],
    "right_wall": [[(1.00, 0.00, -1.04), (1.00, 0.00, 0.99), (1.00, 1.99, 0.99), (1.00, 1.99, -1.04)]],
    "left_wall": [[(-1.01, 0.00, 0.99), (-0.99, 0.00, -1.04), (-1.02, 1.99, -1.04), (-1.02, 1.99, 0.99)]],
    "short_box": [
        [(0.53, 0.60, 0.75), (0.70, 0.60, 0.17), (0.13, 0.60, 0.00), (-0.05, 0.60, 0.57)],
        [(-0.05, 0.00, 0.57), (-0.05, 0.60, 0.57), (0.13, 0.60, 0.00), (0.13, 0.00, 0.00)],
        [(0.53, 0.00, 0.75), (0.53, 0.60, 0.75), (-0.05, 0.60, 0.57), (-0.05, 0.00, 0.57)],
        [(0.70, 0.00, 0.17), (0.70, 0.60, 0.17), (0.53, 0.60, 0.75), (0.53, 0.00, 0.75)],
        [(0.13, 0.00, 0.00), (0.13, 0.60, 0.00), (0.70, 0.60, 0.17), (0.70, 0.00, 0.17)],
    ],
    "tall_box": [
        [(-0.53, 1.20, 0.09), (0.04, 1.20, -0.09), (-0.14, 1.20, -0.67), (-0.71, 1.20, -0.49)],
        [(-0.53, 0.00, 0.09), (-0.53, 1.20, 0.09), (-0.71, 1.20, -0.49), (-0.71, 0.00, -0.49)],
        [(-0.71, 0.00, -0.49), (-0.71, 1.20, -0.49), (-0.14, 1.20, -0.67), (-0.14, 0.00, -0.67)],
        [(-0.14, 0.00, -0.67), (-0.14, 1.20, -0.67), (0.04, 1.20, -0.09), (0.04, 0.00, -0.09)],
        [(0.04, 0.00, -0.09), (0.04, 1.20, -0.09), (-0.53, 1.20, 0.09), (-0.53, 0.00, 0.09)],
    ],
    "light": [[(-0.24, 1.98, 0.16), (-0.24, 1.98, -0.22), (0.23, 1.98, -0.22), (0.23, 1.98, 0.16)]],
}

_CORNELL_COLORS = {
    "white": (0.725, 0.710, 0.680),
    "green": (0.140, 0.450, 0.091),
    "red": (0.630, 0.065, 0.050),
}

_CORNELL_SURFACE_OF = {
    "floor": "white", "ceiling": "white", "back_wall": "white", "right_wall": "green",
    "left_wall": "red", "short_box": "white", "tall_box": "white",
}


def _fmt(x: float) -> str:
    return repr(float(x))


def _mesh_props(quads) -> tuple[str, str]:
    positions, indices = [], []
    for q in quads:
        base = len(positions) // 3
        for v in q:
            positions.extend(v)
        indices.extend([base, base + 1, base + 2, base, base + 2, base + 3])
    return ", ".join(_fmt(p) for p in positions), ", ".join(str(i) for i in indices)


def cornell_box(resolution=(512, 512), spp=16, depth=10, rr_depth=0, rr_threshold=0.95,
                integrator="WavePath", seed=19980810, output="cornell.exr", surface="Matte") -> str:
    """Configs C1 (512x512 @16) and C2 (1024x1024 @4096). ``surface`` may be "Matte" or "Disney"
    (the latter is only used by tests to exercise the Disney closure on simple geometry)."""
    out = []
    for name, rgb in _CORNELL_COLORS.items():
        key = "Kd" if surface == "Matte" else "color"
        out.append(f"Surface {name} : {surface} {{ {key} : Constant {{ v {{ {_fmt(rgb[0])}, {_fmt(rgb[1])}, {_fmt(rgb[2])} }} }} }}")
    out.append("Light area_light : Diffuse { emission : Constant { v { 17.0, 12.0, 4.0 } } }")
    shape_names = []
    for name, quads in _CORNELL_QUADS.items():
        positions, indices = _mesh_props(quads)
        binding = "light { @area_light }" if name == "light" else f"surface {{ @{_CORNELL_SURFACE_OF[name]} }}"
        out.append(f"Shape {name} : InlineMesh {{\n  positions {{ {positions} }}\n  indices {{ {indices} }}\n  {binding}\n}}")
        shape_names.append(f"@{name}")
    out.append(f"""Camera camera : Pinhole {{
  position {{ -0.01, 0.995, 5.0 }}
  front {{ 0.0, 0.0, -1.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 27.8 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}""")
    out.append(f"""render {{
  integrator : {integrator} {{
    depth {{ {int(depth)} }}
    rr_depth {{ {int(rr_depth)} }}
    rr_threshold {{ {_fmt(rr_threshold)} }}
    sampler : Independent {{ seed {{ {int(seed)} }} }}
  }}
  cameras {{ @camera }}
  shapes {{ {", ".join(shape_names)} }}
}}""")
    return "\n".join(out) + "\n"


def instanced_spheres(resolution=(1920, 1080), spp=1024, seed=1, depth=10, rr_depth=0, rr_threshold=0.95,
                      big_subdivision=7, big_count=4, small_subdivision=3, small_count=60, medium=False,
                      integrator=None, sampler_seed=19980810, output="spheres.exr", emissive=0, shared_light_node=False,
                      emission_spread=True, time=0.0) -> str:
    """Configs C3 (1920x1080 @1024), C4 (+ homogeneous medium, depth 8, 3840x2160 @4096) and C5.
    4 x 327 680 + 60 x 1 280 + 2 (ground) + 4 (lights) = 1 387 526 instanced triangles.

    ``emissive=K`` also makes the first K small spheres one-sided emitters (see ``many_lights``): each with its own Light node whose
    emission is log-uniform over two orders of magnitude (``emission_spread``) or 4.0, or all K sharing one node of emission 4.0
    (``shared_light_node``).  The defaults emit the scene without them, unchanged.

    ``time`` makes the scene one frame of an animation: every ``big_*`` / ``small_*`` instance is translated by ``time`` x its own
    horizontal velocity (up to 1 unit per unit of time per axis, from a random stream of its own), so that the frames of one
    ``seed`` share their meshes, surfaces, lights and instance order.  ``time=0.0`` emits the text of the still scene."""
    rng = np.random.default_rng(seed)
    velocity_rng = np.random.default_rng([seed, 2])
    out = []
    emitter_of = {}
    if emissive:
        assert not (shared_light_node and emission_spread), "a shared light node has one emission"
        levels = np.random.default_rng(seed + 7919).uniform(-1.0, 1.0, emissive) if emission_spread else np.zeros(emissive)
        for i in range(emissive):
            node = "sphere_light" if shared_light_node else f"sphere_light_{i}"
            emitter_of[i] = node
            if i == 0 or not shared_light_node:
                v = 4.0 * 10.0 ** levels[i]
                out.append(f"Light {node} : Diffuse {{ emission : Constant {{ v {{ {_fmt(v)}, {_fmt(0.8 * v)}, {_fmt(0.6 * v)} }} }} two_sided {{ false }} }}")
    # 8 Disney surfaces, parameters ~ U[0,1]
    for i in range(8):
        color = rng.uniform(0.0, 1.0, 3)
        metallic, roughness, specular_tint, clearcoat, sheen = rng.uniform(0.0, 1.0, 5)
        out.append(
            f"Surface disney_{i} : Disney {{\n"
            f"  color : Constant {{ v {{ {_fmt(color[0])}, {_fmt(color[1])}, {_fmt(color[2])} }} }}\n"
            f"  metallic : Constant {{ v {{ {_fmt(metallic)} }} }}\n"
            f"  roughness : Constant {{ v {{ {_fmt(roughness)} }} }}\n"
            f"  specular_tint : Constant {{ v {{ {_fmt(specular_tint)} }} }}\n"
            f"  clearcoat : Constant {{ v {{ {_fmt(clearcoat)} }} }}\n"
            f"  sheen : Constant {{ v {{ {_fmt(sheen)} }} }}\n"
            f"}}")
    out.append("Surface ground_surface : Disney { color : Constant { v { 0.6, 0.6, 0.6 } } roughness : Constant { v { 0.8 } } }")
    # each light shape has its own Light node (the uniform light sampler counts light NODES,
    # src/lightsamplers/uniform.cpp:34-38)
    out.append("Light light_a : Diffuse { emission : Constant { v { 20.0, 20.0, 20.0 } } two_sided { false } }")
    out.append("Light light_b : Diffuse { emission : Constant { v { 20.0, 20.0, 20.0 } } two_sided { false } }")
    out.append(f"Shape big_sphere : Sphere {{ subdivision {{ {int(big_subdivision)} }} }}")
    out.append(f"Shape small_sphere : Sphere {{ subdivision {{ {int(small_subdivision)} }} }}")
    shapes = []
    # ground quad (y = 0), facing up
    g = 12.0
    pos, idx = _mesh_props([[(-g, 0.0, g), (g, 0.0, g), (g, 0.0, -g), (-g, 0.0, -g)]])
    out.append(f"Shape ground : InlineMesh {{ positions {{ {pos} }} indices {{ {idx} }} surface {{ @ground_surface }} }}")
    shapes.append("@ground")
    # two one-sided quad lights above the scene, facing down
    for name, (cx, cz) in (("a", (-3.0, 1.0)), ("b", (3.5, -2.0))):
        h, s = 9.0, 1.5
        pos, idx = _mesh_props([[(cx - s, h, cz + s), (cx - s, h, cz - s), (cx + s, h, cz - s), (cx + s, h, cz + s)]])
        out.append(f"Shape light_shape_{name} : InlineMesh {{ positions {{ {pos} }} indices {{ {idx} }} light {{ @light_{name} }} }}")
        shapes.append(f"@light_shape_{name}")

    def add_instance(name, base, scale_range, surface_index, light=None):
        p = rng.uniform(-4.0, 4.0, 3)
        s = rng.uniform(*scale_range)
        p[1] = abs(p[1]) + s  # keep spheres above the ground plane
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        angle = rng.uniform(0.0, 360.0)
        velocity = velocity_rng.uniform(-1.0, 1.0, 2)
        if time != 0.0:
            p[0] += time * velocity[0]
            p[2] += time * velocity[1]
        out.append(
            f"Shape {name} : Instance {{\n"
            f"  shape {{ @{base} }}\n"
            f"  surface {{ @disney_{surface_index} }}\n"
            + (f"  light {{ @{light} }}\n" if light else "") +
            f"  transform : SRT {{ scale {{ {_fmt(s)} }} rotate {{ {_fmt(axis[0])}, {_fmt(axis[1])}, {_fmt(axis[2])}, {_fmt(angle)} }} "
            f"translate {{ {_fmt(p[0])}, {_fmt(p[1])}, {_fmt(p[2])} }} }}\n"
            f"}}")
        shapes.append(f"@{name}")

    for i in range(big_count):
        add_instance(f"big_{i}", "big_sphere", (0.7, 1.0), i % 8)
    for i in range(small_count):
        add_instance(f"small_{i}", "small_sphere", (0.2, 0.5), int(rng.integers(0, 8)), emitter_of.get(i))

    out.append(f"""Camera camera : Pinhole {{
  position {{ 0.0, 3.0, 12.0 }}
  look_at {{ 0.0, 1.5, 0.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 45.0 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}""")
    if integrator is None:
        integrator = "MegaVPTNaive" if medium else "WavePath"
    medium_line = ""
    if medium:
        medium_line = ("  environment_medium : Homogeneous {\n"
                       "    sigma_a : Constant { v { 0.01, 0.01, 0.01 } }\n"
                       "    sigma_s : Constant { v { 0.05, 0.05, 0.05 } }\n"
                       "    phasefunction : HenyeyGreenstein { g { 0.3 } }\n"
                       "  }\n")
    out.append(f"""render {{
  integrator : {integrator} {{
    depth {{ {int(depth)} }}
    rr_depth {{ {int(rr_depth)} }}
    rr_threshold {{ {_fmt(rr_threshold)} }}
    sampler : Independent {{ seed {{ {int(sampler_seed)} }} }}
  }}
{medium_line}  cameras {{ @camera }}
  shapes {{ {", ".join(shapes)} }}
}}""")
    return "\n".join(out) + "\n"


def many_lights(resolution=(1920, 1080), spp=64, count=48, shared_node=False, spread=True, **kw) -> str:
    """The many-light frame of the light tree (option "light_tree"): the C3 scene with its two quad lights and ``count`` of its small
    spheres emissive, with emission over two orders of magnitude (``spread``).  ``shared_node=True``: the spheres share one Light
    node, which the reference's uniform sampler counts once (only the first is ever sampled by next-event estimation)."""
    kw.setdefault("big_subdivision", 5)
    return instanced_spheres(resolution=resolution, spp=spp, emissive=count, shared_light_node=shared_node,
                             emission_spread=spread and not shared_node, output="many_lights.exr", **kw)


def near_light(resolution=(512, 512), spp=16, depth=10, rr_depth=0, rr_threshold=0.95, seed=19980810, irradiance=False,
               output="near_light.exr", glossy_desk=False) -> str:
    """The frame of solid-angle light sampling (option "light_solid_angle"): a Matte room with a desk under a one-sided 1.0 x 0.6
    panel light 0.3 above the desk top, so that the panel is large and close seen from the desk and the walls next to it.

    ``glossy_desk=True``: the frame of resampled light sampling (option "light_candidates"): the same room with a glossy Disney desk
    (roughness 0.15, metallic 0.6), whose lobe under the panel decides which light samples matter.

    ``irradiance=True``: one one-sided triangle light of emission 4 facing down 0.5 above a Matte plane of albedo 0.5, seen from a
    pinhole 0.3 above the plane looking straight down (the light is behind it), ``depth`` 2: every pixel is (0.5 / pi) * E, E the
    light's irradiance at the plane point (Lambert's polygon formula), blurred only by the pixel's box filter."""
    out = []
    if irradiance:
        out.append("Surface plane_surface : Matte { Kd : Constant { v { 0.5, 0.5, 0.5 } } }")
        out.append("Light tri_light : Diffuse { emission : Constant { v { 4.0, 4.0, 4.0 } } two_sided { false } }")
        g = 10.0
        pos, idx = _mesh_props([[(-g, 0.0, g), (g, 0.0, g), (g, 0.0, -g), (-g, 0.0, -g)]])
        out.append(f"Shape plane : InlineMesh {{ positions {{ {pos} }} indices {{ {idx} }} surface {{ @plane_surface }} }}")
        tri = [(-0.9, 0.5, 0.8), (-0.7, 0.5, -1.0), (1.1, 0.5, 0.1)]  # cross(p1 - p0, p2 - p0) points down: it lights the plane
        pos = ", ".join(_fmt(c) for v in tri for c in v)
        out.append(f"Shape light : InlineMesh {{ positions {{ {pos} }} indices {{ 0, 1, 2 }} light {{ @tri_light }} }}")
        shapes = ["@plane", "@light"]
        camera = "position { 0.0, 0.3, 0.0 }\n  front { 0.0, -1.0, 0.0 }\n  up { 0.0, 0.0, -1.0 }\n  fov { 60.0 }"
        depth = 2
    else:
        shapes = _matte_room(out, "Light panel_light : Diffuse { emission : Constant { v { 6.0, 5.5, 4.5 } } two_sided { false } }",
                             glossy_desk)
        pos, idx = _mesh_props([[(-0.5, 1.0, -0.1), (-0.5, 1.0, -0.7), (0.5, 1.0, -0.7), (0.5, 1.0, -0.1)]])  # facing down
        out.append(f"Shape panel : InlineMesh {{ positions {{ {pos} }} indices {{ {idx} }} light {{ @panel_light }} }}")
        shapes.append("@panel")
        camera = _MATTE_ROOM_CAMERA
    return _matte_room_render(out, shapes, camera, resolution, spp, depth, rr_depth, rr_threshold, seed, output)


_MATTE_ROOM_CAMERA = "position { 0.0, 1.1, 3.4 }\n  front { 0.0, -0.08, -1.0 }\n  up { 0.0, 1.0, 0.0 }\n  fov { 38.0 }"


def _matte_room(out, light_line, glossy_desk=False):
    """The Matte room of ``near_light`` and ``emissive_globe``: its surfaces, the Light node ``light_line``, then its walls and desk.
    ``glossy_desk``: the desk is a glossy Disney surface of the same colour.  Returns the shape references."""
    colors = {"white": (0.725, 0.710, 0.680), "green": (0.140, 0.450, 0.091), "red": (0.630, 0.065, 0.050), "desk": (0.55, 0.45, 0.35)}
    for name, rgb in colors.items():
        color = f"{_fmt(rgb[0])}, {_fmt(rgb[1])}, {_fmt(rgb[2])}"
        if name == "desk" and glossy_desk:
            out.append(f"Surface desk : Disney {{ color : Constant {{ v {{ {color} }} }} metallic : Constant {{ v {{ 0.6 }} }} "
                       f"roughness : Constant {{ v {{ 0.15 }} }} }}")
        else:
            out.append(f"Surface {name} : Matte {{ Kd : Constant {{ v {{ {color} }} }} }}")
    out.append(light_line)
    x0, x1, y0, y1, z0, z1 = -1.0, 1.0, 0.0, 2.0, -1.0, 1.0
    quads = {  # (name, surface, [4 vertices])
        "floor": ("white", [(x0, y0, z1), (x1, y0, z1), (x1, y0, z0), (x0, y0, z0)]),
        "ceiling": ("white", [(x0, y1, z1), (x0, y1, z0), (x1, y1, z0), (x1, y1, z1)]),
        "back_wall": ("white", [(x0, y0, z0), (x1, y0, z0), (x1, y1, z0), (x0, y1, z0)]),
        "left_wall": ("red", [(x0, y0, z1), (x0, y0, z0), (x0, y1, z0), (x0, y1, z1)]),
        "right_wall": ("green", [(x1, y0, z0), (x1, y0, z1), (x1, y1, z1), (x1, y1, z0)]),
        "desk_top": ("desk", [(-0.7, 0.7, 0.1), (0.7, 0.7, 0.1), (0.7, 0.7, -0.9), (-0.7, 0.7, -0.9)]),
        "desk_front": ("desk", [(-0.7, 0.0, 0.1), (0.7, 0.0, 0.1), (0.7, 0.7, 0.1), (-0.7, 0.7, 0.1)]),
    }
    shapes = []
    for name, (surface, q) in quads.items():
        pos, idx = _mesh_props([q])
        out.append(f"Shape {name} : InlineMesh {{ positions {{ {pos} }} indices {{ {idx} }} surface {{ @{surface} }} }}")
        shapes.append(f"@{name}")
    return shapes


def _matte_room_render(out, shapes, camera, resolution, spp, depth, rr_depth, rr_threshold, seed, output) -> str:
    out.append(f"""Camera camera : Pinhole {{
  {camera}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}""")
    out.append(f"""render {{
  integrator : WavePath {{
    depth {{ {int(depth)} }}
    rr_depth {{ {int(rr_depth)} }}
    rr_threshold {{ {_fmt(rr_threshold)} }}
    sampler : Independent {{ seed {{ {int(seed)} }} }}
  }}
  cameras {{ @camera }}
  shapes {{ {", ".join(shapes)} }}
}}""")
    return "\n".join(out) + "\n"


def _icosphere(subdivision: int):
    """The unit icosphere of ``subdivision`` levels as (positions [n, 3], triangles [m, 3]), wound so that cross(p1 - p0, p2 - p0)
    points outwards: each level splits every triangle into four at its edges' midpoints, pushed onto the sphere."""
    t = (1.0 + 5.0 ** 0.5) / 2.0
    verts = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
             (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    verts = [tuple(np.array(v, np.float64) / np.linalg.norm(v)) for v in verts]
    tris = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
            (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    for _ in range(int(subdivision)):
        mid = {}

        def midpoint(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                m = np.add(verts[a], verts[b])
                verts.append(tuple(m / np.linalg.norm(m)))
                mid[key] = len(verts) - 1
            return mid[key]

        new = []
        for a, b, c in tris:
            ab, bc, ca = midpoint(a, b), midpoint(b, c), midpoint(c, a)
            new += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        tris = new
    return np.array(verts, np.float64), np.array(tris, np.int64)


def emissive_globe(resolution=(512, 512), spp=16, subdivision=5, transform="uniform", depth=10, rr_depth=0, rr_threshold=0.95,
                   seed=19980810, output="emissive_globe.exr", wobble=None) -> str:
    """The frame of the triangle-level light trees (option "light_tree_triangles"): ``near_light``'s Matte room lit only by a
    one-sided emissive icosphere of radius 0.25 (``subdivision`` levels) whose lowest point hangs 0.15 above the desk top.  Seen
    from the desk, most of the globe faces away: an emitter whose triangles are picked by area wastes most of its shadow rays.

    ``transform`` places the globe: "uniform" (an SRT of uniform scale), "stretched" (a Matrix of non-uniform scale 0.3 / 0.2 /
    0.25 under a rotation) or "mirrored" (a Matrix of negative determinant that mirrors x, applied to an icosphere wound inwards,
    so that its world-space triangles face outwards as the others do).

    ``wobble`` (a float) deforms the globe: it is ``_icosphere``'s InlineMesh with every vertex v scaled radially by
    1 + wobble * sin(3 v.x + 2 v.y) * cos(4 v.z), under the same ``transform``.  Frames of different ``wobble`` share their mesh
    layout and triangles (lrk_update_meshes); None keeps the text of the undeformed globe."""
    out = []
    shapes = _matte_room(out, "Light globe_light : Diffuse { emission : Constant { v { 9.0, 8.0, 6.5 } } two_sided { false } }")
    desk_top, gap = 0.7, 0.15

    def globe_mesh(inwards=False):
        if wobble is None and not inwards:
            return f"Shape globe_mesh : Sphere {{ subdivision {{ {int(subdivision)} }} }}"
        v, f = _icosphere(subdivision)
        if wobble is not None:
            v = v * (1.0 + float(wobble) * np.sin(3.0 * v[:, 0] + 2.0 * v[:, 1]) * np.cos(4.0 * v[:, 2]))[:, None]
        pos = ", ".join(_fmt(c) for c in v.reshape(-1))
        idx = ", ".join(str(int(i)) for i in (f[:, ::-1] if inwards else f).reshape(-1))
        return f"Shape globe_mesh : InlineMesh {{ positions {{ {pos} }} indices {{ {idx} }} }}"

    if transform == "uniform":
        r = 0.25
        out.append(globe_mesh())
        place = f"transform : SRT {{ scale {{ {_fmt(r)} }} translate {{ 0.0, {_fmt(desk_top + gap + r)}, -0.4 }} }}"
    elif transform in ("stretched", "mirrored"):
        if transform == "stretched":
            out.append(globe_mesh())
            a, b = np.radians(35.0), np.radians(20.0)
            rz = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
            ry = np.array([[np.cos(b), 0.0, np.sin(b)], [0.0, 1.0, 0.0], [-np.sin(b), 0.0, np.cos(b)]])
            m = ry @ rz @ np.diag([0.3, 0.2, 0.25])
        else:
            out.append(globe_mesh(inwards=True))  # wound inwards: the mirror turns them outwards
            m = np.diag([-0.25, 0.25, 0.25])
        low = np.linalg.norm(m[1])  # the lowest point of the ellipsoid lies |row y| below its centre
        t = (0.0, desk_top + gap + low, -0.4)
        rows = [list(m[i]) + [t[i]] for i in range(3)] + [[0.0, 0.0, 0.0, 1.0]]
        place = "transform : Matrix { m { " + ", ".join(_fmt(x) for row in rows for x in row) + " } }"
    else:
        raise ValueError(f"transform is 'uniform', 'stretched' or 'mirrored', not {transform!r}")
    out.append(f"Shape globe : Instance {{ shape {{ @globe_mesh }} light {{ @globe_light }} {place} }}")
    shapes.append("@globe")
    return _matte_room_render(out, shapes, _MATTE_ROOM_CAMERA, resolution, spp, depth, rr_depth, rr_threshold, seed, output)


def wavy_sheet_grid(segments, amplitude, time):
    """The sheet of ``wavy_sheet``: (positions [v, 3], normals [v, 3], uvs [v, 2], triangles [t, 3]) of a grid of ``segments``
    quads over [-0.5, 0.5]^2 in the x-z plane, raised by the wave y = amplitude sin(kx x + w t) cos(kz z + w t / 2)."""
    nx, nz = int(segments[0]), int(segments[1])
    x, z = np.meshgrid(np.linspace(-0.5, 0.5, nx + 1), np.linspace(-0.5, 0.5, nz + 1))
    kx, kz, w = 2.0 * np.pi * 1.5, 2.0 * np.pi, 2.0 * np.pi * 0.5
    y = amplitude * np.sin(kx * x + w * time) * np.cos(kz * z + 0.5 * w * time)
    dydx = amplitude * kx * np.cos(kx * x + w * time) * np.cos(kz * z + 0.5 * w * time)
    dydz = -amplitude * kz * np.sin(kx * x + w * time) * np.sin(kz * z + 0.5 * w * time)
    n = np.stack([-dydx, np.ones_like(y), -dydz], axis=-1)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    p = np.stack([x, y, z], axis=-1)
    uv = np.stack([x + 0.5, z + 0.5], axis=-1)
    a = (np.arange(nz)[:, None] * (nx + 1) + np.arange(nx)[None, :]).reshape(-1)
    b, c, d = a + 1, a + nx + 2, a + nx + 1
    tris = np.stack([np.stack([a, d, c], -1), np.stack([a, c, b], -1)], axis=1).reshape(-1, 3)  # cross(p1 - p0, p2 - p0) points up
    return p.reshape(-1, 3), n.reshape(-1, 3), uv.reshape(-1, 2), tris


def wavy_sheet(resolution=(64, 48), spp=4, segments=(24, 16), amplitude=0.08, time=0.0, emissive=False, depth=6, rr_depth=0,
               rr_threshold=0.95, seed=19980810, output="wavy_sheet.exr") -> str:
    """The frame of mesh deformation (lrk_update_meshes): ``near_light``'s Matte room with one Matte sheet of ``segments`` quads
    (an InlineMesh with normals and uvs) instanced twice through one mesh - above the desk and leaning on the floor - lit by a
    quad light under the ceiling.  ``time`` moves only the sheet's vertex positions and normals, by a travelling wave of height
    ``amplitude``: every frame of one parameter set has the same mesh layout, triangles and instance order.  ``emissive=True``
    makes the sheet a two-sided light and drops the ceiling light."""
    out = []
    light = "Light sheet_light : Diffuse { emission : Constant { v { 4.0, 3.6, 3.0 } } two_sided { true } }" if emissive else \
        "Light lamp_light : Diffuse { emission : Constant { v { 14.0, 12.0, 9.0 } } }"
    shapes = _matte_room(out, light)
    if not emissive:
        pos, idx = _mesh_props([[(-0.3, 1.98, 0.2), (-0.3, 1.98, -0.3), (0.3, 1.98, -0.3), (0.3, 1.98, 0.2)]])
        out.append(f"Shape lamp : InlineMesh {{ positions {{ {pos} }} indices {{ {idx} }} light {{ @lamp_light }} }}")
        shapes.append("@lamp")
        out.append("Surface sheet : Matte { Kd : Constant { v { 0.3, 0.45, 0.7 } } }")
    p, n, uv, tris = wavy_sheet_grid(segments, amplitude, time)
    fmt = lambda arr: ", ".join(_fmt(c) for c in np.asarray(arr).reshape(-1))  # noqa: E731
    out.append(f"Shape sheet_mesh : InlineMesh {{ positions {{ {fmt(p)} }} normals {{ {fmt(n)} }} uvs {{ {fmt(uv)} }} "
               f"indices {{ {', '.join(str(int(i)) for i in tris.reshape(-1))} }} }}")
    carry = "light { @sheet_light }" if emissive else "surface { @sheet }"
    places = ["scale { 0.9 } rotate { 1.0, 0.0, 0.0, 12.0 } translate { -0.2, 1.15, -0.35 }",
              "scale { 0.8 } rotate { 0.0, 0.0, 1.0, 35.0 } translate { 0.55, 0.3, 0.35 }"]
    for k, place in enumerate(places):
        out.append(f"Shape sheet_{k} : Instance {{ shape {{ @sheet_mesh }} {carry} transform : SRT {{ {place} }} }}")
        shapes.append(f"@sheet_{k}")
    return _matte_room_render(out, shapes, _MATTE_ROOM_CAMERA, resolution, spp, depth, rr_depth, rr_threshold, seed, output)


def textured_materials(resolution=(64, 40), spp=4, depth=6, rr_depth=0, rr_threshold=0.95, seed=19980810, assets="tests/golden/assets",
                       output="texmat.exr", integrator="WavePath") -> str:
    """SURVEY.md §8 row f3 with image-textured parameters: four uv-mapped panels - Mirror (colour + roughness images), Glass (Kr, Kt
    and roughness images), Plastic (Kd, sigma_a, thickness and roughness images) and Metal (named copper, Kd + roughness images) -
    in a Matte room, so that the closure context of each is derived per hit from texels (mirror.cpp:142-162, glass.cpp:236-279,
    plastic.cpp:252-291, metal.cpp:273-310)."""
    a = assets
    img = lambda f, enc="sRGB", extra="": f'Image {{ file {{ "{a}/{f}" }} encoding {{ "{enc}" }} {extra}}}'  # noqa: E731
    out = [
        "Surface white : Matte { Kd : Constant { v { 0.725, 0.71, 0.68 } } }",
        "Surface blue : Matte { Kd : Constant { v { 0.15, 0.25, 0.65 } } }",
        f"Surface t_mirror : Mirror {{ color : {img('checker_rgb8.png')} roughness : {img('rough_gray8.png', 'linear', 'uv_scale { 2.0 } ')} }}",
        f"Surface t_glass : Glass {{ Kr : {img('palette4.png')} Kt : {img('checker_rgb8.png', 'sRGB', 'uv_scale { 3.0 } ')} "
        f"roughness : {img('rough_gray8.png', 'linear')} remap_roughness {{ false }} eta : Constant {{ v {{ 1.4 }} }} }}",
        f"Surface t_plastic : Plastic {{ Kd : {img('ramp_rgba16.png', 'linear')} sigma_a : {img('palette4.png', 'linear', 'uv_scale { 2.0 } ')} "
        f"thickness : {img('rough_gray8.png', 'linear', 'uv_offset { 0.25, 0.1 } ')} roughness : {img('rough_gray8.png', 'linear')} eta : Constant {{ v {{ 1.5 }} }} }}",
        f"Surface t_metal : Metal {{ eta {{ \"Cu\" }} Kd : {img('checker_rgb8.png', 'sRGB', 'uv_scale { 2.0 } ')} roughness : {img('rough_gray8.png', 'linear', 'uv_scale { 1.5 } ')} }}",
        "Light area_light : Diffuse { emission : Constant { v { 17.0, 14.0, 10.0 } } }",
    ]
    shapes = []

    def quad(name, pts, surface=None, light=None, uvs=False):
        pos, idx = _mesh_props([pts])
        attach = f"surface {{ @{surface} }}" if surface else f"light {{ @{light} }}"
        uv = " uvs { 0.0, 0.0,  1.0, 0.0,  1.0, 1.0,  0.0, 1.0 }" if uvs else ""
        out.append(f"Shape {name} : InlineMesh {{ positions {{ {pos} }}{uv} indices {{ {idx} }} {attach} }}")
        shapes.append(f"@{name}")

    quad("floor", [(-2.0, 0.0, 1.5), (2.0, 0.0, 1.5), (2.0, 0.0, -1.5), (-2.0, 0.0, -1.5)], "white")
    quad("ceiling", [(-2.0, 2.5, 1.5), (-2.0, 2.5, -1.5), (2.0, 2.5, -1.5), (2.0, 2.5, 1.5)], "white")
    quad("back", [(-2.0, 0.0, -1.5), (2.0, 0.0, -1.5), (2.0, 2.5, -1.5), (-2.0, 2.5, -1.5)], "blue")
    quad("left", [(-2.0, 0.0, 1.5), (-2.0, 0.0, -1.5), (-2.0, 2.5, -1.5), (-2.0, 2.5, 1.5)], "white")
    quad("right", [(2.0, 0.0, -1.5), (2.0, 0.0, 1.5), (2.0, 2.5, 1.5), (2.0, 2.5, -1.5)], "white")
    quad("lamp", [(-0.6, 2.49, 0.4), (-0.6, 2.49, -0.4), (0.6, 2.49, -0.4), (0.6, 2.49, 0.4)], light="area_light")
    for i, surface in enumerate(["t_mirror", "t_glass", "t_plastic", "t_metal"]):
        x0 = -1.8 + 0.92 * i
        z0, z1 = (-0.2, -0.5) if i % 2 == 0 else (-0.6, -0.3)  # slightly turned panels
        quad(f"panel_{i}", [(x0, 0.15, z0), (x0 + 0.8, 0.15, z1), (x0 + 0.8, 1.55, z1 - 0.25), (x0, 1.55, z0 - 0.25)], surface, uvs=True)
    out.append(f"""Camera camera : Pinhole {{
  position {{ 0.0, 1.1, 4.6 }}
  look_at {{ 0.0, 0.85, 0.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 40.0 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}""")
    out.append(f"""render {{
  integrator : {integrator} {{
    depth {{ {int(depth)} }}
    rr_depth {{ {int(rr_depth)} }}
    rr_threshold {{ {_fmt(rr_threshold)} }}
    sampler : Independent {{ seed {{ {int(seed)} }} }}
  }}
  cameras {{ @camera }}
  shapes {{ {", ".join(shapes)} }}
}}""")
    return "\n".join(out) + "\n"


def media_box(resolution=(64, 64), spp=4, depth=8, rr_depth=0, rr_threshold=0.95, seed=19980810, output="media.exr",
              environment_medium=False, skip_quirk=False) -> str:
    """Row a22 beyond config C4: media bound to shapes (MegaVPTNaive's medium tracker).  The Cornell box whose short box is a
    smooth Glass shell around a dense, coloured medium and whose tall box is a rough Glass shell around a second medium; with
    ``environment_medium`` the room itself is filled with a thin third medium (registered last: highest medium tag), otherwise
    the environment medium is a Vacuum node.
    ``skip_quirk`` gives the tall box's medium priority 0 and tag 1: inside it `true_hit(tag)` (mega_vpt_naive.cpp:387 compares
    the TAG with the current priority) is false for its own boundary and the path leaves straight through, without refraction."""
    out = []
    for name, rgb in _CORNELL_COLORS.items():
        out.append(f"Surface {name} : Matte {{ Kd : Constant {{ v {{ {_fmt(rgb[0])}, {_fmt(rgb[1])}, {_fmt(rgb[2])} }} }} }}")
    out.append('Surface shell_smooth : Glass { eta { "BK7" } }')
    out.append("Surface shell_rough : Glass { Kr : Constant { v { 1.0, 0.95, 0.9 } } Kt : Constant { v { 0.9, 0.95, 1.0 } } "
               "roughness : Constant { v { 0.25 } } eta { 1.33 } }")
    out.append("Medium fog_dense : Homogeneous {\n  priority { 2 }\n  sigma_a : Constant { v { 0.4, 0.8, 2.5 } }\n"
               "  sigma_s : Constant { v { 2.0, 3.0, 1.5 } }\n  phasefunction : HenyeyGreenstein { g { 0.5 } }\n}")
    out.append(f"Medium fog_light : Homogeneous {{\n  priority {{ {0 if skip_quirk else 1} }}\n  sigma_a : Constant {{ v {{ 0.3, 0.1, 0.1 }} }}\n"
               "  sigma_s : Constant { v { 0.8, 0.9, 1.2 } }\n  phasefunction : HenyeyGreenstein { g { 0.0 } }\n}")
    out.append("Light area_light : Diffuse { emission : Constant { v { 17.0, 12.0, 4.0 } } }")
    shape_names = []
    for name, quads in _CORNELL_QUADS.items():
        positions, indices = _mesh_props(quads)
        if name == "light":
            binding = "light { @area_light }"
        elif name == "short_box":
            binding = "surface { @shell_smooth }\n  medium { @fog_dense }"
        elif name == "tall_box":
            binding = "surface { @shell_rough }\n  medium { @fog_light }"
        else:
            binding = f"surface {{ @{_CORNELL_SURFACE_OF[name]} }}"
        out.append(f"Shape {name} : InlineMesh {{\n  positions {{ {positions} }}\n  indices {{ {indices} }}\n  {binding}\n}}")
        shape_names.append(f"@{name}")
    out.append(f"""Camera camera : Pinhole {{
  position {{ -0.01, 0.995, 5.0 }}
  front {{ 0.0, 0.0, -1.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 27.8 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}""")
    # the reference needs SOME environment medium as soon as two media are registered: the tracker's initialisation dispatches on
    # the environment medium's tag and an invalid tag runs into the dispatch's unreachable() (mega_vpt_naive.cpp:184-190)
    medium_line = "  environment_medium : Vacuum {}\n"
    if environment_medium:
        medium_line = ("  environment_medium : Homogeneous {\n    priority { 1 }\n"
                       "    sigma_a : Constant { v { 0.02, 0.02, 0.02 } }\n"
                       "    sigma_s : Constant { v { 0.08, 0.08, 0.1 } }\n"
                       "    phasefunction : HenyeyGreenstein { g { 0.3 } }\n"
                       "  }\n")
    out.append(f"""render {{
  integrator : MegaVPTNaive {{
    depth {{ {int(depth)} }}
    rr_depth {{ {int(rr_depth)} }}
    rr_threshold {{ {_fmt(rr_threshold)} }}
    sampler : Independent {{ seed {{ {int(seed)} }} }}
  }}
{medium_line}  cameras {{ @camera }}
  shapes {{ {", ".join(shape_names)} }}
}}""")
    return "\n".join(out) + "\n"


def textured_room(resolution=(96, 64), spp=8, depth=6, rr_depth=0, rr_threshold=0.95, seed=19980810,
                  assets="tests/golden/assets", output="textured.exr", integrator="WavePath", wrappers=False,
                  mesh_files=True, textured_light=False) -> str:
    """SURVEY.md §8 row f1 in one small scene: image-textured Matte and Disney parameters (PNG 8/16-bit, grey, palette; all
    four address modes, point + bilinear filters, sRGB + linear encodings, uv scale/offset) on an InlineMesh with uvs and
    on mesh FILES (Wavefront OBJ without normals, binary PLY).  `assets` is relative to the directory the scene is loaded from.
    ``wrappers=True`` adds the surface wrappers of src/base/surface.h:160-275: a normal-mapped floor, a cut-out screen with an
    alpha texture (stochastic alpha test inside closest-hit and any-hit traversal) and a half-transparent cube (constant opacity).
    ``textured_light=True`` gives the lamp an image emission (src/lights/diffuse.cpp:74: evaluated at the uv of the emitter hit or of
    the sampled light point, src/lightsamplers/uniform.cpp:108-123)."""
    a = assets.rstrip("/")
    emission = "Constant { v { 14.0, 13.0, 11.0 } }"
    lamp_uvs = ""
    if textured_light:
        emission = f'Image {{ file {{ "{a}/checker_rgb8.png" }} address {{ "repeat" }} filter {{ "bilinear" }} uv_scale {{ 2.0 }} uv_offset {{ 0.3, 0.1 }} scale {{ 20.0 }} }}'
        lamp_uvs = "\n  uvs { 0.0, 0.0,  0.0, 1.0,  1.0, 1.0,  1.0, 0.0 }"
    floor_extra = cube_extra = screen = screen_ref = ""
    # mesh_files=False: the two file meshes become inline panels with uvs (the reference build under oracle/ref has no
    # `Mesh` plugin: it needs assimp)
    cube_geometry = f'Mesh {{\n  file {{ "{a}/cube.obj" }}'
    tetra_geometry = f'Mesh {{\n  file {{ "{a}/tetra_binary.ply" }}\n  flip_uv {{ true }}'
    if not mesh_files:
        cube_geometry = ("InlineMesh {\n  positions { -0.5, -0.5, 0.5,  0.5, -0.5, 0.5,  0.5, 0.5, 0.5,  -0.5, 0.5, 0.5,  0.5, -0.5, -0.5,  0.5, 0.5, -0.5 }\n"
                         "  uvs { 0.0, 0.0,  1.0, 0.0,  1.0, 1.0,  0.0, 1.0,  2.0, 0.0,  2.0, 1.0 }\n  indices { 0, 1, 2, 0, 2, 3, 1, 4, 5, 1, 5, 2 }")
        tetra_geometry = ("InlineMesh {\n  positions { -0.5, 0.0, 0.4,  0.5, 0.0, 0.4,  0.0, 0.9, 0.0,  0.0, 0.0, -0.5 }\n"
                          "  uvs { 0.0, 0.0,  1.0, 0.0,  0.5, 1.0,  0.5, -0.3 }\n  indices { 0, 1, 2, 1, 3, 2, 3, 0, 2 }")
    if wrappers:
        floor_extra = f'normal_map : Image {{ file {{ "{a}/normal_rgb8.png" }} encoding {{ "linear" }} uv_scale {{ 4.0 }} }} normal_map_strength {{ 0.8 }}'
        cube_extra = "opacity : Constant { v { 0.5 } }"
        screen = f"""
Surface screen_s : Matte {{
  Kd : Constant {{ v {{ 0.8, 0.75, 0.2 }} }}
  alpha : Image {{ file {{ "{a}/alpha_gray8.png" }} encoding {{ "linear" }} uv_scale {{ 2.0 }} }}
}}
Shape screen : InlineMesh {{
  positions {{ 0.2, 0.0, 1.0,  1.6, 0.0, 0.6,  1.6, 1.3, 0.6,  0.2, 1.3, 1.0 }}
  uvs {{ 0.0, 0.0,  1.0, 0.0,  1.0, 1.0,  0.0, 1.0 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  surface {{ @screen_s }}
}}"""
        screen_ref = ", @screen"
    return f"""
Surface floor_s : Matte {{
  Kd : Image {{ file {{ "{a}/checker_rgb8.png" }} address {{ "repeat" }} filter {{ "bilinear" }} uv_scale {{ 2.0, 3.0 }} uv_offset {{ 0.25, 0.0 }} }}
  {floor_extra}
}}
Surface wall_s : Matte {{
  Kd : Image {{ file {{ "{a}/ramp_rgba16.png" }} address {{ "edge" }} encoding {{ "linear" }} scale {{ 0.9 }} }}
  sigma : Image {{ file {{ "{a}/rough_gray8.png" }} encoding {{ "linear" }} filter {{ "point" }} }}
}}
Surface cube_s : Disney {{
  color : Image {{ file {{ "{a}/checker_rgb8.png" }} address {{ "mirror" }} filter {{ "point" }} uv_scale {{ 1.5 }} }}
  roughness : Image {{ file {{ "{a}/rough_gray8.png" }} encoding {{ "linear" }} address {{ "repeat" }} }}
  metallic : Constant {{ v {{ 0.2 }} }}
  clearcoat : Constant {{ v {{ 0.5 }} }}
  {cube_extra}
}}
Surface tetra_s : Matte {{
  Kd : Image {{ file {{ "{a}/palette4.png" }} address {{ "zero" }} encoding {{ "gamma" }} gamma {{ 2.0 }} }}
}}
Light area_light : Diffuse {{ emission : {emission} }}
Shape floor : InlineMesh {{
  positions {{ -2.0, 0.0, 2.0,  2.0, 0.0, 2.0,  2.0, 0.0, -2.0,  -2.0, 0.0, -2.0 }}
  uvs {{ 0.0, 0.0,  1.0, 0.0,  1.0, 1.0,  0.0, 1.0 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  surface {{ @floor_s }}
}}
Shape wall : InlineMesh {{
  positions {{ -2.0, 0.0, -2.0,  2.0, 0.0, -2.0,  2.0, 2.5, -2.0,  -2.0, 2.5, -2.0 }}
  uvs {{ -0.2, -0.2,  1.2, -0.2,  1.2, 1.2,  -0.2, 1.2 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  surface {{ @wall_s }}
}}
Shape cube : {cube_geometry}
  surface {{ @cube_s }}
  transform : SRT {{ scale {{ 0.8 }} rotate {{ 0.0, 1.0, 0.0, 30.0 }} translate {{ -0.6, 0.4, -0.3 }} }}
}}
Shape tetra : {tetra_geometry}
  surface {{ @tetra_s }}
  transform : SRT {{ scale {{ 1.1 }} translate {{ 0.5, 0.0, -0.2 }} }}
}}
{screen}
Shape lamp : InlineMesh {{
  positions {{ -0.6, 2.4, 0.4,  -0.6, 2.4, -0.4,  0.6, 2.4, -0.4,  0.6, 2.4, 0.4 }}{lamp_uvs}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  light {{ @area_light }}
}}
Camera camera : Pinhole {{
  position {{ 0.0, 1.4, 4.2 }}
  front {{ 0.0, -0.2, -1.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 40.0 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}
render {{
  integrator : {integrator} {{
    depth {{ {int(depth)} }}
    rr_depth {{ {int(rr_depth)} }}
    rr_threshold {{ {_fmt(rr_threshold)} }}
    sampler : Independent {{ seed {{ {int(seed)} }} }}
  }}
  cameras {{ @camera }}
  shapes {{ @floor, @wall, @cube, @tetra, @lamp{screen_ref} }}
}}
"""


def environment_scene(resolution=(64, 40), spp=8, depth=5, rr_depth=0, rr_threshold=0.95, seed=19980810, assets="tests/golden/assets",
                      emission="image", area_light=True, environment_weight=0.5, compensate_mis=True, output="env.exr",
                      sky_file="sky.pfm") -> str:
    """SURVEY.md §8 rows a12 / f3: a Spherical environment light (src/environments/spherical.cpp) — image emission with the
    importance map, or a constant one — next to an optional area light (uniform light sampler, environment_weight), seen by a
    Matte sphere on a Disney floor."""
    a = assets.rstrip("/")
    if emission == "image":
        # sky.exr holds the same texels as sky.pfm (the reference's image reader has no PFM decoder)
        em = f'emission : Image {{ file {{ "{a}/{sky_file}" }} encoding {{ "linear" }} address {{ "repeat" }} }}'
    else:
        em = f"emission : Constant {{ v {{ {_fmt(emission[0])}, {_fmt(emission[1])}, {_fmt(emission[2])} }} }}"
    light = lamp = lamp_ref = ""
    if area_light:
        light = "Light area_light : Diffuse { emission : Constant { v { 9.0, 8.0, 6.0 } } }"
        lamp = """Shape lamp : InlineMesh {
  positions { -0.4, 2.2, 0.4,  -0.4, 2.2, -0.4,  0.4, 2.2, -0.4,  0.4, 2.2, 0.4 }
  indices { 0, 1, 2, 0, 2, 3 }
  light { @area_light }
}"""
        lamp_ref = ", @lamp"
    return f"""
Surface ball_s : Matte {{ Kd : Constant {{ v {{ 0.8, 0.8, 0.8 }} }} }}
Surface floor_s : Disney {{ color : Constant {{ v {{ 0.5, 0.45, 0.4 }} }} roughness : Constant {{ v {{ 0.6 }} }} }}
{light}
Shape ball : Sphere {{ subdivision {{ 3 }} surface {{ @ball_s }} transform : SRT {{ scale {{ 0.7 }} translate {{ 0.0, 0.7, 0.0 }} }} }}
Shape floor : InlineMesh {{
  positions {{ -3.0, 0.0, 3.0,  3.0, 0.0, 3.0,  3.0, 0.0, -3.0,  -3.0, 0.0, -3.0 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  surface {{ @floor_s }}
}}
{lamp}
Camera camera : Pinhole {{
  position {{ 0.0, 1.2, 4.0 }}
  front {{ 0.0, -0.12, -1.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 42.0 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}
render {{
  integrator : WavePath {{
    depth {{ {int(depth)} }}
    rr_depth {{ {int(rr_depth)} }}
    rr_threshold {{ {_fmt(rr_threshold)} }}
    sampler : Independent {{ seed {{ {int(seed)} }} }}
    light_sampler : Uniform {{ environment_weight {{ {_fmt(environment_weight)} }} }}
  }}
  environment : Spherical {{
    {em}
    scale {{ 1.0 }}
    compensate_mis {{ {"true" if compensate_mis else "false"} }}
    transform : SRT {{ rotate {{ 0.0, 1.0, 0.0, 40.0 }} }}
  }}
  cameras {{ @camera }}
  shapes {{ @ball, @floor{lamp_ref} }}
}}
"""


def layered_box(**kw) -> str:
    """Row f3's Layered surface (src/surfaces/layered.cpp) on three of the materials box's balls: a rough Glass coat over a Matte base
    with a tinted, forward-scattering slab between them (two evaluate samples); a Glass coat over a Mirror base with a black albedo
    (the slab only attenuates: the reference's `albedo.is_zero()` branch); a Plastic coat over Matte with the node's defaults."""
    src = materials_box(**kw)
    layered = [
        "Surface l_coat : Glass { roughness : Constant { v { 0.2 } } eta : Constant { v { 1.5 } } }",
        "Surface l_base : Matte { Kd : Constant { v { 0.8, 0.3, 0.2 } } }",
        "Surface l_base_mirror : Mirror { color : Constant { v { 0.9, 0.85, 0.6 } } roughness : Constant { v { 0.3 } } }",
        "Surface l_coat_plastic : Plastic { Kd : Constant { v { 0.3, 0.6, 0.3 } } roughness : Constant { v { 0.25 } } }",
        "Surface m_mirror : Layered { top { @l_coat } bottom { @l_base } thickness : Constant { v { 0.05 } } g : Constant { v { 0.3 } } "
        "albedo : Constant { v { 0.6, 0.7, 0.9 } } max_depth { 8 } samples { 2 } }",
        "Surface m_glass : Layered { top { @l_coat } bottom { @l_base_mirror } thickness : Constant { v { 0.02 } } "
        "albedo : Constant { v { 0.0, 0.0, 0.0 } } max_depth { 6 } }",
        "Surface m_plastic : Layered { top { @l_coat_plastic } bottom { @l_base } }",
    ]
    out = []
    for line in src.split("\n"):
        if line.startswith("Surface m_mirror :"):
            out += layered
        elif line.startswith("Surface m_glass :"):
            continue
        elif line.startswith("Surface m_plastic :"):
            continue
        elif line.startswith("sigma_a : Constant") and out and out[-1].startswith("Surface m_plastic : Layered"):
            continue
        else:
            out.append(line)
    return "\n".join(out)


def materials_box(resolution=(32, 24), spp=4, depth=8, rr_depth=0, rr_threshold=0.95, seed=19980810, subdivision=2,
                  integrator="WavePath", output="materials.exr", mix=False) -> str:
    """SURVEY.md §8 row f3: a Cornell-like box with one Loop-subdivision sphere per closure of src/surfaces -
    Mirror, Glass (built-in bk7), rough Glass, Plastic, Metal (custom eta list) - on a Matte floor, plus a mirror back wall."""
    out = [
        "Surface white : Matte { Kd : Constant { v { 0.725, 0.71, 0.68 } } }",
        "Surface red : Matte { Kd : Constant { v { 0.63, 0.065, 0.05 } } }",
        "Surface green : Plastic { Kd : Constant { v { 0.14, 0.45, 0.091 } } roughness : Constant { v { 0.3 } } }",
        "Surface wall_mirror : Mirror { color : Constant { v { 0.9, 0.9, 0.95 } } roughness : Constant { v { 0.05 } } }",
        "Surface m_mirror : Mirror { Kd : Constant { v { 0.95, 0.8, 0.6 } } }",
        "Surface m_glass : Glass { eta { \"BK7\" } }",
        "Surface m_rough_glass : Glass { Kr : Constant { v { 1.0, 0.9, 0.9 } } Kt : Constant { v { 0.7, 0.9, 1.0 } } "
        "eta : Constant { v { 1.33 } } roughness : Constant { v { 0.4, 0.2 } } }",
        "Surface m_plastic : Plastic { Kd : Constant { v { 0.2, 0.3, 0.8 } } roughness : Constant { v { 0.15 } } "
        "sigma_a : Constant { v { 0.3, 0.1, 0.05 } } thickness : Constant { v { 0.5 } } eta : Constant { v { 1.45 } } }",
        "Surface m_metal : Metal { eta { 350.0, 0.2, 1.9, 500.0, 0.35, 2.4, 600.0, 0.25, 3.0, 850.0, 0.2, 5.0 } "
        "roughness : Constant { v { 0.25 } } Kd : Constant { v { 1.0, 0.85, 0.6 } } }",
        "Light area_light : Diffuse { emission : Constant { v { 17.0, 14.0, 10.0 } } }",
        f"Shape ball : Sphere {{ subdivision {{ {int(subdivision)} }} }}",
    ]
    ball_surfaces = ["m_mirror", "m_glass", "m_rough_glass", "m_plastic", "m_metal"]
    floor_surface = "white"
    if mix:  # src/surfaces/mix.cpp: a matte/mirror blend, a plastic/glass blend (refraction events), the default ratio
        out += [
            "Surface mx_matte_mirror : Mix { a { @red } b { @m_mirror } ratio : Constant { v { 0.3 } } }",
            "Surface mx_glass_plastic : Mix { a { @m_rough_glass } b { @m_plastic } ratio : Constant { v { 0.65 } } }",
            "Surface mx_floor : Mix { a { @white } b { @m_metal } }",
        ]
        ball_surfaces = ["mx_matte_mirror", "m_glass", "mx_glass_plastic", "m_plastic", "mx_matte_mirror"]
        floor_surface = "mx_floor"
    shapes = []

    def quad(name, pts, surface=None, light=None):
        pos, idx = _mesh_props([pts])
        attach = f"surface {{ @{surface} }}" if surface else f"light {{ @{light} }}"
        out.append(f"Shape {name} : InlineMesh {{ positions {{ {pos} }} indices {{ {idx} }} {attach} }}")
        shapes.append(f"@{name}")

    quad("floor", [(-2.0, 0.0, 1.5), (2.0, 0.0, 1.5), (2.0, 0.0, -1.5), (-2.0, 0.0, -1.5)], floor_surface)
    quad("ceiling", [(-2.0, 2.5, 1.5), (-2.0, 2.5, -1.5), (2.0, 2.5, -1.5), (2.0, 2.5, 1.5)], "white")
    quad("back", [(-2.0, 0.0, -1.5), (2.0, 0.0, -1.5), (2.0, 2.5, -1.5), (-2.0, 2.5, -1.5)], "wall_mirror")
    quad("left", [(-2.0, 0.0, 1.5), (-2.0, 0.0, -1.5), (-2.0, 2.5, -1.5), (-2.0, 2.5, 1.5)], "red")
    quad("right", [(2.0, 0.0, -1.5), (2.0, 0.0, 1.5), (2.0, 2.5, 1.5), (2.0, 2.5, -1.5)], "green")
    quad("lamp", [(-0.6, 2.49, 0.4), (-0.6, 2.49, -0.4), (0.6, 2.49, -0.4), (0.6, 2.49, 0.4)], light="area_light")
    for i, surface in enumerate(ball_surfaces):
        x = -1.5 + 0.75 * i
        z = 0.3 if i % 2 == 0 else -0.4
        out.append(f"Shape ball_{i} : Instance {{ shape {{ @ball }} surface {{ @{surface} }} "
                   f"transform : SRT {{ scale {{ 0.33 }} translate {{ {_fmt(x)}, 0.33, {_fmt(z)} }} }} }}")
        shapes.append(f"@ball_{i}")
    out.append(f"""Camera camera : Pinhole {{
  position {{ 0.0, 1.2, 5.2 }}
  look_at {{ 0.0, 0.9, 0.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 38.0 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}""")
    out.append(f"""render {{
  integrator : {integrator} {{
    depth {{ {int(depth)} }}
    rr_depth {{ {int(rr_depth)} }}
    rr_threshold {{ {_fmt(rr_threshold)} }}
    sampler : Independent {{ seed {{ {int(seed)} }} }}
  }}
  cameras {{ @camera }}
  shapes {{ {", ".join(shapes)} }}
}}""")
    return "\n".join(out) + "\n"


def flatten_stress(resolution=(32, 24), spp=4, depth=6, output="flatten.exr") -> str:
    """Host-side flattening (SURVEY.md §8 row a23) in one scene: Group / Instance nesting with SRT, Matrix and Stack transforms,
    surface and light overrides down the hierarchy, an invisible shape that still casts no shadow, vertex normals with a
    shadow-terminator factor and an intersection-offset factor, a two-sided light as an instanced shape, a render-level
    shadow_terminator default."""
    return f"""
Surface white : Matte {{ Kd : Constant {{ v {{ 0.75, 0.75, 0.75 }} }} }}
Surface blue : Matte {{ Kd : Constant {{ v {{ 0.15, 0.25, 0.7 }} }} sigma : Constant {{ v {{ 0.4 }} }} }}
Surface gold : Disney {{ color : Constant {{ v {{ 0.9, 0.7, 0.2 }} }} metallic : Constant {{ v {{ 0.9 }} }} roughness : Constant {{ v {{ 0.35 }} }} }}
Light lamp_light : Diffuse {{ emission : Constant {{ v {{ 12.0, 11.0, 10.0 }} }} two_sided {{ true }} }}
Light small_light : Diffuse {{ emission : Constant {{ v {{ 3.0, 6.0, 9.0 }} }} scale {{ 2.0 }} }}
Transform lamp_tilt : SRT {{ rotate {{ 1.0, 0.0, 0.0, 90.0 }} scale {{ 1.6 }} }}
Transform lamp_lift : SRT {{ translate {{ 0.0, 2.6, 0.0 }} }}
Shape floor : InlineMesh {{
  positions {{ -3.0, 0.0, 3.0,  3.0, 0.0, 3.0,  3.0, 0.0, -3.0,  -3.0, 0.0, -3.0 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  surface {{ @white }}
}}
Shape bump : InlineMesh {{
  positions {{ -0.6, 0.0, 0.6,  0.6, 0.0, 0.6,  0.6, 0.0, -0.6,  -0.6, 0.0, -0.6,  0.0, 0.7, 0.0 }}
  normals {{ -0.6, 0.5, 0.6,  0.6, 0.5, 0.6,  0.6, 0.5, -0.6,  -0.6, 0.5, -0.6,  0.0, 1.0, 0.0 }}
  uvs {{ 0.0, 0.0,  1.0, 0.0,  1.0, 1.0,  0.0, 1.0,  0.5, 0.5 }}
  indices {{ 0, 1, 4,  1, 2, 4,  2, 3, 4,  3, 0, 4 }}
  surface {{ @blue }}
  shadow_terminator {{ 0.6 }}
  intersection_offset {{ 0.3 }}
}}
Shape quad : InlineMesh {{
  positions {{ -0.5, -0.5, 0.0,  0.5, -0.5, 0.0,  0.5, 0.5, 0.0,  -0.5, 0.5, 0.0 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
}}
Shape gold_bump : Instance {{
  shape {{ @bump }}
  surface {{ @gold }}
  transform : SRT {{ scale {{ 0.7, 1.3, 0.7 }} rotate {{ 0.0, 1.0, 0.0, 25.0 }} translate {{ 1.4, 0.0, -0.4 }} }}
}}
Shape lamp : Instance {{
  shape {{ @quad }}
  light {{ @lamp_light }}
  transform : Stack {{ transforms {{ @lamp_tilt, @lamp_lift }} }}
}}
Shape pair : Group {{
  shapes {{ @bump, @gold_bump }}
  transform : Matrix {{ m {{ 0.8, 0.0, 0.0, -1.5,   0.0, 0.8, 0.0, 0.0,   0.0, 0.0, 0.8, 0.8,   0.0, 0.0, 0.0, 1.0 }} }}
}}
Shape pair_again : Instance {{
  shape {{ @pair }}
  surface {{ @white }}
  transform : SRT {{ translate {{ 2.2, 0.0, -1.6 }} rotate {{ 0.0, 1.0, 0.0, -40.0 }} }}
}}
Shape hidden_wall : Instance {{
  shape {{ @quad }}
  surface {{ @blue }}
  visible {{ false }}
  transform : SRT {{ scale {{ 3.0 }} translate {{ 0.0, 1.0, 1.5 }} }}
}}
Shape small_lamp : Instance {{
  shape {{ @quad }}
  light {{ @small_light }}
  surface {{ @white }}
  transform : SRT {{ scale {{ 0.5 }} rotate {{ 0.0, 1.0, 0.0, 180.0 }} translate {{ -2.0, 1.0, -2.5 }} }}
}}
Camera camera : Pinhole {{
  position {{ 0.5, 2.2, 5.5 }}
  look_at {{ 0.0, 0.6, 0.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 42.0 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}
render {{
  integrator : WavePath {{
    depth {{ {int(depth)} }}
    rr_depth {{ 1 }}
    sampler : Independent {{ seed {{ 7 }} }}
  }}
  shadow_terminator {{ 0.25 }}
  cameras {{ @camera }}
  shapes {{ @floor, @pair, @pair_again, @gold_bump, @lamp, @hidden_wall, @small_lamp }}
}}
"""


def subdivision_scene(resolution=(64, 48), spp=4, depth=5, output="subdiv.exr", integrator="WavePath") -> str:
    """The `LoopSubdiv` shape (src/shapes/loop_subdiv.cpp): Loop subdivision to the limit surface with limit normals of
    a closed cube (valence-4/5 extraordinary vertices), a tetrahedron (valence 3: the 3/16 rule), an OPEN two-triangle sheet
    (boundary and corner rules, valence-2 corners) and an open fan of five triangles (boundary valence 3, interior valence 5);
    level 0 passes the base mesh through."""
    return f"""
Surface white : Matte {{ Kd : Constant {{ v {{ 0.75, 0.75, 0.75 }} }} }}
Surface blue : Disney {{ color : Constant {{ v {{ 0.2, 0.35, 0.8 }} }} roughness : Constant {{ v {{ 0.35 }} }} metallic : Constant {{ v {{ 0.1 }} }} }}
Surface orange : Matte {{ Kd : Constant {{ v {{ 0.85, 0.45, 0.12 }} }} sigma : Constant {{ v {{ 20.0 }} }} }}
Surface steel : Metal {{ eta {{ 350.0, 0.2, 1.9, 500.0, 0.35, 2.4, 600.0, 0.25, 3.0, 850.0, 0.2, 5.0 }} roughness : Constant {{ v {{ 0.25 }} }} }}
Light area_light : Diffuse {{ emission : Constant {{ v {{ 15.0, 14.0, 12.0 }} }} }}
Shape floor : InlineMesh {{
  positions {{ -3.0, 0.0, 3.0,  3.0, 0.0, 3.0,  3.0, 0.0, -3.0,  -3.0, 0.0, -3.0 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  surface {{ @white }}
}}
Shape lamp : InlineMesh {{
  positions {{ -0.8, 3.0, 0.8,  -0.8, 3.0, -0.8,  0.8, 3.0, -0.8,  0.8, 3.0, 0.8 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  light {{ @area_light }}
}}
Shape cube : LoopSubdiv {{
  mesh : InlineMesh {{
    positions {{ -0.5, -0.5, 0.5,  0.5, -0.5, 0.5,  0.5, 0.5, 0.5,  -0.5, 0.5, 0.5,  -0.5, -0.5, -0.5,  0.5, -0.5, -0.5,  0.5, 0.5, -0.5,  -0.5, 0.5, -0.5 }}
    indices {{ 0, 1, 2, 0, 2, 3,  1, 5, 6, 1, 6, 2,  5, 4, 7, 5, 7, 6,  4, 0, 3, 4, 3, 7,  3, 2, 6, 3, 6, 7,  4, 5, 1, 4, 1, 0 }}
  }}
  level {{ 3 }}
  surface {{ @blue }}
  transform : SRT {{ scale {{ 1.2 }} rotate {{ 0.0, 1.0, 0.0, 25.0 }} translate {{ -1.1, 0.62, 0.0 }} }}
}}
Shape tetra : LoopSubdiv {{
  shape : InlineMesh {{
    positions {{ 0.0, 1.0, 0.0,  -0.9, -0.4, 0.55,  0.9, -0.4, 0.55,  0.0, -0.4, -1.0 }}
    indices {{ 0, 1, 2,  0, 2, 3,  0, 3, 1,  1, 3, 2 }}
  }}
  level {{ 2 }}
  surface {{ @orange }}
  transform : SRT {{ scale {{ 0.9 }} translate {{ 0.9, 0.55, -0.4 }} }}
}}
Shape sheet : LoopSubdiv {{
  base : InlineMesh {{
    positions {{ -0.6, 0.0, 0.5,  0.6, 0.0, 0.5,  0.6, 0.9, 0.1,  -0.6, 0.9, 0.1 }}
    indices {{ 0, 1, 2, 0, 2, 3 }}
  }}
  level {{ 2 }}
  surface {{ @steel }}
  transform : SRT {{ rotate {{ 0.0, 1.0, 0.0, -20.0 }} translate {{ 0.2, 0.02, 1.3 }} }}
}}
Shape fan : LoopSubdiv {{
  mesh : InlineMesh {{
    positions {{ 0.0, 0.5, 0.0,  0.6, 0.0, 0.0,  0.3, 0.0, 0.55,  -0.3, 0.0, 0.55,  -0.6, 0.0, 0.0,  -0.3, 0.0, -0.55,  0.3, 0.0, -0.55 }}
    indices {{ 0, 1, 2,  0, 2, 3,  0, 3, 4,  0, 4, 5,  0, 5, 6 }}
  }}
  level {{ 1 }}
  shadow_terminator {{ 0.5 }}
  surface {{ @white }}
  transform : SRT {{ translate {{ -0.3, 0.01, -1.6 }} }}
}}
Shape passthrough : LoopSubdiv {{
  mesh : InlineMesh {{
    positions {{ 1.6, 0.0, -1.8,  2.4, 0.0, -1.8,  2.0, 1.2, -1.8 }}
    normals {{ 0.0, 0.3, 1.0,  0.2, 0.0, 1.0,  -0.2, 0.1, 1.0 }}
    indices {{ 0, 1, 2 }}
  }}
  level {{ 0 }}
  surface {{ @orange }}
}}
Camera camera : Pinhole {{
  position {{ 0.0, 2.2, 5.2 }}
  front {{ 0.0, -0.32, -1.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 42.0 }}
  spp {{ {spp} }}
  film : Color {{ resolution {{ {resolution[0]}, {resolution[1]} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}
render {{
  integrator : {integrator} {{
    depth {{ {depth} }}
    rr_depth {{ 0 }}
    rr_threshold {{ 0.95 }}
    sampler : Independent {{ seed {{ 19980810 }} }}
  }}
  cameras {{ @camera }}
  shapes {{ @floor, @lamp, @cube, @tetra, @sheet, @fan, @passthrough }}
}}
"""


def swizzle_scene(resolution=(64, 48), spp=4, output="swizzle.exr", assets="tests/golden/assets", integrator="WavePath") -> str:
    """The `Swizzle` texture (src/textures/swizzle.cpp) on the textured room: reordered image channels ("bgr" of an sRGB PNG,
    "gbr" of a gamma-decoded palette PNG), one channel of a four-channel 16-bit image as a scalar parameter (index list form),
    a swizzled constant, and a swizzle of a swizzle."""
    src = textured_room(resolution=resolution, spp=spp, mesh_files=False, assets=assets, output=output, integrator=integrator)
    a = assets.rstrip("/")

    def swap(text, old, new):
        assert text.count(old) == 1, old
        return text.replace(old, new)

    src = swap(src, f'Kd : Image {{ file {{ "{a}/checker_rgb8.png" }} address {{ "repeat" }} filter {{ "bilinear" }} uv_scale {{ 2.0, 3.0 }} uv_offset {{ 0.25, 0.0 }} }}',
               f'Kd : Swizzle {{ base : Image {{ file {{ "{a}/checker_rgb8.png" }} address {{ "repeat" }} filter {{ "bilinear" }} uv_scale {{ 2.0, 3.0 }} uv_offset {{ 0.25, 0.0 }} }} swizzle {{ "bgr" }} }}')
    src = swap(src, f'sigma : Image {{ file {{ "{a}/rough_gray8.png" }} encoding {{ "linear" }} filter {{ "point" }} }}',
               f'sigma : Swizzle {{ base : Image {{ file {{ "{a}/ramp_rgba16.png" }} encoding {{ "linear" }} scale {{ 40.0 }} }} swizzle {{ 1 }} }}')
    src = swap(src, 'metallic : Constant { v { 0.2 } }',
               'metallic : Swizzle { base : Swizzle { base : Constant { v { 0.9, 0.2, 0.5 } } swizzle { 2, 0, 1 } } swizzle { "z" } }')
    src = swap(src, f'Kd : Image {{ file {{ "{a}/palette4.png" }} address {{ "zero" }} encoding {{ "gamma" }} gamma {{ 2.0 }} }}',
               f'Kd : Swizzle {{ base : Image {{ file {{ "{a}/palette4.png" }} address {{ "zero" }} encoding {{ "gamma" }} gamma {{ 2.0 }} }} swizzle {{ "gbr" }} }}')
    return src


def checkerboard_scene(resolution=(64, 48), spp=4, output="checker.exr", assets="tests/golden/assets", integrator="WavePath") -> str:
    """The `Checkerboard` texture (src/textures/checkerboard.cpp) with constant squares on the textured room: RGB squares with
    an anisotropic scale, a scalar parameter (Oren-Nayar sigma), the default off texture (black)."""
    src = textured_room(resolution=resolution, spp=spp, mesh_files=False, assets=assets, output=output, integrator=integrator)
    a = assets.rstrip("/")

    def swap(text, old, new):
        assert text.count(old) == 1, old
        return text.replace(old, new)

    src = swap(src, f'Kd : Image {{ file {{ "{a}/checker_rgb8.png" }} address {{ "repeat" }} filter {{ "bilinear" }} uv_scale {{ 2.0, 3.0 }} uv_offset {{ 0.25, 0.0 }} }}',
               'Kd : Checkerboard { on : Constant { v { 0.8, 0.2, 0.2 } } off : Constant { v { 0.1, 0.1, 0.6 } } scale { 5.0, 7.0 } }')
    src = swap(src, f'sigma : Image {{ file {{ "{a}/rough_gray8.png" }} encoding {{ "linear" }} filter {{ "point" }} }}',
               'sigma : Checkerboard { on : Constant { v { 35.0 } } off : Constant { v { 0.0 } } scale { 3.0 } }')
    src = swap(src, f'Kd : Image {{ file {{ "{a}/palette4.png" }} address {{ "zero" }} encoding {{ "gamma" }} gamma {{ 2.0 }} }}',
               'Kd : Checkerboard { on : Constant { v { 0.9, 0.85, 0.3 } } scale { 2.5 } }')
    return src


IMAGE_FORMAT_FILES = ("bmp_rgb24.bmp", "bmp_pal8.bmp", "bmp_pal4.bmp", "bmp_pal1.bmp", "bmp_rgba32_topdown.bmp", "bmp_rgbx32.bmp", "bmp_rgb565.bmp",
                      "bmp_rgb555.bmp", "tga_rgb24.tga", "tga_rgba32_rle_topdown.tga", "tga_grey8.tga", "tga_grey_alpha16.tga", "tga_mapped8.tga",
                      "tga_rgb15.tga")
# the JPEG decoding paths of csrc/host/jpegload.cpp (grey, each chroma layout and its upsampling filter, progressive, RGB stored as such)
JPEG_FORMAT_FILES = ("jpg_grey.jpg", "jpg_444.jpg", "jpg_422.jpg", "jpg_420.jpg", "jpg_440.jpg", "jpg_411.jpg", "jpg_420_restart_optimized.jpg",
                     "jpg_420_low_quality.jpg", "jpg_progressive_420.jpg", "jpg_progressive_444_restart.jpg", "jpg_progressive_grey.jpg",
                     "jpg_progressive_440_restart.jpg", "jpg_rgb_by_ids.jpg", "jpg_rgb_by_adobe_marker.jpg", "jpg_444_q100_noise.jpg")


def image_formats_scene(resolution=(80, 48), spp=2, output="formats.exr", assets="tests/golden/assets", integrator="WavePath",
                        files=IMAGE_FORMAT_FILES) -> str:
    """One point-sampled Matte panel per BMP / TGA storage variant of tests/golden/assets (5 x 3 panels facing the camera, lit by an
    area light behind it): the film is a function of every texel the readers of csrc/host/imageload.cpp produce, next to what
    stb_image hands the reference for the same files."""
    a = assets.rstrip("/")
    parts, names = [], []
    for k, name in enumerate(files):
        col, row = k % 5, k // 5
        x0, y0 = -2.5 + col * 1.0 + 0.05, 1.9 - row * 1.0 + 0.05
        x1, y1 = x0 + 0.9, y0 - 0.9
        encoding = ("linear", "sRGB")[k % 2]
        parts.append(f'''
Surface s{k} : Matte {{ Kd : Image {{ file {{ "{a}/{name}" }} filter {{ "point" }} address {{ "edge" }} encoding {{ "{encoding}" }} }} }}
Shape p{k} : InlineMesh {{
  positions {{ {_fmt(x0)}, {_fmt(y1)}, 0.0,  {_fmt(x1)}, {_fmt(y1)}, 0.0,  {_fmt(x1)}, {_fmt(y0)}, 0.0,  {_fmt(x0)}, {_fmt(y0)}, 0.0 }}
  uvs {{ 0.0, 1.0,  1.0, 1.0,  1.0, 0.0,  0.0, 0.0 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  surface {{ @s{k} }}
}}''')
        names.append(f"@p{k}")
    return "".join(parts) + f'''
Light area_light : Diffuse {{ emission : Constant {{ v {{ 30.0 }} }} }}
Shape lamp : InlineMesh {{
  positions {{ -1.5, 3.5, 4.0,  1.5, 3.5, 4.0,  1.5, 2.5, 5.0,  -1.5, 2.5, 5.0 }}
  indices {{ 0, 1, 2, 0, 2, 3 }}
  light {{ @area_light }}
}}
Camera camera : Pinhole {{
  position {{ 0.0, 0.4, 5.2 }}
  front {{ 0.0, 0.0, -1.0 }}
  up {{ 0.0, 1.0, 0.0 }}
  fov {{ 38.0 }}
  spp {{ {int(spp)} }}
  film : Color {{ resolution {{ {int(resolution[0])}, {int(resolution[1])} }} }}
  filter : Box {{ radius {{ 0.5 }} }}
  file {{ "{output}" }}
}}
render {{
  integrator : {integrator} {{
    depth {{ 3 }}
    sampler : Independent {{ seed {{ 7 }} }}
  }}
  cameras {{ @camera }}
  shapes {{ {", ".join(names)}, @lamp }}
}}
'''
