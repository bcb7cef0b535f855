"""Scenes of the renderer's tests (tests/test_render_host.py, tests/test_gpu_render.py) and of its reference fixtures
(tools/make_render_goldens.py -> tests/golden/render_<name>.npz for every entry of SCENES).

PRIMITIVES: every primitive type and a mesh on a plane, materials with specular / shininess / emission, a directional, a spot and a
point light with non-default attenuation, cutoff and exponent, a light that casts no shadow, a tracking camera and a targeted light on
a moving body, a fixed perspective camera, an orthographic one and a sensorsize / focalpixel one, and geoms outside groups 0-2.
"""

PRIMITIVES = """
<mujoco model="render_primitives">
  <visual><headlight ambient="0.15 0.15 0.15" diffuse="0.3 0.3 0.3" specular="0.2 0.2 0.2"/></visual>
  <default>
    <default class="shiny"><geom material="gloss"/></default>
    <light attenuation="1 0.05 0.01"/>
  </default>
  <asset>
    <material name="gloss" rgba="0.8 0.2 0.2 1" specular="0.9" shininess="0.8"/>
    <material name="glow" rgba="0.2 0.8 0.3 1" emission="0.6" specular="0.1" shininess="0.2"/>
    <material name="floor" rgba="0.6 0.6 0.65 1"/>
    <mesh name="tet" vertex="0 0 0  0.3 0 0  0 0.3 0  0 0 0.3"/>
  </asset>
  <worldbody>
    <light name="sun" directional="true" pos="0 0 5" dir="0.3 0.2 -1" diffuse="0.5 0.5 0.5" castshadow="true"/>
    <light name="spot" type="spot" pos="1 -1 3" dir="-0.3 0.3 -1" cutoff="35" exponent="4" diffuse="0.6 0.5 0.4" specular="0.4 0.4 0.4" ambient="0.05 0.05 0.05"/>
    <light name="bulb" type="point" pos="-1 1 1.5" castshadow="false" diffuse="0.3 0.3 0.5" attenuation="1 0.2 0.05"/>
    <camera name="overview" pos="0 -3.2 2.2" xyaxes="1 0 0 0 0.55 0.83" fovy="50" resolution="31 23"/>
    <camera name="ortho" pos="0 0 4" projection="orthographic" fovy="4" resolution="17 13"/>
    <camera name="sensor" pos="2.2 -2.2 2.2" xyaxes="0.707 0.707 0 -0.5 0.5 0.707" sensorsize="0.006 0.004" focalpixel="20 20" resolution="25 19"/>
    <geom name="floor" type="plane" size="0 0 0.1" material="floor"/>
    <geom name="box" type="box" pos="0.7 0.4 0.25" size="0.2 0.15 0.25" euler="0 0 30" class="shiny"/>
    <geom name="cyl" type="cylinder" pos="-0.7 0.5 0.3" size="0.18 0.3" material="glow"/>
    <geom name="ell" type="ellipsoid" pos="-0.6 -0.5 0.3" size="0.25 0.15 0.3" rgba="0.2 0.3 0.9 1"/>
    <geom name="tet" type="mesh" mesh="tet" pos="0.5 -0.6 0.01" rgba="0.9 0.8 0.2 1"/>
    <geom name="hidden" type="sphere" pos="0 0 1.8" size="0.3" group="4" rgba="1 0 1 1"/>
    <body name="mover" pos="0 0 0.6">
      <joint name="slide" type="slide" axis="1 0 0"/>
      <joint name="hinge" type="hinge" axis="0 1 0"/>
      <geom name="ball" type="sphere" size="0.2" rgba="0.9 0.9 0.9 1"/>
      <geom name="cap" type="capsule" fromto="0 0 0.2 0 0 0.6" size="0.08" class="shiny"/>
    </body>
    <camera name="tracker" mode="trackcom" pos="0 -2 1.2" xyaxes="1 0 0 0 0.5 0.87" resolution="21 15"/>
    <light name="follow" mode="targetbody" target="mover" pos="0 2 2" diffuse="0.2 0.2 0.2" cutoff="60"/>
  </worldbody>
</mujoco>
"""

# No lights (the 0.3 ambient fallback) and no headlight; one camera inside the sphere
NOLIGHT = """
<mujoco model="render_nolight">
  <visual><headlight active="0"/></visual>
  <worldbody>
    <camera name="inside" pos="0 0 0.5" resolution="15 11"/>
    <camera name="outside" pos="0 -2 0.5" xyaxes="1 0 0 0 0 1" resolution="19 13"/>
    <geom name="floor" type="plane" size="3 3 0.1" rgba="0.5 0.5 0.5 1"/>
    <geom name="shell" type="sphere" pos="0 0 0.5" size="0.4" rgba="0.8 0.3 0.3 1"/>
    <body name="b" pos="0.6 0 0.3">
      <freejoint/>
      <geom type="box" size="0.1 0.1 0.1" rgba="0.2 0.7 0.2 1"/>
    </body>
  </worldbody>
</mujoco>
"""

NWORLD = 3


def qpos(mjm, nworld, seed):
  """seeded joint positions: the first two qpos entries (PRIMITIVES: the moving body's slide and hinge; NOLIGHT: the free box's x, y)
  moved by up to 0.3 in every world"""
  import numpy as np

  rng = np.random.default_rng(seed)
  q = np.tile(np.asarray(mjm.qpos0, dtype=np.float64), (nworld, 1))
  q[:, :2] += rng.uniform(-0.3, 0.3, size=(nworld, 2))
  return q


def batch_fields(mjm, sc):
  """per-world values of the fields named in sc["batch"] ({field: entries}): entry 0 is the model's value, the others seeded"""
  import numpy as np

  rng = np.random.default_rng(sc.get("seed", 0) + 100)
  out = {}
  for k, n in sc.get("batch", {}).items():
    base = np.asarray(getattr(mjm, k), dtype=np.float64)
    v = np.repeat(base[None], n, axis=0)
    for i in range(1, n):
      if k in ("geom_rgba", "mat_rgba"):
        v[i, ..., :3] = rng.uniform(0.1, 0.9, size=v[i, ..., :3].shape)
      elif k == "light_diffuse":
        v[i] = base * rng.uniform(0.3, 0.8)
      elif k == "cam_fovy":
        v[i] = base * 0.7
    out[k] = np.asarray(v, dtype=np.float32).astype(np.float64)
  return out


_ALL = dict(render_rgb=True, render_depth=True, render_seg=True)
_NO_HEADLIGHT = PRIMITIVES.replace('<headlight ambient="0.15 0.15 0.15"', '<headlight active="0" ambient="0.15 0.15 0.15"')
# the reference fixtures: every scene renders rgb, depth and segmentation of its active cameras in NWORLD worlds
SCENES = {
  # every primitive and a mesh on a plane, materials, directional / spot / point lights, the orthographic and sensorsize / focalpixel
  # cameras, the tracking camera and the targeted light on the moving body; shadows off
  "primitives": dict(xml=PRIMITIVES, kwargs=dict(_ALL)),
  "shadows": dict(xml=PRIMITIVES, kwargs=dict(_ALL, use_shadows=True), seed=1),
  # headlight off with lights; specular, emission and per-light ambient off; groups 0, 2 and 4; cameras by name
  "switches": dict(xml=_NO_HEADLIGHT, kwargs=dict(_ALL, enable_specular=False, enable_emission=False, enable_per_light_ambient=False,
                                                  enabled_geom_groups=[0, 2, 4], cam_active=["overview", "tracker"]), seed=2),
  "no_ambient": dict(xml=PRIMITIVES, kwargs=dict(_ALL, use_ambient_lighting=False, use_shadows=True, cam_active=["overview", "sensor"]), seed=3),
  # per-world geom_rgba / mat_rgba / light_diffuse / cam_fovy (rays computed per world)
  "per_world": dict(xml=PRIMITIVES, kwargs=dict(_ALL, use_precomputed_rays=False, cam_active=["overview", "tracker"]), seed=4,
                    batch=dict(geom_rgba=2, mat_rgba=2, light_diffuse=2, cam_fovy=2)),
  # no lights (the ambient fallback), no headlight; a camera inside a sphere, culled and not
  "nolight": dict(xml=NOLIGHT, kwargs=dict(_ALL)),
  "nolight_nocull": dict(xml=NOLIGHT, kwargs=dict(_ALL, enable_backface_culling=False), seed=5),
}
