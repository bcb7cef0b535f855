"""Scenes whose mesh hulls exceed the fixed multi-contact buffers of the CCD_MESH = 1 collision build (a hull polygon of more than 32
vertices, or a hull vertex shared by more than 16 polygons), with the meshes generated here as inline `vertex=` assets.

- prism48 / prism64 / prism96: N-gon prisms (cylinder hulls) cap-down on the floor (plane-mesh) and on a box (face-face, the large polygon on
  one side), cap-to-cap on a fixed prism (large polygons on both sides), and tilted onto their rim on a box (the edge-face branches).
- cone: 24-segment cones apex-down on a box (a hull vertex of degree 24, the one-vertex feature) and on the floor.
- uvsphere: 32-segment UV spheres pole-down on a box and on a fixed 48-gon prism (pole degree 32), and on the floor.
- mixed: in-cap hulls (cubes, a 16-gon prism) next to one 64-gon prism; MIXED_INCAP is the same model without the large prism.
- sensors: distance / normal / fromto sensors between two 64-gon prisms and between a prism and a cone.

Every scene runs 8 worlds from seeded poses (SCENES[name]["cfg"]), so that contacts differ per world.
"""
import numpy as np

NWORLD = 8


def _fmt(v):
  return " ".join(f"{x:.6f}" for x in np.asarray(v, dtype=np.float64).reshape(-1))


def prism(n, r=0.08, h=0.04):
  """Vertices of an n-gon prism around z: two n-gon caps at z = -h and z = +h."""
  a = 2 * np.pi * np.arange(n) / n
  ring = np.stack([r * np.cos(a), r * np.sin(a)], axis=1)
  return np.concatenate([np.c_[ring, -h * np.ones(n)], np.c_[ring, h * np.ones(n)]])


def cone(n, r=0.06, h=0.05):
  """Apex at z = -h (shared by the n side triangles) and an n-gon base at z = +h."""
  a = 2 * np.pi * np.arange(n) / n
  return np.concatenate([[[0.0, 0.0, -h]], np.c_[r * np.cos(a), r * np.sin(a), h * np.ones(n)]])


def uvsphere(nseg, nring=8, radius=0.06):
  """Poles on z (each shared by nseg triangles) and nring - 1 rings of nseg vertices."""
  out = [[0.0, 0.0, -radius], [0.0, 0.0, radius]]
  for i in range(1, nring):
    th = np.pi * i / nring
    a = 2 * np.pi * np.arange(nseg) / nseg
    out.extend(np.c_[radius * np.sin(th) * np.cos(a), radius * np.sin(th) * np.sin(a), -radius * np.cos(th) * np.ones(nseg)].tolist())
  return np.asarray(out)


_HEAD = """<mujoco>
  <option timestep="0.002" iterations="50"/>
  <default><geom friction="0.9 0.01 0.002" density="600"/></default>"""

DEPTH = 0.0005  # every resting hull starts this far into its support


def prism_xml(n):
  r, h, tilt = 0.08, 0.04, 20.0
  tz = h * np.cos(np.radians(tilt)) + r * np.sin(np.radians(tilt))
  return f"""{_HEAD}
  <asset><mesh name="prism" vertex="{_fmt(prism(n, r, h))}"/></asset>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 .05"/>
    <geom name="table" type="box" size="0.15 0.15 0.05" pos="0.5 0 0.05"/>
    <geom name="ramp" type="box" size="0.15 0.15 0.05" pos="0 -0.6 0.05"/>
    <geom name="base" type="mesh" mesh="prism" pos="0 0.6 {h:.6f}"/>
    <body pos="-0.5 0 {h - DEPTH:.6f}"><freejoint/><geom name="on_floor" type="mesh" mesh="prism"/></body>
    <body pos="0.5 0 {0.1 + h - DEPTH:.6f}" euler="0 0 7"><freejoint/><geom name="on_table" type="mesh" mesh="prism"/></body>
    <body pos="0.01 0.6 {3 * h - DEPTH:.6f}" euler="0 0 3"><freejoint/><geom name="on_base" type="mesh" mesh="prism"/></body>
    <body pos="0 -0.6 {0.1 + tz - DEPTH:.6f}" euler="0 {tilt} 0"><freejoint/><geom name="on_rim" type="mesh" mesh="prism"/></body>
  </worldbody>
</mujoco>"""


def cone_xml(n=24):
  h = 0.05
  return f"""{_HEAD}
  <asset><mesh name="cone" vertex="{_fmt(cone(n, 0.06, h))}"/></asset>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 .05"/>
    <geom name="table" type="box" size="0.15 0.15 0.05" pos="0.5 0 0.05"/>
    <body pos="0.5 0 {0.1 + h - DEPTH:.6f}"><freejoint/><geom name="apex_on_table" type="mesh" mesh="cone"/></body>
    <body pos="-0.5 0 {h - DEPTH:.6f}" euler="0 0 11"><freejoint/><geom name="apex_on_floor" type="mesh" mesh="cone"/></body>
  </worldbody>
</mujoco>"""


def uvsphere_xml(nseg=32):
  rad, h = 0.06, 0.04
  return f"""{_HEAD}
  <asset>
    <mesh name="ball" vertex="{_fmt(uvsphere(nseg, 8, rad))}"/>
    <mesh name="prism" vertex="{_fmt(prism(48, 0.08, h))}"/>
  </asset>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 .05"/>
    <geom name="table" type="box" size="0.15 0.15 0.05" pos="0.5 0 0.05"/>
    <geom name="base" type="mesh" mesh="prism" pos="0 0.6 {h:.6f}"/>
    <body pos="0.5 0 {0.1 + rad - DEPTH:.6f}"><freejoint/><geom name="pole_on_table" type="mesh" mesh="ball"/></body>
    <body pos="0 0.6 {2 * h + rad - DEPTH:.6f}"><freejoint/><geom name="pole_on_prism" type="mesh" mesh="ball"/></body>
    <body pos="-0.5 0 {rad - DEPTH:.6f}"><freejoint/><geom name="pole_on_floor" type="mesh" mesh="ball"/></body>
  </worldbody>
</mujoco>"""


def mixed_xml(large=True):
  h, cube = 0.04, "-1 -1 -1  1 -1 -1  -1 1 -1  1 1 -1  -1 -1 1  1 -1 1  -1 1 1  1 1 1"
  big = f"""
    <body pos="0 -0.6 {h - DEPTH:.6f}"><freejoint/><geom name="big" type="mesh" mesh="big"/></body>""" if large else ""
  big_asset = f"""
    <mesh name="big" vertex="{_fmt(prism(64, 0.08, h))}"/>""" if large else ""
  return f"""{_HEAD}
  <asset>
    <mesh name="cube" vertex="{cube}" scale="0.1 0.08 0.05"/>
    <mesh name="small" vertex="{_fmt(prism(16, 0.06, h))}"/>{big_asset}
  </asset>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 .05"/>
    <geom name="table" type="box" size="0.15 0.15 0.05" pos="0.5 0 0.05"/>
    <body pos="-0.5 0 {0.05 - DEPTH:.6f}"><freejoint/><geom name="cube_a" type="mesh" mesh="cube"/></body>
    <body pos="-0.48 0.01 {0.15 - 2 * DEPTH:.6f}" euler="0 0 25"><freejoint/><geom name="cube_b" type="mesh" mesh="cube"/></body>
    <body pos="0.5 0 {0.1 + h - DEPTH:.6f}" euler="0 0 5"><freejoint/><geom name="small_on_table" type="mesh" mesh="small"/></body>
    <body pos="0 0.6 {0.05 - DEPTH:.6f}"><freejoint/><geom name="box_on_floor" type="box" size="0.05 0.05 0.05"/></body>{big}
  </worldbody>
</mujoco>"""


def sensors_xml():
  h = 0.04
  return f"""{_HEAD}
  <asset>
    <mesh name="prism" vertex="{_fmt(prism(64, 0.08, h))}"/>
    <mesh name="cone" vertex="{_fmt(cone(24, 0.06, 0.05))}"/>
  </asset>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 .05"/>
    <body pos="-0.2 0 {h - DEPTH:.6f}"><freejoint/><geom name="p1" type="mesh" mesh="prism"/></body>
    <body pos="0.0 0 {3 * h + 0.01:.6f}" euler="0 25 0"><freejoint/><geom name="p2" type="mesh" mesh="prism"/></body>
    <body pos="0.25 0.05 {0.05 - DEPTH:.6f}"><freejoint/><geom name="c1" type="mesh" mesh="cone"/></body>
  </worldbody>
  <sensor>
    <distance geom1="p1" geom2="p2" cutoff="1"/>
    <normal geom1="p1" geom2="p2" cutoff="1"/>
    <fromto geom1="p1" geom2="p2" cutoff="1"/>
    <distance geom1="p2" geom2="c1" cutoff="1"/>
    <fromto geom1="c1" geom2="p2" cutoff="1"/>
  </sensor>
</mujoco>"""


_CFG = dict(nconmax=48, njmax=256, key=None, qpos_noise=0.0004, qvel_noise=0.05, ctrl_noise=0.0, exact_world0=False)
# name -> xml, the compiled npolygonmax / nmeshdegmax it is designed for, and the fixture's state / capacity settings
SCENES = {
  "prism48": dict(xml=prism_xml(48), npolygonmax=48, nmeshdegmax=3, cfg=_CFG),
  "prism64": dict(xml=prism_xml(64), npolygonmax=64, nmeshdegmax=3, cfg=_CFG),
  "prism96": dict(xml=prism_xml(96), npolygonmax=96, nmeshdegmax=3, cfg=_CFG),
  "cone": dict(xml=cone_xml(24), npolygonmax=24, nmeshdegmax=24, cfg=_CFG),
  "uvsphere": dict(xml=uvsphere_xml(32), npolygonmax=48, nmeshdegmax=32, cfg=_CFG),
  "mixed": dict(xml=mixed_xml(True), npolygonmax=64, nmeshdegmax=3, cfg=_CFG),
  "sensors": dict(xml=sensors_xml(), npolygonmax=64, nmeshdegmax=24, cfg=_CFG),
}
MIXED_INCAP = mixed_xml(False)  # the mixed scene without its large prism: every hull within the fixed buffers


def load(name):
  from mujoco_warp_b200._src import mjcf

  return mjcf.load_string(SCENES[name]["xml"] if name in SCENES else name)


def seeded(mjm, name):
  """The scene's per-world starting state (qpos, qvel, ctrl, qacc_warmstart), exactly representable in fp32."""
  from tests import util

  cfg = {k: v for k, v in SCENES[name]["cfg"].items() if k not in ("nconmax", "njmax")}
  qpos, qvel, ctrl, warm = util.seeded_state(mjm, NWORLD, seed=4321, **cfg)
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(qpos), f32(qvel), f32(ctrl), f32(warm)
