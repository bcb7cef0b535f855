"""The scene of the batched frame-sensor fixture (tools/make_sensor_goldens.py, tests/golden/sensor_batched.npz) and of the tests
that read it.

A free body and a hinged two-link arm, each carrying geoms, sites and a camera with rotated local frames, no collisions.  framequat,
framepos and framexaxis of every object type (body, xbody, geom, site, camera), in the world frame and against every reference type.
`batched` turns body_iquat, geom_quat, site_quat and cam_quat per world: each entry is the nominal quaternion times a different small
rotation, and the reference reads entry w % nb, so world 3 of 4 sees a different local frame from world 0 on every object."""

import numpy as np

NWORLD = 4
NB = 3  # batch entries: fewer than the worlds, so world 3 reads entry 0 again

OBJ = (("body", "arm1"), ("xbody", "free"), ("geom", "g_arm2"), ("site", "s_free"), ("camera", "c_arm2"))

XML = """
<mujoco model="sensor_batched">
  <option timestep="0.004"/>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <body name="free" pos="0.3 -0.2 1.0" euler="10 -20 30">
      <freejoint/>
      <geom name="g_free" type="box" size="0.05 0.08 0.03" pos="0.02 0 0" euler="5 10 15" mass="0.6"/>
      <geom type="sphere" size="0.03" pos="-0.06 0.04 0.02" mass="0.3"/>
      <site name="s_free" pos="0.05 0.02 -0.01" euler="30 0 -40"/>
      <camera name="c_free" pos="0 -0.2 0.1" euler="70 0 10"/>
    </body>
    <body name="arm1" pos="-0.4 0 0.8" euler="0 15 0">
      <joint name="h1" type="hinge" axis="0 1 0"/>
      <geom name="g_arm1" type="capsule" fromto="0 0 0 0.3 0.02 0" size="0.03" mass="0.5"/>
      <geom type="box" size="0.02 0.04 0.02" pos="0.1 0.03 0" euler="0 0 25" mass="0.2"/>
      <site name="s_arm1" pos="0.15 0 0.03" euler="-15 25 5"/>
      <body name="arm2" pos="0.3 0 0" euler="20 0 0">
        <joint name="h2" type="hinge" axis="1 0 0"/>
        <geom name="g_arm2" type="capsule" fromto="0 0 0 0 0.25 0" size="0.025" euler="0 0 10" mass="0.4"/>
        <geom type="sphere" size="0.02" pos="0.03 0.2 0.01" mass="0.15"/>
        <site name="s_arm2" pos="0 0.2 0" euler="40 -10 20"/>
        <camera name="c_arm2" pos="0 0.1 0.1" euler="-30 20 0"/>
      </body>
    </body>
  </worldbody>
  <sensor>
    {sensors}
  </sensor>
</mujoco>"""


def sensors():
  out = []
  for ot, on in OBJ:
    for kind in ("framequat", "framepos", "framexaxis"):
      out.append(f'<{kind} objtype="{ot}" objname="{on}"/>')
      for rt, rn in OBJ:
        out.append(f'<{kind} objtype="{ot}" objname="{on}" reftype="{rt}" refname="{rn}"/>')
  return "\n    ".join(out)


def load():
  from mujoco_warp_b200._src import mjcf

  return mjcf.load_string(XML.format(sensors=sensors()))


def _qmul(u, v):
  w1, x1, y1, z1 = np.moveaxis(u, -1, 0)
  w2, x2, y2, z2 = np.moveaxis(v, -1, 0)
  return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                   w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1)


def batched(mjm, nb=NB, seed=5):
  """Per-world body_iquat, geom_quat, site_quat and cam_quat (nb, n, 4): the nominal entry times a small rotation of its own, unit
  length and fp32-representable (so the GPU holds exactly what the fixture's reference run read)."""
  rng = np.random.default_rng(seed)
  out = {}
  for n in ("body_iquat", "geom_quat", "site_quat", "cam_quat"):
    q0 = np.asarray(getattr(mjm, n), dtype=np.float64).reshape(-1, 4)
    d = np.concatenate([np.ones((nb, len(q0), 1)), rng.uniform(-0.3, 0.3, (nb, len(q0), 3))], -1)
    q = _qmul(np.broadcast_to(q0, d.shape), d / np.linalg.norm(d, axis=-1, keepdims=True))
    out[n] = (q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(np.float32).astype(np.float64)
  return out


def state(mjm, nworld=NWORLD, seed=9):
  """Per-world qpos (the free body moved and turned, both hinges bent) and qvel, fp32-representable."""
  from tests import util

  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=None, seed=seed, qpos_noise=0.3, qvel_noise=1.0, exact_world0=False)
  q = qpos[:, 3:7]
  qpos[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(qpos), f32(qvel)
