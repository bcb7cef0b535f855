"""Scenes and seeded inputs of the body-stage fixtures (rne_postconstraint, subtree_vel, jac, xfrc_accumulate, tendon, deriv_smooth_vel),
shared by tools/make_body_stage_goldens.py and the tests that read tests/golden/body_stage_<scene>.npz.

Each scene: (loader, per_world).  per_world scenes batch body_mass, body_inertia and dof_damping over the worlds."""

import numpy as np

from tests import fluid_scenes, util

NWORLD = 4

# a free box on a hinged arm with a tendon, an affine position servo and a velocity servo: dof and tendon damping, implicitfast
TENDON_ACTUATOR_XML = """
<mujoco model="tendon_actuator">
  <option timestep="0.004" integrator="implicitfast"/>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 .05"/>
    <body name="a0" pos="0 0 0.6">
      <joint name="a0" type="hinge" axis="0 1 0" damping="0.3" armature="0.01"/>
      <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.03" mass="0.5"/>
      <body name="a1" pos="0.2 0 0">
        <joint name="a1" type="hinge" axis="0 1 0" damping="0.1"/>
        <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.025" mass="0.3"/>
        <body name="a2" pos="0.2 0 0">
          <joint name="a2" type="slide" axis="1 0 0" damping="0.2"/>
          <geom type="box" size="0.03 0.03 0.03" mass="0.2"/>
        </body>
      </body>
    </body>
    <body name="free" pos="0.5 0 0.2">
      <freejoint/>
      <geom type="box" size="0.05 0.04 0.03" mass="0.4"/>
    </body>
  </worldbody>
  <tendon>
    <fixed name="t0" damping="0.4"><joint joint="a0" coef="1"/><joint joint="a1" coef="-0.5"/></fixed>
    <fixed name="t1" damping="0.25"><joint joint="a1" coef="0.7"/><joint joint="a2" coef="2"/></fixed>
  </tendon>
  <actuator>
    <position joint="a0" kp="20" kv="2"/>
    <velocity joint="a1" kv="1.5"/>
    <general tendon="t1" gaintype="affine" gainprm="3 0.5 -0.4" biastype="affine" biasprm="0.1 -2 -0.3"/>
  </actuator>
</mujoco>"""


def _humanoid(cone):
  from mujoco_warp_b200._src import mjcf

  mjm = mjcf.load_any(util.HUMANOID)
  mjm.opt.cone = cone
  return mjm


def _load_string(xml):
  from mujoco_warp_b200._src import mjcf

  return mjcf.load_string(xml)


def _water(integrator):
  return fluid_scenes.ellipsoid_xml(integrator).replace('density="1.2" viscosity="0.00002"', 'density="1000" viscosity="0.001"')


def _g1():
  from mujoco_warp_b200._src import mjcf

  return mjcf.load_any(util.G1)


SCENES = {
  "humanoid_pyramidal": (lambda: _humanoid(0), False),
  "humanoid_elliptic": (lambda: _humanoid(1), False),
  "equality": (lambda: _load_string(util.EQUALITY_XML), False),
  "tendon_actuator": (lambda: _load_string(TENDON_ACTUATOR_XML), False),
  "fluid": (lambda: _load_string(fluid_scenes.ellipsoid_xml("implicitfast")), False),
  # the ellipsoid model in water: its B is far from symmetric, which implicitfast symmetrizes and the other integrators do not
  "fluid_water_euler": (lambda: _load_string(_water("Euler")), False),
  "fluid_water_rk4": (lambda: _load_string(_water("RK4")), False),
  "fluid_water_implicitfast": (lambda: _load_string(_water("implicitfast")), False),
  "batched": (lambda: _load_string(TENDON_ACTUATOR_XML), True),
  "g1": (_g1, False),
}


SCENES_BATCHED = {k: v[1] for k, v in SCENES.items()}


def load(name):
  return SCENES[name][0]()


def seeded(mjm, nworld=NWORLD, seed=7):
  """qpos / qvel / ctrl (util.seeded_state; a humanoid or G1 is lowered onto the floor so its feet touch), act, xfrc_applied on three
  bodies per world, the jac points and bodies (world 0 asks for body 0) and a non-zero qfrc for xfrc_accumulate."""
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld, seed=seed)
  if mjm.njnt and int(mjm.jnt_type[0]) == 0 and mjm.nbody > 20:
    qpos[:, 2] -= 0.03
  rng = np.random.default_rng(seed + 1)
  act = rng.uniform(-0.5, 0.5, (nworld, mjm.na)) if mjm.na else np.zeros((nworld, 0))
  xfrc = np.zeros((nworld, mjm.nbody, 6))
  for w in range(nworld):
    for b in rng.choice(np.arange(1, mjm.nbody), size=min(3, mjm.nbody - 1), replace=False):
      xfrc[w, b, :3] = rng.uniform(-5.0, 5.0, 3)
      xfrc[w, b, 3:] = rng.uniform(-0.5, 0.5, 3)
  body = rng.integers(0, mjm.nbody, nworld).astype(np.int32)
  body[0] = 0
  point = rng.uniform(-0.5, 0.5, (nworld, 3)) + np.array([0.0, 0.0, 0.8])
  qfrc = rng.uniform(-1.0, 1.0, (nworld, mjm.nv))
  return dict(qpos=qpos, qvel=qvel, ctrl=ctrl, act=act, xfrc_applied=xfrc, body=body, point=point, qfrc=qfrc)


def batched(mjm, nworld=NWORLD, seed=3):
  """Per-world body_mass, body_inertia and dof_damping: the nominal values scaled per world."""
  rng = np.random.default_rng(seed)
  s = rng.uniform(0.7, 1.4, (nworld, 1))
  mass = np.asarray(mjm.body_mass, dtype=np.float64)[None] * s
  inertia = np.asarray(mjm.body_inertia, dtype=np.float64)[None] * s[:, :, None]
  damping = np.asarray(mjm.dof_damping, dtype=np.float64)[None] * rng.uniform(0.5, 2.0, (nworld, 1))
  return mass, inertia, damping
