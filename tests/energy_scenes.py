"""Scenes for potential / kinetic energy (tests/test_energy_*.py, tests/test_gpu_energy.py, tools/make_energy_goldens.py).

Each scene is a model, the enable / disable flags it runs with, and the Model fields it randomises per world.  Worlds start from seeded
per-world qpos / qvel (fp32-representable).  The joint scenes have no contacts (no geom collides), so their steps are smooth.
"""
import numpy as np

NWORLD = 3
ENBL_ENERGY = 1 << 1
DSBL_SPRING, DSBL_GRAVITY = 1 << 5, 1 << 7

# hinge / slide / ball / free joints with stiffness; hinge and slide with a spring reference away from qpos0
JOINTS = """
<mujoco model="energy_joints">
  <option timestep="0.002" integrator="{integrator}"/>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <body name="h" pos="0 0 1">
      <joint name="hinge" type="hinge" axis="0 1 0" stiffness="3" springref="20" damping="0"/>
      <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03"/>
      <body name="s" pos="0.3 0 0">
        <joint name="slide" type="slide" axis="1 0 0" stiffness="40" springref="0.05"/>
        <geom type="box" size="0.05 0.04 0.03"/>
        <body name="b" pos="0.1 0 0">
          <joint name="ball" type="ball" stiffness="2"/>
          <geom type="capsule" fromto="0 0 0 0 0 -0.2" size="0.02"/>
        </body>
      </body>
    </body>
    <body name="f" pos="1 0 1">
      <joint name="free" type="free" stiffness="5"/>
      <geom type="box" size="0.1 0.07 0.05"/>
    </body>
    <body name="plain" pos="-1 0 1">
      <joint name="h2" type="hinge" axis="1 0 0"/>
      <geom type="capsule" fromto="0 0 0 0 0.2 0" size="0.02"/>
    </body>
  </worldbody>
  {sensors}
</mujoco>"""

# fixed tendons with stiffness: a two-sided dead band, a single spring length, and one without stiffness
TENDON = """
<mujoco model="energy_tendon">
  <option timestep="0.002"/>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <body name="a0" pos="0 0 0.6">
      <joint name="a0" type="hinge" axis="0 1 0"/>
      <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.03"/>
      <body name="a1" pos="0.2 0 0">
        <joint name="a1" type="hinge" axis="0 1 0"/>
        <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.025"/>
      </body>
    </body>
    <body name="s" pos="-0.4 0 0.3">
      <joint name="pz" type="slide" axis="0 0 1"/>
      <geom type="box" size="0.05 0.04 0.02"/>
    </body>
  </worldbody>
  <tendon>
    <fixed name="band" stiffness="20" springlength="-0.1 0.1"><joint joint="a0" coef="0.5"/><joint joint="a1" coef="-0.5"/><joint joint="pz" coef="0.3"/></fixed>
    <fixed name="point" stiffness="7" springlength="0.05"><joint joint="a1" coef="1"/><joint joint="pz" coef="0.7"/></fixed>
    <fixed name="slack"><joint joint="pz" coef="2"/></fixed>
  </tendon>
</mujoco>"""

SENSORS = """<sensor>
    <jointpos joint="hinge"/>
    <e_potential name="pot"/>
    <e_kinetic name="kin"/>
    <e_potential name="pot_cut" cutoff="0.5"/>
    <e_kinetic name="kin_cut" cutoff="0.05"/>
    <clock/>
  </sensor>"""


def joints_xml(integrator="Euler", sensors=False):
  return JOINTS.format(integrator=integrator, sensors=SENSORS if sensors else "")


def load(name):
  """The scene's compiled model, with its enable / disable flags applied."""
  from mujoco_warp_b200._src import mjcf
  from tests import util

  src, enable, disable = SCENES[name][:3]
  mjm = mjcf.load_any(src) if src in (util.HUMANOID, util.G1) else mjcf.load_string(src)
  mjm.opt.enableflags = int(mjm.opt.enableflags) | enable
  mjm.opt.disableflags = int(mjm.opt.disableflags) | disable
  return mjm


def per_world_inputs(name, mjm, nworld=NWORLD, seed=11):
  """{Model field: (nworld, ...) float64, fp32-representable} the scene randomises per world."""
  rng = np.random.default_rng(seed)
  tile = lambda a: np.repeat(np.asarray(a, dtype=np.float64)[None], nworld, axis=0)
  fields = SCENES[name][3]
  out = {}
  if "body_mass" in fields:
    out["body_mass"] = tile(mjm.body_mass) * rng.uniform(0.6, 1.6, (nworld, mjm.nbody))
  if "jnt_stiffness" in fields:
    out["jnt_stiffness"] = tile(mjm.jnt_stiffness) * rng.uniform(0.5, 2.0, (nworld, mjm.njnt))
  if "qpos_spring" in fields:
    qs = tile(mjm.qpos_spring)
    for j in range(mjm.njnt):
      a, t = int(mjm.jnt_qposadr[j]), int(mjm.jnt_type[j])
      if t == 0:
        qs[:, a : a + 3] += rng.normal(0, 0.1, (nworld, 3))
      if t in (0, 1):
        r = a + 3 if t == 0 else a
        q = rng.normal(0, 0.3, (nworld, 4))
        q[:, 0] += 1.0
        qs[:, r : r + 4] = q / np.linalg.norm(q, axis=1, keepdims=True)
      else:
        qs[:, a] += rng.normal(0, 0.2, nworld)
    out["qpos_spring"] = qs
  if "tendon_lengthspring" in fields:
    # per world: a band the tendon sits inside, one above it and one below it (and the single-length spring moved about)
    ls = tile(mjm.tendon_lengthspring)
    shift = np.array([0.0, 0.3, -0.3])[np.arange(nworld) % 3]
    ls[:, 0, :] += shift[:, None]
    ls[:, 1, :] += rng.normal(0, 0.05, (nworld, 1))
    out["tendon_lengthspring"] = ls
  return {k: v.astype(np.float32).astype(np.float64) for k, v in out.items()}


def _scenes():
  from tests import util

  per = ("body_mass", "jnt_stiffness", "qpos_spring")
  return {
    # name: (model, enable, disable, per-world fields)
    "humanoid": (util.HUMANOID, ENBL_ENERGY, 0, ("body_mass",)),
    "joints": (joints_xml(), ENBL_ENERGY, 0, per),
    "tendon": (TENDON, ENBL_ENERGY, 0, ("body_mass", "tendon_lengthspring")),
    "g1": (util.G1, ENBL_ENERGY, 0, ()),
    "sensors_off": (joints_xml(sensors=True), 0, 0, per),
    "sensors_on": (joints_xml(sensors=True), ENBL_ENERGY, 0, per),
    "sensors_nogravity": (joints_xml(sensors=True), ENBL_ENERGY, DSBL_GRAVITY, per),
    "sensors_nospring": (joints_xml(sensors=True), 0, DSBL_SPRING, per),
    "joints_rk4": (joints_xml("RK4"), ENBL_ENERGY, 0, per),
    "joints_implicitfast": (joints_xml("implicitfast"), ENBL_ENERGY, 0, per),
  }


SCENES = _scenes()


def seeded_state(mjm, nworld=NWORLD):
  """Per-world qpos / qvel, fp32-representable (world 0 moves as well)."""
  from tests import util

  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=0 if mjm.nkey else None, seed=2024, qpos_noise=0.2, qvel_noise=1.0, exact_world0=False)
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(qpos), f32(qvel)
