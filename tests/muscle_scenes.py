"""Scenes for muscle actuators (tests/test_muscle_host.py, tests/test_gpu_muscle.py, tools/make_muscle_goldens.py, tools/muscle_bench.py).

MUSCLES covers the muscle model's branches on one small model without collisions:
- muscles on a hinge, a slide and a limited fixed tendon, with lengthrange taken from the limits (a negative gear swaps the ends);
- force < 0 (peak force scale / acc0) and force > 0; tausmooth 0 and > 0;
- actearly, actlimited and ctrllimited on and off; an agonist / antagonist pair on one hinge;
- a <general> muscle with raw parameters and an explicit lengthrange, and a class default.
It runs once per integrator.  The humanoid scene puts an agonist / antagonist muscle pair in place of each of the humanoid's motors;
`humanoid_affine` is the same model with affine actuators and filter dynamics in place of the muscles (the benchmark's baseline).
Worlds start from seeded per-world qpos / qvel / act and take a seeded per-world ctrl in [-0.2, 1.2] each step.
"""
import numpy as np

NWORLD = 3

MUSCLES = """
<mujoco model="muscles">
  <option timestep="0.002" integrator="{integrator}"/>
  <default>
    <geom contype="0" conaffinity="0"/>
    <default class="slow"><muscle timeconst="0.02 0.08" force="35"/></default>
  </default>
  <worldbody>
    <body name="arm" pos="0 0 1">
      <joint name="elbow" type="hinge" axis="0 1 0" range="-70 85" limited="true" damping="0.05"/>
      <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03" mass="0.8"/>
      <body name="hand" pos="0.3 0 0">
        <joint name="wrist" type="hinge" axis="0 1 0" range="-45 45" limited="true" damping="0.02"/>
        <geom type="capsule" fromto="0 0 0 0.12 0 0" size="0.02" mass="0.3"/>
      </body>
    </body>
    <body name="sled" pos="0 0.5 1">
      <joint name="slide" type="slide" axis="1 0 0" range="-0.2 0.25" limited="true" damping="0.5"/>
      <geom type="box" size="0.05 0.05 0.05" mass="1.2"/>
    </body>
    <body name="free" pos="0 1 1">
      <joint name="loose" type="slide" axis="0 0 1" damping="0.3"/>
      <geom type="box" size="0.04 0.04 0.04" mass="0.6"/>
    </body>
  </worldbody>
  <tendon>
    <fixed name="coupled" range="-0.9 1.1" limited="true">
      <joint joint="elbow" coef="0.6"/>
      <joint joint="wrist" coef="0.4"/>
    </fixed>
  </tendon>
  <actuator>
    <muscle name="flexor" joint="elbow" gear="2"/>
    <muscle name="extensor" joint="elbow" gear="-2" tausmooth="0.3" actearly="true"/>
    <muscle name="sled" joint="slide" class="slow" ctrllimited="true" ctrlrange="0 1" actlimited="true" actrange="0 1"/>
    <muscle name="tendon" tendon="coupled" range="0.6 1.2" lmin="0.4" lmax="1.8" vmax="2" fpmax="1.5" fvmax="1.4" scale="150"/>
    <general name="raw" joint="loose" dyntype="muscle" gaintype="muscle" biastype="muscle" lengthrange="-0.1 0.3"
             dynprm="0.015 0.05 0.1" gainprm="0.8 1.1 20 100 0.5 1.6 1.5 1.3 1.2" biasprm="0.8 1.1 20 100 0.5 1.6 1.5 1.3 1.2" actearly="true"/>
    <motor name="motor" joint="wrist" gear="0.5"/>
  </actuator>
  <sensor>
    <actuatorfrc actuator="flexor"/>
    <actuatorfrc actuator="tendon"/>
    <jointactuatorfrc joint="elbow"/>
    <jointpos joint="elbow"/>
  </sensor>
</mujoco>"""


def muscles(integrator="Euler"):
  from mujoco_warp_b200._src import mjcf

  return mjcf.load_string(MUSCLES.format(integrator=integrator))


def _pairs(mjm, muscle):
  """The humanoid with two actuators per motor (gear +g and -g on the motor's joint): muscles, or affine actuators with filter dynamics
  of the same time constant.  acc0 is the motor's (it does not depend on the sign of the gear)."""
  from mujoco_warp_b200._src import constants as C

  nu0 = int(mjm.nu)
  rep = lambda a: np.repeat(np.asarray(a), 2, axis=0)
  nu = 2 * nu0
  sign = np.tile([1.0, -1.0], nu0)
  mjm.nu = nu
  mjm.na = nu
  mjm.actuator_trntype = rep(mjm.actuator_trntype)
  mjm.actuator_trnid = rep(mjm.actuator_trnid)
  mjm.actuator_gear = rep(mjm.actuator_gear) * sign[:, None]
  mjm.actuator_acc0 = rep(mjm.actuator_acc0)
  mjm.actuator_dyntype = np.full(nu, C.DYN_MUSCLE if muscle else C.DYN_FILTER, dtype=np.int32)
  mjm.actuator_gaintype = np.full(nu, C.GAIN_MUSCLE if muscle else C.GAIN_AFFINE, dtype=np.int32)
  mjm.actuator_biastype = np.full(nu, C.BIAS_MUSCLE if muscle else C.BIAS_AFFINE, dtype=np.int32)
  dyn = np.zeros((nu, 10))
  dyn[:, :2] = (0.01, 0.04)
  prm = np.zeros((nu, 10))
  if muscle:
    prm[:, :9] = (0.75, 1.05, -1.0, 200.0, 0.5, 1.6, 1.5, 1.3, 1.2)
    bias = prm.copy()
  else:
    dyn[:, 0] = 0.02
    prm[:, 0], prm[:, 1] = 1.0, -0.001
    bias = np.zeros((nu, 10))
    bias[:, 1], bias[:, 2] = -0.002, -0.0005
  mjm.actuator_dynprm, mjm.actuator_gainprm, mjm.actuator_biasprm = dyn, prm, bias
  mjm.actuator_ctrllimited = np.ones(nu, dtype=bool)
  mjm.actuator_ctrlrange = np.tile([0.0, 1.0], (nu, 1))
  mjm.actuator_forcelimited = np.zeros(nu, dtype=bool)
  mjm.actuator_forcerange = np.zeros((nu, 2))
  mjm.actuator_actlimited = np.zeros(nu, dtype=bool)
  mjm.actuator_actrange = np.zeros((nu, 2))
  mjm.actuator_actadr = np.arange(nu, dtype=np.int32)
  mjm.actuator_actnum = np.ones(nu, dtype=np.int32)
  mjm.actuator_actearly = np.zeros(nu, dtype=bool)
  rng = np.asarray(mjm.jnt_range)[np.asarray(mjm.actuator_trnid)[:, 0]]
  g = np.asarray(mjm.actuator_gear)[:, 0:1]
  mjm.actuator_lengthrange = np.where(g > 0, rng * g, rng[:, ::-1] * g)
  nkey = int(getattr(mjm, "nkey", 0))
  if nkey:  # keyframes: each motor's ctrl for both actuators of its pair, activations at rest
    mjm.key_ctrl = np.repeat(np.asarray(mjm.key_ctrl).reshape(nkey, nu0), 2, axis=1)
    mjm.key_act = np.zeros((nkey, nu))
  names = getattr(getattr(mjm, "names", None), "actuator", None)
  if names is not None:
    mjm.names.actuator = [f"{n}_{s}" for n in names for s in ("pos", "neg")]
  return mjm


def humanoid(muscle=True):
  from mujoco_warp_b200._src import mjcf
  from tests import util

  mjm = mjcf.load_any(util.HUMANOID)
  assert np.all(np.asarray(mjm.jnt_limited)[np.asarray(mjm.actuator_trnid)[:, 0]]), "every humanoid motor drives a limited joint"
  return _pairs(mjm, muscle)


# name: (model source, steps)
SCENES = {
  "euler": (lambda: muscles("Euler"), 12),
  "implicitfast": (lambda: muscles("implicitfast"), 10),
  "implicit": (lambda: muscles("implicit"), 10),
  "rk4": (lambda: muscles("RK4"), 8),
  "humanoid": (humanoid, 6),
}


def load(name):
  return SCENES[name][0]()


def seeded(mjm, nsteps, nworld=NWORLD, seed=5):
  """Per-world qpos / qvel / act and a per-world, per-step ctrl (nsteps, nworld, nu), fp32-representable."""
  from tests import util

  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=0 if getattr(mjm, "nkey", 0) else None, seed=seed, qpos_noise=0.1, qvel_noise=0.5, exact_world0=False)
  rng = np.random.default_rng(seed)
  act = rng.uniform(0.0, 1.0, (nworld, int(mjm.na)))
  ctrl = rng.uniform(-0.2, 1.2, (nsteps, nworld, int(mjm.nu)))
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(qpos), f32(qvel), f32(act), f32(ctrl)
