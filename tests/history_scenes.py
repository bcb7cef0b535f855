"""Scenes for actuator and sensor delays (tests/test_history_*.py, tests/test_gpu_history.py, tools/make_history_goldens.py).

Every scene runs at a timestep of 2^-9 s, so that d.time, the stamps in the buffers and every delay (a multiple of a quarter step) are
exact in fp32 and fp64 alike: a zero-order-hold read lands in the same bracket in the fp64 reference and on the GPU.  No geom collides in
the small scenes, so their steps are smooth.  Worlds start from seeded per-world qpos / qvel and take a seeded per-world ctrl each step.
"""
import numpy as np

NWORLD = 3
DT = 2.0**-9

# slide joints driven by actuators with zero-order-hold, linear and cubic delays, different nsample, a history-only actuator
# (delay 0) and an undelayed one; delayed scalar sensors of the three stages, a history-only sensor and a defaults class
ACTUATORS = """
<mujoco model="history_actuators">
  <option timestep="{dt}" integrator="{integrator}"/>
  <default>
    <geom contype="0" conaffinity="0"/>
    <default class="lagged"><motor nsample="4" interp="zoh" delay="{d25}"/></default>
  </default>
  <worldbody>
    <body name="a" pos="0 0 1"><joint name="a" type="slide" axis="1 0 0" damping="0.5"/><geom type="box" size="0.05 0.05 0.05" mass="1"/></body>
    <body name="b" pos="0 0.3 1"><joint name="b" type="slide" axis="1 0 0" damping="0.5"/><geom type="box" size="0.05 0.05 0.05" mass="1.5"/></body>
    <body name="c" pos="0 0.6 1"><joint name="c" type="hinge" axis="0 0 1" damping="0.1"/><geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.03" mass="0.7"/></body>
    <body name="e" pos="0 0.9 1"><joint name="e" type="slide" axis="1 0 0"/><geom type="box" size="0.05 0.05 0.05" mass="2"/></body>
    <body name="f" pos="0 1.2 1"><joint name="f" type="slide" axis="0 1 0"/><geom type="box" size="0.05 0.05 0.05" mass="1"/></body>
  </worldbody>
  <actuator>
    <motor name="zoh" joint="a" class="lagged"/>
    <motor name="linear" joint="b" nsample="3" interp="linear" delay="{d15}" ctrlrange="-1.5 1.5" ctrllimited="true"/>
    <motor name="cubic" joint="c" nsample="6" interp="cubic" delay="{d225}"/>
    <motor name="record" joint="e" nsample="2"/>
    <motor name="direct" joint="f"/>
  </actuator>
  <sensor>
    <jointpos name="qa" joint="a" nsample="3" interp="zoh" delay="{d15}"/>
    <jointvel name="vb" joint="b" nsample="4" interp="linear" delay="{d1}"/>
    <actuatorfrc name="fc" actuator="cubic" nsample="5" interp="cubic" delay="{d275}"/>
    <jointpos name="qe" joint="e" nsample="2"/>
    <jointpos name="qf" joint="f"/>
  </sensor>
</mujoco>"""

# filter and integrator activation dynamics fed a delayed ctrl
DYNAMICS = """
<mujoco model="history_dynamics">
  <option timestep="{dt}" integrator="{integrator}"/>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <body name="a" pos="0 0 1"><joint name="a" type="slide" axis="1 0 0"/><geom type="box" size="0.05 0.05 0.05" mass="1"/></body>
    <body name="b" pos="0 0.3 1"><joint name="b" type="slide" axis="1 0 0"/><geom type="box" size="0.05 0.05 0.05" mass="1"/></body>
  </worldbody>
  <actuator>
    <general name="filter" joint="a" dyntype="filter" dynprm="0.01" nsample="4" interp="linear" delay="{d15}"/>
    <general name="integrator" joint="b" dyntype="integrator" nsample="3" interp="zoh" delay="{d2}" actlimited="true" actrange="-0.2 0.2"/>
  </actuator>
  <sensor><actuatorfrc actuator="filter" nsample="3" delay="{d1}"/></sensor>
</mujoco>"""

# vector sensors (ballangvel, framequat) with delays, and an interval sensor whose phase init_sensor_history sets
VECTORS = """
<mujoco model="history_vectors">
  <option timestep="{dt}" integrator="{integrator}" gravity="0 0 -9.81"/>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <body name="p" pos="0 0 1">
      <joint name="ball" type="ball" damping="0.01"/>
      <geom type="capsule" fromto="0 0 0 0.3 0.1 -0.2" size="0.03" mass="1"/>
      <site name="tip" pos="0.3 0.1 -0.2"/>
    </body>
    <body name="h" pos="0.5 0 1"><joint name="h" type="hinge" axis="0 1 0"/><geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.03" mass="0.5"/></body>
  </worldbody>
  <actuator><motor joint="h" nsample="3" delay="{d1}" interp="linear"/></actuator>
  <sensor>
    <ballangvel name="w" joint="ball" nsample="4" interp="linear" delay="{d15}"/>
    <framequat name="q" objtype="site" objname="tip" nsample="5" interp="cubic" delay="{d225}"/>
    <framepos name="held" objtype="site" objname="tip" nsample="2" interval="{d3} {d1}"/>
    <framepos name="both" objtype="site" objname="tip" nsample="3" interp="linear" delay="{d1}" interval="{d2}"/>
  </sensor>
</mujoco>"""


def xml(template, integrator="Euler"):
  d = {f"d{k}": repr(float(v) * DT) for k, v in (("1", 1), ("15", 1.5), ("2", 2), ("225", 2.25), ("25", 2.5), ("275", 2.75), ("3", 3))}
  return template.format(dt=repr(DT), integrator=integrator, **d)


def humanoid():
  """The humanoid with every actuator delayed by two steps (4 samples, linear) and every sensor by one (3 samples, zero-order hold)."""
  from mujoco_warp_b200._src import mjcf
  from tests import util

  mjm = mjcf.load_any(util.HUMANOID)
  mjm.opt.timestep = DT
  delay_all(mjm, 2 * DT, 4, 1, 1 * DT, 3, 0)
  return mjm


def delay_all(mjm, act_delay, act_n, act_interp, sens_delay=0.0, sens_n=0, sens_interp=0):
  """Delays every actuator (and every sensor) of a compiled model in place and lays out its buffers."""
  from mujoco_warp_b200._src import mjcf

  nu, ns = int(mjm.nu), int(getattr(mjm, "nsensor", 0))
  mjm.actuator_history = np.tile(np.array([act_n, act_interp], dtype=np.int32), (nu, 1))
  mjm.actuator_delay = np.full(nu, float(act_delay))
  mjm.sensor_history = np.tile(np.array([sens_n, sens_interp], dtype=np.int32), (ns, 1))
  mjm.sensor_delay = np.full(ns, float(sens_delay))
  mjm.sensor_interval = np.zeros((ns, 2))
  if not hasattr(mjm, "sensor_dim"):
    mjm.sensor_dim = np.zeros(0, dtype=np.int32)
  mjcf.set_history_layout(mjm)


# name: (model source, steps).  Each scene steps more often than its largest nsample, so every ring wraps.
SCENES = {
  "actuators": (lambda: xml(ACTUATORS), 14),
  "actuators_rk4": (lambda: xml(ACTUATORS, "RK4"), 10),
  "actuators_implicitfast": (lambda: xml(ACTUATORS, "implicitfast"), 10),
  "dynamics": (lambda: xml(DYNAMICS), 12),
  "vectors": (lambda: xml(VECTORS), 14),
  "humanoid": (humanoid, 6),
}


def load(name):
  from mujoco_warp_b200._src import mjcf

  src = SCENES[name][0]()
  return mjcf.load_string(src) if isinstance(src, str) else src


def seeded(mjm, nsteps, nworld=NWORLD, seed=7):
  """Per-world qpos / qvel and a per-world, per-step ctrl (nsteps, nworld, nu), fp32-representable."""
  from tests import util

  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=0 if mjm.nkey else None, seed=seed, qpos_noise=0.1, qvel_noise=0.5, exact_world0=False)
  rng = np.random.default_rng(seed)
  ctrl = rng.uniform(-1.0, 1.0, (nsteps, nworld, int(mjm.nu)))
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(qpos), f32(qvel), f32(ctrl)


def interval_phase(nworld=NWORLD):
  """Per-world phase of the `held` interval sensor of VECTORS: the last time it was due, before and after t = 0."""
  return np.array([-DT, 0.0, DT])[np.arange(nworld) % 3]
