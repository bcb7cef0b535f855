"""Scenes of the make_constraint fixtures (tools/make_constraint_goldens.py) and of the GPU tests that use them.

  sparse   the tendon scene (arms, gripper, tendon friction, tendon limits, a two-tendon and a single-tendon equality) plus a connect, a weld
           and a limited ball joint, under jacobian="sparse": every row kind a sparse model can hold goes through the CSR view
  batched  the tendon scene with dof friction on a1, per-world dof_frictionloss / tendon_frictionloss (world 1 zeroes the nominally
           positive a1 and t_fric entries, world 2 makes the nominally zero f1 and t_spring entries positive) and per-world eq_data,
           jnt_range, jnt_margin, dof_solref and geom_friction
"""

import numpy as np

from tests import util

NWORLD = 3


def xml(name):
  x = util.tendon_xml()
  if name == "sparse":
    x = x.replace('<option timestep="0.004"', '<option jacobian="sparse" timestep="0.004"')
    x = x.replace('<body name="ball" pos="0.3 0.4 0.049"><freejoint/><geom type="sphere" size="0.05" mass="0.2"/></body>',
                  '<body name="ball" pos="0.3 0.4 0.049"><freejoint/><geom type="sphere" size="0.05" mass="0.2"/></body>'
                  '<body name="bb" pos="0.8 0 0.6"><freejoint/><geom type="box" size="0.03 0.03 0.03" mass="0.1"/></body>'
                  '<body name="pend" pos="-0.8 0 0.8"><joint name="bj" type="ball" limited="true" range="0 20"/>'
                  '<geom type="capsule" fromto="0 0 0 0 0 -0.2" size="0.02" mass="0.1"/></body>')
    x = x.replace("</equality>", '<connect body1="bb" body2="a2" anchor="0 0 0"/><weld body1="bb" body2="ball" torquescale="0.5"/></equality>')
    x = x.replace('active="false"', "")
    x = x[: x.index("<keyframe>")] + x[x.index("</keyframe>") + len("</keyframe>") :]
  else:
    x = x.replace('<joint name="a1" type="hinge" axis="0 1 0" damping="0.05"', '<joint name="a1" type="hinge" axis="0 1 0" damping="0.05" frictionloss="0.15"')
  return x


def load(name):
  from mujoco_warp_b200._src import mjcf

  return mjcf.load_string(xml(name))


def state(mjm, name):
  qpos, qvel, ctrl, warm = util.seeded_state(mjm, NWORLD, key=0 if name == "batched" else None, seed=99, qpos_noise=0.05, qvel_noise=0.5,
                                             ctrl_noise=0.5, exact_world0=False)
  qpos[:, 0] = (1.2, -1.6, 1.0)  # with a1 = -0.6: t_lim = (a0 - a1) / 2 past its upper end, past its lower end, past its upper end
  qpos[:, 1] = -0.6
  if name == "sparse":  # the limited ball joint (range 20 degrees) turned 30, 10 and 45 degrees about a tilted axis
    ang = np.radians([30.0, 10.0, 45.0])
    ax = np.array([0.6, 0.0, 0.8])
    qpos[:, -4:] = np.concatenate([np.cos(ang / 2)[:, None], np.sin(ang / 2)[:, None] * ax[None]], axis=1)
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(qpos), f32(qvel), f32(ctrl), f32(warm)


def batched(mjm):
  """{field: (NWORLD, ...) per-world values} of the batched scene."""
  out = {}
  fl = np.repeat(np.asarray(mjm.dof_frictionloss, dtype=np.float64)[None], NWORLD, 0)
  a1, f1 = int(mjm.jnt_dofadr[1]), int(mjm.jnt_dofadr[4])
  assert fl[0, a1] > 0 and fl[0, f1] == 0
  fl[1, a1] = 0.0
  fl[2, f1] = 0.25
  out["dof_frictionloss"] = fl
  tf = np.repeat(np.asarray(mjm.tendon_frictionloss, dtype=np.float64)[None], NWORLD, 0)
  assert tf[0, 2] > 0 and tf[0, 1] == 0  # t_fric, t_spring
  tf[1, 2] = 0.0
  tf[2, 1] = 0.3
  out["tendon_frictionloss"] = tf
  ed = np.repeat(np.asarray(mjm.eq_data, dtype=np.float64).reshape(1, mjm.neq, 11), NWORLD, 0)
  ed[:, 0, 0] = (0.0, 0.01, -0.02)
  ed[:, 0, 1] = (1.0, 0.8, 1.2)
  out["eq_data"] = ed
  rng = np.repeat(np.asarray(mjm.jnt_range, dtype=np.float64).reshape(1, mjm.njnt, 2), NWORLD, 0)
  rng[:, 4] = ((-0.03, 0.03), (-0.02, 0.025), (-0.035, 0.01))
  rng[:, 5] = ((-0.03, 0.03), (-0.01, 0.02), (-0.025, 0.03))
  out["jnt_range"] = rng
  mg = np.repeat(np.asarray(mjm.jnt_margin, dtype=np.float64)[None], NWORLD, 0)
  mg[:, 4] = (0.0, 0.004, 0.002)
  out["jnt_margin"] = mg
  sr = np.repeat(np.asarray(mjm.dof_solref, dtype=np.float64).reshape(1, mjm.nv, 2), NWORLD, 0)
  sr[1] = (0.05, 0.9)
  sr[2] = (-500.0, -20.0)
  out["dof_solref"] = sr
  gf = np.repeat(np.asarray(mjm.geom_friction, dtype=np.float64).reshape(1, mjm.ngeom, 3), NWORLD, 0)
  gf[:, :, 0] *= np.asarray([1.0, 0.6, 1.4])[:, None]
  out["geom_friction"] = gf
  return {k: np.asarray(v, dtype=np.float32).astype(np.float64) for k, v in out.items()}
