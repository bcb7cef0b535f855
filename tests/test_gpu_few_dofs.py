"""GPU parity for a model with more bodies than dofs: a cart-pole with welded links (nbody 8, nv 2).

k_velocity's shared-memory layout lets cfrc_int reuse cdof_dot's slot (6 nv words); with 6 nbody > 6 nv that slot has to be sized
for cfrc_int, or cfrc_int runs into cacc.  Every smooth field, cacc and cfrc_int included, is compared with the oracle after the
fused forward() and after the stages called one by one."""
import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu

CARTPOLE_XML = """
<mujoco model="cartpole_links">
  <option timestep="0.01"/>
  <worldbody>
    <body name="rail" pos="0 0 1">
      <geom type="box" size="2 0.02 0.02" contype="0" conaffinity="0" mass="1"/>
    </body>
    <body name="cart" pos="0 0 1">
      <joint name="slider" type="slide" axis="1 0 0" damping="0.1"/>
      <geom type="box" size="0.2 0.1 0.05" mass="1" contype="0" conaffinity="0"/>
      <body name="lamp" pos="0 0 0.1">
        <geom type="sphere" size="0.03" mass="0.05" contype="0" conaffinity="0"/>
      </body>
      <body name="pole" pos="0 0 0">
        <joint name="hinge" type="hinge" axis="0 1 0" damping="0.01"/>
        <geom type="capsule" fromto="0 0 0 0 0 0.6" size="0.04" mass="0.3" contype="0" conaffinity="0"/>
        <body name="mid" pos="0.05 0 0.3">
          <geom type="box" size="0.02 0.02 0.02" mass="0.05" contype="0" conaffinity="0"/>
        </body>
        <body name="tip" pos="0 0 0.6" quat="0.92388 0 0.38268 0">
          <geom type="sphere" size="0.06" mass="0.2" contype="0" conaffinity="0"/>
          <body name="tag" pos="0.05 0 0">
            <geom type="sphere" size="0.02" mass="0.02" contype="0" conaffinity="0"/>
          </body>
        </body>
      </body>
    </body>
  </worldbody>
  <actuator>
    <motor joint="slider" gear="10" ctrlrange="-1 1" ctrllimited="true"/>
  </actuator>
</mujoco>
"""

NWORLD, NCONMAX, NJMAX = 64, 4, 8


def _setup(mjw, mjm, m, seed):
  d = mjw.make_data(mjm, nworld=NWORLD, nconmax=NCONMAX, njmax=NJMAX, m=m)
  o = util.make_oracle(mjm, NWORLD, NCONMAX, NJMAX)
  qpos, qvel, ctrl, warm = util.seeded_state(mjm, NWORLD, seed=seed)
  f32 = lambda a: a.astype(np.float32)
  for name, val in (("qpos", qpos), ("qvel", qvel), ("ctrl", ctrl), ("qacc_warmstart", warm)):
    getattr(d, name).copy_(torch.from_numpy(f32(val)))
  o.set_state(qpos=f32(qpos), qvel=f32(qvel), ctrl=f32(ctrl), qacc_warmstart=f32(warm))
  return d, o


@pytest.mark.parametrize("stagewise", [False, True], ids=["forward", "stages"])
def test_more_bodies_than_dofs_matches_oracle(built, stagewise):
  import mujoco_warp_b200 as mjw

  mjm = mjw.mjcf.load_string(CARTPOLE_XML)
  assert mjm.nbody > mjm.nv and 6 * mjm.nbody > ((6 * mjm.nv + 3) & ~3)
  m = mjw.put_model(mjm)
  d, o = _setup(mjw, mjm, m, seed=11)
  if stagewise:
    for fn in (mjw.kinematics, mjw.com_pos, mjw.camlight, mjw.crb, mjw.collision, mjw.make_constraint, mjw.transmission,
               mjw.fwd_velocity, mjw.rne, mjw.fwd_actuation, mjw.fwd_acceleration, mjw.solve):
      fn(m, d)
  else:
    mjw.forward(m, d)
  o.forward()
  torch.cuda.synchronize()
  for name in util.SMOOTH_FIELDS:
    got = getattr(d, name).cpu().numpy()
    util.assert_close(name, got.reshape(o.d[name].shape), o.d[name], atol=5e-4, rtol=5e-4)
  util.assert_close("qacc", d.qacc.cpu().numpy(), o.d["qacc"], atol=5e-3, rtol=5e-3)
