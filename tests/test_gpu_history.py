"""Actuator and sensor delays on the GPU (k_history.cu through step, forward, step1 / step2, inverse and the public history functions).

- The scenes of tests/history_scenes.py against the reference's own results (tests/golden/history_*.npz), step by step from the reference's
  state: d.history, the delayed actuator forces, the delayed / held sensors and the state after each step (Euler, implicitfast, RK4,
  filter and integrator dynamics, vector and interval sensors, the humanoid with per-world ctrl); forward, inverse, step1 + step2.
- read_ctrl / read_sensor / init_ctrl_history / init_sensor_history against the reference at off-grid times.
- Without a reference: a zero-order-hold delay of k steps is, bit for bit, an undelayed run fed the ctrl k steps late.
- get_state -> set_state reproduces the next steps bit for bit; 2048 worlds on two world halves equal one stream; the launch count.
"""
import os

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src.types import State
from tests import history_scenes as H

pytestmark = pytest.mark.gpu

STATE = ("time", "qpos", "qvel", "act", "qacc_warmstart", "ctrl", "history")
# fp32 against the fp64 reference after one step from the same state.  Buffers hold ctrl values and stamps exactly; sensor values and
# the state carry the fp32 chain of one step (the humanoid's contacts and solver: looser).
TOL = {"history": 2e-5, "actuator_force": 2e-5, "sensordata": 2e-4, "qpos": 2e-5, "qvel": 2e-4, "act": 2e-5, "time": 0.0}
HUMANOID_TOL = {"history": 2e-5, "actuator_force": 2e-5, "time": 0.0, "qpos": 2e-3}


def _golden(name):
  return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"history_{name}.npz"))


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).cuda()


def setup(scene, nworld=H.NWORLD):
  import mujoco_warp_b200 as mjw

  g, mjm = _golden(scene), H.load(scene)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, nconmax=int(g["in/nconmax"]), njmax=int(g["in/njmax"]), m=m)
  return mjw, g, mjm, m, d


def _load_state(d, g, prefix):
  for f in STATE:
    getattr(d, f).copy_(_t(g[prefix + f]).reshape(getattr(d, f).shape))


def _compare(d, g, prefix, tol, what):
  for f, t in tol.items():
    got, want = _np(getattr(d, f)).reshape(g[prefix + f].shape), g[prefix + f]
    scale = max(1.0, float(np.abs(want).max(initial=0)))
    assert np.abs(got - want).max(initial=0) <= t * scale, f"{what}: {f} off by {np.abs(got - want).max()}"


@pytest.mark.parametrize("scene", list(H.SCENES))
def test_gpu_history_steps_meet_the_reference(built, scene):
  mjw, g, mjm, m, d = setup(scene)
  tol = HUMANOID_TOL if scene == "humanoid" else TOL
  for k in range(H.SCENES[scene][1]):
    _load_state(d, g, f"step/{k}/in_")
    mjw.step(m, d)
    _compare(d, g, f"step/{k}/out_", tol, f"{scene} step {k}")


@pytest.mark.parametrize("scene", ["actuators", "dynamics", "vectors"])
def test_gpu_history_split_step_meets_the_reference(built, scene):
  """step1, then the ctrl, then step2: the sensor stage functions and fwd_actuation / euler carry the delays as step does."""
  mjw, g, mjm, m, d = setup(scene)
  for k in range(H.SCENES[scene][1]):
    _load_state(d, g, f"step/{k}/in_")
    ctrl = d.ctrl.clone()
    d.ctrl.zero_()
    mjw.step1(m, d)
    d.ctrl.copy_(ctrl)
    mjw.step2(m, d)
    _compare(d, g, f"step/{k}/out_", TOL, f"{scene} split step {k}")


@pytest.mark.parametrize("scene", ["actuators", "vectors", "dynamics"])
def test_gpu_history_forward_and_inverse_meet_the_reference(built, scene):
  """forward() replaces the sensors and records them but never inserts ctrl; inverse() does the same for its sensors."""
  mjw, g, mjm, m, d = setup(scene)
  _load_state(d, g, "step/0/in_")
  h0 = d.history.clone()
  mjw.forward(m, d)
  _compare(d, g, "forward/", {"history": TOL["history"], "sensordata": TOL["sensordata"], "actuator_force": TOL["actuator_force"]}, f"{scene} forward")
  d.history.copy_(h0)
  mjw.inverse(m, d)
  _compare(d, g, "inverse/", {"history": TOL["history"], "sensordata": TOL["sensordata"]}, f"{scene} inverse")


@pytest.mark.parametrize("scene", ["actuators", "vectors"])
def test_gpu_history_functions_meet_the_reference(built, scene):
  mjw, g, mjm, m, d = setup(scene)
  mjw.init_ctrl_history(m, d, 0, _t(g["init/ctrl_times"]), _t(g["init/ctrl_values"]))
  if "init/sensor_id" in g:
    mjw.init_sensor_history(m, d, int(g["init/sensor_id"]), None, _t(g["init/sensor_values"]), _t(g["init/sensor_phase"]))
  np.testing.assert_allclose(_np(d.history), g["init/history"], rtol=1e-6, atol=1e-7)
  last = H.SCENES[scene][1] - 1
  for f in ("history", "time", "ctrl", "sensordata"):
    getattr(d, f).copy_(_t(g[f"step/{last}/out_{f}"]).reshape(getattr(d, f).shape))
  tq = _t(g["fn/time"])
  for u in range(m.nu):
    for interp in (-1, 0, 1, 2):
      res = torch.full((d.nworld,), float("nan"), device="cuda")
      mjw.read_ctrl(m, d, u, tq, interp, res)
      np.testing.assert_allclose(_np(res), g[f"fn/read_ctrl/{u}/{interp}"], rtol=1e-5, atol=1e-6, err_msg=f"read_ctrl {u} {interp}")
  for s in range(m.nsensor):
    for interp in (-1, 0, 1, 2):
      res = torch.full((d.nworld, int(mjm.sensor_dim[s])), float("nan"), device="cuda")
      mjw.read_sensor(m, d, s, tq, interp, res)
      np.testing.assert_allclose(_np(res), g[f"fn/read_sensor/{s}/{interp}"], rtol=1e-5, atol=1e-6, err_msg=f"read_sensor {s} {interp}")
  mjw.init_ctrl_history(m, d, 0, _t(g["fn/init_ctrl_times"]), _t(g["fn/init_ctrl_values"]))
  mjw.init_sensor_history(m, d, 0, _t(g["fn/init_sensor_times"]), _t(g["fn/init_sensor_values"]), _t(g["fn/init_sensor_phase"]))
  np.testing.assert_allclose(_np(d.history), g["fn/init_history"], rtol=1e-6, atol=1e-7)


def test_gpu_history_function_refusals(built):
  mjw, g, mjm, m, d = setup("actuators")
  with pytest.raises(ValueError, match="strictly increasing"):
    mjw.init_ctrl_history(m, d, 0, _t([0.0, 0.0, 1.0, 2.0]), _t(np.zeros((d.nworld, 4))))
  with pytest.raises(ValueError, match="no history buffer"):
    mjw.init_ctrl_history(m, d, 4, None, _t(np.zeros((d.nworld, 1))))
  with pytest.raises(ValueError, match="out of range"):
    mjw.read_ctrl(m, d, 5, _t(np.zeros(d.nworld)), -1, _t(np.zeros(d.nworld)))


SHIFT = """
<mujoco>
  <option timestep="{dt}"/>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <body pos="0 0 1"><joint name="a" type="hinge" axis="0 1 0" damping="0.2"/><geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03" mass="1"/></body>
  </worldbody>
  <actuator><motor joint="a" {attrs}/></actuator>
  <sensor><jointpos joint="a"/></sensor>
</mujoco>"""


@pytest.mark.parametrize("k", [1, 3])
def test_gpu_zoh_delay_is_a_shifted_ctrl(built, k):
  """After init_ctrl_history with stamps -(n-1) dt .. 0 and zeros, a zero-order-hold delay of k steps reproduces, bit for bit, the
  undelayed model fed the same ctrl sequence k steps later with zeros first.  Needs no reference."""
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import mjcf

  n, nworld, nsteps = k + 2, 4, 100
  ctrl = np.random.default_rng(k).uniform(-1, 1, (nsteps, nworld)).astype(np.float32)
  shifted = np.concatenate([np.zeros((k, nworld), np.float32), ctrl[:-k]])
  runs = []
  for attrs, seq in ((f'nsample="{n}" interp="zoh" delay="{k * H.DT!r}"', ctrl), ("", shifted)):
    mjm = mjcf.load_string(SHIFT.format(dt=repr(H.DT), attrs=attrs))
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=nworld, m=m)
    if attrs:
      mjw.init_ctrl_history(m, d, 0, _t(-H.DT * np.arange(n - 1, -1, -1)), _t(np.zeros((nworld, n))))
    qs = []
    for j in range(nsteps):
      d.ctrl.copy_(_t(seq[j]).reshape(nworld, 1))
      mjw.step(m, d)
      qs.append(_np(d.qpos).copy())
    runs.append(np.array(qs))
  assert np.abs(runs[0]).max() > 1e-3
  np.testing.assert_array_equal(runs[0], runs[1])


def test_gpu_history_state_round_trip(built):
  """get_state -> steps -> set_state -> the same steps reproduces every output bit for bit (the buffers are part of the state)."""
  mjw, g, mjm, m, d = setup("vectors")
  _load_state(d, g, "step/0/in_")
  for _ in range(3):
    mjw.step(m, d)
  sig = int(State.TIME | State.QPOS | State.QVEL | State.ACT | State.HISTORY | State.WARMSTART | State.CTRL)
  width = 1 + m.nq + m.nv + m.na + m.nhistory + m.nv + m.nu
  st = torch.zeros((d.nworld, width), device="cuda")
  mjw.get_state(m, d, st, sig)
  assert torch.equal(st[:, 1 + m.nq + m.nv + m.na : 1 + m.nq + m.nv + m.na + m.nhistory], d.history)
  runs = []
  for _ in range(2):
    mjw.set_state(m, d, st, sig)
    out = []
    for _ in range(6):
      mjw.step(m, d)
      out.append(torch.cat([d.qpos, d.qvel, d.history, d.sensordata], dim=1).clone())
    runs.append(torch.stack(out))
  assert torch.equal(runs[0], runs[1])


def test_gpu_history_two_halves_equal_one_stream(built):
  """2048 humanoid worlds with every actuator delayed and per-world ctrl: the two world halves compute what one stream computes."""
  import mujoco_warp_b200 as mjw

  mjm = H.load("humanoid")
  nworld, nsteps = 2048, 6
  qpos, qvel, ctrl = H.seeded(mjm, nsteps, nworld)
  outs = []
  for split in ("2", "1"):
    os.environ["MJB_SPLIT"] = split
    try:
      m = mjw.put_model(mjm)
      d = mjw.make_data(mjm, nworld=nworld, nconmax=24, njmax=64, m=m)
    finally:
      os.environ.pop("MJB_SPLIT")
    d.qpos.copy_(_t(qpos))
    d.qvel.copy_(_t(qvel))
    for j in range(nsteps):
      d.ctrl.copy_(_t(ctrl[j]))
      mjw.step(m, d)
    outs.append([_np(x) for x in (d.qpos, d.qvel, d.history, d.actuator_force)])
  for a, b in zip(*outs):
    np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("scene, nworld, per_step", [("actuators", 8, 3), ("actuators_rk4", 8, 9), ("humanoid", 2048, 4)])
def test_gpu_history_launch_count(built, scene, nworld, per_step):
  """A history model launches, per forward pass and world half, one delayed-ctrl read and one sensor kernel (if it has delayed sensors),
  and one ctrl insert per step; the same model without delays launches the parent's kernels.  The count is the captured graph's."""
  from tests.test_gpu_launch_count import _captured_kernels

  import mujoco_warp_b200 as mjw

  counts = []
  for delayed in (True, False):
    mjm = H.load(scene)
    if not delayed:
      H.delay_all(mjm, 0.0, 0, 0)
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=nworld, m=m)
    mjw.step(m, d)
    kernels = _captured_kernels(lambda: mjw.step(m, d))
    assert mjw.last_launch_count() == kernels
    counts.append(kernels)
  assert counts[0] == counts[1] + per_step
