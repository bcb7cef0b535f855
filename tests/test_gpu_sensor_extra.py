"""The magnetometer, camprojection, insidesite, tendon limit and tendonactfrc sensors on the GPU (k_sensor's EXTRA build).

- The scenes of tests/sensor_extra_scenes.py against the reference's own sensordata (tests/golden/sensor_extra_*.npz): forward from the
  seeded state and every step from the reference's state (Euler, implicitfast, RK4, per-world opt.magnetic / cam_fovy / cam_intrinsic,
  each sensor alone).  insidesite must match exactly (the scenes keep every point away from the site surfaces).
- sensor_pos / sensor_vel / sensor_acc called alone fill their stage's slots as forward does; DSBL_SENSOR leaves every slot untouched.
- tendonactfrc (an ordered sum) and every other slot are bit-identical run to run; opt.magnetic follows assignment and override_model.
- A model with the new sensors launches as many kernels per step as the same model without them.
"""
import os

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from tests import sensor_extra_scenes as S

pytestmark = pytest.mark.gpu

STATE = ("time", "qpos", "qvel", "qacc_warmstart", "ctrl", "history")
# fp32 against the fp64 reference after forward or one step from the same state: the tolerance of the muscle and contact-sensor replays,
# relative to the largest value of each sensor (camprojection reads hundreds of pixels)
TOL = 2e-4


def _golden(name):
  return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"sensor_extra_{name}.npz"))


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).cuda()


def setup(scene):
  import mujoco_warp_b200 as mjw

  g, mjm = _golden(scene), S.load(scene)
  m = mjw.put_model(mjm)
  if S.SCENES[scene][2]:
    m.opt.magnetic, m.cam_fovy, m.cam_intrinsic = _t(g["in/magnetic"]), _t(g["in/cam_fovy"]), _t(g["in/cam_intrinsic"])
  d = mjw.make_data(mjm, nworld=S.NWORLD, nconmax=int(g["in/nconmax"]), njmax=int(g["in/njmax"]), m=m)
  return mjw, g, mjm, m, d


def _load_state(d, g, prefix):
  for f in STATE:
    getattr(d, f).copy_(_t(g[prefix + f]).reshape(getattr(d, f).shape))


def _compare(mjm, got, want, what):
  for s in range(mjm.nsensor):
    a, n = int(mjm.sensor_adr[s]), int(mjm.sensor_dim[s])
    x, y = got[:, a : a + n], want[:, a : a + n]
    if int(mjm.sensor_type[s]) == C.SENS_INSIDESITE:
      np.testing.assert_array_equal(x, y, err_msg=f"{what}: insidesite sensor {s}")
    else:
      err = np.abs(x - y).max()
      assert err <= TOL * max(1.0, float(np.abs(y).max())), f"{what}: sensor {s} (type {int(mjm.sensor_type[s])}) off by {err}"


@pytest.mark.parametrize("scene", list(S.SCENES))
def test_gpu_sensor_extra_forward_and_steps_meet_the_reference(built, scene):
  mjw, g, mjm, m, d = setup(scene)
  _load_state(d, g, "start/")
  mjw.forward(m, d)
  _compare(mjm, _np(d.sensordata), g["forward/sensordata"], f"{scene} forward")
  for k in range(S.SCENES[scene][1]):
    _load_state(d, g, f"step/{k}/in_")
    mjw.step(m, d)
    _compare(mjm, _np(d.sensordata), g[f"step/{k}/out_sensordata"], f"{scene} step {k}")


@pytest.mark.parametrize("scene", ["all_euler", "batched"])
def test_gpu_sensor_extra_stage_calls_fill_their_slots(built, scene):
  """sensor_pos / sensor_vel / sensor_acc after forward's stages write exactly what forward wrote into their stage's slots (undelayed
  sensors; a delayed slot reads the history, which these calls advance) and leave the other slots alone."""
  mjw, g, mjm, m, d = setup(scene)
  _load_state(d, g, "start/")
  mjw.forward(m, d)
  ref = d.sensordata.clone()
  stage = np.asarray(mjm.sensor_needstage)
  undelayed = np.asarray(mjm.sensor_history)[:, 0] == 0
  for st, call in ((1, mjw.sensor_pos), (2, mjw.sensor_vel), (3, mjw.sensor_acc)):
    _load_state(d, g, "start/")
    d.sensordata.fill_(-7.0)
    call(m, d)
    got = d.sensordata.clone()
    for s in range(mjm.nsensor):
      a, n = int(mjm.sensor_adr[s]), int(mjm.sensor_dim[s])
      if stage[s] == st and undelayed[s]:
        assert torch.equal(got[:, a : a + n], ref[:, a : a + n]), f"{scene}: stage {st} call, sensor {s}"
      elif stage[s] != st:
        assert bool((got[:, a : a + n] == -7.0).all()), f"{scene}: stage {st} call wrote sensor {s} of stage {stage[s]}"


def test_gpu_sensor_extra_disabled_leaves_slots(built):
  mjw, g, mjm, m, d = setup("all_euler")
  m.opt.disableflags = int(m.opt.disableflags) | C.DSBL_SENSOR
  _load_state(d, g, "start/")
  d.sensordata.fill_(3.5)
  mjw.forward(m, d)
  mjw.step(m, d)
  assert bool((d.sensordata == 3.5).all())


def test_gpu_sensor_extra_bit_identical_reruns(built):
  mjw, g, mjm, m, d = setup("all_euler")
  runs = []
  for _ in range(2):
    _load_state(d, g, "step/0/in_")
    for _ in range(3):
      mjw.step(m, d)
    runs.append(d.sensordata.clone())
  assert torch.equal(runs[0], runs[1])
  frc = [s for s in range(mjm.nsensor) if int(mjm.sensor_type[s]) == C.SENS_TENDONACTFRC]
  assert frc and bool((runs[0][:, [int(mjm.sensor_adr[s]) for s in frc]] != 0).any())


def test_gpu_magnetic_follows_assignment_and_override(built):
  import mujoco_warp_b200 as mjw

  mjm = S.load("alone_magnetometer")
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=4, m=m)
  mjw.forward(m, d)
  R = _np(d.site_xmat)[:, list(mjm.names.site).index("tip")]
  want = lambda mag: np.einsum("wji,wj->wi", R, np.broadcast_to(mag, (4, 3)))
  np.testing.assert_allclose(_np(d.sensordata), want(np.asarray(mjm.opt.magnetic)), atol=1e-6)
  mjw.override_model(m, ["opt.magnetic = 0.5 0 -1"])
  mjw.forward(m, d)
  np.testing.assert_allclose(_np(d.sensordata), want(np.array([0.5, 0.0, -1.0])), atol=1e-6)
  per_world = np.array([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0], [1.0, 1.0, 1.0]])
  m.opt.magnetic = _t(per_world)
  mjw.forward(m, d)
  np.testing.assert_allclose(_np(d.sensordata), want(per_world), atol=1e-6)


def test_gpu_sensor_extra_launch_count(built):
  """The EXTRA build replaces k_sensor; it adds no launch.  (The scene's delayed sensors are left out: their history buffers add the
  history kernel's launch, as for any delayed sensor.)"""
  import mujoco_warp_b200 as mjw

  counts = []
  undelayed = ([x for x in S.ALL_SENSORS if "nsample" not in x], tuple(g for g in S.MAGNETOMETERS if g[2] == 0))
  for sensors, mags in ((['<jointpos joint="j1"/>'], ()), undelayed):
    mjm = S._load("Euler", sensors, mags)
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=8, m=m)
    mjw.step(m, d)
    counts.append(mjw.last_launch_count())
  assert counts[0] == counts[1]
