"""<contact> sensors on the GPU (k_sensor_contact).

- Teacher-forced: after forward / step, the GPU's own contact pool and efc_force go through the fp64 restatement of
  tests/contact_sensor_oracle.py; found matches exactly, the rest to 1e-5 relative / 1e-6 absolute (per slot, up to the order of
  matches whose sort criteria tie in fp32).  Every fixture scene, the site volumes, an overflowing capacity with netforce and num past
  it, per-world Model fields, and 8192 worlds of the humanoid with foot sensors.
- The reference's own sensordata (tests/golden/contact_sensor_*.npz) for each world whose contact count matches the fixture's.
- OVF_CONTACT_MATCH exactly when the matches exceed the capacity; override_model of opt.contact_sensor_maxmatch; bit-identical reruns.
- step, step1 + step2, RK4, sensor_acc and inverse all write the slots; DSBL_SENSOR leaves them alone.
- One more launch than the same model without contact sensors; the benchmark humanoid's count is unchanged.
"""
import glob
import os

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf
from tests import contact_sensor_oracle as O
from tests import contact_sensor_scenes as S
from tests import util
from tests.test_gpu_launch_count import _captured_kernels

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
OVF = 1 << 6
RTOL, ATOL = 1e-5, 1e-6


def _np(t):
  return t.detach().cpu().numpy()


def _setup(mjm, nworld, njmax=256, seed=3, batch_sizes=None, qpos_noise=0.01):
  import mujoco_warp_b200 as mjw

  m = mjw.put_model(mjm, batch_sizes=batch_sizes) if batch_sizes else mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m, nconmax=16, njmax=njmax)
  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=None, seed=seed, qpos_noise=qpos_noise, qvel_noise=0.3, exact_world0=False)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  return mjw, m, d


def _contacts(d):
  n = int(_np(d.nacon)[0])
  return {k: _np(getattr(d.contact, k))[:n].astype(np.float64 if getattr(d.contact, k).is_floating_point() else np.int64)
          for k in ("dist", "pos", "frame", "friction", "dim", "geom", "efc_address", "worldid", "type")}


def _history(mjm):
  h = getattr(mjm, "sensor_history", None)
  return np.zeros(mjm.nsensor, dtype=int) if h is None else np.asarray(h)[:, 0]


def teacher_forced(mjm, m, d, worlds=None):
  """the restatement fed the GPU's contacts and efc_force, world by world, against d.sensordata and the overflow bit"""
  torch.cuda.synchronize()
  con, force, sd, ovf = _contacts(d), _np(d.efc.force).astype(np.float64), _np(d.sensordata).astype(np.float64), _np(d.overflow)
  sxp, sxm = _np(d.site_xpos).astype(np.float64), _np(d.site_xmat).astype(np.float64).reshape(d.nworld, -1, 9)
  hist = _history(mjm)
  nslot = 0
  for w in worlds if worlds is not None else range(d.nworld):
    res, o = O.world_sensors(mjm, O.world_contacts(con, w), force[w], d.njmax, int(m.opt.contact_sensor_maxmatch), sxp[w], sxm[w])
    assert bool(ovf[w] & OVF) == o, w
    for s, r in res.items():
      if hist[s] > 0:
        continue
      got = sd[w, mjm.sensor_adr[s] : mjm.sensor_adr[s] + mjm.sensor_dim[s]]
      if mjm.sensor_intprm[s][0] & 1 and (r["reduce"] == 3 or r["matches"]):
        assert got[0] == r["nmatch"], (w, mjm.names.sensor[s])  # found is the exact count
      O.check_sensor(got, r, RTOL, ATOL, what=f"world {w} sensor {mjm.names.sensor[s]}")
      nslot += min(len(r["matches"]), r["num"])
  return nslot


SCENE_IDS = list(S.SCENES)


@pytest.mark.parametrize("scene", SCENE_IDS)
def test_teacher_forced_scenes(built, scene):
  xml, njmax = S.SCENES[scene]
  mjm = mjcf.load_string(xml)
  mjw, m, d = _setup(mjm, 64, njmax=njmax)
  mjw.forward(m, d)
  assert teacher_forced(mjm, m, d) > 0
  for _ in range(3):
    d.overflow.zero_()  # the bits accumulate over calls; the check wants this step's
    mjw.step(m, d)
    teacher_forced(mjm, m, d)


def test_teacher_forced_overflow_with_netforce_and_num_past_capacity(built):
  mjm = mjcf.load_string(S.overflow_xml(maxmatch=3, netforce=True))
  mjw, m, d = _setup(mjm, 64)
  mjw.forward(m, d)
  teacher_forced(mjm, m, d)
  ovf = _np(d.overflow) & OVF
  assert ovf.any() and not ovf.all()  # some worlds have more than 3 contacts, some not
  # decision 3: netforce sums the 3 stored matches; slots past them are zero even where more matched (num 6 > maxmatch)
  sd = _np(d.sensordata)
  s = mjm.names.sensor.index("all_none_6")
  size = mjcf.contact_slot_size(int(mjm.sensor_intprm[s][0]))
  assert np.all(sd[ovf > 0, mjm.sensor_adr[s] + 3 * size : mjm.sensor_adr[s] + 6 * size] == 0)


def test_teacher_forced_batched_model_fields(built):
  mjm = mjcf.load_string(S.SCENES["pyramidal"][0])
  nworld = 32
  mjw, m, d = _setup(mjm, nworld, batch_sizes={"geom_friction": nworld, "geom_size": nworld})
  rng = np.random.default_rng(5)
  fr = m.geom_friction.clone()
  fr[:, :, 0] = torch.from_numpy(rng.uniform(0.2, 1.5, (nworld, mjm.ngeom)).astype(np.float32)).cuda()
  m.geom_friction.copy_(fr)
  size = m.geom_size.clone()
  size[:, 2, 0] *= torch.from_numpy(rng.uniform(0.9, 1.1, nworld).astype(np.float32)).cuda()  # the ball's radius
  m.geom_size.copy_(size)
  mjw.forward(m, d)
  mjw.step(m, d)
  d.overflow.zero_()
  mjw.step(m, d)
  teacher_forced(mjm, m, d)


def test_teacher_forced_humanoid_8192_worlds(built):
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200.scenes import WORKLOADS

  mjm = S.humanoid()
  wl = WORKLOADS["humanoid"]
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=8192, m=m, nconmax=wl["nconmax"], njmax=wl["njmax"])
  qpos, qvel, _, _ = util.seeded_state(mjm, 8192, key=0, seed=11, qpos_noise=0.02, qvel_noise=0.3)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  for _ in range(20):
    mjw.step(m, d)
  d.overflow.zero_()
  mjw.forward(m, d)
  found = _np(d.sensordata)[:, mjm.sensor_adr]
  assert (found > 0).mean() > 0.5  # most worlds stand on at least one foot
  assert teacher_forced(mjm, m, d) > 0


GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "contact_sensor_*.npz")))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[15:-4] for p in GOLDEN])
def test_reference_fixtures(built, path):
  """forward from the fixture's state; worlds with the fixture's contact count are compared with the reference's sensordata (slots
  order-free for reduce none, whose pool order may differ; tie groups for the sorted ones).  Contacts and forces are fp32 here."""
  name = os.path.basename(path)[len("contact_sensor_"):-4]
  z = np.load(path)
  xml, njmax = S.SCENES[name]
  mjm = mjcf.load_string(xml)
  nworld = z["in/qpos"].shape[0]
  mjw, m, d = _setup(mjm, nworld, njmax=njmax)
  d.qpos.copy_(torch.from_numpy(z["in/qpos"].astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(z["in/qvel"].astype(np.float32)))
  d.qacc_warmstart.copy_(torch.from_numpy(z["in/qacc_warmstart"].astype(np.float32)))
  mjw.forward(m, d)
  torch.cuda.synchronize()
  con = _contacts(d)
  gcon = {k: z[f"forward/con_{k}"] for k in ("dist", "pos", "frame", "friction", "dim", "geom", "efc_address", "worldid", "type")}
  sd = _np(d.sensordata).astype(np.float64)
  hist = _history(mjm)
  compared = 0
  for w in range(nworld):
    gw = O.world_contacts(gcon, w)
    if len(gw["dist"]) != int((con["worldid"] == w).sum()):
      continue
    res, ovf = O.world_sensors(mjm, gw, z["forward/efc_force"][w], njmax, int(z["maxmatch"]), z["forward/site_xpos"][w], z["forward/site_xmat"][w].reshape(-1, 9))
    assert bool(_np(d.overflow)[w] & OVF) == ovf
    for s, r in res.items():
      got = sd[w, mjm.sensor_adr[s] : mjm.sensor_adr[s] + mjm.sensor_dim[s]]
      want = z["forward/sensordata"][w, mjm.sensor_adr[s] : mjm.sensor_adr[s] + mjm.sensor_dim[s]]
      scale = 1.0 + np.abs(want).max()
      if hist[s] > 0:
        np.testing.assert_allclose(got, want, rtol=2e-3, atol=2e-3 * scale)
        continue
      # the restatement meets the reference's own data (tests/test_contact_sensor_host.py); its slots give the tie groups here
      O.check_sensor(got, r, rtol=2e-3, atol=2e-3 * scale, order_free=r["reduce"] == 0, what=f"world {w} sensor {mjm.names.sensor[s]}")
      compared += 1
  assert compared > 0


def test_override_maxmatch_takes_effect(built):
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(S.overflow_xml(maxmatch=3, netforce=True))
  _, m, d = _setup(mjm, 64)
  assert m.opt.contact_sensor_maxmatch == 3
  mjw.forward(m, d)
  torch.cuda.synchronize()
  assert (_np(d.overflow) & OVF).any()
  mjw.override_model(m, {"opt.contact_sensor_maxmatch": 64})
  assert m.opt.contact_sensor_maxmatch == 64
  d.overflow.zero_()
  mjw.forward(m, d)
  assert not (_np(d.overflow) & OVF).any()
  teacher_forced(mjm, m, d)
  with pytest.raises(ValueError, match="contact_sensor_maxmatch"):
    mjw.override_model(m, {"opt.contact_sensor_maxmatch": 0})


def test_two_runs_are_bit_identical(built):
  for xml in (S.SCENES["pyramidal"][0], S.overflow_xml(maxmatch=3, netforce=True)):
    mjm = mjcf.load_string(xml)
    out = []
    for _ in range(2):
      mjw, m, d = _setup(mjm, 256)
      for _ in range(5):
        mjw.step(m, d)
      torch.cuda.synchronize()
      out.append(_np(d.sensordata).copy())
    assert np.array_equal(out[0], out[1])


def _fresh(mjm, **kw):
  mjw, m, d = _setup(mjm, 16, **kw)
  d.sensordata.fill_(-7.0)
  return mjw, m, d


def _contact_slots(mjm, d):
  torch.cuda.synchronize()
  sd = _np(d.sensordata)
  cols = np.concatenate([np.arange(a, a + n) for a, n, t in zip(mjm.sensor_adr, mjm.sensor_dim, mjm.sensor_type) if t == C.SENS_CONTACT])
  return sd[:, cols]


@pytest.mark.parametrize("entry", ["step", "step1_step2", "rk4", "sensor_acc", "inverse"])
def test_every_entry_point_fills_the_slots(built, entry):
  xml = S.SCENES["pyramidal"][0]
  if entry == "rk4":
    xml = xml.replace('<option timestep="0.004"', '<option timestep="0.004" integrator="RK4"')
  mjm = mjcf.load_string(xml)
  mjw, m, d = _fresh(mjm)
  if entry in ("step", "rk4"):
    mjw.step(m, d)
  elif entry == "step1_step2":
    mjw.step1(m, d)
    d.sensordata.fill_(-7.0)  # step2 runs the acceleration stage, where the contact sensors are
    mjw.step2(m, d)
  elif entry == "sensor_acc":
    mjw.forward(m, d)
    d.sensordata.fill_(-7.0)
    mjw.sensor_acc(m, d)
  else:
    mjw.forward(m, d)
    d.sensordata.fill_(-7.0)
    mjw.inverse(m, d)
  assert not (_contact_slots(mjm, d) == -7.0).any()
  if entry in ("sensor_acc", "inverse"):
    teacher_forced(mjm, m, d)


def test_dsbl_sensor_leaves_the_slots(built):
  mjm = mjcf.load_string(S.SCENES["pyramidal"][0])
  mjm.opt.disableflags |= C.DSBL_SENSOR
  mjw, m, d = _fresh(mjm)
  mjw.step(m, d)
  assert (_contact_slots(mjm, d) == -7.0).all()


def test_launch_counts(built):
  import mujoco_warp_b200 as mjw
  from tests.test_oracle_golden_pipeline import load_scene

  counts = {}
  for name, mjm in (("plain", load_scene("humanoid")), ("feet", S.humanoid())):
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=8, m=m)
    mjw.step(m, d)
    n = _captured_kernels(lambda: mjw.step(m, d))
    mjw.step(m, d)
    assert mjw.last_launch_count() == n
    counts[name] = n
  assert counts["plain"] == 6
  # k_sensor runs for any model with sensors, k_sensor_contact once more for its contact sensors
  assert counts["feet"] == counts["plain"] + 2
  mjm = S.humanoid()
  mjm.opt.disableflags |= C.DSBL_SENSOR
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=8, m=m)
  mjw.step(m, d)
  assert mjw.last_launch_count() == counts["plain"] + 1
