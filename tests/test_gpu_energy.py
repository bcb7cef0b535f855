"""Potential and kinetic energy on the GPU (k_energy.cu through mjw.energy_pos / energy_vel, forward, step, step1, inverse, sensor_pos).

- The scenes of tests/energy_scenes.py against the reference's own results (tests/golden/energy_*.npz): forward, energy_pos / energy_vel
  and one step, per world, with per-world body_mass / jnt_stiffness / qpos_spring / tendon_lengthspring.
- Which call writes what (flag on / off, energy sensors present or not, DSBL_SENSOR), the launch count, run-time toggling of the flag,
  CUDA-graph replay, bit-reproducibility, 2048 worlds on two world halves.
- Independent invariants: kinetic energy against the bodies' 1/2 cvel' I cvel, and drift of the total energy under RK4.
"""
import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from tests import energy_oracle, energy_scenes, util
from tests.test_energy_vectors import energy_sensors, load

pytestmark = pytest.mark.gpu

# fp32 against the fp64 reference, as a fraction of sum |term| (each body's gravity term, each spring term, each product
# qvel_i M_ij qvel_j / 2): every term carries a few ulps of relative error from the fp32 chain that produced its inputs (kinematics down
# the tree for xipos and ten_length, crb for M), and the sum adds one ulp per term.  The largest gap reference_gaps() observed on an H100
# is 1.8e-7 (sensors_nogravity; humanoid 1.4e-7, G1 7.7e-8), so FWD_TOL is about 5x that.  After an RK4 step d.energy is the last
# stage's, whose state comes from three fp32 solves: 6.2e-5 observed (joints_rk4), so STEP_TOL is about 5x that.
FWD_TOL = 1e-6
STEP_TOL = 3e-4
SENTINEL = 12345.0


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def setup(scene, nworld=energy_scenes.NWORLD, mjm=None):
  import mujoco_warp_b200 as mjw

  g, mjm_, inputs = load(scene)
  mjm = mjm or mjm_
  m = mjw.put_model(mjm, batch_sizes={f: nworld for f in inputs})
  for f, v in inputs.items():
    getattr(m, f).copy_(torch.from_numpy(np.asarray(v, dtype=np.float32)).reshape(getattr(m, f).shape))
  d = mjw.make_data(mjm, nworld=nworld, nconmax=int(g["in/nconmax"]), njmax=int(g["in/njmax"]), m=m)
  d.qpos.copy_(torch.from_numpy(g["in/qpos"].astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(g["in/qvel"].astype(np.float32)))
  return mjw, g, mjm, inputs, m, d


def scales(mjm, inputs, g, w):
  """sum |term| of world w's potential and kinetic energy"""
  grav, spring = energy_oracle.potential_terms(mjm, inputs, w, g["in/qpos"][w], g["forward/xipos"][w], g["forward/ten_length"][w])
  return float(np.abs(grav).sum() + np.abs(spring).sum()) + 1e-6, float(np.abs(energy_oracle.kinetic_terms(mjm, g["in/qvel"][w], g["forward/M"][w])).sum()) + 1e-6


def reference_gaps(scene):
  """{stage: max over worlds and terms of |GPU - reference| / sum |term|} for forward, energy_pos / energy_vel, step and the sensors."""
  mjw, g, mjm, inputs, m, d = setup(scene)
  sensors = energy_sensors(mjm)
  gaps = {}

  def gap(key, got, want, sens_got=None, sens_want=None):
    e = 0.0
    for w in range(energy_scenes.NWORLD):
      sp, sk = scales(mjm, inputs, g, w)
      e = max(e, abs(got[w, 0] - want[w, 0]) / sp, abs(got[w, 1] - want[w, 1]) / sk)
      for slot, typ, _ in sensors if sens_got is not None else ():
        e = max(e, abs(sens_got[w, slot] - sens_want[w, slot]) / (sp if typ == C.SENS_E_POTENTIAL else sk))
    gaps[key] = e

  d.energy.fill_(SENTINEL)
  mjw.forward(m, d)
  gap("forward", _np(d.energy), g["forward/energy"], _np(d.sensordata), g["forward/sensordata"])
  d.energy.fill_(float("nan"))
  mjw.energy_pos(m, d)
  mjw.energy_vel(m, d)
  gap("direct", _np(d.energy), g["direct/energy"])
  mjw.step(m, d)
  gap("step", _np(d.energy), g["step/energy"], _np(d.sensordata), g["step/sensordata"])
  return gaps


@pytest.mark.parametrize("scene", sorted(energy_scenes.SCENES))
def test_gpu_energy_meets_the_reference(built, scene):
  gaps = reference_gaps(scene)
  step_tol = STEP_TOL if load(scene)[1].opt.integrator == C.INT_RK4 else FWD_TOL
  for key, e in gaps.items():
    assert e <= (step_tol if key == "step" else FWD_TOL), f"{scene}/{key}: {e:.3g} of sum |term|"


def test_gpu_energy_functions_with_the_flag_off(built):
  """energy_pos / energy_vel compute their own component whatever the flag says, and nothing else."""
  mjw, g, mjm, inputs, m, d = setup("sensors_off")
  mjw.fwd_position(m, d)
  d.energy.fill_(SENTINEL)
  mjw.energy_pos(m, d)
  e = _np(d.energy)
  assert (e[:, 1] == SENTINEL).all()
  mjw.energy_vel(m, d)
  e = _np(d.energy)
  for w in range(energy_scenes.NWORLD):
    sp, sk = scales(mjm, inputs, g, w)
    assert abs(e[w, 0] - g["direct/energy"][w, 0]) <= FWD_TOL * sp and abs(e[w, 1] - g["direct/energy"][w, 1]) <= FWD_TOL * sk
  assert mjw.last_launch_count() == 1


def _flags(m, enable=None, disable=None):
  """set ENBL_ENERGY to `enable` (0 or ENBL_ENERGY) and, if given, the disable flags"""
  if enable is not None:
    m.opt.enableflags = (int(m.opt.enableflags) & ~C.ENBL_ENERGY) | int(enable)
  if disable is not None:
    m.opt.disableflags = int(disable)


@pytest.mark.parametrize("call", ["forward", "step", "step1"])
def test_gpu_energy_pipeline_cells(built, call):
  """forward / step / step1: flag on -> both terms (and sensors); off with energy sensors -> sensors report, d.energy zeroed; off without
  them -> d.energy untouched.  With DSBL_SENSOR and the flag on, d.energy is still computed and the sensor slots are left alone."""
  mjw, g, mjm, inputs, m, d = setup("sensors_on")
  slots = [s for s, _, _ in energy_sensors(mjm)]
  want = g["direct/energy"]
  qpos, qvel = d.qpos.clone(), d.qvel.clone()

  def run():
    d.qpos.copy_(qpos)
    d.qvel.copy_(qvel)
    d.energy.fill_(SENTINEL)
    d.sensordata.fill_(SENTINEL)
    getattr(mjw, call)(m, d)
    return _np(d.energy), _np(d.sensordata)[:, slots]

  base = int(m.opt.disableflags)
  e, s = run()  # flag on, sensors
  np.testing.assert_allclose(e, want, rtol=1e-4)
  assert (s != SENTINEL).all()
  _flags(m, enable=0)
  e, s = run()  # flag off, sensors
  assert (e == 0.0).all() and (s != SENTINEL).all()
  _flags(m, enable=C.ENBL_ENERGY, disable=base | C.DSBL_SENSOR)
  e, s = run()  # flag on, sensors disabled: computed anyway, slots untouched (step1 zeroes sensordata first, as the reference does)
  np.testing.assert_allclose(e, want, rtol=1e-4)
  assert (s == (0.0 if call == "step1" else SENTINEL)).all()
  # flag off, no energy sensor
  mjw, g, mjm, inputs, m, d = setup("joints")
  _flags(m, enable=0)
  d.energy.fill_(SENTINEL)
  getattr(mjw, call)(m, d)
  assert (_np(d.energy) == SENTINEL).all()


@pytest.mark.parametrize("call", ["inverse", "sensor_pos"])
def test_gpu_energy_sensor_calls(built, call):
  """inverse and sensor_pos compute energy only for the energy sensors (and only their terms), whatever the flag says."""
  mjw, g, mjm, inputs, m, d = setup("sensors_off")
  mjw.forward(m, d)
  for enable in (0, C.ENBL_ENERGY):
    _flags(m, enable=enable)
    d.energy.fill_(SENTINEL)
    d.sensordata.fill_(SENTINEL)
    getattr(mjw, call)(m, d)
    np.testing.assert_allclose(_np(d.energy), g["direct/energy"], rtol=1e-4)
    assert (_np(d.sensordata)[:, [s for s, _, _ in energy_sensors(mjm)]] != SENTINEL).all()
  _flags(m, disable=int(m.opt.disableflags) | C.DSBL_SENSOR)
  d.energy.fill_(SENTINEL)
  getattr(mjw, call)(m, d)
  assert (_np(d.energy) == SENTINEL).all()
  # no energy sensor: nothing, flag or not
  mjw, g, mjm, inputs, m, d = setup("joints")
  mjw.forward(m, d)
  d.energy.fill_(SENTINEL)
  getattr(mjw, call)(m, d)
  assert (_np(d.energy) == SENTINEL).all()


@pytest.mark.parametrize("scene,nworld,per_pass", [("joints", 8, 1), ("joints_rk4", 8, 4), ("sensors_off", 8, 1), ("humanoid", 2048, 2)])
def test_gpu_energy_launch_count(built, scene, nworld, per_pass):
  """The flag off without energy sensors launches what the step launched before; with the flag (or an energy sensor) one k_energy more
  per forward pass and world half.  The count is the captured graph's kernel count."""
  from tests.test_gpu_launch_count import _captured_kernels

  import mujoco_warp_b200 as mjw

  _, mjm, _ = load(scene)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m)
  counts = {}
  for enable in (0, C.ENBL_ENERGY):
    _flags(m, enable=enable)
    mjw.step(m, d)
    kernels = _captured_kernels(lambda: mjw.step(m, d))
    assert mjw.last_launch_count() == kernels
    counts[enable] = kernels
  if scene.startswith("sensors"):
    assert counts[C.ENBL_ENERGY] == counts[0]
    _, mjm0, _ = load("joints")
    m0 = mjw.put_model(mjm0)
    d0 = mjw.make_data(mjm0, nworld=nworld, m=m0)
    _flags(m0, enable=0)
    mjw.step(m0, d0)
    # the sensor model launches k_sensor and k_energy on top of the sensor-free model's step
    assert counts[0] == _captured_kernels(lambda: mjw.step(m0, d0)) + 2 * per_pass
  else:
    assert counts[C.ENBL_ENERGY] == counts[0] + per_pass


def test_gpu_energy_toggle_without_reallocation(built):
  mjw, g, mjm, inputs, m, d = setup("joints")
  _flags(m, enable=0)
  mjw.forward(m, d)
  ptr, nkeep_m, nkeep_d = d.energy.data_ptr(), len(m._keep), len(d._keep)
  d.energy.fill_(SENTINEL)
  mjw.forward(m, d)
  assert (_np(d.energy) == SENTINEL).all()
  m.opt.enableflags = int(m.opt.enableflags) | C.ENBL_ENERGY
  mjw.forward(m, d)
  np.testing.assert_allclose(_np(d.energy), g["direct/energy"], rtol=1e-4)
  assert d.energy.data_ptr() == ptr and len(m._keep) == nkeep_m and len(d._keep) == nkeep_d
  # rebinding d.energy rebinds the kernel's pointer
  fresh = torch.full_like(d.energy, SENTINEL)
  d.energy = fresh
  mjw.forward(m, d)
  np.testing.assert_allclose(_np(fresh), g["direct/energy"], rtol=1e-4)


def test_gpu_energy_graph_replay_and_reproducibility(built):
  mjw, g, mjm, inputs, m, d = setup("humanoid", nworld=energy_scenes.NWORLD)
  qpos, qvel = d.qpos.clone(), d.qvel.clone()

  def reset():
    d.qpos.copy_(qpos)
    d.qvel.copy_(qvel)

  mjw.step(m, d)
  first = d.energy.clone()
  reset()
  mjw.step(m, d)
  assert torch.equal(d.energy, first)  # two runs are bit-identical
  reset()
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    mjw.step(m, d)
  reset()
  d.energy.fill_(SENTINEL)
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(d.energy, first)


def test_gpu_energy_every_world_of_two_halves(built):
  """2048 worlds run as two world halves: every world's energy is its own, against the fp64 formulas on the GPU's own intermediates."""
  import mujoco_warp_b200 as mjw

  _, mjm, _ = load("humanoid")
  nworld = 2048
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, nconmax=24, njmax=64, m=m)
  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, seed=5, qvel_noise=1.0)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  d.energy.fill_(float("nan"))
  mjw.forward(m, d)
  e, xipos, M, qp, qv = _np(d.energy), _np(d.xipos), _np(d.M), _np(d.qpos), _np(d.qvel)
  assert np.isfinite(e).all()
  for w in list(range(0, nworld, 97)) + [nworld // 2 - 1, nworld // 2, nworld - 1]:
    grav, spring = energy_oracle.potential_terms(mjm, {}, w, qp[w], xipos[w], np.zeros(0))
    kt = energy_oracle.kinetic_terms(mjm, qv[w], M[w])
    # only the fp32 sums differ from the fp64 ones here: at most about one ulp per term
    assert abs(e[w, 0] - (grav.sum() + spring.sum())) <= 1e-5 * (np.abs(grav).sum() + np.abs(spring).sum()), w
    assert abs(e[w, 1] - kt.sum()) <= 1e-5 * np.abs(kt).sum(), w


@pytest.mark.parametrize("scene", ["humanoid", "g1"])
def test_gpu_kinetic_energy_equals_the_bodies(built, scene):
  """1/2 qvel' M qvel minus the armature's share equals sum_b 1/2 cvel_b' I_b cvel_b from d.cvel and d.cinert (com-frame inertia)."""
  mjw, g, mjm, inputs, m, d = setup(scene)
  mjw.forward(m, d)
  e, cinert, cvel, qv = _np(d.energy), _np(d.cinert), _np(d.cvel), _np(d.qvel)
  arm = np.asarray(mjm.dof_armature, dtype=np.float64)
  for w in range(energy_scenes.NWORLD):
    body = 0.0
    for b in range(1, mjm.nbody):
      ci, cv = cinert[w, b], cvel[w, b]
      I = np.array([[ci[0], ci[3], ci[4]], [ci[3], ci[1], ci[5]], [ci[4], ci[5], ci[2]]])
      wv, lv = cv[:3], cv[3:]
      body += 0.5 * (wv @ I @ wv) + lv @ np.cross(wv, ci[6:9]) + 0.5 * ci[9] * lv @ lv
    joint = e[w, 1] - 0.5 * float(np.sum(arm * qv[w] * qv[w]))
    assert joint == pytest.approx(body, rel=1e-4), (w, joint, body)


def test_gpu_energy_drift_under_rk4(built):
  """No contacts, damping or actuation, RK4 at dt = 2 ms, the model's own (unbatched) parameters: the total energy of every world stays
  within 2e-4 of its scale (sum |term|) over 400 steps.  The fp64 CPU oracle drifts by about 1.3e-5 of the scale on these states; the
  rest of the bound is fp32 rounding.  (After an RK4 step d.energy is the last stage's; the energy of the state the step reached is
  evaluated on its own.)"""
  import mujoco_warp_b200 as mjw

  g, mjm, _ = load("joints_rk4")
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=energy_scenes.NWORLD, nconmax=4, njmax=16, m=m)
  d.qpos.copy_(torch.from_numpy(g["in/qpos"].astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(g["in/qvel"].astype(np.float32)))

  def energy_now():
    mjw.fwd_position(m, d)
    mjw.energy_pos(m, d)
    mjw.energy_vel(m, d)
    return _np(d.energy)

  e0 = energy_now()
  total0 = e0.sum(axis=1)
  scale = np.abs(e0).sum(axis=1)
  drift = np.zeros(energy_scenes.NWORLD)
  for _ in range(400):
    mjw.step(m, d)
    drift = np.maximum(drift, np.abs(energy_now().sum(axis=1) - total0))
  assert (drift <= 2e-4 * scale).all(), drift / scale
  assert np.abs(_np(d.qvel)).max() > 0.1  # the worlds moved
