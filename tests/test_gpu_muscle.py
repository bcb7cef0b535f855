"""Muscle actuators on the GPU (mjb_muscle.cuh in k_velocity's actuation stage, k_set_length_range through set_length_range).

- The scenes of tests/muscle_scenes.py against the reference's own results (tests/golden/muscle_*.npz), step by step from the reference's
  state (Euler, implicitfast, implicit, RK4, the humanoid with a muscle pair per motor); forward, inverse, step1 + step2.
- Per-world gainprm / biasprm / actuator_acc0 / actuator_lengthrange against the fp64 actuation of tests/muscle_oracle.py, world by world,
  and whole batched steps (Euler, implicitfast, implicit, RK4) against its fp64 step (the pipeline oracle plus the muscle forces).
- set_length_range against the reference and the oracle, with per-world jnt_range / tendon_range / gear; set_const then step reads the
  new acc0.
- Two runs are bit-identical; inverse reports forward's actuator forces; a muscle model launches the kernels of its affine twin.
"""
import os

import numpy as np
import pytest
import torch

from tests import muscle_oracle as O
from tests import muscle_scenes as S

pytestmark = pytest.mark.gpu

STATE = ("time", "qpos", "qvel", "act", "qacc_warmstart", "ctrl")
# fp32 against the fp64 reference after one step from the same state, the tolerances of the other golden replays.  Every scene,
# the humanoid and RK4 included, stays within them by two or more orders of magnitude (largest seen on an H100: qvel 1.3e-6 relative,
# the humanoid; 4.1e-7 elsewhere).
TOL = {"actuator_force": 2e-5, "act_dot": 2e-5, "qfrc_actuator": 2e-5, "act": 2e-5, "qpos": 2e-5, "qvel": 2e-4, "sensordata": 2e-4, "time": 1e-7}


def _golden(name):
  return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"muscle_{name}.npz"))


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).cuda()


def setup(scene, nworld=S.NWORLD, batch_sizes=None):
  import mujoco_warp_b200 as mjw

  g, mjm = _golden(scene), S.load(scene)
  m = mjw.put_model(mjm, batch_sizes=batch_sizes)
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


@pytest.mark.parametrize("scene", list(S.SCENES))
def test_gpu_muscle_steps_meet_the_reference(built, scene):
  mjw, g, mjm, m, d = setup(scene)
  for k in range(S.SCENES[scene][1]):
    _load_state(d, g, f"step/{k}/in_")
    mjw.step(m, d)
    _compare(d, g, f"step/{k}/out_", TOL, f"{scene} step {k}")


@pytest.mark.parametrize("scene", ["euler", "implicit"])
def test_gpu_muscle_split_step_meets_the_reference(built, scene):
  """step1, then the ctrl, then step2: fwd_actuation and the integrators carry the muscles as step does."""
  mjw, g, mjm, m, d = setup(scene)
  for k in range(S.SCENES[scene][1]):
    _load_state(d, g, f"step/{k}/in_")
    ctrl = d.ctrl.clone()
    d.ctrl.zero_()
    mjw.step1(m, d)
    d.ctrl.copy_(ctrl)
    mjw.step2(m, d)
    _compare(d, g, f"step/{k}/out_", TOL, f"{scene} split step {k}")


@pytest.mark.parametrize("scene", list(S.SCENES))
def test_gpu_muscle_forward_and_inverse(built, scene):
  """forward meets the reference; inverse at forward's qacc reports the same actuator forces and act_dot."""
  mjw, g, mjm, m, d = setup(scene)
  _load_state(d, g, "start/")
  mjw.forward(m, d)
  tol = {f: TOL[f] for f in ("actuator_force", "act_dot", "qfrc_actuator")}
  _compare(d, g, "forward/", tol, f"{scene} forward")
  fwd_force, fwd_act_dot = d.actuator_force.clone(), d.act_dot.clone()
  d.actuator_force.zero_()
  d.act_dot.zero_()
  mjw.inverse(m, d)
  assert torch.equal(d.actuator_force, fwd_force), f"{scene}: inverse's actuator_force differs from forward's"
  assert torch.equal(d.act_dot, fwd_act_dot), f"{scene}: inverse's act_dot differs from forward's"
  _compare(d, g, "inverse/", {"actuator_force": TOL["actuator_force"], "act_dot": TOL["act_dot"]}, f"{scene} inverse")


def _oracle_check(mjm, m, d, what, tol=2e-5):
  """actuator_force and act_dot of every world against the fp64 oracle at the GPU's own lengths, velocities, ctrl and act, with each
  world's entry of the (possibly batched) muscle fields."""
  nw = d.nworld
  row = lambda x, w: _np(x)[w % x.shape[0]]
  L, V, ctrl, act = _np(d.actuator_length), _np(d.actuator_velocity), _np(d.ctrl), _np(d.act)
  force, act_dot = _np(d.actuator_force), _np(d.act_dot)
  for w in range(nw):
    want_ad, want_f = O.actuation(mjm, ctrl[w], act[w], L[w], V[w], float(mjm.opt.timestep), gainprm=row(m.actuator_gainprm, w), biasprm=row(m.actuator_biasprm, w),
                                  acc0=row(m.actuator_acc0, w), lengthrange=row(m.actuator_lengthrange, w))
    scale = max(1.0, float(np.abs(want_f).max()))
    assert np.abs(force[w] - want_f).max() <= tol * scale, f"{what} world {w}: actuator_force off by {np.abs(force[w] - want_f).max()}"
    assert np.abs(act_dot[w] - want_ad).max() <= tol * max(1.0, float(np.abs(want_ad).max())), f"{what} world {w}: act_dot"


@pytest.mark.parametrize("scene", ["euler", "humanoid"])
def test_gpu_muscle_per_world_fields_meet_the_oracle(built, scene):
  nworld = 5
  fields = ("actuator_gainprm", "actuator_biasprm", "actuator_acc0", "actuator_lengthrange")
  mjw, g, mjm, m, d = setup(scene, nworld=nworld, batch_sizes={f: nworld for f in fields})
  rng = np.random.default_rng(1)
  s = torch.from_numpy(rng.uniform(0.7, 1.3, (nworld, 1))).float().cuda()
  m.actuator_acc0 = m.actuator_acc0 * s
  m.actuator_lengthrange = m.actuator_lengthrange * s[:, :, None]
  gp = m.actuator_gainprm.clone()
  gp[:, :, 2] = torch.where(gp[:, :, 2] > 0, gp[:, :, 2] * s, gp[:, :, 2])  # positive peak forces scaled, acc0-scaled ones kept
  gp[:, :, 7] *= s[:, :1]  # fpmax
  m.actuator_gainprm = gp
  m.actuator_biasprm = gp.clone()
  qpos, qvel, act, ctrl = S.seeded(mjm, 1, nworld=nworld, seed=11)
  d.qpos.copy_(_t(qpos))
  d.qvel.copy_(_t(qvel))
  d.act.copy_(_t(act))
  d.ctrl.copy_(_t(ctrl[0]))
  mjw.forward(m, d)
  _oracle_check(mjm, m, d, scene)
  # each world equals an unbatched model carrying that world's values
  for w in (0, 3):
    m1 = mjw.put_model(mjm)
    for f in fields:
      setattr(m1, f, getattr(m, f)[w : w + 1].clone())
    d1 = mjw.make_data(mjm, nworld=1, nconmax=int(g["in/nconmax"]), njmax=int(g["in/njmax"]), m=m1)
    for f in ("qpos", "qvel", "act", "ctrl"):
      getattr(d1, f).copy_(getattr(d, f)[w : w + 1])
    mjw.forward(m1, d1)
    assert torch.equal(d1.actuator_force[0], d.actuator_force[w]), f"{scene} world {w}"


def test_gpu_set_length_range_meets_the_reference(built):
  for scene in ("euler", "humanoid"):
    mjw, g, mjm, m, d = setup(scene, batch_sizes={"actuator_lengthrange": S.NWORLD})
    m.actuator_lengthrange.fill_(-7.0)
    mjw.set_length_range(m, d)
    np.testing.assert_allclose(_np(m.actuator_lengthrange), g["lengthrange/single"], rtol=1e-6, err_msg=scene)
    nb = {"jnt_range": S.NWORLD, "actuator_gear": S.NWORLD, "actuator_lengthrange": S.NWORLD}
    if int(getattr(mjm, "ntendon", 0)):
      nb["tendon_range"] = S.NWORLD
    mjw, g, mjm, m, d = setup(scene, batch_sizes=nb)
    m.jnt_range = _t(g["lengthrange/jnt_range"])
    if int(getattr(mjm, "ntendon", 0)):
      m.tendon_range = _t(g["lengthrange/tendon_range"])
    m.actuator_gear = _t(g["lengthrange/gear"])
    mjw.set_length_range(m, d, -1)
    np.testing.assert_allclose(_np(m.actuator_lengthrange), g["lengthrange/batched"], rtol=1e-6, err_msg=scene)
    # an unbatched output takes world 0's result; a wrong index or an output wider than the Data is refused
    mjw, g, mjm, m, d = setup(scene)
    mjw.set_length_range(m, d, 0)
    np.testing.assert_allclose(_np(m.actuator_lengthrange), g["lengthrange/single"][:1], rtol=1e-6)
    with pytest.raises(ValueError, match="index"):
      mjw.set_length_range(m, d, int(mjm.nu))
    m.actuator_lengthrange = m.actuator_lengthrange.repeat(S.NWORLD + 1, 1, 1)
    with pytest.raises(ValueError, match="per-world entries"):
      mjw.set_length_range(m, d)


def test_gpu_set_const_then_step_reads_the_new_acc0(built):
  """Doubling a world's body masses changes its acc0 through set_const; the next forward scales that world's force < 0 muscles by it."""
  nworld = 3
  mjw, g, mjm, m, d = setup("euler", nworld=nworld, batch_sizes={"body_mass": nworld, "body_inertia": nworld, "actuator_acc0": nworld})
  m.body_mass[1] *= 2.0
  m.body_inertia[1] *= 2.0
  _load_state(d, g, "start/")
  mjw.forward(m, d)
  before = d.actuator_force.clone()
  mjw.set_const(m, d)
  acc0 = _np(m.actuator_acc0)
  assert np.allclose(acc0[0], acc0[2]) and np.all(np.abs(acc0[1] - 0.5 * acc0[0]) <= 1e-5 * acc0[0]), acc0
  _load_state(d, g, "start/")
  mjw.forward(m, d)
  _oracle_check(mjm, m, d, "after set_const")
  neg = np.asarray(mjm.actuator_gainprm)[:, 2] < 0
  neg &= np.asarray(mjm.actuator_gaintype) == 2
  f0, f1 = _np(before), _np(d.actuator_force)
  # worlds 0 and 2 keep their acc0 up to the fp32 recomputation
  np.testing.assert_allclose(f1[[0, 2]], f0[[0, 2]], rtol=1e-4, atol=1e-6)
  moved = np.abs(f1[1, neg]) > 1e-6
  np.testing.assert_allclose(f1[1, neg][moved], 2.0 * f0[1, neg][moved], rtol=1e-4)


@pytest.mark.parametrize("scene", ["implicit", "humanoid"])
def test_gpu_muscle_runs_are_bit_identical(built, scene):
  runs = []
  for _ in range(2):
    mjw, g, mjm, m, d = setup(scene)
    _load_state(d, g, "start/")
    for _ in range(5):
      mjw.step(m, d)
    runs.append([getattr(d, f).clone() for f in ("qpos", "qvel", "act", "actuator_force")])
  for a, b in zip(*runs):
    assert torch.equal(a, b)


def test_gpu_muscle_model_launches_the_kernels_of_its_affine_twin(built):
  """The muscle humanoid launches, per step, the kernels of the same model with affine actuators and filter dynamics (the humanoid
  without activations launches the count tests/test_gpu_launch_count.py holds it to)."""
  from tests.test_gpu_launch_count import _captured_kernels

  import mujoco_warp_b200 as mjw

  counts = []
  for muscle in (True, False):
    mjm = S.humanoid(muscle)
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=64, m=m)
    mjw.step(m, d)
    counts.append(_captured_kernels(lambda: mjw.step(m, d)))
    assert mjw.last_launch_count() == counts[-1]
  assert counts[0] == counts[1], counts


@pytest.mark.parametrize("scene", ["euler", "implicitfast", "implicit", "rk4"])
def test_gpu_muscle_batched_steps_meet_the_fp64_oracle(built, scene):
  """Steps with per-world muscle fields, each from the GPU's own state, against the fp64 step of every world."""
  nworld = 4
  fields = ("actuator_gainprm", "actuator_biasprm", "actuator_acc0", "actuator_lengthrange")
  mjw, g, mjm, m, d = setup(scene, nworld=nworld, batch_sizes={f: nworld for f in fields})
  s = torch.tensor([[1.0], [0.8], [1.25], [0.9]], device="cuda")
  m.actuator_acc0 = m.actuator_acc0 * s
  m.actuator_lengthrange = m.actuator_lengthrange * s[:, :, None]
  gp = m.actuator_gainprm.clone()
  gp[:, :, 2] = torch.where(gp[:, :, 2] > 0, gp[:, :, 2] * s, gp[:, :, 2])
  gp[:, :, 8] = torch.where(gp[:, :, 8] > 0, gp[:, :, 8] * s.sqrt(), gp[:, :, 8])  # fvmax
  m.actuator_gainprm = gp
  m.actuator_biasprm = gp.clone()
  o = O.MuscleStep(mjm, nworld, int(g["in/nconmax"]), int(g["in/njmax"]), muscle_fields={f: _np(getattr(m, f)) for f in fields})
  qpos, qvel, act, ctrl = S.seeded(mjm, 3, nworld=nworld, seed=13)
  d.qpos.copy_(_t(qpos))
  d.qvel.copy_(_t(qvel))
  d.act.copy_(_t(act))
  for k in range(3):
    d.ctrl.copy_(_t(ctrl[k]))
    state = {f: _np(getattr(d, f)) for f in STATE}
    want = dict(zip(("time", "qpos", "qvel", "act", "act_dot", "actuator_force"),
                    o.step(state["time"], state["qpos"], state["qvel"], state["act"], state["ctrl"], state["qacc_warmstart"])))
    mjw.step(m, d)
    for f, t in (("time", 1e-7), ("qpos", TOL["qpos"]), ("qvel", TOL["qvel"]), ("act", TOL["act"]), ("act_dot", TOL["act_dot"]), ("actuator_force", TOL["actuator_force"])):
      got = _np(getattr(d, f)).reshape(np.shape(want[f]))
      scale = max(1.0, float(np.abs(want[f]).max()))
      assert np.abs(got - want[f]).max() <= t * scale, f"{scene} step {k}: {f} off by {np.abs(got - want[f]).max()} (scale {scale})"
