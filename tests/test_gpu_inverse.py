"""Inverse dynamics on the GPU (mjw.inverse, reference inverse.py:148) checked against forward dynamics and the integrators.

- Round trip (reference inverse_test.py:66): forward() finds the qacc that the applied, actuator and passive forces produce, so
  inverse() at that qacc must give back qfrc_inverse = qfrc_smooth - qfrc_passive + qfrc_bias (= qfrc_applied + qfrc_actuator +
  J^T xfrc_applied) and forward's qfrc_constraint, to within what the solver leaves of its gradient.
- Discrete round trip: qacc = (qvel_next - qvel) / h of one step, with ENBL_INVDISCRETE, recovers the same forces (Euler with dof
  damping, implicitfast) and leaves d.qacc bit-identical.
- Zeroing (reference inverse_test.py:118), batched fields, the world split, graph capture and the launch count.
"""
import numpy as np
import pytest
import torch

from tests import util
from tests.test_gpu_launch_count import _captured_kernels
from tests.test_oracle_golden_pipeline import load_scene

pytestmark = pytest.mark.gpu


def _seeded(mjw, mjm, nworld, m=None, seed=42, xfrc=True, **kw):
  m = m or mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m, **kw)
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld, seed=seed)
  rng = np.random.default_rng(seed + 1)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  d.ctrl.copy_(torch.from_numpy(ctrl.astype(np.float32)))
  d.qfrc_applied.copy_(torch.from_numpy(rng.uniform(-0.5, 0.5, (nworld, mjm.nv)).astype(np.float32)))
  if xfrc:
    d.xfrc_applied[:, 1:].copy_(torch.from_numpy(rng.uniform(-0.5, 0.5, (nworld, mjm.nbody - 1, 6)).astype(np.float32)))
  if getattr(mjm, "na", 0):
    d.act.copy_(torch.from_numpy(util.seeded_act(mjm, nworld).astype(np.float32)))
  return m, d


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _scale(*arrays):
  return max(1.0, *(float(np.abs(a).max(initial=0.0)) for a in arrays))


@pytest.mark.parametrize("scene,nworld", [("humanoid", 1024), ("g1", 64), ("mixed_elliptic", 64), ("three_humanoids", 64), ("equality", 64), ("tendons", 64), ("sensors", 64)])
def test_inverse_of_forward_gives_back_the_applied_forces(built, scene, nworld):
  import mujoco_warp_b200 as mjw

  mjm = load_scene(scene)
  m, d = _seeded(mjw, mjm, nworld)
  # twice: in the equality scene the first pass after seeding the state gives other equality-row aref than every later one, and
  # inverse() repeats the position stage
  mjw.forward(m, d)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  qacc, qfc_fwd, sens_fwd = _np(d.qacc), _np(d.qfrc_constraint), _np(d.sensordata)
  want = _np(d.qfrc_smooth) - _np(d.qfrc_passive) + _np(d.qfrc_bias)
  d.qfrc_inverse.fill_(float("nan"))
  d.qfrc_constraint.fill_(float("nan"))
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  assert np.array_equal(_np(d.qacc), qacc)
  assert (_np(d.solver_niter) == 0).all()
  got, qfc = _np(d.qfrc_inverse), _np(d.qfrc_constraint)
  # the solver stops at its tolerance: M qacc - qfrc_smooth - qfrc_constraint is its remaining gradient (reference test: 5e-3)
  tol = 5e-3 * _scale(want, qfc_fwd, _np(d.qfrc_bias))
  err, err_c = np.abs(got - want).max(), np.abs(qfc - qfc_fwd).max()
  print(f"{scene}: max |qfrc_inverse - applied| {err:.3g}, |qfrc_constraint - forward's| {err_c:.3g}, tolerance {tol:.3g}")
  assert err <= tol and err_c <= tol
  if mjm.nsensordata:
    np.testing.assert_allclose(_np(d.sensordata), sens_fwd, atol=5e-3 * _scale(sens_fwd), rtol=5e-3)


@pytest.mark.parametrize("scene,eulerdamp", [("actuators", True), ("actuators", False), ("actuators_implicitfast", True), ("tendons_implicitfast", True), ("g1", True)])
def test_discrete_inverse_recovers_the_forces_of_a_step(built, scene, eulerdamp):
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import constants as C

  mjm = load_scene(scene)
  if not eulerdamp:
    mjm.opt.disableflags = int(mjm.opt.disableflags) | C.DSBL_EULERDAMP
  else:
    mjm.opt.disableflags = int(mjm.opt.disableflags) & ~C.DSBL_EULERDAMP
  mjm.opt.enableflags = int(mjm.opt.enableflags) | C.ENBL_INVDISCRETE
  nworld = 32
  m, d = _seeded(mjw, mjm, nworld)
  state = {f: getattr(d, f).clone() for f in ("qpos", "qvel", "act", "time", "qacc_warmstart")}
  mjw.step(m, d)
  torch.cuda.synchronize()
  qvel_next = d.qvel.clone()
  for f, v in state.items():
    getattr(d, f).copy_(v)
  d.qacc.copy_((qvel_next - state["qvel"]) / float(mjm.opt.timestep))
  qacc = d.qacc.clone()
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  assert torch.equal(d.qacc, qacc)  # d.qacc is the discrete one, untouched
  want = _np(d.qfrc_smooth) - _np(d.qfrc_passive) + _np(d.qfrc_bias)
  got = _np(d.qfrc_inverse)
  # fp32: (qvel_next - qvel) / h carries about eps32 |qvel_next| / h of rounding per dof, which M multiplies (at most its entry sum per
  # world); the rest is what the solver leaves of its gradient (5e-4 of scale)
  eps = float(np.finfo(np.float32).eps)
  msum = float(np.abs(_np(d.M)).sum(axis=1).max())
  tol = 5e-4 * _scale(want, _np(d.qfrc_constraint), _np(d.qfrc_bias)) + 16 * eps * float(np.abs(_np(qvel_next)).max()) / float(mjm.opt.timestep) * msum
  err = np.abs(got - want).max()
  print(f"{scene} eulerdamp={eulerdamp}: max |qfrc_inverse - applied| {err:.3g}, tolerance {tol:.3g}")
  assert err <= tol
  if eulerdamp:
    # negative control: without the conversion the same qacc must miss by more than the tolerance
    m.opt.enableflags = int(m.opt.enableflags) & ~C.ENBL_INVDISCRETE
    mjw.inverse(m, d)
    torch.cuda.synchronize()
    err_off = np.abs(_np(d.qfrc_inverse) - want).max()
    print(f"  without INVDISCRETE: {err_off:.3g}")
    assert err_off > tol


def test_discrete_inverse_rejects_rk4_and_implicit(built):
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import constants as C

  for scene in ("mixed_rk4", "mixed_implicit"):
    mjm = load_scene(scene)
    mjm.opt.enableflags = int(mjm.opt.enableflags) | C.ENBL_INVDISCRETE
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=2, m=m)
    with pytest.raises(NotImplementedError, match="INVDISCRETE"):
      mjw.inverse(m, d)
    mjm.opt.enableflags = 0
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=2, m=m)
    mjw.inverse(m, d)  # continuous-time inverse dynamics works with every integrator


_SPHERE = """
<mujoco>
  <option solver="CG"/>
  <worldbody>
    <geom type="plane" size="10 10 .001"/>
    <body name="sphere" pos="0 0 0.04">
      <freejoint/>
      <geom type="sphere" size="0.05" mass="1.0"/>
    </body>
  </worldbody>
</mujoco>
"""


def _spheres(n):
  bodies = "".join(f'<body pos="{0.2 * i} 0 0.04"><freejoint/><geom type="sphere" size="0.05" mass="1.0"/></body>' for i in range(n))
  return _SPHERE.replace('<body name="sphere" pos="0 0 0.04">\n      <freejoint/>\n      <geom type="sphere" size="0.05" mass="1.0"/>\n    </body>', bodies)


@pytest.mark.parametrize("nsphere", [1, 6])  # 6 free spheres: nv = 36, a sparse model (CSR view of efc.J, the nv > 32 kernel)
def test_qfrc_constraint_is_zeroed_without_rows(built, nsphere):
  """reference inverse_test.py:118: in contact, then teleported away from it (CG; dense and sparse)."""
  import mujoco_warp_b200 as mjw

  mjm = mjw.mjcf.load_string(_spheres(nsphere))
  m = mjw.put_model(mjm)
  assert m.is_sparse == (nsphere > 1)
  d = mjw.make_data(mjm, nworld=4, m=m)
  d.qpos.zero_()
  for i in range(nsphere):
    d.qpos[:, 7 * i] = 0.2 * i
    d.qpos[:, 7 * i + 3] = 1.0
    d.qpos[:, 7 * i + 2] = 0.04
  d.qvel.zero_()
  d.qacc.zero_()
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  assert (_np(d.nefc) > 0).all()
  assert np.abs(_np(d.qfrc_constraint)).max(axis=1).min() > 1.0
  for i in range(nsphere):
    d.qpos[:, 7 * i + 2] = 1.0
  d.qfrc_constraint.fill_(float("nan"))
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  assert (_np(d.nefc) == 0).all()
  assert (_np(d.qfrc_constraint) == 0).all()
  np.testing.assert_allclose(_np(d.qfrc_inverse), _np(d.qfrc_bias) + _np(d.efc.Ma) - _np(d.qfrc_passive), rtol=0, atol=0)


def test_batched_damping_matches_per_world_models(built):
  """dof_damping batched over the worlds: discrete Euler inverse dynamics of world w equals a one-world run on w's values."""
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import constants as C

  mjm = load_scene("actuators")
  mjm.opt.disableflags = int(mjm.opt.disableflags) & ~C.DSBL_EULERDAMP
  mjm.opt.enableflags = int(mjm.opt.enableflags) | C.ENBL_INVDISCRETE
  nworld = 4
  m = mjw.put_model(mjm, batch_sizes={"dof_damping": nworld})
  scale = np.array([0.5, 1.0, 2.0, 4.0], dtype=np.float32)
  m.dof_damping.mul_(torch.from_numpy(scale[:, None]).cuda())
  m, d = _seeded(mjw, mjm, nworld, m=m)
  qacc = torch.from_numpy(np.random.default_rng(7).uniform(-2, 2, (nworld, mjm.nv)).astype(np.float32)).cuda()
  d.qacc.copy_(qacc)
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  for w in range(nworld):
    m1 = mjw.put_model(mjm)
    m1.dof_damping.mul_(float(scale[w]))
    d1 = mjw.make_data(mjm, nworld=1, m=m1)
    for f in ("qpos", "qvel", "ctrl", "act", "qfrc_applied", "xfrc_applied"):
      getattr(d1, f).copy_(getattr(d, f)[w : w + 1])
    d1.qacc.copy_(qacc[w : w + 1])
    mjw.inverse(m1, d1)
    torch.cuda.synchronize()
    for f in ("qfrc_inverse", "qfrc_constraint"):
      np.testing.assert_allclose(_np(getattr(d, f))[w], _np(getattr(d1, f))[0], rtol=2e-5, atol=2e-6, err_msg=f"world {w}: {f}")
  assert np.abs(_np(d.qfrc_inverse)[0] - _np(d.qfrc_inverse)[3]).max() > 1e-3


def test_world_split_is_bit_identical(built, monkeypatch):
  import mujoco_warp_b200 as mjw

  mjm = load_scene("humanoid")
  out = []
  for split in ("1", "2"):
    monkeypatch.setenv("MJB_SPLIT", split)
    m, d = _seeded(mjw, mjm, 2048)
    mjw.forward(m, d)
    mjw.inverse(m, d)
    torch.cuda.synchronize()
    out.append({f: _np(getattr(d, f)) for f in ("qfrc_inverse", "qfrc_constraint", "nefc")} | {"force": _np(d.efc.force), "state": _np(d.efc.state)})
  for f in out[0]:
    assert np.array_equal(out[0][f], out[1][f]), f


@pytest.mark.parametrize("scene,nworld,discrete", [("humanoid", 8, False), ("humanoid", 2048, False), ("sensors", 8, False), ("g1", 8, False), ("actuators_implicitfast", 8, True)])
def test_inverse_captures_in_a_graph_and_counts_its_kernels(built, scene, nworld, discrete):
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import constants as C

  mjm = load_scene(scene)
  if discrete:
    mjm.opt.enableflags = int(mjm.opt.enableflags) | C.ENBL_INVDISCRETE
  m, d = _seeded(mjw, mjm, nworld)
  mjw.forward(m, d)
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  eager = _np(d.qfrc_inverse)
  kernels = _captured_kernels(lambda: mjw.inverse(m, d))
  assert mjw.last_launch_count() == kernels
  assert kernels == (5 + (1 if mjm.nsensor else 0) + (1 if mjm.nv > 32 else 0)) * (2 if nworld >= 1024 else 1)
  d.qfrc_inverse.zero_()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    mjw.inverse(m, d)
  g.replay()
  torch.cuda.synchronize()
  assert np.array_equal(_np(d.qfrc_inverse), eager)
