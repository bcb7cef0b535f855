"""rne_postconstraint, subtree_vel, jac, xfrc_accumulate, tendon and deriv_smooth_vel on the GPU (k_body_stages.cu).

- Every scene of tests/body_stage_scenes.py against the reference's own outputs (tests/golden/body_stage_*.npz): forward from the seeded
  state, then each function.  Values that follow from the positions and velocities alone are held tightly; cacc / cfrc_int / cfrc_ext
  go through the fp32 constraint solve and get the looser tolerance of a solved force.
- rne_postconstraint / subtree_vel write bit for bit what forward writes for a model whose sensors need them, and also run for a model
  without sensors and under DSBL_SENSOR.
- jac against the velocities in cvel, xfrc_accumulate against jac, None outputs, NaN rows for a bad body id, bit-identical reruns, a CUDA
  graph replay, launch counts, and a trajectory unchanged by calling the six functions between steps.
"""
import os

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from tests import body_stage_scenes as S
from tests import util

pytestmark = pytest.mark.gpu

# fp32 against the fp64 reference, relative to the largest magnitude of each output (at least 1): kinematic quantities; forces that
# come out of the constraint solve
TOL_KIN = 2e-4
TOL_SOLVED = 1e-2


def _golden(name):
  return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"body_stage_{name}.npz"))


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _t(a, dtype=torch.float32):
  return torch.from_numpy(np.ascontiguousarray(np.asarray(a))).to(dtype).cuda()


def setup(scene):
  import mujoco_warp_b200 as mjw

  g, mjm = _golden(scene), S.load(scene)
  m = mjw.put_model(mjm)
  if S.SCENES[scene][1]:
    m.body_mass, m.body_inertia, m.dof_damping = _t(g["in/body_mass"]), _t(g["in/body_inertia"]), _t(g["in/dof_damping"])
  d = mjw.make_data(mjm, nworld=S.NWORLD, nconmax=int(g["in/nconmax"]), njmax=int(g["in/njmax"]), m=m)
  for f in ("qpos", "qvel", "ctrl", "act", "xfrc_applied"):
    getattr(d, f).copy_(_t(g[f"in/{f}"]).reshape(getattr(d, f).shape))
  return mjw, g, mjm, m, d


def _outputs(mjw, m, d, g, mjm):
  """the six functions after forward; returns {name: array}"""
  nw = d.nworld
  mjw.forward(m, d)
  mjw.rne_postconstraint(m, d)
  mjw.subtree_vel(m, d)
  mjw.tendon(m, d)
  jacp = torch.zeros((nw, 3, mjm.nv), device="cuda")
  jacr = torch.zeros((nw, 3, mjm.nv), device="cuda")
  mjw.jac(m, d, jacp, jacr, _t(g["in/point"]), _t(g["in/body"], torch.int32))
  qfrc = _t(g["in/qfrc"])
  mjw.xfrc_accumulate(m, d, qfrc)
  deriv = torch.zeros((nw, m.nC), device="cuda")
  mjw.deriv_smooth_vel(m, d, deriv)
  out = {f: getattr(d, f).clone() for f in ("cacc", "cfrc_int", "cfrc_ext", "subtree_linvel", "subtree_angmom", "ten_length", "ten_J")}
  out.update(jacp=jacp, jacr=jacr, qfrc=qfrc, deriv=deriv)
  return out


def _close(name, got, want, tol):
  got, want = _np(got).reshape(want.shape), np.asarray(want, dtype=np.float64)
  if want.size == 0:
    return
  err = np.abs(got - want).max()
  assert err <= tol * max(1.0, float(np.abs(want).max())), f"{name}: off by {err} (largest {np.abs(want).max()})"


@pytest.mark.parametrize("scene", list(S.SCENES))
def test_gpu_body_stages_meet_the_reference(built, scene):
  mjw, g, mjm, m, d = setup(scene)
  out = _outputs(mjw, m, d, g, mjm)
  torch.cuda.synchronize()
  _close(f"{scene} M", d.M, g["fwd/M"], TOL_KIN)
  for f in ("subtree_linvel", "subtree_angmom", "ten_length", "ten_J", "jacp", "jacr", "qfrc", "deriv"):
    _close(f"{scene} {f}", out[f], g[f"out/{f}"], TOL_KIN)
  for f in ("cacc", "cfrc_int", "cfrc_ext"):
    _close(f"{scene} {f}", out[f], g[f"out/{f}"], TOL_SOLVED)
  # rerun: bit-identical
  again = _outputs(mjw, m, d, g, mjm)
  for f in out:
    assert torch.equal(out[f], again[f]) or (torch.isnan(out[f]) == torch.isnan(again[f])).all(), f"{scene} {f} differs run to run"


def _sensor_scene(disable_sensor=False):
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import mjcf

  mjm = mjcf.load_string(util.sensor_xml())
  m = mjw.put_model(mjm)
  if disable_sensor:
    m.opt.disableflags = int(m.opt.disableflags) | C.DSBL_SENSOR
  d = mjw.make_data(mjm, nworld=8, nconmax=16, njmax=64, m=m)
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, 8)
  for f, v in (("qpos", qpos), ("qvel", qvel), ("ctrl", ctrl)):
    getattr(d, f).copy_(_t(v))
  d.xfrc_applied[:, 1:, :] = 0.3
  return mjw, mjm, m, d


def test_gpu_body_stages_match_the_sensor_path(built):
  """A model with accelerometer / force / subtree sensors: forward writes cacc .. subtree_angmom through k_sensor; the two calls run the
  same code and reproduce them bit for bit.  Under DSBL_SENSOR and for a model without sensors they still run."""
  mjw, mjm, m, d = _sensor_scene()
  mjw.forward(m, d)
  fields = ("cacc", "cfrc_int", "cfrc_ext", "subtree_linvel", "subtree_angmom")
  ref = {f: getattr(d, f).clone() for f in fields}
  for f in fields:
    getattr(d, f).fill_(float("nan"))
  mjw.rne_postconstraint(m, d)
  mjw.subtree_vel(m, d)
  for f in fields:
    assert torch.equal(getattr(d, f), ref[f]), f
  # DSBL_SENSOR: forward skips nothing it needs, the calls still write the same values
  mjw2, _, m2, d2 = _sensor_scene(disable_sensor=True)
  mjw2.forward(m2, d2)
  for f in fields:
    getattr(d2, f).fill_(float("nan"))
  mjw2.rne_postconstraint(m2, d2)
  mjw2.subtree_vel(m2, d2)
  for f in fields:
    assert torch.equal(getattr(d2, f), ref[f]), f"DSBL_SENSOR {f}"
  # nsensor == 0 (the humanoid)
  g_mjw, g, mjm_h, m_h, d_h = setup("humanoid_pyramidal")
  assert getattr(mjm_h, "nsensor", 0) == 0
  g_mjw.forward(m_h, d_h)
  for f in fields:
    getattr(d_h, f).fill_(float("nan"))
  g_mjw.rne_postconstraint(m_h, d_h)
  g_mjw.subtree_vel(m_h, d_h)
  for f in fields:
    assert bool(torch.isfinite(getattr(d_h, f)).all()), f


def test_gpu_jac_meets_cvel_and_xfrc_meets_jac(built):
  mjw, g, mjm, m, d = setup("humanoid_pyramidal")
  mjw.forward(m, d)
  nw, nb, nv = d.nworld, mjm.nbody, mjm.nv
  cvel, xipos, scom, qvel = _np(d.cvel).reshape(nw, nb, 6), _np(d.xipos).reshape(nw, nb, 3), _np(d.subtree_com).reshape(nw, nb, 3), _np(d.qvel)
  root = np.asarray(mjm.body_rootid)
  xfrc_sum = np.zeros((nw, nv))
  for b in range(nb):
    body = torch.full((nw,), b, dtype=torch.int32, device="cuda")
    point = _t(xipos[:, b])
    jacp = torch.zeros((nw, 3, nv), device="cuda")
    jacr = torch.zeros((nw, 3, nv), device="cuda")
    mjw.jac(m, d, jacp, jacr, point, body)
    jp, jr = _np(jacp), _np(jacr)
    lin = cvel[:, b, 3:] - np.cross(xipos[:, b] - scom[:, root[b]], cvel[:, b, :3])
    np.testing.assert_allclose(np.einsum("wkv,wv->wk", jp, qvel), lin, atol=2e-4 * max(1.0, np.abs(lin).max()))
    np.testing.assert_allclose(np.einsum("wkv,wv->wk", jr, qvel), cvel[:, b, :3], atol=2e-4 * max(1.0, np.abs(cvel[:, b, :3]).max()))
    f = _np(d.xfrc_applied).reshape(nw, nb, 6)[:, b]
    xfrc_sum += np.einsum("wkv,wk->wv", jp, f[:, :3]) + np.einsum("wkv,wk->wv", jr, f[:, 3:])
    # either output may be None and gives the same values in the other
    for p_on, r_on in ((True, False), (False, True), (False, False)):
      jp2 = torch.zeros_like(jacp) if p_on else None
      jr2 = torch.zeros_like(jacr) if r_on else None
      mjw.jac(m, d, jp2, jr2, point, body)
      if p_on:
        assert torch.equal(jp2, jacp)
      if r_on:
        assert torch.equal(jr2, jacr)
  qfrc = torch.zeros((nw, nv), device="cuda")
  mjw.xfrc_accumulate(m, d, qfrc)
  np.testing.assert_allclose(_np(qfrc), xfrc_sum, atol=2e-4 * max(1.0, np.abs(xfrc_sum).max()))


def test_gpu_jac_bad_body_gives_nan_rows(built):
  mjw, g, mjm, m, d = setup("humanoid_pyramidal")
  mjw.forward(m, d)
  nw, nv = d.nworld, mjm.nv
  body = torch.tensor([1, -1, mjm.nbody, 2], dtype=torch.int32, device="cuda")
  jacp = torch.zeros((nw, 3, nv), device="cuda")
  jacr = torch.zeros((nw, 3, nv), device="cuda")
  mjw.jac(m, d, jacp, jacr, torch.zeros((nw, 3), device="cuda"), body)
  torch.cuda.synchronize()
  for w in range(nw):
    bad = w in (1, 2)
    assert bool(torch.isnan(jacp[w]).all()) == bad and bool(torch.isnan(jacr[w]).all()) == bad
    assert bool(torch.isfinite(jacp[w]).all()) != bad


def test_gpu_body_stages_argument_checks(built):
  mjw, g, mjm, m, d = setup("equality")
  nw, nv = d.nworld, mjm.nv
  point, body = torch.zeros((nw, 3), device="cuda"), torch.zeros((nw,), dtype=torch.int32, device="cuda")
  with pytest.raises(ValueError, match="jacp"):
    mjw.jac(m, d, torch.zeros((nw, 3, nv + 1), device="cuda"), None, point, body)
  with pytest.raises(ValueError, match="body"):
    mjw.jac(m, d, None, None, point, body.long())
  with pytest.raises(ValueError, match="point"):
    mjw.jac(m, d, None, None, point.cpu(), body)
  with pytest.raises(ValueError, match="qfrc"):
    mjw.xfrc_accumulate(m, d, torch.zeros((nw, nv), device="cuda").t())
  with pytest.raises(ValueError, match="out"):
    mjw.deriv_smooth_vel(m, d, torch.zeros((nw, m.nC), device="cuda", dtype=torch.float64))


def test_gpu_body_stages_launch_counts(built):
  mjw, g, mjm, m, d = setup("tendon_actuator")
  nw, nv = d.nworld, mjm.nv
  mjw.forward(m, d)
  calls = (
    lambda: mjw.rne_postconstraint(m, d), lambda: mjw.subtree_vel(m, d), lambda: mjw.tendon(m, d),
    lambda: mjw.jac(m, d, torch.zeros((nw, 3, nv), device="cuda"), None, torch.zeros((nw, 3), device="cuda"), torch.ones((nw,), dtype=torch.int32, device="cuda")),
    lambda: mjw.xfrc_accumulate(m, d, torch.zeros((nw, nv), device="cuda")), lambda: mjw.deriv_smooth_vel(m, d, torch.zeros((nw, m.nC), device="cuda")),
  )
  for c in calls:
    c()
    assert mjw.last_launch_count() == 1
  mjw_h, _, _, m_h, d_h = setup("humanoid_pyramidal")
  mjw_h.tendon(m_h, d_h)
  assert mjw_h.last_launch_count() == 0


def test_gpu_body_stages_graph_replay_and_unchanged_trajectory(built):
  mjw, g, mjm, m, d = setup("humanoid_pyramidal")
  nw, nv = d.nworld, mjm.nv
  start = {f: getattr(d, f).clone() for f in ("qpos", "qvel", "ctrl", "act", "xfrc_applied", "qacc_warmstart", "time")}

  def reset():
    for f, v in start.items():
      getattr(d, f).copy_(v)

  point, body = _t(g["in/point"]), _t(g["in/body"], torch.int32)
  jacp, jacr = torch.zeros((nw, 3, nv), device="cuda"), torch.zeros((nw, 3, nv), device="cuda")
  qfrc, deriv = torch.zeros((nw, nv), device="cuda"), torch.zeros((nw, m.nC), device="cuda")

  def six():
    mjw.rne_postconstraint(m, d)
    mjw.subtree_vel(m, d)
    mjw.tendon(m, d)
    mjw.jac(m, d, jacp, jacr, point, body)
    qfrc.zero_()
    mjw.xfrc_accumulate(m, d, qfrc)
    mjw.deriv_smooth_vel(m, d, deriv)

  # stepping with the six calls in between gives the trajectory of stepping alone, bit for bit
  reset()
  for _ in range(5):
    mjw.step(m, d)
  plain = d.qpos.clone(), d.qvel.clone()
  reset()
  for _ in range(5):
    mjw.step(m, d)
    six()
  assert torch.equal(d.qpos, plain[0]) and torch.equal(d.qvel, plain[1])
  # eager step + six, then the same captured in a CUDA graph and replayed from the same state
  reset()
  mjw.step(m, d)
  six()
  eager = [t.clone() for t in (jacp, jacr, qfrc, deriv, d.cfrc_ext, d.cacc, d.cfrc_int, d.subtree_linvel, d.subtree_angmom, d.qpos)]
  reset()
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    mjw.step(m, d)
    six()
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    mjw.step(m, d)
    six()
  reset()
  graph.replay()
  torch.cuda.synchronize()
  got = [jacp, jacr, qfrc, deriv, d.cfrc_ext, d.cacc, d.cfrc_int, d.subtree_linvel, d.subtree_angmom, d.qpos]
  for a, b in zip(eager, got):
    assert torch.equal(a, b)
