"""set_const on the GPU (k_set_const.cu through mjw.set_const / set_const_0 / set_const_spring / set_const_fixed).

- The scenes of tests/set_const_scenes.py with per-world inputs and every output batched: each world's entry against the numpy
  per-world oracle (tests/set_const_oracle.py), and the reference's own set_const on the same scenes (tests/golden/set_const_*.npz,
  tools/make_set_const_goldens.py), which the oracle meets at 1e-9 in the CPU suite (tests/test_set_const_vectors.py).
- Unmodified models (humanoid, G1, three_humanoids, the equality and tendon scenes): set_const reproduces put_model's values; the
  bodies where the reference's translational / rotational fallback applies and this repo's compiler has none are named.
- restore=True leaves the restore fields bit-identical to the position stages and factor_m at d.qpos; d.qpos comes back bit-exactly in
  every mode; a second call is bit-identical to the first; the launch count does not depend on the model; the C entry point replays
  from a CUDA graph with the same result.
- End to end: four worlds with scaled masses and inertias, set_const, forward and four steps match a model compiled with those masses.
"""
import copy

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import mjcf
from tests import set_const_oracle, set_const_scenes, util
from tests.test_gpu_golden_pipeline import close

pytestmark = pytest.mark.gpu

# fp32 against fp64, as a fraction of max(1, max |field|): the largest gap observed on an H100 is 8.3e-7 (dof_invweight0 of the mixed
# scene; actuator_acc0 7.8e-7, tendon_invweight0 7.3e-7, body_invweight0 5.7e-7, meaninertia 1.7e-7 relative, poses <= 1.4e-7), so 5x that
REF_TOL = 4e-6
# put_model's values come from this repo's fp64 compiler, rounded to fp32: the largest gap observed on an H100 is 1.1e-5 (actuator_acc0 of
# three_humanoids; dof_invweight0 6.4e-6 on the humanoid, every pose and mass <= 1.6e-7), so about 4.5x that
PUT_MODEL_TOL = 5e-5
RESTORE_FIELDS = ("xpos", "xquat", "xmat", "xipos", "ximat", "xanchor", "xaxis", "geom_xpos", "geom_xmat", "site_xpos", "site_xmat", "cam_xpos",
                  "cam_xmat", "light_xpos", "light_xdir", "subtree_com", "cinert", "cdof", "ten_length", "ten_J", "crb", "M", "qLD", "actuator_length",
                  "actuator_moment", "moment_rownnz", "moment_rowadr", "moment_colind")


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _batched_model(mjw, mjm, inputs, nworld):
  """put_model with the scene's inputs per world and every set_const output batched to nworld."""
  sizes = {f: nworld for f in inputs}
  for f in set_const_scenes.OUTPUTS:
    sizes.setdefault(f, nworld)
  m = mjw.put_model(mjm, batch_sizes=sizes)
  for f, v in inputs.items():
    getattr(m, f).copy_(torch.from_numpy(np.asarray(v, dtype=np.float32)).reshape(getattr(m, f).shape))
  return m


@pytest.mark.parametrize("scene", sorted(set_const_scenes.SCENES))
def test_gpu_set_const_matches_the_per_world_oracle(built, scene):
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(set_const_scenes.SCENES[scene])
  nworld = set_const_scenes.NWORLD
  inputs = set_const_scenes.per_world_inputs(scene, mjm)
  batched = scene != "unbatched"
  m = _batched_model(mjw, mjm, inputs, nworld) if batched else mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m)
  # fp32 inputs on both sides
  f32 = {f: np.asarray(v, dtype=np.float32).astype(np.float64) for f, v in inputs.items()}
  want = set_const_oracle.oracle(mjm, f32, nworld if batched else 1)
  mjw.set_const(m, d)
  torch.cuda.synchronize()
  for f in set_const_scenes.OUTPUTS:
    got = _np(getattr(m, f))
    w = want[f].reshape(got.shape)
    scale = max(1.0, float(np.abs(w).max())) if w.size else 1.0
    close(f"{scene}/{f}", got, w, atol=REF_TOL * scale)
  close(f"{scene}/meaninertia", _np(m.stat.meaninertia)[0], want["meaninertia"], atol=0, rtol=REF_TOL)


VECTOR_CASES = [(sc, c) for sc in sorted(set_const_scenes.SCENES) for c in ("set_const", "set_const_0", "set_const_spring")
                if c == "set_const" or sc in ("tendon", "dampratio")]


def reference_gap(scene, call):
  """{field: max |GPU - reference| / max(1, max |reference|)} of `call` on a fixture scene, and the same for meaninertia."""
  import mujoco_warp_b200 as mjw
  from tests.test_set_const_vectors import load

  g, mjm, inputs = load(scene)
  nworld = set_const_scenes.NWORLD
  m = mjw.put_model(mjm) if scene == "unbatched" else _batched_model(mjw, mjm, inputs, nworld)
  d = mjw.make_data(mjm, nworld=nworld, m=m)
  getattr(mjw, call)(m, d)
  torch.cuda.synchronize()
  gap = {}
  for f in set_const_scenes.OUTPUTS:
    want = g[f"{call}/{f}"]
    if want.size:
      gap[f] = float(np.abs(_np(getattr(m, f)).reshape(want.shape) - want).max()) / max(1.0, float(np.abs(want).max()))
  if call != "set_const_spring":
    want = float(g[f"{call}/meaninertia"][0])
    gap["meaninertia"] = abs(float(m.stat.meaninertia[0]) - want) / want
  return gap


@pytest.mark.parametrize("scene,call", VECTOR_CASES)
def test_gpu_set_const_meets_the_reference(built, scene, call):
  """The reference's own set_const (fp64, under the warp shim) on the fixture scenes, every output batched per world."""
  for f, e in reference_gap(scene, call).items():
    assert e <= REF_TOL, f"{scene}/{call}/{f}: {e:.3g} of scale > {REF_TOL}"


# bodies of unmodified models where one invweight0 component is below MINVAL and the reference copies the other one over
FALLBACK_BODIES = {"humanoid": [], "g1": [], "three_humanoids": [], "equality": ["s1", "s2", "s3"], "tendons": ["palm", "f1", "f2"]}
AIMED_LIGHTS = {"humanoid": ["spotlight"], "g1": [], "three_humanoids": ["spotlight"], "equality": [], "tendons": []}


def _scene(name):
  return {"humanoid": lambda: mjcf.load_any(util.HUMANOID), "g1": lambda: mjcf.load_any(util.G1), "three_humanoids": lambda: mjcf.load_any(util.THREE_HUMANOIDS),
          "equality": lambda: mjcf.load_string(util.EQUALITY_XML), "tendons": lambda: mjcf.load_string(util.tendon_xml())}[name]()


@pytest.mark.parametrize("scene", sorted(FALLBACK_BODIES))
def test_gpu_set_const_reproduces_put_model(built, scene):
  import mujoco_warp_b200 as mjw

  mjm = _scene(scene)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=4, m=m)
  before = {f: _np(getattr(m, f)) for f in set_const_scenes.OUTPUTS}
  mi = float(m.stat.meaninertia[0])
  mjw.set_const(m, d)
  torch.cuda.synchronize()
  bw = before["body_invweight0"].copy()
  tr, rot = bw[0, :, 0], bw[0, :, 1]
  fb = ((tr < 1e-15) & (rot > 1e-15)) | ((rot < 1e-15) & (tr > 1e-15))
  assert [mjm.names.body[b] for b in np.nonzero(fb)[0]] == FALLBACK_BODIES[scene]
  bw[0, fb] = np.maximum(tr, rot)[fb, None]
  before["body_invweight0"] = bw
  # light_dir0 of a light aimed at a body is the direction the position stage computes at qpos0 (set_const.py:469); this repo's
  # compiler stores the light's own direction for every mode.  Only track / trackcom lights read light_dir0.
  aimed = np.isin(np.asarray(mjm.light_mode), (3, 4)) & (np.asarray(mjm.light_targetbodyid) >= 0)
  assert [mjm.names.light[i] for i in np.nonzero(aimed)[0]] == AIMED_LIGHTS[scene]
  before["light_dir0"][:, aimed] = _np(m.light_dir0)[:, aimed]
  for f in set_const_scenes.OUTPUTS:
    got = _np(getattr(m, f))
    scale = max(1.0, float(np.abs(before[f]).max())) if before[f].size else 1.0
    close(f"{scene}/{f}", got, before[f], atol=PUT_MODEL_TOL * scale)
  assert abs(float(m.stat.meaninertia[0]) - mi) <= PUT_MODEL_TOL * mi


def _restore_state(m, d):
  return {f: getattr(d, f).clone() for f in RESTORE_FIELDS + ("qpos",)}


@pytest.mark.parametrize("scene,fn", [(s, f) for s in ("humanoid", "tendons", "equality") for f in ("set_const", "set_const_0")] + [("tendons", "set_const_spring")])
def test_gpu_set_const_restores_the_state(built, scene, fn):
  import mujoco_warp_b200 as mjw

  mjm = _scene(scene)
  nworld = 6
  m = mjw.put_model(mjm, batch_sizes={"body_mass": 4, "dof_invweight0": 4, "body_subtreemass": 4, "tendon_lengthspring": 3})
  m.body_mass.mul_(torch.linspace(0.7, 1.4, 4, device=m.body_mass.device)[:, None])
  d = mjw.make_data(mjm, nworld=nworld, m=m)
  mjw.set_const(m, d)  # the new constants first: the position stages below read body_subtreemass and the camera / light poses
  qpos = util.seeded_state(mjm, nworld)[0]
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  mjw.fwd_position(m, d)
  mjw.factor_m(m, d)
  want = _restore_state(m, d)
  getattr(mjw, fn)(m, d)
  torch.cuda.synchronize()
  for f, v in want.items():
    assert torch.equal(getattr(d, f), v), f"{fn}: {f} not restored"
  getattr(mjw, fn)(m, d, restore=False)
  assert torch.equal(d.qpos, want["qpos"])


@pytest.mark.parametrize("scene", ["humanoid", "tendons", "g1"])
def test_gpu_set_const_second_call_is_bit_identical(built, scene):
  import mujoco_warp_b200 as mjw

  mjm = _scene(scene)
  nworld = 8
  m = mjw.put_model(mjm, batch_sizes={"body_mass": nworld, **{f: nworld for f in set_const_scenes.OUTPUTS}})
  m.body_mass.mul_(torch.linspace(0.6, 1.5, nworld, device=m.body_mass.device)[:, None])
  d = mjw.make_data(mjm, nworld=nworld, m=m)
  mjw.set_const(m, d)
  first = {f: getattr(m, f).clone() for f in set_const_scenes.OUTPUTS}
  mi = m.stat.meaninertia.clone()
  nkeep = len(m._keep)
  mjw.set_const(m, d)
  torch.cuda.synchronize()
  assert len(m._keep) == nkeep  # handing meaninertia back does not pin another tensor per call
  for f, v in first.items():
    assert torch.equal(getattr(m, f), v), f
  assert torch.equal(m.stat.meaninertia, mi)


def test_gpu_set_const_launch_count_does_not_depend_on_the_model(built):
  import mujoco_warp_b200 as mjw

  counts = []
  for scene in ("humanoid", "three_humanoids"):
    mjm = _scene(scene)
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=16, m=m)
    mjw.set_const(m, d)
    counts.append(mjw.last_launch_count())
  assert counts[0] == counts[1] == 8, counts


def test_gpu_set_const_replays_from_a_cuda_graph(built):
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import _lib

  mjm = _scene("humanoid")
  nworld = 64
  m = mjw.put_model(mjm, batch_sizes={"body_mass": nworld, **{f: nworld for f in set_const_scenes.OUTPUTS}})
  m.body_mass.mul_(torch.linspace(0.6, 1.5, nworld, device=m.body_mass.device)[:, None])
  d = mjw.make_data(mjm, nworld=nworld, m=m)
  start = {f: getattr(m, f).clone() for f in set_const_scenes.OUTPUTS}
  mjw.set_const(m, d)
  want = {f: getattr(m, f).clone() for f in set_const_scenes.OUTPUTS}
  want_mi = m.stat.meaninertia.clone()
  want_state = _restore_state(m, d)
  for f, v in start.items():
    getattr(m, f).copy_(v)
  L = _lib.lib()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    _lib.check(L.mjb_set_const(m._handle, d._handle, 7, 1, torch.cuda.current_stream().cuda_stream))
  for f, v in start.items():
    assert torch.equal(getattr(m, f), v), "capture must not execute"
  g.replay()
  torch.cuda.synchronize()
  for f, v in want.items():
    assert torch.equal(getattr(m, f), v), f
  assert torch.equal(m.stat.meaninertia, want_mi)
  for f, v in want_state.items():
    assert torch.equal(getattr(d, f), v), f


def test_gpu_set_const_end_to_end_scaled_masses(built):
  """Four worlds with per-world mass / inertia scales, set_const, forward + 4 steps: each world matches a model compiled with its masses."""
  import mujoco_warp_b200 as mjw

  mjm = _scene("humanoid")
  nworld, nstep = 4, 4
  scales = np.array([1.0, 1.35, 0.7, 1.8])
  m = mjw.put_model(mjm, batch_sizes={"body_mass": nworld, "body_inertia": nworld, **{f: nworld for f in set_const_scenes.OUTPUTS}})
  m.body_mass.mul_(torch.from_numpy(scales.astype(np.float32)).cuda()[:, None])
  m.body_inertia.mul_(torch.from_numpy(scales.astype(np.float32)).cuda()[:, None, None])
  d = mjw.make_data(mjm, nworld=nworld, nconmax=32, njmax=128, m=m)
  qpos, qvel, ctrl, warm = util.seeded_state(mjm, nworld)
  stale = {f: _np(getattr(m, f)) for f in ("body_subtreemass", "dof_invweight0", "body_invweight0")}
  mjw.set_const(m, d)

  def run(m, d, w):
    for name, val in (("qpos", qpos), ("qvel", qvel), ("ctrl", ctrl), ("qacc_warmstart", warm)):
      getattr(d, name).copy_(torch.from_numpy(np.asarray(val[w] if w is not None else val, dtype=np.float32)).reshape(getattr(d, name).shape))
    mjw.forward(m, d)
    out = [(_np(d.qacc), _np(d.qvel), _np(d.qpos))]
    for _ in range(nstep):
      mjw.step(m, d)
      out.append((_np(d.qacc), _np(d.qvel), _np(d.qpos)))
    return out

  got = run(m, d, None)
  dt = float(mjm.opt.timestep)
  for w, s in enumerate(scales):
    mv = copy.deepcopy(mjm)
    mv.body_mass = np.asarray(mjm.body_mass) * s
    mv.body_inertia = np.asarray(mjm.body_inertia) * s
    sub = np.array(mv.body_mass, dtype=np.float64)
    for b in range(mv.nbody - 1, 0, -1):
      sub[mv.body_parentid[b]] += sub[b]
    mv.body_subtreemass = sub
    mjcf._set_const(mv)
    mw_ = mjw.put_model(mv)
    dw = mjw.make_data(mv, nworld=1, nconmax=32, njmax=128, m=mw_)
    want = run(mw_, dw, slice(w, w + 1))
    for f in ("body_subtreemass", "dof_invweight0"):
      assert np.abs(stale[f][w] - np.asarray(getattr(mv, f))).max() > 1e-3 * np.abs(getattr(mv, f)).max() or s == 1.0, f
      close(f"w{w}/{f}", _np(getattr(m, f))[w], np.asarray(getattr(mv, f)), atol=2e-5 * np.abs(getattr(mv, f)).max(), rtol=2e-4)
    ascale = max(1.0, float(np.abs(want[0][0]).max()))
    close(f"w{w}/forward/qacc", got[0][0][w], want[0][0][0], atol=5e-3 * ascale)
    for k in range(1, nstep + 1):
      vtol = k * (dt * 5e-3 * ascale + 1e-4)
      close(f"w{w}/step{k}/qvel", got[k][1][w], want[k][1][0], atol=vtol, rtol=1e-3)
      close(f"w{w}/step{k}/qpos", got[k][2][w], want[k][2][0], atol=dt * vtol + 2e-5, rtol=1e-5)
