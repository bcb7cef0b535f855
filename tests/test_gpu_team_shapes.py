"""The team kernels (k_position, k_velocity, k_velocity_fluid) at 8, 16 and 32 lanes per world and in every shared-memory layout
regime, held to the fp64 oracle, to backward-error bounds, to the stage-by-stage API and to themselves across world orders.

Each scene of tests/team_scenes.py runs at 1 world, at a count that leaves a partial last warp group and at one that leaves a
partial last block (the idle teams of a partial group recompute the last valid world and store nothing; the bulk copies fall back
to lane loops).  The launch shape that ran is read back from `team_residency(m, d, shapes=True)` and collected, and the last test
checks that every instance ran at every lane count.  Warps per block: small world counts tie every choice, and ties go to two-warp
blocks; one-warp blocks need more worlds than fit on the SMs at once, and `test_one_warp_blocks_at_many_worlds` reaches them.
Four-warp blocks are not reachable with these scenes on an H100: team_shape picks them only when they fit more warps on an SM than
two-warp blocks do, and at 8 lanes per world the registers (k_velocity's instances use about 128 per thread, k_position's 64) cap
both at the same warps per SM, while at 16 and 32 lanes four of these worlds' warps exceed a block's 200 KB or fit no better.
"""
import os

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import mjcf
from tests import team_scenes as T
from tests import util
from tests.test_gpu_golden_pipeline import close

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NWORLDS = (1, 5, 11)
NCONMAX, NJMAX = 4, 8
BAND = 5e-4  # the smooth-field band of the other parity tests (test_gpu_parity.py, smooth_test.py:32-38 of the reference)
TENDON_FIELDS = ("ten_length", "ten_J", "ten_velocity")
STAGES = ("kinematics", "com_pos", "camlight", "crb", "factor_m", "transmission", "com_vel", "passive", "rne", "fwd_actuation", "fwd_acceleration")
# Backward-error constant: the bounds below are c * n * eps32 * (...).  Cholesky's rounding-error analysis gives
# |U^T U - M| <= gamma_{n+1} |U^T| |U| and, for the solve, (M + dM) x = b with |dM| <= gamma_{3n+1} |U^T| |U| (Higham, Accuracy and
# Stability of Numerical Algorithms, 2nd ed., Thms 10.3 and 10.4), gamma_k = k eps / (1 - k eps).  c = 4 covers the 3n + 1 of the solve,
# the rounding of qfrc_smooth itself and |U^T| |U| <= |M|-sized terms (Cauchy-Schwarz on the columns of U); a wrong entry of the
# factor or a wrong right-hand side is off by O(1) relative, many orders above it.
C_BACKWARD = 4.0
EPS32 = float(np.finfo(np.float32).eps)

SHAPES = []  # (kernel, instance, lpw, wpb, scene, nworld) of every launch shape that ran in this module


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


@pytest.fixture(scope="module")
def models(built):
  import mujoco_warp_b200 as mjw

  out = {}
  for name, (xml, *_rest) in T.SCENES.items():
    mjm = mjcf.load_string(xml)
    out[name] = (mjw, mjm, mjw.put_model(mjm))
  return out


def _inputs(mjm, nworld, seed):
  """Seeded fp32-representable state, ctrl, and applied forces: xfrc_applied only in every other world (teams of one warp differ)."""
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld, key=None, seed=seed, qpos_noise=0.1, qvel_noise=0.3, ctrl_noise=0.8, exact_world0=False)
  rng = np.random.default_rng(seed + 1)
  xfrc = np.zeros((nworld, mjm.nbody, 6))
  moving = np.nonzero(np.asarray(mjm.body_weldid) != 0)[0]
  xfrc[1::2, moving[:: max(1, len(moving) // 7)]] = rng.uniform(-0.5, 0.5, (len(range(1, nworld, 2)), len(moving[:: max(1, len(moving) // 7)]), 6))
  qapp = 0.1 * rng.uniform(-1, 1, (nworld, mjm.nv))
  f32 = lambda a: a.astype(np.float32)
  return dict(qpos=f32(qpos), qvel=f32(qvel), ctrl=f32(ctrl), xfrc_applied=f32(xfrc), qfrc_applied=f32(qapp))


def _data(mjw, mjm, m, inp):
  nworld = inp["qpos"].shape[0]
  d = mjw.make_data(mjm, nworld=nworld, nconmax=NCONMAX, njmax=NJMAX, m=m)
  for k, v in inp.items():
    getattr(d, k).copy_(torch.from_numpy(v).reshape(getattr(d, k).shape))
  return d


def _record(mjw, m, d, scene):
  sh = mjw.team_residency(m, d, shapes=True)
  for kernel, s in sh.items():
    assert s["worlds_per_sm"] > 0, (kernel, s)
    SHAPES.append((kernel, s["instance"], s["lpw"], s["wpb"], scene, d.nworld))
  return sh


def _outputs(mjm, d):
  names = util.SMOOTH_FIELDS + ["site_xpos", "site_xmat", "qacc"] + (list(TENDON_FIELDS) if mjm.ntendon else [])
  return {n: _np(getattr(d, n)) for n in names}


def _trees(mjm):
  """(first dof, dofs, qLD offset) of every kinematic tree."""
  off, out = 0, []
  for a, n in zip(mjm.tree_dofadr, mjm.tree_dofnum):
    out.append((int(a), int(n), off))
    off += int(n) * int(n)
  return out


def _dense_m(mjm, Mw):
  """One world's M (CSR lower triangle, M_rowadr / M_colind) as a dense symmetric nv x nv matrix."""
  nv = mjm.nv
  A = np.zeros((nv, nv))
  for i in range(nv):
    for e in range(mjm.M_rowadr[i], mjm.M_rowadr[i] + mjm.M_rownnz[i]):
      A[i, mjm.M_colind[e]] = A[mjm.M_colind[e], i] = Mw[e]
  return A


def backward_errors(mjm, M, qLD, qacc_smooth, qfrc_smooth):
  """Worst ratio, over worlds and trees, of each backward error to its bound c n eps32 (...), all in fp64 from the given fp32 outputs:
  "factor": |U^T U - M| / (|U^T| |U|) per tree; "solve": |M qacc_smooth - qfrc_smooth| / (|M| |qacc_smooth| + |qfrc_smooth|)."""
  worst = {"factor": 0.0, "solve": 0.0}
  for w in range(M.shape[0]):
    A = _dense_m(mjm, M[w])
    for a, n, off in _trees(mjm):
      U = qLD[w, off : off + n * n].reshape(n, n)
      assert not np.tril(U, -1).any(), "qLD: nonzero below the diagonal"
      Mt = A[a : a + n, a : a + n]
      bound = C_BACKWARD * n * EPS32 * (np.abs(U).T @ np.abs(U)) + 1e-30
      worst["factor"] = max(worst["factor"], float((np.abs(U.T @ U - Mt) / bound).max()))
      x, f = qacc_smooth[w, a : a + n], qfrc_smooth[w, a : a + n]
      bound = C_BACKWARD * n * EPS32 * (np.abs(Mt) @ np.abs(x) + np.abs(f)) + 1e-30
      worst["solve"] = max(worst["solve"], float((np.abs(Mt @ x - f) / bound).max()))
  return worst


@pytest.mark.parametrize("nworld", NWORLDS)
@pytest.mark.parametrize("scene", sorted(T.SCENES))
def test_scene(models, scene, nworld):
  """Shape, oracle, backward error, stages and world independence of one scene at one world count."""
  mjw, mjm, m = models[scene]
  _, _, pos_lanes, vel_lanes, instance = T.SCENES[scene]
  inp = _inputs(mjm, nworld, seed=100 + nworld)
  d = _data(mjw, mjm, m, inp)
  sh = _record(mjw, m, d, scene)
  assert (sh["position"]["lpw"], sh["velocity"]["lpw"], sh["velocity"]["instance"]) == (pos_lanes, vel_lanes, instance), sh
  mjw.forward(m, d)
  torch.cuda.synchronize()
  got = _outputs(mjm, d)
  assert int(d.nefc.cpu().max()) == 0

  # backward error of the factor and the solve, from the kernel's own outputs
  worst = backward_errors(mjm, got["M"].reshape(nworld, -1), got["qLD"].reshape(nworld, -1), got["qacc_smooth"], got["qfrc_smooth"])
  for k, v in worst.items():
    assert v <= 1.0, f"{scene} nworld={nworld}: {k} backward error is {v:.3g} x its bound"

  # the fp64 oracle on the same fp32-rounded inputs
  if scene not in T.ILL_CONDITIONED:
    o = util.make_oracle(mjm, nworld, NCONMAX, NJMAX)
    o.set_state(qpos=inp["qpos"], qvel=inp["qvel"], ctrl=inp["ctrl"])
    o.d["xfrc_applied"][:] = inp["xfrc_applied"]
    o.d["qfrc_applied"][:] = inp["qfrc_applied"]
    o.forward()
    for name, v in got.items():
      if name == "qacc":
        continue
      util.assert_close(f"{scene}/{nworld}/{name}", v.reshape(o.d[name].shape), o.d[name], atol=BAND, rtol=BAND)

  # the public stages one by one: bit-identical to the fused forward (actuator / tendon velocities are fwd_velocity's, an input here)
  d2 = _data(mjw, mjm, m, inp)
  d2.actuator_velocity.copy_(d.actuator_velocity)
  if mjm.ntendon:
    d2.ten_velocity.copy_(d.ten_velocity)
  for fn in STAGES:
    getattr(mjw, fn)(m, d2)
  torch.cuda.synchronize()
  for name, v in _outputs(mjm, d2).items():
    if name != "qacc":
      np.testing.assert_array_equal(v, got[name], err_msg=f"{scene}/{nworld}: stages vs forward: {name}")

  # world independence: reversed world order, and every world alone, give the same bits
  if nworld > 1:
    perm = np.arange(nworld)[::-1].copy()
    d3 = _data(mjw, mjm, m, {k: v[perm] for k, v in inp.items()})
    mjw.forward(m, d3)
    torch.cuda.synchronize()
    for name, v in _outputs(mjm, d3).items():
      np.testing.assert_array_equal(v, got[name][perm], err_msg=f"{scene}/{nworld}: reversed worlds: {name}")
    for w in sorted({0, 1, nworld - 1}):
      d1 = _data(mjw, mjm, m, {k: v[w : w + 1] for k, v in inp.items()})
      mjw.forward(m, d1)
      torch.cuda.synchronize()
      for name, v in _outputs(mjm, d1).items():
        np.testing.assert_array_equal(v[0], got[name][w], err_msg=f"{scene}/{nworld}: world {w} alone: {name}")


def test_world_counts_leave_partial_groups_and_blocks():
  """Every scene's counts include one with a partial last warp group (where a group has more than one world) and one with a partial
  last block, for both kernels, in the shapes that actually ran."""
  ran = {}
  for kernel, _inst, lpw, wpb, scene, nworld in SHAPES:
    ran.setdefault((scene, kernel), []).append((lpw, wpb, nworld))
  assert len(ran) == 2 * len(T.SCENES), sorted(ran)
  for key, runs in ran.items():
    G = 32 // runs[0][0]
    if G > 1:
      assert any(n % G for _, _, n in runs), (key, runs)
    assert any(-(-n // G) % wpb for _, wpb, n in runs), (key, runs)


@pytest.mark.parametrize("scene", sorted(T.FLUID))
def test_fluid_at_every_lane_count(built, scene):
  """k_velocity_fluid at 8, 16 and 32 lanes: tests/fluid_scenes.py's chain and ellipsoid scenes padded with static bodies after their
  own, held to the reference's forward values (tests/golden/fluid_*.npz) on the original dofs and bodies at test_gpu_fluid's bands."""
  import mujoco_warp_b200 as mjw

  base, xml, _regime, lpw, nbody0 = T.FLUID[scene]
  g = np.load(os.path.join(GOLD, f"fluid_{base}.npz"))
  mjm = mjcf.load_string(xml)
  m = mjw.put_model(mjm)
  nworld = g["in/qpos"].shape[0]
  d = mjw.make_data(mjm, nworld=nworld, nconmax=int(g["in/nconmax"]), njmax=int(g["in/njmax"]), m=m)
  f32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
  d.qpos.copy_(f32(g["in/qpos"])); d.qvel.copy_(f32(g["in/qvel"])); d.qacc_warmstart.copy_(f32(g["in/qacc_warmstart"]))
  if mjm.nu:
    d.ctrl.copy_(f32(g["in/ctrl"]))
  sh = _record(mjw, m, d, f"fluid_{scene}")
  assert (sh["velocity"]["instance"], sh["velocity"]["lpw"]) == ("fluid", lpw), sh
  mjw.forward(m, d)
  torch.cuda.synchronize()
  for f in ("qfrc_fluid", "qfrc_passive", "qacc_smooth", "cvel", "qfrc_bias"):
    want = g[f"forward/{f}"].reshape(nworld, -1)
    got = _np(getattr(d, f))
    if f == "cvel":
      assert not got[:, nbody0:].any()  # static bodies do not move
      got = got[:, :nbody0]
    close(f"{scene}/forward/{f}", got.reshape(nworld, -1), want, atol=5e-4 * max(1.0, float(np.abs(want).max())))
  scale = max(1.0, float(np.abs(g["forward/qacc"]).max()))
  close(f"{scene}/forward/qacc", _np(d.qacc), g["forward/qacc"], atol=5e-3 * scale)


def test_one_warp_blocks_at_many_worlds(models):
  """One-warp blocks: team_shape picks them only when they need fewer residency rounds than two-warp blocks, which takes more worlds
  than fit on the SMs at once (the wide scene's 60-70 KB worlds: three one-warp blocks per SM, one two-warp block).  Its worlds
  match the same worlds run alone."""
  mjw, mjm, m = models["wide"]
  nworld = 600
  inp = _inputs(mjm, nworld, seed=7)
  d = _data(mjw, mjm, m, inp)
  sh = _record(mjw, m, d, "wide")
  assert sh["position"]["wpb"] == sh["velocity"]["wpb"] == 1, sh
  mjw.forward(m, d)
  torch.cuda.synchronize()
  got = _outputs(mjm, d)
  for w in (0, 1, nworld - 1):
    d1 = _data(mjw, mjm, m, {k: v[w : w + 1] for k, v in inp.items()})
    mjw.forward(m, d1)
    torch.cuda.synchronize()
    for name, v in _outputs(mjm, d1).items():
      np.testing.assert_array_equal(v[0], got[name][w], err_msg=f"wide/{nworld}: world {w} alone: {name}")


def test_every_instance_ran_at_every_lane_count():
  ran = {(k, i, l) for k, i, l, *_ in SHAPES}
  want = {("position", "plain", l) for l in (8, 16, 32)} | {("velocity", i, l) for i in ("plain", "pext", "fluid") for l in (8, 16, 32)}
  assert want <= ran, sorted(want - ran)
  assert {w for *_, w, _s, _n in SHAPES} == {1, 2}  # four-warp blocks: see the module docstring
  rows = sorted({(k, i, l, w, s) for k, i, l, w, s, _ in SHAPES})
  print("\nkernel | instance | lanes | warps/block | scene")
  for r in rows:
    print(" | ".join(map(str, r)))
