"""The benchmark workload as benchmarked: humanoid, nworld = 8192, nconmax = 24, njmax = 64, squat keyframe, Halton ctrl noise,
CUDA-graph replay of the world-split pipeline -- 400 steps, i.e. into the regime where the humanoid has collapsed onto the floor
and rows are cut at njmax (the state bench.py times).  Every 20 steps the fp32 build of the oracle takes ONE step from the GPU's own
state (teacher forcing: a free-running comparison of two fp32 implementations of a contact-rich system diverges chaotically after a
few dozen steps, which says nothing about either) and must agree per world: exact nefc / ne / nf / nl, exact contact count,
exact overflow bits raised by the step, state within the fp32 band.  Contact make / break decisions sit at |dist - margin| ~ 1e-7
boundaries, so a handful of worlds per checkpoint may legitimately differ by one contact: worlds with a contact within 1e-6 of its margin
on either side may differ in up to 0.1 % of the worlds (at least 4), any other difference in up to 0.25 %.

Also covers the world-split pipeline (MJB_SPLIT = 1, 2, 3 on internal streams, plain launches and graph replay) on the same
state: per-world results must be bit-identical whatever the split (ADVICE r1: the default split was never tested)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu

NWORLD, NCONMAX, NJMAX = 8192, 24, 64
EDGE = 1e-6  # |dist - margin| of a contact whose make / break decision is a matter of fp32 rounding (a few ulp of a body position)


def _bench_state(mjw, mjm, m, nworld):
  from mujoco_warp_b200._src.mjcf import MjDataLite, reset_data_keyframe

  mjd = MjDataLite(mjm)
  reset_data_keyframe(mjm, mjd, 0)
  d = mjw.put_data(mjm, mjd, nworld=nworld, nconmax=NCONMAX, njmax=NJMAX, m=m)
  center = torch.from_numpy(np.asarray(mjd.ctrl, dtype=np.float32)).cuda()
  return d, center


@pytest.mark.parametrize("nworld,njmax,nsteps", [(NWORLD, NJMAX, 400), (1024, 40, 400)], ids=["bench_config", "njmax40_truncation"])
def test_bench_config_lockstep_vs_fp32_oracle(built, nworld, njmax, nsteps):
  """(8192, 64): the benchmark configuration.  (1024, 40): same run with a row capacity the collapsed humanoid exceeds, so that the
  njmax truncation path (rows cut, contact.efc_address = -1, NEFC overflow bit; constraint.py:2048,2712) is exercised in lockstep."""
  import mujoco_warp_b200 as mjw

  global NJMAX
  NWORLD_, NJMAX_SAVE = nworld, NJMAX
  NJMAX = njmax
  try:
    _lockstep(mjw, NWORLD_, njmax, nsteps)
  finally:
    NJMAX = NJMAX_SAVE


def _lockstep(mjw, NWORLD, njmax, nsteps):
  mjm = mjw.mjcf.load_any(util.HUMANOID)
  m = mjw.put_model(mjm)
  d, center = _bench_state(mjw, mjm, m, NWORLD)
  o = util.make_oracle(mjm, NWORLD, NCONMAX, njmax, dtype=np.float32)
  stream = torch.cuda.Stream()
  budget = max(2, NWORLD // 400)  # 0.25 % of the worlds per checkpoint (observed: up to 10 of 8192 while the humanoid is falling, step ~100)
  # worlds whose difference comes with a contact at its margin (below).  Observed on an H100 over the 20 checkpoints: at most 6 of 8192
  # worlds (step 99; 1-4 at ten others, none at the remaining nine) and 3 of 1024 with njmax 40 (steps 99 and 299), while the other
  # differences stayed at 0 of 8192 and at most 1 of 1024
  edge_budget = max(4, NWORLD // 1000)
  seen_overflow, max_nefc = 0, 0
  with torch.cuda.stream(stream):
    mjw.step(m, d)  # warm-up launch configures shared memory sizes before capture
    d2, _ = _bench_state(mjw, mjm, m, NWORLD)
    for n in ("qpos", "qvel", "ctrl", "qacc_warmstart", "time"):
      getattr(d, n).copy_(getattr(d2, n))
    d.overflow.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
      mjw.step(m, d)
    for i in range(nsteps):
      mjw.ctrl_noise(m, d, i, center)
      check = i % 20 == 19
      if check:
        stream.synchronize()
        state = {n: getattr(d, n).cpu().numpy().copy() for n in ("qpos", "qvel", "ctrl", "qacc_warmstart")}
        d.overflow.zero_()
      g.replay()
      if not check:
        continue
      stream.synchronize()
      o.set_state(**state)
      o.d["overflow"][:] = 0
      o.step()
      nacon = int(d.nacon.cpu()[0])
      wid = d.contact.worldid[:nacon].cpu().numpy()
      ncon_gpu = np.bincount(wid, minlength=NWORLD)
      # worlds with a contact within fp32 rounding of its margin on either side count against `edge_budget`, all others against `budget`
      edge = np.zeros(NWORLD, dtype=bool)
      np.logical_or.at(edge, wid, (d.contact.dist[:nacon] - d.contact.includemargin[:nacon]).abs().cpu().numpy() < EDGE)
      live = np.arange(o.d["con_dist"].shape[1])[None, :] < o.d["ncon"][:, None]
      edge |= (live & (np.abs(o.d["con_dist"] - o.d["con_includemargin"]) < EDGE)).any(axis=1)
      for f, gpu in (("nefc", d.nefc), ("ne", d.ne), ("nf", d.nf), ("nl", d.nl), ("contact count", ncon_gpu)):
        differ = (gpu.cpu().numpy() if isinstance(gpu, torch.Tensor) else gpu) != o.d["ncon" if f == "contact count" else f]
        bad, at_edge = int((differ & ~edge).sum()), int((differ & edge).sum())
        assert bad <= budget, f"step {i}: {f} differs in {bad} worlds without a contact at its margin (budget {budget})"
        assert at_edge <= edge_budget, f"step {i}: {f} differs in {at_edge} worlds with a contact at its margin (budget {edge_budget})"
      same = (d.nefc.cpu().numpy() == o.d["nefc"]) & (ncon_gpu == o.d["ncon"])
      # overflow bits of this step (njmax truncation -> NEFC ...); the line-search budget bit may differ at rounding level
      mask = ~int(mjw.OverflowType.LS_ITERATIONS)
      ovf_gpu, ovf_cpu = d.overflow.cpu().numpy() & mask, o.d["overflow"] & mask
      assert int((ovf_gpu != ovf_cpu)[same].sum()) == 0, f"step {i}: overflow bits differ"
      seen_overflow += int((ovf_gpu != 0).sum())
      max_nefc = max(max_nefc, int(d.nefc.max().cpu()))
      util.assert_close(f"qpos@{i}", d.qpos.cpu().numpy()[same], o.d["qpos"][same], atol=2e-4, rtol=2e-4)
      util.assert_close(f"qvel@{i}", d.qvel.cpu().numpy()[same], o.d["qvel"][same], atol=2e-2, rtol=1e-2)
      assert not np.isnan(d.qpos.cpu().numpy()).any()
  assert max_nefc >= 40, f"the run never reached the contact-rich regime (max nefc {max_nefc})"
  if njmax < 64:
    assert seen_overflow > 0, "the truncation variant never exceeded njmax"


SPLIT_SCRIPT = r"""
import os, sys, json
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import mujoco_warp_b200 as mjw
from mujoco_warp_b200._src.mjcf import MjDataLite, reset_data_keyframe
from tests import util
scene, nworld, graph = sys.argv[2], int(sys.argv[3]), sys.argv[4] == "1"
if scene == "humanoid":
  mjm = mjw.mjcf.load_any(util.HUMANOID); nconmax, njmax = 24, 64
else:
  mjm = mjw.mjcf.load_string(util.MIXED_XML.replace('<option timestep="0.004"', '<option integrator="RK4" timestep="0.004"')); nconmax, njmax = 32, 128
m = mjw.put_model(mjm)
qpos, qvel, ctrl, warm = util.seeded_state(mjm, nworld, key=0, seed=7, qpos_noise=0.01)
d = mjw.make_data(mjm, nworld=nworld, nconmax=nconmax, njmax=njmax, m=m)
f32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
def reset():
  d.qpos.copy_(f32(qpos)); d.qvel.copy_(f32(qvel)); d.qacc_warmstart.copy_(f32(warm)); d.time.zero_()
  if mjm.nu: d.ctrl.copy_(f32(ctrl))
reset()
stream = torch.cuda.Stream()
with torch.cuda.stream(stream):
  mjw.step(m, d)
  reset()
  if graph:
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
      mjw.step(m, d)
    for _ in range(6): g.replay()
  else:
    for _ in range(6): mjw.step(m, d)
  stream.synchronize()
n = int(d.nacon.cpu()[0])
wid = d.contact.worldid[:n].cpu().numpy()
order = np.lexsort((np.arange(n), wid))  # contacts grouped by world, pool order inside a world
np.savez(sys.argv[5], qpos=d.qpos.cpu().numpy(), qvel=d.qvel.cpu().numpy(), nefc=d.nefc.cpu().numpy(), force=d.efc.force.cpu().numpy(),
         ncon=np.bincount(wid, minlength=nworld), cdist=d.contact.dist[:n].cpu().numpy()[order], cgeom=d.contact.geom[:n].cpu().numpy()[order], niter=d.solver_niter.cpu().numpy())
"""


@pytest.mark.parametrize("scene", ["humanoid", "mixed_rk4"])
def test_world_split_pipeline_is_bit_identical(built, scene, tmp_path):
  """MJB_SPLIT is read when Data is finalised, so every variant runs in its own process."""
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  script = tmp_path / "split_run.py"
  script.write_text(SPLIT_SCRIPT)
  nworld = 2048
  outs = {}
  # the third knob is MJB_FORK: k_velocity on its own stream next to k_collision -> k_constraint (MJB_FORK=1) or the serial chain (default)
  for split, graph, fork in (("1", "0", "0"), ("1", "0", "1"), ("2", "0", "1"), ("3", "0", "1"), ("2", "1", "1"), ("3", "1", "1"), ("2", "1", "0")):
    out = tmp_path / f"s{split}g{graph}f{fork}.npz"
    env = dict(os.environ, MJB_SPLIT=split, MJB_FORK=fork)
    subprocess.check_call([sys.executable, str(script), root, scene, str(nworld), graph, str(out)], env=env)
    outs[(split, graph, fork)] = np.load(out)
  ref = outs[("1", "0", "0")]
  assert ref["nefc"].max() > 0 and ref["ncon"].max() > 0
  for key, got in outs.items():
    for f in ref.files:
      np.testing.assert_array_equal(got[f], ref[f], err_msg=f"MJB_SPLIT={key[0]} graph={key[1]} MJB_FORK={key[2]}: {f}")
  # and the unsplit run agrees with the oracle (fp32 build) on the integer outputs after the same 6 steps from the same state
  import mujoco_warp_b200 as mjw

  if scene == "humanoid":
    mjm = mjw.mjcf.load_any(util.HUMANOID); nconmax, njmax = 24, 64
  else:
    mjm = mjw.mjcf.load_string(util.MIXED_XML.replace('<option timestep="0.004"', '<option integrator="RK4" timestep="0.004"')); nconmax, njmax = 32, 128
  qpos, qvel, ctrl, warm = util.seeded_state(mjm, nworld, key=0, seed=7, qpos_noise=0.01)
  o = util.make_oracle(mjm, nworld, nconmax, njmax, dtype=np.float32)
  kw = dict(qpos=qpos.astype(np.float32), qvel=qvel.astype(np.float32), qacc_warmstart=warm.astype(np.float32))
  if mjm.nu:
    kw["ctrl"] = ctrl.astype(np.float32)
  o.set_state(**kw)
  for _ in range(6):
    o.step()
  bad = int((ref["nefc"] != o.d["nefc"]).sum())
  assert bad <= max(2, nworld // 100), bad  # six free-running steps: make / break decisions at rounding-level boundaries
  util.assert_close("qpos vs oracle", ref["qpos"], o.d["qpos"], atol=2e-3, rtol=2e-3)
