"""mjw.inverse on the GPU against the reference's own inverse dynamics (tests/golden/inverse_vectors.npz, tools/make_inverse_goldens.py).

Each scene is set to the fixture's state, `d.qacc` to the fixture's acceleration (forward's converged one, then a noisy one that puts rows
in every state; discrete-time under ENBL_INVDISCRETE for the `_disc` scenes), and `inverse` is compared at the tolerances
test_gpu_golden_pipeline.py uses for the same fields: constraint-row quantities within 5e-3 of the force scale, `solver_niter` exact,
row states exact off the knife edge (rows whose reference state flips under a 1e-6 relative nudge of qacc).  Worlds whose row count
differs from the reference's are skipped, as in the pipeline test, and at most a quarter of them may be.
"""
import os

import numpy as np
import pytest
import torch

from tests import util
from tests.test_oracle_golden_pipeline import load_scene

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inverse_vectors.npz")
DSBL_EULERDAMP, ENBL_INVDISCRETE = 1 << 15, 1 << 3


def _scene(name):
  base = name.replace("_disc_noeulerdamp", "").replace("_disc", "")
  mjm = load_scene(base)
  if "_disc" in name:
    mjm.opt.enableflags = int(mjm.opt.enableflags) | ENBL_INVDISCRETE
  if name.endswith("_noeulerdamp"):
    mjm.opt.disableflags = int(mjm.opt.disableflags) | DSBL_EULERDAMP
  return mjm


def _names():
  return sorted({k.split("/")[0] for k in np.load(GOLD).files})


@pytest.mark.parametrize("name", _names())
def test_gpu_inverse_matches_reference(built, name):
  import mujoco_warp_b200 as mjw

  g = np.load(GOLD)
  mjm = _scene(name)
  p = lambda k: g[f"{name}/{k}"]
  nworld = p("in/qpos").shape[0]
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, nconmax=int(p("in/nconmax")), njmax=int(p("in/njmax")), m=m)
  f32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
  d.qpos.copy_(f32(p("in/qpos"))); d.qvel.copy_(f32(p("in/qvel"))); d.qfrc_applied.copy_(f32(p("in/qfrc_applied")))
  if mjm.nu:
    d.ctrl.copy_(f32(p("in/ctrl")))
  if f"{name}/in/act" in g:
    d.act.copy_(f32(p("in/act")))
  if f"{name}/in/mocap_pos" in g:
    d.mocap_pos.copy_(f32(p("in/mocap_pos"))); d.mocap_quat.copy_(f32(p("in/mocap_quat")))
  nv = mjm.nv
  mjw.forward(m, d)  # as the fixture was made: forward, then inverse on the same Data
  # touch sensors: the reference's inverse adds them onto sensordata without clearing it (sensor_acc after forward's values), so its
  # touch entries depend on the Data's history; every other sensor is compared
  touch = np.zeros(int(mjm.nsensordata), bool)
  for i in range(int(mjm.nsensor)):
    if int(mjm.sensor_type[i]) == 0:
      touch[int(mjm.sensor_adr[i]) : int(mjm.sensor_adr[i]) + int(mjm.sensor_dim[i])] = True
  skipped = total = 0
  for kind in ("conv", "noisy"):
    q = lambda k: g[f"{name}/{kind}/{k}"]
    qacc = f32(q("in_qacc")).cuda()
    d.qacc.copy_(qacc)
    d.solver_niter.fill_(-1)
    mjw.inverse(m, d)
    torch.cuda.synchronize()
    assert torch.equal(d.qacc, qacc)
    assert (d.solver_niter.cpu().numpy() == 0).all()
    nefc, want_nefc = d.nefc.cpu().numpy().reshape(-1), q("nefc").reshape(-1)
    qfc_want, inv_want = q("qfrc_constraint").reshape(nworld, nv), q("qfrc_inverse").reshape(nworld, nv)
    scale = max(1.0, float(np.abs(inv_want).max()), float(np.abs(qfc_want).max()))
    got_inv, got_qfc = d.qfrc_inverse.cpu().numpy(), d.qfrc_constraint.cpu().numpy()
    got_ma = d.efc.Ma.cpu().numpy()
    force, state = d.efc.force.cpu().numpy(), d.efc.state.cpu().numpy()
    for w in range(nworld):
      total += 1
      if nefc[w] != want_nefc[w]:
        skipped += 1
        continue
      n = min(int(nefc[w]), d.njmax)
      util.assert_close(f"{kind} qfrc_inverse w{w}", got_inv[w], inv_want[w], atol=5e-3 * scale, rtol=0)
      util.assert_close(f"{kind} qfrc_constraint w{w}", got_qfc[w], qfc_want[w], atol=5e-3 * scale, rtol=0)
      util.assert_close(f"{kind} efc_Ma w{w}", got_ma[w], q("efc_Ma").reshape(nworld, -1)[w, :nv], atol=5e-3 * scale, rtol=0)
      knife = q("knife")[w, :n].astype(bool)
      want_st = q("efc_state")[w, :n]
      bad = (state[w, :n] != want_st) & ~knife
      assert not bad.any(), f"{kind} world {w}: row states differ at rows {np.nonzero(bad)[0]}: {state[w, :n][bad]} vs {want_st[bad]}"
      util.assert_close(f"{kind} efc_force w{w}", force[w, :n][~knife], q("efc_force")[w, :n][~knife], atol=5e-3 * scale, rtol=0)
    if mjm.nsensordata:
      sens = q("sensordata").reshape(nworld, -1)
      sens = sens[:, ~touch]
      util.assert_close(f"{kind} sensordata", d.sensordata.cpu().numpy()[:, ~touch], sens, atol=5e-3 * max(1.0, float(np.abs(sens).max())), rtol=0)
  assert skipped <= total // 4, f"{skipped} of {total} world-cases differ in nefc"
