"""make_constraint (k_constraint, and k_efc_csr for sparse models) alone, against tests/constraint_oracle.py fed the GPU's own inputs.

Each case runs forward(), poisons every output of the stage (efc float fields NaN, efc type / id, the row counts, contact.efc_address
and the CSR arrays a sentinel), calls make_constraint alone and compares world by world with the fp64 restatement evaluated on the
positions, velocities and contacts read back from Data.  Every row below min(nefc, njmax) must have been written.

Tolerance: |got - want| <= 64 eps32 magnitude, magnitude being the sum of the absolute values of the terms that formed the value
(propagated through every operation by the oracle).  The kernel evaluates the same expressions as the oracle, each fp32 operation
adding at most eps32 times the magnitude of its operands; the longest chains (the weld's rotational rows: a quaternion product of a
quaternion product, summed over dofs, then efc_row's impedance and reference) are a few tens of operations deep, and powf / atan2f
add a few ulp.  64 covers that depth with room, and is still ~1e-5 of the magnitude: a dropped term, a wrong sign, a wrong world's
parameter or a missing factor moves a value by a sizeable fraction of it.

Activation decisions sit at least 1e-5 from their thresholds in every scene (the oracle asserts it), so fp32 and fp64 take the same
branches and the comparison is deterministic."""

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf
from tests import constraint_oracle as co
from tests import util

pytestmark = pytest.mark.gpu

EPS32 = float(np.finfo(np.float32).eps)
TOL = 64 * EPS32
POISON = -7777


def selected(m):
  """CPU restatement of launch_constraint's instantiation choice <EQ, BAT>: EQ for equalities, limited ball joints or tendons, BAT when any
  per-world float field holds more than one entry."""
  from mujoco_warp_b200._src import io

  bat = any(isinstance(getattr(m, n, None), torch.Tensor) and getattr(m, n).dim() >= 1 and getattr(m, n).shape[0] > 1
            for n in io._FLOAT_FIELDS + list(io._BATCHABLE_EXTRA))
  return (m.neq > 0 or len(m._tables["jnt_limited_ball_adr"]) > 0 or m.ntendon > 0, bat)


def poison(d, sparse):
  for f in ("pos", "margin", "D", "vel", "aref", "frictionloss"):
    getattr(d.efc, f).fill_(float("nan"))
  (d.efc.J_dense if sparse else d.efc.J).fill_(float("nan"))
  d.efc.type.fill_(POISON); d.efc.id.fill_(POISON)
  for f in ("ne", "nf", "nl", "nefc"):
    getattr(d, f).fill_(POISON)
  d.contact.efc_address.fill_(POISON)
  if sparse:
    d.efc.J.fill_(float("nan"))
    for f in ("J_rownnz", "J_rowadr", "J_colind"):
      getattr(d.efc, f).fill_(POISON)


def world_inputs(mjm, d, w):
  g = lambda f: getattr(d, f)[w].cpu().numpy().astype(np.float64)
  st = {f: g(f) for f in ("qpos", "qvel", "xpos", "xmat", "xquat", "cdof", "cvel", "cdof_dot", "subtree_com")}
  st["ten_length"] = g("ten_length") if mjm.ntendon else np.zeros(0)
  st["eq_active"] = d.eq_active[w].cpu().numpy() if int(getattr(mjm, "neq", 0)) else np.zeros(0)
  ids = util.world_contacts(d, w)
  st["con_id"] = ids
  c = d.contact
  for f in ("dist", "includemargin", "dim", "geom", "pos", "frame", "friction", "solref", "solreffriction", "solimp"):
    x = getattr(c, f)[torch.as_tensor(ids, dtype=torch.long, device=c.dist.device)].cpu().numpy()
    st["con_" + f] = x.astype(np.float64) if x.dtype.kind == "f" else x
  return st


def close(name, got, want, mag):
  got = np.asarray(got, dtype=np.float64)
  assert np.isfinite(got).all(), f"{name}: unwritten (NaN) entries at {np.argwhere(~np.isfinite(got))[:4].tolist()}"
  err = np.abs(got - want)
  bad = err > TOL * mag + 1e-30
  assert not bad.any(), f"{name}: at {np.argwhere(bad)[0].tolist()}: got {got[bad][0]:.9g}, want {want[bad][0]:.9g}, magnitude {mag[bad][0]:.3g}"


def run(mjm, nworld, njmax, nconmax=32, qpos=None, qvel=None, batched=None, eq_active=None, disable=0, njmax_nnz=None, expect=None):
  """forward, poison, make_constraint, compare every world with the oracle; returns (m, d)."""
  import mujoco_warp_b200 as mjw

  batched = batched or {}
  m = mjw.put_model(mjm, batch_sizes={n: x.shape[0] for n, x in batched.items()})
  for n, x in batched.items():
    getattr(m, n).copy_(torch.as_tensor(np.asarray(x, dtype=np.float32)))
  if expect is not None:
    assert selected(m) == expect, f"k_constraint<EQ, BAT> = {selected(m)}, the case is meant for {expect}"
  d = mjw.make_data(mjm, nworld=nworld, nconmax=nconmax, njmax=njmax, njmax_nnz=njmax_nnz, m=m)
  if qpos is not None:
    d.qpos.copy_(torch.as_tensor(np.asarray(qpos, dtype=np.float32)))
  if qvel is not None:
    d.qvel.copy_(torch.as_tensor(np.asarray(qvel, dtype=np.float32)))
  if eq_active is not None:
    d.eq_active.copy_(torch.as_tensor(np.asarray(eq_active)).to(d.eq_active.dtype))
  mjw.forward(m, d)
  if disable:  # after forward(): make_constraint alone runs with the flag
    m.opt.disableflags = int(m.opt.disableflags) | disable
    mjm.opt.disableflags = int(mjm.opt.disableflags) | disable
  sparse = hasattr(d.efc, "J_dense")
  poison(d, sparse)
  mjw.make_constraint(m, d)
  torch.cuda.synchronize()
  nv = mjm.nv
  J = (d.efc.J_dense if sparse else d.efc.J).cpu().numpy()
  cnt = {f: getattr(d, f).cpu().numpy().reshape(-1) for f in ("ne", "nf", "nl", "nefc")}
  efc = {f: getattr(d.efc, f).cpu().numpy() for f in ("pos", "margin", "D", "vel", "aref", "frictionloss", "type", "id")}
  adr = d.contact.efc_address.cpu().numpy()
  if sparse:
    Jsp, rownnz, rowadr, colind = d.efc.J.cpu().numpy()[:, 0], d.efc.J_rownnz.cpu().numpy(), d.efc.J_rowadr.cpu().numpy(), d.efc.J_colind.cpu().numpy()[:, 0]
    ovf = d.overflow.cpu().numpy()
  total, Rs = 0, []
  for w in range(nworld):
    R = co.make_constraint(co.world_model(mjm, batched, w), world_inputs(mjm, d, w), njmax)
    for f in ("ne", "nf", "nl", "nefc"):
      assert int(cnt[f][w]) == getattr(R, f), f"w{w} {f}: {int(cnt[f][w])} vs {getattr(R, f)}"
    nr = min(R.nefc, njmax)
    total += nr
    Rs.append(R)
    a = co.arrays(R, nv)
    np.testing.assert_array_equal(efc["type"][w, :nr], a["type"][:nr], err_msg=f"w{w} efc.type")
    np.testing.assert_array_equal(efc["id"][w, :nr], a["id"][:nr], err_msg=f"w{w} efc.id")
    close(f"w{w} efc.J", J[w, :nr, :nv], a["J"][:nr], a["J_mag"][:nr])
    for f in ("pos", "margin", "D", "vel", "aref", "frictionloss"):
      close(f"w{w} efc.{f}", efc[f][w, :nr], a[f][:nr], a[f + "_mag"][:nr])
    for i, cid in enumerate(world_inputs(mjm, d, w)["con_id"]):  # the addresses of an active contact's rows (-1 past njmax)
      ndim = sum(1 for r in R.rows if r["type"] >= C.CNSTR_CONTACT_FRICTIONLESS and r["id"] == cid)
      np.testing.assert_array_equal(adr[cid, :ndim], R.efc_address[i, :ndim], err_msg=f"w{w} contact {cid} efc_address")
    if sparse:
      nnz, radr, cols, vals, over = co.csr(co.world_model(mjm, batched, w), R, njmax, d.njmax_nnz)
      np.testing.assert_array_equal(rownnz[w, :nr], np.where(nnz < 0, POISON, nnz), err_msg=f"w{w} J_rownnz")
      fit = radr >= 0
      np.testing.assert_array_equal(rowadr[w, :nr], np.where(fit, radr, POISON), err_msg=f"w{w} J_rowadr (a row that does not fit has none)")
      assert bool(ovf[w] & C.OVF_NJMAX_NNZ) == over, f"w{w}: OVF_NJMAX_NNZ {bool(ovf[w] & C.OVF_NJMAX_NNZ)}, want {over}"
      for r in np.nonzero(fit)[0]:
        sl = slice(radr[r], radr[r] + nnz[r])
        np.testing.assert_array_equal(colind[w, sl], cols[r], err_msg=f"w{w} row {r} J_colind")
        close(f"w{w} row {r} CSR values", Jsp[w, sl], np.array([x.v for x in vals[r]]), np.array([x.m for x in vals[r]]))
  assert total > 0 or disable & C.DSBL_CONSTRAINT
  return m, d, Rs


def _lowered_humanoid(nworld, seed=7):
  mjm = mjcf.load_any(util.HUMANOID)
  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=0, seed=seed, qpos_noise=0.003, qvel_noise=0.3, exact_world0=False)
  qpos[:, :7] = mjm.key_qpos[0][:7]
  qpos[:, 2] -= 0.002 + 0.0005 * np.arange(nworld)  # feet clearly in the floor: no contact near its activation threshold
  return mjm, qpos, qvel


@pytest.mark.parametrize("nworld", [1, 5, 33])
def test_humanoid(built, nworld):
  mjm, qpos, qvel = _lowered_humanoid(nworld)
  run(mjm, nworld, 128, 24, qpos, qvel, expect=(False, False))


def test_humanoid_batched(built):
  """Per-world impedance parameters: solimp power 1, 2 and 3 (the general powf path), negative (direct) solref, scaled invweights."""
  nworld = 33
  mjm, qpos, qvel = _lowered_humanoid(nworld)
  w = np.arange(nworld)
  solimp = np.repeat(np.asarray(mjm.jnt_solimp, dtype=np.float64)[None], nworld, 0)
  solimp[:, :, 4] = np.asarray([1.0, 2.0, 3.0])[w % 3][:, None]
  solimp[:, :, 2] = 0.2  # limit rows within the impedance width, so the power matters
  solref = np.repeat(np.asarray(mjm.jnt_solref, dtype=np.float64)[None], nworld, 0)
  solref[w % 4 == 3] = (-3000.0, -40.0)
  inv = np.asarray(mjm.body_invweight0, dtype=np.float64)[None] * (1.0 + 0.05 * w)[:, None, None]
  qpos[:, 7:] += 0.4 * np.sign(np.random.default_rng(3).uniform(-1, 1, qpos[:, 7:].shape))  # push joints into their limits
  run(mjm, nworld, 192, 24, qpos, qvel, batched={"jnt_solimp": solimp, "jnt_solref": solref, "body_invweight0": inv}, expect=(False, True))


def _equality(nworld, seed=11):
  mjm = mjcf.load_string(util.EQUALITY_XML)
  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=0, seed=seed, qpos_noise=0.02, qvel_noise=0.5, exact_world0=False)
  return mjm, qpos, qvel


@pytest.mark.parametrize("nworld", [1, 5])
def test_equality_sparse(built, nworld):
  """Connect, weld (torquescale, Jdot v with nonzero cvel), joint equalities with and without joint2, the ball limit; nv = 33, so the
  CSR view is checked too."""
  mjm, qpos, qvel = _equality(nworld)
  run(mjm, nworld, 64, 16, qpos, qvel, expect=(True, False))


def test_equality_active_per_world(built):
  mjm, qpos, qvel = _equality(5)
  act = np.ones((5, mjm.neq), dtype=bool)
  for w in range(5):
    act[w, w % mjm.neq] = False
    act[w, (w + 3) % mjm.neq] = w % 2 == 0
  run(mjm, 5, 64, 16, qpos, qvel, eq_active=act, expect=(True, False))


def test_equality_batched(built):
  nworld = 33
  mjm, qpos, qvel = _equality(nworld)
  w = np.arange(nworld)
  eq_solref = np.repeat(np.asarray(mjm.eq_solref, dtype=np.float64).reshape(1, mjm.neq, 2), nworld, 0)
  eq_solref[w % 3 == 1] = (-2000.0, -30.0)
  eq_solimp = np.repeat(np.asarray(mjm.eq_solimp, dtype=np.float64).reshape(1, mjm.neq, 5), nworld, 0)
  eq_solimp[:, :, 2] = 0.5
  eq_solimp[:, :, 4] = np.asarray([1.0, 2.0, 2.5])[w % 3][:, None]
  inv = np.asarray(mjm.body_invweight0, dtype=np.float64)[None] * (1.0 + 0.03 * w)[:, None, None]
  run(mjm, nworld, 64, 16, qpos, qvel, batched={"eq_solref": eq_solref, "eq_solimp": eq_solimp, "body_invweight0": inv}, expect=(True, True))


@pytest.mark.parametrize("njmax", [2, 3, 4, 9, 12, 13])
def test_equality_blocks_at_njmax(built, njmax):
  """Rows: connect 0-2 and 3-5, welds 6-11 and 12-17.  njmax 3 / 12 end a connect / weld block exactly at njmax, 2 / 4 / 9 / 13 cut one:
  every row below njmax is written, the counts are the untruncated ones."""
  mjm, qpos, qvel = _equality(3)
  _, _, Rs = run(mjm, 3, njmax, 16, qpos, qvel)
  for R in Rs:  # the layout the parameters are chosen for: equalities 0 and 4 (connect), 1 and 6 (weld)
    assert [r["id"] for r in R.rows[:18]] == [0] * 3 + [4] * 3 + [1] * 6 + [6] * 6 and R.nefc > njmax


@pytest.mark.parametrize("jac", ["dense", "sparse"])
def test_tendons(built, jac):
  """Tendon friction, tendon limits (both sides), tendon equalities with a polynomial in a second tendon; jacobian="sparse" writes their
  CSR rows from ten_J_colind."""
  mjm = mjcf.load_string(util.tendon_xml().replace('<option timestep="0.004"', f'<option jacobian="{jac}" timestep="0.004"'))
  qpos, qvel, _, _ = util.seeded_state(mjm, 5, key=0, seed=5, qpos_noise=0.05, qvel_noise=0.5, exact_world0=False)
  qpos[:, 0] = np.where(np.arange(5) % 2 == 0, 1.2, -1.6)  # t_lim = (a0 - a1) / 2 beyond either end of its range
  act = np.ones((5, mjm.neq), dtype=bool)
  run(mjm, 5, 64, 16, qpos, qvel, eq_active=act, expect=(True, False))


def test_tendons_csr_overflow(built):
  """njmax_nnz edges on the sparse tendon scene: at the exact size every row fits; one less and the last row is counted (rownnz) but not
  placed (no rowadr), with OVF_NJMAX_NNZ raised."""
  mjm = mjcf.load_string(util.tendon_xml().replace('<option timestep="0.004"', '<option jacobian="sparse" timestep="0.004"'))
  qpos, qvel, _, _ = util.seeded_state(mjm, 1, key=0, seed=5, qpos_noise=0.05, qvel_noise=0.5, exact_world0=False)
  qpos[:, 0] = 1.2
  act = np.ones((1, mjm.neq), dtype=bool)
  _, d, _ = run(mjm, 1, 64, 16, qpos, qvel, eq_active=act)
  nr = int(d.nefc.cpu()[0])
  need = int(d.efc.J_rowadr.cpu()[0, nr - 1] + d.efc.J_rownnz.cpu()[0, nr - 1])
  run(mjm, 1, 64, 16, qpos, qvel, eq_active=act, njmax_nnz=need)
  run(mjm, 1, 64, 16, qpos, qvel, eq_active=act, njmax_nnz=need - 1)


@pytest.mark.parametrize("cone", ["pyramidal", "elliptic"])
def test_mixed(built, cone):
  """Contacts of condim 1, 3, 4 and 6, dof friction loss, slide / hinge limits; elliptic with impratio 2."""
  x = util.MIXED_XML if cone == "pyramidal" else util.MIXED_XML.replace('<option timestep="0.004"', '<option cone="elliptic" impratio="2" timestep="0.004"')
  mjm = mjcf.load_string(x)
  qpos, qvel, _, _ = util.seeded_state(mjm, 5, key=0, seed=1234, qpos_noise=0.01, qvel_noise=0.3, exact_world0=False)
  run(mjm, 5, 128, 32, qpos, qvel)


def test_rake_more_than_32_contacts(built):
  """40 contacts in one world (two batches of the contact-row builder), condim 1, 3 and 4 mixed; then njmax cuts a contact's rows."""
  mjm = mjcf.load_string(util.rake_xml().replace('<body name="rake" pos="0 0 0.049">', '<body name="rake" pos="0 0 0.0487">'))
  _, _, Rs = run(mjm, 2, 256, 64)
  assert all(len(R.efc_address) > 32 for R in Rs)
  rows = Rs[0].rows  # njmax one row into world 0's first contact of 6 rows past row 64: its rows straddle njmax
  njmax = next(r + 1 for r in range(64, len(rows) - 5) if rows[r]["type"] >= C.CNSTR_CONTACT_FRICTIONLESS and rows[r]["id"] != rows[r - 1]["id"]
               and all(x["id"] == rows[r]["id"] for x in rows[r : r + 6]))
  _, _, Rs = run(mjm, 2, njmax, 64)
  assert rows[njmax - 1]["id"] == rows[njmax]["id"] and Rs[0].nefc > njmax


def test_nefc_equals_njmax(built):
  mjm, qpos, qvel = _lowered_humanoid(1)
  _, d, _ = run(mjm, 1, 128, 24, qpos, qvel)
  n = int(d.nefc.cpu()[0])
  run(mjm, 1, n, 24, qpos, qvel)
  run(mjm, 1, n - 1, 24, qpos, qvel)


@pytest.mark.parametrize("flag", ["CONSTRAINT", "EQUALITY", "FRICTIONLOSS", "LIMIT", "CONTACT", "REFSAFE"])
def test_disable_flags(built, flag):
  mjm = mjcf.load_string(util.MIXED_XML)
  qpos, qvel, _, _ = util.seeded_state(mjm, 3, key=0, seed=1234, qpos_noise=0.01, qvel_noise=0.3, exact_world0=False)
  run(mjm, 3, 128, 32, qpos, qvel, disable=getattr(C, "DSBL_" + flag))
  mjm, qpos, qvel = _equality(3)
  run(mjm, 3, 64, 16, qpos, qvel, disable=getattr(C, "DSBL_" + flag))


def _batched_scene():
  from tests import constraint_scenes as S

  mjm = S.load("batched")
  qpos, qvel, _, _ = S.state(mjm, "batched")
  return S, mjm, qpos, qvel


@pytest.mark.parametrize("nworld", [3, 33])
def test_per_world_friction_and_limits(built, nworld):
  """Per-world dof_frictionloss / tendon_frictionloss (a world without the nominal rows, a world with rows on nominally frictionless dofs
  and tendons), eq_data, jnt_range, jnt_margin, dof_solref and geom_friction: k_constraint<true, true>."""
  S, mjm, qpos, qvel = _batched_scene()
  rep = lambda a: np.resize(a, (nworld,) + a.shape[1:])
  _, d, _ = run(mjm, nworld, 64, 16, rep(qpos), rep(qvel), batched={k: v for k, v in S.batched(mjm).items()}, expect=(True, True))
  np.testing.assert_array_equal(d.nf.cpu().numpy()[:3], [2, 0, 4])


def test_per_world_friction_end_to_end(built):
  """World w of the batched model against a one-world model holding w's values (assigned, so the friction tables are rebuilt): the same
  rows, and the solver reads the friction-loss rows as such (qacc and efc.force within the solver band)."""
  import mujoco_warp_b200 as mjw

  S, mjm, qpos, qvel = _batched_scene()
  vals = S.batched(mjm)
  m = mjw.put_model(mjm, batch_sizes={k: S.NWORLD for k in vals})
  for k, v in vals.items():
    getattr(m, k).copy_(torch.as_tensor(v, dtype=torch.float32))
  d = mjw.make_data(mjm, nworld=S.NWORLD, nconmax=16, njmax=64, m=m)
  d.qpos.copy_(torch.as_tensor(qpos, dtype=torch.float32)); d.qvel.copy_(torch.as_tensor(qvel, dtype=torch.float32))
  mjw.forward(m, d)
  for w in range(S.NWORLD):
    m1 = mjw.put_model(mjm)
    for k, v in vals.items():
      setattr(m1, k, torch.as_tensor(v[w : w + 1], dtype=torch.float32, device=d.qpos.device).contiguous())
    d1 = mjw.make_data(mjm, nworld=1, nconmax=16, njmax=64, m=m1)
    d1.qpos.copy_(torch.as_tensor(qpos[w : w + 1], dtype=torch.float32)); d1.qvel.copy_(torch.as_tensor(qvel[w : w + 1], dtype=torch.float32))
    mjw.forward(m1, d1)
    torch.cuda.synchronize()
    for f in ("ne", "nf", "nl", "nefc"):
      assert int(getattr(d1, f).cpu()[0]) == int(getattr(d, f).cpu()[w]), f"w{w} {f}"
    n = int(d1.nefc.cpu()[0])
    np.testing.assert_array_equal(d1.efc.type[0, :n].cpu().numpy(), d.efc.type[w, :n].cpu().numpy())
    fl = d.efc.frictionloss[w, :n].cpu().numpy()
    assert (fl > 0).sum() == int(d.nf.cpu()[w])
    fscale = max(1.0, float(d.efc.force[w, :n].abs().max()))
    util.assert_close(f"w{w} efc.force", d1.efc.force[0, :n].cpu().numpy(), d.efc.force[w, :n].cpu().numpy(), atol=5e-3 * fscale, rtol=0)
    qscale = max(1.0, float(d.qacc[w].abs().max()))
    util.assert_close(f"w{w} qacc", d1.qacc[0].cpu().numpy(), d.qacc[w].cpu().numpy(), atol=5e-3 * qscale, rtol=0)
  nf = d.nf.cpu().numpy()
  np.testing.assert_array_equal(nf, [2, 0, 4])
  st = d.efc.state.cpu().numpy()
  force, floss = d.efc.force.cpu().numpy(), d.efc.frictionloss.cpu().numpy()
  for w in (0, 2):  # friction-loss rows are solved as such: a friction state, and |force| bounded by the row's friction loss
    sl = slice(int(d.ne.cpu()[w]), int(d.ne.cpu()[w]) + int(nf[w]))
    assert set(st[w, sl].tolist()) <= {C.STATE_LINEARNEG, C.STATE_LINEARPOS, C.STATE_QUADRATIC}
    assert (np.abs(force[w, sl]) <= floss[w, sl] * (1 + 1e-6)).all() and (floss[w, sl] > 0).all()


def test_rebinding_friction_refreshes_rows(built):
  """Assigning dof_frictionloss / tendon_frictionloss rebuilds the rows make_constraint emits: a friction row appears on a nominally
  frictionless dof and tendon, and the nominal ones go."""
  S, mjm, qpos, qvel = _batched_scene()
  import mujoco_warp_b200 as mjw

  m = mjw.put_model(mjm)
  fl = np.zeros((1, mjm.nv)); fl[0, 4] = 0.2
  tf = np.zeros((1, mjm.ntendon)); tf[0, 1] = 0.3
  dev = m.dof_frictionloss.device
  m.dof_frictionloss = torch.as_tensor(fl, dtype=torch.float32, device=dev)
  m.tendon_frictionloss = torch.as_tensor(tf, dtype=torch.float32, device=dev)
  mjm.dof_frictionloss, mjm.tendon_frictionloss = fl[0], tf[0]
  d = mjw.make_data(mjm, nworld=1, nconmax=16, njmax=64, m=m)
  d.qpos.copy_(torch.as_tensor(qpos[:1], dtype=torch.float32)); d.qvel.copy_(torch.as_tensor(qvel[:1], dtype=torch.float32))
  mjw.forward(m, d)
  poison(d, False)
  mjw.make_constraint(m, d)
  torch.cuda.synchronize()
  R = co.make_constraint(co.world_model(mjm), world_inputs(mjm, d, 0), 64)
  assert int(d.nf.cpu()[0]) == R.nf == 2
  ids = [(r["type"], r["id"]) for r in R.rows[R.ne : R.ne + R.nf]]
  assert ids == [(C.CNSTR_FRICTION_DOF, 4), (C.CNSTR_FRICTION_TENDON, 1)]
  n = R.nefc
  np.testing.assert_array_equal(d.efc.type[0, :n].cpu().numpy(), [r["type"] for r in R.rows])
  np.testing.assert_array_equal(d.efc.id[0, :n].cpu().numpy(), [r["id"] for r in R.rows])
