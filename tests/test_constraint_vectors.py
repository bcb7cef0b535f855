"""tests/constraint_oracle.py against the reference's own constraint rows (tests/golden/pipeline_*.npz, tools/make_pipeline_goldens.py).

The oracle is fed each fixture's own state, so only its arithmetic is under test: integer outputs (counts, row types and ids, contact
efc addresses) exactly, floats to 1e-12 of their magnitude.  Two states per fixture:
  forward  the rows forward() built from the seeded state; the constraint stage runs before the velocity stage, so cvel and cdof_dot
           are still the zeros make_data left;
  step{s}  the rows step s built (s >= 1, not for RK4): qpos / qvel / cvel / cdof_dot as step s - 1 left them, positions as step s
           computed them -- nonzero cvel, so the weld's Jdot * v term and the ball / free joints' cdof_dot are exercised."""

import os

import numpy as np
import pytest

from tests import constraint_oracle as co
from tests.test_oracle_golden_pipeline import GOLD_DIR, SCENES, load_scene

REL = 1e-12


def world_state(mjm, g, tag, prev, w):
  wid = g[f"{tag}/con_worldid"]
  ids = np.nonzero(wid == w)[0]
  st = {f: g[f"{tag}/{f}"][w] for f in ("xpos", "xmat", "xquat", "cdof", "subtree_com")}
  st["ten_length"] = g[f"{tag}/ten_length"][w] if f"{tag}/ten_length" in g else np.zeros(0)
  if prev is None:
    st["qpos"], st["qvel"] = g["in/qpos"][w], g["in/qvel"][w]
    st["cvel"], st["cdof_dot"] = np.zeros((mjm.nbody, 6)), np.zeros((mjm.nv, 6))
  else:
    st.update({f: g[f"{prev}/{f}"][w] for f in ("qpos", "qvel", "cvel", "cdof_dot")})
  st["eq_active"] = np.asarray(getattr(mjm, "eq_active0", np.ones(int(getattr(mjm, "neq", 0)), dtype=bool)))
  st["con_id"] = ids
  for f in ("dist", "includemargin", "dim", "geom", "pos", "frame", "friction", "solref", "solreffriction", "solimp"):
    st["con_" + f] = g[f"{tag}/con_{f}"][ids]
  return st


def tags(g, name=""):
  yield "forward", None
  if name.endswith("rk4"):  # an RK4 step's snapshot holds the positions of its last stage, not those its constraint rows were built from
    return
  s = 1
  while f"step{s}/efc_type" in g:
    yield f"step{s}", f"step{s - 1}"
    s += 1


def check(name, got, want, mag, rel=REL):
  err = np.abs(np.asarray(got, dtype=np.float64) - want)
  tol = rel * np.maximum(mag, 1.0)
  bad = err > tol
  assert not bad.any(), f"{name}: worst at {np.argwhere(bad)[0]}: got {np.asarray(got)[bad][0]!r}, want {want[bad][0]!r}, mag {mag[bad][0]:.3g}"


@pytest.mark.parametrize("name", SCENES)
def test_oracle_matches_reference_rows(name):
  g = np.load(os.path.join(GOLD_DIR, f"pipeline_{name}.npz"))
  mjm = load_scene(name)
  njmax = int(g["in/njmax"])
  nworld = g["in/qpos"].shape[0]
  m = co.world_model(mjm)
  checked = 0
  for tag, prev in tags(g, name):
    for w in range(nworld):
      try:
        R = co.make_constraint(m, world_state(mjm, g, tag, prev, w), njmax)
      except co.KnifeEdge:
        continue  # a decision within rounding of its threshold: the reference may have taken either side
      for f, n in (("ne", R.ne), ("nf", R.nf), ("nl", R.nl), ("nefc", R.nefc)):
        assert n == int(g[f"{tag}/{f}"].reshape(-1)[w]), f"{name} {tag} w{w}: {f} {n} vs {int(g[f'{tag}/{f}'].reshape(-1)[w])}"
      nr = min(R.nefc, njmax)
      a = co.arrays(R, mjm.nv)
      np.testing.assert_array_equal(a["type"][:nr], g[f"{tag}/efc_type"][w, :nr], err_msg=f"{name} {tag} w{w} type")
      np.testing.assert_array_equal(a["id"][:nr], g[f"{tag}/efc_id"][w, :nr], err_msg=f"{name} {tag} w{w} id")
      check(f"{name} {tag} w{w} J", g[f"{tag}/efc_J"][w, :nr, : mjm.nv], a["J"][:nr], a["J_mag"][:nr])
      for f in ("pos", "margin", "vel", "frictionloss", "D", "aref"):
        check(f"{name} {tag} w{w} {f}", g[f"{tag}/efc_{f}"][w, :nr], a[f][:nr], a[f + "_mag"][:nr])
      ids = R.efc_address.shape[0]
      if ids:
        want = g[f"{tag}/con_efc_address"][np.nonzero(g[f"{tag}/con_worldid"] == w)[0]]
        np.testing.assert_array_equal(R.efc_address[:, : want.shape[1]], want, err_msg=f"{name} {tag} w{w} efc_address")
        assert (R.efc_address[:, want.shape[1] :] == -1).all()
      checked += 1
  assert checked >= nworld, f"{name}: only {checked} world states away from every knife edge"


def test_oracle_covers_row_kinds():
  """The fixtures above hold every kind of row the oracle builds (so none of its branches is checked by nothing)."""
  seen = set()
  for name in SCENES:
    g = np.load(os.path.join(GOLD_DIR, f"pipeline_{name}.npz"))
    for tag, _ in tags(g, name):
      t = g[f"{tag}/efc_type"]
      n = np.minimum(g[f"{tag}/nefc"].reshape(-1), t.shape[1])
      for w in range(t.shape[0]):
        seen |= set(int(x) for x in t[w, : n[w]])
  from mujoco_warp_b200._src import constants as C

  want = {C.CNSTR_EQUALITY, C.CNSTR_FRICTION_DOF, C.CNSTR_FRICTION_TENDON, C.CNSTR_LIMIT_JOINT, C.CNSTR_LIMIT_TENDON, C.CNSTR_CONTACT_FRICTIONLESS,
          C.CNSTR_CONTACT_PYRAMIDAL, C.CNSTR_CONTACT_ELLIPTIC}
  assert want <= seen, f"row kinds no fixture holds: {sorted(want - seen)}"


BATCHED = ("dof_frictionloss", "tendon_frictionloss", "eq_data", "jnt_range", "jnt_margin", "dof_solref", "geom_friction")


@pytest.mark.parametrize("name", ["sparse", "batched"])
def test_oracle_matches_reference_constraint_fixtures(name):
  """tests/golden/constraint_*.npz (tools/make_constraint_goldens.py): a sparse scene with every row kind, its CSR view as the reference wrote
  it, and a scene with per-world friction loss (rows appear and disappear per world), eq_data, jnt_range, jnt_margin, dof_solref and
  geom_friction."""
  from tests import constraint_scenes as S

  g = np.load(os.path.join(GOLD_DIR, f"constraint_{name}.npz"))
  mjm = S.load(name)
  njmax = int(g["in/njmax"])
  batched = {k: g[f"in/{k}"] for k in BATCHED if f"in/{k}" in g}
  assert (name == "batched") == bool(batched)
  kinds = set()
  for w in range(g["in/qpos"].shape[0]):
    m = co.world_model(mjm, batched, w)
    R = co.make_constraint(m, world_state(mjm, g, "forward", None, w), njmax)
    for f, n in (("ne", R.ne), ("nf", R.nf), ("nl", R.nl), ("nefc", R.nefc)):
      assert n == int(g[f"forward/{f}"].reshape(-1)[w]), f"{name} w{w}: {f} {n} vs {int(g[f'forward/{f}'].reshape(-1)[w])}"
    nr = min(R.nefc, njmax)
    a = co.arrays(R, mjm.nv)
    kinds |= set(a["type"].tolist())
    np.testing.assert_array_equal(a["type"][:nr], g["forward/efc_type"][w, :nr], err_msg=f"{name} w{w} type")
    np.testing.assert_array_equal(a["id"][:nr], g["forward/efc_id"][w, :nr], err_msg=f"{name} w{w} id")
    check(f"{name} w{w} J", g["forward/efc_J"][w, :nr, : mjm.nv], a["J"][:nr], a["J_mag"][:nr])
    for f in ("pos", "margin", "vel", "frictionloss", "D", "aref"):
      check(f"{name} w{w} {f}", g[f"forward/efc_{f}"][w, :nr], a[f][:nr], a[f + "_mag"][:nr])
    if "csr/J_rownnz" in g:
      nnz, adr, cols, vals, over = co.csr(m, R, njmax, g["csr/J"].shape[2])
      assert not over
      np.testing.assert_array_equal(nnz, g["csr/J_rownnz"][w, :nr], err_msg=f"{name} w{w} rownnz")
      np.testing.assert_array_equal(adr, g["csr/J_rowadr"][w, :nr], err_msg=f"{name} w{w} rowadr")
      for r in range(nr):
        sl = slice(adr[r], adr[r] + nnz[r])
        np.testing.assert_array_equal(cols[r], g["csr/J_colind"][w, 0, sl], err_msg=f"{name} w{w} row {r} colind")
        check(f"{name} w{w} row {r} CSR values", g["csr/J"][w, 0, sl], np.array([x.v for x in vals[r]]), np.array([x.m for x in vals[r]]))
  from mujoco_warp_b200._src import constants as C

  if name == "sparse":  # every row kind a sparse model can hold, incl. both tendon equality forms
    assert {C.CNSTR_EQUALITY, C.CNSTR_FRICTION_TENDON, C.CNSTR_LIMIT_JOINT, C.CNSTR_LIMIT_TENDON, C.CNSTR_CONTACT_PYRAMIDAL} <= kinds
  else:  # per-world friction: world 1 has no friction rows, world 2 has the two nominally frictionless ones as well
    np.testing.assert_array_equal(g["forward/nf"].reshape(-1), [2, 0, 4])
