"""The numpy per-world oracle (tests/set_const_oracle.py) against the reference's own set_const (tests/golden/set_const_*.npz, written by
tools/make_set_const_goldens.py: io.put_model -> make_data -> set_const / set_const_0 / set_const_spring under tools/warp_shim.py, in
double precision, with the scene's inputs and every output batched per world).  Met to 1e-9 of each field's scale."""
import os

import numpy as np
import pytest

from mujoco_warp_b200._src import mjcf
from tests import set_const_oracle, set_const_scenes

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ZERO = ("tendon_length0", "eq_data", "dof_invweight0", "body_invweight0", "tendon_invweight0", "cam_pos0", "cam_poscom0", "cam_mat0", "light_pos0",
        "light_poscom0", "light_dir0", "actuator_acc0", "actuator_biasprm")


def load(scene):
  g = np.load(os.path.join(GOLD, f"set_const_{scene}.npz"))
  mjm = mjcf.load_string(set_const_scenes.SCENES[scene])
  inputs = {k[3:]: g[k] for k in g.files if k.startswith("in/")}
  return g, mjm, inputs


def expected(mjm, inputs, call, nworld):
  """The oracle's outputs of `call` for worlds [0, nworld): (fields, meaninertia of world 0)."""
  if call == "set_const":
    o = set_const_oracle.oracle(mjm, inputs, nworld)
    return {f: o[f] for f in set_const_scenes.OUTPUTS}, o["meaninertia"]
  # set_const_0 / set_const_spring alone: body_subtreemass stays the compiled one; each part writes its own fields only
  nominal = np.asarray(mjm.body_subtreemass, dtype=np.float64)
  per = [set_const_oracle.world(mjm, inputs, w, subtreemass=nominal) for w in range(nworld)]
  fields = ZERO if call == "set_const_0" else ("tendon_lengthspring",)
  return {f: np.stack([p[f] for p in per]) for f in fields}, per[0]["meaninertia"] if call == "set_const_0" else None


CASES = [(s, c) for s in sorted(set_const_scenes.SCENES) for c in ("set_const", "set_const_0", "set_const_spring")
         if c == "set_const" or s in ("tendon", "dampratio")]


@pytest.mark.parametrize("scene,call", CASES)
def test_oracle_meets_the_reference(scene, call):
  g, mjm, inputs = load(scene)
  nworld = 1 if scene == "unbatched" else set_const_scenes.NWORLD
  want, mi = expected(mjm, inputs, call, nworld)
  for f, w in want.items():
    got = g[f"{call}/{f}"]
    if not got.size:
      continue
    scale = max(1.0, float(np.abs(got).max()))
    np.testing.assert_allclose(w.reshape(got.shape), got, atol=1e-9 * scale, rtol=0, err_msg=f"{scene}/{call}/{f}")
  if mi is not None:
    np.testing.assert_allclose(mi, g[f"{call}/meaninertia"][0], rtol=1e-12)


def test_fixtures_cover_the_cases_of_the_issue():
  """Aimed lights, target cameras, weld quaternions cleared and set, the invweight0 fallback, resolved tendon springs, dampratio."""
  g, mjm, _ = load("camlight")
  assert {3, 4} <= set(np.asarray(mjm.light_mode)[np.asarray(mjm.light_targetbodyid) >= 0].tolist())
  assert {1, 2, 3, 4} <= set(np.asarray(mjm.cam_mode).tolist())
  g, mjm, inputs = load("equality")
  assert (inputs["eq_data"][:, 2, 6:10] == 0).all() and (np.abs(g["set_const/eq_data"][:, 2, 6:10]).sum(axis=1) > 0).all()
  np.testing.assert_allclose(np.linalg.norm(g["set_const/eq_data"][:, 1, 6:10], axis=1), 1.0, atol=1e-12)
  g, mjm, _ = load("static")
  bw = g["set_const/body_invweight0"]
  slider = mjm.names.body.index("slider")
  assert (bw[:, slider, 0] == bw[:, slider, 1]).all() and (bw[:, slider] > 0).all()
  g, mjm, inputs = load("tendon")
  assert (g["set_const_spring/tendon_lengthspring"][:, 0] != -1).all() and (inputs["tendon_lengthspring"][:, 0] == -1).all()
  g, mjm, _ = load("dampratio")
  assert (g["set_const/actuator_biasprm"][:, :3, 2] < 0).all()
