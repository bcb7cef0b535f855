"""set_const without a GPU: the numpy per-world oracle and the Python wrapper's checks against a stub of the C library.

- On unmodified models the oracle (tests/set_const_oracle.py) reproduces the compiler's derived fields, except where the reference
  differs from this repo's compiler on purpose (the invweight0 fallback of set_const.py:366-370, camera / light targets).
- Per-world inputs change the per-world outputs, and entries follow their own world's inputs.
- The wrapper: argument types, Data of another Model, an output with more entries than worlds (ValueError), the part bits passed to
  the library and the meaninertia hand-over.
"""
import numpy as np
import pytest

from mujoco_warp_b200._src import mjcf
from tests import set_const_oracle, set_const_scenes


@pytest.mark.parametrize("scene", ["chain", "mixed", "equality", "tendon"])
def test_oracle_reproduces_the_compiler(scene):
  mjm = mjcf.load_string(set_const_scenes.SCENES[scene])
  o = set_const_oracle.oracle(mjm, {}, 1)
  for f in ("body_subtreemass", "dof_invweight0", "tendon_invweight0", "tendon_length0", "actuator_acc0", "eq_data", "tendon_lengthspring"):
    want = np.asarray(getattr(mjm, f), dtype=np.float64).reshape(o[f][0].shape)
    np.testing.assert_allclose(o[f][0], want, atol=1e-9, rtol=1e-9, err_msg=f)
  assert abs(o["meaninertia"] - mjm.stat.meaninertia) <= 1e-9 * mjm.stat.meaninertia
  bw = np.asarray(mjm.body_invweight0)
  fb = ((bw[:, 0] < 1e-15) & (bw[:, 1] > 1e-15)) | ((bw[:, 1] < 1e-15) & (bw[:, 0] > 1e-15))
  want = bw.copy()
  want[fb] = bw[fb].max(axis=1)[:, None]
  np.testing.assert_allclose(o["body_invweight0"][0], want, atol=1e-9, rtol=1e-9)


def test_oracle_fallback_bodies_of_the_static_scene():
  mjm = mjcf.load_string(set_const_scenes.STATIC)
  o = set_const_oracle.oracle(mjm, {}, 1)["body_invweight0"][0]
  names = mjm.names.body
  for b in range(mjm.nbody):
    if names[b] in ("world", "wall"):
      assert (o[b] == 0).all(), names[b]
    elif names[b] in ("slider", "rider", "xy"):  # slide joints only: no rotational weight, the translational one is copied over
      assert o[b, 0] > 0 and o[b, 1] == o[b, 0], names[b]
    else:
      assert o[b, 0] > 0 and o[b, 1] > 0 and o[b, 0] != o[b, 1], names[b]


@pytest.mark.parametrize("scene", ["chain", "mixed", "tendon", "dampratio", "equality"])
def test_oracle_entries_follow_their_world(scene):
  mjm = mjcf.load_string(set_const_scenes.SCENES[scene])
  inputs = set_const_scenes.per_world_inputs(scene, mjm)
  o = set_const_oracle.oracle(mjm, inputs, set_const_scenes.NWORLD)
  for w in range(set_const_scenes.NWORLD):
    one = set_const_oracle.world(mjm, inputs, w)
    for f in set_const_scenes.OUTPUTS:
      np.testing.assert_array_equal(o[f][w], one[f])
  changed = {f for f in set_const_scenes.OUTPUTS if o[f].size and np.abs(o[f][1] - o[f][0]).max() > 1e-9}
  assert {"dof_invweight0", "body_invweight0"} <= changed or scene == "equality", changed
  if scene == "dampratio":
    bp = o["actuator_biasprm"]
    assert (bp[:, :3, 2] < 0).all() and (bp[:, 3:, 2] == np.asarray(mjm.actuator_biasprm)[3:, 2]).all()
  if scene == "tendon":
    assert "tendon_lengthspring" in changed
  if scene == "equality":
    q = o["eq_data"][:, 1, 6:10]
    np.testing.assert_allclose(np.linalg.norm(q, axis=1), 1.0, atol=1e-12)


@pytest.fixture
def stub(monkeypatch):
  import torch

  from mujoco_warp_b200._src import _lib
  from mujoco_warp_b200._src import io as mio

  calls = []

  class Stub:
    def __getattr__(self, name):
      def f(*a, **k):
        calls.append((name, a))
        return 1 if name in ("mjb_model_create", "mjb_data_create") else 0

      return f

  class Stream:
    cuda_stream = 0

    def synchronize(self):
      calls.append(("synchronize", ()))

  monkeypatch.setattr(mio, "_require_cuda", lambda: torch.device("cpu"))
  monkeypatch.setattr(_lib, "lib", lambda: Stub())
  monkeypatch.setattr(torch.cuda, "current_stream", lambda: Stream())
  return calls


def test_wrapper_checks_and_calls(stub):
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import io as mio

  mjm = mjcf.load_string(set_const_scenes.CHAIN)
  m = mio.put_model(mjm, batch_sizes={"body_mass": 4, "dof_invweight0": 4, "actuator_acc0": 2})
  assert tuple(m.actuator_acc0.shape) == (2, mjm.nu)
  d = mio.make_data(mjm, nworld=4, m=m)
  with pytest.raises(TypeError):
    mjw.set_const(m, None)
  stub.clear()
  mjw.set_const(m, d)
  sc = [a for n, a in stub if n == "mjb_set_const"]
  assert len(sc) == 1 and sc[0][2:4] == (3, 1)  # fixed | 0: without tendons nothing depends on qpos_spring
  assert ("synchronize", ()) in stub and any(n == "mjb_model_set_float" and a[1] == b"meaninertia" for n, a in stub)
  stub.clear()
  mjw.set_const_fixed(m, d)
  assert [a[2:4] for n, a in stub if n == "mjb_set_const"] == [(1, 0)] and ("synchronize", ()) not in stub
  stub.clear()
  mjw.set_const_spring(m, d)  # no tendons: nothing to do
  assert not stub
  stub.clear()
  mjw.set_const_0(m, d, restore=False)
  assert [a[2:4] for n, a in stub if n == "mjb_set_const"] == [(2, 0)]
  d2 = mio.make_data(mjm, nworld=2, m=m)
  with pytest.raises(ValueError, match="dof_invweight0 has 4 per-world entries but Data has 2 worlds"):
    mjw.set_const(m, d2)
  mjw.set_const_fixed(m, d2)  # body_subtreemass is unbatched: fine
  other = mio.put_model(mjm)
  other._handle = 2
  with pytest.raises(ValueError, match="different Model"):
    mjw.set_const(other, d)
  with pytest.raises(ValueError, match="not a batched array field"):
    mio.put_model(mjm, batch_sizes={"body_parentid": 2})
