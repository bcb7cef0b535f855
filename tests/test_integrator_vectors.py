"""The fp64 restatement of the integration stage (tests/integrator_oracle.py) without a GPU.

- Against the reference's own fixtures: step0's qLU and qvel of the implicit and implicitfast pipeline scenes, fed the fixtures' forward()
  fields with right-hand side M qacc.
- Against the C oracle's step for every integrator on the mixed, tendons, actuators and cross-tree scenes (RK4: the restatement's
  bookkeeping over the oracle's forward at each stage state).
- Its d(qfrc_bias)/d(qvel) against the central difference of the oracle's qfrc_bias, which is exact up to rounding: RNE is quadratic in qvel.
- The cross-tree scene: a tendon actuator whose moment row spans two kinematic trees puts qDeriv entries in both trees' blocks.
"""
import os

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf
from tests import integrator_oracle as O
from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))
INTEGRATORS = {"Euler": C.INT_EULER, "RK4": C.INT_RK4, "implicit": C.INT_IMPLICIT, "implicitfast": C.INT_IMPLICITFAST}

# A fixed tendon over ja2 (tree 0) and jb, jb2 (tree 1), driven by a position servo with kv: its moment row spans both trees.
CROSSTREE_XML = """<mujoco model="crosstree"><option timestep="0.004" integrator="{integrator}"/>
<worldbody>
  <body name="a1" pos="0 0 1"><joint name="ja1" type="hinge" axis="0 1 0" damping="0.3"/><geom type="capsule" fromto="0 0 0 .2 0 0" size=".02" mass=".5"/>
    <body name="a2" pos=".2 0 0"><joint name="ja2" type="hinge" axis="0 1 0" damping="0.1"/><geom type="capsule" fromto="0 0 0 .2 0 0" size=".02" mass=".3"/></body>
  </body>
  <body name="b1" pos="0 .5 1"><joint name="jb" type="slide" axis="0 0 1" damping="0.5"/><geom type="box" size=".05 .05 .05" mass=".4"/>
    <body name="b2" pos="0 0 -.1"><joint name="jb2" type="hinge" axis="1 0 0"/><geom type="capsule" fromto="0 0 0 0 0 -.2" size=".02" mass=".2"/></body>
  </body>
</worldbody>
<tendon><fixed name="x" damping="0.4"><joint joint="ja2" coef="1"/><joint joint="jb" coef="-0.5"/><joint joint="jb2" coef="0.8"/></fixed></tendon>
<actuator><position tendon="x" kp="5" kv="2"/></actuator></mujoco>"""


def load(scene, integrator):
  xml = {"mixed": lambda i: util.MIXED_XML.replace('<option timestep="0.004"', f'<option integrator="{i}" timestep="0.004"'),
         "actuators": util.actuators_xml, "tendons": util.tendon_xml, "crosstree": lambda i: CROSSTREE_XML.format(integrator=i)}[scene]
  return mjcf.load_string(xml(integrator))


@pytest.mark.parametrize("name", ["mixed_implicit", "actuators_implicit", "tendons_implicit", "actuators_implicitfast", "tendons_implicitfast"])
def test_restatement_meets_the_reference_fixtures(name):
  scene, integrator = name.split("_")
  g = np.load(os.path.join(HERE, "golden", f"pipeline_{name}.npz"))
  mjm = load(scene, integrator)
  nworld = g["in/qpos"].shape[0]
  for w in range(nworld):
    f = {k.split("/")[1]: g[k][w] for k in g if k.startswith("forward/") and g[k].ndim and g[k].shape[0] == nworld}
    f["ctrl"] = g["in/ctrl"][w]
    _, qvel, qpos, act = O.integrate(mjm, f, INTEGRATORS[integrator])
    want = g["step0/qvel"][w]
    assert np.abs(qvel - want).max() <= 1e-9 * max(1.0, np.abs(want).max()), (name, w)
    assert np.abs(qpos - g["step0/qpos"][w]).max() <= 1e-9, (name, w)
    if act is not None:
      assert np.abs(act - g["step0/act"][w]).max() <= 1e-9, (name, w)
    if integrator == "implicit":
      want = g["step0/qLU"][w]
      got = O.lu_d(mjm, O.matrix_a(mjm, f, C.INT_IMPLICIT))
      assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max(), (name, w)


def _state(mjm, nworld, seed):
  rng = np.random.default_rng(seed)
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld, seed=seed, exact_world0=False)
  act = util.seeded_act(mjm, nworld, seed=seed)
  return qpos, qvel, ctrl, act, rng


@pytest.mark.parametrize("scene", ["mixed", "tendons", "actuators", "crosstree"])
@pytest.mark.parametrize("integrator", list(INTEGRATORS))
def test_restatement_meets_the_oracle_step(scene, integrator):
  mjm = load(scene, integrator)
  nworld = 2
  qpos, qvel, ctrl, act, _ = _state(mjm, nworld, 7)
  o = util.make_oracle(mjm, nworld, 32, 128)
  o.set_state(qpos=qpos, qvel=qvel, ctrl=ctrl, act=act)
  o.forward()
  fields = [{k: v[w].copy() for k, v in o.d.items()} for w in range(nworld)]
  o.set_state(qpos=qpos, qvel=qvel, ctrl=ctrl, act=act)
  o.step()
  for w in range(nworld):
    if integrator == "RK4":
      def fwd(q, v, a):
        o1 = util.make_oracle(mjm, 1, 32, 128)
        o1.set_state(qpos=q[None], qvel=v[None], ctrl=ctrl[w : w + 1], act=a[None])
        o1.forward()
        return {"qacc": o1.d["qacc"][0].copy(), "act_dot": o1.d["act_dot"][0].copy()}
      qp, qv, ac, _ = O.rk4(mjm, {"qpos": qpos[w], "qvel": qvel[w], "act": act[w]}, fwd)
    else:
      _, qv, qp, ac = O.integrate(mjm, fields[w], INTEGRATORS[integrator])
    scale = max(1.0, np.abs(o.d["qvel"][w]).max())
    assert np.abs(qv - o.d["qvel"][w]).max() <= 1e-10 * scale, (scene, integrator, w)
    assert np.abs(qp - o.d["qpos"][w]).max() <= 1e-10, (scene, integrator, w)
    if ac is not None and len(ac):
      assert np.abs(ac - o.d["act"][w]).max() <= 1e-10, (scene, integrator, w)


@pytest.mark.parametrize("scene", ["mixed", "tendons", "actuators", "crosstree"])
def test_rne_velocity_derivative_is_the_central_difference(scene):
  """qfrc_bias is quadratic in qvel at fixed qpos, so (bias(v + h e_k) - bias(v - h e_k)) / 2h is its derivative up to rounding.  Every
  joint type of the scenes (free, ball, hinge, slide) agrees with the restatement's column k."""
  mjm = load(scene, "implicit")
  qpos, qvel, ctrl, act, _ = _state(mjm, 1, 11)
  o = util.make_oracle(mjm, 1, 32, 128)
  o.set_state(qpos=qpos, qvel=qvel, ctrl=ctrl, act=act)
  o.forward()
  D = O.drne_dqvel(mjm, {k: v[0] for k, v in o.d.items()})
  h = 0.5
  fd = np.zeros_like(D)
  for k in range(mjm.nv):
    bias = []
    for s in (1.0, -1.0):
      v = qvel.copy()
      v[0, k] += s * h
      o.set_state(qpos=qpos, qvel=v, ctrl=ctrl, act=act)
      o.forward()
      bias.append(o.d["qfrc_bias"][0].copy())
    fd[:, k] = (bias[0] - bias[1]) / (2 * h)
  assert np.abs(D - fd).max() <= 1e-10 * max(1.0, np.abs(fd).max()), np.abs(D - fd).max()


def test_crosstree_actuator_terms_land_in_both_trees():
  """The tendon actuator's kv and the tendon damping put qDeriv entries on dofs of tree 0 (ja2) and of tree 1 (jb, jb2): a kernel that
  assigns the actuator to the tree of its first dof drops tree 1's entries."""
  mjm = load("crosstree", "implicitfast")
  assert int(mjm.ntree) == 2 and list(mjm.ten_J_colind) == [1, 2, 3] and list(mjm.tree_dofadr) == [0, 2]
  qpos, qvel, ctrl, act, _ = _state(mjm, 1, 3)
  o = util.make_oracle(mjm, 1, 8, 16)
  o.set_state(qpos=qpos, qvel=qvel, ctrl=ctrl)
  o.forward()
  f = {k: v[0] for k, v in o.d.items()}
  terms = O.qderiv_terms(mjm, f)
  rows = sorted({i for i, _, _ in terms})
  assert rows == [1, 2, 3], rows  # ja2 in tree 0; jb, jb2 in tree 1 (with the off-diagonal (jb2, jb))
  assert (3, 2) in {(i, j) for i, j, _ in terms}
  A = O.matrix_a(mjm, f, C.INT_IMPLICITFAST)
  M = O.dense_m(mjm, f["M"])
  assert abs(A[3, 2] - M[3, 2]) > 1e-3  # the coupling of jb and jb2 through the actuator and the tendon damper
  assert np.all(A[:2, 2:] == 0) and np.all(A[2:, :2] == 0)  # nothing couples the two trees: M has no entry there
