"""The reference's own energy (tests/golden/energy_*.npz, tools/make_energy_goldens.py) against an fp64 numpy restatement of its formulas
(tests/energy_oracle.py), per world, to 1e-9: energy_pos / energy_vel, what forward leaves in d.energy and in the energy sensors, and
what one step leaves there."""
import os

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from tests import energy_oracle, energy_scenes, util

TOL = 1e-9


def load(scene):
  g = np.load(os.path.join(util.ROOT, "tests", "golden", f"energy_{scene}.npz"))
  mjm = energy_scenes.load(scene)
  inputs = {k[3:]: g[k] for k in g.files if k.startswith("in/") and k[3:] not in ("qpos", "qvel", "nconmax", "njmax")}
  return g, mjm, inputs


def energy_sensors(mjm):
  """[(slot, type, cutoff)] of the model's e_potential / e_kinetic sensors"""
  st = np.asarray(mjm.sensor_type) if mjm.nsensor else np.zeros(0, dtype=int)
  return [(int(mjm.sensor_adr[s]), int(st[s]), float(mjm.sensor_cutoff[s])) for s in range(mjm.nsensor) if st[s] in (C.SENS_E_POTENTIAL, C.SENS_E_KINETIC)]


def sensor_value(e, typ, cutoff):
  x = e[0] if typ == C.SENS_E_POTENTIAL else e[1]
  return float(np.clip(x, -cutoff, cutoff)) if cutoff > 0 else x


@pytest.mark.parametrize("scene", sorted(energy_scenes.SCENES))
def test_energy_oracle_meets_the_reference(scene):
  g, mjm, inputs = load(scene)
  flag = bool(int(mjm.opt.enableflags) & C.ENBL_ENERGY)
  sensors = energy_sensors(mjm)
  for w in range(energy_scenes.NWORLD):
    want = energy_oracle.energy(mjm, inputs, g, w)
    np.testing.assert_allclose(g["direct/energy"][w], want, rtol=TOL, atol=TOL, err_msg=f"{scene} w{w} energy_pos / energy_vel")
    # forward: both terms with the flag; without it the reference zeroes d.energy (forward.py:1332)
    np.testing.assert_allclose(g["forward/energy"][w], want if flag else (0.0, 0.0), rtol=TOL, atol=TOL, err_msg=f"{scene} w{w} forward")
    for slot, typ, cutoff in sensors:
      assert abs(g["forward/sensordata"][w, slot] - sensor_value(want, typ, cutoff)) <= TOL * max(1.0, abs(want[0]) + abs(want[1])), (scene, w, slot)
      assert abs(g["step/sensordata"][w, slot] - sensor_value(want, typ, cutoff)) <= TOL * max(1.0, abs(want[0]) + abs(want[1])), (scene, w, slot)
    if mjm.opt.integrator == C.INT_RK4:
      # rungekutta4 calls forward for every stage: d.energy is the last stage's, not the state the step started from
      assert np.abs(g["step/energy"][w] - want).max() > 1e-6, (scene, w)
    else:
      np.testing.assert_allclose(g["step/energy"][w], want if flag else (0.0, 0.0), rtol=TOL, atol=TOL, err_msg=f"{scene} w{w} step")


def test_energy_fixtures_cover_the_cases():
  """Every term is non-trivial somewhere: springs of each joint type, tendons inside / above / below their dead band, clipping cutoffs."""
  g, mjm, inputs = load("tendon")
  ls = inputs["tendon_lengthspring"].reshape(energy_scenes.NWORLD, -1, 2)
  L = g["forward/ten_length"][:, 0]
  assert {int(np.sign(L[w] - ls[w, 0, 1]) if L[w] > ls[w, 0, 1] else np.sign(L[w] - ls[w, 0, 0]) if L[w] < ls[w, 0, 0] else 0) for w in range(3)} == {-1, 0, 1}
  g, mjm, inputs = load("sensors_on")
  clipped = [(w, slot) for w in range(3) for slot, typ, c in energy_sensors(mjm) if c > 0 and abs(sensor_value(g["direct/energy"][w], typ, 0.0)) > c]
  assert len(clipped) >= 2, clipped
  for w in range(3):
    grav, spring = energy_oracle.potential_terms(mjm, inputs, w, g["in/qpos"][w], g["forward/xipos"][w], g["forward/ten_length"][w])
    assert len(spring) == 5 and (spring > 0).all()  # hinge, slide, ball, free translation, free rotation
  g, mjm, _ = load("g1")
  assert mjm.nv == 35
