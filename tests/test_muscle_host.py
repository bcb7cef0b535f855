"""Muscle actuators without a GPU.

- The device source of the muscle model (mujoco_warp_b200/csrc/mjb_muscle.cuh, compiled as host C++ by tests/host_harness/muscle_host.cpp)
  against the known answers of the reference's util_misc_test.py (gain-length curve, Millard dynamics with and without smoothing, the
  smoothed time scale) and against the fp64 restatement of tests/muscle_oracle.py on random inputs.
- The compiler: the <muscle> shortcut's defaults and attributes, class defaults, <general> with muscle types and raw parameters, the
  lengthrange rules and the "lengthrange" refusal; put_model's refusal of DC-motor and user types.
- The fp64 oracle against the reference's own results (tests/golden/muscle_*.npz, tools/make_muscle_goldens.py): act_dot and
  actuator_force of forward, and of every Euler / implicit step, from the reference's state.
"""
import ctypes
import os
import subprocess
import types

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io, mjcf
from tests import muscle_oracle as O
from tests import muscle_scenes as S

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_harness", "muscle_host.cpp")
OUT = os.path.join(HERE, "host_harness", "_build", "libmuscle_host.so")


@pytest.fixture(scope="module")
def mlib():
  os.makedirs(os.path.dirname(OUT), exist_ok=True)
  cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
  subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", OUT], check=True)
  lib = ctypes.CDLL(OUT)
  fp, cf = ctypes.c_void_p, ctypes.c_float
  for name, args in (("mh_gain_length", [cf] * 3), ("mh_gain", [cf] * 5 + [fp]), ("mh_bias", [cf] * 4 + [fp]), ("mh_timescale", [cf] * 4),
                     ("mh_dynamics", [cf, cf, fp])):
    getattr(lib, name).argtypes = args
    getattr(lib, name).restype = cf
  return lib


def _prm(p):
  a = np.zeros(10, dtype=np.float32)
  a[: len(p)] = p
  return a, a.ctypes.data_as(ctypes.c_void_p)


def _millard(ctrl, act, prm):
  """util_misc_test.py:230-244: the unsmoothed Millard dynamics, as the reference's test states it."""
  ctrlclamp, actclamp = np.clip(ctrl, 0.0, 1.0), np.clip(act, 0.0, 1.0)
  tau = prm[0] * (0.5 + 1.5 * actclamp) if ctrlclamp > act else prm[1] / (0.5 + 1.5 * actclamp)
  return (ctrlclamp - act) / np.maximum(O.MJ_MINVAL, tau)


@pytest.mark.parametrize("length,want", [(0.0, 0.0), (0.5, 0.0), (0.75, 0.5), (1.0, 1.0), (1.25, 0.5), (1.5, 0.0), (2.0, 0.0)])
def test_gain_length_known_answers(mlib, length, want):
  assert mlib.mh_gain_length(length, 0.5, 1.5) == pytest.approx(want, abs=1e-6)
  assert O.gain_length(length, 0.5, 1.5) == pytest.approx(want, abs=1e-12)


def test_dynamics_known_answers(mlib):
  # tausmooth = 0: exactly the Millard dynamics, over the reference's grid of ctrl and act
  a, p = _prm([0.01, 0.04, 0.0])
  for ctrl in (-0.1, 0.0, 0.4, 0.5, 1.0, 1.1):
    for act in (-0.1, 0.0, 0.4, 0.5, 1.0, 1.1):
      want = _millard(ctrl, act, a.astype(np.float64))
      assert mlib.mh_dynamics(ctrl, act, p) == pytest.approx(want, rel=1e-6, abs=1e-6), (ctrl, act)
      assert O.dynamics(ctrl, act, a.astype(np.float64)) == pytest.approx(want, rel=1e-12, abs=1e-12)
  # tausmooth > 0: just outside the smoothing band the Millard value again
  a, p = _prm([0.01, 0.04, 0.2])
  for ctrl in (0.4 - 1e-6, 0.6 + 1e-6):
    assert mlib.mh_dynamics(ctrl, 0.5, p) == pytest.approx(_millard(ctrl, 0.5, a.astype(np.float64)), rel=1e-5)


@pytest.mark.parametrize("dctrl", [0.0, 0.1, 0.2, 1.0, 1.1])
def test_timescale_known_answers(mlib, dctrl):
  # symmetric around dctrl = 0: the mean of the two sides is the mean of the time constants
  lower, upper = mlib.mh_timescale(-dctrl, 0.2, 0.3, 0.2), mlib.mh_timescale(dctrl, 0.2, 0.3, 0.2)
  assert 0.5 * (lower + upper) == pytest.approx(0.25, abs=1e-6)


def test_device_source_matches_fp64_oracle(mlib):
  rng = np.random.default_rng(3)
  worst = 0.0
  for _ in range(3000):
    prm = np.array([rng.uniform(0.4, 0.9), rng.uniform(1.05, 1.5), rng.choice([-1.0, rng.uniform(1, 100)]), rng.uniform(10, 300),
                    rng.uniform(0.2, 0.8), rng.uniform(1.2, 2.0), rng.uniform(0.5, 3), rng.uniform(0.5, 2), rng.uniform(1.1, 2)])
    a, p = _prm(prm)
    prm = a[:9].astype(np.float64)
    lr = np.sort(rng.uniform(-2, 2, 2)).astype(np.float32)
    acc0 = np.float32(rng.uniform(0.1, 500))
    length = np.float32(rng.uniform(lr[0] - 0.5, lr[1] + 0.5))
    vel = np.float32(rng.normal(0, 2))
    scale = max(1.0, abs(O.gain(length, vel, lr, acc0, prm)), abs(O.bias(length, lr, acc0, prm)))
    g = mlib.mh_gain(length, vel, lr[0], lr[1], acc0, p)
    b = mlib.mh_bias(length, lr[0], lr[1], acc0, p)
    worst = max(worst, abs(g - O.gain(length, vel, lr, acc0, prm)) / scale, abs(b - O.bias(length, lr, acc0, prm)) / scale)
    dp, dpp = _prm([rng.uniform(0.005, 0.05), rng.uniform(0.02, 0.1), rng.choice([0.0, rng.uniform(0.01, 0.5)])])
    ctrl, act = np.float32(rng.uniform(-0.3, 1.3)), np.float32(rng.uniform(-0.1, 1.1))
    want = O.dynamics(ctrl, act, dp.astype(np.float64))
    worst = max(worst, abs(mlib.mh_dynamics(ctrl, act, dpp) - want) / max(1.0, abs(want)))
  assert worst < 2e-5, worst


def _xml(actuators, extra=""):
  return f"""<mujoco><default>{extra}</default><worldbody><body><joint name="h" type="hinge" range="-1 2" limited="true"/>
  <joint name="free" type="slide"/><geom type="sphere" size="0.1" mass="1"/></body></worldbody>
  <tendon><fixed name="t" range="-0.5 0.7" limited="true"><joint joint="h" coef="2"/></fixed><fixed name="u"><joint joint="h" coef="1"/></fixed></tendon>
  <compiler angle="radian"/><actuator>{actuators}</actuator></mujoco>"""


def test_compiler_muscle_shortcut():
  m = mjcf.load_string(_xml('<muscle joint="h"/><muscle joint="h" gear="-3" timeconst="0.02 0.05" tausmooth="0.2" range="0.6 1.3" force="40" '
                            'scale="100" lmin="0.3" lmax="1.9" vmax="2" fpmax="1.1" fvmax="1.5"/>'
                            '<muscle class="m" tendon="t"/>', '<default class="m"><muscle force="7" timeconst="0.03"/></default>'))
  assert list(m.actuator_dyntype) == [C.DYN_MUSCLE] * 3 and list(m.actuator_gaintype) == [C.GAIN_MUSCLE] * 3 and list(m.actuator_biastype) == [C.BIAS_MUSCLE] * 3
  np.testing.assert_array_equal(m.actuator_dynprm[0, :3], [0.01, 0.04, 0.0])
  np.testing.assert_array_equal(m.actuator_gainprm[0, :9], [0.75, 1.05, -1, 200, 0.5, 1.6, 1.5, 1.3, 1.2])
  np.testing.assert_array_equal(m.actuator_dynprm[1, :3], [0.02, 0.05, 0.2])
  np.testing.assert_array_equal(m.actuator_gainprm[1, :9], [0.6, 1.3, 40, 100, 0.3, 1.9, 2, 1.1, 1.5])
  np.testing.assert_array_equal(m.actuator_dynprm[2, :3], [0.03, 0.04, 0.0])  # class default: timeconst's second value from MuJoCo's
  assert m.actuator_gainprm[2, 2] == 7
  np.testing.assert_array_equal(m.actuator_biasprm, m.actuator_gainprm)
  assert m.na == 3 and list(m.actuator_actadr) == [0, 1, 2]
  # lengthrange: the joint / tendon limits times gear[0], ends swapped for a negative gear
  np.testing.assert_allclose(m.actuator_lengthrange, [[-1, 2], [-6, 3], [-0.5, 0.7]])


def test_compiler_general_muscle_and_lengthrange_rules():
  m = mjcf.load_string(_xml('<general joint="free" dyntype="muscle" gaintype="muscle" biastype="muscle" gainprm="0.7 1.2 5 100 0.5 1.6 1.5 1.3 1.2" '
                            'biasprm="0.7 1.2 5 100 0.5 1.6 1.5 1.3 1.2" dynprm="0.02 0.03 0.1" lengthrange="-0.2 0.4"/>'
                            '<muscle joint="h" lengthrange="0.1 0.3"/><motor joint="free"/><general joint="h" gaintype="muscle"/>'))
  np.testing.assert_array_equal(m.actuator_gainprm[0, :9], [0.7, 1.2, 5, 100, 0.5, 1.6, 1.5, 1.3, 1.2])
  np.testing.assert_array_equal(m.actuator_dynprm[0, :3], [0.02, 0.03, 0.1])
  assert m.actuator_gaintype[3] == C.GAIN_MUSCLE and m.actuator_biastype[3] == C.BIAS_NONE and m.actuator_dyntype[3] == C.DYN_NONE
  # explicit ranges are kept; a non-muscle keeps (0, 0); a gain-only muscle on a limited joint takes the limits
  np.testing.assert_allclose(m.actuator_lengthrange, [[-0.2, 0.4], [0.1, 0.3], [0, 0], [-1, 2]])
  io._validate(m)


@pytest.mark.parametrize("act", ['<muscle joint="free"/>', '<muscle tendon="u"/>', '<general joint="free" biastype="muscle"/>'])
def test_compiler_refuses_a_muscle_without_lengthrange(act):
  with pytest.raises(NotImplementedError, match="lengthrange"):
    mjcf.load_string(_xml(act))


def test_compiler_refuses_unknown_types_by_name():
  for attr, name in (('gaintype="dcmotor"', "gaintype 'dcmotor'"), ('biastype="user"', "biastype 'user'"), ('dyntype="user"', "dyntype 'user'")):
    with pytest.raises(NotImplementedError, match=name):
      mjcf.load_string(_xml(f'<general joint="h" {attr}/>'))


def test_muscle_on_spatial_tendon_is_still_refused_by_name():
  xml = """<mujoco><worldbody><body><joint type="slide"/><geom type="sphere" size=".1"/><site name="s"/></body><site name="w" pos="1 0 0"/></worldbody>
  <tendon><spatial name="sp"><site site="s"/><site site="w"/></spatial></tendon><actuator><muscle tendon="sp" lengthrange="0 1"/></actuator></mujoco>"""
  with pytest.raises(NotImplementedError, match="spatial"):
    mjcf.load_string(xml)


@pytest.mark.parametrize("field,value,msg", [("actuator_gaintype", 3, r"actuator gain type\(s\) \[3\] are not implemented"),
                                             ("actuator_gaintype", 4, r"actuator gain type\(s\) \[4\] are not implemented"),
                                             ("actuator_biastype", 3, r"actuator bias type\(s\) \[3\] are not implemented"),
                                             ("actuator_dyntype", 5, r"actuator dynamics type\(s\) \[5\] are not implemented"),
                                             ("actuator_dyntype", 6, r"actuator dynamics type\(s\) \[6\] are not implemented")])
def test_put_model_still_refuses_dcmotor_and_user_types(field, value, msg):
  m = S.load("euler")
  getattr(m, field)[0] = value
  with pytest.raises(NotImplementedError, match=msg):
    io._validate(m)


def _lengths(mjm, qpos, qvel):
  """actuator_length / velocity of joint (hinge / slide) and fixed-tendon transmissions."""
  nu = int(mjm.nu)
  L, V = np.zeros(nu), np.zeros(nu)
  for i in range(nu):
    j, g = int(mjm.actuator_trnid[i, 0]), float(mjm.actuator_gear[i, 0])
    if mjm.actuator_trntype[i] == C.TRN_JOINT:
      L[i], V[i] = g * qpos[mjm.jnt_qposadr[j]], g * qvel[mjm.jnt_dofadr[j]]
    else:
      for k in range(int(mjm.tendon_adr[j]), int(mjm.tendon_adr[j] + mjm.tendon_num[j])):
        jj = int(mjm.wrap_objid[k])
        L[i] += g * mjm.wrap_prm[k] * qpos[mjm.jnt_qposadr[jj]]
        V[i] += g * mjm.wrap_prm[k] * qvel[mjm.jnt_dofadr[jj]]
  return L, V


@pytest.mark.parametrize("scene", list(S.SCENES))
def test_oracle_meets_the_reference(scene):
  g = np.load(os.path.join(HERE, "golden", f"muscle_{scene}.npz"))
  mjm = S.load(scene)
  dt = float(mjm.opt.timestep)
  cases = [("start/", "forward/")] + ([(f"step/{k}/in_", f"step/{k}/out_") for k in range(S.SCENES[scene][1])] if scene != "rk4" else [])
  for pin, pout in cases:
    for w in range(S.NWORLD):
      L, V = _lengths(mjm, g[pin + "qpos"][w], g[pin + "qvel"][w])
      act_dot, force = O.actuation(mjm, g[pin + "ctrl"][w], g[pin + "act"][w], L, V, dt)
      scale = max(1.0, float(np.abs(g[pout + "actuator_force"][w]).max()))
      np.testing.assert_allclose(force, g[pout + "actuator_force"][w], rtol=0, atol=1e-9 * scale, err_msg=f"{scene} {pout} world {w}")
      np.testing.assert_allclose(act_dot, g[pout + "act_dot"][w], rtol=0, atol=1e-9 * max(1.0, float(np.abs(act_dot).max())), err_msg=f"{scene} {pout} world {w}")
  # set_length_range: the model's sources, and per-world jnt_range / tendon_range / gear
  nt = int(getattr(mjm, "ntendon", 0))
  for w in range(S.NWORLD):
    want = O.length_range(mjm.actuator_trntype, mjm.actuator_trnid[:, 0], mjm.actuator_gear[:, 0], mjm.jnt_limited, mjm.jnt_range,
                          mjm.tendon_limited if nt else [], mjm.tendon_range if nt else [])
    np.testing.assert_allclose(g["lengthrange/single"][w], want, rtol=1e-12)
    want = O.length_range(mjm.actuator_trntype, mjm.actuator_trnid[:, 0], g["lengthrange/gear"][w, :, 0], mjm.jnt_limited, g["lengthrange/jnt_range"][w],
                          mjm.tendon_limited if nt else [], g["lengthrange/tendon_range"][w])
    np.testing.assert_allclose(g["lengthrange/batched"][w], want, rtol=1e-12)


@pytest.mark.parametrize("scene", ["euler", "implicitfast", "implicit", "rk4"])
def test_full_step_oracle_meets_the_reference(scene):
  """The fp64 muscle step (pipeline oracle plus the muscle forces as applied forces) against every step of the reference's fixtures."""
  g = np.load(os.path.join(HERE, "golden", f"muscle_{scene}.npz"))
  mjm = S.load(scene)
  o = O.MuscleStep(mjm, S.NWORLD, int(g["in/nconmax"]), int(g["in/njmax"]))
  for k in range(S.SCENES[scene][1]):
    p = f"step/{k}/in_"
    t, qpos, qvel, act, act_dot, force = o.step(g[p + "time"], g[p + "qpos"], g[p + "qvel"], g[p + "act"], g[p + "ctrl"], g[p + "qacc_warmstart"])
    q = f"step/{k}/out_"
    for name, got, tol in (("time", t, 1e-12), ("qpos", qpos, 1e-7), ("qvel", qvel, 1e-5), ("act", act, 1e-9), ("act_dot", act_dot, 1e-7),
                           ("actuator_force", force, 1e-7)):
      want = g[q + name].reshape(np.shape(got))
      assert np.abs(got - want).max() <= tol * max(1.0, float(np.abs(want).max())), f"{scene} step {k} {name}: {np.abs(got - want).max()}"


@pytest.mark.parametrize("act", ['<muscle joint="h" gear="0"/>', '<muscle joint="free" lengthrange="0.3 0.3"/>', '<muscle joint="free" lengthrange="0.4 -0.2"/>',
                                 '<general joint="h" gaintype="muscle" lengthrange="1 0"/>'])
def test_compiler_refuses_an_empty_or_reversed_lengthrange(act):
  with pytest.raises(ValueError, match="lengthrange"):
    mjcf.load_string(_xml(act))


def test_put_model_refuses_an_empty_lengthrange():
  m = S.load("euler")
  m.actuator_lengthrange[3] = (0.5, 0.5)
  with pytest.raises(ValueError, match=r"muscle actuator\(s\) \[3\]"):
    io._validate(m)
  m = S.humanoid()
  del m.actuator_lengthrange  # a model saved without the field: every muscle's range is (0, 0)
  with pytest.raises(ValueError, match="lengthrange"):
    io._validate(m)
