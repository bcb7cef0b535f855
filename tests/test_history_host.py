"""Actuator and sensor delays without a GPU.

- The compiler: nsample / interp / delay / interval on actuators and sensors, through defaults classes, and the buffer layout.
- The refusals: a delay or interval without samples, negative values, an unknown interp, per-world delays.
- get_state / set_state: State.HISTORY is nhistory wide.
- The device source of the ring buffers (mujoco_warp_b200/csrc/mjb_history.cuh, compiled as host C++ by tests/host_harness/history_host.cpp)
  replays the reference's own vectors (tests/golden/history_*.npz, tools/make_history_goldens.py): the delayed ctrl each step, the ctrl
  insert, the sensor delay / interval rule with its insert, and read_ctrl / read_sensor at off-grid times.
"""
import ctypes
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import io, mjcf
from tests import history_scenes as H

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_harness", "history_host.cpp")
OUT = os.path.join(HERE, "host_harness", "_build", "libhistory_host.so")
DT = H.DT


@pytest.fixture(scope="module")
def hlib():
  os.makedirs(os.path.dirname(OUT), exist_ok=True)
  cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
  subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", OUT], check=True)
  lib = ctypes.CDLL(OUT)
  fp, ci, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
  lib.hh_read.argtypes = [fp, ci, ci, cf, ci, fp]
  lib.hh_insert.argtypes = [fp, ci, ci, cf, fp]
  lib.hh_sensor.argtypes = [fp, ci, ci, ci, cf, cf, cf, fp]
  return lib


def _p(a):
  return a.ctypes.data_as(ctypes.c_void_p)


def _golden(name):
  return np.load(os.path.join(HERE, "golden", f"history_{name}.npz"))


def test_compiler_fields_and_layout():
  m = H.load("actuators")
  np.testing.assert_array_equal(m.actuator_history, [[4, 0], [3, 1], [6, 2], [2, 0], [0, 0]])  # actuator 0 from the defaults class
  np.testing.assert_allclose(m.actuator_delay, np.array([2.5, 1.5, 2.25, 0, 0]) * DT)
  np.testing.assert_array_equal(m.sensor_history, [[3, 0], [4, 1], [5, 2], [2, 0], [0, 0]])
  # [user, cursor, times[n], values[n dim]]: actuators first, in index order, then sensors; -1 without a buffer
  np.testing.assert_array_equal(m.actuator_historyadr, [0, 10, 18, 32, -1])
  np.testing.assert_array_equal(m.sensor_historyadr, [38, 46, 56, 68, -1])
  assert m.nhistory == 74
  v = H.load("vectors")
  np.testing.assert_allclose(v.sensor_interval, np.array([[0, 0], [0, 0], [3, 1], [2, 0]]) * DT)
  np.testing.assert_array_equal(v.sensor_historyadr, [8, 8 + 2 + 4 * (1 + 3), 26 + 2 + 5 * (1 + 4), 53 + 2 + 2 * (1 + 3)])
  assert v.nhistory == 63 + 2 + 3 * (1 + 3)
  for name in H.SCENES:
    io._validate(H.load(name))


def test_sensor_defaults_and_no_history_model():
  x = """<mujoco><default><sensor nsample="2" interp="linear" delay="0.01"/><default class="c"><sensor nsample="5" interval="0.1 0.05"/></default></default>
  <worldbody><body><joint name="j" type="slide"/><geom size=".1" mass="1"/></body></worldbody>
  <sensor><jointpos joint="j"/><jointvel joint="j" class="c"/><jointpos joint="j" nsample="0" delay="0"/></sensor></mujoco>"""
  m = mjcf.load_string(x)
  np.testing.assert_array_equal(m.sensor_history, [[2, 1], [5, 1], [0, 1]])
  np.testing.assert_allclose(m.sensor_delay, [0.01, 0.01, 0.0])
  np.testing.assert_allclose(m.sensor_interval, [[0, 0], [0.1, 0.05], [0, 0]])
  np.testing.assert_array_equal(m.sensor_historyadr, [0, 6, -1])
  plain = mjcf.load_string("<mujoco><worldbody><body><joint name='j' type='slide'/><geom size='.1' mass='1'/></body></worldbody><actuator><motor joint='j'/></actuator></mujoco>")
  assert plain.nhistory == 0 and plain.actuator_historyadr.tolist() == [-1]


@pytest.mark.parametrize("attrs, match", [
  ('delay="0.02"', "delay > 0 needs a history buffer"),
  ('nsample="0" delay="0.02" interp="linear"', "delay > 0 needs a history buffer"),
  ('nsample="-1"', "nsample must be >= 0"),
  ('nsample="2" delay="-0.01"', "delay must be >= 0"),
])
def test_actuator_refusals(attrs, match):
  x = f"""<mujoco><worldbody><body><joint name="s" type="slide"/><geom size=".1" mass="1"/></body></worldbody>
  <actuator><motor name="m" joint="s" {attrs}/></actuator></mujoco>"""
  with pytest.raises(ValueError, match=f"actuator 0 \\('m'\\): {match}"):
    io._validate(mjcf.load_string(x))


@pytest.mark.parametrize("attrs, match", [
  ('interval="0.1"', "interval > 0 needs a history buffer"),
  ('nsample="2" interval="-0.1"', "interval period must be >= 0"),
  ('delay="0.01"', "delay > 0 needs a history buffer"),
])
def test_sensor_refusals(attrs, match):
  x = f"""<mujoco><worldbody><body><joint name="s" type="slide"/><geom size=".1" mass="1"/></body></worldbody>
  <sensor><jointpos name="p" joint="s" {attrs}/></sensor></mujoco>"""
  with pytest.raises(ValueError, match=f"sensor 0 \\('p'\\): {match}"):
    io._validate(mjcf.load_string(x))


def test_unknown_interp_is_refused():
  x = """<mujoco><worldbody><body><joint name="s" type="slide"/><geom size=".1" mass="1"/></body></worldbody>
  <actuator><motor joint="s" nsample="2" interp="spline"/></actuator></mujoco>"""
  with pytest.raises(ValueError, match="interp must be one of"):
    mjcf.load_string(x)


@pytest.mark.parametrize("field", ["actuator_delay", "sensor_delay"])
def test_delays_are_not_per_world(field):
  with pytest.raises(ValueError, match=f"'{field}' is shared by all worlds"):
    io.put_model(H.load("actuators"), batch_sizes={field: 4})


def test_state_history_width():
  from mujoco_warp_b200._src.forward import _state_fields
  from mujoco_warp_b200._src.types import State

  mjm = H.load("vectors")
  nw = 2
  d = types.SimpleNamespace(nworld=nw, history=torch.arange(nw * mjm.nhistory, dtype=torch.float32).reshape(nw, -1), act=torch.zeros(nw, 0),
                            qpos=torch.zeros(nw, mjm.nq), time=torch.zeros(nw))
  f = _state_fields(None, d, int(State.HISTORY))
  assert len(f) == 1 and tuple(f[0].shape) == (nw, mjm.nhistory)
  widths = [x.shape[1] for x in _state_fields(None, d, int(State.TIME | State.QPOS | State.ACT | State.HISTORY))]
  assert widths == [1, mjm.nq, 0, mjm.nhistory]  # the reference's bit order: TIME, QPOS, QVEL, ACT, HISTORY, ...


def _fresh_at(before, after, n, dim, t):
  """The value a step inserted at stamp t into a buffer (among equal stamps, the slot it changed), zeros if none."""
  val = lambda buf, i: buf[2 + n + i * dim : 2 + n + (i + 1) * dim]
  hit = [i for i in range(n) if abs(after[2 + i] - t) < 1e-9]
  hit = sorted(hit, key=lambda i: np.array_equal(val(before, i), val(after, i)))
  return val(after, hit[0]).copy() if hit else np.zeros(dim)


@pytest.mark.parametrize("scene", ["actuators", "dynamics", "vectors"])
def test_device_buffers_replay_the_reference_steps(hlib, scene):
  g, mjm = _golden(scene), H.load(scene)
  ah, aadr, adelay = mjm.actuator_history, mjm.actuator_historyadr, mjm.actuator_delay
  sh, sadr, sdelay, sint = mjm.sensor_history, mjm.sensor_historyadr, mjm.sensor_delay, mjm.sensor_interval
  checked = 0
  for k in range(H.SCENES[scene][1]):
    hin, hout = g[f"step/{k}/in_history"], g[f"step/{k}/out_history"]
    for w in range(H.NWORLD):
      t = float(g[f"step/{k}/in_time"][w])
      buf = hin[w].astype(np.float32).copy()
      for u in range(mjm.nu):
        n = int(ah[u, 0])
        if n == 0:
          continue
        b = buf[aadr[u] :]
        if adelay[u] > 0 and mjm.actuator_dyntype[u] == 0:  # a motor's force is its delayed ctrl
          v = np.zeros(1, np.float32)
          hlib.hh_read(_p(b), n, 1, np.float32(t - adelay[u]), int(ah[u, 1]), _p(v))
          np.testing.assert_allclose(v[0], g[f"step/{k}/out_actuator_force"][w, u], rtol=2e-6, atol=2e-6, err_msg=f"{scene} step {k} world {w} actuator {u}")
        c = np.array([g[f"step/{k}/in_ctrl"][w, u]], np.float32)
        hlib.hh_insert(_p(b), n, 1, np.float32(t), _p(c))
        checked += 1
      for s in range(int(mjm.nsensor)):
        n, dim = int(sh[s, 0]), int(mjm.sensor_dim[s])
        if n == 0:
          continue
        b = buf[sadr[s] :]
        data = _fresh_at(hin[w, sadr[s] :], hout[w, sadr[s] :], n, dim, t).astype(np.float32)
        hlib.hh_sensor(_p(b), n, dim, int(sh[s, 1]), np.float32(sdelay[s]), np.float32(sint[s, 0]), np.float32(t), _p(data))
        a = int(mjm.sensor_adr[s])
        np.testing.assert_allclose(data, g[f"step/{k}/out_sensordata"][w, a : a + dim], rtol=1e-5, atol=1e-6, err_msg=f"{scene} step {k} world {w} sensor {s}")
        checked += 1
      np.testing.assert_allclose(buf, hout[w], rtol=1e-6, atol=1e-7, err_msg=f"{scene} step {k} world {w} history")
  assert checked > 0


@pytest.mark.parametrize("scene", ["actuators", "vectors"])
def test_device_reads_replay_the_reference_functions(hlib, scene):
  g, mjm = _golden(scene), H.load(scene)
  last = H.SCENES[scene][1] - 1
  hist, tq = g[f"step/{last}/out_history"], g["fn/time"]
  for kind, count in (("ctrl", mjm.nu), ("sensor", mjm.nsensor)):
    for i in range(int(count)):
      hh = (mjm.actuator_history if kind == "ctrl" else mjm.sensor_history)[i]
      if hh[0] == 0:
        continue
      adr = (mjm.actuator_historyadr if kind == "ctrl" else mjm.sensor_historyadr)[i]
      delay = (mjm.actuator_delay if kind == "ctrl" else mjm.sensor_delay)[i]
      dim = 1 if kind == "ctrl" else int(mjm.sensor_dim[i])
      for interp in (-1, 0, 1, 2):
        want = g[f"fn/read_{kind}/{i}/{interp}"].reshape(H.NWORLD, dim)
        for w in range(H.NWORLD):
          out = np.zeros(dim, np.float32)
          hlib.hh_read(_p(hist[w, adr:].astype(np.float32)), int(hh[0]), dim, np.float32(tq[w] - delay), int(hh[1] if interp < 0 else interp), _p(out))
          np.testing.assert_allclose(out, want[w], rtol=1e-5, atol=1e-6, err_msg=f"{kind} {i} interp {interp} world {w}")
