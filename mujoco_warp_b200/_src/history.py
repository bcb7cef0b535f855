"""Actuator and sensor delays: the public functions of the reference's history.py (:634 read_ctrl, :718 read_sensor, :796
init_ctrl_history, :881 init_sensor_history), one kernel launch each (k_history.cu) on the current torch CUDA stream.

The buffers themselves live in `d.history` (nworld, nhistory); `forward` / `step` read and fill them.  Arrays are torch tensors
where the reference takes `wp.array`s.
"""

from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .types import Data, Model

MJ_MINVAL = 1e-15


def _f32(name, t, numel):
  if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or t.numel() != numel:
    raise ValueError(f"{name}: expected a contiguous CUDA float32 tensor with {numel} entries")
  return t.data_ptr()


def _check(m: Model, d: Data, kind: str, i: int):
  if d._model is not m and d._model._handle != m._handle:
    raise ValueError("Data was created for a different Model")
  n = m.nu if kind == "actuator" else m.nsensor
  if not 0 <= int(i) < n:
    raise ValueError(f"{kind} id {i} out of range [0, {n})")
  return int(m._history[kind + "_history"][int(i), 0]), (1 if kind == "actuator" else int(m._mjm.sensor_dim[int(i)]))


def _read(name, m, d, kind, i, time, interp, result):
  _, dim = _check(m, d, kind, i)
  if int(interp) not in (-1, 0, 1, 2):
    raise ValueError(f"interp must be -1 (the model's), 0 (zoh), 1 (linear) or 2 (cubic), got {interp}")
  args = (_f32("time", time, d.nworld), int(interp), _f32("result", result, d.nworld * dim))
  _lib.check(getattr(_lib.lib(), name)(m._handle, d._handle, int(i), *args, torch.cuda.current_stream().cuda_stream))


def _times(times, nsample):
  """Device pointer of the stamps, or None for -MJ_MAXVAL stamps; refuses stamps that are not strictly increasing (history.py:816-820)."""
  if times is None:
    return None
  t = times.detach().cpu().numpy().astype(np.float64).reshape(-1)
  for k in range(len(t) - 1):
    if t[k + 1] - t[k] < MJ_MINVAL:
      raise ValueError(f"times must be strictly increasing, got times[{k}]={t[k]} >= times[{k + 1}]={t[k + 1]}")
  return _f32("times", times, nsample)


def read_ctrl(m: Model, d: Data, ctrlid: int, time: torch.Tensor, interp: int, result: torch.Tensor):
  """Delayed ctrl of actuator `ctrlid` in every world: its buffer read at time[w] - actuator_delay into result (nworld,), with interp
  -1 (the model's), 0 zero-order hold, 1 linear or 2 cubic; d.ctrl[:, ctrlid] for an actuator without a buffer (history.py:634)."""
  _read("mjb_read_ctrl", m, d, "actuator", ctrlid, time, interp, result)


def read_sensor(m: Model, d: Data, sensorid: int, time: torch.Tensor, interp: int, result: torch.Tensor):
  """Delayed value of sensor `sensorid` in every world: its buffer read at time[w] - sensor_delay into result (nworld, dim); the current
  sensordata for a sensor without a buffer (history.py:718)."""
  _read("mjb_read_sensor", m, d, "sensor", sensorid, time, interp, result)


def init_ctrl_history(m: Model, d: Data, ctrlid: int, times: torch.Tensor | None, values: torch.Tensor):
  """Fills the buffer of actuator `ctrlid` in every world from times (nsample,), strictly increasing, or None (every stamp
  -MJ_MAXVAL) and values (nworld, nsample), newest last; the user slot is kept (history.py:796).  ValueError if the times are not
  strictly increasing or the actuator has no buffer."""
  n, _ = _check(m, d, "actuator", ctrlid)
  if n == 0:
    raise ValueError(f"actuator {ctrlid} has no history buffer (nsample = 0)")
  ptimes = _times(times, n)
  _lib.check(_lib.lib().mjb_init_ctrl_history(m._handle, d._handle, int(ctrlid), ptimes, _f32("values", values, d.nworld * n), torch.cuda.current_stream().cuda_stream))


def init_sensor_history(m: Model, d: Data, sensorid: int, times: torch.Tensor | None, values: torch.Tensor, phase: torch.Tensor):
  """Fills the buffer of sensor `sensorid` in every world from times (nsample,) or None and values (nworld, nsample * dim), newest
  last; the user slot becomes phase[w], the last time an interval sensor was due (history.py:881)."""
  n, dim = _check(m, d, "sensor", sensorid)
  if n == 0:
    raise ValueError(f"sensor {sensorid} has no history buffer (nsample = 0)")
  ptimes = _times(times, n)
  _lib.check(_lib.lib().mjb_init_sensor_history(m._handle, d._handle, int(sensorid), ptimes, _f32("values", values, d.nworld * n * dim), _f32("phase", phase, d.nworld),
                                                torch.cuda.current_stream().cuda_stream))
