"""Recompute the Model constants the compiler derives from other Model fields (reference set_const.py:613-950).

After a user changes `body_mass`, `body_inertia`, `body_ipos`, `qpos0`, `dof_armature`, ... -- per world, for domain randomisation --
the derived fields the kernels read every step (`body_subtreemass`, the constraint weights `dof_invweight0` / `body_invweight0` /
`tendon_invweight0`, `stat.meaninertia`, `eq_data`, the camera / light reference poses, ...) describe the old model until these
functions recompute them.  Each is one call through the C-ABI (`mjb_set_const`, `k_set_const.cu`) on the current torch CUDA stream.

Batched outputs: entry i of a derived field is computed from world i, for i below that field's leading size; a field left unbatched
gets world 0's result.  An output field with more entries than `d.nworld` raises `ValueError`.

`stat.meaninertia` stays a Model scalar, as the solver reads it: the C call writes world 0's value to `m.stat.meaninertia` on the
device, and these wrappers then synchronise the stream once and hand the value to the library.  So the Python functions cannot be
captured in a CUDA graph; the C entry point `mjb_set_const` can (it neither allocates nor synchronises), after which the caller
assigns `m.stat.meaninertia` itself.
"""

from __future__ import annotations

import torch

from . import _lib
from .types import Data, Model

FIXED, ZERO, SPRING = 1, 2, 4  # MJB_SET_CONST_FIXED / _0 / _SPRING (include/mjb200.h)

_OUTPUTS = {
  FIXED: ("body_subtreemass",),
  ZERO: ("tendon_length0", "eq_data", "dof_invweight0", "body_invweight0", "tendon_invweight0", "cam_pos0", "cam_poscom0", "cam_mat0",
         "light_pos0", "light_poscom0", "light_dir0", "actuator_acc0", "actuator_biasprm"),
  SPRING: ("tendon_lengthspring",),
}


def output_fields(parts: int):
  """The Model fields a call with `parts` (FIXED | ZERO | SPRING) writes, besides `stat.meaninertia` (ZERO)."""
  return tuple(f for p in (FIXED, ZERO, SPRING) if parts & p for f in _OUTPUTS[p])


def _set_const(m: Model, d: Data, parts: int, restore: bool):
  if not isinstance(m, Model) or not isinstance(d, Data):
    raise TypeError(f"expected (Model, Data), got ({type(m).__name__}, {type(d).__name__})")
  if d._model is not m and d._model._handle != m._handle:
    raise ValueError("Data was created for a different Model")
  if parts & SPRING and m.ntendon == 0:
    parts &= ~SPRING  # set_const.py:853: nothing depends on qpos_spring without tendons
    if not parts:
      return
  for name in output_fields(parts):
    n = int(getattr(m, name).shape[0])
    if n > d.nworld:
      raise ValueError(f"Model.{name} has {n} per-world entries but Data has {d.nworld} worlds: entry i is computed from world i")
  stream = torch.cuda.current_stream()
  _lib.check(_lib.lib().mjb_set_const(m._handle, d._handle, parts, int(bool(restore)), stream.cuda_stream))
  if parts & ZERO:
    stream.synchronize()
    m.stat.meaninertia = m.stat.meaninertia  # the Statistic hook passes world 0's new value to the solver's scalar


def set_const_fixed(m: Model, d: Data):
  """body_subtreemass from body_mass (set_const.py:613)."""
  _set_const(m, d, FIXED, False)


def set_const_0(m: Model, d: Data, restore: bool = True):
  """The fields that depend on qpos0 (set_const.py:634): stat.meaninertia, tendon_length0, eq_data (connect / weld anchors and relative
  pose; a weld whose quaternion is set is only normalised), dof_invweight0, body_invweight0, tendon_invweight0, cam_pos0 / poscom0 /
  mat0, light_pos0 / poscom0 / dir0, actuator_acc0 and the dampratio form of position actuators (actuator_biasprm[2]).  d.qpos is
  restored; with `restore`, the position stages and the factor of M are recomputed at it."""
  _set_const(m, d, ZERO, restore)


def set_const_spring(m: Model, d: Data, restore: bool = True):
  """tendon_lengthspring entries that are (-1, -1) become the tendon length at qpos_spring (set_const.py:847)."""
  _set_const(m, d, SPRING, restore)


def set_const(m: Model, d: Data, restore: bool = True):
  """set_const_fixed, set_const_0 and set_const_spring, then (with `restore`) the position stages and the factor of M at d.qpos
  (set_const.py:881).  Call it after changing body masses, inertias, qpos0, qpos_spring, armature, eq_data or dampratio actuators."""
  _set_const(m, d, FIXED | ZERO | SPRING, restore)


def set_length_range(m: Model, d: Data, index: int = -1):
  """actuator_lengthrange from the joint and tendon limits (set_const.py:952): an actuator on a limited joint or limited fixed tendon
  gets the limit range times gear[0], ends swapped for a negative gear; every other actuator gets (0, 0).  As in the reference, every
  actuator is computed whatever `index` is (-1 or an actuator id).  Entry i of a batched `m.actuator_lengthrange` is computed from
  world i; call it after changing `jnt_range`, `tendon_range` or `actuator_gear` of a model with muscles."""
  if not isinstance(m, Model) or not isinstance(d, Data):
    raise TypeError(f"expected (Model, Data), got ({type(m).__name__}, {type(d).__name__})")
  if d._model is not m and d._model._handle != m._handle:
    raise ValueError("Data was created for a different Model")
  if not -1 <= int(index) < m.nu:
    raise ValueError(f"index must be -1 or an actuator id in [0, {m.nu}), got {index}")
  if m.nu == 0:
    return
  n = int(m.actuator_lengthrange.shape[0])
  if n > d.nworld:
    raise ValueError(f"Model.actuator_lengthrange has {n} per-world entries but Data has {d.nworld} worlds: entry i is computed from world i")
  _lib.check(_lib.lib().mjb_set_length_range(m._handle, d._handle, int(index), torch.cuda.current_stream().cuda_stream))
