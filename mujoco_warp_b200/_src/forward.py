"""Public pipeline functions: step, forward and the individually callable stages.

Same names and `(m, d)` signatures as /root/reference/mujoco_warp/__init__.py:26-123 (forward.py:1368 step, :1341 forward,
:635 fwd_position, smooth.py kinematics/com_pos/camlight/crb/factor_m/transmission, collision_driver.py:884 collision,
constraint.py:4897 make_constraint, forward.py:732/1152/1290 fwd_velocity/fwd_actuation/fwd_acceleration, solver.py:3671 solve,
forward.py:387 euler).  Each is one call through the C-ABI on the current torch CUDA stream; `d` is mutated in place;
nothing synchronises the device, so sequences are capturable with torch.cuda.graphs.
"""

from __future__ import annotations

import torch

from . import _lib
from .types import Data, Model


def _call(name: str, m: Model, d: Data):
  if d._model is not m and d._model._handle != m._handle:
    raise ValueError("Data was created for a different Model")
  stream = torch.cuda.current_stream().cuda_stream
  _lib.check(getattr(_lib.lib(), name)(m._handle, d._handle, stream))


def step(m: Model, d: Data):
  """Advance simulation (forward dynamics + Euler integration)."""
  _call("mjb_step", m, d)


def forward(m: Model, d: Data):
  """Forward dynamics."""
  _call("mjb_forward", m, d)


def fwd_position(m: Model, d: Data):
  """Position-dependent computations (kinematics .. make_constraint, transmission)."""
  _call("mjb_fwd_position", m, d)


def kinematics(m: Model, d: Data):
  _call("mjb_kinematics", m, d)


def com_pos(m: Model, d: Data):
  _call("mjb_com_pos", m, d)


def camlight(m: Model, d: Data):
  _call("mjb_camlight", m, d)


def crb(m: Model, d: Data):
  _call("mjb_crb", m, d)


def factor_m(m: Model, d: Data):
  _call("mjb_factor_m", m, d)


def transmission(m: Model, d: Data):
  _call("mjb_transmission", m, d)


def collision(m: Model, d: Data):
  _call("mjb_collision", m, d)


def make_constraint(m: Model, d: Data):
  _call("mjb_make_constraint", m, d)


def fwd_velocity(m: Model, d: Data):
  _call("mjb_fwd_velocity", m, d)


def fwd_actuation(m: Model, d: Data):
  _call("mjb_fwd_actuation", m, d)


def fwd_acceleration(m: Model, d: Data):
  _call("mjb_fwd_acceleration", m, d)


def solve(m: Model, d: Data):
  _call("mjb_solve", m, d)


def euler(m: Model, d: Data):
  _call("mjb_euler", m, d)


def sensor_pos(m: Model, d: Data):
  """Position-stage sensors (reference sensor.py:810); forward() / step() already evaluate every stage after the solver."""
  _call("mjb_sensor_pos", m, d)


def sensor_vel(m: Model, d: Data):
  """Velocity-stage sensors, with subtree_vel when a sensor needs it (reference sensor.py:1432)."""
  _call("mjb_sensor_vel", m, d)


def sensor_acc(m: Model, d: Data):
  """Acceleration-stage sensors, with the cacc part of rne_postconstraint when an accelerometer needs it (reference sensor.py:2512)."""
  _call("mjb_sensor_acc", m, d)


def energy_pos(m: Model, d: Data):
  """Potential energy into d.energy[:, 0] (reference sensor.py:2934): -sum_b body_mass[b] gravity . xipos[b] unless gravity is
  disabled, plus 1/2 k x^2 of every joint spring (hinge / slide: q - qpos_spring; ball / free: the rotation from qpos_spring, and the
  free joint's translation) and fixed-tendon spring (x: the length outside the springlength dead band) unless springs are disabled.
  Reads the last position stage; runs whatever `EnableBit.ENERGY` says."""
  _call("mjb_energy_pos", m, d)


def energy_vel(m: Model, d: Data):
  """Kinetic energy 1/2 qvel . (M qvel) into d.energy[:, 1] (reference sensor.py:3004), with the M (armature included) of the last crb.
  Runs whatever `EnableBit.ENERGY` says."""
  _call("mjb_energy_vel", m, d)


def rungekutta4(m: Model, d: Data):
  """Runge-Kutta 4 integrator, to be called after forward() (reference forward.py:523); the model must use the RK4 integrator."""
  from . import constants as C

  if m.opt.integrator != C.INT_RK4:
    raise NotImplementedError("rungekutta4(): the model was put with another integrator (the RK scratch is allocated per model)")
  _call("mjb_rungekutta4", m, d)


def implicit(m: Model, d: Data):
  """Integrates implicitly in velocity (reference forward.py:578): the full velocity derivative with an LU solve when the model's
  integrator is IMPLICIT, the symmetric implicitfast variant when it is IMPLICITFAST.  (The reference also runs the implicitfast branch
  for Euler / RK4 models; here the factor-and-solve scratch is sized by the model's integrator at put_model, so those raise.)"""
  from . import constants as C

  if m.opt.integrator not in (C.INT_IMPLICITFAST, C.INT_IMPLICIT):
    raise NotImplementedError("implicit(): the model was put with the Euler / RK4 integrator (scratch is sized per integrator)")
  _call("mjb_implicit", m, d)


def fwd_kinematics(m: Model, d: Data):
  """kinematics, com_pos, camlight (reference forward.py:613-632; no flex / tendon in this version)."""
  kinematics(m, d)
  com_pos(m, d)
  camlight(m, d)


def com_vel(m: Model, d: Data):
  """Body velocities cvel and cdof_dot (reference smooth.py:2261)."""
  _call("mjb_com_vel", m, d)


def passive(m: Model, d: Data):
  """Passive joint forces: springs and dampers (reference passive.py:1257)."""
  _call("mjb_passive", m, d)


def rne(m: Model, d: Data, flg_acc: bool = False):
  """Bias forces by recursive Newton-Euler (reference smooth.py:1499)."""
  if flg_acc:
    raise NotImplementedError("rne(flg_acc=True) is not implemented")
  _call("mjb_rne", m, d)


def _vec_call(name: str, m: Model, d: Data, out: torch.Tensor, inp: torch.Tensor):
  for t in (out, inp):
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or tuple(t.shape) != (d.nworld, m.nv):
      raise ValueError(f"expected a contiguous CUDA float32 tensor of shape ({d.nworld}, {m.nv})")
  stream = torch.cuda.current_stream().cuda_stream
  _lib.check(getattr(_lib.lib(), name)(m._handle, d._handle, out.data_ptr(), inp.data_ptr(), stream))


def solve_m(m: Model, d: Data, x: torch.Tensor, y: torch.Tensor):
  """x = M^-1 y using the factor in d.qLD (reference smooth.py:3214)."""
  _vec_call("mjb_solve_m", m, d, x, y)


def mul_m(m: Model, d: Data, res: torch.Tensor, vec: torch.Tensor):
  """res = M vec (reference support.py:153)."""
  _vec_call("mjb_mul_m", m, d, res, vec)


def contact_force(m: Model, d: Data, contact_ids: torch.Tensor, to_world_frame: bool, force: torch.Tensor):
  """6D force / torque of the listed contacts into force (n, 6), in the contact frame unless to_world_frame
  (reference support.py:445; contact ids index the global contact pool)."""
  n = int(contact_ids.numel())
  if contact_ids.dtype != torch.int32 or not contact_ids.is_cuda or not contact_ids.is_contiguous():
    raise ValueError("contact_ids: expected a contiguous CUDA int32 tensor")
  if force.dtype != torch.float32 or not force.is_cuda or not force.is_contiguous() or tuple(force.shape) != (n, 6):
    raise ValueError(f"force: expected a contiguous CUDA float32 tensor of shape ({n}, 6)")
  stream = torch.cuda.current_stream().cuda_stream
  _lib.check(_lib.lib().mjb_contact_force(m._handle, d._handle, contact_ids.data_ptr(), n, int(bool(to_world_frame)), force.data_ptr(), stream))


def rne_postconstraint(m: Model, d: Data):
  """Per-body accelerations d.cacc, internal wrenches d.cfrc_int and external wrenches d.cfrc_ext (applied, connect / weld equality and
  contact) after the constraint solve (reference smooth.py:1744).  Reads the finished forward pass; runs whatever the model's sensors or
  DisableBit.SENSOR say.  Equality and contact wrenches are summed in row and contact-pool order, so the result is bit-reproducible."""
  _call("mjb_rne_postconstraint", m, d)


def subtree_vel(m: Model, d: Data):
  """Subtree linear velocity d.subtree_linvel and angular momentum d.subtree_angmom of every body (reference smooth.py:3614).  Reads the
  last position and velocity stages; runs whatever the model's sensors or DisableBit.SENSOR say."""
  _call("mjb_subtree_vel", m, d)


def tendon(m: Model, d: Data):
  """Fixed-tendon lengths d.ten_length and Jacobians d.ten_J at the current qpos (reference smooth.py:4197); only fixed tendons exist here,
  so there are no wrap outputs.  Launches nothing for a model without tendons."""
  _call("mjb_tendon", m, d)


def _check_f32(name: str, t, shape):
  if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
    raise ValueError(f"{name}: expected a contiguous CUDA float32 tensor of shape {tuple(shape)}")


def jac(m: Model, d: Data, jacp: torch.Tensor | None, jacr: torch.Tensor | None, point: torch.Tensor, body: torch.Tensor):
  """Translational (jacp) and rotational (jacr) Jacobian of a world-frame point on a body, one per world (reference support.py:583).

  point: (nworld, 3) float32; body: (nworld,) int32 body ids; jacp / jacr: (nworld, 3, nv) float32 outputs, either may be None.  Every
  entry is written: columns of dofs that do not move the body are 0.  A body id outside [0, nbody) cannot be checked without a
  synchronisation: that world's rows are written as NaN instead.  A model without dofs launches nothing."""
  nw = d.nworld
  _check_f32("point", point, (nw, 3))
  if not isinstance(body, torch.Tensor) or body.dtype != torch.int32 or not body.is_cuda or not body.is_contiguous() or tuple(body.shape) != (nw,):
    raise ValueError(f"body: expected a contiguous CUDA int32 tensor of shape ({nw},)")
  for name, t in (("jacp", jacp), ("jacr", jacr)):
    if t is not None:
      _check_f32(name, t, (nw, 3, m.nv))
  stream = torch.cuda.current_stream().cuda_stream
  ptr = lambda t: t.data_ptr() if t is not None else None
  _lib.check(_lib.lib().mjb_jac(m._handle, d._handle, ptr(jacp), ptr(jacr), point.data_ptr(), body.data_ptr(), stream))


def xfrc_accumulate(m: Model, d: Data, qfrc: torch.Tensor):
  """Adds d.xfrc_applied, mapped to joint space through each body's Jacobian at its centre of mass, into qfrc (nworld, nv) float32
  (reference support.py:314).  Bodies are summed in index order, so the result is bit-reproducible."""
  _check_f32("qfrc", qfrc, (d.nworld, m.nv))
  stream = torch.cuda.current_stream().cuda_stream
  _lib.check(_lib.lib().mjb_xfrc_accumulate(m._handle, d._handle, qfrc.data_ptr(), stream))


def deriv_smooth_vel(m: Model, d: Data, out: torch.Tensor):
  """out (nworld, nC) float32 = M - dt qDeriv in the layout of d.M (M_rowadr / M_colind), for any integrator (reference
  derivative.py:1117).  qDeriv holds the derivatives of the smooth forces with respect to qvel: affine actuator gain / bias (unless
  DisableBit.ACTUATION), dof and tendon damping (unless DisableBit.DAMPER), and the fluid forces of a model that has them.  As in the
  reference, an ellipsoid's fluid derivative is symmetrized when the model's integrator is implicitfast and used as it stands otherwise."""
  _check_f32("out", out, (d.nworld, m.nC))
  stream = torch.cuda.current_stream().cuda_stream
  _lib.check(_lib.lib().mjb_deriv_smooth_vel(m._handle, d._handle, out.data_ptr(), stream))


_STATE_ORDER = ("TIME", "QPOS", "QVEL", "ACT", "HISTORY", "WARMSTART", "CTRL", "QFRC_APPLIED", "XFRC_APPLIED", "EQ_ACTIVE", "MOCAP_POS", "MOCAP_QUAT", "USERDATA")


def _state_fields(m: Model, d: Data, sig: int):
  """(tensor, width) of every state component selected by sig, in bit order (reference support.py:722-790)."""
  from .types import State

  if sig >= (1 << int(State.NSTATE)):
    raise ValueError(f"invalid state signature {sig} >= 2^mjNSTATE")
  nw = d.nworld
  out = []
  for name in _STATE_ORDER:
    if not (int(getattr(State, name)) & sig):
      continue
    t = {
      "TIME": lambda: d.time.reshape(nw, 1), "QPOS": lambda: d.qpos, "QVEL": lambda: d.qvel, "WARMSTART": lambda: d.qacc_warmstart,
      "CTRL": lambda: d.ctrl, "QFRC_APPLIED": lambda: d.qfrc_applied, "XFRC_APPLIED": lambda: d.xfrc_applied.reshape(nw, -1),
      "ACT": lambda: d.act, "HISTORY": lambda: d.history, "EQ_ACTIVE": lambda: d.eq_active.reshape(nw, -1), "MOCAP_POS": lambda: d.mocap_pos.reshape(nw, -1), "MOCAP_QUAT": lambda: d.mocap_quat.reshape(nw, -1),
    }.get(name)
    if t is None:  # USERDATA: no user data in this build (width 0)
      continue
    out.append(t())
  return out


def get_state(m: Model, d: Data, state: torch.Tensor, sig: int, active: torch.Tensor = None):
  """Copy the state components selected by the State bit flags in sig from Data into state (nworld, size), concatenated in
  bit order; worlds whose `active` entry is False are left untouched (reference support.py:674)."""
  fields = _state_fields(m, d, int(sig))
  if not fields:
    return
  cat = torch.cat([f.to(torch.float32) for f in fields], dim=1)
  dst = state[:, : cat.shape[1]]
  dst.copy_(cat if active is None else torch.where(active.reshape(-1, 1).bool(), cat, dst))


def set_state(m: Model, d: Data, state: torch.Tensor, sig: int, active: torch.Tensor = None):
  """Inverse of get_state (reference support.py:829)."""
  adr = 0
  for f in _state_fields(m, d, int(sig)):
    w = f.shape[1]
    src = state[:, adr : adr + w].to(f.dtype)
    f.copy_(src if active is None else torch.where(active.reshape(-1, 1).bool(), src, f))
    adr += w


def step1(m: Model, d: Data):
  """First half of a split step, before the user sets controls (reference forward.py:1384 step1: position and velocity stages
  with their sensors, and energy).  With `EnableBit.ENERGY` set d.energy gets both terms; without it a model with e_potential /
  e_kinetic sensors ends with d.energy zeroed, as the reference leaves it, and any other model leaves d.energy untouched."""
  from . import constants as C

  fwd_position(m, d)
  if getattr(m, "nsensor", 0):
    d.sensordata.zero_()
    sensor_pos(m, d)
  energy_on = bool(m.opt.enableflags & C.ENBL_ENERGY)
  if energy_on:
    energy_pos(m, d)
  elif len(m.sensor_energy_adr):
    d.energy.zero_()
  fwd_velocity(m, d)
  if getattr(m, "nsensor", 0):
    sensor_vel(m, d)
  if energy_on:
    energy_vel(m, d)


def step2(m: Model, d: Data):
  """Second half of a split step (reference forward.py step2)."""
  from . import constants as C

  fwd_actuation(m, d)
  fwd_acceleration(m, d)
  solve(m, d)
  if getattr(m, "nsensor", 0):
    sensor_acc(m, d)
  if m.opt.integrator in (C.INT_IMPLICITFAST, C.INT_IMPLICIT):
    implicit(m, d)
  else:
    euler(m, d)


def ctrl_noise(m: Model, d: Data, step_index: int, ctrl_center: torch.Tensor | None = None, noise_std: float = 0.01, noise_rate: float = 0.1):
  """Harness OU control noise (reference cli.py:103-145), deterministic Halton sequence per (step, world, actuator)."""
  stream = torch.cuda.current_stream().cuda_stream
  ptr = ctrl_center.data_ptr() if ctrl_center is not None else None
  _lib.check(_lib.lib().mjb_ctrl_noise(m._handle, d._handle, ptr, int(step_index), float(noise_std), float(noise_rate), stream))


def last_launch_count() -> int:
  return int(_lib.lib().mjb_last_launch_count())


KERNEL_NAMES = ("position", "collision", "constraint", "velocity", "solver", "integrate")


def step_profile(m: Model, d: Data):
  """One step's kernel chain over all worlds with a CUDA event after each stage group; returns {group: ms} for the groups of
  KERNEL_NAMES.  `constraint` includes the CSR view of sparse models, `solver` the sensors, `integrate` every integrator kernel.
  RK4 models profile one forward pass and the Euler update.  Synchronises (profiling aid)."""
  import ctypes

  out = (ctypes.c_float * 6)()
  stream = torch.cuda.current_stream().cuda_stream
  _lib.check(_lib.lib().mjb_step_profile(m._handle, d._handle, stream, out))
  return dict(zip(KERNEL_NAMES, [float(x) for x in out]))


def collision_kernel(m: Model) -> str:
  """Name of the kernel the collision stage launches for m: "k_collision" (no mesh geoms), "k_collision_mesh", or "k_collision_mesh_large"
  (a hull polygon of more than 32 vertices or a hull vertex in more than 16 polygons: multi-contact buffers sized from the model, in global
  scratch that make_data allocates; the collision sensors then run the same build).  Its time is step_profile()'s "collision"."""
  name = _lib.lib().mjb_collision_kernel(m._handle)
  if name is None:
    _lib.check(-1)
  return name.decode()


TEAM_INSTANCES = ("plain", "pext", "fluid")


def team_residency(m: Model, d: Data, shapes: bool = False):
  """Worlds per SM resident at once in the launch shape of k_position / k_velocity for all of d's worlds (occupancy API);
  returns {"position": n, "velocity": n}.  With shapes=True each kernel maps to the launch shape as well:
  {"worlds_per_sm": n, "lpw": lanes per world, "wpb": warps per block, "block_bytes": shared memory per block,
  "instance": "plain" | "pext" | "fluid" (k_position is always "plain")}."""
  import ctypes

  f = _lib.lib().mjb_team_residency
  f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
  pos, vel, sh = ctypes.c_int(), ctypes.c_int(), (ctypes.c_int * 8)()
  _lib.check(f(m._handle, d._handle, ctypes.byref(pos), ctypes.byref(vel), sh))
  if not shapes:
    return {"position": pos.value, "velocity": vel.value}
  return {k: {"worlds_per_sm": n, "lpw": sh[i], "wpb": sh[i + 1], "block_bytes": sh[i + 2], "instance": TEAM_INSTANCES[sh[i + 3]]}
          for k, n, i in (("position", pos.value, 0), ("velocity", vel.value, 4))}
