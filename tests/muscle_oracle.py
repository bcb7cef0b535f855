"""fp64 restatement of MuJoCo's muscle model and of the actuation stage for muscles (tests/test_muscle_host.py, tests/test_gpu_muscle.py).

Written from the formulas (MuJoCo's engine_util_misc.c / the reference's util_misc.py:455-600 and forward.py:800-1040): the length-gain
and force-velocity curves, the passive force, the Millard activation dynamics with quintic-sigmoid smoothing, and the force of one
actuator from its ctrl, activation, length and velocity.  `fp32=True` evaluates the same expressions in float32.

`MuscleStep` is a whole fp64 step of a muscle model, per world: the pipeline oracle (oracle/orc.py) with the muscles taken out of the
model and their forces, computed here, applied as generalized forces.  The pipeline oracle itself has no muscle model: a model with
muscles must go through `MuscleStep`, never to orc.Oracle directly, whose actuation would give the muscles zero force.
"""
import numpy as np

MJ_MINVAL = 1e-15


def _f(fp32):
  return np.float32 if fp32 else np.float64


def gain_length(L, lmin, lmax, fp32=False):
  t = _f(fp32)
  L, lmin, lmax = t(L), t(lmin), t(lmax)
  if lmin > L or L > lmax:
    return t(0)
  a, b = t(0.5) * (lmin + t(1)), t(0.5) * (t(1) + lmax)
  mv = t(MJ_MINVAL)
  if L <= a:
    x = (L - lmin) / max(mv, a - lmin)
    return t(0.5) * x * x
  if L <= 1:
    x = (t(1) - L) / max(mv, t(1) - a)
    return t(1) - t(0.5) * x * x
  if L <= b:
    x = (L - t(1)) / max(mv, b - t(1))
    return t(1) - t(0.5) * x * x
  x = (lmax - L) / max(mv, lmax - b)
  return t(0.5) * x * x


def _force_L0(prm, lr, acc0, fp32):
  t = _f(fp32)
  mv = t(MJ_MINVAL)
  force = t(prm[3]) / max(mv, t(acc0)) if prm[2] < 0 else t(prm[2])
  L0 = (t(lr[1]) - t(lr[0])) / max(mv, t(prm[1]) - t(prm[0]))
  return force, L0


def gain(length, velocity, lr, acc0, prm, fp32=False):
  t = _f(fp32)
  mv = t(MJ_MINVAL)
  force, L0 = _force_L0(prm, lr, acc0, fp32)
  L = t(prm[0]) + (t(length) - t(lr[0])) / max(mv, L0)
  V = t(velocity) / max(mv, L0 * t(prm[6]))
  FL = gain_length(L, prm[4], prm[5], fp32)
  fvmax = t(prm[8])
  y = fvmax - t(1)
  if V <= -1:
    FV = t(0)
  elif V <= 0:
    FV = (V + t(1)) * (V + t(1))
  elif V <= y:
    FV = fvmax - (y - V) * (y - V) / max(mv, y)
  else:
    FV = fvmax
  return -force * FL * FV


def bias(length, lr, acc0, prm, fp32=False):
  t = _f(fp32)
  mv = t(MJ_MINVAL)
  force, L0 = _force_L0(prm, lr, acc0, fp32)
  L = t(prm[0]) + (t(length) - t(lr[0])) / max(mv, L0)
  b = t(0.5) * (t(1) + t(prm[5]))
  fpmax = t(prm[7])
  if L <= 1:
    return t(0)
  if L <= b:
    x = (L - t(1)) / max(mv, b - t(1))
    return -force * fpmax * t(0.5) * x * x
  x = (L - b) / max(mv, b - t(1))
  return -force * fpmax * (t(0.5) + x)


def sigmoid(x, fp32=False):
  t = _f(fp32)
  x = t(x)
  if x <= 0:
    return t(0)
  if x >= 1:
    return t(1)
  return x * x * x * (t(3) * x * (t(2) * x - t(5)) + t(10))


def timescale(dctrl, tau_act, tau_deact, smooth_width, fp32=False):
  t = _f(fp32)
  if t(smooth_width) < t(MJ_MINVAL):
    return t(tau_act) if dctrl > 0 else t(tau_deact)
  return t(tau_deact) + (t(tau_act) - t(tau_deact)) * sigmoid(t(dctrl) / t(smooth_width) + t(0.5), fp32)


def dynamics(ctrl, act, prm, fp32=False):
  t = _f(fp32)
  ctrlclamp = min(max(t(ctrl), t(0)), t(1))
  actclamp = min(max(t(act), t(0)), t(1))
  tau_act = t(prm[0]) * (t(0.5) + t(1.5) * actclamp)
  tau_deact = t(prm[1]) / (t(0.5) + t(1.5) * actclamp)
  dctrl = ctrlclamp - t(act)
  tau = timescale(dctrl, tau_act, tau_deact, prm[2], fp32)
  return dctrl / max(t(MJ_MINVAL), tau)


def actuation(mjm, ctrl, act, length, velocity, timestep, gainprm=None, biasprm=None, acc0=None, lengthrange=None):
  """(act_dot, actuator_force) of one world in fp64 (forward.py:776-1040) for a model whose actuators are muscles, fixed / affine
  gain and affine bias, with NONE / INTEGRATOR / FILTER / FILTEREXACT / MUSCLE dynamics.  gainprm / biasprm / acc0 / lengthrange
  default to the model's (pass a world's row of a batched field instead)."""
  from mujoco_warp_b200._src import constants as C

  nu, na = int(mjm.nu), int(mjm.na)
  gp = np.asarray(mjm.actuator_gainprm if gainprm is None else gainprm, dtype=np.float64).reshape(nu, 10)
  bp = np.asarray(mjm.actuator_biasprm if biasprm is None else biasprm, dtype=np.float64).reshape(nu, 10)
  a0 = np.asarray(mjm.actuator_acc0 if acc0 is None else acc0, dtype=np.float64).reshape(nu)
  lr = np.asarray(mjm.actuator_lengthrange if lengthrange is None else lengthrange, dtype=np.float64).reshape(nu, 2)
  dp = np.asarray(mjm.actuator_dynprm, dtype=np.float64).reshape(nu, 10)
  act_dot, force = np.zeros(na), np.zeros(nu)
  for i in range(nu):
    c = float(ctrl[i])
    if mjm.actuator_ctrllimited[i]:
      c = min(max(c, mjm.actuator_ctrlrange[i][0]), mjm.actuator_ctrlrange[i][1])
    ca = c
    adr = int(mjm.actuator_actadr[i])
    dyn = int(mjm.actuator_dyntype[i])
    if na and adr >= 0:
      last = adr + int(mjm.actuator_actnum[i]) - 1
      a = float(act[last])
      ad = 0.0
      if dyn == C.DYN_INTEGRATOR:
        ad = c
      elif dyn in (C.DYN_FILTER, C.DYN_FILTEREXACT):
        ad = (c - a) / max(dp[i, 0], MJ_MINVAL)
      elif dyn == C.DYN_MUSCLE:
        ad = dynamics(c, a, dp[i])
      act_dot[last] = ad
      if mjm.actuator_actearly[i]:
        if dyn == C.DYN_FILTEREXACT:
          tau = max(MJ_MINVAL, dp[i, 0])
          ca = a + ad * tau * (1.0 - np.exp(-timestep / tau))
        else:
          ca = a + ad * timestep
        if mjm.actuator_actlimited[i]:
          ca = min(max(ca, mjm.actuator_actrange[i][0]), mjm.actuator_actrange[i][1])
      else:
        ca = a
    g, b = 0.0, 0.0
    gt, bt = int(mjm.actuator_gaintype[i]), int(mjm.actuator_biastype[i])
    if gt == C.GAIN_FIXED:
      g = gp[i, 0]
    elif gt == C.GAIN_AFFINE:
      g = gp[i, 0] + gp[i, 1] * length[i] + gp[i, 2] * velocity[i]
    elif gt == C.GAIN_MUSCLE:
      g = gain(length[i], velocity[i], lr[i], a0[i], gp[i])
    if bt == C.BIAS_AFFINE:
      b = bp[i, 0] + bp[i, 1] * length[i] + bp[i, 2] * velocity[i]
    elif bt == C.BIAS_MUSCLE:
      b = bias(length[i], lr[i], a0[i], bp[i])
    f = g * ca + b
    if mjm.actuator_forcelimited[i]:
      f = min(max(f, mjm.actuator_forcerange[i][0]), mjm.actuator_forcerange[i][1])
    force[i] = f
  return act_dot, force


def length_range(trntype, trnid, gear0, jnt_limited, jnt_range, tendon_limited, tendon_range):
  """set_length_range of one world (set_const.py:573-607): (nu, 2)."""
  from mujoco_warp_b200._src import constants as C

  out = np.zeros((len(trntype), 2))
  for i, (t, j, g) in enumerate(zip(trntype, trnid, gear0)):
    rng = None
    if t == C.TRN_JOINT and jnt_limited[j]:
      rng = jnt_range[j]
    elif t == C.TRN_TENDON and len(tendon_limited) and tendon_limited[j]:
      rng = tendon_range[j]
    if rng is not None:
      out[i] = (rng[0] * g, rng[1] * g) if g > 0 else (rng[1] * g, rng[0] * g)
  return out


def lengths(mjm, qpos, qvel):
  """actuator_length / velocity (nu) and the moment rows (nu, nv) of joint (hinge / slide) and fixed-tendon transmissions."""
  from mujoco_warp_b200._src import constants as C

  nu, nv = int(mjm.nu), int(mjm.nv)
  mom = np.zeros((nu, nv))
  for i in range(nu):
    j, g = int(mjm.actuator_trnid[i, 0]), float(mjm.actuator_gear[i, 0])
    if mjm.actuator_trntype[i] == C.TRN_JOINT:
      if mjm.jnt_type[j] not in (C.JNT_HINGE, C.JNT_SLIDE):
        raise NotImplementedError("muscle oracle: hinge / slide joint transmissions only")
      mom[i, mjm.jnt_dofadr[j]] = g
    else:
      for k in range(int(mjm.tendon_adr[j]), int(mjm.tendon_adr[j] + mjm.tendon_num[j])):
        mom[i, mjm.jnt_dofadr[int(mjm.wrap_objid[k])]] += g * mjm.wrap_prm[k]
  # hinge / slide only: qpos and qvel share the dof index order through jnt_qposadr / jnt_dofadr
  q = np.zeros(nv)
  for j in range(int(mjm.njnt)):
    q[mjm.jnt_dofadr[j]] = qpos[mjm.jnt_qposadr[j]]
  return mom @ q, mom @ np.asarray(qvel, dtype=np.float64), mom


class MuscleStep:
  """fp64 step of a model with muscles: the pipeline oracle (oracle/orc.py) runs the model with every muscle's gain, bias and
  activation removed, and the muscles' forces, computed here by `actuation` at each evaluated state with each world's muscle
  fields, enter it as qfrc_applied (moment^T force).  Activations advance here: Euler / implicitfast / implicit add dt act_dot (muscle
  actuators contribute nothing to the implicit velocity derivative, derivative.py:69-104), RK4 restates forward.py:520-560 stage by
  stage through the oracle's forward.  Models whose stateful actuators are all muscles, on hinge / slide joints and fixed tendons."""

  def __init__(self, mjm, nworld, nconmax, njmax, muscle_fields=None):
    import copy

    from tests import util

    self.mjm, self.nworld = mjm, nworld
    nu = int(mjm.nu)
    self.muscle = (np.asarray(mjm.actuator_gaintype) == 2) | (np.asarray(mjm.actuator_biastype) == 2) | (np.asarray(mjm.actuator_dyntype) == 4)
    if np.any(~self.muscle & (np.asarray(mjm.actuator_actadr) >= 0)):
      raise NotImplementedError("muscle oracle: every stateful actuator must be a muscle")
    s = copy.copy(mjm)
    s.na = 0
    for n, v in (("actuator_gaintype", 0), ("actuator_biastype", 0), ("actuator_dyntype", 0), ("actuator_actadr", -1), ("actuator_actnum", 0)):
      a = np.array(getattr(mjm, n)).copy()
      a[self.muscle] = v
      setattr(s, n, a)
    gp = np.array(mjm.actuator_gainprm, dtype=np.float64).copy()
    gp[self.muscle] = 0.0
    s.actuator_gainprm = gp
    self.orc = util.make_oracle(s, nworld, nconmax, njmax)
    # each world's row of the muscle fields: a given (nb, ...) array is read as entry w % nb, as the kernels read batched fields
    given = dict(muscle_fields or {})
    self.fields = {}
    for n, shape in (("actuator_gainprm", (nu, 10)), ("actuator_biasprm", (nu, 10)), ("actuator_acc0", (nu,)), ("actuator_lengthrange", (nu, 2))):
      a = np.asarray(given.get(n, getattr(mjm, n)), dtype=np.float64).reshape((-1,) + shape)
      self.fields[n] = a[np.arange(nworld) % a.shape[0]]

  def _forces(self, w, qpos, qvel, ctrl, act):
    L, V, mom = lengths(self.mjm, qpos, qvel)
    f = self.fields
    act_dot, force = actuation(self.mjm, ctrl, act, L, V, float(self.mjm.opt.timestep), gainprm=f["actuator_gainprm"][w], biasprm=f["actuator_biasprm"][w],
                               acc0=f["actuator_acc0"][w], lengthrange=f["actuator_lengthrange"][w])
    return act_dot, force, mom[self.muscle].T @ force[self.muscle]

  def _clamp(self, act):
    out = act.copy()
    m = self.mjm
    for i in range(int(m.nu)):
      a = int(m.actuator_actadr[i])
      if a >= 0 and m.actuator_actlimited[i]:
        out[..., a] = np.clip(out[..., a], m.actuator_actrange[i][0], m.actuator_actrange[i][1])
    return out

  def step(self, time, qpos, qvel, act, ctrl, qacc_warmstart):
    """One step of every world from the given state: (time, qpos, qvel, act, act_dot, actuator_force)."""
    o, nw, dt = self.orc, self.nworld, float(self.mjm.opt.timestep)
    qpos, qvel, act, ctrl = (np.asarray(x, dtype=np.float64).reshape(nw, -1) for x in (qpos, qvel, act, ctrl))
    o.set_state(qpos=qpos, qvel=qvel, ctrl=ctrl, qacc_warmstart=np.asarray(qacc_warmstart).reshape(nw, -1), time=np.asarray(time).reshape(o.d["time"].shape))

    def evaluate(qp, qv, ac):
      ad, fo = np.zeros_like(act), np.zeros_like(ctrl)
      for w in range(nw):
        ad[w], fo[w], o.d["qfrc_applied"][w] = self._forces(w, qp[w], qv[w], ctrl[w], ac[w])
      return ad, fo

    if int(self.mjm.opt.integrator) != 1:  # Euler, implicit, implicitfast: the oracle's own step at constant muscle forces
      act_dot, force = evaluate(qpos, qvel, act)
      o.step()
      return o.d["time"].reshape(nw).copy(), o.d["qpos"].copy(), o.d["qvel"].copy(), self._clamp(act + dt * act_dot), act_dot, force
    A, B = (0.5, 0.5, 1.0), (1 / 6, 1 / 3, 1 / 3, 1 / 6)
    act_dot, force = evaluate(qpos, qvel, act)
    o.forward()
    qv, qacc = qvel.copy(), o.d["qacc"].copy()
    qvel_rk, qacc_rk, act_dot_rk = B[0] * qv, B[0] * qacc, B[0] * act_dot
    for i in range(3):
      qp_i, qv_i, ac_i = qpos + A[i] * dt * qv, qvel + A[i] * dt * qacc, act + A[i] * dt * act_dot
      o.set_state(qpos=qp_i, qvel=qv_i)
      act_dot, force = evaluate(qp_i, qv_i, ac_i)
      o.forward()
      qv, qacc = qv_i, o.d["qacc"].copy()
      qvel_rk, qacc_rk, act_dot_rk = qvel_rk + B[i + 1] * qv, qacc_rk + B[i + 1] * qacc, act_dot_rk + B[i + 1] * act_dot
    t = np.asarray(time, dtype=np.float64).reshape(nw) + dt
    return t, qpos + dt * qvel_rk, qvel + dt * qacc_rk, self._clamp(act + dt * act_dot_rk), act_dot_rk, force
