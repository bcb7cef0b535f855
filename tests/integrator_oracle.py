"""fp64 restatement of the integration stage (Euler with and without eulerdamp, implicitfast, implicit, RK4 bookkeeping).

Every function takes one world's Data fields as a dict `f` of numpy arrays, so it can be fed either a fixture's fields or the GPU's own
fp32 outputs of forward(); nothing is recomputed upstream of the integrator.  Matrices are dense (nv, nv) in fp64:

- A = M + dt diag(dof_damping) (Euler with eulerdamp); A = M - dt qDeriv (implicitfast: affine actuator gain / bias times the moments,
  skipped when the force sits at or beyond its forcerange, the actearly activation, dof and tendon damping), with entries only where M has
  them -- i.e. at (i, j) with j == i or j an ancestor dof of i -- whatever tree owns them;
- implicit: the same qDeriv minus dt d(qfrc_bias)/d(qvel), taken column by column from cdof, cdof_dot, cvel, cinert and qvel, in the
  D-structure (i and j on one chain), and its LU from the last dof to the first (U unit upper), as the reference stores qLU;
- the velocity and position advance (free, ball, hinge, slide), next_act, and RK4's bookkeeping over a caller-supplied forward().
"""
import numpy as np

from mujoco_warp_b200._src import constants as C

MJ_MINVAL = 1e-15


def ancestors(mjm):
  """anc[i, j]: dof j is dof i or an ancestor dof of it (the M sparsity pattern, lower triangle)."""
  nv = int(mjm.nv)
  anc = np.zeros((nv, nv), dtype=bool)
  for i in range(nv):
    j = i
    while j >= 0:
      anc[i, j] = True
      j = int(mjm.dof_parentid[j])
  return anc


def dense_m(mjm, M):
  """Symmetric dense M from its nC entries (rows at M_rowadr, columns M_colind)."""
  nv = int(mjm.nv)
  A = np.zeros((nv, nv))
  for r in range(nv):
    for e in range(int(mjm.M_rowadr[r]), int(mjm.M_rowadr[r] + mjm.M_rownnz[r])):
      c = int(mjm.M_colind[e])
      A[r, c] = A[c, r] = float(M[e])
  return A


def moment_cols(mjm):
  """The dofs of each actuator's moment row, in the order of Data.actuator_moment (joint dofs, or the tendon's ten_J_colind row)."""
  trntype = np.asarray(getattr(mjm, "actuator_trntype", np.zeros(mjm.nu, dtype=np.int32)))
  out = []
  for a in range(int(mjm.nu)):
    t = int(mjm.actuator_trnid[a, 0])
    if trntype[a] == C.TRN_TENDON:
      adr = int(mjm.ten_J_rowadr[t])
      out.append([int(c) for c in mjm.ten_J_colind[adr : adr + int(mjm.ten_J_rownnz[t])]])
    else:
      nd = {C.JNT_FREE: 6, C.JNT_BALL: 3}.get(int(mjm.jnt_type[t]), 1)
      out.append(list(range(int(mjm.jnt_dofadr[t]), int(mjm.jnt_dofadr[t]) + nd)))
  return out


def ten_j0(mjm):
  """Constant Jacobian rows of the fixed tendons, dense (ntendon, nv)."""
  nt = int(getattr(mjm, "ntendon", 0))
  J = np.zeros((nt, int(mjm.nv)))
  for t in range(nt):
    for k in range(int(mjm.tendon_adr[t]), int(mjm.tendon_adr[t] + mjm.tendon_num[t])):
      J[t, int(mjm.jnt_dofadr[int(mjm.wrap_objid[k])])] = float(mjm.wrap_prm[k])
  return J


def next_act(mjm, a, act, act_dot, scale=1.0, clamp=True, dynprm=None, actrange=None):
  """support.py next_act: one step of actuator a's activation (exact for filterexact), clamped to actrange when clamp and actlimited."""
  dynprm = np.asarray(mjm.actuator_dynprm if dynprm is None else dynprm, dtype=np.float64)
  actrange = np.asarray(mjm.actuator_actrange if actrange is None else actrange, dtype=np.float64)
  dt = float(mjm.opt.timestep)
  if int(mjm.actuator_dyntype[a]) == C.DYN_FILTEREXACT:
    tau = max(MJ_MINVAL, float(dynprm[a, 0]))
    r = act + scale * act_dot * tau * (1.0 - np.exp(-dt / tau))
  else:
    r = act + scale * act_dot * dt
  if clamp and int(mjm.actuator_actlimited[a]):
    r = min(max(r, float(actrange[a, 0])), float(actrange[a, 1]))
  return r


def qderiv_terms(mjm, f, prm=None):
  """The terms of -qDeriv as a list of (i, j, value) on M's lower pattern (j == i or an ancestor of i), in the kernels' order: actuators,
  then tendon damping.  dof damping is left to the caller.  prm: per-world overrides of actuator_gainprm / biasprm / tendon_damping."""
  prm = prm or {}
  flags = int(mjm.opt.disableflags)
  anc = ancestors(mjm)
  out = []
  if mjm.nu and not flags & C.DSBL_ACTUATION:
    gainprm = np.asarray(prm.get("actuator_gainprm", mjm.actuator_gainprm), dtype=np.float64)
    biasprm = np.asarray(prm.get("actuator_biasprm", mjm.actuator_biasprm), dtype=np.float64)
    cols = moment_cols(mjm)
    adr = 0
    for a in range(int(mjm.nu)):
      nnz = len(cols[a])
      mom = np.asarray(f["actuator_moment"], dtype=np.float64)[adr : adr + nnz]
      adr += nnz
      gain = gainprm[a, 2] if int(mjm.actuator_gaintype[a]) == C.GAIN_AFFINE else 0.0
      bias = biasprm[a, 2] if int(mjm.actuator_biastype[a]) == C.BIAS_AFFINE else 0.0
      if gain == 0.0 and bias == 0.0:
        continue
      if int(mjm.actuator_forcelimited[a]):
        frc, (lo, hi) = float(f["actuator_force"][a]), mjm.actuator_forcerange[a]
        if frc <= lo or frc >= hi:  # at the bound the clamped force does not depend on the velocity
          continue
      vel = bias
      if gain != 0.0:
        if getattr(mjm, "na", 0) and int(mjm.actuator_dyntype[a]) != C.DYN_NONE:
          last = int(mjm.actuator_actadr[a] + mjm.actuator_actnum[a] - 1)
          act = float(f["act"][last])
          if int(mjm.actuator_actearly[a]):
            act = next_act(mjm, a, act, float(f["act_dot"][last]))
          vel += gain * act
        else:
          vel += gain * float(f["ctrl"][a])
      for i in range(nnz):
        for j in range(i + 1):
          di, dj = cols[a][i], cols[a][j]
          if anc[di, dj]:
            out.append((di, dj, -mom[i] * mom[j] * vel))
  if getattr(mjm, "ntendon", 0) and not flags & C.DSBL_DAMPER:
    kd = np.asarray(prm.get("tendon_damping", mjm.tendon_damping), dtype=np.float64).reshape(-1)
    J = ten_j0(mjm)
    for t in range(int(mjm.ntendon)):
      if kd[t] == 0.0:
        continue
      nz = np.nonzero(J[t])[0]
      for i in nz:
        for j in nz:
          if j <= i and anc[i, j]:
            out.append((int(i), int(j), J[t, i] * J[t, j] * kd[t]))
  return out


def matrix_a(mjm, f, integrator, prm=None, absolute=False):
  """Dense A in fp64 for Euler with eulerdamp (integrator EULER), IMPLICITFAST or IMPLICIT; with absolute, every term by its absolute
  value (the scale of A's rounding error)."""
  prm = prm or {}
  dt = float(mjm.opt.timestep)
  ab = np.abs if absolute else (lambda x: x)
  A = ab(dense_m(mjm, f["M"]))
  if not int(mjm.opt.disableflags) & C.DSBL_DAMPER:
    A += dt * np.diag(ab(np.asarray(prm.get("dof_damping", mjm.dof_damping), dtype=np.float64).reshape(-1)))
  if integrator == C.INT_EULER:
    return A
  for i, j, v in qderiv_terms(mjm, f, prm):
    A[i, j] += dt * ab(v)
    if i != j:
      A[j, i] += dt * ab(v)
  if integrator == C.INT_IMPLICIT:
    D = drne_dqvel(mjm, f, absolute)
    chain = ancestors(mjm)
    chain = chain | chain.T
    A += (dt if absolute else -dt) * np.where(chain, D, 0.0)
  return A


# spatial algebra, (angular, linear)
def _inert(c, absolute=False):
  """6x6 matrix of a vec10 inertia (I xx yy zz xy xz yz, h, mass) acting on a motion vector."""
  i = np.asarray(c, dtype=np.float64)
  ab = np.abs if absolute else (lambda x: x)
  return ab(np.array([
    [i[0], i[3], i[4], 0.0, -i[8], i[7]],
    [i[3], i[1], i[5], i[8], 0.0, -i[6]],
    [i[4], i[5], i[2], -i[7], i[6], 0.0],
    [0.0, i[8], -i[7], i[9], 0.0, 0.0],
    [-i[8], 0.0, i[6], 0.0, i[9], 0.0],
    [i[7], -i[6], 0.0, 0.0, 0.0, i[9]],
  ]))


def _cross(a, b, absolute):
  if absolute:  # the components' terms by absolute value
    return np.array([a[1] * b[2] + a[2] * b[1], a[2] * b[0] + a[0] * b[2], a[0] * b[1] + a[1] * b[0]])
  return np.cross(a, b)


def _mcross(u, v, absolute=False):
  return np.concatenate([_cross(u[:3], v[:3], absolute), _cross(u[3:], v[:3], absolute) + _cross(u[:3], v[3:], absolute)])


def _fcross(v, f, absolute=False):
  return np.concatenate([_cross(v[:3], f[:3], absolute) + _cross(v[3:], f[3:], absolute), _cross(v[:3], f[3:], absolute)])


def drne_dqvel(mjm, f, absolute=False):
  """Dense d(qfrc_bias)/d(qvel) (nv, nv) at fixed positions, from cdof, cdof_dot, cvel, cinert and qvel; with absolute, the sum of the
  absolute values of every product that enters each entry (the scale of its rounding error).

  qfrc_bias_i = cdof_i . cfrc(subtree of i's body), cfrc_b = I_b cacc_b + cvel_b x* I_b cvel_b, cacc_b = cacc_parent + sum_j cdof_dot_j
  qvel_j with cdof_dot_j = (velocity before dof j) x cdof_j (zero for the free joint's translational dofs), cvel_b = cvel_parent + sum_j
  cdof_j qvel_j.  A joint's dofs enter the velocity after all of its cdof_dot terms; a free joint's translational dofs before its
  rotational ones."""
  nv, nb = int(mjm.nv), int(mjm.nbody)
  ab = np.abs if absolute else (lambda x: x)
  cdof = ab(np.asarray(f["cdof"], dtype=np.float64).reshape(nv, 6))
  cdd = ab(np.asarray(f["cdof_dot"], dtype=np.float64).reshape(nv, 6))
  cvel = ab(np.asarray(f["cvel"], dtype=np.float64).reshape(nb, 6))
  cinert = np.asarray(f["cinert"], dtype=np.float64).reshape(nb, 10)
  qvel = ab(np.asarray(f["qvel"], dtype=np.float64))
  D = np.zeros((nv, nv))
  for k in range(nv):
    dv, da, dfrc = np.zeros((nb, 6)), np.zeros((nb, 6)), np.zeros((nb, 6))
    for b in range(1, nb):
      p = int(mjm.body_parentid[b])
      cv, ca = dv[p].copy(), da[p].copy()
      dof = int(mjm.body_dofadr[b])
      for j in range(int(mjm.body_jntadr[b]), int(mjm.body_jntadr[b] + mjm.body_jntnum[b])):
        jt = int(mjm.jnt_type[j])
        if jt == C.JNT_FREE:
          for a in range(3):
            if k == dof + a:
              cv += cdof[k]
              ca += cdd[k]
          rot = range(dof + 3, dof + 6)
        else:
          rot = range(dof, dof + (3 if jt == C.JNT_BALL else 1))
        for a in rot:
          ca += _mcross(cv, cdof[a], absolute) * qvel[a]
          if k == a:
            ca += cdd[k]
        for a in rot:
          if k == a:
            cv += cdof[k]
        dof += 6 if jt == C.JNT_FREE else len(rot)
      I = _inert(cinert[b], absolute)
      dv[b], da[b] = cv, ca
      dfrc[b] = I @ ca + _fcross(cv, I @ cvel[b], absolute) + _fcross(cvel[b], I @ cv, absolute)
    for b in range(nb - 1, 0, -1):
      p = int(mjm.body_parentid[b])
      if p > 0:
        dfrc[p] += dfrc[b]
    for i in range(nv):
      D[i, k] = cdof[i] @ dfrc[int(mjm.dof_bodyid[i])]
  return D


def lu_d(mjm, A):
  """The reference's LU of A in the D-structure (from the last dof to the first, U unit upper, L lower with the diagonal), as the
  qLU entries at D_rowadr / D_colind."""
  L = A.copy()
  nv = int(mjm.nv)
  for i in range(nv - 1, 0, -1):
    for j in range(i):
      if L[j, i] != 0.0:
        L[j, i] /= L[i, i]
        L[j, :i] -= L[i, :i] * L[j, i]
  out = np.zeros(int(mjm.D_rowadr[-1] + mjm.D_rownnz[-1]))
  for r in range(nv):
    for e in range(int(mjm.D_rowadr[r]), int(mjm.D_rowadr[r] + mjm.D_rownnz[r])):
      out[e] = L[r, int(mjm.D_colind[e])]
  return out


def lu_factors(mjm, LU):
  """(L, U) dense from qLU entries: L lower with the diagonal, U unit upper."""
  nv = int(mjm.nv)
  F = np.zeros((nv, nv))
  for r in range(nv):
    for e in range(int(mjm.D_rowadr[r]), int(mjm.D_rowadr[r] + mjm.D_rownnz[r])):
      F[r, int(mjm.D_colind[e])] = LU[e]
  return np.tril(F), np.triu(F, 1) + np.eye(nv)


def quat_integrate(q, w, dt):
  """normalize(normalize(q) * exp(w dt / 2)), w in the local frame; w = 0 leaves the normalized q."""
  q = np.asarray(q, dtype=np.float64)
  q = q / np.linalg.norm(q)
  n = np.linalg.norm(w)
  if n == 0.0:
    return q
  ax = np.asarray(w, dtype=np.float64) / n
  s, c = np.sin(0.5 * dt * n), np.cos(0.5 * dt * n)
  r = np.array([c, *(ax * s)])
  p = np.array([q[0] * r[0] - q[1:] @ r[1:], *(q[0] * r[1:] + r[0] * q[1:] + np.cross(q[1:], r[1:]))])
  return p / np.linalg.norm(p)


def next_position(mjm, qpos, qvel, dt):
  qpos = np.asarray(qpos, dtype=np.float64).copy()
  for j in range(int(mjm.njnt)):
    t, qa, da = int(mjm.jnt_type[j]), int(mjm.jnt_qposadr[j]), int(mjm.jnt_dofadr[j])
    if t == C.JNT_FREE:
      qpos[qa : qa + 3] += dt * qvel[da : da + 3]
      qpos[qa + 3 : qa + 7] = quat_integrate(qpos[qa + 3 : qa + 7], qvel[da + 3 : da + 6], dt)
    elif t == C.JNT_BALL:
      qpos[qa : qa + 4] = quat_integrate(qpos[qa : qa + 4], qvel[da : da + 3], dt)
    else:
      qpos[qa] += dt * qvel[da]
  return qpos


def solve_trees(mjm, A, b):
  """x = A^-1 b tree by tree (A is block diagonal over the trees)."""
  x = np.zeros(int(mjm.nv))
  for s, n in zip(mjm.tree_dofadr, mjm.tree_dofnum):
    s, n = int(s), int(n)
    x[s : s + n] = np.linalg.solve(A[s : s + n, s : s + n], b[s : s + n])
  return x


def advance(mjm, f, qacc):
  """qvel + dt qacc, the positions integrated with that velocity, the activations by next_act."""
  dt = float(mjm.opt.timestep)
  qvel = np.asarray(f["qvel"], dtype=np.float64) + dt * qacc
  act = None
  if getattr(mjm, "na", 0):
    act = np.asarray(f["act"], dtype=np.float64).copy()
    for a in range(int(mjm.nu)):
      for j in range(int(mjm.actuator_actadr[a]), int(mjm.actuator_actadr[a] + mjm.actuator_actnum[a])) if mjm.actuator_actadr[a] >= 0 else ():
        act[j] = next_act(mjm, a, float(f["act"][j]), float(f["act_dot"][j]), dynprm=f.get("actuator_dynprm"), actrange=f.get("actuator_actrange"))
  return qvel, next_position(mjm, f["qpos"], qvel, dt), act


def integrate(mjm, f, integrator, prm=None):
  """One integrator step from one world's forward() fields: (qacc solved, qvel, qpos, act).  b = efc_Ma, or M qacc without it."""
  b = np.asarray(f["efc_Ma"], dtype=np.float64) if "efc_Ma" in f else dense_m(mjm, f["M"]) @ np.asarray(f["qacc"], dtype=np.float64)
  if integrator == C.INT_EULER and int(mjm.opt.disableflags) & (C.DSBL_EULERDAMP | C.DSBL_DAMPER):
    x = np.asarray(f["qacc"], dtype=np.float64)
  else:
    x = solve_trees(mjm, matrix_a(mjm, f, integrator, prm), b)
  return (x,) + advance(mjm, f, x)


def rk4(mjm, state, forward):
  """forward.py rungekutta4 on one world: state = dict(qpos, qvel, act); forward(qpos, qvel, act) -> dict(qacc, act_dot) evaluated at a
  stage state.  The first evaluation is at the initial state.  Returns (qpos, qvel, act, act_dot)."""
  dt = float(mjm.opt.timestep)
  A, B = (0.5, 0.5, 1.0), (1 / 6, 1 / 3, 1 / 3, 1 / 6)
  q0, v0 = np.asarray(state["qpos"], dtype=np.float64), np.asarray(state["qvel"], dtype=np.float64)
  a0 = np.asarray(state.get("act", np.zeros(0)), dtype=np.float64)
  na = len(a0)
  qpos, qvel, act = q0, v0, a0
  vsum, asum, adsum = np.zeros_like(v0), np.zeros_like(v0), np.zeros(na)
  for s in range(4):
    out = forward(qpos, qvel, act)
    vsum += B[s] * qvel
    asum += B[s] * out["qacc"]
    adsum += B[s] * out.get("act_dot", np.zeros(na))
    if s < 3:
      qpos = next_position(mjm, q0, A[s] * qvel, dt)
      act = a0.copy()
      for a in range(int(mjm.nu)) if na else ():
        for j in range(int(mjm.actuator_actadr[a]), int(mjm.actuator_actadr[a] + mjm.actuator_actnum[a])) if mjm.actuator_actadr[a] >= 0 else ():
          act[j] = next_act(mjm, a, a0[j], out["act_dot"][j], A[s], clamp=False)
      qvel = v0 + A[s] * dt * out["qacc"]
  act = a0.copy()
  for a in range(int(mjm.nu)) if na else ():
    for j in range(int(mjm.actuator_actadr[a]), int(mjm.actuator_actadr[a] + mjm.actuator_actnum[a])) if mjm.actuator_actadr[a] >= 0 else ():
      act[j] = next_act(mjm, a, a0[j], adsum[j], 1.0)
  return next_position(mjm, q0, vsum, dt), v0 + dt * asum, act, adsum
