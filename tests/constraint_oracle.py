"""An fp64 restatement of make_constraint (k_constraint.cu) and of the CSR view of its Jacobian (k_efc_csr, k_support.cu) for ONE world.

Inputs are the world's own arrays (what the position and velocity stages left in Data, and the world's contacts in pool order) and the
model as that world sees it (entry w % nb of every batched field, `world_model`).  The output is every row in this library's
deterministic order -- equality rows (connect, weld, joint, tendon passes over the equalities), dof friction loss, tendon friction loss,
ball limits, slide / hinge limits, tendon limits, contacts in pool order -- which is also the order the reference produces when its
kernels run one thread after the other, so the same code is held to the reference's fixtures.

Every float output comes with a magnitude: the sum of the absolute values of the terms that formed it, propagated through each
operation (class E).  A kernel that evaluates the same expressions in fp32 differs from the fp64 value by at most a small multiple of
eps32 * magnitude, whatever cancellation happened; tests derive their tolerances from it.

Activation decisions (limit pos < 0, contact dist - includemargin < 0, the side of a joint / tendon limit, the ball joint's angle wrap) are
asserted to be at least MARGIN away from their threshold: a scene that drifts onto a knife edge fails here with a clear message instead of
letting fp32 and fp64 take different branches."""

import math

import numpy as np

from mujoco_warp_b200._src import constants as C

MARGIN = 1e-5


class KnifeEdge(AssertionError):
  pass


def _edge(x, what):
  if abs(x) < MARGIN:
    raise KnifeEdge(f"{what}: {x:.3g} is within {MARGIN} of its threshold")


class E:
  """A value and the magnitude of the terms that formed it."""

  __slots__ = ("v", "m")

  def __init__(self, v, m=None):
    self.v = float(v)
    self.m = abs(self.v) if m is None else float(m)

  def __add__(self, o):
    o = _e(o)
    return E(self.v + o.v, self.m + o.m)

  __radd__ = __add__

  def __sub__(self, o):
    o = _e(o)
    return E(self.v - o.v, self.m + o.m)

  def __rsub__(self, o):
    return _e(o) - self

  def __neg__(self):
    return E(-self.v, self.m)

  def __mul__(self, o):
    o = _e(o)
    return E(self.v * o.v, self.m * o.m)

  __rmul__ = __mul__

  def __truediv__(self, o):
    o = _e(o)
    q = self.v / o.v
    return E(q, self.m / abs(o.v) + abs(q) * o.m / abs(o.v))

  def __rtruediv__(self, o):
    return _e(o) / self


def _e(x):
  return x if isinstance(x, E) else E(x)


def esqrt(a):
  r = math.sqrt(max(a.v, 0.0))
  return E(r, r + (a.m / (2.0 * r) if r > 0 else math.sqrt(a.m)))


def emax(a, b):
  a, b = _e(a), _e(b)
  return a if a.v >= b.v else b


def emin(a, b):
  a, b = _e(a), _e(b)
  return a if a.v <= b.v else b


def eclip(a, lo, hi):
  return emin(emax(a, lo), hi)


def v3(a):
  return [_e(x) for x in np.asarray(a, dtype=np.float64).reshape(3)]


def cross(a, b):
  return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def dot(a, b):
  return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def add(a, b):
  return [x + y for x, y in zip(a, b)]


def sub(a, b):
  return [x - y for x, y in zip(a, b)]


def scl(a, s):
  return [x * s for x in a]


def matvec(R, a):
  R = np.asarray(R, dtype=np.float64).reshape(3, 3)
  return [R[i, 0] * a[0] + R[i, 1] * a[1] + R[i, 2] * a[2] for i in range(3)]


def qmul(u, v):
  return [u[0] * v[0] - u[1] * v[1] - u[2] * v[2] - u[3] * v[3], u[0] * v[1] + u[1] * v[0] + u[2] * v[3] - u[3] * v[2],
          u[0] * v[2] - u[1] * v[3] + u[2] * v[0] + u[3] * v[1], u[0] * v[3] + u[1] * v[2] - u[2] * v[1] + u[3] * v[0]]


def qconj(q):
  return [q[0], -q[1], -q[2], -q[3]]


def q_axis(a):
  return [E(0.0), a[0], a[1], a[2]]


class Rows:
  pass


def world_model(mjm, batched=None, w=0):
  """A dict view of the model as world w sees it: batched[name] is an (nb, ...) array and world w reads entry w % nb."""
  batched = batched or {}

  class V:
    def __getattr__(self, n):
      if n in batched:
        x = np.asarray(batched[n])
        return x[w % x.shape[0]]
      return getattr(mjm, n)

  return V()


def _isdofancestor(m, b, dof):
  """dof moves body b: dof lies on the dof chain from b's weld body up to the root."""
  b = int(m.body_weldid[b])
  da = int(m.body_dofadr[b]) + int(m.body_dofnum[b]) - 1
  while da >= 0:
    if da == dof:
      return True
    da = int(m.dof_parentid[da])
  return False


def tendon_J(m, t):
  """Fixed tendon t's Jacobian row (nv,) from its wraps (the last joint wrap that hits a dof sets the entry)."""
  J = np.zeros(int(m.nv))
  for k in range(int(m.tendon_adr[t]), int(m.tendon_adr[t]) + int(m.tendon_num[t])):
    J[int(m.jnt_dofadr[int(m.wrap_objid[k])])] = float(np.asarray(m.wrap_prm).reshape(-1)[k])
  return J


def make_constraint(m, st, njmax):
  """st: dict with qpos, qvel, xpos (nbody, 3), xmat (nbody, 9), xquat (nbody, 4), cdof (nv, 6), cvel (nbody, 6), cdof_dot (nv, 6),
  subtree_com (nbody, 3), ten_length (ntendon,), eq_active (neq,) and the world's contacts: con_id (pool ids) and con_dist, con_includemargin,
  con_dim, con_geom, con_pos, con_frame, con_friction, con_solref, con_solreffriction, con_solimp, each (ncon, ...).  m: world_model()."""
  nv, nbody = int(m.nv), int(m.nbody)
  opt = m.opt
  dsbl = int(opt.disableflags)
  timestep = float(np.asarray(opt.timestep).reshape(-1)[0])
  impratio_invsqrt = 1.0 / math.sqrt(float(opt.impratio))
  qpos = np.asarray(st["qpos"], dtype=np.float64)
  qvel = np.asarray(st["qvel"], dtype=np.float64)
  xpos = np.asarray(st["xpos"], dtype=np.float64).reshape(nbody, 3)
  xmat = np.asarray(st["xmat"], dtype=np.float64).reshape(nbody, 9)
  xquat = np.asarray(st["xquat"], dtype=np.float64).reshape(nbody, 4)
  cdof = np.asarray(st["cdof"], dtype=np.float64).reshape(nv, 6)
  cvel = np.asarray(st["cvel"], dtype=np.float64).reshape(nbody, 6)
  cdof_dot = np.asarray(st["cdof_dot"], dtype=np.float64).reshape(nv, 6)
  scom = np.asarray(st["subtree_com"], dtype=np.float64).reshape(nbody, 3)
  ten_length = np.asarray(st.get("ten_length", np.zeros(0)), dtype=np.float64).reshape(-1)
  R = Rows()
  R.rows = []  # dicts: type, id, J (list of E, nv), pos, margin, vel, frictionloss, D, aref (E)
  R.ne = R.nf = R.nl = 0
  R.nefc = 0
  ncon = len(st.get("con_id", []))
  R.efc_address = -np.ones((ncon, 10), dtype=np.int64)  # a contact has at most 10 rows (pyramidal condim 6)

  def efc_row(pos_aref, pos_imp, invweight, solref, solimp, margin, vel, frictionloss, type_, id_, J):
    solref = [float(x) for x in np.asarray(solref).reshape(2)]
    solimp = [float(x) for x in np.asarray(solimp).reshape(5)]
    pos_aref, pos_imp, invweight, vel = _e(pos_aref), _e(pos_imp), _e(invweight), _e(vel)
    timeconst, dampratio = solref
    if not dsbl & C.DSBL_REFSAFE:
      timeconst = max(timeconst, 2.0 * timestep)
    dmin = min(max(solimp[0], C.MJ_MINIMP), C.MJ_MAXIMP)
    dmax = min(max(solimp[1], C.MJ_MINIMP), C.MJ_MAXIMP)
    width, mid, power = max(C.MJ_MINVAL, solimp[2]), min(max(solimp[3], C.MJ_MINIMP), C.MJ_MAXIMP), max(1.0, solimp[4])
    k = 1.0 / (dmax * dmax * timeconst * timeconst * dampratio * dampratio)
    b = 2.0 / (dmax * timeconst)
    if solref[0] <= 0:
      k = -solref[0] / (dmax * dmax)
    if solref[1] <= 0:
      b = -solref[1] / dmax
    imp_x = E(abs(pos_imp.v), pos_imp.m) / width
    lower = imp_x.v < mid
    bx, bc = (imp_x, mid) if lower else (1.0 - imp_x, 1.0 - mid)
    if power == 2.0:
      t = bx * bx / bc
    elif power == 1.0:
      t = bx
    else:  # x^p / c^(p-1): relative error p times that of x
      tv = bx.v ** power / bc ** (power - 1.0)
      t = E(tv, abs(tv) * (1.0 + power * bx.m / max(abs(bx.v), 1e-300)))
    imp_y = t if lower else 1.0 - t
    imp = eclip(dmin + imp_y * (dmax - dmin), dmin, dmax)
    if imp_x.v > 1.0:
      imp = E(dmax)
    D = 1.0 / emax(invweight * (1.0 - imp) / imp, C.MJ_MINVAL)
    R.rows.append(dict(type=type_, id=id_, J=J, pos=pos_aref + margin, margin=_e(margin), vel=vel, frictionloss=_e(frictionloss), D=D,
                       aref=-k * imp * pos_aref - b * vel))

  def jvel(J):
    s = E(0.0, 0.0)
    for c in range(nv):
      s = s + J[c] * qvel[c]
    return s

  def jac_cols(point, b, dof):
    """jp, jr, dp, dr of dof for the world point on body b (zeros when dof does not move b)."""
    z = [E(0.0)] * 3
    if not _isdofancestor(m, b, dof):
      return z, z, z, z
    off = sub(point, v3(scom[int(m.body_rootid[b])]))
    cang, clin = v3(cdof[dof, :3]), v3(cdof[dof, 3:])
    jp, jr = add(clin, cross(cang, off)), cang
    cvb = cvel[b]
    pvel = sub(v3(cvb[3:]), cross(off, v3(cvb[:3])))
    j = int(m.dof_jntid[dof])
    jt = int(m.jnt_type[j])
    if jt == C.JNT_BALL or (jt == C.JNT_FREE and dof >= int(m.jnt_dofadr[j]) + 3):
      u = cvel[int(m.dof_bodyid[dof])]
      u0, u1, c0, c1 = v3(u[:3]), v3(u[3:]), v3(cdof[dof, :3]), v3(cdof[dof, 3:])
      cdd = cross(u0, c0) + add(cross(u1, c0), cross(u0, c1))
    else:
      cdd = [_e(x) for x in cdof_dot[dof]]
    dp = add(add(cdd[3:], cross(cdd[:3], off)), cross(cang, pvel))
    return jp, jr, dp, cdd[:3]

  # ---- equality rows
  eq_active = np.asarray(st.get("eq_active", np.zeros(0)), dtype=bool).reshape(-1)
  neq = int(getattr(m, "neq", 0))
  if neq and not dsbl & (C.DSBL_CONSTRAINT | C.DSBL_EQUALITY):
    eq_type = np.asarray(m.eq_type)
    data_all = np.asarray(m.eq_data, dtype=np.float64).reshape(neq, 11)
    for want in (C.EQ_CONNECT, C.EQ_WELD, C.EQ_JOINT, C.EQ_TENDON):
      for e in range(neq):
        if int(eq_type[e]) != want or not eq_active[e]:
          continue
        data = data_all[e]
        o1, o2 = int(m.eq_obj1id[e]), int(m.eq_obj2id[e])
        solref, solimp = np.asarray(m.eq_solref).reshape(neq, 2)[e], np.asarray(m.eq_solimp).reshape(neq, 5)[e]
        if want == C.EQ_TENDON:
          pos1 = E(ten_length[o1]) - float(m.tendon_length0[o1])
          J1 = tendon_J(m, o1)
          if o2 > -1:
            invweight = float(m.tendon_invweight0[o1]) + float(m.tendon_invweight0[o2])
            dif = E(ten_length[o2]) - float(m.tendon_length0[o2])
            dif2 = dif * dif
            dif3 = dif2 * dif
            pos = pos1 - (data[0] + data[1] * dif + data[2] * dif2 + data[3] * dif3 + data[4] * (dif3 * dif))
            deriv = data[1] + 2.0 * data[2] * dif + 3.0 * data[3] * dif2 + 4.0 * data[4] * dif3
            J2 = tendon_J(m, o2)
            J = [E(J1[c]) - (deriv * J2[c] if deriv.v != 0 else 0.0) for c in range(nv)]
          else:
            invweight, pos, deriv = float(m.tendon_invweight0[o1]), pos1 - data[0], E(0.0)
            J = [E(J1[c]) for c in range(nv)]
          efc_row(pos, pos, invweight, solref, solimp, 0.0, jvel(J), 0.0, C.CNSTR_EQUALITY, e, J)
          R.rows[-1]["eq_tendon"] = (o1, o2 if deriv.v != 0 else -1)
          continue
        if want == C.EQ_JOINT:
          d1, q1 = int(m.jnt_dofadr[o1]), int(m.jnt_qposadr[o1])
          J = [E(0.0)] * nv
          J[d1] = E(1.0)
          if o2 > -1:
            q2, d2 = int(m.jnt_qposadr[o2]), int(m.jnt_dofadr[o2])
            dif = E(qpos[q2]) - float(m.qpos0[q2])
            rhs = data[0] + dif * (data[1] + dif * (data[2] + dif * (data[3] + dif * data[4])))
            deriv2 = data[1] + dif * (2.0 * data[2] + dif * (3.0 * data[3] + dif * 4.0 * data[4]))
            pos = E(qpos[q1]) - float(m.qpos0[q1]) - rhs
            vel = E(qvel[d1]) - qvel[d2] * deriv2
            invweight = float(m.dof_invweight0[d1]) + float(m.dof_invweight0[d2])
            J[d2] = -deriv2
          else:
            pos = E(qpos[q1]) - float(m.qpos0[q1]) - data[0]
            vel, invweight = E(qvel[d1]), float(m.dof_invweight0[d1])
          efc_row(pos, pos, invweight, solref, solimp, 0.0, vel, 0.0, C.CNSTR_EQUALITY, e, J)
          continue
        nrow = 3 if want == C.EQ_CONNECT else 6
        b1, b2 = o1, o2
        a1, a2 = v3(data[0:3]), v3(data[3:6])
        p1 = add(v3(xpos[b1]), matvec(xmat[b1], a1 if want == C.EQ_CONNECT else a2))
        p2 = add(v3(xpos[b2]), matvec(xmat[b2], a2 if want == C.EQ_CONNECT else a1))
        xq1, xq2 = [_e(x) for x in xquat[b1]], [_e(x) for x in xquat[b2]]
        relpose = [_e(x) for x in data[6:10]]
        ts = float(data[10]) if want == C.EQ_WELD else 0.0
        quat = qmul(xq1, relpose) if want == C.EQ_WELD else [E(1.0), E(0.0), E(0.0), E(0.0)]
        quat1 = qconj(xq2) if want == C.EQ_WELD else [E(1.0), E(0.0), E(0.0), E(0.0)]
        Jrows = [[E(0.0)] * nv for _ in range(nrow)]
        Jdotp, Jdotr0 = [E(0.0, 0.0)] * 3, [E(0.0, 0.0)] * 3
        for c in range(nv):
          jp1, jr1, dp1, dr1 = jac_cols(p1, b1, c)
          jp2, jr2, dp2, dr2 = jac_cols(p2, b2, c)
          jdp = sub(jp1, jp2)
          for k in range(3):
            Jrows[k][c] = jdp[k]
          Jdotp = add(Jdotp, scl(sub(dp1, dp2), qvel[c]))
          if want == C.EQ_WELD:
            jdr = scl(qmul(qmul(quat1, q_axis(scl(sub(jr1, jr2), ts))), quat)[1:], 0.5)
            for k in range(3):
              Jrows[3 + k][c] = jdr[k]
            Jdotr0 = add(Jdotr0, scl(sub(dr1, dr2), qvel[c]))
        cpos = sub(p1, p2)
        crot, Jdotr = [E(0.0)] * 3, [E(0.0)] * 3
        if want == C.EQ_WELD:
          crot = scl(qmul(quat1, quat)[1:], ts)
          om1, om2 = v3(cvel[b1, :3]), v3(cvel[b2, :3])
          dom = sub(om1, om2)
          qdot0r = qmul([x * 0.5 for x in qmul(q_axis(om1), xq1)], relpose)
          qdot1 = [x * 0.5 for x in qmul(q_axis(om2), xq2)]
          t1 = qmul(qmul(qconj(qdot1), q_axis(dom)), quat)[1:]
          t2 = qmul(qmul(qconj(xq2), q_axis(Jdotr0)), quat)[1:]
          t3 = qmul(qmul(qconj(xq2), q_axis(dom)), qdot0r)[1:]
          Jdotr = scl(add(add(t1, t2), t3), 0.5 * ts)
        pos_imp = esqrt(dot(cpos, cpos) + dot(crot, crot))
        iw_t = float(m.body_invweight0[b1][0]) + float(m.body_invweight0[b2][0])
        iw_r = float(m.body_invweight0[b1][1]) + float(m.body_invweight0[b2][1])
        for k in range(nrow):
          rot = k >= 3
          kk = k - 3 if rot else k
          efc_row((crot if rot else cpos)[kk], pos_imp, iw_r if rot else iw_t, solref, solimp, 0.0, jvel(Jrows[k]), 0.0, C.CNSTR_EQUALITY, e, Jrows[k])
          R.rows[-1]["aref"] = R.rows[-1]["aref"] - (Jdotr if rot else Jdotp)[kk]
          R.rows[-1]["eq_chain"] = (b1, b2)
  R.ne = len(R.rows)

  # ---- friction loss: dofs, then tendons, wherever this world's value is positive
  if not dsbl & (C.DSBL_CONSTRAINT | C.DSBL_FRICTIONLOSS):
    fl = np.asarray(m.dof_frictionloss, dtype=np.float64).reshape(-1)
    for dof in range(nv):
      if fl[dof] > 0:
        J = [E(1.0) if c == dof else E(0.0) for c in range(nv)]
        efc_row(0.0, 0.0, float(m.dof_invweight0[dof]), np.asarray(m.dof_solref).reshape(nv, 2)[dof], np.asarray(m.dof_solimp).reshape(nv, 5)[dof],
                0.0, E(qvel[dof]), fl[dof], C.CNSTR_FRICTION_DOF, dof, J)
    nt = int(getattr(m, "ntendon", 0))
    tfl = np.asarray(m.tendon_frictionloss, dtype=np.float64).reshape(-1) if nt else np.zeros(0)
    for t in range(nt):
      if tfl[t] > 0:
        J = [E(x) for x in tendon_J(m, t)]
        efc_row(0.0, 0.0, float(m.tendon_invweight0[t]), np.asarray(m.tendon_solref_fri).reshape(nt, 2)[t],
                np.asarray(m.tendon_solimp_fri).reshape(nt, 5)[t], 0.0, jvel(J), tfl[t], C.CNSTR_FRICTION_TENDON, t, J)
  R.nf = len(R.rows) - R.ne

  # ---- limits: ball, slide / hinge, tendon
  if not dsbl & (C.DSBL_CONSTRAINT | C.DSBL_LIMIT):
    jt = np.asarray(m.jnt_type)
    lim = np.asarray(m.jnt_limited).astype(bool)
    rng = np.asarray(m.jnt_range, dtype=np.float64).reshape(-1, 2)
    jm = np.asarray(m.jnt_margin, dtype=np.float64).reshape(-1)
    jsr, jsi = np.asarray(m.jnt_solref).reshape(-1, 2), np.asarray(m.jnt_solimp).reshape(-1, 5)
    for j in np.nonzero(lim & (jt == C.JNT_BALL))[0]:
      qa, da = int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])
      q = qpos[qa : qa + 4] / np.linalg.norm(qpos[qa : qa + 4])
      s2 = float(np.linalg.norm(q[1:]))
      axis, angle = np.zeros(3), E(0.0)
      if s2 != 0.0:
        speed = 2.0 * math.atan2(s2, q[0])
        _edge(speed - math.pi, f"ball joint {j}: rotation angle vs pi")
        if speed > math.pi:
          speed -= 2.0 * math.pi
        v = q[1:] * (speed / s2)
        a = float(np.linalg.norm(v))
        angle = E(a, a + 4.0 * a)  # normalize, atan2, the wrap and the norm: a few rounding steps of the angle itself
        axis = v / a if a != 0 else v
      pos = E(max(rng[j, 0], rng[j, 1])) - angle - jm[j]
      _edge(pos.v, f"ball joint {j} limit")
      if pos.v >= 0:
        continue
      J = [E(0.0)] * nv
      for k in range(3):
        J[da + k] = E(-axis[k], abs(axis[k]) * 4.0)
      vel = -(E(axis[0], abs(axis[0])) * qvel[da] + E(axis[1], abs(axis[1])) * qvel[da + 1] + E(axis[2], abs(axis[2])) * qvel[da + 2])
      efc_row(pos, pos, float(m.dof_invweight0[da]), jsr[j], jsi[j], jm[j], vel, 0.0, C.CNSTR_LIMIT_JOINT, int(j), J)
    for j in np.nonzero(lim & ((jt == C.JNT_SLIDE) | (jt == C.JNT_HINGE)))[0]:
      qv = qpos[int(m.jnt_qposadr[j])]
      dmin, dmax = E(qv) - rng[j, 0], E(rng[j, 1]) - qv
      _edge(dmin.v - dmax.v, f"joint {j}: limit side")
      pos = emin(dmin, dmax) - jm[j]
      _edge(pos.v, f"joint {j} limit")
      if pos.v >= 0:
        continue
      da = int(m.jnt_dofadr[j])
      s = 1.0 if dmin.v < dmax.v else -1.0
      J = [E(0.0)] * nv
      J[da] = E(s)
      efc_row(pos, pos, float(m.dof_invweight0[da]), jsr[j], jsi[j], jm[j], E(s * qvel[da]), 0.0, C.CNSTR_LIMIT_JOINT, int(j), J)
    nt = int(getattr(m, "ntendon", 0))
    for t in range(nt):
      if not int(np.asarray(m.tendon_limited)[t]):
        continue
      tr = np.asarray(m.tendon_range, dtype=np.float64).reshape(nt, 2)[t]
      tm = float(np.asarray(m.tendon_margin).reshape(-1)[t])
      dmin, dmax = E(ten_length[t]) - tr[0], E(tr[1]) - ten_length[t]
      _edge(dmin.v - dmax.v, f"tendon {t}: limit side")
      pos = emin(dmin, dmax) - tm
      _edge(pos.v, f"tendon {t} limit")
      if pos.v >= 0:
        continue
      s = 1.0 if dmin.v < dmax.v else -1.0
      J = [E(s * x) for x in tendon_J(m, t)]
      efc_row(pos, pos, float(m.tendon_invweight0[t]), np.asarray(m.tendon_solref_lim).reshape(nt, 2)[t], np.asarray(m.tendon_solimp_lim).reshape(nt, 5)[t],
              tm, jvel(J), 0.0, C.CNSTR_LIMIT_TENDON, t, J)
  R.nl = len(R.rows) - R.ne - R.nf

  # ---- contacts, in pool order
  if not dsbl & (C.DSBL_CONSTRAINT | C.DSBL_CONTACT):
    elliptic = int(opt.cone) == C.CONE_ELLIPTIC
    for i in range(ncon):
      pos = E(st["con_dist"][i]) - float(st["con_includemargin"][i])
      _edge(pos.v, f"contact {int(st['con_id'][i])}: dist - includemargin")
      if pos.v >= 0:
        continue
      condim = int(st["con_dim"][i])
      ndim = condim if elliptic else (1 if condim == 1 else 2 * (condim - 1))
      g1, g2 = (int(x) for x in st["con_geom"][i])
      b1, b2 = int(m.geom_bodyid[g1]), int(m.geom_bodyid[g2])
      cpos = v3(st["con_pos"][i])
      frame = np.asarray(st["con_frame"][i], dtype=np.float64).reshape(9)
      fri = np.asarray(st["con_friction"][i], dtype=np.float64).reshape(5)
      off1, off2 = sub(cpos, v3(scom[int(m.body_rootid[b1])])), sub(cpos, v3(scom[int(m.body_rootid[b2])]))
      P = [[E(0.0)] * nv for _ in range(6)]
      for dd in range(nv):
        ang, lin = v3(cdof[dd, :3]), v3(cdof[dd, 3:])
        jp, jr = [E(0.0)] * 3, [E(0.0)] * 3
        if _isdofancestor(m, b2, dd):
          jp, jr = add(lin, cross(ang, off2)), ang
        if _isdofancestor(m, b1, dd):
          jp, jr = sub(jp, add(lin, cross(ang, off1))), sub(jr, ang)
        for k in range(3):
          P[k][dd] = dot(jp, v3(frame[3 * k : 3 * k + 3]))
          P[3 + k][dd] = dot(jr, v3(frame[3 * k : 3 * k + 3]))
      iw0 = float(m.body_invweight0[b1][0]) + float(m.body_invweight0[b2][0])
      typ = C.CNSTR_CONTACT_FRICTIONLESS if condim == 1 else (C.CNSTR_CONTACT_ELLIPTIC if elliptic else C.CNSTR_CONTACT_PYRAMIDAL)
      for dim in range(ndim):
        if elliptic:
          J = P[dim]
        elif condim > 1:
          f = fri[dim // 2] * (-1.0 if dim & 1 else 1.0)
          J = [P[0][c] + P[dim // 2 + 1][c] * f for c in range(nv)]
        else:
          J = P[0]
        invweight, pos_aref = E(iw0), pos
        ref = np.asarray(st["con_solref"][i], dtype=np.float64)
        if elliptic:
          if dim > 0:
            sf = np.asarray(st["con_solreffriction"][i], dtype=np.float64)
            if sf[0] != 0 or sf[1] != 0:
              ref = sf
            invweight = invweight * impratio_invsqrt * impratio_invsqrt
            if dim > 1:
              invweight = invweight * (fri[0] * fri[0] / (fri[dim - 1] * fri[dim - 1]))
            pos_aref = E(0.0)
        elif condim > 1:
          invweight = invweight + fri[0] * fri[0] * invweight
          invweight = invweight * 2.0 * fri[0] * fri[0] * impratio_invsqrt * impratio_invsqrt
        if len(R.rows) < njmax:
          R.efc_address[i, dim] = len(R.rows)
        efc_row(pos_aref, pos, invweight, ref, st["con_solimp"][i], float(st["con_includemargin"][i]), jvel(J), 0.0, typ, int(st["con_id"][i]), J)
        R.rows[-1]["con_bodies"] = (b1, b2)
  R.nefc = len(R.rows)
  return R


def arrays(R, nv):
  """Rows -> dict of arrays (value and magnitude) over every row, njmax not applied."""
  n = len(R.rows)
  out = {"type": np.array([r["type"] for r in R.rows], dtype=np.int64), "id": np.array([r["id"] for r in R.rows], dtype=np.int64)}
  out["J"] = np.array([[x.v for x in r["J"]] for r in R.rows]).reshape(n, nv)
  out["J_mag"] = np.array([[x.m for x in r["J"]] for r in R.rows]).reshape(n, nv)
  for f in ("pos", "margin", "vel", "frictionloss", "D", "aref"):
    out[f] = np.array([r[f].v for r in R.rows])
    out[f + "_mag"] = np.array([r[f].m for r in R.rows])
  return out


def csr(m, R, njmax, njmax_nnz):
  """The reference's CSR view of the first min(nefc, njmax) rows: rownnz, rowadr (-1 where the row did not fit), colind, values.  A
  tendon equality row that does not fit gets no rownnz either (-1 here; constraint.py:758-760)."""
  nv = int(m.nv)

  def chain(b):
    b = int(m.body_weldid[b])
    return int(m.body_dofadr[b]) + int(m.body_dofnum[b]) - 1

  def walk(da1, da2, stop_common):
    out = []
    while da1 >= 0 or da2 >= 0:
      da = max(da1, da2)
      if stop_common and da1 == da and da2 == da:
        break
      if da1 == da:
        da1 = int(m.dof_parentid[da1])
      if da2 == da:
        da2 = int(m.dof_parentid[da2])
      out.append(da)
    return out

  def tcols(t):
    a = int(m.ten_J_rowadr[t])
    return [int(x) for x in np.asarray(m.ten_J_colind)[a : a + int(m.ten_J_rownnz[t])]]

  nrow = min(R.nefc, njmax)
  rownnz, rowadr = np.zeros(nrow, dtype=np.int64), -np.ones(nrow, dtype=np.int64)
  colind, vals = [], []
  base = 0
  for r in range(nrow):
    row = R.rows[r]
    typ, id_ = row["type"], row["id"]
    J = [x.v for x in row["J"]]
    reserve = None
    if typ == C.CNSTR_EQUALITY:
      et = int(np.asarray(m.eq_type)[id_])
      if et == C.EQ_JOINT:
        o2 = int(m.eq_obj2id[id_])
        cols = [int(m.jnt_dofadr[int(m.eq_obj1id[id_])])] + ([int(m.jnt_dofadr[o2])] if o2 > -1 else [])
      elif et == C.EQ_TENDON:
        t1, t2 = row["eq_tendon"]
        merged = sorted(set(tcols(t1)) | (set(tcols(t2)) if t2 > -1 else set()))
        reserve = len(merged)
        cols = [c for c in merged if J[c] != 0.0]
      else:
        b1, b2 = row["eq_chain"]
        cols = walk(chain(b1), chain(b2), False)
    elif typ == C.CNSTR_FRICTION_DOF:
      cols = [id_]
    elif typ == C.CNSTR_LIMIT_JOINT:
      da = int(m.jnt_dofadr[id_])
      cols = [da, da + 1, da + 2] if int(m.jnt_type[id_]) == C.JNT_BALL else [da]
    elif typ in (C.CNSTR_FRICTION_TENDON, C.CNSTR_LIMIT_TENDON):
      cols = tcols(id_)
    else:
      b1, b2 = row["con_bodies"]
      cols = walk(chain(b1), chain(b2), True)
    reserve = len(cols) if reserve is None else reserve
    rownnz[r] = len(cols)
    if base + reserve <= njmax_nnz:
      rowadr[r] = base
      colind.append(cols)
      vals.append([row["J"][c] for c in cols])
    else:
      colind.append(None)
      vals.append(None)
      if typ == C.CNSTR_EQUALITY and int(np.asarray(m.eq_type)[id_]) == C.EQ_TENDON:
        rownnz[r] = -1
    base += reserve
  return rownnz, rowadr, colind, vals, base > njmax_nnz
