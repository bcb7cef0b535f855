"""An fp64 restatement of k_sensor (k_sensor.cu, with mjb_sensor_extra.cuh and the touch sensor's site ray of mjb_ray.cuh) for ONE world.

Inputs are the world's own arrays -- what the launches before k_sensor left in Data (kinematics, cdof / cinert / cvel / cdof_dot, tendon
and actuator lengths, velocities and forces, qacc, the constraint rows and the world's contacts in pool order) -- and the model as that
world sees it (entry w % nb of every batched field, constraint_oracle.world_model).  The output is what one launch writes: the
prerequisites it computes before the sensors (subtree_linvel / subtree_angmom, k_body_subtree_vel.cuh; cacc / cfrc_ext / cfrc_int,
k_body_rne_post.cuh) and every sensordata slot of the types k_sensor carries, cutoff applied (reference sensor.py:57-113).  The slots of
the collision, contact and energy sensors belong to other kernels and are left out.

Every float carries a magnitude (constraint_oracle.E): the sum of the absolute values of the terms that formed it.  The kernel
evaluates the same expressions in fp32, so it differs from the fp64 value by a small multiple of eps32 * magnitude.

Decisions are asserted to be at least MARGIN (relative to the scale of the compared quantities) from their thresholds, or KnifeEdge is
raised: touch's normal-force sign, every geometric comparison of the touch ray against its site volume, insidesite's inside test,
camprojection's depth clamp and the cutoff clamps."""

import math

import numpy as np

from mujoco_warp_b200._src import constants as C
from tests.constraint_oracle import MARGIN, E, KnifeEdge, cross, matvec, qconj, qmul, v3

REAL, POSITIVE, AXIS, QUATERNION = 0, 1, 2, 3
# the slots other kernels write (k_sensor_collision, k_sensor_contact, k_energy)
OTHER_KERNELS = (C.SENS_GEOMDIST, C.SENS_GEOMNORMAL, C.SENS_GEOMFROMTO, C.SENS_CONTACT, C.SENS_E_POTENTIAL, C.SENS_E_KINETIC, C.SENS_RANGEFINDER)
EXTRA = (C.SENS_MAGNETOMETER, C.SENS_CAMPROJECTION, C.SENS_INSIDESITE, C.SENS_TENDONLIMITPOS, C.SENS_TENDONLIMITVEL, C.SENS_TENDONLIMITFRC,
         C.SENS_TENDONACTFRC)
STAGE_BIT = {1: 1, 2: 2, 3: 4}


def _edge(x, scale, what):
  if abs(x) < MARGIN * max(scale, 1e-300):
    raise KnifeEdge(f"{what}: {x:.3g} is within {MARGIN} x {scale:.3g} of its threshold")


def _a(x):
  return np.asarray(x, dtype=np.float64)


def _vec(x):
  return [E(float(v)) for v in _a(x).reshape(-1)]


def add(a, b):
  return [x + y for x, y in zip(a, b)]


def sub(a, b):
  return [x - y for x, y in zip(a, b)]


def scl(a, s):
  return [x * s for x in a]


def mat_t_vec(R, a):
  return matvec(_a(R).reshape(3, 3).T, a)


# ------------------------------------------------------------------ prerequisites


def subtree_vel(m, st):
  """k_body_subtree_vel.cuh (reference smooth.py:3500-3612) -> subtree_linvel, subtree_angmom: lists of nbody E-vectors."""
  nb = int(m.nbody)
  root, parent = np.asarray(m.body_rootid), np.asarray(m.body_parentid)
  mass, smass, inertia = _a(m.body_mass), _a(m.body_subtreemass), _a(m.body_inertia).reshape(nb, 3)
  cvel, xipos, ximat, com = _a(st["cvel"]).reshape(nb, 6), _a(st["xipos"]).reshape(nb, 3), _a(st["ximat"]).reshape(nb, 9), _a(st["subtree_com"]).reshape(nb, 3)
  lin, ang, blin = [], [], []
  for b in range(nb):
    w = v3(cvel[b, :3])
    lb = sub(v3(cvel[b, 3:]), cross(sub(v3(xipos[b]), v3(com[root[b]])), w))
    dv = mat_t_vec(ximat[b], w)
    dv = [dv[k] * inertia[b, k] for k in range(3)]
    lin.append(scl(lb, mass[b]))
    ang.append(matvec(ximat[b].reshape(3, 3), dv))
    blin.append(lb)
  children = [[] for _ in range(nb)]
  for b in range(1, nb):
    children[parent[b]].append(b)
  for b in range(nb - 1, -1, -1):  # children before parents (a child's id is larger than its parent's)
    s = lin[b]
    for c in children[b]:
      s = add(s, scl(lin[c], smass[c]))
    lin[b] = scl(s, 1.0 / max(C.MJ_MINVAL, smass[b]))
  for b in range(1, nb):
    ang[b] = add(ang[b], cross(sub(v3(xipos[b]), v3(com[b])), scl(sub(blin[b], lin[b]), mass[b])))
  for b in range(nb - 1, -1, -1):
    s = ang[b]
    for c in children[b]:
      s = add(add(s, ang[c]), cross(sub(v3(com[c]), v3(com[b])), scl(sub(lin[c], lin[b]), smass[c])))
    ang[b] = s
  return lin, ang


def contact_force(m, st, i, njmax):
  """The contact's 6-vector in its frame from efc_force (support.py contact_force_fn, rows at or past njmax read as 0)."""
  force = _a(st["efc_force"])
  adr = np.asarray(st["con_efc_address"][i]).reshape(-1)
  dim = int(st["con_dim"][i])
  fc = [E(0.0) for _ in range(6)]
  f = lambda a: E(force[a]) if 0 <= a < njmax else E(0.0)
  if adr[0] < 0:
    return fc
  if int(m.opt.cone) == C.CONE_PYRAMIDAL:
    if dim == 1:
      fc[0] = f(adr[0])
    else:
      fr = _a(st["con_friction"][i]).reshape(-1)
      for k in range(dim - 1):
        d1, d2 = f(2 * k + adr[0]), f(2 * k + adr[0] + 1)
        fc[0] = fc[0] + d1 + d2
        fc[k + 1] = (d1 - d2) * fr[k]
  else:
    for k in range(dim):
      if adr[k] >= 0:
        fc[k] = f(adr[k])
  return fc


def rne_post(m, st, njmax):
  """k_body_rne_post.cuh (reference smooth.py:1743 rne_postconstraint) -> cacc, cfrc_ext, cfrc_int: lists of nbody E 6-vectors."""
  nb, nv = int(m.nbody), int(m.nv)
  root, parent = np.asarray(m.body_rootid), np.asarray(m.body_parentid)
  xipos, com = _a(st["xipos"]).reshape(nb, 3), _a(st["subtree_com"]).reshape(nb, 3)
  xpos, xmat = _a(st["xpos"]).reshape(nb, 3), _a(st["xmat"]).reshape(nb, 9)
  xfrc = _a(st.get("xfrc_applied", np.zeros((nb, 6)))).reshape(nb, 6)
  zero6 = lambda: [E(0.0) for _ in range(6)]
  cext = [zero6()]
  for b in range(1, nb):
    f = v3(xfrc[b, :3])
    t = sub(v3(xfrc[b, 3:]), cross(sub(v3(com[root[b]]), v3(xipos[b])), f))
    cext.append(t + f)
  force = _a(st["efc_force"])
  ne_rows = min(int(st["ne"]), njmax)
  fr = lambda r: E(force[r]) if r < ne_rows else E(0.0)
  eq_type, eq_data = np.asarray(m.eq_type) if int(m.neq) else [], _a(m.eq_data).reshape(-1, 11) if int(m.neq) else None
  e = 0
  while e < ne_rows:
    eid = int(st["efc_id"][e])
    typ = int(eq_type[eid])
    if typ not in (C.EQ_CONNECT, C.EQ_WELD):
      break
    f = [fr(e), fr(e + 1), fr(e + 2)]
    tq = [fr(e + 3), fr(e + 4), fr(e + 5)] if typ == C.EQ_WELD else [E(0.0)] * 3
    for side, b in enumerate((int(m.eq_obj1id[eid]), int(m.eq_obj2id[eid]))):
      if b == 0:
        continue
      anchor = eq_data[eid, 0:3] if (typ == C.EQ_CONNECT) == (side == 0) else eq_data[eid, 3:6]
      pos = add(matvec(xmat[b].reshape(3, 3), v3(anchor)), v3(xpos[b]))
      t = sub(tq, cross(sub(v3(com[root[b]]), pos), f))
      cext[b] = [c - x if side else c + x for c, x in zip(cext[b], t + f)]
    e += 3 if typ == C.EQ_CONNECT else 6
  geom_body = np.asarray(m.geom_bodyid)
  for i in range(len(st["con_geom"])):
    g = np.asarray(st["con_geom"][i]).reshape(2)
    id1, id2 = int(geom_body[g[0]]), int(geom_body[g[1]])
    if id1 == 0 and id2 == 0:
      continue
    fc = contact_force(m, st, i, njmax)
    R = _a(st["con_frame"][i]).reshape(3, 3)
    fw = matvec(R.T, fc[:3])
    tw = matvec(R.T, fc[3:])
    pos = v3(st["con_pos"][i])
    for side, b in enumerate((id1, id2)):
      if b == 0:
        continue
      t = sub(tw, cross(sub(v3(com[root[b]]), pos), fw))
      cext[b] = [c + x if side else c - x for c, x in zip(cext[b], t + fw)]
  grav = [E(0.0)] * 3 if int(m.opt.disableflags) & C.DSBL_GRAVITY else [E(-g) for g in _a(m.opt.gravity).reshape(3)]
  cacc = [[E(0.0)] * 3 + grav]
  cdof, cdd = _a(st["cdof"]).reshape(nv, 6), _a(st["cdof_dot"]).reshape(nv, 6)
  qvel, qacc = _a(st["qvel"]).reshape(nv), _a(st["qacc"]).reshape(nv)
  for b in range(1, nb):
    a = list(cacc[parent[b]])
    for j in range(int(m.body_dofnum[b])):
      dof = int(m.body_dofadr[b]) + j
      a = [a[k] + E(cdd[dof, k]) * qvel[dof] + E(cdof[dof, k]) * qacc[dof] for k in range(6)]
    cacc.append(a)
  cinert, cvel = _a(st["cinert"]).reshape(nb, 10), _a(st["cvel"]).reshape(nb, 6)
  cint = [zero6()]
  for b in range(1, nb):
    f = inert_vec(cinert[b], cacc[b])
    iv = inert_vec(cinert[b], _vec(cvel[b]))
    v = _vec(cvel[b])
    g = add(cross(v[:3], iv[:3]), cross(v[3:], iv[3:])) + cross(v[:3], iv[3:])
    cint.append([f[k] + g[k] - cext[b][k] for k in range(6)])
  for b in range(nb - 1, 0, -1):
    cint[parent[b]] = add(cint[parent[b]], cint[b])
  return cacc, cext, cint


def inert_vec(i, v):
  i = [E(x) for x in i]
  return [i[0] * v[0] + i[3] * v[1] + i[4] * v[2] - i[8] * v[4] + i[7] * v[5], i[3] * v[0] + i[1] * v[1] + i[5] * v[2] + i[8] * v[3] - i[6] * v[5],
          i[4] * v[0] + i[5] * v[1] + i[2] * v[2] - i[7] * v[3] + i[6] * v[4], i[8] * v[1] - i[7] * v[2] + i[9] * v[3],
          i[6] * v[2] - i[8] * v[0] + i[9] * v[4], i[7] * v[0] - i[6] * v[1] + i[9] * v[5]]


# ------------------------------------------------------------------ the touch sensor's ray against its site volume (mjb_ray.cuh)


def _quad(a, b, c, what):
  """Roots of a x^2 + 2 b x + c (mjb_ray.cuh ray_quad), or None when the discriminant is negative (asserted off its edge)."""
  det = b * b - a * c
  _edge(det, b * b + abs(a * c), what + " discriminant")
  if det < C.MJ_MINVAL:
    return None
  det = math.sqrt(det)
  den = 1.0 / a if a != 0 else 0.0
  return (-b - det) * den, (-b + det) * den


def _ge0(x, what):
  _edge(x, 1.0, what)
  return x >= 0


def _first(xx, what):
  """ray_quad's result: the smaller root if non-negative, else the larger, else -1."""
  if xx is None:
    return -1.0
  if _ge0(xx[0], what + " near root"):
    return xx[0]
  return xx[1] if _ge0(xx[1], what + " far root") else -1.0


def _sphere_hit(pos, r2, pnt, vec, what):
  dif = pnt - pos
  return _first(_quad(vec @ vec, vec @ dif, dif @ dif - r2, what), what) >= 0


def ray_hit(pos, mat, size, pnt, vec, typ):
  """Whether the ray pnt + x vec (x >= 0) meets the site volume: ray_geom<false> >= 0 for sphere, capsule, ellipsoid, cylinder and box."""
  pos, mat, size, pnt, vec = _a(pos), _a(mat).reshape(3, 3), _a(size), _a(pnt), _a(vec)
  if typ == C.GEOM_SPHERE:
    return _sphere_hit(pos, size[0] ** 2, pnt, vec, "sphere")
  lp, lv = mat.T @ (pnt - pos), mat.T @ vec
  if typ == C.GEOM_CAPSULE:
    if not _sphere_hit(pos, (size[0] + size[1]) ** 2, pnt, vec, "capsule bound"):
      return False
    hit = False
    r2, h = size[0] ** 2, size[1]
    a, b, c = lv[0] ** 2 + lv[1] ** 2, lv[0] * lp[0] + lv[1] * lp[1], lp[0] ** 2 + lp[1] ** 2 - r2
    sol = _first(_quad(a, b, c, "capsule side"), "capsule side")
    if sol >= 0:
      z = h - abs(lp[2] + sol * lv[2])
      _edge(z, h, "capsule side height")
      hit = z >= 0
    a += lv[2] ** 2
    for sgn in (1.0, -1.0):  # top cap: both roots with z >= h; bottom cap: z <= -h
      ld = lp - np.array([0.0, 0.0, sgn * h])
      xx = _quad(a, lv @ ld, ld @ ld - r2, "capsule cap")
      for x in xx if xx is not None else ():
        if _ge0(x, "capsule cap root"):
          z = sgn * (lp[2] + x * lv[2]) - h
          _edge(z, h, "capsule cap height")
          hit |= z >= 0
    return hit
  if typ == C.GEOM_ELLIPSOID:
    si = np.array([1.0 / s ** 2 if s != 0 else 0.0 for s in size])
    return _first(_quad((si * lv) @ lv, (si * lv) @ lp, (si * lp) @ lp - 1.0, "ellipsoid"), "ellipsoid") >= 0
  if typ == C.GEOM_CYLINDER:
    if not _sphere_hit(pos, size[0] ** 2 + size[1] ** 2, pnt, vec, "cylinder bound"):
      return False
    hit = False
    r2, h = size[0] ** 2, size[1]
    if abs(lv[2]) > C.MJ_MINVAL:
      for side in (-1.0, 1.0):
        sol = (side * h - lp[2]) / lv[2]
        if _ge0(sol, "cylinder cap root"):
          p = lp[:2] + sol * lv[:2]
          _edge(r2 - p @ p, r2, "cylinder cap radius")
          hit |= p @ p <= r2
    sol = _first(_quad(lv[0] ** 2 + lv[1] ** 2, lv[0] * lp[0] + lv[1] * lp[1], lp[0] ** 2 + lp[1] ** 2 - r2, "cylinder side"), "cylinder side")
    if sol >= 0:
      z = h - abs(lp[2] + sol * lv[2])
      _edge(z, h, "cylinder side height")
      hit |= z >= 0
    return hit
  if typ == C.GEOM_BOX:
    if not _sphere_hit(pos, size @ size, pnt, vec, "box bound"):
      return False
    hit = False
    for i in range(3):
      if abs(lv[i]) <= C.MJ_MINVAL:
        continue
      for side in (-1.0, 1.0):
        sol = (side * size[i] - lp[i]) / lv[i]
        if not _ge0(sol, "box face root"):
          continue
        i0, i1 = (1 if i == 0 else 0), (1 if i == 2 else 2)
        m0, m1 = size[i0] - abs(lp[i0] + sol * lv[i0]), size[i1] - abs(lp[i1] + sol * lv[i1])
        _edge(m0, size[i0], "box face extent")
        _edge(m1, size[i1], "box face extent")
        hit |= m0 >= 0 and m1 >= 0
    return hit
  return False


def touch(m, st, sid, njmax):
  """sensor.py:2063: the summed normal force of the site body's contacts whose force ray meets the site volume."""
  site = int(m.sensor_objid[sid])
  body = int(m.site_bodyid[site])
  geom_body = np.asarray(m.geom_bodyid)
  force = _a(st["efc_force"])
  f = lambda a: force[a] if 0 <= a < njmax else 0.0
  sxpos, sxmat = _a(st["site_xpos"]).reshape(-1, 3)[site], _a(st["site_xmat"]).reshape(-1, 9)[site]
  size = _a(m.site_size).reshape(-1, 3)[site]
  total = E(0.0)
  for i in range(len(st["con_geom"])):
    g = np.asarray(st["con_geom"][i]).reshape(2)
    b1, b2 = int(geom_body[g[0]]), int(geom_body[g[1]])
    adr = np.asarray(st["con_efc_address"][i]).reshape(-1)
    if adr[0] < 0 or body not in (b1, b2):
      continue
    terms = [f(adr[0])]
    if int(m.opt.cone) == C.CONE_PYRAMIDAL:
      terms += [f(a) for a in adr[1 : 2 * (int(st["con_dim"][i]) - 1)]]  # rows cut by njmax (address -1 or >= njmax) read as 0
    nf = sum(terms)
    if any(t < 0 for t in terms):  # a sum of non-negative forces is positive in any precision exactly when one term is
      _edge(nf, sum(abs(t) for t in terms), "touch normal force")
    if nf <= 0:
      continue
    ray = _a(st["con_frame"][i]).reshape(3, 3)[0] * nf
    ray = ray / np.linalg.norm(ray)
    if body == b2:
      ray = -ray
    if ray_hit(sxpos, sxmat, size, _a(st["con_pos"][i]), ray, int(m.site_type[site])):
      total = total + E(nf, sum(abs(t) for t in terms))
  return [total]


# ------------------------------------------------------------------ the other sensors


def _obj_pos(st, ot, i):
  key = {C.OBJ_BODY: "xipos", C.OBJ_XBODY: "xpos", C.OBJ_GEOM: "geom_xpos", C.OBJ_SITE: "site_xpos", C.OBJ_CAMERA: "cam_xpos"}[ot]
  return _a(st[key]).reshape(-1, 3)[i]


def _obj_mat(st, ot, i):
  key = {C.OBJ_BODY: "ximat", C.OBJ_XBODY: "xmat", C.OBJ_GEOM: "geom_xmat", C.OBJ_SITE: "site_xmat", C.OBJ_CAMERA: "cam_xmat"}[ot]
  return _a(st[key]).reshape(-1, 9)[i]


def _obj_body(m, ot, i):
  if ot in (C.OBJ_BODY, C.OBJ_XBODY):
    return i
  return int({C.OBJ_GEOM: m.geom_bodyid, C.OBJ_SITE: m.site_bodyid, C.OBJ_CAMERA: m.cam_bodyid}[ot][i])


def _obj_quat(m, st, ot, i):
  """sensor.py:342-373: the body's xquat times the object's local quaternion (body_iquat, geom_quat, site_quat, cam_quat)."""
  q = _vec(_a(st["xquat"]).reshape(-1, 4)[_obj_body(m, ot, i)])
  local = {C.OBJ_BODY: "body_iquat", C.OBJ_GEOM: "geom_quat", C.OBJ_SITE: "site_quat", C.OBJ_CAMERA: "cam_quat"}.get(ot)
  return qmul(q, _vec(_a(getattr(m, local)).reshape(-1, 4)[i])) if local else q


def _frame_vel(m, st, ot, i):
  """(ang, lin) of the object's point: the body's cvel shifted from its root's subtree com to the object."""
  b = _obj_body(m, ot, i)
  cv = _a(st["cvel"]).reshape(-1, 6)[b]
  ang, pos = v3(cv[:3]), v3(_obj_pos(st, ot, i))
  com = v3(_a(st["subtree_com"]).reshape(-1, 3)[int(m.body_rootid[b])])
  return ang, sub(v3(cv[3:]), cross(sub(pos, com), ang)), pos


def _limit(st, typ, idx, which, njmax):
  """sensor.py:228 / :1028 / :1640: the last limit row of the object below njmax, else 0."""
  e0 = int(st["ne"]) + int(st["nf"])
  out = E(0.0)
  for e in range(e0, min(e0 + int(st["nl"]), njmax)):
    if int(st["efc_id"][e]) == idx and int(st["efc_type"][e]) == typ:
      out = (E(st["efc_pos"][e]) - E(st["efc_margin"][e])) if which == 0 else E(st["efc_vel"][e] if which == 1 else st["efc_force"][e])
  return [out]


def _inside(pos, mat, size, typ, p):
  """mjb_sensor_contact.cuh contact_inside_site (util_misc.py:676 inside_geom), every comparison asserted off its edge."""
  v = p - pos
  if typ == C.GEOM_SPHERE:
    x = size[0] ** 2 - v @ v
    _edge(x, size[0] ** 2, "insidesite sphere")
    return x > 0
  l = mat.reshape(3, 3).T @ v
  if typ == C.GEOM_CAPSULE:
    z = l[2] - min(max(l[2], -size[1]), size[1])
    x = size[0] ** 2 - (l[0] ** 2 + l[1] ** 2 + z * z)
    _edge(x, size[0] ** 2, "insidesite capsule")
    return x > 0
  if typ == C.GEOM_ELLIPSOID:
    x = 1.0 - np.sum((l / size) ** 2)
    _edge(x, 1.0, "insidesite ellipsoid")
    return x > 0
  if typ == C.GEOM_CYLINDER:
    a, r = size[1] - abs(l[2]), size[0] ** 2 - l[0] ** 2 - l[1] ** 2
    _edge(a, size[1], "insidesite cylinder height")
    _edge(r, size[0] ** 2, "insidesite cylinder radius")
    return a > 0 and r > 0
  if typ == C.GEOM_BOX:
    x = size - np.abs(l)
    for k in range(3):
      _edge(x[k], size[k], "insidesite box")
    return bool((x > 0).all())
  if typ == C.GEOM_PLANE:
    _edge(l[2], 1.0, "insidesite plane")
    return l[2] < 0
  return False


def _camprojection(m, st, site, cam):
  """sensor.py:131: pixel coordinates of the site in the camera's image."""
  R = _a(st["cam_xmat"]).reshape(-1, 9)[cam]
  v = mat_t_vec(R, sub(v3(_a(st["site_xpos"]).reshape(-1, 3)[site]), v3(_a(st["cam_xpos"]).reshape(-1, 3)[cam])))
  res = np.asarray(m.cam_resolution).reshape(-1, 2)[cam].astype(np.float64)
  ss = _a(m.cam_sensorsize).reshape(-1, 2)[cam]
  if ss[0] != 0 and ss[1] != 0:
    intr = _a(m.cam_intrinsic).reshape(-1, 4)[cam]
    fx, fy = E(intr[0]) / (ss[0] + C.MJ_MINVAL) * res[0], E(intr[1]) / (ss[1] + C.MJ_MINVAL) * res[1]
  else:
    fovy = float(_a(m.cam_fovy).reshape(-1)[cam])
    t = math.tan(fovy * math.pi / 360.0)
    fx = fy = E(0.5 / t * res[1], 0.5 / t * res[1] * (1.0 + math.pi / 360.0 * abs(fovy) * (1.0 + t * t) / t))
  den = v[2]
  _edge(abs(den.v) - C.MJ_MINVAL, 1.0, "camprojection depth clamp")
  return [-fx * v[0] / den + 0.5 * res[0], fy * v[1] / den + 0.5 * res[1]]


def sensor_value(m, st, s, njmax, pre):
  """The unclipped E values of sensor s; pre: the in-launch prerequisites (subtree_vel / rne_post results)."""
  t, i = int(m.sensor_type[s]), int(m.sensor_objid[s])
  ot, rt, rid = int(m.sensor_objtype[s]), int(m.sensor_reftype[s]), int(m.sensor_refid[s])
  g = lambda k, n: _a(st[k]).reshape(-1, n)
  site_r = lambda: g("site_xmat", 9)[i]
  if t == C.SENS_JOINTPOS:
    return [E(st["qpos"][int(m.jnt_qposadr[i])])]
  if t == C.SENS_TENDONPOS:
    return [E(st["ten_length"][i])]
  if t == C.SENS_ACTUATORPOS:
    return [E(st["actuator_length"][i])]
  if t == C.SENS_BALLQUAT:
    a = int(m.jnt_qposadr[i])
    q = _vec(st["qpos"][a : a + 4])
    n = math.sqrt(sum(x.v ** 2 for x in q))
    return [x / n for x in q]
  if t == C.SENS_FRAMEPOS:
    r = v3(_obj_pos(st, ot, i))
    return mat_t_vec(_obj_mat(st, rt, rid), sub(r, v3(_obj_pos(st, rt, rid)))) if rid > -1 else r
  if t in (C.SENS_FRAMEXAXIS, C.SENS_FRAMEYAXIS, C.SENS_FRAMEZAXIS):
    r = v3(_obj_mat(st, ot, i).reshape(3, 3)[:, t - C.SENS_FRAMEXAXIS])
    return mat_t_vec(_obj_mat(st, rt, rid), r) if rid > -1 else r
  if t == C.SENS_FRAMEQUAT:
    q = _obj_quat(m, st, ot, i)
    return qmul(qconj(_obj_quat(m, st, rt, rid)), q) if rid > -1 else q
  if t == C.SENS_SUBTREECOM:
    return v3(g("subtree_com", 3)[i])
  if t == C.SENS_CLOCK:
    return [E(float(np.asarray(st["time"]).reshape(-1)[0]))]
  if t in (C.SENS_JOINTLIMITPOS, C.SENS_JOINTLIMITVEL, C.SENS_JOINTLIMITFRC):
    return _limit(st, C.CNSTR_LIMIT_JOINT, i, t - C.SENS_JOINTLIMITPOS, njmax)
  if t == C.SENS_JOINTVEL:
    return [E(st["qvel"][int(m.jnt_dofadr[i])])]
  if t == C.SENS_TENDONVEL:
    return [E(st["ten_velocity"][i])]
  if t == C.SENS_ACTUATORVEL:
    return [E(st["actuator_velocity"][i])]
  if t == C.SENS_BALLANGVEL:
    a = int(m.jnt_dofadr[i])
    return _vec(st["qvel"][a : a + 3])
  if t in (C.SENS_FRAMELINVEL, C.SENS_FRAMEANGVEL):
    ang, lin, pos = _frame_vel(m, st, ot, i)
    if rid < 0:
      return lin if t == C.SENS_FRAMELINVEL else ang
    rang, rlin, rpos = _frame_vel(m, st, rt, rid)
    rel = add(sub(lin, rlin), cross(sub(pos, rpos), rang)) if t == C.SENS_FRAMELINVEL else sub(ang, rang)
    return mat_t_vec(_obj_mat(st, rt, rid), rel)
  if t == C.SENS_SUBTREELINVEL:
    return pre["subtree_linvel"][i]
  if t == C.SENS_SUBTREEANGMOM:
    return pre["subtree_angmom"][i]
  if t == C.SENS_GYRO:
    return mat_t_vec(site_r(), v3(g("cvel", 6)[int(m.site_bodyid[i]), :3]))
  if t in (C.SENS_VELOCIMETER, C.SENS_ACCELEROMETER):
    ang, lin, _ = _frame_vel(m, st, C.OBJ_SITE, i)
    if t == C.SENS_VELOCIMETER:
      return mat_t_vec(site_r(), lin)
    b = int(m.site_bodyid[i])
    ca = pre["cacc"][b]
    dif = sub(v3(g("site_xpos", 3)[i]), v3(g("subtree_com", 3)[int(m.body_rootid[b])]))
    acc = mat_t_vec(site_r(), sub(ca[3:], cross(dif, ca[:3])))
    return add(acc, cross(mat_t_vec(site_r(), ang), mat_t_vec(site_r(), lin)))
  if t in (C.SENS_FRAMELINACC, C.SENS_FRAMEANGACC):
    b = _obj_body(m, ot, i)
    ca = pre["cacc"][b]
    if t == C.SENS_FRAMEANGACC:
      return ca[:3]
    ang, lin, pos = _frame_vel(m, st, ot, i)
    off = sub(pos, v3(g("subtree_com", 3)[int(m.body_rootid[b])]))
    return add(sub(ca[3:], cross(off, ca[:3])), cross(ang, lin))
  if t == C.SENS_TOUCH:
    return touch(m, st, s, njmax)
  if t in (C.SENS_FORCE, C.SENS_TORQUE):
    b = int(m.site_bodyid[i])
    cf = pre["cfrc_int"][b]
    if t == C.SENS_FORCE:
      return mat_t_vec(site_r(), cf[3:])
    dif = sub(v3(g("site_xpos", 3)[i]), v3(g("subtree_com", 3)[int(m.body_rootid[b])]))
    return mat_t_vec(site_r(), sub(cf[:3], cross(dif, cf[3:])))
  if t == C.SENS_ACTUATORFRC:
    return [E(st["actuator_force"][i])]
  if t == C.SENS_JOINTACTFRC:
    return [E(st["qfrc_actuator"][int(m.jnt_dofadr[i])])]
  if t == C.SENS_MAGNETOMETER:
    return mat_t_vec(site_r(), v3(_a(m.opt.magnetic).reshape(3)))
  if t == C.SENS_CAMPROJECTION:
    return _camprojection(m, st, i, rid)
  if t == C.SENS_INSIDESITE:
    p = _obj_pos(st, ot, i)
    if ot == C.OBJ_BODY and i > 0 and float(m.body_mass[i]) < C.MJ_MINVAL and float(m.body_subtreemass[i]) >= C.MJ_MINVAL:
      p = g("subtree_com", 3)[i]
    inside = _inside(g("site_xpos", 3)[rid], g("site_xmat", 9)[rid], _a(m.site_size).reshape(-1, 3)[rid], int(m.site_type[rid]), _a(p))
    return [E(1.0 if inside else 0.0)]
  if t in (C.SENS_TENDONLIMITPOS, C.SENS_TENDONLIMITVEL, C.SENS_TENDONLIMITFRC):
    return _limit(st, C.CNSTR_LIMIT_TENDON, i, t - C.SENS_TENDONLIMITPOS, njmax)
  if t == C.SENS_TENDONACTFRC:
    out = E(0.0)
    trn, trnid = np.asarray(m.actuator_trntype), np.asarray(m.actuator_trnid).reshape(-1, 2)
    for a in range(int(m.nu)):
      if int(trn[a]) == C.TRN_TENDON and int(trnid[a, 0]) == i:
        out = out + E(st["actuator_force"][a])
    return [out]
  raise NotImplementedError(f"sensor type {t}")


def cutoff(m, s, vals, fp32=True):
  """sensor.py:57-113: cutoff > 0 clamps REAL data to [-c, c] and POSITIVE data from above; AXIS and QUATERNION data are not clamped.
  fp32: clamp to the fp32 cutoff the kernel holds (else to the model's own value, as the fp64 reference does)."""
  c = float(_a(m.sensor_cutoff).reshape(-1)[s])
  c = float(np.float32(c)) if fp32 else c
  dt = int(m.sensor_datatype[s])
  if c <= 0 or dt not in (REAL, POSITIVE):
    return vals
  out = []
  for x in vals:
    _edge(x.v - c, max(c, x.m), f"sensor {s} cutoff")
    if dt == REAL:
      _edge(x.v + c, max(c, x.m), f"sensor {s} cutoff")
    out.append(E(c) if x.v > c else (E(-c) if dt == REAL and x.v < -c else x))
  return out


def carried(m, s, extra):
  """Whether k_sensor (with `extra`: its EXTRA build) writes sensor s."""
  t = int(m.sensor_type[s])
  return t not in OTHER_KERNELS and (extra or t not in EXTRA)


def sensor(m, st, njmax, stages=7, sensors=None, fp32_cutoff=True):
  """The fields one k_sensor launch with `stages` (1 pos | 2 vel | 4 acc) writes for this world, as {name: (value, magnitude)}:
  subtree_linvel / subtree_angmom (nbody, 3) when the velocity stage runs and a subtree velocity sensor exists, cacc / cfrc_ext /
  cfrc_int (nbody, 6) when the acceleration stage runs and an accelerometer, force, torque or frame acceleration sensor exists, and
  sensordata (nsensordata,) with NaN in every slot the launch leaves alone.  st: the world's arrays (see the module docstring): qpos,
  qvel, qacc, time, xpos / xquat / xmat / xipos / ximat, geom / site / cam xpos and xmat, subtree_com, cdof, cinert, cvel, cdof_dot,
  ten_length / ten_velocity, actuator_length / velocity / force, qfrc_actuator, xfrc_applied, efc_force / pos / margin / vel / type / id,
  ne / nf / nl and the contacts (con_geom, con_dim, con_frame, con_pos, con_friction, con_efc_address); a sensor reads only what its
  type needs.  sensors: restrict to these sensor ids (default: every one k_sensor's build for this model writes).  fp32_cutoff: see
  cutoff()."""
  nb = int(m.nbody)
  stype = np.asarray(m.sensor_type).reshape(-1)
  extra = bool(np.isin(stype, EXTRA).any())
  out, pre = {}, {}
  to_arr = lambda rows, n: (np.array([[x.v for x in r] for r in rows]).reshape(nb, n), np.array([[x.m for x in r] for r in rows]).reshape(nb, n))
  if stages & 2 and np.isin(stype, (C.SENS_SUBTREELINVEL, C.SENS_SUBTREEANGMOM)).any():
    pre["subtree_linvel"], pre["subtree_angmom"] = subtree_vel(m, st)
    out["subtree_linvel"], out["subtree_angmom"] = to_arr(pre["subtree_linvel"], 3), to_arr(pre["subtree_angmom"], 3)
  if stages & 4 and np.isin(stype, (C.SENS_ACCELEROMETER, C.SENS_FORCE, C.SENS_TORQUE, C.SENS_FRAMELINACC, C.SENS_FRAMEANGACC)).any():
    pre["cacc"], cext, pre["cfrc_int"] = rne_post(m, st, njmax)
    out["cacc"], out["cfrc_ext"], out["cfrc_int"] = to_arr(pre["cacc"], 6), to_arr(cext, 6), to_arr(pre["cfrc_int"], 6)
  n = int(m.nsensordata)
  val, mag = np.full(n, np.nan), np.full(n, np.nan)
  if not int(m.opt.disableflags) & C.DSBL_SENSOR:
    for s in range(len(stype)) if sensors is None else sensors:
      if not carried(m, s, extra) or not stages & STAGE_BIT[int(m.sensor_needstage[s])]:
        continue
      vals = cutoff(m, s, sensor_value(m, st, s, njmax, pre), fp32_cutoff)
      a, dim = int(m.sensor_adr[s]), int(m.sensor_dim[s])
      assert len(vals) == dim, f"sensor {s}: {len(vals)} values for dim {dim}"
      val[a : a + dim], mag[a : a + dim] = [x.v for x in vals], [x.m for x in vals]
  out["sensordata"] = (val, mag)
  return out
