"""fp64 restatement of the <contact> sensor (reference sensor.py:1810-2010, :2315-2510, support.py:326-397, util_misc.py:676).

`world_sensors` is a function of one world's contact arrays and efc_force, so that it can be fed either a reference fixture's contacts
or the GPU's own.  It returns, per contact sensor, the stored matches in slot order and the sensordata the sensor writes, following the
decisions documented in INTEGRATION.md:
  1. with more matches than num, the first num matches in pool order (reduce none);
  2. sort ties break by pool index;
  3. matches past maxmatch are counted (found, the overflow flag) but never read: netforce sums the stored ones, and slots past them are 0;
  4. netforce with num > 1 zeroes slots 2..num;
  5. a match's direction travels with it through the sort.
`reference_dir=True` restates the reference's fifth behaviour instead: its sort permutes the contact ids but not the directions, so slot
i takes the direction of the i-th match in pool order."""

import numpy as np

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf

def contact_force(cone, njmax, force, adr, mu, dim):
  """contact-frame force / torque (6) of one contact; rows cut by njmax read 0"""
  f = np.zeros(6)
  if adr[0] < 0:
    return f
  if cone == C.CONE_PYRAMIDAL:
    if dim == 1:
      f[0] = force[adr[0]] if adr[0] < njmax else 0.0
      return f
    for i in range(dim - 1):
      a = 2 * i + adr[0]
      d1 = force[a] if a < njmax else 0.0
      d2 = force[a + 1] if a + 1 < njmax else 0.0
      f[0] += d1 + d2
      f[i + 1] = (d1 - d2) * mu[i]
  else:
    for i in range(dim):
      if 0 <= adr[i] < njmax:
        f[i] = force[adr[i]]
  return f


def inside_site(pos, mat, size, typ, p):
  v = np.asarray(p, float) - pos
  if typ == C.GEOM_SPHERE:
    return v @ v < size[0] ** 2
  l = np.asarray(mat).reshape(3, 3).T @ v
  if typ == C.GEOM_CAPSULE:
    z = l[2] - np.clip(l[2], -size[1], size[1])
    return l[0] ** 2 + l[1] ** 2 + z * z < size[0] ** 2
  if typ == C.GEOM_ELLIPSOID:
    s = l / size
    return s @ s < 1.0
  if typ == C.GEOM_CYLINDER:
    return abs(l[2]) < size[1] and l[0] ** 2 + l[1] ** 2 < size[0] ** 2
  if typ == C.GEOM_BOX:
    return bool(np.all(np.abs(l) < size))
  if typ == C.GEOM_PLANE:
    return l[2] < 0.0
  return False


def side_match(parent, body, geom, typ, oid):
  if typ in (C.OBJ_UNKNOWN, C.OBJ_SITE):
    return True
  if typ == C.OBJ_GEOM:
    return oid == geom
  if typ == C.OBJ_BODY:
    return oid == body
  if typ == C.OBJ_XBODY:
    while body > oid:
      body = parent[body]
    return body == oid
  return False


def match_dir(parent, otype, oid, rtype, rid, g1, b1, g2, b2):
  """0 (no match) or the direction +-1 (sensor.py:2398-2436)"""
  if otype == C.OBJ_UNKNOWN and rtype == C.OBJ_UNKNOWN:
    return 1
  m11, m12 = side_match(parent, b1, g1, otype, oid), side_match(parent, b2, g2, otype, oid)
  m21, m22 = side_match(parent, b1, g1, rtype, rid), side_match(parent, b2, g2, rtype, rid)
  if (not m11 and not m12) or (not m21 and not m22):
    return 0
  if otype != C.OBJ_UNKNOWN and rtype != C.OBJ_UNKNOWN:
    regular, reverse = m11 and m22, m12 and m21
    if not regular and not reverse:
      return 0
    return -1 if reverse and not regular else 1
  if otype != C.OBJ_UNKNOWN:
    return 1 if m11 else -1
  return 1 if m22 else -1


def slot(dataspec, nmatch, d, f, dist, pos, frame):
  frame = np.asarray(frame, float).reshape(3, 3)
  out = []
  if dataspec & 1:
    out.append(float(nmatch))
  if dataspec & 2:
    out += [f[0], f[1], d * f[2]]
  if dataspec & 4:
    out += [f[3], f[4], d * f[5]]
  if dataspec & 8:
    out.append(dist)
  if dataspec & 16:
    out += list(pos)
  if dataspec & 32:
    out += list(d * frame[0])
  if dataspec & 64:
    out += list(d * frame[1])
  return np.array(out, dtype=float)


def netforce(dataspec, nmatch, items):
  """items: (dir, f6, pos, frame) of the stored matches"""
  net_pos, net_f, net_t, total = np.zeros(3), np.zeros(3), np.zeros(3), 0.0
  for d, f, pos, frame in items:
    R = np.asarray(frame, float).reshape(3, 3)
    w = np.linalg.norm(f[:3])
    net_pos += w * np.asarray(pos)
    total += w
    fg, tg = R.T @ (d * f[:3]), R.T @ (d * f[3:])
    net_f += fg
    net_t += tg + np.cross(pos, fg)
  net_pos /= max(total, 1e-15)
  net_t -= np.cross(net_pos, net_f)
  out = []
  if dataspec & 1:
    out.append(float(nmatch))
  if dataspec & 2:
    out += list(net_f)
  if dataspec & 4:
    out += list(net_t)
  if dataspec & 8:
    out.append(0.0)
  if dataspec & 16:
    out += list(net_pos)
  if dataspec & 32:
    out += [1.0, 0.0, 0.0]
  if dataspec & 64:
    out += [0.0, 1.0, 0.0]
  return np.array(out, dtype=float)


def netforce_scale(dataspec, items):
  """per entry of the netforce slot, the magnitude of the terms summed into it: fp32 cancellation makes a component's rounding error
  proportional to this, not to the (possibly much smaller) result.  Torque: every contact's |torque| + |pos| |force| and the centroid
  term |c| |F|; force: the sum of |force|; centroid: the largest |pos|."""
  f_sum, t_sum, p_max, w_sum, wp = 0.0, 0.0, 0.0, 0.0, np.zeros(3)
  for _, f, pos, _ in items:
    fn, pn = np.linalg.norm(f[:3]), np.linalg.norm(pos)
    f_sum += fn
    t_sum += np.linalg.norm(f[3:]) + pn * fn
    p_max = max(p_max, pn)
  t_sum += p_max * f_sum
  out = []
  if dataspec & 1:
    out.append(0.0)
  if dataspec & 2:
    out += [f_sum] * 3
  if dataspec & 4:
    out += [t_sum] * 3
  if dataspec & 8:
    out.append(0.0)
  if dataspec & 16:
    out += [p_max] * 3
  out += [0.0] * (3 * (bool(dataspec & 32) + bool(dataspec & 64)))
  return np.array(out, dtype=float)


def world_sensors(mjm, con, efc_force, njmax, maxmatch, site_xpos, site_xmat, reference_dir=False):
  """One world.  con: that world's contacts in pool order, dict of dist (n), pos (n, 3), frame (n, 9), friction (n, 5), dim (n),
  geom (n, 2), efc_address (n, k), type (n).  Returns ({sensor id: result}, overflow), result = dict(nmatch, reduce, num, size,
  matches: [(pool index within con, criterion, dir)] in slot order, slots: the slot vector of every stored match in that order,
  data: the sensor's sensordata, scale: netforce_scale of the netforce slot, 0 elsewhere)."""
  cone = int(mjm.opt.cone)
  parent, gbody = np.asarray(mjm.body_parentid), np.asarray(mjm.geom_bodyid)
  intprm = np.asarray(mjm.sensor_intprm).reshape(-1, 3)
  stype = np.asarray(mjm.sensor_type)
  n = len(con["dist"])
  frames = np.asarray(con["frame"], float).reshape(n, 9)
  forces = [contact_force(cone, njmax, efc_force, np.asarray(con["efc_address"][c]), np.asarray(con["friction"][c], float), int(con["dim"][c])) for c in range(n)]
  out, overflow = {}, False
  for s in np.nonzero(stype == C.SENS_CONTACT)[0]:
    dataspec, reduce, num = (int(x) for x in intprm[s])
    otype, oid = int(mjm.sensor_objtype[s]), int(mjm.sensor_objid[s])
    rtype, rid = int(mjm.sensor_reftype[s]), int(mjm.sensor_refid[s])
    size = mjcf.contact_slot_size(dataspec)
    matches = []
    for c in range(n):
      if not int(con["type"][c]) & C.CONTACT_TYPE_CONSTRAINT:
        continue
      if otype == C.OBJ_SITE and not inside_site(site_xpos[oid], site_xmat[oid], np.asarray(mjm.site_size)[oid], int(np.asarray(mjm.site_type)[oid]), con["pos"][c]):
        continue
      g1, g2 = int(con["geom"][c][0]), int(con["geom"][c][1])
      d = match_dir(parent, otype, oid, rtype, rid, g1, int(gbody[g1]), g2, int(gbody[g2]))
      if d == 0:
        continue
      crit = 0.0
      if reduce == 1:
        crit = float(con["dist"][c])
      elif reduce == 2:
        crit = -float(forces[c][:3] @ forces[c][:3])
      matches.append((c, crit, float(d)))
    nmatch = len(matches)
    overflow |= nmatch > maxmatch
    stored = matches[:maxmatch]
    if reduce in (1, 2):
      order = sorted(range(len(stored)), key=lambda i: (stored[i][1], stored[i][0]))
      dirs = [m[2] for m in stored]
      stored = [stored[i] for i in order]
      if reference_dir:
        stored = [(c, crit, dirs[i]) for i, (c, crit, _) in enumerate(stored)]
    slots = [slot(dataspec, nmatch, d, forces[c], float(con["dist"][c]), np.asarray(con["pos"][c], float), frames[c]) for c, _, d in stored]
    data, scale = np.zeros(num * size), np.zeros(num * size)
    if reduce == 3:
      items = [(d, forces[c], np.asarray(con["pos"][c], float), frames[c]) for c, _, d in stored]
      data[:size], scale[:size] = netforce(dataspec, nmatch, items), netforce_scale(dataspec, items)
    else:
      for i in range(min(len(stored), num)):
        data[i * size : (i + 1) * size] = slots[i]
    out[int(s)] = dict(nmatch=nmatch, reduce=reduce, num=num, size=size, matches=stored, slots=slots, data=data, scale=scale)
  return out, overflow


def world_contacts(con_all, w):
  """the contacts of world w (in pool order) from a pool of several worlds' contacts (dict of arrays with a worldid entry)"""
  idx = np.nonzero(np.asarray(con_all["worldid"]) == w)[0]
  return {k: np.asarray(v)[idx] for k, v in con_all.items()}


def tie_groups(crit, rel=1e-5, abs_=1e-7):
  """for sorted criteria, the group index of each position: consecutive entries whose criteria agree within the tolerance share a group"""
  g, out = 0, []
  for i, c in enumerate(crit):
    if i and abs(c - crit[i - 1]) > abs_ + rel * max(abs(c), abs(crit[i - 1])):
      g += 1
    out.append(g)
  return out


def check_sensor(got, res, rtol, atol, order_free=False, what=""):
  """got: a sensor's sensordata from the device; res: world_sensors' result.  Slot i must equal the restatement's slot i, or, where the
  restatement's criteria tie (mindist / maxforce) or with `order_free`, the slot of any match of that tie group / of any stored match.
  Slots past the stored matches are 0."""
  size, num, reduce = res["size"], res["num"], res["reduce"]
  got = np.asarray(got, float)
  if reduce == 3:  # sums: the error bound grows with the magnitude of the summed terms (netforce_scale), 30 fp32 ulps of it
    err, bound = np.abs(got - res["data"]), atol + rtol * np.abs(res["data"]) + 2e-6 * res["scale"]
    assert np.all(err <= bound), f"{what}: netforce {got} vs {res['data']}, error {err} above {bound}"
    return
  nslot = min(len(res["matches"]), num)
  # mindist criteria are the contacts' own dist values, so its ties are exact and break by pool index; maxforce's are recomputed in fp64
  crit = [m[1] for m in res["matches"]]
  groups = tie_groups(crit, rel=0.0, abs_=0.0) if reduce == 1 and not order_free else tie_groups(crit) if reduce in (1, 2) else list(range(len(crit)))
  for i in range(num):
    g = got[i * size : (i + 1) * size]
    if i >= nslot:
      assert np.all(g == 0.0), f"{what}: slot {i} past the matches is not zero: {g}"
      continue
    cands = range(len(res["slots"])) if order_free else [j for j in range(len(res["slots"])) if groups[j] == groups[i]]
    ok = any(np.allclose(g, res["slots"][j], rtol=rtol, atol=atol) for j in cands)
    assert ok, f"{what}: slot {i} {g} matches none of {[res['slots'][j] for j in cands]}"
