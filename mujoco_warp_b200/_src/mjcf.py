"""Mini MJCF compiler: MJCF XML -> MjModel-like numpy object (host side, not the hot path).

The reference delegates model compilation to the `mujoco` C library
(`/root/reference/mujoco_warp/_src/cli.py:78-100`: MjSpec.from_file -> compile), which is not
installed in this image.  This module restates the documented MuJoCo compilation semantics for the
MJCF subset used by the BASELINE scenes (defaults/classes, fromto capsules, spheres, boxes, planes,
hinge/slide/ball/free joints, motor/position/velocity/general actuators, cameras/lights, keyframes,
contact excludes, explicit <inertial>).  Its output exposes MjModel-named numpy attributes so that
`io.put_model` can copy fields by name exactly like `/root/reference/mujoco_warp/_src/io.py:426`.

Constants that need computation rather than parsing (body inertia from geoms, subtreemass,
rbound/aabb, invweight0, meaninertia, cam/light reference poses, CSR sparsity of M) are derived here;
SURVEY.md Appendix C lists them.  `put_model` also accepts a real `mujoco.MjModel` when that package
exists, so this compiler is a stand-in, not a fork of the API.
"""

from __future__ import annotations

import math
import os
import xml.etree.ElementTree as ET
from types import SimpleNamespace

import numpy as np

from . import constants as C

# ----------------------------------------------------------------------------------------------
# small math helpers (float64)
# ----------------------------------------------------------------------------------------------


def _vec(s, n=None, default=None):
  if s is None:
    return None if default is None else np.array(default, dtype=np.float64)
  v = np.array([float(x) for x in s.split()], dtype=np.float64)
  if n is not None and v.size < n and default is not None:
    d = np.array(default, dtype=np.float64)
    d[: v.size] = v
    v = d
  return v


def quat_mul(a, b):
  return np.array(
    [
      a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
      a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
      a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
      a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0],
    ]
  )


def quat_to_mat(q):
  w, x, y, z = q
  return np.array(
    [
      [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
      [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
      [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z],
    ]
  )


def mat_to_quat(R):
  """Rotation matrix -> unit quaternion (w,x,y,z), w >= 0 branch-stable."""
  t = np.trace(R)
  if t > 0:
    s = math.sqrt(t + 1.0) * 2
    q = np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
  elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
    s = math.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) * 2
    q = np.array([(R[2, 1] - R[1, 2]) / s, 0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s])
  elif R[1, 1] > R[2, 2]:
    s = math.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) * 2
    q = np.array([(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s])
  else:
    s = math.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) * 2
    q = np.array([(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s])
  q /= np.linalg.norm(q)
  if q[0] < 0:
    q = -q
  return q


def rot_vec(q, v):
  return quat_to_mat(q) @ v


def axis_angle_quat(axis, angle):
  axis = np.asarray(axis, dtype=np.float64)
  n = np.linalg.norm(axis)
  if n < 1e-14:
    return np.array([1.0, 0, 0, 0])
  axis = axis / n
  return np.concatenate([[math.cos(angle / 2)], math.sin(angle / 2) * axis])


def z2quat(vec):
  """Quaternion rotating the z axis onto `vec` (MuJoCo mjuu_z2quat semantics)."""
  vec = np.asarray(vec, dtype=np.float64)
  n = np.linalg.norm(vec)
  if n < 1e-14:
    return np.array([1.0, 0, 0, 0])
  vec = vec / n
  axis = np.cross([0.0, 0.0, 1.0], vec)
  a = np.linalg.norm(axis)
  if a < 1e-10:
    if vec[2] < 0:
      return np.array([0.0, 1.0, 0.0, 0.0])
    return np.array([1.0, 0, 0, 0])
  ang = math.atan2(a, vec[2])
  return axis_angle_quat(axis / a, ang)


def _frame_quat(attr, compiler):
  """Resolve quat / axisangle / euler / xyaxes / zaxis orientation attributes."""
  deg = compiler["angle"] == "degree"
  if "quat" in attr:
    q = _vec(attr["quat"])
    return q / np.linalg.norm(q)
  if "axisangle" in attr:
    v = _vec(attr["axisangle"])
    ang = math.radians(v[3]) if deg else v[3]
    return axis_angle_quat(v[:3], ang)
  if "euler" in attr:
    e = _vec(attr["euler"])
    if deg:
      e = np.radians(e)
    seq = compiler["eulerseq"]
    q = np.array([1.0, 0, 0, 0])
    for i, ch in enumerate(seq):
      ax = {"x": [1, 0, 0], "y": [0, 1, 0], "z": [0, 0, 1]}[ch.lower()]
      qi = axis_angle_quat(ax, e[i])
      q = quat_mul(q, qi) if ch.islower() else quat_mul(qi, q)
    return q / np.linalg.norm(q)
  if "xyaxes" in attr:
    v = _vec(attr["xyaxes"])
    x = v[:3] / np.linalg.norm(v[:3])
    y = v[3:] - x * np.dot(x, v[3:])
    y = y / np.linalg.norm(y)
    z = np.cross(x, y)
    return mat_to_quat(np.stack([x, y, z], axis=1))
  if "zaxis" in attr:
    return z2quat(_vec(attr["zaxis"]))
  return np.array([1.0, 0, 0, 0])


# ----------------------------------------------------------------------------------------------
# geom helpers
# ----------------------------------------------------------------------------------------------

_GEOM_TYPES = {
  "plane": C.GEOM_PLANE,
  "hfield": C.GEOM_HFIELD,
  "sphere": C.GEOM_SPHERE,
  "capsule": C.GEOM_CAPSULE,
  "ellipsoid": C.GEOM_ELLIPSOID,
  "cylinder": C.GEOM_CYLINDER,
  "box": C.GEOM_BOX,
  "mesh": C.GEOM_MESH,
}


def _geom_volume_inertia(gtype, size):
  """Volume and unit-density principal inertia of a primitive in its own frame."""
  r = size[0]
  if gtype == C.GEOM_SPHERE:
    vol = 4.0 / 3.0 * math.pi * r**3
    i = 0.4 * vol * r * r
    return vol, np.array([i, i, i])
  if gtype == C.GEOM_CAPSULE:
    h = 2.0 * size[1]
    vc = math.pi * r * r * h
    vs = 4.0 / 3.0 * math.pi * r**3
    ixy = vc * (3 * r * r + h * h) / 12.0 + vs * (0.4 * r * r + 0.375 * r * h + 0.25 * h * h)
    iz = vc * r * r / 2.0 + vs * 0.4 * r * r
    return vc + vs, np.array([ixy, ixy, iz])
  if gtype == C.GEOM_CYLINDER:
    h = 2.0 * size[1]
    vol = math.pi * r * r * h
    ixy = vol * (3 * r * r + h * h) / 12.0
    return vol, np.array([ixy, ixy, vol * r * r / 2.0])
  if gtype == C.GEOM_BOX:
    a, b, c = size
    vol = 8.0 * a * b * c
    return vol, vol / 3.0 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
  if gtype == C.GEOM_ELLIPSOID:
    a, b, c = size
    vol = 4.0 / 3.0 * math.pi * a * b * c
    return vol, vol / 5.0 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
  return 0.0, np.zeros(3)


def fluid_semiaxes(gtype, size):
  """Semi-axes of the ellipsoid the fluid model puts in place of a geom (reference passive.py:46 geom_semiaxes)."""
  if gtype == C.GEOM_SPHERE:
    return np.array([size[0], size[0], size[0]], dtype=np.float64)
  if gtype == C.GEOM_CAPSULE:
    return np.array([size[0], size[0], size[1] + size[0]], dtype=np.float64)
  if gtype == C.GEOM_CYLINDER:
    return np.array([size[0], size[0], size[1]], dtype=np.float64)
  return np.asarray(size, dtype=np.float64)[:3].copy()


def _carlson_rd(x, y, z):
  """Carlson's symmetric elliptic integral R_D(x, y, z) = 3/2 int_0^inf dt / ((t + z) sqrt((t + x)(t + y)(t + z))), by duplication."""
  s, fac = 0.0, 1.0
  for _ in range(100):
    mu = (x + y + 3.0 * z) / 5.0
    ex, ey, ez = (mu - x) / mu, (mu - y) / mu, (mu - z) / mu
    if max(abs(ex), abs(ey), abs(ez)) < 1e-4:
      break
    sx, sy, sz = math.sqrt(x), math.sqrt(y), math.sqrt(z)
    lam = sx * (sy + sz) + sy * sz
    s += fac / (sz * (z + lam))
    fac *= 0.25
    x, y, z = 0.25 * (x + lam), 0.25 * (y + lam), 0.25 * (z + lam)
  ea, eb = ex * ey, ez * ez
  ec, ed = ea - eb, ea - 6.0 * eb
  ee = ed + ec + ec
  series = 1.0 + ed * (-3.0 / 14.0 + 9.0 / 88.0 * ed - 4.5 / 26.0 * ez * ee) + ez * (ee / 6.0 + ez * (-9.0 / 22.0 * ec + ez * 3.0 / 26.0 * ea))
  return 3.0 * s + fac * series / (mu * math.sqrt(mu))


def fluid_kappa(s):
  """Lamb's added-mass integrals kappa_i = a b c int_0^inf dl / ((a_i^2 + l) sqrt((a^2 + l)(b^2 + l)(c^2 + l))) of an ellipsoid with
  semi-axes s = (a, b, c).  They sum to 2; a sphere has 2/3 on every axis."""
  a2 = [float(v) * float(v) for v in s]
  abc = float(s[0]) * float(s[1]) * float(s[2])
  return np.array([abc * 2.0 / 3.0 * _carlson_rd(a2[(i + 1) % 3], a2[(i + 2) % 3], a2[i]) for i in range(3)])


def geom_fluid_row(gtype, size, fluidshape, fluidcoef):
  """One row of Model.geom_fluid (12 numbers, MuJoCo's layout): [0] the ellipsoid-model flag, [1:6] blunt drag, slender drag, angular
  drag, Kutta lift and Magnus lift coefficients, [6:9] virtual mass and [9:12] virtual inertia of the geom's fluid ellipsoid per unit
  fluid density.  A geom with fluidshape="none" gets a row of zeros."""
  row = np.zeros(12)
  if fluidshape != "ellipsoid":
    return row
  s = fluid_semiaxes(gtype, size)
  k = fluid_kappa(s)
  vol = 4.0 / 3.0 * math.pi * s[0] * s[1] * s[2]
  row[0] = 1.0
  row[1:6] = fluidcoef
  row[6:9] = vol * k / np.maximum(C.MJ_MINVAL, 2.0 - k)
  sq = s * s
  for i in range(3):  # Lamb's added moment of inertia about axis i, from the two other axes j, k
    j, l = (i + 1) % 3, (i + 2) % 3
    num = (sq[j] - sq[l]) ** 2 * abs(k[l] - k[j])
    den = max(C.MJ_MINVAL, abs(2.0 * (sq[j] - sq[l]) + (sq[j] + sq[l]) * (k[j] - k[l])))
    row[9 + i] = vol * num / den / 5.0
  return row


def _geom_rbound(gtype, size):
  if gtype == C.GEOM_SPHERE:
    return size[0]
  if gtype == C.GEOM_CAPSULE:
    return size[0] + size[1]
  if gtype == C.GEOM_CYLINDER:
    return math.sqrt(size[0] ** 2 + size[1] ** 2)
  if gtype == C.GEOM_ELLIPSOID:
    return max(size)
  if gtype == C.GEOM_BOX:
    return float(np.linalg.norm(size))
  return 0.0  # plane / hfield: 0 marks "unbounded" (reference collision_driver.py:318-320)


def _geom_aabb(gtype, size):
  """(center[3], halfsize[3]) in the geom frame."""
  if gtype == C.GEOM_SPHERE:
    hs = [size[0]] * 3
  elif gtype == C.GEOM_CAPSULE:
    hs = [size[0], size[0], size[0] + size[1]]
  elif gtype == C.GEOM_CYLINDER:
    hs = [size[0], size[0], size[1]]
  elif gtype in (C.GEOM_ELLIPSOID, C.GEOM_BOX):
    hs = list(size)
  else:
    hs = [C.MJ_MAXVAL, C.MJ_MAXVAL, C.MJ_MAXVAL]
  return np.array([0.0, 0.0, 0.0] + hs)


# ----------------------------------------------------------------------------------------------
# defaults
# ----------------------------------------------------------------------------------------------

_ACT_TAGS = ("general", "motor", "position", "velocity", "intvelocity", "damper", "cylinder", "muscle", "adhesion")
# the <muscle> shortcut's scalar parameters after range, in gainprm / biasprm order, with MuJoCo's defaults
_MUSCLE_DEFAULTS = (("force", -1.0), ("scale", 200.0), ("lmin", 0.5), ("lmax", 1.6), ("vmax", 1.5), ("fpmax", 1.3), ("fvmax", 1.2))
# <contact> sensor: data keywords in their canonical order (bit i of sensor_intprm[0]) with the floats each adds to a slot, and the
# reductions (sensor_intprm[1]); reference sensor.py:1816-1851, :2448-2494
CONTACT_DATA = (("found", 1), ("force", 3), ("torque", 3), ("dist", 1), ("pos", 3), ("normal", 3), ("tangent", 3))
CONTACT_REDUCE = ("none", "mindist", "maxforce", "netforce")
CONTACT_SENSOR_MAXMATCH = 64  # matches kept per contact sensor and world unless <numeric name="contact_sensor_maxmatch"> says otherwise


def contact_slot_size(dataspec: int) -> int:
  return sum(n for i, (_, n) in enumerate(CONTACT_DATA) if dataspec >> i & 1)


# the object attributes of the camprojection / insidesite / tendon sensors: (attribute, object type, name list) of the
# sensor's object, then of its reference object (None: no reference)
_EXTRA_SENSOR_ATTRS = {
  "camprojection": (("site", C.OBJ_SITE, "site"), ("camera", C.OBJ_CAMERA, "camera")),
  "insidesite": (("objname", None, None), ("site", C.OBJ_SITE, "site")),
  **{t: (("tendon", C.OBJ_TENDON, "tendon"), None) for t in ("tendonlimitpos", "tendonlimitvel", "tendonlimitfrc", "tendonactfrc")},
}


def _extra_sensor_objects(e, names, objtypes, what):
  """((objtype, objid), (reftype, refid)) of a camprojection / insidesite / tendon sensor element; ValueError naming the
  sensor for a missing attribute, an unknown name or an insidesite objtype other than body, xbody, geom, site or camera."""
  out = []
  for spec in _EXTRA_SENSOR_ATTRS[e.tag]:
    if spec is None:
      out.append((C.OBJ_UNKNOWN, -1))
      continue
    attr, typ, lst = spec
    if typ is None:  # insidesite's object: objtype= and objname=
      if e.get("objtype") is None:
        raise ValueError(f"{what}: missing attribute objtype")
      if e.get("objtype") not in objtypes:
        raise ValueError(f"{what}: objtype '{e.get('objtype')}' is not one of {', '.join(objtypes)}")
      typ, lst = objtypes[e.get("objtype")]
    if e.get(attr) is None:
      raise ValueError(f"{what}: missing attribute {attr}")
    lst_names = getattr(names, lst)
    if e.get(attr) not in lst_names:
      raise ValueError(f"{what}: unknown {lst} '{e.get(attr)}' in {attr}")
    out.append((typ, lst_names.index(e.get(attr))))
  return out


def contact_intprm(data, reduce, num, what):
  """(dataspec, reduce, num) of a <contact> sensor's data / reduce / num attributes; ValueError naming `what` for an unknown or
  out-of-order data keyword, an unknown reduce value or num < 1."""
  keys = [k for k, _ in CONTACT_DATA]
  words = str(data).split()
  if not words:
    raise ValueError(f"{what}: data must list at least one of {' '.join(keys)}")
  for w in words:
    if w not in keys:
      raise ValueError(f"{what}: unknown data keyword '{w}' (expected some of {' '.join(keys)}, in that order)")
  idx = [keys.index(w) for w in words]
  if any(b <= a for a, b in zip(idx, idx[1:])):
    raise ValueError(f"{what}: data keywords '{data}' must appear once each, in the order {' '.join(keys)}")
  if reduce not in CONTACT_REDUCE:
    raise ValueError(f"{what}: unknown reduce '{reduce}' (expected one of {', '.join(CONTACT_REDUCE)})")
  try:
    n = int(num)
  except ValueError:
    raise ValueError(f"{what}: num must be an integer >= 1, got '{num}'") from None
  if n < 1:
    raise ValueError(f"{what}: num must be >= 1, got {n}")
  return (sum(1 << i for i in idx), CONTACT_REDUCE.index(reduce), n)


def contact_sensor_maxmatch(mjm) -> int:
  """Option.contact_sensor_maxmatch of a compiled model: its <numeric name="contact_sensor_maxmatch"> (reference io.py:409-413), else 64"""
  names = list(getattr(getattr(mjm, "names", None), "numeric", None) or [])
  if "contact_sensor_maxmatch" not in names:
    return CONTACT_SENSOR_MAXMATCH
  i = names.index("contact_sensor_maxmatch")
  if int(mjm.numeric_size[i]) < 1:
    raise ValueError('numeric contact_sensor_maxmatch: needs one value (data="N")')
  v = float(mjm.numeric_data[int(mjm.numeric_adr[i])])
  if v != int(v) or v < 1:
    raise ValueError(f"numeric contact_sensor_maxmatch: must be an integer >= 1, got {v:g}")
  return int(v)


# delay / history attributes of actuators and sensors; interp keywords as in the reference's history.py:88 (0 zoh, 1 linear, 2 cubic)
_HISTORY_KEYS = ("nsample", "interp", "delay", "interval")
_INTERP = {"zoh": 0, "linear": 1, "cubic": 2}


def _history_attrs(a, what, interval):
  """((nsample, interp), delay, (period, phase)) of an actuator or sensor element.  Range checks (negative values, a delay or interval
  without samples) are io._validate's, so that they also hold for models that do not come from this compiler."""
  interp = a.get("interp", "zoh")
  if interp not in _INTERP:
    raise ValueError(f"{what}: interp must be one of {sorted(_INTERP)}, got '{interp}'")
  iv = np.zeros(2)
  if interval and "interval" in a:
    v = _vec(a["interval"])
    if v.size not in (1, 2):
      raise ValueError(f"{what}: interval takes 'period [phase]', got '{a['interval']}'")
    iv[: v.size] = v
  return (int(a.get("nsample", 0)), _INTERP[interp]), float(a.get("delay", 0.0)), iv


def set_history_layout(m):
  """actuator_historyadr / sensor_historyadr / nhistory of the delay buffers (reference history.py): one buffer per actuator or sensor
  with nsample > 0, [user, cursor, times[n], values[n * dim]] (dim 1 for actuators), actuators in index order, then sensors; -1 for
  the others."""
  adr = 0
  out = {}
  for kind, hist, dims in (("actuator", m.actuator_history, np.ones(len(m.actuator_history), dtype=int)), ("sensor", m.sensor_history, m.sensor_dim)):
    a = -np.ones(len(hist), dtype=np.int32)
    for i, (n, dim) in enumerate(zip(np.asarray(hist).reshape(-1, 2)[:, 0], np.asarray(dims).reshape(-1))):
      if n > 0:
        a[i] = adr
        adr += 2 + int(n) * (1 + int(dim))
    out[kind] = a
  m.actuator_historyadr, m.sensor_historyadr, m.nhistory = out["actuator"], out["sensor"], adr


# The renderer's fields of <camera>, <light> and <visual><headlight>, with the defaults of MuJoCo's XML reference (not checked
# against MuJoCo's own compiler, which is not available here).
_CAMERA_FIELDS = (("projection", (), np.int32), ("fovy", (), np.float64), ("resolution", (2,), np.int32), ("sensorsize", (2,), np.float64), ("intrinsic", (4,), np.float64))
_LIGHT_FIELDS = (("type", (), np.int32), ("castshadow", (), np.int32), ("active", (), np.int32), ("attenuation", (3,), np.float64), ("cutoff", (), np.float64),
                 ("exponent", (), np.float64), ("ambient", (3,), np.float64), ("diffuse", (3,), np.float64), ("specular", (3,), np.float64))
_TEX_ROLES = ("user", "rgb", "occlusion", "roughness", "metallic", "normal", "opacity", "emissive", "rgba", "orm")  # mjtTextureRole
_LIGHT_TYPES = {"spot": 0, "directional": 1, "point": 2, "image": 3}
_HEADLIGHT_DEFAULTS = (("active", 1), ("ambient", np.full(3, 0.1)), ("diffuse", np.full(3, 0.4)), ("specular", np.full(3, 0.5)))


def _camera_optics(a):
  """projection, fovy, resolution, sensorsize and intrinsic [fx, fy, cx, cy] (length units) of a resolved <camera>"""
  ortho = a.get("projection", "orthographic" if a.get("orthographic") == "true" else "perspective")
  if ortho not in ("perspective", "orthographic"):
    raise ValueError(f"camera projection must be 'perspective' or 'orthographic', got {ortho!r}")
  res = _vec(a.get("resolution"), 2, default=[1, 1])
  sensor = _vec(a.get("sensorsize"), 2, default=[0, 0])
  intr = np.concatenate([_vec(a.get("focal"), 2, default=[0, 0]), _vec(a.get("principal"), 2, default=[0, 0])])
  fp, pp = _vec(a.get("focalpixel"), 2, default=[0, 0]), _vec(a.get("principalpixel"), 2, default=[0, 0])
  if fp.any():
    intr[:2] = fp / res * sensor
  if pp.any():
    intr[2:] = pp / res * sensor
  return dict(projection=int(ortho == "orthographic"), fovy=float(a.get("fovy", 45.0)), resolution=res.astype(np.int32), sensorsize=sensor, intrinsic=intr)


def _light_optics(a):
  """type, castshadow, active, attenuation, cutoff, exponent and the ambient / diffuse / specular colours of a resolved <light>"""
  kind = a.get("type", "directional" if a.get("directional") == "true" else "spot")
  if kind not in _LIGHT_TYPES:
    raise ValueError(f"light type must be one of {sorted(_LIGHT_TYPES)}, got {kind!r}")
  return dict(type=_LIGHT_TYPES[kind], castshadow=int(a.get("castshadow", "true") == "true"), active=int(a.get("active", "true") == "true"),
              attenuation=_vec(a.get("attenuation"), 3, default=[1, 0, 0]), cutoff=float(a.get("cutoff", 45.0)), exponent=float(a.get("exponent", 10.0)),
              ambient=_vec(a.get("ambient"), 3, default=[0, 0, 0]), diffuse=_vec(a.get("diffuse"), 3, default=[0.7, 0.7, 0.7]),
              specular=_vec(a.get("specular"), 3, default=[0.3, 0.3, 0.3]))


class _Defaults:
  def __init__(self):
    self.classes = {"main": {}}
    self.parent = {"main": None}

  def parse(self, elem, parent="main"):
    name = elem.get("class", "main") if parent is not None else "main"
    if name not in self.classes:
      self.classes[name] = {}
      self.parent[name] = parent
    for child in elem:
      if child.tag == "default":
        self.parse(child, name)
      else:
        tag = "actuator" if child.tag in _ACT_TAGS else child.tag
        self.classes[name].setdefault(tag, {}).update(child.attrib)

  def resolve(self, tag, cls):
    tag = "actuator" if tag in _ACT_TAGS else tag
    chain = []
    c = cls if cls in self.classes else "main"
    while c is not None:
      chain.append(c)
      c = self.parent[c]
    out = {}
    for c in reversed(chain):
      out.update(self.classes[c].get(tag, {}))
    return out


# ----------------------------------------------------------------------------------------------
# compiler
# ----------------------------------------------------------------------------------------------


def _expand_includes(root, basedir):
  for parent in list(root.iter()):
    for i, child in enumerate(list(parent)):
      if child.tag == "include":
        sub = ET.parse(os.path.join(basedir, child.get("file"))).getroot()
        _expand_includes(sub, basedir)
        parent.remove(child)
        for j, sc in enumerate(list(sub)):
          parent.insert(i + j, sc)
  return root


# ----------------------------------------------------------------------------------------------
# composite elements: <frame>, <replicate>, <attach model=...> are expanded into plain bodies before compilation
# ----------------------------------------------------------------------------------------------

_ORIENT_ATTRS = ("quat", "axisangle", "euler", "xyaxes", "zaxis")
_NAME_REFS = ("joint", "body1", "body2", "geom1", "geom2", "target", "site", "body", "objname", "refname", "joint1", "joint2")


def _fmt(v):
  return " ".join(repr(float(x)) for x in np.asarray(v).reshape(-1))


def _bake_frame(elem, fpos, fquat, compiler):
  """Express a body / geom / site / camera / light given in a frame (fpos, fquat) in the frame's parent."""
  a = elem.attrib
  if elem.tag == "light":
    a["pos"] = _fmt(fpos + rot_vec(fquat, _vec(a.get("pos"), default=[0, 0, 0])))
    a["dir"] = _fmt(rot_vec(fquat, _vec(a.get("dir"), default=[0, 0, -1])))
    return
  if "fromto" in a:
    ft = _vec(a["fromto"])
    a["fromto"] = _fmt(np.concatenate([fpos + rot_vec(fquat, ft[:3]), fpos + rot_vec(fquat, ft[3:])]))
    return
  q = quat_mul(fquat, _frame_quat(a, compiler))
  for k in _ORIENT_ATTRS:
    a.pop(k, None)
  a["pos"] = _fmt(fpos + rot_vec(fquat, _vec(a.get("pos"), default=[0, 0, 0])))
  a["quat"] = _fmt(q / np.linalg.norm(q))


def _rename(elem, prefix, suffix):
  """prefix + name + suffix on every name and name reference of a subtree."""
  if not prefix and not suffix:
    return
  for e in elem.iter():
    for k in ("name",) + _NAME_REFS:
      if k in e.attrib:
        e.set(k, prefix + e.get(k) + suffix)


def _expand_composites(root, basedir):
  """<frame> children are re-expressed in the parent frame; <replicate> repeats its children `count` times with cumulative
  offset / euler increments and a name suffix `sep + index`; <attach model= body= prefix=> grafts a body subtree of another
  MJCF file (declared in <asset><model/>) together with the actuators, contact pairs / excludes and keyframes that refer to it.
  The attached file's <default> tree is adopted when the host file has none (anything else raises); its <option> is not
  imported (as in MuJoCo).  Keyframes: each attachment contributes its file's keyframes, the rest of qpos keeps qpos0."""
  if not any(e.tag in ("frame", "replicate", "attach") for e in root.iter()):
    return root
  compiler = {"angle": "degree", "eulerseq": "xyz"}
  for ce in root.findall("compiler"):
    compiler["angle"] = ce.get("angle", compiler["angle"]); compiler["eulerseq"] = ce.get("eulerseq", compiler["eulerseq"])
  models = {}
  for asset in root.findall("asset"):
    for me in list(asset.findall("model")):
      models[me.get("name")] = os.path.join(basedir or "", me.get("file"))
      asset.remove(me)
  ident = (np.zeros(3), np.array([1.0, 0, 0, 0]))
  extra = {"actuator": [], "contact": [], "keyframe": []}

  def section(tag):
    sec = root.find(tag)
    if sec is None:
      sec = ET.SubElement(root, tag)
    return sec

  def attach(elem, fpos, fquat, suffix):
    import copy

    if elem.get("model") not in models:
      raise NotImplementedError("<attach> needs model= naming an <asset><model file=.../> entry")
    path = models[elem.get("model")]
    child = ET.parse(path).getroot()
    _expand_includes(child, os.path.dirname(os.path.abspath(path)))
    for tag in ("tendon", "equality", "sensor"):
      if child.find(tag) is not None and len(child.find(tag)):
        raise NotImplementedError(f"<attach>: <{tag}> of the attached model is not supported")
    for ce in child.findall("compiler"):
      if ce.get("angle", "degree") != compiler["angle"] or ce.get("eulerseq", "xyz") != compiler["eulerseq"]:
        raise NotImplementedError("<attach>: the attached model uses different compiler angle / eulerseq settings")
    body = next((b for b in child.iter("body") if b.get("name") == elem.get("body")), None)
    if body is None:
      raise ValueError(f"<attach>: body {elem.get('body')} not found in {path}")
    if child.find("default") is not None:
      if root.find("default") is not None and root.find("default") is not child.find("default") and not root.find("default").get("_adopted"):
        raise NotImplementedError("<attach>: both files define <default>s")
      if root.find("default") is None:
        d = copy.deepcopy(child.find("default")); d.set("_adopted", "1"); root.append(d)
    prefix = elem.get("prefix", "")
    graft = copy.deepcopy(body)
    _bake_frame(graft, fpos, fquat, compiler)
    _rename(graft, prefix, suffix)
    for tag in ("actuator", "contact"):
      sec = child.find(tag)
      for e in (list(sec) if sec is not None else []):
        e2 = copy.deepcopy(e); _rename(e2, prefix, suffix); extra[tag].append(e2)
    # keyframes of the attached file, restricted to the grafted subtree's joints (free-joint root poses move with the frame)
    def qsize(j):
      return {"free": 7, "ball": 4}.get(j.get("type", "hinge") if j.tag == "joint" else "free", 1)

    off, found = 0, False
    for b in child.iter("body"):  # document order = qpos order
      if b is body:
        found = True
        break
      if any(anc is b for anc in []) :
        pass
      off += sum(qsize(j) for j in b if j.tag in ("joint", "freejoint"))
    sub_joints = [j for b in body.iter("body") for j in b if j.tag in ("joint", "freejoint")]
    size = sum(qsize(j) for j in sub_joints)
    free_root = bool(sub_joints) and sub_joints[0] in list(body) and qsize(sub_joints[0]) == 7
    ke = child.find("keyframe")
    for k in (ke.findall("key") if ke is not None and found else []):
      if "qpos" not in k.attrib:
        continue
      q = _vec(k.get("qpos"))[off : off + size].copy()
      if free_root:
        q[:3] = fpos + rot_vec(fquat, q[:3]); q[3:7] = quat_mul(fquat, q[3:7] / np.linalg.norm(q[3:7]))
      pk = ET.Element("key", {"name": prefix + k.get("name", "key") + suffix, "_part_body": graft.get("name"), "_part_qpos": _fmt(q)})
      extra["keyframe"].append(pk)
    return graft

  def expand(parent, fpos, fquat, suffix):
    """children of `parent`, with frames / replicates / attaches resolved; (fpos, fquat) is the pending frame of `parent`'s children."""
    import copy

    out = []
    for ch in list(parent):
      if ch.tag == "frame":
        p = fpos + rot_vec(fquat, _vec(ch.get("pos"), default=[0, 0, 0])); q = quat_mul(fquat, _frame_quat(ch.attrib, compiler))
        out += expand(ch, p, q, suffix)
      elif ch.tag == "replicate":
        n = int(ch.get("count")); sep = ch.get("sep", ""); width = len(str(n - 1))
        off = _vec(ch.get("offset"), default=[0, 0, 0]); rq = _frame_quat({k: v for k, v in ch.attrib.items() if k == "euler"}, compiler)
        p, q = fpos.copy(), fquat.copy()
        for i in range(n):
          out += expand(copy.deepcopy(ch), p, q, suffix + sep + str(i).zfill(width))
          p = p + rot_vec(q, off); q = quat_mul(q, rq)
      elif ch.tag == "attach":
        g = attach(ch, fpos, fquat, suffix)
        g[:] = expand(g, *ident, "")
        out.append(g)
      else:
        if ch.tag in ("body", "geom", "site", "camera", "light") and (fpos.any() or not np.allclose(fquat, ident[1])):
          _bake_frame(ch, fpos, fquat, compiler)
        if suffix:
          for k in ("name",) + _NAME_REFS:
            if k in ch.attrib:
              ch.set(k, ch.get(k) + suffix)
        if ch.tag == "body":
          ch[:] = expand(ch, *ident, suffix)
        out.append(ch)
    return out

  for wb in root.findall("worldbody"):
    wb[:] = expand(wb, *ident, "")
  for tag, elems in extra.items():
    if elems:
      sec = section(tag)
      for e in elems:
        sec.append(e)
  d = root.find("default")
  if d is not None:
    d.attrib.pop("_adopted", None)
  return root


def _merge_toplevel(root):
  """Merge repeated top-level sections (from includes) into one element per tag."""
  merged = {}
  for child in list(root):
    if child.tag in merged and child.tag in ("worldbody", "asset", "actuator", "keyframe", "contact", "sensor", "default"):
      tgt = merged[child.tag]
      for sc in list(child):
        tgt.append(sc)
      root.remove(child)
    else:
      merged.setdefault(child.tag, child)
  return root


def load(path: str):
  """Compile an MJCF file into an MjModel-like object."""
  root = ET.parse(path).getroot()
  _expand_includes(root, os.path.dirname(os.path.abspath(path)))
  _expand_composites(root, os.path.dirname(os.path.abspath(path)))
  _load_mesh_files(root, os.path.dirname(os.path.abspath(path)))
  return compile_xml(root)


def _load_mesh_files(root, basedir):
  """Mesh assets given by `file=` (OBJ / STL under <compiler meshdir>): the vertex / face data is read here and attached to the
  element as inline `vertex=` / `face=` data, which is what the compiler consumes.  Files that do not exist are left alone (only
  visual geoms may then refer to the asset)."""
  from . import mesh as _mesh

  meshdir = ""
  for ce in root.iter("compiler"):
    meshdir = ce.get("meshdir", ce.get("assetdir", meshdir))
  for asset in root.iter("asset"):
    for me in asset.findall("mesh"):
      if "vertex" in me.attrib or "file" not in me.attrib:
        continue
      path = os.path.join(basedir, meshdir, me.get("file"))
      if not os.path.exists(path):
        continue
      v, f = _mesh.read_file(path)
      me.set("vertex", " ".join(repr(float(x)) for x in v.reshape(-1)))
      if len(f):
        me.set("face", " ".join(str(int(x)) for x in f.reshape(-1)))
      if "name" not in me.attrib:
        me.set("name", os.path.splitext(os.path.basename(me.get("file")))[0])


def load_string(xml: str):
  return compile_xml(ET.fromstring(xml))


def compile_xml(root):
  # a model included inside <mujoco> contributes its own top-level sections
  flat = ET.Element("mujoco", root.attrib)
  for child in list(root):
    if child.tag == "mujoco":
      for sc in child:
        flat.append(sc)
    else:
      flat.append(child)
  root = _merge_toplevel(flat)

  # top-level sections: the ones compiled below, the ones without influence on the dynamics (visual, statistic, custom, size), and the ones
  # whose content cannot be dropped without changing the simulation
  for child in root:
    if not isinstance(child.tag, str):
      continue
    if child.tag in ("deformable", "extension"):
      if len(child):
        raise NotImplementedError(f"<{child.tag}> (flex / skin / plugin declarations) is not supported by this compiler")
    elif child.tag not in ("compiler", "option", "size", "visual", "statistic", "default", "asset", "worldbody", "contact", "equality", "tendon",
                           "actuator", "sensor", "keyframe", "custom"):
      raise NotImplementedError(f"unknown top-level element <{child.tag}>")
  compiler = {"angle": "degree", "eulerseq": "xyz", "autolimits": True, "inertiafromgeom": "auto", "boundmass": 0.0, "boundinertia": 0.0}
  for ce in root.findall("compiler"):
    if "angle" in ce.attrib:
      compiler["angle"] = ce.get("angle")
    if "eulerseq" in ce.attrib:
      compiler["eulerseq"] = ce.get("eulerseq")
    if "autolimits" in ce.attrib:
      compiler["autolimits"] = ce.get("autolimits") == "true"
    if "inertiafromgeom" in ce.attrib:
      compiler["inertiafromgeom"] = ce.get("inertiafromgeom")
    if "boundmass" in ce.attrib:
      compiler["boundmass"] = float(ce.get("boundmass"))
    if "boundinertia" in ce.attrib:
      compiler["boundinertia"] = float(ce.get("boundinertia"))
  deg = compiler["angle"] == "degree"

  # ---- options
  opt = SimpleNamespace(
    timestep=0.002,
    tolerance=1e-8,
    ls_tolerance=0.01,
    gravity=np.array([0.0, 0.0, -9.81]),
    integrator=C.INT_EULER,
    cone=C.CONE_PYRAMIDAL,
    solver=C.SOL_NEWTON,
    ccd_iterations=35,
    ccd_tolerance=1e-6,
    iterations=100,
    ls_iterations=50,
    disableflags=0,
    enableflags=0,
    impratio=1.0,
    jacobian=C.JAC_AUTO,
    density=0.0,
    viscosity=0.0,
    wind=np.zeros(3),
    magnetic=np.array([0.0, -0.5, 0.0]),
    noslip_iterations=0,
    noslip_tolerance=1e-6,
    o_margin=0.0,
  )
  known_option = {"timestep", "tolerance", "ls_tolerance", "impratio", "ccd_tolerance", "iterations", "ls_iterations", "ccd_iterations", "gravity", "integrator",
                  "cone", "solver", "jacobian", "density", "viscosity", "wind", "magnetic", "noslip_iterations", "noslip_tolerance", "o_margin", "o_solref",
                  "o_solimp", "o_friction", "sdf_iterations", "sdf_initpoints", "actuatorgroupdisable", "apirate", "mpr_iterations", "mpr_tolerance"}
  for oe in root.findall("option"):
    a = oe.attrib
    unknown = sorted(set(a) - known_option)
    if unknown:
      raise ValueError(f"<option>: unknown attribute(s) {unknown}")
    for k in ("density", "viscosity", "noslip_tolerance", "o_margin"):
      if k in a:
        setattr(opt, k, float(a[k]))
    if "noslip_iterations" in a:
      opt.noslip_iterations = int(a["noslip_iterations"])
    for k in ("wind", "magnetic"):
      if k in a:
        setattr(opt, k, _vec(a[k]))
    if "ccd_iterations" in a:
      opt.ccd_iterations = int(a["ccd_iterations"])
    for k in ("timestep", "tolerance", "ls_tolerance", "impratio", "ccd_tolerance"):
      if k in a:
        setattr(opt, k, float(a[k]))
    for k in ("iterations", "ls_iterations"):
      if k in a:
        setattr(opt, k, int(a[k]))
    if "gravity" in a:
      opt.gravity = _vec(a["gravity"])
    if "integrator" in a:
      opt.integrator = {"Euler": C.INT_EULER, "RK4": C.INT_RK4, "implicit": C.INT_IMPLICIT, "implicitfast": C.INT_IMPLICITFAST}[a["integrator"]]
    if "cone" in a:
      opt.cone = {"pyramidal": C.CONE_PYRAMIDAL, "elliptic": C.CONE_ELLIPTIC}[a["cone"]]
    if "solver" in a:
      opt.solver = {"PGS": 0, "CG": C.SOL_CG, "Newton": C.SOL_NEWTON}[a["solver"]]
    if "jacobian" in a:
      opt.jacobian = {"dense": C.JAC_DENSE, "sparse": C.JAC_SPARSE, "auto": C.JAC_AUTO}[a["jacobian"]]
    for fe in oe.findall("flag"):
      for k, v in fe.attrib.items():
        if k in C.DISABLE_FLAGS:
          if v == "disable":
            opt.disableflags |= C.DISABLE_FLAGS[k]
        elif k in C.ENABLE_FLAGS:
          if v == "enable":
            opt.enableflags |= C.ENABLE_FLAGS[k]

  # ---- defaults
  dflt = _Defaults()
  for de in root.findall("default"):
    dflt.parse(de, None)

  bodies, joints, geoms, sites, cams, lights = [], [], [], [], [], []
  skipped_mesh_geoms = 0
  # mesh assets with inline vertex data (files are resolved by load(); assets whose data is unavailable stay unknown and
  # only visual geoms may refer to them)
  meshes, mesh_names = [], []
  for asset in root.findall("asset"):
    for me in asset.findall("mesh"):
      if "vertex" not in me.attrib:
        continue
      from . import mesh as _mesh

      faces = _vec(me.get("face")).astype(int).reshape(-1, 3) if "face" in me.attrib else None
      ma = dflt.resolve("mesh", me.get("class", "main"))
      ma.update(me.attrib)
      if ma.get("inertia", "convex") not in ("convex", "legacy", "exact"):
        raise NotImplementedError(f"mesh inertia='{ma.get('inertia')}' is not supported")
      # inertia="convex": mass properties of the hull; otherwise those of the given faces (closed, outward-oriented surfaces)
      meshes.append(_mesh.process(_vec(me.get("vertex")).reshape(-1, 3), None if ma.get("inertia") == "convex" else faces, _vec(ma.get("scale"), 3, default=[1, 1, 1])))
      mesh_names.append(me.get("name", f"mesh{len(mesh_names)}"))

  # materials: the colour (a fully transparent material hides its geoms from rays) and the renderer's specular / shininess /
  # emission, with MuJoCo's defaults.  A texture reference is only recorded (mat_texid): the renderer refuses textured materials.
  tex_names = [te.get("name", f"texture{i}") for i, te in enumerate(e for asset in root.findall("asset") for e in asset.findall("texture"))]
  mat_names, mat_rgba, mat_light = [], [], []
  for asset in root.findall("asset"):
    for me in asset.findall("material"):
      ma = dflt.resolve("material", me.get("class", "main"))
      ma.update(me.attrib)
      mat_names.append(me.get("name", f"material{len(mat_names)}"))
      mat_rgba.append(_vec(ma.get("rgba"), 4, default=[1, 1, 1, 1]))
      # mat_texid (nmat, mjNTEXROLE): texture= fills the RGB role, each <layer texture= role=> its role
      texid = [-1] * len(_TEX_ROLES)
      for role, tex in [("rgb", ma.get("texture"))] + [(la.get("role", "rgb"), la.get("texture")) for la in me.findall("layer")]:
        if tex is not None:
          if role not in _TEX_ROLES:
            raise ValueError(f"material layer role must be one of {list(_TEX_ROLES)}, got {role!r}")
          texid[_TEX_ROLES.index(role)] = tex_names.index(tex) if tex in tex_names else len(tex_names)
      mat_light.append((float(ma.get("specular", 0.5)), float(ma.get("shininess", 0.5)), float(ma.get("emission", 0.0)), *texid))

  def attrs(elem, childclass):
    cls = elem.get("class", childclass)
    out = dflt.resolve(elem.tag, cls if cls is not None else "main")
    out.update(elem.attrib)
    return out

  def add_body(elem, parentid, childclass):
    nonlocal skipped_mesh_geoms
    bid = len(bodies)
    if parentid < 0:
      b = dict(name="world", parentid=0, pos=np.zeros(3), quat=np.array([1.0, 0, 0, 0]), inertial=None, gravcomp=0.0, mocap=False)
    else:
      b = dict(
        name=elem.get("name", f"body{bid}"),
        parentid=parentid,
        pos=_vec(elem.get("pos"), default=[0, 0, 0]),
        quat=_frame_quat(elem.attrib, compiler),
        inertial=None,
        gravcomp=float(elem.get("gravcomp", 0.0)),
        mocap=elem.get("mocap", "false") == "true",
      )
      childclass = elem.get("childclass", childclass)
    b["jntadr"], b["jntnum"], b["geomadr"], b["geomnum"] = -1, 0, -1, 0
    bodies.append(b)
    for child in elem:
      tag = child.tag
      if tag == "inertial":
        a = child.attrib
        pos = _vec(a.get("pos"), default=[0, 0, 0])
        quat = _frame_quat(a, compiler)
        mass = float(a["mass"])
        if "diaginertia" in a:
          inertia = _vec(a["diaginertia"])
        else:
          f = _vec(a["fullinertia"])
          full = np.array([[f[0], f[3], f[4]], [f[3], f[1], f[5]], [f[4], f[5], f[2]]])
          full = quat_to_mat(quat) @ full @ quat_to_mat(quat).T
          inertia, quat = _principal(full)
        b["inertial"] = (pos, quat, mass, inertia)
      elif tag in ("joint", "freejoint"):
        a = attrs(child, childclass) if tag == "joint" else dict(child.attrib, type="free")
        jtype = {"free": C.JNT_FREE, "ball": C.JNT_BALL, "slide": C.JNT_SLIDE, "hinge": C.JNT_HINGE}[a.get("type", "hinge")]
        rng = _vec(a.get("range"), default=[0, 0])
        if jtype in (C.JNT_HINGE, C.JNT_BALL) and deg:
          rng = np.radians(rng)
        lim = a.get("limited", "auto")
        limited = (lim == "true") or (lim == "auto" and compiler["autolimits"] and "range" in a)
        afr = _vec(a.get("actuatorfrcrange"), default=[0, 0])
        afl = a.get("actuatorfrclimited", "auto")
        actfrclimited = (afl == "true") or (afl == "auto" and compiler["autolimits"] and "actuatorfrcrange" in a)
        ref = float(a.get("ref", 0.0))
        sref = float(a.get("springref", 0.0))
        if jtype == C.JNT_HINGE and deg:
          ref, sref = math.radians(ref), math.radians(sref)
        axis = _vec(a.get("axis"), default=[0, 0, 1])
        if jtype in (C.JNT_FREE, C.JNT_BALL):
          axis = np.array([0.0, 0.0, 1.0])
        else:
          axis = axis / np.linalg.norm(axis)
        j = dict(
          name=a.get("name", f"joint{len(joints)}"),
          type=jtype,
          bodyid=bid,
          pos=_vec(a.get("pos"), default=[0, 0, 0]),
          axis=axis,
          range=rng,
          limited=bool(limited),
          stiffness=float(a.get("stiffness", 0.0)),
          damping=float(a.get("damping", 0.0)),
          armature=float(a.get("armature", 0.0)),
          frictionloss=float(a.get("frictionloss", 0.0)),
          margin=float(a.get("margin", 0.0)),
          ref=ref,
          springref=sref,
          solreflimit=_vec(a.get("solreflimit"), default=C.DEFAULT_SOLREF),
          solimplimit=_vec(a.get("solimplimit"), 5, default=C.DEFAULT_SOLIMP),
          solreffriction=_vec(a.get("solreffriction"), default=C.DEFAULT_SOLREF),
          solimpfriction=_vec(a.get("solimpfriction"), 5, default=C.DEFAULT_SOLIMP),
          actfrclimited=bool(actfrclimited),
          actfrcrange=afr,
          actgravcomp=a.get("actuatorgravcomp", "false") == "true",
        )
        if jtype == C.JNT_FREE:
          j.update(limited=False, stiffness=float(a.get("stiffness", 0.0)), damping=float(a.get("damping", 0.0)), armature=float(a.get("armature", 0.0)))
        if b["jntnum"] == 0:
          b["jntadr"] = len(joints)
        b["jntnum"] += 1
        joints.append(j)
      elif tag == "geom":
        a = attrs(child, childclass)
        gtype = _GEOM_TYPES[a.get("type", "sphere")]
        if "mesh" in a and "type" not in a:
          gtype = C.GEOM_MESH
        dataid = -1
        if gtype == C.GEOM_MESH and a.get("mesh") in mesh_names:
          dataid = mesh_names.index(a.get("mesh"))
        elif gtype == C.GEOM_MESH:
          # the asset's data is not available (e.g. visual STL files outside the tree): only visual (non-colliding, massless) geoms can be skipped
          if int(a.get("contype", 1)) == 0 and int(a.get("conaffinity", 1)) == 0 and (float(a.get("density", 1000)) == 0 or "mass" in a and float(a["mass"]) == 0):
            skipped_mesh_geoms += 1
            continue
          raise NotImplementedError("colliding / massive mesh geoms need the mesh asset's vertex data (inline `vertex=` or a readable file)")
        size = _vec(a.get("size"), 3, default=[0, 0, 0])
        pos = _vec(a.get("pos"), default=[0, 0, 0])
        quat = _frame_quat(a, compiler)
        if dataid >= 0:  # the geom frame is the mesh frame (centre of mass, principal axes): compose with the asset's transform
          md = meshes[dataid]
          pos = pos + rot_vec(quat, md["pos"])
          quat = quat_mul(quat, md["quat"])
          size = md["aabb_size"].copy()
        if "fromto" in a:
          ft = _vec(a["fromto"])
          vec = ft[0:3] - ft[3:6]
          pos = 0.5 * (ft[0:3] + ft[3:6])
          quat = z2quat(vec)
          half = 0.5 * np.linalg.norm(vec)
          if gtype in (C.GEOM_CAPSULE, C.GEOM_CYLINDER):
            size = np.array([size[0], half, 0.0])
          elif gtype in (C.GEOM_BOX, C.GEOM_ELLIPSOID):
            size = np.array([size[0], size[0], half])
        fr = _vec(a.get("friction"), 3, default=C.DEFAULT_FRICTION)
        g = dict(
          name=a.get("name", f"geom{len(geoms)}"),
          type=gtype,
          bodyid=bid,
          size=size,
          pos=pos,
          quat=quat,
          contype=int(a.get("contype", 1)),
          conaffinity=int(a.get("conaffinity", 1)),
          condim=int(a.get("condim", 3)),
          priority=int(a.get("priority", 0)),
          friction=fr,
          solmix=float(a.get("solmix", 1.0)),
          solref=_vec(a.get("solref"), default=C.DEFAULT_SOLREF),
          solimp=_vec(a.get("solimp"), 5, default=C.DEFAULT_SOLIMP),
          margin=float(a.get("margin", 0.0)),
          gap=float(a.get("gap", 0.0)),
          density=float(a.get("density", 1000.0)),
          mass=float(a["mass"]) if "mass" in a else None,
          group=int(a.get("group", 0)),
          rgba=_vec(a.get("rgba"), 4, default=[0.5, 0.5, 0.5, 1.0]),
          matid=mat_names.index(a["material"]) if a.get("material") in mat_names else -1,
          dataid=dataid,
          fluid=geom_fluid_row(gtype, size, a.get("fluidshape", "none"), _vec(a.get("fluidcoef"), 5, default=C.DEFAULT_FLUIDCOEF)),
        )
        if a.get("fluidshape", "none") not in ("none", "ellipsoid"):
          raise ValueError(f"geom fluidshape must be 'none' or 'ellipsoid', got {a['fluidshape']!r}")
        if b["geomnum"] == 0:
          b["geomadr"] = len(geoms)
        b["geomnum"] += 1
        geoms.append(g)
      elif tag == "site":
        a = attrs(child, childclass)
        if "fromto" in a:
          raise NotImplementedError("site fromto is not supported by this compiler")
        ssize = np.full(3, 0.005)
        sv = _vec(a.get("size"), default=[])
        ssize[: len(sv)] = sv
        sites.append(dict(name=a.get("name", f"site{len(sites)}"), bodyid=bid, pos=_vec(a.get("pos"), default=[0, 0, 0]), quat=_frame_quat(a, compiler),
                          type=_GEOM_TYPES[a.get("type", "sphere")], size=ssize))
      elif tag == "camera":
        a = attrs(child, childclass)
        cams.append(dict(name=a.get("name", f"cam{len(cams)}"), bodyid=bid, pos=_vec(a.get("pos"), default=[0, 0, 0]), quat=_frame_quat(a, compiler), mode=C.CAMLIGHT_MODES[a.get("mode", "fixed")], target=a.get("target"),
                         **_camera_optics(a)))
      elif tag == "light":
        a = attrs(child, childclass)
        d = _vec(a.get("dir"), default=[0, 0, -1])
        lights.append(dict(name=a.get("name", f"light{len(lights)}"), bodyid=bid, pos=_vec(a.get("pos"), default=[0, 0, 0]), dir=d / np.linalg.norm(d), mode=C.CAMLIGHT_MODES[a.get("mode", "fixed")], target=a.get("target"),
                           **_light_optics(a)))
      elif tag == "body":
        pass
      elif tag in ("flexcomp", "composite", "plugin"):
        # deformable / procedurally generated bodies would change the dynamics if they were dropped: say so instead
        raise NotImplementedError(f"<{tag}> inside <body> is not supported by this compiler (flex / composite / plugin bodies)")
      elif not isinstance(tag, str) or tag in ("frame", "replicate", "attach"):
        pass  # comments; composite wrappers are expanded before this pass
      else:
        raise NotImplementedError(f"unknown element <{tag}> inside <body>")
    for child in elem:
      if child.tag == "body":
        add_body(child, bid, childclass)

  # MuJoCo numbers bodies depth-first with all of a body's own elements before its children,
  # but children are visited in document order AFTER the parent's elements: emulate by recursion.
  wb = root.find("worldbody")
  add_body(wb, -1, None)

  nbody, njnt, ngeom = len(bodies), len(joints), len(geoms)

  m = SimpleNamespace()
  m.opt = opt
  m.skipped_mesh_geoms = skipped_mesh_geoms
  m.names = SimpleNamespace(
    body=[b["name"] for b in bodies], joint=[j["name"] for j in joints], geom=[g["name"] for g in geoms],
    site=[s["name"] for s in sites], camera=[c["name"] for c in cams], light=[l["name"] for l in lights],
  )

  # ---- bodies
  m.nbody = nbody
  m.body_parentid = np.array([b["parentid"] for b in bodies], dtype=np.int32)
  m.body_pos = np.array([b["pos"] for b in bodies])
  m.body_quat = np.array([b["quat"] for b in bodies])
  m.body_jntnum = np.array([b["jntnum"] for b in bodies], dtype=np.int32)
  m.body_jntadr = np.array([b["jntadr"] for b in bodies], dtype=np.int32)
  m.body_geomnum = np.array([b["geomnum"] for b in bodies], dtype=np.int32)
  m.body_geomadr = np.array([b["geomadr"] for b in bodies], dtype=np.int32)
  m.body_gravcomp = np.array([b["gravcomp"] for b in bodies])
  mocapid = -np.ones(nbody, dtype=np.int32)
  nm = 0
  for i, b in enumerate(bodies):
    if b["mocap"]:
      mocapid[i] = nm
      nm += 1
  m.body_mocapid = mocapid
  m.nmocap = nm

  # ---- joints / dofs
  m.njnt = njnt
  m.jnt_type = np.array([j["type"] for j in joints], dtype=np.int32)
  m.jnt_bodyid = np.array([j["bodyid"] for j in joints], dtype=np.int32)
  qn = {C.JNT_FREE: 7, C.JNT_BALL: 4, C.JNT_SLIDE: 1, C.JNT_HINGE: 1}
  vn = {C.JNT_FREE: 6, C.JNT_BALL: 3, C.JNT_SLIDE: 1, C.JNT_HINGE: 1}
  qadr, dadr = [], []
  nq = nv = 0
  for j in joints:
    qadr.append(nq)
    dadr.append(nv)
    nq += qn[j["type"]]
    nv += vn[j["type"]]
  m.nq, m.nv = nq, nv
  m.jnt_qposadr = np.array(qadr, dtype=np.int32)
  m.jnt_dofadr = np.array(dadr, dtype=np.int32)
  m.jnt_pos = np.array([j["pos"] for j in joints]).reshape(njnt, 3)
  m.jnt_axis = np.array([j["axis"] for j in joints]).reshape(njnt, 3)
  m.jnt_range = np.array([j["range"] for j in joints]).reshape(njnt, 2)
  m.jnt_limited = np.array([j["limited"] for j in joints], dtype=bool)
  m.jnt_stiffness = np.array([j["stiffness"] for j in joints])
  m.jnt_margin = np.array([j["margin"] for j in joints])
  m.jnt_solref = np.array([j["solreflimit"] for j in joints]).reshape(njnt, 2)
  m.jnt_solimp = np.array([j["solimplimit"] for j in joints]).reshape(njnt, 5)
  m.jnt_actfrclimited = np.array([j["actfrclimited"] for j in joints], dtype=bool)
  m.jnt_actfrcrange = np.array([j["actfrcrange"] for j in joints]).reshape(njnt, 2)
  m.jnt_actgravcomp = np.array([j["actgravcomp"] for j in joints], dtype=np.int32)

  m.body_dofnum = np.zeros(nbody, dtype=np.int32)
  m.body_dofadr = -np.ones(nbody, dtype=np.int32)
  for ji, j in enumerate(joints):
    b = j["bodyid"]
    if m.body_dofnum[b] == 0:
      m.body_dofadr[b] = dadr[ji]
    m.body_dofnum[b] += vn[j["type"]]

  dof_bodyid, dof_jntid = [], []
  dof_armature, dof_damping, dof_frictionloss = [], [], []
  dof_solref, dof_solimp = [], []
  qpos0 = np.zeros(nq)
  qpos_spring = np.zeros(nq)
  for ji, j in enumerate(joints):
    for _ in range(vn[j["type"]]):
      dof_bodyid.append(j["bodyid"])
      dof_jntid.append(ji)
      dof_armature.append(j["armature"])
      dof_damping.append(j["damping"])
      dof_frictionloss.append(j["frictionloss"])
      dof_solref.append(j["solreffriction"])
      dof_solimp.append(j["solimpfriction"])
    qa = qadr[ji]
    b = bodies[j["bodyid"]]
    if j["type"] == C.JNT_FREE:
      qpos0[qa : qa + 3] = b["pos"]
      qpos0[qa + 3 : qa + 7] = b["quat"]
      qpos_spring[qa : qa + 7] = qpos0[qa : qa + 7]
    elif j["type"] == C.JNT_BALL:
      qpos0[qa : qa + 4] = [1, 0, 0, 0]
      qpos_spring[qa : qa + 4] = [1, 0, 0, 0]
    else:
      qpos0[qa] = j["ref"]
      qpos_spring[qa] = j["springref"]
  m.qpos0, m.qpos_spring = qpos0, qpos_spring
  m.dof_bodyid = np.array(dof_bodyid, dtype=np.int32)
  m.dof_jntid = np.array(dof_jntid, dtype=np.int32)
  m.dof_armature = np.array(dof_armature)
  m.dof_damping = np.array(dof_damping)
  m.dof_frictionloss = np.array(dof_frictionloss)
  m.dof_solref = np.array(dof_solref).reshape(nv, 2)
  m.dof_solimp = np.array(dof_solimp).reshape(nv, 5)

  # dof_parentid: previous dof in the same body, else last dof of the nearest ancestor with dofs
  dof_parentid = -np.ones(nv, dtype=np.int32)
  for d in range(nv):
    b = m.dof_bodyid[d]
    if d > m.body_dofadr[b]:
      dof_parentid[d] = d - 1
    else:
      p = m.body_parentid[b]
      while p > 0 and m.body_dofnum[p] == 0:
        p = m.body_parentid[p]
      if p > 0 or (p == 0 and m.body_dofnum[0] > 0):
        if m.body_dofnum[p] > 0:
          dof_parentid[d] = m.body_dofadr[p] + m.body_dofnum[p] - 1
  m.dof_parentid = dof_parentid

  # rootid / weldid / treeid
  rootid = np.zeros(nbody, dtype=np.int32)
  weldid = np.zeros(nbody, dtype=np.int32)
  for b in range(1, nbody):
    p = m.body_parentid[b]
    rootid[b] = b if p == 0 else rootid[p]
    weldid[b] = b if m.body_jntnum[b] > 0 else weldid[p]
  m.body_rootid, m.body_weldid = rootid, weldid
  treeid = -np.ones(nbody, dtype=np.int32)
  ntree = 0
  tree_dofadr, tree_dofnum = [], []
  for b in range(1, nbody):
    p = m.body_parentid[b]
    if m.body_dofnum[b] > 0 and (p == 0 or treeid[p] < 0) and weldid[b] == b:
      treeid[b] = ntree
      tree_dofadr.append(int(m.body_dofadr[b]))
      tree_dofnum.append(0)
      ntree += 1
    elif p > 0:
      treeid[b] = treeid[p]
  m.ntree = ntree
  m.body_treeid = treeid
  m.dof_treeid = np.array([treeid[b] for b in m.dof_bodyid], dtype=np.int32)
  for d in range(nv):
    tree_dofnum[m.dof_treeid[d]] += 1
  m.tree_dofadr = np.array(tree_dofadr, dtype=np.int32)
  m.tree_dofnum = np.array(tree_dofnum, dtype=np.int32)

  # CSR lower-triangular M: row i holds ancestors of dof i in ascending order, diagonal last
  rownnz, rowadr, colind = [], [], []
  adr = 0
  for i in range(nv):
    chain = []
    d = i
    while d >= 0:
      chain.append(d)
      d = dof_parentid[d]
    chain.reverse()
    rownnz.append(len(chain))
    rowadr.append(adr)
    colind.extend(chain)
    adr += len(chain)
  m.M_rownnz = np.array(rownnz, dtype=np.int32)
  m.M_rowadr = np.array(rowadr, dtype=np.int32)
  m.M_colind = np.array(colind, dtype=np.int32)
  m.nC = m.nM = adr
  m.dof_Madr = (m.M_rowadr + m.M_rownnz - 1).astype(np.int32)
  d_structure(m)

  # ---- geoms
  m.ngeom = ngeom
  m.geom_type = np.array([g["type"] for g in geoms], dtype=np.int32)
  m.geom_bodyid = np.array([g["bodyid"] for g in geoms], dtype=np.int32)
  m.geom_contype = np.array([g["contype"] for g in geoms], dtype=np.int32)
  m.geom_conaffinity = np.array([g["conaffinity"] for g in geoms], dtype=np.int32)
  m.geom_condim = np.array([g["condim"] for g in geoms], dtype=np.int32)
  m.geom_priority = np.array([g["priority"] for g in geoms], dtype=np.int32)
  m.geom_dataid = np.array([g["dataid"] for g in geoms], dtype=np.int32).reshape(ngeom)
  m.geom_group = np.array([g["group"] for g in geoms], dtype=np.int32).reshape(ngeom)
  m.geom_matid = np.array([g["matid"] for g in geoms], dtype=np.int32).reshape(ngeom)
  m.geom_rgba = np.array([g["rgba"] for g in geoms]).reshape(ngeom, 4)
  m.geom_fluid = np.array([g["fluid"] for g in geoms]).reshape(ngeom, 12)
  m.nmat = len(mat_names)
  m.mat_rgba = np.array(mat_rgba).reshape(m.nmat, 4)
  ml = np.array(mat_light, dtype=np.float64).reshape(m.nmat, 3 + len(_TEX_ROLES))
  m.mat_specular, m.mat_shininess, m.mat_emission = ml[:, 0].copy(), ml[:, 1].copy(), ml[:, 2].copy()
  m.mat_texid = ml[:, 3:].astype(np.int32)
  m.names.material = list(mat_names)
  m.geom_size = np.array([g["size"] for g in geoms]).reshape(ngeom, 3)
  m.geom_pos = np.array([g["pos"] for g in geoms]).reshape(ngeom, 3)
  m.geom_quat = np.array([g["quat"] for g in geoms]).reshape(ngeom, 4)
  m.geom_friction = np.array([g["friction"] for g in geoms]).reshape(ngeom, 3)
  m.geom_solmix = np.array([g["solmix"] for g in geoms])
  m.geom_solref = np.array([g["solref"] for g in geoms]).reshape(ngeom, 2)
  m.geom_solimp = np.array([g["solimp"] for g in geoms]).reshape(ngeom, 5)
  m.geom_margin = np.array([g["margin"] for g in geoms])
  m.geom_gap = np.array([g["gap"] for g in geoms])
  m.geom_rbound = np.array([meshes[g["dataid"]]["rbound"] if g["dataid"] >= 0 else _geom_rbound(g["type"], g["size"]) for g in geoms])
  m.geom_aabb = np.array([np.concatenate([meshes[g["dataid"]]["aabb_center"], meshes[g["dataid"]]["aabb_size"]]) if g["dataid"] >= 0
                          else _geom_aabb(g["type"], g["size"]) for g in geoms]).reshape(ngeom, 6)

  # ---- body inertial properties
  mass = np.zeros(nbody)
  ipos = np.zeros((nbody, 3))
  iquat = np.tile(np.array([1.0, 0, 0, 0]), (nbody, 1))
  inertia = np.zeros((nbody, 3))
  for bi, b in enumerate(bodies):
    use_geoms = compiler["inertiafromgeom"] == "true" or (compiler["inertiafromgeom"] == "auto" and b["inertial"] is None)
    if not use_geoms:
      if b["inertial"] is not None:
        ipos[bi], iquat[bi], mass[bi], inertia[bi] = b["inertial"]
      continue
    if bi == 0:
      continue
    gs = [g for g in geoms if g["bodyid"] == bi]
    tot, com = 0.0, np.zeros(3)
    parts = []
    for g in gs:
      vol, iu = (meshes[g["dataid"]]["volume"], meshes[g["dataid"]]["inertia"]) if g["dataid"] >= 0 else _geom_volume_inertia(g["type"], g["size"])
      if vol <= 0:
        continue
      gm = g["mass"] if g["mass"] is not None else g["density"] * vol
      if gm <= 0:
        continue
      parts.append((gm, g["pos"], quat_to_mat(g["quat"]), iu * (gm / vol)))
      tot += gm
      com += gm * g["pos"]
    if tot <= 0:
      continue
    com /= tot
    full = np.zeros((3, 3))
    for gm, gp, R, ig in parts:
      d = gp - com
      full += R @ np.diag(ig) @ R.T + gm * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
    inertia[bi], iquat[bi] = _principal(full)
    mass[bi], ipos[bi] = tot, com
  if compiler["boundmass"] > 0:
    mass[1:] = np.maximum(mass[1:], compiler["boundmass"])
  if compiler["boundinertia"] > 0:
    inertia[1:] = np.maximum(inertia[1:], compiler["boundinertia"])
  m.body_mass, m.body_ipos, m.body_iquat, m.body_inertia = mass, ipos, iquat, inertia
  sub = mass.copy()
  for b in range(nbody - 1, 0, -1):
    sub[m.body_parentid[b]] += sub[b]
  m.body_subtreemass = sub

  # ---- sites / cameras / lights
  m.nsite = len(sites)
  m.site_bodyid = np.array([s["bodyid"] for s in sites], dtype=np.int32)
  m.site_pos = np.array([s["pos"] for s in sites]).reshape(m.nsite, 3)
  m.site_quat = np.array([s["quat"] for s in sites]).reshape(m.nsite, 4)
  m.site_type = np.array([s["type"] for s in sites], dtype=np.int32).reshape(m.nsite)
  m.site_size = np.array([s["size"] for s in sites], dtype=np.float64).reshape(m.nsite, 3)

  def body_id(name):
    return m.names.body.index(name) if name is not None else -1

  m.ncam = len(cams)
  m.cam_mode = np.array([c["mode"] for c in cams], dtype=np.int32)
  m.cam_bodyid = np.array([c["bodyid"] for c in cams], dtype=np.int32)
  m.cam_targetbodyid = np.array([body_id(c["target"]) for c in cams], dtype=np.int32)
  m.cam_pos = np.array([c["pos"] for c in cams]).reshape(m.ncam, 3)
  m.cam_quat = np.array([c["quat"] for c in cams]).reshape(m.ncam, 4)
  m.nlight = len(lights)
  m.light_mode = np.array([l["mode"] for l in lights], dtype=np.int32)
  m.light_bodyid = np.array([l["bodyid"] for l in lights], dtype=np.int32)
  m.light_targetbodyid = np.array([body_id(l["target"]) for l in lights], dtype=np.int32)
  m.light_pos = np.array([l["pos"] for l in lights]).reshape(m.nlight, 3)
  m.light_dir = np.array([l["dir"] for l in lights]).reshape(m.nlight, 3)
  # the renderer's camera and light fields (MuJoCo's names and defaults)
  for n, shape, dt in _CAMERA_FIELDS:
    setattr(m, "cam_" + n, np.array([c[n] for c in cams], dtype=dt).reshape((m.ncam,) + shape))
  for n, shape, dt in _LIGHT_FIELDS:
    setattr(m, "light_" + n, np.array([l[n] for l in lights], dtype=dt).reshape((m.nlight,) + shape))
  hl = dict(_HEADLIGHT_DEFAULTS)
  vis_e = root.find("visual")
  hl_e = vis_e.find("headlight") if vis_e is not None else None
  if hl_e is not None:
    hl.update({k: (int(hl_e.get(k)) if k == "active" else _vec(hl_e.get(k), 3)) for k in hl if k in hl_e.attrib})
  m.vis = SimpleNamespace(headlight=SimpleNamespace(**hl))

  # ---- tendons: fixed tendons (linear combinations of scalar joint positions); spatial tendons are not compiled
  tens = []
  te = root.find("tendon")
  for child in (list(te) if te is not None else []):
    if child.tag != "fixed":
      raise NotImplementedError(f"<tendon><{child.tag}>: only fixed tendons are supported")
    a = dflt.resolve("tendon", child.get("class", "main"))
    a.update(child.attrib)
    path = []
    for w in child:
      if w.tag != "joint":
        raise NotImplementedError(f"fixed tendon element <{w.tag}>")
      j = m.names.joint.index(w.get("joint"))
      if m.jnt_type[j] not in (C.JNT_SLIDE, C.JNT_HINGE):
        raise ValueError("fixed tendons combine slide / hinge joints")
      path.append((j, float(w.get("coef", 1.0))))
    if float(a.get("armature", 0.0)) != 0.0:
      raise NotImplementedError("tendon armature is not supported")
    rng = _vec(a.get("range"), 2, default=[0, 0])
    lim = a.get("limited", "auto")
    sl = _vec(a.get("springlength"), default=[-1.0])
    tens.append(dict(
      name=a.get("name", f"tendon{len(tens)}"), path=path, range=rng,
      limited=(lim == "true") or (lim == "auto" and compiler["autolimits"] and "range" in a),
      margin=float(a.get("margin", 0.0)), stiffness=float(a.get("stiffness", 0.0)), damping=float(a.get("damping", 0.0)),
      frictionloss=float(a.get("frictionloss", 0.0)), springlength=(sl if sl.size == 2 else np.array([sl[0], sl[0]])),
      solref_lim=_vec(a.get("solreflimit", "0.02 1")), solimp_lim=_vec(a.get("solimplimit", "0.9 0.95 0.001 0.5 2")),
      solref_fri=_vec(a.get("solreffriction", "0.02 1")), solimp_fri=_vec(a.get("solimpfriction", "0.9 0.95 0.001 0.5 2")),
      actfrcrange=_vec(a.get("actuatorfrcrange"), 2, default=[0, 0]),
      actfrclimited=(a.get("actuatorfrclimited", "auto") == "true") or (a.get("actuatorfrclimited", "auto") == "auto" and compiler["autolimits"] and "actuatorfrcrange" in a),
    ))
  nt = len(tens)
  m.ntendon = nt
  m.names.tendon = [t["name"] for t in tens]
  m.tendon_num = np.array([len(t["path"]) for t in tens], dtype=np.int32)
  m.tendon_adr = (np.concatenate(([0], np.cumsum(m.tendon_num)[:-1])) if nt else np.zeros(0)).astype(np.int32)
  m.nwrap = int(m.tendon_num.sum()) if nt else 0
  m.wrap_type = np.full(m.nwrap, C.WRAP_JOINT, dtype=np.int32)
  m.wrap_objid = np.array([j for t in tens for j, _ in t["path"]], dtype=np.int32)
  m.wrap_prm = np.array([c for t in tens for _, c in t["path"]], dtype=np.float64)
  m.tendon_limited = np.array([t["limited"] for t in tens], dtype=bool)
  m.tendon_range = np.array([t["range"] for t in tens], dtype=np.float64).reshape(nt, 2)
  m.tendon_margin = np.array([t["margin"] for t in tens], dtype=np.float64)
  m.tendon_stiffness = np.array([t["stiffness"] for t in tens], dtype=np.float64)
  m.tendon_damping = np.array([t["damping"] for t in tens], dtype=np.float64)
  m.tendon_armature = np.zeros(nt)
  m.tendon_frictionloss = np.array([t["frictionloss"] for t in tens], dtype=np.float64)
  m.tendon_lengthspring = np.array([t["springlength"] for t in tens], dtype=np.float64).reshape(nt, 2)  # (-1, -1) -> length0 in _set_const
  m.tendon_solref_lim = np.array([t["solref_lim"] for t in tens], dtype=np.float64).reshape(nt, 2)
  m.tendon_solimp_lim = np.array([t["solimp_lim"] for t in tens], dtype=np.float64).reshape(nt, 5)
  m.tendon_solref_fri = np.array([t["solref_fri"] for t in tens], dtype=np.float64).reshape(nt, 2)
  m.tendon_solimp_fri = np.array([t["solimp_fri"] for t in tens], dtype=np.float64).reshape(nt, 5)
  m.tendon_actfrclimited = np.array([t["actfrclimited"] for t in tens], dtype=bool)
  m.tendon_actfrcrange = np.array([t["actfrcrange"] for t in tens], dtype=np.float64).reshape(nt, 2)
  m.tendon_length0 = np.zeros(nt)
  m.tendon_invweight0 = np.zeros(nt)
  # sparsity of the tendon Jacobian (MjModel ten_J_rownnz / rowadr / colind): the dofs of a fixed tendon's joints, ascending
  rows = [sorted({int(m.jnt_dofadr[j]) for j, _ in t["path"]}) for t in tens]
  m.ten_J_rownnz = np.array([len(r) for r in rows], dtype=np.int32)
  m.ten_J_rowadr = (np.concatenate(([0], np.cumsum(m.ten_J_rownnz)[:-1])) if nt else np.zeros(0)).astype(np.int32)
  m.ten_J_colind = np.array([c for r in rows for c in r], dtype=np.int32)
  m.nJten = int(m.ten_J_rownnz.sum()) if nt else 0

  # ---- actuators
  acts = []
  ae = root.find("actuator")
  if ae is not None:
    for child in ae:
      if child.tag not in _ACT_TAGS:
        continue
      a = dflt.resolve(child.tag, child.get("class", "main"))
      a.update(child.attrib)
      acts.append((child.tag, a))
  nu = len(acts)
  m.nu = nu
  m.na = 0
  m.actuator_trntype = np.zeros(nu, dtype=np.int32)
  m.actuator_dyntype = np.zeros(nu, dtype=np.int32)
  m.actuator_gaintype = np.zeros(nu, dtype=np.int32)
  m.actuator_biastype = np.zeros(nu, dtype=np.int32)
  m.actuator_trnid = -np.ones((nu, 2), dtype=np.int32)
  m.actuator_gear = np.zeros((nu, 6))
  m.actuator_gainprm = np.zeros((nu, 10))
  m.actuator_biasprm = np.zeros((nu, 10))
  m.actuator_dynprm = np.zeros((nu, 10))
  m.actuator_ctrllimited = np.zeros(nu, dtype=bool)
  m.actuator_ctrlrange = np.zeros((nu, 2))
  m.actuator_forcelimited = np.zeros(nu, dtype=bool)
  m.actuator_forcerange = np.zeros((nu, 2))
  m.actuator_actlimited = np.zeros(nu, dtype=bool)
  m.actuator_actrange = np.zeros((nu, 2))
  m.actuator_actadr = -np.ones(nu, dtype=np.int32)
  m.actuator_actnum = np.zeros(nu, dtype=np.int32)
  m.actuator_actearly = np.zeros(nu, dtype=bool)
  m.names.actuator = []
  m.actuator_history = np.zeros((nu, 2), dtype=np.int32)
  m.actuator_delay = np.zeros(nu)
  m.actuator_lengthrange = np.zeros((nu, 2))
  dyn_names = {"none": C.DYN_NONE, "integrator": C.DYN_INTEGRATOR, "filter": C.DYN_FILTER, "filterexact": C.DYN_FILTEREXACT, "muscle": C.DYN_MUSCLE}
  gain_names = {"fixed": C.GAIN_FIXED, "affine": C.GAIN_AFFINE, "muscle": C.GAIN_MUSCLE}
  bias_names = {"none": C.BIAS_NONE, "affine": C.BIAS_AFFINE, "muscle": C.BIAS_MUSCLE}
  for i, (tag, a) in enumerate(acts):
    m.names.actuator.append(a.get("name", f"actuator{i}"))
    m.actuator_history[i], m.actuator_delay[i], _ = _history_attrs(a, f"actuator '{m.names.actuator[-1]}'", interval=False)
    if "tendon" in a:
      m.actuator_trntype[i] = C.TRN_TENDON
      m.actuator_trnid[i, 0] = m.names.tendon.index(a["tendon"])
    elif "joint" in a:
      m.actuator_trntype[i] = C.TRN_JOINT
      m.actuator_trnid[i, 0] = m.names.joint.index(a["joint"])
    else:
      raise NotImplementedError(f"actuator transmission other than joint / tendon is not supported: {a}")
    gear = _vec(a.get("gear"), 6, default=[1, 0, 0, 0, 0, 0])
    m.actuator_gear[i] = gear
    m.actuator_gainprm[i, 0] = 1.0
    m.actuator_dynprm[i, 0] = 1.0
    if tag == "general":
      dyn = a.get("dyntype", "none")
      if dyn not in dyn_names:
        raise NotImplementedError(f"actuator dyntype '{dyn}' is not supported (none, integrator, filter, filterexact, muscle are)")
      m.actuator_dyntype[i] = dyn_names[dyn]
      if "dynprm" in a:
        dp = _vec(a["dynprm"])
        m.actuator_dynprm[i, :] = 0
        m.actuator_dynprm[i, : dp.size] = dp
      gt, bt = a.get("gaintype", "fixed"), a.get("biastype", "none")
      if gt not in gain_names:
        raise NotImplementedError(f"actuator gaintype '{gt}' is not supported (fixed, affine, muscle are)")
      if bt not in bias_names:
        raise NotImplementedError(f"actuator biastype '{bt}' is not supported (none, affine, muscle are)")
      m.actuator_gaintype[i] = gain_names[gt]
      m.actuator_biastype[i] = bias_names[bt]
      if "gainprm" in a:
        gp = _vec(a["gainprm"])
        m.actuator_gainprm[i, :] = 0
        m.actuator_gainprm[i, : gp.size] = gp
      if "biasprm" in a:
        bp = _vec(a["biasprm"])
        m.actuator_biasprm[i, : bp.size] = bp
    elif tag == "motor":
      pass
    elif tag == "position":
      kp = float(a.get("kp", 1.0))
      kv = float(a.get("kv", 0.0))
      m.actuator_gainprm[i, 0] = kp
      m.actuator_biastype[i] = C.BIAS_AFFINE
      m.actuator_biasprm[i, 1] = -kp
      m.actuator_biasprm[i, 2] = -kv
      if "dampratio" in a:
        raise NotImplementedError("<position dampratio> is not supported")
      tc = float(a.get("timeconst", 0.0))
      if tc > 0:  # first-order filter on the target, integrated exactly
        m.actuator_dyntype[i] = C.DYN_FILTEREXACT
        m.actuator_dynprm[i, 0] = tc
    elif tag == "intvelocity":  # integrated-velocity servo: the activation is the position target
      kp = float(a.get("kp", 1.0))
      kv = float(a.get("kv", 0.0))
      m.actuator_dyntype[i] = C.DYN_INTEGRATOR
      m.actuator_gainprm[i, 0] = kp
      m.actuator_biastype[i] = C.BIAS_AFFINE
      m.actuator_biasprm[i, 1] = -kp
      m.actuator_biasprm[i, 2] = -kv
      if "actrange" not in a:
        raise ValueError("<intvelocity> requires actrange")
      a.setdefault("actlimited", "true")
    elif tag == "damper":  # force = -kv * velocity * ctrl
      kv = float(a.get("kv", 1.0))
      m.actuator_gaintype[i] = C.GAIN_AFFINE
      m.actuator_gainprm[i, :] = 0
      m.actuator_gainprm[i, 2] = -kv
      if "ctrlrange" not in a:
        raise ValueError("<damper> requires ctrlrange")
      a.setdefault("ctrllimited", "true")
    elif tag == "velocity":
      kv = float(a.get("kv", 1.0))
      m.actuator_gainprm[i, 0] = kv
      m.actuator_biastype[i] = C.BIAS_AFFINE
      m.actuator_biasprm[i, 2] = -kv
    elif tag == "muscle":  # MuJoCo's <muscle> shortcut: dynprm = (timeconst, tausmooth), gainprm = biasprm = the 9 muscle parameters
      m.actuator_dyntype[i], m.actuator_gaintype[i], m.actuator_biastype[i] = C.DYN_MUSCLE, C.GAIN_MUSCLE, C.BIAS_MUSCLE
      m.actuator_dynprm[i, :] = 0
      m.actuator_dynprm[i, :2] = _vec(a.get("timeconst"), 2, default=[0.01, 0.04])
      m.actuator_dynprm[i, 2] = float(a.get("tausmooth", 0.0))
      m.actuator_gainprm[i, :] = 0
      m.actuator_gainprm[i, :2] = _vec(a.get("range"), 2, default=[0.75, 1.05])
      for k, (key, val) in enumerate(_MUSCLE_DEFAULTS):
        m.actuator_gainprm[i, 2 + k] = float(a.get(key, val))
      m.actuator_biasprm[i, :] = m.actuator_gainprm[i]
    else:
      raise NotImplementedError(f"actuator shortcut <{tag}> is not supported")
    if "lengthrange" in a:
      m.actuator_lengthrange[i] = _vec(a["lengthrange"], 2)
    m.actuator_actearly[i] = a.get("actearly", "false") == "true"
    if m.actuator_dyntype[i] != C.DYN_NONE or int(a.get("actdim", -1)) > 0:
      m.actuator_actnum[i] = int(a.get("actdim", -1)) if int(a.get("actdim", -1)) > 0 else 1
      m.actuator_actadr[i] = m.na
      m.na += int(m.actuator_actnum[i])
    for rng, lim in (("ctrlrange", "ctrllimited"), ("forcerange", "forcelimited"), ("actrange", "actlimited")):
      if rng in a:
        getattr(m, "actuator_" + rng)[i] = _vec(a[rng])
      l = a.get(lim, "auto")
      getattr(m, "actuator_" + lim)[i] = (l == "true") or (l == "auto" and compiler["autolimits"] and rng in a)

  _set_length_range(m, [tag for tag, _ in acts], ["lengthrange" in a for _, a in acts])

  # ---- contact excludes / pairs
  excl, pairs = [], []
  ce = root.find("contact")
  if ce is not None:
    for child in ce:
      if child.tag == "exclude":
        b1, b2 = body_id(child.get("body1")), body_id(child.get("body2"))
        excl.append((min(b1, b2) << 16) + max(b1, b2))
        excl.append((max(b1, b2) << 16) + min(b1, b2))
      elif child.tag == "pair":
        a = dflt.resolve("pair", child.get("class", "main"))
        a.update(child.attrib)
        g1, g2 = m.names.geom.index(a["geom1"]), m.names.geom.index(a["geom2"])
        # attributes left unset are derived from the two geoms the way MuJoCo's compiler does for explicit pairs:
        # condim / friction = max, solref / solimp mixed by solmix, margin / gap = max
        mix = m.geom_solmix[g1] / max(m.geom_solmix[g1] + m.geom_solmix[g2], C.MJ_MINVAL)
        fmax = np.maximum(m.geom_friction[g1], m.geom_friction[g2])
        fr = _vec(a.get("friction"), 5, [fmax[0], fmax[0], fmax[1], fmax[2], fmax[2]])
        if "friction" in a:
          given = len(a["friction"].split())
          if given == 1:
            fr[1] = fr[0]
        pairs.append(dict(
          geom1=g1, geom2=g2, dim=int(a.get("condim", max(m.geom_condim[g1], m.geom_condim[g2]))), friction=fr,
          solref=_vec(a.get("solref"), 2, mix * m.geom_solref[g1] + (1 - mix) * m.geom_solref[g2]),
          solreffriction=_vec(a.get("solreffriction"), 2, [0.0, 0.0]),
          solimp=_vec(a.get("solimp"), 5, mix * m.geom_solimp[g1] + (1 - mix) * m.geom_solimp[g2]),
          margin=float(a.get("margin", max(m.geom_margin[g1], m.geom_margin[g2]))), gap=float(a.get("gap", max(m.geom_gap[g1], m.geom_gap[g2]))),
        ))
  m.exclude_signature = np.array(excl, dtype=np.int64)
  m.nexclude = len(excl) // 2
  m.npair = len(pairs)
  m.pair_geom1 = np.array([p["geom1"] for p in pairs], dtype=np.int32)
  m.pair_geom2 = np.array([p["geom2"] for p in pairs], dtype=np.int32)
  m.pair_dim = np.array([p["dim"] for p in pairs], dtype=np.int32)
  m.pair_friction = np.array([p["friction"] for p in pairs], dtype=np.float64).reshape(m.npair, 5)
  m.pair_solref = np.array([p["solref"] for p in pairs], dtype=np.float64).reshape(m.npair, 2)
  m.pair_solreffriction = np.array([p["solreffriction"] for p in pairs], dtype=np.float64).reshape(m.npair, 2)
  m.pair_solimp = np.array([p["solimp"] for p in pairs], dtype=np.float64).reshape(m.npair, 5)
  m.pair_margin = np.array([p["margin"] for p in pairs], dtype=np.float64)
  m.pair_gap = np.array([p["gap"] for p in pairs], dtype=np.float64)

  # ---- equality constraints: connect / weld between bodies, joint coupling (tendon / flex equalities are not compiled)
  eqs = []
  ee = root.find("equality")
  if ee is not None:
    for child in ee:
      if child.tag not in ("connect", "weld", "joint", "tendon"):
        raise NotImplementedError(f"equality type <{child.tag}> is not supported")
      a = dflt.resolve("equality", child.get("class", "main"))
      a.update(child.attrib)
      data = np.zeros(11)
      if child.tag == "joint":
        etype, otype = C.EQ_JOINT, C.OBJ_JOINT
        o1 = m.names.joint.index(a["joint1"])
        o2 = m.names.joint.index(a["joint2"]) if "joint2" in a else -1
        data[:5] = _vec(a.get("polycoef", "0 1 0 0 0"))
      elif child.tag == "tendon":
        etype, otype = C.EQ_TENDON, C.OBJ_TENDON
        o1 = m.names.tendon.index(a["tendon1"])
        o2 = m.names.tendon.index(a["tendon2"]) if "tendon2" in a else -1
        data[:5] = _vec(a.get("polycoef", "0 1 0 0 0"))
      else:
        if "site1" in a:
          raise NotImplementedError("site-based connect / weld equalities are not supported")
        etype, otype = (C.EQ_CONNECT if child.tag == "connect" else C.EQ_WELD), C.OBJ_BODY
        o1 = m.names.body.index(a["body1"])
        o2 = m.names.body.index(a["body2"]) if "body2" in a else 0
        if child.tag == "connect":
          data[:3] = _vec(a["anchor"])
        else:
          data[:3] = _vec(a.get("anchor", "0 0 0"))
          if "relpose" in a:
            rp = _vec(a["relpose"])
            data[3:6], data[6:10] = rp[:3], rp[3:7]
          data[10] = float(a.get("torquescale", 1.0))
      eqs.append(dict(type=etype, objtype=otype, obj1=o1, obj2=o2, data=data, active=a.get("active", "true") == "true",
                      solref=_vec(a.get("solref", "0.02 1")), solimp=_vec(a.get("solimp", "0.9 0.95 0.001 0.5 2"))))
  m.neq = len(eqs)
  m.eq_type = np.array([e["type"] for e in eqs], dtype=np.int32)
  m.eq_objtype = np.array([e["objtype"] for e in eqs], dtype=np.int32)
  m.eq_obj1id = np.array([e["obj1"] for e in eqs], dtype=np.int32)
  m.eq_obj2id = np.array([e["obj2"] for e in eqs], dtype=np.int32)
  m.eq_active0 = np.array([e["active"] for e in eqs], dtype=bool)
  m.eq_solref = np.array([e["solref"] for e in eqs], dtype=np.float64).reshape(m.neq, 2)
  m.eq_solimp = np.array([e["solimp"] for e in eqs], dtype=np.float64).reshape(m.neq, 5)
  m.eq_data = np.array([e["data"] for e in eqs], dtype=np.float64).reshape(m.neq, 11)

  # unused families (sizes only; SURVEY.md Appendix C)
  m.nflex = m.nhfield = 0

  # ---- mesh tables (reference types.py:1214-1235), concatenated over the assets
  m.nmesh = len(meshes)
  m.names.mesh = list(mesh_names)
  cat = lambda key, dt, width=None: (np.concatenate([np.asarray(md[key]).reshape(-1, width) if width else np.asarray(md[key]).reshape(-1) for md in meshes]).astype(dt)
                                     if meshes else np.zeros((0, width) if width else 0, dtype=dt))
  count = lambda key, per=1: np.array([len(np.asarray(md[key]).reshape(-1)) // per for md in meshes], dtype=np.int32)
  adr = lambda n: (np.concatenate(([0], np.cumsum(n)[:-1])) if len(n) else np.zeros(0)).astype(np.int32)
  m.mesh_vertnum = count("vert", 3); m.mesh_vertadr = adr(m.mesh_vertnum); m.mesh_vert = cat("vert", np.float64, 3)
  m.mesh_facenum = count("face", 3); m.mesh_faceadr = adr(m.mesh_facenum); m.mesh_face = cat("face", np.int32, 3)
  m.mesh_graphadr = adr(count("graph")); m.mesh_graph = cat("graph", np.int32)
  m.mesh_pos = cat("pos", np.float64, 3); m.mesh_quat = cat("quat", np.float64, 4)
  m.mesh_polynum = count("polyvertnum"); m.mesh_polyadr = adr(m.mesh_polynum)
  m.mesh_polynormal = cat("polynormal", np.float64, 3)
  m.mesh_polyvertnum = cat("polyvertnum", np.int32)
  m.mesh_polyvertadr = adr(m.mesh_polyvertnum)  # addresses into mesh_polyvert run over all meshes
  m.mesh_polyvert = cat("polyvert", np.int32)
  m.mesh_polymapnum = cat("polymapnum", np.int32)
  m.mesh_polymapadr = adr(m.mesh_polymapnum)
  m.mesh_polymap = cat("polymap", np.int32)
  m.nmeshvert, m.nmeshface, m.nmeshgraph, m.nmeshpoly = len(m.mesh_vert), len(m.mesh_face), len(m.mesh_graph), len(m.mesh_polynormal)
  m.nmeshpolyvert, m.nmeshpolymap, m.nmeshnormal = len(m.mesh_polyvert), len(m.mesh_polymap), 0
  m.npolygonmax = int(m.mesh_polyvertnum.max()) if m.nmesh else 0  # most vertices in one hull polygon / most polygons at one vertex
  m.nmeshdegmax = int(m.mesh_polymapnum.max()) if m.nmesh else 0

  # ---- sensors (MuJoCo mjtSensor / mjtDataType / mjtStage values; element tag -> type, object kind, dim, datatype, stage)
  S = C
  table = {
    "jointpos": (S.SENS_JOINTPOS, "joint", 1, 0, 1), "jointvel": (S.SENS_JOINTVEL, "joint", 1, 0, 2),
    "tendonpos": (S.SENS_TENDONPOS, "tendon", 1, 0, 1), "tendonvel": (S.SENS_TENDONVEL, "tendon", 1, 0, 2),
    "actuatorpos": (S.SENS_ACTUATORPOS, "actuator", 1, 0, 1), "actuatorvel": (S.SENS_ACTUATORVEL, "actuator", 1, 0, 2),
    "actuatorfrc": (S.SENS_ACTUATORFRC, "actuator", 1, 0, 3), "jointactuatorfrc": (S.SENS_JOINTACTFRC, "joint", 1, 0, 3),
    "jointlimitpos": (S.SENS_JOINTLIMITPOS, "joint", 1, 0, 1), "jointlimitvel": (S.SENS_JOINTLIMITVEL, "joint", 1, 0, 2),
    "jointlimitfrc": (S.SENS_JOINTLIMITFRC, "joint", 1, 0, 3),
    "ballquat": (S.SENS_BALLQUAT, "joint", 4, 3, 1), "ballangvel": (S.SENS_BALLANGVEL, "joint", 3, 0, 2),
    "gyro": (S.SENS_GYRO, "site", 3, 0, 2), "velocimeter": (S.SENS_VELOCIMETER, "site", 3, 0, 2), "accelerometer": (S.SENS_ACCELEROMETER, "site", 3, 0, 3),
    "touch": (S.SENS_TOUCH, "site", 1, 1, 3), "force": (S.SENS_FORCE, "site", 3, 0, 3), "torque": (S.SENS_TORQUE, "site", 3, 0, 3),
    "subtreecom": (S.SENS_SUBTREECOM, "body", 3, 0, 1), "subtreelinvel": (S.SENS_SUBTREELINVEL, "body", 3, 0, 2),
    "subtreeangmom": (S.SENS_SUBTREEANGMOM, "body", 3, 0, 2), "clock": (S.SENS_CLOCK, None, 1, 0, 1),
    "framepos": (S.SENS_FRAMEPOS, "obj", 3, 0, 1), "framexaxis": (S.SENS_FRAMEXAXIS, "obj", 3, 2, 1), "frameyaxis": (S.SENS_FRAMEYAXIS, "obj", 3, 2, 1),
    "framezaxis": (S.SENS_FRAMEZAXIS, "obj", 3, 2, 1),
    "framequat": (S.SENS_FRAMEQUAT, "obj", 4, 3, 1), "framelinvel": (S.SENS_FRAMELINVEL, "obj", 3, 0, 2), "frameangvel": (S.SENS_FRAMEANGVEL, "obj", 3, 0, 2),
    "framelinacc": (S.SENS_FRAMELINACC, "obj", 3, 0, 3), "frameangacc": (S.SENS_FRAMEANGACC, "obj", 3, 0, 3),
    # collision sensors between two geoms or bodies: signed distance, unit normal (AXIS), and the two witness points
    "distance": (S.SENS_GEOMDIST, "pair", 1, 0, 1), "normal": (S.SENS_GEOMNORMAL, "pair", 3, 2, 1), "fromto": (S.SENS_GEOMFROMTO, "pair", 6, 0, 1),
    # potential and kinetic energy of the whole model (no object)
    "e_potential": (S.SENS_E_POTENTIAL, None, 1, 0, 1), "e_kinetic": (S.SENS_E_KINETIC, None, 1, 0, 1),
    # contacts matched against up to two sides; dim is num x the slot size of its data keywords (below)
    "contact": (S.SENS_CONTACT, "contact", 0, 0, 3),
    # a site's pixel in a camera's image, an object's point inside a site's volume (0 / 1).  `<magnetometer>` stays in
    # sensor_unsupported: put_model runs magnetometers of models that carry them in their arrays (sensor_type MAGNETOMETER on a site).
    "camprojection": (S.SENS_CAMPROJECTION, "extra", 2, 0, 1),
    "insidesite": (S.SENS_INSIDESITE, "extra", 1, 0, 1),
    # a tendon's limit row (distance - margin, velocity, force; 0 without an active row) and the force of the actuators on it
    "tendonlimitpos": (S.SENS_TENDONLIMITPOS, "extra", 1, 0, 1), "tendonlimitvel": (S.SENS_TENDONLIMITVEL, "extra", 1, 0, 2),
    "tendonlimitfrc": (S.SENS_TENDONLIMITFRC, "extra", 1, 0, 3), "tendonactfrc": (S.SENS_TENDONACTFRC, "extra", 1, 0, 3),
  }
  objkind = {"tendon": (C.OBJ_TENDON, "tendon"), "joint": (C.OBJ_JOINT, "joint"), "actuator": (C.OBJ_ACTUATOR, "actuator"), "site": (C.OBJ_SITE, "site"), "body": (C.OBJ_BODY, "body")}
  objtypes = {"body": (C.OBJ_BODY, "body"), "xbody": (C.OBJ_XBODY, "body"), "geom": (C.OBJ_GEOM, "geom"), "site": (C.OBJ_SITE, "site"), "camera": (C.OBJ_CAMERA, "camera")}
  sens, unsupported = [], []
  contact_sides = ((("site", C.OBJ_SITE), ("geom1", C.OBJ_GEOM), ("body1", C.OBJ_BODY), ("subtree1", C.OBJ_XBODY)),
                   (("geom2", C.OBJ_GEOM), ("body2", C.OBJ_BODY), ("subtree2", C.OBJ_XBODY)))
  nsens = root.find("sensor")
  for e in (list(nsens) if nsens is not None else []):
    has_ref = "reftype" in e.attrib or "refname" in e.attrib
    if e.tag not in table or (has_ref and e.tag not in ("framepos", "framequat", "framexaxis", "frameyaxis", "framezaxis", "framelinvel", "frameangvel")):
      unsupported.append(e.tag)
      continue
    stype, kind, dim, datatype, stage = table[e.tag]
    rtype, rid = C.OBJ_UNKNOWN, -1
    if has_ref:
      rtype, rlst = objtypes[e.get("reftype")]
      rid = getattr(m.names, rlst).index(e.get("refname"))
    if kind is None:
      otype, oid = C.OBJ_UNKNOWN, -1
    elif kind == "pair":  # exactly one of geom<k> / body<k> for each side; the second side is the reference object
      sides = []
      for k in ("1", "2"):
        given = [x for x in ("geom", "body") if x + k in e.attrib]
        if len(given) != 1:
          raise ValueError(f"{e.tag} sensor '{e.get('name', f'sensor{len(sens)}')}': give exactly one of geom{k} / body{k}")
        otype_k, lst = objtypes[given[0]]
        sides.append((otype_k, getattr(m.names, lst).index(e.get(given[0] + k))))
      (otype, oid), (rtype, rid) = sides
    elif kind == "contact":
      sname = e.get("name", f"sensor{len(sens)}")
      sides = []
      for side in contact_sides:
        given = [(a, t) for a, t in side if a in e.attrib]
        if len(given) > 1:
          raise ValueError(f"contact sensor '{sname}': give at most one of {' / '.join(a for a, _ in side)}, got {' and '.join(a for a, _ in given)}")
        if not given:
          sides.append((C.OBJ_UNKNOWN, -1))
          continue
        attr, t = given[0]
        lst = {C.OBJ_SITE: "site", C.OBJ_GEOM: "geom"}.get(t, "body")
        names = getattr(m.names, lst)
        if e.get(attr) not in names:
          raise ValueError(f"contact sensor '{sname}': unknown {lst} '{e.get(attr)}' in {attr}")
        sides.append((t, names.index(e.get(attr))))
      (otype, oid), (rtype, rid) = sides
      intprm = contact_intprm(e.get("data", "found"), e.get("reduce", "none"), e.get("num", "1"), f"contact sensor '{sname}'")
      dim = intprm[2] * contact_slot_size(intprm[0])
    elif kind == "extra":
      (otype, oid), (rtype, rid) = _extra_sensor_objects(e, m.names, objtypes, f"{e.tag} sensor '{e.get('name', f'sensor{len(sens)}')}'")
    elif kind == "obj":
      otype, lst = objtypes[e.get("objtype")]
      oid = getattr(m.names, lst).index(e.get("objname"))
    else:
      otype, lst = objkind[kind]
      oid = getattr(m.names, lst).index(e.get(kind))
    sname = e.get("name", f"sensor{len(sens)}")
    ha = {k: v for k, v in dflt.resolve("sensor", e.get("class", "main")).items() if k in _HISTORY_KEYS}
    ha.update(e.attrib)
    hist, delay, interval = _history_attrs(ha, f"sensor '{sname}'", interval=True)
    sens.append(dict(name=sname, type=stype, objtype=otype, objid=oid, reftype=rtype, refid=rid, dim=dim, datatype=datatype, needstage=stage,
                     cutoff=float(e.get("cutoff", 0.0)), noise=float(e.get("noise", 0.0)), history=hist, delay=delay, interval=interval,
                     intprm=intprm if kind == "contact" else (0, 0, 0)))
  m.nsensor = len(sens)
  m.sensor_unsupported = unsupported  # put_model refuses these (they would silently read zero otherwise)
  m.names.sensor = [x["name"] for x in sens]
  for key in ("type", "objtype", "objid", "reftype", "refid", "dim", "datatype", "needstage"):
    setattr(m, "sensor_" + key, np.array([x[key] for x in sens], dtype=np.int32).reshape(m.nsensor))
  m.sensor_intprm = np.array([x["intprm"] for x in sens], dtype=np.int32).reshape(m.nsensor, 3)
  m.sensor_cutoff = np.array([x["cutoff"] for x in sens], dtype=np.float64).reshape(m.nsensor)
  m.sensor_noise = np.array([x["noise"] for x in sens], dtype=np.float64).reshape(m.nsensor)
  m.sensor_adr = (np.concatenate(([0], np.cumsum(m.sensor_dim)[:-1])) if m.nsensor else np.zeros(0)).astype(np.int32)
  m.nsensordata = int(m.sensor_dim.sum()) if m.nsensor else 0
  m.sensor_history = np.array([x["history"] for x in sens], dtype=np.int32).reshape(m.nsensor, 2)
  m.sensor_delay = np.array([x["delay"] for x in sens], dtype=np.float64).reshape(m.nsensor)
  m.sensor_interval = np.array([x["interval"] for x in sens], dtype=np.float64).reshape(m.nsensor, 2)
  set_history_layout(m)

  # ---- <custom><numeric>: MjModel's numeric_adr / numeric_size / numeric_data; the contact sensors read contact_sensor_maxmatch from it
  nums = [n for c in root.findall("custom") for n in c.findall("numeric")]
  vals = [np.array([float(x) for x in n.get("data", "").split()], dtype=np.float64) for n in nums]
  for n, v in zip(nums, vals):
    size = int(n.get("size", len(v)))
    v.resize(max(size, len(v)), refcheck=False)
  m.nnumeric = len(nums)
  m.names.numeric = [n.get("name", "") for n in nums]
  m.numeric_size = np.array([len(v) for v in vals], dtype=np.int32)
  m.numeric_adr = (np.concatenate(([0], np.cumsum(m.numeric_size)[:-1])) if nums else np.zeros(0)).astype(np.int32)
  m.numeric_data = np.concatenate(vals) if nums else np.zeros(0)
  contact_sensor_maxmatch(m)

  # ---- keyframes
  keys = []
  ke = root.find("keyframe")
  if ke is not None:
    for k in ke.findall("key"):
      keys.append(k)
  m.nkey = len(keys)
  m.key_time = np.zeros(m.nkey)
  m.key_qpos = np.tile(qpos0, (m.nkey, 1)).reshape(m.nkey, nq)
  m.key_qvel = np.zeros((m.nkey, nv))
  m.key_ctrl = np.zeros((m.nkey, nu))
  m.key_act = np.zeros((m.nkey, m.na))
  m.names.key = []
  for i, k in enumerate(keys):
    m.names.key.append(k.get("name", f"key{i}"))
    if "time" in k.attrib:
      m.key_time[i] = float(k.get("time"))
    if "_part_body" in k.attrib:  # keyframe of an attached model: only that subtree's joints, the rest stays at qpos0
      v = _vec(k.get("_part_qpos"))
      b0 = m.names.body.index(k.get("_part_body"))
      adr = int(m.jnt_qposadr[m.body_jntadr[b0]])
      m.key_qpos[i, adr : adr + v.size] = v
      continue
    for nm_, arr in (("qpos", m.key_qpos), ("qvel", m.key_qvel), ("ctrl", m.key_ctrl), ("act", m.key_act)):
      if nm_ in k.attrib:
        v = _vec(k.get(nm_))
        if v.size != arr.shape[1]:
          raise ValueError(f"keyframe {i} {nm_} has {v.size} values, expected {arr.shape[1]}")
        arr[i] = v

  _set_const(m)
  return m


def _principal(full):
  """Principal inertia (descending) and the quaternion of the principal frame."""
  w, V = np.linalg.eigh(0.5 * (full + full.T))
  order = np.argsort(-w)
  w, V = w[order], V[:, order]
  if np.linalg.det(V) < 0:
    V[:, 2] = -V[:, 2]
  return w, mat_to_quat(V)


# ----------------------------------------------------------------------------------------------
# constants that need a forward pass at qpos0 (MuJoCo mj_setConst semantics; the reference
# re-derives the same quantities on device in /root/reference/mujoco_warp/_src/set_const.py)
# ----------------------------------------------------------------------------------------------


def kinematics_np(m, qpos):
  """Host FK at `qpos` (used for make_data static geoms and set_const)."""
  nb = m.nbody
  xpos = np.zeros((nb, 3))
  xquat = np.tile(np.array([1.0, 0, 0, 0]), (nb, 1))
  xanchor = np.zeros((m.njnt, 3))
  xaxis = np.zeros((m.njnt, 3))
  for b in range(1, nb):
    p = m.body_parentid[b]
    ja, jn = m.body_jntadr[b], m.body_jntnum[b]
    if jn == 1 and m.jnt_type[ja] == C.JNT_FREE:
      qa = m.jnt_qposadr[ja]
      xpos[b] = qpos[qa : qa + 3]
      q = qpos[qa + 3 : qa + 7]
      xquat[b] = q / np.linalg.norm(q)
      xanchor[ja] = xpos[b]
      xaxis[ja] = m.jnt_axis[ja]
      continue
    pos = rot_vec(xquat[p], m.body_pos[b]) + xpos[p]
    quat = quat_mul(xquat[p], m.body_quat[b])
    for j in range(ja, ja + jn):
      qa = m.jnt_qposadr[j]
      anchor = rot_vec(quat, m.jnt_pos[j]) + pos
      axis = rot_vec(quat, m.jnt_axis[j])
      t = m.jnt_type[j]
      if t == C.JNT_BALL:
        ql = qpos[qa : qa + 4]
        quat = quat_mul(quat, ql / np.linalg.norm(ql))
        pos = anchor - rot_vec(quat, m.jnt_pos[j])
      elif t == C.JNT_SLIDE:
        pos = pos + axis * (qpos[qa] - m.qpos0[qa])
      elif t == C.JNT_HINGE:
        quat = quat_mul(quat, axis_angle_quat(m.jnt_axis[j], qpos[qa] - m.qpos0[qa]))
        pos = anchor - rot_vec(quat, m.jnt_pos[j])
      xanchor[j], xaxis[j] = anchor, axis
    xpos[b] = pos
    xquat[b] = quat / np.linalg.norm(quat)
  out = SimpleNamespace(xpos=xpos, xquat=xquat, xanchor=xanchor, xaxis=xaxis)
  out.xmat = np.array([quat_to_mat(q) for q in xquat])
  out.xipos = np.array([xpos[b] + rot_vec(xquat[b], m.body_ipos[b]) for b in range(nb)])
  out.ximat = np.array([quat_to_mat(quat_mul(xquat[b], m.body_iquat[b])) for b in range(nb)])
  out.geom_xpos = np.array([xpos[m.geom_bodyid[g]] + rot_vec(xquat[m.geom_bodyid[g]], m.geom_pos[g]) for g in range(m.ngeom)]).reshape(m.ngeom, 3)
  out.geom_xmat = np.array([quat_to_mat(quat_mul(xquat[m.geom_bodyid[g]], m.geom_quat[g])) for g in range(m.ngeom)]).reshape(m.ngeom, 3, 3)
  out.site_xpos = np.array([xpos[m.site_bodyid[s]] + rot_vec(xquat[m.site_bodyid[s]], m.site_pos[s]) for s in range(m.nsite)]).reshape(m.nsite, 3)
  out.site_xmat = np.array([quat_to_mat(quat_mul(xquat[m.site_bodyid[s]], m.site_quat[s])) for s in range(m.nsite)]).reshape(m.nsite, 3, 3)
  # subtree com
  sc = out.xipos * m.body_mass[:, None]
  for b in range(nb - 1, 0, -1):
    sc[m.body_parentid[b]] += sc[b]
  for b in range(nb):
    if m.body_subtreemass[b] > 0:
      sc[b] = sc[b] / m.body_subtreemass[b]
    else:
      sc[b] = out.xipos[b]
  out.subtree_com = sc
  return out


def _body_jacobians(m, kin, point_of_body):
  """World-frame translational/rotational Jacobians (3 x nv each) of point_of_body[b] on body b."""
  nv = m.nv
  jacp = np.zeros((m.nbody, 3, nv))
  jacr = np.zeros((m.nbody, 3, nv))
  for b in range(1, m.nbody):
    bb = b
    while bb > 0:
      ja, jn = m.body_jntadr[bb], m.body_jntnum[bb]
      for j in range(ja, ja + jn):
        d = m.jnt_dofadr[j]
        t = m.jnt_type[j]
        r = point_of_body[b] - kin.xanchor[j]
        if t == C.JNT_FREE:
          jacp[b, :, d : d + 3] = np.eye(3)
          R = kin.xmat[bb]
          for k in range(3):
            jacr[b, :, d + 3 + k] = R[:, k]
            jacp[b, :, d + 3 + k] = np.cross(R[:, k], point_of_body[b] - kin.xpos[bb])
        elif t == C.JNT_BALL:
          R = kin.xmat[bb]
          for k in range(3):
            jacr[b, :, d + k] = R[:, k]
            jacp[b, :, d + k] = np.cross(R[:, k], r)
        elif t == C.JNT_SLIDE:
          jacp[b, :, d] = kin.xaxis[j]
        else:
          jacr[b, :, d] = kin.xaxis[j]
          jacp[b, :, d] = np.cross(kin.xaxis[j], r)
      bb = m.body_parentid[bb]
  return jacp, jacr


def dense_inertia_np(m, kin):
  """Joint-space inertia at the configuration in `kin` via sum_b J_b^T I_b J_b (+ armature)."""
  jacp, jacr = _body_jacobians(m, kin, kin.xipos)
  M = np.diag(m.dof_armature.astype(np.float64))
  for b in range(1, m.nbody):
    Ib = kin.ximat[b] @ np.diag(m.body_inertia[b]) @ kin.ximat[b].T
    M = M + m.body_mass[b] * jacp[b].T @ jacp[b] + jacr[b].T @ Ib @ jacr[b]
  return M, jacp, jacr


def _set_eq_data0(m, kin):
  """Connect / weld anchors and relative pose at qpos0 (reference set_const.py:78-153, MuJoCo mj_setConst)."""
  xmat = np.asarray(kin.xmat).reshape(m.nbody, 3, 3)
  for e in range(m.neq):
    o1, o2, data = int(m.eq_obj1id[e]), int(m.eq_obj2id[e]), m.eq_data[e]
    if m.eq_type[e] == C.EQ_CONNECT:
      pos = kin.xpos[o1] + xmat[o1] @ data[0:3]  # anchor given in body1's frame
      data[3:6] = xmat[o2].T @ (pos - kin.xpos[o2])
    elif m.eq_type[e] == C.EQ_WELD:
      quat = data[6:10]
      if quat @ quat > 0:
        data[6:10] = quat / np.linalg.norm(quat)
      else:
        pos = kin.xpos[o2] + xmat[o2] @ data[0:3]  # anchor given in body2's frame
        data[3:6] = xmat[o1].T @ (pos - kin.xpos[o1])
        q1 = kin.xquat[o1]
        data[6:10] = quat_mul(np.array([q1[0], -q1[1], -q1[2], -q1[3]]), kin.xquat[o2])


def _tendon_row(m, t):
  """Dense moment row (nv) of fixed tendon t."""
  J = np.zeros(m.nv)
  for k in range(m.tendon_adr[t], m.tendon_adr[t] + m.tendon_num[t]):
    J[m.jnt_dofadr[m.wrap_objid[k]]] += m.wrap_prm[k]
  return J


def _set_length_range(m, tags, explicit):
  """actuator_lengthrange: an explicit `lengthrange` is kept; otherwise a muscle on a limited joint or limited fixed tendon gets the
  limit range times gear[0], ends swapped for a negative gear (the rule of the reference's set_const.py:573-607; MuJoCo's compiler
  finds the range by simulation instead).  Any other actuator keeps (0, 0).  A muscle with neither is refused by name."""
  for i in range(m.nu):
    muscle = m.actuator_gaintype[i] == C.GAIN_MUSCLE or m.actuator_biastype[i] == C.BIAS_MUSCLE
    if not muscle:
      continue
    if explicit[i]:
      _check_muscle_lengthrange(m, i, tags[i])
      continue
    j, gear = int(m.actuator_trnid[i, 0]), float(m.actuator_gear[i, 0])
    if m.actuator_trntype[i] == C.TRN_JOINT and m.jnt_limited[j]:
      rng = m.jnt_range[j]
    elif m.actuator_trntype[i] == C.TRN_TENDON and m.tendon_limited[j]:
      rng = m.tendon_range[j]
    else:
      raise NotImplementedError(f"muscle actuator '{m.names.actuator[i]}' ({tags[i]}) needs a lengthrange: give lengthrange= or put it on a limited "
                                "joint or tendon (the simulation-based lengthrange computation is not implemented)")
    m.actuator_lengthrange[i] = (rng[0] * gear, rng[1] * gear) if gear > 0 else (rng[1] * gear, rng[0] * gear)
    _check_muscle_lengthrange(m, i, tags[i])


def _check_muscle_lengthrange(m, i, tag):
  """A muscle's optimum length is (lengthrange[1] - lengthrange[0]) / (range[1] - range[0]): an empty or reversed lengthrange (equal
  limits, gear 0, or an explicit range given backwards) would divide by MJ_MINVAL in the muscle curves."""
  lo, hi = m.actuator_lengthrange[i]
  if not lo < hi:
    raise ValueError(f"muscle actuator '{m.names.actuator[i]}' ({tag}): lengthrange must satisfy lengthrange[0] < lengthrange[1], got ({lo}, {hi})")


def _set_const(m):
  kin = kinematics_np(m, m.qpos0)
  nv = m.nv
  if getattr(m, "neq", 0):
    _set_eq_data0(m, kin)
  m.body_invweight0 = np.zeros((m.nbody, 2))
  m.dof_invweight0 = np.zeros(nv)
  m.actuator_acc0 = np.zeros(m.nu)
  if nv > 0:
    M, jacp, jacr = dense_inertia_np(m, kin)
    Minv = np.linalg.inv(M)
    m.stat = SimpleNamespace(meaninertia=max(C.MJ_MINVAL, float(np.trace(M)) / nv))
    for b in range(1, m.nbody):
      if m.body_weldid[b] == 0:
        continue
      A = jacp[b] @ Minv @ jacp[b].T
      B = jacr[b] @ Minv @ jacr[b].T
      m.body_invweight0[b, 0] = np.trace(A) / 3.0
      m.body_invweight0[b, 1] = np.trace(B) / 3.0
    dg = np.diag(Minv)
    for j in range(m.njnt):
      d = m.jnt_dofadr[j]
      t = m.jnt_type[j]
      if t == C.JNT_FREE:
        m.dof_invweight0[d : d + 3] = dg[d : d + 3].mean()
        m.dof_invweight0[d + 3 : d + 6] = dg[d + 3 : d + 6].mean()
      elif t == C.JNT_BALL:
        m.dof_invweight0[d : d + 3] = dg[d : d + 3].mean()
      else:
        m.dof_invweight0[d] = dg[d]
    for t in range(getattr(m, "ntendon", 0)):  # fixed tendons: length and moment are linear in the joint positions
      J = _tendon_row(m, t)
      m.tendon_length0[t] = sum(m.wrap_prm[k] * m.qpos0[m.jnt_qposadr[m.wrap_objid[k]]] for k in range(m.tendon_adr[t], m.tendon_adr[t] + m.tendon_num[t]))
      m.tendon_invweight0[t] = float(J @ Minv @ J)
      if m.tendon_lengthspring[t, 0] == -1.0 and m.tendon_lengthspring[t, 1] == -1.0:
        m.tendon_lengthspring[t] = m.tendon_length0[t]
    for i in range(m.nu):
      mom = np.zeros(nv)
      j = m.actuator_trnid[i, 0]
      if m.actuator_trntype[i] == C.TRN_TENDON:
        mom = m.actuator_gear[i, 0] * _tendon_row(m, j)
      else:
        mom[m.jnt_dofadr[j]] = m.actuator_gear[i, 0]
      m.actuator_acc0[i] = np.linalg.norm(Minv @ mom)
  else:
    m.stat = SimpleNamespace(meaninertia=1.0)

  # camera / light reference poses at qpos0 (used by track/trackcom modes; reference smooth.py:858-983)
  cam_xpos = np.array([kin.xpos[m.cam_bodyid[c]] + rot_vec(kin.xquat[m.cam_bodyid[c]], m.cam_pos[c]) for c in range(m.ncam)]).reshape(m.ncam, 3)
  cam_xmat = np.array([quat_to_mat(quat_mul(kin.xquat[m.cam_bodyid[c]], m.cam_quat[c])) for c in range(m.ncam)]).reshape(m.ncam, 3, 3)
  m.cam_pos0 = np.array([cam_xpos[c] - kin.xpos[m.cam_bodyid[c]] for c in range(m.ncam)]).reshape(m.ncam, 3)
  m.cam_poscom0 = np.array([cam_xpos[c] - kin.subtree_com[m.cam_bodyid[c]] for c in range(m.ncam)]).reshape(m.ncam, 3)
  m.cam_mat0 = cam_xmat
  l_xpos = np.array([kin.xpos[m.light_bodyid[l]] + rot_vec(kin.xquat[m.light_bodyid[l]], m.light_pos[l]) for l in range(m.nlight)]).reshape(m.nlight, 3)
  l_xdir = np.array([rot_vec(kin.xquat[m.light_bodyid[l]], m.light_dir[l]) for l in range(m.nlight)]).reshape(m.nlight, 3)
  m.light_pos0 = np.array([l_xpos[l] - kin.xpos[m.light_bodyid[l]] for l in range(m.nlight)]).reshape(m.nlight, 3)
  m.light_poscom0 = np.array([l_xpos[l] - kin.subtree_com[m.light_bodyid[l]] for l in range(m.nlight)]).reshape(m.nlight, 3)
  m.light_dir0 = l_xdir


class MjDataLite:
  """Minimal stand-in for mujoco.MjData: the state inputs put_data reads."""

  def __init__(self, m):
    self.qpos = m.qpos0.copy()
    self.qvel = np.zeros(m.nv)
    self.ctrl = np.zeros(m.nu)
    self.act = np.zeros(m.na)
    self.qacc_warmstart = np.zeros(m.nv)
    self.qfrc_applied = np.zeros(m.nv)
    self.xfrc_applied = np.zeros((m.nbody, 6))
    self.time = 0.0


def reset_data_keyframe(m, d: MjDataLite, key: int):
  d.qpos[:] = m.key_qpos[key]
  d.qvel[:] = m.key_qvel[key]
  d.ctrl[:] = m.key_ctrl[key]
  if getattr(m, "na", 0):
    d.act[:] = np.asarray(m.key_act)[key]
  d.time = float(m.key_time[key])
  d.qacc_warmstart[:] = 0


# ----------------------------------------------------------------------------------------------
# compiled-model (de)serialisation: lets a model compiled where the MJCF (or `mujoco`) is available
# travel as one .npz of MjModel-named arrays (SURVEY.md Appendix C "escape hatch")
# ----------------------------------------------------------------------------------------------


def d_structure(m):
  """MjModel's D-structure (dof-dof sparsity of the velocity derivatives, both triangles): row i lists the dofs coupled to dof i --
  ancestors, itself, descendants -- in ascending order; mapM2D sends entry (i, j) to the entry (max, min) of the lower-triangular M."""
  nv = int(m.nv)
  rows = [[] for _ in range(nv)]
  for i in range(nv):
    for k in range(int(m.M_rownnz[i])):
      e = int(m.M_rowadr[i]) + k
      j = int(m.M_colind[e])
      rows[i].append((j, e))
      if j != i:
        rows[j].append((i, e))
  rows = [sorted(r) for r in rows]
  m.D_rownnz = np.array([len(r) for r in rows], dtype=np.int32)
  m.D_rowadr = np.concatenate([[0], np.cumsum(m.D_rownnz)[:-1]]).astype(np.int32) if nv else np.zeros(0, np.int32)
  m.D_diag = np.array([[c for c, _ in r].index(i) for i, r in enumerate(rows)], dtype=np.int32)
  m.D_colind = np.array([c for r in rows for c, _ in r], dtype=np.int32)
  m.mapM2D = np.array([e for r in rows for _, e in r], dtype=np.int32)
  m.nD = int(m.D_rownnz.sum())


def save_npz(m, path: str):
  out = {}
  for k, v in vars(m).items():
    if k in ("opt", "stat", "names"):
      for kk, vv in vars(v).items():
        out[f"{k}.{kk}"] = np.asarray(vv)
    elif k == "vis":
      for kk, vv in vars(v.headlight).items():
        out[f"vis.headlight.{kk}"] = np.asarray(vv)
    else:
      out[k] = np.asarray(v)
  np.savez_compressed(path, **out)


def load_npz(path: str):
  z = np.load(path, allow_pickle=False)
  m = SimpleNamespace(opt=SimpleNamespace(), stat=SimpleNamespace(), names=SimpleNamespace())
  for k in z.files:
    v = z[k]
    tgt, name = m, k
    if k.startswith("vis.headlight."):
      if not hasattr(m, "vis"):
        m.vis = SimpleNamespace(headlight=SimpleNamespace())
      tgt, name = m.vis.headlight, k[len("vis.headlight."):]
      setattr(tgt, name, v.item() if v.ndim == 0 else v)
      continue
    if "." in k:
      grp, name = k.split(".", 1)
      tgt = getattr(m, grp)
    if grp_is_names(k):
      v = [str(s) for s in v.tolist()]
    elif v.ndim == 0:
      v = v.item()
    setattr(tgt, name, v)
  if not hasattr(m, "D_rownnz"):  # files written before the compiler stored the D-structure
    d_structure(m)
  return m


def grp_is_names(k: str) -> bool:
  return k.startswith("names.")


def load_any(path: str):
  """Load a model from .xml (compile) or .npz (precompiled)."""
  return load_npz(path) if path.endswith(".npz") else load(path)
