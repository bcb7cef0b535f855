"""Host <-> device conversion: put_model, make_data, put_data, reset_data.

Mirrors /root/reference/mujoco_warp/_src/io.py (put_model :259, make_data :1680, put_data :1890, reset_data :2435):
same signatures, same Model/Data field names and world-major layout, `torch.Tensor` as the device-array container.
`mjm` is either a real `mujoco.MjModel` (when that package is importable) or the object produced by
`mujoco_warp_b200.mjcf.load` (MjModel-named numpy attributes); fields are copied by name exactly like io.py:426.

Derived index tables are recomputed here for the warp-per-world kernels (tree levels, child lists, CSR entry rows,
symmetric gather tables for M*v, per-tree factor offsets, filtered NXN pairs, limited-joint list ...).
"""

from __future__ import annotations

import weakref

import numpy as np
import torch

from . import _lib
from . import constants as C
from . import mjcf
from . import types

_FLOAT_FIELDS = [
  "qpos0", "qpos_spring", "body_pos", "body_quat", "body_ipos", "body_iquat", "body_mass", "body_subtreemass",
  "body_inertia", "body_invweight0", "body_gravcomp", "jnt_pos", "jnt_axis", "jnt_stiffness", "jnt_range", "jnt_margin", "jnt_solref",
  "jnt_solimp", "jnt_actfrcrange", "dof_armature", "dof_damping", "dof_invweight0", "dof_frictionloss", "dof_solref",
  "dof_solimp", "geom_size", "geom_aabb", "geom_rbound", "geom_pos", "geom_quat", "geom_friction", "geom_margin",
  "geom_gap", "geom_solmix", "geom_solref", "geom_solimp", "actuator_gear", "actuator_gainprm", "actuator_biasprm",
  "actuator_ctrlrange", "actuator_forcerange", "cam_pos", "cam_quat", "cam_poscom0", "cam_pos0", "cam_mat0",
  "light_pos", "light_dir", "light_poscom0", "light_pos0", "light_dir0", "site_pos", "site_quat",
]
_INT_FIELDS = [
  "body_parentid", "body_rootid", "body_weldid", "body_mocapid", "body_jntnum", "body_jntadr", "body_dofnum", "body_dofadr",
  "jnt_type", "jnt_qposadr", "jnt_dofadr", "jnt_bodyid", "jnt_actfrclimited", "jnt_actgravcomp",
  "dof_bodyid", "dof_jntid", "dof_parentid", "M_rownnz", "M_rowadr", "M_colind", "tree_dofadr", "tree_dofnum",
  "geom_type", "geom_condim", "geom_bodyid", "geom_priority",
  "actuator_trnid", "actuator_gaintype", "actuator_biastype", "actuator_ctrllimited", "actuator_forcelimited",
  "cam_mode", "cam_bodyid", "cam_targetbodyid", "light_mode", "light_bodyid", "light_targetbodyid", "site_bodyid",
]
_TENDON_FLOATS = (("tendon_range", 2), ("tendon_margin", 1), ("tendon_stiffness", 1), ("tendon_damping", 1), ("tendon_frictionloss", 1), ("tendon_lengthspring", 2),
                  ("tendon_length0", 1), ("tendon_invweight0", 1), ("tendon_solref_lim", 2), ("tendon_solimp_lim", 5), ("tendon_solref_fri", 2), ("tendon_solimp_fri", 5), ("tendon_actfrcrange", 2))
# float fields outside _FLOAT_FIELDS that carry the reference's `*` leading dimension as well
_BATCHABLE_EXTRA = ("eq_solref", "eq_solimp", "eq_data", "pair_friction", "pair_solref", "pair_solreffriction", "pair_solimp", "pair_margin", "pair_gap",
                    "actuator_dynprm", "actuator_actrange", "geom_rgba", "mat_rgba", "actuator_acc0", "actuator_lengthrange") + tuple(n for n, _ in _TENDON_FLOATS)
# the renderer's float Model fields that carry the reference's `*` leading dimension (types.py cam_fovy ... mat_emission)
_RENDER_FLOATS = ("cam_fovy", "cam_intrinsic", "light_attenuation", "light_cutoff", "light_exponent", "light_ambient", "light_diffuse", "light_specular",
                  "mat_specular", "mat_shininess", "mat_emission")
# per-world float fields the magnetometer and camprojection sensors read (types.py opt.magnetic, cam_fovy, cam_intrinsic)
_SENSOR_BATCHED = ("magnetic", "cam_fovy", "cam_intrinsic")
# sensor types k_sensor runs in its EXTRA build only, with the object type each reads and its reference object's (None: none)
_EXTRA_SENSORS = {
  C.SENS_MAGNETOMETER: ((C.OBJ_SITE,), None), C.SENS_CAMPROJECTION: ((C.OBJ_SITE,), (C.OBJ_CAMERA,)),
  C.SENS_INSIDESITE: ((C.OBJ_BODY, C.OBJ_XBODY, C.OBJ_GEOM, C.OBJ_SITE, C.OBJ_CAMERA), (C.OBJ_SITE,)),
  **{t: ((C.OBJ_TENDON,), None) for t in (C.SENS_TENDONLIMITPOS, C.SENS_TENDONLIMITVEL, C.SENS_TENDONLIMITFRC, C.SENS_TENDONACTFRC)},
}
_SIZES = ["nq", "nv", "nu", "na", "nbody", "njnt", "ngeom", "nsite", "ncam", "nlight", "ntree", "nkey", "nmocap", "neq", "ntendon", "nflex"]

_SUPPORTED_PAIRS = {
  (C.GEOM_PLANE, C.GEOM_SPHERE), (C.GEOM_PLANE, C.GEOM_CAPSULE), (C.GEOM_SPHERE, C.GEOM_SPHERE),
  (C.GEOM_SPHERE, C.GEOM_CAPSULE), (C.GEOM_CAPSULE, C.GEOM_CAPSULE),
  # box / cylinder / ellipsoid primitives (collision_driver.py:47-81: the pairs the reference routes to primitive functions)
  (C.GEOM_PLANE, C.GEOM_ELLIPSOID), (C.GEOM_PLANE, C.GEOM_CYLINDER), (C.GEOM_PLANE, C.GEOM_BOX),
  (C.GEOM_SPHERE, C.GEOM_CYLINDER), (C.GEOM_SPHERE, C.GEOM_BOX), (C.GEOM_CAPSULE, C.GEOM_BOX),
  (C.GEOM_PLANE, C.GEOM_MESH),  # plane_convex (collision_primitive.py:52), in the mesh build of the collision kernel
}
# pairs the reference sends to GJK / EPA (collision_driver.py:47-81) that are built here: analytic convex geoms, single contact
_CONVEX_PAIRS = {
  (C.GEOM_SPHERE, C.GEOM_ELLIPSOID), (C.GEOM_CAPSULE, C.GEOM_ELLIPSOID), (C.GEOM_CAPSULE, C.GEOM_CYLINDER), (C.GEOM_ELLIPSOID, C.GEOM_ELLIPSOID),
  (C.GEOM_ELLIPSOID, C.GEOM_CYLINDER), (C.GEOM_ELLIPSOID, C.GEOM_BOX), (C.GEOM_CYLINDER, C.GEOM_CYLINDER), (C.GEOM_CYLINDER, C.GEOM_BOX),
  # mesh geoms (hull-vertex support function, mesh multi-contact): collision_gjk.py:116, collision_convex.py:1190
  (C.GEOM_SPHERE, C.GEOM_MESH), (C.GEOM_CAPSULE, C.GEOM_MESH), (C.GEOM_ELLIPSOID, C.GEOM_MESH), (C.GEOM_CYLINDER, C.GEOM_MESH),
  (C.GEOM_BOX, C.GEOM_MESH), (C.GEOM_MESH, C.GEOM_MESH),
}


def _require_cuda():
  if not torch.cuda.is_available():
    raise RuntimeError("mujoco_warp_b200 runs its step path on a CUDA (sm_90a) device only; no CPU fallback exists")
  return torch.device("cuda", torch.cuda.current_device())


def is_sparse(mjm) -> bool:
  """io.py:153-160."""
  jac = getattr(mjm.opt, "jacobian", C.JAC_AUTO)
  if jac == C.JAC_AUTO:
    return mjm.nv > 32
  return jac == C.JAC_SPARSE


def _get_padded_sizes(nv: int, njmax: int, sparse: bool, tile_size: int = 16, augment_cholesky: bool = False):
  """io.py:1268-1275."""

  def round_up(x, m):
    return ((x + m - 1) // m) * m

  njmax_padded = round_up(njmax, tile_size)
  nv_padded = round_up(nv + int(augment_cholesky), tile_size) if (sparse or nv > 32) else round_up(nv, 4)
  return njmax_padded, nv_padded


def _default_size(base: float) -> int:
  valid = (2 + (np.arange(19) % 2)) * (2 ** (np.arange(19) // 2 + 3))
  return int(base) if base > valid[-1] else int(valid[np.searchsorted(valid, base)])


def _default_nconmax(mjm) -> int:
  return _default_size(45)  # io.py:1284-1297 without hfield/flex/sdf terms


def _default_njmax(mjm) -> int:
  return _default_size(53)  # io.py:1299-1311


def _np(mjm, name):
  return np.asarray(getattr(mjm, name))


def derive_tables(mjm) -> dict:
  """Index tables for the kernels (host, numpy)."""
  nbody, nv, ngeom, njnt, nu = mjm.nbody, mjm.nv, mjm.ngeom, mjm.njnt, mjm.nu
  parent = _np(mjm, "body_parentid")
  t = {}
  # tree levels (reference body_tree, io.py:495-500) and child lists
  depth = np.zeros(nbody, dtype=np.int32)
  for b in range(1, nbody):
    depth[b] = depth[parent[b]] + 1
  nlevel = int(depth.max()) + 1
  order = np.argsort(depth, kind="stable").astype(np.int32)
  t["level_body"] = order
  t["level_adr"] = np.searchsorted(depth[order], np.arange(nlevel + 1)).astype(np.int32)
  t["nlevel"] = nlevel
  t["body_tree"] = [order[t["level_adr"][l] : t["level_adr"][l + 1]] for l in range(nlevel)]
  children = [[] for _ in range(nbody)]
  for b in range(1, nbody):
    children[parent[b]].append(b)
  t["body_childadr"] = np.concatenate([[0], np.cumsum([len(c) for c in children])]).astype(np.int32)
  t["body_childid"] = np.array([c for cs in children for c in cs] + ([0] if nbody == 1 else []), dtype=np.int32)
  # CSR entry rows (reference M_hinit_i) and symmetric gather tables (reference M_mulm_*, io.py:1029-1050)
  rownnz, rowadr, colind = _np(mjm, "M_rownnz"), _np(mjm, "M_rowadr"), _np(mjm, "M_colind")
  nC = int(rownnz.sum())
  entry_row = np.zeros(nC, dtype=np.int32)
  gather = [[] for _ in range(nv)]
  for i in range(nv):
    for k in range(rownnz[i]):
      e = rowadr[i] + k
      j = colind[e]
      entry_row[e] = i
      gather[i].append((j, e))
      if j != i:
        gather[j].append((i, e))
  t["nC"] = nC
  t["M_entry_row"] = entry_row
  t["mulm_rowadr"] = np.concatenate([[0], np.cumsum([len(g) for g in gather])]).astype(np.int32)
  t["mulm_col"] = np.array([c for g in gather for c, _ in sorted(g)], dtype=np.int32)
  t["mulm_madr"] = np.array([e for g in gather for _, e in sorted(g)], dtype=np.int32)
  # per-tree dense factor blocks (io.py:173-211; every block <= M_BLOCK_DENSE_MAX uses the dense path here)
  tadr, tnum = _np(mjm, "tree_dofadr"), _np(mjm, "tree_dofnum")
  off, qadr = 0, []
  for n in tnum:
    qadr.append(off)
    off += int(n) * int(n)
  t["tree_qLDadr"] = np.array(qadr if qadr else [0], dtype=np.int32)
  t["qld_total"] = off
  t["maxtree"] = int(tnum.max()) if len(tnum) else 0
  # longest dof chain (a dof and its ancestors): bounds the nonzeros of one constraint Jacobian row (two bodies' chains)
  dpar = _np(mjm, "dof_parentid")
  depth = np.zeros(max(nv, 1), dtype=np.int64)
  for i in range(nv):
    depth[i] = 1 + (depth[dpar[i]] if dpar[i] >= 0 else 0)
  t["max_dof_chain"] = int(depth.max()) if nv else 0
  blk = np.zeros(max(nv, 1), dtype=np.int32)
  for a, n, q in zip(tadr, tnum, qadr):
    blk[a : a + n] = q
  t["qLD_block_adr"] = blk
  # dof-ancestor mask (io.py:536-549)
  anc = np.zeros((nbody, nv), dtype=np.int32)
  dofnum, dofadr, dparent = _np(mjm, "body_dofnum"), _np(mjm, "body_dofadr"), _np(mjm, "dof_parentid")
  for bodyid in range(nbody):
    b = bodyid
    while b > 0 and dofnum[b] == 0:
      b = parent[b]
    if dofnum[b] == 0:
      continue
    d = dofadr[b] + dofnum[b] - 1
    while d >= 0:
      anc[bodyid, d] = 1
      d = dparent[d]
  t["body_isdofancestor"] = anc
  # filtered NXN geom pairs (io.py:551-640)
  filterparent = not (mjm.opt.disableflags & C.DSBL_FILTERPARENT)
  g1, g2 = np.triu_indices(ngeom, k=1)
  gb = _np(mjm, "geom_bodyid")
  weld = _np(mjm, "body_weldid")
  b1, b2 = gb[g1], gb[g2]
  w1, w2 = weld[b1], weld[b2]
  wp1, wp2 = weld[parent[w1]], weld[parent[w2]]
  ct, ca = _np(mjm, "geom_contype"), _np(mjm, "geom_conaffinity")
  mask = ((ct[g1] & ca[g2]) | (ct[g2] & ca[g1])).astype(bool)
  self_col = w1 == w2
  parent_child = filterparent & (w1 != 0) & (w2 != 0) & ((w1 == wp2) | (w2 == wp1))
  excl_sig = np.asarray(getattr(mjm, "exclude_signature", np.zeros(0, dtype=np.int64)))
  exclude = np.isin((b1.astype(np.int64) << 16) + b2, excl_sig)
  pairid = -np.ones(len(g1), dtype=np.int32)
  pairid[~(mask & ~self_col & ~parent_child & ~exclude)] = -2
  for i in range(int(getattr(mjm, "npair", 0))):  # explicit <pair>s override the filters (reference io.py:577-583)
    a, b = sorted((int(mjm.pair_geom1[i]), int(mjm.pair_geom2[i])))
    pairid[(a * (2 * ngeom - a - 3)) // 2 + b - 1] = i
  include = pairid > -2
  t["nxn_geom_pair"] = np.stack((g1, g2), axis=1).astype(np.int32)
  t["nxn_pairid"] = np.stack((pairid, -np.ones(len(g1), dtype=np.int32)), axis=1).astype(np.int32)
  t["nxn_geom_pair_filtered"] = t["nxn_geom_pair"][include]
  t["nxn_pairid_filtered"] = t["nxn_pairid"][include]
  gt = _np(mjm, "geom_type")

  def trid(i, j):
    i, j = (j, i) if j < i else (i, j)
    return (i * (2 * C.NGEOMTYPES - i - 1)) // 2 + j

  t["has_convex_pair"] = 0
  nboxbox = nconvex = 0
  counts = np.zeros(C.NGEOMTYPES * (C.NGEOMTYPES + 1) // 2, dtype=int)
  for a, b in t["nxn_geom_pair_filtered"]:
    counts[trid(gt[a], gt[b])] += 1
    key = (min(gt[a], gt[b]), max(gt[a], gt[b]))
    if key == (C.GEOM_BOX, C.GEOM_BOX):
      # box-box is a primitive pair only with native CCD disabled (collision_driver.py:868-870); otherwise GJK / EPA + multi-contact
      if not (int(mjm.opt.disableflags) & C.DSBL_NATIVECCD):
        t["has_convex_pair"] = 1
        nboxbox += 1
        nconvex += 1
    elif key in _CONVEX_PAIRS:
      t["has_convex_pair"] = 1
      nconvex += 1
    elif key not in _SUPPORTED_PAIRS:
      raise NotImplementedError(f"collision between geom types {key} is not implemented in this version (supported: {sorted(_SUPPORTED_PAIRS | _CONVEX_PAIRS)})")
  t["geom_pair_type_count"] = tuple(int(c) for c in counts)
  # EPA gets 16 iterations when every convex pair of the model is box-box (collision_convex.py:1223)
  t["epa_iterations"] = 16 if nboxbox == nconvex else int(getattr(mjm.opt, "ccd_iterations", 35))
  if nboxbox:  # reference io.py:685-712: native box-box CCD does not support margins
    for a, b in t["nxn_geom_pair_filtered"]:
      if gt[a] == C.GEOM_BOX and gt[b] == C.GEOM_BOX and (float(mjm.geom_margin[a]) != 0.0 or float(mjm.geom_margin[b]) != 0.0):
        raise NotImplementedError("box-box geom pair has non-zero margin with NATIVECCD enabled. Set margin to 0 or disable NATIVECCD.")
    for i in range(int(getattr(mjm, "npair", 0))):
      if gt[mjm.pair_geom1[i]] == C.GEOM_BOX and gt[mjm.pair_geom2[i]] == C.GEOM_BOX and float(mjm.pair_margin[i]) != 0.0:
        raise NotImplementedError("box-box contact pair has non-zero margin with NATIVECCD enabled. Set margin to 0 or disable NATIVECCD.")
  # constraint source lists
  jt = _np(mjm, "jnt_type")
  lim = np.asarray(_np(mjm, "jnt_limited")).astype(bool)
  t["jnt_limited_slide_hinge_adr"] = np.nonzero(lim & ((jt == C.JNT_SLIDE) | (jt == C.JNT_HINGE)))[0].astype(np.int32)
  t["jnt_limited_ball_adr"] = np.nonzero(lim & (jt == C.JNT_BALL))[0].astype(np.int32)
  t["dof_fricloss_adr"] = np.nonzero(_np(mjm, "dof_frictionloss") > 0)[0].astype(np.int32)
  # constant sparsity of the actuator moment (joint transmission)
  trnid = _np(mjm, "actuator_trnid").reshape(nu, 2)
  jdof = _np(mjm, "jnt_dofadr")
  nnz_of = {C.JNT_FREE: 6, C.JNT_BALL: 3, C.JNT_SLIDE: 1, C.JNT_HINGE: 1}
  rn, ra, ci = [], [], []
  for a in range(nu):
    trn = int(_np(mjm, "actuator_trntype")[a])
    if trn == C.TRN_TENDON:  # the moment row is the tendon's Jacobian row (smooth.py:2508-2525)
      t_ = int(trnid[a, 0])
      adr_, n = int(_np(mjm, "ten_J_rowadr")[t_]), int(_np(mjm, "ten_J_rownnz")[t_])
      ra.append(len(ci)); rn.append(n)
      ci.extend(int(x) for x in _np(mjm, "ten_J_colind")[adr_ : adr_ + n])
      continue
    if trn != C.TRN_JOINT:
      raise NotImplementedError("only joint and tendon transmissions are implemented")
    jtype = int(jt[trnid[a, 0]])
    if jtype == C.JNT_BALL:
      raise NotImplementedError("ball-joint actuator transmission is not implemented")
    n = nnz_of[jtype]
    ra.append(len(ci))
    rn.append(n)
    ci.extend(range(jdof[trnid[a, 0]], jdof[trnid[a, 0]] + n))
  t["moment_rownnz0"] = np.array(rn if rn else [0], dtype=np.int32)
  t["moment_rowadr0"] = np.array(ra if ra else [0], dtype=np.int32)
  t["moment_colind0"] = np.array(ci if ci else [0], dtype=np.int32)
  t["nJmom"] = len(ci)
  # reverse table: for every dof the (actuator, moment index) pairs that act on it, in actuator order
  rev = [[] for _ in range(nv)]
  for a in range(nu):
    for k in range(rn[a]):
      rev[ci[ra[a] + k]].append((a, ra[a] + k))
  t["dofact_adr"] = np.concatenate([[0], np.cumsum([len(r) for r in rev])]).astype(np.int32)
  t["dofact_act"] = np.array([a for r in rev for a, _ in r] or [0], dtype=np.int32)
  t["dofact_mom"] = np.array([i for r in rev for _, i in r] or [0], dtype=np.int32)
  nmaxcondim = int(_np(mjm, "geom_condim").max()) if ngeom else 1
  if getattr(mjm, "npair", 0):
    nmaxcondim = max(nmaxcondim, int(np.asarray(mjm.pair_dim).max()))
  t["nmaxcondim"] = nmaxcondim
  t["nmaxpyramid"] = max(1, 2 * (nmaxcondim - 1))
  # energy sensors (reference io.py:893-894): k_energy writes their slots, k_sensor skips them
  stype = np.asarray(mjm.sensor_type).reshape(-1) if int(getattr(mjm, "nsensor", 0)) else np.zeros(0, dtype=int)
  t["sensor_energy_adr"] = np.nonzero(np.isin(stype, (C.SENS_E_POTENTIAL, C.SENS_E_KINETIC)))[0].astype(np.int32)
  t["sensor_e_potential"] = bool((stype == C.SENS_E_POTENTIAL).any())
  t["sensor_e_kinetic"] = bool((stype == C.SENS_E_KINETIC).any())
  return t


_COLLISION_SENSORS = (C.SENS_GEOMDIST, C.SENS_GEOMNORMAL, C.SENS_GEOMFROMTO)


def _sensor_collision_tables(mjm, t) -> dict:
  """The geom pairs of the distance / normal / fromto sensors (reference io.py:586-628), kept apart from nxn_pairid.

  sensor_collision_start_adr: for every (sensor, geom1, geom2) in the sensors' loop order (body sensors expand over body_geomadr /
  body_geomnum), the index of that geom pair among the nsensorcollision unique pairs, numbered in first-seen order.  The kernel's own tables:
  sensor_collision_pair (nsensorcollision, 4): both geoms in the order the narrowphase takes them (geom types ascending) and the pair's
  explicit <pair> id or -1 (its margin), and the pair's rank among the pairs that run GJK / EPA or -1 (its scratch slot); sensor_collision_id / _adr: the collision sensors and their first entry of the start_adr list;
  sensor_collision_flip: whether an entry's geom1 comes second in narrowphase order (the reduction then reverses normal and fromto)."""
  nsensor, ngeom = int(getattr(mjm, "nsensor", 0)), int(mjm.ngeom)
  stype = np.asarray(mjm.sensor_type).reshape(-1) if nsensor else np.zeros(0, dtype=int)
  sensors = np.nonzero(np.isin(stype, _COLLISION_SENSORS))[0]
  gt, gadr, gnum = _np(mjm, "geom_type"), _np(mjm, "body_geomadr"), _np(mjm, "body_geomnum")

  def geoms(objtype, objid):
    return range(int(gadr[objid]), int(gadr[objid] + gnum[objid])) if objtype == C.OBJ_BODY else range(int(objid), int(objid) + 1)

  nativeccd = not (int(mjm.opt.disableflags) & C.DSBL_NATIVECCD)
  is_ccd = lambda key: key in _CONVEX_PAIRS or (key == (C.GEOM_BOX, C.GEOM_BOX) and nativeccd)
  nccd = 0
  first = {}  # upper-triangular pair index -> collision id
  pairs, start_adr, flip, adr = [], [], [], []
  for s in sensors:
    adr.append(len(start_adr))
    for g1 in geoms(int(mjm.sensor_objtype[s]), int(mjm.sensor_objid[s])):
      for g2 in geoms(int(mjm.sensor_reftype[s]), int(mjm.sensor_refid[s])):
        a, b = min(g1, g2), max(g1, g2)
        idx = (a * (2 * ngeom - a - 3)) // 2 + b - 1
        if idx not in first:
          key = (min(gt[a], gt[b]), max(gt[a], gt[b]))
          if a == b or not (key in _SUPPORTED_PAIRS or key in _CONVEX_PAIRS or key == (C.GEOM_BOX, C.GEOM_BOX)):
            names = ("plane", "hfield", "sphere", "capsule", "ellipsoid", "cylinder", "box", "mesh", "sdf")
            raise NotImplementedError(f"collision sensor {s}: no collider for the geom types {names[key[0]]} and {names[key[1]]} (geoms {a} and {b})")
          first[idx] = len(pairs)
          lo, hi = (b, a) if gt[a] > gt[b] else (a, b)
          pairs.append((lo, hi, int(t["nxn_pairid"][idx, 0]) if t["nxn_pairid"][idx, 0] >= 0 else -1, nccd if is_ccd(key) else -1))
          nccd += is_ccd(key)
        start_adr.append(first[idx])
        flip.append(int(gt[g1] > gt[g2] or (gt[g1] == gt[g2] and g1 > g2)))
  adr.append(len(start_adr))
  # EPA iterations as the reference counts them over its pair list, which includes the sensor pairs (collision_convex.py:1223)
  convex = [(min(gt[a], gt[b]), max(gt[a], gt[b])) for a, b in list(t["nxn_geom_pair_filtered"]) + [p[:2] for p in pairs]]
  convex = [k for k in convex if is_ccd(k)]
  epa = 16 if all(k == (C.GEOM_BOX, C.GEOM_BOX) for k in convex) else int(getattr(mjm.opt, "ccd_iterations", 35))
  i32 = lambda x, shape: np.asarray(x, dtype=np.int32).reshape(shape)
  return dict(nsensorcollision=len(pairs), sensor_collision_start_adr=i32(start_adr, -1), sensor_collision_pair=i32(pairs, (len(pairs), 4)),
              sensor_collision_id=i32(sensors, -1), sensor_collision_adr=i32(adr, -1), sensor_collision_flip=i32(flip, -1), sensor_collision_epa_iterations=epa,
              nsensorcollision_ccd=nccd)


def _has_fluid(o) -> bool:
  """io.py:471: the model has fluid forces."""
  return bool(np.any(np.asarray(getattr(o, "wind", 0.0)) != 0.0) or float(getattr(o, "density", 0.0)) > 0.0 or float(getattr(o, "viscosity", 0.0)) > 0.0)


def _validate(mjm):
  """Feature checks in the spirit of io.py:284-363: fail loudly on anything the kernels do not cover."""
  o = mjm.opt
  if o.integrator not in (C.INT_EULER, C.INT_RK4, C.INT_IMPLICIT, C.INT_IMPLICITFAST):
    raise NotImplementedError(f"unknown integrator {o.integrator}")
  if o.integrator == C.INT_IMPLICIT and 18 * mjm.nbody * 32 * 4 > 200 * 1024:
    raise NotImplementedError(f"implicit integrator: the velocity-derivative scratch of {mjm.nbody} bodies exceeds one block's shared memory (use implicitfast)")
  if o.cone not in (C.CONE_PYRAMIDAL, C.CONE_ELLIPTIC):
    raise NotImplementedError(f"unknown friction cone {o.cone}")
  if o.solver not in (C.SOL_NEWTON, C.SOL_CG):
    raise NotImplementedError("only the Newton and CG solvers are implemented in this version (no PGS)")
  # features the kernels do not evaluate must fail here, not silently change the simulation (ADVICE r1)
  if _has_fluid(o) and o.integrator == C.INT_IMPLICIT:
    raise NotImplementedError("fluid forces (opt.density / viscosity / wind) with the implicit integrator are not implemented (use implicitfast, Euler or RK4)")
  if int(getattr(o, "noslip_iterations", 0)) > 0:
    raise NotImplementedError("the noslip solver (opt.noslip_iterations > 0) is not implemented")
  unsupported_enable = int(o.enableflags) & (C.ENBL_OVERRIDE | C.ENBL_FWDINV | C.ENBL_SLEEP)
  if unsupported_enable:
    names = [n for n, b in C.ENABLE_FLAGS.items() if unsupported_enable & b]
    raise NotImplementedError(f"enable flag(s) {names} are not implemented (contact override, fwdinv, sleeping)")
  if getattr(mjm, "nu", 0):
    gt, bt = np.asarray(mjm.actuator_gaintype), np.asarray(mjm.actuator_biastype)
    if not np.isin(gt, (C.GAIN_FIXED, C.GAIN_AFFINE, C.GAIN_MUSCLE)).all():
      raise NotImplementedError(f"actuator gain type(s) {sorted(set(gt[~np.isin(gt, (C.GAIN_FIXED, C.GAIN_AFFINE, C.GAIN_MUSCLE))].tolist()))} are not implemented (fixed, affine and muscle are)")
    if not np.isin(bt, (C.BIAS_NONE, C.BIAS_AFFINE, C.BIAS_MUSCLE)).all():
      raise NotImplementedError(f"actuator bias type(s) {sorted(set(bt[~np.isin(bt, (C.BIAS_NONE, C.BIAS_AFFINE, C.BIAS_MUSCLE))].tolist()))} are not implemented (none, affine and muscle are)")
    dyn = np.asarray(getattr(mjm, "actuator_dyntype", np.zeros(mjm.nu)))
    if not np.isin(dyn, (C.DYN_NONE, C.DYN_INTEGRATOR, C.DYN_FILTER, C.DYN_FILTEREXACT, C.DYN_MUSCLE)).all():
      raise NotImplementedError(f"actuator dynamics type(s) {sorted(set(dyn[~np.isin(dyn, (0, 1, 2, 3, 4))].tolist()))} are not implemented (none, integrator, filter, filterexact, muscle are)")
    muscle = np.isin(gt, (C.GAIN_MUSCLE,)) | np.isin(bt, (C.BIAS_MUSCLE,))
    if muscle.any():
      # the muscle curves divide by the optimum length (lengthrange[1] - lengthrange[0]) / (range[1] - range[0]) (util_misc.py:500)
      lr = np.asarray(getattr(mjm, "actuator_lengthrange", np.zeros((mjm.nu, 2))), dtype=np.float64).reshape(mjm.nu, 2)
      bad = np.nonzero(muscle & ~(lr[:, 0] < lr[:, 1]))[0]
      if len(bad):
        raise ValueError(f"muscle actuator(s) {bad.tolist()}: actuator_lengthrange must satisfy lengthrange[0] < lengthrange[1] (got {lr[bad].tolist()})")
  for n in ("dof_dampingpoly", "jnt_stiffnesspoly"):
    if hasattr(mjm, n) and np.any(np.asarray(getattr(mjm, n)) != 0):
      raise NotImplementedError(f"{n}: polynomial stiffness / damping is not implemented")
  gt_ = np.asarray(mjm.geom_type)
  if np.isin(gt_, (C.GEOM_HFIELD, C.GEOM_SDF)).any():
    raise NotImplementedError("height-field / SDF geoms are not implemented (plane, sphere, capsule, ellipsoid, cylinder, box and mesh geoms are)")
  if mjm.nv > 128:
    # the dense per-world Hessian and its factor live in one warp's shared memory; make_data reports the exact per-kernel need
    raise NotImplementedError("nv > 128 is not supported in this version (dense per-world Jacobian/Hessian in shared memory)")
  if getattr(mjm, "ntendon", 0):
    if not np.all(np.asarray(mjm.wrap_type) == C.WRAP_JOINT):
      raise NotImplementedError("spatial tendons (site / geom / pulley wraps) are not implemented; fixed tendons are")
    for n in ("tendon_armature", "tendon_stiffnesspoly", "tendon_dampingpoly"):
      if hasattr(mjm, n) and np.any(np.asarray(getattr(mjm, n)) != 0):
        raise NotImplementedError(f"{n} is not implemented")
  for n in ("nflex",):
    if getattr(mjm, n, 0):
      raise NotImplementedError(f"{n} > 0 is not supported in this version")
  if getattr(mjm, "neq", 0):
    et, ot = np.asarray(mjm.eq_type), np.asarray(mjm.eq_objtype)
    if not np.isin(et, (C.EQ_CONNECT, C.EQ_WELD, C.EQ_JOINT, C.EQ_TENDON)).all():
      raise NotImplementedError("only connect / weld / joint / tendon equality constraints are implemented")
    if (ot[np.isin(et, (C.EQ_CONNECT, C.EQ_WELD))] != C.OBJ_BODY).any():
      raise NotImplementedError("site-based connect / weld equality constraints are not implemented")
  if int(np.asarray(mjm.tree_dofnum).max(initial=0)) > 64:
    raise NotImplementedError("kinematic trees with more than 64 dofs are not supported (dense per-tree Cholesky)")
  _validate_history(mjm)


def history_fields(mjm) -> dict:
  """The delay / history fields of an MjModel-like object (reference types.py:1306-1329), with empty defaults for models saved
  before they existed."""
  nu, ns = int(mjm.nu), int(getattr(mjm, "nsensor", 0))
  g = lambda n, shape, dt: np.asarray(getattr(mjm, n, np.zeros(shape)), dtype=dt).reshape(shape)
  return dict(
    actuator_history=g("actuator_history", (nu, 2), np.int32), actuator_historyadr=np.asarray(getattr(mjm, "actuator_historyadr", -np.ones(nu)), dtype=np.int32).reshape(nu),
    actuator_delay=g("actuator_delay", (nu,), np.float64), sensor_history=g("sensor_history", (ns, 2), np.int32),
    sensor_historyadr=np.asarray(getattr(mjm, "sensor_historyadr", -np.ones(ns)), dtype=np.int32).reshape(ns), sensor_delay=g("sensor_delay", (ns,), np.float64),
    sensor_interval=g("sensor_interval", (ns, 2), np.float64), nhistory=int(getattr(mjm, "nhistory", 0)),
  )


def _contact_sensor_intprm(mjm) -> np.ndarray:
  """sensor_intprm (nsensor, 3) of a model, after checking every <contact> sensor's entries: known data bits and reduce, num >= 1, dim
  equal to num times the slot size, and objects of the kinds and ranges the compiler emits.  ValueError naming the sensor otherwise."""
  ns = int(getattr(mjm, "nsensor", 0))
  stype = np.asarray(mjm.sensor_type).reshape(ns) if ns else np.zeros(0, dtype=int)
  intprm = np.asarray(getattr(mjm, "sensor_intprm", np.zeros((ns, 3))), dtype=np.int64).reshape(ns, -1)[:, :3] if ns else np.zeros((0, 3))
  names = list(getattr(getattr(mjm, "names", None), "sensor", None) or [f"sensor{i}" for i in range(ns)])
  counts = {C.OBJ_SITE: int(getattr(mjm, "nsite", 0)), C.OBJ_GEOM: int(mjm.ngeom), C.OBJ_BODY: int(mjm.nbody), C.OBJ_XBODY: int(mjm.nbody)}
  for s in np.nonzero(stype == C.SENS_CONTACT)[0]:
    what = f"contact sensor '{names[s]}'"
    dataspec, reduce, num = (int(x) for x in intprm[s])
    if dataspec < 1 or dataspec >= 1 << len(mjcf.CONTACT_DATA):
      raise ValueError(f"{what}: unknown data bits {dataspec:#x} (found force torque dist pos normal tangent are bits 0-6)")
    if not 0 <= reduce < len(mjcf.CONTACT_REDUCE):
      raise ValueError(f"{what}: unknown reduce {reduce} (expected 0 none, 1 mindist, 2 maxforce or 3 netforce)")
    if num < 1:
      raise ValueError(f"{what}: num must be >= 1, got {num}")
    if int(mjm.sensor_dim[s]) != num * mjcf.contact_slot_size(dataspec):
      raise ValueError(f"{what}: dim {int(mjm.sensor_dim[s])} is not num ({num}) x the slot size ({mjcf.contact_slot_size(dataspec)}) of its data")
    for side, kinds, typ, oid in ((1, (C.OBJ_SITE, C.OBJ_GEOM, C.OBJ_BODY, C.OBJ_XBODY), int(mjm.sensor_objtype[s]), int(mjm.sensor_objid[s])),
                                  (2, (C.OBJ_GEOM, C.OBJ_BODY, C.OBJ_XBODY), int(getattr(mjm, "sensor_reftype", np.zeros(ns))[s]), int(getattr(mjm, "sensor_refid", -np.ones(ns))[s]))):
      if typ == C.OBJ_UNKNOWN:
        continue
      if typ not in kinds:
        raise ValueError(f"{what}: side {side} has object type {typ}; expected none or one of {kinds}")
      if not 0 <= oid < counts[typ]:
        raise ValueError(f"{what}: side {side} names an unknown object (id {oid})")
  out = np.zeros((ns, 3), dtype=np.int32)
  contact = stype == C.SENS_CONTACT
  out[contact] = intprm[contact]
  return out


def _validate_extra_sensors(mjm):
  """Checks the object kinds and ids of the magnetometer / camprojection / insidesite / tendon sensors again, for models that did not come
  from this package's compiler.  Returns whether the model has one (k_sensor's EXTRA build)."""
  ns = int(getattr(mjm, "nsensor", 0))
  stype = np.asarray(mjm.sensor_type).reshape(ns) if ns else np.zeros(0, dtype=int)
  counts = {C.OBJ_BODY: int(mjm.nbody), C.OBJ_XBODY: int(mjm.nbody), C.OBJ_GEOM: int(mjm.ngeom), C.OBJ_SITE: int(getattr(mjm, "nsite", 0)),
            C.OBJ_CAMERA: int(getattr(mjm, "ncam", 0)), C.OBJ_TENDON: int(getattr(mjm, "ntendon", 0))}
  names = getattr(getattr(mjm, "names", None), "sensor", None)
  found = False
  for s in range(ns):
    if int(stype[s]) not in _EXTRA_SENSORS:
      continue
    found = True
    what = f"sensor {s}" + (f" ('{names[s]}')" if names is not None and s < len(names) else "")
    for side, kinds, typ, oid in (("object", _EXTRA_SENSORS[int(stype[s])][0], int(mjm.sensor_objtype[s]), int(mjm.sensor_objid[s])),
                                  ("reference", _EXTRA_SENSORS[int(stype[s])][1], int(getattr(mjm, "sensor_reftype", np.zeros(ns))[s]),
                                   int(getattr(mjm, "sensor_refid", -np.ones(ns))[s]))):
      if kinds is None:
        continue
      if typ not in kinds:
        raise ValueError(f"{what}: {side} type {typ}; expected one of {kinds}")
      if not 0 <= oid < counts[typ]:
        raise ValueError(f"{what}: {side} names an unknown object (id {oid})")
  return found


def _validate_history(mjm):
  """Refuses, by name, delays and intervals the history buffers would not honour: the reference silently reads the undelayed value
  when nsample is 0 (history.py:380), and negative sizes / times have no meaning."""
  h = history_fields(mjm)
  names = getattr(getattr(mjm, "names", None), "__dict__", {})
  for kind, n in (("actuator", int(mjm.nu)), ("sensor", int(getattr(mjm, "nsensor", 0)))):
    hist, delay = h[kind + "_history"], h[kind + "_delay"]
    period = h["sensor_interval"][:, 0] if kind == "sensor" else np.zeros(n)
    for i in range(n):
      what = f"{kind} {i}" + (f" ('{names[kind][i]}')" if kind in names and i < len(names[kind]) else "")
      if hist[i, 0] < 0:
        raise ValueError(f"{what}: nsample must be >= 0, got {hist[i, 0]}")
      if hist[i, 1] not in (0, 1, 2):
        raise ValueError(f"{what}: interp must be 0 (zoh), 1 (linear) or 2 (cubic), got {hist[i, 1]}")
      if delay[i] < 0:
        raise ValueError(f"{what}: delay must be >= 0, got {delay[i]}")
      if period[i] < 0:
        raise ValueError(f"{what}: interval period must be >= 0, got {period[i]}")
      if hist[i, 0] == 0 and (delay[i] > 0 or period[i] > 0):
        field = "delay" if delay[i] > 0 else "interval"
        raise ValueError(f"{what}: {field} > 0 needs a history buffer (nsample > 0); with nsample = 0 it would be ignored")


def render_fields(mjm) -> dict:
  """The camera, light and material fields the renderer reads (MjModel names); models compiled before they existed get MuJoCo's
  defaults (perspective 45-degree cameras of resolution 1 x 1 without a sensor, spot lights of diffuse 0.7 / specular 0.3 that cast
  shadows, materials of specular 0.5 / shininess 0.5 without emission or texture).  mat_texid has MuJoCo's layout, one column per texture role."""
  nc, nl, nm = int(getattr(mjm, "ncam", 0)), int(getattr(mjm, "nlight", 0)), int(getattr(mjm, "nmat", 0))

  def g(name, n, shape, default, dt):
    v = getattr(mjm, name, None)
    return np.ascontiguousarray((np.broadcast_to(np.asarray(default), (n,) + shape) if v is None else np.asarray(v)).astype(dt).reshape((n,) + shape))

  return dict(
    cam_projection=g("cam_projection", nc, (), 0, np.int32), cam_fovy=g("cam_fovy", nc, (), 45.0, np.float64),
    cam_resolution=g("cam_resolution", nc, (2,), 1, np.int32), cam_sensorsize=g("cam_sensorsize", nc, (2,), 0.0, np.float64),
    cam_intrinsic=g("cam_intrinsic", nc, (4,), 0.0, np.float64),
    light_type=g("light_type", nl, (), 0, np.int32), light_castshadow=g("light_castshadow", nl, (), 1, np.int32), light_active=g("light_active", nl, (), 1, np.int32),
    light_attenuation=g("light_attenuation", nl, (3,), [1.0, 0.0, 0.0], np.float64), light_cutoff=g("light_cutoff", nl, (), 45.0, np.float64),
    light_exponent=g("light_exponent", nl, (), 10.0, np.float64), light_ambient=g("light_ambient", nl, (3,), 0.0, np.float64),
    light_diffuse=g("light_diffuse", nl, (3,), 0.7, np.float64), light_specular=g("light_specular", nl, (3,), 0.3, np.float64),
    mat_specular=g("mat_specular", nm, (), 0.5, np.float64), mat_shininess=g("mat_shininess", nm, (), 0.5, np.float64), mat_emission=g("mat_emission", nm, (), 0.0, np.float64),
    mat_texid=g("mat_texid", nm, (10,), -1, np.int32),  # (nmat, mjNTEXROLE)
  )


def _ptr_tensor(x: torch.Tensor) -> torch.Tensor:
  """A contiguous tensor with a valid device pointer (empty tables get a 1-element dummy)."""
  assert x.is_contiguous()
  if x.numel() == 0:
    return torch.zeros(1, dtype=x.dtype, device=x.device)
  return x


def put_model(mjm, batch_sizes=None) -> types.Model:
  """Creates a device Model from an MjModel-like object (reference io.py:259).

  batch_sizes: optional {field: n} for the float Model fields the reference marks with a `*` leading dimension (types.py:822-833):
  the field is allocated with n entries (each a copy of the model's value) and world w reads entry w % n -- write per-world values
  into `m.<field>` (in place, or by assigning a tensor with a different leading size) for domain randomisation."""
  batch_sizes = dict(batch_sizes or {})
  for name, size in batch_sizes.items():
    if name in ("actuator_delay", "sensor_delay"):
      raise ValueError(f"Model field {name!r} is shared by all worlds (the reference has no per-world delays); it cannot be batched.")
    if name not in _FLOAT_FIELDS and name not in _BATCHABLE_EXTRA and name not in _RENDER_FLOATS:
      raise ValueError(f"Model field {name!r} is not a batched array field.")
    if int(size) < 1:
      raise ValueError(f"batch_sizes[{name!r}] must be positive, got {size}.")
  dev = _require_cuda()
  L = _lib.lib()
  _validate(mjm)
  t = derive_tables(mjm)
  # The reference switches to a CSR constraint Jacobian for nv > 32 (io.py:153-160).  The kernels here always work on dense rows;
  # for a sparse model Data.efc carries the reference's CSR arrays (J_rownnz / J_rowadr / J_colind / J) written by k_efc_csr after
  # make_constraint, and the dense rows live in Data.efc.J_dense.
  sparse = is_sparse(mjm)
  m = types.Model()
  for n in _SIZES:
    setattr(m, n, int(getattr(mjm, n, 0)))
  m.nC = m.nM = t["nC"]
  m.nJmom = t["nJmom"]
  m.nmaxcondim, m.nmaxpyramid = t["nmaxcondim"], t["nmaxpyramid"]
  m.is_sparse = sparse
  m.nv_pad = _get_padded_sizes(m.nv, 0, False)[1]  # row stride of the dense working Jacobian
  m.qLD_block_total = t["qld_total"]
  m.geom_pair_type_count = t["geom_pair_type_count"]
  m.nbranch = int((t["body_childadr"][1:] - t["body_childadr"][:-1] == 0)[1:].sum()) if m.nbody > 1 else 0

  o = mjm.opt
  tol = max(float(o.tolerance), 1e-6)  # io.py:401 float32 clamp
  f32 = lambda x: torch.tensor(np.asarray(x, dtype=np.float32).reshape(1, *np.shape(x)), device=dev)
  m.opt = types.Option(
    timestep=f32(o.timestep), tolerance=f32(tol), ls_tolerance=f32(o.ls_tolerance), gravity=f32(np.asarray(o.gravity)),
    integrator=int(o.integrator), cone=int(o.cone), solver=int(o.solver), iterations=int(o.iterations), ls_iterations=int(o.ls_iterations),
    disableflags=int(o.disableflags), enableflags=int(o.enableflags), impratio_invsqrt=f32(1.0 / np.sqrt(o.impratio)),
    broadphase=types.BroadphaseType(int(getattr(o, "broadphase", 0))), broadphase_filter=int(getattr(o, "broadphase_filter", C.BF_PLANE | C.BF_SPHERE | C.BF_OBB)),
    graph_conditional=False, run_collision_detection=True, warn_overflow=False,
    # model constants here, one value for every world (the reference indexes them per world)
    density=f32(float(getattr(o, "density", 0.0))), viscosity=f32(float(getattr(o, "viscosity", 0.0))),
    wind=f32(np.asarray(getattr(o, "wind", np.zeros(3)), dtype=np.float64).reshape(3)),
    # (nb, 3): world w reads entry w % nb (assign an (nworld, 3) tensor for per-world fields); MuJoCo's default for older models
    magnetic=f32(np.asarray(getattr(o, "magnetic", (0.0, -0.5, 0.0)), dtype=np.float64).reshape(3)),
  )
  if len(t["nxn_geom_pair_filtered"]) >= 250_000:
    # the reference switches to sweep-and-prune here (io.py:631-636); this build keeps one world's geoms and pair list in one
    # warp's shared memory, which such a model does not fit.  opt.broadphase = SAP_* is honoured for models that do fit.
    raise NotImplementedError("models with >= 250k candidate geom pairs are not supported in this version")
  m.stat = types.Statistic(meaninertia=f32(mjm.stat.meaninertia))

  keep = []

  def dev_f(arr, batched=True, name=None):
    a = np.ascontiguousarray(np.asarray(arr, dtype=np.float32))
    x = torch.from_numpy(a).to(dev)
    if not batched:
      return x
    nb = int(batch_sizes.get(name, 1)) if name else 1
    return x.unsqueeze(0).repeat(nb, *([1] * x.dim())).contiguous()

  def dev_i(arr):
    a = np.ascontiguousarray(np.asarray(arr).astype(np.int32))
    return torch.from_numpy(a).to(dev)

  for n in _FLOAT_FIELDS:
    setattr(m, n, dev_f(getattr(mjm, n), name=n))
  for n in _INT_FIELDS:
    setattr(m, n, dev_i(getattr(mjm, n)))
  # stateful actuators (forward.py:135-218, 800-963): activation layout and dynamics parameters
  nu_ = int(mjm.nu)
  m.actuator_dyntype = dev_i(getattr(mjm, "actuator_dyntype", np.zeros(nu_)))
  m.actuator_actadr = dev_i(getattr(mjm, "actuator_actadr", -np.ones(nu_)))
  m.actuator_actnum = dev_i(getattr(mjm, "actuator_actnum", np.zeros(nu_)))
  m.actuator_actlimited = dev_i(np.asarray(getattr(mjm, "actuator_actlimited", np.zeros(nu_))).astype(np.int32))
  m.actuator_actearly = dev_i(np.asarray(getattr(mjm, "actuator_actearly", np.zeros(nu_))).astype(np.int32))
  m.actuator_dynprm = dev_f(np.asarray(getattr(mjm, "actuator_dynprm", np.zeros((nu_, 10)))).reshape(nu_, 10), name="actuator_dynprm")
  # acceleration of a unit actuator force at qpos0 (set_const.py:493-504): the force scale of muscles with force < 0
  m.actuator_acc0 = dev_f(np.asarray(getattr(mjm, "actuator_acc0", np.zeros(nu_))).reshape(nu_), name="actuator_acc0")
  # feasible length range (types.py:1315): the muscles' optimum length and normalized length (util_misc.py:481-558)
  m.actuator_lengthrange = dev_f(np.asarray(getattr(mjm, "actuator_lengthrange", np.zeros((nu_, 2)))).reshape(nu_, 2), name="actuator_lengthrange")
  m.actuator_actrange = dev_f(np.asarray(getattr(mjm, "actuator_actrange", np.zeros((nu_, 2)))).reshape(nu_, 2), name="actuator_actrange")
  # fixed tendons (smooth.py:3658; constraint.py:642, 1867, 2243; passive.py:208): path, Jacobian sparsity and constant entries
  nt = int(getattr(mjm, "ntendon", 0))
  m.ntendon, m.nJten, m.nwrap = nt, (int(getattr(mjm, "nJten", 0)) if nt else 0), (int(getattr(mjm, "nwrap", 0)) if nt else 0)
  m.actuator_trntype = dev_i(getattr(mjm, "actuator_trntype", np.zeros(nu_)))
  for n in ("ten_J_rownnz", "ten_J_rowadr", "ten_J_colind", "tendon_adr", "tendon_num", "wrap_objid"):
    setattr(m, n, dev_i(getattr(mjm, n) if nt else np.zeros(0)))
  m.tendon_limited = dev_i(np.asarray(mjm.tendon_limited).astype(np.int32) if nt else np.zeros(0))
  m.tendon_actfrclimited = dev_i(np.asarray(getattr(mjm, "tendon_actfrclimited", np.zeros(nt))).astype(np.int32) if nt else np.zeros(0))
  m.wrap_prm = dev_f(mjm.wrap_prm if nt else np.zeros(0), batched=False)
  tenJ0 = np.zeros(m.nJten)
  for t_ in range(nt):  # the last joint wrap that hits a dof sets the entry (the reference assigns, it does not accumulate)
    for k in range(int(mjm.tendon_adr[t_]), int(mjm.tendon_adr[t_]) + int(mjm.tendon_num[t_])):
      dof = int(mjm.jnt_dofadr[int(mjm.wrap_objid[k])])
      row = np.asarray(mjm.ten_J_colind)[int(mjm.ten_J_rowadr[t_]) : int(mjm.ten_J_rowadr[t_]) + int(mjm.ten_J_rownnz[t_])]
      tenJ0[int(mjm.ten_J_rowadr[t_]) + int(np.nonzero(row == dof)[0][0])] = float(mjm.wrap_prm[k])
  m.ten_J0 = dev_f(tenJ0, batched=False)
  for n, k in _TENDON_FLOATS:
    setattr(m, n, dev_f(np.asarray(getattr(mjm, n)).reshape((nt, k) if k > 1 else (nt,)) if nt else np.zeros((0, k) if k > 1 else 0), name=n))
  m.ntenfric = int((np.asarray(mjm.tendon_frictionloss) > 0).sum()) if nt else 0
  m.jnt_limited = dev_i(np.asarray(mjm.jnt_limited).astype(np.int32))
  m.body_tree = tuple(dev_i(x) for x in t["body_tree"])
  for n in ("body_childadr", "body_childid", "level_adr", "level_body", "M_entry_row", "mulm_rowadr", "mulm_col", "mulm_madr", "tree_qLDadr",
            "qLD_block_adr", "jnt_limited_slide_hinge_adr", "jnt_limited_ball_adr", "dof_fricloss_adr", "moment_rownnz0", "moment_rowadr0", "moment_colind0",
            "dofact_adr", "dofact_act", "dofact_mom",
            "nxn_geom_pair", "nxn_pairid", "nxn_geom_pair_filtered", "nxn_pairid_filtered"):
    setattr(m, n, dev_i(t[n]))
  m.M_hinit_i = m.M_entry_row
  # D-structure (types.py:1343-1347): the dofs coupled to each dof, both triangles; identical to the symmetric gather rows of mul_m
  m.D_rowadr, m.D_colind, m.mapM2D = m.mulm_rowadr[:-1], m.mulm_col, m.mulm_madr
  m.D_rownnz = dev_i(np.diff(t["mulm_rowadr"]))
  m.D_diag = dev_i(np.array([list(t["mulm_col"][t["mulm_rowadr"][i] : t["mulm_rowadr"][i + 1]]).index(i) for i in range(m.nv)], dtype=np.int32))
  m.nD = int(t["mulm_rowadr"][-1])
  # equality constraints (connect / weld / joint): eq_* as in the reference Model (types.py), data per world-batch slot 0
  neq = int(getattr(mjm, "neq", 0))
  m.neq = neq
  nsensor = int(getattr(mjm, "nsensor", 0))
  unsupported = [str(x) for x in np.asarray(getattr(mjm, "sensor_unsupported", []), dtype=object).reshape(-1)]
  if unsupported:
    raise NotImplementedError(f"sensor types not implemented in this version: {sorted(set(unsupported))}")
  m.nsensor, m.nsensordata = nsensor, int(getattr(mjm, "nsensordata", 0)) if nsensor else 0
  for n in ("sensor_type", "sensor_datatype", "sensor_needstage", "sensor_objtype", "sensor_objid", "sensor_dim", "sensor_adr"):
    setattr(m, n, dev_i(getattr(mjm, n) if nsensor else np.zeros(0)))
  m.sensor_reftype = dev_i(getattr(mjm, "sensor_reftype", np.zeros(nsensor)) if nsensor else np.zeros(0))
  m.sensor_refid = dev_i(getattr(mjm, "sensor_refid", -np.ones(nsensor)) if nsensor else np.zeros(0))
  m.sensor_cutoff = dev_f(np.asarray(mjm.sensor_cutoff) if nsensor else np.zeros(0), batched=False)
  nsite = int(getattr(mjm, "nsite", 0))
  m.site_type = dev_i(getattr(mjm, "site_type", np.full(nsite, C.GEOM_SPHERE)))  # fixtures compiled before sites carried a shape: MuJoCo's default
  m.site_size = dev_f(getattr(mjm, "site_size", np.full((nsite, 3), 0.005)), batched=False)
  stype = np.asarray(mjm.sensor_type) if nsensor else np.zeros(0, dtype=int)
  m.sensor_subtree_vel = bool(np.isin(stype, (C.SENS_SUBTREELINVEL, C.SENS_SUBTREEANGMOM)).any())  # reference io.py:896-897
  m.sensor_extra = _validate_extra_sensors(mjm)
  m.sensor_rne_postconstraint = bool(np.isin(stype, (C.SENS_ACCELEROMETER, C.SENS_FORCE, C.SENS_TORQUE, C.SENS_FRAMELINACC, C.SENS_FRAMEANGACC)).any())  # :900
  # <contact> sensors (reference io.py:409-413, :441, :898): their ids, [dataspec, reduce, num] per sensor, and the match capacity
  sensor_intprm = _contact_sensor_intprm(mjm)
  m.sensor_intprm = dev_i(sensor_intprm)
  m.sensor_contact_adr = dev_i(np.nonzero(stype == C.SENS_CONTACT)[0])
  m.nsensorcontact = int(m.sensor_contact_adr.numel())
  m.opt.contact_sensor_maxmatch = mjcf.contact_sensor_maxmatch(mjm)
  sc = _sensor_collision_tables(mjm, t)
  m.nsensorcollision, m.sensor_collision_epa_iterations, m.nsensorcollision_ccd = (sc.pop(k) for k in ("nsensorcollision", "sensor_collision_epa_iterations", "nsensorcollision_ccd"))
  for n, x in sc.items():
    setattr(m, n, dev_i(x))
  m.sensor_energy_adr = dev_i(t["sensor_energy_adr"])
  m.sensor_e_potential, m.sensor_e_kinetic = t["sensor_e_potential"], t["sensor_e_kinetic"]
  # delay / history buffers (reference types.py:1306-1329); a real MjModel's addresses are taken as given
  hf = history_fields(mjm)
  m.nhistory = hf.pop("nhistory")
  for n, x in hf.items():
    setattr(m, n, dev_i(x) if x.dtype == np.int32 else dev_f(x, batched=False))
  m.sensor_history_id = dev_i(np.nonzero(hf["sensor_history"][:, 0] > 0)[0])  # the sensors k_history_sensor runs over
  m._history = hf  # host copies: the public history functions check sizes against them
  m.eq_type = dev_i(mjm.eq_type if neq else np.zeros(0))
  m.eq_obj1id = dev_i(mjm.eq_obj1id if neq else np.zeros(0))
  m.eq_obj2id = dev_i(mjm.eq_obj2id if neq else np.zeros(0))
  m.eq_objtype = dev_i(mjm.eq_objtype if neq else np.zeros(0))
  m.eq_solref = dev_f(np.asarray(mjm.eq_solref).reshape(neq, 2) if neq else np.zeros((0, 2)), name="eq_solref")
  m.eq_solimp = dev_f(np.asarray(mjm.eq_solimp).reshape(neq, 5) if neq else np.zeros((0, 5)), name="eq_solimp")
  m.eq_data = dev_f(np.asarray(mjm.eq_data).reshape(neq, 11) if neq else np.zeros((0, 11)), name="eq_data")
  # explicit contact pairs (reference Model.pair_*)
  npair = int(getattr(mjm, "npair", 0))
  m.npair = npair
  m.pair_dim = dev_i(mjm.pair_dim if npair else np.zeros(0))
  m.pair_geom1 = dev_i(mjm.pair_geom1 if npair else np.zeros(0))
  m.pair_geom2 = dev_i(mjm.pair_geom2 if npair else np.zeros(0))
  for n, k in (("pair_friction", 5), ("pair_solref", 2), ("pair_solreffriction", 2), ("pair_solimp", 5)):
    setattr(m, n, dev_f(np.asarray(getattr(mjm, n)).reshape(npair, k) if npair else np.zeros((0, k)), name=n))
  for n in ("pair_margin", "pair_gap"):
    setattr(m, n, dev_f(np.asarray(getattr(mjm, n)) if npair else np.zeros(0), name=n))
  # mesh assets (reference Model.mesh_*, types.py): vertex blocks, hull graphs for hill-climbing support queries, hull polygons
  nmesh = int(getattr(mjm, "nmesh", 0))
  m.nmesh = nmesh
  # most vertices in one hull polygon / most hull polygons at one vertex: past 32 / 16 the collision stage runs the build whose multi-contact
  # buffers are sized from these (make_data allocates its scratch)
  m.npolygonmax = int(getattr(mjm, "npolygonmax", 0)) if nmesh else 0
  m.nmeshdegmax = int(getattr(mjm, "nmeshdegmax", 0)) if nmesh else 0
  if nmesh and int(np.asarray(mjm.mesh_vertnum).max()) > 0xFFFF:
    raise NotImplementedError(f"mesh with {int(np.asarray(mjm.mesh_vertnum).max())} vertices: the convex collision packs mesh vertex ids in 16 bits (at most 65535)")
  m.geom_dataid = dev_i(getattr(mjm, "geom_dataid", -np.ones(m.ngeom)))
  for n in ("mesh_vertadr", "mesh_vertnum", "mesh_graphadr", "mesh_graph", "mesh_polynum", "mesh_polyadr", "mesh_polyvertadr", "mesh_polyvertnum",
            "mesh_polyvert", "mesh_polymapadr", "mesh_polymapnum", "mesh_polymap"):
    setattr(m, n, dev_i(getattr(mjm, n) if nmesh else np.zeros(0)))
  m.mesh_vert = dev_f(np.asarray(mjm.mesh_vert).reshape(-1, 3) if nmesh else np.zeros((0, 3)), batched=False)
  m.mesh_polynormal = dev_f(np.asarray(mjm.mesh_polynormal).reshape(-1, 3) if nmesh else np.zeros((0, 3)), batched=False)
  # ray casting (reference ray.py:53 _ray_eliminate, :629 ray_mesh): geom visibility, groups and materials, and the mesh triangles.
  # Models saved before these fields existed get MuJoCo's defaults: opaque grey geoms in group 0, no materials.
  ng = m.ngeom
  m.geom_group = dev_i(getattr(mjm, "geom_group", np.zeros(ng)))
  m.geom_matid = dev_i(getattr(mjm, "geom_matid", -np.ones(ng)))
  m.geom_rgba = dev_f(np.asarray(getattr(mjm, "geom_rgba", np.tile([0.5, 0.5, 0.5, 1.0], (ng, 1)))).reshape(ng, 4), name="geom_rgba")
  m.nmat = int(getattr(mjm, "nmat", 0))
  m.mat_rgba = dev_f(np.asarray(mjm.mat_rgba).reshape(m.nmat, 4) if m.nmat else np.zeros((0, 4)), name="mat_rgba")
  # the renderer's camera, light and material fields (render.py); read at each render() call, so they are not bound to the handle
  for n, x in render_fields(mjm).items():
    setattr(m, n, dev_f(x, name=n) if n in _RENDER_FLOATS else (dev_f(x, batched=False) if x.dtype == np.float64 else dev_i(x)))
  m.mesh_faceadr = dev_i(getattr(mjm, "mesh_faceadr", np.zeros(nmesh)) if nmesh else np.zeros(0))
  m.mesh_face = dev_i(np.asarray(getattr(mjm, "mesh_face", np.zeros((0, 3)))).reshape(-1, 3) if nmesh else np.zeros((0, 3)))
  m.nmeshface = int(m.mesh_face.shape[0])
  # fluid forces (io.py:471, 523-530).  Models saved without geom_fluid have no ellipsoid geoms.
  m.has_fluid = _has_fluid(o)
  geom_fluid = np.asarray(getattr(mjm, "geom_fluid", np.zeros((ng, 12))), dtype=np.float64).reshape(ng, 12)
  m.geom_fluid = dev_f(geom_fluid, batched=False)
  ellipsoid = np.zeros(m.nbody, dtype=bool)
  ellipsoid[np.asarray(mjm.geom_bodyid)[geom_fluid[:, 0] > 0]] = True
  box = ~ellipsoid & (np.asarray(mjm.body_mass) > 0.0)
  box[0] = False
  m.body_fluid_ellipsoid = torch.from_numpy(ellipsoid).to(dev)
  m.body_fluid_ellipsoid_adr = dev_i(np.nonzero(ellipsoid)[0])
  m.body_fluid_box_adr = dev_i(np.nonzero(box)[0])
  m.body_fluid = dev_i(np.where(ellipsoid, 1, np.where(box, 2, 0)))  # the kernels' per-body model: 0 none, 1 ellipsoid, 2 inertia box
  m.body_geomadr = dev_i(mjm.body_geomadr)
  m.body_geomnum = dev_i(mjm.body_geomnum)
  m.M_mulm_rowadr, m.M_mulm_col, m.M_mulm_madr = m.mulm_rowadr, m.mulm_col, m.mulm_madr
  anc_pad = np.zeros((m.nbody, m.nv_pad), dtype=np.int32)
  anc_pad[:, : m.nv] = t["body_isdofancestor"]
  m.body_isdofancestor = dev_i(anc_pad).reshape(m.nbody, m.nv_pad)
  m._isdofancestor_nv = dev_i(t["body_isdofancestor"])
  # host copies the harness reads
  m._mjm = mjm
  m._tables = t

  # ---- bind to the C ABI
  h = L.mjb_model_create()
  m._handle = h
  ints = dict(
    nq=m.nq, nv=m.nv, nu=m.nu, nbody=m.nbody, njnt=m.njnt, ngeom=m.ngeom, nsite=m.nsite, ncam=m.ncam, nlight=m.nlight, nC=m.nC, ntree=m.ntree,
    nJmom=m.nJmom, nlevel=t["nlevel"], nxn_npair=len(t["nxn_geom_pair_filtered"]), nlimit=len(t["jnt_limited_slide_hinge_adr"]),
    nfricdof=len(t["dof_fricloss_adr"]), nmaxpyramid=m.nmaxpyramid, integrator=m.opt.integrator, cone=m.opt.cone, solver=m.opt.solver,
    iterations=m.opt.iterations, ls_iterations=m.opt.ls_iterations, disableflags=m.opt.disableflags, enableflags=m.opt.enableflags,
    broadphase=int(m.opt.broadphase), broadphase_filter=m.opt.broadphase_filter, qld_total=t["qld_total"], maxtree=t["maxtree"],
    has_multicontact_geom=int(np.isin(_np(mjm, "geom_type"), (C.GEOM_ELLIPSOID, C.GEOM_CYLINDER, C.GEOM_BOX, C.GEOM_MESH)).any()), nmesh=nmesh, na=m.na, ntendon=m.ntendon, nJten=m.nJten, ntenfric=m.ntenfric, nwrap=m.nwrap,
    nmocap=int(getattr(mjm, "nmocap", 0)), npair=npair, has_convex_pair=t["has_convex_pair"], ccd_iterations=int(getattr(o, "ccd_iterations", 35)), epa_iterations=t["epa_iterations"], nsensor=m.nsensor, nsensordata=m.nsensordata, nmat=m.nmat, nmeshface=m.nmeshface, sensor_subtree_vel=int(m.sensor_subtree_vel), sensor_rne_postconstraint=int(m.sensor_rne_postconstraint), neq=neq, nlimit_ball=len(t["jnt_limited_ball_adr"]), has_fluid=int(m.has_fluid), has_gravcomp=int((np.asarray(mjm.body_gravcomp) != 0).any() or (np.asarray(mjm.jnt_stiffness)[np.isin(np.asarray(mjm.jnt_type), (C.JNT_FREE, C.JNT_BALL))] != 0).any()),
  )
  for k, v in ints.items():
    _lib.check(L.mjb_model_set_int(h, k.encode(), int(v)))
  for k, v in (("nsensorcollision", m.nsensorcollision), ("nsensorcollision_sensor", len(m.sensor_collision_id)), ("sensor_collision_epa_iterations", m.sensor_collision_epa_iterations),
               ("nsensorcollision_ccd", m.nsensorcollision_ccd), ("nsensor_energy", len(t["sensor_energy_adr"])),
               ("sensor_e_potential", m.sensor_e_potential), ("sensor_e_kinetic", m.sensor_e_kinetic),
               ("nsensorcontact", m.nsensorcontact), ("contact_sensor_maxmatch", m.opt.contact_sensor_maxmatch), ("nhistory", m.nhistory), ("nactuator_history", int((hf["actuator_history"][:, 0] > 0).sum())), ("nsensor_history", len(m.sensor_history_id)),
               ("npolygonmax", m.npolygonmax), ("nmeshdegmax", m.nmeshdegmax), ("sensor_extra", int(m.sensor_extra))):
    _lib.check(L.mjb_model_set_int(h, k.encode(), int(v)))
  g = np.asarray(o.gravity, dtype=np.float64)
  floats = dict(timestep=o.timestep, tolerance=tol, ls_tolerance=o.ls_tolerance, impratio_invsqrt=1.0 / np.sqrt(o.impratio),
                meaninertia=mjm.stat.meaninertia, gravity_x=g[0], gravity_y=g[1], gravity_z=g[2], ccd_tolerance=float(getattr(o, "ccd_tolerance", 1e-6)))
  wind = np.asarray(getattr(o, "wind", np.zeros(3)), dtype=np.float64).reshape(3)
  floats.update(density=float(getattr(o, "density", 0.0)), viscosity=float(getattr(o, "viscosity", 0.0)), wind_x=wind[0], wind_y=wind[1], wind_z=wind[2])
  for k, v in floats.items():
    _lib.check(L.mjb_model_set_float(h, k.encode(), float(v)))
  dev_names = {
    "jnt_limited_adr": m.jnt_limited_slide_hinge_adr, "nxn_geom_pair": m.nxn_geom_pair_filtered, "nxn_pairid": m.nxn_pairid_filtered,
    "body_isdofancestor": m._isdofancestor_nv, "meaninertia": m.stat.meaninertia,  # set_const writes world 0's meaninertia here
    "magnetic": m.opt.magnetic,
  }
  for n in (_FLOAT_FIELDS + _INT_FIELDS + ["body_childadr", "body_childid", "level_adr", "level_body", "M_entry_row", "mulm_rowadr", "mulm_col",
                                         "mulm_madr", "tree_qLDadr", "dof_fricloss_adr", "moment_rownnz0", "moment_rowadr0", "moment_colind0",
                                         "dofact_adr", "dofact_act", "dofact_mom", "eq_type", "eq_obj1id", "eq_obj2id", "eq_solref", "eq_solimp", "eq_data",
                                         "jnt_limited_ball_adr", "pair_dim", "pair_friction", "pair_solref", "pair_solreffriction", "pair_solimp",
                                         "pair_margin", "pair_gap", "sensor_type", "sensor_datatype", "sensor_needstage", "sensor_objtype", "sensor_objid", "sensor_reftype", "sensor_refid",
                                         "sensor_dim", "sensor_adr", "sensor_cutoff", "site_type", "site_size", "geom_dataid", "mesh_vertadr", "mesh_vertnum", "mesh_graphadr", "mesh_graph",
                                         "mesh_polynum", "mesh_polyadr", "mesh_polyvertadr", "mesh_polyvertnum", "mesh_polyvert", "mesh_polymapadr", "mesh_polymapnum",
                                         "mesh_polymap", "mesh_vert", "mesh_polynormal", "actuator_dyntype", "actuator_actadr", "actuator_actnum",
                                         "actuator_actlimited", "actuator_actearly", "actuator_dynprm", "actuator_actrange", "actuator_trntype",
                                         "ten_J_rownnz", "ten_J_rowadr", "ten_J_colind", "tendon_adr", "tendon_num", "wrap_objid", "tendon_limited", "tendon_actfrclimited", "wrap_prm", "ten_J0",
                                         "geom_group", "geom_matid", "geom_rgba", "mat_rgba", "mesh_faceadr", "mesh_face",
                                         "geom_fluid", "body_fluid", "body_geomadr", "body_geomnum", "sensor_collision_start_adr", "sensor_collision_pair",
                                         "sensor_collision_id", "sensor_collision_adr", "sensor_collision_flip", "actuator_acc0", "actuator_lengthrange", "jnt_limited", "sensor_energy_adr",
                                         "actuator_history", "actuator_historyadr", "actuator_delay", "sensor_history", "sensor_historyadr", "sensor_delay",
                                         "sensor_interval", "sensor_history_id", "sensor_contact_adr", "sensor_intprm",
                                         "cam_fovy", "cam_intrinsic", "cam_sensorsize", "cam_resolution"]
                                        + [n for n, _ in _TENDON_FLOATS]):
    dev_names.setdefault(n, getattr(m, n))
  for n, x in dev_names.items():
    x = _ptr_tensor(x)
    keep.append(x)
    nb = int(x.shape[0]) if (n in _FLOAT_FIELDS or n in _BATCHABLE_EXTRA or n in _SENSOR_BATCHED) and x.dim() >= 1 and x.numel() > 0 else 1
    _lib.check(L.mjb_model_set_array_batched(h, n.encode(), x.data_ptr(), nb, int(x.numel() // max(nb, 1))))
  _lib.check(L.mjb_model_finalize(h))
  m._keep = keep
  weakref.finalize(m, L.mjb_model_destroy, h)
  _install_model_rebind(m, L, set(dev_names) - {"jnt_limited_adr", "nxn_geom_pair", "nxn_pairid", "body_isdofancestor", "meaninertia", "magnetic"}, set(ints))
  return m


_OPT_FLOATS = {"timestep": "timestep", "tolerance": "tolerance", "ls_tolerance": "ls_tolerance", "impratio_invsqrt": "impratio_invsqrt", "ccd_tolerance": "ccd_tolerance",
               "density": "density", "viscosity": "viscosity"}
_OPT_INTS = ("integrator", "cone", "solver", "iterations", "ls_iterations", "disableflags", "enableflags", "broadphase", "broadphase_filter", "ccd_iterations",
             "contact_sensor_maxmatch")


def _check_like(name, new, old):
  if not isinstance(new, torch.Tensor):
    raise TypeError(f"{name}: expected a torch.Tensor like the bound one ({tuple(old.shape)}, {old.dtype}), got {type(new).__name__}; use .copy_() to write values")
  if new.shape != old.shape or new.dtype != old.dtype or new.device != old.device:
    raise ValueError(f"{name}: replacement must match the bound tensor: shape {tuple(old.shape)} {old.dtype} on {old.device}, got {tuple(new.shape)} {new.dtype} on {new.device}")
  return new.contiguous()


def _install_model_rebind(m: types.Model, L, arrays, ints):
  """Assignments to bound Model / Option / Statistic fields reach the C handle (ADVICE r1: they used to be silent no-ops)."""
  h = m._handle

  def model_hook(name, value):
    if name in arrays and name in m.__dict__:
      old = m.__dict__[name]
      batchable = name in _FLOAT_FIELDS or name in _BATCHABLE_EXTRA or name in _SENSOR_BATCHED
      if batchable and isinstance(value, torch.Tensor) and value.dim() == old.dim() and value.shape[1:] == old.shape[1:] and value.shape[0] >= 1:
        # a per-world (batched) field may change its leading size: world w reads entry w % size (reference types.py:822-833)
        if value.dtype != old.dtype or value.device != old.device:
          raise ValueError(f"Model.{name}: replacement must be {old.dtype} on {old.device}")
        value = value.contiguous()
      else:
        value = _check_like("Model." + name, value, old)
      x = _ptr_tensor(value)
      m._keep.append(x)
      nb = int(x.shape[0]) if batchable and x.numel() > 0 else 1
      _lib.check(L.mjb_model_set_array_batched(h, name.encode(), x.data_ptr(), nb, int(x.numel() // max(nb, 1))))
    elif name in ints and name in m.__dict__ and isinstance(m.__dict__[name], int):
      raise AttributeError(f"Model.{name} is a compiled size / table constant and cannot be reassigned; build a new Model with put_model")
    return value

  def opt_hook(name, value):
    if name in _OPT_FLOATS:
      v = float(value.reshape(-1)[0]) if isinstance(value, torch.Tensor) else float(value)
      if name == "tolerance":
        v = max(v, 1e-6)
      _lib.check(L.mjb_model_set_float(h, _OPT_FLOATS[name].encode(), v))
      return torch.full((1,), v, dtype=torch.float32, device=m.opt.__dict__[name].device) if not isinstance(value, torch.Tensor) else value
    if name in ("gravity", "wind"):
      g = value.reshape(-1)[:3].tolist() if isinstance(value, torch.Tensor) else [float(x) for x in value]
      for k, v in zip((f"{name}_x", f"{name}_y", f"{name}_z"), g):
        _lib.check(L.mjb_model_set_float(h, k.encode(), float(v)))
      return value if isinstance(value, torch.Tensor) else torch.tensor([g], dtype=torch.float32, device=m.opt.__dict__[name].device)
    if name == "magnetic":  # per world like the batched Model fields: (nb, 3), world w reads entry w % nb
      old = m.opt.__dict__[name]
      x = value if isinstance(value, torch.Tensor) else torch.tensor(np.asarray(value, dtype=np.float32), device=old.device)
      x = x.to(dtype=old.dtype, device=old.device).reshape(-1, 3).contiguous()
      if x.shape[0] < 1:
        raise ValueError(f"opt.magnetic: expected (nb, 3) with nb >= 1, got {tuple(value.shape) if isinstance(value, torch.Tensor) else np.shape(value)}")
      m._keep.append(x)
      _lib.check(L.mjb_model_set_array_batched(h, b"magnetic", x.data_ptr(), int(x.shape[0]), 3))
      return x
    if name in _OPT_INTS:
      if name == "integrator" and int(value) not in (C.INT_EULER, C.INT_IMPLICIT, C.INT_IMPLICITFAST, C.INT_RK4):
        raise NotImplementedError(f"integrator {value} not implemented")
      if name == "contact_sensor_maxmatch" and int(value) < 1:
        raise ValueError(f"opt.contact_sensor_maxmatch must be >= 1, got {int(value)}")
      if name in ("integrator", "cone", "solver") and int(value) != int(m.opt.__dict__[name]):
        raise NotImplementedError(f"opt.{name} selects kernel instantiations and scratch sizes fixed at put_model / make_data; rebuild the Model to change it")
      _lib.check(L.mjb_model_set_int(h, name.encode(), int(value)))
    return value

  def stat_hook(name, value):
    if name == "meaninertia":
      v = float(value.reshape(-1)[0]) if isinstance(value, torch.Tensor) else float(value)
      _lib.check(L.mjb_model_set_float(h, b"meaninertia", v))
      old = m.stat.__dict__.get("meaninertia")
      if (isinstance(value, torch.Tensor) and value.numel() >= 1 and value.device.type != "cpu" and value.dtype == torch.float32
          and (not isinstance(old, torch.Tensor) or value.data_ptr() != old.data_ptr())):
        x = _ptr_tensor(value.contiguous())
        m._keep.append(x)
        _lib.check(L.mjb_model_set_array(h, b"meaninertia", x.data_ptr(), 1))  # set_const's output follows the Statistic's tensor
    return value

  object.__setattr__(m, "_rebind", model_hook)
  object.__setattr__(m.opt, "_rebind", opt_hook)
  object.__setattr__(m.stat, "_rebind", stat_hook)


# --------------------------------------------------------------------------------------------- Data


def _data_spec(m: types.Model, nworld, naconmax, njmax, njmax_pad):
  """name -> (dtype, shape) for top-level Data fields (reference types.py:2230-2374)."""
  f, i = torch.float32, torch.int32
  nb, nv, nq, nu, nj, ng = m.nbody, m.nv, m.nq, m.nu, m.njnt, m.ngeom
  return {
    "solver_niter": (i, (nworld,)), "ne": (i, (nworld,)), "nf": (i, (nworld,)), "nl": (i, (nworld,)), "nefc": (i, (nworld,)),
    "ten_length": (f, (nworld, m.ntendon)), "ten_J": (f, (nworld, m.nJten)), "ten_velocity": (f, (nworld, m.ntendon)),
    "time": (f, (nworld,)), "qpos": (f, (nworld, nq)), "qvel": (f, (nworld, nv)), "act": (f, (nworld, m.na)),
    "qacc_warmstart": (f, (nworld, nv)), "ctrl": (f, (nworld, nu)), "qfrc_applied": (f, (nworld, nv)), "xfrc_applied": (f, (nworld, nb, 6)),
    "qacc": (f, (nworld, nv)), "act_dot": (f, (nworld, m.na)), "sensordata": (f, (nworld, getattr(m, "nsensordata", 0))), "subtree_linvel": (f, (nworld, nb, 3)), "subtree_angmom": (f, (nworld, nb, 3)),
    "xpos": (f, (nworld, nb, 3)), "xquat": (f, (nworld, nb, 4)), "xmat": (f, (nworld, nb, 3, 3)), "xipos": (f, (nworld, nb, 3)),
    "ximat": (f, (nworld, nb, 3, 3)), "xanchor": (f, (nworld, nj, 3)), "xaxis": (f, (nworld, nj, 3)),
    "geom_xpos": (f, (nworld, ng, 3)), "geom_xmat": (f, (nworld, ng, 3, 3)), "site_xpos": (f, (nworld, m.nsite, 3)), "site_xmat": (f, (nworld, m.nsite, 3, 3)),
    "cam_xpos": (f, (nworld, m.ncam, 3)), "cam_xmat": (f, (nworld, m.ncam, 3, 3)), "light_xpos": (f, (nworld, m.nlight, 3)), "light_xdir": (f, (nworld, m.nlight, 3)),
    "subtree_com": (f, (nworld, nb, 3)), "cdof": (f, (nworld, nv, 6)), "cinert": (f, (nworld, nb, 10)),
    "actuator_length": (f, (nworld, nu)), "moment_rownnz": (i, (nworld, nu)), "moment_rowadr": (i, (nworld, nu)),
    "moment_colind": (i, (nworld, m.nJmom)), "actuator_moment": (f, (nworld, m.nJmom)),
    "crb": (f, (nworld, nb, 10)), "M": (f, (nworld, m.nC)), "qLD": (f, (nworld, m.qLD_block_total)), "qLDiagInv": (f, (nworld, nv)), "qLU": (f, (nworld, m.nD)),
    "actuator_velocity": (f, (nworld, nu)), "cvel": (f, (nworld, nb, 6)), "cdof_dot": (f, (nworld, nv, 6)),
    "qfrc_bias": (f, (nworld, nv)), "qfrc_spring": (f, (nworld, nv)), "qfrc_damper": (f, (nworld, nv)), "qfrc_gravcomp": (f, (nworld, nv)),
    "qfrc_fluid": (f, (nworld, nv)), "qfrc_adhesion": (f, (nworld, nv)), "qfrc_passive": (f, (nworld, nv)),
    "actuator_force": (f, (nworld, nu)), "qfrc_actuator": (f, (nworld, nv)), "qfrc_smooth": (f, (nworld, nv)), "qacc_smooth": (f, (nworld, nv)),
    "qfrc_constraint": (f, (nworld, nv)), "qfrc_inverse": (f, (nworld, nv)), "cacc": (f, (nworld, nb, 6)), "cfrc_int": (f, (nworld, nb, 6)),
    "cfrc_ext": (f, (nworld, nb, 6)), "energy": (f, (nworld, 2)), "history": (f, (nworld, m.nhistory)),
    "nacon": (i, (1,)), "ncollision": (i, (1,)), "overflow": (i, (nworld,)),
    "eq_active": (i, (nworld, getattr(m, "neq", 0))),  # the reference stores bool; int32 0/1 here (one word per flag)
    "mocap_pos": (f, (nworld, m.nmocap, 3)), "mocap_quat": (f, (nworld, m.nmocap, 4)),
  }


def _contact_spec(m, naconmax):
  f, i = torch.float32, torch.int32
  return {
    "dist": (f, (naconmax,)), "pos": (f, (naconmax, 3)), "frame": (f, (naconmax, 3, 3)), "includemargin": (f, (naconmax,)),
    "friction": (f, (naconmax, 5)), "solref": (f, (naconmax, 2)), "solreffriction": (f, (naconmax, 2)), "solimp": (f, (naconmax, 5)),
    "dim": (i, (naconmax,)), "geom": (i, (naconmax, 2)), "efc_address": (i, (naconmax, m.nmaxpyramid)), "worldid": (i, (naconmax,)),
    "type": (i, (naconmax,)), "geomcollisionid": (i, (naconmax,)),
  }


def _efc_spec(m, nworld, njmax, njmax_pad):
  f, i = torch.float32, torch.int32
  return {
    "type": (i, (nworld, njmax)), "id": (i, (nworld, njmax)), "J": (f, (nworld, njmax_pad, m.nv_pad)), "pos": (f, (nworld, njmax)),
    "margin": (f, (nworld, njmax)), "D": (f, (nworld, njmax_pad)), "vel": (f, (nworld, njmax)), "aref": (f, (nworld, njmax)),
    "frictionloss": (f, (nworld, njmax)), "force": (f, (nworld, njmax)), "state": (i, (nworld, njmax_pad)), "Ma": (f, (nworld, nv_of(m))),
    "Jqvel": (f, (nworld, njmax)),
  }


def nv_of(m):
  return m.nv


_BOUND_TOP = [
  "time", "qpos", "qvel", "ctrl", "qacc_warmstart", "qfrc_applied", "xfrc_applied", "qacc", "xpos", "xquat", "xmat", "xipos", "ximat", "xanchor",
  "xaxis", "geom_xpos", "geom_xmat", "site_xpos", "site_xmat", "cam_xpos", "cam_xmat", "light_xpos", "light_xdir", "subtree_com", "cdof", "cinert",
  "crb", "M", "qLD", "actuator_length", "actuator_moment", "actuator_velocity", "cvel", "cdof_dot", "qfrc_bias", "qfrc_spring", "qfrc_damper",
  "qfrc_gravcomp", "qfrc_passive", "actuator_force", "qfrc_actuator", "qfrc_smooth", "qacc_smooth", "qfrc_constraint", "qfrc_inverse", "cacc", "cfrc_int",
  "ne", "nf", "nl", "nefc", "nacon", "ncollision", "solver_niter", "overflow", "moment_rownnz", "moment_rowadr", "moment_colind", "eq_active", "mocap_pos", "mocap_quat", "sensordata", "subtree_linvel", "subtree_angmom", "cfrc_ext",
  "act", "act_dot", "ten_length", "ten_J", "ten_velocity", "qLU", "qfrc_fluid", "energy", "history",
]
_BOUND_EFC = ["J", "pos", "margin", "D", "vel", "aref", "frictionloss", "force", "Ma", "type", "id", "state"]
_BOUND_CONTACT = ["dist", "pos", "frame", "includemargin", "friction", "solref", "solreffriction", "solimp", "dim", "geom", "efc_address", "worldid", "type", "geomcollisionid"]


def _alloc(spec, dev):
  out = {}
  for name, (dt, shape) in spec.items():
    out[name] = torch.zeros(shape, dtype=dt, device=dev)
  return out


def make_data(mjm, nworld: int = 1, nconmax=None, nccdmax=None, njmax=None, njmax_nnz=None, naconmax=None, naccdmax=None, nvmax=None, m: types.Model = None) -> types.Data:
  """Creates a zero-initialised device Data at qpos0 (reference io.py:1680).  `m` (optional) reuses an existing device Model."""
  dev = _require_cuda()
  if m is None:
    m = put_model(mjm)
  L = _lib.lib()
  nconmax = _default_nconmax(mjm) if nconmax is None else int(nconmax)
  njmax = _default_njmax(mjm) if njmax is None else int(njmax)
  if nworld < 1:
    raise ValueError("nworld must be >= 1")
  if nconmax < 0 or njmax < 0:
    raise ValueError("nconmax and njmax must be >= 0")
  naconmax = nworld * nconmax if naconmax is None else int(naconmax)
  njmax_pad, nv_pad = _get_padded_sizes(m.nv, njmax, False)
  if m.is_sparse:
    if njmax_nnz is None:
      # every row fits: a row touches at most the dof chains of two bodies (the reference's default is a tighter heuristic,
      # io.py:1468; pass njmax_nnz to reproduce a particular capacity)
      t = m._tables
      njmax_nnz = njmax * min(m.nv, 2 * int(t["max_dof_chain"]))
    njmax_nnz = int(njmax_nnz)
  else:
    njmax_nnz = 0
  d = types.Data(nworld=nworld, naconmax=naconmax, naccdmax=0, njmax=njmax, njmax_pad=njmax_pad, njmax_nnz=njmax_nnz, nvmax=m.nv, nconmax=nconmax)
  for k, v in _alloc(_data_spec(m, nworld, naconmax, njmax, njmax_pad), dev).items():
    setattr(d, k, v)
  d.contact = types.Contact(**_alloc(_contact_spec(m, max(naconmax, 1)), dev))
  d.efc = types.Constraint(**_alloc(_efc_spec(m, nworld, max(njmax, 1), max(njmax_pad, 1)), dev))
  i32 = torch.int32
  if m.is_sparse:  # reference io.py:1803-1812: J becomes the CSR value array; the dense rows stay available as J_dense
    d.efc.J_dense = d.efc.J
    d.efc.J = torch.zeros((nworld, 1, max(njmax_nnz, 1)), dtype=torch.float32, device=dev)
    d.efc.J_rownnz = torch.zeros((nworld, max(njmax, 1)), dtype=i32, device=dev)
    d.efc.J_rowadr = torch.zeros((nworld, max(njmax, 1)), dtype=i32, device=dev)
    d.efc.J_colind = torch.zeros((nworld, 1, max(njmax_nnz, 1)), dtype=i32, device=dev)
  else:
    d.efc.J_rownnz = torch.zeros((nworld, 0), dtype=i32, device=dev)
    d.efc.J_rowadr = torch.zeros((nworld, 0), dtype=i32, device=dev)
    d.efc.J_colind = torch.zeros((nworld, 0, 0), dtype=i32, device=dev)
  # state at qpos0; static geom poses from one host kinematics pass (io.py:1815-1848)
  qpos0 = np.asarray(mjm.qpos0, dtype=np.float64)
  d.qpos.copy_(torch.from_numpy(np.tile(qpos0.astype(np.float32), (nworld, 1))))
  kin = mjcf.kinematics_np(mjm, qpos0) if hasattr(mjm, "names") else _host_kinematics(mjm, qpos0)
  d.geom_xpos.copy_(torch.from_numpy(np.tile(kin.geom_xpos.astype(np.float32), (nworld, 1, 1))))
  d.geom_xmat.copy_(torch.from_numpy(np.tile(kin.geom_xmat.astype(np.float32), (nworld, 1, 1, 1))))
  d.xquat[..., 0] = 1.0
  if getattr(m, "neq", 0):
    d.eq_active.copy_(torch.from_numpy(np.tile(np.asarray(mjm.eq_active0).astype(np.int32), (nworld, 1))))
  _reset_mocap(mjm, d)
  _bind(m, d, L)
  return d


def _reset_mocap(mjm, d):
  """mocap poses start at the bodies' model pose (reference io.py:1824-1846)"""
  if not getattr(mjm, "nmocap", 0):
    return
  mid = np.asarray(mjm.body_mocapid)
  mb = np.nonzero(mid >= 0)[0]
  order = mb[np.argsort(mid[mb])]
  d.mocap_pos.copy_(torch.from_numpy(np.tile(np.asarray(mjm.body_pos, dtype=np.float32)[order], (d.nworld, 1, 1))))
  d.mocap_quat.copy_(torch.from_numpy(np.tile(np.asarray(mjm.body_quat, dtype=np.float32)[order], (d.nworld, 1, 1))))


def _host_kinematics(mjm, qpos):
  import mujoco  # real MjModel path

  mjd = mujoco.MjData(mjm)
  mjd.qpos[:] = qpos
  mujoco.mj_kinematics(mjm, mjd)
  from types import SimpleNamespace

  return SimpleNamespace(geom_xpos=np.array(mjd.geom_xpos), geom_xmat=np.array(mjd.geom_xmat).reshape(-1, 3, 3))


def _bind(m: types.Model, d: types.Data, L):
  h = L.mjb_data_create(d.nworld, d.nconmax, d.naconmax, d.njmax, d.njmax_pad, m.nv_pad)
  d._handle = h
  d._model = m
  d._keep = []

  def reg(cname, x):
    x = _ptr_tensor(x)
    d._keep.append(x)
    _lib.check(L.mjb_data_set_array(h, cname.encode(), x.data_ptr()))

  for n in _BOUND_TOP:
    reg(n, getattr(d, n))
  for n in _BOUND_EFC:
    reg("efc_" + n, d.efc.J_dense if (n == "J" and m.is_sparse) else getattr(d.efc, n))
  reg("efc_Jsp", d.efc.J if m.is_sparse else torch.zeros(1, dtype=torch.float32, device=d.efc.J.device))
  for n in ("J_rownnz", "J_rowadr", "J_colind"):
    reg("efc_" + n, getattr(d.efc, n))
  _lib.check(L.mjb_data_set_int(h, b"njmax_nnz", int(d.njmax_nnz)))
  for n in _BOUND_CONTACT:
    reg("contact_" + n, getattr(d.contact, n))
  _lib.check(L.mjb_data_finalize(h, m._handle))
  weakref.finalize(d, L.mjb_data_destroy, h)

  def make_hook(struct, prefix, names):
    def hook(name, value):
      if name in names and name in struct.__dict__:
        value = _check_like(f"{type(struct).__name__}.{name}", value, struct.__dict__[name])
        x = _ptr_tensor(value)
        d._keep.append(x)
        _lib.check(L.mjb_data_set_array(h, (prefix + name).encode(), x.data_ptr()))
      return value

    return hook

  object.__setattr__(d, "_rebind", make_hook(d, "", set(_BOUND_TOP)))
  object.__setattr__(d.efc, "_rebind", make_hook(d.efc, "efc_", (set(_BOUND_EFC) - {"J"}) if m.is_sparse else set(_BOUND_EFC)))
  object.__setattr__(d.contact, "_rebind", make_hook(d.contact, "contact_", set(_BOUND_CONTACT)))


def put_data(mjm, mjd, nworld: int = 1, nconmax=None, nccdmax=None, njmax=None, njmax_nnz=None, naconmax=None, naccdmax=None, nvmax=None, m: types.Model = None) -> types.Data:
  """Moves host state (MjData-like: qpos, qvel, ctrl, qacc_warmstart, time, ...) to a device Data tiled over nworld (io.py:1890)."""
  d = make_data(mjm, nworld, nconmax, nccdmax, njmax, njmax_nnz, naconmax, naccdmax, nvmax, m=m)
  for name in ("qpos", "qvel", "ctrl", "qacc_warmstart", "qfrc_applied", "xfrc_applied", "act", "history"):
    if hasattr(mjd, name) and getattr(d, name).numel():
      src = np.asarray(getattr(mjd, name), dtype=np.float32)
      dst = getattr(d, name)
      dst.copy_(torch.from_numpy(np.broadcast_to(src, (nworld,) + src.shape).copy()).reshape(dst.shape))
  d.time.fill_(float(getattr(mjd, "time", 0.0)))
  return d


def reset_data(m: types.Model, d: types.Data):
  """Resets every world to qpos0 with zero velocity/ctrl/time (reference io.py:2435, all worlds).  d.history (the actuator and sensor
  delay buffers) is left untouched, as the reference leaves it; refill it with init_ctrl_history / init_sensor_history."""
  mjm = m._mjm
  d.qpos.copy_(torch.from_numpy(np.tile(np.asarray(mjm.qpos0, dtype=np.float32), (d.nworld, 1))))
  for n in ("qvel", "ctrl", "qacc_warmstart", "qacc", "qfrc_applied", "xfrc_applied", "time", "act", "act_dot"):
    getattr(d, n).zero_()
  for n in ("overflow", "solver_niter", "nefc", "ne", "nf", "nl", "nacon", "ncollision"):
    getattr(d, n).zero_()
  if getattr(m, "neq", 0):
    d.eq_active.copy_(torch.from_numpy(np.tile(np.asarray(mjm.eq_active0).astype(np.int32), (d.nworld, 1))))
  _reset_mocap(mjm, d)


def reset_data_keyframe(m: types.Model, d: types.Data, key):
  """Resets worlds to a keyframe (reference io.py:2797): an int resets every world (ValueError if out of range); an integer
  tensor of shape (nworld,) resets each world to its own keyframe and leaves worlds with an out-of-range index untouched."""
  mjm = m._mjm
  nkey = int(mjm.nkey)
  if isinstance(key, (int, np.integer)):
    if key < 0 or key >= nkey:
      raise ValueError(f"key ({int(key)}) must be in [0, {nkey}).")
    keys = torch.full((d.nworld,), int(key), dtype=torch.int64, device=d.qpos.device)
  elif isinstance(key, torch.Tensor):
    if tuple(key.shape) != (d.nworld,):
      raise ValueError(f"key array must have shape ({d.nworld},), got {tuple(key.shape)}.")
    if key.dtype not in (torch.int32, torch.int64):
      raise ValueError(f"key array must be of integer type, got {key.dtype}.")
    keys = key.to(device=d.qpos.device, dtype=torch.int64)
  else:
    raise ValueError(f"key must be an int or a tensor, got {type(key)}.")
  valid = (keys >= 0) & (keys < nkey)
  if not bool(valid.any()):
    return
  idx = keys.clamp(0, max(nkey - 1, 0))
  dev = d.qpos.device
  f32 = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).to(dev)
  sel = lambda new, old: torch.where(valid.reshape((-1,) + (1,) * (old.dim() - 1)), new, old)
  d.qpos.copy_(sel(f32(mjm.key_qpos)[idx], d.qpos))
  d.qvel.copy_(sel(f32(mjm.key_qvel)[idx], d.qvel))
  if m.nu:
    d.ctrl.copy_(sel(f32(mjm.key_ctrl)[idx], d.ctrl))
  d.time.copy_(sel(f32(mjm.key_time)[idx], d.time))
  if m.na:
    d.act.copy_(sel(f32(np.asarray(mjm.key_act).reshape(nkey, m.na))[idx], d.act))
  for n in ("qacc_warmstart", "qacc", "qfrc_applied", "xfrc_applied", "act_dot"):
    t = getattr(d, n)
    t.copy_(sel(torch.zeros_like(t), t))
  for n in ("overflow", "solver_niter", "nefc", "ne", "nf", "nl"):
    t = getattr(d, n)
    t.copy_(sel(torch.zeros_like(t), t))
  if getattr(m, "neq", 0):
    d.eq_active.copy_(sel(torch.from_numpy(np.asarray(mjm.eq_active0).astype(np.int32)).to(dev).expand(d.nworld, -1), d.eq_active))


_GET_FIELDS = (
  "qpos", "qvel", "ctrl", "qacc_warmstart", "qfrc_applied", "xfrc_applied", "qacc", "xpos", "xquat", "xmat", "xipos", "ximat", "xanchor", "xaxis",
  "geom_xpos", "geom_xmat", "site_xpos", "site_xmat", "cam_xpos", "cam_xmat", "light_xpos", "light_xdir", "subtree_com", "cdof", "cinert", "crb",
  "actuator_length", "actuator_velocity", "actuator_force", "cvel", "cdof_dot", "qfrc_bias", "qfrc_spring", "qfrc_damper", "qfrc_passive",
  "qfrc_actuator", "qfrc_smooth", "qacc_smooth", "qfrc_constraint", "cacc", "cfrc_int", "qLD", "actuator_moment",
)


def get_data_into(result, mjm, d: types.Data, world_id: int = 0):
  """Copies one world of a device Data into a host MjData-like object (reference io.py:2184): state and every computed field
  by MjData name, `M` as MuJoCo's CSR values, the world's contacts (`result.contact` as a dict of arrays, in pool order) and
  its constraint rows (`efc_*`, with `efc_J` dense nefc x nv); `ncon`, `nefc`, `ne`, `nf`, `nl`, `time`, `solver_niter`."""
  w = int(world_id)
  if not 0 <= w < d.nworld:
    raise ValueError(f"world_id {w} out of range [0, {d.nworld})")
  nacon = min(int(d.nacon.cpu()[0]), d.naconmax)
  nefc = min(int(d.nefc[w].cpu()), d.njmax)
  for name in _GET_FIELDS:
    setattr(result, name, getattr(d, name)[w].cpu().numpy().astype(np.float64))
  if d.history.shape[1] > 0:  # reference io.py:2322
    result.history = d.history[w].cpu().numpy().astype(np.float64)
  result.qM = d.M[w].cpu().numpy().astype(np.float64)
  result.M = result.qM
  result.time = float(d.time[w].cpu())
  result.solver_niter = int(d.solver_niter[w].cpu())
  result.ne, result.nf, result.nl, result.nefc = int(d.ne[w].cpu()), int(d.nf[w].cpu()), int(d.nl[w].cpu()), nefc
  ids = torch.nonzero(d.contact.worldid[:nacon] == w).reshape(-1)
  result.ncon = int(ids.numel())
  con = {}
  for name in ("dist", "pos", "frame", "includemargin", "friction", "solref", "solreffriction", "solimp", "dim", "geom", "efc_address"):
    con[name] = getattr(d.contact, name)[ids].cpu().numpy()
  result.contact = con
  nv = mjm.nv
  result.efc_J = (d.efc.J_dense if hasattr(d.efc, "J_dense") else d.efc.J)[w, :nefc, :nv].cpu().numpy().astype(np.float64)
  for name in ("pos", "margin", "D", "vel", "aref", "frictionloss", "force"):
    setattr(result, "efc_" + name, getattr(d.efc, name)[w, :nefc].cpu().numpy().astype(np.float64))
  for name in ("type", "id", "state"):
    setattr(result, "efc_" + name, getattr(d.efc, name)[w, :nefc].cpu().numpy())
  return result


def override_model(model, overrides):
  """Overrides model parameters (reference io.py:2933): `overrides` is a dict or a sequence of "key = value" strings such as
  "opt.iterations = 1", "opt.cone = pyramidal", "opt.disableflags = contact | spring".  Works on a device Model (the assignment goes
  through the rebinding hooks, so the C handle follows) and on a host MjModel-like object; fields that exist only on the other kind
  are skipped like in the reference."""
  enum_fields = {
    "opt.broadphase": types.BroadphaseType, "opt.broadphase_filter": types.BroadphaseFilter, "opt.cone": types.ConeType,
    "opt.disableflags": types.DisableBit, "opt.enableflags": types.EnableBit, "opt.integrator": types.IntegratorType, "opt.solver": types.SolverType,
  }
  mj_enum_fields = {"opt.jacobian": {"DENSE": C.JAC_DENSE, "SPARSE": C.JAC_SPARSE, "AUTO": C.JAC_AUTO}}
  mjw_only = {"opt.broadphase", "opt.broadphase_filter", "opt.graph_conditional", "opt.contact_sensor_maxmatch"}
  mj_only = {"opt.jacobian", "vis.quality.offsamples"}
  is_device = isinstance(model, types.Model)
  if not isinstance(overrides, dict):
    parsed = {}
    for o in overrides:
      if "=" not in o:
        raise ValueError(f"Invalid override format: {o}")
      k, v = o.split("=", 1)
      parsed[k.strip()] = v.strip()
    overrides = parsed
  for key, val in overrides.items():
    if key in ("opt.ls_parallel", "opt.ls_parallel_min_step"):
      raise ValueError(f"{key.split('.')[1]} was removed in MuJoCo Warp 3.9.1.")
    if (key in mjw_only and not is_device) or (key in mj_only and is_device):
      continue
    obj, attrs = model, key.split(".")
    for i, attr in enumerate(attrs):
      if not hasattr(obj, attr):
        raise ValueError(f"Unrecognized model field: {key}")
      if i < len(attrs) - 1:
        obj = getattr(obj, attr)
        continue
      cur = getattr(obj, attr)
      if key in mj_enum_fields and isinstance(val, str):
        member = val.strip().upper()
        if member not in mj_enum_fields[key]:
          raise ValueError(f"Unrecognized enum value for {key}: {member}")
        val = mj_enum_fields[key][member]
      elif key in enum_fields and isinstance(val, str):
        acc = 0
        for member in val.split("|"):
          member = member.strip().upper()
          if member not in enum_fields[key].__members__:
            raise ValueError(f"Unrecognized enum value for {enum_fields[key].__name__}: {member}")
          acc |= int(enum_fields[key][member])
        val = acc
      elif isinstance(cur, bool) and isinstance(val, str):
        if val.upper() not in ("TRUE", "FALSE"):
          raise ValueError(f"Unrecognized value for field: {key}")
        val = val.upper() == "TRUE"
      elif isinstance(cur, torch.Tensor) and isinstance(val, str):
        floats = [float(p) for p in val.strip("[]").split()]
        val = torch.tensor(floats, dtype=cur.dtype, device=cur.device).reshape(cur.shape)
      elif isinstance(cur, np.ndarray) and isinstance(val, str):
        val = np.array([float(p) for p in val.strip("[]").split()], dtype=cur.dtype)
      elif isinstance(cur, torch.Tensor):
        val = torch.as_tensor(val, dtype=cur.dtype, device=cur.device).reshape(cur.shape)
      else:
        val = type(cur)(val)
      setattr(obj, attr, val)


def load_trajectory(npz_path: str, mjm, mjd) -> np.ndarray:
  """Loads a ctrl sequence and samples it on the model timestep with zero-order hold (reference io.py:3067-3113).

  Sets mjd.qpos/qvel from the file's first frame when present.  `times` holds one timestamp per control or the
  interval boundaries (one extra)."""
  data = np.load(npz_path)
  ctrl, times = data["ctrl"], data["times"]
  if ctrl.ndim != 2 or len(ctrl) == 0:
    raise ValueError(f"ctrl must have shape (nstep, nu) with nstep > 0, got {ctrl.shape}")
  if ctrl.shape[1] != mjm.nu:
    raise ValueError(f"ctrl shape {ctrl.shape} does not match model nu={mjm.nu}")
  if times.ndim != 1 or len(times) not in (len(ctrl), len(ctrl) + 1):
    raise ValueError(f"times shape {times.shape} must contain {len(ctrl)} or {len(ctrl) + 1} timestamps")
  if not np.all(np.isfinite(times)):
    raise ValueError("times must be finite")
  intervals = np.diff(times)
  if np.any(intervals <= 0):
    raise ValueError("times must be strictly increasing")
  if "qpos" in data and data["qpos"].shape[1] == mjm.nq:
    mjd.qpos[:] = data["qpos"][0]
  if "qvel" in data and data["qvel"].shape[1] == mjm.nv:
    mjd.qvel[:] = data["qvel"][0]
  if len(times) == len(ctrl):
    final_dt = intervals[-1] if len(intervals) else mjm.opt.timestep
    times = np.append(times, times[-1] + final_dt)
  n_steps = int(np.round((times[-1] - times[0]) / mjm.opt.timestep))
  sample_times = times[0] + (np.arange(n_steps) + 1e-7) * mjm.opt.timestep
  return ctrl[np.searchsorted(times, sample_times, side="right") - 1]
