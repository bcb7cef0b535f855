"""A numpy per-world restatement of set_const (reference set_const.py:35-950) on top of mjcf.kinematics_np / dense_inertia_np.

`oracle(mjm, inputs, nworld)` evaluates set_const(m, d) with every output field batched to nworld: world w uses the model with the
per-world inputs of `inputs` (field -> (nworld, ...)) at entry w, and its results are entry w of each output.  Dense M^-1 in double
precision; camera / light poses at qpos0 follow the reference's camlight (smooth.py _cam_local_to_global / _light_local_to_global).
"""
import copy

import numpy as np

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf

MJ_MINVAL = 1e-15


def _world_model(mjm, inputs, w):
  mw = copy.copy(mjm)
  for f, v in inputs.items():
    setattr(mw, f, np.array(v[w], dtype=np.float64))
  for f in ("body_mass", "qpos0", "qpos_spring", "eq_data", "tendon_lengthspring", "actuator_biasprm", "cam_pos0", "cam_poscom0", "cam_mat0",
            "light_pos0", "light_poscom0", "light_dir0"):
    if hasattr(mw, f):
      setattr(mw, f, np.array(getattr(mw, f), dtype=np.float64))
  return mw


def _subtreemass(mw):
  sub = np.array(mw.body_mass, dtype=np.float64)
  for b in range(mw.nbody - 1, 0, -1):
    sub[mw.body_parentid[b]] += sub[b]
  return sub


def _camlight(mw, kin):
  """cam_xpos / cam_xmat / light_xpos / light_xdir at the configuration of kin (reference smooth.py camlight)."""
  cam_xpos, cam_xmat = np.zeros((mw.ncam, 3)), np.zeros((mw.ncam, 3, 3))
  cam_pos0 = np.asarray(mw.cam_pos0).reshape(-1, 3)
  cam_poscom0 = np.asarray(mw.cam_poscom0).reshape(-1, 3)
  cam_mat0 = np.asarray(mw.cam_mat0).reshape(-1, 3, 3)
  for c in range(mw.ncam):
    b, mode, tb = mw.cam_bodyid[c], mw.cam_mode[c], mw.cam_targetbodyid[c]
    fixed_pose = lambda: (kin.xpos[b] + mjcf.rot_vec(kin.xquat[b], mw.cam_pos[c]), mjcf.quat_to_mat(mjcf.quat_mul(kin.xquat[b], mw.cam_quat[c])))
    if mode in (C.CAMLIGHT_TARGETBODY, C.CAMLIGHT_TARGETBODYCOM) and tb < 0:
      cam_xpos[c], cam_xmat[c] = fixed_pose()
    elif mode == C.CAMLIGHT_TRACK:
      cam_xpos[c], cam_xmat[c] = kin.xpos[b] + cam_pos0[c], cam_mat0[c]
    elif mode == C.CAMLIGHT_TRACKCOM:
      cam_xpos[c], cam_xmat[c] = kin.subtree_com[b] + cam_poscom0[c], cam_mat0[c]
    elif mode in (C.CAMLIGHT_TARGETBODY, C.CAMLIGHT_TARGETBODYCOM):
      cam_xpos[c] = kin.xpos[b] + mjcf.rot_vec(kin.xquat[b], mw.cam_pos[c])
      pos = kin.subtree_com[tb] if mode == C.CAMLIGHT_TARGETBODYCOM else kin.xpos[tb]
      n = lambda v: v / np.linalg.norm(v)
      m3 = n(cam_xpos[c] - pos)
      m1 = n(np.cross([0.0, 0.0, 1.0], m3))
      m2 = n(np.cross(m3, m1))
      cam_xmat[c] = np.stack([m1, m2, m3], axis=1)
    else:
      cam_xpos[c], cam_xmat[c] = fixed_pose()
  light_xpos, light_xdir = np.zeros((mw.nlight, 3)), np.zeros((mw.nlight, 3))
  light_pos0 = np.asarray(mw.light_pos0).reshape(-1, 3)
  light_poscom0 = np.asarray(mw.light_poscom0).reshape(-1, 3)
  light_dir0 = np.asarray(mw.light_dir0).reshape(-1, 3)
  for i in range(mw.nlight):
    b, mode = mw.light_bodyid[i], mw.light_mode[i]
    if mode == C.CAMLIGHT_TRACK:
      light_xpos[i], light_xdir[i] = kin.xpos[b] + light_pos0[i], light_dir0[i]
    elif mode == C.CAMLIGHT_TRACKCOM:
      light_xpos[i], light_xdir[i] = kin.subtree_com[b] + light_poscom0[i], light_dir0[i]
    elif mode in (C.CAMLIGHT_TARGETBODY, C.CAMLIGHT_TARGETBODYCOM) and mw.light_targetbodyid[i] >= 0:
      tb = mw.light_targetbodyid[i]
      light_xpos[i] = kin.xpos[b] + mjcf.rot_vec(kin.xquat[b], mw.light_pos[i])
      pos = kin.subtree_com[tb] if mode == C.CAMLIGHT_TARGETBODYCOM else kin.xpos[tb]
      light_xdir[i] = (pos - light_xpos[i]) / np.linalg.norm(pos - light_xpos[i])
    else:  # fixed, or aimed at no body
      light_xpos[i] = kin.xpos[b] + mjcf.rot_vec(kin.xquat[b], mw.light_pos[i])
      light_xdir[i] = mjcf.rot_vec(kin.xquat[b], mw.light_dir[i])
  return cam_xpos, cam_xmat, light_xpos, light_xdir


def _moment_rows(mw):
  """Dense actuator moment rows at any configuration (joint and fixed-tendon transmissions are configuration independent)."""
  rows = np.zeros((mw.nu, mw.nv))
  for i in range(mw.nu):
    j, g = mw.actuator_trnid[i, 0], mw.actuator_gear[i, 0]
    if mw.actuator_trntype[i] == C.TRN_TENDON:
      rows[i] = g * mjcf._tendon_row(mw, j)
    else:
      rows[i, mw.jnt_dofadr[j]] = g
  return rows


def _ten_length(mw, qpos, t):
  return sum(mw.wrap_prm[k] * qpos[mw.jnt_qposadr[mw.wrap_objid[k]]] for k in range(mw.tendon_adr[t], mw.tendon_adr[t] + mw.tendon_num[t]))


def world(mjm, inputs, w, subtreemass=None):
  """set_const's outputs of world w (a dict), with body_subtreemass as the chain sees it (default: world w's own)."""
  mw = _world_model(mjm, inputs, w)
  out = {"body_subtreemass": _subtreemass(mw)}
  mw.body_subtreemass = out["body_subtreemass"] if subtreemass is None else subtreemass
  nv, nbody = mw.nv, mw.nbody
  kin = mjcf.kinematics_np(mw, mw.qpos0)
  M, jacp, jacr = mjcf.dense_inertia_np(mw, kin)
  Minv = np.linalg.inv(M)
  out["meaninertia"] = np.trace(M) / nv
  dg = np.diag(Minv)
  dofw = np.zeros(nv)
  for j in range(mw.njnt):
    a, t = mw.jnt_dofadr[j], mw.jnt_type[j]
    if t == C.JNT_FREE:
      dofw[a : a + 3], dofw[a + 3 : a + 6] = dg[a : a + 3].mean(), dg[a + 3 : a + 6].mean()
    elif t == C.JNT_BALL:
      dofw[a : a + 3] = dg[a : a + 3].mean()
    else:
      dofw[a] = dg[a]
  out["dof_invweight0"] = dofw
  bw = np.zeros((nbody, 2))
  for b in range(1, nbody):
    if mw.body_weldid[b] == 0:
      continue
    tr, rot = np.trace(jacp[b] @ Minv @ jacp[b].T) / 3, np.trace(jacr[b] @ Minv @ jacr[b].T) / 3
    if tr < MJ_MINVAL and rot > MJ_MINVAL:
      tr = rot
    elif rot < MJ_MINVAL and tr > MJ_MINVAL:
      rot = tr
    bw[b] = tr, rot
  out["body_invweight0"] = bw
  nt = int(getattr(mw, "ntendon", 0))
  out["tendon_length0"] = np.array([_ten_length(mw, mw.qpos0, t) for t in range(nt)])
  out["tendon_invweight0"] = np.array([mjcf._tendon_row(mw, t) @ Minv @ mjcf._tendon_row(mw, t) for t in range(nt)])
  if int(getattr(mw, "neq", 0)):
    mw.eq_data = np.array(mw.eq_data, dtype=np.float64).reshape(mw.neq, 11)
    mjcf._set_eq_data0(mw, kin)
    out["eq_data"] = mw.eq_data
  else:
    out["eq_data"] = np.zeros((0, 11))
  cam_xpos, cam_xmat, light_xpos, light_xdir = _camlight(mw, kin)
  tgt = lambda tb, b: tb if tb >= 0 else b
  out["cam_pos0"] = np.array([cam_xpos[c] - kin.xpos[mw.cam_bodyid[c]] for c in range(mw.ncam)]).reshape(mw.ncam, 3)
  out["cam_poscom0"] = np.array([cam_xpos[c] - kin.subtree_com[tgt(mw.cam_targetbodyid[c], mw.cam_bodyid[c])] for c in range(mw.ncam)]).reshape(mw.ncam, 3)
  out["cam_mat0"] = cam_xmat.reshape(mw.ncam, 3, 3)
  out["light_pos0"] = np.array([light_xpos[i] - kin.xpos[mw.light_bodyid[i]] for i in range(mw.nlight)]).reshape(mw.nlight, 3)
  out["light_poscom0"] = np.array([light_xpos[i] - kin.subtree_com[tgt(mw.light_targetbodyid[i], mw.light_bodyid[i])] for i in range(mw.nlight)]).reshape(mw.nlight, 3)
  out["light_dir0"] = light_xdir.reshape(mw.nlight, 3)
  mom = _moment_rows(mw)
  out["actuator_acc0"] = np.array([np.linalg.norm(Minv @ mom[i]) for i in range(mw.nu)])
  bp = np.array(mw.actuator_biasprm, dtype=np.float64).reshape(mw.nu, 10)
  gp = np.asarray(mw.actuator_gainprm, dtype=np.float64).reshape(mw.nu, 10)
  dM0 = np.diag(M)
  for i in range(mw.nu):
    if mw.actuator_biastype[i] != C.BIAS_AFFINE or abs(gp[i, 0] + bp[i, 1]) > MJ_MINVAL or bp[i, 2] <= 0:
      continue
    mass = sum(dM0[j] / mom[i, j] ** 2 for j in range(nv) if abs(mom[i, j]) > MJ_MINVAL)
    bp[i, 2] = -bp[i, 2] * 2 * np.sqrt(gp[i, 0] * mass)
  out["actuator_biasprm"] = bp
  ls = np.array(mw.tendon_lengthspring, dtype=np.float64).reshape(nt, 2) if nt else np.zeros((0, 2))
  for t in range(nt):
    if ls[t, 0] == -1.0 and ls[t, 1] == -1.0:
      ls[t] = _ten_length(mw, mw.qpos_spring, t)
  out["tendon_lengthspring"] = ls
  return out


def oracle(mjm, inputs, nworld):
  """{field: (nworld, ...)} plus "meaninertia" (world 0) for set_const with every output batched to nworld."""
  per = [world(mjm, inputs, w) for w in range(nworld)]
  out = {k: np.stack([p[k] for p in per]) for k in per[0] if k != "meaninertia"}
  out["meaninertia"] = per[0]["meaninertia"]
  return out
