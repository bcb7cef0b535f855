"""Host-side checks of the body-stage functions (rne_postconstraint, subtree_vel, jac, xfrc_accumulate, tendon, deriv_smooth_vel).

- The Python wrappers refuse bad arguments with a ValueError before they reach the C library (a stub library records every call).
- An fp64 numpy restatement of jac and xfrc_accumulate, fed the reference's own kinematics, reproduces the reference's outputs in
  tests/golden/body_stage_*.npz: the per-dof formula the kernels share is the reference's.
- The device fragments themselves (k_body_subtree_vel.cuh, k_body_rne_post.cuh, k_body_jac.cuh, k_body_xfrc.cuh), built for the host by
  tests/host_harness/body_stages_host.cpp with the warp's lanes as threads, reproduce the same fixtures from the reference's kinematics:
  subtree_vel, jac and xfrc_accumulate in every scene; rne_postconstraint in the scenes without equality rows or contacts (the GPU tests
  cover those).
- The public names are exported.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from tests import body_stage_scenes as S


def _golden(name):
  return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"body_stage_{name}.npz"))


def _ancestor(mjm):
  """body_isdofancestor[b, dof]: dof moves body b"""
  nb, nv = mjm.nbody, mjm.nv
  anc = np.zeros((nb, nv), dtype=bool)
  for b in range(nb):
    p = b
    while p > 0:
      anc[b, np.asarray(mjm.dof_bodyid) == p] = True
      p = int(mjm.body_parentid[p])
  return anc


def jac_np(mjm, cdof, scom, point, body):
  """support.py:506 jac_dof for every dof: (3, nv) translational and rotational Jacobians of point on body"""
  nv = mjm.nv
  jp, jr = np.zeros((3, nv)), np.zeros((3, nv))
  anc = _ancestor(mjm)[body]
  off = point - scom[int(mjm.body_rootid[body])]
  for v in np.nonzero(anc)[0]:
    jr[:, v] = cdof[v, :3]
    jp[:, v] = cdof[v, 3:] + np.cross(cdof[v, :3], off)
  return jp, jr


def xfrc_np(mjm, cdof, scom, xipos, xfrc):
  """support.py:273-301 _apply_ft: J^T xfrc_applied summed over the bodies each dof moves"""
  q = np.zeros(mjm.nv)
  for b in range(1, mjm.nbody):
    jp, jr = jac_np(mjm, cdof, scom, xipos[b], b)
    q += jp.T @ xfrc[b, :3] + jr.T @ xfrc[b, 3:]
  return q


@pytest.mark.parametrize("scene", list(S.SCENES))
def test_jac_and_xfrc_restatement_meets_the_reference(scene):
  g, mjm = _golden(scene), S.load(scene)
  cdof, scom, xipos = g["fwd/cdof"], g["fwd/subtree_com"], g["fwd/xipos"]
  for w in range(S.NWORLD):
    jp, jr = jac_np(mjm, cdof[w], scom[w], g["in/point"][w], int(g["in/body"][w]))
    np.testing.assert_allclose(jp, g["out/jacp"][w], atol=1e-9)
    np.testing.assert_allclose(jr, g["out/jacr"][w], atol=1e-9)
    q = g["in/qfrc"][w] + xfrc_np(mjm, cdof[w], scom[w], xipos[w], g["in/xfrc_applied"][w])
    np.testing.assert_allclose(q, g["out/qfrc"][w], atol=1e-9)
  assert int(g["in/body"][0]) == 0 and not g["out/jacp"][0].any()
  assert np.abs(g["in/xfrc_applied"]).max() > 0 and not np.allclose(g["out/qfrc"], g["in/qfrc"])


def test_body_stage_fixtures_cover_the_issue_cases():
  """contacts in the humanoid and G1 scenes, equality rows, tendons, fluid and per-world fields"""
  assert int(_golden("humanoid_pyramidal")["fwd/nacon"][0]) > 0 and int(_golden("g1")["fwd/nacon"][0]) > 0
  assert (_golden("equality")["fwd/ne"] > 0).all()
  assert _golden("tendon_actuator")["out/ten_length"].shape[1] == 2
  assert S.load("g1").nv > 32
  # the water scenes tell the symmetrized fluid derivative of implicitfast from the plain one of Euler / RK4
  e, f = _golden("fluid_water_euler")["out/deriv"], _golden("fluid_water_implicitfast")["out/deriv"]
  assert np.abs(e - f).max() > 5e-3 * np.abs(e).max()  # 25 times the GPU tests' tolerance
  b = _golden("batched")
  assert not np.allclose(b["in/body_mass"][0], b["in/body_mass"][1])


class _Stub:
  def __init__(self):
    self.calls = []

  def __getattr__(self, name):
    def f(*a, **k):
      self.calls.append(name)
      return 0

    return f


class _Fake:
  def __init__(self, nworld, nv, nC):
    self.nworld, self.nv, self.nC, self._handle, self._model = nworld, nv, nC, 1, None


def test_wrappers_refuse_bad_arguments_before_the_library(monkeypatch):
  from mujoco_warp_b200._src import _lib
  from mujoco_warp_b200._src import forward as F

  stub = _Stub()
  monkeypatch.setattr(_lib, "lib", lambda: stub)
  m, d = _Fake(4, 9, 30), _Fake(4, 9, 30)
  f32 = lambda *s: torch.zeros(s, dtype=torch.float32)
  i32 = torch.zeros(4, dtype=torch.int32)
  bad = [
    lambda: F.jac(m, d, f32(4, 3, 9), None, f32(4, 3), i32),  # host tensors
    lambda: F.jac(m, d, None, None, f32(4, 2), i32),
    lambda: F.jac(m, d, None, None, f32(4, 3), torch.zeros(4, dtype=torch.int64)),
    lambda: F.jac(m, d, f32(4, 3, 8), None, f32(4, 3), i32),
    lambda: F.jac(m, d, None, f32(3, 9, 4).permute(2, 0, 1), f32(4, 3), i32),
    lambda: F.xfrc_accumulate(m, d, f32(4, 8)),
    lambda: F.xfrc_accumulate(m, d, torch.zeros((4, 9), dtype=torch.float64)),
    lambda: F.deriv_smooth_vel(m, d, f32(4, 29)),
    lambda: F.deriv_smooth_vel(m, d, f32(30, 4).t()),
  ]
  for call in bad:
    with pytest.raises(ValueError):
      call()
  assert stub.calls == []


def test_public_names():
  import mujoco_warp_b200 as mjw

  for name in ("rne_postconstraint", "subtree_vel", "jac", "xfrc_accumulate", "tendon", "deriv_smooth_vel", "ObjType"):
    assert hasattr(mjw, name), name
  assert int(mjw.ObjType.BODY) == 1 and int(mjw.ObjType.XBODY) == 2 and int(mjw.ObjType.GEOM) == 5 and int(mjw.ObjType.SITE) == 6
  assert int(mjw.ObjType.CAMERA) == 7 and int(mjw.ObjType.FLEX) == 9 and int(mjw.ObjType.UNKNOWN) == 0
  from mujoco_warp_b200._src import _lib

  declared = set(_lib.exported_symbols_in_header())
  for f in ("mjb_rne_postconstraint", "mjb_subtree_vel", "mjb_jac", "mjb_xfrc_accumulate", "mjb_tendon", "mjb_deriv_smooth_vel"):
    assert f in declared, f


HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_harness", "body_stages_host.cpp")
OUT = os.path.join(HERE, "host_harness", "_build", "libbody_stages_host.so")
IARRS = ["body_parentid", "body_rootid", "body_dofnum", "body_dofadr", "body_childadr", "body_childid", "level_adr", "level_body", "dof_bodyid",
         "body_isdofancestor"]
FARRS = ["body_mass", "body_inertia", "body_subtreemass"]
DARRS = ["cvel", "ximat", "xipos", "subtree_com", "cdof", "cdof_dot", "cinert", "qvel", "qacc", "xfrc_applied", "xmat", "xpos"]


@pytest.fixture(scope="module")
def harness():
  os.makedirs(os.path.dirname(OUT), exist_ok=True)
  cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
  subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-std=c++20", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", OUT, "-lpthread"],
                 check=True)
  L = ctypes.CDLL(OUT)
  for f in ("bsh_subtree_vel", "bsh_rne_postconstraint", "bsh_jac", "bsh_xfrc_accumulate"):
    getattr(L, f).restype = None
  return L


class _World:
  """the ctypes arguments of one world of a fixture: sizes, gravity and the model / data arrays (fp32 copies kept alive)"""

  def __init__(self, mjm, g, w):
    from mujoco_warp_b200._src import io as mio

    t = mio.derive_tables(mjm)
    src = lambda k: t[k] if k in t else getattr(mjm, k)
    self.keep = []
    ptr = lambda a, ty: self._keep(np.ascontiguousarray(a, dtype=ty)).ctypes.data_as(ctypes.c_void_p)
    self.sizes = (ctypes.c_int * 4)(mjm.nbody, mjm.nv, int(t["nlevel"]), 0)
    self.gravity = (ctypes.c_float * 3)(*[float(x) for x in mjm.opt.gravity])
    self.iarr = (ctypes.c_void_p * len(IARRS))(*[ptr(np.asarray(src(k)).reshape(-1), np.int32) for k in IARRS])
    farr = {k: np.asarray(getattr(mjm, k)) for k in FARRS}
    if S.SCENES_BATCHED.get(g["_scene"], False):
      farr["body_mass"], farr["body_inertia"] = g["in/body_mass"][w], g["in/body_inertia"][w]
    self.farr = (ctypes.c_void_p * len(FARRS))(*[ptr(farr[k].reshape(-1), np.float32) for k in FARRS])
    dat = {k: g[f"fwd/{k}"][w] for k in DARRS if f"fwd/{k}" in g}
    dat["qvel"], dat["xfrc_applied"] = g["in/qvel"][w], g["in/xfrc_applied"][w]
    self.darr = (ctypes.c_void_p * len(DARRS))(*[ptr(np.asarray(dat[k]).reshape(-1), np.float32) for k in DARRS])

  def _keep(self, a):
    self.keep.append(a)
    return a

  def args(self):
    return (self.sizes, self.gravity, self.iarr, self.farr, self.darr)


def _fixture(scene):
  g = dict(_golden(scene))
  g["_scene"] = scene
  return g


def _f32(shape):
  return np.zeros(shape, dtype=np.float32)


def _p(a):
  return a.ctypes.data_as(ctypes.c_void_p)


def _near(name, got, want, tol=2e-4):
  err = np.abs(got - want).max() if want.size else 0.0
  assert err <= tol * max(1.0, float(np.abs(want).max()) if want.size else 1.0), f"{name}: off by {err}"


@pytest.mark.parametrize("scene", list(S.SCENES))
def test_device_fragments_on_the_host_meet_the_reference(harness, scene):
  g, mjm = _fixture(scene), S.load(scene)
  nb, nv = mjm.nbody, mjm.nv
  for w in range(S.NWORLD):
    W = _World(mjm, g, w)
    lin, ang = _f32((nb, 3)), _f32((nb, 3))
    harness.bsh_subtree_vel(*W.args(), _p(lin), _p(ang))
    _near(f"{scene} w{w} subtree_linvel", lin, g["out/subtree_linvel"][w])
    _near(f"{scene} w{w} subtree_angmom", ang, g["out/subtree_angmom"][w])
    jp, jr = _f32((3, nv)), _f32((3, nv))
    pt = np.ascontiguousarray(g["in/point"][w], dtype=np.float32)
    harness.bsh_jac(*W.args(), _p(pt), int(g["in/body"][w]), _p(jp), _p(jr))
    _near(f"{scene} w{w} jacp", jp, g["out/jacp"][w])
    _near(f"{scene} w{w} jacr", jr, g["out/jacr"][w])
    q = np.ascontiguousarray(g["in/qfrc"][w], dtype=np.float32)
    harness.bsh_xfrc_accumulate(*W.args(), _p(q))
    _near(f"{scene} w{w} qfrc", q, g["out/qfrc"][w])
    if int(g["fwd/ne"][w]) == 0 and int(g["fwd/nacon"][0]) == 0:
      cacc, cint, cext = _f32((nb, 6)), _f32((nb, 6)), _f32((nb, 6))
      harness.bsh_rne_postconstraint(*W.args(), _p(cacc), _p(cint), _p(cext))
      _near(f"{scene} w{w} cfrc_ext", cext, g["out/cfrc_ext"][w])
      _near(f"{scene} w{w} cacc", cacc, g["out/cacc"][w])
      _near(f"{scene} w{w} cfrc_int", cint, g["out/cfrc_int"][w])
