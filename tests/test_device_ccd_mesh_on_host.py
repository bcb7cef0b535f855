"""Mesh geoms in the CUDA convex-collision header (mjb_ccd.cuh built with CCD_MESH=1), run on the host through tests/host_harness:
hull-vertex support function (exhaustive and hull-graph hill climbing, cached start vertex), discrete GJK / EPA and mesh multi-contact
against the oracle, which is pinned on the reference pipeline's `mesh` scene.  The product library is still built without CCD_MESH (the
collision kernel does not carry mesh tables yet); this keeps the device routines ready and checked."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from mujoco_warp_b200._src import mjcf
from oracle import orc
from tests import util
from tests.test_device_ccd_on_host import CSRC, HERE, SRC, rand_rot
from tests.test_oracle_gjk_vectors import CASES, check, posed_geoms

OUT = os.path.join(HERE, "host_harness", "_build", "libccd_host_mesh.so")
GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH = 2, 3, 4, 5, 6, 7
V, F, I = ctypes.c_void_p, ctypes.c_float, ctypes.c_int


class Desc(ctypes.Structure):
  _fields_ = [("type", I), ("vertnum", I), ("polynum", I), ("pad", I)] + [(n, V) for n in (
    "size", "pos", "mat", "vert", "polynormal", "graph", "polyvertadr", "polyvertnum", "polyvert", "polymapadr", "polymapnum", "polymap")]


@pytest.fixture(scope="module")
def hlib():
  deps = [SRC] + [os.path.join(CSRC, f) for f in ("mjb_ccd.cuh", "mjb_colliders.cuh", "mjb_math.cuh", "mjb_types.cuh")]
  if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-DCCD_MESH=1", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", OUT], check=True)
  lib = ctypes.CDLL(OUT)
  lib.hccd_pair.restype = ctypes.c_int
  lib.hccd_pair.argtypes = [I, V, V, V, I, V, V, V, F, F, F, I, I, V, V, V, V]
  lib.hccd_desc.restype = ctypes.c_int
  lib.hccd_desc.argtypes = [V, V, F, F, F, I, I, V, V, V, V]
  return lib


@pytest.fixture(scope="module")
def model():
  return mjcf.load_string(util.mesh_xml())


def make_desc(mjm, g, pos, mat, real):
  """Descriptor of geom g posed at (pos, mat): mesh tables offset to the geom's mesh the way the oracle's fill_cgeom does."""
  keep = []
  def ptr(a, dt):
    a = np.ascontiguousarray(np.asarray(a).astype(dt)); keep.append(a)
    return a.ctypes.data_as(V)
  d = Desc()
  d.type = int(mjm.geom_type[g])
  d.size, d.pos, d.mat = ptr(mjm.geom_size[g], real), ptr(pos, real), ptr(np.asarray(mat).reshape(-1), real)
  if d.type == GEOM_MESH:
    mid = int(mjm.geom_dataid[g]); vadr, padr = int(mjm.mesh_vertadr[mid]), int(mjm.mesh_polyadr[mid])
    d.vertnum, d.polynum = int(mjm.mesh_vertnum[mid]), int(mjm.mesh_polynum[mid])
    d.vert = ptr(np.asarray(mjm.mesh_vert).reshape(-1, 3)[vadr:], real)
    d.polynormal = ptr(np.asarray(mjm.mesh_polynormal).reshape(-1, 3)[padr:], real)
    gadr = int(mjm.mesh_graphadr[mid])
    d.graph = ptr(np.asarray(mjm.mesh_graph)[gadr:], np.int32) if gadr >= 0 else None
    d.polyvertadr, d.polyvertnum = ptr(np.asarray(mjm.mesh_polyvertadr)[padr:], np.int32), ptr(np.asarray(mjm.mesh_polyvertnum)[padr:], np.int32)
    d.polyvert = ptr(mjm.mesh_polyvert, np.int32)
    d.polymapadr, d.polymapnum = ptr(np.asarray(mjm.mesh_polymapadr)[vadr:], np.int32), ptr(np.asarray(mjm.mesh_polymapnum)[vadr:], np.int32)
    d.polymap = ptr(mjm.mesh_polymap, np.int32)
  return d, keep


def run_pair(hlib, mjm, g1, p1, m1, g2, p2, m2, iterations=35):
  out = {}
  for tag, real in (("dev", np.float32), ("o32", np.float32), ("o64", np.float64)):
    d1, k1 = make_desc(mjm, g1, p1, m1, real)
    d2, k2 = make_desc(mjm, g2, p2, m2, real)
    dist = np.zeros(1, real); w1 = np.zeros((4, 3), real); w2 = np.zeros((4, 3), real); ovf = np.zeros(1, np.int32)
    P = lambda a: a.ctypes.data_as(V)
    if tag == "dev":
      n = hlib.hccd_desc(ctypes.byref(d1), ctypes.byref(d2), 0.0, 1e-6, 1e30, iterations, iterations, P(dist), P(w1), P(w2), P(ovf))
    else:
      lib = orc._lib(np.dtype(real).itemsize)
      c_real = ctypes.c_double if real is np.float64 else ctypes.c_float
      lib.orc_ccd_desc.restype = ctypes.c_int
      lib.orc_ccd_desc.argtypes = [V, V, c_real, c_real, c_real, I, I, I, V, V, V, V]
      n = lib.orc_ccd_desc(ctypes.byref(d1), ctypes.byref(d2), 0.0, 1e-6, 1e30, iterations, iterations, 1, P(dist), P(w1), P(w2), P(ovf))
    out[tag] = (float(dist[0]), int(n), w1.astype(np.float64), w2.astype(np.float64), int(ovf[0]))
  return out


def same_points(a, b, n, tol):
  """Two contact sets agree as sets (the order follows polygon vertex order on both sides, so in practice it is the same order too)."""
  a, b = a[:n], b[:n]
  used = set()
  for p in a:
    j = min((k for k in range(n) if k not in used), key=lambda k: np.linalg.norm(b[k] - p))
    assert np.linalg.norm(b[j] - p) <= tol, (a, b)
    used.add(j)


@pytest.mark.parametrize("name", sorted(CASES))
def test_mesh_build_keeps_the_analytic_vectors(hlib, name):
  """The CCD_MESH build (16-bit vertex ids, larger polygon buffers) gives the reference's answers on the known-answer vectors too."""
  from tests.test_device_ccd_on_host import device_ccd

  case = CASES[name]
  g1, g2 = posed_geoms(case)
  dist, ncon, w1, w2, ovf = device_ccd(hlib, g1, g2, iterations=case.get("iterations", 35))
  assert ovf == 0
  exp = dict(case)
  if g1[0] == GEOM_BOX and g2[0] == GEOM_BOX and not case.get("multiccd", False):
    exp.pop("ncon", None)
  if dist == 0.0 and "dist_less" in exp:
    return
  check(exp, dist, ncon, w1, w2)


def scene_pose(mjm):
  kin = mjcf.kinematics_np(mjm, mjm.qpos0)
  return np.asarray(kin.geom_xpos, dtype=np.float64).reshape(-1, 3), np.asarray(kin.geom_xmat, dtype=np.float64).reshape(-1, 9)


def test_mesh_pairs_of_the_scene(hlib, model):
  """Every mesh-involving convex pair of the `mesh` fixture scene at its initial pose (resting / slightly penetrating stacks)."""
  mjm = model
  xpos, xmat = scene_pose(mjm)
  names = {n: i for i, n in enumerate(mjm.geom_names)} if hasattr(mjm, "geom_names") else None
  ng = mjm.ngeom
  npen = nmulti = 0
  for g1 in range(ng):
    for g2 in range(ng):
      t1, t2 = int(mjm.geom_type[g1]), int(mjm.geom_type[g2])
      if g1 == g2 or t1 > t2 or (t1 == t2 and g1 > g2) or t2 != GEOM_MESH or t1 < GEOM_SPHERE:
        continue
      if np.linalg.norm(xpos[g1] - xpos[g2]) > 0.4:
        continue
      r = run_pair(hlib, mjm, g1, xpos[g1], xmat[g1], g2, xpos[g2], xmat[g2])
      dd, dn, dw1, dw2, dovf = r["dev"]
      od, on, ow1, ow2, oovf = r["o64"]
      assert dovf == 0 and oovf == 0
      curved = t1 in (GEOM_ELLIPSOID,)
      assert abs(dd - od) <= (2e-3 if curved else 2e-5), (g1, g2, dd, od)
      if od < 0:
        npen += 1
        assert dn == on, (g1, g2, dn, on)
        if on > 1:
          nmulti += 1
          same_points(0.5 * (dw1 + dw2), 0.5 * (ow1 + ow2), on, 1e-4)
  print('scene pairs: penetrating', npen, 'multi-contact', nmulti)
  assert npen >= 4 and nmulti >= 2, (npen, nmulti)


def test_mesh_pairs_random_poses(hlib, model):
  """Random relative poses of (wedge | cube | blob | box) against (cube | blob | wedge): depth, contact count and contact patch vs the fp64 oracle; the fp32
  oracle as a second opinion where fp32 and fp64 take different branches at a degenerate feature."""
  mjm = model
  types = np.asarray(mjm.geom_type)
  meshes = [g for g in range(mjm.ngeom) if types[g] == GEOM_MESH]
  firsts = meshes + [g for g in range(mjm.ngeom) if types[g] in (GEOM_BOX, GEOM_SPHERE, GEOM_CAPSULE, GEOM_CYLINDER)]
  rng = np.random.default_rng(11)
  ntot = nhit = nagree = 0
  for g1 in firsts:
    for g2 in meshes:
      if g1 == g2 or (types[g1] == GEOM_MESH and g1 > g2):
        continue
      for _ in range(12):
        p1, m1 = np.zeros(3), rand_rot(rng)
        p2, m2 = rng.normal(size=3) * 0.08, rand_rot(rng)
        r = run_pair(hlib, mjm, g1, p1, m1, g2, p2, m2)
        dd, dn, dw1, dw2, dovf = r["dev"]
        od, on, ow1, ow2, oovf = r["o64"]
        fd, fn, fw1, fw2, _ = r["o32"]
        assert dovf == 0
        ntot += 1
        ok64 = abs(dd - od) <= 5e-5 and (od >= 0 or dn == on)
        ok32 = abs(dd - fd) <= 5e-5 and (fd >= 0 or dn == fn)
        assert ok64 or ok32, (g1, g2, (dd, dn), (od, on), (fd, fn))
        nagree += ok64
        if od < 0 and ok64:
          nhit += 1
          if on > 1:
            same_points(0.5 * (dw1 + dw2), 0.5 * (ow1 + ow2), on, 2e-4)
  print('random poses:', ntot, 'penetrating', nhit, 'agree with fp64 oracle', nagree)
  assert nhit >= 30 and nagree >= 0.95 * ntot, (ntot, nhit, nagree)


def test_mesh_build_compiles_for_sm_90a(tmp_path):
  """The CCD_MESH build is device code first: nvcc cross-compiles a one-thread-per-pair kernel around it for sm_90a (no GPU needed)."""
  import shutil

  nvcc = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
  if not os.path.exists(nvcc):
    pytest.skip("nvcc not available")
  src = os.path.join(HERE, "host_harness", "ccd_mesh_device_check.cu")
  r = subprocess.run([nvcc, "-c", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-o", str(tmp_path / "check.o"), src], capture_output=True, text=True)
  assert r.returncode == 0, r.stderr[-2000:]
  assert "k_ccd_mesh_pairs" in r.stderr and "0 bytes spill stores" in r.stderr


def test_plane_mesh_matches_oracle(hlib, model):
  """plane_convex for mesh geoms (exhaustive and hull-graph variants): same vertices picked, same depths / positions as the oracle."""
  mjm = model
  types = np.asarray(mjm.geom_type)
  rng = np.random.default_rng(3)
  hlib.hplane_mesh.restype = None
  hlib.hplane_mesh.argtypes = [V, V, V, V, V]
  ncontact = nfour = 0
  for g in [g for g in range(mjm.ngeom) if types[g] == GEOM_MESH]:
    for trial in range(40):
      # half the trials rest a face / edge nearly flat on the plane (several vertices within the 1e-3 band), the others are random tilts
      mat = rand_rot(rng) if trial % 2 else np.eye(3).reshape(-1)
      if trial % 4 == 0:
        mat = np.array([[1, 0, 0], [0, -1, 0], [0, 0, -1]], dtype=np.float64).reshape(-1)
      pos = np.array([0.0, 0.0, rng.uniform(-0.02, 0.06)])
      n_world, plane_pos = np.array([0.0, 0.0, 1.0]), np.zeros(3)
      res = {}
      for tag, real in (("dev", np.float32), ("o32", np.float32), ("o64", np.float64)):
        d, keep = make_desc(mjm, g, pos, mat, real)
        dist = np.zeros(4, real); p4 = np.zeros((4, 3), real)
        nw, pp = np.ascontiguousarray(n_world.astype(real)), np.ascontiguousarray(plane_pos.astype(real))
        P = lambda a: a.ctypes.data_as(V)
        if tag == "dev":
          hlib.hplane_mesh(P(nw), P(pp), ctypes.byref(d), P(dist), P(p4))
        else:
          lib = orc._lib(np.dtype(real).itemsize)
          lib.orc_plane_convex_desc.restype = None
          lib.orc_plane_convex_desc.argtypes = [V, V, V, V, V]
          lib.orc_plane_convex_desc(P(nw), P(pp), ctypes.byref(d), P(dist), P(p4))
        res[tag] = (dist.astype(np.float64), p4.astype(np.float64))
      dd, dp = res["dev"]
      ok = False
      for tag in ("o64", "o32"):  # near-ties between vertices in the band can resolve differently in fp32 and fp64
        od, op = res[tag]
        if np.array_equal(dd < 1e9, od < 1e9) and np.allclose(dd[dd < 1e9], od[od < 1e9], atol=2e-6) and np.allclose(dp, op, atol=2e-6):
          ok = True
      assert ok, (g, trial, res)
      ncontact += int((dd < 1e9).sum() > 0)
      nfour += int((dd < 1e9).sum() == 4)
  print("plane-mesh trials with contacts:", ncontact, "with four:", nfour)
  assert ncontact >= 60 and nfour >= 10
