"""The CCD_MESH = 2 build of mjb_ccd.cuh (multi-contact buffers sized from the model, the build k_collision_mesh_large.cu and
k_sensor_collision_large.cu run), compiled as host C++ through tests/host_harness/ccd_large_host.cpp, on the large-hull scenes of
tests/mesh_hull_scenes.py: every mesh pair of every world at the reference's forward() pose against the reference's contacts
(tests/golden/mesh_hull_*.npz, tools/make_mesh_hull_goldens.py) and against the fp64 oracle, whose fixed buffers hold hulls up to 64 / 32
(so every scene but prism96).  Tolerances are those of tests/test_device_ccd_mesh_on_host.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import orc
from tests import mesh_hull_scenes as S
from tests.test_device_ccd_mesh_on_host import hlib, make_desc, same_points  # noqa: F401  (hlib: the CCD_MESH = 1 build, a fixture)
from tests.test_device_ccd_on_host import CSRC, HERE

SRC = os.path.join(HERE, "host_harness", "ccd_large_host.cpp")
OUT = os.path.join(HERE, "host_harness", "_build", "libccd_host_mesh_large.so")
GOLD = os.path.join(HERE, "golden")
GEOM_PLANE, GEOM_SPHERE, GEOM_MESH = 0, 2, 7
ORACLE_POLY, ORACLE_DEG = 64, 32  # oracle/oracle_ccd.h CCD_MAXPOLY / CCD_MAXDEG
V, F, I = ctypes.c_void_p, ctypes.c_float, ctypes.c_int


@pytest.fixture(scope="module")
def llib():
  deps = [SRC] + [os.path.join(CSRC, f) for f in ("mjb_ccd.cuh", "mjb_colliders.cuh", "mjb_math.cuh", "mjb_types.cuh")]
  if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-DCCD_MESH=2", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", OUT], check=True)
  lib = ctypes.CDLL(OUT)
  lib.hccd_large_desc.restype = I
  lib.hccd_large_desc.argtypes = [V, V, F, F, F, I, I, I, I, V, V, V, V]
  lib.hplane_mesh_large.restype = None
  lib.hplane_mesh_large.argtypes = [V, V, V, V, V]
  return lib


P = lambda a: a.ctypes.data_as(V)


def large_pair(llib, mjm, g1, p1, m1, g2, p2, m2, iterations=35):
  d1, k1 = make_desc(mjm, g1, p1, m1, np.float32)
  d2, k2 = make_desc(mjm, g2, p2, m2, np.float32)
  dist = np.zeros(1, np.float32); w1 = np.zeros((4, 3), np.float32); w2 = np.zeros((4, 3), np.float32); ovf = np.zeros(1, np.int32)
  n = llib.hccd_large_desc(ctypes.byref(d1), ctypes.byref(d2), 0.0, 1e-6, 1e30, iterations, iterations, int(mjm.npolygonmax), int(mjm.nmeshdegmax),
                           P(dist), P(w1), P(w2), P(ovf))
  return float(dist[0]), int(n), w1.astype(np.float64), w2.astype(np.float64), int(ovf[0])


def oracle_pair(mjm, g1, p1, m1, g2, p2, m2, iterations=35):
  d1, k1 = make_desc(mjm, g1, p1, m1, np.float64)
  d2, k2 = make_desc(mjm, g2, p2, m2, np.float64)
  dist = np.zeros(1); w1 = np.zeros((4, 3)); w2 = np.zeros((4, 3)); ovf = np.zeros(1, np.int32)
  lib = orc._lib(8)
  lib.orc_ccd_desc.restype = I
  lib.orc_ccd_desc.argtypes = [V, V, ctypes.c_double, ctypes.c_double, ctypes.c_double, I, I, I, V, V, V, V]
  n = lib.orc_ccd_desc(ctypes.byref(d1), ctypes.byref(d2), 0.0, 1e-6, 1e30, iterations, iterations, 1, P(dist), P(w1), P(w2), P(ovf))
  return float(dist[0]), int(n), w1, w2, int(ovf[0])


def pairs(mjm):
  """Mesh geom pairs in narrowphase order (the lower geom type first) on different bodies: convex pairs and plane-mesh."""
  t, b = np.asarray(mjm.geom_type), np.asarray(mjm.geom_bodyid)
  out = []
  for g1 in range(mjm.ngeom):
    for g2 in range(mjm.ngeom):
      if g1 == g2 or b[g1] == b[g2] or (b[g1] == 0 and b[g2] == 0) or t[g2] != GEOM_MESH or t[g1] > t[g2] or (t[g1] == t[g2] and g1 > g2):
        continue
      if t[g1] == GEOM_PLANE or t[g1] >= GEOM_SPHERE:
        out.append((g1, g2))
  return out


@pytest.mark.parametrize("name", list(S.SCENES))
def test_scene_compiles_to_its_design_sizes(name):
  mjm = S.load(name)
  assert (int(mjm.npolygonmax), int(mjm.nmeshdegmax)) == (S.SCENES[name]["npolygonmax"], S.SCENES[name]["nmeshdegmax"])
  assert int(mjm.npolygonmax) > 32 or int(mjm.nmeshdegmax) > 16  # past the CCD_MESH = 1 buffers


@pytest.mark.parametrize("name", list(S.SCENES))
def test_large_build_matches_reference_contacts_and_oracle(llib, name):
  mjm = S.load(name)
  g = np.load(os.path.join(GOLD, f"mesh_hull_{name}.npz"))
  xpos, xmat = g["forward/geom_xpos"], g["forward/geom_xmat"].reshape(S.NWORLD, -1, 9)
  cg, cd, cp, cf, cw = (g[f"forward/con_{f}"] for f in ("geom", "dist", "pos", "frame", "worldid"))
  real = cd < 0.0  # margin and gap are zero: the reference's sensor-pair contacts are the ones at or past zero
  with_oracle = int(mjm.npolygonmax) <= ORACLE_POLY and int(mjm.nmeshdegmax) <= ORACLE_DEG
  types = np.asarray(mjm.geom_type)
  nmulti = nplane = 0
  for w in range(S.NWORLD):
    for g1, g2 in pairs(mjm):
      sel = np.nonzero(real & (cw == w) & (cg[:, 0] == g1) & (cg[:, 1] == g2))[0]
      if types[g1] == GEOM_PLANE:
        d, keep = make_desc(mjm, g2, xpos[w, g2], xmat[w, g2], np.float32)
        dist = np.zeros(4, np.float32); p4 = np.zeros((4, 3), np.float32)
        nw, pp = np.ascontiguousarray(xmat[w, g1].reshape(3, 3)[:, 2].astype(np.float32)), np.ascontiguousarray(xpos[w, g1].astype(np.float32))
        llib.hplane_mesh_large(P(nw), P(pp), ctypes.byref(d), P(dist), P(p4))
        hit = dist < 0.0
        assert hit.sum() == len(sel), (name, w, g1, g2, dist, cd[sel])
        if len(sel):
          nplane += 1
          same_points(p4[hit].astype(np.float64), cp[sel], len(sel), 1e-4)
          np.testing.assert_allclose(np.sort(dist[hit]), np.sort(cd[sel]), atol=2e-5)
        continue
      dd, dn, dw1, dw2, dovf = large_pair(llib, mjm, g1, xpos[w, g1], xmat[w, g1], g2, xpos[w, g2], xmat[w, g2])
      assert dovf == 0, (name, w, g1, g2, dovf)
      n = dn if dd < 0.0 else 0
      assert n == len(sel), (name, w, g1, g2, dd, dn, cd[sel])
      if n == 0:
        continue
      nmulti += n > 1
      assert np.abs(cd[sel] - dd).max() <= 2e-5, (name, w, g1, g2, dd, cd[sel])
      same_points(0.5 * (dw1 + dw2), cp[sel], n, 1e-4)
      # the normal is the difference of two fp32 witness points about 5e-4 apart: each carries ~1e-7 of rounding
      nrm = (dw1[0] - dw2[0]) / np.linalg.norm(dw1[0] - dw2[0])
      assert np.abs(cf[sel].reshape(n, 9)[:, :3] - nrm).max() <= 2e-3, (name, w, g1, g2)
      if with_oracle:
        od, on, ow1, ow2, oovf = oracle_pair(mjm, g1, xpos[w, g1], xmat[w, g1], g2, xpos[w, g2], xmat[w, g2])
        assert oovf == 0 and on == dn and abs(od - dd) <= 2e-5, (name, w, g1, g2, (dd, dn), (od, on))
        same_points(0.5 * (dw1 + dw2), 0.5 * (ow1 + ow2), on, 1e-4)
  print(name, "multi-contact pairs", nmulti, "plane-mesh pairs", nplane)
  assert nmulti + nplane >= S.NWORLD


def test_in_cap_pairs_equal_the_in_cap_build(llib, hlib):  # noqa: F811
  """The mixed scene's pairs of in-cap hulls (cubes, a 16-gon prism) in the large build give exactly the CCD_MESH = 1 build's answer."""
  mjm = S.load("mixed")
  g = np.load(os.path.join(GOLD, "mesh_hull_mixed.npz"))
  xpos, xmat = g["forward/geom_xpos"], g["forward/geom_xmat"].reshape(S.NWORLD, -1, 9)
  big = mjm.geom_names.index("big") if hasattr(mjm, "geom_names") else int(np.nonzero(np.asarray(mjm.geom_dataid) == 2)[0][0])
  ncheck = 0
  for w in range(S.NWORLD):
    for g1, g2 in pairs(mjm):
      if big in (g1, g2) or int(mjm.geom_type[g1]) == GEOM_PLANE:
        continue
      lg = large_pair(llib, mjm, g1, xpos[w, g1], xmat[w, g1], g2, xpos[w, g2], xmat[w, g2])
      d1, k1 = make_desc(mjm, g1, xpos[w, g1], xmat[w, g1], np.float32)
      d2, k2 = make_desc(mjm, g2, xpos[w, g2], xmat[w, g2], np.float32)
      dist = np.zeros(1, np.float32); w1 = np.zeros((4, 3), np.float32); w2 = np.zeros((4, 3), np.float32); ovf = np.zeros(1, np.int32)
      n = hlib.hccd_desc(ctypes.byref(d1), ctypes.byref(d2), 0.0, 1e-6, 1e30, 35, 35, P(dist), P(w1), P(w2), P(ovf))
      assert (lg[0], lg[1], lg[4]) == (float(dist[0]), int(n), int(ovf[0])), (w, g1, g2)
      np.testing.assert_array_equal(lg[2], w1.astype(np.float64)); np.testing.assert_array_equal(lg[3], w2.astype(np.float64))
      ncheck += lg[0] < 0
  assert ncheck >= S.NWORLD


def test_large_build_compiles_for_sm_90a(tmp_path):
  """The kernels of the large build cross-compile for sm_90a, and their stack frame does not depend on the model's hull sizes."""
  import re
  import shutil

  nvcc = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
  if not os.path.exists(nvcc):
    pytest.skip("nvcc not available")
  frames = {}
  for src in ("k_collision_mesh_large.cu", "k_sensor_collision_large.cu"):
    r = subprocess.run([nvcc, "-std=c++17", "-O3", "-cubin", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-o", str(tmp_path / "k.cubin"),
                        os.path.join(CSRC, src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for m in re.finditer(r"Function properties for (\S*(?:k_collision_mesh_large|k_sensor_collision_large)I\S*)\n\s*(\d+) bytes stack frame", r.stderr):
      frames[m.group(1)] = int(m.group(2))
  assert len(frames) == 4, frames
  assert max(frames.values()) <= 2048, frames  # CCD_MESH = 1 holds its 32 / 16 buffers on the stack: about 4 KB
