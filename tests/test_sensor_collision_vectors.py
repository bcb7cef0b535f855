"""The collision-sensor device source (mjb_sensor_collision.cuh) compiled as host C++, replayed on the reference-generated fixtures.

tests/golden/sensor_collision_*.npz (tools/make_sensor_collision_goldens.py) hold, after forward and after each step, the geom poses and the
sensordata the reference computed from them.  From those poses the host build of the sensor pairs' colliders and of the per-sensor reduction
reproduces every collision sensor: distances to 1e-4 of the scene's geom size; fromto points to 1e-4 of it and normals to 1e-3 for primitive
pairs, 1e-2 and 2e-2 for GJK / EPA pairs (ccd_sensors says why); normal and fromto entries the fixture tool marks as knife-edge, where the
witness points nearly coincide and the normal is not determined in fp32, are skipped.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io, mjcf
from tests import sensor_collision_scenes as scenes

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_harness", "sensor_collision_host.cpp")
BUILD = os.path.join(HERE, "host_harness", "_build")
GOLD = os.path.join(HERE, "golden")
TAGS = ["forward", "step0", "step1", "step2"]


@pytest.fixture(scope="module")
def lib():
  os.makedirs(BUILD, exist_ok=True)
  out = os.path.join(BUILD, "sensor_collision_host.so")
  deps = [SRC] + [os.path.join(HERE, "..", "mujoco_warp_b200", "csrc", f) for f in ("mjb_sensor_collision.cuh", "mjb_ccd.cuh", "mjb_colliders.cuh", "mjb_math.cuh", "mjb_types.cuh")]
  if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(p) for p in deps):
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-std=c++17", "-DCCD_MESH=1", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", out], check=True)
  L = ctypes.CDLL(out)
  L.hsc_set_int.argtypes = [ctypes.c_char_p, ctypes.c_int]
  L.hsc_set_float.argtypes = [ctypes.c_char_p, ctypes.c_float]
  L.hsc_set_array.argtypes = [ctypes.c_char_p, ctypes.c_void_p]
  L.hsc_run.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
  return L


def _bind(L, mjm, keep):
  sc = io._sensor_collision_tables(mjm, io.derive_tables(mjm))
  ints = dict(ngeom=mjm.ngeom, nsensor=mjm.nsensor, nsensordata=mjm.nsensordata, disableflags=int(mjm.opt.disableflags),
              ccd_iterations=int(mjm.opt.ccd_iterations), nsensorcollision=sc["nsensorcollision"], nsensorcollision_sensor=len(sc["sensor_collision_id"]),
              nsensorcollision_ccd=sc["nsensorcollision_ccd"], sensor_collision_epa_iterations=sc["sensor_collision_epa_iterations"])
  for k, v in ints.items():
    assert L.hsc_set_int(k.encode(), int(v)) == 0, k
  assert L.hsc_set_float(b"ccd_tolerance", float(mjm.opt.ccd_tolerance)) == 0
  npair = int(getattr(mjm, "npair", 0))
  arrays = {n: (np.asarray(getattr(mjm, n)), np.int32) for n in ("geom_type", "geom_dataid", "sensor_type", "sensor_datatype", "sensor_adr", "sensor_dim")}
  arrays.update({n: (np.asarray(getattr(mjm, n)), np.float32) for n in ("geom_size", "geom_margin", "sensor_cutoff")})
  arrays["pair_margin"] = (np.asarray(mjm.pair_margin) if npair else np.zeros(1), np.float32)
  for n in ("mesh_vertadr", "mesh_vertnum", "mesh_graphadr", "mesh_graph", "mesh_polynum", "mesh_polyadr", "mesh_polyvertadr", "mesh_polyvertnum",
            "mesh_polyvert", "mesh_polymapadr", "mesh_polymapnum", "mesh_polymap"):
    arrays[n] = (np.asarray(getattr(mjm, n)) if mjm.nmesh else np.zeros(1), np.int32)
  for n in ("mesh_vert", "mesh_polynormal"):
    arrays[n] = (np.asarray(getattr(mjm, n)) if mjm.nmesh else np.zeros(1), np.float32)
  for n in ("sensor_collision_start_adr", "sensor_collision_pair", "sensor_collision_id", "sensor_collision_adr", "sensor_collision_flip"):
    arrays[n] = (sc[n], np.int32)
  for n, (x, dt) in arrays.items():
    x = np.ascontiguousarray(np.asarray(x, dtype=dt).reshape(-1) if np.asarray(x).size else np.zeros(1, dtype=dt))
    keep.append(x)
    assert L.hsc_set_array(n.encode(), x.ctypes.data) == 0, n


def _size_scale(mjm):
  gt = np.asarray(mjm.geom_type)
  return float(np.asarray(mjm.geom_size)[gt != C.GEOM_PLANE].max())


def ccd_sensors(mjm):
  """Sensors with a GJK / EPA pair.  Where the closest features of two convex shapes are faces or edges, the closest points form a set, and
  fp32 and fp64 GJK stop at different members of it; on curved surfaces the distance is second order in the direction, so EPA's fp32
  direction settles to ~1e-2 (witness points to ~1e-3 of the size) while the distance agrees to 1e-5.  Their fromto points are held to 1e-2 of the geom size, normals to 2e-2."""
  sc = io._sensor_collision_tables(mjm, io.derive_tables(mjm))
  ccd = sc["sensor_collision_pair"][:, 3] >= 0
  out = np.zeros(mjm.nsensor, dtype=bool)
  for i, s in enumerate(sc["sensor_collision_id"]):
    e0, e1 = sc["sensor_collision_adr"][i], sc["sensor_collision_adr"][i + 1]
    out[s] = ccd[sc["sensor_collision_start_adr"][e0:e1]].any()
  return out


def compare(mjm, got, want, knife, size, label, ccd_witness=1e-2):
  """distances to 1e-4 of `size`; fromto points to 1e-4 of it and normals to 1e-3, 1e-2 and 2e-2 for GJK / EPA sensors (ccd_sensors)"""
  ccd = ccd_sensors(mjm)
  for s in range(mjm.nsensor):
    a, n, t = int(mjm.sensor_adr[s]), int(mjm.sensor_dim[s]), int(mjm.sensor_type[s])
    g, w = got[:, a : a + n], want[:, a : a + n]
    if t == C.SENS_GEOMNORMAL:
      ok = ~knife[:, s]
      np.testing.assert_allclose(g[ok], w[ok], atol=2e-2 if ccd[s] else 1e-3, rtol=0, err_msg=f"{label} sensor {s} (normal)")
    elif t == C.SENS_GEOMFROMTO:
      ok = ~knife[:, s]
      np.testing.assert_allclose(g[ok], w[ok], atol=(ccd_witness if ccd[s] else 1e-4) * size, rtol=0, err_msg=f"{label} sensor {s} (fromto)")
    else:
      np.testing.assert_allclose(g, w, atol=1e-4 * size, rtol=0, err_msg=f"{label} sensor {s} (distance)")


@pytest.mark.parametrize("scene", sorted(scenes.SCENES))
def test_host_build_reproduces_reference_sensordata(lib, scene):
  g = np.load(os.path.join(GOLD, f"sensor_collision_{scene}.npz"))
  mjm = mjcf.load_string(scenes.SCENES[scene])
  keep = []
  _bind(lib, mjm, keep)
  size = _size_scale(mjm)
  for tag in TAGS:
    want = g[f"{tag}/sensordata"]
    nworld = want.shape[0]
    xpos = np.ascontiguousarray(g[f"{tag}/geom_xpos"], dtype=np.float32)
    xmat = np.ascontiguousarray(g[f"{tag}/geom_xmat"], dtype=np.float32)
    got = np.full((nworld, mjm.nsensordata), np.nan, dtype=np.float32)
    assert lib.hsc_run(nworld, xpos.ctypes.data, xmat.ctypes.data, got.ctypes.data) == 0
    compare(mjm, got.astype(np.float64), want, g[f"knife/{tag}"], size, f"{scene}/{tag}")


def test_fixtures_cover_every_route():
  """The fixtures reach negative distances (EPA and primitive overlaps), the contact pool holds CONSTRAINT | SENSOR contacts of a pair that
  is both, and a parent-child pair the contact filter excludes is still sensed."""
  neg = {}
  for scene in scenes.SCENES:
    g = np.load(os.path.join(GOLD, f"sensor_collision_{scene}.npz"))
    mjm = mjcf.load_string(scenes.SCENES[scene])
    dist = g["forward/sensordata"][:, np.asarray(mjm.sensor_adr)[np.asarray(mjm.sensor_type) == C.SENS_GEOMDIST]]
    neg[scene] = bool((dist < 0).any())
    if scene == "contact":
      assert (g["forward/con_type"] == 3).any()  # ContactType.CONSTRAINT | SENSOR
      t = io.derive_tables(mjm)
      arm, base = mjm.names.geom.index("arm"), mjm.names.geom.index("base")
      a, b = sorted((arm, base))
      assert t["nxn_pairid"][(a * (2 * mjm.ngeom - a - 3)) // 2 + b - 1, 0] == -2  # filtered as parent-child
  assert neg["overlap"] and neg["contact"]
