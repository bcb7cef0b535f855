"""Fluid forces without a GPU: the compiler's geom_fluid (Lamb's added-mass integrals), put_model's refusal of fluid with the implicit
integrator, and the device header mjb_fluid.cuh compiled as host C++ against the reference-generated fixtures (tests/golden/fluid_*.npz)."""
import ctypes
import math
import os
import subprocess
import types

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io, mjcf
from tests import fluid_scenes

HERE = os.path.dirname(os.path.abspath(__file__))
HARNESS = os.path.join(HERE, "host_harness")
BUILD = os.path.join(HARNESS, "_build")
CSRC = os.path.join(HERE, "..", "mujoco_warp_b200", "csrc")
GOLD = os.path.join(HERE, "golden")


def _row(gtype, size):
  return mjcf.geom_fluid_row(gtype, size, "ellipsoid", C.DEFAULT_FLUIDCOEF)


def test_sphere_kappa_is_two_thirds_virtual_mass_half_volume():
  r = 0.3
  np.testing.assert_allclose(mjcf.fluid_kappa([r, r, r]), [2 / 3] * 3, rtol=1e-12)
  row = _row(C.GEOM_SPHERE, [r, 0, 0])
  vol = 4 / 3 * math.pi * r**3
  assert row[0] == 1.0
  np.testing.assert_allclose(row[1:6], C.DEFAULT_FLUIDCOEF)
  np.testing.assert_allclose(row[6:9], [vol / 2] * 3, rtol=1e-12)
  np.testing.assert_array_equal(row[9:12], 0.0)


@pytest.mark.parametrize("ratio", [1.5, 3.0, 10.0])
def test_spheroids_match_lambs_closed_forms(ratio):
  # prolate a > b = c (Lamb, Hydrodynamics §373): alpha0 along the long axis, beta0 = gamma0 across it
  a, b = ratio, 1.0
  e = math.sqrt(1 - (b / a) ** 2)
  L = math.log((1 + e) / (1 - e))
  alpha0 = 2 * (1 - e * e) / e**3 * (0.5 * L - e)
  beta0 = 1 / e**2 - (1 - e * e) / (2 * e**3) * L
  np.testing.assert_allclose(mjcf.fluid_kappa([a, b, b]), [alpha0, beta0, beta0], rtol=1e-10)
  # oblate a = b > c: gamma0 along the short axis
  c = 1.0 / ratio
  e = math.sqrt(1 - c * c)
  gamma0 = 2 / e**2 * (1 - math.sqrt(1 - e * e) / e * math.asin(e))
  alpha0 = math.sqrt(1 - e * e) / e**3 * math.asin(e) - (1 - e * e) / e**2
  np.testing.assert_allclose(mjcf.fluid_kappa([1.0, 1.0, c]), [alpha0, alpha0, gamma0], rtol=1e-10)
  # virtual mass V k / (2 - k); added moment about the symmetry axis vanishes, about a cross axis it is Lamb's
  k = mjcf.fluid_kappa([a, b, b])
  row = _row(C.GEOM_ELLIPSOID, [a, b, b])
  vol = 4 / 3 * math.pi * a * b * b
  np.testing.assert_allclose(row[6:9], vol * k / (2 - k), rtol=1e-12)
  assert abs(row[9]) < 1e-12 * vol
  want = vol / 5 * (b * b - a * a) ** 2 * (k[0] - k[1]) / (2 * (b * b - a * a) + (b * b + a * a) * (k[1] - k[0]))
  np.testing.assert_allclose(row[10:12], [abs(want)] * 2, rtol=1e-10)


def test_permuting_semiaxes_permutes_outputs():
  s = np.array([0.3, 0.1, 0.2])
  base = _row(C.GEOM_ELLIPSOID, s)
  for p in ([1, 2, 0], [2, 0, 1], [0, 2, 1]):
    r = _row(C.GEOM_ELLIPSOID, s[p])
    np.testing.assert_allclose(r[6:9], base[6:9][p], rtol=1e-12)
    np.testing.assert_allclose(r[9:12], base[9:12][p], rtol=1e-10)


def test_fluidshape_none_and_defaults_from_classes():
  m = mjcf.load_string(fluid_scenes.ellipsoid_xml())
  gf = np.asarray(m.geom_fluid)
  assert gf.shape == (m.ngeom, 12)
  plain = [g for g in range(m.ngeom) if gf[g, 0] == 0]
  assert len(plain) == 1 and np.all(gf[plain[0]] == 0)  # the class "plain" geom
  np.testing.assert_allclose(gf[0, 1:6], [0.4, 0.3, 1.2, 0.8, 1.1])  # from the default class
  np.testing.assert_allclose(gf[1, 1:6], [0.5, 0.2, 1.5, 1.3, 0.7])  # the geom's own fluidcoef
  with pytest.raises(ValueError, match="fluidshape"):
    mjcf.load_string(fluid_scenes.sphere_xml().replace('density="2000.0"', 'density="2000.0" fluidshape="box"'))


def test_saved_model_without_geom_fluid_has_no_ellipsoid_geoms(tmp_path):
  m = mjcf.load_string(fluid_scenes.chain_xml())
  del m.geom_fluid
  mjcf.save_npz(m, str(tmp_path / "m.npz"))
  assert not hasattr(mjcf.load_npz(str(tmp_path / "m.npz")), "geom_fluid")  # put_model then takes zeros (io.py)


def test_fluid_with_implicit_integrator_is_refused_by_name():
  m = mjcf.load_string(fluid_scenes.chain_xml("implicit"))
  with pytest.raises(NotImplementedError, match="fluid.*implicit"):
    io._validate(m)
  io._validate(mjcf.load_string(fluid_scenes.chain_xml("implicitfast")))  # implicitfast, Euler and RK4 are accepted
  io._validate(mjcf.load_string(fluid_scenes.chain_xml("RK4")))


def _host_lib():
  src, out = os.path.join(HARNESS, "fluid_host.cpp"), os.path.join(BUILD, "libfluid_host.so")
  deps = [src] + [os.path.join(CSRC, f) for f in ("mjb_fluid.cuh", "mjb_math.cuh", "mjb_types.cuh")]
  if not os.path.exists(out) or any(os.path.getmtime(p) > os.path.getmtime(out) for p in deps):
    os.makedirs(BUILD, exist_ok=True)
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-std=c++17", "-ffp-contract=off", f"-I{cuda_inc}", src, "-o", out], check=True)
  return ctypes.CDLL(out)


def fluid_tables(mjm):
  """put_model's per-body fluid model (io.py): 1 ellipsoid, 2 inertia box, 0 none."""
  gf = np.asarray(getattr(mjm, "geom_fluid", np.zeros((mjm.ngeom, 12)))).reshape(mjm.ngeom, 12)
  ell = np.zeros(mjm.nbody, dtype=bool)
  ell[np.asarray(mjm.geom_bodyid)[gf[:, 0] > 0]] = True
  box = ~ell & (np.asarray(mjm.body_mass) > 0)
  box[0] = False
  return gf, np.where(ell, 1, np.where(box, 2, 0)).astype(np.int32)


@pytest.mark.parametrize("scene", sorted(fluid_scenes.SCENES))
def test_host_header_reproduces_reference_qfrc_fluid(scene):
  z = np.load(os.path.join(GOLD, f"fluid_{scene}.npz"))
  mjm = mjcf.load_string(fluid_scenes.SCENES[scene][0])
  lib = _host_lib()
  gf, body_fluid = fluid_tables(mjm)
  anc = io.derive_tables(mjm)["body_isdofancestor"]
  F = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.float64).astype(np.float32))
  I = lambda a: np.ascontiguousarray(np.asarray(a).astype(np.int32))
  keep = []
  P = lambda a: (keep.append(a), a.ctypes.data_as(ctypes.c_void_p))[1]
  for tag in ["forward"] + [f"step{s}" for s in range(4)]:
    nworld = z[f"{tag}/cvel"].shape[0]
    out = np.zeros((nworld, mjm.nv), dtype=np.float32)
    wind = F(np.asarray(mjm.opt.wind).reshape(3))
    lib.hfluid_qfrc(mjm.nv, mjm.nbody, mjm.ngeom, P(I(mjm.body_rootid)), P(I(mjm.dof_bodyid)), P(I(anc)), P(F(mjm.body_mass)), P(F(mjm.body_inertia)),
                    P(I(mjm.geom_type)), P(F(mjm.geom_size)), P(I(body_fluid)), P(I(mjm.body_geomadr)), P(I(mjm.body_geomnum)), P(F(gf)),
                    ctypes.c_float(float(mjm.opt.density)), ctypes.c_float(float(mjm.opt.viscosity)), P(wind), nworld,
                    P(F(z[f"{tag}/cvel"])), P(F(z[f"{tag}/xipos"])), P(F(z[f"{tag}/ximat"])), P(F(z[f"{tag}/geom_xpos"])), P(F(z[f"{tag}/geom_xmat"])),
                    P(F(z[f"{tag}/subtree_com"])), P(F(z[f"{tag}/cdof"])), out.ctypes.data_as(ctypes.c_void_p))
    want = z[f"{tag}/qfrc_fluid"]
    scale = max(1e-6, float(np.abs(want).max()))
    np.testing.assert_allclose(out, want, rtol=0, atol=1e-5 * scale, err_msg=f"{scene} {tag}")
