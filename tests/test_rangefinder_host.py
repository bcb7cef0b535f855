"""The rangefinder sensor without a GPU.

- put_model's rangefinder tables (nrangefinder, sensor_rangefinder_adr, rangefinder_sensor_adr, sensor_rangefinder_bodyid) against the
  reference's own, stored in every fixture (tests/golden/rangefinder_*.npz, tools/make_rangefinder_goldens.py); the refusals of
  camera-attached, out-of-range and multi-output rangefinders by name; a rangefinder does not select k_sensor's EXTRA build.
- The fp64 restatement of the reference's ray casting (tests/host_harness/ray_oracle.c), fed each fixture state's site and geom poses,
  with the cutoff applied, against the fixture's rangefinder slots; and the closest-hit scan the GPU kernels share
  (mujoco_warp_b200/csrc/mjb_ray.cuh ray_scan, compiled as host C++ by tests/host_harness/rangefinder_host.cpp) against the same slots in
  fp32, where only knife-edge rays are excused.
"""
import glob
import os

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io
from tests import rangefinder_scenes as S
from tests import test_ray_vectors as RV

HERE = os.path.dirname(os.path.abspath(__file__))
SCENES = list(S.SCENES)


def golden(name):
  return np.load(os.path.join(HERE, "golden", f"rangefinder_{name}.npz"))


def scan_lib():
  import ctypes

  lib = RV._compile(os.path.join(RV.HARNESS, "rangefinder_host.cpp"), os.path.join(RV.BUILD, "librangefinder_host.so"),
                    ["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-ffp-contract=off",
                     "-I" + os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")])
  assert isinstance(lib, ctypes.CDLL)
  return lib


class _WorldModel:
  """The model as world w sees it: per-world geom_size / geom_rgba of the batched fixture in place of the nominal ones."""

  def __init__(self, mjm, **over):
    self._m, self._over = mjm, over

  def __getattr__(self, name):
    return self._over[name] if name in self._over else getattr(self._m, name)


def states(z, nsteps):
  """(tag, sensordata, site_xpos, site_xmat, geom_xpos, geom_xmat, knife) of the forward state and of every step"""
  pre = ["forward/"] + [f"step/{k}/out_" for k in range(nsteps)]
  knife = ["forward/knife"] + [f"step/{k}/knife" for k in range(nsteps)]
  for p, kn in zip(pre, knife):
    yield (p, z[p + "sensordata"], z[p + "site_xpos"], z[p + "site_xmat"], z[p + "geom_xpos"], z[p + "geom_xmat"], z[kn])


def cutoff(x, c, dt):
  """sensor.py:57-81 _write_scalar: REAL data clamped to [-c, c], POSITIVE data from above, for c > 0"""
  x = np.array(x, dtype=np.float64)
  for r in range(x.shape[-1]):
    if c[r] > 0 and dt[r] == 0:
      x[..., r] = np.clip(x[..., r], -c[r], c[r])
    elif c[r] > 0 and dt[r] == 1:
      x[..., r] = np.minimum(x[..., r], c[r])
  return x


def rangefinder_values(fn, real, mjm, z, site_xpos, site_xmat, geom_xpos, geom_xmat, per_world):
  """(nworld, nrangefinder) slots from `fn` (ray_oracle_rays or hrf_scan) on the given poses, with the cutoff applied"""
  t = io.rangefinder_tables(mjm)
  adr = t["sensor_rangefinder_adr"]
  site = np.asarray(mjm.sensor_objid)[adr]
  nworld = site_xpos.shape[0]
  pnt = site_xpos[:, site]
  vec = np.asarray(site_xmat).reshape(nworld, -1, 3, 3)[:, site][..., 2]
  gxmat = np.asarray(geom_xmat).reshape(nworld, -1, 9)
  if per_world:
    dist = np.concatenate([RV.cast(fn, real, _WorldModel(mjm, geom_rgba=z["in/geom_rgba"][w]), geom_xpos[w : w + 1], gxmat[w : w + 1], pnt[w : w + 1],
                                   vec[w : w + 1], [-1] * 6, 1, t["sensor_rangefinder_bodyid"], geom_size=z["in/geom_size"][w])[0] for w in range(nworld)])
  else:
    dist = RV.cast(fn, real, mjm, geom_xpos, gxmat, pnt, vec, [-1] * 6, 1, t["sensor_rangefinder_bodyid"])[0]
  return cutoff(dist, np.asarray(mjm.sensor_cutoff)[adr], np.asarray(mjm.sensor_datatype)[adr])


@pytest.mark.parametrize("name", SCENES)
def test_tables_match_reference(name):
  mjm, z = S.load(name), golden(name)
  t = io.rangefinder_tables(mjm)
  assert t["nrangefinder"] == int(z["ref/nrangefinder"]) > 0
  for f in ("sensor_rangefinder_adr", "rangefinder_sensor_adr", "sensor_rangefinder_bodyid"):
    np.testing.assert_array_equal(t[f], z[f"ref/{f}"], err_msg=f)
    assert t[f].dtype == np.int32
  # a rangefinder alone does not select k_sensor's EXTRA build: k_sensor keeps skipping its slot
  assert not io._validate_extra_sensors(mjm)


def test_scenes_cover_the_cases():
  mjm = S.load("primitives")
  t = io.rangefinder_tables(mjm)
  assert t["sensor_rangefinder_adr"][0] == 0 and list(t["rangefinder_sensor_adr"]).count(-1) == 3  # inserted before and between other sensors
  body = list(mjm.names.body)
  assert 0 in t["sensor_rangefinder_bodyid"] and body.index("inner") in t["sensor_rangefinder_bodyid"]  # world-body site, site inside a sphere
  many = io.rangefinder_tables(S.load("many"))["nrangefinder"]
  assert many >= 200 and (S.NWORLD * many) % 128 != 0 and many % 32 != 0  # warps straddle worlds, the last block is partial
  z = golden("primitives")
  sd = z["forward/sensordata"][:, np.asarray(mjm.sensor_adr)[t["sensor_rangefinder_adr"]]]
  assert (sd == -1).any() and (sd > 0).any()
  cut = np.asarray(mjm.sensor_cutoff)[t["sensor_rangefinder_adr"]]
  assert (sd[:, cut == 0.3] == 0.3).any()  # the cutoff below the hit distance engages


@pytest.mark.parametrize("field,value,msg", [
  ("sensor_objtype", C.OBJ_CAMERA, "object type 7"), ("sensor_objid", 10_000, "unknown object"), ("sensor_dim", 3, "one output"),
])
def test_refusals_name_the_sensor(field, value, msg):
  mjm = S.load("primitives")
  s = int(io.rangefinder_tables(mjm)["sensor_rangefinder_adr"][2])
  a = np.asarray(getattr(mjm, field)).copy()
  a[s] = value
  setattr(mjm, field, a)
  with pytest.raises(ValueError, match=f"sensor {s} \\('{mjm.names.sensor[s]}'\\).*{msg}"):
    io._validate_extra_sensors(mjm)


def test_world_count_refused_past_int_range():
  io.check_rangefinder_worlds(8192, 210)
  with pytest.raises(ValueError, match="nrangefinder"):
    io.check_rangefinder_worlds(2**22, 2**10)


def _check_scene(name, fn, real, atol):
  mjm, z = S.load(name), golden(name)
  _, nsteps, per_world = S.SCENES[name]
  t = io.rangefinder_tables(mjm)
  adr = t["sensor_rangefinder_adr"]
  hist = np.asarray(mjm.sensor_history).reshape(-1, 2)[adr, 0]
  slot = np.asarray(mjm.sensor_adr)[adr]
  compared = 0
  for tag, sd, sx, sm, gx, gm, knife in states(z, nsteps):
    got = rangefinder_values(fn, real, mjm, z, sx, sm, gx, gm, per_world)
    ok = ~knife & (hist == 0)[None]  # delayed slots hold the history's value
    exp = sd[:, slot]
    err = np.abs(got - exp)[ok]
    assert (err <= atol + (1e-5 if real == np.float32 else 0.0) * np.abs(exp[ok])).all(), f"{name} {tag}: max error {err.max()}"
    compared += int(ok.sum())
  assert compared >= (nsteps + 1) * S.NWORLD, f"{name}: only {compared} slots compared"


@pytest.mark.parametrize("name", SCENES)
def test_fp64_oracle_meets_reference(name):
  _check_scene(name, RV.oracle_lib(np.float64).ray_oracle_rays, np.float64, 1e-9)


@pytest.mark.parametrize("name", SCENES)
def test_shared_scan_meets_reference(name):
  _check_scene(name, scan_lib().hrf_scan, np.float32, 1e-5)


def test_fixtures_present():
  assert sorted(os.path.basename(p) for p in glob.glob(os.path.join(HERE, "golden", "rangefinder_*.npz"))) == sorted(f"rangefinder_{n}.npz" for n in SCENES)
