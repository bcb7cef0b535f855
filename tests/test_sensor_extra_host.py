"""The magnetometer, camprojection, insidesite, tendon limit and tendonactfrc sensors without a GPU.

- The compiler: type, object and reference, dim, datatype and stage of each new element, and every refusal by name; put_model's check
  of the object kinds and ids again on a model that did not come from the compiler.  rangefinder, tactile and magnetometer stay
  refused by the compiler; a magnetometer carried in the sensor arrays passes put_model's check.
- The device source of mjb_sensor_extra.cuh, compiled as host C++ (tests/host_harness/sensor_extra_host.cpp), against the reference's
  own sensordata (tests/golden/sensor_extra_*.npz, tools/make_sensor_extra_goldens.py), fed the fixture's site / camera poses and
  actuator forces; the tendon limit sensors' row scan, restated, against the same data from the fixture's efc rows.
"""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io, mjcf
from tests import sensor_extra_scenes as S

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_harness", "sensor_extra_host.cpp")
OUT = os.path.join(HERE, "host_harness", "_build", "libsensor_extra_host.so")
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "sensor_extra_*.npz")))

XML = """<mujoco><worldbody><body name="b" pos="0 0 1"><joint name="j" type="slide"/><geom name="g" size=".1"/>
<site name="s" type="box" size=".2 .2 .2"/><camera name="c" pos="0 -1 0"/></body></worldbody>
<tendon><fixed name="t" limited="true" range="-1 1"><joint joint="j" coef="1"/></fixed></tendon><actuator><motor tendon="t"/></actuator>
<sensor><jointpos joint="j"/>{sensors}</sensor></mujoco>"""


def _compile(sensors):
  return mjcf.load_string(XML.format(sensors=sensors))


@pytest.mark.parametrize("elem,stype,obj,ref,dim,stage", [
  ('<camprojection site="s" camera="c"/>', C.SENS_CAMPROJECTION, (C.OBJ_SITE, 0), (C.OBJ_CAMERA, 0), 2, 1),
  ('<insidesite objtype="body" objname="b" site="s"/>', C.SENS_INSIDESITE, (C.OBJ_BODY, 1), (C.OBJ_SITE, 0), 1, 1),
  ('<insidesite objtype="xbody" objname="b" site="s"/>', C.SENS_INSIDESITE, (C.OBJ_XBODY, 1), (C.OBJ_SITE, 0), 1, 1),
  ('<insidesite objtype="geom" objname="g" site="s"/>', C.SENS_INSIDESITE, (C.OBJ_GEOM, 0), (C.OBJ_SITE, 0), 1, 1),
  ('<insidesite objtype="site" objname="s" site="s"/>', C.SENS_INSIDESITE, (C.OBJ_SITE, 0), (C.OBJ_SITE, 0), 1, 1),
  ('<insidesite objtype="camera" objname="c" site="s"/>', C.SENS_INSIDESITE, (C.OBJ_CAMERA, 0), (C.OBJ_SITE, 0), 1, 1),
  ('<tendonlimitpos tendon="t"/>', C.SENS_TENDONLIMITPOS, (C.OBJ_TENDON, 0), (C.OBJ_UNKNOWN, -1), 1, 1),
  ('<tendonlimitvel tendon="t"/>', C.SENS_TENDONLIMITVEL, (C.OBJ_TENDON, 0), (C.OBJ_UNKNOWN, -1), 1, 2),
  ('<tendonlimitfrc tendon="t"/>', C.SENS_TENDONLIMITFRC, (C.OBJ_TENDON, 0), (C.OBJ_UNKNOWN, -1), 1, 3),
  ('<tendonactfrc tendon="t"/>', C.SENS_TENDONACTFRC, (C.OBJ_TENDON, 0), (C.OBJ_UNKNOWN, -1), 1, 3),
])
def test_compiler_mapping(elem, stype, obj, ref, dim, stage):
  m = _compile(elem)
  assert m.sensor_unsupported == []
  assert int(m.sensor_type[1]) == stype and int(m.sensor_datatype[1]) == 0 and int(m.sensor_needstage[1]) == stage
  assert (int(m.sensor_objtype[1]), int(m.sensor_objid[1])) == obj
  assert (int(m.sensor_reftype[1]), int(m.sensor_refid[1])) == ref
  assert int(m.sensor_dim[1]) == dim and int(m.sensor_adr[1]) == 1 and m.nsensordata == 1 + dim
  assert io._validate_extra_sensors(m)


@pytest.mark.parametrize("elem,msg", [
  ('<camprojection name="cp" site="s"/>', "camprojection sensor 'cp': missing attribute camera"),
  ('<camprojection name="cp" site="s" camera="x"/>', "camprojection sensor 'cp': unknown camera 'x'"),
  ('<insidesite name="in" objtype="joint" objname="j" site="s"/>', "insidesite sensor 'in': objtype 'joint'"),
  ('<insidesite name="in" objname="g" site="s"/>', "insidesite sensor 'in': missing attribute objtype"),
  ('<insidesite name="in" objtype="geom" objname="g" site="g"/>', "insidesite sensor 'in': unknown site 'g'"),
  ('<insidesite name="in" objtype="geom" objname="zz" site="s"/>', "insidesite sensor 'in': unknown geom 'zz'"),
  ('<tendonlimitpos name="tl" tendon="u"/>', "tendonlimitpos sensor 'tl': unknown tendon 'u'"),
  ('<tendonactfrc name="ta"/>', "tendonactfrc sensor 'ta': missing attribute tendon"),
])
def test_compiler_refusals(elem, msg):
  with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)")):
    _compile(elem)


@pytest.mark.parametrize("elem,tag", [('<rangefinder site="s"/>', "rangefinder"), ('<tactile geom="g" mesh="m"/>', "tactile"), ('<magnetometer site="s"/>', "magnetometer")])
def test_compiler_still_refuses(elem, tag):
  assert _compile(elem).sensor_unsupported == [tag]


def test_put_model_checks_magnetometer_arrays():
  """A magnetometer carried in the arrays (MuJoCo's layout) passes the check on a site and is refused on anything else."""
  m = S.add_magnetometers(_compile(""), [("s", 0.0, 0, 0.0)])
  assert int(m.sensor_type[1]) == C.SENS_MAGNETOMETER and int(m.sensor_adr[1]) == 1 and m.nsensordata == 4 and io._validate_extra_sensors(m)
  m.sensor_objtype[1] = C.OBJ_BODY
  with pytest.raises(ValueError, match="object type 1"):
    io._validate_extra_sensors(m)


@pytest.mark.parametrize("field,value,msg", [
  ("sensor_objtype", C.OBJ_GEOM, "object type 5"), ("sensor_objid", 3, "object names an unknown object"),
  ("sensor_reftype", C.OBJ_SITE, "reference type 6"), ("sensor_refid", 2, "reference names an unknown object"),
])
def test_put_model_rechecks_objects(field, value, msg):
  m = _compile('<camprojection name="cp" site="s" camera="c"/>')
  getattr(m, field)[1] = value
  with pytest.raises(ValueError, match=f"sensor 1 \\('cp'\\): {msg}"):
    io._validate_extra_sensors(m)


def test_models_without_the_new_sensors_keep_the_plain_build():
  assert not io._validate_extra_sensors(_compile('<tendonpos tendon="t"/>'))


# ---------------------------------------------------------------- the device source on the host


@pytest.fixture(scope="module")
def hlib():
  os.makedirs(os.path.dirname(OUT), exist_ok=True)
  cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
  subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", OUT], check=True)
  lib = ctypes.CDLL(OUT)
  p, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
  for name, args, res in (("hse_magnetometer", [p, p, p], None), ("hse_camprojection", [p, p, p, f, p, p, p, p], None),
                          ("hse_insidesite", [i, i, p, p, f, f, p, p, p, i], i), ("hse_tendon_actfrc", [i, p, p, p, i], f)):
    getattr(lib, name).argtypes = args
    getattr(lib, name).restype = res
  return lib


def _f(a):
  return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def _i(a):
  return np.ascontiguousarray(np.asarray(a, dtype=np.int32))


def _ptr(a):
  return a.ctypes.data_as(ctypes.c_void_p)


def test_fixtures_present():
  assert {os.path.basename(p)[len("sensor_extra_"):-4] for p in GOLDEN} == set(S.SCENES)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_device_source_matches_reference(hlib, path):
  name = os.path.basename(path)[len("sensor_extra_"):-4]
  z = np.load(path)
  mjm = S.load(name)
  nw = S.NWORLD
  mag = z["in/magnetic"] if "in/magnetic" in z else np.tile(mjm.opt.magnetic, (nw, 1))
  fovy = z["in/cam_fovy"] if "in/cam_fovy" in z else np.tile(mjm.cam_fovy, (nw, 1))
  intr = z["in/cam_intrinsic"] if "in/cam_intrinsic" in z else np.tile(mjm.cam_intrinsic, (nw, 1, 1))
  want = z["forward/sensordata"]
  pos_arrays = {C.OBJ_BODY: "xipos", C.OBJ_XBODY: "xpos", C.OBJ_GEOM: "geom_xpos", C.OBJ_SITE: "site_xpos", C.OBJ_CAMERA: "cam_xpos"}
  checked = active = 0
  for s in range(mjm.nsensor):
    if int(mjm.sensor_history[s, 0]) > 0:  # forward reports a delayed sensor's history, not its fresh value
      continue
    t, oid, rid, adr, dim = (int(x[s]) for x in (mjm.sensor_type, mjm.sensor_objid, mjm.sensor_refid, mjm.sensor_adr, mjm.sensor_dim))
    cutoff, ot = float(mjm.sensor_cutoff[s]), int(mjm.sensor_objtype[s])
    for w in range(nw):
      out = np.zeros(3, dtype=np.float32)
      if t == C.SENS_MAGNETOMETER:
        hlib.hse_magnetometer(_ptr(_f(z["forward/site_xmat"][w, oid])), _ptr(_f(mag[w])), _ptr(out))
      elif t == C.SENS_CAMPROJECTION:
        hlib.hse_camprojection(_ptr(_f(z["forward/site_xpos"][w, oid])), _ptr(_f(z["forward/cam_xpos"][w, rid])), _ptr(_f(z["forward/cam_xmat"][w, rid])),
                               float(fovy[w, rid]), _ptr(_f(intr[w, rid])), _ptr(_f(mjm.cam_sensorsize[rid])), _ptr(_i(mjm.cam_resolution[rid])), _ptr(out))
      elif t == C.SENS_INSIDESITE:
        out[0] = hlib.hse_insidesite(ot, oid, _ptr(_f(z[f"forward/{pos_arrays[ot]}"][w, oid])), _ptr(_f(z["forward/subtree_com"][w, oid if ot in (C.OBJ_BODY, C.OBJ_XBODY) else 0])),
                                     float(mjm.body_mass[oid]) if ot == C.OBJ_BODY else 0.0, float(mjm.body_subtreemass[oid]) if ot == C.OBJ_BODY else 0.0,
                                     _ptr(_f(z["forward/site_xpos"][w, rid])), _ptr(_f(z["forward/site_xmat"][w, rid])), _ptr(_f(mjm.site_size[rid])), int(mjm.site_type[rid]))
      elif t in (C.SENS_TENDONLIMITPOS, C.SENS_TENDONLIMITVEL, C.SENS_TENDONLIMITFRC):  # k_sensor's scan, restated: the tendon's limit row, else 0
        e0 = int(z["forward/ne"][w] + z["forward/nf"][w])
        for e in range(e0, min(e0 + int(z["forward/nl"][w]), int(z["in/njmax"]))):
          if int(z["forward/efc_id"][w, e]) == oid and int(z["forward/efc_type"][w, e]) == C.CNSTR_LIMIT_TENDON:
            out[0] = {C.SENS_TENDONLIMITPOS: z["forward/efc_pos"][w, e] - z["forward/efc_margin"][w, e], C.SENS_TENDONLIMITVEL: z["forward/efc_vel"][w, e],
                      C.SENS_TENDONLIMITFRC: z["forward/efc_force"][w, e]}[t]
            active += 1
      elif t == C.SENS_TENDONACTFRC:
        out[0] = hlib.hse_tendon_actfrc(int(mjm.nu), _ptr(_i(mjm.actuator_trntype)), _ptr(_i(mjm.actuator_trnid)), _ptr(_f(z["forward/actuator_force"][w])), oid)
      else:
        continue
      got = out[:dim].astype(np.float64)
      if cutoff > 0:
        got = np.clip(got, -cutoff, cutoff)
      ref = want[w, adr : adr + dim]
      if t == C.SENS_INSIDESITE:
        np.testing.assert_array_equal(got, ref, err_msg=f"sensor {s} world {w}")
      else:
        np.testing.assert_allclose(got, ref, rtol=2e-5, atol=2e-5 * max(1.0, float(np.abs(ref).max())), err_msg=f"sensor {s} world {w}")
      checked += 1
  assert checked > 0
  if any(int(x) in (C.SENS_TENDONLIMITPOS, C.SENS_TENDONLIMITVEL, C.SENS_TENDONLIMITFRC) for x in mjm.sensor_type):
    assert active > 0, "no world has an active tendon limit row"
