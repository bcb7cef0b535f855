"""<contact> sensors without a GPU.

- The compiler: objtype / reftype / intprm / dim / adr of every side and data combination, the numeric contact_sensor_maxmatch, and every
  refusal by name, in the compiler and again at put_model's check of the arrays.
- The fp64 restatement (tests/contact_sensor_oracle.py) against the reference's own sensordata (tests/golden/contact_sensor_*.npz,
  tools/make_contact_sensor_goldens.py), fed the fixture's contacts and efc_force, with the reference's one divergent behaviour (the
  direction not following its contact through the sort) restated.
- The device source of mjb_sensor_contact.cuh, compiled as host C++ (tests/host_harness/sensor_contact_host.cpp), against the
  restatement on random contacts.
"""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io, mjcf
from tests import contact_sensor_oracle as O
from tests import contact_sensor_scenes as S

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_harness", "sensor_contact_host.cpp")
OUT = os.path.join(HERE, "host_harness", "_build", "libsensor_contact_host.so")
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "contact_sensor_*.npz")))

XML = """<mujoco><worldbody><geom name="floor" type="plane" size="5 5 .1"/>
<body name="a" pos="0 0 .1"><freejoint/><geom name="ga" type="box" size=".1 .1 .1"/><site name="s" type="box" size=".2 .2 .2"/>
<body name="a2" pos="0 0 .3"><joint name="h" type="hinge"/><geom name="ga2" type="sphere" size=".05"/></body></body></worldbody>
{custom}<sensor><jointpos joint="h"/>{sensors}</sensor></mujoco>"""


def _compile(sensors, custom=""):
  return mjcf.load_string(XML.format(sensors=sensors, custom=custom))


@pytest.mark.parametrize("sides,obj,ref", [
  ("", (C.OBJ_UNKNOWN, -1), (C.OBJ_UNKNOWN, -1)),
  ('site="s"', (C.OBJ_SITE, 0), (C.OBJ_UNKNOWN, -1)),
  ('geom1="ga"', (C.OBJ_GEOM, 1), (C.OBJ_UNKNOWN, -1)),
  ('body1="a"', (C.OBJ_BODY, 1), (C.OBJ_UNKNOWN, -1)),
  ('subtree1="a"', (C.OBJ_XBODY, 1), (C.OBJ_UNKNOWN, -1)),
  ('geom2="floor"', (C.OBJ_UNKNOWN, -1), (C.OBJ_GEOM, 0)),
  ('body1="a2" body2="world"', (C.OBJ_BODY, 2), (C.OBJ_BODY, 0)),
  ('geom1="floor" subtree2="a"', (C.OBJ_GEOM, 0), (C.OBJ_XBODY, 1)),
])
def test_compiler_sides(sides, obj, ref):
  m = _compile(f'<contact {sides}/>')
  assert (int(m.sensor_objtype[1]), int(m.sensor_objid[1])) == obj
  assert (int(m.sensor_reftype[1]), int(m.sensor_refid[1])) == ref
  assert int(m.sensor_type[1]) == C.SENS_CONTACT and int(m.sensor_datatype[1]) == 0 and int(m.sensor_needstage[1]) == 3
  assert m.sensor_intprm.tolist() == [[0, 0, 0], [1, 0, 1]]  # defaults: found, none, num 1; other sensors zeros
  assert int(m.sensor_dim[1]) == 1 and int(m.sensor_adr[1]) == 1


@pytest.mark.parametrize("data,bits,size", [
  ("found", 1, 1), ("force", 2, 3), ("torque", 4, 3), ("dist", 8, 1), ("pos", 16, 3), ("normal", 32, 3), ("tangent", 64, 3),
  (S.ALL, 127, 17), ("found dist normal", 1 + 8 + 32, 5),
])
@pytest.mark.parametrize("reduce", list(mjcf.CONTACT_REDUCE))
def test_compiler_intprm_and_dim(data, bits, size, reduce):
  m = _compile(f'<contact data="{data}" reduce="{reduce}" num="3"/><contact data="found"/>')
  assert m.sensor_intprm[1].tolist() == [bits, mjcf.CONTACT_REDUCE.index(reduce), 3]
  assert m.sensor_dim.tolist() == [1, 3 * size, 1]
  assert m.sensor_adr.tolist() == [0, 1, 1 + 3 * size]
  assert m.nsensordata == 2 + 3 * size
  np.testing.assert_array_equal(io._contact_sensor_intprm(m), m.sensor_intprm)


@pytest.mark.parametrize("attrs,msg", [
  ('site="s" geom1="ga"', "at most one of site / geom1 / body1 / subtree1"),
  ('body1="a" subtree1="a"', "at most one of site / geom1 / body1 / subtree1"),
  ('geom2="ga" body2="a"', "at most one of geom2 / body2 / subtree2"),
  ('data="force found"', "in the order found force torque"),
  ('data="found found"', "in the order found force torque"),
  ('data="foundx"', "unknown data keyword 'foundx'"),
  ('data=""', "at least one of"),
  ('reduce="min"', "unknown reduce 'min'"),
  ('num="0"', "num must be >= 1"),
  ('geom1="nope"', "unknown geom 'nope'"),
  ('body2="nope"', "unknown body 'nope'"),
  ('site="nope"', "unknown site 'nope'"),
])
def test_compiler_refusals_name_the_sensor(attrs, msg):
  with pytest.raises(ValueError, match="contact sensor 'bad'") as e:
    _compile(f'<contact name="bad" {attrs}/>')
  assert msg in str(e.value)


@pytest.mark.parametrize("field,value,msg", [
  ("intprm", (0, 0, 1), "unknown data bits"), ("intprm", (128, 0, 1), "unknown data bits"), ("intprm", (1, 4, 1), "unknown reduce"),
  ("intprm", (1, 0, 0), "num must be >= 1"), ("dim", 2, "not num"), ("objtype", C.OBJ_JOINT, "object type"),
  ("objid", 7, "unknown object"), ("reftype", C.OBJ_SITE, "object type"),
])
def test_put_model_checks_the_arrays_again(field, value, msg):
  m = _compile('<contact name="c" body1="a" body2="world"/>')
  if field == "intprm":
    m.sensor_intprm[1] = value
  else:
    getattr(m, "sensor_" + field)[1] = value
  with pytest.raises(ValueError, match=f"contact sensor 'c'.*{msg}"):
    io._contact_sensor_intprm(m)


def test_numeric_maxmatch():
  assert mjcf.contact_sensor_maxmatch(_compile("<contact/>")) == 64
  m = _compile("<contact/>", '<custom><numeric name="other" data="1 2"/><numeric name="contact_sensor_maxmatch" data="5"/></custom>')
  assert mjcf.contact_sensor_maxmatch(m) == 5 and m.numeric_adr.tolist() == [0, 2] and m.numeric_data.tolist() == [1, 2, 5]
  for bad in ("0", "-3", "2.5"):
    with pytest.raises(ValueError, match="contact_sensor_maxmatch"):
      _compile("<contact/>", f'<custom><numeric name="contact_sensor_maxmatch" data="{bad}"/></custom>')


def test_other_missing_sensor_types_are_still_refused_by_name():
  m = mjcf.load_string(XML.format(custom="", sensors='<contact/><rangefinder site="s"/><magnetometer site="s"/>'))
  assert sorted(m.sensor_unsupported) == ["magnetometer", "rangefinder"] and int(m.sensor_type[1]) == C.SENS_CONTACT


# ---------------------------------------------------------------- restatement against the reference's own results


def golden_worlds(z, mjm, tag):
  """(w, contacts of world w, efc_force row, site_xpos, site_xmat) for each world of a fixture's snapshot"""
  con = {k: z[f"{tag}/con_{k}"] for k in ("dist", "pos", "frame", "friction", "dim", "geom", "efc_address", "worldid", "type")}
  for w in range(z[f"{tag}/qpos"].shape[0]):
    yield w, O.world_contacts(con, w), z[f"{tag}/efc_force"][w], z[f"{tag}/site_xpos"][w], z[f"{tag}/site_xmat"][w].reshape(-1, 9)


def _history(mjm):
  h = getattr(mjm, "sensor_history", None)
  return np.zeros(mjm.nsensor, dtype=int) if h is None else np.asarray(h)[:, 0]


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[15:-4] for p in GOLDEN])
def test_restatement_meets_the_reference(path):
  name = os.path.basename(path)[len("contact_sensor_"):-4]
  z = np.load(path)
  mjm = mjcf.load_string(S.SCENES[name][0])
  njmax, maxmatch = int(z["njmax"]), int(z["maxmatch"])
  assert maxmatch == mjcf.contact_sensor_maxmatch(mjm)
  hist = _history(mjm)
  nchecked = 0
  for tag in ["forward"] + [f"step{i}" for i in range(3)]:
    for w, con, force, sxp, sxm in golden_worlds(z, mjm, tag):
      res, ovf = O.world_sensors(mjm, con, force, njmax, maxmatch, sxp, sxm, reference_dir=True)
      assert bool(z[f"{tag}/overflow"][w] & (1 << 6)) == ovf, (tag, w)
      for s, r in res.items():
        if hist[s] > 0:
          continue  # a delayed sensor reports its buffer
        got = z[f"{tag}/sensordata"][w, mjm.sensor_adr[s] : mjm.sensor_adr[s] + mjm.sensor_dim[s]]
        np.testing.assert_allclose(r["data"], got, rtol=1e-9, atol=1e-9, err_msg=f"{tag} world {w} sensor {mjm.names.sensor[s]}")
        nchecked += 1
  assert nchecked > 0


def test_fixtures_exercise_every_decision_edge():
  """the fixtures hold overflowing worlds, worlds with more matches than num and fewer, cut rows and both directions"""
  z = np.load(os.path.join(HERE, "golden", "contact_sensor_overflow.npz"))
  assert (z["forward/overflow"] & (1 << 6)).any()
  z = np.load(os.path.join(HERE, "golden", "contact_sensor_njmax.npz"))
  assert (z["forward/con_efc_address"][:, 0] == -1).any() or (z["forward/con_efc_address"] >= int(z["njmax"])).any()


# ---------------------------------------------------------------- the device source on the host


@pytest.fixture(scope="module")
def hlib():
  os.makedirs(os.path.dirname(OUT), exist_ok=True)
  cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
  subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", OUT], check=True)
  lib = ctypes.CDLL(OUT)
  p, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
  for name, args, res in (("hsc_force", [i, i, p, p, p, i, p], None), ("hsc_inside", [p, p, p, i, p], i), ("hsc_match", [p, i, i, i, i, i, i, i, i], i),
                          ("hsc_slot_size", [i], i), ("hsc_slot", [i, i, f, p, f, p, p, p], None), ("hsc_netforce", [i, i, i, p, p, p, p, p], None),
                          ("hsc_sort", [p, p, p, i], None)):
    getattr(lib, name).argtypes = args
    getattr(lib, name).restype = res
  return lib


def _ptr(a):
  return a.ctypes.data_as(ctypes.c_void_p)


def test_device_force_decode_matches_restatement(hlib):
  rng = np.random.default_rng(1)
  for cone in (C.CONE_PYRAMIDAL, C.CONE_ELLIPTIC):
    for _ in range(300):
      dim = int(rng.choice([1, 3, 4, 6]))
      nrow = dim if cone == C.CONE_ELLIPTIC else (1 if dim == 1 else 2 * (dim - 1))
      njmax = int(rng.integers(4, 16))
      base = int(rng.integers(0, njmax + 2))
      adr = np.array([base + k if base + k < njmax else -1 for k in range(nrow)] + [-1] * (10 - nrow), dtype=np.int32)
      if rng.random() < 0.1:
        adr[:] = -1
      force = rng.normal(size=njmax).astype(np.float32)
      mu = rng.uniform(0.1, 1.0, 5).astype(np.float32)
      out = np.zeros(6, dtype=np.float32)
      hlib.hsc_force(cone, njmax, _ptr(force), _ptr(adr), _ptr(mu), dim, _ptr(out))
      want = O.contact_force(cone, njmax, force.astype(float), adr, mu.astype(float), dim)
      np.testing.assert_allclose(out, want, rtol=1e-6, atol=1e-6)


def test_device_site_volumes_match_restatement(hlib):
  rng = np.random.default_rng(2)
  for typ in (C.GEOM_SPHERE, C.GEOM_CAPSULE, C.GEOM_ELLIPSOID, C.GEOM_CYLINDER, C.GEOM_BOX):
    agree = 0
    for _ in range(500):
      q = rng.normal(size=4)
      q /= np.linalg.norm(q)
      w, x, y, zq = q
      mat = np.array([[1 - 2 * (y * y + zq * zq), 2 * (x * y - zq * w), 2 * (x * zq + y * w)], [2 * (x * y + zq * w), 1 - 2 * (x * x + zq * zq), 2 * (y * zq - x * w)],
                      [2 * (x * zq - y * w), 2 * (y * zq + x * w), 1 - 2 * (x * x + y * y)]], dtype=np.float32)
      pos, size, p = (rng.normal(size=3) * 0.1).astype(np.float32), rng.uniform(0.05, 0.3, 3).astype(np.float32), (rng.normal(size=3) * 0.3).astype(np.float32)
      got = hlib.hsc_inside(_ptr(pos), _ptr(mat.reshape(-1)), _ptr(size), typ, _ptr(p))
      want = O.inside_site(pos.astype(float), mat.astype(float), size.astype(float), typ, p.astype(float))
      agree += int(bool(got) == bool(want))
    assert agree >= 498, (typ, agree)  # fp32 against fp64 on the boundary


def test_device_matching_matches_restatement(hlib):
  parent = np.array([0, 0, 1, 2, 1, 0, 5], dtype=np.int32)  # two trees: 1-2-3, 1-4 and 5-6
  gbody = np.arange(7)
  kinds = [(C.OBJ_UNKNOWN, -1), (C.OBJ_SITE, 0)] + [(t, i) for t in (C.OBJ_GEOM, C.OBJ_BODY, C.OBJ_XBODY) for i in range(7)]
  for ot, oi in kinds:
    for rt, ri in [k for k in kinds if k[0] != C.OBJ_SITE]:
      for g1 in range(7):
        for g2 in range(7):
          got = hlib.hsc_match(_ptr(parent), ot, oi, rt, ri, g1, int(gbody[g1]), g2, int(gbody[g2]))
          assert got == O.match_dir(parent, ot, oi, rt, ri, g1, int(gbody[g1]), g2, int(gbody[g2])), (ot, oi, rt, ri, g1, g2)


def test_device_sort_is_by_criterion_then_pool_index(hlib):
  rng = np.random.default_rng(3)
  for n in list(range(1, 70)) + [127, 128, 129, 500]:
    cid = np.sort(rng.choice(10 * n, n, replace=False)).astype(np.int32)  # stored in pool order
    crit = rng.choice([-1.0, 0.0, 0.5, 2.0], n).astype(np.float32) if n % 2 else rng.normal(size=n).astype(np.float32)
    dirs = rng.choice([-1.0, 1.0], n).astype(np.float32)
    want = sorted(zip(crit.tolist(), cid.tolist(), dirs.tolist()))
    hlib.hsc_sort(_ptr(cid), _ptr(crit), _ptr(dirs), n)
    assert list(zip(crit.tolist(), cid.tolist(), dirs.tolist())) == want, n


def test_device_slots_match_restatement(hlib):
  rng = np.random.default_rng(4)
  for _ in range(200):
    dataspec = int(rng.integers(1, 128))
    size = hlib.hsc_slot_size(dataspec)
    assert size == mjcf.contact_slot_size(dataspec)
    n = int(rng.integers(0, 6))
    dirs = rng.choice([-1.0, 1.0], n).astype(np.float32)
    f = rng.normal(size=(n, 6)).astype(np.float32)
    pos = rng.normal(size=(n, 3)).astype(np.float32)
    fr = np.stack([np.linalg.qr(rng.normal(size=(3, 3)))[0].T.reshape(-1) for _ in range(n)]).astype(np.float32) if n else np.zeros((0, 9), np.float32)
    dist = rng.normal(size=n).astype(np.float32)
    for i in range(n):
      out = np.zeros(size, dtype=np.float32)
      hlib.hsc_slot(dataspec, n + 2, float(dirs[i]), _ptr(f[i]), float(dist[i]), _ptr(pos[i]), _ptr(fr[i]), _ptr(out))
      np.testing.assert_allclose(out, O.slot(dataspec, n + 2, float(dirs[i]), f[i].astype(float), float(dist[i]), pos[i].astype(float), fr[i]), rtol=1e-6, atol=1e-6)
    out = np.zeros(size, dtype=np.float32)
    hlib.hsc_netforce(dataspec, n + 2, n, _ptr(dirs), _ptr(np.ascontiguousarray(f)), _ptr(np.ascontiguousarray(pos)), _ptr(np.ascontiguousarray(fr)), _ptr(out))
    want = O.netforce(dataspec, n + 2, [(float(dirs[i]), f[i].astype(float), pos[i].astype(float), fr[i]) for i in range(n)])
    np.testing.assert_allclose(out, want, rtol=2e-5, atol=2e-5)
