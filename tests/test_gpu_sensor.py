"""k_sensor against tests/sensor_oracle.py fed the GPU's own inputs, at every instantiation, stage call, lane and launch shape.

Each case runs forward(), reads back what the launches before k_sensor left in Data and compares every world's sensordata slots (the
ones k_sensor writes) and the fields the same launch computes first (subtree_linvel / subtree_angmom, cacc / cfrc_ext / cfrc_int) with
the fp64 restatement.  Then it poisons sensordata and those fields with NaN and calls sensor_pos, sensor_vel and sensor_acc one after
the other: each call writes its own stage's slots (matching the oracle) and leaves the later stages' slots poisoned, and after the
three calls every slot and field is bit-identical to what forward() wrote.

Tolerance: |got - want| <= 64 eps32 magnitude (constraint_oracle.E).  The longest chains (the accelerometer: cacc summed down the tree,
rotated, plus a cross product of two rotated velocities; cfrc_int summed up the tree) are a few tens of fp32 operations deep.  A
transposed rotation, a dropped cross term, another world's model entry or a wrong row moves a value by a sizeable fraction of its
magnitude.  Decisions (touch's force sign and ray hits, insidesite, the cutoff clamps) sit at least 1e-5 from their thresholds in
every scene (the oracle raises otherwise), so fp32 and fp64 take the same branches."""

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf
from tests import constraint_oracle as co
from tests import sensor_oracle as so
from tests import util

pytestmark = pytest.mark.gpu

EPS32 = float(np.finfo(np.float32).eps)
TOL = 64 * EPS32
DATA = ("qpos", "qvel", "qacc", "time", "xpos", "xquat", "xmat", "xipos", "ximat", "geom_xpos", "geom_xmat", "site_xpos", "site_xmat", "cam_xpos",
        "cam_xmat", "subtree_com", "cdof", "cinert", "cvel", "cdof_dot", "ten_length", "ten_velocity", "actuator_length", "actuator_velocity",
        "actuator_force", "qfrc_actuator", "xfrc_applied", "ne", "nf", "nl")
EFC = ("force", "pos", "margin", "vel", "type", "id")
CON = ("geom", "dim", "frame", "pos", "friction", "efc_address")
LAUNCH = ("subtree_linvel", "subtree_angmom", "cacc", "cfrc_ext", "cfrc_int")


def selected(m, mjm):
  """CPU restatement of launch_sensor's instantiation choice <BAT, EXTRA>: BAT when any per-world float field holds more than one entry,
  EXTRA when the model has a magnetometer, camprojection, insidesite, tendon limit or tendonactfrc sensor."""
  from mujoco_warp_b200._src import io

  def many(x):
    return isinstance(x, torch.Tensor) and x.dim() >= 1 and x.shape[0] > 1

  names = io._FLOAT_FIELDS + list(io._BATCHABLE_EXTRA) + list(io._RENDER_FLOATS)
  bat = any(many(getattr(m, n, None)) for n in names) or many(m.opt.magnetic)
  return bat, bool(np.isin(np.asarray(mjm.sensor_type), so.EXTRA).any())


def _np(t):
  return t.detach().cpu().numpy()


def read_back(d):
  """Every input of the oracle, for all worlds at once."""
  h = {f: _np(getattr(d, f)) for f in DATA}
  h.update({"efc_" + f: _np(getattr(d.efc, f)) for f in EFC})
  n = int(_np(d.nacon)[0])
  h["con_worldid"] = _np(d.contact.worldid)[:n]
  h.update({"con_" + f: _np(getattr(d.contact, f))[:n] for f in CON})
  return h


def world_inputs(h, w):
  st = {f: (h[f][w] if h[f].ndim and h[f].shape[0] else h[f]) for f in h if not f.startswith("con_")}
  for f in ("ne", "nf", "nl"):
    st[f] = int(h[f].reshape(-1)[w])
  ids = np.nonzero(h["con_worldid"] == w)[0]
  for f in CON:
    st["con_" + f] = h["con_" + f][ids]
  st["time"] = h["time"].reshape(-1)[w]
  return st


def close(name, got, want, mag):
  got = np.asarray(got, dtype=np.float64)
  assert np.isfinite(got).all(), f"{name}: unwritten (NaN) entries at {np.argwhere(~np.isfinite(got))[:4].tolist()}"
  bad = np.abs(got - want) > TOL * mag + 1e-30
  assert not bad.any(), f"{name}: at {np.argwhere(bad)[0].tolist()}: got {got[bad][0]:.9g}, want {want[bad][0]:.9g}, magnitude {mag[bad][0]:.3g}"


def compare(mjm, batched, d, njmax, worlds, stages=7, fields=None):
  """sensordata (slots the oracle writes for `stages`) and the in-launch fields of every world in `worlds` against the oracle; the slots
  and fields the launch leaves alone must still hold their poison (NaN) when `fields` is given (the stage-call checks)."""
  h = read_back(d)
  sd = _np(d.sensordata)
  got_f = {f: _np(getattr(d, f)) for f in LAUNCH}
  out = {}
  for w in worlds:
    R = so.sensor(co.world_model(mjm, batched, w), world_inputs(h, w), njmax, stages=stages)
    out[w] = R
    val, mag = R["sensordata"]
    done = ~np.isnan(val)
    close(f"w{w} sensordata (stages {stages})", sd[w][done], val[done], mag[done])
    if fields is not None:
      mine = owned(mjm)
      left = mine & ~done
      assert np.isnan(sd[w][left]).all(), f"w{w}: stages {stages} wrote slots {np.nonzero(left & ~np.isnan(sd[w]))[0].tolist()} of a later stage"
    for f in LAUNCH:
      if f in R:
        close(f"w{w} {f}", got_f[f][w].reshape(R[f][0].shape), *R[f])
      elif fields is not None and f in fields:
        assert np.isnan(got_f[f][w]).all(), f"w{w}: {f} written by stages {stages}"
  return out


def owned(mjm):
  """The sensordata slots k_sensor writes."""
  extra = bool(np.isin(np.asarray(mjm.sensor_type), so.EXTRA).any())
  mask = np.zeros(int(mjm.nsensordata), dtype=bool)
  for s in range(int(mjm.nsensor)):
    if so.carried(mjm, s, extra):
      mask[int(mjm.sensor_adr[s]) : int(mjm.sensor_adr[s]) + int(mjm.sensor_dim[s])] = True
  return mask


def run(mjm, nworld, njmax=128, nconmax=64, qpos=None, qvel=None, batched=None, expect=None, worlds=None, disable=0):
  """forward, compare; poison, sensor_pos / sensor_vel / sensor_acc, compare each; the three calls reproduce forward bit for bit."""
  import mujoco_warp_b200 as mjw

  batched = batched or {}
  m = mjw.put_model(mjm, batch_sizes={n: x.shape[0] for n, x in batched.items()})
  for n, x in batched.items():
    getattr(m, n).copy_(torch.as_tensor(np.asarray(x, dtype=np.float32)))
  if expect is not None:
    assert selected(m, mjm) == expect, f"k_sensor<BAT, EXTRA> = {selected(m, mjm)}, the case is meant for {expect}"
  d = mjw.make_data(mjm, nworld=nworld, nconmax=nconmax, njmax=njmax, m=m)
  if qpos is not None:
    d.qpos.copy_(torch.as_tensor(np.asarray(qpos, dtype=np.float32)))
  if qvel is not None:
    d.qvel.copy_(torch.as_tensor(np.asarray(qvel, dtype=np.float32)))
  mjw.forward(m, d)
  torch.cuda.synchronize()
  worlds = range(nworld) if worlds is None else worlds
  if disable:  # after forward(): the stage calls alone run with the flag
    m.opt.disableflags = int(m.opt.disableflags) | disable
    mjm.opt.disableflags = int(mjm.opt.disableflags) | disable
  ref = compare(mjm, batched, d, njmax, worlds) if not disable else None
  fwd = {f: getattr(d, f).clone() for f in ("sensordata",) + LAUNCH}
  for f in ("sensordata",) + LAUNCH:
    getattr(d, f).fill_(float("nan"))
  for stages, call in ((1, mjw.sensor_pos), (3, mjw.sensor_vel), (7, mjw.sensor_acc)):
    call(m, d)
    torch.cuda.synchronize()
    last = compare(mjm, batched, d, njmax, worlds, stages=stages, fields=LAUNCH)
  written = set(next(iter(last.values())))  # sensordata and the in-launch fields this model's launch computes
  if not disable:
    for f, x in fwd.items():
      if f not in written:
        continue
      a, b = _np(getattr(d, f)), _np(x)
      assert np.array_equal(a, b, equal_nan=True), f"{f}: sensor_pos + sensor_vel + sensor_acc differ from forward at {np.argwhere(~((a == b) | (np.isnan(a) & np.isnan(b))))[:4].tolist()}"
  else:
    assert np.isnan(_np(d.sensordata)).all(), "DSBL_SENSOR: sensordata written"
  return m, d, ref


# ---------------------------------------------------------------- scenes


def _state(mjm, nworld, seed=1234, noise=0.01, vel=0.3):
  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=0, seed=seed, qpos_noise=noise, qvel_noise=vel, exact_world0=False)
  return qpos, qvel


def sensor_scene(extra=False, cone="pyramidal", sensors=None, cutoff=False):
  """util.sensor_xml(): every core type, five touch site shapes on contacting bodies, joint limits, both cones; `extra` adds an
  insidesite sensor (the EXTRA build, for its core types); `sensors` replaces the sensor block."""
  x = util.sensor_xml()
  if cone == "elliptic":
    x = x.replace('<option timestep="0.004"', '<option cone="elliptic" impratio="2" timestep="0.004"')
  add = ""
  if extra:  # cap0's frame origin lies at the centre of its capsule site; st0 lies 0.05 from ball0's, far outside tz_sph
    add += '<insidesite objtype="xbody" objname="cap0" site="tz_cap"/> <insidesite objtype="site" objname="st0" site="tz_cyl"/>'
  if cutoff:
    add += CUTOFF
  if sensors is not None:
    i, j = x.index("<sensor>"), x.index("</sensor>")
    x = x[: i + len("<sensor>")] + sensors + x[j:]
  elif add:
    x = x.replace("<clock name=\"clk\"/>", "<clock name=\"clk\"/>" + add)
  return mjcf.load_string(x)


# cutoff on each datatype: REAL clamped on both sides, POSITIVE (touch) from above, AXIS and QUATERNION data never
CUTOFF = ('<framepos objtype="site" objname="imu" cutoff="0.05"/> <framelinvel objtype="site" objname="imu" cutoff="0.02"/>'
          '<touch site="tz_box" cutoff="0.5"/> <framexaxis objtype="site" objname="imu" cutoff="0.1"/>'
          '<framequat objtype="site" objname="imu" cutoff="0.1"/> <ballquat joint="ball" cutoff="0.05"/>')

OBJ = (("body", "pend"), ("xbody", "cap0"), ("geom", "c1"), ("site", "imu"), ("camera", "c0"))


def _quats(mjm, nb, seed=5):
  """Per-world body_iquat, geom_quat, site_quat and cam_quat: each entry turned by a different small rotation."""
  rng = np.random.default_rng(seed)
  out = {}
  for n in ("body_iquat", "geom_quat", "site_quat", "cam_quat"):
    q0 = np.asarray(getattr(mjm, n), dtype=np.float64).reshape(-1, 4)
    q = np.empty((nb,) + q0.shape)
    for k in range(nb):
      d = np.concatenate([np.ones((len(q0), 1)), rng.uniform(-0.3, 0.3, (len(q0), 3))], 1)
      d /= np.linalg.norm(d, axis=1, keepdims=True)
      q[k] = _qmul_np(q0, d)
    out[n] = q / np.linalg.norm(q, axis=-1, keepdims=True)
  return out


def _qmul_np(u, v):
  w1, x1, y1, z1 = u.T
  w2, x2, y2, z2 = v.T
  return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                   w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], 1)


def pair_sensors():
  """framepos, framexaxis, framequat, framelinvel and frameangvel for every object type against every reference type."""
  out = []
  for ot, on in OBJ:
    for rt, rn in OBJ:
      for kind in ("framepos", "framexaxis", "framequat", "framelinvel", "frameangvel"):
        out.append(f'<{kind} objtype="{ot}" objname="{on}" reftype="{rt}" refname="{rn}"/>')
    for kind in ("framepos", "frameyaxis", "framezaxis", "framequat", "framelinvel", "frameangvel", "framelinacc", "frameangacc"):
      out.append(f'<{kind} objtype="{ot}" objname="{on}"/>')
  return " ".join(out)


# ---------------------------------------------------------------- cases


@pytest.mark.parametrize("bat", [False, True])
@pytest.mark.parametrize("extra", [False, True])
def test_instantiations(built, extra, bat):
  """All four k_sensor<BAT, EXTRA>; the batched model turns every local frame per world, so framequat reads each world's body_iquat,
  geom_quat, site_quat and cam_quat."""
  mjm = sensor_scene(extra=extra)
  nworld = 5
  qpos, qvel = _state(mjm, nworld)
  run(mjm, nworld, qpos=qpos, qvel=qvel, batched=_quats(mjm, 3) if bat else None, expect=(bat, extra))


@pytest.mark.parametrize("nworld", [1, 3, 7, 33])
def test_world_counts(built, nworld):
  """Per-world frames with nb = 3, which does not divide 7 or 33."""
  mjm = sensor_scene()
  qpos, qvel = _state(mjm, nworld)
  run(mjm, nworld, qpos=qpos, qvel=qvel, batched=_quats(mjm, 3), expect=(True, False))


def test_split_worlds(built):
  """1025 worlds: forward runs two halves of 513 and 512 worlds on their own streams, and k_sensor's second launch starts at world 513."""
  mjm = sensor_scene()
  nworld = 1025
  qpos, qvel = _state(mjm, nworld)
  worlds = list(range(4)) + list(range(505, 521)) + list(range(1017, 1025))
  run(mjm, nworld, qpos=qpos, qvel=qvel, batched=_quats(mjm, 3), expect=(True, False), worlds=worlds)


POOL = ['<jointpos joint="hinge"/>', '<framequat objtype="site" objname="imu" reftype="body" refname="ball0"/>', '<gyro site="imu"/>',
        '<accelerometer site="st0"/>', '<subtreeangmom body="arm"/>', '<touch site="tz_cap"/>', '<framelinvel objtype="geom" objname="tip"/>',
        '<force site="imu"/>', '<ballquat joint="ball"/>', '<jointlimitfrc joint="slide"/>', '<clock/>', '<torque site="st0"/>',
        '<framexaxis objtype="camera" objname="c0" reftype="xbody" refname="fore"/>', '<subtreelinvel body="fore"/>', '<velocimeter site="imu"/>',
        '<framelinacc objtype="body" objname="ball1"/>', '<actuatorfrc actuator="p_hinge"/>']


@pytest.mark.parametrize("nsensor", [31, 32, 33, 70])
def test_sensor_counts(built, nsensor):
  """The lane loop at one warp's worth of sensors, one more, and more than two."""
  mjm = sensor_scene(sensors=" ".join(POOL[i % len(POOL)] for i in range(nsensor)))
  assert int(mjm.nsensor) == nsensor
  qpos, qvel = _state(mjm, 3)
  run(mjm, 3, qpos=qpos, qvel=qvel)


def test_batched_frames_meet_the_reference(built):
  """The scene of tests/golden/sensor_batched.npz (per-world body_iquat / geom_quat / site_quat / cam_quat, nb = 3 over 4 worlds; frame
  sensors of every object type against every reference type) from the fixture's state: the oracle fed the GPU's inputs as everywhere
  here, and the reference's own sensordata within fp32 rounding of unit-scale kinematics."""
  import os

  from tests import sensor_scenes as S

  g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sensor_batched.npz"))
  mjm = S.load()
  batched = {k: g[f"in/{k}"] for k in ("body_iquat", "geom_quat", "site_quat", "cam_quat")}
  _, d, _ = run(mjm, S.NWORLD, njmax=8, nconmax=4, qpos=g["in/qpos"], qvel=g["in/qvel"], batched=batched, expect=(True, False))
  want = g["forward/sensordata"]
  err = np.abs(_np(d.sensordata) - want)
  assert err.max() <= 2e-5 * max(1.0, np.abs(want).max()), f"sensordata off the reference by {err.max():.3g} at {np.unravel_index(err.argmax(), err.shape)}"


def test_every_object_and_reference_type(built):
  """Every objtype x reftype pair the frame sensors accept, per-world frames."""
  mjm = sensor_scene(sensors=pair_sensors())
  qpos, qvel = _state(mjm, 4)
  run(mjm, 4, qpos=qpos, qvel=qvel, batched=_quats(mjm, 4), expect=(True, False))


def test_many_bodies(built):
  """1100 static bodies, each with a site and a framepos sensor on every 50th: 12 nbody floats of dynamic shared memory exceed 48 KB, so
  the launch takes the opt-in path; subtree and acceleration sensors make k_sensor run subtree_vel and rne_postconstraint over them."""
  n = 1100
  bodies = "".join(f'<body name="b{i}" pos="{0.01 * (i % 40):.2f} {0.01 * (i // 40):.2f} 2"><site name="s{i}" pos="0 0 0.01"/></body>' for i in range(n))
  sensors = "".join(f'<framepos objtype="site" objname="s{i}" reftype="site" refname="imu"/>' for i in range(0, n, 50))
  sensors += '<subtreelinvel body="ball0"/> <subtreeangmom body="arm"/> <accelerometer site="imu"/> <force site="st0"/> <touch site="tz_sph"/>'
  x = util.sensor_xml().replace("</worldbody>", bodies + "</worldbody>")
  i, j = x.index("<sensor>"), x.index("</sensor>")
  mjm = mjcf.load_string(x[: i + len("<sensor>")] + sensors + x[j:])
  assert int(mjm.nbody) > 1024 and 12 * int(mjm.nbody) * 4 > 48 * 1024
  qpos, qvel = _state(mjm, 2)
  run(mjm, 2, qpos=qpos, qvel=qvel)


def _rows(mjm, nworld=3, cone="pyramidal", njmax=256):
  import mujoco_warp_b200 as mjw

  qpos, qvel = _state(mjm, nworld)
  slide = int(mjm.jnt_qposadr[list(np.asarray(mjm.jnt_type)).index(C.JNT_SLIDE)])
  qpos[:, slide] = np.where(np.arange(nworld) % 2 == 0, -0.25, 0.08)  # the slide and the hinge past either end of their ranges
  qpos[:, slide + 1] = np.where(np.arange(nworld) % 2 == 0, 1.2, -0.8)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, nconmax=64, njmax=njmax, m=m)
  d.qpos.copy_(torch.as_tensor(qpos, dtype=torch.float32)); d.qvel.copy_(torch.as_tensor(qvel, dtype=torch.float32))
  mjw.forward(m, d)
  torch.cuda.synchronize()
  return qpos, qvel, read_back(d)


def test_limit_rows_at_njmax(built):
  """The joint-limit sensors with their rows inside njmax, straddling it (the first limit row inside, the second past) and past it
  (ne + nf >= njmax)."""
  mjm = sensor_scene()
  qpos, qvel, h = _rows(mjm)
  e0 = int(h["ne"][0] + h["nf"][0])
  nl = int(h["nl"][0])
  assert nl >= 2 and (h["efc_type"][0, e0 : e0 + nl] == C.CNSTR_LIMIT_JOINT).all(), "the case needs both joint limits active in world 0"
  for njmax in (e0 + nl, e0 + 1, e0, e0 - 1):
    run(mjm, 3, njmax=njmax, qpos=qpos, qvel=qvel)


@pytest.mark.parametrize("cone", ["pyramidal", "elliptic"])
def test_touch(built, cone):
  """Touch under both cones: contacts of condim 3, 4 and 6 (condim 1: the rake below), the sensor body as the contact's first and as
  its second body."""
  mjm = sensor_scene(cone=cone)
  qpos, qvel = _state(mjm, 5)
  _, d, ref = run(mjm, 5, qpos=qpos, qvel=qvel)
  h = read_back(d)
  sides, dims = set(), set()
  gb = np.asarray(mjm.geom_bodyid)
  touch_bodies = {int(mjm.site_bodyid[int(mjm.sensor_objid[s])]) for s in range(mjm.nsensor) if int(mjm.sensor_type[s]) == C.SENS_TOUCH}
  for c in range(len(h["con_worldid"])):
    b = gb[h["con_geom"][c]]
    a = h["con_efc_address"][c, 0]
    w = h["con_worldid"][c]
    if a < 0 or h["efc_force"][w, a] <= 0:
      continue
    dims.add(int(h["con_dim"][c]))
    sides |= {k for k in (0, 1) if int(b[k]) in touch_bodies}
  assert sides == {0, 1} and dims >= {3, 4, 6}, f"sensor body sides {sides}, condims {dims}"


@pytest.mark.parametrize("cone", ["pyramidal", "elliptic"])
def test_touch_more_than_32_contacts(built, cone):
  """A touch site around the rake under both cones: 40 contacts of condim 1, 3 and 4 in one world (elliptic condim 1: touch reads the
  normal row alone), the pool interleaving two worlds' contacts."""
  x = util.rake_xml().replace('<body name="rake" pos="0 0 0.049">', '<body name="rake" pos="0 0 0.0487">')
  if cone == "elliptic":
    x = x.replace('<option timestep="0.002"', '<option cone="elliptic" timestep="0.002"')
  x = x.replace("<freejoint/>", '<freejoint/><site name="zone" type="box" size="0.6 0.6 0.2" pos="0.42 0.24 0"/>')
  x = x.replace("</worldbody>", '</worldbody><sensor><touch site="zone"/><touch site="zone" cutoff="3"/></sensor>')
  mjm = mjcf.load_string(x)
  assert int(mjm.opt.cone) == (C.CONE_ELLIPTIC if cone == "elliptic" else C.CONE_PYRAMIDAL)
  _, d, _ = run(mjm, 2, njmax=256, nconmax=128)
  h = read_back(d)
  assert (np.bincount(h["con_worldid"], minlength=2) > 32).all() and set(h["con_dim"].tolist()) == {1, 3, 4}
  one = [c for c in range(len(h["con_worldid"])) if h["con_dim"][c] == 1 and h["efc_force"][h["con_worldid"][c], h["con_efc_address"][c, 0]] > 0]
  assert one, "no condim-1 contact carries a normal force"


def test_touch_rows_cut_by_njmax(built):
  """Pyramidal rows of a touch-sensed contact cut by njmax: the rows past it (address -1) add nothing to the normal force, the rows
  below it do."""
  mjm = sensor_scene()
  qpos, qvel, h = _rows(mjm)
  gb = np.asarray(mjm.geom_bodyid)
  touch_bodies = {int(mjm.site_bodyid[int(mjm.sensor_objid[s])]) for s in range(mjm.nsensor) if int(mjm.sensor_type[s]) == C.SENS_TOUCH}
  w0 = np.nonzero(h["con_worldid"] == 0)[0]
  k = next(c for c in w0 if h["con_dim"][c] >= 3 and h["con_efc_address"][c, 0] >= 0 and touch_bodies & set(gb[h["con_geom"][c]].tolist())
           and h["efc_force"][0, h["con_efc_address"][c, 0]] > 0)
  a0, nrow = int(h["con_efc_address"][k, 0]), 2 * (int(h["con_dim"][k]) - 1)
  for njmax in (a0 + 1, a0 + 3):
    _, d, _ = run(mjm, 3, njmax=njmax, qpos=qpos, qvel=qvel)
    h2 = read_back(d)  # the same contact, found by its world and geoms: worlds take their pool blocks in no fixed order
    k2 = [c for c in np.nonzero(h2["con_worldid"] == 0)[0] if (h2["con_geom"][c] == h["con_geom"][k]).all()]
    assert len(k2) == 1
    adr = h2["con_efc_address"][k2[0], :nrow]
    assert adr[0] == a0 and (adr[njmax - a0 :] == -1).all() and (adr[: njmax - a0] >= 0).all(), f"njmax {njmax}: addresses {adr}"
    assert _np(d.efc.force)[0, a0] > 0


def test_cutoff(built):
  """cutoff on REAL (both sides), POSITIVE (from above), AXIS and QUATERNION data (never); cutoff 0 elsewhere."""
  mjm = sensor_scene(cutoff=True)
  dt = {int(mjm.sensor_datatype[s]) for s in range(mjm.nsensor) if float(mjm.sensor_cutoff[s]) > 0}
  assert dt == {so.REAL, so.POSITIVE, so.AXIS, so.QUATERNION}
  qpos, qvel = _state(mjm, 5, vel=1.0)
  _, d, _ = run(mjm, 5, qpos=qpos, qvel=qvel)
  sd = _np(d.sensordata)
  clamped_touch = False
  for s in range(mjm.nsensor):  # the REAL cutoffs clamp in some world on each side
    c = float(mjm.sensor_cutoff[s])
    if c > 0 and int(mjm.sensor_datatype[s]) == so.REAL and int(mjm.sensor_type[s]) == C.SENS_FRAMEPOS:
      x = sd[:, int(mjm.sensor_adr[s]) : int(mjm.sensor_adr[s]) + 3]
      assert (x == np.float32(c)).any() and (x == -np.float32(c)).any()
    if c == 0.5 and int(mjm.sensor_type[s]) == C.SENS_TOUCH:  # and the POSITIVE one of CUTOFF (touch) from above
      assert (sd[:, int(mjm.sensor_adr[s])] == np.float32(c)).any()
      clamped_touch = True
  assert clamped_touch


def test_disabled(built):
  """DSBL_SENSOR: sensordata keeps its poison; subtree_linvel / subtree_angmom and cacc / cfrc_ext / cfrc_int are still computed
  (tests/test_gpu_body_stages.py) and match the oracle."""
  mjm = sensor_scene()
  qpos, qvel = _state(mjm, 3)
  try:
    run(mjm, 3, qpos=qpos, qvel=qvel, disable=C.DSBL_SENSOR)
  finally:
    mjm.opt.disableflags = int(mjm.opt.disableflags) & ~C.DSBL_SENSOR
