"""tests/sensor_oracle.py against the reference's own sensordata and in-launch fields (tests/golden/*.npz).

The oracle is fed each fixture's own state, so only its arithmetic is under test: every sensordata slot k_sensor writes, and cacc /
cfrc_ext / cfrc_int / subtree_linvel / subtree_angmom, to 1e-9 of their magnitude (the fixtures hold fp64 results of the unmodified
reference).  States:
  forward  what forward() computed from the seeded state;
  step{s}  what step s's forward computed: positions, velocities-derived fields, the solver's qacc and rows as stored at step s, with
           qpos / qvel / time as the previous snapshot left them (the step then integrates them)."""

import os

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from tests import constraint_oracle as co
from tests import sensor_oracle as so
from tests.test_oracle_golden_pipeline import GOLD_DIR, SCENES, load_scene

REL = 1e-9
KIN = ("xpos", "xquat", "xmat", "xipos", "ximat", "geom_xpos", "geom_xmat", "site_xpos", "site_xmat", "cam_xpos", "cam_xmat", "subtree_com",
       "cdof", "cinert", "cvel", "cdof_dot", "qacc", "ten_length", "ten_velocity", "actuator_length", "actuator_velocity", "actuator_force",
       "qfrc_actuator")
EFC = ("efc_force", "efc_pos", "efc_margin", "efc_vel", "efc_type", "efc_id")
CON = ("geom", "dim", "frame", "pos", "friction", "efc_address")


def world_state(g, tag, prev, w, xfrc=None):
  """World w's sensor inputs from fixture snapshot `tag`, with qpos / qvel / time from `prev` (None: the fixture's own)."""
  st = {f: g[f"{tag}/{f}"][w] for f in KIN + EFC if f"{tag}/{f}" in g}
  for f in ("qpos", "qvel", "time"):
    src = f"{prev}/{f}" if prev else f"{tag}/{f}"
    if src in g:
      st[f] = np.asarray(g[src]).reshape(g[src].shape[0], -1)[w]
  for f in ("ne", "nf", "nl"):
    if f"{tag}/{f}" in g:
      st[f] = int(np.asarray(g[f"{tag}/{f}"]).reshape(-1)[w])
  if f"{tag}/con_worldid" in g:
    n = int(np.asarray(g[f"{tag}/nacon"]).reshape(-1)[0])
    ids = np.nonzero(g[f"{tag}/con_worldid"][:n] == w)[0]
    for f in CON:
      st["con_" + f] = g[f"{tag}/con_{f}"][ids]
  if xfrc is not None:
    st["xfrc_applied"] = xfrc[w]
  return st


def check(name, got, want, mag, rel=REL):
  err = np.abs(np.asarray(got, dtype=np.float64) - want)
  bad = err > rel * np.maximum(mag, 1.0)
  assert not bad.any(), f"{name}: worst at {np.argwhere(bad)[0]}: got {np.asarray(got)[bad][0]!r}, want {want[bad][0]!r}, mag {mag[bad][0]:.3g}"


def compare_sensors(mjm, g, name, tags, batched=None, only=None):
  """Every slot the oracle writes against the fixture's sensordata; returns the sensor types compared.  A world state whose decisions sit
  on a knife edge is skipped, but at least as many states as the fixture has worlds must have been compared."""
  njmax = int(g["in/njmax"])
  seen, checked = set(), 0
  for tag, prev, key in tags:
    want_all = g[key]
    for w in range(want_all.shape[0]):
      m = co.world_model(mjm, batched, w)
      sens = [s for s in range(mjm.nsensor) if only is None or int(mjm.sensor_type[s]) in only]
      try:
        val, mag = so.sensor(m, world_state(g, tag, prev, w), njmax, sensors=sens, fp32_cutoff=False)["sensordata"]
      except co.KnifeEdge:
        continue  # a decision within rounding of its threshold: the reference may have taken either side
      done = ~np.isnan(val)
      check(f"{name} {tag} w{w} sensordata", want_all[w][done], val[done], mag[done])
      seen |= {int(mjm.sensor_type[s]) for s in sens if done[int(mjm.sensor_adr[s])]}
      checked += 1
  assert checked >= want_all.shape[0], f"{name}: only {checked} world states away from every knife edge"
  return seen


def _pipeline_tags(g):
  yield "forward", None, "forward/sensordata"
  s, prev = 0, "forward"
  while f"step{s}/sensordata" in g:
    yield f"step{s}", prev, f"step{s}/sensordata"
    prev, s = f"step{s}", s + 1


SENSOR_SCENES = [n for n in SCENES if "sensordata" in "".join(np.load(os.path.join(GOLD_DIR, f"pipeline_{n}.npz")).files)]


@pytest.mark.parametrize("name", SENSOR_SCENES)
def test_oracle_matches_pipeline_sensordata(name):
  """Every pipeline fixture with sensors, at forward and at every stored step."""
  g = np.load(os.path.join(GOLD_DIR, f"pipeline_{name}.npz"))
  mjm = load_scene(name)
  seen = compare_sensors(mjm, g, name, list(_pipeline_tags(g)))
  if name == "sensors":  # the scene carries one sensor of every core type
    core = {int(t) for t in np.asarray(mjm.sensor_type)}
    assert core <= seen, f"types never compared: {sorted(core - seen)}"


def test_pipeline_sensors_cover_every_core_type_and_reference():
  """pipeline_sensors holds every sensor type k_sensor's plain build carries, objects of every type and every reference-frame type."""
  mjm = load_scene("sensors")
  core = {C.SENS_JOINTPOS, C.SENS_ACTUATORPOS, C.SENS_BALLQUAT, C.SENS_FRAMEPOS, C.SENS_FRAMEXAXIS, C.SENS_FRAMEYAXIS, C.SENS_FRAMEZAXIS,
          C.SENS_FRAMEQUAT, C.SENS_SUBTREECOM, C.SENS_CLOCK, C.SENS_JOINTLIMITPOS, C.SENS_JOINTLIMITVEL, C.SENS_JOINTLIMITFRC, C.SENS_JOINTVEL,
          C.SENS_ACTUATORVEL, C.SENS_BALLANGVEL, C.SENS_FRAMELINVEL, C.SENS_FRAMEANGVEL, C.SENS_SUBTREELINVEL, C.SENS_SUBTREEANGMOM,
          C.SENS_GYRO, C.SENS_VELOCIMETER, C.SENS_ACCELEROMETER, C.SENS_FRAMELINACC, C.SENS_FRAMEANGACC, C.SENS_TOUCH, C.SENS_FORCE,
          C.SENS_TORQUE, C.SENS_ACTUATORFRC, C.SENS_JOINTACTFRC}
  assert core <= {int(t) for t in mjm.sensor_type}
  ref = {int(t) for t, r in zip(mjm.sensor_reftype, mjm.sensor_refid) if r >= 0}
  assert {C.OBJ_BODY, C.OBJ_XBODY, C.OBJ_GEOM, C.OBJ_SITE, C.OBJ_CAMERA} <= ref
  touch_sites = {int(mjm.site_type[i]) for t, i in zip(mjm.sensor_type, mjm.sensor_objid) if t == C.SENS_TOUCH}
  assert touch_sites == {C.GEOM_SPHERE, C.GEOM_CAPSULE, C.GEOM_ELLIPSOID, C.GEOM_CYLINDER, C.GEOM_BOX}


def test_oracle_matches_batched_frames():
  """tests/golden/sensor_batched.npz (tools/make_sensor_goldens.py): per-world body_iquat, geom_quat, site_quat and cam_quat with nb = 3
  over 4 worlds; framequat, framepos and framexaxis of every object type, alone and against every reference type.  Each world is fed
  the model as it sees it (entry w % nb), and the same slots miss the reference when fed the nominal model."""
  from tests import sensor_scenes as S

  g = np.load(os.path.join(GOLD_DIR, "sensor_batched.npz"))
  mjm = S.load()
  batched = {k: g[f"in/{k}"] for k in ("body_iquat", "geom_quat", "site_quat", "cam_quat")}
  assert all(v.shape[0] == S.NB for v in batched.values()) and g["forward/sensordata"].shape[0] == S.NWORLD > S.NB
  seen = compare_sensors(mjm, g, "batched", [("forward", None, "forward/sensordata")], batched=batched)
  assert {C.SENS_FRAMEQUAT, C.SENS_FRAMEPOS, C.SENS_FRAMEXAXIS} <= seen
  refs = {(int(mjm.sensor_objtype[s]), int(mjm.sensor_reftype[s])) for s in range(mjm.nsensor) if int(mjm.sensor_type[s]) == C.SENS_FRAMEQUAT}
  kinds = {C.OBJ_BODY, C.OBJ_XBODY, C.OBJ_GEOM, C.OBJ_SITE, C.OBJ_CAMERA}
  assert {(o, r) for o in kinds for r in kinds | {C.OBJ_UNKNOWN}} <= refs
  for w in range(S.NWORLD):  # the per-world entries matter: the nominal model gives another framequat in every world
    val, _ = so.sensor(co.world_model(mjm, None, w), world_state(g, "forward", None, w), int(g["in/njmax"]), fp32_cutoff=False)["sensordata"]
    q = [int(mjm.sensor_adr[s]) for s in range(mjm.nsensor) if int(mjm.sensor_type[s]) == C.SENS_FRAMEQUAT]
    assert np.abs(val[q] - g["forward/sensordata"][w][q]).max() > 1e-2


def _extra_names():
  from tests import sensor_extra_scenes as S

  return list(S.SCENES)


@pytest.mark.parametrize("scene", _extra_names())
def test_oracle_matches_sensor_extra_fixtures(scene):
  """Every sensor_extra_* fixture at forward: magnetometer, camprojection (fovy and intrinsic paths, per-world fovy / intrinsic /
  magnetic), insidesite on every object and site type, tendon limit pos / vel / frc and tendonactfrc, each with cutoffs."""
  from tests import sensor_extra_scenes as S

  g = np.load(os.path.join(GOLD_DIR, f"sensor_extra_{scene}.npz"))
  mjm = S.load(scene)
  batched = {}
  if S.SCENES[scene][2]:
    batched = {"cam_fovy": g["in/cam_fovy"], "cam_intrinsic": g["in/cam_intrinsic"]}
  extra_types = set(so.EXTRA) | {C.SENS_JOINTPOS}
  n = g["forward/sensordata"].shape[0]
  seen = set()
  for w in range(n):
    m = co.world_model(mjm, batched, w)
    if "in/magnetic" in g:
      m = _with_magnetic(m, mjm, g["in/magnetic"][w])
    st = world_state(g, "forward", None, w)
    st["qpos"] = g["start/qpos"][w]
    # delayed sensors report their history buffer (tests/test_gpu_history.py), not this launch's value
    sens = [s for s in range(mjm.nsensor) if int(mjm.sensor_type[s]) in extra_types and int(mjm.sensor_historyadr[s]) < 0]
    val, mag = so.sensor(m, st, int(g["in/njmax"]), sensors=sens, fp32_cutoff=False)["sensordata"]
    done = ~np.isnan(val)
    check(f"{scene} w{w}", g["forward/sensordata"][w][done], val[done], mag[done])
    seen |= {int(mjm.sensor_type[s]) for s in sens}
  assert seen


def _with_magnetic(m, mjm, mag):
  class O:
    def __getattr__(self, k):
      return mag if k == "magnetic" else getattr(mjm.opt, k)

  class V:
    opt = O()

    def __getattr__(self, k):
      return getattr(m, k)

  return V()


BODY_STAGE = ("humanoid_pyramidal", "humanoid_elliptic", "g1", "equality", "tendon_actuator", "batched", "fluid")


@pytest.mark.parametrize("scene", BODY_STAGE)
def test_oracle_matches_body_stage_fixtures(scene):
  """cacc / cfrc_ext / cfrc_int / subtree_linvel / subtree_angmom of tests/golden/body_stage_*.npz (the reference's rne_postconstraint and
  subtree_vel after forward), for the worlds whose fixture holds every input the restatement reads."""
  from tests import body_stage_scenes as S

  g = np.load(os.path.join(GOLD_DIR, f"body_stage_{scene}.npz"))
  mjm = S.load(scene)
  njmax = int(g["in/njmax"])
  checked = 0
  for w in range(g["in/qpos"].shape[0]):
    st = {k.split("/")[1]: g[k][w] for k in g.files if k.startswith("fwd/") and g[k].ndim and g[k].shape[0] == g["in/qpos"].shape[0]}
    st["qvel"], st["xfrc_applied"] = g["in/qvel"][w], g["in/xfrc_applied"][w]
    m = co.world_model(mjm, {k: g[f"in/{k}"] for k in ("body_mass", "body_inertia") if f"in/{k}" in g}, w)
    lin, ang = so.subtree_vel(m, st)
    for f, x in (("subtree_linvel", lin), ("subtree_angmom", ang)):
      check(f"{scene} w{w} {f}", g[f"out/{f}"][w], np.array([[e.v for e in r] for r in x]), np.array([[e.m for e in r] for r in x]))
    nacon, ne = int(np.asarray(g["fwd/nacon"]).reshape(-1)[0]), int(np.asarray(g["fwd/ne"]).reshape(-1)[w])
    if nacon or ne:
      continue  # the fixture keeps no efc_force / contacts: cfrc_ext would need them
    st.update(ne=0, efc_force=np.zeros(1), efc_id=np.zeros(1, int), con_geom=[])
    cacc, cext, cint = so.rne_post(m, st, njmax)
    for f, x in (("cacc", cacc), ("cfrc_ext", cext), ("cfrc_int", cint)):
      check(f"{scene} w{w} {f}", g[f"out/{f}"][w], np.array([[e.v for e in r] for r in x]), np.array([[e.m for e in r] for r in x]))
    checked += 1
  if scene in ("fluid", "tendon_actuator"):
    assert checked, f"{scene}: no world without contacts or equality rows"
