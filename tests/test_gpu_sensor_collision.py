"""Distance / normal / fromto sensors on the GPU (k_sensor_collision).

- Analytic cases: two spheres (dist = |c1 - c2| - r1 - r2, witness points on the surfaces) and a sphere over a plane.
- Swapping geom1 and geom2 negates the normal and swaps the halves of fromto; a body sensor is the minimum over its geoms; the cutoff.
- DSBL_SENSOR leaves the slots alone; the sensors change nothing of the physics; per-world geom_size gives per-world distances.
- One extra launch for a model with collision sensors and none otherwise; CUDA-graph capture; 8192 worlds, finite and deterministic.
"""
import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf
from tests import sensor_collision_scenes as scenes
from tests import util
from tests.test_gpu_launch_count import _captured_kernels

pytestmark = pytest.mark.gpu


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _setup(xml, nworld, seed=3, batch_sizes=None, noise=0.3):
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(xml)
  m = mjw.put_model(mjm, batch_sizes=batch_sizes) if batch_sizes else mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m, nconmax=16, njmax=64)
  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=None, seed=seed, qpos_noise=noise, qvel_noise=0.5, exact_world0=False)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  return mjw, mjm, m, d


def _slots(mjm, d):
  s = _np(d.sensordata)
  return [s[:, a : a + n] for a, n in zip(mjm.sensor_adr, mjm.sensor_dim)]


def test_spheres_and_plane_analytic(built):
  r1, r2 = 0.1, 0.15
  mjw, mjm, m, d = _setup(scenes.spheres_xml(r1, r2), 64)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  x = _np(d.geom_xpos)
  ca, cb = x[:, 1], x[:, 2]
  dist, normal, fromto, dist_ba, normal_ba, fromto_ba, dfloor, ftfloor, nfloor = _slots(mjm, d)
  want = np.linalg.norm(cb - ca, axis=1) - r1 - r2
  np.testing.assert_allclose(dist[:, 0], want, atol=2e-6)
  u = (cb - ca) / np.linalg.norm(cb - ca, axis=1, keepdims=True)
  assert (want < 0).any() and (want > 0).any()
  # normal = normalize(to - from): from a to b when the spheres are apart, reversed when they overlap (the witness points cross);
  # |to - from| = |dist|, so fp32 cancellation leaves it ~1e-7 / |dist| accurate: compared where the spheres are 2 cm from touching
  far = np.abs(want) > 0.02
  assert far.sum() > 32
  np.testing.assert_allclose(normal[far], (u * np.sign(want)[:, None])[far], atol=1e-5)
  np.testing.assert_allclose(fromto[:, :3], ca + r1 * u, atol=2e-6)  # on sphere a's surface, towards b
  np.testing.assert_allclose(fromto[:, 3:], cb - r2 * u, atol=2e-6)  # on sphere b's surface, towards a
  # swapping geom1 and geom2: the same distance, the normal negated, the fromto halves swapped
  np.testing.assert_array_equal(dist_ba, dist)
  np.testing.assert_allclose(normal_ba, -normal, atol=1e-6)
  np.testing.assert_allclose(fromto_ba, np.concatenate([fromto[:, 3:], fromto[:, :3]], axis=1), atol=1e-6)
  # the floor is the plane z = 0: sphere a's height minus its radius, from the floor straight up
  np.testing.assert_allclose(dfloor[:, 0], ca[:, 2] - r1, atol=2e-6)
  np.testing.assert_allclose(ftfloor[:, :2], ca[:, :2], atol=2e-6)
  np.testing.assert_allclose(ftfloor[:, 2], 0.0, atol=2e-6)
  np.testing.assert_allclose(ftfloor[:, 3:], ca - [0, 0, r1], atol=2e-6)
  np.testing.assert_allclose(nfloor, np.tile([0.0, 0.0, -1.0], (64, 1)), atol=1e-6)  # geom1 = a: from the sphere to the floor


def test_overlapping_spheres_have_negative_distance(built):
  mjw, mjm, m, d = _setup(scenes.spheres_xml(0.3, 0.3), 8, noise=0.0)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  x = _np(d.geom_xpos)
  want = np.linalg.norm(x[:, 2] - x[:, 1], axis=1) - 0.6
  assert (want < 0).all()
  np.testing.assert_allclose(_slots(mjm, d)[0][:, 0], want, atol=2e-6)


def test_body_sensor_is_the_minimum_over_its_geoms(built):
  xml = scenes.pair_xml("sphere", "sphere", "box", "capsule")
  extra = '<distance geom1="obj0" geom2="objobj0" cutoff="10"/><distance geom1="obj0" geom2="objobj1" cutoff="10"/><distance geom1="obj0" body2="objobj" cutoff="10"/>'
  xml = xml.replace("<sensor>", "<sensor>" + extra)
  mjw, mjm, m, d = _setup(xml, 32, noise=0.2)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  a, b, body = _slots(mjm, d)[:3]
  np.testing.assert_array_equal(body[:, 0], np.minimum(a[:, 0], b[:, 0]))


def test_cutoff_clamps_and_zeroes(built):
  mjw, mjm, m, d = _setup(scenes.spheres_xml(cutoff=0.01), 16, noise=0.0)  # the spheres are 0.08 apart, the floor 0.4 below
  mjw.forward(m, d)
  torch.cuda.synchronize()
  dist, normal, fromto = _slots(mjm, d)[:3]
  np.testing.assert_array_equal(dist, np.float32(0.01))
  np.testing.assert_array_equal(normal, 0.0)
  np.testing.assert_array_equal(fromto, 0.0)


def test_disabled_sensors_leave_the_slots_alone(built):
  mjw, mjm, m, d = _setup(scenes.spheres_xml(), 8)
  m.opt.disableflags = int(C.DSBL_SENSOR)
  d.sensordata.fill_(7.0)
  mjw.forward(m, d)
  mjw.step(m, d)
  torch.cuda.synchronize()
  assert (d.sensordata == 7.0).all()


def _run_physics(xml, nworld, steps):
  mjw, mjm, m, d = _setup(xml, nworld, noise=0.05)
  for _ in range(steps):
    mjw.step(m, d)
  torch.cuda.synchronize()
  n = int(d.nacon.item())
  out = {f: _np(getattr(d, f)) for f in ("qpos", "qvel", "qacc", "nefc")}
  out["efc_force"] = _np(d.efc.force)
  out["contact_dist"], out["contact_pos"], out["contact_geom"] = _np(d.contact.dist)[:n], _np(d.contact.pos)[:n], _np(d.contact.geom)[:n]
  out["nacon"] = n
  return out, mjw.last_launch_count()


def test_sensors_change_nothing_of_the_physics_and_add_one_launch(built, monkeypatch):
  monkeypatch.setenv("MJB_SPLIT", "1")  # one stream, so that the contact pool order is the same in both runs
  with_s, n_with = _run_physics(scenes.spheres_xml(contact=True), 64, 50)
  without, n_without = _run_physics(scenes.spheres_xml(contact=True, sensors=False), 64, 50)
  assert with_s["nacon"] > 0
  for k in with_s:
    assert np.array_equal(with_s[k], without[k]), k
  # the model without sensors has no k_sensor either: one k_sensor and one k_sensor_collision launch more
  assert n_with == n_without + 2
  framepos = scenes.spheres_xml(contact=True, sensors=False).replace("</mujoco>", '<sensor><framepos objtype="body" objname="a"/></sensor></mujoco>')
  assert _run_physics(framepos, 64, 1)[1] == n_without + 1


def test_per_world_geom_size(built):
  nworld = 16
  mjw, mjm, m, d = _setup(scenes.spheres_xml(), nworld, batch_sizes={"geom_size": nworld}, noise=0.0)
  r = 0.05 + 0.005 * np.arange(nworld)
  sizes = np.repeat(np.asarray(mjm.geom_size)[None], nworld, axis=0)
  sizes[:, 1, 0] = r
  m.geom_size.copy_(torch.as_tensor(sizes, dtype=torch.float32))
  mjw.forward(m, d)
  torch.cuda.synchronize()
  x = _np(d.geom_xpos)
  np.testing.assert_allclose(_slots(mjm, d)[0][:, 0], np.linalg.norm(x[:, 2] - x[:, 1], axis=1) - r - 0.15, atol=2e-6)


@pytest.mark.parametrize("types", [("sphere", "capsule", "box", "ellipsoid"), ("box", "cylinder", "mesh", "box")], ids=["primitive_convex", "mesh"])
def test_8192_worlds_finite_deterministic_and_captured(built, types):
  xml = scenes.pair_xml(*types)
  if "mesh" in types:
    xml = xml.replace("<worldbody>", '<asset><mesh name="m" vertex="0 0 0  .1 0 0  0 .1 0  0 0 .1  .05 .05 .05"/></asset><worldbody>').replace(
      'type="mesh" size=".09 .09 .09"', 'type="mesh" mesh="m"')
  runs = []
  for _ in range(2):
    mjw, mjm, m, d = _setup(xml, 8192, noise=0.4)
    mjw.forward(m, d)
    mjw.step(m, d)
    torch.cuda.synchronize()
    runs.append(_np(d.sensordata))
  assert np.isfinite(runs[0]).all()
  assert np.array_equal(runs[0], runs[1])
  kernels = _captured_kernels(lambda: mjw.step(m, d))
  assert mjw.last_launch_count() == kernels
  mjw2, _, m2, d2 = _setup(xml, 8192, noise=0.4)
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    mjw.step(m, d)
  for name in ("qpos", "qvel", "qacc_warmstart", "time"):
    getattr(d, name).copy_(getattr(d2, name))
  d.sensordata.zero_()
  g.replay()
  mjw2.step(m2, d2)
  torch.cuda.synchronize()
  assert np.array_equal(_np(d.sensordata), _np(d2.sensordata))


def test_fromto_is_not_clamped_by_the_cutoff(built):
  # cutoff 0.2: the spheres are 0.08 apart, so the sensors see them; the witness points lie at heights 0.5-0.6, above the cutoff
  r1, r2 = 0.1, 0.15
  mjw, mjm, m, d = _setup(scenes.spheres_xml(r1, r2, cutoff=0.2), 8, noise=0.0)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  x = _np(d.geom_xpos)
  ca, cb = x[:, 1], x[:, 2]
  u = (cb - ca) / np.linalg.norm(cb - ca, axis=1, keepdims=True)
  dist, normal, fromto = _slots(mjm, d)[:3]
  assert (dist[:, 0] < 0.2).all() and (np.abs(fromto) > 0.2).any()
  np.testing.assert_allclose(fromto[:, :3], ca + r1 * u, atol=2e-6)
  np.testing.assert_allclose(fromto[:, 3:], cb - r2 * u, atol=2e-6)


@pytest.mark.parametrize("scene", sorted(scenes.SCENES))
def test_gpu_matches_reference_fixture(built, scene):
  """Every fixture through the public API, teacher-forced: the positions the reference's forward and steps started from, then the collision
  sensors at the host-replay bands and the contacts against the fixture's CONSTRAINT-typed ones (its SENSOR-only contacts do not exist here)."""
  import os

  import mujoco_warp_b200 as mjw

  from tests.test_sensor_collision_vectors import GOLD, TAGS, _size_scale, compare

  g = np.load(os.path.join(GOLD, f"sensor_collision_{scene}.npz"))
  mjm = mjcf.load_string(scenes.SCENES[scene])
  nworld = g["in/qpos"].shape[0]
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m, nconmax=64, njmax=256)
  for tag in TAGS:
    d.qpos.copy_(torch.from_numpy(np.asarray(g["in/qpos" if tag == "forward" else f"{tag}/qpos_before"], dtype=np.float32)))
    d.qvel.copy_(torch.from_numpy(np.asarray(g["in/qvel"], dtype=np.float32)))
    mjw.forward(m, d)
    torch.cuda.synchronize()
    # the geom poses are this build's fp32 kinematics, not the fixture's: a GJK witness point that slides along a face moves further (2e-2)
    compare(mjm, _np(d.sensordata), g[f"{tag}/sensordata"], g[f"knife/{tag}"], _size_scale(mjm), f"{scene}/{tag}", ccd_witness=2e-2)
    # contacts: the fixture's constraint contacts (type bit 1), per world and geom pair, against ours
    keep = (g[f"{tag}/con_type"] & 1) != 0
    want = sorted(zip(g[f"{tag}/con_worldid"][keep].tolist(), map(tuple, g[f"{tag}/con_geom"][keep].tolist()), g[f"{tag}/con_geomcollisionid"][keep].tolist(),
                      g[f"{tag}/con_dist"][keep].tolist()))
    n = int(d.nacon.item())
    got = sorted(zip(_np(d.contact.worldid)[:n].astype(int).tolist(), map(tuple, _np(d.contact.geom)[:n].astype(int).tolist()),
                     _np(d.contact.geomcollisionid)[:n].astype(int).tolist(), _np(d.contact.dist)[:n].tolist()))
    assert [w[:3] for w in want] == [x[:3] for x in got], f"{scene}/{tag}"
    np.testing.assert_allclose([x[3] for x in got], [w[3] for w in want], atol=1e-4 * _size_scale(mjm))
