"""Mesh hulls past the fixed multi-contact buffers on the GPU (k_collision_mesh_large, k_sensor_collision_large): the scenes of
tests/mesh_hull_scenes.py against the reference's fixtures (tests/golden/mesh_hull_*.npz, tools/make_mesh_hull_goldens.py) with the
tolerances tests/test_gpu_golden_pipeline.py uses for its `mesh` scene, the mixed scene's in-cap pairs against the in-cap build, and the
dispatch: models within 32 / 16 keep k_collision_mesh."""
import os

import numpy as np
import pytest
import torch

from tests import mesh_hull_scenes as S
from tests import util

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PTOL = 5e-3  # flat-on-flat contacts: EPA in fp32 and in double stop at different points of the same patch (test_gpu_golden_pipeline.py)


def close(name, got, want, atol, rtol=0.0):
  got = np.asarray(got, dtype=np.float64)
  util.assert_close(name, got, np.asarray(want, dtype=np.float64).reshape(got.shape), atol=atol, rtol=rtol)


def setup(name, nworld=S.NWORLD, xml=None):
  import mujoco_warp_b200 as mjw

  mjm = S.load(xml or name)
  cfg = S.SCENES[name]["cfg"]
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, nconmax=cfg["nconmax"], njmax=cfg["njmax"], m=m)
  return mjw, mjm, m, d


def load_state(d, qpos, qvel, warm):
  f32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
  d.qpos.copy_(f32(qpos)); d.qvel.copy_(f32(qvel)); d.qacc_warmstart.copy_(f32(warm))


def world_pairs(d, w):
  """World w's contacts grouped by geom pair: {(g1, g2): [(dist, pos, normal), ...]}."""
  c, out = d.contact, {}
  for i in util.world_contacts(d, w):
    key = tuple(int(x) for x in c.geom[i].cpu().numpy())
    out.setdefault(key, []).append((float(c.dist[i]), c.pos[i].cpu().numpy().astype(np.float64), c.frame[i].cpu().numpy().reshape(-1)[:3].astype(np.float64)))
  return out


def match(name, got, want, dtol, ptol):
  """Two contact lists of one geom pair agree as sets: every wanted contact has its own got contact within ptol, at depth dtol."""
  assert len(got) == len(want), (name, len(got), len(want))
  used = set()
  for wd, wp, wn in want:
    j = min((k for k in range(len(got)) if k not in used), key=lambda k: float(np.abs(got[k][1] - wp).sum()))
    used.add(j)
    gd, gp, gn = got[j]
    assert abs(gd - wd) <= dtol and np.abs(gp - wp).max() <= ptol and np.abs(gn - wn).max() <= ptol, (name, (gd, gp, gn), (wd, wp, wn))


@pytest.mark.parametrize("name", list(S.SCENES))
def test_scene_runs_the_large_build_and_matches_the_reference(built, name):
  mjw, mjm, m, d = setup(name)
  assert mjw.collision_kernel(m) == "k_collision_mesh_large"
  g = np.load(os.path.join(GOLD, f"mesh_hull_{name}.npz"))
  load_state(d, g["in/qpos"], g["in/qvel"], g["in/qacc_warmstart"])
  mjw.forward(m, d)
  torch.cuda.synchronize()
  assert (d.overflow.cpu().numpy() == 0).all()
  # contacts: the reference's pool also holds its sensor pairs' contacts (ContactType.SENSOR, at or past zero distance here)
  cg, cd, cp, cf, cw = (g[f"forward/con_{f}"] for f in ("geom", "dist", "pos", "frame", "worldid"))
  real = cd < 0.0
  assert int(d.nacon.cpu()[0]) == int(real.sum())
  for w in range(S.NWORLD):
    got = world_pairs(d, w)
    want = {}
    for i in np.nonzero(real & (cw == w))[0]:
      want.setdefault(tuple(int(x) for x in cg[i]), []).append((float(cd[i]), cp[i], cf[i].reshape(-1)[:3]))
    assert sorted(got) == sorted(want), (w, sorted(got), sorted(want))
    for key in want:
      match(f"w{w} {key}", got[key], want[key], 5e-4, PTOL)
  if g["forward/sensordata"].size:
    close("sensordata", d.sensordata.cpu().numpy(), g["forward/sensordata"], atol=5e-4, rtol=5e-4)
  np.testing.assert_array_equal(d.nefc.cpu().numpy().reshape(-1), g["forward/nefc"].reshape(-1))
  # collision() alone writes the same contacts, bit for bit
  before = [world_pairs(d, w) for w in range(S.NWORLD)]
  mjw.collision(m, d)
  torch.cuda.synchronize()
  for w in range(S.NWORLD):
    after = world_pairs(d, w)
    assert sorted(after) == sorted(before[w])
    for key in after:
      match(f"rerun w{w} {key}", after[key], before[w][key], 0.0, 0.0)
  # teacher-forced steps (test_gpu_golden_pipeline.py): step s starts from the reference's state after step s - 1
  dt = float(np.asarray(mjm.opt.timestep))
  s = 0
  while f"step{s}/qpos" in g:
    if s > 0:
      load_state(d, g[f"step{s - 1}/qpos"], g[f"step{s - 1}/qvel"], g[f"step{s - 1}/qacc_warmstart"])
      d.time.copy_(torch.from_numpy(np.asarray(g[f"step{s - 1}/time"], dtype=np.float32).reshape(-1)))
    mjw.step(m, d)
    torch.cuda.synchronize()
    same = d.nefc.cpu().numpy().reshape(-1) == g[f"step{s}/nefc"].reshape(-1)
    assert same.sum() >= S.NWORLD - 2, (s, d.nefc.cpu().numpy(), g[f"step{s}/nefc"])
    ascale = max(1.0, float(np.abs(g[f"step{s}/qacc"]).max()))
    vtol = dt * 1e-2 * ascale + 1e-4
    close(f"step{s}/qvel", d.qvel.cpu().numpy()[same], g[f"step{s}/qvel"][same], atol=vtol, rtol=1e-3)
    close(f"step{s}/qpos", d.qpos.cpu().numpy()[same], g[f"step{s}/qpos"][same], atol=dt * vtol + 2e-5, rtol=1e-5)
    if g[f"step{s}/sensordata"].size:
      close(f"step{s}/sensordata", d.sensordata.cpu().numpy()[same], g[f"step{s}/sensordata"][same], atol=5e-4, rtol=5e-4)
    s += 1
  assert s >= 3 and ((d.overflow.cpu().numpy() & ~(1 << 10)) == 0).all()


def test_mixed_in_cap_pairs_agree_with_the_in_cap_build(built):
  """The mixed scene without its 64-gon prism runs k_collision_mesh; the pairs it shares with the full scene (run by
  k_collision_mesh_large) give the same contacts, world by world."""
  mjw, mjm, m, d = setup("mixed")
  _, mjm0, m0, d0 = setup("mixed", xml=S.MIXED_INCAP)
  assert mjw.collision_kernel(m) == "k_collision_mesh_large" and mjw.collision_kernel(m0) == "k_collision_mesh"
  qpos, qvel, ctrl, warm = S.seeded(mjm, "mixed")
  assert mjm0.nq == mjm.nq - 7 and mjm0.ngeom == mjm.ngeom - 1  # the large prism is the last body and geom
  load_state(d, qpos, qvel, warm)
  load_state(d0, qpos[:, :-7], qvel[:, :-6], warm[:, :-6])
  mjw.kinematics(m, d); mjw.kinematics(m0, d0)
  mjw.collision(m, d); mjw.collision(m0, d0)
  torch.cuda.synchronize()
  big = mjm.ngeom - 1
  nshared = 0
  for w in range(S.NWORLD):
    full = {k: v for k, v in world_pairs(d, w).items() if big not in k}
    incap = world_pairs(d0, w)
    assert sorted(full) == sorted(incap), w
    for key in incap:
      match(f"w{w} {key}", full[key], incap[key], 1e-6, 1e-6)
      nshared += len(incap[key])
  assert nshared >= 4 * S.NWORLD


def test_large_sensor_kernel_and_launch_names(built):
  """torch.profiler sees k_collision_mesh_large and k_sensor_collision_large in a step of the sensors scene; bench.py's convex_mesh
  workload (hulls within 32 / 16) still launches the in-cap kernels and none of the large ones."""
  from torch.profiler import ProfilerActivity, profile

  from mujoco_warp_b200._src import mjcf
  from mujoco_warp_b200.scenes import WORKLOADS

  mjw, mjm, m, d = setup("sensors")
  g = np.load(os.path.join(GOLD, "mesh_hull_sensors.npz"))
  load_state(d, g["in/qpos"], g["in/qvel"], g["in/qacc_warmstart"])
  mjw.step(m, d)
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    mjw.step(m, d)
    torch.cuda.synchronize()
  names = " ".join(e.key for e in prof.key_averages())
  assert "k_collision_mesh_large" in names and "k_sensor_collision_large" in names, names

  wl = WORKLOADS["convex_mesh"]
  cm = mjcf.load_any(wl["model"])
  assert int(cm.npolygonmax) <= 32 and int(cm.nmeshdegmax) <= 16
  mc = mjw.put_model(cm)
  dc = mjw.make_data(cm, nworld=64, nconmax=wl["nconmax"], njmax=wl["njmax"], m=mc)
  assert mjw.collision_kernel(mc) == "k_collision_mesh"
  prof_ms = mjw.step_profile(mc, dc)
  assert prof_ms["collision"] > 0.0
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    mjw.step(mc, dc)
    torch.cuda.synchronize()
  names = " ".join(e.key for e in prof.key_averages())
  assert "k_collision<" in names and "_large" not in names, names
