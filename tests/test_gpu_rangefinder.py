"""The rangefinder sensor on the GPU (k_sensor_rangefinder).

- Every scene of tests/rangefinder_scenes.py against the reference's own sensordata (tests/golden/rangefinder_*.npz): forward from the
  seeded state and every step from the reference's state (Euler, implicitfast, implicit, RK4, per-world geom_size / geom_rgba, meshes,
  delayed sensors, 210 rangefinders), at test_gpu_ray's fp32 tolerances; only knife-edge rays are excused.
- On every step, the fp64 ray oracle (tests/host_harness/ray_oracle.c) fed the GPU's own site and geom poses meets sensordata.
- On these scenes sensordata is bit-identical to rays(m, d, site_xpos, site z axis, None, True, site body) with the cutoff applied, after
  forward, step1, sensor_pos, inverse and a world-split forward (1025 worlds, two world ranges); and bit-identical run to run and under
  graph replay.  (Both kernels run the same scan, compiled separately: elsewhere a distance may differ from rays() in the last bits.)
- read_sensor of a delayed rangefinder meets the delay fixture's sensordata.
- DSBL_SENSOR: the slots keep their sentinel and the kernel is not launched.  Launch counts: one more per position-stage sensor call
  with rangefinders, none more without them.
"""
import os

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io, mjcf
from tests import rangefinder_scenes as S
from tests import test_rangefinder_host as H

pytestmark = pytest.mark.gpu

STATE = ("time", "qpos", "qvel", "qacc_warmstart", "ctrl", "history")


def _t(a):
  return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).cuda()


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def setup(scene, nworld=S.NWORLD, rows=True):
  import mujoco_warp_b200 as mjw

  g = H.golden(scene)
  mjm = S.load(scene) if rows else mjcf.load_string(S.xml(S.INTEGRATORS.get(scene, "Euler"), mesh=scene == "mesh"))
  per_world = S.SCENES[scene][2]
  m = mjw.put_model(mjm, batch_sizes={"geom_size": S.NWORLD, "geom_rgba": S.NWORLD} if per_world else None)
  if per_world:
    m.geom_size.copy_(_t(g["in/geom_size"]))
    m.geom_rgba.copy_(_t(g["in/geom_rgba"]))
  d = mjw.make_data(mjm, nworld=nworld, nconmax=int(g["in/nconmax"]), njmax=int(g["in/njmax"]), m=m)
  return mjw, g, mjm, m, d


def _load_state(d, g, prefix):
  for f in STATE:
    a = np.asarray(g[prefix + f])
    reps = d.nworld // a.shape[0] + 1 if a.ndim and a.shape[0] == S.NWORLD else 1
    a = np.concatenate([a] * reps)[: d.nworld] if reps > 1 else a
    getattr(d, f).copy_(_t(a).reshape(getattr(d, f).shape))


def _tables(mjm):
  t = io.rangefinder_tables(mjm)
  adr = t["sensor_rangefinder_adr"]
  return t, adr, np.asarray(mjm.sensor_adr)[adr], np.asarray(mjm.sensor_history).reshape(-1, 2)[adr, 0]


def _rays_slots(mjw, mjm, m, d):
  """rays() from every rangefinder site along its z axis on the same Data, with the cutoff applied in fp32"""
  t, adr, _, _ = _tables(mjm)
  site = torch.from_numpy(np.asarray(mjm.sensor_objid)[adr].astype(np.int64)).cuda()
  nw, nrf = d.nworld, len(adr)
  pnt = d.site_xpos.reshape(nw, -1, 3)[:, site].contiguous()
  vec = d.site_xmat.reshape(nw, -1, 9)[:, site][..., [2, 5, 8]].contiguous()
  dist = torch.empty((nw, nrf), dtype=torch.float32, device="cuda")
  gid = torch.empty((nw, nrf), dtype=torch.int32, device="cuda")
  nrm = torch.empty((nw, nrf, 3), dtype=torch.float32, device="cuda")
  mjw.rays(m, d, pnt, vec, None, True, _t(t["sensor_rangefinder_bodyid"]).int(), dist, gid, nrm)
  c, dt = np.asarray(mjm.sensor_cutoff, dtype=np.float32)[adr], np.asarray(mjm.sensor_datatype)[adr]
  for r in range(nrf):
    if c[r] > 0 and dt[r] == 0:
      dist[:, r] = dist[:, r].clamp(-float(c[r]), float(c[r]))
    elif c[r] > 0 and dt[r] == 1:
      dist[:, r] = torch.minimum(dist[:, r], torch.tensor(float(c[r]), device="cuda"))
  return dist.cpu().numpy()


def _slots(mjm, d):
  _, _, slot, _ = _tables(mjm)
  return d.sensordata.cpu().numpy()[:, slot]


def _compare(got, want, knife, what, datol=1e-5):
  ok = ~knife
  err = np.abs(got - want)[ok]
  assert (err <= datol + 1e-5 * np.abs(want[ok])).all(), f"{what}: max error {err.max()} at {np.argwhere(~(np.abs(got - want) <= datol + 1e-5 * np.abs(want)) & ok)[:5].tolist()}"
  assert ((got == -1) == (want == -1))[ok].all(), f"{what}: hit / miss differs"


def _oracle(mjm, g, d, per_world):
  """the fp64 oracle fed the GPU's own site and geom poses, with the cutoff applied"""
  nw = d.nworld
  return H.rangefinder_values(H.RV.oracle_lib(np.float64).ray_oracle_rays, np.float64, mjm, g, _np(d.site_xpos), _np(d.site_xmat).reshape(nw, -1, 9),
                              _np(d.geom_xpos), _np(d.geom_xmat).reshape(nw, -1, 9), per_world)


@pytest.mark.parametrize("scene", list(S.SCENES))
def test_scene_meets_reference(scene):
  mjw, g, mjm, m, d = setup(scene)
  _, nsteps, per_world = S.SCENES[scene]
  _, adr, slot, hist = _tables(mjm)
  delayed = (hist > 0)[None]
  anyknife = g["forward/knife"].copy()
  for k in range(nsteps):
    anyknife |= g[f"step/{k}/knife"]
  _load_state(d, g, "start/")
  d.ctrl.copy_(_t(g["in/ctrl"][0]))
  mjw.forward(m, d)
  torch.cuda.synchronize()
  got = _slots(mjm, d)
  _compare(got, g["forward/sensordata"][:, slot], g["forward/knife"] | (delayed & anyknife), f"{scene} forward")
  np.testing.assert_array_equal(got[:, ~delayed[0]], _rays_slots(mjw, mjm, m, d)[:, ~delayed[0]])
  for k in range(nsteps):
    _load_state(d, g, f"step/{k}/in_")
    mjw.step(m, d)
    torch.cuda.synchronize()
    got = _slots(mjm, d)
    _compare(got, g[f"step/{k}/out_sensordata"][:, slot], g[f"step/{k}/knife"] | (delayed & anyknife), f"{scene} step {k}")
    # fed its own inputs: the poses this step's sensors read are still in Data (the integrator does not touch them)
    exp = _oracle(mjm, g, d, per_world)
    _compare(got[:, ~delayed[0]], exp[:, ~delayed[0]], g[f"step/{k}/knife"][:, ~delayed[0]], f"{scene} step {k} vs fp64 oracle on its own poses")
    np.testing.assert_array_equal(got[:, ~delayed[0]], _rays_slots(mjw, mjm, m, d)[:, ~delayed[0]])


@pytest.mark.parametrize("scene", ["primitives", "mesh", "batched"])
def test_stage_calls_match_rays_bitwise(scene):
  mjw, g, mjm, m, d = setup(scene)
  _, _, slot, _ = _tables(mjm)
  _load_state(d, g, "start/")
  mjw.forward(m, d)
  ref = _rays_slots(mjw, mjm, m, d)
  np.testing.assert_array_equal(_slots(mjm, d), ref)
  for call in (lambda: mjw.sensor_pos(m, d), lambda: mjw.inverse(m, d), lambda: mjw.step1(m, d)):
    d.sensordata[:, slot] = float("nan")
    call()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(_slots(mjm, d), ref)
  # run to run
  d.sensordata.fill_(float("nan"))
  mjw.forward(m, d)
  np.testing.assert_array_equal(_slots(mjm, d), ref)


def test_discrete_inverse_writes_the_same_slots():
  mjw, g, mjm, m, d = setup("implicitfast")
  _, _, slot, _ = _tables(mjm)
  _load_state(d, g, "start/")
  mjw.forward(m, d)
  ref = _slots(mjm, d)
  m.opt.enableflags = int(m.opt.enableflags) | C.ENBL_INVDISCRETE
  d.sensordata[:, slot] = float("nan")
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  np.testing.assert_array_equal(_slots(mjm, d), ref)


def test_world_split_matches_single_range():
  """1025 worlds: forward runs two world ranges (513 + 512) on their own streams; every world matches rays() and the 3-world run"""
  mjw, g, mjm, m, d = setup("many", nworld=1025)
  _load_state(d, g, "start/")
  mjw.forward(m, d)
  torch.cuda.synchronize()
  got = _slots(mjm, d)
  np.testing.assert_array_equal(got, _rays_slots(mjw, mjm, m, d))
  _, _, _, m3, d3 = setup("many")
  _load_state(d3, g, "start/")
  mjw.forward(m3, d3)
  small = _slots(mjm, d3)
  for w in (0, 1, 2, 513, 514, 515, 1023, 1024):
    np.testing.assert_array_equal(got[w], small[w % S.NWORLD])


def test_read_sensor_meets_delay_golden():
  mjw, g, mjm, m, d = setup("delay")
  _, adr, slot, hist = _tables(mjm)
  nsteps = S.SCENES["delay"][1]
  for k in range(nsteps):
    _load_state(d, g, f"step/{k}/in_")
    mjw.step(m, d)
  torch.cuda.synchronize()
  knife = np.zeros_like(g["forward/knife"])
  for k in range(nsteps):
    knife |= g[f"step/{k}/knife"]
  res = torch.zeros((d.nworld, 1), dtype=torch.float32, device="cuda")
  t_sensed = _t(g[f"step/{nsteps - 1}/in_time"])  # the time the last step's sensors ran at (the step then advanced d.time)
  for r in np.nonzero(hist > 0)[0]:
    mjw.read_sensor(m, d, int(adr[r]), t_sensed, 0, res)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(res.cpu().numpy()[:, 0], _slots(mjm, d)[:, r])
    _compare(res.cpu().numpy()[:, 0], g[f"step/{nsteps - 1}/out_sensordata"][:, slot[r]], knife[:, r], f"read_sensor {adr[r]}")


def test_dsbl_sensor_leaves_slots_and_skips_the_kernel():
  mjw, g, mjm, m, d = setup("primitives")
  _, _, slot, _ = _tables(mjm)
  _load_state(d, g, "start/")
  mjw.sensor_pos(m, d)
  on = mjw.last_launch_count()
  m.opt.disableflags = int(m.opt.disableflags) | C.DSBL_SENSOR
  d.sensordata.fill_(-7.0)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  assert (_slots(mjm, d) == -7.0).all()
  mjw.sensor_pos(m, d)
  torch.cuda.synchronize()
  assert (_slots(mjm, d) == -7.0).all()
  m.opt.disableflags = int(m.opt.disableflags) & ~C.DSBL_SENSOR
  mjw.sensor_pos(m, d)
  assert mjw.last_launch_count() == on


# position-stage sensor calls per step: RK4 evaluates the sensors at each of its four stages
SENSOR_CALLS_PER_STEP = {"primitives": 1, "rk4": 4, "implicit": 1}


@pytest.mark.parametrize("scene", list(SENSOR_CALLS_PER_STEP))
def test_launch_count(scene):
  """one more launch per position-stage sensor call with rangefinders; the model without them launches what it did before"""
  counts = {}
  for rows in (True, False):
    mjw, g, mjm, m, d = setup(scene, rows=rows)
    _load_state(d, g, "start/")
    c = {}
    for name, call in (("forward", mjw.forward), ("step", mjw.step), ("sensor_pos", mjw.sensor_pos), ("sensor_vel", mjw.sensor_vel),
                       ("sensor_acc", mjw.sensor_acc), ("inverse", mjw.inverse)):
      call(m, d)
      c[name] = mjw.last_launch_count()
    m.opt.disableflags = int(m.opt.disableflags) | C.DSBL_SENSOR
    mjw.sensor_pos(m, d)
    c["sensor_pos_disabled"] = mjw.last_launch_count()
    counts[rows] = c
  torch.cuda.synchronize()
  for name in ("forward", "step", "sensor_pos", "inverse"):
    assert counts[True][name] == counts[False][name] + (SENSOR_CALLS_PER_STEP[scene] if name == "step" else 1), (name, counts)
  for name in ("sensor_vel", "sensor_acc", "sensor_pos_disabled"):
    assert counts[True][name] == counts[False][name], (name, counts)


def test_graph_replay_is_bitwise():
  mjw, g, mjm, m, d = setup("mesh")
  _load_state(d, g, "step/0/in_")
  stream = torch.cuda.Stream()
  with torch.cuda.stream(stream):
    mjw.step(m, d)
    stream.synchronize()
    _load_state(d, g, "step/0/in_")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
      mjw.step(m, d)
    outs = []
    for _ in range(2):
      _load_state(d, g, "step/0/in_")
      stream.synchronize()
      graph.replay()
      stream.synchronize()
      outs.append(d.sensordata.cpu().numpy().copy())
  _load_state(d, g, "step/0/in_")
  mjw.step(m, d)
  torch.cuda.synchronize()
  np.testing.assert_array_equal(outs[0], outs[1])
  np.testing.assert_array_equal(outs[0], d.sensordata.cpu().numpy())
