"""Fluid forces on the GPU (k_velocity_fluid, and the fluid derivatives of implicitfast in k_euler_fluid / k_inverse_fluid).

- The reference's own pipeline (tests/golden/fluid_*.npz, tools/make_fluid_goldens.py), teacher-forced like test_gpu_golden_pipeline:
  qfrc_fluid, qfrc_passive and qacc_smooth at the smooth-field band, qacc at the solver band, the stepped state at dt times that.
- Invariants: a body moving at v in still fluid feels what the body at rest feels in a wind of -v; a sphere falling in a viscous
  fluid settles at the inertia-box model's terminal speed; forward then inverse gives back the applied forces (continuous time and
  the implicitfast ENBL_INVDISCRETE round trip).
- 4096 worlds: bit-identical from run to run, under graph capture and with the world split; no extra launch.
"""
import os

import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf
from tests import fluid_scenes, util
from tests.test_gpu_golden_pipeline import close
from tests.test_gpu_launch_count import _captured_kernels

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("scene", sorted(fluid_scenes.SCENES))
def test_gpu_matches_reference_fluid(built, scene):
  import mujoco_warp_b200 as mjw

  g = np.load(os.path.join(GOLD, f"fluid_{scene}.npz"))
  mjm = mjcf.load_string(fluid_scenes.SCENES[scene][0])
  m = mjw.put_model(mjm)
  nworld = g["in/qpos"].shape[0]
  d = mjw.make_data(mjm, nworld=nworld, nconmax=int(g["in/nconmax"]), njmax=int(g["in/njmax"]), m=m)
  f32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
  d.qpos.copy_(f32(g["in/qpos"])); d.qvel.copy_(f32(g["in/qvel"])); d.qacc_warmstart.copy_(f32(g["in/qacc_warmstart"]))
  if mjm.nu:
    d.ctrl.copy_(f32(g["in/ctrl"]))
  mjw.forward(m, d)
  torch.cuda.synchronize()
  for f in ("qfrc_fluid", "qfrc_passive", "qacc_smooth", "cvel", "qfrc_bias"):
    want = g[f"forward/{f}"].reshape(nworld, -1)
    close(f"forward/{f}", _np(getattr(d, f)).reshape(nworld, -1), want, atol=5e-4 * max(1.0, float(np.abs(want).max())))
  if scene == "wind_only":  # wind alone moves nothing: the forces scale with density and viscosity
    assert not d.qfrc_fluid.any()
  scale = max(1.0, float(np.abs(g["forward/qacc"]).max()))
  close("forward/qacc", _np(d.qacc), g["forward/qacc"], atol=5e-3 * scale)
  dt = float(np.asarray(mjm.opt.timestep))
  for s in range(4):
    if s > 0:
      d.qpos.copy_(f32(g[f"step{s - 1}/qpos"])); d.qvel.copy_(f32(g[f"step{s - 1}/qvel"]))
      d.qacc_warmstart.copy_(f32(g[f"step{s - 1}/qacc_warmstart"]))
      d.time.copy_(f32(np.asarray(g[f"step{s - 1}/time"]).reshape(-1)))
    mjw.step(m, d)
    torch.cuda.synchronize()
    ascale = max(1.0, float(np.abs(g[f"step{s}/qacc"]).max()))
    vtol = dt * 5e-3 * ascale + 1e-4
    close(f"step{s}/qvel", _np(d.qvel), g[f"step{s}/qvel"], atol=vtol, rtol=1e-3)
    close(f"step{s}/qpos", _np(d.qpos), g[f"step{s}/qpos"], atol=dt * vtol + 2e-5, rtol=1e-5)


def _state(mjw, mjm, nworld, seed=7):
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m, nconmax=4, njmax=16)
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld, key=None, seed=seed, qvel_noise=1.0, exact_world0=False)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  if mjm.nu:
    d.ctrl.copy_(torch.from_numpy(ctrl.astype(np.float32)))
  rng = np.random.default_rng(seed)
  d.qfrc_applied.copy_(torch.from_numpy(rng.uniform(-0.2, 0.2, (nworld, mjm.nv)).astype(np.float32)))
  return m, d


@pytest.mark.parametrize("scene", ["chain", "ellipsoid"])
def test_moving_body_feels_the_wind_of_minus_its_velocity(built, scene):
  import mujoco_warp_b200 as mjw

  v = np.array([0.7, -0.4, 0.25])
  still = mjcf.load_string(fluid_scenes.SCENES[scene][0])
  still.opt.wind = np.zeros(3)
  windy = mjcf.load_string(fluid_scenes.SCENES[scene][0])
  windy.opt.wind = -v
  free = [int(a) for t, a in zip(still.jnt_type, still.jnt_dofadr) if t == C.JNT_FREE]
  out = []
  for mjm, vel in ((still, v), (windy, np.zeros(3))):
    m, d = _state(mjw, mjm, 8)
    d.qvel.zero_()
    for a in free:  # the free joints' linear velocity: every body translates at vel
      d.qvel[:, a : a + 3] = torch.from_numpy(vel.astype(np.float32))
    mjw.forward(m, d)
    torch.cuda.synchronize()
    out.append(_np(d.qfrc_fluid))
  assert np.abs(out[0]).max() > 1e-4
  np.testing.assert_allclose(out[0], out[1], rtol=1e-4, atol=1e-5 * np.abs(out[0]).max())


def test_falling_sphere_settles_at_terminal_speed(built):
  import mujoco_warp_b200 as mjw

  r, rho, mu, g = 0.05, 2000.0, 2.0, 9.81
  mjm = mjcf.load_string(fluid_scenes.sphere_xml(radius=r, density_geom=rho, viscosity=mu))
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=4, m=m, nconmax=4, njmax=16)
  for _ in range(5000):  # 10 s, about 14 time constants
    mjw.step(m, d)
  torch.cuda.synchronize()
  # passive.py inertia box of a solid sphere: every side sqrt(2.4) r, viscous drag 3 pi diam mu v (no density: no quadratic term)
  mass = rho * 4.0 / 3.0 * np.pi * r**3
  diam = np.sqrt(2.4) * r
  v_terminal = mass * g / (3.0 * np.pi * diam * mu)
  np.testing.assert_allclose(_np(d.qvel)[:, 2], -v_terminal, rtol=1e-3)
  np.testing.assert_allclose(_np(d.qvel)[:, [0, 1, 3, 4, 5]], 0.0, atol=1e-6)


@pytest.mark.parametrize("scene", ["chain", "ellipsoid", "chain_rk4"])
def test_inverse_of_forward_gives_back_the_applied_forces(built, scene):
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(fluid_scenes.SCENES[scene][0])
  m, d = _state(mjw, mjm, 64)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  want = _np(d.qfrc_smooth) - _np(d.qfrc_passive) + _np(d.qfrc_bias)
  fluid = _np(d.qfrc_fluid)
  assert np.abs(fluid).max() > 1e-3
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  np.testing.assert_allclose(_np(d.qfrc_fluid), fluid, rtol=0, atol=0)  # inverse recomputes the same passive forces
  scale = max(1.0, float(np.abs(want).max()))
  np.testing.assert_allclose(_np(d.qfrc_inverse), want, rtol=0, atol=1e-4 * scale)


@pytest.mark.parametrize("xml", [fluid_scenes.chain_xml("implicitfast"), fluid_scenes.ellipsoid_xml("implicitfast")], ids=["chain", "ellipsoid"])
def test_discrete_inverse_of_an_implicitfast_step_gives_back_the_applied_forces(built, xml):
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(xml)
  mjm.opt.enableflags = int(mjm.opt.enableflags) | C.ENBL_INVDISCRETE
  m, d = _state(mjw, mjm, 64)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  qpos0, qvel0 = d.qpos.clone(), d.qvel.clone()
  want = _np(d.qfrc_smooth) - _np(d.qfrc_passive) + _np(d.qfrc_bias)  # no contacts: qfrc_constraint is zero
  mjw.step(m, d)
  torch.cuda.synchronize()
  h = float(np.asarray(mjm.opt.timestep))
  qacc_disc = (d.qvel - qvel0) / h
  d.qpos.copy_(qpos0); d.qvel.copy_(qvel0); d.qacc.copy_(qacc_disc)
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  scale = max(1.0, float(np.abs(want).max()))
  np.testing.assert_allclose(_np(d.qfrc_inverse), want, rtol=0, atol=2e-3 * scale)
  assert np.array_equal(_np(d.qacc), _np(qacc_disc))


def _run(mjw, mjm, nworld, steps=3):
  m, d = _state(mjw, mjm, nworld)
  for _ in range(steps):
    mjw.step(m, d)
  torch.cuda.synchronize()
  return m, d, {f: _np(getattr(d, f)) for f in ("qpos", "qvel", "qfrc_fluid", "qfrc_passive", "qacc")}


@pytest.mark.parametrize("scene", ["chain", "ellipsoid_implicitfast"])
def test_fluid_at_4096_worlds_is_deterministic_split_and_captured(built, monkeypatch, scene):
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(fluid_scenes.SCENES[scene][0])
  runs = []
  for split in ("1", "2", "2"):
    monkeypatch.setenv("MJB_SPLIT", split)
    runs.append(_run(mjw, mjm, 4096)[2])
  for f in runs[0]:
    assert np.array_equal(runs[0][f], runs[1][f]), f
    assert np.array_equal(runs[1][f], runs[2][f]), f
  m, d, _ = _run(mjw, mjm, 4096, steps=0)
  kernels = _captured_kernels(lambda: mjw.step(m, d))
  assert mjw.last_launch_count() == kernels
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    mjw.step(m, d)
  m2, d2, _ = _run(mjw, mjm, 4096, steps=0)
  for name in ("qpos", "qvel", "qacc_warmstart", "ctrl", "qfrc_applied", "time"):
    getattr(d, name).copy_(getattr(d2, name))
  g.replay()
  mjw.step(m2, d2)
  torch.cuda.synchronize()
  for f in ("qpos", "qvel", "qfrc_fluid"):
    assert np.array_equal(_np(getattr(d, f)), _np(getattr(d2, f))), f
  # the same launches as the model without fluid forces
  plain = mjcf.load_string(fluid_scenes.SCENES[scene][0])
  plain.opt.density, plain.opt.viscosity, plain.opt.wind = 0.0, 0.0, np.zeros(3)
  mp, dp = _state(mjw, plain, 4096)
  mjw.step(mp, dp)
  assert mjw.last_launch_count() == kernels
  assert not dp.qfrc_fluid.any()
