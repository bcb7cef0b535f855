"""The integrator kernels (k_euler, k_euler_flat, k_implicit, k_next_act, k_rk_stage) against the fp64 restatement of
tests/integrator_oracle.py fed the kernels' own inputs: forward() runs on the GPU, its outputs are snapshot, then only the integrator runs.

Bounds come from rounding analysis, not from the observed errors (eps = 2^-24, n the tree size):
- qvel: Higham's componentwise forward error of the solve, dt |A^-1| (3 n eps (Aabs |x| + |b|)), with Aabs the matrix assembled from the
  absolute values of its terms (so the assembly's rounding is covered too), plus 2 eps (|qvel'| + dt |x|) for the update;
- qLU (implicit): the backward error of the factors, |U L - A64| <= 3 n eps |U| |L| + 8 eps Aabs (the elimination runs from the last dof,
  so A = U L with U unit upper);
- hinge / slide positions: 2 eps (|qpos'| + dt |qvel'|); quaternions: 16 eps from the fp64 integral of the kernel's fp32 inputs, up to sign;
- qacc_warmstart == qacc and time + dt exactly.
Each check prints its worst ratio to its bound.
"""
import numpy as np
import pytest
import torch

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import mjcf
from tests import integrator_oracle as O
from tests import util
from tests.test_integrator_vectors import load

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24
FIELDS = ("qpos", "qvel", "qacc", "M", "ctrl", "act", "act_dot", "actuator_moment", "actuator_force", "cdof", "cdof_dot", "cvel", "cinert", "time")
RAN = set()


def chain_xml(n, integrator="Euler", eulerdamp=True):
  """n hinge joints in one chain (one tree of n dofs), alternating axes, damped, no contacts."""
  body = ""
  for i in reversed(range(n)):
    ax = ("0 1 0", "1 0 0", "0 0 1")[i % 3]
    body = (f'<body pos="{0.1 if i else 0} 0 0"><joint type="hinge" axis="{ax}" damping="{0.05 + 0.01 * (i % 5)}" armature="0.002"/>'
            f'<geom type="capsule" fromto="0 0 0 .1 0 0" size=".01" mass="{0.1 + 0.002 * i}" contype="0" conaffinity="0"/>{body}</body>')
  flag = "" if eulerdamp else '<flag eulerdamp="disable"/>'
  return f'<mujoco><option timestep="0.002" integrator="{integrator}">{flag}</option><worldbody>{body}</worldbody></mujoco>'


JOINTS_XML = """<mujoco><option timestep="0.004" gravity="0 0 0">{flag}</option><worldbody>
  <body><freejoint/><geom type="box" size=".1 .07 .05" mass="1" contype="0" conaffinity="0"/></body>
  <body pos="1 0 0"><joint type="ball" damping="{damp}"/><geom type="capsule" fromto="0 0 0 0 0 -.3" size=".02" contype="0" conaffinity="0"/>
    <body pos="0 0 -.3"><joint type="hinge" axis="0 1 0" damping="{damp}"/><geom type="capsule" fromto="0 0 0 .2 0 0" size=".02" contype="0" conaffinity="0"/></body></body>
  <body pos="0 1 0"><joint type="slide" axis="1 0 0" damping="{damp}"/><geom type="sphere" size=".05" contype="0" conaffinity="0"/></body>
</worldbody></mujoco>"""


def _np(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _setup(mjw, mjm, nworld, seed, m=None, qvel_noise=0.8, njmax=128):
  m = m or mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, nconmax=32, njmax=njmax, m=m)
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld, seed=seed, qvel_noise=qvel_noise, exact_world0=False)
  for name, v in (("qpos", qpos), ("qvel", qvel), ("ctrl", ctrl)):
    getattr(d, name).copy_(torch.from_numpy(v.astype(np.float32)))
  if getattr(mjm, "na", 0):
    d.act.copy_(torch.from_numpy(util.seeded_act(mjm, nworld, seed=seed).astype(np.float32)))
  return m, d


def _snapshot(d):
  s = {k: _np(getattr(d, k)) for k in FIELDS}
  s["efc_Ma"] = _np(d.efc.Ma)[:, : s["qvel"].shape[1]]
  return s


def _world(s, w):
  return {k: v[w] for k, v in s.items()}


def check_step(mjm, s, out, integrator, worlds, label):
  """out: the kernel's qvel, qpos, qacc_warmstart, time (and qLU for implicit) after the integrator, s: its inputs."""
  dt = float(mjm.opt.timestep)
  worst = {"qvel": 0.0, "qpos": 0.0, "quat": 0.0, "qLU": 0.0}
  for w in worlds:
    f = _world(s, w)
    np.testing.assert_array_equal(out["qacc_warmstart"][w], f["qacc"], err_msg=f"{label} world {w}: qacc_warmstart")
    assert np.float32(out["time"][w]) == np.float32(np.float32(f["time"]) + np.float32(dt)), f"{label} world {w}: time"
    flat = integrator == C.INT_EULER and int(mjm.opt.disableflags) & (C.DSBL_EULERDAMP | C.DSBL_DAMPER)
    if flat:
      x, bq = f["qacc"], np.zeros(mjm.nv)
    else:
      A = O.matrix_a(mjm, f, integrator)
      Aabs = O.matrix_a(mjm, f, integrator, absolute=True)
      x = O.solve_trees(mjm, A, f["efc_Ma"])
      bq = np.zeros(mjm.nv)
      for st, n in zip(mjm.tree_dofadr, mjm.tree_dofnum):
        sl = slice(int(st), int(st + n))
        Ainv = np.abs(np.linalg.inv(A[sl, sl]))
        bq[sl] = dt * Ainv @ (3 * int(n) * EPS * (Aabs[sl, sl] @ np.abs(x[sl]) + np.abs(f["efc_Ma"][sl])))
      if integrator == C.INT_IMPLICIT:
        L, U = O.lu_factors(mjm, out["qLU"][w])
        bound = 3 * mjm.nv * EPS * (np.abs(U) @ np.abs(L)) + 8 * EPS * Aabs
        chain = O.ancestors(mjm) | O.ancestors(mjm).T
        r = np.where(chain, np.abs(U @ L - A) / (bound + 1e-30), 0.0)
        worst["qLU"] = max(worst["qLU"], float(r.max()))
    qvel = f["qvel"] + dt * x
    bound = bq + 2 * EPS * (np.abs(qvel) + dt * np.abs(x)) + 1e-30
    worst["qvel"] = max(worst["qvel"], float((np.abs(out["qvel"][w] - qvel) / bound).max()))
    # positions: the fp64 integral of the kernel's own fp32 velocity
    want = O.next_position(mjm, f["qpos"], out["qvel"][w], dt)
    for j in range(mjm.njnt):
      t, qa, da = int(mjm.jnt_type[j]), int(mjm.jnt_qposadr[j]), int(mjm.jnt_dofadr[j])
      if t in (C.JNT_FREE, C.JNT_BALL):
        q0 = qa + 3 if t == C.JNT_FREE else qa
        got, ref = out["qpos"][w, q0 : q0 + 4], want[q0 : q0 + 4]
        worst["quat"] = max(worst["quat"], min(np.abs(got - ref).max(), np.abs(got + ref).max()) / (16 * EPS))
        lin = range(qa, qa + 3) if t == C.JNT_FREE else ()
      else:
        lin = (qa,)
      for k in lin:
        v = out["qvel"][w, da + (k - qa)]
        worst["qpos"] = max(worst["qpos"], abs(out["qpos"][w, k] - want[k]) / (2 * EPS * (abs(want[k]) + dt * abs(v)) + 1e-30))
  print(f"{label}: worst ratio to bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
  for k, v in worst.items():
    assert v <= 1.0, f"{label}: {k} error is {v:.3g} x its bound"


def run_case(mjw, mjm, nworld, seed, label, m=None, prepare=None, njmax=128):
  m, d = _setup(mjw, mjm, nworld, seed, m=m, njmax=njmax)
  if prepare:
    prepare(d)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  s = _snapshot(d)
  integ = int(mjm.opt.integrator)
  if integ in (C.INT_IMPLICIT, C.INT_IMPLICITFAST):
    mjw.implicit(m, d)
  else:
    mjw.euler(m, d)
  torch.cuda.synchronize()
  out = {k: _np(getattr(d, k)) for k in ("qvel", "qpos", "qacc_warmstart", "time", "qLU")}
  check_step(mjm, s, out, integ, range(nworld), label)
  return m, d, s, out


def _path(mjm):
  integ = int(mjm.opt.integrator)
  if integ == C.INT_IMPLICIT:
    return "k_implicit/%d" % ((mjm.nv + 31) // 32)
  if integ == C.INT_EULER and int(mjm.opt.disableflags) & (C.DSBL_EULERDAMP | C.DSBL_DAMPER):
    return "k_euler_flat"
  return "k_euler/%s/%s" % ("warp" if int(max(mjm.tree_dofnum)) > 32 else "reg", "implicitfast" if integ == C.INT_IMPLICITFAST else "euler")


@pytest.mark.parametrize("n", [1, 40, 64])
@pytest.mark.parametrize("integrator", ["Euler", "implicitfast", "implicit"])
def test_chain(built, n, integrator):
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(chain_xml(n, integrator))
  run_case(mjw, mjm, 3, n, f"chain{n} {integrator}")
  RAN.add(_path(mjm))


@pytest.mark.parametrize("integrator", ["Euler", "implicitfast"])
def test_humanoid_27_dofs(built, integrator):
  import mujoco_warp_b200 as mjw

  mjm = mjw.mjcf.load_any(util.HUMANOID)
  mjm.opt.disableflags = int(mjm.opt.disableflags) & ~C.DSBL_EULERDAMP
  mjm.opt.integrator = C.INT_EULER if integrator == "Euler" else C.INT_IMPLICITFAST
  run_case(mjw, mjm, 5, 2, f"humanoid {integrator}")
  RAN.add(_path(mjm))


def test_three_humanoids_implicit_three_column_passes(built):
  import mujoco_warp_b200 as mjw

  mjm = mjw.mjcf.load_any(util.THREE_HUMANOIDS)
  mjm.opt.integrator = C.INT_IMPLICIT
  assert mjm.nv > 64
  run_case(mjw, mjm, 3, 4, "three_humanoids implicit")
  RAN.add(_path(mjm))


@pytest.mark.parametrize("scene,integrator", [("crosstree", "implicitfast"), ("crosstree", "implicit"), ("crosstree", "Euler"), ("actuators", "implicitfast"),
                                              ("actuators", "implicit"), ("actuators", "Euler"), ("tendons", "implicitfast"), ("tendons", "implicit")])
def test_scenes(built, scene, integrator):
  """Tendon damping, the cross-tree tendon actuator, stateful actuators (filterexact with actlimited, integrator dynamics, actearly)."""
  import mujoco_warp_b200 as mjw

  mjm = load(scene, integrator)
  _, d, s, _ = run_case(mjw, mjm, 3, 9, f"{scene} {integrator}")
  if getattr(mjm, "na", 0):  # k_next_act: the activations of the step
    act = _np(d.act)
    for w in range(3):
      want = O.advance(mjm, _world(s, w), np.zeros(mjm.nv))[2]
      np.testing.assert_allclose(act[w], want, rtol=4 * EPS, atol=4 * EPS, err_msg=f"{scene} {integrator} world {w}: act")
    RAN.add("k_next_act")


@pytest.mark.parametrize("flag", ["DSBL_DAMPER", "DSBL_ACTUATION"])
def test_disable_flags(built, flag):
  import mujoco_warp_b200 as mjw

  mjm = load("actuators", "implicitfast")
  mjm.opt.disableflags = int(mjm.opt.disableflags) | getattr(C, flag)
  run_case(mjw, mjm, 3, 10, f"actuators implicitfast {flag}")


@pytest.mark.parametrize("eulerdamp", [True, False])
def test_joint_types_and_quaternion_edges(built, eulerdamp):
  """free, ball, hinge and slide joints; per world: omega = 0, |omega| dt ~ 1e-8, |omega| dt > pi, and a stored quaternion that is not unit
  length.  eulerdamp=False runs k_euler_flat, True k_euler."""
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(JOINTS_XML.format(flag="" if eulerdamp else '<flag eulerdamp="disable"/>', damp=0.3))

  def prepare(d):
    qvel, qpos = _np(d.qvel), _np(d.qpos)
    dt = float(mjm.opt.timestep)
    qvel[0, 3:9] = 0.0
    qvel[1, 3:9] = np.array([1.0, -2.0, 2.0, 0.6, 0.0, -0.8]) * (1e-8 / 3 / dt)
    qvel[2, 3:9] = np.array([1.0, 2.0, -2.0, -0.6, 0.8, 0.0]) * (4.0 / 3 / dt)
    qpos[3, 3:7] *= 1.7
    qpos[3, 7:11] *= 0.6
    d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
    d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))

  run_case(mjw, mjm, 4, 12, f"joints eulerdamp={eulerdamp}", prepare=prepare)
  RAN.add(_path(mjm))


def _batched(mjw, mjm, fields, nworld, seed, nstep):
  """World w of a batched model against a single-world model holding w's values; fields: name -> leading size."""
  m = mjw.put_model(mjm, batch_sizes=fields)
  rng = np.random.default_rng(seed)
  scale = {}
  for f, n in fields.items():
    t = getattr(m, f)
    sc = rng.uniform(0.6, 1.5, size=(n,) + (1,) * (t.dim() - 1)).astype(np.float32)
    scale[f] = sc
    t.mul_(torch.from_numpy(sc).cuda())
  m, d = _setup(mjw, mjm, nworld, seed, m=m)
  init = {k: getattr(d, k).clone() for k in ("qpos", "qvel", "ctrl", "act")}
  for _ in range(nstep):
    mjw.step(m, d)
  torch.cuda.synchronize()
  got = {k: _np(getattr(d, k)) for k in ("qpos", "qvel", "act")}
  for w in range(nworld):
    m1 = mjw.put_model(mjm)
    for f, n in fields.items():
      getattr(m1, f).mul_(torch.from_numpy(scale[f][w % n : w % n + 1]).cuda())
    d1 = mjw.make_data(mjm, nworld=1, nconmax=32, njmax=128, m=m1)
    for k, v in init.items():
      getattr(d1, k).copy_(v[w : w + 1])
    for _ in range(nstep):
      mjw.step(m1, d1)
    torch.cuda.synchronize()
    for k, v in got.items():
      np.testing.assert_allclose(v[w], _np(getattr(d1, k))[0], rtol=2e-5, atol=2e-6, err_msg=f"world {w}: {k}")
  return got


@pytest.mark.parametrize("integrator", ["Euler", "RK4"])
def test_batched_activation_parameters(built, integrator):
  """actuator_dynprm (the filterexact / filter time constants) and actuator_actrange (the final clamp) per world."""
  import mujoco_warp_b200 as mjw

  mjm = load("actuators", integrator)
  got = _batched(mjw, mjm, {"actuator_dynprm": 3, "actuator_actrange": 3}, 3, 21, 4)
  assert np.abs(got["act"] - got["act"][0]).max() > 1e-5
  if integrator == "RK4":
    RAN.add("k_rk_stage/batched")


@pytest.mark.parametrize("integrator", ["implicitfast", "implicit"])
def test_batched_derivative_parameters(built, integrator):
  import mujoco_warp_b200 as mjw

  mjm = load("tendons", integrator)
  _batched(mjw, mjm, {"dof_damping": 3, "tendon_damping": 3, "actuator_gainprm": 3, "actuator_biasprm": 3}, 3, 22, 3)
  mjm = load("crosstree", integrator)
  _batched(mjw, mjm, {"dof_damping": 3, "tendon_damping": 3, "actuator_gainprm": 3, "actuator_biasprm": 3}, 3, 23, 3)


def test_rk4_matches_a_composition_of_forward_calls(built):
  """rungekutta4 against RK4 composed in fp64 from GPU forward() calls at the fp64-composed stage states.  The stage states differ from the
  kernel's by rounding, and how much forward() amplifies that is measured: the band is 4x the spread of the same composition with the
  states of stages 1-3 perturbed by +-1 ulp (stage 0 is the initial state, which the kernel evaluates exactly).  On top of it, the rounding of the kernel's own fp32 bookkeeping: 4 eps (|x_t0| + g sum_s B_s |rate_s|),
  with rate qvel for qpos, qacc for qvel and act_dot for act, and g = dt -- for a filterexact activation g = tau (1 - e^-x), x = dt / tau,
  times the condition number 1 + e^-x / (1 - e^-x) of that difference, which expf's rounding enters."""
  import mujoco_warp_b200 as mjw

  mjm = load("actuators", "RK4")
  mjm.opt.disableflags = int(mjm.opt.disableflags) | C.DSBL_CONSTRAINT
  nworld = 3
  dt = float(mjm.opt.timestep)
  m, d = _setup(mjw, mjm, nworld, 31)
  init = {k: _np(getattr(d, k)) for k in ("qpos", "qvel", "ctrl", "act")}
  mjw.forward(m, d)
  mjw.rungekutta4(m, d)
  torch.cuda.synchronize()
  got = {k: _np(getattr(d, k)) for k in ("qpos", "qvel", "act")}
  de = mjw.make_data(mjm, nworld=1, nconmax=32, njmax=128, m=m)

  def composed(w, ulp, rates=None):
    stage = [0]

    def fwd(q, v, a):
      for k, x in (("qpos", q), ("qvel", v), ("act", a)):
        x32 = x.astype(np.float32)
        if ulp and stage[0] > 0:
          x32 = np.nextafter(x32, np.float32(np.inf) if ulp > 0 else np.float32(-np.inf))
        getattr(de, k).copy_(torch.from_numpy(x32[None]))
      de.ctrl.copy_(torch.from_numpy(init["ctrl"][w : w + 1].astype(np.float32)))
      mjw.forward(m, de)
      out = {"qacc": _np(de.qacc)[0], "act_dot": _np(de.act_dot)[0]}
      stage[0] += 1
      if rates is not None:
        rates.append((np.abs(v), np.abs(out["qacc"]), np.abs(out["act_dot"])))
      return out
    return O.rk4(mjm, {"qpos": init["qpos"][w], "qvel": init["qvel"][w], "act": init["act"][w]}, fwd)

  worst = {"qpos": 0.0, "qvel": 0.0, "act": 0.0}
  B = (1 / 6, 1 / 3, 1 / 3, 1 / 6)
  for w in range(nworld):
    rates = []
    base = composed(w, 0, rates)
    spread = [np.maximum(np.abs(composed(w, 1)[i] - base[i]), np.abs(composed(w, -1)[i] - base[i])) for i in range(3)]
    qpos_rate = np.zeros(mjm.nq)
    for j in range(mjm.njnt):  # the hinge / slide positions of this scene advance by dt qvel
      qpos_rate[mjm.jnt_qposadr[j]] = sum(b * r[0][mjm.jnt_dofadr[j]] for b, r in zip(B, rates))
    g = np.full(mjm.na, dt)
    for a in range(mjm.nu):
      if mjm.actuator_actadr[a] >= 0 and mjm.actuator_dyntype[a] == C.DYN_FILTEREXACT:
        tau = float(mjm.actuator_dynprm[a, 0])
        e = np.exp(-dt / tau)
        g[mjm.actuator_actadr[a]] = tau * (1 - e) * (1 + e / (1 - e))
    own = (4 * EPS * (np.abs(init["qpos"][w]) + dt * qpos_rate), 4 * EPS * (np.abs(init["qvel"][w]) + dt * sum(b * r[1] for b, r in zip(B, rates))),
           4 * EPS * (np.abs(init["act"][w]) + g * sum(b * r[2] for b, r in zip(B, rates))))
    for i, k in enumerate(("qpos", "qvel", "act")):
      band = 4 * spread[i] + own[i] + 1e-30
      r = np.abs(got[k][w] - base[i]) / band
      if r.max() > worst[k]:
        worst[k] = float(r.max())
        print(f"rk4 world {w} {k}[{int(r.argmax())}]: kernel {got[k][w][r.argmax()]:.9g} composed {base[i][r.argmax()]:.9g} spread {spread[i][r.argmax()]:.3g} own {own[i][r.argmax()]:.3g}")
  print("rk4 composition: worst ratio to the band " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
  for k, v in worst.items():
    assert v <= 1.0, f"rk4 {k}: {v:.3g} x its band"


@pytest.mark.parametrize("nworld", [1, 7, 1031])
def test_world_counts_match_worlds_run_alone(built, nworld):
  """k_euler_flat, bit for bit.  step() at 1031 worlds runs two world halves (the second with w0 != 0); its result must equal forward() at
  the same world count followed by euler() over all worlds at once (w0 = 0), and every world must equal the same world advanced from the
  same forward() outputs in a batch of five."""
  import mujoco_warp_b200 as mjw

  mjm = mjcf.load_string(JOINTS_XML.format(flag='<flag eulerdamp="disable"/>', damp=0.3))
  m, d = _setup(mjw, mjm, nworld, 41)
  init = {k: getattr(d, k).clone() for k in ("qpos", "qvel")}
  _, ds = _setup(mjw, mjm, nworld, 41, m=m)
  mjw.step(m, ds)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  fwd = {k: getattr(d, k).clone() for k in ("qpos", "qvel", "qacc", "time")}
  mjw.euler(m, d)
  torch.cuda.synchronize()
  keys = ("qpos", "qvel", "time", "qacc_warmstart")
  got = {k: getattr(d, k).cpu().numpy() for k in keys}
  for k in keys:
    np.testing.assert_array_equal(getattr(ds, k).cpu().numpy(), got[k], err_msg=f"step() at {nworld} worlds vs forward() + euler(): {k}")
  assert torch.equal(init["qpos"], fwd["qpos"]) and torch.equal(init["qvel"], fwd["qvel"])
  for w0 in sorted({0, nworld // 2, max(0, nworld - 5)}):
    ws = list(range(w0, min(nworld, w0 + 5)))
    d1 = mjw.make_data(mjm, nworld=len(ws), nconmax=32, njmax=128, m=m)
    for k, v in fwd.items():
      getattr(d1, k).copy_(v[ws])
    mjw.euler(m, d1)
    torch.cuda.synchronize()
    for k in keys:
      np.testing.assert_array_equal(got[k][ws], getattr(d1, k).cpu().numpy(), err_msg=f"worlds {ws}: {k}")
  RAN.add("k_euler_flat")


def trees_xml(trees, integrator):
  """One hinge chain per entry of trees; entry k of a chain's list is the number of hinge joints of its k-th body."""
  def chain(njs, first):
    body = ""
    for i in reversed(range(len(njs))):
      joints = "".join(f'<joint type="hinge" axis="{("0 1 0", "1 0 0", "0 0 1")[(i + k) % 3]}" damping="0.05"/>' for k in range(njs[i]))
      body = (f'<body pos="{0.1 if i else 0} {first if i == 0 else 0} 0">{joints}'
              f'<geom type="capsule" fromto="0 0 0 .1 0 0" size=".01" mass="{0.1 + 0.002 * i}" contype="0" conaffinity="0"/>{body}</body>')
    return body
  bodies = "".join(chain(njs, 0.5 * t) for t, njs in enumerate(trees))
  return f'<mujoco><option timestep="0.002" integrator="{integrator}"/><worldbody>{bodies}</worldbody></mujoco>'


def test_implicit_shared_memory_limit(built):
  """k_implicit keeps qLU's tree blocks, the right-hand side and 18 nbody x 32 floats of scratch in one block's shared memory.
  - 87 bodies (nbody 88, two chains of 43 and 44 hinges) is the most put_model accepts, and it fits and runs correctly (three column passes);
  - one body more is refused by put_model's scratch check;
  - at nbody 88, trees of 64 and 58 dofs (bodies with two hinges) pass put_model but not the launch's check of the whole layout, which
    refuses the model by name before launching anything."""
  import mujoco_warp_b200 as mjw

  r4 = lambda k: -(-k // 4) * 4
  words = lambda sizes, nbody: r4(sum(n * n for n in sizes)) + r4(sum(sizes)) + 18 * nbody * 32
  assert words((43, 44), 88) * 4 <= 227 * 1024 and 18 * 88 * 32 * 4 <= 200 * 1024 < 18 * 89 * 32 * 4
  mjm = mjcf.load_string(trees_xml([[1] * 43, [1] * 44], "implicit"))
  assert mjm.nbody == 88 and mjm.nv == 87
  run_case(mjw, mjm, 2, 88, "nbody 88 implicit (largest)", njmax=8)
  RAN.add(_path(mjm))
  with pytest.raises(NotImplementedError, match="velocity-derivative scratch of 89 bodies"):
    mjw.put_model(mjcf.load_string(trees_xml([[1] * 44, [1] * 44], "implicit")))
  mjm = mjcf.load_string(trees_xml([[2] * 21 + [1] * 22, [2] * 14 + [1] * 30], "implicit"))
  assert mjm.nbody == 88 and list(mjm.tree_dofnum) == [64, 58] and words((64, 58), 88) * 4 > 227 * 1024
  m, d = _setup(mjw, mjm, 2, 89, njmax=8)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  qvel = d.qvel.clone()
  with pytest.raises(RuntimeError, match="velocity-derivative scratch"):
    mjw.implicit(m, d)
  assert mjw.last_launch_count() == 0
  torch.cuda.synchronize()
  assert torch.equal(d.qvel, qvel)


def test_crosstree_discrete_inverse(built):
  """k_inverse's discrete-time conversion (ENBL_INVDISCRETE, implicitfast) on the cross-tree scene: given the discrete acceleration the
  restatement's implicitfast step takes, qacc_cont = M^-1 A qacc, so qfrc_inverse must give back the applied and actuator forces.  The
  scene has no constraint rows, so the only error is fp32 rounding; the tendon actuator's entries of tree 1, which a per-first-dof tree
  assignment drops, move qfrc_inverse by far more than the tolerance (checked below)."""
  import mujoco_warp_b200 as mjw

  mjm = load("crosstree", "implicitfast")
  mjm.opt.enableflags = int(mjm.opt.enableflags) | C.ENBL_INVDISCRETE
  nworld = 3
  m, d = _setup(mjw, mjm, nworld, 51)
  rng = np.random.default_rng(52)
  d.qfrc_applied.copy_(torch.from_numpy(rng.uniform(-0.5, 0.5, (nworld, mjm.nv)).astype(np.float32)))
  mjw.forward(m, d)
  torch.cuda.synchronize()
  s = _snapshot(d)
  assert int(_np(d.nefc).max()) == 0
  qacc_disc = np.stack([O.solve_trees(mjm, O.matrix_a(mjm, _world(s, w), C.INT_IMPLICITFAST), s["efc_Ma"][w]) for w in range(nworld)])
  d.qacc.copy_(torch.from_numpy(qacc_disc.astype(np.float32)))
  mjw.inverse(m, d)
  torch.cuda.synchronize()
  want = _np(d.qfrc_smooth) - _np(d.qfrc_passive) + _np(d.qfrc_bias)
  got = _np(d.qfrc_inverse)
  dt = float(mjm.opt.timestep)
  worst = 0.0
  for w in range(nworld):
    f = _world(s, w)
    x = qacc_disc[w].astype(np.float32).astype(np.float64)
    Aabs = O.matrix_a(mjm, f, C.INT_IMPLICITFAST, absolute=True)
    M = O.dense_m(mjm, f["M"])
    # A x in fp32 (assembly and product), M^-1 of it by Cholesky and M times that again, each a few n eps of its absolute terms
    tol = 16 * mjm.nv * EPS * (Aabs @ np.abs(x) + np.abs(M) @ (np.abs(np.linalg.inv(M)) @ (Aabs @ np.abs(x))) + np.abs(want[w])) + 1e-30
    worst = max(worst, float((np.abs(got[w] - want[w]) / tol).max()))
    # negative control: the actuator's entries on tree 1's dofs (jb, jb2) change qfrc_inverse by dt dA x
    dA = np.zeros((mjm.nv, mjm.nv))
    for i, j, v in O.qderiv_terms(mjm, f, {"tendon_damping": np.zeros(mjm.ntendon)}):
      if i >= int(mjm.tree_dofadr[1]):
        dA[i, j] += dt * v
        if i != j:
          dA[j, i] += dt * v
    assert np.abs(dA @ x).max() > 10 * tol.max(), (np.abs(dA @ x).max(), tol.max())
  print(f"crosstree discrete inverse: worst ratio to bound {worst:.3f}")
  assert worst <= 1.0, worst


def test_every_path_ran():
  """Every integrator path above ran in this session (run the file as a whole)."""
  want = {"k_euler/reg/euler", "k_euler/warp/euler", "k_euler/reg/implicitfast", "k_euler/warp/implicitfast", "k_euler_flat", "k_implicit/3",
          "k_rk_stage/batched", "k_next_act"}
  if not RAN:
    pytest.skip("no integrator test ran in this session")
  assert want <= RAN, sorted(want - RAN)
