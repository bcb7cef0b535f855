"""Actuator and sensor delay fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_history_goldens.py [scene ...]   # writes tests/golden/history_<scene>.npz

For every scene of tests/history_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data (NWORLD
worlds), seeded per-world qpos / qvel, then
- `init/*`: init_ctrl_history of actuator 0 with per-world values at the stamps -(n-1) dt .. 0, and (VECTORS) init_sensor_history of
  the interval sensor `held` with -MJ_MAXVAL stamps and a per-world phase;
- `forward/*` and `inverse/*`: d.history, d.sensordata and d.actuator_force after forward.forward / inverse.inverse from that state
  (the history is put back after each, so the steps start from `init`);
- `step/<k>/in_*` and `step/<k>/out_*` for each step k: the state before (time, qpos, qvel, act, qacc_warmstart, ctrl, history) and
  after one forward.step (the same plus sensordata and actuator_force), so that a test can replay every step from the reference's state;
- `fn/*` after the last step: history.read_ctrl / read_sensor of every actuator / sensor at off-grid times with interp -1 / 0 / 1 / 2,
  then init_ctrl_history / init_sensor_history of actuator 0 / sensor 0 at off-grid stamps (`fn/init_*`).
One process per scene, as in make_pipeline_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import io as mio  # noqa: E402
from tests import history_scenes as H  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402

BIG = ("humanoid",)  # scenes with contacts: the contact and row capacities of the pipeline goldens
STATE = ("time", "qpos", "qvel", "act", "qacc_warmstart", "ctrl", "history")


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  hist = warp_shim.load_reference_module("history")
  inverse = warp_shim.load_reference_module("inverse")
  mjm = H.load(name)
  nsteps = H.SCENES[name][1]
  nworld = H.NWORLD
  nconmax, njmax = (32, 128) if name in BIG else (4, 16)
  t0 = time.time()
  ad = ref_runner.MjModelAdapter(mjm, defaults={"nJmom": mio.derive_tables(mjm)["nJmom"]})
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=nworld, nconmax=nconmax, njmax=njmax)
  qpos, qvel, ctrl = H.seeded(mjm, nsteps)
  d.qpos.a[...] = qpos
  d.qvel.a[...] = qvel
  d.ctrl.a[...] = ctrl[0]
  out = {"in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax), "in/ctrl": ctrl}
  arr = lambda x: wp.array(np.asarray(x, dtype=np.float64), dtype=float)

  n0 = int(mjm.actuator_history[0, 0])
  times = -H.DT * np.arange(n0 - 1, -1, -1)
  vals = np.random.default_rng(11).uniform(-1, 1, (nworld, n0))
  hist.init_ctrl_history(m, d, 0, arr(times), wp.array(vals, dtype=float))
  out["init/ctrl_times"], out["init/ctrl_values"] = times, vals
  names = list(mjm.names.sensor) if int(getattr(mjm, "nsensor", 0)) else []
  if "held" in names:
    sid = names.index("held")
    n, dim = int(mjm.sensor_history[sid, 0]), int(mjm.sensor_dim[sid])
    svals = np.random.default_rng(12).uniform(-1, 1, (nworld, n * dim))
    phase = H.interval_phase(nworld)
    hist.init_sensor_history(m, d, sid, None, wp.array(svals, dtype=float), arr(phase))
    out["init/sensor_id"], out["init/sensor_values"], out["init/sensor_phase"] = np.array(sid), svals, phase
  out["init/history"] = d.history.numpy().copy()

  h0 = d.history.numpy().copy()
  for tag, call in (("forward", lambda: fwd.forward(m, d)), ("inverse", lambda: inverse.inverse(m, d))):
    call()
    for f in ("history", "sensordata", "actuator_force"):
      out[f"{tag}/{f}"] = getattr(d, f).numpy().copy()
    d.history.a[...] = h0

  for k in range(nsteps):
    d.ctrl.a[...] = ctrl[k]
    for f in STATE:
      out[f"step/{k}/in_{f}"] = getattr(d, f).numpy().copy()
    fwd.step(m, d)
    for f in STATE + ("sensordata", "actuator_force"):
      out[f"step/{k}/out_{f}"] = getattr(d, f).numpy().copy()

  if name in ("actuators", "vectors"):
    # off-grid query times, different per world, inside and outside each buffer's span
    tq = d.time.numpy()[0] - H.DT * np.array([0.3, 1.7, 2.9])[:nworld]
    out["fn/time"] = tq
    for u in range(int(mjm.nu)):
      for interp in (-1, 0, 1, 2):
        res = wp.zeros(nworld, dtype=float)
        hist.read_ctrl(m, d, u, arr(tq), interp, res)
        out[f"fn/read_ctrl/{u}/{interp}"] = res.numpy().copy()
    for s in range(len(names)):
      for interp in (-1, 0, 1, 2):
        res = wp.zeros((nworld, int(mjm.sensor_dim[s])), dtype=float)
        hist.read_sensor(m, d, s, arr(tq), interp, res)
        out[f"fn/read_sensor/{s}/{interp}"] = res.numpy().copy()
    stamps = H.DT * (np.arange(n0) * 1.37 - 0.41)
    cvals = np.random.default_rng(13).uniform(-2, 2, (nworld, n0))
    hist.init_ctrl_history(m, d, 0, arr(stamps), wp.array(cvals, dtype=float))
    out["fn/init_ctrl_times"], out["fn/init_ctrl_values"] = stamps, cvals
    if names:
      n, dim = int(mjm.sensor_history[0, 0]), int(mjm.sensor_dim[0])
      sstamps = H.DT * (np.arange(n) * 0.83 + 0.2)
      svals = np.random.default_rng(14).uniform(-2, 2, (nworld, n * dim))
      phase = np.array([0.25, -0.5, 1.0])[:nworld] * H.DT
      hist.init_sensor_history(m, d, 0, arr(sstamps), wp.array(svals, dtype=float), arr(phase))
      out["fn/init_sensor_times"], out["fn/init_sensor_values"], out["fn/init_sensor_phase"] = sstamps, svals, phase
    out["fn/init_history"] = d.history.numpy().copy()

  path = os.path.join(ROOT, "tests", "golden", f"history_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: nhistory {m.nhistory}, {nsteps} steps, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(H.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
