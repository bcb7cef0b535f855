"""Muscle actuator fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_muscle_goldens.py [scene ...]   # writes tests/golden/muscle_<scene>.npz

For every scene of tests/muscle_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data (NWORLD
worlds), seeded per-world qpos / qvel / act, then
- `forward/*` and `inverse/*`: act_dot, actuator_force, qfrc_actuator and sensordata after forward.forward / inverse.inverse from the
  seeded state with the first step's ctrl;
- `step/<k>/in_*` and `step/<k>/out_*` for each step k: the state before (time, qpos, qvel, act, qacc_warmstart, ctrl) and after one
  forward.step (the same plus act_dot, actuator_force, qfrc_actuator and sensordata), so that a test can replay every step;
- `lengthrange/*`: set_const.set_length_range into a per-world output, from the model's sources (`single`) and from per-world jnt_range,
  tendon_range and actuator_gear (each world's ranges scaled and gears flipped differently; `batched`), next to those inputs.
One process per scene, as in make_history_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import io as mio  # noqa: E402
from tests import muscle_scenes as S  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402

BIG = ("humanoid",)
STATE = ("time", "qpos", "qvel", "act", "qacc_warmstart", "ctrl")
OUT = ("act_dot", "actuator_force", "qfrc_actuator", "sensordata")


def batched_lengthrange_inputs(mjm, nworld=S.NWORLD):
  """Per-world jnt_range / tendon_range (scaled by 1, 1.5, 0.5, ...) and actuator_gear (sign flipped in odd worlds, scaled in world 2)."""
  scale = np.array([1.0, 1.5, 0.5, 2.0])[np.arange(nworld) % 4]
  jr = np.asarray(mjm.jnt_range, dtype=np.float64)[None] * scale[:, None, None]
  tr = np.asarray(getattr(mjm, "tendon_range", np.zeros((0, 2))), dtype=np.float64).reshape(-1, 2)[None] * scale[:, None, None]
  gear = np.repeat(np.asarray(mjm.actuator_gear, dtype=np.float64)[None], nworld, axis=0)
  gear[1::2, :, 0] *= -1.0
  if nworld > 2:
    gear[2, :, 0] *= 0.75
  return jr, tr, gear


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  inverse = warp_shim.load_reference_module("inverse")
  set_const = warp_shim.load_reference_module("set_const")
  mjm = S.load(name)
  nsteps = S.SCENES[name][1]
  nworld = S.NWORLD
  nconmax, njmax = (32, 128) if name in BIG else (4, 32)
  t0 = time.time()
  ad = ref_runner.MjModelAdapter(mjm, defaults={"nJmom": mio.derive_tables(mjm)["nJmom"]})
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=nworld, nconmax=nconmax, njmax=njmax)
  qpos, qvel, act, ctrl = S.seeded(mjm, nsteps)
  d.qpos.a[...] = qpos
  d.qvel.a[...] = qvel
  d.act.a[...] = act
  d.ctrl.a[...] = ctrl[0]
  out = {"in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax), "in/ctrl": ctrl, "in/act": act}
  for f in STATE:
    out[f"start/{f}"] = getattr(d, f).numpy().copy()

  for tag, call in (("forward", lambda: fwd.forward(m, d)), ("inverse", lambda: inverse.inverse(m, d))):
    for f in STATE:
      getattr(d, f).a[...] = out[f"start/{f}"]
    call()
    for f in OUT:
      out[f"{tag}/{f}"] = getattr(d, f).numpy().copy()
  for f in STATE:
    getattr(d, f).a[...] = out[f"start/{f}"]

  for k in range(nsteps):
    d.ctrl.a[...] = ctrl[k]
    for f in STATE:
      out[f"step/{k}/in_{f}"] = getattr(d, f).numpy().copy()
    fwd.step(m, d)
    for f in STATE + OUT:
      out[f"step/{k}/out_{f}"] = getattr(d, f).numpy().copy()

  # set_length_range writes one entry per world (the reference's launch is nworld x nu): a per-world output, first from the model's
  # own sources, then from per-world ones
  m.actuator_lengthrange = wp.array(np.zeros((nworld, int(mjm.nu), 2)), dtype=wp.vec2)
  set_const.set_length_range(m, d)
  out["lengthrange/single"] = m.actuator_lengthrange.numpy().copy()
  jr, tr, gear = batched_lengthrange_inputs(mjm)
  m.jnt_range = wp.array(jr, dtype=wp.vec2)
  if int(getattr(mjm, "ntendon", 0)):
    m.tendon_range = wp.array(tr, dtype=wp.vec2)
  m.actuator_gear = wp.array(gear, dtype=wp.spatial_vector)
  m.actuator_lengthrange = wp.array(np.zeros((nworld, int(mjm.nu), 2)), dtype=wp.vec2)
  set_const.set_length_range(m, d)
  out["lengthrange/jnt_range"], out["lengthrange/tendon_range"], out["lengthrange/gear"] = jr, tr, gear
  out["lengthrange/batched"] = m.actuator_lengthrange.numpy().copy()

  path = os.path.join(ROOT, "tests", "golden", f"muscle_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: nu {mjm.nu}, na {mjm.na}, {nsteps} steps, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(S.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
