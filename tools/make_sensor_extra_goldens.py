"""Magnetometer / camprojection / insidesite / tendon limit / tendonactfrc fixtures from the reference's own code, executed on the CPU
through tools/warp_shim.py.

  python tools/make_sensor_extra_goldens.py [scene ...]   # writes tests/golden/sensor_extra_<scene>.npz

For every scene of tests/sensor_extra_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data (NWORLD
worlds), seeded per-world qpos / qvel (and, for `batched`, per-world opt.magnetic, cam_fovy and cam_intrinsic, stored under `in/`), then
- `forward/*`: sensordata and the inputs the sensors read (site / camera poses, efc rows, actuator_force) after forward.forward from the
  seeded state with the first step's ctrl;
- `step/<k>/in_*` and `step/<k>/out_*` for each step k: the state before (time, qpos, qvel, qacc_warmstart, ctrl, history) and after one
  forward.step (the same plus sensordata), so that a test can replay every step.
One process per scene, as in make_muscle_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import io as mio  # noqa: E402
from tests import sensor_extra_scenes as S  # noqa: E402
from tools import ref_runner  # noqa: E402

STATE = ("time", "qpos", "qvel", "qacc_warmstart", "ctrl", "history")
OUT = ("sensordata",)
INPUTS = ("site_xpos", "site_xmat", "cam_xpos", "cam_xmat", "xpos", "xipos", "geom_xpos", "subtree_com", "actuator_force", "ne", "nf", "nl")
EFC = ("type", "id", "pos", "margin", "vel", "force")


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  mjm = S.load(name)
  _, nsteps, per_world = S.SCENES[name]
  nworld = S.NWORLD
  nconmax, njmax = 4, 16
  t0 = time.time()
  ad = ref_runner.MjModelAdapter(mjm, defaults={"nJmom": mio.derive_tables(mjm)["nJmom"]})
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=nworld, nconmax=nconmax, njmax=njmax)
  out = {"in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax)}
  if per_world:
    mag, fovy, intr = S.batched(mjm)
    m.opt.magnetic = wp.array(mag, dtype=wp.vec3)
    m.cam_fovy = wp.array(fovy, dtype=float)
    m.cam_intrinsic = wp.array(intr, dtype=wp.vec4)
    out["in/magnetic"], out["in/cam_fovy"], out["in/cam_intrinsic"] = mag, fovy, intr
  qpos, qvel, ctrl = S.seeded(mjm, nsteps)
  d.qpos.a[...] = qpos
  d.qvel.a[...] = qvel
  d.ctrl.a[...] = ctrl[0]
  out["in/ctrl"] = ctrl
  for f in STATE:
    out[f"start/{f}"] = getattr(d, f).numpy().copy()

  fwd.forward(m, d)
  for f in OUT + INPUTS:
    out[f"forward/{f}"] = getattr(d, f).numpy().copy()
  for f in EFC:
    out[f"forward/efc_{f}"] = getattr(d.efc, f).numpy().copy()
  for f in STATE:
    getattr(d, f).a[...] = out[f"start/{f}"]

  for k in range(nsteps):
    d.ctrl.a[...] = ctrl[k]
    for f in STATE:
      out[f"step/{k}/in_{f}"] = getattr(d, f).numpy().copy()
    fwd.step(m, d)
    for f in STATE + OUT:
      out[f"step/{k}/out_{f}"] = getattr(d, f).numpy().copy()

  path = os.path.join(ROOT, "tests", "golden", f"sensor_extra_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: nsensor {mjm.nsensor}, {nsteps} steps, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(S.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
