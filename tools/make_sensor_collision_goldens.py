"""Collision-sensor fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_sensor_collision_goldens.py [scene ...]   # writes tests/golden/sensor_collision_<scene>.npz

For every scene of tests/sensor_collision_scenes.SCENES the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data ->
forward.forward, then NSTEP x forward.step, from seeded states (3 worlds).  Stored after forward and after each step: the geom poses and
sensordata the step computed (before it integrated), the contact arrays with contact.type (the reference's pool also holds the
sensor pairs' ContactType.SENSOR contacts), and the state.  `knife/<tag>` marks (world, sensor) entries whose normal is not determined
to fp32 precision: |distance| below 1e-3 (the witness points nearly coincide).  One process per scene, as in make_pipeline_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import constants as C  # noqa: E402
from mujoco_warp_b200._src import mjcf  # noqa: E402
from tests import sensor_collision_scenes, util  # noqa: E402
from tools import ref_runner  # noqa: E402

NSTEP = 3
NWORLD = 3
CON = ["dist", "pos", "frame", "geom", "worldid", "geomcollisionid", "type"]


def snapshot(mjm, d, out, tag):
  for f in ("geom_xpos", "geom_xmat", "sensordata"):
    out[f"{tag}/{f}"] = getattr(d, f).numpy()
  nacon = int(d.nacon.numpy()[0])
  out[f"{tag}/nacon"] = np.array(nacon)
  for f in CON:
    out[f"{tag}/con_{f}"] = getattr(d.contact, f).numpy()[:nacon]
  for f in ("qpos", "qvel", "qacc_warmstart", "time"):
    out[f"{tag}/{f}"] = getattr(d, f).numpy()
  dist = out[f"{tag}/sensordata"][:, np.asarray(mjm.sensor_adr)]
  out[f"knife/{tag}"] = (np.abs(dist) < 1e-3) & np.isin(np.asarray(mjm.sensor_type), (C.SENS_GEOMNORMAL, C.SENS_GEOMFROMTO))[None]


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  mjm = mjcf.load_string(sensor_collision_scenes.SCENES[name])
  t0 = time.time()
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  qpos, qvel, _, warm = (f32(a) for a in util.seeded_state(mjm, NWORLD, key=None, seed=1234, qpos_noise=0.05, qvel_noise=0.3, exact_world0=False))
  ad = ref_runner.MjModelAdapter(mjm)
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=NWORLD, nconmax=64, njmax=256)
  d.qpos.a[...] = qpos; d.qvel.a[...] = qvel; d.qacc_warmstart.a[...] = warm
  out = {"in/qpos": qpos, "in/qvel": qvel, "in/qacc_warmstart": warm}
  fwd.forward(m, d)
  snapshot(mjm, d, out, "forward")
  for s in range(NSTEP):
    qpos_before = d.qpos.numpy().copy()
    fwd.step(m, d)
    snapshot(mjm, d, out, f"step{s}")
    out[f"step{s}/qpos_before"] = qpos_before
  path = os.path.join(ROOT, "tests", "golden", f"sensor_collision_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: {mjm.nsensor} sensors, nacon {int(out['forward/nacon'])}, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; "
        f"MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(sensor_collision_scenes.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
