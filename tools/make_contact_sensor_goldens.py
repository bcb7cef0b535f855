"""Contact-sensor fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_contact_sensor_goldens.py [scene ...]   # writes tests/golden/contact_sensor_<scene>.npz

For every scene of tests/contact_sensor_scenes.SCENES the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data ->
forward.forward, then NSTEP x forward.step, from seeded states (3 worlds).  Stored after forward and after each step: the state, the
contact arrays (dist, pos, frame, friction, dim, geom, efc_address, worldid, type), efc_force and sensordata.  The shim runs a launch's
threads in index order and its tile_sort is stable, so the reference's matches come out in pool order and its sort ties break by pool
index, as here.  MuJoCo's mj_name2id is a stub in the shim; the model's <numeric> names are looked up directly so that
contact_sensor_maxmatch reaches the reference.  One process per scene, as in make_pipeline_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import mjcf  # noqa: E402
from tests import contact_sensor_scenes, util  # noqa: E402
from tools import ref_runner  # noqa: E402

NSTEP = 3
NWORLD = 3
CON = ["dist", "pos", "frame", "friction", "dim", "geom", "efc_address", "worldid", "type"]


def snapshot(d, out, tag):
  for f in ("site_xpos", "site_xmat", "sensordata"):
    out[f"{tag}/{f}"] = getattr(d, f).numpy()
  nacon = int(d.nacon.numpy()[0])
  out[f"{tag}/nacon"] = np.array(nacon)
  for f in CON:
    out[f"{tag}/con_{f}"] = getattr(d.contact, f).numpy()[:nacon]
  out[f"{tag}/efc_force"] = d.efc.force.numpy()
  out[f"{tag}/overflow"] = d.overflow.numpy()
  for f in ("qpos", "qvel", "qacc_warmstart", "time"):
    out[f"{tag}/{f}"] = getattr(d, f).numpy()


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  xml, njmax = contact_sensor_scenes.SCENES[name]
  mjm = mjcf.load_string(xml)
  mj = sys.modules["mujoco"]
  mj.mj_name2id = lambda m, t, n: (list(mjm.names.numeric).index(n) if t == mj.mjtObj.mjOBJ_NUMERIC and n in list(mjm.names.numeric) else -1)
  t0 = time.time()
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  qpos, qvel, _, warm = (f32(a) for a in util.seeded_state(mjm, NWORLD, key=None, seed=1234, qpos_noise=0.01, qvel_noise=0.3, exact_world0=False))
  ad = ref_runner.MjModelAdapter(mjm)
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=NWORLD, nconmax=64, njmax=njmax)
  d.qpos.a[...] = qpos; d.qvel.a[...] = qvel; d.qacc_warmstart.a[...] = warm
  out = {"in/qpos": qpos, "in/qvel": qvel, "in/qacc_warmstart": warm, "njmax": np.array(njmax), "maxmatch": np.array(int(m.opt.contact_sensor_maxmatch))}
  fwd.forward(m, d)
  snapshot(d, out, "forward")
  for s in range(NSTEP):
    fwd.step(m, d)
    snapshot(d, out, f"step{s}")
  path = os.path.join(ROOT, "tests", "golden", f"contact_sensor_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: {mjm.nsensor} sensors, nacon {int(out['forward/nacon'])}, maxmatch {int(out['maxmatch'])}, {os.path.getsize(path) // 1024} KiB, "
        f"{time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(contact_sensor_scenes.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
