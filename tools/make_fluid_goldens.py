"""Fluid-force fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_fluid_goldens.py [scene ...]   # writes tests/golden/fluid_<scene>.npz

For every scene of tests/fluid_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data -> forward.forward,
then NSTEP x forward.step, from seeded states (3 worlds).  The snapshot of make_pipeline_goldens.py is stored after forward and after
each step, plus qfrc_fluid.  The file names stay outside the pipeline_* glob: the fp64 C oracle has no fluid model.
One process per scene, as in make_pipeline_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import mjcf  # noqa: E402
from tests import fluid_scenes, util  # noqa: E402
from tools import make_pipeline_goldens as pg  # noqa: E402
from tools import ref_runner  # noqa: E402

NSTEP = 4


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  xml, nworld = fluid_scenes.SCENES[name]
  mjm = mjcf.load_string(xml)
  t0 = time.time()
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  qpos, qvel, ctrl, warm = (f32(a) for a in util.seeded_state(mjm, nworld, key=None, seed=1234, qpos_noise=0.05, qvel_noise=1.0, ctrl_noise=0.5, exact_world0=False))
  ad = ref_runner.MjModelAdapter(mjm)
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=nworld, nconmax=4, njmax=16)
  d.qpos.a[...] = qpos; d.qvel.a[...] = qvel; d.qacc_warmstart.a[...] = warm
  if mjm.nu:
    d.ctrl.a[...] = ctrl
  out = {"in/qpos": qpos, "in/qvel": qvel, "in/ctrl": ctrl, "in/qacc_warmstart": warm, "in/nconmax": np.array(4), "in/njmax": np.array(16)}
  fwd.forward(m, d)
  pg.snapshot(mjm, d, out, "forward")
  out["forward/qfrc_fluid"] = d.qfrc_fluid.numpy()
  for s in range(NSTEP):
    fwd.step(m, d)
    pg.snapshot(mjm, d, out, f"step{s}")
    out[f"step{s}/qfrc_fluid"] = d.qfrc_fluid.numpy()
  path = os.path.join(ROOT, "tests", "golden", f"fluid_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: |qfrc_fluid| max {np.abs(out['forward/qfrc_fluid']).max():.3g}, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; "
        f"MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(fluid_scenes.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
