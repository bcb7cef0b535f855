"""Reference fixtures for the large-hull mesh scenes (tests/mesh_hull_scenes.py), from the reference's own pipeline on the CPU.

  python tools/make_mesh_hull_goldens.py [scene ...]    # writes tests/golden/mesh_hull_<scene>.npz

The UNMODIFIED reference (io.put_model -> io.make_data -> forward.forward, then forward.step; its collision pipeline sizes the mesh
multi-contact buffers from the model, collision_convex.py:1229-1236) runs in double precision through tools/warp_shim.py on the model
compiled by mujoco_warp_b200._src.mjcf, from the scene's seeded states.  The fixture holds the inputs and the fields of
tools/make_pipeline_goldens.py after forward() and after each of NSTEP step() calls: contacts, constraint rows, sensordata, state.
"""

import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import mesh_hull_scenes as S  # noqa: E402
from tools import ref_runner  # noqa: E402
from tools.make_pipeline_goldens import snapshot  # noqa: E402

NSTEP = 4


def main(name):
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  t0 = time.time()
  mjm = S.load(name)
  cfg = S.SCENES[name]["cfg"]
  qpos, qvel, ctrl, warm = S.seeded(mjm, name)
  ad = ref_runner.MjModelAdapter(mjm)
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=S.NWORLD, nconmax=cfg["nconmax"], njmax=cfg["njmax"])
  d.qpos.a[...] = qpos; d.qvel.a[...] = qvel; d.qacc_warmstart.a[...] = warm
  if mjm.nu:
    d.ctrl.a[...] = ctrl
  out = {"in/qpos": qpos, "in/qvel": qvel, "in/ctrl": ctrl, "in/qacc_warmstart": warm, "in/nconmax": np.array(cfg["nconmax"]), "in/njmax": np.array(cfg["njmax"])}
  fwd.forward(m, d)
  snapshot(mjm, d, out, "forward")
  out["forward/overflow"] = d.overflow.numpy()
  for s in range(NSTEP):
    fwd.step(m, d)
    snapshot(mjm, d, out, f"step{s}")
    out[f"step{s}/overflow"] = d.overflow.numpy()
  path = os.path.join(ROOT, "tests", "golden", f"mesh_hull_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: nacon {int(out['forward/nacon'])}, nefc {out['forward/nefc'].ravel()}, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s")


if __name__ == "__main__":
  # one process per scene: the reference keeps process-global kernel state (see tools/make_pipeline_goldens.py)
  names = sys.argv[1:] or list(S.SCENES)
  if len(names) == 1:
    main(names[0])
  else:
    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
