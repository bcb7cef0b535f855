"""The batched frame-sensor fixture from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_sensor_goldens.py   # writes tests/golden/sensor_batched.npz

The UNMODIFIED reference runs the scene of tests/sensor_scenes.py in double precision: io.put_model with per-world body_iquat, geom_quat,
site_quat and cam_quat (sensor_scenes.batched, stored under `in/`), io.make_data, the seeded state, then forward.forward.  `forward/*`
holds what forward left (tools/make_pipeline_goldens.py's snapshot), sensordata included.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import sensor_scenes as S  # noqa: E402
from tools import ref_runner  # noqa: E402
from tools.make_pipeline_goldens import snapshot  # noqa: E402


def main():
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  mjm = S.load()
  nconmax, njmax = 4, 8
  t0 = time.time()
  ad = ref_runner.MjModelAdapter(mjm)
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=S.NWORLD, nconmax=nconmax, njmax=njmax)
  out = {"in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax)}
  for k, v in S.batched(mjm).items():
    setattr(m, k, wp.array(v, dtype=wp.quat))
    out[f"in/{k}"] = v
  qpos, qvel = S.state(mjm)
  d.qpos.a[...] = qpos; d.qvel.a[...] = qvel
  out.update({"in/qpos": qpos, "in/qvel": qvel})
  fwd.forward(m, d)
  snapshot(mjm, d, out, "forward")
  out["forward/sensordata"] = d.sensordata.numpy().copy()
  path = os.path.join(ROOT, "tests", "golden", "sensor_batched.npz")
  np.savez_compressed(path, **out)
  print(f"sensor_batched: nsensor {mjm.nsensor}, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  main()
