"""Times the step with fluid forces against the same model without them.

  python tools/fluid_bench.py [--reps 30] [--warmup 5]

Workloads:
- humanoid at 8192 worlds (bench.py's model, nconmax / njmax and keyframe, 50 bench-style steps with control noise first) in air --
  density 1.2, viscosity 1.8e-5, the inertia-box model on every body -- against the same model with neither;
- the ellipsoid-model scene of tests/fluid_scenes.py (every geom type) at 8192 worlds, Euler and implicitfast, against itself without fluid.
The two models of a pair are stepped alternately, each step timed with CUDA events; `step_profile` gives k_velocity's time (the
`velocity` group) and the integrator's.  Prints one JSON line with the card name and its power limit, read in the same run.
"""

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mujoco_warp_b200 as mjw  # noqa: E402
from mujoco_warp_b200._src.mjcf import MjDataLite, load_any, load_string, reset_data_keyframe  # noqa: E402
from mujoco_warp_b200.scenes import WORKLOADS  # noqa: E402
from tests import fluid_scenes, util  # noqa: E402


def humanoid(nworld, fluid):
  wl = WORKLOADS["humanoid"]
  mjm = load_any(wl["model"])
  if fluid:
    mjm.opt.density, mjm.opt.viscosity = 1.2, 1.8e-5
  mjd = MjDataLite(mjm)
  if mjm.nkey > 0:
    reset_data_keyframe(mjm, mjd, 0)
  m = mjw.put_model(mjm)
  d = mjw.put_data(mjm, mjd, nworld=nworld, nconmax=wl["nconmax"], njmax=wl["njmax"], m=m)
  for s in range(50):
    mjw.ctrl_noise(m, d, s)
    mjw.step(m, d)
  torch.cuda.synchronize()
  return m, d


def ellipsoid(nworld, fluid, integrator):
  mjm = load_string(fluid_scenes.ellipsoid_xml(integrator))
  if not fluid:
    mjm.opt.density, mjm.opt.viscosity, mjm.opt.wind = 0.0, 0.0, np.zeros(3)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m, nconmax=4, njmax=16)
  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=None, seed=3, qvel_noise=1.0, exact_world0=False)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  torch.cuda.synchronize()
  return m, d


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def pair(make, reps, warmup):
  runs = {"fluid": make(True), "none": make(False)}
  for _ in range(warmup):
    for m, d in runs.values():
      mjw.step(m, d)
  ms = {k: [] for k in runs}
  for _ in range(reps):  # alternate, so that clock drift hits both alike
    for k, (m, d) in runs.items():
      ms[k].append(timed(lambda: mjw.step(m, d)))
  out = {}
  for k, (m, d) in runs.items():
    prof = [mjw.step_profile(m, d) for _ in range(5)]
    out[k] = dict(step_ms_median=round(float(np.median(ms[k])), 4), step_ms_spread=round(float(np.percentile(ms[k], 90) - np.percentile(ms[k], 10)), 4),
                  k_velocity_ms=round(float(np.median([p["velocity"] for p in prof])), 4), integrate_ms=round(float(np.median([p["integrate"] for p in prof])), 4),
                  finite=bool(torch.isfinite(d.qpos).all()))
  return out


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--reps", type=int, default=30)
  p.add_argument("--warmup", type=int, default=5)
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q}
  res["humanoid_8192_air"] = pair(lambda f: humanoid(8192, f), a.reps, a.warmup)
  res["ellipsoid_8192_euler"] = pair(lambda f: ellipsoid(8192, f, "Euler"), a.reps, a.warmup)
  res["ellipsoid_8192_implicitfast"] = pair(lambda f: ellipsoid(8192, f, "implicitfast"), a.reps, a.warmup)
  print(json.dumps(res))


if __name__ == "__main__":
  main()
