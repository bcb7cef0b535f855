"""Times the step of the muscle humanoid against the same model with affine actuators, on one GPU.

  python tools/muscle_bench.py [--nworld 8192] [--reps 30] [--warmup 5] [--out profiles/muscle_bench_h100.json]

Both models are tests/muscle_scenes.py's humanoid with two actuators per motor (42 actuators, 42 activations): muscles, or affine gain
and bias with filter dynamics.  Each gets its own Data from the same seeded state and ctrl; their steps alternate and each is timed
with CUDA events.  Prints one JSON line with the card name and its power limit, read in the same run, and writes it to --out when given.
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
from tests import muscle_scenes, util  # noqa: E402


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--nworld", type=int, default=8192)
  p.add_argument("--reps", type=int, default=30)
  p.add_argument("--warmup", type=int, default=5)
  p.add_argument("--out", default=None)
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  runs = {}
  for key, muscle in (("affine", False), ("muscle", True)):
    mjm = muscle_scenes.humanoid(muscle)
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=a.nworld, nconmax=24, njmax=64, m=m)
    qpos, qvel, _, _ = util.seeded_state(mjm, a.nworld)
    ctrl = np.random.default_rng(0).uniform(0.0, 1.0, (a.nworld, mjm.nu))
    for name, val in (("qpos", qpos), ("qvel", qvel), ("ctrl", ctrl)):
      getattr(d, name).copy_(torch.from_numpy(np.asarray(val, dtype=np.float32)))
    runs[key] = (mjm, m, d)
  for _ in range(a.warmup):
    for _, m, d in runs.values():
      mjw.step(m, d)
  ms = {k: [] for k in runs}
  for _ in range(a.reps):
    for key, (_, m, d) in runs.items():
      ms[key].append(timed(lambda: mjw.step(m, d)))
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q, "nworld": a.nworld, "nu": int(runs["muscle"][0].nu),
         "qpos_finite": {k: bool(torch.isfinite(d.qpos).all()) for k, (_, _, d) in runs.items()}}
  for k, v in ms.items():
    med = float(np.median(v))
    res[f"{k}_step_ms_median"] = round(med, 4)
    res[f"{k}_step_ms_spread"] = round(float(np.percentile(v, 90) - np.percentile(v, 10)), 4)
    res[f"{k}_env_steps_per_s"] = round(a.nworld / (med * 1e-3))
  res["muscle_minus_affine_ms_median"] = round(float(np.median(np.asarray(ms["muscle"]) - np.asarray(ms["affine"]))), 4)
  line = json.dumps(res)
  print(line)
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
