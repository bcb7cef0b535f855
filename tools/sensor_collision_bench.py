"""Times the step with distance / normal / fromto sensors against the same model without them.

  python tools/sensor_collision_bench.py [--reps 30] [--warmup 5]

Workloads, 8192 worlds each: the three-body scene of tests/sensor_collision_scenes.py (36 sensors over 5 unique geom pairs) with
primitive pairs only (sphere, sphere, box, capsule) and with GJK / EPA pairs (ellipsoid, cylinder, box, box), each against the same
scene with its sensor block removed.  The two models of a pair are stepped alternately, each step timed with CUDA events.  Prints one
JSON line with the card name and its power limit, read in the same run.
"""

import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mujoco_warp_b200 as mjw  # noqa: E402
from mujoco_warp_b200._src.mjcf import load_string  # noqa: E402
from tests import sensor_collision_scenes as scenes  # noqa: E402
from tests import util  # noqa: E402


def make(xml, nworld):
  mjm = load_string(xml)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, m=m, nconmax=4, njmax=16)
  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=None, seed=3, qpos_noise=0.3, qvel_noise=0.5, exact_world0=False)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  torch.cuda.synchronize()
  return mjm, m, d


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def pair(xml, nworld, reps, warmup):
  runs = {"sensors": make(xml, nworld), "none": make(re.sub(r"<sensor>.*</sensor>", "", xml, flags=re.S), nworld)}
  for _ in range(warmup):
    for _, m, d in runs.values():
      mjw.step(m, d)
  ms = {k: [] for k in runs}
  for _ in range(reps):  # alternate, so that clock drift hits both alike
    for k, (_, m, d) in runs.items():
      ms[k].append(timed(lambda: mjw.step(m, d)))
  out = {"nsensor": int(runs["sensors"][0].nsensor), "nsensorcollision": int(runs["sensors"][1].nsensorcollision)}
  for k, (_, m, d) in runs.items():
    mjw.step(m, d)
    out[k] = dict(step_ms_median=round(float(np.median(ms[k])), 4), step_ms_spread=round(float(np.percentile(ms[k], 90) - np.percentile(ms[k], 10)), 4),
                  launches=mjw.last_launch_count(), finite=bool(torch.isfinite(d.sensordata).all() and torch.isfinite(d.qpos).all()))
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
  res["primitive_8192"] = pair(scenes.pair_xml("sphere", "sphere", "box", "capsule"), 8192, a.reps, a.warmup)
  res["convex_8192"] = pair(scenes.pair_xml("ellipsoid", "cylinder", "box", "box"), 8192, a.reps, a.warmup)
  print(json.dumps(res))


if __name__ == "__main__":
  main()
