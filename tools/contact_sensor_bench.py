"""Times the humanoid's step with and without four <contact> foot sensors, and the contact-sensor kernel itself.

  python tools/contact_sensor_bench.py [--reps 50] [--warmup 10] [--out profiles/contact_sensor_bench_h100.json]

Workload: the benchmark humanoid (tests/contact_sensor_scenes.humanoid) at 8192 worlds, keyframe 0 with seeded noise, with four sensors
(subtree1 on each foot, data "found force", reduce netforce and maxforce) against the same model without sensors.  The two models are
stepped alternately, each step timed with CUDA events; k_sensor_contact's own time is the sum of its kernel records in a torch.profiler
trace of `--prof` steps.  Writes one JSON object with the card name and its power limit, read in the same run.
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
from mujoco_warp_b200.scenes import WORKLOADS  # noqa: E402
from tests import contact_sensor_scenes as scenes  # noqa: E402
from tests import util  # noqa: E402
from tests.test_oracle_golden_pipeline import load_scene  # noqa: E402

NWORLD = 8192


def make(mjm):
  wl = WORKLOADS["humanoid"]
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=NWORLD, m=m, nconmax=wl["nconmax"], njmax=wl["njmax"])
  qpos, qvel, _, _ = util.seeded_state(mjm, NWORLD, key=0, seed=11, qpos_noise=0.02, qvel_noise=0.3)
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


def kernel_us(m, d, nstep):
  from torch.profiler import ProfilerActivity, profile

  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(nstep):
      mjw.step(m, d)
    torch.cuda.synchronize()
  tot = {}
  for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA and "k_sensor" in e.name:
      key = "k_sensor_contact" if "k_sensor_contact" in e.name else "k_sensor"
      tot[key] = tot.get(key, 0.0) + e.device_time
  return {k: round(v / nstep, 2) for k, v in tot.items()}


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--reps", type=int, default=50)
  p.add_argument("--warmup", type=int, default=10)
  p.add_argument("--prof", type=int, default=10)
  p.add_argument("--out", default=os.path.join("profiles", "contact_sensor_bench_h100.json"))
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  runs = {"feet_sensors": make(scenes.humanoid()), "no_sensors": make(load_scene("humanoid"))}
  for _ in range(a.warmup):
    for m, d in runs.values():
      mjw.step(m, d)
  ms = {k: [] for k in runs}
  for _ in range(a.reps):  # alternate, so that clock drift hits both alike
    for k, (m, d) in runs.items():
      ms[k].append(timed(lambda: mjw.step(m, d)))
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q, "nworld": NWORLD, "reps": a.reps,
         "workload": "humanoid (benchmark model), keyframe 0 + seeded noise; feet_sensors: subtree1 on foot_right / foot_left, data found force, netforce and maxforce"}
  for k, (m, d) in runs.items():
    mjw.step(m, d)
    res[k] = dict(step_ms_median=round(float(np.median(ms[k])), 4), step_ms_p10=round(float(np.percentile(ms[k], 10)), 4),
                  step_ms_p90=round(float(np.percentile(ms[k], 90)), 4), launches=mjw.last_launch_count(),
                  kernel_us_per_step=kernel_us(m, d, a.prof), finite=bool(torch.isfinite(d.sensordata).all() and torch.isfinite(d.qpos).all()))
  sd = runs["feet_sensors"][1].sensordata.cpu().numpy()
  res["feet_sensors"]["worlds_with_foot_contact"] = int((sd[:, 0] > 0).sum())
  res["step_ms_delta_median"] = round(res["feet_sensors"]["step_ms_median"] - res["no_sensors"]["step_ms_median"], 4)
  line = json.dumps(res)
  print(line)
  os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
  with open(a.out, "w") as f:
    f.write(line + "\n")


if __name__ == "__main__":
  main()
