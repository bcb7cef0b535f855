"""Times the step with and without actuator and sensor delays, on one GPU.

  python tools/history_bench.py [--reps 30] [--warmup 5] [--out FILE]

Workloads: the humanoid at 8192 worlds and unitree G1 at 4096, from seeded states.  Each runs two Models of the same robot, one as
compiled and one with every actuator delayed by two timesteps (nsample 4, linear) and every sensor by two timesteps (nsample 4,
linear), each with its own Data; their steps alternate and each is timed with CUDA events.  A separate torch.profiler pass over a few
delayed steps reports the k_history kernels' own device time per step.  Prints one JSON line with the card name and its power limit,
read in the same run, and writes it to --out when given.
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
from tests import history_scenes, util  # noqa: E402


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def workload(path, nworld, nconmax, njmax, reps, warmup):
  runs = {}
  for key in ("off", "on"):
    mjm = mjw.mjcf.load_any(path)
    if key == "on":
      dt = float(mjm.opt.timestep)
      history_scenes.delay_all(mjm, 2 * dt, 4, 1, 2 * dt, 4, 1)
    m = mjw.put_model(mjm)
    d = mjw.make_data(mjm, nworld=nworld, nconmax=nconmax, njmax=njmax, m=m)
    qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld)
    for name, val in (("qpos", qpos), ("qvel", qvel), ("ctrl", ctrl)):
      getattr(d, name).copy_(torch.from_numpy(val.astype(np.float32)))
    runs[key] = (mjm, m, d)
  launches = {}
  for _ in range(warmup):
    for key, (_, m, d) in runs.items():
      mjw.step(m, d)
      launches[key] = mjw.last_launch_count()
  ms = {"off": [], "on": []}
  for _ in range(reps):
    for key, (_, m, d) in runs.items():
      ms[key].append(timed(lambda: mjw.step(m, d)))
  torch.cuda.synchronize()
  mjm, m, d = runs["on"]
  nprof = 10
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(nprof):
      mjw.step(m, d)
    torch.cuda.synchronize()
  kernels = {}
  for e in prof.key_averages():
    if "k_history" in e.key:
      name = e.key.split("k_history")[1].split("(")[0].split("E")[0]
      kernels["k_history" + name] = round(e.device_time_total / 1000.0 / nprof, 4)
  out = {"nworld": nworld, "nu": mjm.nu, "nsensor": int(getattr(mjm, "nsensor", 0)), "nhistory": int(m.nhistory),
         "launches_off": launches["off"], "launches_on": launches["on"], "qpos_finite": bool(torch.isfinite(d.qpos).all()),
         "history_kernels_ms_per_step": kernels}
  for k, v in ms.items():
    out[f"step_{k}_ms_median"] = round(float(np.median(v)), 4)
    out[f"step_{k}_ms_spread"] = round(float(np.percentile(v, 90) - np.percentile(v, 10)), 4)
  out["on_minus_off_ms_median"] = round(float(np.median(np.asarray(ms["on"]) - np.asarray(ms["off"]))), 4)
  return out


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--reps", type=int, default=30)
  p.add_argument("--warmup", type=int, default=5)
  p.add_argument("--out", default=None)
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q}
  res["humanoid_8192"] = workload(util.HUMANOID, 8192, 24, 64, a.reps, a.warmup)
  res["g1_4096"] = workload(util.G1, 4096, 48, 192, a.reps, a.warmup)
  line = json.dumps(res)
  print(line)
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
