"""Times mjw.inverse against mjw.forward from one state, and k_inverse against k_solver, on the benchmark configurations.

  python tools/inverse_bench.py [--reps 30] [--warmup 5]

Workloads: humanoid at 8192 worlds and g1 at 4096 (bench.py's models, nconmax / njmax and keyframe, 50 bench-style steps with control
noise from the keyframe).  From that state `forward` and `inverse` (at forward's qacc) are called alternately, each timed with CUDA
events; neither changes the state the other reads, so every call starts from the same one.  Kernel times come from one
torch.profiler trace of a forward and an inverse call (k_inverse, k_solver).  Prints one JSON line with the card name and its power
limit, read in the same run.
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
from mujoco_warp_b200._src.mjcf import MjDataLite, load_any, reset_data_keyframe  # noqa: E402
from mujoco_warp_b200.scenes import WORKLOADS  # noqa: E402


def state(workload, nworld, steps=50):
  wl = WORKLOADS[workload]
  mjm = load_any(wl["model"])
  mjd = MjDataLite(mjm)
  if mjm.nkey > 0:
    reset_data_keyframe(mjm, mjd, 0)
  m = mjw.put_model(mjm)
  d = mjw.put_data(mjm, mjd, nworld=nworld, nconmax=wl["nconmax"], njmax=wl["njmax"], m=m)
  for s in range(steps):
    mjw.ctrl_noise(m, d, s)
    mjw.step(m, d)
  mjw.forward(m, d)
  torch.cuda.synchronize()
  return m, d


def timed(fn, reps):
  ms = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    ms.append(a.elapsed_time(b))
  return ms


def kernel_us(m, d):
  from torch.profiler import ProfilerActivity, profile

  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    mjw.forward(m, d)
    mjw.inverse(m, d)
    torch.cuda.synchronize()
  out = {}
  for e in prof.events():
    for k in ("k_inverse", "k_solver"):
      if k in e.name:
        out[k] = out.get(k, 0.0) + e.device_time_total if hasattr(e, "device_time_total") else out.get(k, 0.0) + e.cuda_time_total
  return {k: round(v, 1) for k, v in out.items()}  # summed over the world halves of the split launch


def run(workload, nworld, reps, warmup):
  m, d = state(workload, nworld)
  for _ in range(warmup):
    mjw.forward(m, d)
    mjw.inverse(m, d)
  fwd, inv = [], []
  for _ in range(reps):  # alternate, so that clock drift hits both alike
    fwd += timed(lambda: mjw.forward(m, d), 1)
    inv += timed(lambda: mjw.inverse(m, d), 1)
  k = kernel_us(m, d)
  return dict(nworld=nworld, forward_ms_median=round(float(np.median(fwd)), 4), inverse_ms_median=round(float(np.median(inv)), 4),
              forward_ms_spread=round(float(np.percentile(fwd, 90) - np.percentile(fwd, 10)), 4),
              inverse_ms_spread=round(float(np.percentile(inv, 90) - np.percentile(inv, 10)), 4), kernel_us=k,
              nefc_mean=round(float(d.nefc.float().mean()), 2))


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
  res["humanoid"] = run("humanoid", 8192, a.reps, a.warmup)
  res["g1"] = run("g1", 4096, a.reps, a.warmup)
  print(json.dumps(res))


if __name__ == "__main__":
  main()
