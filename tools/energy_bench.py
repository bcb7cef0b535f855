"""Times the step with energy off and on, on one GPU.

  python tools/energy_bench.py [--reps 30] [--warmup 5] [--out FILE]

Workloads: the humanoid and unitree G1, each at 8192 worlds, from seeded states.  One Model per workload; `m.opt.enableflags` is toggled
between calls, so the off and on steps alternate on the same Data (turning energy on adds one k_energy launch per world half after the
sensors).  Each step is timed with CUDA events.  Prints one JSON line with the card name and its power limit, read in the same run, and
writes it to --out when given.
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
from mujoco_warp_b200._src import constants as C  # noqa: E402
from tests import util  # noqa: E402


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def workload(path, nworld, nconmax, njmax, reps, warmup):
  mjm = mjw.mjcf.load_any(path)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=nworld, nconmax=nconmax, njmax=njmax, m=m)
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld)
  for name, val in (("qpos", qpos), ("qvel", qvel), ("ctrl", ctrl)):
    getattr(d, name).copy_(torch.from_numpy(val.astype(np.float32)))
  off, on = int(m.opt.enableflags) & ~C.ENBL_ENERGY, int(m.opt.enableflags) | C.ENBL_ENERGY
  launches = {}
  for flags in (off, on) * warmup:
    m.opt.enableflags = flags
    mjw.step(m, d)
    launches["off" if flags == off else "on"] = mjw.last_launch_count()
  ms = {"off": [], "on": []}
  for _ in range(reps):
    for key, flags in (("off", off), ("on", on)):
      m.opt.enableflags = flags
      ms[key].append(timed(lambda: mjw.step(m, d)))
  torch.cuda.synchronize()
  out = {"nworld": nworld, "nv": mjm.nv, "nbody": mjm.nbody, "launches_off": launches["off"], "launches_on": launches["on"],
         "energy_finite": bool(torch.isfinite(d.energy).all())}
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
  res["g1_8192"] = workload(util.G1, 8192, 48, 192, a.reps, a.warmup)
  line = json.dumps(res)
  print(line)
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
