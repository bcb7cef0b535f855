"""Times a scene of 64-gon prism hulls (k_collision_mesh_large: multi-contact buffers in global scratch) against the same scene rebuilt with
32-gon prisms (k_collision_mesh: buffers on the stack), at 8192 worlds.

  python tools/mesh_hull_bench.py [--reps 50] [--warmup 10] [--prof 10] [--out profiles/mesh_hull_bench_h100.json]

Scene: tests/mesh_hull_scenes.prism_xml(n) -- prisms on the floor, on a box, cap-to-cap on a fixed prism and tilted onto their rim on a box;
about 14 contacts per world -- from seeded poses.  The two models are stepped alternately, each step timed with CUDA events (env-steps/s =
worlds / step time); the collision kernel's own time is the sum of its records in a torch.profiler trace of `--prof` steps (at 8192 worlds the
step runs two world halves on two streams, so this sum of both halves' kernels can exceed the step's wall time).  Writes one
JSON object with the card name and its power limit, read in the same run.
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
from mujoco_warp_b200._src import mjcf  # noqa: E402
from tests import mesh_hull_scenes as S  # noqa: E402
from tests import util  # noqa: E402

NWORLD = 8192


def make(n):
  mjm = mjcf.load_string(S.prism_xml(n))
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=NWORLD, m=m, nconmax=24, njmax=96)
  qpos, qvel, _, _ = util.seeded_state(mjm, NWORLD, key=None, seed=11, qpos_noise=0.0004, qvel_noise=0.05, exact_world0=False)
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


def collision_us(m, d, nstep):
  from torch.profiler import ProfilerActivity, profile

  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(nstep):
      mjw.step(m, d)
    torch.cuda.synchronize()
  tot, names = 0.0, set()
  for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA and "k_collision" in e.name:
      tot += e.device_time
      names.add(re.search(r"k_collision\w*", e.name).group(0))
  return round(tot / nstep, 2), sorted(names)


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--reps", type=int, default=50)
  p.add_argument("--warmup", type=int, default=10)
  p.add_argument("--prof", type=int, default=10)
  p.add_argument("--out", default=os.path.join("profiles", "mesh_hull_bench_h100.json"))
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  runs = {"prism64_large_build": make(64), "prism32_in_cap_build": make(32)}
  for _ in range(a.warmup):
    for m, d in runs.values():
      mjw.step(m, d)
  ms = {k: [] for k in runs}
  for _ in range(a.reps):  # alternate, so that clock drift hits both alike
    for k, (m, d) in runs.items():
      ms[k].append(timed(lambda: mjw.step(m, d)))
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q, "nworld": NWORLD, "reps": a.reps,
         "workload": "tests/mesh_hull_scenes.prism_xml(n): 4 free n-gon prisms per world (floor, box, cap-to-cap, rim on a box), seeded poses"}
  for k, (m, d) in runs.items():
    us, names = collision_us(m, d, a.prof)
    med = float(np.median(ms[k]))
    res[k] = dict(collision_kernel=mjw.collision_kernel(m), kernel_names=names, collision_us_per_step=us,
                  step_ms_median=round(med, 4), step_ms_p10=round(float(np.percentile(ms[k], 10)), 4), step_ms_p90=round(float(np.percentile(ms[k], 90)), 4),
                  env_steps_per_s_median=round(NWORLD / med * 1e3), nacon=int(d.nacon.cpu()[0]), overflow_worlds=int((d.overflow != 0).sum()),
                  finite=bool(torch.isfinite(d.qpos).all()))
  line = json.dumps(res)
  print(line)
  os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
  with open(a.out, "w") as f:
    f.write(line + "\n")


if __name__ == "__main__":
  main()
