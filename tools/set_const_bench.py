"""Times set_const against one step on one GPU.

  python tools/set_const_bench.py [--reps 20] [--warmup 3]

Workloads: the humanoid at 8192 worlds and unitree G1 at 4096, with body_mass scaled per world and every field set_const writes
batched to nworld (each world's constants computed and stored).  set_const is timed through its C entry point (all three parts and
the restore, CUDA events; the Python wrapper adds one stream synchronise for meaninertia) and through the Python wrapper (host clock
around the call, which ends in that synchronise); the step is timed with CUDA events.  Calls alternate between the two.  Prints one
JSON line with the card name and its power limit, read in the same run.
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mujoco_warp_b200 as mjw  # noqa: E402
from mujoco_warp_b200._src import _lib  # noqa: E402
from tests import set_const_scenes, util  # noqa: E402


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def workload(path, nworld, nconmax, njmax, reps, warmup):
  mjm = mjw.mjcf.load_any(path)
  m = mjw.put_model(mjm, batch_sizes={"body_mass": nworld, **{f: nworld for f in set_const_scenes.OUTPUTS}})
  m.body_mass.mul_(torch.linspace(0.8, 1.25, nworld, device=m.body_mass.device)[:, None])
  d = mjw.make_data(mjm, nworld=nworld, nconmax=nconmax, njmax=njmax, m=m)
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, nworld)
  for name, val in (("qpos", qpos), ("qvel", qvel), ("ctrl", ctrl)):
    getattr(d, name).copy_(torch.from_numpy(val.astype(np.float32)))
  L = _lib.lib()
  c_call = lambda: _lib.check(L.mjb_set_const(m._handle, d._handle, 7, 1, torch.cuda.current_stream().cuda_stream))
  for _ in range(warmup):
    mjw.set_const(m, d)
    mjw.step(m, d)
  ms = {"set_const_c": [], "set_const_py": [], "step": []}
  for _ in range(reps):
    ms["set_const_c"].append(timed(c_call))
    launches = mjw.last_launch_count()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mjw.set_const(m, d)
    ms["set_const_py"].append((time.perf_counter() - t0) * 1e3)
    ms["step"].append(timed(lambda: mjw.step(m, d)))
  out = {"nworld": nworld, "nv": mjm.nv, "nbody": mjm.nbody, "nu": mjm.nu, "set_const_launches": launches,
         "finite": bool(all(torch.isfinite(getattr(m, f)).all() for f in ("dof_invweight0", "body_invweight0", "actuator_acc0")))}
  for k, v in ms.items():
    out[f"{k}_ms_median"] = round(float(np.median(v)), 4)
    out[f"{k}_ms_spread"] = round(float(np.percentile(v, 90) - np.percentile(v, 10)), 4)
  return out


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--reps", type=int, default=20)
  p.add_argument("--warmup", type=int, default=3)
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q}
  res["humanoid_8192"] = workload(util.HUMANOID, 8192, 24, 64, a.reps, a.warmup)
  res["g1_4096"] = workload(util.G1, 4096, 48, 192, a.reps, a.warmup)
  print(json.dumps(res))


if __name__ == "__main__":
  main()
