"""Times mjw.rays (k_ray.cu) with CUDA events: median ms per call over repeated calls after warm-up, and rays per second.

  python tools/ray_bench.py [--reps 50] [--warmup 10]

Workloads: the humanoid at 8192 worlds from the bench keyframe (with qpos noise) casting an 11 x 17 downward height-scan grid
(187 rays, 0.1 m apart) from each world's torso; convex_mesh at 2048 worlds casting 64 rays per world (an 8 x 8 downward grid
from each world's first body).  Prints one JSON line with the card name and its power limit, read in the same run.
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


def state(workload, nworld):
  wl = WORKLOADS[workload]
  mjm = load_any(wl["model"])
  mjd = MjDataLite(mjm)
  if mjm.nkey > 0:
    reset_data_keyframe(mjm, mjd, 0)
  m = mjw.put_model(mjm)
  d = mjw.put_data(mjm, mjd, nworld=nworld, nconmax=wl["nconmax"], njmax=wl["njmax"], m=m)
  g = torch.Generator(device="cuda").manual_seed(0)
  d.qpos.add_(0.02 * torch.randn(d.qpos.shape, device="cuda", generator=g))
  mjw.forward(m, d)
  return mjm, m, d


def grid(d, body, nx, ny, spacing=0.1):
  c = d.xpos[:, body]
  gx, gy = torch.meshgrid((torch.arange(nx, device="cuda") - nx // 2) * spacing, (torch.arange(ny, device="cuda") - ny // 2) * spacing, indexing="ij")
  off = torch.stack([gx.reshape(-1), gy.reshape(-1), torch.zeros(nx * ny, device="cuda")], 1)
  pnt = (c[:, None, :] + off[None]).contiguous()
  vec = torch.tensor([0.0, 0.0, -1.0], device="cuda").expand(pnt.shape).contiguous()
  return pnt, vec


def time_rays(m, d, pnt, vec, reps, warmup):
  n = pnt.shape[1]
  bx = torch.full((n,), -1, dtype=torch.int32, device="cuda")
  out = (torch.empty(d.nworld, n, device="cuda"), torch.empty(d.nworld, n, dtype=torch.int32, device="cuda"), torch.empty(d.nworld, n, 3, device="cuda"))
  for _ in range(warmup):
    mjw.rays(m, d, pnt, vec, None, True, bx, *out)
  ms = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    mjw.rays(m, d, pnt, vec, None, True, bx, *out)
    b.record()
    b.synchronize()
    ms.append(a.elapsed_time(b))
  med = float(np.median(ms))
  return dict(nworld=d.nworld, nray=n, ngeom=int(d._model.ngeom), ms_median=round(med, 4), ms_min=round(float(np.min(ms)), 4),
              rays_per_s=float(f"{d.nworld * n / (med * 1e-3):.4g}"), hit_fraction=round(float((out[1] >= 0).float().mean()), 4))


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--reps", type=int, default=50)
  p.add_argument("--warmup", type=int, default=10)
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q}
  mjm, m, d = state("humanoid", 8192)
  pnt, vec = grid(d, mjm.names.body.index("torso"), 11, 17)
  res["humanoid_height_scan"] = time_rays(m, d, pnt, vec, a.reps, a.warmup)
  mjm, m, d = state("convex_mesh", 2048)
  pnt, vec = grid(d, 1, 8, 8)
  res["convex_mesh_64"] = time_rays(m, d, pnt, vec, a.reps, a.warmup)
  print(json.dumps(res))


if __name__ == "__main__":
  main()
