"""Times a rendered frame (mjw.refit_bvh + mjw.render, k_render.cu) against a physics step with CUDA events.

  python tools/render_bench.py [--reps 30] [--warmup 5] [--out render_bench.json]

Workloads: the humanoid (test_data/humanoid.npz, bench keyframe with qpos noise) at 8192 and 1024 worlds, its camera 0 at 64 x 64;
three frame kinds: rgb + depth without shadows, rgb + depth with shadows, segmentation only.  Frames and steps alternate in one
loop, each timed by its own event pair, so the cost of a frame next to a step is read from the same conditions.  Prints one JSON
line (and writes it to --out) with the card name and its power limit, read in the same run.
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

RES = (64, 64)
KINDS = {"rgb_depth": dict(render_rgb=True, render_depth=True, render_seg=False, use_shadows=False),
         "rgb_depth_shadows": dict(render_rgb=True, render_depth=True, render_seg=False, use_shadows=True),
         "seg_only": dict(render_rgb=False, render_depth=False, render_seg=True, use_shadows=False)}


def state(nworld):
  wl = WORKLOADS["humanoid"]
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


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn()
  b.record()
  return a, b


def run(nworld, kind, reps, warmup):
  mjm, m, d = state(nworld)
  rc = mjw.create_render_context(mjm, nworld=nworld, cam_active=[0], cam_res=RES, **KINDS[kind])
  frame = lambda: (mjw.refit_bvh(m, d, rc), mjw.render(m, d, rc))
  step = lambda: mjw.step(m, d)
  for _ in range(warmup):
    step()
    frame()
  ev = []
  for _ in range(reps):
    ev.append((timed(step), timed(frame)))
  torch.cuda.synchronize()
  step_ms = [s[0].elapsed_time(s[1]) for s, _ in ev]
  frame_ms = [f[0].elapsed_time(f[1]) for _, f in ev]
  med = float(np.median(frame_ms))
  pixels = nworld * RES[0] * RES[1]
  hit = float((rc.seg_data[..., 0] >= 0).float().mean()) if rc.render_seg[0] else float((rc.depth_data > 0).float().mean())
  return dict(nworld=nworld, kind=kind, ngeom_rendered=rc.bvh_ngeom, nlight=int(mjm.nlight), frame_ms_median=round(med, 4),
              frame_ms_min=round(float(np.min(frame_ms)), 4), frame_ms_max=round(float(np.max(frame_ms)), 4), step_ms_median=round(float(np.median(step_ms)), 4),
              frame_over_step=round(med / float(np.median(step_ms)), 3), pixels_per_s=float(f"{pixels / (med * 1e-3):.4g}"), hit_fraction=round(hit, 4),
              buffer_bytes=int(sum(x.numel() * x.element_size() for x in (rc.rgb_data, rc.depth_data, rc.seg_data))))


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
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q, "camera": 0, "resolution": list(RES), "reps": a.reps, "warmup": a.warmup,
         "runs": [run(n, k, a.reps, a.warmup) for n in (8192, 1024) for k in KINDS]}
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
