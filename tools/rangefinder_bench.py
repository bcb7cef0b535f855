"""Times the rangefinder sensor (k_sensor_rangefinder.cu) on the benchmark humanoid and writes one JSON result.

  python tools/rangefinder_bench.py [--nworld 8192] [--reps 50] [--rounds 5] [--out profiles/rangefinder_bench_h100.json]

Workload: benchmarks/humanoid/humanoid.xml from tests/golden/reference_models.tar.xz, compiled by this package's compiler with an 11 x 17
grid of downward sites 0.1 m apart on the torso (the height scan of tools/ray_bench.py), at nworld worlds from the squat keyframe with
qpos noise.  The same compiled model is run with the 187 sites carrying rangefinders and without those sensor rows.  Recorded:
- k_sensor_rangefinder's device time per launch, from torch.profiler over `reps` sensor_pos calls, and sensor_pos with and without the
  rows from CUDA events;
- step with and without the rows, alternated `rounds` times, `reps` steps per timing (CUDA events);
- rays() on the same rays (CUDA events), for comparison;
- the card's name and power limit, read in the same run.
"""

import argparse
import json
import os
import re
import subprocess
import sys
import tarfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mujoco_warp_b200 as mjw  # noqa: E402
from mujoco_warp_b200._src import io, mjcf  # noqa: E402
from mujoco_warp_b200._src.mjcf import MjDataLite, reset_data_keyframe  # noqa: E402
from tests import rangefinder_scenes as S  # noqa: E402

NX, NY, SPACING = 11, 17, 0.1


def humanoid_with_sites():
  with tarfile.open(os.path.join(ROOT, "tests", "golden", "reference_models.tar.xz")) as t:
    xml = t.extractfile("benchmarks/humanoid/humanoid.xml").read().decode()
  sites = "".join(f'<site name="rf{i}_{j}" pos="{(i - NX // 2) * SPACING:.2f} {(j - NY // 2) * SPACING:.2f} 0" euler="180 0 0" size="0.005"/>'
                  for i in range(NX) for j in range(NY))
  xml, n = re.subn(r'(<body name="torso"[^>]*>)', lambda mt: mt.group(1) + sites, xml, count=1)
  assert n == 1
  return xml


def data(mjm, m, nworld):
  mjd = MjDataLite(mjm)
  reset_data_keyframe(mjm, mjd, 0)
  d = mjw.put_data(mjm, mjd, nworld=nworld, nconmax=24, njmax=64, m=m)
  g = torch.Generator(device="cuda").manual_seed(0)
  d.qpos.add_(0.02 * torch.randn(d.qpos.shape, device="cuda", generator=g))
  mjw.forward(m, d)
  return d


def events(fn, reps):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(reps):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b) / reps


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--nworld", type=int, default=8192)
  p.add_argument("--reps", type=int, default=50)
  p.add_argument("--rounds", type=int, default=5)
  p.add_argument("--out", default=os.path.join(ROOT, "profiles", "rangefinder_bench_h100.json"))
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q, "nworld": a.nworld, "nrangefinder": NX * NY}
  xml = humanoid_with_sites()
  plain = mjcf.load_string(xml)
  rf = S.add_rangefinders(mjcf.load_string(xml), [(f"rf{i}_{j}", 0.0, 0, 0.0, 0.0, None) for i in range(NX) for j in range(NY)])
  assert io.rangefinder_tables(rf)["nrangefinder"] == NX * NY
  runs = {}
  for name, mjm in (("with", rf), ("without", plain)):
    m = mjw.put_model(mjm)
    runs[name] = (mjm, m, data(mjm, m, a.nworld))
  for name, (mjm, m, d) in runs.items():  # warm-up of every shape the timed windows use
    for _ in range(5):
      mjw.step(m, d)
      mjw.sensor_pos(m, d)
  torch.cuda.synchronize()

  # k_sensor_rangefinder's device time (profiler, a run of its own) and sensor_pos with / without the rows (events)
  mjm, m, d = runs["with"]
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(a.reps):
      mjw.sensor_pos(m, d)
    torch.cuda.synchronize()
  ev = [e for e in prof.key_averages() if "k_sensor_rangefinder" in e.key]
  assert ev, "k_sensor_rangefinder did not run"
  us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in ev) / sum(e.count for e in ev)
  res["k_sensor_rangefinder_us"] = round(us, 2)
  res["k_sensor_rangefinder_launches"] = int(sum(e.count for e in ev))
  res["rangefinder_rays_per_s"] = float(f"{a.nworld * NX * NY / (us * 1e-6):.4g}")
  res["sensor_pos_ms"] = {k: round(events(lambda: mjw.sensor_pos(v[1], v[2]), a.reps), 4) for k, v in runs.items()}

  # step with and without the rows, alternated
  step = {"with": [], "without": []}
  for _ in range(a.rounds):
    for k, (_, m_, d_) in runs.items():
      step[k].append(events(lambda: mjw.step(m_, d_), a.reps))
  res["step_ms"] = {k: dict(median=round(float(np.median(v)), 4), all=[round(x, 4) for x in v]) for k, v in step.items()}
  res["step_overhead_ms"] = round(float(np.median(step["with"]) - np.median(step["without"])), 4)

  # rays() on the same rays
  t = io.rangefinder_tables(mjm)
  site = torch.from_numpy(np.asarray(mjm.sensor_objid)[t["sensor_rangefinder_adr"]].astype(np.int64)).cuda()
  pnt = d.site_xpos[:, site].contiguous()
  vec = d.site_xmat.reshape(d.nworld, -1, 9)[:, site][..., [2, 5, 8]].contiguous()
  bx = torch.from_numpy(t["sensor_rangefinder_bodyid"]).cuda()
  n = NX * NY
  out = (torch.empty(d.nworld, n, device="cuda"), torch.empty(d.nworld, n, dtype=torch.int32, device="cuda"), torch.empty(d.nworld, n, 3, device="cuda"))
  for _ in range(5):
    mjw.rays(m, d, pnt, vec, None, True, bx, *out)
  res["rays_ms"] = round(events(lambda: mjw.rays(m, d, pnt, vec, None, True, bx, *out), a.reps), 4)
  mjw.sensor_pos(m, d)
  torch.cuda.synchronize()
  sd = d.sensordata[:, torch.from_numpy(np.asarray(mjm.sensor_adr)[t["sensor_rangefinder_adr"]].astype(np.int64)).cuda()]
  res["matches_rays_bitwise"] = bool(torch.equal(sd, out[0]))
  if not res["matches_rays_bitwise"]:
    bad = (sd != out[0]).nonzero()
    res["mismatch"] = dict(n=int(bad.shape[0]), max_abs=float((sd - out[0]).abs().max()),
                           first=[[int(w), int(r), float(sd[w, r]), float(out[0][w, r]), int(out[1][w, r])] for w, r in bad[:8].tolist()])
  res["hit_fraction"] = round(float((out[1] >= 0).float().mean()), 4)
  print(json.dumps(res))
  os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
  with open(a.out, "w") as f:
    json.dump(res, f, indent=1)


if __name__ == "__main__":
  main()
