"""Times k_sensor with and without the magnetometer / camprojection / insidesite / tendon limit / tendonactfrc sensors.

  python tools/sensor_extra_bench.py [--reps 50] [--warmup 10] [--prof 10] [--out profiles/sensor_extra_bench_h100.json]

Workloads, 8192 worlds each, every pair stepped alternately and each step timed with CUDA events; k_sensor's own time per step is the
sum of its kernel records in a torch.profiler trace of `--prof` steps, taken after the timed steps:
- humanoid: the benchmark humanoid (keyframe 0 with seeded noise; it has no sites and no tendons) with one sphere site at each body's
  frame, and per site a magnetometer, a camprojection into camera 0 and an insidesite (the body's xbody in the next body's site)
  against the same model with a jointpos sensor only (k_sensor's plain build);
- tendon: the arm / sled scene of tests/sensor_extra_scenes.py with all its new sensors (tendon limit pos / vel / frc and tendonactfrc
  on both tendons among them) against the same scene with a jointpos sensor only.
Writes one JSON object with the card name and its power limit, read in the same run.
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
from mujoco_warp_b200._src import mjcf  # noqa: E402
from mujoco_warp_b200.scenes import HUMANOID, WORKLOADS  # noqa: E402
from tests import sensor_extra_scenes as scenes  # noqa: E402
from tests import util  # noqa: E402

NWORLD = 8192


def _set_sensors(m, rows):
  """rows: (type, objtype, objid, reftype, refid, dim, stage)"""
  n = len(rows)
  col = lambda k: np.array([r[k] for r in rows], dtype=np.int32)
  m.nsensor = n
  m.names.sensor = [f"s{i}" for i in range(n)]
  m.sensor_type, m.sensor_objtype, m.sensor_objid, m.sensor_reftype, m.sensor_refid, m.sensor_dim, m.sensor_needstage = (col(k) for k in range(7))
  m.sensor_datatype = np.zeros(n, dtype=np.int32)
  m.sensor_intprm = np.zeros((n, 3), dtype=np.int32)
  m.sensor_cutoff, m.sensor_noise = np.zeros(n), np.zeros(n)
  m.sensor_adr = np.concatenate(([0], np.cumsum(m.sensor_dim)[:-1])).astype(np.int32)
  m.nsensordata = int(m.sensor_dim.sum())
  m.sensor_history = np.zeros((n, 2), dtype=np.int32)
  m.sensor_delay, m.sensor_interval = np.zeros(n), np.zeros((n, 2))
  m.sensor_unsupported = []
  return m


def humanoid(extra):
  m = mjcf.load_any(HUMANOID)
  assert m.nsensor == 0 and m.nsite == 0 and m.ncam > 0
  nb = int(m.nbody)
  m.nsite = nb - 1  # one site at each body's frame
  m.names.site = [f"site_{b}" for b in range(1, nb)]
  m.site_bodyid = np.arange(1, nb, dtype=np.int32)
  m.site_pos, m.site_quat = np.zeros((nb - 1, 3)), np.tile([1.0, 0.0, 0.0, 0.0], (nb - 1, 1))
  m.site_type, m.site_size = np.full(nb - 1, C.GEOM_SPHERE, dtype=np.int32), np.full((nb - 1, 3), 0.1)
  rows = [(C.SENS_JOINTPOS, C.OBJ_JOINT, 1, 0, -1, 1, 1)]
  if extra:
    for s in range(nb - 1):
      rows += [(C.SENS_MAGNETOMETER, C.OBJ_SITE, s, 0, -1, 3, 1), (C.SENS_CAMPROJECTION, C.OBJ_SITE, s, C.OBJ_CAMERA, 0, 2, 1),
               (C.SENS_INSIDESITE, C.OBJ_XBODY, s + 1, C.OBJ_SITE, (s + 1) % (nb - 1), 1, 1)]
  return _set_sensors(m, rows), dict(key=0, qpos_noise=0.02, qvel_noise=0.3), WORKLOADS["humanoid"]


def tendon(extra):
  return (scenes._load("Euler") if extra else scenes._load("Euler", ['<jointpos joint="j1"/>'], ())), dict(key=None, qpos_noise=0.1, qvel_noise=0.5), dict(nconmax=4, njmax=16)


def make(mjm, state, sizes):
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=NWORLD, m=m, nconmax=sizes["nconmax"], njmax=sizes["njmax"])
  qpos, qvel, _, _ = util.seeded_state(mjm, NWORLD, seed=11, **state)
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
    if e.device_type == torch.autograd.DeviceType.CUDA and "k_sensor" in e.name and "k_sensor_" not in e.name:  # either build of k_sensor
      tot["k_sensor"] = tot.get("k_sensor", 0.0) + e.device_time
  return {k: round(v / nstep, 2) for k, v in tot.items()}


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--reps", type=int, default=50)
  p.add_argument("--warmup", type=int, default=10)
  p.add_argument("--prof", type=int, default=10)
  p.add_argument("--out", default=os.path.join("profiles", "sensor_extra_bench_h100.json"))
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q, "nworld": NWORLD, "reps": a.reps}
  for wl, build in (("humanoid", humanoid), ("tendon", tendon)):
    runs = {"extra_sensors": make(*build(True)), "plain": make(*build(False))}
    for _ in range(a.warmup):
      for m, d in runs.values():
        mjw.step(m, d)
    ms = {k: [] for k in runs}
    for _ in range(a.reps):  # alternate, so that clock drift hits both alike
      for k, (m, d) in runs.items():
        ms[k].append(timed(lambda: mjw.step(m, d)))
    out = {}
    for k, (m, d) in runs.items():
      mjw.step(m, d)
      out[k] = dict(nsensor=int(m.nsensor), step_ms_median=round(float(np.median(ms[k])), 4), step_ms_p10=round(float(np.percentile(ms[k], 10)), 4),
                    step_ms_p90=round(float(np.percentile(ms[k], 90)), 4), launches=mjw.last_launch_count(), kernel_us_per_step=kernel_us(m, d, a.prof),
                    finite=bool(torch.isfinite(d.sensordata).all() and torch.isfinite(d.qpos).all()))
    out["step_ms_delta_median"] = round(out["extra_sensors"]["step_ms_median"] - out["plain"]["step_ms_median"], 4)
    res[wl] = out
    del runs
    torch.cuda.empty_cache()
  line = json.dumps(res)
  print(line)
  os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
  with open(a.out, "w") as f:
    f.write(line + "\n")


if __name__ == "__main__":
  main()
