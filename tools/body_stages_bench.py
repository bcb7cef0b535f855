"""Times step alone and step followed by each of rne_postconstraint, subtree_vel, jac, xfrc_accumulate and deriv_smooth_vel.

  python tools/body_stages_bench.py [--reps 50] [--warmup 10] [--prof 10] [--out profiles/body_stages_bench_h100.json]

Workloads: the benchmark humanoid and G1, 8192 worlds each, from seeded states with non-zero xfrc_applied on every body.  The six variants
alternate in one run after warm-up, each timed with CUDA events; each new kernel's own time is the mean of its records in a
torch.profiler trace of `--prof` calls.  jac asks for one body per world (the last body) and writes jacp and jacr.  For scale, each
kernel's record carries the bytes it must at least write, the write rate that implies, and whether the kernel is memory- or latency-bound:
memory-bound when that rate reaches a quarter of the card's DRAM bandwidth (HBM_GBPS; the kernel's reads of the same order come on top),
latency-bound otherwise (a warp walks a world's tree level by level, or a thread its dof's bodies, and the memory system idles).
`--bench-ab DIR` records the humanoid rate of alternating `bench.py` runs of the parent build and this one, read from the last JSON line of
DIR/bench_parent_<k>.log and DIR/bench_new_<k>.log.  Writes one JSON object with the card name and power limit, read in the same run.
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
from mujoco_warp_b200._src import mjcf  # noqa: E402
from mujoco_warp_b200.scenes import G1, HUMANOID  # noqa: E402
from tests import util  # noqa: E402

NWORLD = 8192
HBM_GBPS = 3350.0  # H100 SXM5 80 GB HBM3, NVIDIA's data sheet


def make(path, nconmax, njmax):
  mjm = mjcf.load_any(path)
  m = mjw.put_model(mjm)
  d = mjw.make_data(mjm, nworld=NWORLD, m=m, nconmax=nconmax, njmax=njmax)
  qpos, qvel, _, _ = util.seeded_state(mjm, NWORLD, seed=11, qpos_noise=0.02, qvel_noise=0.3)
  d.qpos.copy_(torch.from_numpy(qpos.astype(np.float32)))
  d.qvel.copy_(torch.from_numpy(qvel.astype(np.float32)))
  d.xfrc_applied[:, 1:, :] = 0.1
  torch.cuda.synchronize()
  return mjm, m, d


def timed(fn):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def kernel_us(fn, name, n):
  from torch.profiler import ProfilerActivity, profile

  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(n):
      fn()
    torch.cuda.synchronize()
  t = [e.device_time for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and name in e.name]
  return round(sum(t) / n, 2) if t else None


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--reps", type=int, default=50)
  p.add_argument("--warmup", type=int, default=10)
  p.add_argument("--prof", type=int, default=10)
  p.add_argument("--out", default=os.path.join("profiles", "body_stages_bench_h100.json"))
  p.add_argument("--bench-ab", default=None, metavar="DIR", help="record alternating bench.py runs of the parent and this build from DIR")
  a = p.parse_args()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ""
  res = {"gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit": q, "nworld": NWORLD, "reps": a.reps}
  for wl, path, nconmax, njmax in (("humanoid", HUMANOID, 24, 64), ("g1", G1, 48, 192)):
    mjm, m, d = make(path, nconmax, njmax)
    nv, nb = mjm.nv, mjm.nbody
    point = d.xipos[:, nb - 1].contiguous()
    body = torch.full((NWORLD,), nb - 1, dtype=torch.int32, device="cuda")
    jacp, jacr = torch.zeros((NWORLD, 3, nv), device="cuda"), torch.zeros((NWORLD, 3, nv), device="cuda")
    qfrc, deriv = torch.zeros((NWORLD, nv), device="cuda"), torch.zeros((NWORLD, m.nC), device="cuda")
    calls = {
      "rne_postconstraint": (lambda: mjw.rne_postconstraint(m, d), "k_rne_postconstraint", 4 * NWORLD * 18 * nb),
      "subtree_vel": (lambda: mjw.subtree_vel(m, d), "k_subtree_vel", 4 * NWORLD * 6 * nb),
      "jac": (lambda: mjw.jac(m, d, jacp, jacr, point, body), "k_jac", 4 * NWORLD * 6 * nv),
      "xfrc_accumulate": (lambda: mjw.xfrc_accumulate(m, d, qfrc), "k_xfrc_accumulate", 4 * NWORLD * 2 * nv),
      "deriv_smooth_vel": (lambda: mjw.deriv_smooth_vel(m, d, deriv), "k_deriv_smooth_vel", 4 * NWORLD * m.nC),
    }
    variants = {"step": lambda: mjw.step(m, d)}
    for k, (fn, _, _) in calls.items():
      variants["step+" + k] = (lambda f: (lambda: (mjw.step(m, d), f())))(fn)
    for _ in range(a.warmup):
      for v in variants.values():
        v()
    ms = {k: [] for k in variants}
    for _ in range(a.reps):  # alternate, so that clock drift hits every variant alike
      for k, v in variants.items():
        ms[k].append(timed(v))
    out = {"nv": nv, "nbody": nb, "nC": int(m.nC)}
    for k in variants:
      out[k] = dict(ms_median=round(float(np.median(ms[k])), 4), ms_p10=round(float(np.percentile(ms[k], 10)), 4), ms_p90=round(float(np.percentile(ms[k], 90)), 4))
    for k, (fn, kname, nbytes) in calls.items():
      us = kernel_us(fn, kname, a.prof)
      gbps = round(nbytes / (us * 1e3), 1) if us else None
      out[k + "_kernel"] = dict(us=us, min_write_bytes=nbytes, write_gbps=gbps,
                                bound=None if gbps is None else ("memory" if gbps >= 0.25 * HBM_GBPS else "latency"))
    out["finite"] = bool(all(torch.isfinite(t).all() for t in (jacp, jacr, qfrc, deriv, d.cfrc_ext, d.qpos)))
    res[wl] = out
    del m, d, jacp, jacr, qfrc, deriv
    torch.cuda.empty_cache()
  if a.bench_ab:
    rates = {}
    for build in ("parent", "new"):
      k = 1
      while os.path.exists(os.path.join(a.bench_ab, f"bench_{build}_{k}.log")):
        last = [ln for ln in open(os.path.join(a.bench_ab, f"bench_{build}_{k}.log")) if ln.startswith("{")][-1]
        rates.setdefault(build, []).append(round(json.loads(last)["value"] / 1e6, 3))
        k += 1
    res["bench_py_humanoid_Menv_steps_s_alternating"] = {"parent": rates.get("parent"), "change": rates.get("new")}
  line = json.dumps(res)
  print(line)
  os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
  with open(a.out, "w") as f:
    f.write(line + "\n")


if __name__ == "__main__":
  main()
