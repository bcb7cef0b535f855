#!/usr/bin/env python
"""bench.py -- env-steps/sec of the batched physics step on humanoid.xml (BASELINE.json metric).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--nworld 8192]
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...

Workload (BASELINE.json configs[1], reference benchmarks/humanoid/__init__.py): humanoid, nworld=8192 per GPU, nconmax=24,
njmax=64, keyframe 0 (squat), Newton / pyramidal / Euler, deterministic Ornstein-Uhlenbeck ctrl noise (cli.py:103-145).
A "step" is one pass of the hot path (ctrl-noise kernel + mjb_step) over all worlds of the rank.  Weak scaling: every rank
owns its own 8192 worlds on its own GPU, no collective inside the step; the timed region is bracketed by barrier +
synchronize, timed with CUDA events, MAX over ranks.

One JSON line on stdout (rank 0).  See DESIGN.md "Measurement" for the roofline / algorithmic-bytes definitions.
"""

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from mujoco_warp_b200.scenes import WORKLOADS  # noqa: E402  (paths + sizes only; the package imports torch lazily)


def metric_name(wl):
  return "env-steps/sec (whole box) on humanoid.xml at nworld=8192 per GPU" if wl == "humanoid" else f"env-steps/sec (whole box) on {wl} at nworld={WORKLOADS[wl]['nworld']} per GPU"


def parse():
  p = argparse.ArgumentParser()
  p.add_argument("--gpus", type=int, default=1)
  p.add_argument("--steps", type=int, default=200)
  p.add_argument("--warmup", type=int, default=20)
  p.add_argument("--impl", default="ours", choices=["ours", "reference"])
  p.add_argument("--workload", default="humanoid", choices=sorted(WORKLOADS), help="BASELINE configs[1] (default), [2] g1, [3] convex_mesh stand-in, three_humanoids")
  p.add_argument("--nworld", type=int, default=None, help="worlds per GPU (default: the workload's)")
  p.add_argument("--no-graph", action="store_true", help="launch kernels directly instead of replaying a CUDA graph")
  p.add_argument("--cpu-sample-worlds", type=int, default=None)
  p.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg (kernel A/B sweeps)")
  p.add_argument("--dump-outputs", metavar="DIR", default=None,
                 help="write the last timed step's outputs (qpos, qvel, qacc, ...) to DIR/<field>.npy")
  a = p.parse_args()
  if a.steps < 1 or a.warmup < 0:
    p.error("--steps must be >= 1 and --warmup >= 0")
  if a.dump_outputs and a.impl != "ours":
    p.error("--dump-outputs writes the GPU arm's outputs; --impl reference has none")
  return a


def usable_cores() -> int:
  """Host cores this process may actually use: min(affinity mask, cgroup cpu quota)."""
  n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
  try:
    quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
    if quota != "max":
      n = min(n, max(1, int(int(quota) / int(period))))
  except Exception:
    pass
  return n


# --------------------------------------------------------------------------------------------- clocks


class ClockSampler:
  """Samples nvidia-smi clocks / throttle reasons during the timed region."""

  Q = "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

  def __init__(self, gpu_index):
    self.gpu, self.rows, self.proc = gpu_index, [], None

  def start(self):
    try:
      self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100"],
                                   stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
      self.t = threading.Thread(target=self._read, daemon=True)
      self.t.start()
    except Exception:
      self.proc = None

  def _read(self):
    for line in self.proc.stdout:
      self.rows.append([x.strip() for x in line.split(",")])

  def stop(self):
    if self.proc is None:
      return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
    self.proc.terminate()
    try:
      self.proc.wait(timeout=2)
    except Exception:
      self.proc.kill()
    sm = [float(r[1]) for r in self.rows if len(r) >= 9 and r[1].replace(".", "").isdigit()]
    mx = [float(r[2]) for r in self.rows if len(r) >= 9 and r[2].replace(".", "").isdigit()]
    reasons = set()
    names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
    for r in self.rows:
      if len(r) >= 9:
        for n, v in zip(names, r[5:9]):
          if v.lower().startswith("active"):
            reasons.add(n)
    return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons), "samples": len(sm)}


def gpu_info(gpu_index):
  """Name and power limit of the card the line was measured on (part of every absolute number it reports)."""
  try:
    out = subprocess.run(["nvidia-smi", f"--id={gpu_index}", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1])}
  except Exception:
    return {"name": None, "power_limit_w": None}


# --------------------------------------------------------------------------------------------- output dump

# What a caller of step(m, d) reads back: the advanced state, its accelerations and constraint forces, the solver's row count.
DUMP_FIELDS = ("qpos", "qvel", "act", "ctrl", "time", "qacc", "qacc_warmstart", "qfrc_constraint", "sensordata", "nefc", "solver_niter")
DUMP_LIMIT = 64 * 2**20


def collect_outputs(d, nworld):
  """DUMP_FIELDS as float32 (counters as float64); above DUMP_LIMIT a seeded sample of worlds, indices in `world_index`."""
  ts = {n: getattr(d, n) for n in DUMP_FIELDS if getattr(d, n).numel()}
  per_world = sum((t.numel() // nworld) * (4 if t.is_floating_point() else 8) for t in ts.values())
  out = {}
  if per_world * nworld > DUMP_LIMIT:
    idx = np.sort(np.random.default_rng(0).choice(nworld, size=DUMP_LIMIT // (per_world + 8), replace=False))
    out["world_index"] = idx.astype(np.float64)
    ts = {n: t[idx] for n, t in ts.items()}
  for n, t in ts.items():
    out[n] = t.cpu().numpy().astype(np.float32 if t.is_floating_point() else np.float64)
  return out


# --------------------------------------------------------------------------------------------- algorithmic bytes


def algorithmic_words(mjm, tabs, ncon_mean, nefc_mean, nv_pad):
  """Per-env-step algorithmic fp32/int32 words per kernel: every Data output written once, every input read once;
  Model constants and workspace count zero (SURVEY.md §8d)."""
  nq, nv, nu, nb, nj, ng = mjm.nq, mjm.nv, mjm.nu, mjm.nbody, mjm.njnt, mjm.ngeom
  ng_dyn = int((np.asarray(mjm.body_weldid)[np.asarray(mjm.geom_bodyid)] != 0).sum())
  nC, nJ, qld = tabs["nC"], tabs["nJmom"], tabs["qld_total"]
  w = {}
  w["position"] = nq + (3 + 4 + 9 + 3 + 9) * nb + 6 * nj + 12 * ng_dyn + 12 * mjm.nsite + 12 * mjm.ncam + 6 * mjm.nlight + (3 + 10) * nb + 6 * nv + 10 * nb + nC + 3 * nu + 2 * nJ
  w["collision"] = 12 * ng + 39 * ncon_mean + 2
  w["constraint"] = nq + nv + 6 * nv + 3 * nb + 39 * ncon_mean + nefc_mean * nv_pad + 8 * nefc_mean + 4 * ncon_mean + 4
  w["velocity"] = nv + 6 * nv + 10 * nb + nu + nC + 2 * nJ + nu + nu + 6 * nb + 6 * nv + 6 * nv + 12 * nb + nu + qld + nv + nv
  w["solver"] = nefc_mean * nv_pad + 3 * nefc_mean + nC + 2 * nv + 3 * nv + 2 * nefc_mean + 1
  w["integrate"] = nq + 2 * nv + nq + 2 * nv + 1
  return w


# --------------------------------------------------------------------------------------------- CPU arm (oracle)


def load_workload(name):
  """Model + initial host state + (optional) control trajectory of a workload."""
  from mujoco_warp_b200._src import io as mio
  from mujoco_warp_b200._src import mjcf
  from mujoco_warp_b200._src.mjcf import MjDataLite, reset_data_keyframe

  wl = WORKLOADS[name]
  mjm = mjcf.load_any(wl["model"])
  mjd = MjDataLite(mjm)
  ctrls = None
  if wl["replay"]:
    ctrls = mio.load_trajectory(wl["replay"], mjm, mjd)
  elif mjm.nkey > 0:
    reset_data_keyframe(mjm, mjd, 0)
  return wl, mjm, mjd, ctrls


def ctrl_noise_np(mjm, ctrl, step, center, noise_std=0.01, noise_rate=0.1):
  """numpy restatement of the harness control noise (reference cli.py:103-145; the GPU arm's k_ctrl_noise): per (world, actuator)
  ctrl <- rate ctrl + (1 - rate) centre + scale halfrange (2 halton((step + 1)(world + 1), actuator + 2) - 1), clipped to ctrlrange."""
  nworld, nu = ctrl.shape
  rate = np.exp(-float(mjm.opt.timestep) / noise_rate)
  scale = noise_std * np.sqrt(1.0 - rate * rate)
  limited = np.asarray(mjm.actuator_ctrllimited).astype(bool)
  lo, hi = np.asarray(mjm.actuator_ctrlrange)[:, 0], np.asarray(mjm.actuator_ctrlrange)[:, 1]
  halfrange = np.where(limited, 0.5 * (hi - lo), 1.0)
  n = np.tile(((step + 1) * (np.arange(nworld, dtype=np.int64) + 1))[:, None], (1, nu))
  base = (np.arange(nu, dtype=np.int64) + 2)[None, :]
  f = 1.0 / base
  h = np.zeros((nworld, nu))
  while (n > 0).any():  # radical inverse, all (world, actuator) pairs at once
    h += f * (n % base)
    n //= base
    f = f / base
  out = rate * ctrl + (1.0 - rate) * center[None, :] + scale * halfrange[None, :] * (2.0 * h - 1.0)
  return np.where(limited[None, :], np.clip(out, lo[None, :], hi[None, :]), out)


def cpu_run(name, nworld, nsteps, nthreads):
  """Times the CPU restatement (oracle, fp64, OpenMP over worlds) on a bounded sample; returns env-steps/s."""
  from tests import util
  from oracle import orc  # noqa: F401  (bench.py's cpu_baseline / --impl reference legs are allowed to use the oracle)

  wl, mjm, mjd, ctrls = load_workload(name)
  o = util.make_oracle(mjm, nworld, wl["nconmax"], wl["njmax"])
  o.set_state(qpos=np.asarray(mjd.qpos), qvel=np.asarray(mjd.qvel), ctrl=np.asarray(mjd.ctrl))
  center = np.asarray(mjd.ctrl, dtype=np.float64)
  o.step(nthreads)
  t0 = time.perf_counter()
  for i in range(nsteps):
    if ctrls is not None:
      o.d["ctrl"][:] = ctrls[i % len(ctrls)]
    elif mjm.nu:  # the same control process as the GPU arm: OU noise around the keyframe controls, Halton sequence (cli.py:103-145)
      o.d["ctrl"][:] = ctrl_noise_np(mjm, o.d["ctrl"], i, center)
    o.step(nthreads)
  dt = time.perf_counter() - t0
  return nworld * nsteps / dt, dt


def run_reference(args):
  """--impl reference: the reference's algorithm on the box's host cores.  The reference itself (Warp + mujoco) cannot be
  installed here (no wheels, no network: DESIGN.md), so this arm times the CPU restatement in oracle/ (kind = "port")."""
  rank = int(os.environ.get("RANK", "0"))
  if rank != 0:
    return
  wl = WORKLOADS[args.workload]
  nworld = args.nworld or wl["nworld"]
  cores = usable_cores()
  nw = args.cpu_sample_worlds or nworld
  for _ in range(max(1, min(args.warmup, 3))):
    cpu_run(args.workload, nw, 1, cores)
  rate, dt = cpu_run(args.workload, nw, args.steps, cores)
  sample = f"{nw} worlds x {args.steps} steps of the oracle (fp64 C, OpenMP {cores} threads) per run"
  line = {
    "impl": "reference", "metric": metric_name(args.workload), "value": rate, "unit": "env-steps/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
    "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
    "config": {"workload": f"{wl['label']}; CPU sample of {nw} worlds per step (bounded sample of nworld={nworld}/GPU), same OU / Halton ctrl noise as the GPU arm" if not wl["replay"] else f"{wl['label']}; CPU sample of {nw} worlds per step"},
    "cpu_baseline": {"value": rate, "unit": "env-steps/s", "cores": cores, "kind": "port", "sample": sample},
    "e2e": {"value": rate, "unit": "env-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    "gpu_launches": 0,
  }
  print(json.dumps(line))


# --------------------------------------------------------------------------------------------- GPU arm

HBM_PEAK_GBS = 3350.0  # H100 SXM data sheet (HBM3); the roofline's denominator


def run_ours(args):
  import torch

  torch.set_num_threads(max(1, min(4, usable_cores())))  # host-side tensor ops in the e2e loop stay within the cpu quota
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import io as mio

  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local = int(os.environ.get("LOCAL_RANK", "0"))
  torch.cuda.set_device(local)
  dist = None
  if world > 1:
    import torch.distributed as dist

    dist.init_process_group("nccl", device_id=torch.device("cuda", local))

  def barrier():
    if dist is not None:
      dist.barrier()
    torch.cuda.synchronize()

  wl, mjm, mjd, ctrls = load_workload(args.workload)
  tabs = mio.derive_tables(mjm)
  m = mjw.put_model(mjm)
  nworld = args.nworld or wl["nworld"]
  NCONMAX, NJMAX = wl["nconmax"], wl["njmax"]
  d = mjw.put_data(mjm, mjd, nworld=nworld, nconmax=NCONMAX, njmax=NJMAX, m=m)
  center = torch.from_numpy(np.asarray(mjd.ctrl, dtype=np.float32)).cuda()
  traj = torch.from_numpy(np.asarray(ctrls, dtype=np.float32)).cuda() if ctrls is not None else None  # (nstep, nu), device resident
  data_mb = sum(t.numel() * t.element_size() for o in (d, d.efc, d.contact) for t in vars(o).values() if isinstance(t, torch.Tensor)) / 2**20
  # timing rule: a per-step working set that fits the L2 (50 MB on an H100) is flushed between timed steps (each step then gets its own event pair)
  l2_mb = torch.cuda.get_device_properties(local).L2_cache_size / 2**20
  flush = torch.empty(256 * 2**20 // 4, dtype=torch.float32, device="cuda") if data_mb <= l2_mb else None
  # ranks use shifted Halton step indices so their noise streams differ
  world_offset = rank * nworld

  stream = torch.cuda.Stream()
  graph = None
  step_idx = [0]
  initial = {n: getattr(d, n).clone() for n in ("qpos", "qvel", "ctrl", "qacc_warmstart", "time", "qacc")}

  def set_ctrl():
    if traj is not None:  # trajectory replay, zero-order hold (cli.py:154-158): every world gets the step's control row
      d.ctrl.copy_(traj[step_idx[0] % traj.shape[0]].unsqueeze(0).expand(nworld, -1))
    elif mjm.nu:
      mjw.ctrl_noise(m, d, step_idx[0] + world_offset, center)

  def one_step():
    set_ctrl()
    if graph is not None:
      graph.replay()
    else:
      mjw.step(m, d)
    step_idx[0] += 1

  with torch.cuda.stream(stream):
    for _ in range(3):
      one_step()
    stream.synchronize()
    launches_per_step = 1 + mjw.last_launch_count()
    if not args.no_graph:
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g, stream=stream):
        mjw.step(m, d)
      graph = g
    # The simulated state inside the timed window is deterministic: the state is put back to the keyframe after graph capture,
    # advanced by exactly `warmup` steps, snapshotted, and restored right before the timed region.  nvidia-smi needs a few hundred
    # ms before its first row, so the same load keeps running (on the live state) until it reports; those extra steps are undone
    # by the restore.
    def snapshot():
      return {n: getattr(d, n).clone() for n in ("qpos", "qvel", "ctrl", "qacc_warmstart", "time", "qacc")}

    def restore(snap):
      for n, v in snap.items():
        getattr(d, n).copy_(v)

    restore(initial)
    step_idx[0] = 0
    sampler = ClockSampler(local)
    if rank == 0:
      sampler.start()
    for _ in range(args.warmup):
      one_step()
    stream.synchronize()
    snap, snap_idx = snapshot(), step_idx[0]
    t_wait = time.perf_counter() + 3.0
    while rank == 0 and sampler.proc is not None and len(sampler.rows) < 1 and time.perf_counter() < t_wait:
      one_step()
      stream.synchronize()
    restore(snap)
    step_idx[0] = snap_idx
    sim_steps_before_timed = snap_idx

    # ---- timed region: K steps, device-resident inputs, CUDA events on the launching stream
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if flush is None:
      e0.record(stream)
      for _ in range(args.steps):
        one_step()
      e1.record(stream)
      stream.synchronize()
      ms = e0.elapsed_time(e1)
    else:
      evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
      for a, b in evs:
        flush.fill_(0.0)
        a.record(stream)
        one_step()
        b.record(stream)
      stream.synchronize()
      ms = sum(a.elapsed_time(b) for a, b in evs)
    barrier()
    outputs = collect_outputs(d, nworld) if args.dump_outputs and rank == 0 else None
    # ---- statistics of the run (untimed), taken from the last timed step
    ncon_mean = float(d.nacon.cpu()[0]) / nworld
    nefc_mean = float(d.nefc.float().mean().cpu())
    niter_mean = float(d.solver_niter.float().mean().cpu())
    niter_hist = torch.bincount(d.solver_niter.clamp(0, 4).long().cpu(), minlength=5).tolist()  # worlds with 0, 1, 2, 3, >= 4 Newton iterations
    ovf = int((d.overflow != 0).sum().cpu())
    ovf_bits = int(np.bitwise_or.reduce(d.overflow.cpu().numpy().astype(np.int64))) if nworld else 0
    nan_worlds = int(torch.isnan(d.qpos).any(dim=1).sum().cpu())
    n_rows, t_wait = len(sampler.rows), time.perf_counter() + 1.0
    while rank == 0 and sampler.proc is not None and len(sampler.rows) <= n_rows and time.perf_counter() < t_wait:
      one_step()  # same load, untimed, until one more 100 ms sample lands after the timed region
      stream.synchronize()
    clocks = sampler.stop() if rank == 0 else None
    restore(snap)  # the per-kernel pass and the e2e loop below start from the same state as the timed region
    step_idx[0] = snap_idx

    # ---- per-kernel durations (separate pass with event pairs around each kernel)
    nprof = 20
    acc = None
    for _ in range(nprof):
      set_ctrl()
      step_idx[0] += 1
      r = mjw.step_profile(m, d)
      acc = r if acc is None else {k: acc[k] + r[k] for k in r}
    kms = {k: v / nprof for k, v in acc.items()}

    # ---- e2e: same metric through the public API with HOST buffers: every step's controls come from pinned host memory (H2D) and
    # every step's qpos + qvel go back to pinned host memory (D2H), all inside the timed region.  The loop is software-pipelined one
    # step deep, as an asynchronous actor would run it: the two copy engines work on their own streams (upload of step k + 1's
    # controls and download of step k - 1's state overlap the kernels of step k; small device-to-device copies decouple the buffers
    # the step graph reads / writes from the ones in flight), and the host consumes the read-back of step k - 1 (event wait, not a
    # stream sync) to produce the controls of step k + 1.
    nbuf, nq_, nv_ = 2, mjm.nq, mjm.nv
    ctrl_host = [torch.empty((nworld, mjm.nu), dtype=torch.float32).pin_memory() for _ in range(nbuf)]
    state_host = [torch.empty((nworld, nq_ + nv_), dtype=torch.float32).pin_memory() for _ in range(nbuf)]
    ctrl_dev = [torch.empty_like(d.ctrl) for _ in range(nbuf)]
    state_dev = [torch.empty((nworld, nq_ + nv_), dtype=torch.float32, device="cuda") for _ in range(nbuf)]
    h2d_done, ctrl_used, snap_done, d2h_done = ([torch.cuda.Event() for _ in range(nbuf)] for _ in range(4))
    s_in, s_out = torch.cuda.Stream(), torch.cuda.Stream()
    for c in ctrl_host:
      c.copy_(d.ctrl.cpu())
    e2e_steps = max(10, args.steps // 2)

    def upload(b):
      with torch.cuda.stream(s_in):
        s_in.wait_event(ctrl_used[b])
        ctrl_dev[b].copy_(ctrl_host[b], non_blocking=True)
        h2d_done[b].record(s_in)

    stream.synchronize()
    barrier()
    t0 = time.perf_counter()
    upload(0)
    tr = [0.0] * 5 if os.environ.get('MJB_E2E_TRACE') else None
    for i in range(e2e_steps):
      b = i % nbuf
      ta = time.perf_counter()
      stream.wait_event(h2d_done[b])
      if mjm.nu:
        d.ctrl.copy_(ctrl_dev[b], non_blocking=True)
      ctrl_used[b].record(stream)
      if graph is not None:
        graph.replay()
      else:
        mjw.step(m, d)
      stream.wait_event(d2h_done[b])  # the download that last read state_dev[b] (step i - 2)
      state_dev[b][:, :nq_].copy_(d.qpos, non_blocking=True)
      state_dev[b][:, nq_:].copy_(d.qvel, non_blocking=True)
      snap_done[b].record(stream)
      with torch.cuda.stream(s_out):
        s_out.wait_event(snap_done[b])
        state_host[b].copy_(state_dev[b], non_blocking=True)
        d2h_done[b].record(s_out)
      tb = time.perf_counter()
      p = (i + 1) % nbuf
      if i > 0:  # host-side policy stand-in on the PREVIOUS step's read-back, while this step runs on the GPU
        d2h_done[p].synchronize()
        tc = time.perf_counter()
        ctrl_host[p].add_(0.001 * float(state_host[p][0, 2])).clamp_(-1, 1)
      else:
        tc = tb
      td = time.perf_counter()
      upload(p)  # controls of step i + 1
      if tr is not None:
        te = time.perf_counter()
        for k, v in enumerate((tb - ta, tc - tb, td - tc, te - td)):
          tr[k] += v
    for e in d2h_done:
      e.synchronize()
    if tr is not None:
      print('e2e host us/step: launch %.1f wait %.1f policy %.1f upload %.1f' % tuple(1e6 * v / e2e_steps for v in tr[:4]), file=sys.stderr)
    stream.synchronize()
    e2e_s = time.perf_counter() - t0
    barrier()

  from mujoco_warp_b200._src import shard  # the measurement path's only collectives: MAX over ranks of the device-timed durations

  ms_max, e2e_ms_max = shard.reduce_max_elapsed(ms, dist), shard.reduce_max_elapsed(e2e_s * 1e3, dist)
  total_worlds = nworld * world
  value = shard.whole_job_rate(nworld * args.steps, ms_max * 1e-3, world)
  e2e_value = shard.whole_job_rate(nworld * e2e_steps, e2e_ms_max * 1e-3, world)

  if rank == 0:
    if outputs is not None:
      os.makedirs(args.dump_outputs, exist_ok=True)
      for n, v in outputs.items():
        np.save(os.path.join(args.dump_outputs, n + ".npy"), v)
    peak = HBM_PEAK_GBS
    words = algorithmic_words(mjm, tabs, ncon_mean, nefc_mean, m.nv_pad)
    top = max(kms, key=kms.get)
    bytes_launch = 4.0 * words[top] * nworld
    achieved = bytes_launch / (kms[top] * 1e-3) / 1e9
    step_bytes = 4.0 * sum(words.values()) * nworld
    cpu = None
    if world == 1 and not args.no_cpu:  # reported baseline, rank 0 at N = 1 only: a bounded sample of the same workload on the host cores
      cores = usable_cores()
      cpu_steps = 50
      nws = args.cpu_sample_worlds or nworld
      rate, dt = cpu_run(args.workload, nws, cpu_steps, cores)
      cpu = {"value": rate, "unit": "env-steps/s", "cores": cores, "kind": "port",
             "sample": f"{nws} worlds x {cpu_steps} steps of the fp64 C oracle (OpenMP {cores} threads), {dt:.1f} s wall"}
    line = {
      "metric": metric_name(args.workload), "value": value, "unit": "env-steps/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
      "ms_per_step": ms_max / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": value / 2729192.0 if args.workload == "humanoid" else None,
      "dtype": "f32", "data": "synthetic",
      "config": {
        "workload": wl["label"] if nworld == wl["nworld"] else wl["label"].replace(f"nworld={wl['nworld']}", f"nworld={nworld}"),
        "cuda_graph": graph is not None, "l2": f"per-step Data working set ({data_mb:.0f} MB of Data tensors at {nworld} worlds) exceeds the {l2_mb:.0f} MB L2; no explicit flush" if flush is None else f"Data tensors are {data_mb:.0f} MB (<= {l2_mb:.0f} MB L2): 256 MB scratch buffer written between timed steps",
        "vs_baseline_note": "2,729,192 steps/s is the reference's only published number (benchmarks/README.md:48), hardware unstated",
        "sim_steps_before_timed": sim_steps_before_timed, "ncon_mean": ncon_mean, "nefc_mean": nefc_mean, "solver_niter_mean": niter_mean, "solver_niter_hist_0_1_2_3_4plus": niter_hist, "overflow_worlds": ovf, "overflow_bits_or": hex(ovf_bits), "nan_worlds": nan_worlds,
      },
      "e2e": {"value": e2e_value, "unit": "env-steps/s", "h2d_bytes_per_step": int(nworld * mjm.nu * 4), "d2h_bytes_per_step": int(nworld * (mjm.nq + mjm.nv) * 4), "steps": e2e_steps,
              "pipeline": "one step deep: host consumes step k-1 while the GPU runs step k; H2D / D2H on their own streams (two pinned buffer sets, event waits)"},
      "gpu_launches": launches_per_step * args.steps,
      "kernel_ms": kms,
      "roofline": {"bound": "hbm", "kernel": "k_" + top, "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                   "peak_source": "H100 SXM data sheet, 3.35 TB/s HBM3 (not a measured peak)",
                   "algorithmic_bytes_per_launch": bytes_launch, "step_algorithmic_bytes": step_bytes,
                   "step_frac": step_bytes / (ms_max / args.steps * 1e-3) / 1e9 / peak},
      "cpu_baseline": cpu,
      "clocks": clocks,
      "device": gpu_info(local),
    }
    print(json.dumps(line))
  if dist is not None:
    dist.destroy_process_group()


if __name__ == "__main__":
  a = parse()
  if a.impl == "reference":
    run_reference(a)
  else:
    run_ours(a)
