"""mjwarp-testspeed compatible benchmark CLI for the H100 step path.

  python -m mujoco_warp_b200.testspeed <model.xml|model.npz> --nworld 8192 --nconmax 24 --njmax 64 [--nstep 1000]
      [--keyframe 0] [--replay traj.npz] [--function step] [--format human|short|json] [--event_trace]
      [--ctrl_noise_std 0.01 --ctrl_noise_rate 0.1] [--measure_solver] [--measure_alloc] [--memory]

Mirrors /root/reference/mujoco_warp/testspeed.py:140-378 and _src/cli.py:34-297: the same flag names, the same timed
region (one CUDA-graph replay of `fn(m, d)` + device sync per step, measured with time.perf_counter; the ctrl-noise kernel
and the host callback are untimed), and the same output keys (`jit_duration`, `run_time`, `steps_per_second`,
`converged_worlds`, `*_memory`, `ncon_mean/p95`, `nefc_mean/p95`, `solver_niter_mean/p95`, flattened event trace in
ns / env-step), so `benchmarks/run.py` can parse it unchanged.
"""

from __future__ import annotations

import argparse
import inspect
import json
import sys
import time

import numpy as np


def _parse(argv):
  p = argparse.ArgumentParser(prog="mjwarp-b200-testspeed")
  p.add_argument("mjcf")
  p.add_argument("--function", default="step")
  p.add_argument("--nworld", type=int, default=8192)
  p.add_argument("--nstep", type=int, default=None)
  p.add_argument("--nconmax", type=int, default=None)
  p.add_argument("--njmax", type=int, default=None)
  p.add_argument("--keyframe", type=int, default=0)
  p.add_argument("--replay", default=None)
  p.add_argument("--ctrl_noise_std", type=float, default=0.01)
  p.add_argument("--ctrl_noise_rate", type=float, default=0.1)
  p.add_argument("--format", default="human", choices=["human", "short", "json"])
  p.add_argument("--event_trace", nargs="?", const="true", default="false")
  p.add_argument("--measure_solver", nargs="?", const="true", default="false")
  p.add_argument("--measure_alloc", nargs="?", const="true", default="false")
  p.add_argument("--memory", nargs="?", const="true", default="false")
  p.add_argument("--device", default="cuda:0")
  p.add_argument("-o", "--override", action="append", default=[], help='model overrides, e.g. -o "opt.iterations = 10" (reference io.py:2933)')
  a = p.parse_args(argv)
  for k in ("event_trace", "measure_solver", "measure_alloc", "memory"):
    setattr(a, k, str(getattr(a, k)).lower() in ("1", "true", "yes"))
  return a


def _memory(obj) -> int:
  import torch

  tot = 0
  for v in vars(obj).values():
    if isinstance(v, torch.Tensor):
      tot += v.numel() * v.element_size()
    elif hasattr(v, "__dict__") and not isinstance(v, type) and type(v).__name__ in ("Contact", "Constraint", "Option", "Statistic"):
      tot += _memory(v)
    elif isinstance(v, (tuple, list)):
      tot += sum(t.numel() * t.element_size() for t in v if isinstance(t, torch.Tensor))
  return tot


def main(argv=None):
  a = _parse(sys.argv[1:] if argv is None else argv)
  import torch

  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src.mjcf import MjDataLite, reset_data_keyframe

  if not torch.cuda.is_available():
    raise ValueError("testspeed available for gpu only")  # same refusal as the reference (testspeed.py:153-154)
  torch.cuda.set_device(torch.device(a.device))
  funcs = {n: f for n, f in inspect.getmembers(mjw, inspect.isfunction) if list(inspect.signature(f).parameters) == ["m", "d"]}
  if a.function not in funcs:
    raise ValueError(f"Unknown function: {a.function} (available: {sorted(funcs)})")
  fn = funcs[a.function]

  if a.format == "human":
    print(f"Loading model from: {a.mjcf}...\n")
  mjm = mjw.mjcf.load_any(a.mjcf)
  mjd = MjDataLite(mjm)
  ctrls = None
  if a.replay:
    ctrls = mjw.load_trajectory(a.replay, mjm, mjd)
    if a.nstep is None:
      a.nstep = len(ctrls)
  elif mjm.nkey > 0 and a.keyframe > -1:
    reset_data_keyframe(mjm, mjd, a.keyframe)
  if a.nstep is None:
    a.nstep = 1000
  free0 = torch.cuda.mem_get_info()[0]
  mjw.override_model(mjm, a.override)
  m = mjw.put_model(mjm)
  mjw.override_model(m, a.override)
  d = mjw.put_data(mjm, mjd, nworld=a.nworld, nconmax=a.nconmax, njmax=a.njmax, m=m)
  timestep = float(m.opt.timestep.cpu()[0])
  if a.format == "human":
    print("Model\n  " + " ".join(f"{f}: {getattr(m, f)}" for f in ("nq", "nv", "nu", "nbody", "ngeom")))
    print(f"Option\n  integrator: {m.opt.integrator} cone: {m.opt.cone} solver: {m.opt.solver} iterations: {m.opt.iterations} ls_iterations: {m.opt.ls_iterations}")
    print(f"Data\n  nworld: {d.nworld} naconmax: {d.naconmax} njmax: {d.njmax}\n")
    print(f"Rolling out {a.nstep} steps at dt = {timestep:g}...")

  center = torch.from_numpy(np.asarray(mjd.ctrl, dtype=np.float32)).cuda()
  # "JIT" = build/load of the sm_90a library + CUDA-graph capture of fn(m, d)
  t0 = time.perf_counter()
  stream = torch.cuda.Stream()
  with torch.cuda.stream(stream):
    fn(m, d)  # warm-up launch (configures dynamic shared memory) before capture
    stream.synchronize()
    # undo the warm-up step's state change so the rollout starts from the requested state
    d2 = mjw.put_data(mjm, mjd, nworld=a.nworld, nconmax=a.nconmax, njmax=a.njmax, m=m)
    for name in ("qpos", "qvel", "ctrl", "qacc_warmstart", "time"):
      getattr(d, name).copy_(getattr(d2, name))
    del d2
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
      fn(m, d)
    stream.synchronize()
    jit_duration = time.perf_counter() - t0

    run_time = 0.0
    nacon, nefc, niter = [], [], []
    trace = {}
    for i in range(a.nstep):
      if ctrls is not None:
        d.ctrl.copy_(torch.from_numpy(np.tile(ctrls[i].astype(np.float32), (a.nworld, 1))))
      elif a.ctrl_noise_std > 0 and m.nu > 0:
        mjw.ctrl_noise(m, d, i, center, a.ctrl_noise_std, a.ctrl_noise_rate)
      stream.synchronize()
      t1 = time.perf_counter()
      graph.replay()
      stream.synchronize()
      run_time += time.perf_counter() - t1
      nacon.append(int(d.nacon.cpu()[0]))
      nefc.append(float(d.nefc.float().mean().cpu()))
      niter.append(float(d.solver_niter.float().mean().cpu()))
    if a.event_trace and a.function == "step":
      # the reference's nested stage keys (warp_util.py:51-145, testspeed.py:75-89), from stage-wise steps (see _src/trace.py)
      acc = None
      ntrace = 10
      for i in range(ntrace):
        fl = mjw.flatten_trace(mjw.event_trace_step(m, d), scale=1e6 / a.nworld)  # ms -> ns per env-step
        acc = fl if acc is None else {k: acc[k] + fl[k] for k in fl}
      trace = {k: v / ntrace for k, v in acc.items()}
      # the fused production step for comparison (kernels of mjb_step timed one by one)
      accp = None
      for i in range(20):
        r = mjw.step_profile(m, d)
        accp = r if accp is None else {k: accp[k] + r[k] for k in r}
      trace.update({f"fused.{k}": 1e6 * v / 20 / a.nworld for k, v in accp.items()})

  nconverged = int((~torch.isnan(d.qpos).any(dim=1)).sum().cpu())
  steps = a.nworld * a.nstep
  model_mem, data_mem = _memory(m), _memory(d)
  total_mem = free0 - torch.cuda.mem_get_info()[0]
  metrics = {
    "jit_duration": jit_duration, "run_time": run_time, "steps_per_second": steps / run_time, "converged_worlds": nconverged,
    "model_memory": model_mem, "data_memory": data_mem, "total_memory": total_mem,
    "ncon_mean": float(np.mean(nacon)) / a.nworld, "ncon_p95": float(np.percentile(nacon, 95)) / a.nworld,
    "nefc_mean": float(np.mean(nefc)), "nefc_p95": float(np.percentile(nefc, 95)),
    "solver_niter_mean": float(np.mean(niter)), "solver_niter_p95": float(np.percentile(niter, 95)),
  }
  if a.format == "human":
    print(f"""
Summary for {d.nworld} parallel rollouts

Total JIT time: {jit_duration:.2f} s
Total simulation time: {run_time:.2f} s
Total steps per second: {steps / run_time:,.0f}
Total realtime factor: {steps * timestep / run_time:,.2f} x
Total time per step: {1e9 * run_time / steps:.2f} ns
Total converged worlds: {nconverged} / {d.nworld}""")
    if trace:
      print("\nEvent trace (ns / env-step):\n")
      for k, v in trace.items():
        print(f"{'  ' * k.count('.')}{k.split('.')[-1]}: {v:.2f}")
    if a.measure_alloc:
      print(f"\nnacon alloc mean {np.mean(nacon):.1f} max {np.max(nacon)} / naconmax {d.naconmax};  nefc mean {np.mean(nefc):.2f} / njmax {d.njmax}")
    if a.measure_solver:
      print(f"solver niter mean {np.mean(niter):.3f} p95 {np.percentile(niter, 95):.3f}")
    if a.memory:
      print(f"Model memory {model_mem / 2**20:.2f} MiB, Data memory {data_mem / 2**20:.2f} MiB, total {total_mem / 2**20:.2f} MiB")
    ovf = int((d.overflow != 0).sum().cpu())
    if ovf:
      print(f"overflow flags set in {ovf} worlds: 0x{int(torch.bitwise_or(d.overflow, torch.zeros_like(d.overflow)).max().cpu()):x}")
  elif a.format == "short":
    for k, v in (metrics | trace).items():
      print(f"{k}: {v}")
  else:
    print(json.dumps(metrics | trace))


if __name__ == "__main__":
  main()
