"""Per-kernel and whole-step timing of the humanoid benchmark state (deterministic: `warm` steps from the squat keyframe).
usage: python tools/ktime.py [nworld] [warm] [reps]   (MJB_LIB selects the library build to time, KT_MODEL / KT_NCONMAX / KT_NJMAX the scene)"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mujoco_warp_b200 as mjw
from mujoco_warp_b200._src.mjcf import MjDataLite, reset_data_keyframe

nworld = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
warm = int(sys.argv[2]) if len(sys.argv) > 2 else 20
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 100
model = os.environ.get("KT_MODEL", os.path.join(os.path.dirname(mjw.__file__), "test_data", "humanoid.npz"))
nconmax, njmax = int(os.environ.get("KT_NCONMAX", 24)), int(os.environ.get("KT_NJMAX", 64))
mjm = mjw.mjcf.load_any(model)
m = mjw.put_model(mjm)
mjd = MjDataLite(mjm)
if mjm.nkey > 0:
  reset_data_keyframe(mjm, mjd, 0)
d = mjw.put_data(mjm, mjd, nworld=nworld, nconmax=nconmax, njmax=njmax, m=m)
center = torch.from_numpy(np.asarray(mjd.ctrl, dtype=np.float32)).cuda()
stream = torch.cuda.Stream()
with torch.cuda.stream(stream):
  for i in range(warm):
    mjw.ctrl_noise(m, d, i, center)
    mjw.step(m, d)
  stream.synchronize()
  snap = {n: getattr(d, n).clone() for n in ("qpos", "qvel", "ctrl", "qacc_warmstart", "time")}
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g, stream=stream):
    mjw.step(m, d)
  for n, v in snap.items():
    getattr(d, n).copy_(v)
  for _ in range(5):
    g.replay()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for n, v in snap.items():
    getattr(d, n).copy_(v)
  e0.record(stream)
  for i in range(reps):
    g.replay()
  e1.record(stream)
  stream.synchronize()
  step_ms = e0.elapsed_time(e1) / reps
  for n, v in snap.items():
    getattr(d, n).copy_(v)
  acc = None
  for i in range(20):
    r = mjw.step_profile(m, d)
    acc = r if acc is None else {k: acc[k] + r[k] for k in r}
  kms = {k: round(v / 20 * 1e3, 1) for k, v in acc.items()}
out = {"cfg": {k: v for k, v in os.environ.items() if k.startswith("MJB_")}, "step_us": round(step_ms * 1e3, 1), "Msteps_s": round(nworld / step_ms / 1e3, 2),
       "kernel_us": kms, "nefc": float(d.nefc.float().mean()), "niter": float(d.solver_niter.float().mean()), "nan": int(torch.isnan(d.qpos).any(dim=1).sum())}
print(json.dumps(out))
