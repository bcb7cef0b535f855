"""Rangefinder fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_rangefinder_goldens.py [scene ...]   # writes tests/golden/rangefinder_<scene>.npz

For every scene of tests/rangefinder_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data (NWORLD
worlds), seeded per-world qpos / qvel (and, for `batched`, per-world geom_size and geom_rgba, stored under `in/`), then
- `forward/*`: sensordata and the poses the rangefinders read (site_xpos / site_xmat / geom_xpos / geom_xmat) after forward.forward from
  the seeded state with the first step's ctrl;
- `step/<k>/in_*` and `step/<k>/out_*` for each step k: the state before (time, qpos, qvel, qacc_warmstart, ctrl, history) and after one
  forward.step (the same plus sensordata and the poses), so that a test can replay every step.
Each state also carries `knife` (nworld, nrangefinder): the rangefinder's ray is knife-edge when a 1e-5 move of its origin (three random
moves, ray.rays on the same poses) changes the geom it hits or its distance by more than 1e-4, or when its distance lies within 1e-5 of
its cutoff.  Only those may come out differently in fp32.  One process per scene, as in make_sensor_extra_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import io as mio  # noqa: E402
from tests import rangefinder_scenes as S  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402

STATE = ("time", "qpos", "qvel", "qacc_warmstart", "ctrl", "history")
POSES = ("site_xpos", "site_xmat", "geom_xpos", "geom_xmat")


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd, ty = ref["io"], ref["forward"], ref["types"]
  rayref = warp_shim.load_reference_module("ray")
  mjm = S.load(name)
  _, nsteps, per_world = S.SCENES[name]
  nworld = S.NWORLD
  nconmax, njmax = 4, 16
  t0 = time.time()
  ad = ref_runner.MjModelAdapter(mjm, defaults={"nJmom": mio.derive_tables(mjm)["nJmom"]})
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=nworld, nconmax=nconmax, njmax=njmax)
  rft = mio.rangefinder_tables(mjm)
  out = {"in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax)}
  # the reference's own rangefinder fields, for the host test of put_model's tables
  out["ref/nrangefinder"] = np.array(int(m.nrangefinder))
  for f in ("sensor_rangefinder_adr", "rangefinder_sensor_adr", "sensor_rangefinder_bodyid"):
    out[f"ref/{f}"] = np.asarray(getattr(m, f).numpy() if hasattr(getattr(m, f), "numpy") else getattr(m, f)).astype(np.int32)
  if per_world:
    size, rgba = S.batched(mjm)
    m.geom_size = wp.array(size, dtype=wp.vec3)
    m.geom_rgba = wp.array(rgba, dtype=wp.vec4)
    out["in/geom_size"], out["in/geom_rgba"] = size, rgba
  qpos, qvel, ctrl = S.seeded(mjm, nsteps)
  d.qpos.a[...] = qpos
  d.qvel.a[...] = qvel
  d.ctrl.a[...] = ctrl[0]
  out["in/ctrl"] = ctrl

  site = np.asarray(mjm.sensor_objid)[rft["sensor_rangefinder_adr"]]
  cutoff = np.asarray(mjm.sensor_cutoff, dtype=np.float64)[rft["sensor_rangefinder_adr"]]
  bodyx = wp.array(rft["sensor_rangefinder_bodyid"], dtype=int)
  rng = np.random.default_rng(7)

  def knife():
    pnt = d.site_xpos.numpy()[:, site].astype(np.float64)
    vec = d.site_xmat.numpy().reshape(nworld, -1, 3, 3)[:, site][..., 2].astype(np.float64)
    nrf = len(site)

    def cast(p):
      dist, gid, nrm = wp.zeros((nworld, nrf), dtype=float), wp.zeros((nworld, nrf), dtype=int), wp.zeros((nworld, nrf), dtype=wp.vec3)
      rayref.rays(m, d, wp.array(p, dtype=wp.vec3), wp.array(vec, dtype=wp.vec3), ty.vec6(*([1e10] * 6)), True, bodyx, dist, gid, nrm)
      return dist.numpy().astype(np.float64), gid.numpy()

    dist, gid = cast(pnt)
    k = (cutoff[None] > 0) & (np.abs(dist - cutoff[None]) < 1e-5)
    for _ in range(3):
      dp = rng.normal(size=pnt.shape)
      d2, g2 = cast(pnt + 1e-5 * dp / np.linalg.norm(dp, axis=-1, keepdims=True))
      k |= (g2 != gid) | (np.abs(d2 - dist) > 1e-4)
    return k

  for f in STATE:
    out[f"start/{f}"] = getattr(d, f).numpy().copy()
  fwd.forward(m, d)
  for f in ("sensordata",) + POSES:
    out[f"forward/{f}"] = getattr(d, f).numpy().copy()
  out["forward/knife"] = knife()
  for f in STATE:
    getattr(d, f).a[...] = out[f"start/{f}"]

  for k in range(nsteps):
    d.ctrl.a[...] = ctrl[k]
    for f in STATE:
      out[f"step/{k}/in_{f}"] = getattr(d, f).numpy().copy()
    fwd.step(m, d)
    for f in STATE + ("sensordata",) + POSES:
      out[f"step/{k}/out_{f}"] = getattr(d, f).numpy().copy()
    out[f"step/{k}/knife"] = knife()

  path = os.path.join(ROOT, "tests", "golden", f"rangefinder_{name}.npz")
  np.savez_compressed(path, **out)
  sd = out["forward/sensordata"][:, np.asarray(mjm.sensor_adr)[rft["sensor_rangefinder_adr"]]]
  nknife = sum(int(out[k].sum()) for k in out if k.endswith("knife"))
  print(f"{name}: nrangefinder {len(site)}, {nsteps} steps, {int((sd >= 0).sum())}/{sd.size} hits at forward, {nknife} knife-edge, "
        f"{os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(S.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
