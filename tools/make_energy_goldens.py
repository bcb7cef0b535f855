"""Energy fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_energy_goldens.py [scene ...]   # writes tests/golden/energy_<scene>.npz

For every scene of tests/energy_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data (NWORLD
worlds), the scene's per-world Model inputs (each field batched to NWORLD), seeded per-world qpos / qvel, then forward.forward,
sensor.energy_pos and sensor.energy_vel on the state forward left (d.energy filled with NaN first), and one forward.step.  Stored:
`in/*` (qpos, qvel, the per-world fields, nconmax / njmax), `forward/energy` and `forward/sensordata`, the intermediates the energy
terms read (`forward/xipos`, `forward/ten_length`, `forward/M` in the reference's layout, `is_sparse`), `direct/energy`, and
`step/energy`, `step/sensordata`, `step/qpos`, `step/qvel`.  One process per scene, as in make_pipeline_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import io as mio  # noqa: E402
from tests import energy_scenes  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402

BIG = ("humanoid", "g1")  # scenes with contacts: the contact and row capacities of the pipeline goldens


def _batch(arr, n):
  """Give a reference Model field a leading (batch) size n, every entry a copy of entry 0."""
  arr.a = np.repeat(arr.a[:1], n, axis=0)
  arr.shape = (n,) + tuple(arr.shape[1:])


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd = ref["io"], ref["forward"]
  sensor = warp_shim.load_reference_module("sensor")
  mjm = energy_scenes.load(name)
  nworld = energy_scenes.NWORLD
  nconmax, njmax = (32, 128) if name in BIG else (4, 16)
  t0 = time.time()
  ad = ref_runner.MjModelAdapter(mjm, defaults={"nJmom": mio.derive_tables(mjm)["nJmom"]})
  m = io.put_model(ad)
  inputs = energy_scenes.per_world_inputs(name, mjm, nworld)
  for f, v in inputs.items():
    arr = getattr(m, f)
    _batch(arr, nworld)
    arr.a[...] = np.asarray(v).reshape(arr.a.shape)
  d = io.make_data(ad, nworld=nworld, nconmax=nconmax, njmax=njmax)
  qpos, qvel = energy_scenes.seeded_state(mjm, nworld)
  d.qpos.a[...] = qpos
  d.qvel.a[...] = qvel
  out = {"in/qpos": qpos, "in/qvel": qvel, "in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax), "is_sparse": np.array(bool(m.is_sparse))}
  for f, v in inputs.items():
    out[f"in/{f}"] = v
  fwd.forward(m, d)
  out["forward/energy"] = d.energy.numpy().copy()
  out["forward/sensordata"] = d.sensordata.numpy().copy()
  out["forward/xipos"] = d.xipos.numpy().copy()
  out["forward/ten_length"] = d.ten_length.numpy().copy()
  out["forward/M"] = d.M.numpy().copy()
  d.energy.a[...] = np.nan
  sensor.energy_pos(m, d)
  sensor.energy_vel(m, d)
  out["direct/energy"] = d.energy.numpy().copy()
  fwd.step(m, d)
  for f in ("energy", "sensordata", "qpos", "qvel"):
    out[f"step/{f}"] = getattr(d, f).numpy().copy()
  path = os.path.join(ROOT, "tests", "golden", f"energy_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: energy {out['direct/energy'].tolist()}, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(energy_scenes.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
