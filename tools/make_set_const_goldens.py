"""set_const fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_set_const_goldens.py [scene ...]   # writes tests/golden/set_const_<scene>.npz

For every scene of tests/set_const_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data
(NWORLD worlds), then the scene's per-world inputs are written into the Model (each input field batched to NWORLD) and every field
set_const writes is batched to NWORLD as well ("unbatched" leaves every field shared), and set_const.set_const runs.  For scenes with
tendons set_const_0 and set_const_spring also run on their own, each from a fresh Model.  Stored per call `<call>/<field>`: every
output field (NWORLD entries, or 1), `<call>/meaninertia` (its NWORLD entries), and `in/<field>` the per-world inputs.
One process per scene, as in make_pipeline_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import io as mio  # noqa: E402
from mujoco_warp_b200._src import mjcf  # noqa: E402
from tests import set_const_scenes  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402


def _batch(arr, n):
  """Give a reference Model field a leading (batch) size n, every entry a copy of entry 0."""
  arr.a = np.repeat(arr.a[:1], n, axis=0)
  arr.shape = (n,) + tuple(arr.shape[1:])


class _KernelShape(tuple):
  """A warp array's shape as a kernel sees it: four entries, 0 past ndim (set_const.py:385 reads ten_J.shape[2] of a 2-D array)."""

  def __getitem__(self, i):
    return 0 if isinstance(i, int) and i >= len(self) else tuple.__getitem__(self, i)


def _model(io, ad, mjm, scene, nworld):
  m = io.put_model(ad)
  if scene != "unbatched":
    inputs = set_const_scenes.per_world_inputs(scene, mjm, nworld)
    for f in set(inputs) | set(set_const_scenes.OUTPUTS) | {"meaninertia"}:
      arr = m.stat.meaninertia if f == "meaninertia" else getattr(m, f)
      _batch(arr, nworld)
      if f in inputs:
        arr.a[...] = np.asarray(inputs[f], dtype=np.float32).astype(np.float64).reshape(arr.a.shape)
  return m


def run(scene):
  wp, ref = ref_runner.setup()
  io = ref["io"]
  sc = warp_shim.load_reference_module("set_const")
  mjm = mjcf.load_string(set_const_scenes.SCENES[scene])
  nworld = set_const_scenes.NWORLD
  t0 = time.time()
  # MjModel.nJmom counts the non-zeros of tendon transmissions too (the adapter's default counts joint transmissions only)
  ad = ref_runner.MjModelAdapter(mjm, defaults={"nJmom": mio.derive_tables(mjm)["nJmom"]})
  out = {}
  for f, v in set_const_scenes.per_world_inputs(scene, mjm, nworld).items():
    out[f"in/{f}"] = np.asarray(v, dtype=np.float32).astype(np.float64)
  calls = ["set_const"] + (["set_const_0", "set_const_spring"] if int(getattr(mjm, "ntendon", 0)) else [])
  for call in calls:
    m = _model(io, ad, mjm, scene, nworld)
    d = io.make_data(ad, nworld=nworld, nconmax=4, njmax=16)
    d.ten_J.shape = _KernelShape(d.ten_J.shape)
    getattr(sc, call)(m, d)
    for f in set_const_scenes.OUTPUTS:
      out[f"{call}/{f}"] = getattr(m, f).numpy()
    out[f"{call}/meaninertia"] = m.stat.meaninertia.numpy()
  path = os.path.join(ROOT, "tests", "golden", f"set_const_{scene}.npz")
  np.savez_compressed(path, **out)
  print(f"{scene}: {len(calls)} call(s), {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or list(set_const_scenes.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
