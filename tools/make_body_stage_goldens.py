"""rne_postconstraint / subtree_vel / jac / xfrc_accumulate / tendon / deriv_smooth_vel fixtures from the reference's own code, executed on
the CPU through tools/warp_shim.py.

  python tools/make_body_stage_goldens.py [scene ...]   # writes tests/golden/body_stage_<scene>.npz

For every scene of tests/body_stage_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data (NWORLD
worlds; for `batched`, per-world body_mass / body_inertia / dof_damping, stored under `in/`), the seeded state and inputs (`in/*`), then
forward.forward followed by each of the six functions.  `fwd/*` holds what forward left that the functions and the tests read; `out/*`
what each function wrote (jacp / jacr for the seeded points and bodies, qfrc after xfrc_accumulate added into the seeded `in/qfrc`,
deriv = M - dt qDeriv).  One process per scene, as in make_muscle_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import io as mio  # noqa: E402
from tests import body_stage_scenes as S  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402

FWD = ("qacc", "M", "cdof", "cvel", "cdof_dot", "cinert", "xipos", "ximat", "xpos", "xmat", "subtree_com", "actuator_force", "ne", "nacon")
OUT = ("cacc", "cfrc_int", "cfrc_ext", "subtree_linvel", "subtree_angmom", "ten_length", "ten_J")


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd, smooth, support = ref["io"], ref["forward"], ref["smooth"], ref["support"]
  derivative = warp_shim.load_reference_module("derivative")
  mjm = S.load(name)
  nworld = S.NWORLD
  nconmax, njmax = 48, 256
  t0 = time.time()
  ad = ref_runner.MjModelAdapter(mjm, defaults={"nJmom": mio.derive_tables(mjm)["nJmom"]})
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=nworld, nconmax=nconmax, njmax=njmax)
  out = {"in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax)}
  if S.SCENES[name][1]:
    mass, inertia, damping = S.batched(mjm)
    m.body_mass = wp.array(mass, dtype=float)
    m.body_inertia = wp.array(inertia, dtype=wp.vec3)
    m.dof_damping = wp.array(damping, dtype=float)
    out["in/body_mass"], out["in/body_inertia"], out["in/dof_damping"] = mass, inertia, damping
  inp = S.seeded(mjm)
  for f in ("qpos", "qvel", "ctrl", "act", "xfrc_applied"):
    getattr(d, f).a[...] = inp[f].reshape(getattr(d, f).a.shape)
  for k, v in inp.items():
    out[f"in/{k}"] = v

  fwd.forward(m, d)
  for f in FWD:
    out[f"fwd/{f}"] = getattr(d, f).numpy().copy()
  smooth.rne_postconstraint(m, d)
  smooth.subtree_vel(m, d)
  smooth.tendon(m, d)
  jacp = wp.zeros((nworld, 3, mjm.nv), dtype=float)
  jacr = wp.zeros((nworld, 3, mjm.nv), dtype=float)
  support.jac(m, d, jacp, jacr, wp.array(inp["point"], dtype=wp.vec3), wp.array(inp["body"], dtype=int))
  qfrc = wp.array(inp["qfrc"], dtype=float)
  support.xfrc_accumulate(m, d, qfrc)
  deriv = wp.zeros(d.M.numpy().shape, dtype=float)
  derivative.deriv_smooth_vel(m, d, deriv)
  for f in OUT:
    out[f"out/{f}"] = getattr(d, f).numpy().copy()
  out["out/jacp"], out["out/jacr"], out["out/qfrc"], out["out/deriv"] = jacp.numpy().copy(), jacr.numpy().copy(), qfrc.numpy().copy(), deriv.numpy().copy()

  path = os.path.join(ROOT, "tests", "golden", f"body_stage_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: nbody {mjm.nbody}, nv {mjm.nv}, contacts {out['fwd/nacon']}, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s")


if __name__ == "__main__":
  names = sys.argv[1:] or list(S.SCENES)
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
