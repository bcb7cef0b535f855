"""Inverse-dynamics fixture from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_inverse_goldens.py          # writes tests/golden/inverse_vectors.npz

For every scene (the scene definitions and seeded states of tools/make_pipeline_goldens.py) the UNMODIFIED reference runs in double
precision: io.put_model -> io.make_data -> forward.forward, then inverse.inverse at two accelerations per scene: the converted `qacc`
of forward ("conv") and that `qacc` plus noise ("noisy"), so that rows land in every state.  The INVDISCRETE variants set
`mjENBL_INVDISCRETE`.  Stored per case: the inputs, every Data field inverse writes, the Jacobian rows and aref, and the knife-edge
rows: rows whose reference state changes under a 1e-6 relative nudge of `qacc` (either sign).  Only those may come out in another
state in fp32.  One process per scene, as in make_pipeline_goldens.py.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import constants as C  # noqa: E402
from tests import util  # noqa: E402
from tools import make_pipeline_goldens as pg  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
OUT = os.path.join(GOLD, "inverse_vectors.npz")
FIELDS = ["qfrc_inverse", "qfrc_constraint", "solver_niter", "sensordata", "qacc", "nefc", "ne", "nf"]
EFC = ["force", "state", "Ma", "aref", "D", "type", "id", "frictionloss"]
# fixture scene -> (pipeline scene, INVDISCRETE, extra disable flags)
SCENES = {
  "humanoid": ("humanoid", False, 0), "humanoid_elliptic": ("humanoid_elliptic", False, 0), "mixed": ("mixed", False, 0),
  "mixed_elliptic": ("mixed_elliptic", False, 0), "equality": ("equality", False, 0), "tendons": ("tendons", False, 0),
  "sensors": ("sensors", False, 0), "g1": ("g1", False, 0), "three_humanoids": ("three_humanoids", False, 0),
  "actuators_disc": ("actuators", True, 0), "actuators_disc_noeulerdamp": ("actuators", True, C.DSBL_EULERDAMP),
  "actuators_implicitfast_disc": ("actuators_implicitfast", True, 0), "tendons_implicitfast_disc": ("tendons_implicitfast", True, 0),
  "g1_disc": ("g1", True, 0),
}


def run(name):
  base, disc, dsbl = SCENES[name]
  wp, ref = ref_runner.setup()
  io, fwd, inv = ref["io"], ref["forward"], warp_shim.load_reference_module("inverse")
  mjm, cfg = next((mm, cc) for n, mm, cc in pg.scenes() if n == base)
  mjm.opt.disableflags = int(mjm.opt.disableflags) | dsbl
  if disc:
    mjm.opt.enableflags = int(mjm.opt.enableflags) | C.ENBL_INVDISCRETE
  nconmax, njmax, key = cfg.pop("nconmax"), cfg.pop("njmax"), cfg.pop("key")
  nworld = cfg.pop("nworld", 3)
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  qpos, qvel, ctrl, _ = (f32(a) for a in util.seeded_state(mjm, nworld, key=key, seed=1234, **cfg))
  if base.startswith("humanoid"):
    qpos[:, :7] = mjm.key_qpos[0][:7]
    qpos[:, 2] -= 0.0005 * np.arange(nworld)
  if base == "three_humanoids":
    for i in range(3):
      sl = slice(28 * i, 28 * (i + 1))
      qpos[:, sl] += mjm.key_qpos[3 * i][sl] - mjm.key_qpos[0][sl]
      qpos[:, 28 * i : 28 * i + 7] = mjm.key_qpos[3 * i][28 * i : 28 * i + 7]
      qpos[:, 28 * i + 2] -= 0.0005 * np.arange(nworld)
  rng = np.random.default_rng(99)
  qfrc_applied = f32(rng.uniform(-0.5, 0.5, (nworld, mjm.nv)))
  ad = ref_runner.MjModelAdapter(mjm)
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=nworld, nconmax=nconmax, njmax=njmax)
  d.qpos.a[...] = qpos; d.qvel.a[...] = qvel; d.qfrc_applied.a[...] = qfrc_applied
  if mjm.nu:
    d.ctrl.a[...] = ctrl
  out = {"in/qpos": qpos, "in/qvel": qvel, "in/ctrl": ctrl, "in/qfrc_applied": qfrc_applied, "in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax)}
  if getattr(mjm, "na", 0):
    act = util.seeded_act(mjm, nworld)
    d.act.a[...] = act
    out["in/act"] = act
  if getattr(mjm, "nmocap", 0):
    r2 = np.random.default_rng(77)
    mp = d.mocap_pos.numpy() + f32(0.03 * r2.uniform(-1, 1, (nworld, mjm.nmocap, 3)))
    mq = d.mocap_quat.numpy() + f32(0.1 * r2.uniform(-1, 1, (nworld, mjm.nmocap, 4)))
    mq = f32(mq / np.linalg.norm(mq, axis=-1, keepdims=True))
    d.mocap_pos.a[...] = mp; d.mocap_quat.a[...] = mq
    out.update({"in/mocap_pos": mp, "in/mocap_quat": mq})
  fwd.forward(m, d)
  qacc_conv = f32(d.qacc.numpy())
  noise = f32(rng.normal(size=qacc_conv.shape) * (0.5 + 0.5 * np.abs(qacc_conv)))
  for kind, qacc in (("conv", qacc_conv), ("noisy", qacc_conv + noise)):
    qacc = f32(qacc)
    states = []
    for nudge in (0.0, 1e-6, -1e-6):
      d.qacc.a[...] = qacc * (1.0 + nudge)
      inv.inverse(m, d)
      states.append(d.efc.state.numpy().copy())
      if nudge == 0.0:
        tag = f"{kind}"
        out[f"{tag}/in_qacc"] = qacc
        for f in FIELDS:
          a = getattr(d, f, None)
          if a is not None and a.a is not None:
            out[f"{tag}/{f}"] = a.numpy().copy()
        for f in EFC:
          out[f"{tag}/efc_{f}"] = getattr(d.efc, f).numpy().copy()
        snap = {}
        pg.snapshot(mjm, d, snap, "x")
        out[f"{tag}/efc_J"] = snap["x/efc_J"][:, :, : mjm.nv]
        for f in ("friction", "dim", "efc_address", "worldid"):  # the elliptic rows' contact data
          out[f"{tag}/con_{f}"] = snap[f"x/con_{f}"]
    out[f"{kind}/knife"] = (states[1] != states[0]) | (states[2] != states[0])
  return out


def main():
  if len(sys.argv) > 1 and sys.argv[1] == "--one":  # child: one scene into a temporary .npz
    name, path = sys.argv[2], sys.argv[3]
    t0 = time.time()
    out = run(name)
    np.savez_compressed(path, **out)
    st = out["noisy/efc_state"]
    print(f"{name}: nefc {out['conv/nefc'].ravel()}, noisy states {np.bincount(st[st >= 0].ravel(), minlength=5)}, "
          f"knife {int(out['conv/knife'].sum())} + {int(out['noisy/knife'].sum())}, {time.time() - t0:.1f} s", flush=True)
    return
  import subprocess
  import tempfile

  names = sys.argv[1:] or list(SCENES)
  allout = dict(np.load(OUT)) if os.path.exists(OUT) and sys.argv[1:] else {}
  with tempfile.TemporaryDirectory() as tmp:
    for n in names:
      p = os.path.join(tmp, n + ".npz")
      subprocess.check_call([sys.executable, os.path.abspath(__file__), "--one", n, p])
      allout = {k: v for k, v in allout.items() if not k.startswith(n + "/")}
      allout.update({f"{n}/{k}": v for k, v in np.load(p).items()})
  np.savez_compressed(OUT, **allout)


if __name__ == "__main__":
  main()
