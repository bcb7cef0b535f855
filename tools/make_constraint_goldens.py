"""make_constraint fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_constraint_goldens.py [scene ...]   # writes tests/golden/constraint_<scene>.npz

For every scene of tests/constraint_scenes.py the UNMODIFIED reference runs in double precision: io.put_model -> io.make_data (for
`batched`, the per-world fields of constraint_scenes.batched, stored under `in/`), the seeded state, then forward.forward.  `forward/*` holds
what forward left (tools/make_pipeline_goldens.py's snapshot: state, contacts, the rows with efc_J densified); for a sparse model
`csr/*` holds the reference's CSR arrays as it wrote them (J_rownnz, J_rowadr, J_colind, J).  One process per scene.
"""

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import constraint_scenes as S  # noqa: E402
from tools import ref_runner  # noqa: E402
from tools.make_pipeline_goldens import snapshot  # noqa: E402


def run(name):
  wp, ref = ref_runner.setup()
  io, fwd, types = ref["io"], ref["forward"], ref["types"]
  mjm = S.load(name)
  nconmax, njmax = 16, 64
  t0 = time.time()
  ad = ref_runner.MjModelAdapter(mjm)
  m = io.put_model(ad)
  d = io.make_data(ad, nworld=S.NWORLD, nconmax=nconmax, njmax=njmax)
  out = {"in/nconmax": np.array(nconmax), "in/njmax": np.array(njmax)}
  if name == "batched":
    dt = {"dof_frictionloss": float, "tendon_frictionloss": float, "jnt_margin": float, "jnt_range": wp.vec2, "dof_solref": wp.vec2,
          "geom_friction": wp.vec3, "eq_data": types.vec11}
    for k, v in S.batched(mjm).items():
      setattr(m, k, wp.array(v, dtype=dt[k]))
      out[f"in/{k}"] = v
  qpos, qvel, ctrl, warm = S.state(mjm, name)
  d.qpos.a[...] = qpos; d.qvel.a[...] = qvel; d.qacc_warmstart.a[...] = warm
  if mjm.nu:
    d.ctrl.a[...] = ctrl
  out.update({"in/qpos": qpos, "in/qvel": qvel, "in/ctrl": ctrl, "in/qacc_warmstart": warm})
  fwd.forward(m, d)
  snapshot(mjm, d, out, "forward")
  if d.efc.J.numpy().shape[1] == 1:
    for f in ("J_rownnz", "J_rowadr", "J_colind", "J"):
      out[f"csr/{f}"] = getattr(d.efc, f).numpy().copy()
  path = os.path.join(ROOT, "tests", "golden", f"constraint_{name}.npz")
  np.savez_compressed(path, **out)
  print(f"{name}: nefc {out['forward/nefc'].ravel()}, ne {out['forward/ne'].ravel()}, nf {out['forward/nf'].ravel()}, nl {out['forward/nl'].ravel()}, "
        f"nacon {int(out['forward/nacon'])}, {os.path.getsize(path) // 1024} KiB, {time.time() - t0:.1f} s; MjModel fallbacks: {len(ad.missing)}")


if __name__ == "__main__":
  names = sys.argv[1:] or ["sparse", "batched"]
  if len(names) == 1:
    run(names[0])
  else:
    import subprocess

    for n in names:
      subprocess.check_call([sys.executable, os.path.abspath(__file__), n])
