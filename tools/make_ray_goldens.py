"""Ray-casting fixture from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_ray_goldens.py          # writes tests/golden/ray_vectors.npz

The UNMODIFIED reference (io.put_model -> io.make_data -> smooth.kinematics -> ray.rays / ray.ray) runs in double precision on
the scene of tests/test_ray_vectors.py (compiled by mujoco_warp_b200._src.mjcf), in NWORLD seeded worlds.  Ray sets, one per
case: rays aimed at every geom (through the centre, grazing, missing, from inside, parallel to a face, pointing away), random
rays, and the geomgroup / flg_static / bodyexclude filters, with a shared (1, nray) and a per-world (nworld, nray) origin.
A ray is marked knife-edge when a 1e-5 move of its origin changes the reference's geom id or its distance by more than 1e-4:
only those may come out differently in fp32.
"""

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mujoco_warp_b200._src import mjcf  # noqa: E402
from tests.test_ray_vectors import NWORLD, RAY_FIELDS, SCENE_XML  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ray_vectors.npz")
f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)  # inputs exactly representable in fp32


def unit(v):
  return v / np.linalg.norm(v, axis=-1, keepdims=True)


def aimed_rays(mjm, xpos, xmat, rng):
  """(nworld, nray, 3) origins / directions aimed at every geom of every world (the cases of the reference's ray_test.py)"""
  pnts, vecs = [], []
  for g in range(mjm.ngeom):
    size = np.asarray(mjm.geom_size[g])
    rad = max(float(np.max(size)), 0.3) if mjm.geom_type[g] != 0 else 0.5
    u = unit(rng.normal(size=3))
    perp = unit(np.cross(u, rng.normal(size=3)))
    for w in range(xpos.shape[0]):
      c, R = xpos[w, g], xmat[w, g].reshape(3, 3)
      if mjm.geom_type[g] == 0:  # plane: from the front side
        uu = unit(R[:, 2] + 0.6 * (u - R[:, 2] * (u @ R[:, 2])))
      else:
        uu = u
      far = c + 3.0 * rad * uu
      pw = [far, far + 0.9 * rad * perp, far + 4.0 * rad * perp, c + 0.1 * rad * perp, c + R @ np.array([-3 * rad, 0.0, size[2] if mjm.geom_type[g] == 6 else 0.2]),
            far]
      vw = [-uu, -uu, -uu, unit(rng.normal(size=3)), R[:, 0], uu]
      if w == 0:
        pnts.append([]), vecs.append([])
      pnts[-1].append(pw), vecs[-1].append(vw)
  # (ngeom, nworld, 6, 3) -> (nworld, ngeom * 6, 3)
  p = np.asarray(pnts).transpose(1, 0, 2, 3).reshape(xpos.shape[0], -1, 3)
  v = np.asarray(vecs).transpose(1, 0, 2, 3).reshape(xpos.shape[0], -1, 3)
  return p, v


def main():
  wp, ref = ref_runner.setup()
  io, smooth = ref["io"], ref["smooth"]
  rayref = warp_shim.load_reference_module("ray")
  ty = ref["types"]
  mjm = mjcf.load_string(SCENE_XML)
  ad = ref_runner.MjModelAdapter(mjm)
  m = io.put_model(ad)
  missing = sorted(ad.missing & set(RAY_FIELDS))
  assert not missing, f"the reference's put_model fell back to defaults for ray fields {missing}: the fixture would be meaningless"

  rng = np.random.default_rng(2024)
  qpos = np.tile(np.asarray(mjm.qpos0, dtype=np.float64), (NWORLD, 1))
  for j in range(mjm.njnt):
    if mjm.jnt_type[j] == 0:  # free joints: move and turn every body differently in every world
      a = int(mjm.jnt_qposadr[j])
      qpos[:, a : a + 3] += rng.uniform(-0.1, 0.1, (NWORLD, 3))
      qpos[:, a + 3 : a + 7] = unit(rng.normal(size=(NWORLD, 4)))
  qpos = f32(qpos)
  d = io.make_data(ad, nworld=NWORLD, nconmax=8, njmax=8)
  d.qpos.a[...] = qpos
  smooth.kinematics(m, d)
  xpos, xmat = f32(d.geom_xpos.numpy()), f32(d.geom_xmat.numpy().reshape(NWORLD, mjm.ngeom, 9))
  # the fixture holds the poses in fp32 and the reference reads them back, so that every implementation sees the same geoms
  d.geom_xpos.a[...] = xpos
  d.geom_xmat.a[...] = xmat.reshape(d.geom_xmat.a.shape)

  def cast(pnt, vec, geomgroup, flg_static, bodyexclude):
    pa, va = wp.array(pnt, dtype=wp.vec3), wp.array(vec, dtype=wp.vec3)
    nray = pnt.shape[1]
    dist, gid, nrm = wp.zeros((NWORLD, nray), dtype=float), wp.zeros((NWORLD, nray), dtype=int), wp.zeros((NWORLD, nray), dtype=wp.vec3)
    rayref.rays(m, d, pa, va, ty.vec6(*geomgroup), bool(flg_static), wp.array(bodyexclude, dtype=int), dist, gid, nrm)
    return dist.numpy().astype(np.float64), gid.numpy().astype(np.int32), nrm.numpy().astype(np.float64).reshape(NWORLD, nray, 3)

  ap, av = aimed_rays(mjm, xpos, xmat, rng)
  nrand = 96
  rp = np.concatenate([rng.uniform([-2.0, -2.0, 0.05], [2.0, 2.0, 1.5], (nrand // 2, 3)), np.tile([[0.0, 0.0, 3.0]], (nrand // 2, 1))])[None]
  rv = unit(np.concatenate([rng.normal(size=(nrand // 2, 3)), np.stack([rng.normal(0, 0.4, nrand // 2), rng.normal(0, 0.4, nrand // 2), -np.ones(nrand // 2)], 1)]))[None]
  nb = mjm.nbody
  cases = {
    "aimed": (ap, av, [-1] * 6, 1, -np.ones(ap.shape[1])),
    "random": (rp, rv, [-1] * 6, 1, -np.ones(nrand)),
    "groups": (rp, rv, [1, 0, 1, 0, 1, 0], 1, -np.ones(nrand)),
    "groups_only2": (rp, rv, [0, 0, 1, -1, 0, 0], 1, -np.ones(nrand)),
    "nostatic": (rp, rv, [-1] * 6, 0, -np.ones(nrand)),
    "bodyexclude": (rp, rv, [-1] * 6, 1, np.arange(nrand) % (nb + 1) - 1),
    "aimed_nostatic_groups": (ap, av, [1, 1, 0, 1, 1, 1], 0, (np.arange(ap.shape[1]) % (nb + 1)) - 1),
  }
  out = {"in/qpos": qpos, "geom_xpos": xpos, "geom_xmat": xmat}
  for name, (p, v, gg, fs, bx) in cases.items():
    p, v, bx = f32(p), f32(unit(v)), np.asarray(bx, dtype=np.int32)
    dist, gid, nrm = cast(p, v, gg, fs, bx)
    knife = np.zeros(dist.shape, dtype=bool)
    for _ in range(3):
      dp = unit(rng.normal(size=p.shape)) * 1e-5
      d2, g2, _ = cast(p + dp, v, gg, fs, bx)
      knife |= (g2 != gid) | (np.abs(d2 - dist) > 1e-4)
    out.update({f"{name}/pnt": p, f"{name}/vec": v, f"{name}/geomgroup": np.asarray(gg, dtype=np.int32), f"{name}/flg_static": np.array(fs),
                f"{name}/bodyexclude": bx, f"{name}/dist": dist, f"{name}/geomid": gid, f"{name}/normal": nrm, f"{name}/knife": knife})
    print(f"{name}: {dist.size} rays, {int((gid >= 0).sum())} hits, {int(knife.sum())} knife-edge, geoms hit {sorted(set(gid.ravel().tolist()))}")
  # ray.ray: one ray per world, bodyexclude as a scalar
  p1, v1 = f32(ap[:, 7:8]), f32(unit(av[:, 7:8]))
  dd, gg_, nn = rayref.ray(m, d, wp.array(p1, dtype=wp.vec3), wp.array(v1, dtype=wp.vec3), bodyexclude=int(mjm.geom_bodyid[0]))
  out.update({"ray/pnt": p1, "ray/vec": v1, "ray/bodyexclude": np.array(int(mjm.geom_bodyid[0])), "ray/dist": dd.numpy().astype(np.float64),
              "ray/geomid": gg_.numpy().astype(np.int32), "ray/normal": nn.numpy().astype(np.float64).reshape(NWORLD, 1, 3)})
  np.savez_compressed(OUT, **out)
  print(f"wrote {OUT} ({os.path.getsize(OUT) // 1024} KiB)")


if __name__ == "__main__":
  main()
