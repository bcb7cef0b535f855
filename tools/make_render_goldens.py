"""Renderer fixtures from the reference's own code, executed on the CPU through tools/warp_shim.py.

  python tools/make_render_goldens.py                 # tests/golden/render_vectors.npz and every scene of tests/render_scenes.SCENES
  python tools/make_render_goldens.py vectors NAME..  # only those (one process each: they run in parallel)

Images: for each scene of tests/render_scenes.SCENES the UNMODIFIED reference (io.put_model -> io.make_data -> smooth.kinematics ->
smooth.camlight -> render_util.create_render_context -> bvh.refit_bvh -> render.render) runs in double precision, with the shim's
brute-force stand-ins for warp's BVH and mesh queries, in NWORLD worlds of seeded joint positions; the poses are rounded to fp32 first
and stored, so that both renderers read the same geoms, cameras and lights (a last-bit difference in a camera's orientation moves the
depth of a ray that grazes the floor far away by more than the tolerance).  rgb_data / depth_data / seg_data are stored raw.  A buffer entry is knife-edge when
moving every camera by 1e-5 (two directions) changes its geom id, its depth by more than 1e-4 relative (at least 1e-4 absolute: rays
that graze the floor far away move more), or a colour channel by more than 2/255; shadow-edge when moving every light's position and
direction by 1e-5 changes its geom id or a channel by more than 2/255.  A depth is also knife-edge when turning every camera by 1e-6 rad (either way about its x and y axes)
changes it by more than 1e-5 relative (ill-conditioned in fp32: rays that graze the floor far away).

Vectors:
The UNMODIFIED reference functions run in double precision on seeded inputs that are exactly representable in fp32:
render_util.py:71 compute_ray (perspective, orthographic and sensorsize / intrinsic cameras at odd resolutions, every pixel of a
few images) and render.py:518 compute_lighting with shadows off (directional, spot and point lights, default and non-default
attenuation, inactive lights, lights behind the surface and outside the spot cone, specular on and off).  With use_shadows off the
lighting closure never casts a ray, so the scene arguments it takes are placeholders.
"""

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import render_scenes  # noqa: E402
from tools import ref_runner, warp_shim  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
OUT = os.path.join(GOLDEN, "render_vectors.npz")
f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)


def unit(v):
  return v / np.linalg.norm(v)


def vectors():
  wp, _ = ref_runner.setup()
  ru = warp_shim.load_reference_module("render_util")
  rd = warp_shim.load_reference_module("render")
  rng = np.random.default_rng(7)

  # compute_ray: (projection, fovy, sensor w, sensor h, img_w, img_h, px, py, znear) and intrinsic [fx, fy, cx, cy]
  cams = [(0, 45.0, 0.0, 0.0, 31, 23, [0, 0, 0, 0], 0.01), (0, 90.0, 0.0, 0.0, 17, 29, [0, 0, 0, 0], 0.05), (1, 45.0, 0.0, 0.0, 11, 7, [0, 0, 0, 0], 0.01),
          (0, 45.0, 0.006, 0.004, 25, 19, [0.0048, 0.0048, 0.0, 0.0], 0.01), (0, 45.0, 0.006, 0.004, 13, 21, [0.004, 0.005, 0.0003, -0.0002], 0.02),
          (0, 60.0, 0.004, 0.004, 9, 9, [0.003, 0.003, 0.0, 0.0], 0.01)]
  rargs, rintr, rays = [], [], []
  for proj, fovy, sw, sh, w, h, intr, zn in cams:
    for py in range(h):
      for px in range(w):
        a = f32([proj, fovy, sw, sh, w, h, px, py, zn])
        i = f32(intr)
        r = ru.compute_ray(int(a[0]), a[1], wp.vec2(a[2], a[3]), wp.vec4(*i), int(a[4]), int(a[5]), int(a[6]), int(a[7]), a[8])
        rargs.append(a), rintr.append(i), rays.append(list(r))

  # compute_lighting with shadows off
  lighting = rd._make_compute_lighting(rd._make_cast_ray((0,), first_hit=True))
  light, surf, flags, out = [], [], [], []
  for k in range(400):
    ltype = int(rng.integers(0, 3))
    n = unit(rng.normal(size=3))
    hit = rng.normal(size=3)
    view = unit(rng.normal(size=3) + n)
    pos = hit + rng.uniform(0.5, 3.0) * unit(rng.normal(size=3) + 1.5 * n)
    ldir = unit(hit - pos + 0.4 * rng.normal(size=3)) if ltype != 1 else unit(-n + 0.8 * rng.normal(size=3))
    default_att = bool(k % 3 == 0)
    att = [1.0, 0.0, 0.0] if default_att else [1.0, rng.uniform(0, 0.3), rng.uniform(0, 0.1)]
    l = f32([float(k % 17 != 0), ltype, 1.0, *pos, *ldir, *att, np.deg2rad(rng.uniform(10, 80)), rng.uniform(0, 20), *rng.uniform(0, 1, 3), *rng.uniform(0, 1, 3)])
    s = f32([*n, *hit, *view, rng.uniform(0, 1), rng.uniform(0, 1) * 128.0])
    fl = [int(k % 5 != 0), int(default_att), int(ltype == 0 or k % 2 == 0)]
    V = lambda a: wp.vec3(*a)
    diff, spec = lighting(None, None, None, None, None, None, None, None, None, False, 0, 0, 0, 0, None, 0, None, None, None, None, None, None,
                          bool(l[0]), int(l[1]), bool(l[2]), V(l[3:6]), V(l[6:9]), V(l[9:12]), l[12], l[13], V(l[14:17]), V(l[17:20]),
                          V(s[0:3]), V(s[3:6]), V(s[6:9]), s[9], s[10], True, bool(fl[0]), bool(fl[1]), bool(fl[2]))
    light.append(l), surf.append(s), flags.append(fl), out.append(list(diff) + list(spec))

  np.savez_compressed(OUT, ray_args=np.array(rargs), ray_intrinsic=np.array(rintr), ray=np.array(rays), light=np.array(light), surf=np.array(surf),
                      light_flags=np.array(flags, dtype=np.int32), lighting=np.array(out))
  print("wrote", OUT, len(rays), "rays,", len(out), "lighting cases")


def scene(name):
  import json
  from types import SimpleNamespace

  from mujoco_warp_b200._src import mjcf

  wp, ref = ref_runner.setup()
  mj = sys.modules["mujoco"]
  mj.mj_forward = lambda m, d: None  # create_render_context's initial BVH bounds are replaced by the refit below
  init = mj.MjData.__init__

  def data_init(self, m):
    init(self, m)
    self.flexvert_xpos = np.zeros((0, 3))

  mj.MjData.__init__ = data_init
  ru, rd, bvh = (warp_shim.load_reference_module(n) for n in ("render_util", "render", "bvh"))
  io, smooth = ref["io"], ref["smooth"]
  sc = render_scenes.SCENES[name]
  mjm = mjcf.load_string(sc["xml"])
  mjm.vis.map = SimpleNamespace(znear=0.01)  # MuJoCo's default; the rays do not depend on it
  mjm.stat.extent = 1.0
  ad = ref_runner.MjModelAdapter(mjm)
  mj.mj_name2id = lambda _m, t, n: mjm.names.camera.index(n) if t == mj.mjtObj.mjOBJ_CAMERA and n in mjm.names.camera else -1
  m = io.put_model(ad)
  nw = render_scenes.NWORLD
  qpos = f32(render_scenes.qpos(mjm, nw, sc.get("seed", 0)))
  d = io.make_data(ad, nworld=nw, nconmax=8, njmax=8)
  d.qpos.a[...] = qpos
  smooth.kinematics(m, d)
  smooth.camlight(m, d)
  for k in ("geom_xpos", "geom_xmat", "cam_xpos", "cam_xmat", "light_xpos", "light_xdir"):
    getattr(d, k).a[...] = f32(getattr(d, k).a)
  out = {"qpos": qpos, "kwargs": np.array(json.dumps(sc["kwargs"]))}
  for k in ("geom_xpos", "geom_xmat", "cam_xpos", "cam_xmat", "light_xpos", "light_xdir"):  # the poses both renderers read
    out["pose/" + k] = np.asarray(getattr(d, k).a, dtype=np.float64).reshape(nw, -1)
  vec = {"geom_rgba": wp.vec4, "mat_rgba": wp.vec4, "light_diffuse": wp.vec3, "cam_fovy": float}
  for k, v in render_scenes.batch_fields(mjm, sc).items():  # per-world Model fields, world w reading entry w % n
    out["batch/" + k] = v
    setattr(m, k, wp.array(v, dtype=vec[k]))
  rc = ru.create_render_context(ad, nworld=nw, **sc["kwargs"])

  def frame():
    bvh.refit_bvh(m, d, rc)
    rd.render(m, d, rc)
    return (rc.rgb_data.numpy().astype(np.int64).reshape(nw, -1), rc.depth_data.numpy().astype(np.float64).reshape(nw, -1),
            rc.seg_data.numpy().astype(np.int64).reshape(nw, -1, 2))

  def channels(rgb):
    return np.stack([(rgb >> s) & 0xFF for s in (16, 8, 0)], -1)

  rgb, depth, seg = frame()
  nrgb, ndepth = rgb.shape[1], depth.shape[1]
  knife_rgb, knife_depth, knife_seg = np.zeros(rgb.shape, bool), np.zeros(depth.shape, bool), np.zeros(seg.shape[:2], bool)
  cam0 = d.cam_xpos.a.copy()
  for off in ([1e-5, 1e-5, 1e-5], [1e-5, -1e-5, 0.0]):
    d.cam_xpos.a[...] = cam0 + np.asarray(off)
    r2, d2, s2 = frame()
    knife_rgb |= (np.abs(channels(r2) - channels(rgb)) > 2).any(-1)
    knife_depth |= np.abs(d2 - depth) > 1e-4 * np.maximum(1.0, np.abs(depth))
    knife_seg |= (s2 != seg).any(-1)
  d.cam_xpos.a[...] = cam0
  # turning every camera by 1e-6 rad (about 16 fp32 ulps of a ray direction) marks the depths fp32 cannot hold to 1e-5: rays that
  # graze a surface far away, where depth = height / cos(angle to the normal) amplifies a direction's rounding
  mat0 = d.cam_xmat.a.copy()
  c, s_ = np.cos(1e-6), np.sin(1e-6)
  rots = [np.array([[1, 0, 0], [0, c, -sg * s_], [0, sg * s_, c]]) for sg in (1, -1)] + [np.array([[c, 0, sg * s_], [0, 1, 0], [-sg * s_, 0, c]]) for sg in (1, -1)]
  for rot in rots:
    d.cam_xmat.a[...] = (mat0.reshape(nw, -1, 3, 3) @ rot).reshape(mat0.shape)
    _, d2, _ = frame()
    knife_depth |= np.abs(d2 - depth) > 1e-5 * np.maximum(1.0, np.abs(depth))
  d.cam_xmat.a[...] = mat0
  shadow_rgb, shadow_seg = np.zeros(rgb.shape, bool), np.zeros(seg.shape[:2], bool)
  if mjm.nlight:
    lp, ldir = d.light_xpos.a.copy(), d.light_xdir.a.copy()
    d.light_xpos.a[...], d.light_xdir.a[...] = lp + 1e-5, ldir + 1e-5
    r2, _, s2 = frame()
    shadow_rgb = (np.abs(channels(r2) - channels(rgb)) > 2).any(-1)
    shadow_seg = (s2 != seg).any(-1)
  # a pixel's geom id decides all three outputs: a pixel marked in one output is marked in every output it appears in
  adr = {k: rc.__dict__[k].numpy() for k in ("rgb_adr", "depth_adr", "seg_adr")}
  res = rc.cam_res.numpy().reshape(-1, 2)
  out.update(rgb=rgb, depth=depth, seg=seg, knife_rgb=knife_rgb, knife_depth=knife_depth, knife_seg=knife_seg, shadow_rgb=shadow_rgb, shadow_seg=shadow_seg,
             rgb_adr=adr["rgb_adr"], depth_adr=adr["depth_adr"], seg_adr=adr["seg_adr"], cam_res=res, cam_id=rc.cam_id_map.numpy())
  path = os.path.join(GOLDEN, f"render_{name}.npz")
  np.savez_compressed(path, **out)
  npix = nw * int(res.prod(axis=1).sum())
  marked = int(knife_rgb.sum() + shadow_rgb.sum()) if nrgb else 0
  print(f"{name}: {npix} pixels, rgb {nrgb}, depth {ndepth}, seg hits {int((seg[..., 0] >= 0).sum())}, marked rgb {marked}, depth {int(knife_depth.sum())}, "
        f"seg {int((knife_seg | shadow_seg).sum())} -> {path}")


if __name__ == "__main__":
  import subprocess

  names = sys.argv[1:]
  if len(names) == 1:
    vectors() if names[0] == "vectors" else scene(names[0])
  else:
    names = names or ["vectors"] + list(render_scenes.SCENES)
    procs = [subprocess.Popen([sys.executable, __file__, n]) for n in names]
    sys.exit(max(p.wait() for p in procs))
