"""Batch rendering on the GPU (create_render_context / refit_bvh / render / get_*), checked without a reference renderer: each
pixel's primary ray, rebuilt from the context's camera-frame rays and the camera poses, is cast through `mjw.rays`, which is pinned
to the reference by tests/golden/ray_vectors.npz.  Geom ids must agree and depth / (-ray_z) must equal the ray distance, except on
knife-edge pixels (a 1e-5 move of the ray origin changes the geom id, or the distance by more than 1e-4 relative: rays that graze the
infinite floor far away move by more than 1e-4 in absolute terms)."""

import numpy as np
import pytest
import torch

from tests import render_scenes

pytestmark = pytest.mark.gpu

NWORLD = 5
ORTHOGRAPHIC = (1,)  # camera ids of the orthographic cameras of render_scenes.PRIMITIVES ("ortho")


def _setup(xml, nworld=NWORLD, batch_sizes=None, seed=0, **kw):
  import mujoco_warp_b200 as mjw

  mjm = mjw.mjcf.load_string(xml)
  m = mjw.put_model(mjm, batch_sizes=batch_sizes)
  d = mjw.make_data(mjm, nworld=nworld, m=m)
  rng = np.random.default_rng(seed)
  q = np.tile(np.asarray(mjm.qpos0, dtype=np.float64), (nworld, 1))
  if mjm.nq:
    q[:, : min(2, mjm.nq)] += rng.uniform(-0.3, 0.3, size=(nworld, min(2, mjm.nq)))
  d.qpos.copy_(torch.from_numpy(q.astype(np.float32)))
  mjw.kinematics(m, d)
  mjw.camlight(m, d)
  kw.setdefault("render_rgb", True)
  kw.setdefault("render_depth", True)
  kw.setdefault("render_seg", True)
  rc = mjw.create_render_context(mjm, nworld=nworld, **kw)
  return mjw, mjm, m, d, rc


def _frame(mjw, m, d, rc):
  mjw.refit_bvh(m, d, rc)
  mjw.render(m, d, rc)
  torch.cuda.synchronize()


def _world_rays(d, rc, c):
  """pnt, vec (nworld, npix, 3) of active camera c's pixels, and the camera-frame z of each ray"""
  cam = int(rc.cam_id_map[c])
  a = int(rc.pix_adr[c])
  w, h = rc.cam_res[c].tolist()
  loc = rc.ray[a : a + w * h]
  xmat = d.cam_xmat[:, cam].reshape(-1, 3, 3)
  vec = torch.einsum("wij,pj->wpi", xmat, loc).contiguous()
  pnt = d.cam_xpos[:, cam].reshape(-1, 1, 3).expand(-1, w * h, 3).contiguous()
  return pnt, vec, loc[:, 2]


def _cast(mjw, m, d, pnt, vec, groups):
  n = pnt.shape[1]
  gg = [1 if g in groups else 0 for g in range(6)]
  dist = torch.empty((d.nworld, n), dtype=torch.float32, device="cuda")
  gid = torch.empty((d.nworld, n), dtype=torch.int32, device="cuda")
  nrm = torch.empty((d.nworld, n, 3), dtype=torch.float32, device="cuda")
  mjw.rays(m, d, pnt, vec, gg, True, torch.full((n,), -1, dtype=torch.int32, device="cuda"), dist, gid, nrm)
  return dist, gid


def _cross_check(mjw, m, d, rc, groups=(0, 1, 2), cams=None):
  """Returns the number of compared pixels; asserts agreement with mjw.rays away from knife edges."""
  compared = 0
  for c in range(rc.nrender) if cams is None else cams:
    pnt, vec, z = _world_rays(d, rc, c)
    dist, gid = _cast(mjw, m, d, pnt, vec, groups)
    edge = torch.zeros_like(gid, dtype=torch.bool)
    for off in ([1e-5, 0, 0], [0, 1e-5, 0], [0, 0, 1e-5], [-1e-5, -1e-5, -1e-5]):
      dd, gg = _cast(mjw, m, d, (pnt + torch.tensor(off, device="cuda")).contiguous(), vec, groups)
      edge |= (gg != gid) | ((dd - dist).abs() > 1e-4 * dist.abs().clamp(min=1.0))
    for off in ([1e-6, 0, 0], [0, 1e-6, 0], [0, 0, 1e-6]):  # a 1e-6 turn of the ray: depths fp32 cannot hold (rays grazing a surface)
      dd, gg = _cast(mjw, m, d, pnt, (vec + torch.tensor(off, device="cuda")).contiguous(), groups)
      edge |= (gg != gid) | ((dd - dist).abs() > 1e-5 * dist.abs().clamp(min=1.0))
    n = pnt.shape[1]
    seg = rc.seg_data[:, int(rc.seg_adr[c]) : int(rc.seg_adr[c]) + n]
    depth = rc.depth_data[:, int(rc.depth_adr[c]) : int(rc.depth_adr[c]) + n]
    ok = ~edge
    if int(rc.cam_id_map[c]) not in ORTHOGRAPHIC:  # an orthographic camera casts one ray per world (render_util.py:88-89)
      assert edge.float().mean() < 0.01, f"camera {c}: {int(edge.sum())} knife-edge pixels"
    assert torch.equal(seg[..., 0][ok], gid[ok]), f"camera {c}: geom ids differ on {int((seg[..., 0] != gid)[ok].sum())} pixels"
    assert torch.equal(seg[..., 1][ok], torch.where(gid[ok] >= 0, 5, -1).to(torch.int32))
    hit = ok & (gid >= 0)
    want = dist * (-z)[None, :]
    # mjw.rays solves the quadratics of spheres, capsules, ellipsoids and cylinders from the camera, where fp32 cancellation costs
    # about (distance / size)^2 ulps (measured up to 3.5e-5 relative here); the renderer solves them from the geom's bounds and is held
    # to the reference at 1e-5 by test_render_matches_reference_images
    torch.testing.assert_close(depth[hit], want[hit], rtol=5e-5, atol=1e-5)
    assert (depth[ok & (gid < 0)] == 0).all()
    compared += int(ok.sum())
  return compared


def test_render_matches_rays():
  mjw, mjm, m, d, rc = _setup(render_scenes.PRIMITIVES)
  _frame(mjw, m, d, rc)
  assert _cross_check(mjw, m, d, rc) > 0
  seg = rc.seg_data[..., 0]
  hidden = mjm.names.geom.index("hidden")
  assert not (seg == hidden).any()
  # every rendered pixel is written: background pixels carry the packed background colour, hits are opaque
  rgb = rc.rgb_data.view(torch.int32)
  miss = rc.seg_data[:, : rgb.shape[1], 0] < 0
  assert (rgb[miss] == np.int32(np.uint32(rc.background_color).view(np.int32))).all()
  assert ((rgb >> 24) & 0xFF == 255).all()


def test_render_groups_and_culling():
  mjw, mjm, m, d, rc = _setup(render_scenes.PRIMITIVES, enabled_geom_groups=[0, 4], cam_active=["overview"])
  _frame(mjw, m, d, rc)
  _cross_check(mjw, m, d, rc, groups=(0, 4))
  # a camera inside a sphere: culled, the sphere's inside is invisible; not culled, every pixel sees it, as the unculled rays do
  for cull in (True, False):
    mjw, mjm, m, d, rc = _setup(render_scenes.NOLIGHT, cam_active=["inside"], enable_backface_culling=cull)
    _frame(mjw, m, d, rc)
    shell = mjm.names.geom.index("shell")
    seg = rc.seg_data[..., 0]
    if cull:
      assert not (seg == shell).any()
    else:
      assert (seg == shell).all()
      _cross_check(mjw, m, d, rc)


def test_render_reads_data_only_and_launches():
  mjw, mjm, m, d, rc = _setup(render_scenes.PRIMITIVES, use_shadows=True)
  before = {k: v.clone() for k, v in vars(d).items() if isinstance(v, torch.Tensor)}
  mjw.refit_bvh(m, d, rc)
  assert mjw.last_launch_count() == 1
  mjw.render(m, d, rc)
  assert mjw.last_launch_count() == 1
  torch.cuda.synchronize()
  for k, v in before.items():
    assert torch.equal(getattr(d, k), v), k
  first = [x.clone() for x in (rc.rgb_data.view(torch.int32), rc.depth_data, rc.seg_data)]
  _frame(mjw, m, d, rc)
  for a, b in zip(first, (rc.rgb_data.view(torch.int32), rc.depth_data, rc.seg_data)):
    assert torch.equal(a, b)  # deterministic


def test_render_shadows_lights_and_switches():
  """Shadows darken pixels without moving any geom; each shading switch changes the image only where it should."""
  base = None
  imgs = {}
  for key, kw in (("plain", {}), ("shadow", dict(use_shadows=True)), ("noamb", dict(use_ambient_lighting=False)), ("nospec", dict(enable_specular=False)),
                  ("noemis", dict(enable_emission=False)), ("noperlight", dict(enable_per_light_ambient=False))):
    mjw, mjm, m, d, rc = _setup(render_scenes.PRIMITIVES, cam_active=["overview"], **kw)
    _frame(mjw, m, d, rc)
    rgb = rc.rgb_data.view(torch.int32)
    imgs[key] = torch.stack([(rgb >> s) & 0xFF for s in (16, 8, 0)], -1).int()
    if base is None:
      base = rc.seg_data.clone()
    assert torch.equal(rc.seg_data, base), key
  for key in ("shadow", "noamb", "nospec", "noemis", "noperlight"):
    diff = imgs[key] - imgs["plain"]
    assert (diff != 0).any(), key
    assert (diff <= 0).all(), key  # each switch removes light


def test_render_no_lights_fallback_and_tracking_camera():
  mjw, mjm, m, d, rc = _setup(render_scenes.NOLIGHT, cam_active=["outside"])
  _frame(mjw, m, d, rc)
  _cross_check(mjw, m, d, rc)
  # no light and no headlight: a hit pixel is 0.3 x its rgba (render.py:967-968)
  rgb = rc.rgb_data.view(torch.int32)
  seg = rc.seg_data[..., 0]
  floor = mjm.names.geom.index("floor")
  px = rgb[seg == floor]
  assert px.numel() > 0 and (((px >> 16) & 0xFF) == int(0.3 * 0.5 * 255)).all()
  # the tracking camera follows the moving body after step()
  mjw, mjm, m, d, rc = _setup(render_scenes.PRIMITIVES, cam_active=["tracker"])
  _frame(mjw, m, d, rc)
  seg0, pos0 = rc.seg_data.clone(), d.cam_xpos[:, mjm.names.camera.index("tracker")].clone()
  d.qvel.copy_(torch.tensor([[1.5, 0.0]] * NWORLD, device="cuda"))
  for _ in range(20):
    mjw.step(m, d)
  _frame(mjw, m, d, rc)
  assert not torch.equal(d.cam_xpos[:, mjm.names.camera.index("tracker")], pos0)
  _cross_check(mjw, m, d, rc)
  assert rc.seg_data.shape == seg0.shape


def test_per_world_fields():
  """World w reads entry w % n of a per-world field; per-world cam_fovy works with use_precomputed_rays=False."""
  mjw, mjm, m, d, rc = _setup(render_scenes.PRIMITIVES, batch_sizes={"geom_rgba": 2, "light_diffuse": 2, "mat_rgba": 2, "cam_fovy": 2}, seed=5,
                              cam_active=["overview"], use_precomputed_rays=False)
  d.qpos.copy_(d.qpos[:1].expand_as(d.qpos))  # one pose in every world
  mjw.kinematics(m, d)
  mjw.camlight(m, d)
  m.geom_rgba[1, :, :3] = torch.rand(mjm.ngeom, 3, device="cuda")
  m.mat_rgba[1, :, :3] = torch.rand(mjm.nmat, 3, device="cuda")
  m.light_diffuse[1] *= 0.5
  _frame(mjw, m, d, rc)
  rgb, seg = rc.rgb_data.view(torch.int32), rc.seg_data
  assert torch.equal(rgb[0], rgb[2]) and torch.equal(rgb[1], rgb[3]) and not torch.equal(rgb[0], rgb[1])
  assert torch.equal(seg[0], seg[1])
  m.cam_fovy[1] = 30.0
  _frame(mjw, m, d, rc)
  assert not torch.equal(rc.seg_data[0], rc.seg_data[1]) and torch.equal(rc.seg_data[0], rc.seg_data[2])
  # world 1 at fovy 30 renders what an unbatched 30-degree camera with precomputed rays renders
  xml = render_scenes.PRIMITIVES.replace('fovy="50" resolution="31 23"', 'fovy="30" resolution="31 23"')
  mjw, mjm2, m2, d2, rc2 = _setup(xml, cam_active=["overview"])
  d2.qpos.copy_(d.qpos)
  mjw.kinematics(m2, d2)
  mjw.camlight(m2, d2)
  _frame(mjw, m2, d2, rc2)
  assert torch.equal(rc2.seg_data[1], rc.seg_data[1])
  torch.testing.assert_close(rc2.depth_data[1], rc.depth_data[1], rtol=1e-6, atol=1e-6)


def test_getters():
  mjw, mjm, m, d, rc = _setup(render_scenes.PRIMITIVES, cam_active=["overview", "sensor"])
  _frame(mjw, m, d, rc)
  for c in range(rc.nrender):
    w, h = rc.cam_res[c].tolist()
    a, n = int(rc.rgb_adr[c]), w * h
    rgb = torch.empty((NWORLD, h, w, 3), device="cuda")
    mjw.get_rgb(rc, c, rgb)
    raw = rc.rgb_data.view(torch.int32)[:, a : a + n].reshape(NWORLD, h, w)
    torch.testing.assert_close(rgb[..., 0], ((raw >> 16) & 0xFF).float() / 255.0)
    torch.testing.assert_close(rgb[..., 2], (raw & 0xFF).float() / 255.0)
    dep = torch.empty((NWORLD, h, w), device="cuda")
    mjw.get_depth(rc, c, 2.0, dep)
    da = int(rc.depth_adr[c])
    torch.testing.assert_close(dep, (rc.depth_data[:, da : da + n] / 2.0).clamp(0, 1).reshape(NWORLD, h, w))
    seg = torch.empty((NWORLD, h, w, 2), dtype=torch.int32, device="cuda")
    mjw.get_segmentation(rc, c, seg)
    sa = int(rc.seg_adr[c])
    assert torch.equal(seg, rc.seg_data[:, sa : sa + n].reshape(NWORLD, h, w, 2))
  with pytest.raises(ValueError, match="leading shape"):
    mjw.get_rgb(rc, 0, torch.empty((NWORLD, 3, 3, 3), device="cuda"))


def test_rays_with_render_context_still_refused():
  mjw, mjm, m, d, rc = _setup(render_scenes.PRIMITIVES, nworld=1)
  p = torch.zeros((1, 1, 3), device="cuda")
  with pytest.raises(NotImplementedError):
    mjw.ray(m, d, p, p, rc=rc)


@pytest.mark.parametrize("name", sorted(render_scenes.SCENES))
def test_render_matches_reference_images(name):
  """tests/golden/render_<name>.npz (tools/make_render_goldens.py: the reference's create_render_context / refit_bvh / render in fp64):
  away from knife-edge and shadow-edge entries, segmentation is equal, depth is within 1e-5 absolute and relative, and each colour
  channel within 2/255.  At most 0.1 % of a buffer's entries may be marked."""
  import json
  import os

  import mujoco_warp_b200 as mjw

  g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"render_{name}.npz"))
  sc = render_scenes.SCENES[name]
  kw = json.loads(str(g["kwargs"]))
  mjm = mjw.mjcf.load_string(sc["xml"])
  batch = {k[len("batch/"):]: g[k] for k in g.files if k.startswith("batch/")}
  m = mjw.put_model(mjm, batch_sizes={k: v.shape[0] for k, v in batch.items()})
  for k, v in batch.items():
    getattr(m, k).copy_(torch.from_numpy(v.astype(np.float32)))
  nw = g["qpos"].shape[0]
  d = mjw.make_data(mjm, nworld=nw, m=m)
  d.qpos.copy_(torch.from_numpy(g["qpos"].astype(np.float32)))
  mjw.kinematics(m, d)
  mjw.camlight(m, d)
  for k in ("geom_xpos", "geom_xmat", "cam_xpos", "cam_xmat", "light_xpos", "light_xdir"):
    # the fixture's fp32 poses (the kinematics agree to the last bits; the renderer alone is under test)
    x = getattr(d, k)
    torch.testing.assert_close(x.reshape(nw, -1).double().cpu(), torch.from_numpy(g["pose/" + k]), rtol=1e-5, atol=1e-5)
    x.copy_(torch.from_numpy(g["pose/" + k].astype(np.float32)).reshape(x.shape))
  rc = mjw.create_render_context(mjm, nworld=nw, **kw)
  for k in ("rgb_adr", "depth_adr", "seg_adr", "cam_res"):
    np.testing.assert_array_equal(getattr(rc, k).cpu().numpy().reshape(g[k].shape), g[k], err_msg=k)
  _frame(mjw, m, d, rc)
  rgb = rc.rgb_data.view(torch.int32).cpu().numpy().astype(np.int64) & 0xFFFFFFFF
  depth, seg = rc.depth_data.cpu().numpy().astype(np.float64), rc.seg_data.cpu().numpy().astype(np.int64)
  mark_rgb, mark_seg, mark_depth = g["knife_rgb"] | g["shadow_rgb"], g["knife_seg"] | g["shadow_seg"], g["knife_depth"]
  for what, mark in (("rgb", mark_rgb), ("depth", mark_depth), ("seg", mark_seg)):
    assert mark.mean() <= 1e-3 if mark.size else True, f"{name}: {int(mark.sum())} of {mark.size} {what} entries marked"
  ok = ~mark_seg
  assert np.array_equal(seg[ok], g["seg"][ok]), f"{name}: segmentation differs on {int((seg != g['seg']).any(-1)[ok].sum())} pixels"
  ok = ~mark_depth
  err = np.abs(depth - g["depth"])[ok]
  bad = np.nonzero(~(err <= 1e-5 + 1e-5 * np.abs(g["depth"][ok])))[0]
  assert not len(bad), f"{name}: depth error {err.max():.3g} at {[(int(i), float(g['depth'][ok][i]), float(depth[ok][i])) for i in bad[:5]]}"
  ch = lambda x: np.stack([(x >> s) & 0xFF for s in (24, 16, 8, 0)], -1)
  cerr = np.abs(ch(rgb) - ch(g["rgb"]))[~mark_rgb]
  assert (cerr <= 2).all(), f"{name}: {int((cerr > 2).any(-1).sum())} pixels differ by more than 2/255 (max {cerr.max()})"
  print(f"{name}: depth max error {err.max() if err.size else 0:.3g}, rgb max channel error {cerr.max() if cerr.size else 0}/255, "
        f"rgb pixels off by 1 or 2: {int((cerr > 0).any(-1).sum())} of {cerr.shape[0]}, marked rgb/depth/seg {int(mark_rgb.sum())}/{int(mark_depth.sum())}/{int(mark_seg.sum())}")
