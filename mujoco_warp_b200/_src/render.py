"""Batch rendering: one RGB, depth and segmentation image per (world, camera), on the GPU (reference render.py, render_util.py, bvh.py).

`create_render_context` lays out the output buffers and the camera rays once; `refit_bvh` writes every world's geom bounds from the
poses of the last kinematics; `render` then shades every pixel in one kernel (k_render.cu).  As in the reference, `render` does not
refit by itself: call `refit_bvh` after the poses change.  `get_rgb` / `get_depth` / `get_segmentation` copy one camera's image out
of the packed buffers.  Nothing here allocates or synchronises after the context exists, so a frame can be captured in a CUDA graph.

Not implemented: textures (a model whose materials reference one needs use_textures=False, which renders the material's rgba), the
skybox, Gaussian splats, flex and height fields.  The reference's BVH is replaced by a bounds test of every enabled geom.
"""

from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .io import render_fields
from .types import Data, Model, RenderContext

_CAMOUT_RGB, _CAMOUT_DEPTH, _CAMOUT_SEG = 1, 2, 16  # mjtCamOutBit


class _Render(ctypes.Structure):
  """include/mjb200.h mjbRender"""

  _fields_ = [(n, ctypes.c_int) for n in ("ncam", "ngeom", "npixel", "nrgb", "ndepth", "nseg")] + [
    (n, ctypes.c_void_p) for n in ("cam_id", "cam_res", "pix_adr", "rgb_adr", "depth_adr", "seg_adr", "ray", "geom_id", "mesh_half", "lower", "upper",
                                   "rgb", "depth", "seg", "cam_projection", "cam_fovy", "cam_sensorsize", "cam_intrinsic")
  ] + [("nb_cam_fovy", ctypes.c_int), ("nb_cam_intrinsic", ctypes.c_int), ("nlight", ctypes.c_int)] + [
    (n, ctypes.c_void_p) for n in ("light_type", "light_castshadow", "light_active", "light_attenuation", "light_cutoff", "light_exponent",
                                   "light_ambient", "light_diffuse", "light_specular")
  ] + [(f"nb_light_{n}", ctypes.c_int) for n in ("attenuation", "cutoff", "exponent", "ambient", "diffuse", "specular")] + [
    (n, ctypes.c_void_p) for n in ("mat_specular", "mat_shininess", "mat_emission")
  ] + [(f"nb_mat_{n}", ctypes.c_int) for n in ("specular", "shininess", "emission")] + [
    (n, ctypes.c_int) for n in ("use_shadows", "use_ambient_lighting", "enable_per_light_ambient", "enable_specular", "enable_emission",
                                "enable_backface_culling", "headlight_active", "light_attenuation_is_default", "has_spot_lights")
  ] + [("background_color", ctypes.c_uint), ("znear", ctypes.c_float)] + [(n, ctypes.c_float * 3) for n in ("headlight_ambient", "headlight_diffuse", "headlight_specular")]


def pack_rgba_to_uint32(r: float, g: float, b: float, a: float) -> int:
  """render_util.py:133: channels in [0, 255] packed as 0xAARRGGBB (truncated)"""
  return (int(a) << 24) | (int(r) << 16) | (int(g) << 8) | int(b)


def _device() -> torch.device:
  return torch.device("cuda", torch.cuda.current_device())


def _stream() -> ctypes.c_void_p:
  return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _per_camera(value, name, ncam, ncam_model, active, default):
  """render_rgb / render_depth / render_seg as render_util.py:514-548 reads them: None (the model's cam_output), a bool, or a list of
  one entry, one per active camera or one per model camera"""
  if value is None:
    return list(default)
  if isinstance(value, (bool, np.bool_)):
    return [bool(value)] * ncam
  value = list(value)
  if len(value) == ncam_model and ncam != ncam_model:
    value = [value[i] for i in active]
  elif len(value) == 1 and ncam > 1:
    value = value * ncam
  if len(value) != ncam:
    raise ValueError(f"{name} length ({len(value)}) does not match active camera count ({ncam}).")
  return [bool(x) for x in value]


def _camera_names(mjm):
  names = getattr(getattr(mjm, "names", None), "camera", None)
  if names is not None:
    return list(names)
  return [mjm.camera(i).name for i in range(int(mjm.ncam))]


def create_render_context(mjm, nworld: int = 1, cam_res=None, render_rgb=None, render_depth=None, render_seg=None, use_textures: bool = True,
                          use_fast_math: bool = True, use_shadows: bool = False, use_ambient_lighting: bool = True, enabled_geom_groups=(0, 1, 2),
                          cam_active=None, background_color=(0.1, 0.1, 0.2, 1.0), flex_render_smooth: bool = True, use_precomputed_rays: bool = True,
                          render_skybox: bool = False, enable_backface_culling: bool = True, enable_specular: bool = True, enable_emission: bool = True,
                          enable_per_light_ambient: bool = True, splat_position=None, splat_rotation=None, splat_scale=None, splat_rgba=None,
                          splat_adr=None, splat_group_id=None) -> RenderContext:
  """Creates a render context on the current CUDA device (reference render_util.py:272; same arguments and meaning).

  cam_active: bools (one per model camera), camera names or camera ids; None = every camera.  cam_res: (width, height) for every
  active camera, or a list of one per active camera; None = the model's cam_resolution.  render_rgb / render_depth / render_seg: a
  bool, or a list per active (or per model) camera; None = the model's cam_output bits (RGB only for models without them).
  use_precomputed_rays: the camera-frame rays are computed once here from the model's cam_fovy / cam_intrinsic; per-world values of
  those fields (put_model batch_sizes) therefore need use_precomputed_rays=False, which computes each world's rays in render().
  use_fast_math and flex_render_smooth only tune the reference's code and are accepted.

  Raises NotImplementedError for use_textures=True on a model whose materials reference a texture (pass use_textures=False to
  render the material's rgba), for render_skybox=True and for any splat_* argument."""
  splats = dict(splat_position=splat_position, splat_rotation=splat_rotation, splat_scale=splat_scale, splat_rgba=splat_rgba, splat_adr=splat_adr,
                splat_group_id=splat_group_id)
  given = [k for k, v in splats.items() if v is not None]
  if given:
    raise NotImplementedError(f"Gaussian splat rendering ({', '.join(given)}) is not implemented")
  if render_skybox:
    raise NotImplementedError("render_skybox=True: skybox rendering is not implemented")
  rf = render_fields(mjm)
  textured = np.nonzero(rf["mat_texid"][:, 1] >= 0)[0]  # the RGB role, the one the reference samples (render.py:926)
  if use_textures and len(textured):
    raise NotImplementedError(f"use_textures=True: textures are not implemented (material(s) {textured.tolist()} reference one); pass use_textures=False to "
                              "render each material's rgba")
  if int(getattr(mjm, "nflex", 0)):
    raise NotImplementedError("flex rendering is not implemented")
  nworld = int(nworld)
  if nworld < 1:
    raise ValueError(f"nworld must be >= 1, got {nworld}")
  ncam_model = int(mjm.ncam)

  if cam_active is None:
    active = list(range(ncam_model))
  elif len(cam_active) > 0 and isinstance(cam_active[0], (bool, np.bool_)):
    if len(cam_active) != ncam_model:
      raise ValueError(f"cam_active must have length {ncam_model} (got {len(cam_active)})")
    active = [int(i) for i in np.nonzero(np.asarray(cam_active, dtype=bool))[0]]
  elif len(cam_active) > 0 and isinstance(cam_active[0], str):
    names = _camera_names(mjm)
    active = []
    for name in cam_active:
      if name not in names:
        raise ValueError(f"Camera '{name}' not found in model.")
      active.append(names.index(name))
  elif len(cam_active) > 0 and isinstance(cam_active[0], (int, np.integer)):
    active = [int(x) for x in cam_active]
    bad = [c for c in active if not 0 <= c < ncam_model]
    if bad:
      raise ValueError(f"cam_active: camera ids {bad} out of range [0, {ncam_model})")
  else:
    raise ValueError(f"Invalid cam_active format: {cam_active}")
  ncam = len(active)

  if cam_res is not None:
    if isinstance(cam_res, tuple):
      cam_res = [cam_res] * ncam
    elif isinstance(cam_res, list) and len(cam_res) == 1 and ncam > 1:
      cam_res = cam_res * ncam
    if len(cam_res) != ncam:
      raise ValueError(f"Camera resolutions count ({len(cam_res)}) does not match active camera count ({ncam}).")
    res = np.asarray(cam_res, dtype=np.int64).reshape(ncam, 2)
  else:
    res = rf["cam_resolution"][active].astype(np.int64).reshape(ncam, 2)
  if (res < 1).any():
    raise ValueError(f"camera resolutions must be at least 1 x 1, got {res.tolist()}")

  out = np.asarray(getattr(mjm, "cam_output", np.full(ncam_model, _CAMOUT_RGB)), dtype=np.int64).reshape(ncam_model)
  flags = {}
  for name, value, bit in (("render_rgb", render_rgb, _CAMOUT_RGB), ("render_depth", render_depth, _CAMOUT_DEPTH), ("render_seg", render_seg, _CAMOUT_SEG)):
    flags[name] = _per_camera(value, name, ncam, ncam_model, active, [bool(out[c] & bit) for c in active])

  npix = res[:, 0] * res[:, 1]
  pix_adr = np.concatenate([[0], np.cumsum(npix)[:-1]]).astype(np.int64) if ncam else np.zeros(0, dtype=np.int64)
  adr = {}
  for name in ("render_rgb", "render_depth", "render_seg"):
    a, n = -np.ones(ncam, dtype=np.int64), 0
    for i in range(ncam):
      if flags[name][i]:
        a[i], n = n, n + int(npix[i])
    adr[name] = (a, n)
  total = int(npix.sum())

  groups = [int(x) for x in enabled_geom_groups]
  geom_group = np.asarray(getattr(mjm, "geom_group", np.zeros(int(mjm.ngeom))), dtype=np.int64).reshape(-1)
  enabled = np.nonzero(np.isin(geom_group, groups))[0]
  nmesh = int(getattr(mjm, "nmesh", 0))
  half = np.zeros((nmesh, 3))
  for i in range(nmesh):  # bvh.py:427 build_mesh_bvh: half the extent of the mesh's vertex box
    v = np.asarray(mjm.mesh_vert).reshape(-1, 3)[int(mjm.mesh_vertadr[i]) : int(mjm.mesh_vertadr[i]) + int(mjm.mesh_vertnum[i])]
    half[i] = 0.5 * (v.max(axis=0) - v.min(axis=0))

  nlight = int(getattr(mjm, "nlight", 0))
  light_type = rf["light_type"]
  hl = getattr(getattr(mjm, "vis", None), "headlight", None)
  hl_get = lambda k, dflt: np.asarray(getattr(hl, k, dflt) if hl is not None else dflt, dtype=np.float64)
  vmap, stat = getattr(getattr(mjm, "vis", None), "map", None), getattr(mjm, "stat", None)
  # the ray direction does not depend on znear (every frustum term scales with it); MuJoCo's value where the model has one
  znear = float(getattr(vmap, "znear", 0.01)) * float(getattr(stat, "extent", 1.0))

  dev = _device()
  i32 = lambda a: torch.as_tensor(np.asarray(a, dtype=np.int32), device=dev)
  f32 = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32), device=dev)
  rgb_adr, nrgb = adr["render_rgb"]
  depth_adr, ndepth = adr["render_depth"]
  seg_adr, nseg = adr["render_seg"]
  bg = [float(x) for x in background_color]
  rc = RenderContext(
    nrender=ncam, cam_id_map=i32(active), cam_res=i32(res), pix_adr=i32(pix_adr), total_rays=total,
    render_rgb=flags["render_rgb"], render_depth=flags["render_depth"], render_seg=flags["render_seg"],
    rgb_adr=i32(rgb_adr), depth_adr=i32(depth_adr), seg_adr=i32(seg_adr),
    rgb_data=torch.zeros((nworld, nrgb), dtype=torch.int32, device=dev).view(torch.uint32),
    depth_data=torch.zeros((nworld, ndepth), dtype=torch.float32, device=dev),
    seg_data=torch.full((nworld, max(nseg, 1), 2), -1, dtype=torch.int32, device=dev),
    bvh_ngeom=len(enabled), enabled_geom_ids=i32(enabled), mesh_bounds_size=f32(half),
    lower=torch.zeros((nworld, len(enabled), 3), dtype=torch.float32, device=dev), upper=torch.zeros((nworld, len(enabled), 3), dtype=torch.float32, device=dev),
    nworld=nworld, use_textures=bool(use_textures), use_fast_math=bool(use_fast_math), use_shadows=bool(use_shadows), use_ambient_lighting=bool(use_ambient_lighting),
    enabled_geom_groups=groups, background_color=pack_rgba_to_uint32(bg[0] * 255.0, bg[1] * 255.0, bg[2] * 255.0, bg[3] * 255.0),
    flex_render_smooth=bool(flex_render_smooth), use_precomputed_rays=bool(use_precomputed_rays), render_skybox=False,
    enable_backface_culling=bool(enable_backface_culling), enable_specular=bool(enable_specular), enable_emission=bool(enable_emission),
    enable_per_light_ambient=bool(enable_per_light_ambient), znear=znear,
    headlight_active=bool(int(hl_get("active", 1))), headlight_ambient=hl_get("ambient", [0.1] * 3).reshape(3).tolist(),
    headlight_diffuse=hl_get("diffuse", [0.4] * 3).reshape(3).tolist(), headlight_specular=hl_get("specular", [0.5] * 3).reshape(3).tolist(),
    light_attenuation_is_default=bool(nlight == 0 or np.allclose(rf["light_attenuation"].astype(np.float32), np.array([1.0, 0.0, 0.0], dtype=np.float32))),
    has_spot_lights=bool(nlight and (light_type == 0).any()),
    ray=torch.zeros((total, 3), dtype=torch.float32, device=dev),
  )
  rc._host = dict(cam_res=res, rgb=rgb_adr, depth=depth_adr, segmentation=seg_adr)  # get_* check shapes without reading the device
  if use_precomputed_rays and total:
    cams = {k: f32(rf[k]) if rf[k].dtype == np.float64 else i32(rf[k]) for k in ("cam_projection", "cam_fovy", "cam_sensorsize", "cam_intrinsic")}
    s = _struct(rc, cams, None)
    _lib.check(_lib.lib().mjb_render_rays(ctypes.byref(s), rc.ray.data_ptr(), _stream()))
  return rc


def _nb(x: torch.Tensor) -> int:
  return max(int(x.shape[0]), 1) if x.dim() > 1 or x.numel() == 0 else 1


def _struct(rc: RenderContext, m, nlight) -> _Render:
  """The mjbRender of rc with the camera / light / material fields of `m` (a Model, or a dict of the camera fields alone).  A batched
  field's leading size is its number of per-world entries."""
  get = (lambda n: m[n]) if isinstance(m, dict) else (lambda n: getattr(m, n))
  s = _Render()
  s.ncam, s.ngeom, s.npixel = rc.nrender, rc.bvh_ngeom, rc.total_rays
  s.nrgb, s.ndepth, s.nseg = int(rc.rgb_data.shape[1]), int(rc.depth_data.shape[1]), int(rc.seg_data.shape[1])
  for n in ("cam_res", "pix_adr", "rgb_adr", "depth_adr", "seg_adr", "lower", "upper"):
    setattr(s, n, getattr(rc, n).data_ptr())
  s.cam_id, s.geom_id, s.mesh_half = rc.cam_id_map.data_ptr(), rc.enabled_geom_ids.data_ptr(), rc.mesh_bounds_size.data_ptr()
  s.ray = rc.ray.data_ptr() if rc.use_precomputed_rays and nlight is not None else None
  s.rgb, s.depth, s.seg = rc.rgb_data.data_ptr(), rc.depth_data.data_ptr(), rc.seg_data.data_ptr()
  for n in ("cam_projection", "cam_sensorsize"):
    setattr(s, n, get(n).data_ptr())
  s.cam_fovy, s.cam_intrinsic = get("cam_fovy").data_ptr(), get("cam_intrinsic").data_ptr()
  # the dict form holds the model's unbatched values: one entry
  s.nb_cam_fovy = 1 if isinstance(m, dict) else _nb(m.cam_fovy)
  s.nb_cam_intrinsic = 1 if isinstance(m, dict) else (int(m.cam_intrinsic.shape[0]) if m.cam_intrinsic.dim() == 3 else 1)
  s.nb_light_cutoff = s.nb_light_exponent = s.nb_light_attenuation = s.nb_light_ambient = s.nb_light_diffuse = s.nb_light_specular = 1
  s.nb_mat_specular = s.nb_mat_shininess = s.nb_mat_emission = 1
  if nlight is not None:
    s.nlight = nlight
    for n in ("light_type", "light_castshadow", "light_active", "light_attenuation", "light_cutoff", "light_exponent", "light_ambient", "light_diffuse",
              "light_specular", "mat_specular", "mat_shininess", "mat_emission"):
      setattr(s, n, get(n).data_ptr())
    for n, vec in (("light_attenuation", True), ("light_ambient", True), ("light_diffuse", True), ("light_specular", True), ("light_cutoff", False),
                   ("light_exponent", False), ("mat_specular", False), ("mat_shininess", False), ("mat_emission", False)):
      x = get(n)
      setattr(s, "nb_" + n, max(int(x.shape[0]), 1) if x.dim() == (3 if vec else 2) else 1)
  s.use_shadows, s.use_ambient_lighting, s.enable_per_light_ambient = int(rc.use_shadows), int(rc.use_ambient_lighting), int(rc.enable_per_light_ambient)
  s.enable_specular, s.enable_emission, s.enable_backface_culling = int(rc.enable_specular), int(rc.enable_emission), int(rc.enable_backface_culling)
  s.headlight_active, s.light_attenuation_is_default, s.has_spot_lights = int(rc.headlight_active), int(rc.light_attenuation_is_default), int(rc.has_spot_lights)
  s.background_color, s.znear = rc.background_color, rc.znear
  s.headlight_ambient[:], s.headlight_diffuse[:], s.headlight_specular[:] = rc.headlight_ambient, rc.headlight_diffuse, rc.headlight_specular
  return s


def _check_pair(m: Model, d: Data, rc: RenderContext):
  if d._model is not m and d._model._handle != m._handle:
    raise ValueError("Data was created for a different Model")
  if rc.nworld != d.nworld:
    raise ValueError(f"the render context was created for {rc.nworld} worlds, the Data has {d.nworld}")


def refit_bvh(m: Model, d: Data, rc: RenderContext):
  """Writes rc.lower / rc.upper, the world-space bounds of every enabled geom in every world, from the geom poses of the last
  kinematics (reference bvh.py:39; the bounds of bvh.py:178 _compute_bvh_bounds).  One kernel launch."""
  _check_pair(m, d, rc)
  s = _struct(rc, m, m.nlight)
  _lib.check(_lib.lib().mjb_refit_bvh(m._handle, d._handle, ctypes.byref(s), _stream()))


def render(m: Model, d: Data, rc: RenderContext):
  """Renders every active camera of every world into rc.rgb_data / depth_data / seg_data (reference render.py:656).

  Reads geom_xpos / geom_xmat, cam_xpos / cam_xmat and light_xpos / light_xdir of the last kinematics and the bounds of the last
  `refit_bvh`; writes no Data field.  One kernel launch."""
  _check_pair(m, d, rc)
  s = _struct(rc, m, m.nlight)
  _lib.check(_lib.lib().mjb_render(m._handle, d._handle, ctypes.byref(s), _stream()))


def _image(rc: RenderContext, camera_index: int, out: torch.Tensor, what: str):
  if not 0 <= camera_index < rc.nrender:
    raise ValueError(f"camera_index {camera_index} out of range [0, {rc.nrender})")
  a = int(rc._host[what][camera_index])
  if a < 0:
    raise ValueError(f"camera {camera_index} does not render {what}")
  w, h = (int(x) for x in rc._host["cam_res"][camera_index])
  if out.shape[:3] != (rc.nworld, h, w):
    raise ValueError(f"{what} output: expected leading shape ({rc.nworld}, {h}, {w}), got {tuple(out.shape)}")
  return a, h * w


def get_rgb(rc: RenderContext, camera_index: int, rgb_out: torch.Tensor):
  """Camera `camera_index`'s RGB image, unpacked to float32 in [0, 1], into rgb_out (nworld, height, width, 3) (render_util.py:181)."""
  a, n = _image(rc, camera_index, rgb_out, "rgb")
  v = rc.rgb_data.view(torch.int32)[:, a : a + n]
  for k, shift in enumerate((16, 8, 0)):
    rgb_out[..., k].copy_(((v >> shift) & 0xFF).to(torch.float32).mul_(1.0 / 255.0).view(rgb_out.shape[:3]))


def get_depth(rc: RenderContext, camera_index: int, depth_scale: float, depth_out: torch.Tensor):
  """Camera `camera_index`'s depth divided by depth_scale and clamped to [0, 1], into depth_out (nworld, height, width)
  (render_util.py:197)."""
  a, n = _image(rc, camera_index, depth_out, "depth")
  depth_out.copy_((rc.depth_data[:, a : a + n] / depth_scale).clamp_(0.0, 1.0).view(depth_out.shape))


def get_segmentation(rc: RenderContext, camera_index: int, seg_out: torch.Tensor):
  """Camera `camera_index`'s (geom id, mjOBJ_GEOM) pairs, (-1, -1) for background, into seg_out (nworld, height, width, 2) int32
  (render_util.py:233)."""
  a, n = _image(rc, camera_index, seg_out, "segmentation")
  seg_out.copy_(rc.seg_data[:, a : a + n].view(seg_out.shape))
