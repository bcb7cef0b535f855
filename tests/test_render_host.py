"""The renderer without a GPU: the compiler's camera / light / material fields, create_render_context's host logic against a stub
library, and a host build of csrc/mjb_render.cuh against the reference's known answers (tests/golden/render_vectors.npz, written
by tools/make_render_goldens.py)."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import render_scenes, util

HERE = os.path.dirname(os.path.abspath(__file__))
HARNESS = os.path.join(HERE, "host_harness")
BUILD = os.path.join(HARNESS, "_build")
CSRC = os.path.join(os.path.dirname(HERE), "mujoco_warp_b200", "csrc")
GOLDEN = os.path.join(HERE, "golden", "render_vectors.npz")


def host_lib():
  src, out = os.path.join(HARNESS, "render_host.cpp"), os.path.join(BUILD, "librender_host.so")
  deps = [src] + [os.path.join(CSRC, f) for f in ("mjb_render.cuh", "mjb_math.cuh", "mjb_types.cuh")]
  if not os.path.exists(out) or any(os.path.getmtime(p) > os.path.getmtime(out) for p in deps):
    os.makedirs(BUILD, exist_ok=True)
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-ffp-contract=off", f"-I{cuda_inc}", src, "-o", out], check=True)
  return ctypes.CDLL(out)


def _ptr(a):
  return a.ctypes.data_as(ctypes.c_void_p)


# ---------------------------------------------------------------- compiler


def test_compiler_fields_and_defaults():
  from mujoco_warp_b200._src import mjcf

  m = mjcf.load_string(render_scenes.PRIMITIVES)
  cam = m.names.camera
  ov, orth, sen, trk = (cam.index(n) for n in ("overview", "ortho", "sensor", "tracker"))
  assert m.cam_projection.tolist() == [0, 1, 0, 0] and m.cam_projection[orth] == 1
  np.testing.assert_array_equal(m.cam_fovy, [50.0, 4.0, 45.0, 45.0])
  np.testing.assert_array_equal(m.cam_resolution[[ov, orth, sen, trk]], [[31, 23], [17, 13], [25, 19], [21, 15]])
  np.testing.assert_array_equal(m.cam_sensorsize[sen], [0.006, 0.004])
  np.testing.assert_array_equal(m.cam_sensorsize[ov], [0.0, 0.0])
  # focalpixel 20 px on a 25 x 19 image of a 6 x 4 mm sensor
  np.testing.assert_allclose(m.cam_intrinsic[sen], [20 / 25 * 0.006, 20 / 19 * 0.004, 0.0, 0.0])
  lt = m.names.light
  sun, spot, bulb, follow = (lt.index(n) for n in ("sun", "spot", "bulb", "follow"))
  assert m.light_type[[sun, spot, bulb, follow]].tolist() == [1, 0, 2, 0]
  assert m.light_castshadow[[sun, bulb, follow]].tolist() == [1, 0, 1] and m.light_active.tolist() == [1, 1, 1, 1]
  np.testing.assert_array_equal(m.light_attenuation[bulb], [1, 0.2, 0.05])
  np.testing.assert_array_equal(m.light_attenuation[sun], [1, 0.05, 0.01])  # <default><light attenuation=...>
  np.testing.assert_array_equal(m.light_cutoff[[spot, bulb, follow]], [35, 45, 60])
  np.testing.assert_array_equal(m.light_exponent[[spot, bulb]], [4, 10])
  np.testing.assert_array_equal(m.light_ambient[spot], [0.05] * 3)
  np.testing.assert_array_equal(m.light_ambient[sun], [0.0] * 3)
  np.testing.assert_array_equal(m.light_diffuse[follow], [0.2] * 3)
  np.testing.assert_array_equal(m.light_specular[[sun, spot]], [[0.3] * 3, [0.4] * 3])
  mats = m.names.material
  gl, gw, fl = (mats.index(n) for n in ("gloss", "glow", "floor"))
  np.testing.assert_array_equal(m.mat_specular[[gl, gw, fl]], [0.9, 0.1, 0.5])
  np.testing.assert_array_equal(m.mat_shininess[[gl, gw, fl]], [0.8, 0.2, 0.5])
  np.testing.assert_array_equal(m.mat_emission[[gl, gw, fl]], [0.0, 0.6, 0.0])
  assert (m.mat_texid == -1).all() and m.mat_texid.shape == (3, 10)
  assert m.geom_matid[m.names.geom.index("cap")] == gl  # <default class="shiny"><geom material=...>
  hl = m.vis.headlight
  assert hl.active == 1
  np.testing.assert_array_equal(np.vstack([hl.ambient, hl.diffuse, hl.specular]), [[0.15] * 3, [0.3] * 3, [0.2] * 3])
  n = mjcf.load_string(render_scenes.NOLIGHT)
  assert n.vis.headlight.active == 0 and n.nlight == 0
  np.testing.assert_array_equal(n.vis.headlight.diffuse, [0.4] * 3)
  np.testing.assert_array_equal(n.cam_fovy, [45.0, 45.0])


def test_compiler_legacy_attributes_classes_and_textures(tmp_path):
  from mujoco_warp_b200._src import mjcf

  xml = """<mujoco><default><camera fovy="30"/><default class="d"><light castshadow="false" type="point"/></default></default>
    <asset><texture name="t" type="2d" builtin="checker" width="8" height="8"/><material name="tm" texture="t"/></asset>
    <worldbody><camera name="o" orthographic="true"/><camera name="p" fovy="70"/><light name="a" directional="true"/><light name="b" class="d" active="false"/>
    <geom type="sphere" size="0.1" material="tm"/></worldbody></mujoco>"""
  m = mjcf.load_string(xml)
  assert m.cam_projection.tolist() == [1, 0]
  np.testing.assert_array_equal(m.cam_fovy, [30.0, 70.0])
  assert m.light_type.tolist() == [1, 2] and m.light_castshadow.tolist() == [1, 0] and m.light_active.tolist() == [1, 0]
  assert m.mat_texid[:, 1].tolist() == [0] and (m.mat_texid[:, [0, *range(2, 10)]] == -1).all()
  with pytest.raises(ValueError, match="projection"):
    mjcf.load_string('<mujoco><worldbody><camera projection="fisheye"/></worldbody></mujoco>')
  with pytest.raises(ValueError, match="light type"):
    mjcf.load_string('<mujoco><worldbody><light type="laser"/></worldbody></mujoco>')
  path = str(tmp_path / "m.npz")
  mjcf.save_npz(m, path)
  r = mjcf.load_npz(path)
  assert r.vis.headlight.active == 1 and r.mat_texid[:, 1].tolist() == [0] and r.light_type.tolist() == [1, 2]


def test_committed_models_get_the_defaults():
  """test_data/*.npz were compiled before the renderer's fields existed: put_model / create_render_context see MuJoCo's defaults."""
  from mujoco_warp_b200._src import io as mio
  from mujoco_warp_b200._src import mjcf

  mjm = mjcf.load_any(util.HUMANOID)
  assert not hasattr(mjm, "cam_fovy") and not hasattr(mjm, "light_type")
  rf = mio.render_fields(mjm)
  nc, nl = mjm.ncam, mjm.nlight
  np.testing.assert_array_equal(rf["cam_fovy"], [45.0] * nc)
  np.testing.assert_array_equal(rf["cam_resolution"], [[1, 1]] * nc)
  np.testing.assert_array_equal(rf["cam_projection"], [0] * nc)
  np.testing.assert_array_equal(rf["light_type"], [0] * nl)
  np.testing.assert_array_equal(rf["light_castshadow"], [1] * nl)
  np.testing.assert_array_equal(rf["light_attenuation"], [[1, 0, 0]] * nl)
  np.testing.assert_array_equal(rf["light_diffuse"], [[0.7] * 3] * nl)
  np.testing.assert_array_equal(rf["light_specular"], [[0.3] * 3] * nl)
  assert rf["mat_texid"].shape == (getattr(mjm, "nmat", 0), 10)


# ---------------------------------------------------------------- create_render_context against a stub library


@pytest.fixture
def stub(monkeypatch):
  import torch

  from mujoco_warp_b200._src import _lib
  from mujoco_warp_b200._src import render as mr

  calls = []

  class Stub:
    def __getattr__(self, name):
      def f(*a, **k):
        calls.append(name)
        return 0

      return f

  monkeypatch.setattr(_lib, "lib", lambda: Stub())
  monkeypatch.setattr(mr, "_device", lambda: torch.device("cpu"))
  monkeypatch.setattr(mr, "_stream", lambda: None)
  return calls


def test_context_layout(stub):
  from mujoco_warp_b200._src import mjcf
  from mujoco_warp_b200._src.render import create_render_context

  mjm = mjcf.load_string(render_scenes.PRIMITIVES)
  rc = create_render_context(mjm, nworld=3, render_rgb=True, render_depth=[True, False, True, False], render_seg=[False, True, True, True])
  npix = [31 * 23, 17 * 13, 25 * 19, 21 * 15]
  assert rc.nrender == 4 and rc.total_rays == sum(npix)
  assert rc.cam_id_map.tolist() == [0, 1, 2, 3]
  assert rc.pix_adr.tolist() == [0, npix[0], npix[0] + npix[1], sum(npix[:3])]
  assert rc.rgb_adr.tolist() == [0, npix[0], npix[0] + npix[1], sum(npix[:3])]
  assert rc.depth_adr.tolist() == [0, -1, npix[0], -1]
  assert rc.seg_adr.tolist() == [-1, 0, npix[1], npix[1] + npix[2]]
  assert tuple(rc.rgb_data.shape) == (3, sum(npix)) and str(rc.rgb_data.dtype) == "torch.uint32"
  assert tuple(rc.depth_data.shape) == (3, npix[0] + npix[2])
  assert tuple(rc.seg_data.shape) == (3, sum(npix[1:]), 2)
  assert tuple(rc.ray.shape) == (sum(npix), 3)
  assert stub.count("mjb_render_rays") == 1
  # groups 0-2: the group-4 sphere is not rendered
  hidden = mjm.names.geom.index("hidden")
  assert hidden not in rc.enabled_geom_ids.tolist() and rc.bvh_ngeom == mjm.ngeom - 1
  assert tuple(rc.lower.shape) == (3, mjm.ngeom - 1, 3)
  rc = create_render_context(mjm, enabled_geom_groups=[4])
  assert rc.enabled_geom_ids.tolist() == [hidden]
  # half the box of the compiled mesh's vertices (the compiler moves them to the mesh's inertial frame, as MuJoCo does)
  v = np.asarray(mjm.mesh_vert).reshape(-1, 3)
  np.testing.assert_allclose(rc.mesh_bounds_size.numpy(), [0.5 * (v.max(axis=0) - v.min(axis=0))], rtol=1e-6)
  assert rc.background_color == (255 << 24) | (int(0.1 * 255) << 16) | (int(0.1 * 255) << 8) | int(0.2 * 255)
  assert rc.headlight_active and rc.headlight_ambient == pytest.approx([0.15] * 3)
  assert not rc.light_attenuation_is_default and rc.has_spot_lights


def test_context_cam_active_and_res(stub):
  from mujoco_warp_b200._src import mjcf
  from mujoco_warp_b200._src.render import create_render_context

  mjm = mjcf.load_string(render_scenes.PRIMITIVES)
  by_bool = create_render_context(mjm, cam_active=[False, True, False, True])
  by_name = create_render_context(mjm, cam_active=["ortho", "tracker"])
  by_id = create_render_context(mjm, cam_active=[1, 3])
  for rc in (by_bool, by_name, by_id):
    assert rc.cam_id_map.tolist() == [1, 3] and rc.cam_res.tolist() == [[17, 13], [21, 15]]
  rc = create_render_context(mjm, cam_active=["tracker"], cam_res=(8, 6), render_depth=[False, False, False, True])
  assert rc.cam_res.tolist() == [[8, 6]] and rc.total_rays == 48 and rc.depth_adr.tolist() == [0]
  rc = create_render_context(mjm, cam_res=[(4, 3), (5, 3), (6, 3), (7, 3)])
  assert rc.cam_res.tolist() == [[4, 3], [5, 3], [6, 3], [7, 3]] and rc.total_rays == 66
  # defaults: the model's resolution, RGB only
  rc = create_render_context(mjm)
  assert rc.render_rgb == [True] * 4 and rc.render_depth == [False] * 4 and rc.render_seg == [False] * 4
  with pytest.raises(ValueError, match="not found"):
    create_render_context(mjm, cam_active=["nope"])
  with pytest.raises(ValueError, match="length"):
    create_render_context(mjm, cam_active=[True, False])
  with pytest.raises(ValueError, match="out of range"):
    create_render_context(mjm, cam_active=[7])
  with pytest.raises(ValueError, match="resolutions count"):
    create_render_context(mjm, cam_res=[(4, 3), (5, 3)])
  with pytest.raises(ValueError, match="render_depth length"):
    create_render_context(mjm, render_depth=[True, False])


def test_context_refusals(stub):
  from mujoco_warp_b200._src import mjcf
  from mujoco_warp_b200._src.render import create_render_context

  mjm = mjcf.load_string(render_scenes.PRIMITIVES)
  with pytest.raises(NotImplementedError, match="render_skybox"):
    create_render_context(mjm, render_skybox=True)
  for k in ("splat_position", "splat_rotation", "splat_scale", "splat_rgba", "splat_adr", "splat_group_id"):
    with pytest.raises(NotImplementedError, match=k):
      create_render_context(mjm, **{k: np.zeros((1, 3))})
  tex = mjcf.load_string("""<mujoco><asset><texture name="t" type="2d" builtin="checker" width="8" height="8"/><material name="tm" texture="t"/></asset>
    <worldbody><camera/><geom type="sphere" size="0.1" material="tm"/></worldbody></mujoco>""")
  with pytest.raises(NotImplementedError, match="use_textures=False"):
    create_render_context(tex)
  rc = create_render_context(tex, use_textures=False, use_fast_math=False, flex_render_smooth=False)
  assert rc.nrender == 1
  # a texture attached through <layer role="rgb"> is refused the same way; one on another role is not sampled by the renderer
  layered = """<mujoco><asset><texture name="t" type="2d" builtin="checker" width="8" height="8"/>
    <material name="tm"><layer texture="t" role="ROLE"/></material></asset><worldbody><camera/><geom type="sphere" size="0.1" material="tm"/></worldbody></mujoco>"""
  with pytest.raises(NotImplementedError, match="use_textures=False"):
    create_render_context(mjcf.load_string(layered.replace("ROLE", "rgb")))
  occ = mjcf.load_string(layered.replace("ROLE", "occlusion"))
  assert occ.mat_texid[0, 2] == 0 and occ.mat_texid[0, 1] == -1
  assert create_render_context(occ).nrender == 1


def test_put_model_render_fields(monkeypatch):
  """put_model uploads the float render fields as batchable (world w reads entry w % n) and refuses integer ones by name."""
  import torch

  from mujoco_warp_b200._src import _lib
  from mujoco_warp_b200._src import io as mio
  from mujoco_warp_b200._src import mjcf

  class Stub:
    def __getattr__(self, name):
      return lambda *a, **k: 1 if name in ("mjb_model_create", "mjb_data_create") else 0

  monkeypatch.setattr(mio, "_require_cuda", lambda: torch.device("cpu"))
  monkeypatch.setattr(_lib, "lib", lambda: Stub())
  mjm = mjcf.load_string(render_scenes.PRIMITIVES)
  m = mio.put_model(mjm, batch_sizes={"cam_fovy": 3, "light_diffuse": 2, "mat_specular": 4, "cam_intrinsic": 5})
  assert tuple(m.cam_fovy.shape) == (3, mjm.ncam) and tuple(m.light_diffuse.shape) == (2, mjm.nlight, 3)
  assert tuple(m.mat_specular.shape) == (4, mjm.nmat) and tuple(m.cam_intrinsic.shape) == (5, mjm.ncam, 4)
  assert tuple(m.light_cutoff.shape) == (1, mjm.nlight) and tuple(m.cam_sensorsize.shape) == (mjm.ncam, 2)
  np.testing.assert_allclose(m.cam_fovy[2].numpy(), mjm.cam_fovy)
  for n in ("light_type", "light_active", "light_castshadow", "geom_matid"):
    with pytest.raises(ValueError, match=n):
      mio.put_model(mjm, batch_sizes={n: 2})


# ---------------------------------------------------------------- host build of mjb_render.cuh


def test_compute_ray_matches_reference():
  g = np.load(GOLDEN)
  lib = host_lib()
  args, intr = g["ray_args"].astype(np.float32), g["ray_intrinsic"].astype(np.float32)
  out = np.zeros((len(args), 3), dtype=np.float32)
  lib.hrender_rays(len(args), _ptr(args), _ptr(intr), _ptr(out))
  # measured: 1.3e-7 absolute on unit vectors (about one fp32 ulp)
  np.testing.assert_allclose(out, g["ray"], rtol=1e-6, atol=2e-7)


def test_lighting_matches_reference():
  g = np.load(GOLDEN)
  lib = host_lib()
  light, surf, flags = g["light"].astype(np.float32), g["surf"].astype(np.float32), np.ascontiguousarray(g["light_flags"], dtype=np.int32)
  out = np.zeros((len(light), 6), dtype=np.float32)
  lib.hrender_lighting(len(light), _ptr(light), _ptr(surf), _ptr(flags), _ptr(out))
  ref = g["lighting"]
  assert (np.abs(ref) > 0).any(axis=1).sum() > len(ref) // 3  # the cases light the surface, not only miss it
  # fp32 against the reference in fp64.  Measured: diffuse 2.7e-6 relative (the spot term's powf, exponents up to 20), specular
  # 1.5e-5 relative (powf(n.h, shininess * 128): an exponent up to 128 multiplies the base's rounding error by as much)
  np.testing.assert_allclose(out[:, :3], ref[:, :3], rtol=5e-6, atol=1e-7)
  np.testing.assert_allclose(out[:, 3:], ref[:, 3:], rtol=2e-5, atol=1e-7)


def test_bounds_contain_the_geom():
  """render_bounds against the box hull of points sampled on each geom's surface (bvh.py:47-174 give tight boxes for sphere,
  capsule, ellipsoid, cylinder and box)."""
  from mujoco_warp_b200._src.mjcf import quat_to_mat

  lib = host_lib()
  rng = np.random.default_rng(3)
  types = np.array([2, 3, 4, 5, 6, 7, 0, 0], dtype=np.int32)
  size = np.array([[0.3, 0, 0], [0.1, 0.4, 0], [0.2, 0.3, 0.5], [0.25, 0.35, 0], [0.1, 0.2, 0.3], [0, 0, 0], [1.5, 2.0, 0.1], [0, 0, 0.1]], dtype=np.float32)
  half = np.array([[0, 0, 0]] * 5 + [[0.2, 0.1, 0.3]] + [[0, 0, 0]] * 2, dtype=np.float32)
  pos = rng.normal(size=(8, 3)).astype(np.float32)
  mat = np.array([quat_to_mat(q / np.linalg.norm(q)).reshape(9) for q in rng.normal(size=(8, 4))], dtype=np.float32)
  out = np.zeros((8, 6), dtype=np.float32)
  lib.hrender_bounds(8, _ptr(types), _ptr(pos), _ptr(mat), _ptr(size), _ptr(half), _ptr(out))
  u = rng.normal(size=(4000, 3))
  u /= np.linalg.norm(u, axis=1, keepdims=True)
  R = mat.reshape(8, 3, 3)
  for i, t in enumerate(types):
    s = size[i].astype(np.float64)
    if t == 2:
      loc = u * s[0]
    elif t == 3:
      loc = u * s[0] + np.outer(np.sign(u[:, 2]), [0, 0, s[1]])
    elif t == 4:
      loc = u * s
    elif t == 5:
      loc = np.c_[u[:, :2] / np.linalg.norm(u[:, :2], axis=1, keepdims=True) * s[0], np.sign(u[:, 2]) * s[1]]
    elif t in (6, 7):
      loc = np.sign(u) * (s if t == 6 else half[i])
    else:
      e = 2 * max(s[0], s[1]) if s[0] > 0 and s[1] > 0 else 1000.0
      loc = np.c_[np.sign(u[:, :2]) * e, np.zeros(len(u))]
    wpts = pos[i] + loc @ R[i].T
    lo, hi = wpts.min(axis=0), wpts.max(axis=0)
    slack = 0.01 if t == 0 else 0.0
    np.testing.assert_allclose(out[i, :3], lo - slack, atol=1e-4 * max(1.0, np.abs(lo).max()), err_msg=str(t)) if t in (0, 6, 7) else None
    assert (out[i, :3] <= lo + 1e-5 * max(1.0, np.abs(lo).max())).all() and (out[i, 3:] >= hi - 1e-5 * max(1.0, np.abs(hi).max())).all(), t
