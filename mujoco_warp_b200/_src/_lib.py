"""ctypes binding of libmjb200.so (the C-ABI in include/mjb200.h).

The library is built in-tree by `__graft_entry__.build()` / `mujoco_warp_b200.build()` with
`nvcc -gencode arch=compute_90a,code=sm_90a`.  There is NO fallback: if the shared object is missing
or a symbol is absent, importing the step path raises.
"""

from __future__ import annotations

import ctypes
import os
import subprocess

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_CSRC = os.path.join(_PKG, "csrc")
LIB_PATH = os.environ.get("MJB_LIB", os.path.join(_PKG, "libmjb200.so"))  # MJB_LIB: A/B-test an alternative build
HEADER_PATH = os.path.join(os.path.dirname(_PKG), "include", "mjb200.h")
SOURCES = ["capi.cu", "k_position.cu", "k_collision.cu", "k_collision_mesh.cu", "k_collision_mesh_large.cu", "k_constraint.cu", "k_velocity.cu", "k_solver.cu", "k_integrate.cu", "k_implicit.cu", "k_support.cu", "k_sensor.cu", "k_sensor_collision.cu", "k_sensor_collision_large.cu", "k_sensor_contact.cu", "k_sensor_rangefinder.cu", "k_ray.cu", "k_inverse.cu", "k_set_const.cu", "k_energy.cu", "k_history.cu", "k_render.cu", "k_body_stages.cu"]
NVCC_FLAGS = ["-std=c++17", "-O3", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "--extended-lambda", "-Xcompiler", "-fPIC", "-shared"]

_lib = None


def _headers():
  return [os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith(".cuh")] + [HEADER_PATH]


def _stale() -> bool:
  if not os.path.exists(LIB_PATH):
    return True
  t = os.path.getmtime(LIB_PATH)
  deps = [os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cu", ".cuh"))] + [HEADER_PATH]
  return any(os.path.getmtime(p) > t for p in deps)


def build(force: bool = False, verbose: bool = False) -> str:
  """Compile every CUDA source for sm_90a into libmjb200.so (nvcc cross-compiles without a GPU).

  One object per translation unit, compiled in parallel and only when the source or a header changed, then linked."""
  if not (force or _stale()):
    return LIB_PATH
  import fcntl
  from concurrent.futures import ThreadPoolExecutor

  lock = open(os.path.join(_CSRC, ".build.lock"), "w")
  fcntl.flock(lock, fcntl.LOCK_EX)  # concurrent builders (pytest-xdist workers) take turns; the later ones find a fresh library
  if not (force or _stale()):
    return LIB_PATH

  nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
  objdir = os.path.join(_CSRC, "_obj")
  os.makedirs(objdir, exist_ok=True)
  hdr_t = max(os.path.getmtime(p) for p in _headers())
  flags = [f for f in NVCC_FLAGS if f != "-shared"] + (["-Xptxas=-v"] if verbose else [])
  # the mesh builds include k_collision.cu / k_sensor_collision.cu
  extra_dep = {"k_collision_mesh.cu": [os.path.join(_CSRC, "k_collision.cu")], "k_collision_mesh_large.cu": [os.path.join(_CSRC, "k_collision.cu")],
               "k_sensor_collision_large.cu": [os.path.join(_CSRC, "k_sensor_collision.cu")]}

  def compile_one(src):
    path, obj = os.path.join(_CSRC, src), os.path.join(objdir, src[:-3] + ".o")
    newest = max([os.path.getmtime(path), hdr_t] + [os.path.getmtime(p) for p in extra_dep.get(src, [])])
    if force or not os.path.exists(obj) or os.path.getmtime(obj) < newest:
      subprocess.check_call([nvcc, *flags, "-c", path, "-o", obj])
    return obj

  with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
    objs = list(ex.map(compile_one, SOURCES))
  subprocess.check_call([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH, *objs])
  return LIB_PATH


def exported_symbols_in_header():
  """Names of the functions include/mjb200.h declares (used by the symbol-coverage test)."""
  import re

  txt = open(HEADER_PATH).read()
  txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
  return sorted(set(re.findall(r"\b(mjb_[a-z_0-9]+)\s*\(", txt)))


def lib():
  """Load libmjb200.so; raises if it is missing (no CPU / eager fallback exists)."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise RuntimeError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). There is no CPU fallback for the step path.")
  L = ctypes.CDLL(LIB_PATH)
  vp, cp, ci, cf = ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_float
  L.mjb_last_error.restype = cp
  L.mjb_version.restype = cp
  L.mjb_model_create.restype = vp
  L.mjb_model_destroy.argtypes = [vp]
  L.mjb_model_set_int.argtypes = [vp, cp, ci]
  L.mjb_model_set_float.argtypes = [vp, cp, cf]
  L.mjb_model_set_array.argtypes = [vp, cp, vp, ci]
  L.mjb_model_set_array_batched.argtypes = [vp, cp, vp, ci, ci]
  L.mjb_model_finalize.argtypes = [vp]
  L.mjb_data_create.restype = vp
  L.mjb_data_create.argtypes = [ci] * 6
  L.mjb_data_destroy.argtypes = [vp]
  L.mjb_data_set_array.argtypes = [vp, cp, vp]
  L.mjb_data_set_int.argtypes = [vp, cp, ci]
  L.mjb_data_finalize.argtypes = [vp, vp]
  for f in STAGE_FUNCS:
    getattr(L, f).argtypes = [vp, vp, vp]
    getattr(L, f).restype = ci
  L.mjb_ctrl_noise.argtypes = [vp, vp, vp, ci, cf, cf, vp]
  for f in ("mjb_solve_m", "mjb_mul_m"):
    getattr(L, f).argtypes = [vp, vp, vp, vp, vp]
    getattr(L, f).restype = ci
  L.mjb_contact_force.argtypes = [vp, vp, vp, ci, ci, vp, vp]
  L.mjb_contact_force.restype = ci
  L.mjb_rays.argtypes = [vp, vp, vp, vp, ci, ci, ctypes.POINTER(ci), ci, vp, vp, vp, vp, vp]
  L.mjb_rays.restype = ci
  for f in ("mjb_refit_bvh", "mjb_render"):
    getattr(L, f).argtypes = [vp, vp, vp, vp]
    getattr(L, f).restype = ci
  L.mjb_render_rays.argtypes = [vp, vp, vp]
  L.mjb_render_rays.restype = ci
  L.mjb_set_const.argtypes = [vp, vp, ci, ci, vp]
  L.mjb_set_const.restype = ci
  L.mjb_set_length_range.argtypes = [vp, vp, ci, vp]
  L.mjb_set_length_range.restype = ci
  for f, args in (("mjb_read_ctrl", [vp, ci, vp]), ("mjb_read_sensor", [vp, ci, vp]), ("mjb_init_ctrl_history", [vp, vp]), ("mjb_init_sensor_history", [vp, vp, vp])):
    getattr(L, f).argtypes = [vp, vp, ci] + args + [vp]
    getattr(L, f).restype = ci
  L.mjb_jac.argtypes = [vp, vp, vp, vp, vp, vp, vp]
  L.mjb_jac.restype = ci
  for f in ("mjb_xfrc_accumulate", "mjb_deriv_smooth_vel"):
    getattr(L, f).argtypes = [vp, vp, vp, vp]
    getattr(L, f).restype = ci
  L.mjb_step_profile.argtypes = [vp, vp, vp, ctypes.POINTER(ctypes.c_float)]
  L.mjb_last_launch_count.restype = ci
  L.mjb_collision_kernel.argtypes = [vp]
  L.mjb_collision_kernel.restype = cp
  _lib = L
  return L


STAGE_FUNCS = [
  "mjb_step", "mjb_forward", "mjb_inverse", "mjb_fwd_position", "mjb_kinematics", "mjb_com_pos", "mjb_camlight", "mjb_crb", "mjb_transmission",
  "mjb_collision", "mjb_make_constraint", "mjb_fwd_velocity", "mjb_fwd_actuation", "mjb_fwd_acceleration", "mjb_factor_m",
  "mjb_solve", "mjb_euler", "mjb_implicit", "mjb_com_vel", "mjb_passive", "mjb_rne", "mjb_rungekutta4", "mjb_sensor_pos", "mjb_sensor_vel", "mjb_sensor_acc",
  "mjb_energy_pos", "mjb_energy_vel", "mjb_rne_postconstraint", "mjb_subtree_vel", "mjb_tendon",
]


def check(rc: int):
  if rc != 0:
    raise RuntimeError("mjb200: " + lib().mjb_last_error().decode())
