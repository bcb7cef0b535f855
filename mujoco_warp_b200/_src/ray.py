"""Ray casting: the closest geom a ray hits, for many rays in every world (reference ray.py:1172 ray, :1219 rays).

Both read the geom poses of the last kinematics (`forward`, `fwd_position`, `kinematics` or `step`) and launch one kernel
(k_ray.cu) on the current torch CUDA stream.  `rays` writes into preallocated outputs and neither allocates nor synchronises,
so it can be captured in a CUDA graph; `ray` allocates its outputs, as the reference's does.  Every geom is tested (there is no
BVH render context) and height fields do not exist in this build.
"""

from __future__ import annotations

import ctypes

import torch

from . import _lib
from .types import Data, Model


def _check(name: str, t: torch.Tensor, dtype: torch.dtype, shape: tuple):
  if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_cuda or not t.is_contiguous() or tuple(t.shape) != shape:
    kind = "float32" if dtype == torch.float32 else "int32"
    got = f"{tuple(t.shape)} {t.dtype} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
    raise ValueError(f"{name}: expected a contiguous CUDA {kind} tensor of shape {shape}, got {got}")


def _geomgroup(geomgroup) -> ctypes.Array:
  g = [-1] * 6 if geomgroup is None else [int(x) for x in geomgroup]
  if len(g) != 6:
    raise ValueError(f"geomgroup: expected 6 entries (one per geom group 0-5; all -1 = no group filter), got {len(g)}")
  return (ctypes.c_int * 6)(*g)


def rays(m: Model, d: Data, pnt: torch.Tensor, vec: torch.Tensor, geomgroup, flg_static: bool, bodyexclude: torch.Tensor, dist: torch.Tensor,
         geomid: torch.Tensor, normal: torch.Tensor, rc=None):
  """Intersects nray rays with the geoms of every world (reference ray.py:1219).

  pnt, vec: ray origins and directions, float32 (1, nray, 3) shared by all worlds or (nworld, nray, 3) per world; the distance
    is in units of |vec|.
  geomgroup: 6 entries, one per geom group (0-5; larger groups count as 5): a geom is skipped when its group's entry is 0; all -1
    (or None) = no group filter.
  flg_static: False skips geoms on static bodies (welded to the world).
  bodyexclude: int32 (nray,): geoms of this body are skipped by that ray (-1: none).
  dist (nworld, nray) float32, geomid (nworld, nray) int32, normal (nworld, nray, 3) float32: the closest hit's distance, geom id and
    world-frame surface normal; dist = -1, geomid = -1 and a zero normal on a miss.  Equally distant hits go to the lowest geom id.
  rc: the reference's BVH render context; not implemented."""
  if rc is not None:
    raise NotImplementedError("rays(rc=...): BVH-accelerated ray casting is not implemented; call without a render context")
  if d._model is not m and d._model._handle != m._handle:
    raise ValueError("Data was created for a different Model")
  if not isinstance(pnt, torch.Tensor) or pnt.dim() != 3 or pnt.shape[0] not in (1, d.nworld):
    got = tuple(pnt.shape) if isinstance(pnt, torch.Tensor) else type(pnt).__name__
    raise ValueError(f"pnt: expected a contiguous CUDA float32 tensor of shape (1, nray, 3) or ({d.nworld}, nray, 3), got {got}")
  nb, nray = int(pnt.shape[0]), int(pnt.shape[1])
  _check("pnt", pnt, torch.float32, (nb, nray, 3))
  _check("vec", vec, torch.float32, (nb, nray, 3))
  _check("bodyexclude", bodyexclude, torch.int32, (nray,))
  _check("dist", dist, torch.float32, (d.nworld, nray))
  _check("geomid", geomid, torch.int32, (d.nworld, nray))
  _check("normal", normal, torch.float32, (d.nworld, nray, 3))
  stream = torch.cuda.current_stream().cuda_stream
  _lib.check(_lib.lib().mjb_rays(m._handle, d._handle, pnt.data_ptr(), vec.data_ptr(), nray, nb, _geomgroup(geomgroup), int(bool(flg_static)),
                                 bodyexclude.data_ptr(), dist.data_ptr(), geomid.data_ptr(), normal.data_ptr(), stream))


def ray(m: Model, d: Data, pnt: torch.Tensor, vec: torch.Tensor, geomgroup=None, flg_static: bool = True, bodyexclude: int = -1, rc=None):
  """One ray per world (reference ray.py:1172): pnt, vec float32 (1, 1, 3) or (nworld, 1, 3).  Returns (dist (nworld, 1),
  geomid (nworld, 1), normal (nworld, 1, 3)), newly allocated; see `rays` for the other arguments."""
  if isinstance(pnt, torch.Tensor) and pnt.dim() == 3 and pnt.shape[1] != 1:
    raise ValueError(f"pnt: ray() casts one ray per world (shape (1, 1, 3) or ({d.nworld}, 1, 3)), got {tuple(pnt.shape)}; use rays() for several")
  dev = pnt.device if isinstance(pnt, torch.Tensor) else torch.device("cuda")
  ex = torch.full((1,), int(bodyexclude), dtype=torch.int32, device=dev)
  dist = torch.empty((d.nworld, 1), dtype=torch.float32, device=dev)
  geomid = torch.empty((d.nworld, 1), dtype=torch.int32, device=dev)
  normal = torch.empty((d.nworld, 1, 3), dtype=torch.float32, device=dev)
  rays(m, d, pnt, vec, geomgroup, flg_static, ex, dist, geomid, normal, rc)
  return dist, geomid, normal
