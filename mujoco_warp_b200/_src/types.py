"""Model / Data / Contact / Constraint / Option containers and enums.

Mirrors the names, shapes and dtypes of /root/reference/mujoco_warp/_src/types.py (Model :982, Data :2075,
Contact :1975, Constraint :2021, Option :836, enums :53-560) for the fields on the step path.  The device-array
container is `torch.Tensor` (CUDA, contiguous, fp32/int32) instead of `wp.array`; vec/mat dtypes flatten to trailing
dims (vec3 -> (...,3), quat -> (...,4), mat33 -> (...,3,3), spatial_vector -> (...,6), vec10 -> (...,10)).
"""

from __future__ import annotations

import enum

from . import constants as C


class JointType(enum.IntEnum):
  FREE = C.JNT_FREE
  BALL = C.JNT_BALL
  SLIDE = C.JNT_SLIDE
  HINGE = C.JNT_HINGE


class GeomType(enum.IntEnum):
  PLANE = C.GEOM_PLANE
  HFIELD = C.GEOM_HFIELD
  SPHERE = C.GEOM_SPHERE
  CAPSULE = C.GEOM_CAPSULE
  ELLIPSOID = C.GEOM_ELLIPSOID
  CYLINDER = C.GEOM_CYLINDER
  BOX = C.GEOM_BOX
  MESH = C.GEOM_MESH
  SDF = C.GEOM_SDF
  FLEX = 9


class ConeType(enum.IntEnum):
  PYRAMIDAL = C.CONE_PYRAMIDAL
  ELLIPTIC = C.CONE_ELLIPTIC


class IntegratorType(enum.IntEnum):
  EULER = C.INT_EULER
  RK4 = C.INT_RK4
  IMPLICIT = C.INT_IMPLICIT
  IMPLICITFAST = C.INT_IMPLICITFAST


class SolverType(enum.IntEnum):
  CG = C.SOL_CG
  NEWTON = C.SOL_NEWTON


class ConstraintType(enum.IntEnum):
  EQUALITY = C.CNSTR_EQUALITY
  FRICTION_DOF = C.CNSTR_FRICTION_DOF
  FRICTION_TENDON = C.CNSTR_FRICTION_TENDON
  LIMIT_JOINT = C.CNSTR_LIMIT_JOINT
  LIMIT_TENDON = C.CNSTR_LIMIT_TENDON
  CONTACT_FRICTIONLESS = C.CNSTR_CONTACT_FRICTIONLESS
  CONTACT_PYRAMIDAL = C.CNSTR_CONTACT_PYRAMIDAL
  CONTACT_ELLIPTIC = C.CNSTR_CONTACT_ELLIPTIC


class ConstraintState(enum.IntEnum):
  SATISFIED = C.STATE_SATISFIED
  QUADRATIC = C.STATE_QUADRATIC
  LINEARNEG = C.STATE_LINEARNEG
  LINEARPOS = C.STATE_LINEARPOS
  CONE = C.STATE_CONE


class DisableBit(enum.IntFlag):
  CONSTRAINT = C.DSBL_CONSTRAINT
  EQUALITY = C.DSBL_EQUALITY
  FRICTIONLOSS = C.DSBL_FRICTIONLOSS
  LIMIT = C.DSBL_LIMIT
  CONTACT = C.DSBL_CONTACT
  SPRING = C.DSBL_SPRING
  DAMPER = C.DSBL_DAMPER
  GRAVITY = C.DSBL_GRAVITY
  CLAMPCTRL = C.DSBL_CLAMPCTRL
  WARMSTART = C.DSBL_WARMSTART
  FILTERPARENT = C.DSBL_FILTERPARENT
  ACTUATION = C.DSBL_ACTUATION
  REFSAFE = C.DSBL_REFSAFE
  SENSOR = C.DSBL_SENSOR
  EULERDAMP = C.DSBL_EULERDAMP
  NATIVECCD = C.DSBL_NATIVECCD
  ISLAND = C.DSBL_ISLAND


class EnableBit(enum.IntFlag):
  ENERGY = C.ENBL_ENERGY
  INVDISCRETE = C.ENBL_INVDISCRETE
  SLEEP = C.ENBL_SLEEP


class OverflowType(enum.IntFlag):
  NEFC = 1 << 0
  NJMAX_NNZ = 1 << 1
  BROADPHASE = 1 << 2
  NARROWPHASE = 1 << 3
  CCD = 1 << 4
  HFIELD = 1 << 5
  CONTACT_MATCH = 1 << 6
  NVMAX = 1 << 7
  EPA_HORIZON = 1 << 8
  ITERATIONS = 1 << 9
  LS_ITERATIONS = 1 << 10


class ObjType(enum.IntEnum):
  """Object types (MuJoCo mjtObj values; reference types.py:651).  XBODY addresses a body's regular frame instead of its inertial one."""

  UNKNOWN = 0
  BODY = 1
  XBODY = 2
  GEOM = 5
  FLEX = 9
  SITE = 6
  CAMERA = 7


class BroadphaseType(enum.IntEnum):
  NXN = 0
  SAP_TILE = 1
  SAP_SEGMENTED = 2


class State(enum.IntEnum):
  """State components as bit flags (reference types.py:712; MuJoCo mjtState with the history element after ACT)."""

  TIME = 1 << 0
  QPOS = 1 << 1
  QVEL = 1 << 2
  ACT = 1 << 3
  HISTORY = 1 << 4
  WARMSTART = 1 << 5
  CTRL = 1 << 6
  QFRC_APPLIED = 1 << 7
  XFRC_APPLIED = 1 << 8
  EQ_ACTIVE = 1 << 9
  MOCAP_POS = 1 << 10
  MOCAP_QUAT = 1 << 11
  USERDATA = 1 << 12
  PLUGIN = 1 << 13
  NSTATE = 14
  PHYSICS = (1 << 0) | (1 << 1) | (1 << 2) | (1 << 3) | (1 << 4)
  FULLPHYSICS = (1 << 0) | (1 << 1) | (1 << 2) | (1 << 3) | (1 << 4) | (1 << 13)
  USER = (1 << 6) | (1 << 7) | (1 << 8) | (1 << 9) | (1 << 10) | (1 << 11) | (1 << 12)
  INTEGRATION = FULLPHYSICS | USER | (1 << 5)


class TrnType(enum.IntEnum):
  JOINT = 0
  JOINTINPARENT = 1
  SLIDERCRANK = 2
  TENDON = 3
  SITE = 4
  BODY = 5


class DynType(enum.IntEnum):
  NONE = 0
  INTEGRATOR = 1
  FILTER = 2
  FILTEREXACT = 3
  MUSCLE = 4


class GainType(enum.IntEnum):
  FIXED = 0
  AFFINE = 1
  MUSCLE = 2


class BiasType(enum.IntEnum):
  NONE = 0
  AFFINE = 1
  MUSCLE = 2


class BroadphaseFilter(enum.IntFlag):
  PLANE = 1
  SPHERE = 2
  AABB = 4
  OBB = 8


class ContactType(enum.IntFlag):
  CONSTRAINT = 1
  SENSOR = 2


class _Struct:
  """Attribute bag with a stable field listing (stands in for the reference's dataclasses).

  The C handle holds raw device pointers / scalar options, so once a struct is bound (io.put_model / io._bind install
  `_rebind`) assigning a field re-registers the new pointer or scalar with the handle after validating shape, dtype and
  device -- `d.qpos = t`, `m.opt.timestep = 0.002`, `m.geom_friction = t` take effect on the next launch exactly like the
  reference, whose kernels read the dataclass fields at launch time.  (A captured CUDA graph keeps the old pointers, the
  same hazard the reference has.)
  """

  def __init__(self, **kw):
    self.__dict__.update(kw)

  def __setattr__(self, name, value):
    hook = self.__dict__.get("_rebind")
    if hook is not None and not name.startswith("_"):
      value = hook(name, value)
    object.__setattr__(self, name, value)

  def fields(self):
    return [k for k in self.__dict__ if not k.startswith("_")]

  def __repr__(self):
    return f"{type(self).__name__}({', '.join(self.fields())})"


class Option(_Struct):
  pass


class Statistic(_Struct):
  pass


class Model(_Struct):
  pass


class Contact(_Struct):
  pass


class Constraint(_Struct):
  pass


class Data(_Struct):
  pass


class RenderContext(_Struct):
  """Render context of `create_render_context` (reference types.py RenderContext): the active cameras, their output buffers and
  the enabled geoms.

  nrender: active cameras; cam_id_map (nrender) their Model camera ids; cam_res (nrender, 2) width, height; pix_adr (nrender) first
  pixel of each camera in `ray`; total_rays: pixels of all active cameras; ray (total_rays, 3) camera-frame ray directions (with
  use_precomputed_rays); render_rgb / render_depth / render_seg (nrender) host bools; rgb_adr / depth_adr / seg_adr (nrender) first
  pixel of each camera in rgb_data / depth_data / seg_data, -1 when the camera does not produce that output; rgb_data (nworld, nrgb)
  uint32 packed 0xAARRGGBB; depth_data (nworld, ndepth) float32; seg_data (nworld, nseg, 2) int32 (geom id, mjOBJ_GEOM), (-1, -1) on a
  miss; bvh_ngeom: enabled geoms; enabled_geom_ids (bvh_ngeom); lower / upper (nworld, bvh_ngeom, 3) world-space geom bounds written by
  `refit_bvh`; mesh_bounds_size (nmesh, 3) half-extent of each mesh's vertex box; the remaining fields are the creation options."""
