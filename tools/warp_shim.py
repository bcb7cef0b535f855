"""Minimal pure-Python stand-in for the `warp` API surface used by the reference's @wp.func-level code.

NVIDIA Warp and MuJoCo are not installable offline, so the reference cannot run as shipped.  Its device functions
(`@wp.func` in collision_primitive_core.py, math.py, the solver's cost functions ...) are however plain Python once
`wp.vec3`, `wp.mat33`, `wp.where`, ... exist.  This module provides those names with VALUE semantics (indexing a matrix
returns a copy, augmented assignment rebinds) and double-precision scalars, and `load_reference_module()` imports a
reference source file from /root/reference UNMODIFIED against it.  It is used only by the golden-vector generators under
tools/ (run in the build container, where /root/reference exists); nothing at test or run time imports it.
"""

import importlib.util
import math as _m
import os
import sys
import types as _t


class Vec:
  __slots__ = ("v",)
  _n = 3
  _conv = float

  def __init__(self, *a):
    n = self._n
    if len(a) == 0:
      self.v = [0.0] * n
    elif len(a) == 1 and isinstance(a[0], Vec):
      self.v = list(a[0].v)
    elif len(a) == 1 and isinstance(a[0], (list, tuple)):
      self.v = [self._conv(x) for x in a[0]]
    elif len(a) == 1 and hasattr(a[0], "__len__"):
      self.v = [self._conv(x) for x in a[0]]
    elif len(a) == 1:
      self.v = [self._conv(a[0])] * n
    else:
      flat = []
      for x in a:  # e.g. spatial_vector(vec3, vec3), quat(vec3, w)
        flat.extend(x.v if isinstance(x, Vec) else [x])
      assert len(flat) == n, (len(flat), n)
      self.v = [self._conv(x) for x in flat]

  def _new(self, vals):
    o = type(self).__new__(type(self))
    o.v = vals
    return o

  def __getitem__(self, i):
    return self.v[i]

  def __setitem__(self, i, x):
    self.v[i] = self._conv(x)

  def __len__(self):
    return len(self.v)

  def __eq__(self, o):
    return isinstance(o, Vec) and self.v == o.v

  def __hash__(self):
    return hash(tuple(self.v))

  def __iter__(self):
    return iter(self.v)

  x = property(lambda s: s.v[0])
  y = property(lambda s: s.v[1])
  z = property(lambda s: s.v[2])
  w = property(lambda s: s.v[3])

  def __neg__(self):
    return self._new([-a for a in self.v])

  def __add__(self, o):
    return self._new([a + b for a, b in zip(self.v, o.v)])

  def __sub__(self, o):
    return self._new([a - b for a, b in zip(self.v, o.v)])

  def __mul__(self, s):
    return self._new([a * s for a in self.v])

  __rmul__ = __mul__

  def __truediv__(self, s):
    return self._new([a / float(s) for a in self.v])

  def __repr__(self):
    return f"vec{len(self.v)}({self.v})"


class Mat:
  __slots__ = ("m",)
  _shape = (3, 3)

  def __init__(self, *a):
    r, c = self._shape
    if len(a) == 0:
      self.m = [[0.0] * c for _ in range(r)]
    elif len(a) == 1 and isinstance(a[0], Mat):
      self.m = [list(row) for row in a[0].m]
    elif len(a) == 1:
      self.m = [[float(a[0])] * c for _ in range(r)]
    else:
      assert len(a) == r * c, (len(a), r, c)
      self.m = [[float(a[i * c + j]) for j in range(c)] for i in range(r)]

  def _new(self, rows):
    o = type(self).__new__(type(self))
    o.m = rows
    return o

  def __getitem__(self, idx):
    if isinstance(idx, tuple):
      if isinstance(idx[0], slice):  # m[:, j]: a copy of column j
        col = [r[idx[1]] for r in self.m[idx[0]]]
        return _vec_cls(len(col))(col)
      return self.m[idx[0]][idx[1]]
    return _vec_cls(len(self.m[idx]))(list(self.m[idx]))  # a COPY of the row

  def __setitem__(self, idx, x):
    if isinstance(idx, tuple):
      self.m[idx[0]][idx[1]] = float(x)
    else:
      self.m[idx] = [float(t) for t in x]

  def __matmul__(self, o):
    if isinstance(o, Vec):
      return _vec_cls(len(self.m))([sum(a * b for a, b in zip(row, o.v)) for row in self.m])
    cols = list(zip(*o.m))
    return _mat_cls(len(self.m), len(cols))._from_rows([[sum(a * b for a, b in zip(row, col)) for col in cols] for row in self.m])

  def __rmatmul__(self, o):  # row vector times matrix
    cols = list(zip(*self.m))
    return _vec_cls(len(cols))([sum(a * b for a, b in zip(o.v, col)) for col in cols])

  def __mul__(self, o):  # warp allows mat * vec as well as scalar scaling
    if isinstance(o, (Vec, Mat)):
      return self.__matmul__(o)
    return self._new([[a * float(o) for a in row] for row in self.m])

  def __rmul__(self, s):
    return self._new([[a * float(s) for a in row] for row in self.m])

  def __add__(self, o):
    return self._new([[a + b for a, b in zip(r1, r2)] for r1, r2 in zip(self.m, o.m)])

  def __sub__(self, o):
    return self._new([[a - b for a, b in zip(r1, r2)] for r1, r2 in zip(self.m, o.m)])

  def __neg__(self):
    return self._new([[-a for a in row] for row in self.m])

  @classmethod
  def _from_rows(cls, rows):
    o = cls.__new__(cls)
    o.m = [list(map(float, r)) for r in rows]
    return o

  def __repr__(self):
    return f"mat({self.m})"


_VEC, _MAT = {}, {}


def _vec_cls(n, conv=float):
  key = (n, conv)
  if key not in _VEC:
    _VEC[key] = type(f"vec{n}{'i' if conv is int else ''}", (Vec,), {"_n": n, "_conv": conv, "_shape_": (n,), "__slots__": ()})
  return _VEC[key]


def _mat_cls(r, c):
  if (r, c) not in _MAT:
    _MAT[(r, c)] = type(f"mat{r}{c}", (Mat,), {"_shape": (r, c), "_shape_": (r, c), "__slots__": ()})
  return _MAT[(r, c)]


def _build_warp():
  wp = _t.ModuleType("warp")
  _overloads = {}

  def func(f):
    """@wp.func: arguments are passed by value; functions of one module that share a name are overloads, picked by arity."""
    import functools

    cands = _overloads.setdefault((f.__module__, f.__qualname__), [])
    cands.append(f)

    @functools.wraps(f)
    def by_value(*a, **k):
      g = f
      n = len(a) + len(k)
      if len(cands) > 1 and f.__code__.co_argcount != n:  # an overload with another arity; a same-named function whose arity fits is itself
        g = next((c for c in reversed(cands) if c.__code__.co_argcount == n), f)  # (kernel builders redefine their nested functions per build)
      return g(*[_wp_copy(x) for x in a], **{n_: _wp_copy(x) for n_, x in k.items()})

    return by_value

  wp.func = func
  wp.kernel = lambda f=None, **k: f if f is not None else (lambda g: g)
  wp.struct = _struct
  wp.set_module_options = lambda *a, **k: None
  wp.static = lambda x: x
  wp.vec2, wp.vec3, wp.vec4 = _vec_cls(2), _vec_cls(3), _vec_cls(4)
  wp.vec2f, wp.vec3f, wp.vec4f, wp.quat, wp.quatf = wp.vec2, wp.vec3, wp.vec4, _vec_cls(4), _vec_cls(4)
  wp.vec2i, wp.vec3i, wp.vec4i = _vec_cls(2, int), _vec_cls(3, int), _vec_cls(4, int)
  wp.spatial_vector = _vec_cls(6)
  wp.mat33, wp.mat33f = _mat_cls(3, 3), _mat_cls(3, 3)
  wp.float32 = wp.float64 = wp.float = float
  wp.int32 = wp.int = int
  wp.bool = bool
  wp.inf, wp.pi = _m.inf, _m.pi
  _install_runtime(wp)
  def _missing(name):  # unused API (textures, bvh, ...) resolves to dummies
    if name.startswith("__"):
      raise AttributeError(name)
    return type(name, (), {})

  wp.__dict__["__getattr__"] = _missing
  tt = _t.ModuleType("warp.types")
  tt.vector = lambda length, dtype=float: _vec_cls(length)
  tt.matrix = lambda shape, dtype=float: _mat_cls(*shape)
  wp.types = tt

  def where(c, a, b):
    return a if c else b

  def _abs(x):
    return x._new([abs(a) for a in x.v]) if isinstance(x, Vec) else abs(x)

  def _ew(f):
    def g(a, b):
      if isinstance(a, Vec):
        return a._new([f(p, q) for p, q in zip(a.v, b.v)])
      return f(a, b)
    return g

  wp.where = where
  wp.abs = _abs
  wp.min, wp.max = _ew(min), _ew(max)
  wp.dot = lambda a, b: sum(p * q for p, q in zip(a.v, b.v))
  wp.cross = lambda a, b: a._new([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])
  wp.length_sq = lambda a: sum(p * p for p in a.v)
  wp.length = lambda a: _m.sqrt(sum(p * p for p in a.v))
  wp.norm_l2 = wp.length

  def normalize(a):
    l = wp.length(a)
    return a / l if l > 0.0 else a._new([0.0] * len(a.v))

  wp.normalize = normalize
  wp.cw_mul = lambda a, b: a._new([p * q for p, q in zip(a.v, b.v)])
  wp.cw_div = lambda a, b: a._new([_wp_div(p, q) for p, q in zip(a.v, b.v)])
  wp.sqrt, wp.sin, wp.cos, wp.atan2, wp.acos, wp.exp, wp.log, wp.pow = _m.sqrt, _m.sin, _m.cos, _m.atan2, _m.acos, _m.exp, _m.log, _m.pow
  wp.tan = _m.tan  # render_util.py compute_ray
  wp.sign = lambda x: x._new([-1.0 if a < 0 else 1.0 for a in x.v]) if isinstance(x, Vec) else (-1.0 if x < 0 else 1.0)  # warp: sign(0) = +1
  wp.clamp = lambda x, lo, hi: min(max(x, lo), hi)
  wp.transpose = lambda a: _mat_cls(len(a.m[0]), len(a.m))._from_rows([list(c) for c in zip(*a.m)])
  wp.matrix_from_rows = lambda *rows: _mat_cls(len(rows), len(rows[0].v))._from_rows([list(r.v) for r in rows])
  wp.matrix_from_cols = lambda *cols: wp.transpose(wp.matrix_from_rows(*cols))
  wp.identity = lambda n, dtype=float: _mat_cls(n, n)._from_rows([[1.0 if i == j else 0.0 for j in range(n)] for i in range(n)])
  # the fluid force derivatives (derivative.py:588-852)
  wp.skew = lambda v: _mat_cls(3, 3)._from_rows([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])
  wp.outer = lambda a, b: _mat_cls(len(a.v), len(b.v))._from_rows([[p * q for q in b.v] for p in a.v])
  return wp


# ---------------------------------------------------------------------------------------------------------------------
# kernel emulation: arrays, launch, tid, atomics, tiles.  One Python call per (world, thread) index; blocks run with
# block_dim = 1, so `for i in range(tid, n, wp.block_dim())` loops cover everything and barriers are no-ops.
import dis as _dis
import itertools as _it

import numpy as _np

_STATE = {"tid": (0,), "block_dim": 1}
_CPU = _t.SimpleNamespace(is_cpu=True, is_cuda=False, sm_count=1, ordinal=0, arch=0)


def _inner(dtype):
  return tuple(getattr(dtype, "_shape_", ()))


def _np_dtype(dtype):
  if dtype in (bool,):
    return _np.bool_
  if dtype in (int,) or (isinstance(dtype, type) and issubclass(dtype, Vec) and dtype._conv is int):
    return _np.int64
  return _np.float64


class array:
  """numpy-backed stand-in for wp.array (any rank); element access returns copies with value semantics"""

  def __init__(self, data=None, dtype=None, shape=None, ndim=None, device=None, **kw):
    self.dtype = dtype if dtype is not None else float
    self._is_batched = False
    self.device = _CPU
    inner = _inner(self.dtype)
    if kw.get("ptr") is not None:  # reinterpretation of another array's storage (same bytes, new dtype / shape)
      self.a = kw["ptr"].a.reshape(tuple(_shape_t(shape)) + inner)
      self.shape = tuple(_shape_t(shape))
      self.ndim = len(self.shape)
      return
    if data is None:
      self.a = None if shape is None else _np.zeros(tuple(_shape_t(shape)) + inner, dtype=_np_dtype(self.dtype))
      self.shape = tuple(_shape_t(shape)) if shape is not None else ()
      self.ndim = ndim if ndim is not None else len(self.shape)
      return
    if isinstance(data, array):
      data = data.a
    a = _np.array(data).astype(_np_dtype(self.dtype))
    if shape is not None:
      a = a.reshape(tuple(_shape_t(shape)) + inner)
    elif inner and a.shape[a.ndim - len(inner):] != inner:
      a = a.reshape((-1,) + inner)
    self.a = a
    self.shape = a.shape[: a.ndim - len(inner)]
    self.ndim = len(self.shape)

  def __class_getitem__(cls, k):
    return cls

  @classmethod
  def _view(cls, a, dtype):
    o = cls.__new__(cls)
    o.dtype, o.a, o._is_batched, o.device = dtype, a, False, _CPU
    inner = _inner(dtype)
    o.shape = a.shape[: a.ndim - len(inner)]
    o.ndim = len(o.shape)
    return o

  @property
  def size(self):
    return int(_np.prod(self.shape)) if self.shape else 0

  @property
  def ptr(self):
    return self

  def reshape(self, shape):
    return array._view(self.a.reshape(tuple(_shape_t(shape)) + _inner(self.dtype)), self.dtype)  # shares storage

  def flatten(self):
    return self.reshape((self.size,))

  def view(self, dtype):
    return array._view(self.a, dtype)

  def _wrap(self, e):
    dt = self.dtype
    if isinstance(dt, type) and issubclass(dt, Vec):
      return dt([dt._conv(x) for x in e])
    if isinstance(dt, type) and issubclass(dt, Mat):
      return dt._from_rows(e.tolist())
    if dt is bool:
      return bool(e)
    if dt is int:
      return int(e)
    return float(e)

  def __getitem__(self, idx):
    if not isinstance(idx, tuple):
      idx = (idx,)
    idx = tuple(int(i) for i in idx)
    for i, n in zip(idx, self.shape):
      if not 0 <= i < n:
        raise IndexError(f"index {idx} out of range for shape {self.shape}")
    if len(idx) == len(self.shape):
      if isinstance(self.dtype, type) and issubclass(self.dtype, Vec) and _component_store(sys._getframe(1)):
        return _ComponentRef(self.a, idx)
      return self._wrap(self.a[idx])
    return array._view(self.a[idx], self.dtype)

  def __setitem__(self, idx, val):
    if not isinstance(idx, tuple):
      idx = (idx,)
    idx = tuple(int(i) for i in idx)
    for i, n in zip(idx, self.shape):
      if not 0 <= i < n:
        raise IndexError(f"index {idx} out of range for shape {self.shape}")
    assert len(idx) == len(self.shape), (idx, self.shape)
    if isinstance(val, Vec):
      self.a[idx] = val.v
    elif isinstance(val, Mat):
      self.a[idx] = val.m
    else:
      self.a[idx] = val

  def numpy(self):
    return _np.array(self.a)

  def zero_(self):
    self.a[...] = 0

  def fill_(self, v):
    if isinstance(v, Vec):
      self.a[...] = v.v
    else:
      self.a[...] = v

  def __len__(self):
    return self.shape[0]


def _shape_t(shape):
  return (shape,) if isinstance(shape, (int, _np.integer)) else tuple(int(x) for x in shape)


class Tile:
  """value-semantics tile: float ndarray for scalar tiles, object ndarray (of Vec / Mat) for vector tiles"""

  def __init__(self, a):
    self.a = a if isinstance(a, _np.ndarray) else _np.array(a, dtype=_np.float64)

  @property
  def shape(self):
    return self.a.shape

  def __getitem__(self, i):
    e = self.a[i]
    if isinstance(e, (Vec, Mat)):
      return _wp_copy(e)
    return float(e) if _np.ndim(e) == 0 else Tile(_np.array(e))

  def __setitem__(self, i, v):
    self.a[i] = v

  def __add__(self, o):
    return Tile(self.a + (o.a if isinstance(o, Tile) else o))

  def __sub__(self, o):
    return Tile(self.a - (o.a if isinstance(o, Tile) else o))

  def __mul__(self, o):
    return Tile(self.a * (o.a if isinstance(o, Tile) else o))

  __rmul__ = __mul__

  def __neg__(self):
    return Tile(-self.a)


def _tile_from(src, dtype):
  """numpy block (outer dims + inner dims of dtype) -> tile backing array"""
  inner = _inner(dtype)
  if not inner:
    return _np.array(src, dtype=_np.float64)
  outer = src.shape[: src.ndim - len(inner)]
  out = _np.empty(outer, dtype=object)
  for i in _np.ndindex(outer):
    out[i] = dtype([dtype._conv(x) for x in src[i]]) if issubclass(dtype, Vec) else dtype._from_rows(src[i].tolist())
  return out


class _ComponentRef:
  """`arr[i]` as the target of a component store `arr[i][k] = v`, which in warp writes into the array (a plain read returns a copy)"""

  __slots__ = ("a", "idx")

  def __init__(self, a, idx):
    self.a, self.idx = a, idx

  def __setitem__(self, k, v):
    self.a[self.idx + (int(k),)] = v


_STORE_CACHE = {}


def _component_store(frame):
  """whether the instruction after the caller's subscript loads one index and stores into the element: `arr[i][k] = v`"""
  key = (frame.f_code, frame.f_lasti)
  if key not in _STORE_CACHE:
    nxt = [ins.opname for ins in _dis.get_instructions(frame.f_code) if ins.offset > frame.f_lasti][:2]
    _STORE_CACHE[key] = len(nxt) == 2 and nxt[0] in ("LOAD_CONST", "LOAD_FAST") and nxt[1] == "STORE_SUBSCR"
  return _STORE_CACHE[key]


_UNPACK_CACHE = {}


def _unpack_count(frame):
  key = (frame.f_code, frame.f_lasti)
  if key not in _UNPACK_CACHE:
    n = None
    for ins in _dis.get_instructions(frame.f_code):
      if ins.offset > frame.f_lasti:
        if ins.opname == "UNPACK_SEQUENCE":
          n = ins.argval
        break
    _UNPACK_CACHE[key] = n
  return _UNPACK_CACHE[key]


def _install_runtime(wp):
  import sys as _sys

  wp.array = array
  wp.array1d = wp.array2d = wp.array3d = wp.array4d = array
  wp.dtype_to_numpy = _np_dtype
  wp.int64, wp.uint32, wp.uint64, wp.int8, wp.uint8 = int, int, int, int, int

  def tid():
    n = _unpack_count(_sys._getframe(1))
    t = _STATE["tid"]
    if n is None:
      return t[0]
    return tuple(t[:n]) if n <= len(t) else tuple(t) + (0,) * (n - len(t))

  wp.tid = tid
  wp.block_dim = lambda: _STATE["block_dim"]

  def launch(kernel, dim=None, inputs=(), outputs=(), block_dim=None, device=None, **kw):
    dims = _shape_t(dim)
    if any(d == 0 for d in dims):
      return
    args = list(inputs) + list(outputs)
    saved = dict(_STATE)
    try:
      for idx in _it.product(*(range(d) for d in dims)):
        _STATE["tid"] = idx
        kernel(*args)
    finally:
      _STATE.update(saved)

  def launch_tiled(kernel, dim=None, inputs=(), outputs=(), block_dim=None, device=None, **kw):
    dims = _shape_t(dim)
    if any(d == 0 for d in dims):
      return
    args = list(inputs) + list(outputs)
    saved = dict(_STATE)
    try:
      for idx in _it.product(*(range(d) for d in dims)):
        _STATE["tid"] = idx + (0,)  # one thread per block
        kernel(*args)
    finally:
      _STATE.update(saved)

  wp.launch, wp.launch_tiled = launch, launch_tiled

  def kernel(f=None, **kw):
    return f if f is not None else (lambda g: g)

  wp.kernel = kernel
  wp.func_native = lambda snippet=None, **kw: (lambda f: (lambda *a, **k: None))
  wp.zeros = lambda shape=None, dtype=float, **kw: array(None, dtype=dtype, shape=shape)
  wp.empty = wp.zeros
  wp.zeros_like = lambda a, **kw: array(None, dtype=a.dtype, shape=a.shape)
  wp.empty_like = wp.zeros_like

  def full(shape=None, value=0, dtype=float, **kw):
    a = array(None, dtype=dtype, shape=shape)
    a.fill_(value)
    return a

  wp.full = full
  wp.ones = lambda shape=None, dtype=float, **kw: full(shape, 1, dtype)
  wp.clone = lambda a, **kw: array._view(_np.array(a.a), a.dtype)

  def copy(dest, src, dest_offset=0, src_offset=0, count=0, **kw):
    if count:
      dest.a.reshape(-1)[dest_offset : dest_offset + count] = src.a.reshape(-1)[src_offset : src_offset + count]
    else:
      dest.a[...] = src.a

  wp.copy = copy

  def _atomic(op):
    def f(arr, *a):
      idx, val = a[:-1], a[-1]
      old = arr[idx if len(idx) > 1 else idx[0]]
      arr[idx if len(idx) > 1 else idx[0]] = op(old, val)
      return old
    return f

  wp.atomic_add = _atomic(lambda o, v: o + v)
  wp.atomic_sub = _atomic(lambda o, v: o - v)
  wp.atomic_max = _atomic(lambda o, v: max(o, v))
  wp.atomic_min = _atomic(lambda o, v: min(o, v))
  wp.atomic_or = _atomic(lambda o, v: o | v)
  wp.add, wp.sub, wp.mul = (lambda a, b: a + b), (lambda a, b: a - b), (lambda a, b: a * b)
  wp.spatial_top = lambda s: _vec_cls(3)([s[0], s[1], s[2]])
  wp.spatial_bottom = lambda s: _vec_cls(3)([s[3], s[4], s[5]])
  wp.quat_rotate = lambda q, v: _quat_rotate(q, v)
  wp.printf = lambda *a: None
  wp.isnan = lambda x: x != x
  wp.ceil, wp.floor, wp.round = _m.ceil, _m.floor, round
  wp.init = lambda: None
  wp.constant = lambda x: x
  wp.get_device = lambda *a: _t.SimpleNamespace(is_cuda=False, is_cpu=True, sm_count=1, arch=0, ordinal=0)
  wp.is_conditional_graph_supported = lambda: False
  wp.ScopedDevice = lambda *a, **k: _Null()
  wp.get_suggested_block_size = lambda kernel, *a, **k: (256, 1184)  # (block size, min grid): only used to partition work
  wp.config = _t.SimpleNamespace(enable_backward=False, quiet=True)

  def capture_while(cond, while_body=None, **kw):
    while bool(cond.a.reshape(-1)[0]):
      while_body(**kw)

  def capture_if(cond, on_true=None, on_false=None, **kw):
    if bool(cond.a.reshape(-1)[0]):
      if on_true:
        on_true(**kw)
    elif on_false:
      on_false(**kw)

  wp.capture_while, wp.capture_if = capture_while, capture_if

  # ---- tiles (numpy semantics; every tile op sees the whole tile)
  def tile_load(arr, shape=None, offset=None, bounds_check=True, **kw):
    shape = _shape_t(shape)
    offset = (0,) * len(shape) if offset is None else _shape_t(offset)
    inner = _inner(arr.dtype)
    out = _np.zeros(shape + inner)
    src = arr.a
    sl_src, sl_dst = [], []
    for o, n, tot in zip(offset, shape, src.shape):
      hi = min(o + n, tot)
      sl_src.append(slice(o, hi)); sl_dst.append(slice(0, max(hi - o, 0)))
    out[tuple(sl_dst)] = src[tuple(sl_src)]
    return Tile(_tile_from(out, arr.dtype))

  def tile_store(arr, t, offset=None, bounds_check=True, **kw):
    shape = t.a.shape
    offset = (0,) * len(shape) if offset is None else _shape_t(offset)
    sl_dst, sl_src = [], []
    for o, n, tot in zip(offset, shape, arr.a.shape):
      hi = min(o + n, tot)
      sl_dst.append(slice(o, hi)); sl_src.append(slice(0, max(hi - o, 0)))
    block = t.a[tuple(sl_src)]
    if block.dtype == object:
      block = _np.array([[*(e.v if isinstance(e, Vec) else sum(e.m, []))] for e in block.reshape(-1)]).reshape(block.shape + _inner(arr.dtype))
    arr.a[tuple(sl_dst)] = block

  wp.tile_load, wp.tile_store = tile_load, tile_store

  def tile_sort(keys, values):
    order = _np.argsort(keys.a, kind="stable")
    keys.a[...] = keys.a[order]; values.a[...] = values.a[order]

  wp.tile_sort = tile_sort

  class _Utils:
    @staticmethod
    def array_scan(src, dst, inclusive=True):
      c = _np.cumsum(src.a.reshape(-1))
      dst.a.reshape(-1)[...] = c if inclusive else _np.concatenate(([0], c[:-1]))

    @staticmethod
    def segmented_sort_pairs(keys, values, count, segment_start_indices, segment_end_indices=None):
      k, v, seg = keys.a.reshape(-1), values.a.reshape(-1), segment_start_indices.a.reshape(-1)
      for i in range(len(seg) - 1):
        lo, hi = int(seg[i]), int(seg[i + 1])
        order = _np.argsort(k[lo:hi], kind="stable")
        k[lo:hi] = k[lo:hi][order]; v[lo:hi] = v[lo:hi][order]

  wp.utils = _Utils
  wp.tile_zeros = lambda shape=None, dtype=float, **kw: Tile(_np.zeros(_shape_t(shape)))
  wp.tile_ones = lambda shape=None, dtype=float, **kw: Tile(_np.ones(_shape_t(shape)))
  wp.tile_arange = lambda *a, dtype=int, **kw: Tile(_np.arange(*a).astype(float))
  wp.tile_transpose = lambda t: Tile(t.a.T)
  wp.tile_matmul = _tile_matmul
  wp.tile_reshape = lambda t, shape=None: Tile(t.a.reshape(_shape_t(shape)))
  wp.tile_broadcast = lambda t, shape=None: Tile(_np.broadcast_to(t.a, _shape_t(shape)).copy())

  def tile_map(op, *ts):
    shape = next(t.a.shape for t in ts if isinstance(t, Tile))
    out = _np.empty(shape, dtype=object)
    for i in _np.ndindex(shape):
      args = []
      for t in ts:
        if isinstance(t, Tile):
          e = t.a[i]
          args.append(_wp_copy(e) if t.a.dtype == object else float(e))
        else:
          args.append(t)  # a scalar / vector broadcast over the tile
      out[i] = op(*args)
    try:
      return Tile(out.astype(_np.float64))
    except (TypeError, ValueError):
      return Tile(out)

  wp.tile_map = tile_map

  def tile_reduce(op, t):
    flat = list(t.a.reshape(-1))
    acc = flat[0]
    for x in flat[1:]:
      acc = op(acc, x)
    o = _np.empty((1,), dtype=object if isinstance(acc, (Vec, Mat)) else _np.float64)
    o[0] = acc
    return Tile(o)

  wp.tile_reduce = tile_reduce
  wp.tile_sum = lambda t: tile_reduce(lambda a, b: a + b, t)

  def tile(x, preserve_type=False):
    o = _np.empty((1,), dtype=object if isinstance(x, (Vec, Mat)) else _np.float64)
    o[0] = x
    return Tile(o)

  class _TileCtor:  # callable (wp.tile(x)) and subscriptable (annotation wp.tile[float, n, m])
    def __call__(self, x, preserve_type=False):
      return tile(x, preserve_type)

    def __getitem__(self, k):
      return Tile

  wp.tile = _TileCtor()
  wp.tile_argmin = lambda t: [int(_np.argmin(t.a))]  # index of the first minimum (ray.py:995)
  wp.tile_extract = lambda t, *i: t[i if len(i) > 1 else i[0]]

  def _sym(a, fill_mode):
    tri = _np.triu(a) if fill_mode == "upper" else _np.tril(a)
    return tri + tri.T - _np.diag(_np.diag(a))

  def tile_cholesky(t, fill_mode="lower"):
    Lm = _np.linalg.cholesky(_sym(t.a, fill_mode))
    return Tile(Lm.T.copy() if fill_mode == "upper" else Lm)

  def tile_cholesky_inplace(t, fill_mode="lower"):
    t.a[...] = tile_cholesky(t, fill_mode).a  # upper: A = U^T U with U stored in the upper triangle

  def tile_cholesky_solve(L, b, fill_mode="lower"):
    Lm = _np.triu(L.a).T if fill_mode == "upper" else _np.tril(L.a)
    y = _np.linalg.solve(Lm, b.a)
    return Tile(_np.linalg.solve(Lm.T, y))

  def tile_load_indexed(arr, idx, shape=None, **kw):
    flat = arr.a.reshape(-1)
    ii = idx.a.astype(_np.int64).reshape(-1)
    ok = (ii >= 0) & (ii < flat.size)
    out = _np.where(ok, flat[_np.clip(ii, 0, max(flat.size - 1, 0))], 0.0)
    return Tile(out.reshape(_shape_t(shape)))

  def tile_scatter_add(t, pos, val, enable=True):
    if enable:
      t.a.reshape(-1)[int(pos)] += val

  def tile_scatter_masked(t, pos, val, mask=True):
    if mask:
      t.a.reshape(-1)[int(pos)] = val

  wp.tile_load_indexed, wp.tile_scatter_add, wp.tile_scatter_masked = tile_load_indexed, tile_scatter_add, tile_scatter_masked

  def tile_view(t, shape=None, offset=None):
    shape = _shape_t(shape)
    offset = (0,) * len(shape) if offset is None else _shape_t(offset)
    return Tile(t.a[tuple(slice(o, o + n) for o, n in zip(offset, shape))])  # numpy view: writes go through

  def tile_assign(dst, src, offset=None):
    offset = (0,) * src.a.ndim if offset is None else _shape_t(offset)
    dst.a[tuple(slice(o, o + n) for o, n in zip(offset, src.a.shape))] = src.a

  def tile_lower_solve_inplace(L, B):
    B.a[...] = _np.linalg.solve(_np.tril(L.a), B.a)

  def tile_upper_solve_inplace(U, B):
    B.a[...] = _np.linalg.solve(_np.triu(U.a), B.a)

  wp.tile_view, wp.tile_assign = tile_view, tile_assign
  wp.tile_lower_solve_inplace, wp.tile_upper_solve_inplace = tile_lower_solve_inplace, tile_upper_solve_inplace
  wp.tile_lower_solve = lambda L, B: Tile(_np.linalg.solve(_np.tril(L.a), B.a))
  wp.tile_upper_solve = lambda U, B: Tile(_np.linalg.solve(_np.triu(U.a), B.a))

  def tile_cholesky_solve_inplace(L, b, fill_mode="lower"):
    b.a[...] = tile_cholesky_solve(L, b, fill_mode).a

  wp.tile_cholesky, wp.tile_cholesky_inplace = tile_cholesky, tile_cholesky_inplace
  wp.tile_cholesky_solve, wp.tile_cholesky_solve_inplace = tile_cholesky_solve, tile_cholesky_solve_inplace
  wp.tile_diag_add = lambda t, d: Tile(t.a + _np.diag(d.a))
  wp.diag = lambda v: _mat_cls(len(v.v), len(v.v))._from_rows([[v.v[i] if i == j else 0.0 for j in range(len(v.v))] for i in range(len(v.v))])


def _tile_matmul(a, b, out=None, alpha=1.0, beta=1.0):
  r = alpha * (a.a @ b.a)
  if out is not None:
    out.a[...] = beta * out.a + r
    return out
  return Tile(r)


def _quat_rotate(q, v):
  # warp quats are (x, y, z, w); the reference uses its own (w, x, y, z) helpers except in a few places
  x, y, z, w = q.v
  c = [y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0]]
  c2 = [y * c[2] - z * c[1], z * c[0] - x * c[2], x * c[1] - y * c[0]]
  return _vec_cls(3)([v[i] + 2.0 * (w * c[i] + c2[i]) for i in range(3)])


class _Null:
  def __enter__(self):
    return self

  def __exit__(self, *a):
    return False


import ast
import builtins as _bi


def _wp_div(a, b):
  """warp's `/`: C integer division (truncation toward zero) when both operands are ints, true division otherwise"""
  if isinstance(a, int) and isinstance(b, int) and not isinstance(a, bool):
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q
  try:
    return a / b
  except ZeroDivisionError:  # IEEE floats, as on the device: +-inf, or nan for 0 / 0
    with _np.errstate(divide="ignore", invalid="ignore"):
      return float(_np.float64(a) / _np.float64(b))


def _wp_mod(a, b):
  """C remainder for ints (sign of the dividend)"""
  if isinstance(a, int) and isinstance(b, int) and not isinstance(a, bool):
    return a - b * _wp_div(a, b)
  return a % b


def _wp_copy(x):
  """`a = b` copies vectors / matrices / structs in warp (value types); Python would alias them"""
  if isinstance(x, Vec):
    return x._new(list(x.v))
  if isinstance(x, Mat):
    return x._new([list(r) for r in x.m])
  if getattr(type(x), "_wp_struct", False):
    o = type(x).__new__(type(x))
    for k, v in x.__dict__.items():
      o.__dict__[k] = _wp_copy(v) if isinstance(v, (Vec, Mat)) or getattr(type(v), "_wp_struct", False) else v
    return o
  return x


def _struct(cls):
  """@wp.struct: fields are zero-initialised on construction, instances have value semantics (see _wp_copy)"""
  import typing

  def __init__(self):
    for name, tp in typing.get_type_hints(cls, include_extras=False).items() if False else cls.__annotations__.items():
      if tp is bool:
        v = False
      elif tp is int:
        v = 0
      elif tp is float:
        v = 0.0
      elif isinstance(tp, type) and issubclass(tp, (Vec, Mat)):
        v = tp()
      elif isinstance(tp, type) and getattr(tp, "_wp_struct", False):
        v = tp()
      else:
        v = None  # arrays are bound by the caller
      setattr(self, name, v)

  cls.__init__ = __init__
  cls._wp_struct = True
  return cls


_bi.__wp_div__, _bi.__wp_mod__, _bi.__wp_copy__ = _wp_div, _wp_mod, _wp_copy


def _is_wp_decorator(dec):
  if isinstance(dec, ast.Call):
    dec = dec.func
  return isinstance(dec, ast.Attribute) and isinstance(dec.value, ast.Name) and dec.value.id == "wp" and dec.attr in ("func", "kernel")


class _WarpSemantics(ast.NodeTransformer):
  """Applied in memory to device code only (functions decorated with @wp.func / @wp.kernel, including nested ones): the
  source files are read unmodified from the reference tree; this restores the places where Python's semantics differ
  from warp's typed semantics -- integer `/` and `%`, boolean-valued `and` / `or`, and value (copy) semantics of vector/matrix assignment."""

  def __init__(self):
    self.depth = 0

  def visit_FunctionDef(self, node):
    dev = any(_is_wp_decorator(d) for d in node.decorator_list)
    if dev:
      self.depth += 1
    self.generic_visit(node)
    if dev:
      self.depth -= 1
    return node

  def visit_BinOp(self, node):
    self.generic_visit(node)
    if self.depth and isinstance(node.op, (ast.Div, ast.Mod)):
      fn = "__wp_div__" if isinstance(node.op, ast.Div) else "__wp_mod__"
      return ast.copy_location(ast.Call(func=ast.Name(id=fn, ctx=ast.Load()), args=[node.left, node.right], keywords=[]), node)
    return node

  def visit_BoolOp(self, node):
    # warp's `and` / `or` yield a bool (float(a & 2 and b & 2) is 1.0); Python's yield one of the operands
    self.generic_visit(node)
    if self.depth:
      return ast.copy_location(ast.Call(func=ast.Name(id="bool", ctx=ast.Load()), args=[node], keywords=[]), node)
    return node

  def visit_AugAssign(self, node):
    self.generic_visit(node)
    if self.depth and isinstance(node.op, (ast.Div, ast.Mod)) and isinstance(node.target, ast.Name):
      fn = "__wp_div__" if isinstance(node.op, ast.Div) else "__wp_mod__"
      load = ast.Name(id=node.target.id, ctx=ast.Load())
      return ast.copy_location(ast.Assign(targets=[node.target], value=ast.Call(func=ast.Name(id=fn, ctx=ast.Load()), args=[load, node.value], keywords=[])), node)
    return node

  def visit_Call(self, node):
    # warp's `bvh_query_next(query, index, max_dist)` writes `index` through a reference: rebound here from the query object
    self.generic_visit(node)
    f = node.func
    if self.depth and isinstance(f, ast.Attribute) and f.attr == "bvh_query_next" and len(node.args) == 3 and isinstance(node.args[1], ast.Name):
      q, idx, dist = node.args
      nxt = ast.Call(func=f, args=[q, dist], keywords=[])
      bind = ast.Compare(left=ast.NamedExpr(target=ast.Name(id=idx.id, ctx=ast.Store()), value=ast.Attribute(value=q, attr="index", ctx=ast.Load())),
                         ops=[ast.IsNot()], comparators=[ast.Constant(value=None)])
      return ast.copy_location(ast.BoolOp(op=ast.And(), values=[nxt, bind]), node)
    return node

  def visit_Assign(self, node):
    self.generic_visit(node)
    # warp's `hit = mesh_query_ray(id, p, v, max_t, t, u, v, sign, n, f)` writes its last six arguments through references
    v = node.value
    if (self.depth and isinstance(v, ast.Call) and isinstance(v.func, ast.Attribute) and v.func.attr == "mesh_query_ray" and len(v.args) == 10
        and len(node.targets) == 1):
      outs = [ast.Name(id=a.id, ctx=ast.Store()) for a in v.args[4:]]
      node.targets = [ast.Tuple(elts=[node.targets[0]] + outs, ctx=ast.Store())]
      v.args = v.args[:4]
      return node
    if self.depth and isinstance(node.value, (ast.Name, ast.Attribute)):
      node.value = ast.copy_location(ast.Call(func=ast.Name(id="__wp_copy__", ctx=ast.Load()), args=[node.value], keywords=[]), node.value)
    return node


# ---------------------------------------------------------------------------------------------------------------------
# brute-force stand-ins for warp's BVH and mesh queries (the renderer: bvh.py, render.py, ray.py ray_mesh_with_bvh).  A BVH only
# prunes candidates, so visiting every leaf whose bounds the ray enters gives the same closest hit (exact ties aside).
_OBJECTS = {}


def _register(obj):
  obj.id = len(_OBJECTS) + 1
  _OBJECTS[obj.id] = obj
  return obj


def _slab(lo, hi, p, v, max_t):
  """the ray p + t v enters the box [lo, hi] at some t < max_t with the box not wholly behind its origin"""
  tmin, tmax = -_m.inf, _m.inf
  for k in range(3):
    if v[k] != 0.0:
      a, b = (lo[k] - p[k]) / v[k], (hi[k] - p[k]) / v[k]
      tmin, tmax = max(tmin, min(a, b)), min(tmax, max(a, b))
    elif p[k] < lo[k] or p[k] > hi[k]:
      return False
  return tmax >= max(tmin, 0.0) and tmin < max_t


class _Bvh:
  def __init__(self, lower, upper, groups=None, constructor=None, **kw):
    self.lower, self.upper, self.groups = lower, upper, groups  # read live: refit() has nothing to do
    _register(self)

  def refit(self):
    pass


class _BvhQuery:
  def __init__(self, bvh, p, v, root):
    lo, hi = bvh.lower.numpy().reshape(-1, 3), bvh.upper.numpy().reshape(-1, 3)
    grp = bvh.groups.numpy().reshape(-1) if bvh.groups is not None else _np.zeros(len(lo), dtype=int)
    self.leaves = [(i, lo[i], hi[i]) for i in range(len(lo)) if int(grp[i]) == int(root)]
    self.p, self.v, self.k, self.index = [float(x) for x in p], [float(x) for x in v], 0, -1

  def next(self, max_t):
    while self.k < len(self.leaves):
      i, lo, hi = self.leaves[self.k]
      self.k += 1
      if _slab(lo, hi, self.p, self.v, max_t):
        self.index = i
        return True
    return False


class _Mesh:
  def __init__(self, points=None, indices=None, **kw):
    self.points = _np.asarray(points.numpy(), dtype=_np.float64).reshape(-1, 3)
    self.tris = _np.asarray(indices.numpy(), dtype=_np.int64).reshape(-1, 3)
    _register(self)


def _mesh_query_ray(mesh_id, p, v, max_t):
    """warp's mesh_query_ray: the closest triangle hit with 0 <= t < max_t, either side; (hit, t, u, v, sign, normal, face), with the
    hit point u p0 + v p1 + (1 - u - v) p2 and the unit face normal cross(p1 - p0, p2 - p0)"""
    mesh = _OBJECTS[int(mesh_id)]
    o, d = _np.array([float(x) for x in p]), _np.array([float(x) for x in v])
    best = None
    for f, (i0, i1, i2) in enumerate(mesh.tris):
      a, b, c = mesh.points[i0], mesh.points[i1], mesh.points[i2]
      e1, e2 = b - a, c - a
      h = _np.cross(d, e2)
      det = e1 @ h
      if det == 0.0:
        continue
      s = o - a
      bu = (s @ h) / det
      q = _np.cross(s, e1)
      bv = (d @ q) / det
      t = (e2 @ q) / det
      if bu < 0.0 or bv < 0.0 or bu + bv > 1.0 or t < 0.0 or t >= max_t:
        continue
      if best is None or t < best[0]:
        best = (t, 1.0 - bu - bv, bu, f)
    vec3 = _vec_cls(3)
    if best is None:
      return False, 0.0, 0.0, 0.0, 0.0, vec3(0.0, 0.0, 0.0), -1
    t, u, w, f = best
    i0, i1, i2 = mesh.tris[f]
    n = _np.cross(mesh.points[i1] - mesh.points[i0], mesh.points[i2] - mesh.points[i0])
    n = n / _np.linalg.norm(n)
    return True, t, u, w, (1.0 if n @ d < 0.0 else -1.0), vec3(*n), f


def _install_render_stand_ins(wp):
  wp.Bvh, wp.Mesh = _Bvh, _Mesh
  wp.bvh_get_group_root = lambda bvh_id, group: int(group)
  wp.bvh_query_ray = lambda bvh_id, p, v, root: _BvhQuery(_OBJECTS[int(bvh_id)], p, v, root)
  wp.bvh_query_next = lambda query, max_t: query.next(max_t)
  wp.mesh_query_ray = _mesh_query_ray
  wp.mesh_query_ray_anyhit = lambda mesh_id, p, v, max_t: _mesh_query_ray(mesh_id, p, v, max_t)[0]


def install(root="/root/reference/mujoco_warp/_src"):
  """Put the shim `warp` into sys.modules and make `mujoco_warp._src.<name>` importable straight from the reference
  source tree (unmodified files; the package __init__ files are skipped).  Returns the fake warp module."""
  import importlib.abc
  import importlib.machinery

  wp = _build_warp()
  _install_render_stand_ins(wp)
  sys.modules["warp"] = wp
  sys.modules["warp.types"] = wp.types
  pkg = _t.ModuleType("mujoco_warp")
  pkg.__path__ = []
  sub = _t.ModuleType("mujoco_warp._src")
  sub.__path__ = []
  sys.modules["mujoco_warp"], sys.modules["mujoco_warp._src"] = pkg, sub
  pkg._src = sub

  class Loader(importlib.machinery.SourceFileLoader):
    def source_to_code(self, data, path, *, _optimize=-1):
      tree = ast.parse(data, filename=path)
      tree = _WarpSemantics().visit(tree)
      ast.fix_missing_locations(tree)
      return compile(tree, path, "exec", dont_inherit=True, optimize=_optimize)

  class Finder(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path=None, target=None):
      pre = "mujoco_warp._src."
      if not fullname.startswith(pre) or "." in fullname[len(pre):]:
        return None
      fn = f"{root}/{fullname[len(pre):]}.py"
      if not os.path.exists(fn):
        return None
      return importlib.util.spec_from_file_location(fullname, fn, loader=Loader(fullname, fn))

  sys.meta_path.insert(0, Finder())
  if "mujoco" not in sys.modules:  # math.py / collision_primitive_core.py only need types' constants; give types a stub mujoco
    _stub_types()
  return wp


def _stub_types():
  """constants-only `mujoco_warp._src.types` for callers that never touch MuJoCo enums (collider goldens)"""
  ty = _t.ModuleType("mujoco_warp._src.types")
  # numeric constants restated from /root/reference/mujoco_warp/_src/types.py:32-56 (MJ_MINVAL = mujoco.mjMINVAL = 1e-15)
  ty.MJ_MINVAL, ty.MJ_MAXVAL, ty.MJ_MINIMP, ty.MJ_MAXIMP, ty.MJ_MINMU = 1e-15, 1e10, 0.0001, 0.9999, 1e-5
  ty.vec5, ty.vec6, ty.vec8, ty.vec10, ty.vec11 = (_vec_cls(n) for n in (5, 6, 8, 10, 11))
  ty.vec10f = ty.vec10
  sys.modules["mujoco_warp._src.types"] = ty
  sys.modules["mujoco_warp._src"].types = ty


def load_reference_module(name):
  """Import /root/reference/mujoco_warp/_src/<name>.py unmodified under the shim (install() must have been called)."""
  import importlib

  return importlib.import_module(f"mujoco_warp._src.{name}")
