"""tree_implicit_a (mujoco_warp_b200/csrc/mjb_implicit_a.cuh) on the CPU: the device source, compiled as host C++ with its 32 lanes as
threads (tests/host_harness/implicit_a_host.cpp), against the fp64 restatement of tests/integrator_oracle.py.

Each tree's block is written into a buffer with a guard region on both sides, as k_euler's shared memory has qvel before A and the
solve's right-hand side after it: nothing may land outside the block.  On the cross-tree scene (a tendon actuator over dofs of two trees)
a kernel that assigns the actuator to the tree of its first dof writes tree 1's entries at tree-0 offsets past the block.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from mujoco_warp_b200._src import constants as C
from mujoco_warp_b200._src import io
from tests import integrator_oracle as O
from tests import util
from tests.test_integrator_vectors import load

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_harness", "implicit_a_host.cpp")
OUT = os.path.join(HERE, "host_harness", "_build", "libimplicit_a_host.so")
IARRS = ["M_rowadr", "M_rownnz", "M_entry_row", "M_colind", "body_isdofancestor", "dof_bodyid", "moment_rowadr0", "moment_rownnz0", "moment_colind0",
         "actuator_gaintype", "actuator_biastype", "actuator_forcelimited", "actuator_dyntype", "actuator_actadr", "actuator_actnum", "actuator_actlimited",
         "actuator_actearly", "ten_J_rowadr", "ten_J_rownnz", "ten_J_colind"]
FARRS = ["dof_damping", "actuator_gainprm", "actuator_biasprm", "actuator_forcerange", "actuator_dynprm", "actuator_actrange", "tendon_damping", "ten_J0"]
DARRS = ["actuator_force", "actuator_moment", "act", "act_dot", "ctrl"]
GUARD = 64
# a moderate value: the stray writes this guards against are accumulations (-= / +=) of terms of order dt, which a huge sentinel would
# absorb in its rounding
SENTINEL = np.float32(3.0)
EPS32 = 2.0 ** -24


@pytest.fixture(scope="module")
def lib():
  os.makedirs(os.path.dirname(OUT), exist_ok=True)
  cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
  subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-std=c++20", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", OUT, "-lpthread"],
                 check=True)
  L = ctypes.CDLL(OUT)
  L.iah_tree_a.restype = None
  return L


def _arrays(mjm, f):
  """The model's tables as the kernels get them (io.derive_tables for the derived ones), fp32 / int32, and one world's data."""
  t = io.derive_tables(mjm)
  nt = int(getattr(mjm, "ntendon", 0))
  tj = O.ten_j0(mjm)
  src = dict(t)
  src.update(body_isdofancestor=util.make_oracle(mjm, 1, 1, 1).tabs["body_isdofancestor"], dof_bodyid=mjm.dof_bodyid, M_rowadr=mjm.M_rowadr,
             M_rownnz=mjm.M_rownnz, M_colind=mjm.M_colind, dof_damping=mjm.dof_damping, tendon_damping=mjm.tendon_damping if nt else np.zeros(1))
  for n in ("ten_J_rowadr", "ten_J_rownnz", "ten_J_colind"):
    src[n] = np.asarray(getattr(mjm, n)) if nt else np.zeros(1)
  src["ten_J0"] = np.array([tj[r, c] for r in range(nt) for c in mjm.ten_J_colind[mjm.ten_J_rowadr[r] : mjm.ten_J_rowadr[r] + mjm.ten_J_rownnz[r]]]) if nt else np.zeros(1)
  for n in IARRS[9:17] + FARRS[1:6]:
    src[n] = getattr(mjm, n)
  assert [int(c) for c in t["moment_colind0"][: t["nJmom"]]] == [c for cols in O.moment_cols(mjm) for c in cols]
  keep = [np.ascontiguousarray(np.asarray(src[n]).astype(np.int32).reshape(-1)) for n in IARRS]
  keep += [np.ascontiguousarray(np.asarray(src[n], dtype=np.float64).astype(np.float32).reshape(-1)) for n in FARRS]
  keep += [np.ascontiguousarray(np.asarray(f[n], dtype=np.float32).reshape(-1)) if len(np.asarray(f[n]).reshape(-1)) else np.zeros(1, np.float32) for n in DARRS]
  P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
  ip = (ctypes.c_void_p * len(IARRS))(*[P(a) for a in keep[: len(IARRS)]])
  fp = (ctypes.c_void_p * len(FARRS))(*[P(a) for a in keep[len(IARRS) : len(IARRS) + len(FARRS)]])
  dp = (ctypes.c_void_p * len(DARRS))(*[P(a) for a in keep[len(IARRS) + len(FARRS) :]])
  sizes = np.array([mjm.nv, mjm.nu, getattr(mjm, "na", 0), nt, t["nJmom"], mjm.opt.disableflags], dtype=np.int32)
  return keep, sizes, ip, fp, dp


def tree_blocks(lib, mjm, f, integrator):
  """Every tree's block through the device source: (list of (start, n, block n x n lower), guard intact)."""
  keep, sizes, ip, fp, dp = _arrays(mjm, f)
  M = np.ascontiguousarray(np.asarray(f["M"], dtype=np.float32))
  fast = integrator == C.INT_IMPLICITFAST
  damper = not (int(mjm.opt.disableflags) & C.DSBL_DAMPER)
  out, intact = [], True
  for start, n in zip(mjm.tree_dofadr, mjm.tree_dofnum):
    start, n = int(start), int(n)
    ld = n | 1
    buf = np.full(GUARD + n * ld + GUARD, SENTINEL, dtype=np.float32)
    lib.iah_tree_a(sizes.ctypes.data_as(ctypes.c_void_p), ctypes.c_float(mjm.opt.timestep), ip, fp, dp, M.ctypes.data_as(ctypes.c_void_p),
                   start, n, ld, int(fast), int(damper), buf[GUARD:].ctypes.data_as(ctypes.c_void_p))
    guard = np.concatenate([buf[:GUARD], buf[GUARD + n * ld :]])
    intact &= bool(np.all(guard.view(np.uint32) == SENTINEL.view(np.uint32)))
    out.append((start, n, np.tril(buf[GUARD : GUARD + n * ld].reshape(n, ld)[:, :n].astype(np.float64))))
  return out, intact


def _fields(mjm, seed, nconmax=32, njmax=128):
  qpos, qvel, ctrl, _ = util.seeded_state(mjm, 1, seed=seed, exact_world0=False)
  act = util.seeded_act(mjm, 1, seed=seed)
  o = util.make_oracle(mjm, 1, nconmax, njmax, dtype=np.float32)
  o.set_state(qpos=qpos, qvel=qvel, ctrl=ctrl, act=act)
  o.forward()
  return {k: v[0].astype(np.float64) for k, v in o.d.items()}


def check_blocks(lib, mjm, f, integrator):
  blocks, intact = tree_blocks(lib, mjm, f, integrator)
  assert intact, "tree_implicit_a wrote outside its tree's block"
  A = O.matrix_a(mjm, f, integrator)
  Aabs = O.matrix_a(mjm, f, integrator, absolute=True)
  worst = 0.0
  for start, n, blk in blocks:
    want, scale = np.tril(A[start : start + n, start : start + n]), np.tril(Aabs[start : start + n, start : start + n])
    # each entry: M plus a handful of fp32 products and sums, each term rounded a few times
    bound = 8 * EPS32 * scale + 1e-30
    worst = max(worst, float((np.abs(blk - want) / bound).max()))
  print(f"tree_implicit_a: worst |A - A64| / (8 eps32 Aabs) = {worst:.3f}")
  assert worst <= 1.0, worst


@pytest.mark.parametrize("scene,integrator", [("crosstree", "implicitfast"), ("crosstree", "Euler"), ("actuators", "implicitfast"),
                                              ("tendons", "implicitfast"), ("mixed", "Euler"), ("mixed", "implicitfast")])
def test_device_source_matches_the_restatement_inside_its_block(lib, scene, integrator):
  mjm = load(scene, integrator)
  check_blocks(lib, mjm, _fields(mjm, 5), int(mjm.opt.integrator))


def test_crosstree_writes_stay_inside_each_block(lib):
  """The guard alone: the tendon actuator's entries of tree 1 (jb, jb2) must not be scattered at tree 0's offsets."""
  mjm = load("crosstree", "implicitfast")
  _, intact = tree_blocks(lib, mjm, _fields(mjm, 5), C.INT_IMPLICITFAST)
  assert intact, "tree_implicit_a wrote outside its tree's block"


@pytest.mark.parametrize("flag", ["DSBL_DAMPER", "DSBL_ACTUATION"])
def test_disable_flags(lib, flag):
  mjm = load("actuators", "implicitfast")
  mjm.opt.disableflags = int(mjm.opt.disableflags) | getattr(C, flag)
  check_blocks(lib, mjm, _fields(mjm, 6), C.INT_IMPLICITFAST)


def test_force_limit_edges(lib):
  """The filterexact actuator a_fex (forcerange -1 1) contributes nothing when its force sits exactly at a bound, and its term when the
  force is one ulp inside it."""
  mjm = load("actuators", "implicitfast")
  f = _fields(mjm, 8)
  a = 2
  assert mjm.actuator_forcelimited[a] and tuple(mjm.actuator_forcerange[a]) == (-1.0, 1.0)
  mjm.actuator_gaintype = np.array(mjm.actuator_gaintype)
  mjm.actuator_gaintype[a] = C.GAIN_AFFINE  # a velocity-dependent gain, so that the skip rule matters
  mjm.actuator_gainprm = np.array(mjm.actuator_gainprm)
  mjm.actuator_gainprm[a, 2] = -0.7
  dof = O.moment_cols(mjm)[a][0]
  for frc, skipped in ((1.0, True), (-1.0, True), (float(np.nextafter(np.float32(1), np.float32(0))), False),
                       (float(np.nextafter(np.float32(-1), np.float32(0))), False)):
    f["actuator_force"][a] = frc
    check_blocks(lib, mjm, f, C.INT_IMPLICITFAST)
    terms = [v for i, j, v in O.qderiv_terms(mjm, f) if i == dof and j == dof]
    assert (len(terms) == 0) == skipped, frc
