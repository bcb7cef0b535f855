"""The shared row rule of the solver and inverse dynamics, compiled as host C++, against the reference's inverse dynamics.

tests/golden/inverse_vectors.npz (tools/make_inverse_goldens.py) holds the reference's own `inverse.inverse` run under the warp shim:
for each scene, at forward's converged `qacc` and at a noisy one (rows in every state), every Data field inverse writes plus the
Jacobian rows, `aref`, `D` and the contact data of the rows.  Here `Jaref = J qacc - aref` is formed from the stored rows (continuous-time
cases only: the discrete ones convert `qacc` first) and fed, rounded to fp32, through `row_force_state` of
mujoco_warp_b200/csrc/mjb_linesearch.cuh: row states must equal the reference's off the knife edge, forces agree to fp32 rounding.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "inverse_vectors.npz")
SRC = os.path.join(HERE, "host_harness", "inverse_rows_host.cpp")
OUT = os.path.join(HERE, "host_harness", "_build", "libinverse_rows_host.so")
CNSTR_CONTACT_ELLIPTIC = 7


def _lib():
  import tempfile

  cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
  out = OUT
  try:
    os.makedirs(os.path.dirname(out), exist_ok=True)
  except OSError:
    out = os.path.join(tempfile.mkdtemp(), "libinverse_rows_host.so")
  if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(SRC), os.path.getmtime(os.path.join(HERE, "..", "mujoco_warp_b200", "csrc", "mjb_linesearch.cuh"))):
    try:
      subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", out], check=True)
    except (OSError, subprocess.CalledProcessError):
      out = os.path.join(tempfile.mkdtemp(), "libinverse_rows_host.so")
      subprocess.run(["g++", "-O1", "-shared", "-fPIC", "-w", "-x", "c++", "-ffp-contract=off", f"-I{cuda_inc}", SRC, "-o", out], check=True)
  L = ctypes.CDLL(out)
  L.irh_rows.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 7
  return L


def _cases():
  g = np.load(GOLD)
  names = sorted({k.split("/")[0] for k in g.files})
  return [(n, kind) for n in names if "disc" not in n for kind in ("conv", "noisy")]


def elliptic_map(g, p, w, nefc, nmaxpyramid, impratio_invsqrt):
  """k_solver's / k_inverse's row -> (contact, component) map of world w, from the fixture's rows and contacts"""
  rinfo, rfri = np.full(nefc, -1, np.int32), np.zeros(nefc, np.float32)
  typ, ids = g[f"{p}/efc_type"][w], g[f"{p}/efc_id"][w]
  adr, dim, fr = g[f"{p}/con_efc_address"], g[f"{p}/con_dim"], g[f"{p}/con_friction"]
  for r in range(nefc):
    if typ[r] != CNSTR_CONTACT_ELLIPTIC:
      continue
    cid = int(ids[r])
    e0, dm = int(np.asarray(adr[cid]).reshape(-1)[0]), int(dim[cid])
    j = r - e0
    rinfo[r] = -2 if (e0 < 0 or e0 + dm > nefc) else ((dm << 4) | j)
    rfri[r] = fr[cid, 0] * impratio_invsqrt if j == 0 else fr[cid, j - 1]
  return rinfo, rfri


@pytest.mark.parametrize("name,kind", _cases())
def test_row_rule_reproduces_reference_rows(name, kind):
  from tests.test_oracle_golden_pipeline import load_scene

  g = np.load(GOLD)
  L = _lib()
  p = f"{name}/{kind}"
  mjm = load_scene(name)
  impratio_invsqrt = np.float32(1.0 / np.sqrt(float(mjm.opt.impratio)))
  ell = int(mjm.opt.cone) == 1
  nmaxpyramid = 1
  J, qacc, aref = g[f"{p}/efc_J"], g[f"{p}/in_qacc"], g[f"{p}/efc_aref"]
  checked = 0
  for w in range(qacc.shape[0]):
    nefc = min(int(g[f"{p}/nefc"].reshape(-1)[w]), aref.shape[1])
    if nefc == 0:
      continue
    jaref = (J[w, :nefc] @ qacc[w] - aref[w, :nefc]).astype(np.float32)
    D = np.ascontiguousarray(g[f"{p}/efc_D"][w, :nefc], dtype=np.float32)
    floss = np.ascontiguousarray(g[f"{p}/efc_frictionloss"][w, :nefc], dtype=np.float32)
    rinfo, rfri = elliptic_map(g, p, w, nefc, nmaxpyramid, impratio_invsqrt) if ell else (None, None)
    force, state = np.zeros(nefc, np.float32), np.zeros(nefc, np.int32)
    ptr = lambda a: a.ctypes.data if a is not None else None
    L.irh_rows(nefc, int(g[f"{p}/ne"].reshape(-1)[w]), int(g[f"{p}/nf"].reshape(-1)[w]), ptr(jaref), ptr(D), ptr(floss), ptr(rinfo), ptr(rfri), ptr(force), ptr(state))
    knife = g[f"{p}/knife"][w, :nefc].astype(bool)
    want_st, want_f = g[f"{p}/efc_state"][w, :nefc], g[f"{p}/efc_force"][w, :nefc]
    assert (state[~knife] == want_st[~knife]).all(), (w, np.nonzero((state != want_st) & ~knife))
    ok = ~knife & (state == want_st)
    scale = max(1.0, float(np.abs(want_f).max()))
    np.testing.assert_allclose(force[ok], want_f[ok], atol=1e-4 * scale, rtol=1e-4, err_msg=f"world {w}")
    checked += int(ok.sum())
  assert checked > 0
