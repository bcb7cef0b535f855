"""Inverse dynamics without a GPU: put_model's feature checks and the C-ABI entry point."""
import ctypes

import pytest


def test_validate_accepts_invdiscrete_and_refuses_fwdinv():
  from mujoco_warp_b200._src import constants as C
  from mujoco_warp_b200._src import io, mjcf
  from tests import util

  mjm = mjcf.load_string(util.actuators_xml("Euler"))
  mjm.opt.enableflags = C.ENBL_INVDISCRETE
  io._validate(mjm)
  mjm.opt.enableflags = C.ENBL_FWDINV
  with pytest.raises(NotImplementedError, match="fwdinv"):
    io._validate(mjm)


def test_inverse_is_exported(built):
  import mujoco_warp_b200 as mjw
  from mujoco_warp_b200._src import _lib

  assert callable(mjw.inverse)
  assert "mjb_inverse" in _lib.exported_symbols_in_header()
  assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "mjb_inverse")
