"""Inverse dynamics: the generalized forces that produce a given acceleration (reference inverse.py:148 inverse).

`inverse(m, d)` runs the position and velocity stages for the state in `d` and then, at the given `d.qacc`, evaluates the
constraint forces the way the solver's first pass does (no iterations: `solver_niter` is 0) and writes
`qfrc_inverse = qfrc_bias + M qacc - qfrc_passive - qfrc_constraint` together with `efc.force`, `efc.state`, `efc.Ma`,
`qfrc_constraint` and the sensors.  It is one call through the C-ABI on the current torch CUDA stream (k_inverse.cu after the
forward kernels), with no allocation and no synchronisation, so it can be captured in a CUDA graph.

With `EnableBit.INVDISCRETE`, `d.qacc` is the discrete-time acceleration of one step, `(qvel_next - qvel) / timestep`: it is first
converted to the continuous-time one, `M^-1 (M + h diag(dof_damping)) qacc` (Euler, unless `DisableBit.EULERDAMP` is set, in which
case it is used as given) or `M^-1 (M - h qDeriv) qacc` (implicitfast), and everything above uses that one.  `d.qacc` itself is left
as it was.  RK4 and the implicit integrator have no discrete form here, as in the reference.
"""

from __future__ import annotations

from . import constants as C
from .forward import _call
from .types import Data, Model


def inverse(m: Model, d: Data):
  """Inverse dynamics: qfrc_inverse and the constraint forces at the given d.qacc."""
  if int(m.opt.enableflags) & C.ENBL_INVDISCRETE and int(m.opt.integrator) in (C.INT_RK4, C.INT_IMPLICIT):
    name = "RK4" if int(m.opt.integrator) == C.INT_RK4 else "implicit"
    raise NotImplementedError(f"discrete inverse dynamics (EnableBit.INVDISCRETE) is not supported by the {name} integrator")
  _call("mjb_inverse", m, d)
