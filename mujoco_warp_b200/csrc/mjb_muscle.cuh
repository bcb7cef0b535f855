// mjb_muscle.cuh -- MuJoCo's muscle model: the active force-length-velocity gain, the passive force and the activation dynamics.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/util_misc.py): :455 muscle_gain_length, :481 muscle_gain, :526 muscle_bias,
// :561 _sigmoid, :574 muscle_dynamics_timescale, :588 muscle_dynamics (Millard et al. 2013 time constants, quintic-sigmoid smoothing).
// Parameters as MuJoCo lays them out: gainprm / biasprm = (range[2], force, scale, lmin, lmax, vmax, fpmax, fvmax), dynprm =
// (tau_act, tau_deact, tausmooth).  A negative force is replaced by scale / acc0.
// Plain functions of scalars (no warp intrinsics, no shared memory), kept in a header so that the same source also compiles as host
// C++: tests/host_harness/muscle_host.cpp checks THIS code against the reference's known answers and an fp64 restatement on the CPU.
#pragma once
#include "mjb_types.cuh"

// normalized length-gain curve: 0 outside [lmin, lmax], 1 at length 1, four half-quadratic pieces in between
__device__ __forceinline__ float muscle_gain_length(float length, float lmin, float lmax) {
  if (lmin > length || length > lmax) return 0.f;
  const float a = 0.5f * (lmin + 1.0f), b = 0.5f * (1.0f + lmax);
  if (length <= a) {
    const float x = (length - lmin) / fmaxf(MJ_MINVAL, a - lmin);
    return 0.5f * x * x;
  } else if (length <= 1.0f) {
    const float x = (1.0f - length) / fmaxf(MJ_MINVAL, 1.0f - a);
    return 1.0f - 0.5f * x * x;
  } else if (length <= b) {
    const float x = (length - 1.0f) / fmaxf(MJ_MINVAL, b - 1.0f);
    return 1.0f - 0.5f * x * x;
  }
  const float x = (lmax - length) / fmaxf(MJ_MINVAL, lmax - b);
  return 0.5f * x * x;
}

// peak force (scale / acc0 for a negative force) and optimum length L0 of a muscle
__device__ __forceinline__ float muscle_force(const float* prm, float acc0) { return prm[2] < 0.f ? prm[3] / fmaxf(MJ_MINVAL, acc0) : prm[2]; }
__device__ __forceinline__ float muscle_L0(const float* prm, float lr0, float lr1) { return (lr1 - lr0) / fmaxf(MJ_MINVAL, prm[1] - prm[0]); }

// active gain: -force * FL(normalized length) * FV(normalized velocity)
__device__ __forceinline__ float muscle_gain(float len, float vel, float lr0, float lr1, float acc0, const float* prm) {
  const float force = muscle_force(prm, acc0), L0 = muscle_L0(prm, lr0, lr1);
  const float lmin = prm[4], lmax = prm[5], vmax = prm[6], fvmax = prm[8];
  const float L = prm[0] + (len - lr0) / fmaxf(MJ_MINVAL, L0);
  const float V = vel / fmaxf(MJ_MINVAL, L0 * vmax);
  const float FL = muscle_gain_length(L, lmin, lmax);
  const float y = fvmax - 1.0f;
  float FV;
  if (V <= -1.0f) FV = 0.f;
  else if (V <= 0.f) FV = (V + 1.0f) * (V + 1.0f);
  else if (V <= y) FV = fvmax - (y - V) * (y - V) / fmaxf(MJ_MINVAL, y);
  else FV = fvmax;
  return -force * FL * FV;
}

// passive force: 0 up to the optimum length, half-quadratic to (1 + lmax) / 2, linear beyond
__device__ __forceinline__ float muscle_bias(float len, float lr0, float lr1, float acc0, const float* prm) {
  const float force = muscle_force(prm, acc0), L0 = muscle_L0(prm, lr0, lr1);
  const float lmax = prm[5], fpmax = prm[7];
  const float L = prm[0] + (len - lr0) / fmaxf(MJ_MINVAL, L0);
  const float b = 0.5f * (1.0f + lmax);
  if (L <= 1.0f) return 0.f;
  if (L <= b) {
    const float x = (L - 1.0f) / fmaxf(MJ_MINVAL, b - 1.0f);
    return -force * fpmax * 0.5f * x * x;
  }
  const float x = (L - b) / fmaxf(MJ_MINVAL, b - 1.0f);
  return -force * fpmax * (0.5f + x);
}

// quintic sigmoid on [0, 1]: f(0) = f'(0) = f''(0) = 0, f(1) = 1, f'(1) = f''(1) = 0
__device__ __forceinline__ float muscle_sigmoid(float x) {
  if (x <= 0.f) return 0.f;
  if (x >= 1.0f) return 1.0f;
  return x * x * x * (3.0f * x * (2.0f * x - 5.0f) + 10.0f);
}

// time constant: hard switch on the sign of dctrl, or a sigmoid blend of width smooth_width around dctrl = 0
__device__ __forceinline__ float muscle_dynamics_timescale(float dctrl, float tau_act, float tau_deact, float smooth_width) {
  if (smooth_width < MJ_MINVAL) return dctrl > 0.f ? tau_act : tau_deact;
  return tau_deact + (tau_act - tau_deact) * muscle_sigmoid(dctrl / smooth_width + 0.5f);
}

// activation derivative: (clamped ctrl - act) / tau, with activation-dependent time constants
__device__ __forceinline__ float muscle_dynamics(float ctrl, float act, const float* prm) {
  const float ctrlclamp = fminf(fmaxf(ctrl, 0.f), 1.0f), actclamp = fminf(fmaxf(act, 0.f), 1.0f);
  const float tau_act = prm[0] * (0.5f + 1.5f * actclamp);
  const float tau_deact = prm[1] / (0.5f + 1.5f * actclamp);
  const float dctrl = ctrlclamp - act;
  const float tau = muscle_dynamics_timescale(dctrl, tau_act, tau_deact, prm[2]);
  return dctrl / fmaxf(MJ_MINVAL, tau);
}
