// Test-only: compiles the muscle model (mujoco_warp_b200/csrc/mjb_muscle.cuh) as plain host C++, so that the device source of the gain,
// bias and activation dynamics is checked against the reference's known answers and an fp64 restatement on the CPU.  Nothing in the
// product path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include "../../mujoco_warp_b200/csrc/mjb_muscle.cuh"

extern "C" float mh_gain_length(float length, float lmin, float lmax) { return muscle_gain_length(length, lmin, lmax); }
extern "C" float mh_gain(float len, float vel, float lr0, float lr1, float acc0, const float* prm) { return muscle_gain(len, vel, lr0, lr1, acc0, prm); }
extern "C" float mh_bias(float len, float lr0, float lr1, float acc0, const float* prm) { return muscle_bias(len, lr0, lr1, acc0, prm); }
extern "C" float mh_timescale(float dctrl, float tau_act, float tau_deact, float smooth_width) {
  return muscle_dynamics_timescale(dctrl, tau_act, tau_deact, smooth_width);
}
extern "C" float mh_dynamics(float ctrl, float act, const float* prm) { return muscle_dynamics(ctrl, act, prm); }
