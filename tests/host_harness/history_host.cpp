// Test-only: compiles the delay ring buffers (mujoco_warp_b200/csrc/mjb_history.cuh) as plain host C++, so that the device source of
// the buffer reads, inserts and the sensor rule replays the reference's own vectors on the CPU.  Nothing in the product path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include "../../mujoco_warp_b200/csrc/mjb_history.cuh"

extern "C" void hh_read(const float* buf, int n, int dim, float t, int interp, float* out) { hist_read(buf, n, dim, t, interp, out); }
extern "C" void hh_insert(float* buf, int n, int dim, float t, const float* value) { hist_insert(buf, n, dim, t, value); }
extern "C" void hh_sensor(float* buf, int n, int dim, int interp, float delay, float period, float t, float* data) {
  float fresh[16];
  hist_sensor(buf, n, dim, interp, delay, period, t, data, fresh);
}
