// k_body_vec.cuh -- the two small vector helpers the k_body_*.cuh fragments call, shared by k_sensor.cu and k_body_stages.cu, which
// include those fragments.
#pragma once
#include "mjb_math.cuh"

static __device__ __forceinline__ float comp3(v3 v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : v.z); }
static __device__ __forceinline__ v3 mat_t_vec(const float* m, v3 v) {  // m^T v
  return mk3(m[0] * v.x + m[3] * v.y + m[6] * v.z, m[1] * v.x + m[4] * v.y + m[7] * v.z, m[2] * v.x + m[5] * v.y + m[8] * v.z);
}
