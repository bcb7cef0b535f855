// Test-only: compiles the magnetometer / camprojection / insidesite / tendonactfrc header (mujoco_warp_b200/csrc/mjb_sensor_extra.cuh)
// as plain host C++, so that the device source runs on the CPU against the reference's fixtures (tests/golden/sensor_extra_*.npz).
// Nothing in the product path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>
using std::max;
using std::min;
static inline float __shfl_xor_sync(unsigned, float v, int) { return v; }
static inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
static inline int __shfl_up_sync(unsigned, int v, int) { return v; }
static inline float __shfl_sync(unsigned, float v, int) { return v; }
static inline int __shfl_sync(unsigned, int v, int) { return v; }
static inline unsigned __ballot_sync(unsigned, int p) { return p ? 1u : 0u; }
static inline void __syncwarp(unsigned = 0xffffffffu) {}
#include "../../mujoco_warp_b200/csrc/mjb_sensor_extra.cuh"

extern "C" void hse_magnetometer(const float* site_xmat, const float* magnetic, float* out) { st3(out, sensor_magnetometer(site_xmat, ld3(magnetic))); }
extern "C" void hse_camprojection(const float* target, const float* cam_pos, const float* cam_mat, float fovy, const float* intrinsic, const float* sensorsize,
                                  const int* res, float* out) {
  sensor_camprojection(ld3(target), ld3(cam_pos), cam_mat, fovy, intrinsic, sensorsize, res, out);
}
extern "C" int hse_insidesite(int objtype, int objid, const float* pos, const float* subtree_com, float body_mass, float body_subtreemass,
                              const float* site_pos, const float* site_mat, const float* site_size, int site_type) {
  const v3 p = sensor_inside_point(objtype, objid, pos, subtree_com, body_mass, body_subtreemass);
  return contact_inside_site(ld3(site_pos), site_mat, ld3(site_size), site_type, p);
}
extern "C" float hse_tendon_actfrc(int nu, const int* trntype, const int* trnid, const float* actuator_force, int tendon) {
  return sensor_tendon_actfrc(nu, trntype, trnid, actuator_force, tendon);
}
