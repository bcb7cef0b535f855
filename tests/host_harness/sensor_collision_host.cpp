// Test-only: compiles the collision-sensor header (mujoco_warp_b200/csrc/mjb_sensor_collision.cuh) as plain host C++, so that the device
// source of the sensor pairs' colliders and of the per-sensor reduction runs on the CPU against the reference-generated fixtures
// (tests/golden/sensor_collision_*.npz).  k_sensor_collision's loop over one world is restated here; nothing in the product path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <vector>
#ifndef __noinline__
#define __noinline__
#endif
using std::max;
using std::min;
// warp intrinsics referenced by helpers in mjb_math.cuh that the routines here never call
static inline float __shfl_xor_sync(unsigned, float v, int) { return v; }
static inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
static inline int __shfl_up_sync(unsigned, int v, int) { return v; }
static inline float __shfl_sync(unsigned, float v, int) { return v; }
static inline int __shfl_sync(unsigned, int v, int) { return v; }
static inline unsigned __ballot_sync(unsigned, int p) { return p ? 1u : 0u; }
static inline void __syncwarp(unsigned = 0xffffffffu) {}
#include "../../mujoco_warp_b200/csrc/mjb_sensor_collision.cuh"

static ModelDev g_m;
static SensorCollisionDev g_c;

// the model fields the routines read, set by name like the C ABI does
extern "C" int hsc_set_int(const char* name, int v) {
#define X(n) if (!strcmp(name, #n)) { g_m.n = v; return 0; }
  X(ngeom) X(nsensor) X(nsensordata) X(disableflags) X(ccd_iterations)
#undef X
#define X(n) if (!strcmp(name, #n)) { g_c.n = v; return 0; }
  MJB_SENSCOL_INTS(X)
#undef X
  return -1;
}
extern "C" int hsc_set_float(const char* name, float v) {
  if (!strcmp(name, "ccd_tolerance")) { g_m.ccd_tolerance = v; return 0; }
  return -1;
}
extern "C" int hsc_set_array(const char* name, const void* p) {
#define X(n) if (!strcmp(name, #n)) { g_m.n = (const int*)p; return 0; }
  X(geom_type) X(geom_dataid) X(mesh_vertadr) X(mesh_vertnum) X(mesh_graphadr) X(mesh_graph) X(mesh_polynum) X(mesh_polyadr) X(mesh_polyvertadr)
  X(mesh_polyvertnum) X(mesh_polyvert) X(mesh_polymapadr) X(mesh_polymapnum) X(mesh_polymap) X(sensor_type) X(sensor_datatype) X(sensor_adr) X(sensor_dim)
#undef X
#define X(n) if (!strcmp(name, #n)) { g_m.n = (const float*)p; return 0; }
  X(geom_size) X(geom_margin) X(pair_margin) X(mesh_vert) X(mesh_polynormal) X(sensor_cutoff)
#undef X
#define X(n) if (!strcmp(name, #n)) { g_c.n = (const int*)p; return 0; }
  MJB_SENSCOL_IARRS(X)
#undef X
  return -1;
}

// k_sensor_collision for every world: the pairs, then the sensors; writes the collision sensors' slots of sensordata (nworld, nsensordata)
// and returns the number of pairs whose EPA horizon overflowed
extern "C" int hsc_run(int nworld, const float* geom_xpos, const float* geom_xmat, float* sensordata) {
  std::vector<float> pairs((size_t)SC_WORDS * max(g_c.nsensorcollision, 1));
  std::vector<float> scratch(ccd_scratch_words(g_c.sensor_collision_epa_iterations) + 64);
  int novf = 0;
  for (int w = 0; w < nworld; w++) {
    for (int p = 0; p < g_c.nsensorcollision; p++) {
      const int* pr = g_c.sensor_collision_pair + SC_PAIR_WORDS * p;
      novf += sensor_pair(g_m, geom_xpos + (size_t)w * 3 * g_m.ngeom, geom_xmat + (size_t)w * 9 * g_m.ngeom, pr[0], pr[1], pr[2],
                          g_c.sensor_collision_epa_iterations, scratch.data(), pairs.data() + SC_WORDS * p);
    }
    for (int i = 0; i < g_c.nsensorcollision_sensor; i++) sensor_collision_reduce(g_m, g_c, i, pairs.data(), sensordata + (size_t)w * g_m.nsensordata);
  }
  return novf;
}
