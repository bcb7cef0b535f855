// Test-only: compiles the contact-sensor header (mujoco_warp_b200/csrc/mjb_sensor_contact.cuh) as plain host C++, so that the device
// source of the force decode, the site volumes, the side matching, the sort and the slot writers runs on the CPU against the fp64
// restatement of tests/contact_sensor_oracle.py.  The sort runs as one lane (its comparators of one step are disjoint, so the lane count
// does not change the result).  Nothing in the product path uses this file.
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
#include "../../mujoco_warp_b200/csrc/mjb_sensor_contact.cuh"

extern "C" void hsc_force(int cone, int njmax, const float* force, const int* adr, const float* mu, int dim, float* out) {
  contact_force_decode(cone, njmax, force, adr, mu, dim, out);
}
extern "C" int hsc_inside(const float* pos, const float* mat, const float* size, int type, const float* p) {
  return contact_inside_site(ld3(pos), mat, ld3(size), type, ld3(p));
}
extern "C" int hsc_match(const int* parent, int otype, int oid, int rtype, int rid, int g1, int b1, int g2, int b2) {
  return contact_match_dir(parent, otype, oid, rtype, rid, g1, b1, g2, b2);
}
extern "C" int hsc_slot_size(int dataspec) { return contact_slot_size(dataspec); }
extern "C" void hsc_slot(int dataspec, int nmatch, float dir, const float* f, float dist, const float* pos, const float* frame, float* out) {
  contact_slot_write(dataspec, nmatch, dir, f, dist, pos, frame, out);
}
// netforce over n matches: dir (n), f (n, 6), pos (n, 3), frame (n, 9)
extern "C" void hsc_netforce(int dataspec, int nmatch, int n, const float* dir, const float* f, const float* pos, const float* frame, float* out) {
  float acc[CNF_WORDS] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int i = 0; i < n; i++) contact_netforce_add(dir[i], f + 6 * i, pos + 3 * i, frame + 9 * i, acc);
  contact_netforce_write(dataspec, nmatch, acc, out);
}
extern "C" void hsc_sort(int* cid, float* crit, float* dir, int n) { contact_sort(cid, crit, dir, n, 0, 1, [] {}); }
