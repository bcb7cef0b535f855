// Test-only: compiles the row rule the solver and inverse dynamics share (MJB_ROW_FORCE_STATE / row_force_state in
// mujoco_warp_b200/csrc/mjb_linesearch.cuh) as plain host C++, so that the device source runs on the CPU against the reference's
// inverse-dynamics fixture (tests/golden/inverse_vectors.npz).  Nothing in the product path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>
#ifndef __noinline__
#define __noinline__
#endif
using std::max;
using std::min;
static inline float __shfl_xor_sync(unsigned, float v, int) { return v; }
static inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
static inline int __shfl_up_sync(unsigned, int v, int) { return v; }
static inline float __shfl_sync(unsigned, float v, int) { return v; }
static inline int __shfl_sync(unsigned, int v, int) { return v; }
static inline unsigned __ballot_sync(unsigned, int p) { return p ? 1u : 0u; }
static inline void __syncwarp(unsigned = 0xffffffffu) {}
#include "../../mujoco_warp_b200/csrc/mjb_linesearch.cuh"

// force / state of rows [0, nefc) of one world at Jaref; rinfo / rfri: the elliptic row map (NULL for models without elliptic cones)
extern "C" void irh_rows(int nefc, int ne, int nf, const float* jaref, const float* D, const float* floss, const int* rinfo, const float* rfri,
                         float* force, int* state) {
  for (int r = 0; r < nefc; r++) {
    float f; int st; bool cone0 = false;
    if (rinfo) row_force_state<true>(r, ne, nf, jaref[r], D[r], floss, rinfo, rfri, jaref, D, f, st, cone0);
    else row_force_state<false>(r, ne, nf, jaref[r], D[r], floss, rinfo, rfri, jaref, D, f, st, cone0);
    force[r] = f; state[r] = st;
  }
}
