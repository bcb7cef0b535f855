// Test-only: compiles the assembly of one tree's block of the velocity-implicit matrix (tree_implicit_a in
// mujoco_warp_b200/csrc/mjb_implicit_a.cuh) as host C++.  The warp's 32 lanes run as 32 threads and __syncwarp is a barrier among them,
// so the lanes split the work exactly as they do on the GPU; the caller's A buffer may carry a guard region around the block, which shows
// writes outside it.  Nothing in the product path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <algorithm>
#include <barrier>
#include <thread>
#include <vector>
using std::max;
using std::min;
static std::barrier<>* g_warp = nullptr;
static inline void __syncwarp(unsigned = 0xffffffffu) { g_warp->arrive_and_wait(); }
static inline float __shfl_xor_sync(unsigned, float v, int) { return v; }
static inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
static inline int __shfl_up_sync(unsigned, int v, int) { return v; }
#include "../../mujoco_warp_b200/csrc/mjb_implicit_a.cuh"

// The int and float arrays of the model in the order of IAH_IARRS / IAH_FARRS, and of one world's data in the order of IAH_DARRS.
#define IAH_IARRS(X) X(M_rowadr) X(M_rownnz) X(M_entry_row) X(M_colind) X(body_isdofancestor) X(dof_bodyid) X(moment_rowadr0) X(moment_rownnz0) \
  X(moment_colind0) X(actuator_gaintype) X(actuator_biastype) X(actuator_forcelimited) X(actuator_dyntype) X(actuator_actadr) X(actuator_actnum) \
  X(actuator_actlimited) X(actuator_actearly) X(ten_J_rowadr) X(ten_J_rownnz) X(ten_J_colind)
#define IAH_FARRS(X) X(dof_damping) X(actuator_gainprm) X(actuator_biasprm) X(actuator_forcerange) X(actuator_dynprm) X(actuator_actrange) \
  X(tendon_damping) X(ten_J0)
#define IAH_DARRS(X) X(actuator_force) X(actuator_moment) X(act) X(act_dot) X(ctrl)

// sizes: nv, nu, na, ntendon, nJmom, disableflags.  Writes the block of tree dofs [start, start + n) (leading dimension ld) at A.
extern "C" void iah_tree_a(const int* sizes, float dt, const int* const* iarr, const float* const* farr, const float* const* darr, const float* M,
                           int start, int n, int ld, int implicitfast, int damper, float* A) {
  ModelDev m;
  memset(&m, 0, sizeof m);
  m.nv = sizes[0]; m.nu = sizes[1]; m.na = sizes[2]; m.ntendon = sizes[3]; m.nJmom = sizes[4]; m.disableflags = sizes[5];
  m.timestep = dt;
  int k = 0;
#define X(f) m.f = iarr[k++];
  IAH_IARRS(X)
#undef X
  k = 0;
#define X(f) m.f = farr[k++];
  IAH_FARRS(X)
#undef X
  DataDev d;
  memset(&d, 0, sizeof d);
  k = 0;
#define X(f) d.f = const_cast<float*>(darr[k++]);
  IAH_DARRS(X)
#undef X
  std::barrier<> warp(32);
  g_warp = &warp;
  std::vector<std::thread> lanes;
  for (int lane = 0; lane < 32; lane++)
    lanes.emplace_back([&, lane] { tree_implicit_a<false>(m, d, 0, M, start, n, ld, dt, implicitfast != 0, damper != 0, A, lane, FluidDev{}); });
  for (auto& t : lanes) t.join();
  g_warp = nullptr;
}
