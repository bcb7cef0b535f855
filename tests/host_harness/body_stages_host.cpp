// Test-only: compiles the statement fragments the body-stage kernels share with k_sensor, k_constraint and k_velocity
// (mujoco_warp_b200/csrc/k_body_subtree_vel.cuh, k_body_rne_post.cuh, k_body_jac.cuh, k_body_xfrc.cuh) as host C++, inside the same
// surroundings k_body_stages.cu gives them, so that the device source runs on the CPU against the reference's fixtures
// (tests/golden/body_stage_*.npz).  The warp fragments run their 32 lanes as 32 threads with __syncwarp as a barrier among them, so the
// lanes split the work exactly as they do on the GPU.  Nothing in the product path uses this file.
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
#include "../../mujoco_warp_b200/csrc/k_body_vec.cuh"
#include "../../mujoco_warp_b200/csrc/mjb_types.cuh"

// The model's int and float arrays in the order of BSH_IARRS / BSH_FARRS, one world's data in the order of BSH_DARRS (each a world's
// slice: the fragments run as world 0).
#define BSH_IARRS(X) X(body_parentid) X(body_rootid) X(body_dofnum) X(body_dofadr) X(body_childadr) X(body_childid) X(level_adr) X(level_body) \
  X(dof_bodyid) X(body_isdofancestor)
#define BSH_FARRS(X) X(body_mass) X(body_inertia) X(body_subtreemass)
#define BSH_DARRS(X) X(cvel) X(ximat) X(xipos) X(subtree_com) X(cdof) X(cdof_dot) X(cinert) X(qvel) X(qacc) X(xfrc_applied) X(xmat) X(xpos)

static void bind(const int* sizes, const float* gravity, const int* const* iarr, const float* const* farr, float* const* darr, ModelDev* m, DataDev* d) {
  memset(m, 0, sizeof *m);
  memset(d, 0, sizeof *d);
  m->nbody = sizes[0]; m->nv = sizes[1]; m->nlevel = sizes[2]; m->disableflags = sizes[3];
  m->gravity_x = gravity[0]; m->gravity_y = gravity[1]; m->gravity_z = gravity[2];
  int k = 0;
#define X(f) m->f = iarr[k++];
  BSH_IARRS(X)
#undef X
  k = 0;
#define X(f) m->f = farr[k++];
  BSH_FARRS(X)
#undef X
  k = 0;
#define X(f) d->f = darr[k++];
  BSH_DARRS(X)
#undef X
  d->nworld = 1;
}

template <class F>
static void run_warp(F body) {
  std::barrier<> warp(32);
  g_warp = &warp;
  std::vector<std::thread> lanes;
  for (int lane = 0; lane < 32; lane++) lanes.emplace_back([&, lane] { body(lane); });
  for (auto& t : lanes) t.join();
  g_warp = nullptr;
}

// sizes: nbody, nv, nlevel, disableflags.  subtree_linvel / subtree_angmom (nbody, 3) of world 0.
extern "C" void bsh_subtree_vel(const int* sizes, const float* gravity, const int* const* iarr, const float* const* farr, float* const* darr,
                                float* subtree_linvel, float* subtree_angmom) {
  ModelDev mm;
  DataDev d;
  bind(sizes, gravity, iarr, farr, darr, &mm, &d);
  d.subtree_linvel = subtree_linvel;
  d.subtree_angmom = subtree_angmom;
  const ModelDev& m = mm;
  std::vector<float> scratch(12 * (size_t)m.nbody);
  float* smem = scratch.data();
  run_warp([&](int lane) {
    const size_t wb = 0;
    const int nb = m.nbody;
#include "../../mujoco_warp_b200/csrc/k_body_subtree_vel.cuh"
  });
}

// rne_postconstraint of world 0 without equality rows or contacts (ne = 0, no contact in the world's block): cfrc_ext from xfrc_applied,
// cacc with qacc, cfrc_int.  Outputs (nbody, 6) each.
extern "C" void bsh_rne_postconstraint(const int* sizes, const float* gravity, const int* const* iarr, const float* const* farr, float* const* darr,
                                       float* cacc, float* cfrc_int, float* cfrc_ext) {
  ModelDev mm;
  DataDev d;
  bind(sizes, gravity, iarr, farr, darr, &mm, &d);
  int zero[2] = {0, 0};
  d.ne = zero; d.world_conadr = zero; d.world_ncon = zero + 1;
  d.cacc = cacc; d.cfrc_int = cfrc_int; d.cfrc_ext = cfrc_ext;
  const ModelDev& m = mm;
  std::vector<float> scratch(12 * (size_t)m.nbody);
  float* smem = scratch.data();
  run_warp([&](int lane) {
    const int w = 0;
    const size_t wb = 0;
    const int nb = m.nbody, nv = m.nv;
#include "../../mujoco_warp_b200/csrc/k_body_rne_post.cuh"
  });
}

static void jac_column(const ModelDev& m, const float* cdof, const float* scom, v3 point, int b, int dof, v3* jp, v3* jr) {
  v3 dp_unused, dr_unused, *dp = &dp_unused, *dr = &dr_unused;
#include "../../mujoco_warp_b200/csrc/k_body_jac.cuh"
}

// jacp / jacr (3, nv) of point on body b in world 0, and qfrc (nv) += J^T xfrc_applied
extern "C" void bsh_jac(const int* sizes, const float* gravity, const int* const* iarr, const float* const* farr, float* const* darr, const float* point,
                        int b, float* jacp, float* jacr) {
  ModelDev m;
  DataDev d;
  bind(sizes, gravity, iarr, farr, darr, &m, &d);
  const int nv = m.nv;
  for (int dof = 0; dof < nv; dof++) {
    v3 jp, jr;
    jac_column(m, d.cdof, d.subtree_com, ld3(point), b, dof, &jp, &jr);
    jacp[dof] = jp.x; jacp[nv + dof] = jp.y; jacp[2 * nv + dof] = jp.z;
    jacr[dof] = jr.x; jacr[nv + dof] = jr.y; jacr[2 * nv + dof] = jr.z;
  }
}
extern "C" void bsh_xfrc_accumulate(const int* sizes, const float* gravity, const int* const* iarr, const float* const* farr, float* const* darr, float* qfrc) {
  ModelDev mm;
  DataDev d;
  bind(sizes, gravity, iarr, farr, darr, &mm, &d);
  const ModelDev& m = mm;
  const size_t wb = 0;
  const int nb = m.nbody;
  const float* cdof = d.cdof;
  for (int dd = 0; dd < m.nv; dd++) {
#include "../../mujoco_warp_b200/csrc/k_body_xfrc.cuh"
    qfrc[dd] += acc;
  }
}
