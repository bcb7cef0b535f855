// k_body_stages.cu -- the individually callable stages that read a finished forward pass: rne_postconstraint, subtree_vel, jac,
// xfrc_accumulate, tendon and deriv_smooth_vel.  One launch each, over d's world range.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): smooth.py:1744 rne_postconstraint, :3614 subtree_vel, :4197 tendon (fixed
// tendons), support.py:583 jac, :314 xfrc_accumulate (apply_ft, :304), derivative.py:1117 deriv_smooth_vel.  rne_postconstraint and
// subtree_vel run the code k_sensor runs for the sensors that need them, whatever the model's sensors are; jac and
// xfrc_accumulate share their per-dof code with k_constraint and k_velocity; tendon writes what k_position writes; deriv_smooth_vel
// builds each tree's block of M - dt qDeriv with the implicitfast integrator's tree_implicit_a.  The shared statements live in the
// k_body_*.cuh fragments, included in place, so that the kernels that had them before compile exactly as they did.
#include <math.h>

#include "k_body_vec.cuh"
#include "mjb_implicit_a.cuh"
#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

namespace {

template <bool BAT>
__global__ void __launch_bounds__(32) k_rne_postconstraint(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d) {
  extern __shared__ float smem[];  // nbody x (cfrc_ext 6 | cacc / cfrc_int 6)
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  const int nb = m.nbody, nv = m.nv;
#include "k_body_rne_post.cuh"
}

template <bool BAT>
__global__ void __launch_bounds__(32) k_subtree_vel(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d) {
  extern __shared__ float smem[];  // nbody x (linvel 3 | angmom 3 | bodyvel lin 3)
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  const int nb = m.nbody;
#include "k_body_subtree_vel.cuh"
}

// Jacobian column `dof` of point on body b, as k_constraint's jac_cols opens (without the time derivative)
__device__ __forceinline__ void jac_column(const ModelDev& m, const float* cdof, const float* scom, v3 point, int b, int dof, v3* jp, v3* jr) {
  v3 dp_unused, dr_unused, *dp = &dp_unused, *dr = &dr_unused;
#include "k_body_jac.cuh"
}

// One thread per (world, dof): consecutive threads store consecutive dofs of a Jacobian row.  A body id outside [0, nbody) gives NaN
// in every entry of the world's rows (nothing is read through it).
__global__ void __launch_bounds__(256) k_jac(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, float* __restrict__ jacp,
                                             float* __restrict__ jacr, const float* __restrict__ point, const int* __restrict__ body) {
  const int nv = m.nv;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)d.wn * nv) return;
  const int wl = (int)(i / nv), dof = (int)(i - (long long)wl * nv), w = d.w0 + wl;
  const size_t wb = (size_t)w;
  const int b = body[w];
  v3 jp, jr;
  if (b < 0 || b >= m.nbody) jp = jr = mk3(NAN, NAN, NAN);
  else jac_column(m, d.cdof + wb * nv * 6, d.subtree_com + wb * m.nbody * 3, ld3(point + 3 * wb), b, dof, &jp, &jr);
  if (jacp) { float* o = jacp + wb * 3 * nv + dof; o[0] = jp.x; o[nv] = jp.y; o[2 * nv] = jp.z; }
  if (jacr) { float* o = jacr + wb * 3 * nv + dof; o[0] = jr.x; o[nv] = jr.y; o[2 * nv] = jr.z; }
}

// One thread per (world, dof): qfrc += J^T xfrc_applied at the dof.
__global__ void __launch_bounds__(256) k_xfrc_accumulate(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, float* __restrict__ qfrc) {
  const int nv = m.nv;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)d.wn * nv) return;
  const int wl = (int)(i / nv), dof = (int)(i - (long long)wl * nv), w = d.w0 + wl;
  const size_t wb = (size_t)w;
  const int nb = m.nbody, dd = dof;
  const float* cdof = d.cdof + wb * nv * 6;
#include "k_body_xfrc.cuh"
  qfrc[wb * nv + dd] += acc;
}

// One thread per (world, tendon): the fixed tendon's length and Jacobian row, as k_position's tendon stage writes them.
template <bool BAT>
__global__ void __launch_bounds__(256) k_tendon(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)d.wn * mp.ntendon) return;
  const int wl = (int)(i / mp.ntendon), t = (int)(i - (long long)wl * mp.ntendon), w = d.w0 + wl;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  d.ten_length[wb * m.ntendon + t] = tendon_length(m, t, d.qpos + wb * m.nq);
  for (int k = m.ten_J_rowadr[t]; k < m.ten_J_rowadr[t] + m.ten_J_rownnz[t]; k++) d.ten_J[wb * m.nJten + k] = m.ten_J0[k];
}

// One warp per world: each tree's block of M - dt qDeriv (the implicitfast terms: affine actuators, dof and tendon damping, and with
// FLUID the fluid forces, their ellipsoid B symmetrized with SYM: a model whose integrator is implicitfast) in shared memory, then its
// lower triangle back to M's CSR entries.
template <bool FLUID, bool SYM, bool BAT>
__global__ void __launch_bounds__(32) k_deriv_smooth_vel(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, float* __restrict__ out,
                                                          const __grid_constant__ FluidDev f) {
  extern __shared__ float smem[];  // maxtree x maxtree
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  const float* Mw = d.M + wb * m.nC;
  float* ow = out + wb * m.nC;
  const bool damper = !(m.disableflags & DSBL_DAMPER);
#pragma unroll 1
  for (int t = 0; t < m.ntree; t++) {
    const int start = m.tree_dofadr[t], n = m.tree_dofnum[t];
    tree_implicit_a<FLUID, SYM>(m, d, wb, Mw, start, n, n, m.timestep, true, damper, smem, lane, f);
    const int e0 = m.M_rowadr[start], e1 = m.M_rowadr[start + n - 1] + m.M_rownnz[start + n - 1];
#pragma unroll 1
    for (int e = e0 + lane; e < e1; e += 32) ow[e] = smem[(m.M_entry_row[e] - start) * n + (m.M_colind[e] - start)];
    __syncwarp();
  }
}

unsigned flat_grid(long long n) { return (unsigned)((n + 255) / 256); }

}  // namespace

cudaError_t launch_rne_postconstraint(const ModelDev& m, const DataDev& d, cudaStream_t s) {
  return launch(m.batched ? k_rne_postconstraint<true> : k_rne_postconstraint<false>, d.wn, 32, (size_t)12 * m.nbody * sizeof(float), s, m, d);
}
cudaError_t launch_subtree_vel(const ModelDev& m, const DataDev& d, cudaStream_t s) {
  return launch(m.batched ? k_subtree_vel<true> : k_subtree_vel<false>, d.wn, 32, (size_t)12 * m.nbody * sizeof(float), s, m, d);
}
// jac and xfrc_accumulate launch nothing for a model without dofs (an empty grid is not a valid launch)
cudaError_t launch_jac(const ModelDev& m, const DataDev& d, float* jacp, float* jacr, const float* point, const int* body, cudaStream_t s) {
  if ((long long)d.wn * m.nv == 0) return cudaSuccess;
  return launch(k_jac, flat_grid((long long)d.wn * m.nv), 256, 0, s, m, d, jacp, jacr, point, body);
}
cudaError_t launch_xfrc_accumulate(const ModelDev& m, const DataDev& d, float* qfrc, cudaStream_t s) {
  if ((long long)d.wn * m.nv == 0) return cudaSuccess;
  return launch(k_xfrc_accumulate, flat_grid((long long)d.wn * m.nv), 256, 0, s, m, d, qfrc);
}
cudaError_t launch_tendon(const ModelDev& m, const DataDev& d, cudaStream_t s) {
  if (m.ntendon == 0) return cudaSuccess;
  return launch(m.batched ? k_tendon<true> : k_tendon<false>, flat_grid((long long)d.wn * m.ntendon), 256, 0, s, m, d);
}
size_t smem_deriv_smooth_vel(const ModelDev& m) { return (size_t)m.maxtree * m.maxtree * sizeof(float); }
cudaError_t launch_deriv_smooth_vel(const ModelDev& m, const DataDev& d, float* out, cudaStream_t s, const FluidDev& f) {
  const size_t smem = smem_deriv_smooth_vel(m);
  if (f.has_fluid && m.integrator == INT_IMPLICITFAST)
    return launch(m.batched ? k_deriv_smooth_vel<true, true, true> : k_deriv_smooth_vel<true, true, false>, d.wn, 32, smem, s, m, d, out, f);
  if (f.has_fluid)
    return launch(m.batched ? k_deriv_smooth_vel<true, false, true> : k_deriv_smooth_vel<true, false, false>, d.wn, 32, smem, s, m, d, out, f);
  return launch(m.batched ? k_deriv_smooth_vel<false, true, true> : k_deriv_smooth_vel<false, true, false>, d.wn, 32, smem, s, m, d, out, f);
}
