// k_velocity.cu -- fused velocity / actuation / acceleration stage.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): forward.py:680 _actuator_velocity; smooth.py:2179-2285 com_vel;
// passive.py:73-206,631-667 (joint springs/dampers, passive sum); smooth.py:1353-1515 rne (incl. 7 per-level atomic
// launches of _cfrc_backward); forward.py:756-1149 fwd_actuation (stateless FIXED/AFFINE gain, NONE/AFFINE bias, joint
// transmission); forward.py:1255-1324 fwd_acceleration with support.py:259-324 xfrc_accumulate and the per-tree dense
// Cholesky factor+solve of M (smooth.py:3227-3265) -- about 30 launches there, one here.
//
// A team of LPW lanes owns one world, a warp owns G = 32 / LPW consecutive worlds (mjb_team.cuh); inputs and outputs move as
// bulk-async (TMA) copies of the contiguous [G][n] blocks.  Tree passes are level-synchronous in shared memory, children
// are gathered by the parent in a fixed order (no float atomics => bit-reproducible), the inertia blocks are factored by the
// team in shared memory directly in the qLD layout (upper factor, row-major), so qLD leaves as one bulk store.

#include "mjb_fluid.cuh"
#include "mjb_math.cuh"
#include "mjb_muscle.cuh"
#include "mjb_team.cuh"
#include "mjb_types.cuh"

namespace {

struct VelLayout { int qvel, cdof, cinert, cvel, cdofdot, cacc, cfrc, qpas, qbias, qact, qsm, qld, x, af, total; };
// Per-world words of shared memory, sized by what is live in each phase: 3.1 KB for the humanoid, so that an SM holds 64 worlds
// at once and 8192 worlds fit on 132 SMs in one round (the kernel is latency bound, DESIGN.md §3).  qfrc_passive and qfrc_bias
// stay live until qfrc_smooth is formed and sit outside the region below: qfrc_smooth is formed in place in qfrc_passive's slot
// (qfrc_passive goes straight to global memory, so no bulk store reads that slot), and the solve's right-hand side / solution
// takes qfrc_bias's slot once its bulk store has drained.  The region holds, in turn:
//  - the tree-pass fields; cfrc_int takes cdof_dot's slot (sized for both) once the cacc pass has read it and its bulk store has
//    drained;
//  - the actuation fields (qfrc_actuator, actuator forces) in the slots of cinert and qvel, both dead after rne and never the
//    source of a bulk store (or past the tree-pass fields when they do not fit there);
//  - the n x n factor (Data.qLD layout), once the bulk stores that read the region have drained; M is scattered into it straight
//    from global memory.  cdof stays intact until then: the applied-wrench term of qfrc_smooth reads it.
__host__ __device__ inline VelLayout vel_layout(const ModelDev& m) {
  VelLayout L;
  int o = 0;
  auto pad = [](int n) { return (n + 3) & ~3; };  // padded: a field's group block [G][n] starts 16 B aligned
  auto take = [&](int n) { int r = o; o += pad(n); return r; };
  L.qpas = take(m.nv); L.qbias = take(m.nv);
  L.qsm = L.qpas; L.x = L.qbias;
  const int a0 = o;
  L.cdof = take(6 * m.nv); L.cinert = take(10 * m.nbody); L.qvel = take(m.nv);
  // cdof_dot's slot also holds cfrc_int later, so it is sized for the larger of the two (models with more bodies than dofs / 6)
  L.cvel = take(6 * m.nbody); L.cdofdot = take(6 * (m.nv > m.nbody ? m.nv : m.nbody)); L.cacc = take(6 * m.nbody);
  L.cfrc = L.cdofdot;
  if (pad(m.nv) + pad(m.nu) <= L.cvel - L.cinert) { L.qact = L.cinert; L.af = L.cinert + pad(m.nv); }
  else { L.qact = take(m.nv); L.af = take(m.nu); }
  L.qld = a0;
  if (o - a0 < pad(m.qld_total)) o = a0 + pad(m.qld_total);
  L.total = o;
  return L;
}

// Dense Cholesky of one tree's inertia block by a team, in the qLD layout: U (n x n, row-major, ld = n) starts as the upper
// triangle of M with zeros below and ends as the factor U with U^T U = M (= the reference's L^T, smooth.py:3227-3265).
// Row j of U needs the columns above it: U[j][i] = (M[j][i] - sum_{k<j} U[k][j] U[k][i]) / U[j][j]; lanes take the entries
// i = j + sub, j + sub + LPW, ... .  The right-hand side rides along as a virtual column i = n (y = U^-T b comes out of the
// same sweep), then the backward substitution U x = y runs column by column.  x holds b on entry, the solution on exit.
template <int LPW>
__device__ __forceinline__ void team_chol_upper(float* U, int n, float* x, bool solve, int sub) {
#pragma unroll 1
  for (int j = 0; j < n; j++) {
    const int iend = solve ? n + 1 : n;
#pragma unroll 1
    for (int i = j + sub; i < iend; i += LPW) {
      const bool rhs = i == n;
      const float* col = rhs ? x : U + i;
      const int cs = rhs ? 1 : n;
      float s0 = rhs ? x[j] : U[j * n + i], s1 = 0.f;
      int k = 0;
#pragma unroll 4
      for (; k + 1 < j; k += 2) {
        s0 -= U[k * n + j] * col[k * cs];
        s1 -= U[(k + 1) * n + j] * col[(k + 1) * cs];
      }
      if (k < j) s0 -= U[k * n + j] * col[k * cs];
      if (rhs) x[j] = s0 + s1; else U[j * n + i] = s0 + s1;
    }
    __syncwarp();
    const float piv = sqrtf(fmaxf(U[j * n + j], MJ_MINVAL)), inv = 1.0f / piv;
    __syncwarp();
#pragma unroll 1
    for (int i = j + sub; i < iend; i += LPW) {
      if (i == n) x[j] *= inv;
      else U[j * n + i] = i == j ? piv : U[j * n + i] * inv;
    }
    __syncwarp();
  }
  if (!solve) return;
#pragma unroll 1
  for (int j = n - 1; j >= 0; j--) {  // backward: U x = y, column j of U
    const float xj = x[j] / U[j * n + j];
    __syncwarp();
#pragma unroll 1
    for (int k = sub; k < j; k += LPW) x[k] -= U[k * n + j] * xj;
    if (sub == 0) x[j] = xj;
    __syncwarp();
  }
}

// PEXT = the model uses gravity compensation or free / ball joint springs (kept out of the plain instantiation).  k_velocity_fluid is
// the instance for models with fluid forces (with PEXT).  Both kernels take the body below as text, so that the plain instances
// compile exactly as they did before the fluid one existed (an inlined shared function compiles to different code).
template <bool PEXT, int LPW, bool BAT>
__global__ void __launch_bounds__(256)
k_velocity(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int mask) {
  constexpr bool FLUID = false;
  [[maybe_unused]] constexpr FluidDev f{};
#include "k_velocity_body.cuh"
}

template <int LPW, bool BAT>
__global__ void __launch_bounds__(256)
k_velocity_fluid(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int mask, const __grid_constant__ FluidDev f) {
  constexpr bool PEXT = true, FLUID = true;
#include "k_velocity_body.cuh"
}

}  // namespace

template <bool PEXT>
static TeamKernel vel_instance(int lpw, bool bat) {
  if (bat) return k_velocity<PEXT, 32, true>;
  return lpw == 8 ? k_velocity<PEXT, 8, false> : lpw == 16 ? k_velocity<PEXT, 16, false> : k_velocity<PEXT, 32, false>;
}
// has_gravcomp also flags free / ball joint springs (io.py put_model); tendons live in the same instantiation
static bool vel_pext(const ModelDev& m) { return m.has_gravcomp || m.ntendon > 0; }
static TeamKernel vel_kernel(const ModelDev& m, int lpw) { return vel_pext(m) ? vel_instance<true>(lpw, m.batched) : vel_instance<false>(lpw, m.batched); }
// models with fluid forces: one instance per lane count with everything the other two cover as well
using FluidKernel = void (*)(ModelDev, DataDev, int, FluidDev);
static FluidKernel vel_kernel_fluid(const ModelDev& m, int lpw) {
  if (m.batched) return k_velocity_fluid<32, true>;
  return lpw == 8 ? k_velocity_fluid<8, false> : lpw == 16 ? k_velocity_fluid<16, false> : k_velocity_fluid<32, false>;
}

size_t smem_velocity(const ModelDev& m, const DataDev& d, const FluidDev& f) {
  const int words = vel_layout(m).total;
  return f.has_fluid ? team_shape(m, d.wn, words, vel_kernel_fluid).block_bytes : team_shape(m, d.wn, words, vel_kernel).block_bytes;
}
cudaError_t launch_velocity(const ModelDev& m, const DataDev& d, int mask, cudaStream_t s, const FluidDev& f) {
  const int words = vel_layout(m).total;
  return f.has_fluid ? team_launch(m, d, words, vel_kernel_fluid, mask, s, f) : team_launch(m, d, words, vel_kernel, mask, s);
}
cudaError_t resident_worlds_velocity(const ModelDev& m, const DataDev& d, int* worlds, int* shape, const FluidDev& f) {
  const int words = vel_layout(m).total;
  shape[3] = f.has_fluid ? 2 : vel_pext(m) ? 1 : 0;
  return f.has_fluid ? team_resident_worlds(m, d, words, vel_kernel_fluid, worlds, shape) : team_resident_worlds(m, d, words, vel_kernel, worlds, shape);
}
