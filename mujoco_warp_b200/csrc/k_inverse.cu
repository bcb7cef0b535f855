// k_inverse.cu -- inverse dynamics after the position and velocity stages: the constraint forces at a GIVEN qacc and
// qfrc_inverse = qfrc_bias + M qacc - qfrc_passive - qfrc_constraint.  One warp per world.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): inverse.py:148 inverse after fwd_position / fwd_velocity: :79-119
// discrete_acc (ENBL_INVDISCRETE: Euler's M + dt diag(damping), implicitfast's M - dt qDeriv, then the M solve), :129 inv_constraint
// (solver.py:3622 init_context with grad=False: Jaref = J qacc - aref, efc_Ma = M qacc, solver.py:1699 _update_constraint_efc, the
// qfrc_constraint = J^T efc_force kernels, solver_niter = 0), support.py:153 mul_m and :59 _qfrc_inverse.
//
// The Jacobian is read twice -- J qacc with lanes over rows, J^T force with lanes over dofs -- and both passes read it through L2 (it
// was written by k_constraint just before): one pass each way over a world's rows is less than a bulk copy into shared memory would
// cost in resident worlds, and the row pass issues one independent float4 load per lane and row chunk.
#include "mjb_implicit_a.cuh"
#include "mjb_launch.cuh"
#include "mjb_linesearch.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

namespace {

__host__ __device__ inline int inv_ld(int n) { return n | 1; }
// Shared-memory slice of one world: qacc (zero-padded to nv_pad), the M^-1 A qacc scratch, Jaref and force per row, the elliptic row map,
// and the per-tree matrix A of the discrete conversion.
struct InvLayout { int qa, y, Jaref, force, rinfo, rfri, A, total; };
__host__ __device__ inline InvLayout inv_layout(const ModelDev& m, const DataDev& d, bool disc) {
  InvLayout L;
  int o = 0;
  auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
  const bool ell = m.cone == CONE_ELLIPTIC;
  L.qa = take(d.nv_pad);
  L.y = take(disc ? m.nv : 0);
  L.Jaref = take(d.njmax);
  L.force = take(d.njmax);
  L.rinfo = take(ell ? d.njmax : 0);
  L.rfri = take(ell ? d.njmax : 0);
  L.A = take(disc ? m.maxtree * inv_ld(m.maxtree) : 0);
  L.total = o;
  return L;
}

// dot of a 16B-aligned J row (global) with the zero-padded qacc in shared memory
__device__ __forceinline__ float row_dot_g(const float* __restrict__ Jr, const float* qa, int nvp) {
  float s = 0.f;
#pragma unroll 4
  for (int k = 0; k < nvp; k += 4) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(Jr + k)), b = *reinterpret_cast<const float4*>(qa + k);
    s += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
  }
  return s;
}

// disc: convert the given (discrete-time) qacc to continuous time first, qacc <- M^-1 A qacc, and write it to qacc_cont.
// qfrc_inverse and qacc_cont are arguments, not DataDev fields: a larger DataDev would move every field of every other kernel.
// FLUID: the implicitfast conversion includes the fluid force derivatives (k_inverse_fluid)
template <bool FLUID, bool ELL, bool BIG, bool BAT>
__device__ __forceinline__ void inverse(const ModelDev& mp, const DataDev& d, float* __restrict__ qfrc_inverse, float* __restrict__ qacc_cont, int disc, const FluidDev& f) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x;  // one warp (one block) owns the world
  const int w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const InvLayout L = inv_layout(mp, d, disc);
  const int nv = m.nv, nvp = d.nv_pad, njmax = d.njmax;
  const size_t wb = (size_t)w;
  float *qa = smem + L.qa, *Jaref = smem + L.Jaref, *force = smem + L.force;

#pragma unroll 1
  for (int i = lane; i < nvp; i += 32) qa[i] = i < nv ? d.qacc[wb * nv + i] : 0.f;
  __syncwarp();

  if (disc) {
    // inverse.py:79-119: qfrc = A qacc with A = M + dt diag(damping) (Euler: only eulerdamp=disable skips it, the damper flag is not
    // read) or M - dt qDeriv (implicitfast), then qacc = M^-1 qfrc through the per-tree factor U (M = U^T U) in Data.qLD
    const bool implicitfast = m.integrator == INT_IMPLICITFAST;
    const bool damper = !implicitfast || !(m.disableflags & DSBL_DAMPER);
    float *y = smem + L.y, *A = smem + L.A;
    const float* Mw = d.M + wb * m.nC;
#pragma unroll 1
    for (int t = 0; t < m.ntree; t++) {
      const int start = m.tree_dofadr[t], n = m.tree_dofnum[t], ld = inv_ld(n);
      tree_implicit_a<FLUID>(m, d, wb, Mw, start, n, ld, m.timestep, implicitfast, damper, A, lane, f);
      __syncwarp();
#pragma unroll 1
      for (int i = lane; i < n; i += 32) {  // A holds the lower triangle
        float s = 0.f;
        for (int j = 0; j <= i; j++) s += A[i * ld + j] * qa[start + j];
        for (int j = i + 1; j < n; j++) s += A[j * ld + i] * qa[start + j];
        y[start + i] = s;
      }
      __syncwarp();
      const float* U = d.qLD + wb * m.qld_total + m.tree_qLDadr[t];
      float* xt = y + start;
#pragma unroll 1
      for (int j = 0; j < n; j++) {  // U^T z = y
        const float zj = xt[j] / U[j * n + j];
        __syncwarp();
        for (int i = j + 1 + lane; i < n; i += 32) xt[i] -= U[j * n + i] * zj;
        if (lane == 0) xt[j] = zj;
        __syncwarp();
      }
#pragma unroll 1
      for (int j = n - 1; j >= 0; j--) {  // U x = z
        const float xj = xt[j] / U[j * n + j];
        __syncwarp();
        for (int i = lane; i < j; i += 32) xt[i] -= U[i * n + j] * xj;
        if (lane == 0) xt[j] = xj;
        __syncwarp();
      }
    }
#pragma unroll 1
    for (int i = lane; i < nv; i += 32) { qa[i] = y[i]; qacc_cont[wb * nv + i] = y[i]; }
    __syncwarp();
  }

  // solver.py:3622 init_context (grad=False): Jaref = J qacc - aref, the row rule, qfrc_constraint = J^T force
  const int nefc = njmax > 0 ? min(d.nefc[w], njmax) : 0;
  const int ne = d.ne[w], nf = d.nf[w];
  const float* Jg = d.efc_J + wb * (size_t)d.njmax_pad * nvp;
  int* rinfo = (int*)(smem + L.rinfo);
  float* rfri = smem + L.rfri;
#pragma unroll 1
  for (int r = lane; r < nefc; r += 32) {
    Jaref[r] = row_dot_g(Jg + (size_t)r * nvp, qa, nvp) - d.efc_aref[wb * njmax + r];
    if (ELL) {  // row -> (contact, component) map, as k_solver builds it; a contact's rows are consecutive (k_constraint.cu)
      int info = -1; float fr = 0.f;
      if (d.efc_type[wb * njmax + r] == CNSTR_CONTACT_ELLIPTIC) {
        const int cid = d.efc_id[wb * njmax + r], e0 = d.contact_efc_address[(size_t)cid * m.nmaxpyramid], dim = d.contact_dim[cid], j = r - e0;
        info = (e0 < 0 || e0 + dim > nefc) ? -2 : ((dim << 4) | j);
        fr = j == 0 ? d.contact_friction[5 * (size_t)cid] * m.impratio_invsqrt : d.contact_friction[5 * (size_t)cid + j - 1];
      }
      rinfo[r] = info; rfri[r] = fr;
    }
  }
  __syncwarp();
  const float* D = d.efc_D + wb * d.njmax_pad;
  const float* floss = d.efc_frictionloss + wb * njmax;
#pragma unroll 1
  for (int r = lane; r < nefc; r += 32) {
    float f; int st; bool cone0 = false;
    row_force_state<ELL>(r, ne, nf, Jaref[r], D[r], floss, rinfo, rfri, Jaref, D, f, st, cone0);
    force[r] = f;
    d.efc_force[wb * njmax + r] = f;
    d.efc_state[wb * d.njmax_pad + r] = st;
  }
  __syncwarp();

  // efc_Ma = M qacc (support.py:153, gather tables), qfrc_constraint = J^T force, qfrc_inverse (inverse.py:59)
  const float* Mw = d.M + wb * m.nC;
#pragma unroll 1
  for (int i = lane; i < nv; i += 32) {
    float ma = 0.f;
    for (int k = m.mulm_rowadr[i]; k < m.mulm_rowadr[i + 1]; k++) ma += Mw[m.mulm_madr[k]] * qa[m.mulm_col[k]];
    float qfc = 0.f;
#pragma unroll 4
    for (int r = 0; r < nefc; r++) qfc += Jg[(size_t)r * nvp + i] * force[r];
    const size_t k = wb * nv + i;
    d.efc_Ma[k] = ma;
    d.qfrc_constraint[k] = qfc;
    qfrc_inverse[k] = d.qfrc_bias[k] + ma - d.qfrc_passive[k] - qfc;
    if (!BIG) break;  // nv <= 32: one dof per lane
  }
  if (lane == 0) d.solver_niter[w] = 0;
}

template <bool ELL, bool BIG, bool BAT>
__global__ void __launch_bounds__(32)
k_inverse(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, float* __restrict__ qfrc_inverse, float* __restrict__ qacc_cont, int disc) {
  inverse<false, ELL, BIG, BAT>(mp, d, qfrc_inverse, qacc_cont, disc, FluidDev{});
}
template <bool ELL, bool BIG, bool BAT>
__global__ void __launch_bounds__(32)
k_inverse_fluid(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, float* __restrict__ qfrc_inverse, float* __restrict__ qacc_cont, int disc,
                const __grid_constant__ FluidDev f) {
  inverse<true, ELL, BIG, BAT>(mp, d, qfrc_inverse, qacc_cont, disc, f);
}

}  // namespace

// Instantiated by what the model can produce: elliptic cones, nv > 32 (more than one dof per lane), per-world (batched) fields, fluid forces.
cudaError_t launch_inverse(const ModelDev& m, const DataDev& d, float* qfrc_inverse, float* qacc_cont, bool disc, cudaStream_t s, const FluidDev& f) {
  const int which = 4 * (m.batched ? 1 : 0) + 2 * (m.nv > 32 ? 1 : 0) + (m.cone == CONE_ELLIPTIC ? 1 : 0);
  static void (*const kerns[8])(ModelDev, DataDev, float*, float*, int) = {
    k_inverse<false, false, false>, k_inverse<true, false, false>, k_inverse<false, true, false>, k_inverse<true, true, false>,
    k_inverse<false, false, true>,  k_inverse<true, false, true>,  k_inverse<false, true, true>,  k_inverse<true, true, true>};
  static void (*const kerns_fluid[8])(ModelDev, DataDev, float*, float*, int, FluidDev) = {
    k_inverse_fluid<false, false, false>, k_inverse_fluid<true, false, false>, k_inverse_fluid<false, true, false>, k_inverse_fluid<true, true, false>,
    k_inverse_fluid<false, false, true>,  k_inverse_fluid<true, false, true>,  k_inverse_fluid<false, true, true>,  k_inverse_fluid<true, true, true>};
  const size_t smem = (size_t)inv_layout(m, d, disc).total * sizeof(float);
  if (f.has_fluid) return launch(kerns_fluid[which], d.wn, 32, smem, s, m, d, qfrc_inverse, qacc_cont, (int)disc, f);
  return launch(kerns[which], d.wn, 32, smem, s, m, d, qfrc_inverse, qacc_cont, (int)disc);
}
