// k_implicit.cu -- the fully implicit-in-velocity integrator's linear solve: qacc = (M - dt (qDeriv_smooth + d RNE / d qvel))^-1 Ma.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): forward.py:578-600 implicit (IntegratorType.IMPLICIT branch), :560-575 _map_m2d,
// derivative.py:1117-1213 deriv_smooth_vel (actuator / damper / tendon-damper velocity derivatives in the sparsity of M),
// derivative.py:321-584 deriv_rne_vel (deriv_rne_cvel_cdof_dot, deriv_rne_cacc_cfrcbody_forward, deriv_rne_cfrcbody_backward,
// deriv_rne_body2jnt_sparse: four (nworld, nbody | nv, nv) scratch arrays of spatial vectors in global memory and 3 nlevel + 1 launches) and
// smooth.py:3376-3497 factor_solve_lu (sparse LU without fill-in, one THREAD per world).
//
// Here one warp owns one world.  The matrix lives in shared memory as dense per-tree blocks (the D-structure -- a dof, its ancestors and its
// descendants -- is exactly what a tree's block holds besides structural zeros).  The RNE derivative is taken one column (dof k) per lane: a
// lane walks the bodies once, forward (d cvel, d cacc, d body force) with its 18 floats per body in shared memory interleaved over lanes, and
// once backward; every lane runs the same joint-type branches, only the "is k one of this joint's dofs" predicates differ.  The LU runs from
// the last dof to the first like the reference's (U unit upper, L lower): entries outside the D-structure never fill in, because two dofs
// that are both ancestors of a third lie on one chain -- so the dense elimination reproduces the sparse one.  Results: Data.qLU (the factors,
// D-structure) and the solved acceleration for the advance kernel (k_integrate.cu).
#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

namespace {

struct ImpLayout { int A, x, scr, total; };
__host__ __device__ inline ImpLayout imp_layout(const ModelDev& m) {
  ImpLayout L;
  int o = 0;
  auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
  L.A = take(m.qld_total);          // per-tree n x n blocks at tree_qLDadr
  L.x = take(m.nv);
  L.scr = take(18 * m.nbody * 32);  // d cvel | d cacc | d cfrc_body: (3, nbody, 6) per lane, lane-interleaved
  L.total = o;
  return L;
}

// block address of (i, j), both dofs of the tree that starts at dof `start` with n dofs
__device__ __forceinline__ int blk(int adr, int start, int n, int i, int j) { return adr + (i - start) * n + (j - start); }

template <bool BAT>
__global__ void __launch_bounds__(32)
k_implicit(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, float* __restrict__ qacc_out) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x;
  const int w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const ImpLayout L = imp_layout(mp);
  float *A = smem + L.A, *x = smem + L.x, *scr = smem + L.scr;
  const int nv = m.nv, nb = m.nbody;
  const size_t wb = (size_t)w;
  const float dt = m.timestep;
  const bool damper = !(m.disableflags & DSBL_DAMPER);

  // ---- M - dt qDeriv_smooth, mirrored into both triangles of the tree blocks (derivative.py:1117-1213, forward.py:560-575)
#pragma unroll 1
  for (int i = lane; i < m.qld_total; i += 32) A[i] = 0.f;
  __syncwarp();
  const float* Mw = d.M + wb * m.nC;
#pragma unroll 1
  for (int t = 0; t < m.ntree; t++) {
    const int start = m.tree_dofadr[t], n = m.tree_dofnum[t], adr = m.tree_qLDadr[t];
    const int e0 = m.M_rowadr[start], e1 = m.M_rowadr[start + n - 1] + m.M_rownnz[start + n - 1];
#pragma unroll 1
    for (int e = e0 + lane; e < e1; e += 32) {
      const int r = m.M_entry_row[e], col = m.M_colind[e];
      const float v = Mw[e] + ((col == r && damper) ? dt * m.dof_damping[r] : 0.f);
      A[blk(adr, start, n, r, col)] = v;
      A[blk(adr, start, n, col, r)] = v;
    }
  }
  __syncwarp();
  if (m.nu > 0 && !(m.disableflags & DSBL_ACTUATION)) {
#pragma unroll 1
    for (int a = 0; a < m.nu; a++) {  // actuators one after the other: fixed accumulation order, no atomics
      const int madr = m.moment_rowadr0[a], nnz = m.moment_rownnz0[a];
      if (nnz == 0) continue;
      const float gain = m.actuator_gaintype[a] == GAIN_AFFINE ? m.actuator_gainprm[10 * a + 2] : 0.f;
      const float bias = m.actuator_biastype[a] == BIAS_AFFINE ? m.actuator_biasprm[10 * a + 2] : 0.f;
      if (bias == 0.f && gain == 0.f) continue;
      if (m.actuator_forcelimited[a]) {
        const float f = d.actuator_force[wb * m.nu + a];
        if (f <= m.actuator_forcerange[2 * a] || f >= m.actuator_forcerange[2 * a + 1]) continue;
      }
      float vel = bias;
      if (gain != 0.f) {  // derivative.py:142-164: the gain multiplies the activation of a stateful actuator
        if (m.na > 0 && m.actuator_dyntype[a] != DYN_NONE) {
          const int last = m.actuator_actadr[a] + m.actuator_actnum[a] - 1;
          const float act = d.act[wb * m.na + last];
          vel += gain * (m.actuator_actearly[a] ? next_act(m, a, act, d.act_dot[wb * m.na + last], 1.0f, m.actuator_actlimited[a] != 0) : act);
        } else vel += gain * d.ctrl[wb * m.nu + a];
      }
      for (int p = lane; p < nnz * nnz; p += 32) {
        const int i = p / nnz, j = p - i * nnz;
        const int di = m.moment_colind0[madr + i], dj = m.moment_colind0[madr + j];
        // entries of the M sparsity pattern only (derivative.py:178-218): dj is di or an ancestor dof of it; mirrored like _map_m2d does
        if (j <= i && m.body_isdofancestor[m.dof_bodyid[di] * nv + dj]) {
          int t = 0;
          while (t + 1 < m.ntree && m.tree_dofadr[t + 1] <= di) t++;
          const int start = m.tree_dofadr[t], n = m.tree_dofnum[t], adr = m.tree_qLDadr[t];
          const float mi = d.actuator_moment[wb * m.nJmom + madr + i], mj = d.actuator_moment[wb * m.nJmom + madr + j];
          const float v = dt * mi * mj * vel;
          A[blk(adr, start, n, di, dj)] -= v;
          if (di != dj) A[blk(adr, start, n, dj, di)] -= v;
        }
      }
      __syncwarp();
    }
  }
  if (m.ntendon > 0 && damper) {  // derivative.py:262-318: tendon damping on the entries of the M sparsity pattern
#pragma unroll 1
    for (int tn = 0; tn < m.ntendon; tn++) {
      const float kd = m.tendon_damping[tn];
      const int tadr = m.ten_J_rowadr[tn], nnz = m.ten_J_rownnz[tn];
      if (kd == 0.f) continue;
      for (int p = lane; p < nnz * nnz; p += 32) {
        const int i = p / nnz, j = p - i * nnz, di = m.ten_J_colind[tadr + i], dj = m.ten_J_colind[tadr + j];
        if (dj <= di && m.body_isdofancestor[m.dof_bodyid[di] * nv + dj]) {
          int t = 0;
          while (t + 1 < m.ntree && m.tree_dofadr[t + 1] <= di) t++;
          const int start = m.tree_dofadr[t], n = m.tree_dofnum[t], adr = m.tree_qLDadr[t];
          const float v = dt * m.ten_J0[tadr + i] * m.ten_J0[tadr + j] * kd;
          A[blk(adr, start, n, di, dj)] += v;
          if (di != dj) A[blk(adr, start, n, dj, di)] += v;
        }
      }
      __syncwarp();
    }
  }

  // ---- minus dt d(qfrc_bias) / d(qvel): lane = column (dof k), 32 columns per pass (derivative.py:321-584)
  const float* cdof = d.cdof + wb * 6 * nv;
  const float* cdd = d.cdof_dot + wb * 6 * nv;
  const float* cvel = d.cvel + wb * 6 * nb;
  const float* cinert = d.cinert + wb * 10 * nb;
  const float* qvel = d.qvel + wb * nv;
  float* Dcvel = scr + lane;                  // element (b, c) at ((b * 6 + c) * 32)
  float* Dcacc = scr + 6 * nb * 32 + lane;
  float* Dcfrc = scr + 12 * nb * 32 + lane;
#define SV(p, b, c) (p)[((b) * 6 + (c)) * 32]
#pragma unroll 1
  for (int k0 = 0; k0 < nv; k0 += 32) {
    const int k = k0 + lane;  // lanes beyond nv carry k = an index no dof has: their derivatives stay zero and nothing is stored
    for (int c = 0; c < 6; c++) { SV(Dcvel, 0, c) = 0.f; SV(Dcacc, 0, c) = 0.f; SV(Dcfrc, 0, c) = 0.f; }
#pragma unroll 1
    for (int b = 1; b < nb; b++) {
      const int pid = m.body_parentid[b];
      float cv[6], ca[6];
      for (int c = 0; c < 6; c++) { cv[c] = SV(Dcvel, pid, c); ca[c] = SV(Dcacc, pid, c); }
      int dof = m.body_dofadr[b];
#pragma unroll 1
      for (int j = m.body_jntadr[b]; j < m.body_jntadr[b] + m.body_jntnum[b]; j++) {
        const int jt = m.jnt_type[j];
        if (jt == JNT_FREE) {
          // rotational dofs first: they enter d cvel before the translational dofs' cdof_dot is differentiated; their own cdof_dot is zero
          if (k >= dof && k < dof + 3) for (int c = 0; c < 6; c++) { cv[c] += cdof[6 * k + c]; ca[c] += cdd[6 * k + c]; }
          for (int a = 3; a < 6; a++) {
            float t6[6];
            motion_cross(cv, cdof + 6 * (dof + a), t6);
            if (k == dof + a) for (int c = 0; c < 6; c++) ca[c] += cdd[6 * k + c];
            const float qv = qvel[dof + a];
            for (int c = 0; c < 6; c++) ca[c] += t6[c] * qv;
          }
          if (k >= dof + 3 && k < dof + 6) for (int c = 0; c < 6; c++) cv[c] += cdof[6 * k + c];
          dof += 6;
        } else {
          const int nd = jt == JNT_BALL ? 3 : 1;
          for (int a = 0; a < nd; a++) {
            float t6[6];
            motion_cross(cv, cdof + 6 * (dof + a), t6);
            if (k == dof + a) for (int c = 0; c < 6; c++) ca[c] += cdd[6 * k + c];
            const float qv = qvel[dof + a];
            for (int c = 0; c < 6; c++) ca[c] += t6[c] * qv;
          }
          if (k >= dof && k < dof + nd) for (int c = 0; c < 6; c++) cv[c] += cdof[6 * k + c];
          dof += nd;
        }
      }
      // d(cfrc_body) = I d cacc + d cvel x* (I cvel) + cvel x* (I d cvel)   (derivative.py:443-459)
      float t1[6], icv[6], idcv[6], x1[6], x2[6];
      inert_vec(cinert + 10 * b, ca, t1);
      inert_vec(cinert + 10 * b, cvel + 6 * b, icv);
      inert_vec(cinert + 10 * b, cv, idcv);
      motion_cross_force(cv, icv, x1);
      motion_cross_force(cvel + 6 * b, idcv, x2);
      for (int c = 0; c < 6; c++) { SV(Dcvel, b, c) = cv[c]; SV(Dcacc, b, c) = ca[c]; SV(Dcfrc, b, c) = t1[c] + x1[c] + x2[c]; }
    }
#pragma unroll 1
    for (int b = nb - 1; b > 0; b--) {  // children into parents (bodies are numbered parents first)
      const int pid = m.body_parentid[b];
      if (pid > 0) for (int c = 0; c < 6; c++) SV(Dcfrc, pid, c) += SV(Dcfrc, b, c);
    }
    if (k < nv) {  // rows coupled to dof k: its D-structure row (= the symmetric gather row of mul_m)
      int t = 0;
      while (t + 1 < m.ntree && m.tree_dofadr[t + 1] <= k) t++;
      const int start = m.tree_dofadr[t], n = m.tree_dofnum[t], adr = m.tree_qLDadr[t];
#pragma unroll 1
      for (int e = m.mulm_rowadr[k]; e < m.mulm_rowadr[k + 1]; e++) {
        const int i = m.mulm_col[e], bi = m.dof_bodyid[i];
        float s = 0.f;
        for (int c = 0; c < 6; c++) s += cdof[6 * i + c] * SV(Dcfrc, bi, c);
        A[blk(adr, start, n, i, k)] -= dt * s;
      }
    }
    __syncwarp();
  }
#undef SV

  // ---- LU from the last dof to the first, then (U + I) y = Ma, L x = y (smooth.py:3376-3478); lanes = rows
#pragma unroll 1
  for (int t = 0; t < m.ntree; t++) {
    const int start = m.tree_dofadr[t], n = m.tree_dofnum[t];
    float* At = A + m.tree_qLDadr[t];
#pragma unroll 1
    for (int i = n - 1; i > 0; i--) {
      const float piv = At[i * n + i];
#pragma unroll 1
      for (int j = lane; j < i; j += 32) {
        const float aji = At[j * n + i];
        if (aji != 0.f) {
          const float lji = aji / piv;
          At[j * n + i] = lji;
#pragma unroll 4
          for (int c = 0; c < i; c++) At[j * n + c] -= At[i * n + c] * lji;
        }
      }
      __syncwarp();
    }
#pragma unroll 1
    for (int i = lane; i < n; i += 32) x[i] = d.efc_Ma[wb * nv + start + i];
    __syncwarp();
#pragma unroll 1
    for (int i = n - 1; i > 0; i--) {  // unit upper triangle, columns from the right
      const float xi = x[i];
      __syncwarp();
      for (int r = lane; r < i; r += 32) x[r] -= At[r * n + i] * xi;
      __syncwarp();
    }
#pragma unroll 1
    for (int i = 0; i < n; i++) {  // lower triangle with its diagonal, columns from the left
      const float xi = x[i] / At[i * n + i];
      __syncwarp();
      if (lane == 0) x[i] = xi;
      for (int r = i + 1 + lane; r < n; r += 32) x[r] -= At[r * n + i] * xi;
      __syncwarp();
    }
#pragma unroll 1
    for (int i = lane; i < n; i += 32) qacc_out[wb * nv + start + i] = x[i];
    // Data.qLU: the factors in the D-structure (types.py:2163)
    const int e0 = m.mulm_rowadr[start], e1 = m.mulm_rowadr[start + n];
#pragma unroll 1
    for (int e = e0 + lane; e < e1; e += 32) {
      int r = start;  // row of entry e
      while (m.mulm_rowadr[r + 1] <= e) r++;
      d.qLU[wb * (size_t)m.mulm_rowadr[nv] + e] = At[(r - start) * n + (m.mulm_col[e] - start)];
    }
    __syncwarp();
  }
}

}  // namespace

size_t smem_implicit(const ModelDev& m) { return (size_t)imp_layout(m).total * sizeof(float); }

cudaError_t launch_implicit_solve(const ModelDev& m, const DataDev& d, float* qacc_out, cudaStream_t s) {
  return launch(m.batched ? k_implicit<true> : k_implicit<false>, d.wn, 32, smem_implicit(m), s, m, d, qacc_out);
}
