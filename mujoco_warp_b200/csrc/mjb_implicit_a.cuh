// mjb_implicit_a.cuh -- one kinematic tree's block of the velocity-implicit matrix A = M + dt diag(damping) (Euler with eulerdamp) or
// A = M - dt qDeriv (implicitfast), shared by the integrator (k_integrate.cu k_euler: qacc = A^-1 M qacc) and inverse dynamics
// (k_inverse.cu: the discrete-to-continuous conversion qacc = M^-1 A qacc).
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): forward.py:391-415 (M + dt diag(damping)), derivative.py:38-176
// _qderiv_actuator_passive_vel, :178-245 moment^T vel moment scatter, :221-245 dof damping, :262-318 tendon damping.
#pragma once
#include "mjb_math.cuh"
#include "mjb_types.cuh"

// Writes the lower triangle of the block of tree dofs [start, start + n) of world wb (Mw: its M values) into A (row-major, leading
// dimension ld; the upper triangle is zeroed).  damper: add dt * dof_damping on the diagonal; implicitfast: subtract dt times the actuator and add dt times the tendon damping
// derivatives on the entries of the M sparsity pattern.  The warp's lanes share the work; ends with the warp converged.
__device__ __forceinline__ void tree_implicit_a(const ModelDev& m, const DataDev& d, size_t wb, const float* Mw, int start, int n, int ld, float dt,
                                                bool implicitfast, bool damper, float* A, int lane) {
  const int nv = m.nv;
#pragma unroll 1
  for (int i = lane; i < n * ld; i += 32) A[i] = 0.f;
  __syncwarp();
  const int e0 = m.M_rowadr[start], e1 = m.M_rowadr[start + n - 1] + m.M_rownnz[start + n - 1];
#pragma unroll 1
  for (int e = e0 + lane; e < e1; e += 32) {
    const int r = m.M_entry_row[e], col = m.M_colind[e];
    A[(r - start) * ld + (col - start)] = Mw[e] + ((col == r && damper) ? dt * m.dof_damping[r] : 0.f);
  }
  __syncwarp();
  if (implicitfast && m.nu > 0 && !(m.disableflags & DSBL_ACTUATION)) {
#pragma unroll 1
    for (int a = 0; a < m.nu; a++) {  // actuators one after the other: fixed accumulation order, no atomics
      const int adr = m.moment_rowadr0[a], nnz = m.moment_rownnz0[a], d0 = m.moment_colind0[adr];
      if (d0 < start || d0 >= start + n) continue;
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
        const int di = m.moment_colind0[adr + i], dj = m.moment_colind0[adr + j];
        // entries of the M sparsity pattern only (derivative.py:178-218: M_elemid < 0 is skipped): dj is di or an ancestor dof
        // of it -- a tendon transmission may couple dofs of sibling bodies, which M does not
        if (j <= i && m.body_isdofancestor[m.dof_bodyid[di] * nv + dj]) {
          const float mi = d.actuator_moment[wb * m.nJmom + adr + i], mj = d.actuator_moment[wb * m.nJmom + adr + j];
          A[(di - start) * ld + (dj - start)] -= dt * mi * mj * vel;
        }
      }
      __syncwarp();
    }
  }
  if (implicitfast && m.ntendon > 0 && damper) {  // derivative.py:262-318: tendon damping on the entries of the M sparsity pattern
#pragma unroll 1
    for (int t = 0; t < m.ntendon; t++) {
      const float kd = m.tendon_damping[t];
      const int adr = m.ten_J_rowadr[t], nnz = m.ten_J_rownnz[t];
      if (kd == 0.f) continue;
      for (int p = lane; p < nnz * nnz; p += 32) {
        const int i = p / nnz, j = p - i * nnz, di = m.ten_J_colind[adr + i], dj = m.ten_J_colind[adr + j];
        if (di >= start && di < start + n && dj <= di && m.body_isdofancestor[m.dof_bodyid[di] * nv + dj])  // dj: di itself or an ancestor dof, i.e. an entry of M
          A[(di - start) * ld + (dj - start)] += dt * m.ten_J0[adr + i] * m.ten_J0[adr + j] * kd;
      }
      __syncwarp();
    }
  }
}
