// mjb_implicit_a.cuh -- one kinematic tree's block of the velocity-implicit matrix A = M + dt diag(damping) (Euler with eulerdamp) or
// A = M - dt qDeriv (implicitfast), shared by the integrator (k_integrate.cu k_euler: qacc = A^-1 M qacc) and inverse dynamics
// (k_inverse.cu: the discrete-to-continuous conversion qacc = M^-1 A qacc).
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): forward.py:391-415 (M + dt diag(damping)), derivative.py:38-176
// _qderiv_actuator_passive_vel, :178-245 moment^T vel moment scatter, :221-245 dof damping, :262-318 tendon damping, and with FLUID
// :935-1117 the fluid force derivatives (_qderiv_ellipsoid_fluid, _qderiv_box_fluid).
#pragma once
#include "mjb_fluid.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

// Writes the lower triangle of the block of tree dofs [start, start + n) of world wb (Mw: its M values) into A (row-major, leading
// dimension ld; the upper triangle is zeroed); f: the model's fluid fields, read with FLUID only.  damper: add dt * dof_damping on the diagonal; implicitfast: subtract dt times the actuator and add dt times the tendon damping
// derivatives on the entries of the M sparsity pattern, and with FLUID (a model with fluid forces) the fluid force derivatives.  The warp's
// lanes share the work; ends with the warp converged.  SYM: the fluid B of an ellipsoid is symmetrized, as implicitfast does
// (derivative.py:800); deriv_smooth_vel for the other integrators leaves it as it stands (the inertia-box B is diagonal either way).
template <bool FLUID = false, bool SYM = true>
__device__ __forceinline__ void tree_implicit_a(const ModelDev& m, const DataDev& d, size_t wb, const float* Mw, int start, int n, int ld, float dt,
                                                bool implicitfast, bool damper, float* A, int lane, const FluidDev& f) {
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
      const int adr = m.moment_rowadr0[a], nnz = m.moment_rownnz0[a];
      // moment_colind0 rows are ascending: skip an actuator with no dof in [start, start + n); one that spans trees stays
      if (nnz == 0 || m.moment_colind0[adr + nnz - 1] < start || m.moment_colind0[adr] >= start + n) continue;
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
        // entries of this tree's block of the M sparsity pattern only (derivative.py:178-218: M_elemid < 0 is skipped): di in the
        // block, dj di or an ancestor dof of it -- a tendon transmission may couple dofs of sibling bodies or of other trees, which
        // M does not
        if (j <= i && di >= start && di < start + n && m.body_isdofancestor[m.dof_bodyid[di] * nv + dj]) {
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
  if (FLUID && implicitfast && f.has_fluid && (f.density > 0.f || f.viscosity > 0.f)) {
    // derivative.py:935-1117: A -= dt J_i^T B J_j for every fluid body b of this tree and every entry (i, j) of M with i a dof of b's
    // chain.  Bodies one after the other, each entry owned by one lane: fixed accumulation order, no atomics.
    const int nb = m.nbody, ng = m.ngeom;
    const float *cvel = d.cvel + wb * 6 * nb, *xipos = d.xipos + wb * nb * 3, *ximat = d.ximat + wb * nb * 9, *stc = d.subtree_com + wb * nb * 3;
    const float *cdof = d.cdof + wb * nv * 6, *gxpos = d.geom_xpos + wb * ng * 3, *gxmat = d.geom_xmat + wb * ng * 9;
    const v3 wind = mk3(f.wind_x, f.wind_y, f.wind_z);
    const bool has_wind = f.wind_x != 0.f || f.wind_y != 0.f || f.wind_z != 0.f;
#pragma unroll 1
    for (int b = 1; b < nb; b++) {
      const int kind = f.body_fluid[b];
      if (kind == FLUID_NONE || !m.body_isdofancestor[b * nv + start]) continue;  // the tree's first dof is an ancestor of all its bodies
      const v3 xip = ld3(xipos + 3 * b), root = ld3(stc + 3 * m.body_rootid[b]);
      v3 ang, lin;
      fluid_body_vel(cvel + 6 * b, xip, root, &ang, &lin);
      if (kind == FLUID_BOX) {
        const float* R = ximat + 9 * b;
        const v3 la = fl_mtv(R, ang), ll = fl_mtv(R, lin) - fl_mtv(R, wind);
        const float lvel[6] = {la.x, la.y, la.z, ll.x, ll.y, ll.z};
        float Bd[6];
        fluid_box_B(m, f, b, lvel, Bd);
#pragma unroll 1
        for (int e = e0 + lane; e < e1; e += 32) {
          const int r = m.M_entry_row[e], col = m.M_colind[e];
          if (!m.body_isdofancestor[b * nv + r]) continue;
          float Ji[6], Jj[6];
          fluid_jac_local(cdof + 6 * r, xip - root, R, Ji);
          fluid_jac_local(cdof + 6 * col, xip - root, R, Jj);
          float c = 0.f;
#pragma unroll
          for (int k = 0; k < 6; k++) c += Ji[k] * (Bd[k] * Jj[k]);
          A[(r - start) * ld + (col - start)] -= dt * c;
        }
      } else {
#pragma unroll 1
        for (int g = f.body_geomadr[b]; g < f.body_geomadr[b] + f.body_geomnum[b]; g++) {
          const float* fl = f.geom_fluid + 12 * g;
          if (fl[0] <= 0.f) continue;
          const float* R = gxmat + 9 * g;
          const v3 gpos = ld3(gxpos + 3 * g);
          const v3 l_ang = fl_mtv(R, ang);
          v3 l_lin = fl_mtv(R, lin + cross(ang, gpos - xip));
          if (has_wind) l_lin = l_lin - fl_mtv(R, wind);
          float B[36];
          fluid_ellipsoid_B<SYM>(fl, fluid_semiaxes(m.geom_type[g], m.geom_size + 3 * g), l_ang, l_lin, f.density, f.viscosity, B);
#pragma unroll 1
          for (int e = e0 + lane; e < e1; e += 32) {
            const int r = m.M_entry_row[e], col = m.M_colind[e];
            if (!m.body_isdofancestor[b * nv + r]) continue;
            float Ji[6], Jj[6];
            fluid_jac_local(cdof + 6 * r, gpos - root, R, Ji);
            fluid_jac_local(cdof + 6 * col, gpos - root, R, Jj);
            float c = 0.f;
#pragma unroll
            for (int k = 0; k < 6; k++) {
              float bj = 0.f;
#pragma unroll
              for (int q = 0; q < 6; q++) bj += B[6 * k + q] * Jj[q];
              c += Ji[k] * bj;
            }
            A[(r - start) * ld + (col - start)] -= dt * c;
          }
        }
      }
    }
    __syncwarp();
  }
}
