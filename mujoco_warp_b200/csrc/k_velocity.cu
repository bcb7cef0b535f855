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

#include "mjb_math.cuh"
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

// PEXT = the model uses gravity compensation or free / ball joint springs (kept out of the plain instantiation)
template <bool PEXT, int LPW, bool BAT>
__global__ void __launch_bounds__(256)
k_velocity(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int mask) {
  extern __shared__ __align__(16) float smem[];
  constexpr int G = 32 / LPW;
  Team<LPW> T;
  T.init(d.w0, d.wn, d.nworld);
  if (T.nvalid <= 0) return;
  MJB_WORLD_MODEL(T.w)
  const int lane = T.lane, sub = T.sub, g = T.g, nval = T.nvalid;
  const bool valid = T.valid;
  const VelLayout L = vel_layout(mp);
  float* S = smem + (size_t)(threadIdx.x >> 5) * ((size_t)L.total * G + 4);  // this warp's slice (+ its mbarrier)
  Stager st;
  st.init(reinterpret_cast<uint64_t*>(S + (size_t)L.total * G), lane);
  const int nv = m.nv, nb = m.nbody, nu = m.nu;
#define FLD(f, n) (S + (size_t)L.f * G + (size_t)g * (n))
  float *qvel = FLD(qvel, nv), *cdof = FLD(cdof, 6 * nv), *cinert = FLD(cinert, 10 * nb), *cvel = FLD(cvel, 6 * nb), *cdofdot = FLD(cdofdot, 6 * nv),
        *cacc = FLD(cacc, 6 * nb), *cfrc = FLD(cfrc, 6 * nb), *q_passive = FLD(qpas, nv), *q_bias = FLD(qbias, nv), *q_act = FLD(qact, nv),
        *q_smooth = FLD(qsm, nv), *qld = FLD(qld, m.qld_total), *x = FLD(x, nv), *aforce = FLD(af, nu);
  const float* Mw = d.M + (size_t)T.w * m.nC;
#undef FLD
  const size_t wg = (size_t)T.wg0;
#define GLOAD(f, field, n) st.load(S + (size_t)L.f * G, d.field + wg * (size_t)(n), nval * (n))
#define GSTORE(field, f, n) st.store(d.field + wg * (size_t)(n), S + (size_t)L.f * G, nval * (n))
  const size_t wb = (size_t)T.w;
  const bool v_all = mask & STG_VELOCITY;  // the sub-stage bits serve the individually callable com_vel / passive / rne

  GLOAD(qvel, qvel, nv); GLOAD(cdof, cdof, 6 * nv);
  if (v_all || (mask & STG_RNE)) GLOAD(cinert, cinert, 10 * nb);
  // Long-latency global reads whose consumers come much later are issued now, into registers: the world's inertia entries
  // (scattered into the factor's layout by the Cholesky phase; MREG * LPW entries are prefetched, the rest is read in place)
  // and the "any applied wrench?" test of fwd_acceleration.
  constexpr int MREG = 32;
  float mreg[MREG];
  const bool fac = mask & (STG_ACCELERATION | STG_FACTOR_ONLY);
#pragma unroll
  for (int k = 0; k < MREG; k++) { const int e = sub + k * LPW; mreg[k] = (fac && e < m.nC) ? Mw[e] : 0.f; }
  bool any_xfrc = false;
  if (mask & STG_ACCELERATION) {
#pragma unroll 4
    for (int i = sub; i < 6 * nb; i += LPW) any_xfrc |= d.xfrc_applied[wb * 6 * nb + i] != 0.f;
  }
  st.load_wait();

  // ------------------------------------------------------------------ fwd_velocity
  if (mask & (STG_VELOCITY | STG_COMVEL | STG_PASSIVE | STG_RNE)) {
    if (v_all)
#pragma unroll 1
    for (int a = valid ? sub : nu; a < nu; a += LPW) {  // actuator velocity = moment . qvel
      const int nnz = d.moment_rownnz[wb * nu + a], adr = d.moment_rowadr[wb * nu + a];
      float vel = 0.f;
      for (int k = 0; k < nnz; k++) vel += d.actuator_moment[wb * m.nJmom + adr + k] * qvel[d.moment_colind[wb * m.nJmom + adr + k]];
      d.actuator_velocity[wb * nu + a] = vel;
    }
    if (PEXT && v_all && m.ntendon > 0) {  // forward.py:706-729 tendon velocity
#pragma unroll 1
      for (int t = valid ? sub : m.ntendon; t < m.ntendon; t += LPW) {
        float vel = 0.f;
        for (int k = m.ten_J_rowadr[t]; k < m.ten_J_rowadr[t] + m.ten_J_rownnz[t]; k++) vel += m.ten_J0[k] * qvel[m.ten_J_colind[k]];
        d.ten_velocity[wb * m.ntendon + t] = vel;
      }
    }
    // com_vel: level-synchronous forward pass
    if (v_all || (mask & STG_COMVEL)) {
    if (sub < 6) cvel[sub] = 0.f;
    __syncwarp();
#pragma unroll 1
    for (int l = 1; l < m.nlevel; l++) {
#pragma unroll 1
      for (int i = m.level_adr[l] + sub; i < m.level_adr[l + 1]; i += LPW) {
        const int b = m.level_body[i], pid = m.body_parentid[b], jntadr = m.body_jntadr[b], jntnum = m.body_jntnum[b];
        int dof = m.body_dofadr[b];
        float cv[6];
#pragma unroll
        for (int k = 0; k < 6; k++) cv[k] = cvel[6 * pid + k];
#pragma unroll 1
        for (int j = jntadr; j < jntadr + jntnum; j++) {
          const int t = m.jnt_type[j];
          if (t == JNT_FREE) {
            for (int q = 0; q < 3; q++) { const float v = qvel[dof + q]; for (int k = 0; k < 6; k++) { cv[k] += cdof[6 * (dof + q) + k] * v; cdofdot[6 * (dof + q) + k] = 0.f; } }
            for (int q = 3; q < 6; q++) motion_cross(cv, cdof + 6 * (dof + q), cdofdot + 6 * (dof + q));
            for (int q = 3; q < 6; q++) { const float v = qvel[dof + q]; for (int k = 0; k < 6; k++) cv[k] += cdof[6 * (dof + q) + k] * v; }
            dof += 6;
          } else if (t == JNT_BALL) {
            for (int q = 0; q < 3; q++) motion_cross(cv, cdof + 6 * (dof + q), cdofdot + 6 * (dof + q));
            for (int q = 0; q < 3; q++) { const float v = qvel[dof + q]; for (int k = 0; k < 6; k++) cv[k] += cdof[6 * (dof + q) + k] * v; }
            dof += 3;
          } else {
            motion_cross(cv, cdof + 6 * dof, cdofdot + 6 * dof);
            const float v = qvel[dof];
            for (int k = 0; k < 6; k++) cv[k] += cdof[6 * dof + k] * v;
            dof += 1;
          }
        }
#pragma unroll
        for (int k = 0; k < 6; k++) cvel[6 * b + k] = cv[k];
      }
      __syncwarp();
    }
    st.store_fence();
    GSTORE(cvel, cvel, 6 * nb); GSTORE(cdof_dot, cdofdot, 6 * nv);
    st.store_commit();
    } else if (mask & STG_RNE) {
      GLOAD(cvel, cvel, 6 * nb); GLOAD(cdofdot, cdof_dot, 6 * nv);
      st.load_wait();
    }

    // passive: joint springs (slide / hinge; ball and free joints through quat_sub) and dampers, gravity compensation
    if (v_all || (mask & STG_PASSIVE)) {
      const bool dsbl_spring = m.disableflags & DSBL_SPRING, dsbl_damper = m.disableflags & DSBL_DAMPER;
      const bool gravcomp = PEXT && m.has_gravcomp && !(m.disableflags & DSBL_GRAVITY) && !(dsbl_spring && dsbl_damper);
#pragma unroll 1
      for (int dd = sub; dd < nv; dd += LPW) {
        const int j = m.dof_jntid[dd], t = m.jnt_type[j];
        float spring = 0.f, damper = 0.f, gc = 0.f;
        if (!(dsbl_spring && dsbl_damper)) {
          const float stiffness = m.jnt_stiffness[j];
          if (stiffness != 0.f && !dsbl_spring) {
            const int qa = m.jnt_qposadr[j], k = dd - m.jnt_dofadr[j];
            if (t == JNT_SLIDE || t == JNT_HINGE) spring = -(d.qpos[wb * m.nq + qa] - m.qpos_spring[qa]) * stiffness;
            else if (!PEXT) {}
            else if (t == JNT_FREE && k < 3) spring = -stiffness * (d.qpos[wb * m.nq + qa + k] - m.qpos_spring[qa + k]);
            else {  // rotational part: -k * quat_sub(q, q_spring) (passive.py:141-183, math.py:161-186)
              const int ra = t == JNT_FREE ? qa + 3 : qa, kk = t == JNT_FREE ? k - 3 : k;
              const q4 rot = qnormalize(ldq(d.qpos + wb * m.nq + ra)), ref = ldq(m.qpos_spring + ra);
              const q4 qd = qmul(mkq(ref.w, -ref.x, -ref.y, -ref.z), rot);
              const float s2 = sqrtf(qd.x * qd.x + qd.y * qd.y + qd.z * qd.z);
              if (s2 != 0.f) {
                float speed = 2.0f * atan2f(s2, qd.w);
                if (speed > 3.14159265358979f) speed -= 2.0f * 3.14159265358979f;
                spring = -stiffness * (kk == 0 ? qd.x : kk == 1 ? qd.y : qd.z) * (speed / s2);
              }
            }
          }
          const float damping = m.dof_damping[dd];
          if (damping != 0.f && !dsbl_damper) damper = -qvel[dd] * damping;
          if (PEXT && m.ntendon > 0) {  // tendon springs (dead band lengthspring) and dampers, J^T force gathered per dof (passive.py:208-272)
#pragma unroll 1
            for (int tn = 0; tn < m.ntendon; tn++) {
              const float ks = m.tendon_stiffness[tn], kd = m.tendon_damping[tn];
              if ((ks == 0.f || dsbl_spring) && (kd == 0.f || dsbl_damper)) continue;
              const float J = tendon_J_at(m, tn, dd);
              if (J == 0.f) continue;
              if (ks != 0.f && !dsbl_spring) {
                const float len = d.ten_length[wb * m.ntendon + tn], lo = m.tendon_lengthspring[2 * tn], hi = m.tendon_lengthspring[2 * tn + 1];
                const float x = len > hi ? len - hi : (len < lo ? len - lo : 0.f);
                spring += J * (-x * ks);
              }
              if (kd != 0.f && !dsbl_damper) {
                float vel = 0.f;
                for (int k = m.ten_J_rowadr[tn]; k < m.ten_J_rowadr[tn] + m.ten_J_rownnz[tn]; k++) vel += m.ten_J0[k] * qvel[m.ten_J_colind[k]];
                damper += J * (-vel * kd);
              }
            }
          }
        }
        if (gravcomp) {  // passive.py:275-303: -gravity * mass * gravcomp at the body's inertial origin, projected on this dof
#pragma unroll 1
          for (int b = 1; b < nb; b++) {
            const float g = m.body_gravcomp[b];
            if (g == 0.f || !m.body_isdofancestor[b * nv + dd]) continue;
            const float sc = -m.body_mass[b] * g;
            const v3 off = ld3(d.xipos + (wb * nb + b) * 3) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
            const v3 jp = ld3(cdof + 6 * dd + 3) + cross(ld3(cdof + 6 * dd), off);
            gc += sc * (jp.x * m.gravity_x + jp.y * m.gravity_y + jp.z * m.gravity_z);
          }
        }
        const float passive = spring + damper + (m.jnt_actgravcomp[j] ? 0.f : gc);
        q_passive[dd] = passive;
        if (valid) {
          d.qfrc_spring[wb * nv + dd] = spring;
          d.qfrc_damper[wb * nv + dd] = damper;
          d.qfrc_gravcomp[wb * nv + dd] = gc;
          d.qfrc_passive[wb * nv + dd] = passive;
        }
      }
    }
    // rne: cacc forward, cfrc per body, backward accumulation, projection
    if (v_all || (mask & STG_RNE)) {
    for (int k = sub; k < 6; k += LPW) cacc[k] = k < 3 ? 0.f : ((m.disableflags & DSBL_GRAVITY) ? 0.f : -(k == 3 ? m.gravity_x : k == 4 ? m.gravity_y : m.gravity_z));
    __syncwarp();
#pragma unroll 1
    for (int l = 1; l < m.nlevel; l++) {
#pragma unroll 1
      for (int i = m.level_adr[l] + sub; i < m.level_adr[l + 1]; i += LPW) {
        const int b = m.level_body[i], pid = m.body_parentid[b];
        float a[6];
#pragma unroll
        for (int k = 0; k < 6; k++) a[k] = cacc[6 * pid + k];
#pragma unroll 1
        for (int q = 0; q < m.body_dofnum[b]; q++) {
          const int dof = m.body_dofadr[b] + q;
          const float v = qvel[dof];
#pragma unroll
          for (int k = 0; k < 6; k++) a[k] += cdofdot[6 * dof + k] * v;
        }
#pragma unroll
        for (int k = 0; k < 6; k++) cacc[6 * b + k] = a[k];
      }
      __syncwarp();
    }
    st.store_wait_read();  // cfrc_int takes cdof_dot's slot: the bulk store of cdof_dot must have read it
#pragma unroll 2
    for (int b = sub; b < nb; b += LPW) {
      float f[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (b > 0) {
        float iv[6], g[6];
        inert_vec(cinert + 10 * b, cacc + 6 * b, f);
        inert_vec(cinert + 10 * b, cvel + 6 * b, iv);
        motion_cross_force(cvel + 6 * b, iv, g);
#pragma unroll
        for (int k = 0; k < 6; k++) f[k] += g[k];
      }
#pragma unroll
      for (int k = 0; k < 6; k++) cfrc[6 * b + k] = f[k];
    }
    __syncwarp();
#pragma unroll 1
    for (int l = m.nlevel - 2; l >= 0; l--) {
#pragma unroll 1
      for (int i = m.level_adr[l] + sub; i < m.level_adr[l + 1]; i += LPW) {
        const int b = m.level_body[i];
        float acc[6];
#pragma unroll
        for (int k = 0; k < 6; k++) acc[k] = cfrc[6 * b + k];
#pragma unroll 1
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) {
          const float* cc = cfrc + 6 * m.body_childid[c];
#pragma unroll
          for (int k = 0; k < 6; k++) acc[k] += cc[k];
        }
#pragma unroll
        for (int k = 0; k < 6; k++) cfrc[6 * b + k] = acc[k];
      }
      __syncwarp();
    }
#pragma unroll 1
    for (int dd = sub; dd < nv; dd += LPW) {
      const float v = dot6(cdof + 6 * dd, cfrc + 6 * m.dof_bodyid[dd]);
      q_bias[dd] = v;
    }
    st.store_fence();
    GSTORE(cacc, cacc, 6 * nb); GSTORE(cfrc_int, cfrc, 6 * nb); GSTORE(qfrc_bias, qbias, nv);
    st.store_commit();
    }
  } else if (mask & STG_ACCELERATION) {
    GLOAD(qpas, qfrc_passive, nv); GLOAD(qbias, qfrc_bias, nv);
    st.load_wait();
  }
  __syncwarp();

  // ------------------------------------------------------------------ fwd_actuation
  if (mask & STG_ACTUATION) {
#pragma unroll 1
    for (int dd = sub; dd < nv; dd += LPW) q_act[dd] = 0.f;
    __syncwarp();
    const bool enabled = nu > 0 && !(m.disableflags & DSBL_ACTUATION);
    // actuator forces; scatter moment^T force by a per-dof gather loop over actuators (deterministic, no atomics)
#pragma unroll 1
    for (int a = sub; a < nu; a += LPW) {
      float force = 0.f;
      if (enabled) {
        float ctrl = d.ctrl[wb * nu + a];
        if (m.actuator_ctrllimited[a] && !(m.disableflags & DSBL_CLAMPCTRL)) ctrl = clampf(ctrl, m.actuator_ctrlrange[2 * a], m.actuator_ctrlrange[2 * a + 1]);
        const float length = d.actuator_length[wb * nu + a], velocity = d.actuator_velocity[wb * nu + a];
        const float *gp = m.actuator_gainprm + 10 * a, *bp = m.actuator_biasprm + 10 * a;
        float gain = 0.f, bias = 0.f;
        if (m.actuator_gaintype[a] == GAIN_FIXED) gain = gp[0];
        else if (m.actuator_gaintype[a] == GAIN_AFFINE) gain = gp[0] + gp[1] * length + gp[2] * velocity;
        if (m.actuator_biastype[a] == BIAS_AFFINE) bias = bp[0] + bp[1] * length + bp[2] * velocity;
        float ctrl_act = ctrl;
        if (m.na > 0 && m.actuator_actadr[a] >= 0) {  // stateful actuator (forward.py:800-963): INTEGRATOR / FILTER / FILTEREXACT
          const int last = m.actuator_actadr[a] + m.actuator_actnum[a] - 1, dyn = m.actuator_dyntype[a];
          const float act = d.act[wb * m.na + last];
          float act_dot = 0.f;
          if (dyn == DYN_INTEGRATOR) act_dot = ctrl;
          else if (dyn == DYN_FILTER || dyn == DYN_FILTEREXACT) act_dot = (ctrl - act) / fmaxf(m.actuator_dynprm[10 * a], MJ_MINVAL);
          if (valid) d.act_dot[wb * m.na + last] = act_dot;
          ctrl_act = m.actuator_actearly[a] ? next_act(m, a, act, act_dot, 1.0f, m.actuator_actlimited[a] != 0) : act;
        }
        force = gain * ctrl_act + bias;
        if (m.actuator_forcelimited[a]) force = clampf(force, m.actuator_forcerange[2 * a], m.actuator_forcerange[2 * a + 1]);
      } else if (m.na > 0 && m.actuator_actadr[a] >= 0 && valid) {
        d.act_dot[wb * m.na + m.actuator_actadr[a] + m.actuator_actnum[a] - 1] = 0.f;  // forward.py:1155: actuation disabled
      }
      if (valid) d.actuator_force[wb * nu + a] = force;
      aforce[a] = force;
    }
    __syncwarp();
    if (PEXT && enabled && m.ntendon > 0) {  // forward.py:1054-1094: the actuators of a force-limited tendon share the tendon's range
#pragma unroll 1
      for (int t = sub; t < m.ntendon; t += LPW) {  // one lane per tendon: the actuator sets of different tendons are disjoint
        if (!m.tendon_actfrclimited[t]) continue;
        float total = 0.f;
        for (int b = 0; b < nu; b++) if (m.actuator_trntype[b] == TRN_TENDON && m.actuator_trnid[2 * b] == t) total += aforce[b];
        const float lo = m.tendon_actfrcrange[2 * t], hi = m.tendon_actfrcrange[2 * t + 1];
        const float sc = total < lo ? lo / total : (total > hi ? hi / total : 1.0f);
        if (sc == 1.0f) continue;
        for (int b = 0; b < nu; b++)
          if (m.actuator_trntype[b] == TRN_TENDON && m.actuator_trnid[2 * b] == t) { aforce[b] *= sc; if (valid) d.actuator_force[wb * nu + b] = aforce[b]; }
      }
      __syncwarp();
    }
    if (enabled) {
#pragma unroll 1
      for (int dd = sub; dd < nv; dd += LPW) {
        float q = 0.f;
        // moment^T force through the per-dof reverse table (entries in actuator order -> fixed summation order, no atomics)
        for (int k = m.dofact_adr[dd]; k < m.dofact_adr[dd + 1]; k++) q += d.actuator_moment[wb * m.nJmom + m.dofact_mom[k]] * aforce[m.dofact_act[k]];
        const int j = m.dof_jntid[dd];
        if (!(m.disableflags & DSBL_GRAVITY) && m.jnt_actgravcomp[j]) q += d.qfrc_gravcomp[wb * nv + dd];
        if (m.jnt_actfrclimited[j]) q = clampf(q, m.jnt_actfrcrange[2 * j], m.jnt_actfrcrange[2 * j + 1]);
        q_act[dd] = q;
      }
    }
    st.store_fence();
    GSTORE(qfrc_actuator, qact, nv);
    st.store_commit();
  } else if (mask & STG_ACCELERATION) {
    GLOAD(qact, qfrc_actuator, nv);
    st.load_wait();
  }
  __syncwarp();

  // ------------------------------------------------------------------ fwd_acceleration (factorize=True)
  if (mask & (STG_ACCELERATION | STG_FACTOR_ONLY)) {
    if (mask & STG_ACCELERATION) {
#pragma unroll 1
      for (int dd = sub; dd < nv; dd += LPW) q_smooth[dd] = q_passive[dd] - q_bias[dd] + q_act[dd] + d.qfrc_applied[wb * nv + dd];
      // xfrc_applied: skipped entirely when the world's applied wrenches are all zero (the common case)
      if (team_any<LPW>(any_xfrc, g)) {
#pragma unroll 1
        for (int dd = sub; dd < nv; dd += LPW) {
          const float* cd = cdof + 6 * dd;
          const int db = m.dof_bodyid[dd];
          float acc = 0.f;
          for (int b = db; b < nb; b++) {
            const float* ft = d.xfrc_applied + (wb * nb + b) * 6;
            if (ft[0] == 0.f && ft[1] == 0.f && ft[2] == 0.f && ft[3] == 0.f && ft[4] == 0.f && ft[5] == 0.f) continue;
            int p = b;
            while (p != 0 && p != db) p = m.body_parentid[p];
            if (p == 0) continue;
            const v3 off = ld3(d.xipos + (wb * nb + b) * 3) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
            const v3 cr = cross(ld3(cd), off);
            acc += cd[3] * ft[0] + cd[4] * ft[1] + cd[5] * ft[2] + cd[0] * ft[3] + cd[1] * ft[4] + cd[2] * ft[5] + dot(cr, ld3(ft));
          }
          q_smooth[dd] += acc;
        }
      }
      __syncwarp();
    }
    // per-tree dense Cholesky of M in the qLD layout (upper factor U, row-major, zeros below), qacc_smooth = M^-1 qfrc_smooth
    const bool acc = mask & STG_ACCELERATION;
    // the factor is built where cdof .. cfrc_int and the actuation fields lived, and the solve vector takes qfrc_bias's slot: the
    // bulk stores that read them must have drained
    st.store_wait_read();
#pragma unroll 1
    for (int i = sub; i < m.qld_total; i += LPW) qld[i] = 0.f;
    if (acc)
#pragma unroll 1
      for (int i = sub; i < nv; i += LPW) x[i] = q_smooth[i];
    __syncwarp();
#pragma unroll 1
    for (int t = 0; t < m.ntree; t++) {
      const int start = m.tree_dofadr[t], n = m.tree_dofnum[t];
      float* U = qld + m.tree_qLDadr[t];
      const int e0 = m.M_rowadr[start], e1 = m.M_rowadr[start + n - 1] + m.M_rownnz[start + n - 1];
      // lower entry (r, c) -> U[c][r]; entries e = sub + k * LPW with k < MREG come from the registers loaded at kernel start
#pragma unroll
      for (int k = 0; k < MREG; k++) {
        const int e = sub + k * LPW;
        if (e >= e0 && e < e1) U[(m.M_colind[e] - start) * n + (m.M_entry_row[e] - start)] = mreg[k];
      }
#pragma unroll 1
      for (int e = max(e0, MREG * LPW) + ((sub - max(e0, MREG * LPW)) % LPW + LPW) % LPW; e < e1; e += LPW)
        U[(m.M_colind[e] - start) * n + (m.M_entry_row[e] - start)] = Mw[e];
      __syncwarp();
      team_chol_upper<LPW>(U, n, x + start, acc, sub);
    }
    st.store_fence();
    if (acc) { GSTORE(qfrc_smooth, qsm, nv); GSTORE(qacc_smooth, x, nv); }
    GSTORE(qLD, qld, m.qld_total);
    st.store_commit();
  }
  st.store_wait_read();  // shared memory must outlive the bulk stores that read it
#undef GLOAD
#undef GSTORE
}

}  // namespace

template <bool PEXT>
static TeamKernel vel_kernel(int lpw, bool bat) {
  if (bat) return k_velocity<PEXT, 32, true>;
  return lpw == 8 ? k_velocity<PEXT, 8, false> : lpw == 16 ? k_velocity<PEXT, 16, false> : k_velocity<PEXT, 32, false>;
}
// has_gravcomp also flags free / ball joint springs (io.py put_model); tendons live in the same instantiation
static TeamKernel vel_kernel(const ModelDev& m, int lpw) {
  return m.has_gravcomp || m.ntendon > 0 ? vel_kernel<true>(lpw, m.batched) : vel_kernel<false>(lpw, m.batched);
}

size_t smem_velocity(const ModelDev& m, const DataDev& d) { return team_shape(m, d.wn, vel_layout(m).total, vel_kernel).block_bytes; }
cudaError_t launch_velocity(const ModelDev& m, const DataDev& d, int mask, cudaStream_t s) { return team_launch(m, d, vel_layout(m).total, vel_kernel, mask, s); }
cudaError_t resident_worlds_velocity(const ModelDev& m, const DataDev& d, int* worlds) { return team_resident_worlds(m, d, vel_layout(m).total, vel_kernel, worlds); }
