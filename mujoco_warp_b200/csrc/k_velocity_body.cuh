// k_velocity_body.cuh -- the body of the velocity kernels (k_velocity.cu), included inside k_velocity and k_velocity_fluid.  It reads
// the kernel's parameters mp, d, mask and f and its compile-time PEXT, FLUID, LPW and BAT.  Not a header of its own: no include guard.
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
      // fluid: each body's world-frame wrench into cacc's slot (dead until rne), then projected per dof below (passive.py:631-666)
      [[maybe_unused]] const bool fluid = FLUID && !(dsbl_spring && dsbl_damper);
      if constexpr (FLUID) if (fluid) {
        const float* cv = (v_all || (mask & STG_COMVEL)) ? cvel : d.cvel + wb * 6 * nb;
        const float *xip = d.xipos + wb * nb * 3, *stc = d.subtree_com + wb * nb * 3;
#pragma unroll 1
        for (int b = sub; b < nb; b += LPW)
          fluid_body_wrench(m, f, b, cv + 6 * b, ld3(xip + 3 * b), d.ximat + (wb * nb + b) * 9, ld3(stc + 3 * m.body_rootid[b]), d.geom_xpos + wb * m.ngeom * 3,
                            d.geom_xmat + wb * m.ngeom * 9, cacc + 6 * b);
        __syncwarp();
      }
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
        float passive = spring + damper + (m.jnt_actgravcomp[j] ? 0.f : gc);
        if constexpr (FLUID) {
          const float fl = fluid ? fluid_project(m, dd, cdof + 6 * dd, cacc, d.xipos + wb * nb * 3, d.subtree_com + wb * nb * 3) : 0.f;
          passive += fl;
          if (valid) f.qfrc_fluid[wb * nv + dd] = fl;
        }
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
        else if (m.actuator_gaintype[a] == GAIN_MUSCLE)  // forward.py:976-980, per-world acc0 and lengthrange
          gain = muscle_gain(length, velocity, m.actuator_lengthrange[2 * a], m.actuator_lengthrange[2 * a + 1], m.actuator_acc0[a], gp);
        if (m.actuator_biastype[a] == BIAS_AFFINE) bias = bp[0] + bp[1] * length + bp[2] * velocity;
        else if (m.actuator_biastype[a] == BIAS_MUSCLE)  // forward.py:1016-1019
          bias = muscle_bias(length, m.actuator_lengthrange[2 * a], m.actuator_lengthrange[2 * a + 1], m.actuator_acc0[a], bp);
        float ctrl_act = ctrl;
        if (m.na > 0 && m.actuator_actadr[a] >= 0) {  // stateful actuator (forward.py:800-963): INTEGRATOR / FILTER / FILTEREXACT / MUSCLE
          const int last = m.actuator_actadr[a] + m.actuator_actnum[a] - 1, dyn = m.actuator_dyntype[a];
          const float act = d.act[wb * m.na + last];
          float act_dot = 0.f;
          if (dyn == DYN_INTEGRATOR) act_dot = ctrl;
          else if (dyn == DYN_FILTER || dyn == DYN_FILTEREXACT) act_dot = (ctrl - act) / fmaxf(m.actuator_dynprm[10 * a], MJ_MINVAL);
          else if (dyn == DYN_MUSCLE) act_dot = muscle_dynamics(ctrl, act, m.actuator_dynprm + 10 * a);
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
#include "k_body_xfrc.cuh"
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
