// k_constraint.cu -- fused make_constraint: equality rows (connect / weld / joint), dof-friction rows, joint-limit rows
// (ball, slide / hinge), contact rows (dense Jacobian).
//
// Replaces (reference, /root/reference/mujoco_warp/_src/constraint.py): :61 _zero_constraint_counts, :156 _equality_connect,
// :966 _equality_weld, :500 _equality_joint (+ support.py:506 jac_dof, :615 jac_dot_dof), :2107 _limit_ball, :1765 _friction_dof,
// :1990 _limit_slide_hinge, :2641 _efc_contact_init, :3751 _efc_contact_jac_dense, :4197 _efc_contact_update and the row
// builder :83-152 _efc_row -- ~16 launches with per-row atomics there, one launch here.
//
// One warp owns one world.  Rows are allocated in a fixed order (friction dofs by dof id, limits by joint id via
// ballot/prefix, contacts in the world's contact order), so efc row order is deterministic (the reference's is
// atomics-dependent; its own tests sort before comparing, constraint_test.py:40-59).  Lanes map to dofs: a J row is a
// single coalesced store, J*qvel is a warp-shuffle reduction; the per-row impedance / reference math of the contact rows runs
// afterwards with lanes = rows of the 32-contact batch (phase C), so its eight per-row stores are coalesced over consecutive rows.

#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

namespace {

// Per-contact record prepared by ONE lane per contact (phase A: every dependent lookup -- pool fields, geom -> body ->
// root -> subtree_com, invweight -- happens in parallel across contacts), then consumed by the whole warp (phase B: lanes =
// dofs).  The reference does the same work with one thread per contact (_efc_contact_init) and one tile per world
// (_efc_contact_jac_dense), re-reading the pool from global memory in every kernel.
constexpr int CR_FRAME = 0, CR_FRI = 9, CR_OFF1 = 14, CR_OFF2 = 17, CR_POS = 20, CR_INC = 21, CR_INVW = 22, CR_SOLREF = 23,
              CR_SOLREFF = 25, CR_SOLIMP = 27, CR_B1 = 32, CR_B2 = 33, CR_BASE = 34, CR_NDIM = 35, CR_CONDIM = 36, CR_WORDS = 37;
// phase B leaves J qvel of the contact's (up to ten) rows where its frame and first offset were: slots 0..8 and 14
__device__ __forceinline__ int cr_vel(int k) { return k < 9 ? CR_FRAME + k : CR_OFF1 + (k - 9); }
__host__ __device__ inline int con_cap(const DataDev& d) { return 2 * d.nconmax > 32 ? 2 * d.nconmax : 32; }  // = collision's per-world cap

struct ConLayout { int cdof, scom, qvel, rec, rowmap, total; };
__host__ __device__ inline ConLayout con_layout(const ModelDev& m, const DataDev& d) {
  ConLayout L;
  int o = 0;
  auto take = [&](int n) { int r = o; o += n; return r; };
  L.cdof = take(6 * m.nv); L.scom = take(3 * m.nbody); L.qvel = take(m.nv); L.rec = take(CR_WORDS * 32);  // one 32-contact batch at a time
  L.rowmap = take(d.njmax < 320 ? d.njmax : 320);  // row of the batch -> contact | dimension << 8 (a batch holds <= 32 x 10 rows, njmax caps them)
  L.total = (o + 3) & ~3;
  return L;
}

// general impedance exponent (solimp[4] other than the default 2 or 1): kept out of line, two powf expansions per inlined copy of efc_row
// were a seventh of the kernel's code
__device__ __noinline__ float imp_pow(float bx, float bc, float power) { return (1.0f / powf(bc, power - 1.0f)) * powf(bx, power); }

// constraint.py:83-152
__device__ void efc_row(const ModelDev& m, const DataDev& d, int w, int efcid, float pos_aref, float pos_imp, float invweight,
                        const float* solref, const float* solimp, float margin, float vel, float frictionloss, int type, int id) {
  float timeconst = solref[0];
  const float dampratio = solref[1];
  if (!(m.disableflags & DSBL_REFSAFE)) timeconst = fmaxf(timeconst, 2.0f * m.timestep);
  const float dmin = clampf(solimp[0], MJ_MINIMP, MJ_MAXIMP), dmax = clampf(solimp[1], MJ_MINIMP, MJ_MAXIMP);
  const float width = fmaxf(MJ_MINVAL, solimp[2]), mid = clampf(solimp[3], MJ_MINIMP, MJ_MAXIMP), power = fmaxf(1.0f, solimp[4]);
  const float dmax_sq = dmax * dmax;
  float k = 1.0f / (dmax_sq * timeconst * timeconst * dampratio * dampratio);
  float b = 2.0f / (dmax * timeconst);
  if (solref[0] <= 0.f) k = -solref[0] / dmax_sq;
  if (solref[1] <= 0.f) b = -solref[1] / dmax;
  const float imp_x = fabsf(pos_imp) / width;
  // x^power / c^(power-1) on the lower branch, mirrored on the upper one; power == 2 (MuJoCo default) and 1 avoid powf
  const bool lower = imp_x < mid;
  const float bx = lower ? imp_x : 1.0f - imp_x, bc = lower ? mid : 1.0f - mid;
  float t;
  if (power == 2.0f) t = bx * bx / bc;
  else if (power == 1.0f) t = bx;
  else t = imp_pow(bx, bc, power);
  const float imp_y = lower ? t : 1.0f - t;
  float imp = clampf(dmin + imp_y * (dmax - dmin), dmin, dmax);
  if (imp_x > 1.0f) imp = dmax;
  const size_t r = (size_t)w * d.njmax + efcid;
  d.efc_D[(size_t)w * d.njmax_pad + efcid] = 1.0f / fmaxf(invweight * (1.0f - imp) / imp, MJ_MINVAL);
  d.efc_vel[r] = vel;
  d.efc_aref[r] = -k * imp * pos_aref - b * vel;
  d.efc_pos[r] = pos_aref + margin;
  d.efc_margin[r] = margin;
  d.efc_frictionloss[r] = frictionloss;
  d.efc_type[r] = type;
  d.efc_id[r] = id;
}


// support.py:506 / :615 -- Jacobian column of a point on body b for dof `dof`, and its time derivative.  cvel / cdof_dot
// are read from Data as the previous velocity stage left them (the reference builds constraints before fwd_velocity too).
__device__ __forceinline__ void jac_cols(const ModelDev& m, const DataDev& d, size_t wb, const float* cdof, const float* scom, v3 point, int b,
                                         int dof, v3* jp, v3* jr, v3* dp, v3* dr) {
#include "k_body_jac.cuh"
  const float* cv = d.cvel + (wb * m.nbody + b) * 6;
  const v3 pvel = ld3(cv + 3) - cross(off, ld3(cv));
  float cdd[6];
  const int j = m.dof_jntid[dof], jt = m.jnt_type[j];
  if (jt == JNT_BALL || (jt == JNT_FREE && dof >= m.jnt_dofadr[j] + 3)) motion_cross(d.cvel + (wb * m.nbody + m.dof_bodyid[dof]) * 6, cd, cdd);
  else for (int i = 0; i < 6; i++) cdd[i] = d.cdof_dot[(wb * m.nv + dof) * 6 + i];
  *dp = ld3(cdd + 3) + cross(ld3(cdd), off) + cross(cang, pvel);
  *dr = ld3(cdd);
}
__device__ __forceinline__ float comp3(v3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
__device__ __forceinline__ q4 quat_mul_axis(q4 q, v3 a) {  // math.py:33
  return mkq(-q.x * a.x - q.y * a.y - q.z * a.z, q.w * a.x + q.y * a.z - q.z * a.y, q.w * a.y + q.z * a.x - q.x * a.z, q.w * a.z + q.x * a.y - q.y * a.x);
}
__device__ __forceinline__ q4 qscale(q4 q, float s) { return mkq(q.w * s, q.x * s, q.y * s, q.z * s); }
__device__ __forceinline__ q4 qconj(q4 q) { return mkq(q.w, -q.x, -q.y, -q.z); }
__device__ __forceinline__ v3 qvec(q4 q) { return mk3(q.x, q.y, q.z); }
__device__ __forceinline__ v3 warp_sum3v(v3 a) { return mk3(warp_sum(a.x), warp_sum(a.y), warp_sum(a.z)); }

// EQ = the model has equality constraints or limited ball joints; plain articulated models (humanoid) use the leaner
// instantiation without that code.
template <bool EQ, bool BAT>
__global__ void __launch_bounds__(64, EQ ? 12 : 16)
k_constraint(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;  // every warp of the block owns one world (its own shared-memory slice)
  const int w = blockIdx.x * (blockDim.x >> 5) + warp + d.w0;
  if (w >= d.nworld || w >= d.w0 + d.wn) return;
  MJB_WORLD_MODEL(w)
  const ConLayout L = con_layout(mp, d);
  float* S = smem + warp * L.total;
  float *cdof = S + L.cdof, *scom = S + L.scom, *qvel = S + L.qvel, *rec = S + L.rec;
  int* rowmap = (int*)(S + L.rowmap);
  const int nv = m.nv, nb = m.nbody, njmax = d.njmax, nvp = d.nv_pad;
  const size_t wb = (size_t)w;
  float* Jw = d.efc_J + wb * (size_t)d.njmax_pad * nvp;   // (nworld, njmax_pad, nv_pad)

  if (m.disableflags & DSBL_CONSTRAINT) {
    if (lane == 0) { d.ne[w] = 0; d.nf[w] = 0; d.nl[w] = 0; d.nefc[w] = 0; }
    return;
  }
  warp_copy(cdof, d.cdof + wb * 6 * nv, 6 * nv, lane);
  warp_copy(scom, d.subtree_com + wb * 3 * nb, 3 * nb, lane);
  warp_copy(qvel, d.qvel + wb * nv, nv, lane);
  __syncwarp();

  int nefc = 0, ne = 0, nf = 0, nl = 0;

  // ---- equality rows, in the reference's launch order: connect, weld, joint (constraint.py:4911-5080).  The warp walks
  // the (few) equalities together; lanes map to dofs for the Jacobian rows and the J*qvel / Jdot*qvel reductions.
  if (EQ && m.neq > 0 && !(m.disableflags & DSBL_EQUALITY)) {
#pragma unroll 1
    for (int pass = 0; pass < 4; pass++) {
#pragma unroll 1
      for (int e = 0; e < m.neq; e++) {
        const int type = m.eq_type[e];
        if (type != (pass == 0 ? EQ_CONNECT : pass == 1 ? EQ_WELD : pass == 2 ? EQ_JOINT : EQ_TENDON) || !d.eq_active[wb * m.neq + e]) continue;
        const float* data = m.eq_data + 11 * e;
        const int o1 = m.eq_obj1id[e], o2 = m.eq_obj2id[e];
        if (type == EQ_TENDON) {  // constraint.py:642-826: tendon length (coupled to a second tendon through a quartic)
          const int efcid = nefc;
          nefc += 1; ne += 1;
          if (efcid >= njmax) continue;
          const float pos1 = d.ten_length[wb * m.ntendon + o1] - m.tendon_length0[o1];
          float pos, invweight, deriv = 0.f;
          if (o2 > -1) {
            invweight = m.tendon_invweight0[o1] + m.tendon_invweight0[o2];
            const float dif = d.ten_length[wb * m.ntendon + o2] - m.tendon_length0[o2], dif2 = dif * dif, dif3 = dif2 * dif, dif4 = dif3 * dif;
            pos = pos1 - (data[0] + data[1] * dif + data[2] * dif2 + data[3] * dif3 + data[4] * dif4);
            deriv = data[1] + 2.0f * data[2] * dif + 3.0f * data[3] * dif2 + 4.0f * data[4] * dif3;
          } else {
            invweight = m.tendon_invweight0[o1];
            pos = pos1 - data[0];
          }
          float Jqvel = 0.f;
#pragma unroll 1
          for (int c = lane; c < nvp; c += 32) {
            float J = 0.f;
            if (c < nv) { J = tendon_J_at(m, o1, c); if (deriv != 0.f) J -= deriv * tendon_J_at(m, o2, c); Jqvel += J * qvel[c]; }
            Jw[(size_t)efcid * nvp + c] = J;
          }
          Jqvel = warp_sum(Jqvel);
          if (lane == 0) efc_row(m, d, w, efcid, pos, pos, invweight, m.eq_solref + 2 * e, m.eq_solimp + 5 * e, 0.f, Jqvel, 0.f, CNSTR_EQUALITY, e);
          continue;
        }
        if (type == EQ_JOINT) {
          const int efcid = nefc;
          nefc += 1; ne += 1;
          if (efcid >= njmax) continue;
          const int d1 = m.jnt_dofadr[o1], q1 = m.jnt_qposadr[o1];
          int d2 = -1;
          float pos, Jqvel, invweight, deriv2 = 0.f;
          if (o2 > -1) {
            const int q2 = m.jnt_qposadr[o2];
            d2 = m.jnt_dofadr[o2];
            const float dif = d.qpos[wb * m.nq + q2] - m.qpos0[q2];
            const float rhs = data[0] + dif * (data[1] + dif * (data[2] + dif * (data[3] + dif * data[4])));
            deriv2 = data[1] + dif * (2.0f * data[2] + dif * (3.0f * data[3] + dif * 4.0f * data[4]));
            pos = d.qpos[wb * m.nq + q1] - m.qpos0[q1] - rhs;
            Jqvel = qvel[d1] - qvel[d2] * deriv2;
            invweight = m.dof_invweight0[d1] + m.dof_invweight0[d2];
          } else {
            pos = d.qpos[wb * m.nq + q1] - m.qpos0[q1] - data[0];
            Jqvel = qvel[d1];
            invweight = m.dof_invweight0[d1];
          }
#pragma unroll 1
          for (int c = lane; c < nvp; c += 32) Jw[(size_t)efcid * nvp + c] = c == d1 ? 1.0f : (c == d2 ? -deriv2 : 0.f);
          if (lane == 0) efc_row(m, d, w, efcid, pos, pos, invweight, m.eq_solref + 2 * e, m.eq_solimp + 5 * e, 0.f, Jqvel, 0.f, CNSTR_EQUALITY, e);
          continue;
        }
        // every row of the block that fits below njmax is written (the reference skips a block that ends at or beyond njmax,
        // constraint.py:228, :1039, which leaves rows the solver reads unwritten)
        const int nrow = type == EQ_CONNECT ? 3 : 6, efcid = nefc, nfit = min(nrow, njmax - efcid);
        nefc += nrow; ne += nrow;
        if (nfit <= 0) continue;
        const int b1 = o1, b2 = o2;
        const v3 a1 = ld3(data), a2 = ld3(data + 3);  // connect: a1 in body1, a2 in body2; weld: data[0:3] is in body2's frame
        const v3 pos1 = ld3(d.xpos + (wb * nb + b1) * 3) + matvec(d.xmat + (wb * nb + b1) * 9, type == EQ_CONNECT ? a1 : a2);
        const v3 pos2 = ld3(d.xpos + (wb * nb + b2) * 3) + matvec(d.xmat + (wb * nb + b2) * 9, type == EQ_CONNECT ? a2 : a1);
        q4 quat = mkq(1.f, 0.f, 0.f, 0.f), quat1 = quat;
        const q4 xq1 = ldq(d.xquat + (wb * nb + b1) * 4), xq2 = ldq(d.xquat + (wb * nb + b2) * 4), relpose = ldq(data + 6);
        float torquescale = 0.f;
        if (type == EQ_WELD) { torquescale = data[10]; quat = qmul(xq1, relpose); quat1 = qconj(xq2); }
        v3 Jqvelp = mk3(0.f, 0.f, 0.f), Jqvelr = Jqvelp, Jdotvp = Jqvelp, Jdotvr0 = Jqvelp;
#pragma unroll 1
        for (int c = lane; c < nvp; c += 32) {
          v3 jdp = mk3(0.f, 0.f, 0.f), jdr = jdp;
          if (c < nv) {
            v3 jp1, jr1, dp1, dr1, jp2, jr2, dp2, dr2;
            jac_cols(m, d, wb, cdof, scom, pos1, b1, c, &jp1, &jr1, &dp1, &dr1);
            jac_cols(m, d, wb, cdof, scom, pos2, b2, c, &jp2, &jr2, &dp2, &dr2);
            const float qv = qvel[c];
            jdp = jp1 - jp2;
            Jqvelp = Jqvelp + jdp * qv; Jdotvp = Jdotvp + (dp1 - dp2) * qv;
            if (type == EQ_WELD) {
              jdr = qvec(qmul(quat_mul_axis(quat1, (jr1 - jr2) * torquescale), quat)) * 0.5f;
              Jqvelr = Jqvelr + jdr * qv; Jdotvr0 = Jdotvr0 + (dr1 - dr2) * qv;
            }
          }
#pragma unroll
          for (int k = 0; k < 6; k++) if (k < nfit) Jw[(size_t)(efcid + k) * nvp + c] = comp3(k < 3 ? jdp : jdr, k < 3 ? k : k - 3);
        }
        Jqvelp = warp_sum3v(Jqvelp); Jdotvp = warp_sum3v(Jdotvp);
        const v3 cpos = pos1 - pos2;
        const float invw_t = m.body_invweight0[2 * b1] + m.body_invweight0[2 * b2];
        v3 crot = mk3(0.f, 0.f, 0.f), Jdotvr = crot;
        if (type == EQ_WELD) {
          Jqvelr = warp_sum3v(Jqvelr); Jdotvr0 = warp_sum3v(Jdotvr0);
          crot = qvec(qmul(quat1, quat)) * torquescale;
          // rotational Jdot*v through the quaternion product rule (constraint.py:1085-1117, 1381-1395)
          const v3 om1 = ld3(d.cvel + (wb * nb + b1) * 6), om2 = ld3(d.cvel + (wb * nb + b2) * 6), dom = om1 - om2;
          const q4 om1q = mkq(0.f, om1.x, om1.y, om1.z), om2q = mkq(0.f, om2.x, om2.y, om2.z), domq = mkq(0.f, dom.x, dom.y, dom.z);
          const q4 qdot0r = qmul(qscale(qmul(om1q, xq1), 0.5f), relpose), qdot1 = qscale(qmul(om2q, xq2), 0.5f);
          const q4 negqdot1 = qconj(qdot1), negq1 = qconj(xq2), djq = mkq(0.f, Jdotvr0.x, Jdotvr0.y, Jdotvr0.z);
          const v3 t1 = qvec(qmul(qmul(negqdot1, domq), quat)), t2 = qvec(qmul(qmul(negq1, djq), quat)), t3 = qvec(qmul(qmul(negq1, domq), qdot0r));
          Jdotvr = (t1 + t2 + t3) * (0.5f * torquescale);
        }
        const float pos_imp = sqrtf(dot(cpos, cpos) + dot(crot, crot));
        if (lane < nfit) {
          const bool rot = lane >= 3;
          const int k = rot ? lane - 3 : lane;
          const float invw = rot ? m.body_invweight0[2 * b1 + 1] + m.body_invweight0[2 * b2 + 1] : invw_t;
          efc_row(m, d, w, efcid + lane, comp3(rot ? crot : cpos, k), pos_imp, invw, m.eq_solref + 2 * e, m.eq_solimp + 5 * e, 0.f,
                  comp3(rot ? Jqvelr : Jqvelp, k), 0.f, CNSTR_EQUALITY, e);
          d.efc_aref[wb * njmax + efcid + lane] -= comp3(rot ? Jdotvr : Jdotvp, k);
        }
      }
    }
  }

  // ---- dof friction loss rows: one per listed dof whose frictionloss is positive in this world (dof_fricloss_adr lists every dof when
  // dof_frictionloss is per world), allocated in dof order by ballot / prefix like the joint limits
  if (!(m.disableflags & DSBL_FRICTIONLOSS)) {
#pragma unroll 1
    for (int i0 = 0; i0 < m.nfricdof; i0 += 32) {
      const int i = i0 + lane, dof = i < m.nfricdof ? m.dof_fricloss_adr[i] : 0;
      const float fl = i < m.nfricdof ? m.dof_frictionloss[dof] : 0.f;
      const unsigned bal = __ballot_sync(FULL_MASK, fl > 0.f);
      const int efcid = nefc + __popc(bal & ((1u << lane) - 1u));
      if (fl > 0.f && efcid < njmax)
        efc_row(m, d, w, efcid, 0.f, 0.f, m.dof_invweight0[dof], m.dof_solref + 2 * dof, m.dof_solimp + 5 * dof, 0.f, qvel[dof], fl,
                CNSTR_FRICTION_DOF, dof);
      unsigned rem = bal;
      while (rem) {  // whole warp writes each row's J
        const int src = __ffs(rem) - 1;
        rem &= rem - 1;
        const int r = __shfl_sync(FULL_MASK, efcid, src), dcol = __shfl_sync(FULL_MASK, dof, src);
        if (r < njmax)
#pragma unroll 1
          for (int c = lane; c < nvp; c += 32) Jw[(size_t)r * nvp + c] = c == dcol ? 1.0f : 0.f;
      }
      const int n = __popc(bal);
      nefc += n; nf += n;
    }
    if (EQ && m.ntenfric > 0) {  // tendon friction loss (constraint.py:1867-1985)
#pragma unroll 1
      for (int t = 0; t < m.ntendon; t++) {
        if (!(m.tendon_frictionloss[t] > 0.f)) continue;
        const int efcid = nefc;
        nefc += 1; nf += 1;
        if (efcid >= njmax) continue;
        float Jqvel = 0.f;
#pragma unroll 1
        for (int c = lane; c < nvp; c += 32) {
          const float J = c < nv ? tendon_J_at(m, t, c) : 0.f;
          if (c < nv) Jqvel += J * qvel[c];
          Jw[(size_t)efcid * nvp + c] = J;
        }
        Jqvel = warp_sum(Jqvel);
        if (lane == 0)
          efc_row(m, d, w, efcid, 0.f, 0.f, m.tendon_invweight0[t], m.tendon_solref_fri + 2 * t, m.tendon_solimp_fri + 5 * t, 0.f, Jqvel,
                  m.tendon_frictionloss[t], CNSTR_FRICTION_TENDON, t);
      }
    }
  }

  // ---- joint limits: ball joints first (constraint.py:2107), then slide / hinge -- the reference's launch order
  if (!(m.disableflags & DSBL_LIMIT)) {
#pragma unroll 1
    for (int li = 0; li < (EQ ? m.nlimit_ball : 0); li++) {
      const int j = m.jnt_limited_ball_adr[li], qa = m.jnt_qposadr[j], dofadr = m.jnt_dofadr[j];
      const q4 q = qnormalize(ldq(d.qpos + wb * m.nq + qa));
      v3 axis = mk3(0.f, 0.f, 0.f);
      float angle = 0.f;
      const float s2 = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z);
      if (s2 != 0.f) {  // math.py:161 quat_to_vel, then normalize_with_norm
        float speed = 2.0f * atan2f(s2, q.w);
        if (speed > 3.14159265358979f) speed -= 2.0f * 3.14159265358979f;
        const v3 v = mk3(q.x, q.y, q.z) * (speed / s2);
        angle = length(v);
        axis = angle == 0.f ? v : v * (1.0f / angle);
      }
      const float margin = m.jnt_margin[j], pos = fmaxf(m.jnt_range[2 * j], m.jnt_range[2 * j + 1]) - angle - margin;
      if (!(pos < 0.f)) continue;
      const int efcid = nefc;
      nefc += 1; nl += 1;
      if (efcid >= njmax) continue;
#pragma unroll 1
      for (int c = lane; c < nvp; c += 32) Jw[(size_t)efcid * nvp + c] = (c >= dofadr && c < dofadr + 3) ? -comp3(axis, c - dofadr) : 0.f;
      if (lane == 0)
        efc_row(m, d, w, efcid, pos, pos, m.dof_invweight0[dofadr], m.jnt_solref + 2 * j, m.jnt_solimp + 5 * j, margin,
                -(axis.x * qvel[dofadr] + axis.y * qvel[dofadr + 1] + axis.z * qvel[dofadr + 2]), 0.f, CNSTR_LIMIT_JOINT, j);
    }
#pragma unroll 1
    for (int l0 = 0; l0 < m.nlimit; l0 += 32) {
      const int li = l0 + lane;
      bool active = false;
      int j = 0, dofadr = 0;
      float pos = 0.f, Jv = 0.f, margin = 0.f;
      if (li < m.nlimit) {
        j = m.jnt_limited_adr[li];
        const float q = d.qpos[wb * m.nq + m.jnt_qposadr[j]];
        margin = m.jnt_margin[j];
        const float dist_min = q - m.jnt_range[2 * j], dist_max = m.jnt_range[2 * j + 1] - q;
        pos = fminf(dist_min, dist_max) - margin;
        active = pos < 0.f;
        Jv = dist_min < dist_max ? 1.0f : -1.0f;
        dofadr = m.jnt_dofadr[j];
      }
      const unsigned bal = __ballot_sync(FULL_MASK, active);
      const int efcid = nefc + __popc(bal & ((1u << lane) - 1u));
      if (active && efcid < njmax)
        efc_row(m, d, w, efcid, pos, pos, m.dof_invweight0[dofadr], m.jnt_solref + 2 * j, m.jnt_solimp + 5 * j, margin,
                Jv * qvel[dofadr], 0.f, CNSTR_LIMIT_JOINT, j);
      unsigned rem = bal;
      while (rem) {  // whole warp writes each active row's J
        const int src = __ffs(rem) - 1;
        rem &= rem - 1;
        const int r = __shfl_sync(FULL_MASK, efcid, src), dcol = __shfl_sync(FULL_MASK, dofadr, src);
        const float jv = __shfl_sync(FULL_MASK, Jv, src);
        if (r < njmax)
#pragma unroll 1
          for (int c = lane; c < nvp; c += 32) Jw[(size_t)r * nvp + c] = c == dcol ? jv : 0.f;
      }
      const int n = __popc(bal);
      nefc += n; nl += n;
    }
    if (EQ && m.ntendon > 0) {  // tendon limits (constraint.py:2243-2375)
#pragma unroll 1
      for (int t = 0; t < m.ntendon; t++) {
        if (!m.tendon_limited[t]) continue;
        const float len = d.ten_length[wb * m.ntendon + t], margin = m.tendon_margin[t];
        const float dist_min = len - m.tendon_range[2 * t], dist_max = m.tendon_range[2 * t + 1] - len;
        const float pos = fminf(dist_min, dist_max) - margin;
        if (!(pos < 0.f)) continue;
        const int efcid = nefc;
        nefc += 1; nl += 1;
        if (efcid >= njmax) continue;
        const float scl = dist_min < dist_max ? 1.0f : -1.0f;
        float Jqvel = 0.f;
#pragma unroll 1
        for (int c = lane; c < nvp; c += 32) {
          const float J = c < nv ? scl * tendon_J_at(m, t, c) : 0.f;
          if (c < nv) Jqvel += J * qvel[c];
          Jw[(size_t)efcid * nvp + c] = J;
        }
        Jqvel = warp_sum(Jqvel);
        if (lane == 0)
          efc_row(m, d, w, efcid, pos, pos, m.tendon_invweight0[t], m.tendon_solref_lim + 2 * t, m.tendon_solimp_lim + 5 * t, margin, Jqvel, 0.f,
                  CNSTR_LIMIT_TENDON, t);
      }
    }
  }

  // ---- contacts
  if (!(m.disableflags & DSBL_CONTACT)) {
    const int cbase = d.world_conadr[w], ncon = min(d.world_ncon[w], con_cap(d)), np = m.nmaxpyramid;
    const bool elliptic = m.cone == CONE_ELLIPTIC;
#pragma unroll 1
    for (int c0 = 0; c0 < ncon; c0 += 32) {
      // ---- phase A: lane = contact (batch of 32)
      const int c = c0 + lane, cid = cbase + c;
      int ndim = 0, condim = 0;
      float includemargin = 0.f, pos = 0.f;
      if (c < ncon) {
        includemargin = d.contact_includemargin[cid];
        pos = d.contact_dist[cid] - includemargin;
        condim = d.contact_dim[cid];
        if (pos < 0.f) ndim = elliptic ? condim : (condim == 1 ? 1 : 2 * (condim - 1));
      }
      const int bstart = nefc;  // first row of this batch
      const int base = nefc + warp_excl_scan(ndim, lane);
      nefc += warp_sum_i(ndim);
      if (c < ncon) {
        float* r = rec + CR_WORDS * lane;
        r[CR_NDIM] = __int_as_float(ndim);
        if (ndim > 0) {
          const int g1 = d.contact_geom[2 * cid], g2 = d.contact_geom[2 * cid + 1], b1 = m.geom_bodyid[g1], b2 = m.geom_bodyid[g2];
          const v3 cpos = ld3(d.contact_pos + 3 * cid);
          for (int k = 0; k < 9; k++) r[CR_FRAME + k] = d.contact_frame[9 * (size_t)cid + k];
          for (int k = 0; k < 5; k++) { r[CR_FRI + k] = d.contact_friction[5 * cid + k]; r[CR_SOLIMP + k] = d.contact_solimp[5 * cid + k]; }
          st3(r + CR_OFF1, cpos - ld3(scom + 3 * m.body_rootid[b1]));
          st3(r + CR_OFF2, cpos - ld3(scom + 3 * m.body_rootid[b2]));
          r[CR_POS] = pos; r[CR_INC] = includemargin;
          r[CR_INVW] = m.body_invweight0[2 * b1] + m.body_invweight0[2 * b2];
          r[CR_SOLREF] = d.contact_solref[2 * cid]; r[CR_SOLREF + 1] = d.contact_solref[2 * cid + 1];
          r[CR_SOLREFF] = d.contact_solreffriction[2 * cid]; r[CR_SOLREFF + 1] = d.contact_solreffriction[2 * cid + 1];
          r[CR_B1] = __int_as_float(b1); r[CR_B2] = __int_as_float(b2);
          r[CR_BASE] = __int_as_float(base); r[CR_CONDIM] = __int_as_float(condim);
          for (int k = 0; k < ndim; k++) {
            d.contact_efc_address[np * cid + k] = base + k < njmax ? base + k : -1;
            if (base + k < njmax) rowmap[base + k - bstart] = lane | (k << 8);
          }
        }
      }
      __syncwarp();
      // ---- phase B: lanes = dofs, the batch's contacts one after the other, every operand already in shared memory
      const int nb_ = min(32, ncon - c0);
#pragma unroll 1
      for (int cb = 0; cb < nb_; cb++) {
      const float* r = rec + CR_WORDS * cb;
      const int ndim = __float_as_int(r[CR_NDIM]);
      if (ndim == 0) continue;
      const int base = __float_as_int(r[CR_BASE]), condim = __float_as_int(r[CR_CONDIM]);
      const int b1 = __float_as_int(r[CR_B1]), b2 = __float_as_int(r[CR_B2]);
      float frame[9], fri[5];
      for (int k = 0; k < 9; k++) frame[k] = r[CR_FRAME + k];
      for (int k = 0; k < 5; k++) fri[k] = r[CR_FRI + k];
      const v3 off1 = ld3(r + CR_OFF1), off2 = ld3(r + CR_OFF2);
      float velp[10];
#pragma unroll
      for (int k = 0; k < 10; k++) velp[k] = 0.f;
#pragma unroll 1
      for (int dd = lane; dd < nvp; dd += 32) {
        v3 jpd = mk3(0.f, 0.f, 0.f), jrd = mk3(0.f, 0.f, 0.f);
        float qv = 0.f;
        if (dd < nv) {
          const v3 ang = ld3(cdof + 6 * dd), lin = ld3(cdof + 6 * dd + 3);
          qv = qvel[dd];
          const int a1 = m.body_isdofancestor[b1 * nv + dd], a2 = m.body_isdofancestor[b2 * nv + dd];
          if (a2) { jpd = lin + cross(ang, off2); jrd = ang; }
          if (a1) { jpd = jpd - (lin + cross(ang, off1)); jrd = jrd - ang; }
        }
        const float p0 = dot(jpd, ld3(frame)), p1 = dot(jpd, ld3(frame + 3)), p2 = dot(jpd, ld3(frame + 6));
        const float r0 = dot(jrd, ld3(frame)), r1 = dot(jrd, ld3(frame + 3)), r2 = dot(jrd, ld3(frame + 6));
        if (!elliptic && ndim == 4) {
          // the common contact (pyramidal, condim 3): rows n + mu1 t1, n - mu1 t1, n + mu2 t2, n - mu2 t2 written out, without the
          // ten-way predicated generic loop below (constraint.py:3851-3868)
          const float J0 = p0 + p1 * fri[0], J1 = p0 + p1 * -fri[0], J2 = p0 + p2 * fri[1], J3 = p0 + p2 * -fri[1];
          float* Jr = Jw + (size_t)base * nvp + dd;
          if (base < njmax) Jr[0] = J0;
          if (base + 1 < njmax) Jr[nvp] = J1;
          if (base + 2 < njmax) Jr[2 * nvp] = J2;
          if (base + 3 < njmax) Jr[3 * nvp] = J3;
          velp[0] += J0 * qv; velp[1] += J1 * qv; velp[2] += J2 * qv; velp[3] += J3 * qv;
          continue;
        }
#pragma unroll
        for (int dim = 0; dim < 10; dim++) {
          if (dim < ndim) {
            float J;
            if (elliptic) {
              J = dim == 0 ? p0 : dim == 1 ? p1 : dim == 2 ? p2 : dim == 3 ? r0 : dim == 4 ? r1 : r2;
            } else {
              J = p0;
              if (condim > 1) {
                const int dimid2 = dim / 2 + 1;
                const float frii = fri[dimid2 - 1] * ((dim & 1) ? -1.0f : 1.0f);
                const float comp = dimid2 == 1 ? p1 : dimid2 == 2 ? p2 : dimid2 == 3 ? r0 : dimid2 == 4 ? r1 : r2;
                J += comp * frii;
              }
            }
            if (base + dim < njmax) Jw[(size_t)(base + dim) * nvp + dd] = J;
            velp[dim] += J * qv;
          }
        }
      }
      // J qvel of the contact's rows, left in the record for phase C (the frame / offset slots are free again: every lane holds its
      // copy in registers).  Four rows -- a pyramidal condim-3 contact -- go through the halving butterfly: 6 SHFL instead of 20.
      __syncwarp();
      float* rv = rec + CR_WORDS * cb;
      if (ndim == 4) {
        const bool b4 = lane & 16, b3 = lane & 8;
        const float w0 = (b4 ? velp[2] : velp[0]) + __shfl_xor_sync(FULL_MASK, b4 ? velp[0] : velp[2], 16);
        const float w1 = (b4 ? velp[3] : velp[1]) + __shfl_xor_sync(FULL_MASK, b4 ? velp[1] : velp[3], 16);
        float t = (b3 ? w1 : w0) + __shfl_xor_sync(FULL_MASK, b3 ? w0 : w1, 8);
        t += __shfl_xor_sync(FULL_MASK, t, 4);
        t += __shfl_xor_sync(FULL_MASK, t, 2);
        t += __shfl_xor_sync(FULL_MASK, t, 1);
        if ((lane & 7) == 0) rv[cr_vel(lane >> 3)] = t;  // row 2 b4 + b3 ended up in lanes 8 (2 b4 + b3) ..
      } else {
#pragma unroll
        for (int dim = 0; dim < 10; dim++) {
          if (dim < ndim) { const float s = warp_sum(velp[dim]); if (lane == dim) rv[cr_vel(dim)] = s; }
        }
      }
      }
      __syncwarp();
      // ---- phase C: lane = row of the batch (constraint.py:4197-4343): impedance / reference of up to 32 rows at a time, the
      // per-row stores coalesced over consecutive rows
      const int nrows_b = min(nefc, njmax) - bstart;
#pragma unroll 1
      for (int rr = lane; rr < nrows_b; rr += 32) {
        const int rm = rowmap[rr], cb = rm & 255, dim = rm >> 8, efcid = bstart + rr;
        const float* r = rec + CR_WORDS * cb;
        const int cid = cbase + c0 + cb, condim = __float_as_int(r[CR_CONDIM]);
        const float pos = r[CR_POS], includemargin = r[CR_INC], myvel = r[cr_vel(dim)];
        float invweight = r[CR_INVW];
        float pos_aref = pos;
        float ref[2] = {r[CR_SOLREF], r[CR_SOLREF + 1]};
        float imp5[5];
        for (int k = 0; k < 5; k++) imp5[k] = r[CR_SOLIMP + k];
        if (elliptic) {
          if (dim > 0) {
            const float s0 = r[CR_SOLREFF], s1 = r[CR_SOLREFF + 1];
            if (s0 != 0.f || s1 != 0.f) { ref[0] = s0; ref[1] = s1; }
            invweight = invweight * m.impratio_invsqrt * m.impratio_invsqrt;
            if (dim > 1) invweight *= r[CR_FRI] * r[CR_FRI] / (r[CR_FRI + dim - 1] * r[CR_FRI + dim - 1]);
            pos_aref = 0.f;
          }
        } else if (condim > 1) {
          const float f0 = r[CR_FRI];
          invweight = invweight + f0 * f0 * invweight;
          invweight = invweight * 2.0f * f0 * f0 * m.impratio_invsqrt * m.impratio_invsqrt;
        }
        const int type = condim == 1 ? CNSTR_CONTACT_FRICTIONLESS : (elliptic ? CNSTR_CONTACT_ELLIPTIC : CNSTR_CONTACT_PYRAMIDAL);
        efc_row(m, d, w, efcid, pos_aref, pos, invweight, ref, imp5, includemargin, myvel, 0.f, type, cid);
      }
      __syncwarp();
    }
  }
  if (lane == 0) { d.ne[w] = ne; d.nf[w] = nf; d.nl[w] = nl; d.nefc[w] = nefc; }
}

}  // namespace

// warps (= worlds) per block: one-warp blocks cap an SM at 32 resident worlds (CTA limit)
constexpr int constraint_wpb() { return 2; }

size_t smem_constraint(const ModelDev& m, const DataDev& d) { return (size_t)con_layout(m, d).total * sizeof(float) * constraint_wpb(); }

cudaError_t launch_constraint(const ModelDev& m, const DataDev& d, cudaStream_t s) {
  const bool eq = m.neq > 0 || m.nlimit_ball > 0 || m.ntendon > 0;
  void (*kern)(ModelDev, DataDev) = eq ? (m.batched ? k_constraint<true, true> : k_constraint<true, false>) : (m.batched ? k_constraint<false, true> : k_constraint<false, false>);
  const int grid = (d.wn + constraint_wpb() - 1) / constraint_wpb();
  return launch(kern, grid, constraint_wpb() * 32, smem_constraint(m, d), s, m, d);
}
