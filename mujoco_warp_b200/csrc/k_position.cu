// k_position.cu -- fused position stage: kinematics -> com_pos -> camlight -> crb (+M) -> transmission.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): smooth.py:46-226 (5 kinematics kernels),
// :686-855 (com_pos: 11 launches with float atomics per tree level), :858-1027 (camlight), :1029-1098 (crb: 10
// launches), :2288-2396 (_transmission, joint transmission).  One warp owns one world: the body tree lives in the
// warp's shared-memory slice, tree passes run level by level with __syncwarp() instead of one launch per level,
// parents gather their children in fixed order (deterministic; no float atomics), and every Data field is written
// once with coalesced row stores.  `mask` selects sub-stages so each public stage function stays individually callable;
// inputs a skipped sub-stage would have produced are re-loaded from Data.

#include "mjb_math.cuh"
#include "mjb_team.cuh"
#include "mjb_types.cuh"

namespace {

struct PosLayout {
  int qpos, xpos, xquat, xipos, xanchor, xaxis, scom, cinert, cdof, buf, arena, gxpos, gxmat, M, total;
};

// Per-world words of shared memory.  Only what later phases read stays resident (body poses, joint anchors / axes, subtree
// com, cinert -> crb in place, cdof); pure outputs pass through space whose bulk store has drained:
//  - the arena holds qpos until the tree pass and the transmission are done, then xmat, then ximat;
//  - geom_xpos and geom_xmat are built from xipos on: xipos, xanchor, xaxis, subtree_com and the arena have all been stored by then;
//  - the crb * cdof scratch and then M are built from xpos on, once the body poses have left.
// 3.3 KB per humanoid world, so that an SM holds 64 worlds at once and 8192 worlds fit on 132 SMs in one round.  That is what
// the kernel time hangs on -- it is latency bound (ncu: one instruction issued per ~13 cycles per warp, long-scoreboard stalls
// on dependent table lookups), so time ~ rounds of resident worlds x per-warp chain (DESIGN.md §3).
__host__ __device__ inline int pad4(int n) { return (n + 3) & ~3; }
__host__ __device__ inline PosLayout pos_layout(const ModelDev& m) {
  PosLayout L;
  int o = 0;
  auto take = [&](int n) { int r = o; o += pad4(n); return r; };  // padded: a field's group block [G][n] starts 16 B aligned
  L.xpos = take(3 * m.nbody); L.xquat = take(4 * m.nbody); L.xipos = take(3 * m.nbody);
  L.xanchor = take(3 * m.njnt); L.xaxis = take(3 * m.njnt); L.scom = take(3 * m.nbody);
  L.arena = take(pad4(m.nq) > pad4(9 * m.nbody) ? m.nq : 9 * m.nbody);
  L.qpos = L.arena;
  L.gxpos = L.xipos; L.gxmat = L.gxpos + pad4(3 * m.ngeom);
  L.buf = L.xpos; L.M = L.buf + pad4(6 * m.nv);
  if (o < L.gxmat + pad4(9 * m.ngeom)) o = L.gxmat + pad4(9 * m.ngeom);
  if (o < L.M + pad4(m.nC)) o = L.M + pad4(m.nC);
  L.cinert = take(10 * m.nbody); L.cdof = take(6 * m.nv);
  L.total = o;
  return L;
}

// LPW lanes per world, G = 32 / LPW worlds per warp (one warp per block).  Shared layout of field f: [G][n_f] at S + L.f * G.
// BAT: per-world (batched) Model fields -- the launcher then uses one world per warp so the world's offsets stay uniform
template <int LPW, bool BAT>
__global__ void __launch_bounds__(256)
k_position(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int mask) {
  extern __shared__ __align__(16) float smem[];
  constexpr int G = 32 / LPW;
  Team<LPW> T;
  T.init(d.w0, d.wn, d.nworld);
  if (T.nvalid <= 0) return;
  MJB_WORLD_MODEL(T.w)
  const int lane = T.lane, sub = T.sub, g = T.g, nval = T.nvalid;
  const bool valid = T.valid;
  const PosLayout L = pos_layout(mp);
  float* S = smem + (size_t)(threadIdx.x >> 5) * ((size_t)L.total * G + 4);  // this warp's slice (+ its mbarrier)
  Stager st;
  st.init(reinterpret_cast<uint64_t*>(S + (size_t)L.total * G), lane);
  const int nb = m.nbody, nj = m.njnt, ng = m.ngeom, nv = m.nv;
  // block (all G worlds) and this team's row of a field
#define BLK(f) (S + (size_t)L.f * G)
#define ROW(blk, n) ((blk) + (size_t)g * (n))
  float *qpos = ROW(BLK(qpos), m.nq), *xpos = ROW(BLK(xpos), 3 * nb), *xquat = ROW(BLK(xquat), 4 * nb), *xipos = ROW(BLK(xipos), 3 * nb),
        *xanchor = ROW(BLK(xanchor), 3 * nj), *xaxis = ROW(BLK(xaxis), 3 * nj), *scom = ROW(BLK(scom), 3 * nb), *cinert = ROW(BLK(cinert), 10 * nb),
        *cdof = ROW(BLK(cdof), 6 * nv);
  float *xmat = ROW(BLK(arena), 9 * nb), *ximat = ROW(BLK(arena), 9 * nb), *gxpos = ROW(BLK(gxpos), 3 * ng), *gxmat = ROW(BLK(gxmat), 9 * ng),
        *buf = ROW(BLK(buf), 6 * nv), *Ms = ROW(BLK(M), m.nC);
  float* crb = cinert;  // accumulated in place once cinert has been stored
  // the G worlds' rows of a Data field are one contiguous block in global memory
  const size_t wg = (size_t)T.wg0;
#define GLOAD(blk, field, n) st.load(blk, d.field + wg * (size_t)(n), nval * (n))
#define GSTORE(field, blk, n) st.store(d.field + wg * (size_t)(n), blk, nval * (n))
  const size_t wb = (size_t)T.w;
  const bool kin = mask & STG_KINEMATICS, com = mask & STG_COM_POS, cam = mask & STG_CAMLIGHT, crbm = mask & STG_CRB;

  // ------------------------------------------------------------------ inputs
  if (mask & (STG_KINEMATICS | STG_TRANSMISSION)) GLOAD(BLK(qpos), qpos, m.nq);
  if (!kin && (com || cam)) {  // a skipped kinematics stage: its outputs come from Data
    GLOAD(BLK(xpos), xpos, 3 * nb); GLOAD(BLK(xquat), xquat, 4 * nb); GLOAD(BLK(xipos), xipos, 3 * nb);
    GLOAD(BLK(xanchor), xanchor, 3 * nj); GLOAD(BLK(xaxis), xaxis, 3 * nj);
  }
  if (!com && (cam || crbm)) { GLOAD(BLK(scom), subtree_com, 3 * nb); GLOAD(BLK(cinert), cinert, 10 * nb); GLOAD(BLK(cdof), cdof, 6 * nv); }
  st.load_wait();

  // ------------------------------------------------------------------ kinematics: tree pass (smooth.py:46-145)
  if (kin) {
    if (sub == 0) { xpos[0] = xpos[1] = xpos[2] = 0.f; xquat[0] = 1.f; xquat[1] = xquat[2] = xquat[3] = 0.f; }
    __syncwarp();
#pragma unroll 1
    for (int l = 1; l < m.nlevel; l++) {
#pragma unroll 1
      for (int i = m.level_adr[l] + sub; i < m.level_adr[l + 1]; i += LPW) {
        const int b = m.level_body[i], pid = m.body_parentid[b], jntadr = m.body_jntadr[b], jntnum = m.body_jntnum[b];
        if (jntnum == 1 && m.jnt_type[jntadr] == JNT_FREE) {
          const int qa = m.jnt_qposadr[jntadr];
          v3 p = ld3(qpos + qa);
          q4 q = qnormalize(ldq(qpos + qa + 3));
          st3(xpos + 3 * b, p); stq(xquat + 4 * b, q);
          st3(xanchor + 3 * jntadr, p); st3(xaxis + 3 * jntadr, ld3(m.jnt_axis + 3 * jntadr));
          continue;
        }
        q4 pq = ldq(xquat + 4 * pid);
        // mocap bodies take their pose from Data.mocap_pos / mocap_quat (smooth.py:104-110)
        const int mc = m.nmocap > 0 ? m.body_mocapid[b] : -1;
        const v3 bpos = mc >= 0 ? ld3(d.mocap_pos + (wb * m.nmocap + mc) * 3) : ld3(m.body_pos + 3 * b);
        const q4 bquat = mc >= 0 ? ldq(d.mocap_quat + (wb * m.nmocap + mc) * 4) : ldq(m.body_quat + 4 * b);
        v3 pos = qrot(pq, bpos) + ld3(xpos + 3 * pid);
        q4 quat = qmul(pq, bquat);
#pragma unroll 1
        for (int j = jntadr; j < jntadr + jntnum; j++) {
          const int qa = m.jnt_qposadr[j], t = m.jnt_type[j];
          v3 jpos = ld3(m.jnt_pos + 3 * j), jax = ld3(m.jnt_axis + 3 * j);
          v3 anchor = qrot(quat, jpos) + pos, axis = qrot(quat, jax);
          if (t == JNT_BALL) {
            quat = qmul(quat, qnormalize(ldq(qpos + qa)));
            pos = anchor - qrot(quat, jpos);
          } else if (t == JNT_SLIDE) {
            pos = pos + axis * (qpos[qa] - m.qpos0[qa]);
          } else if (t == JNT_HINGE) {
            quat = qmul(quat, axis_angle_quat(jax, qpos[qa] - m.qpos0[qa]));
            pos = anchor - qrot(quat, jpos);
          }
          st3(xanchor + 3 * j, anchor); st3(xaxis + 3 * j, axis);
        }
        st3(xpos + 3 * b, pos); stq(xquat + 4 * b, qnormalize(quat));
      }
      __syncwarp();
    }
  }

  // ------------------------------------------------------------------ tendon (smooth.py:3658-3692, 4197: fixed tendons)
  if (kin && m.ntendon > 0) {
#pragma unroll 1
    for (int t = valid ? sub : m.ntendon; t < m.ntendon; t += LPW) {
      d.ten_length[wb * m.ntendon + t] = tendon_length(m, t, qpos);
      for (int k = m.ten_J_rowadr[t]; k < m.ten_J_rowadr[t] + m.ten_J_rownnz[t]; k++) d.ten_J[wb * m.nJten + k] = m.ten_J0[k];
    }
  }

  // ------------------------------------------------------------------ transmission (joint / tendon transmission; smooth.py:2288-2396)
  if (mask & STG_TRANSMISSION) {
#pragma unroll 1
    for (int a = valid ? sub : m.nu; a < m.nu; a += LPW) {
      if (m.ntendon > 0 && m.actuator_trntype[a] == TRN_TENDON) {  // smooth.py:2508-2525: length and moment of the tendon, times gear[0]
        const int t = m.actuator_trnid[2 * a], adr = m.moment_rowadr0[a], nnz = m.moment_rownnz0[a], tadr = m.ten_J_rowadr[t];
        const float gear0 = m.actuator_gear[6 * a];
        d.actuator_length[wb * m.nu + a] = tendon_length(m, t, qpos) * gear0;
        d.moment_rownnz[wb * m.nu + a] = nnz;
        d.moment_rowadr[wb * m.nu + a] = adr;
        for (int k = 0; k < nnz; k++) {
          d.moment_colind[wb * m.nJmom + adr + k] = m.moment_colind0[adr + k];
          d.actuator_moment[wb * m.nJmom + adr + k] = m.ten_J0[tadr + k] * gear0;
        }
        continue;
      }
      const int j = m.actuator_trnid[2 * a], t = m.jnt_type[j], adr = m.moment_rowadr0[a], nnz = m.moment_rownnz0[a];
      const float* gear = m.actuator_gear + 6 * a;
      d.actuator_length[wb * m.nu + a] = (t == JNT_SLIDE || t == JNT_HINGE) ? qpos[m.jnt_qposadr[j]] * gear[0] : 0.f;
      d.moment_rownnz[wb * m.nu + a] = nnz;
      d.moment_rowadr[wb * m.nu + a] = adr;
#pragma unroll 1
      for (int k = 0; k < nnz; k++) {
        d.moment_colind[wb * m.nJmom + adr + k] = m.moment_colind0[adr + k];
        d.actuator_moment[wb * m.nJmom + adr + k] = gear[k];
      }
    }
  }

  __syncwarp();  // tendon / transmission lanes are done reading qpos: the arena it lives in is about to take xmat (found by racecheck)

  // ------------------------------------------------------------------ kinematics: per-body frames, sites
  if (kin) {
#pragma unroll 2
    for (int b = sub; b < nb; b += LPW) {
      q4 q = ldq(xquat + 4 * b);
      quat_to_mat(q, xmat + 9 * b);
      st3(xipos + 3 * b, ld3(xpos + 3 * b) + qrot(q, ld3(m.body_ipos + 3 * b)));
    }
#pragma unroll 1
    for (int s = valid ? sub : m.nsite; s < m.nsite; s += LPW) {
      const int b = m.site_bodyid[s];
      q4 q = ldq(xquat + 4 * b);
      float mat[9];
      st3(d.site_xpos + (wb * m.nsite + s) * 3, ld3(xpos + 3 * b) + qrot(q, ld3(m.site_pos + 3 * s)));
      quat_to_mat(qmul(q, ldq(m.site_quat + 4 * s)), mat);
      for (int k = 0; k < 9; k++) d.site_xmat[(wb * m.nsite + s) * 9 + k] = mat[k];
    }
    st.store_fence();
    GSTORE(xpos, BLK(xpos), 3 * nb); GSTORE(xquat, BLK(xquat), 4 * nb); GSTORE(xmat, BLK(arena), 9 * nb); GSTORE(xipos, BLK(xipos), 3 * nb);
    GSTORE(xanchor, BLK(xanchor), 3 * nj); GSTORE(xaxis, BLK(xaxis), 3 * nj);
    st.store_commit();
    if (!com) {  // kinematics alone: the inertial frames follow xmat through the arena (otherwise the cinert loop below produces them)
      st.store_wait_read();
#pragma unroll 2
      for (int b = sub; b < nb; b += LPW) quat_to_mat(qmul(ldq(xquat + 4 * b), ldq(m.body_iquat + 4 * b)), ximat + 9 * b);
      st.store_fence();
      GSTORE(ximat, BLK(arena), 9 * nb);
      st.store_commit();
    }
  }
  __syncwarp();

  // ------------------------------------------------------------------ com_pos (smooth.py:686-855)
  if (com) {
#pragma unroll 2
    for (int b = sub; b < nb; b += LPW) st3(scom + 3 * b, ld3(xipos + 3 * b) * m.body_mass[b]);
    __syncwarp();
#pragma unroll 1
    for (int l = m.nlevel - 2; l >= 0; l--) {
#pragma unroll 1
      for (int i = m.level_adr[l] + sub; i < m.level_adr[l + 1]; i += LPW) {
        const int b = m.level_body[i];
        v3 acc = ld3(scom + 3 * b);
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) acc = acc + ld3(scom + 3 * m.body_childid[c]);
        st3(scom + 3 * b, acc);
      }
      __syncwarp();
    }
#pragma unroll 2
    for (int b = sub; b < nb; b += LPW) {
      const float ms = m.body_subtreemass[b];
      if (ms != 0.f) st3(scom + 3 * b, ld3(scom + 3 * b) * (1.0f / ms));
    }
    __syncwarp();
    if (kin) st.store_wait_read();  // xmat has left the arena (long ago: the subtree-com passes ran in between); ximat takes its place
#pragma unroll 2
    for (int b = sub; b < nb; b += LPW) {  // cinert (smooth.py:733); the inertial frame is built here, on its way out through the arena
      float* mat = ximat + 9 * b;
      quat_to_mat(qmul(ldq(xquat + 4 * b), ldq(m.body_iquat + 4 * b)), mat);
      const v3 inert = ld3(m.body_inertia + 3 * b);
      const float mass = m.body_mass[b];
      const v3 dif = ld3(xipos + 3 * b) - ld3(scom + 3 * m.body_rootid[b]);
      float* r = cinert + 10 * b;
      // mat * diag(inert) * mat^T, symmetric
      const float a0 = mat[0] * inert.x, a1 = mat[1] * inert.y, a2 = mat[2] * inert.z;
      const float b0 = mat[3] * inert.x, b1 = mat[4] * inert.y, b2 = mat[5] * inert.z;
      const float c0 = mat[6] * inert.x, c1 = mat[7] * inert.y, c2 = mat[8] * inert.z;
      r[0] = a0 * mat[0] + a1 * mat[1] + a2 * mat[2] + mass * (dif.y * dif.y + dif.z * dif.z);
      r[1] = b0 * mat[3] + b1 * mat[4] + b2 * mat[5] + mass * (dif.x * dif.x + dif.z * dif.z);
      r[2] = c0 * mat[6] + c1 * mat[7] + c2 * mat[8] + mass * (dif.x * dif.x + dif.y * dif.y);
      r[3] = a0 * mat[3] + a1 * mat[4] + a2 * mat[5] - mass * dif.x * dif.y;
      r[4] = a0 * mat[6] + a1 * mat[7] + a2 * mat[8] - mass * dif.x * dif.z;
      r[5] = b0 * mat[6] + b1 * mat[7] + b2 * mat[8] - mass * dif.y * dif.z;
      r[6] = mass * dif.x; r[7] = mass * dif.y; r[8] = mass * dif.z; r[9] = mass;
    }
#pragma unroll 2
    for (int j = sub; j < nj; j += LPW) {  // cdof (smooth.py:779)
      const int b = m.jnt_bodyid[j], t = m.jnt_type[j];
      int dof = m.jnt_dofadr[j];
      const v3 offset = ld3(scom + 3 * m.body_rootid[b]) - ld3(xanchor + 3 * j);
      if (t == JNT_FREE || t == JNT_BALL) {
        float xm[9];
        quat_to_mat(ldq(xquat + 4 * b), xm);
        if (t == JNT_FREE) {
          for (int k = 0; k < 18; k++) cdof[6 * dof + k] = 0.f;
          cdof[6 * dof + 3] = 1.f; cdof[6 * (dof + 1) + 4] = 1.f; cdof[6 * (dof + 2) + 5] = 1.f;
          dof += 3;
        }
        for (int k = 0; k < 3; k++) {
          v3 col = matcol(xm, k);
          st3(cdof + 6 * (dof + k), col); st3(cdof + 6 * (dof + k) + 3, cross(col, offset));
        }
      } else if (t == JNT_SLIDE) {
        st3(cdof + 6 * dof, mk3(0.f, 0.f, 0.f)); st3(cdof + 6 * dof + 3, ld3(xaxis + 3 * j));
      } else {
        v3 ax = ld3(xaxis + 3 * j);
        st3(cdof + 6 * dof, ax); st3(cdof + 6 * dof + 3, cross(ax, offset));
      }
    }
    st.store_fence();
    GSTORE(subtree_com, BLK(scom), 3 * nb); GSTORE(cinert, BLK(cinert), 10 * nb); GSTORE(cdof, BLK(cdof), 6 * nv);
    if (kin) GSTORE(ximat, BLK(arena), 9 * nb);
    st.store_commit();
  }
  __syncwarp();

  // ------------------------------------------------------------------ camlight (smooth.py:858-1027)
  if (mask & STG_CAMLIGHT) {
#pragma unroll 1
    for (int c = valid ? sub : m.ncam; c < m.ncam; c += LPW) {
      const int mode = m.cam_mode[c], b = m.cam_bodyid[c], tb = m.cam_targetbodyid[c];
      const bool is_target = mode == CAM_TARGETBODY || mode == CAM_TARGETBODYCOM;
      v3 p; float mat[9];
      if (mode == CAM_TRACK) {
        for (int k = 0; k < 9; k++) mat[k] = m.cam_mat0[9 * c + k];
        p = ld3(xpos + 3 * b) + ld3(m.cam_pos0 + 3 * c);
      } else if (mode == CAM_TRACKCOM) {
        for (int k = 0; k < 9; k++) mat[k] = m.cam_mat0[9 * c + k];
        p = ld3(scom + 3 * b) + ld3(m.cam_poscom0 + 3 * c);
      } else if (is_target && tb >= 0) {
        q4 q = ldq(xquat + 4 * b);
        p = ld3(xpos + 3 * b) + qrot(q, ld3(m.cam_pos + 3 * c));
        v3 tp = mode == CAM_TARGETBODYCOM ? ld3(scom + 3 * tb) : ld3(xpos + 3 * tb);
        v3 m3 = normalize(p - tp), m1 = normalize(cross(mk3(0.f, 0.f, 1.f), m3)), m2 = normalize(cross(m3, m1));
        mat[0] = m1.x; mat[1] = m2.x; mat[2] = m3.x; mat[3] = m1.y; mat[4] = m2.y; mat[5] = m3.y; mat[6] = m1.z; mat[7] = m2.z; mat[8] = m3.z;
      } else {
        q4 q = ldq(xquat + 4 * b);
        p = ld3(xpos + 3 * b) + qrot(q, ld3(m.cam_pos + 3 * c));
        quat_to_mat(qmul(q, ldq(m.cam_quat + 4 * c)), mat);
      }
      st3(d.cam_xpos + (wb * m.ncam + c) * 3, p);
      for (int k = 0; k < 9; k++) d.cam_xmat[(wb * m.ncam + c) * 9 + k] = mat[k];
    }
#pragma unroll 1
    for (int l = valid ? sub : m.nlight; l < m.nlight; l += LPW) {
      const int mode = m.light_mode[l], b = m.light_bodyid[l], tb = m.light_targetbodyid[l];
      const bool is_target = mode == CAM_TARGETBODY || mode == CAM_TARGETBODYCOM;
      v3 p, dir;
      bool norm = true;
      q4 q = ldq(xquat + 4 * b);
      if (is_target && tb < 0) {
        p = ld3(xpos + 3 * b) + qrot(q, ld3(m.light_pos + 3 * l)); dir = qrot(q, ld3(m.light_dir + 3 * l)); norm = false;
      } else if (mode == CAM_TRACK) {
        dir = ld3(m.light_dir0 + 3 * l); p = ld3(xpos + 3 * b) + ld3(m.light_pos0 + 3 * l);
      } else if (mode == CAM_TRACKCOM) {
        dir = ld3(m.light_dir0 + 3 * l); p = ld3(scom + 3 * b) + ld3(m.light_poscom0 + 3 * l);
      } else if (is_target) {
        p = ld3(xpos + 3 * b) + qrot(q, ld3(m.light_pos + 3 * l));
        v3 tp = mode == CAM_TARGETBODYCOM ? ld3(scom + 3 * tb) : ld3(xpos + 3 * tb);
        dir = tp - p;
      } else {
        p = ld3(xpos + 3 * b) + qrot(q, ld3(m.light_pos + 3 * l)); dir = qrot(q, ld3(m.light_dir + 3 * l));
      }
      if (norm) dir = normalize(dir);
      st3(d.light_xpos + (wb * m.nlight + l) * 3, p);
      st3(d.light_xdir + (wb * m.nlight + l) * 3, dir);
    }
  }


  // ------------------------------------------------------------------ kinematics: geom poses (from xipos on, once xipos .. ximat have been stored)
  if (kin) {
    st.store_wait_read();
#pragma unroll 2
    for (int gi = sub; gi < ng; gi += LPW) {
      const int b = m.geom_bodyid[gi];
      if (m.body_weldid[b] == 0 && (m.nmocap == 0 || m.body_mocapid[m.body_rootid[b]] == -1)) {  // static geom: keeps the pose computed at make_data (smooth.py:197-200)
        for (int k = 0; k < 3; k++) gxpos[3 * gi + k] = d.geom_xpos[(wb * ng + gi) * 3 + k];
        for (int k = 0; k < 9; k++) gxmat[9 * gi + k] = d.geom_xmat[(wb * ng + gi) * 9 + k];
      } else {
        q4 q = ldq(xquat + 4 * b);
        st3(gxpos + 3 * gi, ld3(xpos + 3 * b) + qrot(q, ld3(m.geom_pos + 3 * gi)));
        quat_to_mat(qmul(q, ldq(m.geom_quat + 4 * gi)), gxmat + 9 * gi);
      }
    }
    st.store_fence();
    GSTORE(geom_xpos, BLK(gxpos), 3 * ng); GSTORE(geom_xmat, BLK(gxmat), 9 * ng);
    st.store_commit();
  }

  // ------------------------------------------------------------------ crb + M (smooth.py:1029-1098)
  if (crbm) {
    st.store_wait_read();  // cinert has been stored: crb accumulates in place; the geom poses have been stored: xpos on (-> buf, M) is free
#pragma unroll 1
    for (int l = m.nlevel - 2; l >= 1; l--) {
#pragma unroll 1
      for (int i = m.level_adr[l] + sub; i < m.level_adr[l + 1]; i += LPW) {
        const int b = m.level_body[i];
        float acc[10];
#pragma unroll
        for (int k = 0; k < 10; k++) acc[k] = crb[10 * b + k];
#pragma unroll 1
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) {
          const float* cc = crb + 10 * m.body_childid[c];
#pragma unroll
          for (int k = 0; k < 10; k++) acc[k] += cc[k];
        }
#pragma unroll
        for (int k = 0; k < 10; k++) crb[10 * b + k] = acc[k];
      }
      __syncwarp();
    }
#pragma unroll 2
    for (int dd = sub; dd < nv; dd += LPW) inert_vec(crb + 10 * m.dof_bodyid[dd], cdof + 6 * dd, buf + 6 * dd);
    __syncwarp();
#pragma unroll 4
    for (int e = sub; e < m.nC; e += LPW) {
      const int i = m.M_entry_row[e], j = m.M_colind[e];
      float v = dot6(cdof + 6 * j, buf + 6 * i);
      if (i == j) v += m.dof_armature[i];
      Ms[e] = v;
    }
    st.store_fence();
    GSTORE(crb, BLK(cinert), 10 * nb); GSTORE(M, BLK(M), m.nC);
    st.store_commit();
  }
  st.store_wait_read();  // shared memory must outlive the bulk stores that read it
#undef GLOAD
#undef GSTORE
#undef BLK
#undef ROW
}

}  // namespace

static TeamKernel pos_kernel(const ModelDev& m, int lpw) {
  return m.batched ? k_position<32, true> : lpw == 8 ? k_position<8, false> : lpw == 16 ? k_position<16, false> : k_position<32, false>;
}

size_t smem_position(const ModelDev& m, const DataDev& d) { return team_shape(m, d.wn, pos_layout(m).total, pos_kernel).block_bytes; }
cudaError_t launch_position(const ModelDev& m, const DataDev& d, int mask, cudaStream_t s) { return team_launch(m, d, pos_layout(m).total, pos_kernel, mask, s); }
cudaError_t resident_worlds_position(const ModelDev& m, const DataDev& d, int* worlds, int* shape) {
  shape[3] = 0;
  return team_resident_worlds(m, d, pos_layout(m).total, pos_kernel, worlds, shape);
}
