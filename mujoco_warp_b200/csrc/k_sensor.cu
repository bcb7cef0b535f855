// k_sensor.cu -- sensors of one world by one warp.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): sensor.py:810 sensor_pos, :1432 sensor_vel, :2512 sensor_acc for the sensor
// types this build carries (joint / actuator / ball readings, gyro, velocimeter, accelerometer, subtree com / linvel / angmom, frame
// position and axes, clock), with their prerequisites smooth.py:3500-3612 subtree_vel (subtree linear velocity and angular momentum) and
// smooth.py:1743 rne_postconstraint (cfrc_ext from applied wrenches, body-to-body connect / weld equalities and contacts; cacc including
// qacc; cfrc_int accumulated up the tree).  Every input a position- or velocity-stage sensor reads is final once its stage has run, so one launch after
// the solver evaluates all three stages (the stage mask lets sensor_pos / sensor_vel / sensor_acc be called on their own).
#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_ray.cuh"
#include "mjb_types.cuh"

namespace {

__device__ __forceinline__ float comp3(v3 v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : v.z); }
__device__ __forceinline__ v3 mat_t_vec(const float* m, v3 v) {  // m^T v
  return mk3(m[0] * v.x + m[3] * v.y + m[6] * v.z, m[1] * v.x + m[4] * v.y + m[7] * v.z, m[2] * v.x + m[5] * v.y + m[8] * v.z);
}

enum { STAGE_POS = 1, STAGE_VEL = 2, STAGE_ACC = 4 };

__device__ __forceinline__ const float* obj_pos(const DataDev& d, const ModelDev& m, size_t wb, int objtype, int id) {
  switch (objtype) {
    case OBJ_BODY: return d.xipos + (wb * m.nbody + id) * 3;
    case OBJ_XBODY: return d.xpos + (wb * m.nbody + id) * 3;
    case OBJ_GEOM: return d.geom_xpos + (wb * m.ngeom + id) * 3;
    case OBJ_SITE: return d.site_xpos + (wb * m.nsite + id) * 3;
    default: return d.cam_xpos + (wb * m.ncam + id) * 3;
  }
}
__device__ __forceinline__ const float* obj_mat(const DataDev& d, const ModelDev& m, size_t wb, int objtype, int id) {
  switch (objtype) {
    case OBJ_BODY: return d.ximat + (wb * m.nbody + id) * 9;
    case OBJ_XBODY: return d.xmat + (wb * m.nbody + id) * 9;
    case OBJ_GEOM: return d.geom_xmat + (wb * m.ngeom + id) * 9;
    case OBJ_SITE: return d.site_xmat + (wb * m.nsite + id) * 9;
    default: return d.cam_xmat + (wb * m.ncam + id) * 9;
  }
}

__device__ __forceinline__ int obj_body(const ModelDev& m, int objtype, int id) {  // sensor.py:1066 / :320
  switch (objtype) {
    case OBJ_BODY: case OBJ_XBODY: return id;
    case OBJ_GEOM: return m.geom_bodyid[id];
    case OBJ_SITE: return m.site_bodyid[id];
    case OBJ_CAMERA: return m.cam_bodyid[id];
    default: return 0;
  }
}

template <bool BAT>
__global__ void __launch_bounds__(32)
k_sensor(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int stages) {
  extern __shared__ float smem[];  // nbody x (linvel 3 | angmom 3 | bodyvel lin 3) or nbody x (cfrc_ext 6 | cacc / cfrc_int 6)
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  const int nb = m.nbody, nv = m.nv;

  if ((stages & STAGE_VEL) && m.sensor_subtree_vel) {  // smooth.py:3500-3612
    float *linvel = smem, *angmom = smem + 3 * nb, *blin = smem + 6 * nb;
    for (int b = lane; b < nb; b += 32) {
      const float* cv = d.cvel + (wb * nb + b) * 6;
      const float* ximat = d.ximat + (wb * nb + b) * 9;
      const v3 ang = ld3(cv), dif = ld3(d.xipos + (wb * nb + b) * 3) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
      const v3 lin = ld3(cv + 3) - cross(dif, ang);
      st3(linvel + 3 * b, lin * m.body_mass[b]);
      v3 dv = mat_t_vec(ximat, ang);
      dv.x *= m.body_inertia[3 * b]; dv.y *= m.body_inertia[3 * b + 1]; dv.z *= m.body_inertia[3 * b + 2];
      st3(angmom + 3 * b, matvec(ximat, dv));
      st3(blin + 3 * b, lin);
    }
    __syncwarp();
    // _linear_momentum: children into parents, deepest level first (fixed child order: no float atomics), then divide by the subtree mass
    for (int lv = m.nlevel - 1; lv >= 0; lv--) {
      for (int i = m.level_adr[lv] + lane; i < m.level_adr[lv + 1]; i += 32) {
        const int b = m.level_body[i];
        v3 s = ld3(linvel + 3 * b);
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) { const int ch = m.body_childid[c]; s = s + ld3(linvel + 3 * ch) * m.body_subtreemass[ch]; }
        st3(linvel + 3 * b, s * (1.0f / fmaxf(MJ_MINVAL, m.body_subtreemass[b])));
      }
      __syncwarp();
    }
    // _angular_momentum: a body's own term, then its (finished) subtree momentum and the orbital term go to the parent
    for (int b = lane; b < nb; b += 32) {
      if (b == 0) continue;
      const v3 dx = ld3(d.xipos + (wb * nb + b) * 3) - ld3(d.subtree_com + (wb * nb + b) * 3);
      const v3 dp = (ld3(blin + 3 * b) - ld3(linvel + 3 * b)) * m.body_mass[b];
      st3(angmom + 3 * b, ld3(angmom + 3 * b) + cross(dx, dp));
    }
    __syncwarp();
    for (int lv = m.nlevel - 1; lv >= 0; lv--) {
      for (int i = m.level_adr[lv] + lane; i < m.level_adr[lv + 1]; i += 32) {
        const int b = m.level_body[i];
        v3 s = ld3(angmom + 3 * b);
        const v3 com = ld3(d.subtree_com + (wb * nb + b) * 3), lv_b = ld3(linvel + 3 * b);
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) {
          const int ch = m.body_childid[c];
          const v3 dx = ld3(d.subtree_com + (wb * nb + ch) * 3) - com, dv = (ld3(linvel + 3 * ch) - lv_b) * m.body_subtreemass[ch];
          s = s + ld3(angmom + 3 * ch) + cross(dx, dv);
        }
        st3(angmom + 3 * b, s);
      }
      __syncwarp();
    }
    for (int i = lane; i < 3 * nb; i += 32) { d.subtree_linvel[wb * 3 * nb + i] = linvel[i]; d.subtree_angmom[wb * 3 * nb + i] = angmom[i]; }
    __syncwarp();
  }

  if ((stages & STAGE_ACC) && m.sensor_rne_postconstraint) {  // smooth.py:1743 rne_postconstraint
    float *cext = smem, *cacc = smem + 6 * nb;  // cfrc_int later reuses the cacc rows
    // cfrc_ext: applied wrenches (:1518) ...
    for (int b = lane; b < nb; b += 32) {
      float o[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (b) {
        const float* x = d.xfrc_applied + (wb * nb + b) * 6;
        const v3 off = ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3) - ld3(d.xipos + (wb * nb + b) * 3);
        const v3 f = ld3(x), t = ld3(x + 3) - cross(off, f);
        o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = f.x; o[4] = f.y; o[5] = f.z;
      }
      for (int k = 0; k < 6; k++) cext[6 * b + k] = o[k];
    }
    __syncwarp();
    // ... connect / weld equalities between bodies (:1562; rows are ordered connect, weld, joint) and contacts (:1660), one after the
    // other in row / pool order so that the sums are reproducible; lanes 0-5 own the six components
    const float* force = d.efc_force + wb * d.njmax;
#pragma unroll 1
    for (int e = 0; e < d.ne[w];) {
      const int id = d.efc_id[wb * d.njmax + e], type = m.eq_type[id];
      if (type != EQ_CONNECT && type != EQ_WELD) break;
      const int nrow = type == EQ_CONNECT ? 3 : 6, b1 = m.eq_obj1id[id], b2 = m.eq_obj2id[id];
      const v3 f = mk3(force[e], force[e + 1], force[e + 2]);
      const v3 tq = type == EQ_WELD ? mk3(force[e + 3], force[e + 4], force[e + 5]) : mk3(0.f, 0.f, 0.f);
      const float* data = m.eq_data + 11 * id;
      for (int side = 0; side < 2; side++) {
        const int b = side ? b2 : b1;
        if (!b) continue;
        const v3 anchor = ld3(data + (((type == EQ_CONNECT) == (side == 0)) ? 0 : 3));
        const v3 pos = matvec(d.xmat + (wb * nb + b) * 9, anchor) + ld3(d.xpos + (wb * nb + b) * 3);
        const v3 dif = ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3) - pos, t = tq - cross(dif, f);
        if (lane < 6) { const float c = lane < 3 ? comp3(t, lane) : comp3(f, lane - 3); cext[6 * b + lane] += side ? -c : c; }
      }
      __syncwarp();
      e += nrow;
    }
    const int c0 = d.world_conadr[w], c1 = c0 + d.world_ncon[w];  // already clamped by k_collision to the per-world cap and the pool
#pragma unroll 1
    for (int c = c0; c < c1; c++) {
      const int id1 = m.geom_bodyid[d.contact_geom[2 * c]], id2 = m.geom_bodyid[d.contact_geom[2 * c + 1]];
      if (id1 == 0 && id2 == 0) continue;
      float fc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // support.py:326-397 contact_force_fn
      const int dim = d.contact_dim[c];
      const int* adr = d.contact_efc_address + (size_t)c * m.nmaxpyramid;
      if (adr[0] >= 0) {
        if (m.cone == CONE_PYRAMIDAL) {
          if (dim == 1) fc[0] = adr[0] < d.njmax ? force[adr[0]] : 0.f;
          else
            for (int i = 0; i < dim - 1; i++) {
              const int a = 2 * i + adr[0];
              const float d1 = a < d.njmax ? force[a] : 0.f, d2 = a + 1 < d.njmax ? force[a + 1] : 0.f;
              fc[0] += d1 + d2; fc[i + 1] = (d1 - d2) * d.contact_friction[5 * (size_t)c + i];
            }
        } else {
          for (int i = 0; i < dim; i++) if (adr[i] >= 0 && adr[i] < d.njmax) fc[i] = force[adr[i]];
        }
      }
      const float* R = d.contact_frame + 9 * (size_t)c;
      const v3 fw = mk3(fc[0] * R[0] + fc[1] * R[3] + fc[2] * R[6], fc[0] * R[1] + fc[1] * R[4] + fc[2] * R[7], fc[0] * R[2] + fc[1] * R[5] + fc[2] * R[8]);
      const v3 tw = mk3(fc[3] * R[0] + fc[4] * R[3] + fc[5] * R[6], fc[3] * R[1] + fc[4] * R[4] + fc[5] * R[7], fc[3] * R[2] + fc[4] * R[5] + fc[5] * R[8]);
      const v3 pos = ld3(d.contact_pos + 3 * (size_t)c);
      for (int side = 0; side < 2; side++) {
        const int b = side ? id2 : id1;
        if (!b) continue;
        const v3 off = ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3) - pos, t = tw - cross(off, fw);
        if (lane < 6) { const float cc = lane < 3 ? comp3(t, lane) : comp3(fw, lane - 3); cext[6 * b + lane] += side ? cc : -cc; }
      }
      __syncwarp();
    }
    // cacc including qacc (:1364-1425 with flg_acc)
    if (lane < 6) cacc[lane] = (lane >= 3 && !(m.disableflags & DSBL_GRAVITY)) ? -(lane == 3 ? m.gravity_x : (lane == 4 ? m.gravity_y : m.gravity_z)) : 0.f;
    __syncwarp();
    for (int lv = 1; lv < m.nlevel; lv++) {
      for (int i = m.level_adr[lv] + lane; i < m.level_adr[lv + 1]; i += 32) {
        const int b = m.level_body[i], pid = m.body_parentid[b];
        float a[6];
        for (int k = 0; k < 6; k++) a[k] = cacc[6 * pid + k];
        for (int j = 0; j < m.body_dofnum[b]; j++) {
          const int dof = m.body_dofadr[b] + j;
          const float qv = d.qvel[wb * nv + dof], qa = d.qacc[wb * nv + dof];
          const float *cd = d.cdof + (wb * nv + dof) * 6, *cdd = d.cdof_dot + (wb * nv + dof) * 6;
          for (int k = 0; k < 6; k++) { a[k] += cdd[k] * qv; a[k] += cd[k] * qa; }
        }
        for (int k = 0; k < 6; k++) cacc[6 * b + k] = a[k];
      }
      __syncwarp();
    }
    for (int i = lane; i < 6 * nb; i += 32) { d.cacc[wb * 6 * nb + i] = cacc[i]; d.cfrc_ext[wb * 6 * nb + i] = cext[i]; }
    __syncwarp();
    // cfrc_int = I cacc + cvel x* (I cvel) - cfrc_ext (:1428), then children into parents, deepest level first (:1453)
    float* cint = cacc;
    for (int b = lane; b < nb; b += 32) {
      float o[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (b) {
        float f[6], iv[6], g[6];
        const float *ci = d.cinert + (wb * nb + b) * 10, *cv = d.cvel + (wb * nb + b) * 6;
        inert_vec(ci, cacc + 6 * b, f); inert_vec(ci, cv, iv); motion_cross_force(cv, iv, g);
        for (int k = 0; k < 6; k++) o[k] = f[k] + g[k] - cext[6 * b + k];
      }
      // (a lane only reads and then overwrites its own body's row)
      for (int k = 0; k < 6; k++) cint[6 * b + k] = o[k];
    }
    __syncwarp();
    for (int lv = m.nlevel - 2; lv >= 0; lv--) {
      for (int i = m.level_adr[lv] + lane; i < m.level_adr[lv + 1]; i += 32) {
        const int b = m.level_body[i];
        float a[6];
        for (int k = 0; k < 6; k++) a[k] = cint[6 * b + k];
        for (int c = m.body_childadr[b]; c < m.body_childadr[b + 1]; c++) { const int ch = m.body_childid[c]; for (int k = 0; k < 6; k++) a[k] += cint[6 * ch + k]; }
        for (int k = 0; k < 6; k++) cint[6 * b + k] = a[k];
      }
      __syncwarp();
    }
    for (int i = lane; i < 6 * nb; i += 32) d.cfrc_int[wb * 6 * nb + i] = cint[i];
    __syncwarp();
  }

  if (m.disableflags & DSBL_SENSOR) return;
  float* out = d.sensordata + wb * m.nsensordata;
  for (int s = lane; s < m.nsensor; s += 32) {
    const int st = m.sensor_needstage[s];
    if (!(stages & (st == 1 ? STAGE_POS : (st == 2 ? STAGE_VEL : STAGE_ACC)))) continue;
    const int t = m.sensor_type[s], id = m.sensor_objid[s], rt = m.sensor_reftype[s], rid = m.sensor_refid[s];  // rid = -1: world frame
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    switch (t) {
      case SENS_JOINTPOS: v[0] = d.qpos[wb * m.nq + m.jnt_qposadr[id]]; break;
      case SENS_TENDONPOS: v[0] = d.ten_length[wb * m.ntendon + id]; break;
      case SENS_ACTUATORPOS: v[0] = d.actuator_length[wb * m.nu + id]; break;
      case SENS_BALLQUAT: { const q4 q = qnormalize(ldq(d.qpos + wb * m.nq + m.jnt_qposadr[id])); v[0] = q.w; v[1] = q.x; v[2] = q.y; v[3] = q.z; break; }
      case SENS_FRAMEPOS: {  // sensor.py:377
        v3 r = ld3(obj_pos(d, m, wb, m.sensor_objtype[s], id));
        if (rid > -1) r = mat_t_vec(obj_mat(d, m, wb, rt, rid), r - ld3(obj_pos(d, m, wb, rt, rid)));
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_FRAMEXAXIS: case SENS_FRAMEYAXIS: case SENS_FRAMEZAXIS: {
        const float* R = obj_mat(d, m, wb, m.sensor_objtype[s], id); const int c = t - SENS_FRAMEXAXIS;
        v3 r = mk3(R[c], R[3 + c], R[6 + c]);
        if (rid > -1) r = mat_t_vec(obj_mat(d, m, wb, rt, rid), r);  // sensor.py:406
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_FRAMEQUAT: {  // sensor.py:342-374 _get_quat
        const int ot = m.sensor_objtype[s];
        const float* local = ot == OBJ_BODY ? m.body_iquat + 4 * id : ot == OBJ_GEOM ? m.geom_quat + 4 * id : ot == OBJ_SITE ? m.site_quat + 4 * id : ot == OBJ_CAMERA ? m.cam_quat + 4 * id : nullptr;
        q4 q = ldq(d.xquat + (wb * nb + obj_body(m, ot, id)) * 4);
        if (local) q = qmul(q, ldq(local));
        if (rid > -1) {  // sensor.py:470-482: conj(refquat) * quat
          const float* rl = rt == OBJ_BODY ? m.body_iquat + 4 * rid : rt == OBJ_GEOM ? m.geom_quat + 4 * rid : rt == OBJ_SITE ? m.site_quat + 4 * rid : rt == OBJ_CAMERA ? m.cam_quat + 4 * rid : nullptr;
          q4 rq = ldq(d.xquat + (wb * nb + obj_body(m, rt, rid)) * 4);
          if (rl) rq = qmul(rq, ldq(rl));
          q = qmul(mkq(rq.w, -rq.x, -rq.y, -rq.z), q);
        }
        v[0] = q.w; v[1] = q.x; v[2] = q.y; v[3] = q.z; break; }
      case SENS_SUBTREECOM: { const float* p = d.subtree_com + (wb * nb + id) * 3; v[0] = p[0]; v[1] = p[1]; v[2] = p[2]; break; }
      case SENS_CLOCK: v[0] = d.time[w]; break;
      case SENS_JOINTLIMITPOS: case SENS_JOINTLIMITVEL: case SENS_JOINTLIMITFRC: {  // sensor.py:228, :1028, :1640: the joint's active limit row, else 0
        const int e0 = d.ne[w] + d.nf[w], e1 = min(e0 + d.nl[w], d.njmax);
        for (int e = e0; e < e1; e++)
          if (d.efc_id[wb * d.njmax + e] == id && d.efc_type[wb * d.njmax + e] == CNSTR_LIMIT_JOINT)
            v[0] = t == SENS_JOINTLIMITPOS ? d.efc_pos[wb * d.njmax + e] - d.efc_margin[wb * d.njmax + e]
                                           : (t == SENS_JOINTLIMITVEL ? d.efc_vel[wb * d.njmax + e] : d.efc_force[wb * d.njmax + e]);
        break; }
      case SENS_JOINTVEL: v[0] = d.qvel[wb * nv + m.jnt_dofadr[id]]; break;
      case SENS_TENDONVEL: v[0] = d.ten_velocity[wb * m.ntendon + id]; break;
      case SENS_ACTUATORVEL: v[0] = d.actuator_velocity[wb * m.nu + id]; break;
      case SENS_BALLANGVEL: { const float* p = d.qvel + wb * nv + m.jnt_dofadr[id]; v[0] = p[0]; v[1] = p[1]; v[2] = p[2]; break; }
      case SENS_FRAMELINVEL: case SENS_FRAMEANGVEL: {  // sensor.py:1108-1293 without a reference frame
        const int ot = m.sensor_objtype[s], b = obj_body(m, ot, id);
        const float* cv = d.cvel + (wb * nb + b) * 6;
        const v3 ang = ld3(cv), pos = ld3(obj_pos(d, m, wb, ot, id));
        const v3 lin = ld3(cv + 3) - cross(pos - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3), ang);
        v3 r = t == SENS_FRAMELINVEL ? lin : ang;
        if (rid > -1) {  // sensor.py:1188-1210, :1255-1291: relative to, and expressed in, the reference frame
          const int rb = obj_body(m, rt, rid);
          const float* rv = d.cvel + (wb * nb + rb) * 6;
          const v3 rang = ld3(rv), rpos = ld3(obj_pos(d, m, wb, rt, rid));
          const v3 rlin = ld3(rv + 3) - cross(rpos - ld3(d.subtree_com + (wb * nb + m.body_rootid[rb]) * 3), rang);
          const v3 rel = t == SENS_FRAMELINVEL ? lin - rlin + cross(pos - rpos, rang) : ang - rang;
          r = mat_t_vec(obj_mat(d, m, wb, rt, rid), rel);
        }
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_SUBTREELINVEL: { const float* p = d.subtree_linvel + (wb * nb + id) * 3; v[0] = p[0]; v[1] = p[1]; v[2] = p[2]; break; }
      case SENS_SUBTREEANGMOM: { const float* p = d.subtree_angmom + (wb * nb + id) * 3; v[0] = p[0]; v[1] = p[1]; v[2] = p[2]; break; }
      case SENS_GYRO: {  // sensor.py:989
        const v3 r = mat_t_vec(d.site_xmat + (wb * m.nsite + id) * 9, ld3(d.cvel + (wb * nb + m.site_bodyid[id]) * 6));
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_VELOCIMETER: {  // sensor.py:964
        const int b = m.site_bodyid[id];
        const float* cv = d.cvel + (wb * nb + b) * 6;
        const v3 dif = ld3(d.site_xpos + (wb * m.nsite + id) * 3) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
        const v3 r = mat_t_vec(d.site_xmat + (wb * m.nsite + id) * 9, ld3(cv + 3) - cross(dif, ld3(cv)));
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_ACCELEROMETER: {  // sensor.py:1510
        const int b = m.site_bodyid[id];
        const float *cv = d.cvel + (wb * nb + b) * 6, *ca = d.cacc + (wb * nb + b) * 6, *R = d.site_xmat + (wb * m.nsite + id) * 9;
        const v3 dif = ld3(d.site_xpos + (wb * m.nsite + id) * 3) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
        const v3 ang = mat_t_vec(R, ld3(cv)), lin = mat_t_vec(R, ld3(cv + 3) - cross(dif, ld3(cv)));
        const v3 acc = mat_t_vec(R, ld3(ca + 3) - cross(dif, ld3(ca))), r = acc + cross(ang, lin);
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_FRAMELINACC: case SENS_FRAMEANGACC: {  // sensor.py:1678-1753
        const int ot = m.sensor_objtype[s], b = obj_body(m, ot, id);
        const float *cv = d.cvel + (wb * nb + b) * 6, *ca = d.cacc + (wb * nb + b) * 6;
        v3 r = ld3(ca);
        if (t == SENS_FRAMELINACC) {
          const v3 off = ld3(obj_pos(d, m, wb, ot, id)) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
          const v3 ang = ld3(cv), lin = ld3(cv + 3) - cross(off, ang);
          r = ld3(ca + 3) - cross(off, r) + cross(ang, lin);
        }
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_TOUCH: {  // sensor.py:2063: normal forces of the sensorised body's contacts whose force ray meets the site volume
        const int body = m.site_bodyid[id];
        const float* force = d.efc_force + wb * d.njmax;
        const int c0 = d.world_conadr[w], c1 = c0 + d.world_ncon[w];  // already clamped by k_collision to the per-world cap and the pool
        float total = 0.f;
        for (int c = c0; c < c1; c++) {
          const int b1 = m.geom_bodyid[d.contact_geom[2 * c]], b2 = m.geom_bodyid[d.contact_geom[2 * c + 1]];
          const int* adr = d.contact_efc_address + (size_t)c * m.nmaxpyramid;
          if (adr[0] < 0 || (body != b1 && body != b2)) continue;
          float nf = adr[0] < d.njmax ? force[adr[0]] : 0.f;  // rows cut by njmax carry address -1 (k_constraint)
          if (m.cone == CONE_PYRAMIDAL) for (int i = 1; i < 2 * (d.contact_dim[c] - 1); i++) nf += (adr[i] >= 0 && adr[i] < d.njmax) ? force[adr[i]] : 0.f;
          if (nf <= 0.f) continue;
          v3 ray = normalize(ld3(d.contact_frame + 9 * (size_t)c) * nf);
          if (body == b2) ray = ray * -1.0f;
          if (ray_geom<false>(ld3(d.site_xpos + (wb * m.nsite + id) * 3), d.site_xmat + (wb * m.nsite + id) * 9, ld3(m.site_size + 3 * id),
                              ld3(d.contact_pos + 3 * (size_t)c), ray, m.site_type[id], nullptr) >= 0.f) total += nf;
        }
        v[0] = total; break; }
      case SENS_FORCE: {  // sensor.py:1542
        const v3 r = mat_t_vec(d.site_xmat + (wb * m.nsite + id) * 9, ld3(d.cfrc_int + (wb * nb + m.site_bodyid[id]) * 6 + 3));
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_TORQUE: {  // sensor.py:1559
        const int b = m.site_bodyid[id];
        const float* cf = d.cfrc_int + (wb * nb + b) * 6;
        const v3 dif = ld3(d.site_xpos + (wb * m.nsite + id) * 3) - ld3(d.subtree_com + (wb * nb + m.body_rootid[b]) * 3);
        const v3 r = mat_t_vec(d.site_xmat + (wb * m.nsite + id) * 9, ld3(cf) - cross(dif, ld3(cf + 3)));
        v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
      case SENS_ACTUATORFRC: v[0] = d.actuator_force[wb * m.nu + id]; break;
      case SENS_JOINTACTFRC: v[0] = d.qfrc_actuator[wb * nv + m.jnt_dofadr[id]]; break;
      default: continue;
    }
    // sensor.py:56-113: cutoff clamps REAL data to [-c, c] and POSITIVE data from above
    const float cutoff = m.sensor_cutoff[s];
    const int dt = m.sensor_datatype[s], adr = m.sensor_adr[s];
    for (int k = 0; k < m.sensor_dim[s]; k++) {
      float x = v[k];
      if (cutoff > 0.f) { if (dt == 0) x = fminf(fmaxf(x, -cutoff), cutoff); else if (dt == 1) x = fminf(x, cutoff); }
      out[adr + k] = x;
    }
  }
}

}  // namespace

cudaError_t launch_sensor(const ModelDev& m, const DataDev& d, int stages, cudaStream_t s, const SensorCollisionDev& c) {
  if (m.nsensor == 0) return cudaSuccess;
  const cudaError_t e = launch(m.batched ? k_sensor<true> : k_sensor<false>, d.wn, 32, (size_t)12 * m.nbody * sizeof(float), s, m, d, stages);
  // k_sensor skips the collision sensors: their slots are k_sensor_collision's
  if (e != cudaSuccess || !(stages & STAGE_POS) || c.nsensorcollision == 0 || (m.disableflags & DSBL_SENSOR)) return e;
  return launch_sensor_collision(m, d, c, s);
}
