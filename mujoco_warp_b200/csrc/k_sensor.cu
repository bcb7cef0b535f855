// k_sensor.cu -- sensors of one world by one warp.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): sensor.py:810 sensor_pos, :1432 sensor_vel, :2512 sensor_acc for the sensor
// types this build carries (joint / actuator / ball readings, gyro, velocimeter, accelerometer, subtree com / linvel / angmom, frame
// position and axes, clock; with EXTRA also magnetometer, camprojection, insidesite, tendon limit pos / vel / frc and tendonactfrc,
// mjb_sensor_extra.cuh), with their prerequisites smooth.py:3500-3612 subtree_vel (subtree linear velocity and angular momentum) and
// smooth.py:1743 rne_postconstraint (cfrc_ext from applied wrenches, body-to-body connect / weld equalities and contacts; cacc including
// qacc; cfrc_int accumulated up the tree), both shared with k_body_stages.cu (k_body_subtree_vel.cuh, k_body_rne_post.cuh).  Every input a position- or velocity-stage sensor reads is final once its stage has run, so one launch after
// the solver evaluates all three stages (the stage mask lets sensor_pos / sensor_vel / sensor_acc be called on their own).  EXTRA is
// chosen per model (ModelDev.sensor_extra), so a model without those sensor types runs the same code as before they existed.
#include "k_body_vec.cuh"
#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_ray.cuh"
#include "mjb_sensor_extra.cuh"
#include "mjb_types.cuh"

namespace {

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

template <bool BAT, bool EXTRA>
__global__ void __launch_bounds__(32)
k_sensor(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int stages) {
  extern __shared__ float smem[];  // nbody x (linvel 3 | angmom 3 | bodyvel lin 3) or nbody x (cfrc_ext 6 | cacc / cfrc_int 6)
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  const int nb = m.nbody, nv = m.nv;

  if ((stages & STAGE_VEL) && m.sensor_subtree_vel) {  // smooth.py:3500-3612
#include "k_body_subtree_vel.cuh"
  }

  if ((stages & STAGE_ACC) && m.sensor_rne_postconstraint) {  // smooth.py:1743 rne_postconstraint
#include "k_body_rne_post.cuh"
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
      default: {
        if (!EXTRA) continue;
        switch (t) {  // mjb_sensor_extra.cuh
          case SENS_MAGNETOMETER: { const v3 r = sensor_magnetometer(d.site_xmat + (wb * m.nsite + id) * 9, ld3(m.magnetic)); v[0] = r.x; v[1] = r.y; v[2] = r.z; break; }
          case SENS_CAMPROJECTION:
            sensor_camprojection(ld3(d.site_xpos + (wb * m.nsite + id) * 3), ld3(d.cam_xpos + (wb * m.ncam + rid) * 3), d.cam_xmat + (wb * m.ncam + rid) * 9, m.cam_fovy[rid],
                                 m.cam_intrinsic + 4 * rid, m.cam_sensorsize + 2 * rid, m.cam_resolution + 2 * rid, v);
            break;
          case SENS_INSIDESITE: {
            const int ot = m.sensor_objtype[s];
            const v3 p = sensor_inside_point(ot, id, obj_pos(d, m, wb, ot, id), d.subtree_com + (wb * nb + id) * 3, ot == OBJ_BODY ? m.body_mass[id] : 0.f,
                                             ot == OBJ_BODY ? m.body_subtreemass[id] : 0.f);
            v[0] = contact_inside_site(ld3(d.site_xpos + (wb * m.nsite + rid) * 3), d.site_xmat + (wb * m.nsite + rid) * 9, ld3(m.site_size + 3 * rid), m.site_type[rid], p) ? 1.f : 0.f;
            break; }
          case SENS_TENDONLIMITPOS: case SENS_TENDONLIMITVEL: case SENS_TENDONLIMITFRC: {  // sensor.py:228, :1028, :1640: the tendon's limit row, else 0
            const int e0 = d.ne[w] + d.nf[w], e1 = min(e0 + d.nl[w], d.njmax);
            for (int e = e0; e < e1; e++)
              if (d.efc_id[wb * d.njmax + e] == id && d.efc_type[wb * d.njmax + e] == CNSTR_LIMIT_TENDON)
                v[0] = t == SENS_TENDONLIMITPOS ? d.efc_pos[wb * d.njmax + e] - d.efc_margin[wb * d.njmax + e]
                                                : (t == SENS_TENDONLIMITVEL ? d.efc_vel[wb * d.njmax + e] : d.efc_force[wb * d.njmax + e]);
            break; }
          case SENS_TENDONACTFRC: v[0] = sensor_tendon_actfrc(m.nu, m.actuator_trntype, m.actuator_trnid, d.actuator_force + wb * m.nu, id); break;
          default: continue;
        }
      }
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
  // models with a magnetometer / camprojection / insidesite / tendon limit / tendonactfrc sensor run the EXTRA build; the others the
  // plain one, whose switch does not know those types
  const cudaError_t e = launch(m.sensor_extra ? (m.batched ? k_sensor<true, true> : k_sensor<false, true>) : (m.batched ? k_sensor<true, false> : k_sensor<false, false>),
                               d.wn, 32, (size_t)12 * m.nbody * sizeof(float), s, m, d, stages);
  // k_sensor skips the collision sensors: their slots are k_sensor_collision's
  if (e != cudaSuccess || !(stages & STAGE_POS) || c.nsensorcollision == 0 || (m.disableflags & DSBL_SENSOR)) return e;
  return launch_sensor_collision(m, d, c, s);
}
