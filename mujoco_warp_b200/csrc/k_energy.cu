// k_energy.cu -- potential and kinetic energy of one world by one warp.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): sensor.py:2773-3019 energy_pos (gravity over the bodies, joint springs and
// fixed-tendon springs) and energy_vel (1/2 qvel . M qvel through support.py:153 mul_m), and the e_potential / e_kinetic branches of
// _sensor_pos (sensor.py:747-752).  The reference accumulates with float atomics; here each lane sums its share of the bodies, joints
// and tendons in index order and the warp reduces by a fixed butterfly, so the result is bit-reproducible.  Polynomial stiffness is
// refused by put_model, so poly_potential (util_misc.py:727) reduces to 1/2 k x^2.
#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

namespace {

// |quat_sub(normalize(q), q_spring)| (math.py:161-186): the angle of the rotation from q_spring to q, as the length of its 3D velocity
__device__ __forceinline__ float quat_sub_length(const float* q, const float* q_spring) {
  const q4 rot = qnormalize(ldq(q)), ref = ldq(q_spring);
  const q4 qd = qmul(mkq(ref.w, -ref.x, -ref.y, -ref.z), rot);
  const v3 axis = mk3(qd.x, qd.y, qd.z);
  const float s2 = length(axis);
  if (s2 == 0.f) return 0.f;
  float speed = 2.0f * atan2f(s2, qd.w);
  if (speed > 3.14159265358979f) speed -= 2.0f * 3.14159265358979f;
  return length(axis * (speed / s2));
}

template <bool BAT>
__global__ void __launch_bounds__(32)
k_energy(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const __grid_constant__ EnergyDev e, int parts) {
  extern __shared__ float v[];  // the world's qvel (kinetic term)
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld || w >= d.w0 + d.wn) return;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  float pot = 0.f, kin = 0.f;
  if (parts & ENERGY_POT) {
    float grav = 0.f, spring = 0.f;
    if (!(m.disableflags & DSBL_GRAVITY)) {  // -sum_b mass_b gravity . xipos_b over the bodies after the world body
      const v3 g = mk3(m.gravity_x, m.gravity_y, m.gravity_z);
      for (int b = 1 + lane; b < m.nbody; b += 32) grav += m.body_mass[b] * dot(g, ld3(d.xipos + (wb * m.nbody + b) * 3));
    }
    if (!(m.disableflags & DSBL_SPRING)) {
      const float* qpos = d.qpos + wb * m.nq;
      for (int j = lane; j < m.njnt; j += 32) {  // sensor.py:2806-2897
        const float k = m.jnt_stiffness[j];
        if (k == 0.f) continue;
        const int qa = m.jnt_qposadr[j], t = m.jnt_type[j];
        if (t == JNT_FREE) {
          const float r0 = length(ld3(qpos + qa) - ld3(m.qpos_spring + qa)), r1 = quat_sub_length(qpos + qa + 3, m.qpos_spring + qa + 3);
          spring += 0.5f * k * r0 * r0 + 0.5f * k * r1 * r1;
        } else if (t == JNT_BALL) {
          const float r = quat_sub_length(qpos + qa, m.qpos_spring + qa);
          spring += 0.5f * k * r * r;
        } else {
          const float x = qpos[qa] - m.qpos_spring[qa];
          spring += 0.5f * k * x * x;
        }
      }
      for (int t = lane; t < m.ntendon; t += 32) {  // sensor.py:2900-2938: the length outside the dead band [lower, upper]
        const float k = m.tendon_stiffness[t];
        if (k == 0.f) continue;
        const float len = d.ten_length[wb * m.ntendon + t], lo = m.tendon_lengthspring[2 * t], hi = m.tendon_lengthspring[2 * t + 1];
        const float x = len > hi ? len - hi : (len < lo ? len - lo : 0.f);
        spring += 0.5f * k * x * x;
      }
    }
    pot = warp_sum(spring) - warp_sum(grav);
  }
  if (parts & ENERGY_KIN) {  // 1/2 qvel . (M qvel), M with armature as crb left it
    warp_copy(v, d.qvel + wb * m.nv, m.nv, lane);
    __syncwarp();
    const float* M = d.M + wb * m.nC;
    float q = 0.f;
    for (int i = lane; i < m.nv; i += 32) q += v[i] * mul_m_row(m, M, v, i);
    kin = 0.5f * warp_sum(q);
  }
  if (parts & ENERGY_SENSOR) {  // sensor.py:747-752, cutoff as for every REAL sensor (:56-113)
    float* out = d.sensordata + wb * m.nsensordata;
    for (int i = lane; i < e.nsensor_energy; i += 32) {
      const int s = e.sensor_energy_adr[i];
      const float c = m.sensor_cutoff[s];
      float x = m.sensor_type[s] == SENS_E_POTENTIAL ? pot : kin;
      if (c > 0.f) x = fminf(fmaxf(x, -c), c);
      out[m.sensor_adr[s]] = x;
    }
  }
  if (lane == 0) {
    float* en = e.energy + 2 * wb;
    if (parts & ENERGY_ZERO) { en[0] = 0.f; en[1] = 0.f; }
    else {
      if (parts & ENERGY_POT) en[0] = pot;
      if (parts & ENERGY_KIN) en[1] = kin;
    }
  }
}

}  // namespace

cudaError_t launch_energy(const ModelDev& m, const DataDev& d, const EnergyDev& e, int parts, cudaStream_t s) {
  if (parts == 0) return cudaSuccess;
  return launch(m.batched ? k_energy<true> : k_energy<false>, d.wn, 32, (m.nv + 4) * sizeof(float), s, m, d, e, parts);
}
