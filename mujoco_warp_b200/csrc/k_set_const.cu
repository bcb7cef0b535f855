// k_set_const.cu -- recomputes the Model constants the compiler derives from other Model fields, per world.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): set_const.py:613 set_const_fixed, :634 set_const_0, :847 set_const_spring,
// :952 set_length_range.
// The reference runs one solve_m launch (plus helpers) per dof, per body x 6 Jacobian rows, per tendon and per actuator.  Here one
// warp per world solves all of these right-hand sides against the factor the world already holds (Data.qLD, per-tree dense upper U
// with M = U^T U, k_support.cu): U is staged in shared memory once, the lanes take one right-hand side each, so every factor read is
// a shared-memory broadcast, and the launch count does not depend on the model's sizes.
//
// Batched outputs: entry i of a derived field is computed from world i, for i below that field's leading size (the reference's
// `worldid % shape[0]`, made deterministic): world w writes entry w of a field only when w < nb of that field.  Inputs are read as
// every kernel reads them (world_model: entry w % nb).
#include "mjb_launch.cuh"
#include "mjb_math.cuh"

namespace {

// ---------------------------------------------------------------- set_const_fixed (set_const.py:35-57, 613-631)
// body_subtreemass of world w < nw: body_mass accumulated up the tree, children before parents (bodies are in topological order).
__global__ void k_set_const_fixed(const __grid_constant__ ModelDev mp, int nw, int nworld) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nw) return;
  const ModelDev m = world_model(mp, w, nworld);
  float* sub = const_cast<float*>(m.body_subtreemass);
  for (int b = 0; b < m.nbody; b++) sub[b] = m.body_mass[b];
  for (int b = m.nbody - 1; b > 0; b--) sub[m.body_parentid[b]] += sub[b];
}

// ---------------------------------------------------------------- set_length_range (set_const.py:573-607, 952-985)
// One thread per (world, actuator) of worlds [0, nw): the range of a limited joint or fixed tendon times gear[0] (ends swapped for a
// negative gear), (0, 0) for any other transmission.  Every actuator is written, muscle or not, as the reference does.
__global__ void k_set_length_range(const __grid_constant__ ModelDev mp, int nw, int nworld) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nw * mp.nu) return;
  const int w = i / mp.nu, a = i - w * mp.nu;
  const ModelDev m = world_model(mp, w, nworld);
  const int trn = m.actuator_trntype[a], id = m.actuator_trnid[2 * a];
  const float gear = m.actuator_gear[6 * a];
  const float* rng = nullptr;
  if (trn == TRN_JOINT && m.jnt_limited[id]) rng = m.jnt_range + 2 * id;
  else if (trn == TRN_TENDON && m.ntendon > 0 && m.tendon_limited[id]) rng = m.tendon_range + 2 * id;
  float lo = 0.f, hi = 0.f;
  if (rng) {
    if (gear > 0.f) { lo = rng[0] * gear; hi = rng[1] * gear; }
    else { lo = rng[1] * gear; hi = rng[0] * gear; }
  }
  float* out = const_cast<float*>(m.actuator_lengthrange) + 2 * a;
  out[0] = lo;
  out[1] = hi;
}

// ---------------------------------------------------------------- qpos swap (set_const.py:59-66, 656-658, 833)
// One thread per (world, qpos entry) of worlds [0, nw); the SAVE modes copy the state to the save buffer first.
__global__ void k_set_const_qpos(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, const SetConstDev c, int mode, int nw) {
  float* __restrict__ save = c.qpos_save;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nw * m.nq) return;
  const int w = i / m.nq, q = i - w * m.nq;
  if (mode == QPOS_RESTORE) { d.qpos[i] = save[i]; return; }
  if (mode != QPOS_LOADSPRING) save[i] = d.qpos[i];
  const bool spring = mode != QPOS_SAVE_LOAD0;
  const float* src = spring ? m.qpos_spring : m.qpos0;
  const int nb = spring ? m.nb_qpos_spring : m.nb_qpos0, bs = spring ? m.bs_qpos_spring : m.bs_qpos0;
  d.qpos[i] = src[(nb > 1 ? (size_t)(w % nb) * bs : 0) + q];
}

// ---------------------------------------------------------------- set_const_spring (set_const.py:156-166)
__global__ void k_set_const_spring(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int nw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nw * mp.ntendon) return;
  const int w = i / mp.ntendon, t = i - w * mp.ntendon;
  const ModelDev m = world_model(mp, w, d.nworld);
  float* ls = const_cast<float*>(m.tendon_lengthspring) + 2 * t;
  if (ls[0] == -1.f && ls[1] == -1.f) {
    const float l = d.ten_length[(size_t)w * m.ntendon + t];
    ls[0] = l;
    ls[1] = l;
  }
}

// ---------------------------------------------------------------- set_const_0 (set_const.py:169-570, 670-831)
// Shared memory of one world, in floats: U (qld_total), the lanes' right-hand sides and solutions, lane-interleaved (2 x 32 nv:
// entry i of lane l at i * 32 + l, so the lanes hit distinct banks), diag(M^-1) (nv) and the body Jacobians' diagonals (6 nbody).
__host__ __device__ inline size_t set_const_words(int qld_total, int nv, int nbody) { return (size_t)qld_total + 64 * (size_t)nv + nv + 6 * (size_t)nbody; }

// Right-hand side r of a world, in the reference's order: the nv unit vectors, 6 Jacobian rows of each body b >= 1 (3 translational,
// 3 rotational, at xipos), the tendon Jacobian rows, the actuator moment rows.  rhs is this lane's column (stride 32), zeroed.
__device__ void build_rhs(const ModelDev& m, const DataDev& d, int w, int r, float* rhs) {
  const size_t wb = (size_t)w;
  if (r < m.nv) { rhs[32 * r] = 1.f; return; }
  r -= m.nv;
  const int nrow_body = 6 * (m.nbody - 1);
  if (r < nrow_body) {  // set_const.py:263-318 _compute_body_jac_row
    const int b = 1 + r / 6, row = r % 6;
    int bb = b;
    while (bb > 0 && m.body_dofnum[bb] == 0) bb = m.body_parentid[bb];
    if (bb == 0) return;
    const v3 offset = ld3(d.xipos + (wb * m.nbody + b) * 3) - ld3(d.subtree_com + (wb * m.nbody + m.body_rootid[b]) * 3);
    for (int dof = m.body_dofadr[bb] + m.body_dofnum[bb] - 1; dof >= 0; dof = m.dof_parentid[dof]) {
      const float* cd = d.cdof + (wb * m.nv + dof) * 6;
      float v;
      if (row < 3) {
        const v3 tmp = cross(ld3(cd), offset);
        v = cd[3 + row] + (row == 0 ? tmp.x : row == 1 ? tmp.y : tmp.z);
      } else {
        v = cd[row - 3];
      }
      rhs[32 * dof] = v;
    }
    return;
  }
  r -= nrow_body;
  if (r < m.ntendon) {  // set_const.py:376-390 _copy_tendon_jacobian
    for (int k = m.ten_J_rowadr[r]; k < m.ten_J_rowadr[r] + m.ten_J_rownnz[r]; k++) rhs[32 * m.ten_J_colind[k]] = d.ten_J[wb * m.nJten + k];
    return;
  }
  r -= m.ntendon;  // set_const.py:473-490 _copy_actuator_moment
  const int adr = d.moment_rowadr[wb * m.nu + r], nnz = d.moment_rownnz[wb * m.nu + r];
  for (int k = adr; k < adr + nnz; k++) rhs[32 * d.moment_colind[wb * m.nJmom + k]] = d.actuator_moment[wb * m.nJmom + k];
}

__global__ void __launch_bounds__(32)
k_set_const(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const SetConstDev c, int nw) {
  extern __shared__ float sm[];
  const int lane = threadIdx.x, w = blockIdx.x;
  if (w >= nw) return;
  const size_t wb = (size_t)w;
  const ModelDev m = world_model(mp, w, d.nworld);
  const int nv = m.nv, nbody = m.nbody;
  float* U = sm;
  float* rhs = U + m.qld_total;
  float* x = rhs + 32 * nv;
  float* diagA = x + 32 * nv;
  float* bodyA = diagA + nv;
  warp_copy(U, d.qLD + wb * m.qld_total, m.qld_total, lane);
  __syncwarp();

  const int nrhs = nv + 6 * (nbody - 1) + m.ntendon + m.nu;
  const bool st_tenw = w < m.nb_tendon_invweight0, st_acc0 = w < c.nb_actuator_acc0;
#pragma unroll 1
  for (int base = 0; base < nrhs; base += 32) {
    const int r = base + lane;
    if (r < nrhs) {
      float* rl = rhs + lane;
      float* xl = x + lane;
      for (int i = 0; i < nv; i++) rl[32 * i] = 0.f;
      build_rhs(m, d, w, r, rl);
      for (int i = 0; i < nv; i++) xl[32 * i] = rl[32 * i];
      // x = M^-1 rhs tree by tree, the arithmetic of k_solve_m (k_support.cu): U^T z = rhs, then U x = z
#pragma unroll 1
      for (int t = 0; t < m.ntree; t++) {
        const int n = m.tree_dofnum[t];
        const float* Ut = U + m.tree_qLDadr[t];
        float* xt = xl + 32 * m.tree_dofadr[t];
#pragma unroll 1
        for (int j = 0; j < n; j++) {
          const float zj = xt[32 * j] / Ut[j * n + j];
          for (int i = j + 1; i < n; i++) xt[32 * i] -= Ut[j * n + i] * zj;
          xt[32 * j] = zj;
        }
#pragma unroll 1
        for (int j = n - 1; j >= 0; j--) {
          const float xj = xt[32 * j] / Ut[j * n + j];
          for (int i = 0; i < j; i++) xt[32 * i] -= Ut[i * n + j] * xj;
          xt[32 * j] = xj;
        }
      }
      // each solution reduced to the scalar it is for, summed in the reference's order
      if (r < nv) {
        diagA[r] = xl[32 * r];  // set_const.py:207-215
      } else if (r < nv + 6 * (nbody - 1)) {  // set_const.py:321-336: J[row] . M^-1 J[row]^T
        float s = 0.f;
        for (int i = 0; i < nv; i++) s += rl[32 * i] * xl[32 * i];
        bodyA[6 + (r - nv)] = s;
      } else if (r < nv + 6 * (nbody - 1) + m.ntendon) {  // set_const.py:393-417
        const int t = r - nv - 6 * (nbody - 1);
        float s = 0.f;
        for (int k = m.ten_J_rowadr[t]; k < m.ten_J_rowadr[t] + m.ten_J_rownnz[t]; k++) s += d.ten_J[wb * m.nJten + k] * xl[32 * m.ten_J_colind[k]];
        if (st_tenw) const_cast<float*>(m.tendon_invweight0)[t] = s;
      } else {  // set_const.py:493-504: || M^-1 moment ||
        const int a = r - nv - 6 * (nbody - 1) - m.ntendon;
        float s = 0.f;
        for (int i = 0; i < nv; i++) s += xl[32 * i] * xl[32 * i];
        if (st_acc0) c.actuator_acc0[(size_t)w * m.nu + a] = sqrtf(s);
      }
    }
  }
  __syncwarp();

  // set_const.py:218-259 dof_invweight0: diag(M^-1), averaged over each half of a free joint and over a ball joint
  if (w < m.nb_dof_invweight0) {
    float* out = const_cast<float*>(m.dof_invweight0);
    for (int i = lane; i < nv; i += 32) {
      const int j = m.dof_jntid[i], type = m.jnt_type[j], adr = m.jnt_dofadr[j];
      float v = diagA[i];
      if (type == JNT_FREE || type == JNT_BALL) {
        const int a = (type == JNT_FREE && i >= adr + 3) ? adr + 3 : adr;
        v = (1.0f / 3.0f) * (diagA[a] + diagA[a + 1] + diagA[a + 2]);
      }
      out[i] = v;
    }
  }
  // set_const.py:339-372 body_invweight0: mean diagonal of the translational / rotational parts, with the MINVAL fallback between them
  if (w < m.nb_body_invweight0) {
    float* out = const_cast<float*>(m.body_invweight0);
    for (int b = lane; b < nbody; b += 32) {
      float tr = 0.f, rot = 0.f;
      if (b > 0 && m.body_weldid[b] != 0) {
        const float* A = bodyA + 6 * b;
        tr = (1.0f / 3.0f) * (A[0] + A[1] + A[2]);
        rot = (1.0f / 3.0f) * (A[3] + A[4] + A[5]);
        if (tr < MJ_MINVAL && rot > MJ_MINVAL) tr = rot;
        else if (rot < MJ_MINVAL && tr > MJ_MINVAL) rot = tr;
      }
      out[2 * b] = tr;
      out[2 * b + 1] = rot;
    }
  }
  // set_const.py:169-190 meaninertia: mean of diag(M), world 0 only (a Model scalar here)
  if (w == 0 && lane == 0) {
    float total = 0.f;
    for (int i = 0; i < nv; i++) total += d.M[wb * m.nC + m.M_rowadr[i] + m.M_rownnz[i] - 1];
    c.meaninertia[0] = nv > 0 ? total / (float)nv : 1.f;
  }
  // set_const.py:69-76 tendon_length0
  if (w < m.nb_tendon_length0)
    for (int t = lane; t < m.ntendon; t += 32) const_cast<float*>(m.tendon_length0)[t] = d.ten_length[wb * m.ntendon + t];
  // set_const.py:79-153 eq_data: connect / weld anchors and the relative pose at qpos0; a weld whose quaternion is set is normalised
  if (w < m.nb_eq_data) {
    for (int e = lane; e < m.neq; e += 32) {
      float* data = const_cast<float*>(m.eq_data) + 11 * e;
      const int type = m.eq_type[e], o1 = m.eq_obj1id[e], o2 = m.eq_obj2id[e];
      const float* xpos = d.xpos + wb * nbody * 3;
      const float* xmat = d.xmat + wb * nbody * 9;
      if (type == EQ_CONNECT) {
        const v3 pos = ld3(xpos + 3 * o1) + matvec(xmat + 9 * o1, ld3(data));
        const v3 p = pos - ld3(xpos + 3 * o2);
        const float* R = xmat + 9 * o2;
        st3(data + 3, mk3(dot(matcol(R, 0), p), dot(matcol(R, 1), p), dot(matcol(R, 2), p)));
      } else if (type == EQ_WELD) {
        const q4 q = ldq(data + 6);
        if (q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z > 0.f) {
          stq(data + 6, qnormalize(q));
        } else {
          const v3 pos = ld3(xpos + 3 * o2) + matvec(xmat + 9 * o2, ld3(data));
          const v3 p = pos - ld3(xpos + 3 * o1);
          const float* R = xmat + 9 * o1;
          st3(data + 3, mk3(dot(matcol(R, 0), p), dot(matcol(R, 1), p), dot(matcol(R, 2), p)));
          const q4 q1 = ldq(d.xquat + (wb * nbody + o1) * 4), q2 = ldq(d.xquat + (wb * nbody + o2) * 4);
          stq(data + 6, qmul(mkq(q1.w, -q1.x, -q1.y, -q1.z), q2));
        }
      }
    }
  }
  // set_const.py:420-469 camera and light reference poses
  for (int i = lane; i < m.ncam; i += 32) {
    const int b = m.cam_bodyid[i], tb = m.cam_targetbodyid[i];
    const v3 p = ld3(d.cam_xpos + (wb * m.ncam + i) * 3);
    if (w < m.nb_cam_pos0) st3(const_cast<float*>(m.cam_pos0) + 3 * i, p - ld3(d.xpos + (wb * nbody + b) * 3));
    if (w < m.nb_cam_poscom0) st3(const_cast<float*>(m.cam_poscom0) + 3 * i, p - ld3(d.subtree_com + (wb * nbody + (tb >= 0 ? tb : b)) * 3));
    if (w < m.nb_cam_mat0)
      for (int k = 0; k < 9; k++) const_cast<float*>(m.cam_mat0)[9 * i + k] = d.cam_xmat[(wb * m.ncam + i) * 9 + k];
  }
  for (int i = lane; i < m.nlight; i += 32) {
    const int b = m.light_bodyid[i], tb = m.light_targetbodyid[i];
    const v3 p = ld3(d.light_xpos + (wb * m.nlight + i) * 3);
    if (w < m.nb_light_pos0) st3(const_cast<float*>(m.light_pos0) + 3 * i, p - ld3(d.xpos + (wb * nbody + b) * 3));
    if (w < m.nb_light_poscom0) st3(const_cast<float*>(m.light_poscom0) + 3 * i, p - ld3(d.subtree_com + (wb * nbody + (tb >= 0 ? tb : b)) * 3));
    if (w < m.nb_light_dir0) st3(const_cast<float*>(m.light_dir0) + 3 * i, ld3(d.light_xdir + (wb * m.nlight + i) * 3));
  }
  // set_const.py:507-570 dampratio of affine-bias actuators (gainprm[0] == -biasprm[1], biasprm[2] > 0), reflected mass from diag(M)
  if (w < m.nb_actuator_biasprm) {
    for (int a = lane; a < m.nu; a += 32) {
      if (m.actuator_biastype[a] != BIAS_AFFINE) continue;
      float* bp = const_cast<float*>(m.actuator_biasprm) + 10 * a;
      const float kp = m.actuator_gainprm[10 * a];
      if (fabsf(kp + bp[1]) > MJ_MINVAL || bp[2] <= 0.f) continue;
      float mass = 0.f;
      const int adr = d.moment_rowadr[wb * m.nu + a], nnz = d.moment_rownnz[wb * m.nu + a];
      for (int k = adr; k < adr + nnz; k++) {
        const int j = d.moment_colind[wb * m.nJmom + k];
        const float mom = d.actuator_moment[wb * m.nJmom + k];
        if (fabsf(mom) > MJ_MINVAL) mass += d.M[wb * m.nC + m.M_rowadr[j] + m.M_rownnz[j] - 1] / (mom * mom);
      }
      bp[2] = -(bp[2] * 2.0f * sqrtf(kp * mass));
    }
  }
}

}  // namespace

size_t smem_set_const(const ModelDev& m) { return sizeof(float) * set_const_words(m.qld_total, m.nv, m.nbody); }

cudaError_t launch_set_const_fixed(const ModelDev& m, int nw, int nworld, cudaStream_t s) {
  return launch(k_set_const_fixed, (nw + 127) / 128, 128, 0, s, m, nw, nworld);
}
cudaError_t launch_set_length_range(const ModelDev& m, int nw, int nworld, cudaStream_t s) {
  const int n = nw * m.nu;
  if (n == 0) return cudaSuccess;
  return launch(k_set_length_range, (n + 127) / 128, 128, 0, s, m, nw, nworld);
}
cudaError_t launch_set_const_qpos(const ModelDev& m, const DataDev& d, const SetConstDev& c, int mode, int nw, cudaStream_t s) {
  const int n = nw * m.nq;
  if (n == 0) return cudaSuccess;  // no joints: qpos0 / qpos_spring and the state are empty
  return launch(k_set_const_qpos, (n + 255) / 256, 256, 0, s, m, d, c, mode, nw);
}
cudaError_t launch_set_const_0(const ModelDev& m, const DataDev& d, const SetConstDev& c, int nw, cudaStream_t s) {
  return launch(k_set_const, nw, 32, smem_set_const(m), s, m, d, c, nw);
}
cudaError_t launch_set_const_spring(const ModelDev& m, const DataDev& d, int nw, cudaStream_t s) {
  const int n = nw * m.ntendon;
  return launch(k_set_const_spring, (n + 127) / 128, 128, 0, s, m, d, nw);
}
