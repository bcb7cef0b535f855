// k_support.cu -- small public utilities that operate on a finished position stage: solve_m and mul_m.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): smooth.py:3214 solve_m (x = M^-1 y through the per-tree factor kept
// in Data.qLD; the reference launches one tile kernel per block size) and support.py:153-256 mul_m (res = M vec through the
// symmetric gather tables of io.py:1029-1050).  One warp per world, like every other stage.
#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_sensor_contact.cuh"
#include "mjb_types.cuh"

namespace {

// ---- CSR view of the constraint Jacobian for models the reference treats as sparse (io.py:153 is_sparse: nv > 32 under jacobian = auto).
// The kernels of this library build and consume a dense efc.J; this pass writes the reference's arrays next to it (types.py:2021-2072:
// J_rownnz, J_rowadr (nworld, njmax), J_colind, J (nworld, 1, njmax_nnz)) with the reference's own sparsity pattern and column order:
//   contact rows      constraint.py:2728-2753 / :3100-3250  dof chains of the two (weld) bodies, descending dof, stopping at the first common dof
//   connect / weld    :262-370 / :1130-1240                  union of the two chains, descending (common ancestors kept)
//   joint equality    :570-606  dof1 [, dof2];   dof friction :1821  dof;   slide / hinge limit :2041  dof;   ball limit :2182  dof, dof + 1, dof + 2
//   tendon friction / limit :1930 / :2315  the tendon's ten_J_colind entries, in their order (zeros kept)
//   tendon equality   :741-800  ascending merge of the two tendons' ten_J_colind (the second only when the polynomial's slope is
//                     nonzero): the whole merge is reserved, the entries whose value is nonzero are stored and counted in rownnz
// Row addresses are the running sum of rownnz in row order (the reference hands them out with an atomic, i.e. in its launch order; run
// sequentially that is the same sequence).  A row that does not fit in njmax_nnz raises OVF_NJMAX_NNZ and stays empty.
__device__ __forceinline__ int chain_start(const ModelDev& m, int body) {
  const int b = m.body_weldid[body];
  return m.body_dofadr[b] + m.body_dofnum[b] - 1;
}
// walks the two dof chains downwards; emit(da) per visited dof.  stop_common: contact rows end at the first dof both chains share.
template <typename F>
__device__ __forceinline__ int chain_walk(const ModelDev& m, int da1, int da2, bool stop_common, F emit) {
  int n = 0;
  while (da1 >= 0 || da2 >= 0) {
    const int da = max(da1, da2);
    if (stop_common && da1 == da && da2 == da) break;
    if (da1 == da) da1 = m.dof_parentid[da1];
    if (da2 == da) da2 = m.dof_parentid[da2];
    emit(da, n);
    n++;
  }
  return n;
}

// ascending merge of the ten_J_colind rows of tendons t1 and t2 (t2 = -1: t1 alone); emit(col, k) per distinct column
template <typename F>
__device__ __forceinline__ int tendon_merge(const ModelDev& m, int t1, int t2, F emit) {
  const int adr1 = m.ten_J_rowadr[t1], n1 = m.ten_J_rownnz[t1], adr2 = t2 > -1 ? m.ten_J_rowadr[t2] : 0, n2 = t2 > -1 ? m.ten_J_rownnz[t2] : 0;
  int p1 = 0, p2 = 0, n = 0;
  while (p1 < n1 || p2 < n2) {
    const int c1 = p1 < n1 ? m.ten_J_colind[adr1 + p1] : INT_MAX, c2 = p2 < n2 ? m.ten_J_colind[adr2 + p2] : INT_MAX, c = min(c1, c2);
    if (c1 == c) p1++;
    if (c2 == c) p2++;
    emit(c, n);
    n++;
  }
  return n;
}

__global__ void __launch_bounds__(32)
k_efc_csr(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d) {
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld || w >= d.w0 + d.wn) return;
  const size_t wb = (size_t)w;
  const int njmax = d.njmax, nvp = d.nv_pad, nrow = min(d.nefc[w], njmax);
  const float* Jd = d.efc_J + wb * (size_t)d.njmax_pad * nvp;
  float* Jv = d.efc_Jsp + wb * (size_t)d.njmax_nnz;
  int* col = d.efc_J_colind + wb * (size_t)d.njmax_nnz;
  int base = 0;
  bool ovf = false;
#pragma unroll 1
  for (int r0 = 0; r0 < nrow; r0 += 32) {
    const int r = r0 + lane;
    // kind 0: listed dofs a1 [, a2] / ball triple; 1: chain union; 2: chain difference; 4: tendon a1 [merged with tendon a2]; 5: tendon a1
    int kind = 0, a1 = -1, a2 = -1, nnz = 0;
    const float* Jr = Jd + (size_t)r * nvp;
    if (r < nrow) {
      const int type = d.efc_type[wb * njmax + r], id = d.efc_id[wb * njmax + r];
      if (type == CNSTR_EQUALITY) {
        const int o1 = m.eq_obj1id[id], o2 = m.eq_obj2id[id];
        if (m.eq_type[id] == EQ_JOINT) { a1 = m.jnt_dofadr[o1]; a2 = o2 > -1 ? m.jnt_dofadr[o2] : -1; nnz = a2 >= 0 ? 2 : 1; }
        else if (m.eq_type[id] == EQ_TENDON) {
          kind = 4; a1 = o1;
          if (o2 > -1) {  // the polynomial's slope, as k_constraint evaluates it
            const ModelDev mw = world_model(m, w, d.nworld);
            const float* data = mw.eq_data + 11 * id;
            const float dif = d.ten_length[wb * m.ntendon + o2] - mw.tendon_length0[o2], dif2 = dif * dif, dif3 = dif2 * dif;
            if (data[1] + 2.0f * data[2] * dif + 3.0f * data[3] * dif2 + 4.0f * data[4] * dif3 != 0.f) a2 = o2;
          }
          nnz = tendon_merge(m, a1, a2, [](int, int) {});
        } else { kind = 1; a1 = chain_start(m, o1); a2 = chain_start(m, o2); }
      } else if (type == CNSTR_FRICTION_DOF) { a1 = id; nnz = 1; }
      else if (type == CNSTR_LIMIT_JOINT) { a1 = m.jnt_dofadr[id]; if (m.jnt_type[id] == JNT_BALL) { kind = 3; nnz = 3; } else nnz = 1; }
      else if (type == CNSTR_FRICTION_TENDON || type == CNSTR_LIMIT_TENDON) { kind = 5; a1 = id; nnz = m.ten_J_rownnz[id]; }
      else { kind = 2; a1 = chain_start(m, m.geom_bodyid[d.contact_geom[2 * (size_t)id]]); a2 = chain_start(m, m.geom_bodyid[d.contact_geom[2 * (size_t)id + 1]]); }
      if (kind == 1 || kind == 2) nnz = chain_walk(m, a1, a2, kind == 2, [](int, int) {});
    }
    const int adr = base + warp_excl_scan(nnz, lane);
    base += warp_sum_i(nnz);
    if (r < nrow) {
      if (kind == 4) {  // rownnz counts the stored (nonzero) entries of the reserved merge; a row that does not fit keeps no rownnz (:758-760)
        int k = 0;
        if (adr + nnz <= d.njmax_nnz) {
          tendon_merge(m, a1, a2, [&](int c, int) { if (Jr[c] != 0.f) { col[adr + k] = c; Jv[adr + k] = Jr[c]; k++; } });
          d.efc_J_rownnz[wb * njmax + r] = k;
        }
      } else {
        d.efc_J_rownnz[wb * njmax + r] = nnz;
      }
      if (adr + nnz > d.njmax_nnz) { ovf = true; continue; }
      d.efc_J_rowadr[wb * njmax + r] = adr;
      if (kind == 1 || kind == 2) chain_walk(m, a1, a2, kind == 2, [&](int da, int k) { col[adr + k] = da; Jv[adr + k] = Jr[da]; });
      else if (kind == 3) { for (int k = 0; k < 3; k++) { col[adr + k] = a1 + k; Jv[adr + k] = Jr[a1 + k]; } }
      else if (kind == 5) { for (int k = 0; k < nnz; k++) { const int c = m.ten_J_colind[m.ten_J_rowadr[a1] + k]; col[adr + k] = c; Jv[adr + k] = Jr[c]; } }
      else if (kind == 0) { col[adr] = a1; Jv[adr] = Jr[a1]; if (nnz == 2) { col[adr + 1] = a2; Jv[adr + 1] = Jr[a2]; } }
    }
  }
  if (__any_sync(FULL_MASK, ovf) && lane == 0) d.overflow[w] |= OVF_NJMAX_NNZ;
}

// qLD holds, per kinematic tree, the dense upper factor U (row-major n x n, zeros below the diagonal) with M = U^T U.
__global__ void __launch_bounds__(32)
k_solve_m(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, float* __restrict__ xo, const float* __restrict__ yi) {
  extern __shared__ float x[];
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  const size_t wb = (size_t)w;
  const int nv = m.nv;
  warp_copy(x, yi + wb * nv, nv, lane);
  __syncwarp();
#pragma unroll 1
  for (int t = 0; t < m.ntree; t++) {
    const int start = m.tree_dofadr[t], n = m.tree_dofnum[t];
    const float* U = d.qLD + wb * m.qld_total + m.tree_qLDadr[t];
    float* xt = x + start;
#pragma unroll 1
    for (int j = 0; j < n; j++) {  // U^T z = y (forward)
      const float zj = xt[j] / U[j * n + j];
      __syncwarp();
      for (int i = j + 1 + lane; i < n; i += 32) xt[i] -= U[j * n + i] * zj;
      if (lane == 0) xt[j] = zj;
      __syncwarp();
    }
#pragma unroll 1
    for (int j = n - 1; j >= 0; j--) {  // U x = z (backward)
      const float xj = xt[j] / U[j * n + j];
      __syncwarp();
      for (int i = lane; i < j; i += 32) xt[i] -= U[i * n + j] * xj;
      if (lane == 0) xt[j] = xj;
      __syncwarp();
    }
  }
  warp_copy(xo + wb * nv, x, nv, lane);
}

__global__ void __launch_bounds__(32)
k_mul_m(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, float* __restrict__ res, const float* __restrict__ vec) {
  extern __shared__ float v[];
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  const size_t wb = (size_t)w;
  warp_copy(v, vec + wb * m.nv, m.nv, lane);
  __syncwarp();
  const float* M = d.M + wb * m.nC;
#pragma unroll 1
  for (int i = lane; i < m.nv; i += 32) res[wb * m.nv + i] = mul_m_row(m, M, v, i);
}

// support.py:326-442 contact_force: 6D force / torque of the listed contacts, in the contact frame unless to_world is set
// (the decode is mjb_sensor_contact.cuh's contact_force_decode).  No adhesion in this build.
__global__ void k_contact_force(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d, const int* __restrict__ contact_ids, int n, int to_world,
                                float* __restrict__ out) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= n) return;
  const int cid = contact_ids[tid];
  if (cid >= d.nacon[0]) return;
  float f[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (cid >= 0) {
    const int w = d.contact_worldid[cid];
    contact_force_decode(m.cone, d.njmax, d.efc_force + (size_t)w * d.njmax, d.contact_efc_address + (size_t)cid * m.nmaxpyramid,
                         d.contact_friction + 5 * (size_t)cid, d.contact_dim[cid], f);
    if (to_world) {  // row vector times the frame matrix, for the force and the torque part
      const float* R = d.contact_frame + 9 * (size_t)cid;
      float t[6];
      for (int k = 0; k < 3; k++) { t[k] = f[0] * R[k] + f[1] * R[3 + k] + f[2] * R[6 + k]; t[3 + k] = f[3] * R[k] + f[4] * R[3 + k] + f[5] * R[6 + k]; }
      for (int k = 0; k < 6; k++) f[k] = t[k];
    }
  }
  for (int k = 0; k < 6; k++) out[6 * (size_t)tid + k] = f[k];
}

}  // namespace

cudaError_t launch_solve_m(const ModelDev& m, const DataDev& d, float* x, const float* y, cudaStream_t s) {
  return launch(k_solve_m, d.wn, 32, (m.nv + 4) * sizeof(float), s, m, d, x, y);
}
cudaError_t launch_mul_m(const ModelDev& m, const DataDev& d, float* res, const float* vec, cudaStream_t s) {
  return launch(k_mul_m, d.wn, 32, (m.nv + 4) * sizeof(float), s, m, d, res, vec);
}
cudaError_t launch_contact_force(const ModelDev& m, const DataDev& d, const int* contact_ids, int n, int to_world, float* out, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  return launch(k_contact_force, (n + 127) / 128, 128, 0, s, m, d, contact_ids, n, to_world, out);
}

cudaError_t launch_efc_csr(const ModelDev& m, const DataDev& d, cudaStream_t s) {
  return launch(k_efc_csr, d.wn, 32, 0, s, m, d);
}
