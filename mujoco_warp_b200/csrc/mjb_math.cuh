// mjb_math.cuh -- device math for the step kernels (fp32).
// Same conventions as the reference's math.py (/root/reference/mujoco_warp/_src/math.py): quaternion (w,x,y,z),
// spatial vector (angular, linear), vec10 inertia, row-major mat33.  Written from the formulas, not from the Warp source.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include "mjb_types.cuh"

#define FULL_MASK 0xffffffffu

struct v3 { float x, y, z; };
struct q4 { float w, x, y, z; };

__device__ __forceinline__ v3 mk3(float x, float y, float z) { v3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ v3 ld3(const float* p) { return mk3(p[0], p[1], p[2]); }
__device__ __forceinline__ void st3(float* p, v3 a) { p[0] = a.x; p[1] = a.y; p[2] = a.z; }
__device__ __forceinline__ v3 operator+(v3 a, v3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ v3 operator-(v3 a, v3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ v3 operator*(v3 a, float s) { return mk3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ v3 operator*(float s, v3 a) { return mk3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ v3 cross(v3 a, v3 b) { return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float length(v3 a) { return sqrtf(dot(a, a)); }
// zero vector stays zero (Warp's normalize semantics)
__device__ __forceinline__ v3 normalize(v3 a) { float l = length(a); return l > 0.f ? a * (1.0f / l) : mk3(0.f, 0.f, 0.f); }

__device__ __forceinline__ q4 mkq(float w, float x, float y, float z) { q4 q; q.w = w; q.x = x; q.y = y; q.z = z; return q; }
__device__ __forceinline__ q4 ldq(const float* p) { return mkq(p[0], p[1], p[2], p[3]); }
__device__ __forceinline__ void stq(float* p, q4 q) { p[0] = q.w; p[1] = q.x; p[2] = q.y; p[3] = q.z; }
__device__ __forceinline__ q4 qnormalize(q4 q) {
  float l = sqrtf(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  if (l > 0.f) { float s = 1.0f / l; return mkq(q.w * s, q.x * s, q.y * s, q.z * s); }
  return mkq(0.f, 0.f, 0.f, 0.f);
}
__device__ __forceinline__ q4 qmul(q4 u, q4 v) {
  return mkq(u.w * v.w - u.x * v.x - u.y * v.y - u.z * v.z, u.w * v.x + u.x * v.w + u.y * v.z - u.z * v.y,
             u.w * v.y - u.x * v.z + u.y * v.w + u.z * v.x, u.w * v.z + u.x * v.y - u.y * v.x + u.z * v.w);
}
__device__ __forceinline__ v3 qrot(q4 q, v3 v) {
  v3 u = mk3(q.x, q.y, q.z);
  float s = q.w;
  return 2.0f * dot(u, v) * u + (s * s - dot(u, u)) * v + 2.0f * s * cross(u, v);
}
__device__ __forceinline__ q4 axis_angle_quat(v3 axis, float angle) {
  float s, c;
  sincosf(angle * 0.5f, &s, &c);
  return mkq(c, axis.x * s, axis.y * s, axis.z * s);
}
__device__ __forceinline__ void quat_to_mat(q4 q, float* m) {
  float q00 = q.w * q.w, q01 = q.w * q.x, q02 = q.w * q.y, q03 = q.w * q.z;
  float q11 = q.x * q.x, q12 = q.x * q.y, q13 = q.x * q.z, q22 = q.y * q.y, q23 = q.y * q.z, q33 = q.z * q.z;
  m[0] = q00 + q11 - q22 - q33; m[1] = 2.f * (q12 - q03); m[2] = 2.f * (q13 + q02);
  m[3] = 2.f * (q12 + q03); m[4] = q00 - q11 + q22 - q33; m[5] = 2.f * (q23 - q01);
  m[6] = 2.f * (q13 - q02); m[7] = 2.f * (q23 + q01); m[8] = q00 - q11 - q22 + q33;
}
__device__ __forceinline__ q4 quat_integrate(q4 q, v3 v, float dt) {
  float n = length(v);
  v3 a = normalize(v);
  q4 r = axis_angle_quat(a, dt * n);
  return qnormalize(qmul(qnormalize(q), r));
}
__device__ __forceinline__ v3 matvec(const float* m, v3 v) {
  return mk3(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[3] * v.x + m[4] * v.y + m[5] * v.z, m[6] * v.x + m[7] * v.y + m[8] * v.z);
}
__device__ __forceinline__ v3 matcol(const float* m, int k) { return mk3(m[k], m[3 + k], m[6 + k]); }

// spatial (6-vector) helpers on float[6]
__device__ __forceinline__ void inert_vec(const float* i, const float* v, float* o) {
  float r0 = i[0] * v[0] + i[3] * v[1] + i[4] * v[2] - i[8] * v[4] + i[7] * v[5];
  float r1 = i[3] * v[0] + i[1] * v[1] + i[5] * v[2] + i[8] * v[3] - i[6] * v[5];
  float r2 = i[4] * v[0] + i[5] * v[1] + i[2] * v[2] - i[7] * v[3] + i[6] * v[4];
  float r3 = i[8] * v[1] - i[7] * v[2] + i[9] * v[3];
  float r4 = i[6] * v[2] - i[8] * v[0] + i[9] * v[4];
  float r5 = i[7] * v[0] - i[6] * v[1] + i[9] * v[5];
  o[0] = r0; o[1] = r1; o[2] = r2; o[3] = r3; o[4] = r4; o[5] = r5;
}
__device__ __forceinline__ void motion_cross(const float* u, const float* v, float* o) {
  v3 u0 = ld3(u), u1 = ld3(u + 3), v0 = ld3(v), v1 = ld3(v + 3);
  v3 a = cross(u0, v0), b = cross(u1, v0) + cross(u0, v1);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = b.x; o[4] = b.y; o[5] = b.z;
}
__device__ __forceinline__ void motion_cross_force(const float* v, const float* f, float* o) {
  v3 v0 = ld3(v), v1 = ld3(v + 3), f0 = ld3(f), f1 = ld3(f + 3);
  v3 a = cross(v0, f0) + cross(v1, f1), b = cross(v0, f1);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = b.x; o[4] = b.y; o[5] = b.z;
}
__device__ __forceinline__ float dot6(const float* a, const float* b) {
  return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5];
}
// contact frame with rows (a, b, c): b orthogonal to a chosen from y or z (reference math.py:203-258)
__device__ __forceinline__ void make_frame(v3 a_in, float* frame) {
  v3 a = normalize(a_in);
  v3 s = (-0.5f < a.y && a.y < 0.5f) ? mk3(0.f, 1.f, 0.f) : mk3(0.f, 0.f, 1.f);
  v3 b = normalize(s - a * dot(a, s));
  if (length(a) == 0.f) b = mk3(0.f, 0.f, 0.f);
  v3 c = cross(a, b);
  st3(frame, a); st3(frame + 3, b); st3(frame + 6, c);
}
__device__ __forceinline__ float safe_div(float x, float y) { return x / (y != 0.f ? y : MJ_MINVAL); }
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
// smooth.py:3658-3692 (fixed tendons): length = sum of coef * joint position over the tendon's joint wraps; the Jacobian entries are
// the constant coefficients (Model.ten_J0, in the sparsity of ten_J_colind)
__device__ __forceinline__ float tendon_length(const ModelDev& m, int t, const float* qpos) {
  float len = 0.f;
#pragma unroll 1
  for (int k = m.tendon_adr[t]; k < m.tendon_adr[t] + m.tendon_num[t]; k++) len += m.wrap_prm[k] * qpos[m.jnt_qposadr[m.wrap_objid[k]]];
  return len;
}
// entry of tendon t's Jacobian row at dof c (0 outside the row's sparsity)
__device__ __forceinline__ float tendon_J_at(const ModelDev& m, int t, int c) {
  const int adr = m.ten_J_rowadr[t], n = m.ten_J_rownnz[t];
  for (int k = 0; k < n; k++) if (m.ten_J_colind[adr + k] == c) return m.ten_J0[adr + k];
  return 0.f;
}
// support.py:153-256 mul_m: row i of M v for one world's M (nC entries) through the symmetric gather tables; v in shared memory
__device__ __forceinline__ float mul_m_row(const ModelDev& m, const float* M, const float* v, int i) {
  float acc = 0.f;
  for (int k = m.mulm_rowadr[i]; k < m.mulm_rowadr[i + 1]; k++) acc += M[m.mulm_madr[k]] * v[m.mulm_col[k]];
  return acc;
}
// support.py:38-64 next_act: one integration step of actuator a's activation (exact for FILTEREXACT), optionally clamped to actrange
__device__ __forceinline__ float next_act(const ModelDev& m, int a, float act, float act_dot, float scale, bool clamp) {
  float r;
  if (m.actuator_dyntype[a] == DYN_FILTEREXACT) {
    const float tau = fmaxf(MJ_MINVAL, m.actuator_dynprm[10 * a]);
    r = act + scale * act_dot * tau * (1.0f - expf(-m.timestep / tau));
  } else r = act + scale * act_dot * m.timestep;
  if (clamp) r = clampf(r, m.actuator_actrange[2 * a], m.actuator_actrange[2 * a + 1]);
  return r;
}
__device__ __forceinline__ v3 closest_segment_point(v3 a, v3 b, v3 pt) {
  v3 ab = b - a;
  float t = dot(pt - a, ab) / (dot(ab, ab) + 1e-6f);
  return a + clampf(t, 0.f, 1.f) * ab;
}

// warp helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}
// exclusive prefix sum over lanes
__device__ __forceinline__ int warp_excl_scan(int v, int lane) {
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(FULL_MASK, x, o); if (lane >= o) x += y; }
  return x - v;
}
// coalesced copy of n floats between a world's global row and its shared staging buffer
__device__ __forceinline__ void warp_copy(float* dst, const float* src, int n, int lane) {
  for (int i = lane; i < n; i += 32) dst[i] = src[i];
}
__device__ __forceinline__ void warp_copy_i(int* dst, const int* src, int n, int lane) {
  for (int i = lane; i < n; i += 32) dst[i] = src[i];
}
