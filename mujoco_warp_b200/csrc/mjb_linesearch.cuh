// mjb_linesearch.cuh -- scalar pieces of the Newton / CG line search (k_solver.cu): per-row cost / gradient / curvature of the piecewise-
// quadratic 1-D cost, shifted by its value at alpha = 0, for equality / friction-loss / inequality rows and for elliptic contacts.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/solver.py): :203 _eval_pt, :425-517 _eval_constraint / the shifted direct and
// friction-loss evaluations, :286-305 _eval_elliptic_reference, :308-320 alpha = 0 value, :329-404 _eval_elliptic_shifted.
// Plain functions of their arguments (no warp intrinsics, no shared memory), kept in a header so that the same source also compiles as
// host C++: tests/host_harness/linesearch_host.cpp runs the reference's elliptic shifted-cost known-answer vectors (solver_test.py:296-350)
// through THIS code on the CPU.
#pragma once
#include "mjb_math.cuh"
#include "mjb_types.cuh"

struct P3 { float c, g, h; };
__device__ __forceinline__ P3 mkp(float c, float g, float h) { P3 p; p.c = c; p.g = g; p.h = h; return p; }
__device__ __forceinline__ P3 operator+(P3 a, P3 b) { return mkp(a.c + b.c, a.g + b.g, a.h + b.h); }


// row kinds by position (solver.py:1751-1755): [0,ne) equality, [ne,ne+nf) friction loss, rest inequality
// shifted evaluation: (cost(alpha) - cost(0), grad, hess) -- solver.py:479-517
__device__ __forceinline__ P3 eval_row(int r, float alpha, int ne, int nf, float D, float f, float jaref, float jv) {
  if (r >= ne + nf) {
    const float x = jaref + alpha * jv, quad0 = 0.5f * D * jaref * jaref, cost0 = jaref < 0.f ? quad0 : 0.f, offset = quad0 - cost0;
    if (x < 0.f) { const float jvD = jv * D, h = jv * jvD, ah = alpha * h; return mkp(alpha * (jvD * jaref + 0.5f * ah) + offset, jvD * jaref + ah, h); }
    return mkp(-cost0, 0.f, 0.f);
  }
  if (r >= ne) {
    const float x = jaref + alpha * jv, rf = safe_div(f, D);
    float c0;
    if (-rf < jaref && jaref < rf) c0 = 0.5f * D * jaref * jaref; else if (jaref <= -rf) c0 = f * (-0.5f * rf - jaref); else c0 = f * (-0.5f * rf + jaref);
    if (-rf < x && x < rf) { const float jvD = jv * D; return mkp(0.5f * D * x * x - c0, jvD * x, jv * jvD); }
    if (x <= -rf) return mkp(f * (-0.5f * rf - x) - c0, -f * jv, 0.f);
    return mkp(f * (-0.5f * rf + x) - c0, f * jv, 0.f);
  }
  const float jvD = jv * D, h = jv * jvD, ah = alpha * h;
  return mkp(alpha * (jvD * jaref + 0.5f * ah), jvD * jaref + ah, h);
}
// absolute evaluation at alpha = 0 (solver.py:570-592)
__device__ __forceinline__ P3 eval_row_zero(int r, int ne, int nf, float D, float f, float jaref, float jv) {
  if (r >= ne + nf) {
    if (jaref < 0.f) { const float jvD = jv * D; return mkp(0.5f * D * jaref * jaref, jvD * jaref, jv * jvD); }
    return mkp(0.f, 0.f, 0.f);
  }
  if (r >= ne) {
    const float rf = safe_div(f, D), x = jaref;
    if (-rf < x && x < rf) { const float jvD = jv * D; return mkp(0.5f * D * x * x, jvD * x, jv * jvD); }
    if (x <= -rf) return mkp(f * (-0.5f * rf - x), -f * jv, 0.f);
    return mkp(f * (-0.5f * rf + x), f * jv, 0.f);
  }
  const float jvD = jv * D;
  return mkp(0.5f * D * jaref * jaref, jvD * jaref, jv * jvD);
}
__device__ __forceinline__ P3 eval_gauss(float q0, float q1, float q2, float alpha) {  // _eval_pt solver.py:203
  const float aq2 = alpha * q2;
  return mkp(alpha * aq2 + alpha * q1 + q0, 2.0f * aq2 + q1, 2.0f * q2);
}
__device__ __forceinline__ bool in_bracket(P3 x, P3 y) { return (x.g < y.g && y.g < 0.f) || (x.g > y.g && y.g > 0.f); }

// ---- force and state of one row at its Jaref (solver.py:1699 _update_constraint_efc), shared by the solver's row pass (k_solver.cu) and
// inverse dynamics (k_inverse.cu).  Row kinds by position as above; with ELL, rows whose rinfo is not -1 belong to an elliptic contact:
// rinfo = -2 (contact cut by njmax: no force) or (dim << 4) | j, and rfri = mu (j = 0) or friction[j - 1].  Jaref, Dv: the world's rows.
// Sets force and st, and cone0 = true when the row is the first row of a contact in the cone zone.  A macro, so that the solver's row pass
// compiles exactly as it did with the rule written out in place (the inlined-function form reorders its branches).
#define MJB_ROW_FORCE_STATE(ELL, r, ne, nf, jaref, D, floss, rinfo, rfri, Jaref, Dv, force, st, cone0)                                          \
  if ((r) < (ne)) { force = -(D) * (jaref); st = ST_QUADRATIC; }                                                                            \
  else if ((r) < (ne) + (nf)) {                                                                                                              \
    const float f_ = (floss)[r], rf_ = safe_div(f_, D);                                                                                      \
    if ((jaref) <= -rf_) { force = f_; st = ST_LINEARNEG; } else if ((jaref) >= rf_) { force = -f_; st = ST_LINEARPOS; }                      \
    else { force = -(D) * (jaref); st = ST_QUADRATIC; }                                                                                      \
  } else if ((ELL) && (rinfo)[r] != -1) {  /* solver.py:455-472 */                                                                           \
    const int info_ = (rinfo)[r];                                                                                                            \
    force = 0.f; st = ST_SATISFIED;                                                                                                          \
    if (info_ >= 0) {                                                                                                                        \
      const int j_ = info_ & 15, dim_ = info_ >> 4, e0_ = (r) - j_;                                                                          \
      const float mu_ = (rfri)[e0_], N_ = (Jaref)[e0_] * mu_;                                                                                \
      float TT_ = 0.f;                                                                                                                       \
      for (int i_ = 1; i_ < dim_; i_++) { const float u_ = (Jaref)[e0_ + i_] * (rfri)[e0_ + i_]; TT_ += u_ * u_; }                          \
      const float T_ = TT_ <= 0.f ? 0.f : sqrtf(TT_);                                                                                        \
      if ((N_ >= mu_ * T_) || (T_ <= 0.f && N_ >= 0.f)) {}                                                                                   \
      else if ((mu_ * N_ + T_ <= 0.f) || (T_ <= 0.f && N_ < 0.f)) { force = -(D) * (jaref); st = ST_QUADRATIC; }                             \
      else {                                                                                                                                 \
        const float dm_ = safe_div((Dv)[e0_], mu_ * mu_ * (1.0f + mu_ * mu_)), fn_ = -dm_ * (N_ - mu_ * T_) * mu_, fr_ = (rfri)[r];          \
        force = j_ == 0 ? fn_ : -safe_div(fn_, T_) * ((jaref) * fr_ * fr_);                                                                   \
        st = ST_CONE;                                                                                                                        \
        cone0 = j_ == 0;                                                                                                                     \
      }                                                                                                                                      \
    }                                                                                                                                        \
  } else if ((jaref) >= 0.f) { force = 0.f; st = ST_SATISFIED; }                                                                             \
  else { force = -(D) * (jaref); st = ST_QUADRATIC; }

template <bool ELL>
__device__ __forceinline__ void row_force_state(int r, int ne, int nf, float jaref, float D, const float* floss, const int* rinfo, const float* rfri,
                                                const float* Jaref, const float* Dv, float& force, int& st, bool& cone0) {
  MJB_ROW_FORCE_STATE(ELL, r, ne, nf, jaref, D, floss, rinfo, rfri, Jaref, Dv, force, st, cone0)
}

// ---- elliptic cone, one contact (quad = cost polynomial of all its rows, (u0, v0, uu), (uv, vv, dm))
struct EllQ { float q0, q1, q2, u0, v0, uu, uv, vv, dm; };
struct EllRef { float cost0, T0, r0; int st; };
// cost / tangential norm / residual / zone at alpha = 0 (solver.py:286-305)
__device__ __forceinline__ EllRef ell_reference(float mu, const EllQ& q) {
  EllRef e; e.T0 = 0.f; e.r0 = 0.f;
  if (q.uu <= 0.f) { const bool neg = q.u0 < 0.f; e.cost0 = neg ? q.q0 : 0.f; e.st = neg ? ST_QUADRATIC : ST_SATISFIED; return e; }
  e.T0 = sqrtf(q.uu);
  if (q.u0 >= mu * e.T0) { e.cost0 = 0.f; e.st = ST_SATISFIED; return e; }
  if (mu * q.u0 + e.T0 <= 0.f) { e.cost0 = q.q0; e.st = ST_QUADRATIC; return e; }
  e.r0 = q.u0 - mu * e.T0; e.cost0 = 0.5f * q.dm * e.r0 * e.r0; e.st = ST_CONE;
  return e;
}
// shifted (cost(alpha) - cost(0), grad, hess) of one elliptic contact (solver.py:329-404)
__device__ __forceinline__ P3 ell_shifted(float mu, const EllQ& q, const EllRef& e, float alpha) {
  const float N = q.u0 + alpha * q.v0, Tsqr_delta = alpha * (2.0f * q.uv + alpha * q.vv), Tsqr = q.uu + Tsqr_delta;
  bool bottom = false;
  float T = 0.f;
  if (Tsqr <= 0.f) bottom = N < 0.f;
  else {
    T = sqrtf(Tsqr);
    if (N >= mu * T) {}  // top zone
    else if (mu * N + T <= 0.f) bottom = true;
    else {
      const float Tinv = 1.0f / T, T1 = (q.uv + alpha * q.vv) * Tinv, T2 = (q.vv - T1 * T1) * Tinv, r = N - mu * T, r1 = q.v0 - mu * T1;
      float cost;
      if (e.st == ST_CONE) { const float Td = Tsqr_delta / (T + e.T0), rd = alpha * q.v0 - mu * Td; cost = 0.5f * q.dm * rd * (2.0f * e.r0 + rd); }
      else if (e.st == ST_QUADRATIC) { const float aq2 = alpha * q.q2, b = mu * N + T; cost = alpha * (aq2 + q.q1) - 0.5f * q.dm * b * b; }
      else cost = 0.5f * q.dm * r * r;
      return mkp(cost, q.dm * r * r1, q.dm * (r1 * r1 + r * (-mu * T2)));
    }
  }
  if (bottom) {
    const float aq2 = alpha * q.q2;
    float cost = alpha * (aq2 + q.q1);
    if (e.st == ST_CONE) { const float b = mu * q.u0 + e.T0; cost += 0.5f * q.dm * b * b; }
    else if (e.st == ST_SATISFIED) cost = 0.5f * q.dm * (1.0f + mu * mu) * (N * N + fmaxf(Tsqr, 0.f));
    return mkp(cost, 2.0f * aq2 + q.q1, 2.0f * q.q2);
  }
  return mkp(-e.cost0, 0.f, 0.f);
}
// absolute value at alpha = 0 (solver.py:308-320)
__device__ __forceinline__ P3 ell_zero(float mu, const EllQ& q) {
  const EllRef e = ell_reference(mu, q);
  if (e.st == ST_QUADRATIC) return mkp(q.q0, q.q1, 2.0f * q.q2);
  if (e.st == ST_CONE) {
    const float Tinv = 1.0f / e.T0, T1 = q.uv * Tinv, T2 = (q.vv - T1 * T1) * Tinv, r1 = q.v0 - mu * T1;
    return mkp(e.cost0, q.dm * e.r0 * r1, q.dm * (r1 * r1 - mu * e.r0 * T2));
  }
  return mkp(0.f, 0.f, 0.f);
}

