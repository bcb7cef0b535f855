// k_solver.cu -- Newton constraint solver as ONE persistent launch (one warp per world -- a team of 2 or 4 warps above
// nv = 32 -- with all state in shared memory).
//
// Replaces (reference, /root/reference/mujoco_warp/_src/solver.py): :3671 solve / :3689 _solve, :3622 init_context,
// :1566 _solve_init_dof, :1609 _solve_init_jaref, support.py:153 mul_m, :1698 _update_constraint_efc,
// :1912 qfrc_constraint, :2119-2199 gradient, :2366 _update_gradient_JTDAJ_dense_tiled, :1951 _update_gradient_h_incremental,
// :2567 _update_gradient_cholesky, :836-1347 _linesearch_iterative_kernel, :3453 _solve_done, and the CUDA-graph `while`
// node (:3717-3726) that relaunches ~10 kernels per iteration until every world is done.
//
// Here a world's Jacobian (nefc x nv), Hessian, its Cholesky factor, CSR inertia and all solver vectors live in the
// warp's shared-memory slice for the whole solve; iterations are a device-side loop, so a world stops as soon as IT has
// converged (no global `nsolving` counter, no graph conditional).  Reductions are warp shuffles; the Hessian is updated
// incrementally from the rows whose QUADRATIC flag flipped (exactly the reference's rule) and refactored in place.
// Algorithm and tolerances follow the reference: exact Newton with the iterative bracketing line search on the
// shifted (cost(alpha) - cost(0)) piecewise-quadratic 1-D cost.  Pyramidal / frictionless / limit / dof-friction rows
// in the default instantiation; k_solver<true> adds elliptic cones (solver.py:286-477 zones, :957-1015 per-contact
// quads, :2443-2565 cone Hessian) with the Hessian rebuilt from M every iteration like the reference's elliptic path.
#include <cstdlib>

#include "mjb_chol.cuh"
#include "mjb_linesearch.cuh"
#include "mjb_team.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

namespace {

// Shared-memory slice of one world.  J rows keep the global stride nv_pad (a multiple of 4 floats), so a row is 16-byte
// aligned: staging is a straight float4 copy and row-times-vector products use LDS.128 (a quarter-warp of 112-byte-strided
// rows is bank-conflict free).  Per-dof vectors are padded to nv_pad with zeros so the float4 loops need no tail handling.
struct SolLayout { int J, vec, H, Lf, M, rowf, rowi, ldJ, ldH, nvp, nrowf, jcap, cgv, red, env, bar, total; };
// rows of shared memory a world gets: d.rowcap for a row-capacity class launch (see launch_solver), else njmax
__host__ __device__ inline int sol_rowcap(const DataDev& d) { return d.rowcap > 0 ? d.rowcap : d.njmax; }
__host__ __device__ inline SolLayout sol_layout(const ModelDev& m, const DataDev& d, bool big) {
  SolLayout L;
  const int cap = sol_rowcap(d);
  int o = 0;
  auto take = [&](int n) { int r = o; o += (n + 3) & ~3; return r; };
  L.nvp = d.nv_pad; L.ldJ = d.nv_pad; L.ldH = m.nv | 1;
  // nv > 32 ("big" models, e.g. unitree G1, three_humanoids): only the first d.jcap Jacobian rows are staged in shared memory,
  // the rest is read from global memory (L2 hits).  d.jcap defaults to 0: occupancy beats the shorter access (see capi.cu).
  L.jcap = big ? (cap < d.jcap ? cap : d.jcap) : cap;
  L.J = take(L.jcap * L.ldJ);
  L.vec = take(7 * L.nvp);  // qacc, Ma, grad, search, mv (= x scratch of the nv > 32 path), qfs, qfc
  L.cgv = take(m.solver == SOL_CG ? 3 * L.nvp : 0);  // CG only: Mgrad, prev_grad, prev_Mgrad
  // nv <= 32: H and its factor are stored as packed lower triangles (register Cholesky path); larger nv keeps nv x ldH
  // H and its factor are packed lower triangles (register Cholesky for nv <= 32, shared-memory Cholesky above)
  const int hsz = m.nv * (m.nv + 1) / 2;
  L.H = take(hsz);
  // nv <= 32: the factor lives in the padded column layout of chol_solve_rows_bcast, and M is kept as a dense packed lower
  // triangle (H starts as a copy of it, M * v needs no index tables); nv > 32: packed factor, CSR M with gather tables
  L.Lf = take(big ? hsz : cholpair_size(m.nv <= 8 ? 8 : m.nv <= 16 ? 16 : m.nv <= 24 ? 24 : m.nv <= 28 ? 28 : 32));  // padded size of the register path (>= colsub_off of the same size)
  L.M = take(big ? m.nC : hsz);
  // Jaref, jv (= hw: the H-update weights live only between update_constraint and update_search), D, force [, floss]
  // elliptic cones add: per-row friction scale, 3 quad words per row (solver.py:1008-1015 layout), row->contact info
  const bool ell = m.cone == CONE_ELLIPTIC;
  L.nrowf = ((m.nfricdof + m.ntenfric) > 0 ? 5 : 4);
  L.rowf = take((L.nrowf + (ell ? 4 : 0)) * cap);
  L.rowi = take((ell ? 3 : 2) * cap);
  L.red = take(big ? 9 * 8 : 0);  // cross-warp reduction scratch of the multi-warp (nv > 32) instantiations
  // nv > 32: nonzero column range of every Jacobian row (lo | hi << 16) and the Hessian's row envelope (first column per row)
  L.env = take(big ? cap + L.nvp : 0);
  L.bar = take(4);  // mbarrier of the bulk-async staging (8 bytes, 16-byte slot)
  L.total = o;
  return L;
}

// ---- team = the NW warps (one block) that own a world.  NW = 1: plain warp primitives.  NW > 1 (models with nv > 32, where a
// world's slice of shared memory caps the SM at a few resident worlds): block barriers, and reductions that finish in shared
// memory in a fixed order so every thread sees the same bits.
template <int NW> __device__ __forceinline__ void tsync() { if (NW == 1) __syncwarp(); else __syncthreads(); }
template <int NW, int N>
__device__ __forceinline__ void tsum_n(float (&v)[N], float* red) {
#pragma unroll
  for (int k = 0; k < N; k++) v[k] = warp_sum(v[k]);
  if (NW == 1) return;
  const int warp = threadIdx.x >> 5;
  __syncthreads();  // the previous reduction's readers are done with `red`
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < N; k++) red[warp * N + k] = v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < N; k++) {
    float t = red[k];
#pragma unroll
    for (int w = 1; w < NW; w++) t += red[w * N + k];
    v[k] = t;
  }
}
template <int NW> __device__ __forceinline__ float tsum(float v, float* red) { float a[1] = {v}; tsum_n<NW, 1>(a, red); return a[0]; }
template <int NW> __device__ __forceinline__ P3 tsum3(P3 p, float* red) { float a[3] = {p.c, p.g, p.h}; tsum_n<NW, 3>(a, red); return mkp(a[0], a[1], a[2]); }
template <int NW> __device__ __forceinline__ void tcopy(float* dst, const float* src, int n, int tid) {
#pragma unroll 1  // n is a per-dof count: one or two trips; the unrolled-by-16 form the compiler picks costs ~45 instructions per call (solver 206 -> 202 us)
  for (int i = tid; i < n; i += 32 * NW) dst[i] = src[i];
}

// dot of a 16B-aligned J row with a zero-padded, 16B-aligned per-dof vector
__device__ __forceinline__ float row_dot(const float* Jr, const float* vec, int nvp) {
  float s = 0.f;
#pragma unroll 4
  for (int k = 0; k < nvp; k += 4) {
    const float4 a = *reinterpret_cast<const float4*>(Jr + k), b = *reinterpret_cast<const float4*>(vec + k);
    s += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
  }
  return s;
}

struct Ctx {
  const ModelDev* m;
  int lane, nv, nvp, nefc, ne, nf, ldJ, ldH;
  float *J, *H, *Lf, *M, *qacc, *Ma, *grad, *search, *mv, *qfs, *x, *qfc;
  float *Jaref, *jv, *D, *force, *floss, *hw;
  int *state, *hidx;
  float search_dot, grad_dot, newton_decrement, improvement;
  // elliptic only: rinfo[r] = -1 (not an elliptic row) | -2 (contact cut by njmax) | (dim << 4) | j;  rfri[r] = mu (j = 0)
  // or friction[j-1];  quad = 3 words per row;  the CONE contacts' primary rows are listed from the END of hidx
  int* rinfo; float *rfri, *quad; int njmax, ncone;
  const float* Jg; int jcap;  // big models: rows >= jcap live in global memory (same leading dimension)
  float* cgv;                 // CG only: Mgrad, prev_grad, prev_Mgrad (nvp each)
  float* red;                 // NW > 1: cross-warp reduction scratch (9 floats per warp)
  int *rng, *fz;              // nv > 32: Jacobian row ranges, Hessian row envelope
  bool env;                   // ranges / envelope in use (several kinematic trees: the Hessian is close to block diagonal)
  float chol_inv;             // nv <= 32: lane j keeps 1 / L_jj of the factor in Lf
  int chol_off;               // nv <= 32: where lane j's column of the factor starts in Lf (paired-column layout)
  bool factored;              // Lf holds the factor of the current H
};
template <bool BIG>
__device__ __forceinline__ const float* jrow(const Ctx& c, int r) {
  if (BIG && r >= c.jcap) return c.Jg + (size_t)r * c.ldJ;
  return c.J + r * c.ldJ;
}
__device__ __forceinline__ EllQ ell_load(const Ctx& c, int r) {
  const float* q = c.quad + 3 * r;
  EllQ e; e.q0 = q[0]; e.q1 = q[1]; e.q2 = q[2]; e.u0 = q[3]; e.v0 = q[4]; e.uu = q[5]; e.uv = q[6]; e.vv = q[7]; e.dm = q[8];
  return e;
}

// res = M vec (support.py:153 mul_m).  nv <= 32: M is a dense packed lower triangle in shared memory, lane i walks row i up to the
// diagonal and column i below it -- no index tables, no global loads (the CSR gather's table lookups were the top long-scoreboard line
// of the solver).  A fully unrolled variant with predicated loads (4 instead of 9 instructions per entry) measured SLOWER: 245 vs 206 us.
// nv > 32: the symmetric gather tables (io.py:1029-1050).
template <int NW, bool BIG>
__device__ __forceinline__ void mul_m(const Ctx& c, const float* vec, float* res) {
  const ModelDev& m = *c.m;
  if (!BIG) {
    const int i = c.lane, nv = c.nv;
    if (i < nv) {
      const float* Mi = c.M + (i * (i + 1)) / 2;
      float acc = 0.f;
      int tk = 0;  // k (k + 1) / 2
#pragma unroll 4
      for (int k = 0; k < nv; k++) {
        const float mk = k <= i ? Mi[k] : c.M[tk + i];
        acc += mk * vec[k];
        tk += k + 1;
      }
      res[i] = acc;
    }
    return;
  }
#pragma unroll 1
  for (int i = c.lane; i < c.nv; i += 32 * NW) {
    float acc = 0.f;
#pragma unroll 4
    for (int k = m.mulm_rowadr[i]; k < m.mulm_rowadr[i + 1]; k++) acc += c.M[m.mulm_madr[k]] * vec[m.mulm_col[k]];
    res[i] = acc;
  }
}

// force/state per row, qfrc_constraint = J^T force, and the list of rows whose QUADRATIC flag changed
// (init=true: list every QUADRATIC row with weight +D).  Returns the list length.
template <bool ELL, bool BIG, int NW>
__device__ __forceinline__ int update_constraint(Ctx& c, bool init) {
  int nlist = 0, ncone = 0;
  if (ELL) init = true;  // elliptic: H is rebuilt from M, so every QUADRATIC row is listed
  // the row pass (a handful of flops per row, ordered compaction by ballot) stays on the first warp of the team
#pragma unroll 1
  for (int r0 = 0; r0 < ((NW == 1 || c.lane < 32) ? c.nefc : 0); r0 += 32) {
    const int r = r0 + c.lane;
    bool flip = false, cone0 = false;
    float wgt = 0.f;
    if (r < c.nefc) {
      const float jaref = c.Jaref[r], D = c.D[r];
      const int old = c.state[r];
      float force; int st;
      if (r < c.ne) { force = -D * jaref; st = ST_QUADRATIC; }
      else if (r < c.ne + c.nf) {
        const float f = c.floss[r], rf = safe_div(f, D);
        if (jaref <= -rf) { force = f; st = ST_LINEARNEG; } else if (jaref >= rf) { force = -f; st = ST_LINEARPOS; } else { force = -D * jaref; st = ST_QUADRATIC; }
      } else if (ELL && c.rinfo[r] != -1) {  // solver.py:455-472
        const int info = c.rinfo[r];
        force = 0.f; st = ST_SATISFIED;
        if (info >= 0) {
          const int j = info & 15, dim = info >> 4, e0 = r - j;
          const float mu = c.rfri[e0], N = c.Jaref[e0] * mu;
          float TT = 0.f;
          for (int i = 1; i < dim; i++) { const float u = c.Jaref[e0 + i] * c.rfri[e0 + i]; TT += u * u; }
          const float T = TT <= 0.f ? 0.f : sqrtf(TT);
          if ((N >= mu * T) || (T <= 0.f && N >= 0.f)) {}
          else if ((mu * N + T <= 0.f) || (T <= 0.f && N < 0.f)) { force = -D * jaref; st = ST_QUADRATIC; }
          else {
            const float dm = safe_div(c.D[e0], mu * mu * (1.0f + mu * mu)), fn = -dm * (N - mu * T) * mu, fr = c.rfri[r];
            force = j == 0 ? fn : -safe_div(fn, T) * (jaref * fr * fr);
            st = ST_CONE;
            cone0 = j == 0;
          }
        }
      } else if (jaref >= 0.f) { force = 0.f; st = ST_SATISFIED; }
      else { force = -D * jaref; st = ST_QUADRATIC; }
      c.force[r] = force; c.state[r] = st;
      const bool nq = st == ST_QUADRATIC, oq = (!init) && old == ST_QUADRATIC;
      flip = nq != oq;
      wgt = nq ? D : -D;
    }
    const unsigned bal = __ballot_sync(FULL_MASK, flip);
    if (flip) { const int p = nlist + __popc(bal & ((1u << c.lane) - 1u)); c.hidx[p] = r; c.hw[p] = wgt; }
    nlist += __popc(bal);
    if (ELL) {
      const unsigned cb = __ballot_sync(FULL_MASK, cone0);
      if (cone0) c.hidx[c.njmax - 1 - (ncone + __popc(cb & ((1u << c.lane) - 1u)))] = r;
      ncone += __popc(cb);
    }
  }
  if (NW > 1) {  // hand the two counts to the other warps
    if (c.lane == 0) { c.red[0] = __int_as_float(nlist); c.red[1] = __int_as_float(ncone); }
    __syncthreads();
    nlist = __float_as_int(c.red[0]); ncone = __float_as_int(c.red[1]);
  }
  c.ncone = ncone;
  tsync<NW>();
#pragma unroll 1
  for (int dd = c.lane; dd < c.nv; dd += 32 * NW) {
    float s = 0.f;
#pragma unroll 8
    for (int r = 0; r < c.nefc; r++) s += jrow<BIG>(c, r)[dd] * c.force[r];
    c.qfc[dd] = s;
  }
  tsync<NW>();
  return nlist;
}

// grad = Ma - qfrc_smooth - qfrc_constraint and its squared norm
template <int NW>
__device__ __forceinline__ void update_grad(Ctx& c) {
  float gd = 0.f;
#pragma unroll 1
  for (int dd = c.lane; dd < c.nv; dd += 32 * NW) { const float g = c.Ma[dd] - c.qfs[dd] - c.qfc[dd]; c.grad[dd] = g; gd += g * g; }
  c.grad_dot = tsum<NW>(gd, c.red);
  tsync<NW>();
}

// Newton direction for nv <= 32: lane i keeps row i of H in registers, adds w * J_r[i] * J_r[:] for every listed row r
// (J_r[:] read with broadcast LDS.128), stores the updated row back, and hands the registers straight to the Cholesky sweep.
// Elliptic cone term of one CONE-state contact as `dim` rank-1 updates (solver.py:2443-2565 regrouped): with
// z0 = mu J0, p = sum_j u_j s_j J_j (u_j = Jaref_j s_j, s_j = friction_j-1),
//   dH = dm [ z0 z0^T - mu/t (z0 p^T + p z0^T) + mu n / t^3 p p^T + (mu^2 - n mu / t) sum_j s_j^2 J_j J_j^T ]
// so row i receives cA_i J0[:] + sum_j c_ji J_j[:].  Returns the per-contact scalars; the caller applies the updates.
struct ConeK { float dm, mu, mu_tinv, munttt, tdiag; int dim; };
__device__ __forceinline__ ConeK cone_scalars(const Ctx& c, int e0) {
  ConeK k;
  k.dim = c.rinfo[e0] >> 4; k.mu = c.rfri[e0];
  const float mu2 = k.mu * k.mu;
  k.dm = safe_div(c.D[e0], mu2 * (1.0f + mu2));
  const float n = c.Jaref[e0] * k.mu;
  float tt = 0.f;
  for (int j = 1; j < k.dim; j++) { const float u = c.Jaref[e0 + j] * c.rfri[e0 + j]; tt += u * u; }
  const float t = fmaxf(sqrtf(tt), MJ_MINVAL), ttt = fmaxf(t * t * t, MJ_MINVAL);
  k.mu_tinv = safe_div(k.mu, t); k.munttt = k.mu * safe_div(n, ttt); k.tdiag = mu2 - n * k.mu_tinv;
  return k;
}
// coefficient of row e0 + j's rank-1 update for Hessian row i, given J0[i], p_i
__device__ __forceinline__ float cone_coef(const Ctx& c, const ConeK& k, int e0, int j, float J0i, float pi, float Jji) {
  if (j == 0) return k.dm * k.mu * (k.mu * J0i - k.mu_tinv * pi);
  const float s = c.rfri[e0 + j], us = c.Jaref[e0 + j] * s * s;
  return k.dm * ((k.munttt * pi - k.mu_tinv * k.mu * J0i) * us + k.tdiag * s * s * Jji);
}

template <int N, bool ELL>
__device__ __forceinline__ float newton_direction_reg(Ctx& c, int nlist, float g) {
  const int lane = c.lane, nv = c.nv;
  float a[N];
  chol_load_rows<N, true>(a, c.H, c.ldH, nv, lane);
  if (nlist > 0) {
#pragma unroll 2
    for (int t = 0; t < nlist; t++) {
      const float* Jr = c.J + c.hidx[t] * c.ldJ;
      const float sc = lane < nv ? c.hw[t] * Jr[lane] : 0.f;
#pragma unroll
      for (int k = 0; k < N; k += 4) {
        const float4 v = *reinterpret_cast<const float4*>(Jr + k);
        a[k] += sc * v.x; a[k + 1] += sc * v.y; a[k + 2] += sc * v.z; a[k + 3] += sc * v.w;
      }
    }
    if (!ELL && lane < nv) {  // elliptic keeps c.H == M: the next iteration rebuilds from it
      const int base = (lane * (lane + 1)) / 2;
#pragma unroll
      for (int k = 0; k < N; k++)
        if (k <= lane) c.H[base + k] = a[k];
    }
    // columns >= nv of rows < nv only ever hold the unused upper triangle; rows >= nv stay identity (sc == 0)
  }
  if (ELL) {
#pragma unroll 1
    for (int t = 0; t < c.ncone; t++) {
      const int e0 = c.hidx[c.njmax - 1 - t];
      const ConeK k = cone_scalars(c, e0);
      if (k.dm == 0.f) continue;
      const float* J0 = c.J + e0 * c.ldJ;
      const float J0i = lane < nv ? J0[lane] : 0.f;
      float pi = 0.f;
      for (int j = 1; j < k.dim; j++) pi += c.Jaref[e0 + j] * c.rfri[e0 + j] * c.rfri[e0 + j] * (lane < nv ? J0[j * c.ldJ + lane] : 0.f);
#pragma unroll 1
      for (int j = 0; j < k.dim; j++) {
        const float* Jr = J0 + j * c.ldJ;
        const float sc = lane < nv ? cone_coef(c, k, e0, j, J0i, pi, Jr[lane]) : 0.f;
#pragma unroll
        for (int q = 0; q < N; q += 4) {
          const float4 v = *reinterpret_cast<const float4*>(Jr + q);
          a[q] += sc * v.x; a[q + 1] += sc * v.y; a[q + 2] += sc * v.z; a[q + 3] += sc * v.w;
        }
      }
    }
  }
#ifdef MJB_CHOL_UNROLLED  // off by default: the straight-line sweep misses the instruction cache (see mjb_chol.cuh)
  return chol_solve_rows_unrolled<N>(a, nv, g, c.Lf, lane);
#else
  c.factored = true;
#ifdef MJB_CHOL_SINGLE  // one column per sweep (humanoid solver 216 us)
  return chol_solve_rows_bcast<N>(a, nv, g, c.Lf, lane, c.chol_inv);
#else
  return chol_solve_rows_pair<N>(a, nv, g, c.Lf, lane, c.chol_inv, c.chol_off);
#endif
#endif
}

// H += sum_list w J J^T (lower triangle), Cholesky, search = -H^-1 grad, Newton decrement
template <bool ELL, bool BIG, int NW, int NREG = 0>
__device__ __forceinline__ void update_search(Ctx& c, int nlist) {
  const int nv = c.nv;
  float sd = 0.f, nd = 0.f;
  if (!BIG) {  // nv <= 32 (launch_solver picks the instantiation)
    const float g = c.lane < nv ? c.grad[c.lane] : 0.f;
    float xx;
    // no row changed state since the last factorisation: H is what was factored, only the right-hand side is new (the reference's
    // stable-state shortcut, solver.py:2145-2159, which reuses the whole direction instead)
#ifdef MJB_CHOL_SINGLE
    if (!ELL && nlist == 0 && c.factored) xx = chol_subst_bcast(nv, g, c.Lf, c.lane, c.chol_inv);
#else
    if (!ELL && nlist == 0 && c.factored) xx = chol_subst_pair(nv, g, c.Lf, c.lane, c.chol_inv, c.chol_off);
#endif
    else if (NREG == 28) xx = newton_direction_reg<28, ELL>(c, nlist, g);  // register-row size fixed by the launcher: one variant in the kernel
    else if (NREG == 32) xx = newton_direction_reg<32, ELL>(c, nlist, g);
    else if (nv <= 8) xx = newton_direction_reg<8, ELL>(c, nlist, g);
    else if (nv <= 16) xx = newton_direction_reg<16, ELL>(c, nlist, g);
    else if (nv <= 24) xx = newton_direction_reg<24, ELL>(c, nlist, g);
    else if (nv <= 28) xx = newton_direction_reg<28, ELL>(c, nlist, g);
    else xx = newton_direction_reg<32, ELL>(c, nlist, g);
    sd = xx * xx; nd = g * xx;
    if (c.lane < nv) c.search[c.lane] = -xx;
  } else {
    // nv > 32: packed lower triangle in shared memory, worked on by the whole team
    constexpr int NT = 32 * NW;
    const int ntri = nv * (nv + 1) / 2;
    float* Hd = ELL ? c.Lf : c.H;  // elliptic: rebuild into Lf from M (c.H) every iteration
    if (ELL) {
#pragma unroll 1
      for (int e = c.lane; e < ntri; e += NT) c.Lf[e] = c.H[e];
      tsync<NW>();
    }
    if (NW == 1) {  // one warp: lane owns rows lane, lane + 32, ...
#pragma unroll 1
      for (int t = 0; t < nlist; t++) {
        const float* Jr = jrow<true>(c, c.hidx[t]);
        const float wt = c.hw[t];
        const int lo = c.env ? (c.rng[c.hidx[t]] & 0xFFFF) : 0, hi = c.env ? (c.rng[c.hidx[t]] >> 16) : nv;  // the row is zero outside [lo, hi)
#pragma unroll 1
        for (int i = lo + ((c.lane - lo) & 31); i < hi; i += 32) {  // row i always belongs to lane i % 32, whatever the row range
          const float sc = wt * Jr[i];
          float* Hi = Hd + (i * (i + 1)) / 2;
          if (sc != 0.f)
#pragma unroll 4
            for (int k = lo; k <= i; k++) Hi[k] += sc * Jr[k];
        }
      }
    } else if (nlist > 0) {  // team: every thread owns entries (i, k) of the triangle and sums the listed rows' contributions
#pragma unroll 1
      for (int e = c.lane; e < ntri; e += NT) {
        int i = (int)((sqrtf(8.0f * (float)e + 1.0f) - 1.0f) * 0.5f);
        while ((i + 1) * (i + 2) / 2 <= e) i++;
        while (i * (i + 1) / 2 > e) i--;
        const int k = e - i * (i + 1) / 2;
        float acc = 0.f;
#pragma unroll 4
        for (int t = 0; t < nlist; t++) { const float* Jr = jrow<true>(c, c.hidx[t]); acc += c.hw[t] * Jr[i] * Jr[k]; }
        Hd[e] += acc;
      }
    }
    if (ELL) {
      tsync<NW>();
#pragma unroll 1
      for (int t = 0; t < c.ncone; t++) {
        const int e0 = c.hidx[c.njmax - 1 - t];
        const ConeK k = cone_scalars(c, e0);
        if (k.dm == 0.f) continue;
        const float* J0 = jrow<true>(c, e0);
#pragma unroll 1
        for (int i = c.lane; i < nv; i += NT) {
          float pi = 0.f;
          for (int q = 1; q < k.dim; q++) pi += c.Jaref[e0 + q] * c.rfri[e0 + q] * c.rfri[e0 + q] * jrow<true>(c, e0 + q)[i];
          float* Hi = Hd + (i * (i + 1)) / 2;
          for (int q = 0; q < k.dim; q++) {
            const float* Jq = jrow<true>(c, e0 + q);
            const float sc = cone_coef(c, k, e0, q, J0[i], pi, Jq[i]);
            for (int kk = 0; kk <= i; kk++) Hi[kk] += sc * Jq[kk];
          }
        }
      }
    }
    tsync<NW>();
    if (!ELL) {
#pragma unroll 1
      for (int e = c.lane; e < ntri; e += NT) c.Lf[e] = c.H[e];
    }
#pragma unroll 1
    for (int dd = c.lane; dd < nv; dd += NT) c.x[dd] = c.grad[dd];
    tsync<NW>();
    if (NW == 1) {
      if (c.env) {
        warp_cholesky_packed_env(c.Lf, nv, c.fz, c.lane);
        warp_chol_solve_packed_env(c.Lf, nv, c.fz, c.x, c.lane);
      } else {
        warp_cholesky_packed(c.Lf, nv, c.lane);
        warp_chol_solve_packed(c.Lf, nv, c.x, c.lane);
      }
    } else {
      team_cholesky_packed<NW>(c.Lf, nv, c.lane);
      team_chol_solve_packed<NW>(c.Lf, nv, c.x, c.lane);
    }
#pragma unroll 1
    for (int dd = c.lane; dd < nv; dd += NT) { const float xx = c.x[dd]; sd += xx * xx; nd += c.grad[dd] * xx; c.search[dd] = -xx; }
  }
  { float a[2] = {sd, nd}; tsum_n<NW, 2>(a, c.red); c.search_dot = a[0]; c.newton_decrement = a[1]; }
  tsync<NW>();
}

template <bool ELL, int NW>
__device__ __forceinline__ P3 eval_total(const Ctx& c, float alpha, float q0, float q1, float q2) {
  P3 s = mkp(0.f, 0.f, 0.f);
#pragma unroll 1
  for (int r = c.lane; r < c.nefc; r += 32 * NW) {
    if (ELL && c.rinfo[r] != -1) {
      if (c.rinfo[r] >= 0 && (c.rinfo[r] & 15) == 0) { const EllQ q = ell_load(c, r); const float mu = c.rfri[r]; s = s + ell_shifted(mu, q, ell_reference(mu, q), alpha); }
    } else s = s + eval_row(r, alpha, c.ne, c.nf, c.D[r], c.floss[r], c.Jaref[r], c.jv[r]);
  }
  return eval_gauss(q0, q1, q2, alpha) + tsum3<NW>(s, c.red);
}

// solver.py:836-1347; returns true when the line search converged
template <bool ELL, bool BIG, int NW>
__device__ __forceinline__ bool linesearch(Ctx& c) {
  const ModelDev& m = *c.m;
  const int nv = c.nv;
  constexpr int NT = 32 * NW;
  mul_m<NW, BIG>(c, c.search, c.mv);
#pragma unroll 1
  for (int r = c.lane; r < c.nefc; r += NT) {
    c.jv[r] = row_dot(jrow<BIG>(c, r), c.search, c.nvp);
  }
  tsync<NW>();
  const float snorm = sqrtf(c.search_dot), scale = m.meaninertia * (float)nv;
  const float gtol = fmaxf(m.tolerance * m.ls_tolerance * snorm * scale, 1e-6f);
  P3 p0s = mkp(0.f, 0.f, 0.f);
  if (ELL) {  // per-contact quads at the primary rows (solver.py:957-1015)
#pragma unroll 1
    for (int r = c.lane; r < c.nefc; r += NT) {
      const int info = c.rinfo[r];
      if (info < 0 || (info & 15) != 0) continue;
      const int dim = info >> 4;
      const float mu = c.rfri[r], ja = c.Jaref[r], jv = c.jv[r], D = c.D[r], jvD = jv * D;
      float q0 = 0.5f * ja * ja * D, q1 = jvD * ja, q2 = 0.5f * jv * jvD, uu = 0.f, uv = 0.f, vv = 0.f;
      for (int j = 1; j < dim; j++) {
        const float jvj = c.jv[r + j], jaj = c.Jaref[r + j], dj = c.D[r + j], DJ = dj * jaj, fj = c.rfri[r + j];
        q0 += 0.5f * jaj * DJ; q1 += jvj * DJ; q2 += 0.5f * jvj * dj * jvj;
        const float uj = jaj * fj, vj = jvj * fj;
        uu += uj * uj; uv += uj * vj; vv += vj * vj;
      }
      float* q = c.quad + 3 * r;
      const float mu2 = mu * mu;
      q[0] = q0; q[1] = q1; q[2] = q2; q[3] = ja * mu; q[4] = jv * mu; q[5] = uu; q[6] = uv; q[7] = vv; q[8] = D / (mu2 * (1.0f + mu2));
    }
    tsync<NW>();
  }
#pragma unroll 1
  for (int r = c.lane; r < c.nefc; r += NT) {
    if (ELL && c.rinfo[r] != -1) {
      if (c.rinfo[r] >= 0 && (c.rinfo[r] & 15) == 0) p0s = p0s + ell_zero(c.rfri[r], ell_load(c, r));
    } else p0s = p0s + eval_row_zero(r, c.ne, c.nf, c.D[r], c.floss[r], c.Jaref[r], c.jv[r]);
  }
  float g1 = 0.f, g2 = 0.f;
#pragma unroll 1
  for (int dd = c.lane; dd < nv; dd += NT) { const float s = c.search[dd]; g1 += s * (c.Ma[dd] - c.qfs[dd]); g2 += 0.5f * s * c.mv[dd]; }
  float q1, q2;
  { float a[5] = {p0s.c, p0s.g, p0s.h, g1, g2}; tsum_n<NW, 5>(a, c.red); p0s = mkp(a[0], a[1], a[2]); q1 = a[3]; q2 = a[4]; }
  const float q0 = 0.f;
  const P3 p0 = mkp(q0 + p0s.c, q1 + p0s.g, 2.0f * q2 + p0s.h);
  const P3 p0_delta = mkp(0.f, p0.g, p0.h);
  const float lo_alpha_in = -safe_div(p0.g, p0.h);
  const P3 lo_in = eval_total<ELL, NW>(c, lo_alpha_in, q0, q1, q2);
  const bool initial_converged = fabsf(lo_in.g) < gtol && lo_in.c < 0.f;
  bool ls_converged = initial_converged;
  float alpha = 0.f, improvement = 0.f;
  if (!initial_converged) {
    const bool lo_less = lo_in.g < p0.g;
    P3 lo = lo_less ? lo_in : p0_delta, hi = lo_less ? p0_delta : lo_in;
    float lo_alpha = lo_less ? lo_alpha_in : 0.f, hi_alpha = lo_less ? 0.f : lo_alpha_in;
#pragma unroll 1
    for (int it = 0; it < m.ls_iterations; it++) {
      const float lo_next_alpha = lo_alpha - safe_div(lo.g, lo.h), hi_next_alpha = hi_alpha - safe_div(hi.g, hi.h), mid_alpha = 0.5f * (lo_alpha + hi_alpha);
      P3 sl = mkp(0.f, 0.f, 0.f), sh = sl, sm = sl;
#pragma unroll 1
      for (int r = c.lane; r < c.nefc; r += NT) {
        if (ELL && c.rinfo[r] != -1) {
          if (c.rinfo[r] >= 0 && (c.rinfo[r] & 15) == 0) {
            const EllQ q = ell_load(c, r); const float mu = c.rfri[r]; const EllRef e = ell_reference(mu, q);
            sl = sl + ell_shifted(mu, q, e, lo_next_alpha); sh = sh + ell_shifted(mu, q, e, hi_next_alpha); sm = sm + ell_shifted(mu, q, e, mid_alpha);
          }
          continue;
        }
        const float D = c.D[r], f = c.floss[r], ja = c.Jaref[r], jv = c.jv[r];
        sl = sl + eval_row(r, lo_next_alpha, c.ne, c.nf, D, f, ja, jv);
        sh = sh + eval_row(r, hi_next_alpha, c.ne, c.nf, D, f, ja, jv);
        sm = sm + eval_row(r, mid_alpha, c.ne, c.nf, D, f, ja, jv);
      }
      {
        float a[9] = {sl.c, sl.g, sl.h, sh.c, sh.g, sh.h, sm.c, sm.g, sm.h};
        tsum_n<NW, 9>(a, c.red);
        sl = mkp(a[0], a[1], a[2]); sh = mkp(a[3], a[4], a[5]); sm = mkp(a[6], a[7], a[8]);
      }
      const P3 lo_next = eval_gauss(q0, q1, q2, lo_next_alpha) + sl;
      const P3 hi_next = eval_gauss(q0, q1, q2, hi_next_alpha) + sh;
      const P3 mid = eval_gauss(q0, q1, q2, mid_alpha) + sm;
      const bool s1 = in_bracket(lo, lo_next); if (s1) { lo = lo_next; lo_alpha = lo_next_alpha; }
      const bool s2 = in_bracket(lo, mid); if (s2) { lo = mid; lo_alpha = mid_alpha; }
      const bool s3 = in_bracket(lo, hi_next); if (s3) { lo = hi_next; lo_alpha = hi_next_alpha; }
      const bool h1 = in_bracket(hi, hi_next); if (h1) { hi = hi_next; hi_alpha = hi_next_alpha; }
      const bool h2 = in_bracket(hi, mid); if (h2) { hi = mid; hi_alpha = mid_alpha; }
      const bool h3 = in_bracket(hi, lo_next); if (h3) { hi = lo_next; hi_alpha = lo_next_alpha; }
      const bool swap_lo = s1 || s2 || s3, swap_hi = h1 || h2 || h3;
      const bool ls_done = (!swap_lo && !swap_hi) || (lo.c < 0.f && lo.g < 0.f && lo.g > -gtol) || (hi.c < 0.f && hi.g > 0.f && hi.g < gtol);
      const bool improved = lo.c < 0.f || hi.c < 0.f, lo_better = lo.c < hi.c;
      if (improved) { alpha = lo_better ? lo_alpha : hi_alpha; improvement = -(lo_better ? lo.c : hi.c); }
      if (ls_done) { ls_converged = true; break; }
    }
  } else {
    alpha = lo_alpha_in; improvement = -lo_in.c;
  }
#pragma unroll 1
  for (int dd = c.lane; dd < nv; dd += NT) { c.qacc[dd] += alpha * c.search[dd]; c.Ma[dd] += alpha * c.mv[dd]; }
#pragma unroll 1
  for (int r = c.lane; r < c.nefc; r += NT) c.Jaref[r] += alpha * c.jv[r];
  c.improvement = improvement;
  tsync<NW>();
  return ls_converged;
}

// Conjugate-gradient direction (solver.py:1665 _solve_init_search_cg, :3295 beta, :3360 search update): Mgrad = M^-1 grad
// through the per-tree factor U (M = U^T U) that fwd_acceleration left in Data.qLD, Polak-Ribiere beta, search update.
// Only the CG instantiations of the kernel contain it.
__device__ __forceinline__ void cg_direction(Ctx& c, const ModelDev& m, const DataDev& d, size_t wb, bool init) {
  const int nv = c.nv, lane = c.lane;
  float *Mg = c.cgv, *pg = c.cgv + c.nvp, *pMg = c.cgv + 2 * c.nvp;
#pragma unroll 1
  for (int dd = lane; dd < nv; dd += 32) Mg[dd] = c.grad[dd];
  __syncwarp();
#pragma unroll 1
  for (int t = 0; t < m.ntree; t++) {
    const int start = m.tree_dofadr[t], n = m.tree_dofnum[t];
    const float* U = d.qLD + wb * m.qld_total + m.tree_qLDadr[t];
    float* xt = Mg + start;
#pragma unroll 1
    for (int j = 0; j < n; j++) {
      const float zj = xt[j] / U[j * n + j];
      __syncwarp();
      for (int i = j + 1 + lane; i < n; i += 32) xt[i] -= U[j * n + i] * zj;
      if (lane == 0) xt[j] = zj;
      __syncwarp();
    }
#pragma unroll 1
    for (int j = n - 1; j >= 0; j--) {
      const float xj = xt[j] / U[j * n + j];
      __syncwarp();
      for (int i = lane; i < j; i += 32) xt[i] -= U[i * n + j] * xj;
      if (lane == 0) xt[j] = xj;
      __syncwarp();
    }
  }
  float beta = 0.f;
  if (!init) {
    float num = 0.f, den = 0.f;
#pragma unroll 1
    for (int dd = lane; dd < nv; dd += 32) { num += c.grad[dd] * (Mg[dd] - pMg[dd]); den += pg[dd] * pMg[dd]; }
    beta = fmaxf(0.f, warp_sum(num) / fmaxf(MJ_MINVAL, warp_sum(den)));
  }
  float sd = 0.f;
#pragma unroll 1
  for (int dd = lane; dd < nv; dd += 32) {
    const float sv = -Mg[dd] + beta * c.search[dd];
    c.search[dd] = sv; sd += sv * sv;
    pg[dd] = c.grad[dd]; pMg[dd] = Mg[dd];
  }
  c.search_dot = warp_sum(sd);
  __syncwarp();
}

// nv <= 32: 16 one-warp blocks per SM need <= 128 registers per thread (the register file is split per scheduler: 136 registers
// already drop an SM from 16 to 12 resident worlds -- measured 206 -> 250 us on the humanoid)
// PLAIN: the model can produce neither equality nor friction-loss rows (no equalities, no dof / tendon frictionloss), so every row is
// an inequality: ne = nf = 0 become compile-time constants and the two other row kinds drop out of the line search and the row pass
template <bool ELL, bool BIG, bool CG, int NW, bool PLAIN = false, int NREG = 0>
__global__ void __launch_bounds__(NW * 32, (NW == 1 && !BIG) ? 16 : 1)
k_solver(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d) {
  extern __shared__ float smem[];
  constexpr int NT = 32 * NW;
  const int lane = threadIdx.x;  // index inside the team of NW warps (one block) that owns the world
  int w = blockIdx.x + d.w0;
  if (d.rowcap > 0) {  // row-capacity class launch: the block's world comes from the class list
    if ((int)blockIdx.x >= d.sol_count[2 * d.split_id + d.sol_class]) return;
    w = d.sol_list[(size_t)d.sol_class * d.nworld + d.w0 + blockIdx.x];
  }
  if (w >= d.nworld) return;
  const SolLayout L = sol_layout(m, d, BIG);
  float* S = smem;
  const int nv = m.nv, njmax = d.njmax, nvp = d.nv_pad;
  const int cap = sol_rowcap(d);  // rows of this world's shared-memory slice (njmax, or the row-capacity class of this launch)
  const size_t wb = (size_t)w;
  Ctx c;
  c.factored = false; c.chol_inv = 1.0f; c.chol_off = 0;
  c.m = &m; c.lane = lane; c.nv = nv; c.nvp = L.nvp; c.ldJ = L.ldJ; c.ldH = L.ldH;
  if (NREG > 0) { c.nvp = NREG; c.ldJ = NREG; }  // the launcher checked nv_pad == NREG: row strides and row-dot trip counts become constants (176 -> 172 us)
  c.J = S + L.J; c.H = S + L.H; c.Lf = S + L.Lf; c.M = S + L.M;
  float* v = S + L.vec;
  const int vp = L.nvp;
  c.qacc = v; c.Ma = v + vp; c.grad = v + 2 * vp; c.search = v + 3 * vp; c.mv = v + 4 * vp; c.x = c.mv; c.qfs = v + 5 * vp; c.qfc = v + 6 * vp;
  float* rf = S + L.rowf;
  c.Jaref = rf; c.jv = rf + cap; c.hw = c.jv; c.D = rf + 2 * cap; c.force = rf + 3 * cap;
  c.floss = (m.nfricdof + m.ntenfric) > 0 ? rf + 4 * cap : c.D;  // never interpreted when the world has no friction rows
  int* ri = (int*)(S + L.rowi);
  c.state = ri; c.hidx = ri + cap;
  c.njmax = cap; c.ncone = 0;
  c.jcap = L.jcap; c.Jg = d.efc_J + wb * (size_t)d.njmax_pad * nvp;
  c.cgv = S + L.cgv;
  c.red = S + L.red;
  c.rng = (int*)(S + L.env); c.fz = c.rng + cap;
  // a single tree with a floating base has a dense envelope (every row reaches the root dofs): bookkeeping would only cost
  c.env = BIG && m.ntree > 1;
  c.rfri = rf + L.nrowf * cap; c.quad = c.rfri + cap; c.rinfo = ri + 2 * cap;

  if (njmax == 0 || nv == 0) {
#pragma unroll 1
    for (int dd = lane; dd < nv; dd += NT) d.qacc[wb * nv + dd] = d.qacc_smooth[wb * nv + dd];
    if (lane == 0) d.solver_niter[w] = 0;
    return;
  }
  const int nefc = min(min(d.nefc[w], njmax), cap);
  c.nefc = nefc; c.ne = PLAIN ? 0 : d.ne[w]; c.nf = PLAIN ? 0 : d.nf[w];

  // ---- stage the world's problem in shared memory.  One warp per world (NW = 1): the Jacobian rows and the per-row vectors are
  // contiguous, 16-byte aligned blocks of the world-major arrays, so one lane issues a bulk-async copy (cp.async.bulk, SASS UBLKCP)
  // for each and the warp waits once on the mbarrier, after it has issued its own small loads -- instead of four dependent
  // load -> store loops in a row.  aref lands in the Jaref slot and is folded in below.
  Stager st;
  const int n4 = (nefc + 3) & ~3, nrow = n4 <= cap ? n4 : nefc;  // whole float4s when the slice has room (the pad is never read)
  if (NW == 1) {
    st.init(reinterpret_cast<uint64_t*>(S + L.bar), lane);
    st.load(c.J, d.efc_J + wb * (size_t)d.njmax_pad * nvp, min(nefc, L.jcap) * nvp);
    st.load(c.D, d.efc_D + wb * d.njmax_pad, nrow);
    st.load(c.Jaref, d.efc_aref + wb * njmax, nrow);
    if ((m.nfricdof + m.ntenfric) > 0) st.load(c.floss, d.efc_frictionloss + wb * njmax, nrow);
  }
  {
    if (NW != 1) {
      const float4* Jg = reinterpret_cast<const float4*>(d.efc_J + wb * (size_t)d.njmax_pad * nvp);
      float4* Js = reinterpret_cast<float4*>(c.J);
#pragma unroll 1
      for (int i = lane; i < min(nefc, L.jcap) * nvp / 4; i += NT) Js[i] = Jg[i];
    }
    for (int i = lane; i < 7 * vp; i += NT) v[i] = 0.f;  // zero padding of every per-dof vector
    tsync<NW>();
#pragma unroll 1
    for (int r = lane; r < nefc; r += NT) {
      if (NW != 1) {
        c.D[r] = d.efc_D[wb * d.njmax_pad + r];
        if ((m.nfricdof + m.ntenfric) > 0) c.floss[r] = d.efc_frictionloss[wb * njmax + r];
      }
      c.state[r] = ST_SATISFIED;
      if (ELL) {  // row -> (contact, component) map; a contact's rows are consecutive (k_constraint.cu)
        int info = -1; float fr = 0.f;
        if (d.efc_type[wb * njmax + r] == CNSTR_CONTACT_ELLIPTIC) {
          const int cid = d.efc_id[wb * njmax + r], e0 = d.contact_efc_address[(size_t)cid * m.nmaxpyramid], dim = d.contact_dim[cid], j = r - e0;
          info = (e0 < 0 || e0 + dim > nefc) ? -2 : ((dim << 4) | j);
          fr = j == 0 ? d.contact_friction[5 * (size_t)cid] * m.impratio_invsqrt : d.contact_friction[5 * (size_t)cid + j - 1];
        }
        c.rinfo[r] = info; c.rfri[r] = fr;
      }
    }
    if (BIG) tcopy<NW>(c.M, d.M + wb * m.nC, m.nC, lane);
    tcopy<NW>(c.qfs, d.qfrc_smooth + wb * nv, nv, lane);
    const float* start = (m.disableflags & DSBL_WARMSTART) ? d.qacc_smooth : d.qacc_warmstart;
    tcopy<NW>(c.qacc, start + wb * nv, nv, lane);
    const int hsz = nv * (nv + 1) / 2;
#pragma unroll 1
    for (int e = lane; e < hsz; e += NT) { c.H[e] = 0.f; if (!BIG) c.M[e] = 0.f; }
  }
  tsync<NW>();
  if (c.env) {
#pragma unroll 1
    for (int i = lane; i < nv; i += NT) c.fz[i] = i;
    tsync<NW>();
  }
  if (!BIG) {  // dense packed M from the CSR values in global memory; H = M
    const float* Mg = d.M + wb * m.nC;
#pragma unroll 4
    for (int e = lane; e < m.nC; e += NT) {
      const int r = m.M_entry_row[e], col = m.M_colind[e];
      const float v = Mg[e];
      c.M[(r * (r + 1)) / 2 + col] = v;
      c.H[(r * (r + 1)) / 2 + col] = v;
    }
  } else {
#pragma unroll 1
    for (int e = lane; e < m.nC; e += NT) {  // lower triangle of M
      const int r = m.M_entry_row[e], col = m.M_colind[e];
      c.H[(r * (r + 1)) / 2 + col] = c.M[e];
      if (c.env) atomicMin(&c.fz[r], col);
    }
  }
  if (NW == 1) st.load_wait();  // staged rows and per-row vectors have landed
  if (c.env) {
    // nonzero column range [lo, hi) of every Jacobian row; rows of one elliptic contact share the union of their ranges (the cone
    // Hessian mixes them); every dof inside a row's range gets that row's lo into its envelope (H = M + sum of w J_r J_r^T terms)
#pragma unroll 1
    for (int r = lane; r < nefc; r += NT) {
      const float* Jr = jrow<BIG>(c, r);
      int lo = nv, hi = 0;
      for (int k = 0; k < nv; k++) if (Jr[k] != 0.f) { lo = min(lo, k); hi = k + 1; }
      if (hi == 0) lo = 0;
      c.rng[r] = lo | (hi << 16);
    }
    tsync<NW>();
    if (ELL) {
#pragma unroll 1
      for (int r = lane; r < nefc; r += NT) {
        const int info = c.rinfo[r];
        if (info < 0 || (info & 15) != 0) continue;
        const int dim = info >> 4;
        int lo = nv, hi = 0;
        for (int j = 0; j < dim; j++) { const int g = c.rng[r + j]; if ((g >> 16) > 0) { lo = min(lo, g & 0xFFFF); hi = max(hi, g >> 16); } }
        if (hi == 0) lo = 0;
        for (int j = 0; j < dim; j++) c.rng[r + j] = lo | (hi << 16);
      }
      tsync<NW>();
    }
#pragma unroll 1
    for (int r = lane; r < nefc; r += NT) {
      const int lo = c.rng[r] & 0xFFFF, hi = c.rng[r] >> 16;
      for (int i = lo; i < hi; i++) atomicMin(&c.fz[i], lo);
    }
  }
#pragma unroll 1
  for (int r = lane; r < nefc; r += NT) {  // Jaref = J qacc - aref
    c.Jaref[r] = row_dot(jrow<BIG>(c, r), c.qacc, c.nvp) - (NW == 1 ? c.Jaref[r] : d.efc_aref[wb * njmax + r]);
  }
  mul_m<NW, BIG>(c, c.qacc, c.Ma);
  tsync<NW>();

  // One call site per phase: iteration -1 is init_context (solver.py:3622), iterations >= 0 are _solver_iteration (:3526).
  // _solve_done's three criteria are OR-ed (:3483-3486), so when `improvement` or `gradient` already satisfies the
  // tolerance the Hessian refactorisation (whose only consumer is the next line search) is skipped.
  const float scale = m.meaninertia * (float)nv;
  int niter = 0, ovf = 0;
  for (int it = -1;; it++) {
    if (it >= 0 && !linesearch<ELL, BIG, NW>(c)) ovf |= OVF_LS_ITERATIONS;
    const int nlist = update_constraint<ELL, BIG, NW>(c, it < 0);
    update_grad<NW>(c);
    if (it >= 0) {
      niter++;
      const float improvement = c.improvement / scale, gradient = sqrtf(c.grad_dot) / scale;
      if (improvement < m.tolerance || gradient < m.tolerance) break;
    } else if (m.iterations == 0) break;
    if (CG) {
      if (it >= 0 && niter == m.iterations) { ovf |= OVF_ITERATIONS; break; }
      cg_direction(c, m, d, wb, it < 0);
      continue;
    }
    if (!CG) update_search<ELL, BIG, NW, NREG>(c, nlist);
    if (it >= 0) {
      if (0.5f * c.newton_decrement / scale < m.tolerance) break;
      if (niter == m.iterations) { ovf |= OVF_ITERATIONS; break; }
    }
  }

  // ---- results
  tcopy<NW>(d.qacc + wb * nv, c.qacc, nv, lane);
  tcopy<NW>(d.efc_Ma + wb * nv, c.Ma, nv, lane);
  tcopy<NW>(d.qfrc_constraint + wb * nv, c.qfc, nv, lane);
#pragma unroll 1
  for (int r = lane; r < nefc; r += NT) { d.efc_force[wb * njmax + r] = c.force[r]; d.efc_state[wb * d.njmax_pad + r] = c.state[r]; }
  if (lane == 0) { d.solver_niter[w] = niter; if (ovf) d.overflow[w] |= ovf; }
}

// Row-capacity classes.  A world's shared-memory slice is dominated by its staged Jacobian, sized for njmax rows although most worlds
// hold far fewer (benchmark humanoid: njmax 64, ~18 rows while it stands): worlds whose row count fits rowcap = njmax / 2 are listed
// here and solved by a launch with the smaller slice -- more of them are resident per SM, which is what the latency-bound solver's
// time hangs on -- the rest by a launch with the full slice.  Lists are filled with one warp-aggregated atomic per warp; the order
// inside a list depends on scheduling, the per-world results do not.
__global__ void __launch_bounds__(256)
k_solver_classify(const __grid_constant__ DataDev d, int cap0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  const bool in = i < d.wn && i + d.w0 < d.nworld;
  const int w = i + d.w0;
  const int cls = in ? (min(d.nefc[w], d.njmax) <= cap0 ? 0 : 1) : -1;
  for (int c = 0; c < 2; c++) {
    const unsigned bal = __ballot_sync(FULL_MASK, cls == c);
    if (!bal) continue;
    int base = 0;
    if (lane == __ffs(bal) - 1) base = atomicAdd(&d.sol_count[2 * d.split_id + c], __popc(bal));
    base = __shfl_sync(FULL_MASK, base, __ffs(bal) - 1);
    if (cls == c) d.sol_list[(size_t)c * d.nworld + d.w0 + base + __popc(bal & ((1u << lane) - 1u))] = w;
  }
}

}  // namespace

// The "big" instantiation (packed Hessian and factor worked on in shared memory, Jacobian rows read through L2, CSR inertia) is mandatory
// above nv = 32; MJB_SOLVER_BIG = 1 selects it for small models too (62 instead of 127 registers, 6.4 instead of 14 KB per world).
static bool solver_big(const ModelDev& m) {
  static int forced = -1;
  if (forced < 0) { const char* e = getenv("MJB_SOLVER_BIG"); forced = e ? atoi(e) : 0; }
  return m.nv > 32 || forced == 1;
}
size_t smem_solver(const ModelDev& m, const DataDev& d) { return (size_t)sol_layout(m, d, solver_big(m)).total * sizeof(float); }

// Warps per world: 1.  For nv > 32 the per-world slice of shared memory (packed Hessian + factor + Jacobian rows) limits an SM to
// a few resident worlds; teams of 2 or 4 warps per world (block barriers, right-looking team Cholesky) are implemented and
// parity-tested but measured slower than one warp per world, so they stay an experiment knob: MJB_SOLVER_WARPS = 1, 2 or 4.
static int solver_warps(const ModelDev& m) {
  if (m.nv <= 32 || m.solver == SOL_CG) return 1;
  static int forced = -1;
  if (forced < 0) { const char* e = getenv("MJB_SOLVER_WARPS"); forced = e ? atoi(e) : 0; }
  if (forced == 1 || forced == 2 || forced == 4) return forced;
  return 1;  // teams of 2 / 4 warps measured slower on unitree G1 and three_humanoids (block barriers per Cholesky column)
}

// row-capacity classes (see k_solver_classify): small-model path with a staged Jacobian, enough rows and worlds to matter
static bool solver_uses_classes(const ModelDev& m, const DataDev& d) {
  static int classes = -1;
  // off by default: measured slower for the humanoid, with every world in the small class and with a mixed population -- the extra
  // resident worlds do not speed the solve up, so its time is not set by the number of worlds in
  // flight the way the position / velocity kernels' is; kept as an experiment knob (MJB_SOLVER_CLASSES=1), parity-tested
  if (classes < 0) { const char* e = getenv("MJB_SOLVER_CLASSES"); classes = e ? atoi(e) : 0; }
  return classes && !solver_big(m) && d.rowcap == 0 && d.njmax >= 32 && d.wn >= 256 && d.sol_list;
}
int solver_launch_count(const ModelDev& m, const DataDev& d) { return solver_uses_classes(m, d) ? 3 : 1; }

cudaError_t launch_solver(const ModelDev& m, const DataDev& d, cudaStream_t s) {
  const size_t smem = smem_solver(m, d);
  const int ell = m.cone == CONE_ELLIPTIC ? 1 : 0, big = solver_big(m) ? 1 : 0, cg = m.solver == SOL_CG ? 1 : 0;
  const int nw = solver_warps(m), team = nw == 4 ? 2 : (nw == 2 ? 1 : 0);
  const int which = cg ? 4 + 2 * big + ell : (big ? 8 + 2 * team + ell : ell);
  static size_t configured[18] = {0};
  static void (*const kerns[14])(ModelDev, DataDev) = {
    k_solver<false, false, false, 1>, k_solver<true, false, false, 1>, nullptr, nullptr,
    k_solver<false, false, true, 1>,  k_solver<true, false, true, 1>,  k_solver<false, true, true, 1>,  k_solver<true, true, true, 1>,
    k_solver<false, true, false, 1>,  k_solver<true, true, false, 1>,  k_solver<false, true, false, 2>, k_solver<true, true, false, 2>,
    k_solver<false, true, false, 4>,  k_solver<true, true, false, 4>};
  void (*kern)(ModelDev, DataDev) = kerns[which];
  int ci = which;
  // no equality and no friction-loss rows possible: the instantiation with ne = nf = 0 compiled in (humanoid solver 202 -> 181 us: the
  // line-search loops lose two of their three row kinds, and with them instructions and instruction-cache footprint)
  const bool plain = m.neq == 0 && m.nfricdof == 0 && m.ntenfric == 0 && m.ntendon == 0;
  if (which == 0 && plain) {
    kern = k_solver<false, false, false, 1, true>; ci = 14;
    // ... and the register-row size fixed (one Hessian / Cholesky variant in the kernel instead of five: 182 -> 178 us)
    if (m.nv > 24 && m.nv <= 28 && d.nv_pad == 28) { kern = k_solver<false, false, false, 1, true, 28>; ci = 15; }
    else if (m.nv > 28 && d.nv_pad == 32) { kern = k_solver<false, false, false, 1, true, 32>; ci = 16; }
  }
  if (which == 8 && plain) { kern = k_solver<false, true, false, 1, true>; ci = 17; }  // nv > 32 (unitree G1, three_humanoids)
  if (smem > 48 * 1024 && smem > configured[ci]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured[ci] = smem;
  }
  const int cap0 = ((d.njmax / 2) + 3) & ~3;
  if (solver_uses_classes(m, d)) {
    cudaError_t e = cudaMemsetAsync(d.sol_count + 2 * d.split_id, 0, 2 * sizeof(int), s);
    if (e != cudaSuccess) return e;
    k_solver_classify<<<(d.wn + 255) / 256, 256, 0, s>>>(d, cap0);
    // the two classes run concurrently (fork / join on the range's auxiliary stream): with different slice sizes they cannot share a
    // launch, and back to back each would pay its own last, partly empty round of resident blocks
    cudaStream_t aux = (cudaStream_t)d.sol_stream;
    cudaEvent_t fork = (cudaEvent_t)d.sol_fork, join = (cudaEvent_t)d.sol_join;
    if ((e = cudaEventRecord(fork, s)) != cudaSuccess) return e;
    if ((e = cudaStreamWaitEvent(aux, fork, 0)) != cudaSuccess) return e;
    DataDev dc = d;
    dc.rowcap = d.njmax; dc.sol_class = 1;
    kern<<<d.wn, nw * 32, smem, aux>>>(m, dc);  // blocks beyond the class count exit at once
    if ((e = cudaEventRecord(join, aux)) != cudaSuccess) return e;
    dc.rowcap = cap0; dc.sol_class = 0;
    kern<<<d.wn, nw * 32, smem_solver(m, dc), s>>>(m, dc);
    if ((e = cudaStreamWaitEvent(s, join, 0)) != cudaSuccess) return e;
    return cudaGetLastError();
  }
  const int grid = d.wn;
  kern<<<grid, nw * 32, smem, s>>>(m, d);
  return cudaGetLastError();
}
