// mjb_chol.cuh -- warp-cooperative dense Cholesky in shared memory.
// Replaces the reference's wp.tile_cholesky_inplace / tile_cholesky_solve (cuSolverDx via libmathdx) call sites:
// smooth.py:1308,3151,3256-3260 (inertia blocks) and solver.py:2595-2597 (Newton Hessian).
// A is n x n with leading dimension ld (choose ld odd so that lane-strided row access is bank-conflict free);
// only the lower triangle is read/written.  One warp, lanes map to rows, left-looking column sweep.
#pragma once
#include "mjb_math.cuh"

// In-place lower Cholesky: A = L L^T.  Returns (via *min_diag) the smallest pivot before sqrt for diagnostics.
__device__ __forceinline__ void warp_cholesky(float* A, int n, int ld, int lane) {
  for (int j = 0; j < n; j++) {
    const float* rj = A + j * ld;
    float s = 0.f;
    for (int k = lane; k < j; k += 32) s += rj[k] * rj[k];
    s = warp_sum(s);
    const float ljj = sqrtf(fmaxf(rj[j] - s, MJ_MINVAL));
    const float inv = 1.0f / ljj;
    for (int i = j + 1 + lane; i < n; i += 32) {
      const float* ri = A + i * ld;
      float t = ri[j];
      for (int k = 0; k < j; k++) t -= ri[k] * rj[k];
      A[i * ld + j] = t * inv;
    }
    __syncwarp();
    if (lane == 0) A[j * ld + j] = ljj;
    __syncwarp();
  }
}

// x <- (L L^T)^-1 x, x in shared memory (length n).
__device__ __forceinline__ void warp_chol_solve(const float* L, int n, int ld, float* x, int lane) {
  for (int j = 0; j < n; j++) {  // forward: L y = b
    const float yj = x[j] / L[j * ld + j];
    __syncwarp();
    for (int i = j + 1 + lane; i < n; i += 32) x[i] -= L[i * ld + j] * yj;
    if (lane == 0) x[j] = yj;
    __syncwarp();
  }
  for (int j = n - 1; j >= 0; j--) {  // backward: L^T x = y
    const float xj = x[j] / L[j * ld + j];
    __syncwarp();
    for (int i = lane; i < j; i += 32) x[i] -= L[j * ld + i] * xj;
    if (lane == 0) x[j] = xj;
    __syncwarp();
  }
}

// Packed-lower-triangle variants (row r starts at r(r+1)/2), used for 32 < n <= 64 where the matrix must stay small enough
// in shared memory for a healthy number of resident warps.
__device__ __forceinline__ void warp_cholesky_packed(float* A, int n, int lane) {
  for (int j = 0; j < n; j++) {
    const float* rj = A + (j * (j + 1)) / 2;
    float s = 0.f;
    for (int k = lane; k < j; k += 32) s += rj[k] * rj[k];
    s = warp_sum(s);
    const float ljj = sqrtf(fmaxf(rj[j] - s, MJ_MINVAL));
    const float inv = 1.0f / ljj;
    for (int i = j + 1 + lane; i < n; i += 32) {
      float* ri = A + (i * (i + 1)) / 2;
      float t = ri[j];
#pragma unroll 4
      for (int k = 0; k < j; k++) t -= ri[k] * rj[k];
      ri[j] = t * inv;
    }
    __syncwarp();
    if (lane == 0) A[(j * (j + 1)) / 2 + j] = ljj;
    __syncwarp();
  }
}
__device__ __forceinline__ void warp_chol_solve_packed(const float* L, int n, float* x, int lane) {
  for (int j = 0; j < n; j++) {  // forward: L y = b
    const float yj = x[j] / L[(j * (j + 1)) / 2 + j];
    __syncwarp();
    for (int i = j + 1 + lane; i < n; i += 32) x[i] -= L[(i * (i + 1)) / 2 + j] * yj;
    if (lane == 0) x[j] = yj;
    __syncwarp();
  }
  for (int j = n - 1; j >= 0; j--) {  // backward: L^T x = y
    const float* rj = L + (j * (j + 1)) / 2;
    const float xj = x[j] / rj[j];
    __syncwarp();
    for (int i = lane; i < j; i += 32) x[i] -= rj[i] * xj;
    if (lane == 0) x[j] = xj;
    __syncwarp();
  }
}

// Envelope (skyline) variants: fz[i] <= i is the first column of row i that can be nonzero (the factor keeps the envelope of the
// matrix), so inner products start at max(fz[i], fz[j]) and rows whose envelope starts past column j are skipped.  For a
// block-diagonal Hessian (independent kinematic trees without a coupling constraint) this is one small factorisation per block.
__device__ __forceinline__ void warp_cholesky_packed_env(float* A, int n, const int* fz, int lane) {
  for (int j = 0; j < n; j++) {
    const float* rj = A + (j * (j + 1)) / 2;
    const int fj = fz[j];
    float s = 0.f;
    for (int k = fj + lane; k < j; k += 32) s += rj[k] * rj[k];
    s = warp_sum(s);
    const float ljj = sqrtf(fmaxf(rj[j] - s, MJ_MINVAL));
    const float inv = 1.0f / ljj;
    for (int i = j + 1 + lane; i < n; i += 32) {
      const int fi = fz[i];
      if (fi > j) continue;  // A[i][j] is outside the envelope: stays 0
      float* ri = A + (i * (i + 1)) / 2;
      float t = ri[j];
#pragma unroll 4
      for (int k = max(fi, fj); k < j; k++) t -= ri[k] * rj[k];
      ri[j] = t * inv;
    }
    __syncwarp();
    if (lane == 0) A[(j * (j + 1)) / 2 + j] = ljj;
    __syncwarp();
  }
}
__device__ __forceinline__ void warp_chol_solve_packed_env(const float* L, int n, const int* fz, float* x, int lane) {
  for (int j = 0; j < n; j++) {  // forward: L y = b
    const float yj = x[j] / L[(j * (j + 1)) / 2 + j];
    __syncwarp();
    for (int i = j + 1 + lane; i < n; i += 32) if (fz[i] <= j) x[i] -= L[(i * (i + 1)) / 2 + j] * yj;
    if (lane == 0) x[j] = yj;
    __syncwarp();
  }
  for (int j = n - 1; j >= 0; j--) {  // backward: L^T x = y
    const float* rj = L + (j * (j + 1)) / 2;
    const float xj = x[j] / rj[j];
    __syncwarp();
    for (int i = fz[j] + lane; i < j; i += 32) x[i] -= rj[i] * xj;
    if (lane == 0) x[j] = xj;
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Register-resident Cholesky for n <= 32: lane i keeps row i of the matrix in registers, columns are eliminated
// right-looking with warp shuffles (no shared-memory round trips, no __syncwarp per column), the forward substitution of
// one right-hand side is folded into the same sweep, the factor is written once to shared memory (for the caller and for
// the transposed read of the backward substitution).  ~N^2/2 SHFL + FFMA instead of ~N^2/2 dependent LDS chains.
//   Hs  : shared, n x n, leading dim ld, lower triangle valid
//   b   : right-hand side element of row `lane` (0 for lane >= n)
//   Ls  : shared scratch (n rows x ldL), receives L (lower triangle); may alias Hs when ldL == ld (each lane only
//         reads and writes its own row)
// returns x[lane] of (L L^T) x = b.
// Lower-triangular element address.  PACKED rows start at the triangular number r(r+1)/2: triangular numbers are distinct
// mod 32 for r < 32, so both the row-wise access (lane = row) and the transposed access (lane = column) stay bank-conflict
// free while the matrix takes n(n+1)/2 words instead of n*ld.
template <bool PACKED>
__device__ __forceinline__ int tri_at(int r, int c, int ld) { return PACKED ? (r * (r + 1)) / 2 + c : r * ld + c; }

// Row loader: a[k] = H[lane][k] for k <= lane < n, identity padding elsewhere.
template <int N, bool PACKED = false>
__device__ __forceinline__ void chol_load_rows(float (&a)[N], const float* Hs, int ld, int n, int lane) {
  const int base = tri_at<PACKED>(lane, 0, ld);
#pragma unroll
  for (int k = 0; k < N; k++) {
    float v = (k == lane) ? 1.0f : 0.f;
    if (lane < n && k <= lane) v = Hs[base + k];
    a[k] = v;
  }
}

// Factor + solve on rows already held in registers (consumes a[]).
template <int N, bool PACKED = false>
__device__ __forceinline__ float chol_solve_rows(float (&a)[N], int n, float b, float* Ls, int ldL, int lane) {
  float myinv = 1.0f;
#pragma unroll
  for (int j = 0; j < N; j++) {
    const float ajj = __shfl_sync(FULL_MASK, a[j], j);
    const float inv = rsqrtf(fmaxf(ajj, MJ_MINVAL));
    a[j] *= inv;
    if (lane == j) myinv = inv;
    const float yj = __shfl_sync(FULL_MASK, b, j) * inv;
    b = lane > j ? b - a[j] * yj : (lane == j ? yj : b);
#pragma unroll
    for (int k = j + 1; k < N; k++) {
      const float lkj = __shfl_sync(FULL_MASK, a[j], k);
      a[k] -= a[j] * lkj;
    }
  }
  if (lane < n) {  // rows >= n are identity padding and are not stored
    const int base = tri_at<PACKED>(lane, 0, ldL);
#pragma unroll
    for (int k = 0; k < N; k++)
      if (k <= lane) Ls[base + k] = a[k];
  }
  __syncwarp();
#pragma unroll
  for (int j = N - 1; j >= 0; j--) {
    const float xj = __shfl_sync(FULL_MASK, b * myinv, j);
    const float ltj = (lane < j && j < n) ? Ls[tri_at<PACKED>(j, lane, ldL)] : 0.f;
    b = lane < j ? b - ltj * xj : (lane == j ? xj : b);
  }
  return b;
}

// 1 / sqrt(x) for x known to be a normal number (callers clamp at MJ_MINVAL): the bare MUFU.RSQ, without the denormal rescaling
// rsqrtf() wraps around it -- same bits for normal inputs.
__device__ __forceinline__ float rsqrt_normal(float x) {
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ---- Factor + solve for n <= 32 with a rolled loop over PAIRS of columns: lane i holds row i in registers, which rotate by two
// after each pair so the next pivots always sit in a[0], a[1].  The per-column bookkeeping (pivot broadcast, reciprocal square root,
// slot arithmetic, barrier, loop control) is paid once per pair, and a row makes one shared-memory round trip per pair.  The pair's
// two factor columns are broadcast to every lane through shared memory (LDS.128 of the same address).  A rolled loop keeps the
// sweep small enough for the instruction cache.  Columns (j, j+1) are eliminated together:
//   l0 = a[0] / sqrt(a00);  l10 = l0 of row j+1;  t1 = a[1] - l0 l10;  l1 = t1 / sqrt(t1 of row j+1)
//   a[k-2] <- a[k] - l0 L[j+k][j] - l1 L[j+k][j+1]     (registers rotate by two)
// Storage of the factor, per pair p (columns 2p, 2p+1, cnt = ne - 2p - 2 rows below the pair, ne = n rounded up to even):
//   [3 pad, L[2p+1][2p]] [P0: L[2p+2+t][2p], pad4(cnt)] [P1: L[2p+2+t][2p+1], pad4(cnt)]
// so both column pieces start 16-byte aligned (LDS.128 broadcasts in the trailing update) and P0[-1] is the in-pair entry.
__host__ __device__ __forceinline__ int cholpair_size(int n) {
  const int ne = (n + 1) & ~1;
  int o = 0;
  for (int c = ne - 2; c >= 0; c -= 2) o += 4 + 2 * ((c + 3) & ~3);
  return o;
}
template <int N>
__device__ __forceinline__ float chol_solve_rows_pair(float (&a)[N], int n, float b, float* Lc, int lane, float& myinv, int& mycol_off) {
  static_assert((N & 1) == 0, "register rows come in even sizes");
  myinv = 1.0f;
  mycol_off = 0;
  const int ne = (n + 1) & ~1;
  int cnt = ne - 2;      // rows below the current pair
  float* P0 = Lc + 4;    // pair block: P0[-1] = in-pair entry, P0[t], P1[t] = P0[pad4(cnt) + t]
#pragma unroll 1
  for (int j = 0; j < ne; j += 2) {
    const int pc = (cnt + 3) & ~3;
    const float a00 = __shfl_sync(FULL_MASK, a[0], j);
    const float inv0 = rsqrt_normal(fmaxf(a00, MJ_MINVAL));
    const float l0 = a[0] * inv0;                       // L[lane][j], lanes >= j
    const float l10 = __shfl_sync(FULL_MASK, l0, j + 1);
    const float t1 = a[1] - l0 * l10;                   // column j+1 after eliminating column j
    const float a11 = __shfl_sync(FULL_MASK, t1, j + 1);
    const float inv1 = rsqrt_normal(fmaxf(a11, MJ_MINVAL));
    const float l1 = t1 * inv1;                         // L[lane][j+1], lanes >= j+1
    if (lane == j) myinv = inv0;
    if (lane == j + 1) myinv = inv1;
    // forward substitution folded in (pivot lanes keep their unscaled b: y = b * myinv)
    const float y0 = __shfl_sync(FULL_MASK, b, j) * inv0;
    b -= lane > j ? l0 * y0 : 0.f;
    const float y1 = __shfl_sync(FULL_MASK, b, j + 1) * inv1;
    b -= lane > j + 1 ? l1 * y1 : 0.f;
    // this lane's column of the factor starts in this pair's block: remember where (backward substitution reads mycol[row])
    if ((lane >> 1) == (j >> 1)) mycol_off = (int)(P0 - Lc) + ((lane & 1) ? pc - (lane + 1) : -(lane + 2));
    if (lane > j && lane < ne) {
      P0[lane - j - 2] = l0;                            // lane j+1 lands on P0[-1]
      if (lane > j + 1) P0[pc + lane - j - 2] = l1;
    }
    __syncwarp();
    const float* P1 = P0 + pc;
#pragma unroll
    for (int k0 = 2; k0 < N; k0 += 4) {
      if (k0 - 2 >= cnt) break;
      const float4 p = *reinterpret_cast<const float4*>(P0 + (k0 - 2));
      const float4 q = *reinterpret_cast<const float4*>(P1 + (k0 - 2));
      a[k0 - 2] = a[k0] - l0 * p.x - l1 * q.x;
      if (k0 + 1 < N) a[k0 - 1] = a[k0 + 1] - l0 * p.y - l1 * q.y;
      if (k0 + 2 < N) a[k0] = a[k0 + 2] - l0 * p.z - l1 * q.z;
      if (k0 + 3 < N) a[k0 + 1] = a[k0 + 3] - l0 * p.w - l1 * q.w;
    }
    P0 += 4 + 2 * pc;
    cnt -= 2;
  }
  // backward substitution: L[j][lane] for lane < j is mycol[j]
  const float* mycol = Lc + mycol_off;
  b *= myinv;  // y
#pragma unroll 1
  for (int j = n - 1; j >= 0; j--) {
    const float xj = __shfl_sync(FULL_MASK, b * myinv, j);
    const float ltj = lane < j ? mycol[j] : 0.f;
    b -= ltj * xj;
  }
  return b * myinv;
}
// Solve only, on the factor chol_solve_rows_pair left in Lc (same operations in the same order as the folded substitutions).
__device__ __forceinline__ float chol_subst_pair(int n, float b, const float* Lc, int lane, float myinv, int mycol_off) {
  const int ne = (n + 1) & ~1;
  int cnt = ne - 2;
  const float* P0 = Lc + 4;
#pragma unroll 1
  for (int j = 0; j < ne; j += 2) {
    const int pc = (cnt + 3) & ~3;
    const float l0 = (lane > j && lane < ne) ? P0[lane - j - 2] : 0.f;
    const float l1 = (lane > j + 1 && lane < ne) ? P0[pc + lane - j - 2] : 0.f;
    const float y0 = __shfl_sync(FULL_MASK, b * myinv, j);
    b -= lane > j ? l0 * y0 : 0.f;
    const float y1 = __shfl_sync(FULL_MASK, b * myinv, j + 1);
    b -= lane > j + 1 ? l1 * y1 : 0.f;
    P0 += 4 + 2 * pc;
    cnt -= 2;
  }
  const float* mycol = Lc + mycol_off;
  b *= myinv;
#pragma unroll 1
  for (int j = n - 1; j >= 0; j--) {
    const float xj = __shfl_sync(FULL_MASK, b * myinv, j);
    const float ltj = lane < j ? mycol[j] : 0.f;
    b -= ltj * xj;
  }
  return b * myinv;
}

template <int N>
__device__ __forceinline__ float chol_solve_reg(const float* Hs, int ld, int n, float b, float* Ls, int ldL, int lane) {
  float a[N];
  chol_load_rows<N>(a, Hs, ld, n, lane);
  return chol_solve_rows<N>(a, n, b, Ls, ldL, lane);
}

// n <= 32 dispatch over padded sizes (warp-uniform branch)
__device__ __forceinline__ float chol_solve_reg_any(const float* Hs, int ld, int n, float b, float* Ls, int ldL, int lane) {
  if (n <= 8) return chol_solve_reg<8>(Hs, ld, n, b, Ls, ldL, lane);
  if (n <= 16) return chol_solve_reg<16>(Hs, ld, n, b, Ls, ldL, lane);
  if (n <= 24) return chol_solve_reg<24>(Hs, ld, n, b, Ls, ldL, lane);
  if (n <= 28) return chol_solve_reg<28>(Hs, ld, n, b, Ls, ldL, lane);
  return chol_solve_reg<32>(Hs, ld, n, b, Ls, ldL, lane);
}
