// mjb_team.cuh -- sub-warp world teams and bulk-async (1-D TMA) staging.
//
// A warp owns G = 32 / LPW consecutive worlds; the LPW lanes of a "team" own one world.  Tree passes (1-4 bodies per
// level) and per-dof / per-row loops then keep most lanes busy, instead of one warp walking one world's tree with 1-4 active
// lanes.  Model loads (same address for every team) coalesce into one request per warp.
//
// Because Data is world-major (types.py:2230-2374 of the reference), the rows of the G worlds of a warp are ONE contiguous
// block of G * n floats per field.  With G * n * 4 a multiple of 16 bytes the block moves with a single
// cp.async.bulk (SASS UBLKCP): global -> shared completes on an mbarrier, shared -> global is a bulk group.  One elected lane
// issues a handful of these per kernel instead of every lane looping LDG -> STS / LDS -> STG over each row.
// Shared layout of a field: [G][n] at S + off * G (off = per-world offset, padded to 4 floats so the block is 16 B aligned).
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

#include "mjb_math.cuh"

template <int LPW>
__device__ __forceinline__ float team_sum(float v) {
#pragma unroll
  for (int o = LPW / 2; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}
template <int LPW>
__device__ __forceinline__ int team_sum_i(int v) {
#pragma unroll
  for (int o = LPW / 2; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}
template <int LPW>
__device__ __forceinline__ bool team_any(bool p, int g) {
  const unsigned b = __ballot_sync(FULL_MASK, p);
  return LPW == 32 ? b != 0u : ((b >> (g * LPW)) & ((1u << (LPW & 31)) - 1u)) != 0u;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Staging of group blocks.  All methods are called by the whole (converged) warp.
struct Stager {
  uint64_t* bar;
  uint32_t phase;
  int lane;
  bool pending_store;

  __device__ __forceinline__ void init(uint64_t* b, int lane_) {
    bar = b; phase = 0; lane = lane_; pending_store = false;
    if (lane == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
  }
  static __device__ __forceinline__ bool bulk_ok(const void* g, const void* s, int nfloats) {
    return (((uintptr_t)g | (uintptr_t)smem_u32(s)) & 15u) == 0 && (nfloats & 3) == 0 && nfloats > 0;
  }
  // global -> shared, n floats
  __device__ __forceinline__ void load(float* s, const float* g, int n) {
    if (bulk_ok(g, s, n)) {
      if (lane == 0) {
        const uint32_t bytes = (uint32_t)n * 4u;
        asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(s)), "l"(g),
                     "r"(bytes), "r"(smem_u32(bar))
                     : "memory");
      }
    } else {
#pragma unroll 1  // cold path: the 16-way unrolled form the compiler picks cost ~55 instructions per call site -- 40 % of k_position's code
      for (int i = lane; i < n; i += 32) s[i] = g[i];
    }
  }
  __device__ __forceinline__ void load_wait() {
    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
    uint32_t ok = 0;
    while (!ok) {
      asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
    }
    phase ^= 1u;
    __syncwarp();
  }
  // generic-proxy writes of every lane become visible to the async proxy; call once before a batch of store()s
  __device__ __forceinline__ void store_fence() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
  }
  // shared -> global, n floats
  __device__ __forceinline__ void store(float* g, const float* s, int n) {
    if (bulk_ok(g, s, n)) {
      if (lane == 0) {
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(g), "r"(smem_u32(s)), "r"((uint32_t)n * 4u) : "memory");
        pending_store = true;
      }
    } else {
#pragma unroll 1
      for (int i = lane; i < n; i += 32) g[i] = s[i];
    }
  }
  __device__ __forceinline__ void store_commit() {
    if (lane == 0 && pending_store) asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
  // the shared source of every committed store has been read (the buffers may be overwritten / the block may exit)
  __device__ __forceinline__ void store_wait_read() {
    if (lane == 0 && pending_store) { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); pending_store = false; }
    __syncwarp();
  }
};

// Launch shape of a team kernel: lanes per world and warps per block, from the per-world shared-memory footprint.
// Default 8 lanes per world (4 worlds per warp) and two-warp blocks: measured best on H100 for the humanoid (DESIGN.md); models
// whose worlds are too large for that fall back to fewer worlds per warp / one-warp blocks.  MJB_LPW_* / MJB_WPB_* override.
struct TeamShape { int lpw, wpb; size_t warp_bytes, block_bytes; };
inline TeamShape team_shape(size_t world_words, const char* env_lpw, const char* env_wpb) {
  constexpr size_t kBlockMax = 200 * 1024;  // leaves room for a second resident block's reserve
  auto bytes = [&](int lpw) { return (world_words * (size_t)(32 / lpw) + 4) * sizeof(float); };
  const char* e = getenv(env_lpw);
  int lpw = e ? atoi(e) : 8;
  if (lpw != 4 && lpw != 8 && lpw != 16 && lpw != 32) lpw = 8;
  while (lpw < 32 && bytes(lpw) > kBlockMax / 2) lpw *= 2;
  e = getenv(env_wpb);
  int wpb = e ? atoi(e) : 2;
  if (wpb < 1) wpb = 1;
  if (wpb > 8) wpb = 8;
  while (wpb > 1 && bytes(lpw) * wpb > kBlockMax) wpb--;
  TeamShape t;
  t.lpw = lpw; t.wpb = wpb; t.warp_bytes = bytes(lpw); t.block_bytes = t.warp_bytes * wpb;
  return t;
}

inline TeamShape team_shape_fixed(size_t world_words, int lpw, int wpb) {
  TeamShape t;
  t.lpw = lpw; t.wpb = wpb; t.warp_bytes = (world_words * (size_t)(32 / lpw) + 4) * sizeof(float);
  while (t.wpb > 1 && t.warp_bytes * t.wpb > 200 * 1024) t.wpb--;
  t.block_bytes = t.warp_bytes * t.wpb;
  return t;
}

// World team of the calling lane.
template <int LPW>
struct Team {
  static constexpr int G = 32 / LPW;
  int lane, sub, g;   // lane in the warp, lane in the team, team in the warp
  int wg0, nvalid;    // first world of the warp's group, worlds of the group that exist
  int w;              // this team's world (clamped to the last valid one: idle teams recompute it and store nothing)
  bool valid;
  __device__ __forceinline__ void init(int w0, int wn, int nworld) {
    lane = threadIdx.x & 31; sub = lane % LPW; g = lane / LPW;
    wg0 = w0 + (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * G;  // warps of a block are independent world groups
    const int wend = min(w0 + wn, nworld);
    nvalid = min(G, wend - wg0);
    valid = g < nvalid;
    w = wg0 + (valid ? g : nvalid - 1);
  }
};
