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
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cuda_runtime.h>

#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

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

// ---------------------------------------------------------------- host side: shape, configuration and launch of a team kernel
// A team kernel (k_position, k_velocity) is one instance per lanes-per-world count, `kernel_of(m, lpw)`, taking (m, d, stage mask),
// with `world_words` floats of shared memory per world.
// Instances may take arguments after the mask (the fluid instances of k_velocity), so the chooser's kernel type is a parameter.
using TeamKernel = void (*)(ModelDev, DataDev, int);
template <class K>
using TeamChooserOf = K (*)(const ModelDev& m, int lpw);

// Launch shape of a team kernel: lanes per world and warps per block, from the per-world shared-memory footprint.
// Default 8 lanes per world (4 worlds per warp); models whose worlds are too large for that fall back to fewer worlds per warp.
// The team kernels are latency bound, so their time is the number of residency rounds (waves of blocks that fit on the SMs at
// once) times one warp's dependent chain (DESIGN.md §3).  The warps per block (1, 2 or 4) are those that need the fewest rounds
// for `nworld` worlds, with as many blocks per SM as its shared memory, register file (registers per thread of the kernel
// instance for lpw), block and warp limits allow; ties go to two-warp blocks.  Batched models have only a 32-lane instance:
// where the footprint alone would give fewer lanes per world, they take 32 lanes in two-warp blocks.
struct TeamShape { int lpw, wpb; size_t block_bytes; };
template <class K>
inline TeamShape team_shape(const ModelDev& m, int nworld, size_t world_words, TeamChooserOf<K> kernel_of) {
  constexpr size_t kBlockMax = 200 * 1024;  // leaves room for a second resident block's reserve
  auto bytes = [&](int lpw) { return (world_words * (size_t)(32 / lpw) + 4) * sizeof(float); };
  int lpw = 8;
  while (lpw < 32 && bytes(lpw) > kBlockMax / 2) lpw *= 2;
  int wpb = 2;
  if (m.batched && lpw < 32) {
    lpw = 32;
  } else {
    const SmLimits& sm = sm_limits();
    const long groups = (nworld + 32 / lpw - 1) / (32 / lpw);
    const int warp_regs = (kernel_regs(kernel_of(m, lpw)) * 32 + 255) & ~255;  // registers are allocated per warp in units of 256
    auto rounds = [&](int w) {
      long per_sm = (long)(sm.smem_per_sm / sm_block_bytes(bytes(lpw) * w));
      per_sm = std::min({per_sm, (long)sm.blocks, (long)(sm.warps / w)});
      if (warp_regs > 0) per_sm = std::min(per_sm, (long)(sm.regs / warp_regs / w));
      const long fit = per_sm * sm.sms, blocks = (groups + w - 1) / w;  // fit: blocks resident at once
      return fit > 0 ? (blocks + fit - 1) / fit : LONG_MAX;
    };
    for (int w : {1, 4})
      if (bytes(lpw) * w <= kBlockMax && rounds(w) < rounds(wpb)) wpb = w;
  }
  while (wpb > 1 && bytes(lpw) * wpb > kBlockMax) wpb--;
  return TeamShape{lpw, wpb, bytes(lpw) * wpb};
}

// Shared-memory carveout (percent of the SM's shared memory) for team blocks of `block_bytes`: the one just large enough for as
// many blocks as fit.  The driver rounds a carveout up to the next shared-memory size the SM supports (CUDA Programming Guide,
// shared memory of compute capabilities 7.x and later), so the blocks that fit stay resident.  A smaller carveout, which the driver
// is free to pick otherwise, would cost resident worlds; a larger one costs L1 that the model-table lookups use (three_humanoids
// k_position, which fits 2 blocks per SM, DESIGN.md §3).
inline int team_carveout(size_t block_bytes) {
  const size_t per_sm = sm_limits().smem_per_sm, block = sm_block_bytes(block_bytes), fit = per_sm / block;
  const size_t pct = fit > 0 ? (100 * fit * block + per_sm - 1) / per_sm : 100;
  return pct < 100 ? (int)pct : (int)cudaSharedmemCarveoutMaxShared;
}

template <class K, class... A>
inline cudaError_t team_launch(const ModelDev& m, const DataDev& d, size_t world_words, TeamChooserOf<K> kernel_of, int mask, cudaStream_t s, const A&... extra) {
  const TeamShape t = team_shape(m, d.wn, world_words, kernel_of);
  const int G = 32 / t.lpw, ngroups = (d.wn + G - 1) / G, grid = (ngroups + t.wpb - 1) / t.wpb;
  return launch(kernel_of(m, t.lpw), grid, 32 * t.wpb, t.block_bytes, team_carveout(t.block_bytes), s, m, d, mask, extra...);
}

// Worlds per SM resident at once (occupancy API) in the launch shape of d's world range, and that shape: shape[0..2] = lanes per
// world, warps per block, block bytes.
template <class K>
inline cudaError_t team_resident_worlds(const ModelDev& m, const DataDev& d, size_t world_words, TeamChooserOf<K> kernel_of, int* worlds, int* shape) {
  const TeamShape t = team_shape(m, d.wn, world_words, kernel_of);
  const K kern = kernel_of(m, t.lpw);
  int blocks = 0;
  cudaError_t e = launch_configure((const void*)kern, t.block_bytes, team_carveout(t.block_bytes));
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kern, 32 * t.wpb, t.block_bytes);
  *worlds = blocks * t.wpb * (32 / t.lpw);
  shape[0] = t.lpw; shape[1] = t.wpb; shape[2] = (int)t.block_bytes;
  return e;
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
