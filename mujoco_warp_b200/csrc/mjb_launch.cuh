// mjb_launch.cuh -- host side of every kernel launch: per-instance configuration, the launch itself and the launch count.
#pragma once
#include <mutex>
#include <unordered_map>
#include <cuda_runtime.h>

// Kernels the calling thread launched since the C-ABI entry point it is in started (mjb_last_launch_count).
inline thread_local int g_launches = 0;

// Per-SM limits of the device, read once per process: SMs, shared memory per SM and the part of it the runtime reserves per
// block, blocks, warps and registers per SM.  Like the per-instance configuration below, this assumes that the GPUs a process
// drives are of one kind (one process per GPU, as bench.py and torchrun run it).
struct SmLimits { int sms; size_t smem_per_sm, reserved_per_block; int blocks, warps, regs; };
inline const SmLimits& sm_limits() {
  static const SmLimits l = [] {
    int dev = 0, sms = 0, smem = 0, reserved = 0, blocks = 0, threads = 0, regs = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev);
    cudaDeviceGetAttribute(&blocks, cudaDevAttrMaxBlocksPerMultiprocessor, dev);
    cudaDeviceGetAttribute(&threads, cudaDevAttrMaxThreadsPerMultiProcessor, dev);
    cudaDeviceGetAttribute(&regs, cudaDevAttrMaxRegistersPerMultiprocessor, dev);
    return SmLimits{sms, (size_t)smem, (size_t)reserved, blocks, threads / 32, regs};
  }();
  return l;
}

// Registers per thread of a kernel instance (0 if unknown: then registers do not limit the shape choice).
template <class K>
inline int kernel_regs(K* kern) {
  cudaFuncAttributes a;
  return cudaFuncGetAttributes(&a, kern) == cudaSuccess ? a.numRegs : 0;
}

// Shared memory an SM sets aside for a block of `bytes`: 128-byte allocation units plus the runtime's per-block reserve.
inline size_t sm_block_bytes(size_t bytes) { return ((bytes + 127) & ~(size_t)127) + sm_limits().reserved_per_block; }

// Configures a kernel instance for blocks of `smem` bytes of dynamic shared memory: above the 48 KB default it opts in to that
// size, raised only when a launch needs more than any before; a `carveout` other than cudaSharedmemCarveoutDefault is set
// whenever it differs from the one set last.  Attributes are per instance, so the cache is keyed by the kernel.
inline cudaError_t launch_configure(const void* kern, size_t smem, int carveout = cudaSharedmemCarveoutDefault) {
  struct Config { size_t smem = 0; int carveout = cudaSharedmemCarveoutDefault; };
  static std::mutex mu;
  static std::unordered_map<const void*, Config> by_kernel;
  std::lock_guard<std::mutex> lock(mu);
  Config& c = by_kernel[kern];
  if (carveout != cudaSharedmemCarveoutDefault && carveout != c.carveout) {
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, carveout);
    if (e != cudaSuccess) return e;
    c.carveout = carveout;
  }
  if (smem > 48 * 1024 && smem > c.smem) {
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    c.smem = smem;
  }
  return cudaSuccess;
}

// Launches kern<<<grid, block, smem, s>>>(args...) after configuring the instance for `smem` (and `carveout`), and counts it.
template <class... P, class... A>
inline cudaError_t launch(void (*kern)(P...), unsigned grid, unsigned block, size_t smem, int carveout, cudaStream_t s, const A&... args) {
  const cudaError_t e = launch_configure((const void*)kern, smem, carveout);
  if (e != cudaSuccess) return e;
  kern<<<grid, block, smem, s>>>(args...);
  g_launches++;
  return cudaGetLastError();
}
template <class... P, class... A>
inline cudaError_t launch(void (*kern)(P...), unsigned grid, unsigned block, size_t smem, cudaStream_t s, const A&... args) {
  return launch(kern, grid, block, smem, cudaSharedmemCarveoutDefault, s, args...);
}
