// Shared device/host helpers for the parl_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/parl_b200.h"

namespace rl {

void set_error(const char* fmt, ...);
int effective_sms(int sms);          // SM count capped by rl_set_sm_limit
int pdl_enabled();                   // 1: chain kernels are launched with programmatic stream serialization

#define RL_CHECK_ARG(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      rl::set_error(__VA_ARGS__);          \
      return RL_ERR_BAD_ARG;               \
    }                                      \
  } while (0)

#define RL_CHECK_LAUNCH(name)                                              \
  do {                                                                     \
    cudaError_t e__ = cudaGetLastError();                                  \
    if (e__ != cudaSuccess) {                                              \
      rl::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return RL_ERR_CUDA;                                                  \
    }                                                                      \
  } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Opt a kernel in to the device's whole dynamic shared-memory range (227 KB minus its static use) ONCE per
// device and never lower it again: the per-launch size is then free to vary with the launch's shapes without
// re-programming the function while another launch of it is still queued.
template <class Kernel>
static inline void opt_in_max_dynamic_smem(Kernel kernel, unsigned long long* done_mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (*done_mask & bit) return;
  int optin = 0;
  cudaFuncAttributes fa;
  if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess &&
      cudaFuncGetAttributes(&fa, kernel) == cudaSuccess)
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
  *done_mask |= bit;
}
#define RL_SMEM_OPTIN(...)                                  \
  do {                                                      \
    static unsigned long long done__ = 0;                   \
    rl::opt_in_max_dynamic_smem(__VA_ARGS__, &done__);      \
  } while (0)

#ifdef __CUDACC__
// Programmatic dependent launch (actor chain: 7 short kernels per env step).  A kernel launched through launch_chain
// may begin while its predecessor in the stream is still draining: its prologue (barrier init,
// tensor-map prefetch, weight loads — nothing a predecessor writes) runs ahead, pdl_wait() then blocks until the
// predecessor grid has completed and its writes are visible, and pdl_trigger() lets the NEXT kernel in the stream start
// its own prologue.  Every kernel launched this way MUST call pdl_wait() before its first access to memory another
// kernel of the stream produces (or still reads) — and before it exits.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_chain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                       Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid, cfg.blockDim = block, cfg.dynamicSmemBytes = smem, cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = attr, cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src) {
  unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// streaming (evict-first) vector store / load for data touched exactly once
__device__ __forceinline__ void st_cs_f4(float4* p, float4 v) { __stcs(p, v); }
__device__ __forceinline__ float4 ld_cs_f4(const float4* p) { return __ldcs(p); }
#endif

}  // namespace rl
