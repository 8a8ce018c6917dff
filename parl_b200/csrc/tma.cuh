// TMA (cp.async.bulk.tensor) + mbarrier helpers for sm_90a, and host-side tensor-map creation
// through the driver entry point (no link-time libcuda dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rl {

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(void* mbar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(mbar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(void* mbar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(mbar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(void* mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(mbar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(void* mbar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LAB_DONE;\n"
      "bra LAB_WAIT;\n"
      "LAB_DONE:\n"
      "}\n" ::"r"(smem_u32(mbar)),
      "r"(parity)
      : "memory");
}

// 2-D tiled load: box at element coordinates (c0 = innermost, c1) -> dense smem tile [box1][box0].
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, void* mbar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(mbar))
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* smem_src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];\n" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1), "r"(smem_u32(smem_src))
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
#endif

// Host: encode a rank-2 float32 tensor map {dim0 (contiguous), dim1} with row pitch `pitch_bytes` and box {box0, box1}.
// Returns 0 on success; on failure `err` (if non-NULL) receives a static message.
inline int make_tensor_map_2d_f32(CUtensorMap* map, const void* base, uint64_t dim0, uint64_t dim1, uint64_t pitch_bytes,
                                  uint32_t box0, uint32_t box1, const char** err, bool as_int32 = false, int l2_promo = 1) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) {
      if (err) *err = "cuTensorMapEncodeTiled entry point unavailable";
      return -1;
    }
    fn = reinterpret_cast<EncodeFn>(p);
  }
  const cuuint64_t gdim[2] = {dim0, dim1};
  const cuuint64_t gstride[1] = {pitch_bytes};
  const cuuint32_t box[2] = {box0, box1};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(map, as_int32 ? CU_TENSOR_MAP_DATA_TYPE_INT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                        const_cast<void*>(base), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                        l2_promo == 2 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                      : (l2_promo == 0 ? CU_TENSOR_MAP_L2_PROMOTION_NONE : CU_TENSOR_MAP_L2_PROMOTION_L2_128B),
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    if (err) *err = "cuTensorMapEncodeTiled failed";
    return -2;
  }
  return 0;
}

// Same, through a small per-thread cache keyed by (base, dims, pitch, box): the loss kernels are launched every
// learner step on the same buffers, and six driver encodes per launch are several microseconds of host time.
inline int cached_tensor_map_2d_f32(CUtensorMap* map, const void* base, uint64_t dim0, uint64_t dim1, uint64_t pitch_bytes,
                                    uint32_t box0, uint32_t box1, const char** err, bool as_int32 = false, int l2_promo = 1) {
  struct Entry {
    const void* base;
    uint64_t dim0, dim1, pitch;
    uint32_t box0, box1;
    bool as_int32;
    int l2_promo;
    CUtensorMap map;
  };
  constexpr int kN = 128;
  static thread_local Entry cache[kN];
  static thread_local int used = 0, next = 0;
  for (int i = 0; i < used; ++i) {
    const Entry& e = cache[i];
    if (e.base == base && e.dim0 == dim0 && e.dim1 == dim1 && e.pitch == pitch_bytes && e.box0 == box0 && e.box1 == box1 &&
        e.as_int32 == as_int32 && e.l2_promo == l2_promo) {
      *map = e.map;
      return 0;
    }
  }
  const int rc = make_tensor_map_2d_f32(map, base, dim0, dim1, pitch_bytes, box0, box1, err, as_int32, l2_promo);
  if (rc) return rc;
  Entry& e = cache[next];
  e.base = base, e.dim0 = dim0, e.dim1 = dim1, e.pitch = pitch_bytes, e.box0 = box0, e.box1 = box1, e.as_int32 = as_int32,
  e.l2_promo = l2_promo, e.map = *map;
  next = (next + 1) % kN;
  if (used < kN) ++used;
  return 0;
}

}  // namespace rl
