// uint8 input windows for the conv1 kernels (K6): the observation stays uint8 in HBM (the frames a PARL actor
// sends are uint8, examples/IMPALA/atari_agent.py:35-42 divides by 255 in the model) and becomes the bf16
// SWIZZLE_128B operand only in shared memory, inside the kernels that consume it.
//
// Per position tile the producer's TMA brings the DENSE uint8 window [wrows][64 B] into a staging ring; 256
// converter threads (4 per row, 16 input bytes each) write the 128-byte bf16 rows of the operand window exactly
// where a SWIZZLE_128B tensor-map load would have put them — 16-byte chunk j of row r lands at chunk j ^ (r & 7)
// (the window base is 1024-byte aligned) — then fence.proxy.async + mbarrier.arrive hand the window to the
// wgmma consumers.  byte -> bf16(byte * scale) uses the same 2^23 magic-number FMA and cvt.rn.bf16x2 as the
// bf16 gather (rl_obs_stack_gather out_dtype 3), so both input forms give bit-identical operands.
#pragma once
#include <cuda.h>
#include <stdint.h>

#include "tma.cuh"

namespace rl {

constexpr int kU8Stages = 3;       // uint8 staging ring depth
constexpr int kU8Threads = 256;    // converter threads (8 warps: two per scheduler, the conversion is issue-bound)

#ifdef __CUDACC__
__device__ __forceinline__ int u8_stage_bytes(int wrows) { return (wrows * 64 + 1023) & ~1023; }

// 16 bytes -> 16 x bf16(byte * scale): per byte one PRMT (2^23 magic number), one FFMA, half a cvt.bf16x2
__device__ __forceinline__ void u8x16_to_bf16(const uint4 in, float scale, float bias, uint32_t (&pk)[8]) {
  const uint32_t w[4] = {in.x, in.y, in.z, in.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float f0 = __fmaf_rn(__uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7540u)), scale, bias);
    const float f1 = __fmaf_rn(__uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7541u)), scale, bias);
    const float f2 = __fmaf_rn(__uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7542u)), scale, bias);
    const float f3 = __fmaf_rn(__uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7543u)), scale, bias);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;\n" : "=r"(pk[2 * i]) : "f"(f1), "f"(f0));
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;\n" : "=r"(pk[2 * i + 1]) : "f"(f3), "f"(f2));
  }
}

// ct in [0, kU8Threads): thread ct handles 16-byte chunk (ct & 3) of rows (ct >> 2) + 64 k.  Three rows per pass with
// all loads issued before the first conversion (wrows <= 192 is one pass).
__device__ __forceinline__ void u8_window_to_bf16_sw128(const unsigned char* __restrict__ stage,
                                                        unsigned char* __restrict__ win, int wrows, int ct, float scale,
                                                        float bias) {
  constexpr int RPP = kU8Threads / 4;            // rows per pass step
  const int q = ct & 3, r0 = ct >> 2;
  // row & 7 == r0 & 7 for every row of this thread (RPP is a multiple of 8): the swizzled chunk offsets are fixed
  const int o0 = ((2 * q) ^ (r0 & 7)) << 4, o1 = ((2 * q + 1) ^ (r0 & 7)) << 4;
  for (int base = r0; base < wrows; base += 3 * RPP) {
    uint4 in[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (base + k * RPP < wrows) in[k] = *reinterpret_cast<const uint4*>(stage + (base + k * RPP) * 64 + q * 16);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (base + k * RPP < wrows) {
        uint32_t pk[8];
        u8x16_to_bf16(in[k], scale, bias, pk);
        unsigned char* drow = win + (base + k * RPP) * 128;
        *reinterpret_cast<uint4*>(drow + o0) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        *reinterpret_cast<uint4*>(drow + o1) = make_uint4(pk[4], pk[5], pk[6], pk[7]);
      }
    }
  }
}
#endif

// Host: tensor map of a uint8 [rows][64] matrix, box {64, box_rows}, dense (no swizzle) rows in shared memory.
inline int make_tensor_map_u8_rows64(CUtensorMap* map, const void* base, uint64_t rows, uint32_t box_rows) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return -1;
    fn = reinterpret_cast<EncodeFn>(p);
  }
  const cuuint64_t gdim[2] = {64, rows};
  const cuuint64_t gstride[1] = {64};
  const cuuint32_t box[2] = {64, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), gdim, gstride, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS
             ? 0
             : -2;
}

}  // namespace rl
