// K6 (convolution weight gradient, TMA-window form) — for a stride-1 NHWC conv written as shifted GEMMs
//     out[q, co] = sum_t sum_ci in[q + off_t, ci] W_t[co, ci]
// the weight gradient is a sum over ALL positions of outer products
//     dW_t[co, ci] = sum_q in[q + off_t, ci] * dout_grid[q, co]
// i.e. per tap a GEMM whose reduction (K) dimension is the position index q.  Both operands are read exactly
// as they lie in HBM — rows = positions, contiguous channels — through the same TMA windows as the forward kernel and
// consumed by wgmma as MN-MAJOR operands: A = input window starting off_t rows down (M = 64 input channels of one
// channel block, SWIZZLE_128B), B = dout tile (N = Cout; SWIZZLE_128B for 64 channels, SWIZZLE_64B for 32), K = 16
// positions per instruction.  Every (tap, channel block) pair is an accumulator "slot" of 64 x Cout fp32 registers
// that stays in the registers of one consumer warpgroup across the CTA's whole persistent loop over position tiles.
// The bias gradient rides along as one more slot whose A operand is a constant tile of ones,
//     D_b[m, co] += sum_q 1 * dout[q, co]        (every row m holds the column sums; row 0 is read back)
// so the gradient grid is not streamed from HBM a second time by a column-sum kernel.  Slots beyond what two
// warpgroups hold (kWgSlots each) are split over CTA groups.  Partials are dumped once per CTA and reduced in fixed
// order by a second kernel (deterministic).
#include <cuda_bf16.h>

#include "common.cuh"
#include "tma.cuh"
#include "u8win.cuh"
#include "wgmma.cuh"

namespace rl {

constexpr int kWgBM = 128;            // positions (K of the GEMM) per tile
constexpr int kWgMaxStages = 6;
constexpr int kWgThreads = 384;       // producer warpgroup (warp 0 active) + 2 consumer warpgroups
constexpr int kWgSlots = 4;           // accumulator slots per consumer warpgroup (4 x 64 x 64 fp32 = 128 registers)
constexpr int kWgMaxCtas = 160;       // grid bound the workspace is sized for

struct WgradArgs {
  float* partials;                    // [gridDim.x][per_group slots][64 rows][COUT]
  int W, KW, ntaps;
  int wrows, num_tiles, stages;
  int ngroups, per_group;             // slot s lives in group s / per_group; CTA b belongs to group b % ngroups
  int bias;                           // 1: the last slot is the bias gradient (column sums of dout)
  float in_scale;                     // U8X: input operand = bf16(byte * in_scale)
};

// U8X (conv1 on the uint8 observation): map_x is the uint8 [Q][64] matrix; the producer fills a dense staging ring
// and 256 more threads convert each window into the bf16 SWIZZLE_128B slot (u8win.cuh).
// DOUT_A (rl_debug_set_wgrad_lane_map(2), Cout = 64, no bias slot): the operand roles swapped — A = dout tile
// (M = 64 output channels), B = shifted input window (N = 64 input channels), accumulator rows = output channels —
// an independent cross-check of the MN-major descriptors in both operand positions.
template <int COUT, int CBLK, bool U8X = false, bool DOUT_A = false>
__global__ void __launch_bounds__(U8X ? kWgThreads + kU8Threads : kWgThreads, 1)
    wgrad_kernel(const __grid_constant__ CUtensorMap map_dout, const __grid_constant__ CUtensorMap map_x, const WgradArgs g) {
  static_assert(!U8X || CBLK == 1, "the uint8 window is one 64-channel block");
  static_assert(!DOUT_A || (COUT == 64 && !U8X), "the swapped-role form is built for 64 output channels");
  constexpr int DOUT_BYTES = kWgBM * COUT * 2;                        // 16 KB (SW128) or 8 KB (SW64)
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  const int win_bytes = (g.wrows * 128 + 1023) & ~1023;
  const int stage_bytes = CBLK * win_bytes + DOUT_BYTES;              // windows first (1024-byte aligned), then dout
  __shared__ __align__(8) unsigned long long full_bar[kWgMaxStages], empty_bar[kWgMaxStages];
  __shared__ __align__(8) unsigned long long u8_full[kU8Stages], u8_empty[kU8Stages];
  const uint32_t nstages = (uint32_t)g.stages;
  const int gid = blockIdx.x % g.ngroups;
  const int cta_in_group = blockIdx.x / g.ngroups, ctas_per_group = (gridDim.x + g.ngroups - 1 - gid) / g.ngroups;
  // constant A operand of the bias-gradient slot: 16 K-rows x 64 bf16 ones, after the stage ring
  unsigned char* s_ones = smem + nstages * stage_bytes;
  unsigned char* sStage = s_ones + 2048;                              // U8X: [kU8Stages][wrows][64 B]
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_dout);
    tma_prefetch_desc(&map_x);
    for (int s = 0; s < kWgMaxStages; ++s) {
      mbar_init(&full_bar[s], U8X ? 1 + kU8Threads : 1);   // U8X: the dout TMA + every converter thread
      mbar_init(&empty_bar[s], 2);                          // one arrival per consumer warpgroup
    }
    for (int s = 0; s < kU8Stages; ++s) {
      mbar_init(&u8_full[s], 1);
      mbar_init(&u8_empty[s], kU8Threads);
    }
    fence_mbar_init();
  }
  if (g.bias) {
    for (int i = threadIdx.x; i < 512; i += blockDim.x) reinterpret_cast<uint32_t*>(s_ones)[i] = 0x3F803F80u;
    fence_proxy_async_smem();               // generic-proxy stores -> visible to the tensor core's async proxy
  }
  __syncthreads();

  if (threadIdx.x < 128) {
    if (threadIdx.x == 0) {
      uint32_t s = 0, par = 1, ss = 0, spar = 1;
      const int sbytes = u8_stage_bytes(g.wrows);
      for (int tile = cta_in_group; tile < g.num_tiles; tile += ctas_per_group) {
        if (U8X) {
          mbar_wait(&u8_empty[ss], spar);
          mbar_arrive_expect_tx(&u8_full[ss], (uint32_t)(g.wrows * 64));
          tma_load_2d(sStage + ss * sbytes, &map_x, 0, tile * kWgBM, &u8_full[ss]);
          if (++ss == kU8Stages) ss = 0, spar ^= 1u;
        }
        mbar_wait(&empty_bar[s], par);
        mbar_arrive_expect_tx(&full_bar[s], (uint32_t)(DOUT_BYTES + (U8X ? 0 : CBLK * g.wrows * 128)));
        unsigned char* st = smem + s * stage_bytes;
        if (!U8X) {
#pragma unroll
          for (int cb = 0; cb < CBLK; ++cb) tma_load_2d(st + cb * win_bytes, &map_x, cb * 64, tile * kWgBM, &full_bar[s]);
        }
        tma_load_2d(st + CBLK * win_bytes, &map_dout, 0, tile * kWgBM, &full_bar[s]);
        if (++s == nstages) s = 0, par ^= 1u;
      }
    }
    return;
  }
  if (U8X && threadIdx.x >= kWgThreads) {
    // uint8 -> bf16 window converters
    const int ct = threadIdx.x - kWgThreads;
    const int sbytes = u8_stage_bytes(g.wrows);
    const float cbias = -8388608.0f * g.in_scale;
    uint32_t s = 0, epar = 1, ss = 0, fpar = 0;
    for (int tile = cta_in_group; tile < g.num_tiles; tile += ctas_per_group) {
      mbar_wait(&u8_full[ss], fpar);
      mbar_wait(&empty_bar[s], epar);            // the MMAs that read this slot have completed
      u8_window_to_bf16_sw128(sStage + ss * sbytes, smem + s * stage_bytes, g.wrows, ct, g.in_scale, cbias);
      fence_proxy_async_smem();
      mbar_arrive(&full_bar[s]);
      mbar_arrive(&u8_empty[ss]);
      if (++s == nstages) s = 0, epar ^= 1u;
      if (++ss == kU8Stages) ss = 0, fpar ^= 1u;
    }
    return;
  }
  // ===== consumers: warpgroup c owns local slots [j0, j0 + nmine) of this CTA's group =====
  const int c = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127;
  const int nslots_all = g.ntaps * CBLK + g.bias;
  const int gs0 = gid * g.per_group, ngs = min(g.per_group, nslots_all - gs0);
  const int half = (ngs + 1) >> 1, j0 = c == 0 ? 0 : half, nmine = c == 0 ? half : ngs - half;
  constexpr uint32_t hiB = COUT == 64 ? kGmmaHiSw128 : kGmmaHiSw64;
  constexpr uint32_t kstepB = COUT == 64 ? 128u : 64u;               // 16 positions of dout rows, 16-byte units
  // Both warpgroups issue `half` MMA chains (a bound that does not depend on the thread index, so the wgmma stay
  // warpgroup-uniform and are not serialised); when ngs is odd the second warpgroup's last chain is a dummy that reads
  // the ones tile and is never written back.
  uint32_t a_off[kWgSlots];        // per slot: window shift + channel block (16-byte units), or the ones tile
  bool is_ones[kWgSlots];
#pragma unroll
  for (int j = 0; j < kWgSlots; ++j) {
    const int slot = gs0 + j0 + j;
    is_ones[j] = slot >= g.ntaps * CBLK || j >= nmine;
    const int tap = slot / CBLK, cb = slot - tap * CBLK, r = tap / g.KW;
    a_off[j] = is_ones[j] ? 0u : (uint32_t)((r * g.W + tap - r * g.KW) * 8 + cb * (win_bytes >> 4));
  }
  const uint32_t lo0 = gmma_lo(smem), stage16 = (uint32_t)stage_bytes >> 4, ones_lo = gmma_lo(s_ones);
  float d[kWgSlots][COUT / 2];
#pragma unroll
  for (int j = 0; j < kWgSlots; ++j)
#pragma unroll
    for (int i = 0; i < COUT / 2; ++i) d[j][i] = 0.f;
  uint32_t s = 0, par = 0;
  for (int tile = cta_in_group; tile < g.num_tiles; tile += ctas_per_group) {
    mbar_wait(&full_bar[s], par);
    wgmma_fence();
    const uint32_t x_lo = lo0 + s * stage16;
    const uint32_t b_lo = x_lo + (uint32_t)((CBLK * win_bytes) >> 4);
#pragma unroll
    for (int j = 0; j < kWgSlots; ++j) {
      if (j < half) {
#pragma unroll
        for (int kk = 0; kk < kWgBM / 16; ++kk) {   // 16 positions = 16 window rows (128 units) per K step
          const uint32_t a_lo = is_ones[j] ? ones_lo : x_lo + a_off[j] + kk * 128u;
          if constexpr (DOUT_A)
            wgmma_bf16<COUT, 1, 1>(d[j], gmma_desc(kGmmaHiSw128, b_lo + kk * kstepB), gmma_desc(kGmmaHiSw128, a_lo), 1u);
          else
            wgmma_bf16<COUT, 1, 1>(d[j], gmma_desc(kGmmaHiSw128, a_lo), gmma_desc(hiB, b_lo + kk * kstepB), 1u);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (t == 0) mbar_arrive(&empty_bar[s]);
    if (++s == nstages) s = 0, par ^= 1u;
  }
#pragma unroll
  for (int j = 0; j < kWgSlots; ++j) {
    wgmma_fence_regs(d[j]);
    if (j < nmine) {
      float* dst = g.partials + ((size_t)blockIdx.x * g.per_group + j0 + j) * 64 * COUT;
#pragma unroll
      for (int i = 0; i < COUT / 2; i += 2)
        *reinterpret_cast<float2*>(dst + gmma_row(t, i) * COUT + gmma_col(t, i)) = make_float2(d[j][i], d[j][i + 1]);
    }
  }
}

// dW[co][(tap, cb, ci)] = sum over the CTAs of the slot's group in index order (deterministic); db[co] from row 0 of
// the bias slot.  dout_rows: the partial tiles are [co][ci] (swapped-role form) instead of [ci][co].
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ partials, int nctas, int ngroups,
                                                           int per_group, int ntaps, int cblk, int cout, int dout_rows,
                                                           float* __restrict__ dw, float* __restrict__ db, int accumulate) {
  const int K = ntaps * cblk * 64;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int slot, row, co;
  if (idx >= cout * K) {
    co = idx - cout * K;
    if (!db || co >= cout) return;
    slot = ntaps * cblk, row = 0;
  } else {
    co = idx / K;
    const int k = idx - co * K;
    slot = k >> 6, row = k & 63;                        // k = (tap * cblk + cb) * 64 + ci
  }
  const int gid = slot / per_group, local = slot - gid * per_group;
  float acc = 0.f;
  const size_t off = dout_rows ? (size_t)co * 64 + row : (size_t)row * cout + co;
  for (int c = gid; c < nctas; c += ngroups) acc += partials[((size_t)c * per_group + local) * 64 * cout + off];
  if (idx >= cout * K) db[co] = accumulate ? db[co] + acc : acc;
  else dw[idx] = accumulate ? dw[idx] + acc : acc;
}

// column sums of a [rows, C] bf16 matrix (bias gradients): deterministic two-stage, 16-byte loads.
// A thread owns 8 adjacent columns (one uint4) and walks the rows of its block's chunk with stride
// (256 / (C/8)) so that a warp reads whole 128-byte lines.
__global__ void __launch_bounds__(256) colsum_bf16_stage1(const __nv_bfloat16* __restrict__ x, long long rows, int C,
                                                          float* __restrict__ part) {
  const int vpr = C >> 3;                              // uint4 vectors per row
  const long long chunk = (rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = (long long)blockIdx.x * chunk, r1 = min(rows, r0 + chunk);
  __shared__ float sm[256][8];
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  if (vpr <= 256) {
    const int nph = 256 / vpr;                         // row phases handled concurrently by the block
    const int v = threadIdx.x % vpr, ph = threadIdx.x / vpr;
    if (ph < nph) {
      const uint4* base = reinterpret_cast<const uint4*>(x) + v;
      for (long long r = r0 + ph; r < r1; r += nph) {
        const uint4 q = __ldcs(base + r * vpr);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[2 * i] += __uint_as_float(w[i] << 16);
          acc[2 * i + 1] += __uint_as_float(w[i] & 0xffff0000u);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) sm[threadIdx.x][i] = acc[i];
    __syncthreads();
    if (threadIdx.x < vpr) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float a = 0.f;
        for (int p = 0; p < nph; ++p) a += sm[p * vpr + threadIdx.x][i];
        part[(size_t)blockIdx.x * C + threadIdx.x * 8 + i] = a;
      }
    }
  } else {
    for (int c = threadIdx.x; c < C; c += 256) {       // very wide matrices: scalar fallback
      float a = 0.f;
      for (long long r = r0; r < r1; ++r) a += __bfloat162float(x[r * C + c]);
      part[(size_t)blockIdx.x * C + c] = a;
    }
  }
}
__global__ void colsum_stage2(const float* __restrict__ part, int nblocks, int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f;
  for (int b = 0; b < nblocks; ++b) a += part[(size_t)b * C + c];
  out[c] = a;
}

static int wg_make_map(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint32_t box_rows,
                       uint32_t box_cols = 64, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
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
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {cols * 2};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS
             ? 0
             : -2;
}

}  // namespace rl

using namespace rl;

// Weight-gradient form.  0 (default): A = input window, B = dout, bias gradient as a slot against a tile of ones;
// 2: for 64 output channels the operand roles swapped (wgrad_kernel<64, CBLK, false, true>), and the bias gradient from
// rl_colsum_bf16 — a cross-check of the default form (Cout = 32 keeps the default roles, the uint8 input the default form).
static int g_wg_form = 0;
extern "C" int rl_debug_set_wgrad_lane_map(int mode) {
  RL_CHECK_ARG(mode == 0 || mode == 2, "wgrad form must be 0 (default) or 2 (swapped operand roles)");
  g_wg_form = mode;
  return RL_OK;
}

static void wgrad_groups(int ntaps, int cblk, int bias, int* ngroups, int* per_group) {
  const int nslots = ntaps * cblk + bias;
  *ngroups = (nslots + 2 * kWgSlots - 1) / (2 * kWgSlots);
  *per_group = (nslots + *ngroups - 1) / *ngroups;
}

// Enough for every call with these filter dimensions: with or without the bias-gradient slot (the slot count, and so
// the slots per CTA group, differ), either form, and the column-sum pass of form 2 (rl_colsum_bf16: 1184 x Cout floats).
extern "C" size_t rl_conv_wgrad_workspace_bytes(int KH, int KW, int Cin) {
  size_t need = (size_t)1184 * 64 * sizeof(float);
  for (int bias = 0; bias <= 1; ++bias) {
    int ngroups = 1, per = 1;
    wgrad_groups(KH * KW, Cin / 64, bias, &ngroups, &per);
    const size_t b = (size_t)kWgMaxCtas * per * 64 * 64 * sizeof(float);
    if (b > need) need = b;
  }
  return need + 4096;
}

static int wgrad_dispatch(const void* dout_grid, const void* in, float* dw_krsc, float* db, int N, int H, int W, int Cin,
                          int Cout, int KH, int KW, int accumulate, void* workspace, size_t workspace_bytes,
                          rl_stream_t stream, int u8in, float in_scale) {
  RL_CHECK_ARG(dout_grid && in && dw_krsc && workspace && N > 0, "conv2d_s1_wgrad: bad argument");
  RL_CHECK_ARG(aligned16(dout_grid) && aligned16(in) && aligned16(workspace), "conv2d_s1_wgrad: alignment");
  RL_CHECK_ARG((Cout == 64 && (Cin == 64 || Cin == 128)) || (Cout == 32 && Cin == 64),
               "conv2d_s1_wgrad: (Cout, Cin) must be (64, 64|128) or (32, 64)");
  const long long Q = (long long)N * H * W;
  RL_CHECK_ARG(Q < (1LL << 31), "conv2d_s1_wgrad: too many positions");
  const int cblk = Cin / 64, ntaps = KH * KW;
  WgradArgs a;
  a.partials = reinterpret_cast<float*>(workspace);
  a.W = W, a.KW = KW, a.ntaps = ntaps, a.wrows = kWgBM + (KH - 1) * W + (KW - 1);
  RL_CHECK_ARG(a.wrows <= 256, "conv2d_s1_wgrad: window too tall");
  const bool legacy = g_wg_form == 2 && !u8in;
  RL_CHECK_ARG(!(legacy && db && accumulate), "conv2d_s1_wgrad: accumulate with a bias gradient needs the default form");
  a.num_tiles = (int)((Q + kWgBM - 1) / kWgBM), a.bias = (db && !legacy) ? 1 : 0, a.in_scale = in_scale;
  wgrad_groups(ntaps, cblk, a.bias, &a.ngroups, &a.per_group);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  sms = effective_sms(sms);
  // CTAs per group: one per position tile at most; the whole grid at most one per SM (and kWgMaxCtas)
  long long per_grp = (sms < kWgMaxCtas ? sms : kWgMaxCtas) / a.ngroups;
  if (per_grp < 1) per_grp = 1;
  if (per_grp > a.num_tiles) per_grp = a.num_tiles;
  const int grid = (int)per_grp * a.ngroups;
  if (workspace_bytes < (size_t)grid * a.per_group * 64 * Cout * sizeof(float)) {
    set_error("conv2d_s1_wgrad: workspace too small");
    return RL_ERR_WORKSPACE;
  }
  alignas(64) CUtensorMap md, mx;
  if (wg_make_map(&md, dout_grid, (uint64_t)Cout, (uint64_t)Q, kWgBM, (uint32_t)Cout,
                  Cout == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B) ||
      (u8in ? make_tensor_map_u8_rows64(&mx, in, (uint64_t)Q, (uint32_t)a.wrows)
            : wg_make_map(&mx, in, (uint64_t)Cin, (uint64_t)Q, (uint32_t)a.wrows))) {
    set_error("conv2d_s1_wgrad: cuTensorMapEncodeTiled failed");
    return RL_ERR_CUDA;
  }
  const size_t win = (size_t)((a.wrows * 128 + 1023) & ~1023);
  const size_t stage = (size_t)cblk * win + (size_t)kWgBM * Cout * 2;
  const size_t u8ring = u8in ? (size_t)kU8Stages * (size_t)((a.wrows * 64 + 1023) & ~1023) : 0;
  const long long nst = (long long)((216 * 1024 - u8ring) / stage);
  a.stages = (int)(nst > kWgMaxStages ? kWgMaxStages : (nst < 2 ? 2 : nst));
  const size_t smem = (size_t)a.stages * stage + 2048 + 1024 + u8ring;   // + the 2 KB tile of ones (+ uint8 staging)
  cudaStream_t st = (cudaStream_t)stream;
  if (u8in) {
    RL_CHECK_ARG(Cout == 32 && cblk == 1, "conv2d_s1_u8in_wgrad: Cout 32, Cin 64");
    auto kern = wgrad_kernel<32, 1, true>;
    RL_SMEM_OPTIN(kern);
    kern<<<grid, kWgThreads + kU8Threads, smem, st>>>(md, mx, a);
  } else if (legacy && Cout == 64 && cblk == 1) {
    auto kern = wgrad_kernel<64, 1, false, true>;
    RL_SMEM_OPTIN(kern);
    kern<<<grid, kWgThreads, smem, st>>>(md, mx, a);
  } else if (legacy && Cout == 64) {
    auto kern = wgrad_kernel<64, 2, false, true>;
    RL_SMEM_OPTIN(kern);
    kern<<<grid, kWgThreads, smem, st>>>(md, mx, a);
  } else if (Cout == 64 && cblk == 1) {
    RL_SMEM_OPTIN(wgrad_kernel<64, 1>);
    wgrad_kernel<64, 1><<<grid, kWgThreads, smem, st>>>(md, mx, a);
  } else if (Cout == 64) {
    RL_SMEM_OPTIN(wgrad_kernel<64, 2>);
    wgrad_kernel<64, 2><<<grid, kWgThreads, smem, st>>>(md, mx, a);
  } else {
    RL_SMEM_OPTIN(wgrad_kernel<32, 1>);
    wgrad_kernel<32, 1><<<grid, kWgThreads, smem, st>>>(md, mx, a);
  }
  const int K = ntaps * cblk * 64;
  wgrad_reduce_kernel<<<(Cout * K + Cout + 255) / 256, 256, 0, st>>>(a.partials, grid, a.ngroups, a.per_group, ntaps, cblk,
                                                                     Cout, legacy && Cout == 64 ? 1 : 0, dw_krsc,
                                                                     a.bias ? db : nullptr, accumulate);
  RL_CHECK_LAUNCH("rl_conv2d_s1_nhwc_bf16_wgrad");
  // swapped-role form: the bias gradient by a column-sum pass (the partials are consumed: the workspace is free again)
  if (db && !a.bias) return rl_colsum_bf16(dout_grid, Q, Cout, db, workspace, workspace_bytes, stream);
  return RL_OK;
}

extern "C" int rl_conv2d_s1_nhwc_bf16_wgrad(const void* dout_grid, const void* in, float* dw_krsc, float* db, int N,
                                            int H, int W, int Cin, int Cout, int KH, int KW, int accumulate,
                                            void* workspace, size_t workspace_bytes, rl_stream_t stream) {
  return wgrad_dispatch(dout_grid, in, dw_krsc, db, N, H, W, Cin, Cout, KH, KW, accumulate, workspace, workspace_bytes,
                        stream, 0, 1.f);
}

extern "C" int rl_conv2d_s1_u8in_bf16_wgrad(const void* dout_grid, const void* in_u8, float in_scale, float* dw_krsc,
                                            float* db, int N, int H, int W, int Cout, int KH, int KW, int accumulate,
                                            void* workspace, size_t workspace_bytes, rl_stream_t stream) {
  RL_CHECK_ARG(Cout == 32 && KH == 2 && KW == 2, "conv2d_s1_u8in_wgrad: built for the 2x2, 64 -> 32 layer (conv1, space-to-depth)");
  return wgrad_dispatch(dout_grid, in_u8, dw_krsc, db, N, H, W, 64, Cout, KH, KW, accumulate, workspace, workspace_bytes,
                        stream, 1, in_scale);
}

extern "C" int rl_colsum_bf16(const void* x, long long rows, int C, float* out, void* workspace, size_t workspace_bytes,
                              rl_stream_t stream) {
  RL_CHECK_ARG(x && out && workspace && rows > 0 && C >= 8 && C % 8 == 0 && aligned16(x) &&
                   ((C / 8) > 256 || 256 % (C / 8) == 0),
               "colsum_bf16: C must be a multiple of 8 with C/8 dividing 256 (or C > 2048)");
  const int nblocks = 1184;
  if (workspace_bytes < (size_t)nblocks * C * sizeof(float)) {
    set_error("colsum_bf16: workspace too small (need %d*C*4 bytes)", nblocks);
    return RL_ERR_WORKSPACE;
  }
  colsum_bf16_stage1<<<nblocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, rows, C, (float*)workspace);
  colsum_stage2<<<(C + 63) / 64, 64, 0, (cudaStream_t)stream>>>((const float*)workspace, nblocks, C, out);
  RL_CHECK_LAUNCH("rl_colsum_bf16");
  return RL_OK;
}
