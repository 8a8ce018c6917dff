// K6 (convolutions, TMA-window form) — stride-1 NHWC bf16 convolution forward on the Hopper tensor cores where the
// A operand is never gathered: a stride-1 conv over the row-major flattened pixel sequence is a sum of SHIFTED GEMMs
//     out[q, :] = bias + sum_{r,s} in[q + r*W + s, :] . W[(r,s)]^T        q = n*H*W + y*W + x
// (positions with y >= Hout or x >= Wout are computed and dropped).  Per 128-position tile ONE 2-D TMA load
// brings the input window rows [q0, q0 + 128 + (KH-1)*W + (KW-1)) into shared memory (SWIZZLE_128B); every
// filter tap then issues wgmma with an smem descriptor that simply starts (r*W+s) rows further down
// (the swizzle phase follows from the absolute shared-memory address).  Each input byte crosses L2->SM once per tile
// instead of once per tap.  Stride-2/4 layers are brought to this form by space-to-depth of their INPUT
// (conv1: rl_obs_stack_gather out_dtype 3; conv2: conv1's epilogue writes the padded 2x2-block layout).
//
// Layers of the Atari actor-critic (a13: benchmark/torch/a2c/atari_model.py:26-44):
//   conv1  8x8/4/p1, 4->32   == 2x2/1 on [21,21,64]   -> [20,20,32] written as s2d2-padded [12,12,128]
//   conv2  4x4/2/p2, 32->64  == 2x2/1 on [12,12,128]  -> [11,11,64]
//   conv3  3x3/1,    64->64  == 3x3/1 on [11,11,64]   -> [9,9,64]
// Roles: warp 0 TMA producer (window ring; the data gradient's ring stage also holds the tile's ReLU mask, rows
// [128 tile, 128 tile + 128) of the saved activation, loaded with the window); consumer warpgroups 1 and 2 take
// alternate tiles of the CTA (weights resident in smem): each issues the tile's wgmma m64nCOUT chains for both 64-row
// halves into two register accumulators and runs the epilogue — one warpgroup's epilogue overlaps the other's MMAs.
// Forward: frees the window slot once the MMAs retire, then bias, ReLU, bf16 and layout-aware stores from the
// registers.  Data gradient: stmatrix of the bf16 tile over its mask, ANDed with the mask words that ldmatrix reads
// from the same place, then 16-byte chunks read back by consecutive threads, the ring stage freed, and the chunks
// stored as contiguous destination runs.
#include <cuda_bf16.h>

#include "common.cuh"
#include "tma.cuh"
#include "u8win.cuh"
#include "wgmma.cuh"

namespace rl {

constexpr int kScBM = 128;
constexpr int kScMaxStages = 8;      // window ring depth is chosen at launch from the shared memory left by the weights
constexpr int kScThreads = 384;      // producer warpgroup (warp 0 active) + 2 consumer warpgroups
constexpr int kScEpiBar = 1;         // named barriers kScEpiBar + c: the epilogue of consumer warpgroup c (128 threads)

struct ShiftConvArgs {
  const float* bias;
  __nv_bfloat16* out;
  int H, W, KH, KW, Hout, Wout;   // input grid per image, filter, valid output grid
  int Q;                           // N * H * W flattened input positions
  int wrows;                       // window rows = 128 + (KH-1)*W + (KW-1)
  int num_tiles, relu;
  int stages;                      // depth of the TMA window ring (2..kScMaxStages)
  int out_mode;                    // 0: NHWC grid [N,OGH,OGW,Cout] (valid y<Hout, x<Wout);
                                   // 1: conv1 -> conv2 s2d2-padded [N,12,12,4*Cout];
                                   // 2: (dgrad of the s2d2 conv) [N,12,12,128] blocks -> grid [N,21,21,32]
  int OGH, OGW;                    // output grid of out_mode 0
  int row_shift;                   // TMA row coordinate of a tile = tile*128 + row_shift (dgrad: -((KH-1)*W+KW-1))
  int flip;                        // 1: tap (r,s) reads window row (KH-1-r)*W + (KW-1-s)  (transposed conv)
  const __nv_bfloat16* mask;       // optional activation on the accumulator grid [Q, COUT]: out *= (mask > 0)
  float in_scale;                  // U8IN: operand = bf16(byte * in_scale)
};

// fp32 pair -> packed bf16x2 (lo = first argument), round-to-nearest-even; the ReLU form clamps in the same instruction
__device__ __forceinline__ uint32_t s_pack_bf16x2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;\n" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
__device__ __forceinline__ uint32_t s_pack_relu_bf16x2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;\n" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

// Byte offset of 16-byte chunk `ch` (columns 8ch .. 8ch + 7) of row `row` in a 128-row bf16 tile of the data gradient:
// 64-column blocks of 128-byte rows, 16 KB apart, in the SWIZZLE_128B layout that a TMA load of the saved activation
// writes (chunk ^ row % 8).  The 8 rows of one stmatrix / ldmatrix matrix, and 8 consecutive chunks of the copy-out,
// fall on distinct banks.
__device__ __forceinline__ uint32_t sc_tile_off(int row, int ch) {
  return (uint32_t)((ch >> 3) * (kScBM * 128) + row * 128 + (((ch & 7) ^ (row & 7)) << 4));
}

// MODE 0: forward  (out = act(acc + bias), ReLU optional)     MODE 1: data gradient (out = acc * (mask > 0), mask optional)
// U8IN (conv1 on the uint8 observation): map_in is the uint8 [Q][64] matrix, the producer fills a dense staging
// ring and 256 more threads convert each window into the bf16 SWIZZLE_128B ring (u8win.cuh).
// map_mask (MODE 1 with a mask): the saved activation [Q, COUT], 64-column x 128-row SWIZZLE_128B boxes.
// The forward stores from the accumulator registers.  The data gradient stages its bf16 tile in shared memory and
// writes it in 16-byte chunks; the forward does not: staging made conv3's MMA-bound forward (N = 64, 3x3) 10-15% and
// the uint8 conv1 forward at the actor batch about 10% slower (H100 80GB HBM3, 400 W).
template <int COUT, int CBLK, int KS, int MODE, bool U8IN = false>
__global__ void __launch_bounds__(U8IN ? kScThreads + kU8Threads : kScThreads, 1)
    shiftconv_fwd_kernel(const __grid_constant__ CUtensorMap map_in, const __grid_constant__ CUtensorMap map_w,
                         const __grid_constant__ CUtensorMap map_mask, const ShiftConvArgs g) {
  static_assert(!U8IN || CBLK == 1, "the uint8 window is one 64-channel block");
  static_assert(MODE == 0 || COUT % 64 == 0, "the data gradient's tile is made of 64-column mask boxes");
  constexpr int W_KB = COUT * 128;                        // one 64-wide weight k-block
  constexpr int OUT_BYTES = kScBM * COUT * 2;             // one bf16 data-gradient tile
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  constexpr int num_kb = KS * KS * CBLK;                  // square KS x KS filter
  const int win_bytes = (g.wrows * 128 + 1023) & ~1023;   // one 64-channel column block of the window
  unsigned char* sW = smem;                               // [num_kb][COUT][128 B]
  unsigned char* sWin = smem + ((num_kb * W_KB + 1023) & ~1023);   // [stages][CBLK][wrows][128 B]
  __shared__ __align__(8) unsigned long long full_bar[kScMaxStages], empty_bar[kScMaxStages], w_bar;
  __shared__ __align__(8) unsigned long long u8_full[kU8Stages], u8_empty[kU8Stages];
  const uint32_t nstages = (uint32_t)g.stages;
  unsigned char* sStage = sWin + nstages * CBLK * win_bytes;       // U8IN: [kU8Stages][wrows][64 B]
  unsigned char* sOut = sWin + nstages * CBLK * win_bytes;         // MODE 1: [stages][OUT_BYTES] mask / output tiles
  const bool has_mask = MODE == 1 && g.mask != nullptr;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_in);
    tma_prefetch_desc(&map_w);
    if (has_mask) tma_prefetch_desc(&map_mask);
    for (int s = 0; s < kScMaxStages; ++s) {
      mbar_init(&full_bar[s], U8IN ? kU8Threads : 1);
      mbar_init(&empty_bar[s], MODE == 0 ? 1 : 128);   // data gradient: every consumer thread, after its copy-out reads
    }
    for (int s = 0; s < kU8Stages; ++s) {
      mbar_init(&u8_full[s], 1);
      mbar_init(&u8_empty[s], kU8Threads);
    }
    mbar_init(&w_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  // resident weights: requested BEFORE the dependency wait (they are written by the operand refresh, at least two
  // kernels back in the stream), so the load overlaps the tail of the previous kernel
  if (threadIdx.x == 128) {
    mbar_arrive_expect_tx(&w_bar, (uint32_t)(num_kb * W_KB));
    for (int kb = 0; kb < num_kb; ++kb) tma_load_2d(sW + kb * W_KB, &map_w, kb * 64, 0, &w_bar);
  }
  pdl_wait();            // chain kernel (launch_chain): the input activations come from the previous kernel
  pdl_trigger();

  if (warp < 4) {
    // ===== TMA producer: one window (CBLK column blocks) per tile =====
    if (warp == 0 && lane == 0) {
      uint32_t s = 0, par = 1;
      if (U8IN) {
        const int sbytes = u8_stage_bytes(g.wrows);
        for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
          mbar_wait(&u8_empty[s], par);
          mbar_arrive_expect_tx(&u8_full[s], (uint32_t)(g.wrows * 64));
          tma_load_2d(sStage + s * sbytes, &map_in, 0, tile * kScBM + g.row_shift, &u8_full[s]);
          if (++s == kU8Stages) s = 0, par ^= 1u;
        }
      } else {
        const uint32_t tx = (uint32_t)(CBLK * g.wrows * 128) + (has_mask ? (uint32_t)OUT_BYTES : 0u);
        for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
          mbar_wait(&empty_bar[s], par);
          mbar_arrive_expect_tx(&full_bar[s], tx);
#pragma unroll
          for (int cb = 0; cb < CBLK; ++cb)
            tma_load_2d(sWin + (s * CBLK + cb) * win_bytes, &map_in, cb * 64, tile * kScBM + g.row_shift, &full_bar[s]);
          if (has_mask) {
            // rows past Q of the last tile are zero-filled (and never stored)
#pragma unroll
            for (int cb = 0; cb < COUT / 64; ++cb)
              tma_load_2d(sOut + s * OUT_BYTES + cb * (kScBM * 128), &map_mask, cb * 64, tile * kScBM, &full_bar[s]);
          }
          if (++s == nstages) s = 0, par ^= 1u;
        }
      }
    }
    return;
  }
  if (U8IN && threadIdx.x >= kScThreads) {
    // ===== uint8 -> bf16 window converters =====
    const int ct = threadIdx.x - kScThreads;
    const int sbytes = u8_stage_bytes(g.wrows);
    const float bias = -8388608.0f * g.in_scale;
    uint32_t s = 0, epar = 1, ss = 0, fpar = 0;
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      mbar_wait(&u8_full[ss], fpar);
      mbar_wait(&empty_bar[s], epar);              // the MMAs that read this window slot have completed
      u8_window_to_bf16_sw128(sStage + ss * sbytes, sWin + s * win_bytes, g.wrows, ct, g.in_scale, bias);
      fence_proxy_async_smem();                    // generic-proxy stores -> visible to the tensor core's async proxy
      mbar_arrive(&full_bar[s]);
      mbar_arrive(&u8_empty[ss]);
      if (++s == nstages) s = 0, epar ^= 1u;
      if (++ss == kU8Stages) ss = 0, fpar ^= 1u;
    }
    return;
  }
  // ===== consumers: warpgroup c takes tiles it = c, c + 2, ... of this CTA =====
  const int c = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127;
  mbar_wait(&w_bar, 0);
  // tap shifts in 16-byte descriptor units (8 per 128-byte window row)
  uint32_t tap_off[KS * KS];
#pragma unroll
  for (int r = 0; r < KS; ++r)
#pragma unroll
    for (int sx = 0; sx < KS; ++sx)
      tap_off[r * KS + sx] = (uint32_t)(g.flip ? (KS - 1 - r) * g.W + (KS - 1 - sx) : r * g.W + sx) * 8u;
  const uint32_t w_lo = gmma_lo(sW), win_lo0 = gmma_lo(sWin);
  const uint32_t win16 = (uint32_t)win_bytes >> 4;
  float bias_r[MODE == 0 ? COUT / 2 : 1];           // bias of the column of each accumulator element
  if (MODE == 0) {
#pragma unroll
    for (int i = 0; i < COUT / 2; ++i) bias_r[i] = __ldg(g.bias + gmma_col(t, i));
  }
  const bool relu = g.relu != 0;
  const int HW = g.H * g.W;
  constexpr int CH = COUT / 8;                      // 16-byte chunks of an output row
  // stmatrix / ldmatrix: lane l addresses row l % 8 of matrix l / 8 = (row half (l / 8) % 2, chunk j + l / 16)
  const int mx_row = 16 * (t >> 5) + (lane & 7) + 8 * ((lane >> 3) & 1), mx_ch = lane >> 4;
  // copy-out: thread t moves chunk t % CH of rows t / CH + RSTEP k, consecutive threads cover a row's chunks in order
  constexpr int RSTEP = kScBM / CH;
  const int cp_ch = t % CH, cp_row = t / CH;
  uint32_t s = (uint32_t)c, full_par = 0;
  for (long long tile = blockIdx.x + (long long)c * gridDim.x; tile < g.num_tiles; tile += 2 * gridDim.x) {
    float d[2][COUT / 2];                            // rows [0, 64) and [64, 128) of the tile
    mbar_wait(&full_bar[s], full_par);
    wgmma_fence();
    const uint32_t a_lo = win_lo0 + s * (CBLK * win16);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int tap = 0; tap < KS * KS; ++tap) {
#pragma unroll
        for (int cb = 0; cb < CBLK; ++cb) {
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_bf16<COUT>(d[h], gmma_desc(kGmmaHiSw128, a_lo + h * 512u + cb * win16 + tap_off[tap] + 2u * k),
                             gmma_desc(kGmmaHiSw128, w_lo + (uint32_t)((tap * CBLK + cb) * (W_KB >> 4) + 2 * k)),
                             (tap | cb | k) != 0 ? 1u : 0u);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(d[0]);
    wgmma_fence_regs(d[1]);
    if constexpr (MODE == 0) {
      // forward: the window slot is free as soon as the MMAs retire; bias + ReLU, bf16, stored from the registers
      if (t == 0) mbar_arrive(&empty_bar[s]);
      s += 2;
      if (s >= nstages) s -= nstages, full_par ^= 1u;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {             // the thread's two rows of this half: r0 and r0 + 8
          const int q = (int)tile * kScBM + 64 * h + gmma_row(t, 2 * rr);
          const int n = q / HW;
          const int rem = q - n * HW;
          const int y = rem / g.W, x = rem - y * g.W;
          const bool valid = q < g.Q && y < g.Hout && x < g.Wout;
          size_t obase;
          if (g.out_mode == 0) {
            obase = ((size_t)(n * g.OGH + y) * g.OGW + x) * COUT;
          } else {
            // conv1 -> conv2 input: zero-padded by 2, 2x2 space-to-depth: [n, (y+2)/2, (x+2)/2, ((y&1)*2 + (x&1))*COUT + c]
            const int yp = y + 2, xp = x + 2;
            obase = (((size_t)n * 12 + (yp >> 1)) * 12 + (xp >> 1)) * (4 * COUT) + (size_t)(((yp & 1) * 2 + (xp & 1)) * COUT);
          }
#pragma unroll
          for (int j = 0; j < CH; ++j) {
            const int i = 4 * j + 2 * rr;
            if (!valid) continue;
            const float v0 = d[h][i] + bias_r[i], v1 = d[h][i + 1] + bias_r[i + 1];
            *reinterpret_cast<uint32_t*>(g.out + obase + gmma_col(t, i)) =
                relu ? s_pack_relu_bf16x2(v0, v1) : s_pack_bf16x2(v0, v1);
          }
        }
      }
    } else {
      // data gradient: the bf16 tile is staged over the tile's mask (or in the mask slot), then copied out
      const unsigned char* tile_p = sOut + s * OUT_BYTES;
      const uint32_t otile = smem_u32(tile_p);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int j = 0; j < CH; j += 2) {
          uint32_t pk[4];                            // matrix m = (row half m % 2, chunk j + m / 2): elements 4j + 2m, +1
#pragma unroll
          for (int m = 0; m < 4; ++m) pk[m] = s_pack_bf16x2(d[h][4 * j + 2 * m], d[h][4 * j + 2 * m + 1]);
          const uint32_t a = otile + sc_tile_off(64 * h + mx_row, j + mx_ch);
          if (has_mask) {
            // ReLU backward: keep the gradient where the saved activation is > 0 — one packed bf16x2 compare per word
            uint32_t mw[4];
            ldmatrix_x4(a, mw);
#pragma unroll
            for (int m = 0; m < 4; ++m)
              pk[m] &= __hgt2_mask(*reinterpret_cast<const __nv_bfloat162*>(&mw[m]), __floats2bfloat162_rn(0.f, 0.f));
          }
          stmatrix_x4(a, pk);
        }
      }
      named_bar_sync(kScEpiBar + c, 128);            // the warpgroup's tile is staged
      uint4 v[CH];
#pragma unroll
      for (int k = 0; k < CH; ++k) v[k] = *reinterpret_cast<const uint4*>(tile_p + sc_tile_off(cp_row + RSTEP * k, cp_ch));
      fence_proxy_async_smem();                      // these generic accesses come before the next TMA write of the slot
      mbar_arrive(&empty_bar[s]);                    // every thread: the window and the mask slot are free
      s += 2;
      if (s >= nstages) s -= nstages, full_par ^= 1u;
      int q = (int)tile * kScBM + cp_row;
      int n = q / HW;
      int y = (q - n * HW) / g.W;
      int x = q - n * HW - y * g.W;
#pragma unroll
      for (int k = 0; k < CH; ++k) {
        const int col = 8 * cp_ch;
        bool ok = q < g.Q;
        size_t dst_off;
        if (g.out_mode == 0) {
          ok = ok && y < g.Hout && x < g.Wout;
          dst_off = ((size_t)(n * g.OGH + y) * g.OGW + x) * COUT + col;
        } else {
          // channel block (dy,dx) of position (Y,X) is pixel (2Y+dy-2, 2X+dx-2) of the 20x20 image, 32 channels
          const int blk = col >> 5, py = 2 * y + (blk >> 1) - 2, px = 2 * x + (blk & 1) - 2;
          ok = ok && py >= 0 && py < 20 && px >= 0 && px < 20;
          dst_off = (((size_t)n * 21 + py) * 21 + px) * 32 + (col & 31);
        }
        if (ok) *reinterpret_cast<uint4*>(g.out + dst_off) = v[k];
        q += RSTEP;
        for (x += RSTEP; x >= g.W; x -= g.W)
          if (++y == g.H) y = 0, ++n;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Column-tap form (rl_debug_set_shiftconv_form(1)): an independent cross-check of the tap / shift bookkeeping of the
// form above.  The KS taps of a filter COLUMN s share no window shift: the tile computes, per column tap s,
//     D_s[p, co] = sum_{r, ci} in[p + r*W, ci] * W[co, (r, s, ci)]
// and the epilogue finishes out[p, co] = sum_s D_s[p + shift(s), co] (shift(s) = s, or KS-1-s for the transposed
// conv), so the column shift is applied to the OUTPUT rows through a shared-memory accumulator instead of to the
// operand descriptor.  A tile of 128 window rows yields 128 - (KS-1) output rows.  Both consumer warpgroups work on
// the same tile (rows [64c, 64c + 64)); the column taps are accumulated in shift order 0, 1, .. into the fp32 tile,
// one 256-thread barrier per phase.
// ---------------------------------------------------------------------------------------------------------------
template <int COUT, int CBLK, int KS, int MODE, bool U8IN = false>
__global__ void __launch_bounds__(U8IN ? kScThreads + kU8Threads : kScThreads, 1)
    shiftconv_coltap_kernel(const __grid_constant__ CUtensorMap map_in, const __grid_constant__ CUtensorMap map_w,
                            const ShiftConvArgs g) {
  static_assert(!U8IN || CBLK == 1, "the uint8 window is one 64-channel block");
  constexpr int W_KB = COUT * 128;
  constexpr int ST = kScBM - (KS - 1);                    // output rows per tile
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  constexpr int num_kb = KS * KS * CBLK;
  const int win_bytes = (g.wrows * 128 + 1023) & ~1023;
  unsigned char* sW = smem;                               // [tap = r*KS + s][CBLK][COUT][128 B]
  unsigned char* sWin = smem + ((num_kb * W_KB + 1023) & ~1023);
  __shared__ __align__(8) unsigned long long full_bar[kScMaxStages], empty_bar[kScMaxStages], w_bar;
  __shared__ __align__(8) unsigned long long u8_full[kU8Stages], u8_empty[kU8Stages];
  const uint32_t nstages = (uint32_t)g.stages;
  unsigned char* sStage = sWin + nstages * CBLK * win_bytes;
  float* sAcc = reinterpret_cast<float*>(sStage + (U8IN ? kU8Stages * u8_stage_bytes(g.wrows) : 0));   // [128][COUT]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_in);
    tma_prefetch_desc(&map_w);
    for (int s = 0; s < kScMaxStages; ++s) {
      mbar_init(&full_bar[s], U8IN ? kU8Threads : 1);
      mbar_init(&empty_bar[s], 1);
    }
    for (int s = 0; s < kU8Stages; ++s) {
      mbar_init(&u8_full[s], 1);
      mbar_init(&u8_empty[s], kU8Threads);
    }
    mbar_init(&w_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 128) {
    mbar_arrive_expect_tx(&w_bar, (uint32_t)(num_kb * W_KB));
    for (int kb = 0; kb < num_kb; ++kb) tma_load_2d(sW + kb * W_KB, &map_w, kb * 64, 0, &w_bar);
  }
  pdl_wait();
  pdl_trigger();

  if (warp < 4) {
    // ===== TMA producer: one window per tile; tiles advance by ST rows =====
    if (warp == 0 && lane == 0) {
      uint32_t s = 0, par = 1;
      if (U8IN) {
        const int sbytes = u8_stage_bytes(g.wrows);
        for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
          mbar_wait(&u8_empty[s], par);
          mbar_arrive_expect_tx(&u8_full[s], (uint32_t)(g.wrows * 64));
          tma_load_2d(sStage + s * sbytes, &map_in, 0, tile * ST + g.row_shift, &u8_full[s]);
          if (++s == kU8Stages) s = 0, par ^= 1u;
        }
      } else {
        for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
          mbar_wait(&empty_bar[s], par);
          mbar_arrive_expect_tx(&full_bar[s], (uint32_t)(CBLK * g.wrows * 128));
#pragma unroll
          for (int cb = 0; cb < CBLK; ++cb)
            tma_load_2d(sWin + (s * CBLK + cb) * win_bytes, &map_in, cb * 64, tile * ST + g.row_shift, &full_bar[s]);
          if (++s == nstages) s = 0, par ^= 1u;
        }
      }
    }
    return;
  }
  if (U8IN && threadIdx.x >= kScThreads) {
    const int ct = threadIdx.x - kScThreads;
    const int sbytes = u8_stage_bytes(g.wrows);
    const float bias = -8388608.0f * g.in_scale;
    uint32_t s = 0, epar = 1, ss = 0, fpar = 0;
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      mbar_wait(&u8_full[ss], fpar);
      mbar_wait(&empty_bar[s], epar);
      u8_window_to_bf16_sw128(sStage + ss * sbytes, sWin + s * win_bytes, g.wrows, ct, g.in_scale, bias);
      fence_proxy_async_smem();
      mbar_arrive(&full_bar[s]);
      mbar_arrive(&u8_empty[ss]);
      if (++s == nstages) s = 0, epar ^= 1u;
      if (++ss == kU8Stages) ss = 0, fpar ^= 1u;
    }
    return;
  }
  // ===== consumers: warpgroup c owns rows [64c, 64c + 64) of every tile of this CTA =====
  const int c = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127;
  mbar_wait(&w_bar, 0);
  uint32_t row_off[KS];                                   // window shift of filter row r, 16-byte units
#pragma unroll
  for (int r = 0; r < KS; ++r) row_off[r] = (uint32_t)((g.flip ? KS - 1 - r : r) * g.W) * 8u;
  const uint32_t w_lo = gmma_lo(sW), win_lo0 = gmma_lo(sWin);
  const uint32_t win16 = (uint32_t)win_bytes >> 4;
  float bias_r[MODE == 0 ? COUT / 2 : 1];
  if (MODE == 0) {
#pragma unroll
    for (int i = 0; i < COUT / 2; ++i) bias_r[i] = __ldg(g.bias + gmma_col(t, i));
  }
  const bool relu = g.relu != 0;
  const bool has_mask = MODE == 1 && g.mask != nullptr;
  const int HW = g.H * g.W;
  uint32_t s = 0, full_par = 0;
  for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
    mbar_wait(&full_bar[s], full_par);
    const uint32_t a_lo = win_lo0 + s * (CBLK * win16) + (uint32_t)c * 512u;
#pragma unroll
    for (int sh = 0; sh < KS; ++sh) {
      const int sc = g.flip ? KS - 1 - sh : sh;          // the column tap whose output shift is sh
      float d[COUT / 2];
      wgmma_fence();
#pragma unroll
      for (int r = 0; r < KS; ++r)
#pragma unroll
        for (int cb = 0; cb < CBLK; ++cb)
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_bf16<COUT>(d, gmma_desc(kGmmaHiSw128, a_lo + cb * win16 + row_off[r] + 2u * k),
                             gmma_desc(kGmmaHiSw128, w_lo + (uint32_t)(((r * KS + sc) * CBLK + cb) * (W_KB >> 4) + 2 * k)),
                             (r | cb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      // both warpgroups: the previous phase's accumulation (or the previous tile's epilogue) is complete
      named_bar_sync(1, 256);
      if (sh == KS - 1 && threadIdx.x == 128) mbar_arrive(&empty_bar[s]);   // every MMA of this window has retired
#pragma unroll
      for (int i = 0; i < COUT / 2; i += 2) {
        const int p = 64 * c + gmma_row(t, i) - sh;       // output row this accumulator row contributes to
        if (p < 0) continue;
        float2* cell = reinterpret_cast<float2*>(sAcc + p * COUT + gmma_col(t, i));
        if (sh == 0) {
          *cell = make_float2(d[i], d[i + 1]);
        } else {
          const float2 o = *cell;
          *cell = make_float2(o.x + d[i], o.y + d[i + 1]);
        }
      }
    }
    if (++s == nstages) s = 0, full_par ^= 1u;
    named_bar_sync(1, 256);
#pragma unroll
    for (int i = 0; i < COUT / 2; i += 2) {
      const int p = 64 * c + gmma_row(t, i), col = gmma_col(t, i);
      const int q = tile * ST + p;
      if (p >= ST || q >= g.Q) continue;
      const float2 v = *reinterpret_cast<const float2*>(sAcc + p * COUT + col);
      const int n = q / HW;
      const int rem = q - n * HW;
      const int y = rem / g.W, x = rem - y * g.W;
      bool ok = y < g.Hout && x < g.Wout;
      size_t dst_off;
      if (g.out_mode == 0) {
        dst_off = ((size_t)(n * g.OGH + y) * g.OGW + x) * COUT + col;
      } else if (g.out_mode == 1) {
        const int yp = y + 2, xp = x + 2;
        dst_off = (((size_t)n * 12 + (yp >> 1)) * 12 + (xp >> 1)) * (4 * COUT) + (size_t)(((yp & 1) * 2 + (xp & 1)) * COUT) + col;
      } else {
        const int blk = col >> 5, py = 2 * y + (blk >> 1) - 2, px = 2 * x + (blk & 1) - 2;
        ok = py >= 0 && py < 20 && px >= 0 && px < 20;
        dst_off = (((size_t)n * 21 + py) * 21 + px) * 32 + (col & 31);
      }
      if (!ok) continue;
      uint32_t pk;
      if (MODE == 0) {
        const float v0 = v.x + bias_r[i], v1 = v.y + bias_r[i + 1];
        pk = relu ? s_pack_relu_bf16x2(v0, v1) : s_pack_bf16x2(v0, v1);
      } else {
        pk = s_pack_bf16x2(v.x, v.y);
        if (has_mask) {
          const uint32_t mw = __ldg(reinterpret_cast<const unsigned int*>(g.mask + (size_t)q * COUT + col));
          pk &= __hgt2_mask(*reinterpret_cast<const __nv_bfloat162*>(&mw), __floats2bfloat162_rn(0.f, 0.f));
        }
      }
      *reinterpret_cast<uint32_t*>(g.out + dst_off) = pk;
    }
  }
}

static int sc_make_map(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint32_t box_rows) {
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
  const cuuint32_t box[2] = {64, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS
             ? 0
             : -2;
}

static size_t u8_ring_bytes(int wrows) { return (size_t)kU8Stages * (size_t)((wrows * 64 + 1023) & ~1023); }

template <int COUT, int CBLK, int KS, int MODE, bool U8IN = false>
static void launch_shiftconv(const CUtensorMap& mi, const CUtensorMap& mw, const CUtensorMap& mm, const ShiftConvArgs& g,
                             int num_kb, int sms, cudaStream_t st) {
  const size_t win = (size_t)((g.wrows * 128 + 1023) & ~1023);
  const size_t tile = MODE == 1 ? (size_t)kScBM * COUT * 2 : 0;      // data gradient: mask / output tile per stage
  const size_t smem = (size_t)((num_kb * COUT * 128 + 1023) & ~1023) + (size_t)g.stages * (CBLK * win + tile) + 1024 +
                      (U8IN ? u8_ring_bytes(g.wrows) : 0);
  auto kern = shiftconv_fwd_kernel<COUT, CBLK, KS, MODE, U8IN>;
  RL_SMEM_OPTIN(kern);
  const int grid = g.num_tiles < sms ? g.num_tiles : sms;
  launch_chain(kern, dim3(grid), dim3(U8IN ? kScThreads + kU8Threads : kScThreads), smem, st, mi, mw, mm, g);
}

template <int COUT, int CBLK, int KS, int MODE, bool U8IN = false>
static void launch_coltap(const CUtensorMap& mi, const CUtensorMap& mw, const ShiftConvArgs& g, int num_kb, int sms,
                          cudaStream_t st) {
  const size_t win = (size_t)((g.wrows * 128 + 1023) & ~1023);
  const size_t smem = (size_t)((num_kb * COUT * 128 + 1023) & ~1023) + (size_t)g.stages * CBLK * win + 1024 +
                      (U8IN ? u8_ring_bytes(g.wrows) : 0) + (size_t)kScBM * COUT * sizeof(float);
  auto kern = shiftconv_coltap_kernel<COUT, CBLK, KS, MODE, U8IN>;
  RL_SMEM_OPTIN(kern);
  const int grid = g.num_tiles < sms ? g.num_tiles : sms;
  launch_chain(kern, dim3(grid), dim3(U8IN ? kScThreads + kU8Threads : kScThreads), smem, st, mi, mw, g);
}

}  // namespace rl

using namespace rl;

// Tile form of the window conv.  0 (default): one MMA chain per filter tap, the shift applied to the operand window
// (shiftconv_fwd_kernel); 1: per filter column, the column shift applied to the output rows (shiftconv_coltap_kernel),
// an independent cross-check of the tap / shift bookkeeping.
static int g_sc_form = 0;
extern "C" int rl_debug_set_shiftconv_form(int form) {
  RL_CHECK_ARG(form == 0 || form == 1, "shiftconv form must be 0 (per-tap) or 1 (column taps)");
  g_sc_form = form;
  return RL_OK;
}

// The descriptor base_offset field stays 0: the swizzle phase follows from the absolute shared-memory address of the
// shifted window row, so setting it would count the phase twice.  Asking for 1 is an error.
extern "C" int rl_debug_set_shiftconv_base_offset(int enable) {
  RL_CHECK_ARG(enable == 0, "shiftconv base_offset must be 0 (the swizzle phase comes from the shared-memory address)");
  return RL_OK;
}

static int shiftconv_launch(const void* in, const void* weight, const float* bias, void* out, int N, int H, int W,
                            int Cin, int Cout, int KH, int KW, int relu, int out_mode, int Hout, int Wout, int OGH, int OGW,
                            int transposed, const void* mask, rl_stream_t stream, const char* name, int u8in = 0,
                            float in_scale = 1.f) {
  RL_CHECK_ARG(in && weight && out && N > 0, "%s: bad argument", name);
  RL_CHECK_ARG(aligned16(in) && aligned16(weight) && aligned16(out) && (!mask || aligned16(mask)),
               "%s: 16-byte alignment required", name);
  RL_CHECK_ARG((Cout == 32 || Cout == 64 || Cout == 128) && (Cin == 64 || Cin == 128),
               "%s: Cin in {64,128}, Cout in {32,64,128}", name);
  RL_CHECK_ARG(KH == KW && (KH == 2 || KH == 3) && KH <= H && KW <= W, "%s: filter must be 2x2 or 3x3", name);
  ShiftConvArgs g;
  g.bias = bias, g.out = (__nv_bfloat16*)out, g.H = H, g.W = W, g.KH = KH, g.KW = KW;
  g.Hout = Hout, g.Wout = Wout, g.OGH = OGH, g.OGW = OGW;
  const long long Q = (long long)N * H * W;
  RL_CHECK_ARG(Q < (1LL << 31), "%s: too many positions", name);
  const int coltap = g_sc_form == 1;
  const int tile_rows = coltap ? kScBM - (KW - 1) : kScBM;            // output rows per 128-row tile
  g.Q = (int)Q, g.wrows = kScBM + (KH - 1) * W + (coltap ? 0 : KW - 1), g.relu = relu, g.out_mode = out_mode;
  g.row_shift = transposed ? -((KH - 1) * W + (KW - 1)) : 0, g.flip = transposed;
  g.mask = (const __nv_bfloat16*)mask, g.in_scale = in_scale;
  RL_CHECK_ARG(g.wrows <= 256, "%s: window of %d rows exceeds the TMA box limit", name, g.wrows);
  g.num_tiles = (int)((Q + tile_rows - 1) / tile_rows);
  const int cblk = Cin / 64, num_kb = KH * KW * cblk;
  const size_t win = (size_t)((g.wrows * 128 + 1023) & ~1023);
  {
    const size_t acc = coltap ? (size_t)kScBM * Cout * sizeof(float) : 0;    // column-tap form: fp32 output tile
    const size_t tile = transposed && !coltap ? (size_t)kScBM * Cout * 2 : 0;  // data gradient: mask / output tile
    const size_t budget = 220 * 1024 - ((size_t)num_kb * Cout * 128 + 2048) - (u8in ? u8_ring_bytes(g.wrows) : 0) - acc;
    long long st = (long long)(budget / ((size_t)cblk * win + tile));
    if (st > kScMaxStages) st = kScMaxStages;
    RL_CHECK_ARG(st >= 2, "%s: weights + windows do not fit in shared memory", name);
    g.stages = (int)st;
  }
  alignas(64) CUtensorMap mi, mw, mm;
  if ((u8in ? make_tensor_map_u8_rows64(&mi, in, (uint64_t)Q, (uint32_t)g.wrows)
            : sc_make_map(&mi, in, (uint64_t)Cin, (uint64_t)Q, (uint32_t)g.wrows)) ||
      sc_make_map(&mw, weight, (uint64_t)KH * KW * Cin, (uint64_t)Cout, (uint32_t)Cout) ||
      // the ReLU mask of a tile: its 128 accumulator rows of the saved activation [Q, Cout]
      (mask && !coltap && sc_make_map(&mm, mask, (uint64_t)Cout, (uint64_t)Q, (uint32_t)kScBM))) {
    set_error("%s: cuTensorMapEncodeTiled failed", name);
    return RL_ERR_CUDA;
  }
  if (!mask || coltap) mm = mi;                 // not read
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  sms = effective_sms(sms);
  cudaStream_t st = (cudaStream_t)stream;
  // instantiations: the layers of the Atari actor-critic and their data gradients (2x2 and 3x3 filters)
  const int key = (u8in ? 1000000 : 0) + (transposed ? 100000 : 0) + Cout * 100 + cblk * 10 + KH;
  if (coltap) {
    switch (key) {
      case 1003212: launch_coltap<32, 1, 2, 0, true>(mi, mw, g, num_kb, sms, st); break;
      case 3212: launch_coltap<32, 1, 2, 0>(mi, mw, g, num_kb, sms, st); break;
      case 6422: launch_coltap<64, 2, 2, 0>(mi, mw, g, num_kb, sms, st); break;
      case 6413: launch_coltap<64, 1, 3, 0>(mi, mw, g, num_kb, sms, st); break;
      case 6412: launch_coltap<64, 1, 2, 0>(mi, mw, g, num_kb, sms, st); break;
      case 6423: launch_coltap<64, 2, 3, 0>(mi, mw, g, num_kb, sms, st); break;
      case 106413: launch_coltap<64, 1, 3, 1>(mi, mw, g, num_kb, sms, st); break;
      case 112812: launch_coltap<128, 1, 2, 1>(mi, mw, g, num_kb, sms, st); break;
      case 106412: launch_coltap<64, 1, 2, 1>(mi, mw, g, num_kb, sms, st); break;
      case 112813: launch_coltap<128, 1, 3, 1>(mi, mw, g, num_kb, sms, st); break;
      default:
        set_error("%s: no instantiation for Cout=%d Cin=%d %dx%d", name, Cout, Cin, KH, KW);
        return RL_ERR_BAD_ARG;
    }
  } else
  switch (key) {
    case 1003212: launch_shiftconv<32, 1, 2, 0, true>(mi, mw, mm, g, num_kb, sms, st); break;  // conv1 fwd, uint8 input
    case 3212: launch_shiftconv<32, 1, 2, 0>(mi, mw, mm, g, num_kb, sms, st); break;          // conv1 fwd
    case 6422: launch_shiftconv<64, 2, 2, 0>(mi, mw, mm, g, num_kb, sms, st); break;          // conv2 fwd
    case 6413: launch_shiftconv<64, 1, 3, 0>(mi, mw, mm, g, num_kb, sms, st); break;          // conv3 fwd
    case 6412: launch_shiftconv<64, 1, 2, 0>(mi, mw, mm, g, num_kb, sms, st); break;
    case 6423: launch_shiftconv<64, 2, 3, 0>(mi, mw, mm, g, num_kb, sms, st); break;
    case 106413: launch_shiftconv<64, 1, 3, 1>(mi, mw, mm, g, num_kb, sms, st); break;        // conv3 dgrad
    case 112812: launch_shiftconv<128, 1, 2, 1>(mi, mw, mm, g, num_kb, sms, st); break;       // conv2 dgrad
    case 106412: launch_shiftconv<64, 1, 2, 1>(mi, mw, mm, g, num_kb, sms, st); break;
    case 112813: launch_shiftconv<128, 1, 3, 1>(mi, mw, mm, g, num_kb, sms, st); break;
    default:
      set_error("%s: no instantiation for Cout=%d Cin=%d %dx%d", name, Cout, Cin, KH, KW);
      return RL_ERR_BAD_ARG;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", name, cudaGetErrorString(e));
    return RL_ERR_CUDA;
  }
  return RL_OK;
}

extern "C" int rl_conv2d_s1_nhwc_bf16_fwd(const void* in, const void* weight_krsc, const float* bias, void* out, int N,
                                          int H, int W, int Cin, int Cout, int KH, int KW, int relu, int out_mode,
                                          rl_stream_t stream) {
  RL_CHECK_ARG(bias, "conv2d_s1: bias required");
  RL_CHECK_ARG(out_mode == 0 || (out_mode == 1 && H - KH + 1 == 20 && W - KW + 1 == 20),
               "conv2d_s1: out_mode 1 is the 20x20 -> [12,12,4*Cout] layout");
  return shiftconv_launch(in, weight_krsc, bias, out, N, H, W, Cin, Cout, KH, KW, relu, out_mode, H - KH + 1, W - KW + 1,
                          H - KH + 1, W - KW + 1, 0, nullptr, stream, "conv2d_s1");
}

extern "C" int rl_conv2d_s1_u8in_bf16_fwd(const void* in_u8, float in_scale, const void* weight_krsc, const float* bias,
                                          void* out, int N, int H, int W, int Cout, int KH, int KW, int relu,
                                          int out_mode, rl_stream_t stream) {
  RL_CHECK_ARG(bias, "conv2d_s1_u8in: bias required");
  RL_CHECK_ARG(Cout == 32 && KH == 2 && KW == 2, "conv2d_s1_u8in: built for the 2x2, 64 -> 32 layer (conv1, space-to-depth)");
  RL_CHECK_ARG(out_mode == 0 || (out_mode == 1 && H - KH + 1 == 20 && W - KW + 1 == 20),
               "conv2d_s1_u8in: out_mode 1 is the 20x20 -> [12,12,4*Cout] layout");
  return shiftconv_launch(in_u8, weight_krsc, bias, out, N, H, W, 64, Cout, KH, KW, relu, out_mode, H - KH + 1,
                          W - KW + 1, H - KH + 1, W - KW + 1, 0, nullptr, stream, "conv2d_s1_u8in", 1, in_scale);
}

extern "C" int rl_conv2d_s1_nhwc_bf16_dgrad(const void* dout_grid, const void* weight_t_krsc, const void* act_mask,
                                            void* din, int N, int H, int W, int Cout, int Cin, int KH, int KW,
                                            int out_mode, int OGH, int OGW, rl_stream_t stream) {
  RL_CHECK_ARG(out_mode == 0 || (out_mode == 2 && H == 12 && W == 12 && Cin == 128),
               "conv2d_s1_dgrad: out_mode 2 is the [12,12,128] -> [21,21,32] layout");
  // the data gradient of a stride-1 conv is the same shifted-GEMM sum run backwards: window starts
  // (KH-1)*W+(KW-1) rows earlier, taps flipped, weights transposed ([Cin, (r,s,co)]); every grid position is an output
  return shiftconv_launch(dout_grid, weight_t_krsc, nullptr, din, N, H, W, Cout, Cin, KH, KW, 0, out_mode, H, W,
                          out_mode == 0 ? OGH : 0, out_mode == 0 ? OGW : 0, 1, act_mask, stream, "conv2d_s1_dgrad");
}
