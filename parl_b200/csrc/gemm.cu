// K6 (dense contractions) — bf16 GEMM on the Hopper tensor cores: C[M,N] = act(A[M,K] · B[N,K]^T + bias)
// with fp32 accumulation in registers.  Used for the linear layers of the policy/value networks
// (a13: benchmark/torch/a2c/atari_model.py:46-49 fc 5184->512 and the heads; forward x·W^T).
//
// sm_90a structure (one 128 x BN output tile per CTA, BK = 64 bf16 = one 128-byte swizzle atom):
//   warp 0        : TMA producer — cp.async.bulk.tensor 2-D tiles of A and B (SWIZZLE_128B) into a
//                   4..8-stage shared-memory ring, completion on per-stage "full" mbarriers
//   warpgroups 1-2: consumers — warpgroup c issues wgmma.mma_async m64nBNk16 for rows [64c, 64c + 64) of the tile
//                   (4 per stage, one stage kept in flight), releases each stage on its "empty" mbarrier once the
//                   MMAs that read it have retired, then runs the epilogue (bias + optional ReLU / ReLU-backward
//                   mask, convert, store) straight from its accumulator registers
// Tensor-pipe bound: 2*M*N*K flops; operand traffic (M*K + N*K)*2 B + M*N*out B.
#include <cuda_bf16.h>

#include "common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace rl {

constexpr int kGemmBM = 128;
constexpr int kGemmBK = 64;          // bf16 elements per k-block = 128 bytes
// ring depth by tile width: the loop is bound by the L2/HBM latency of the TMA loads (bytes in flight per SM), so the
// ring takes what shared memory allows — 8 stages up to BN = 64, 6 at BN = 128, 4 at BN = 256 (~200 KB)
__host__ __device__ constexpr int gemm_stages(int bn) { return bn <= 64 ? 8 : (bn <= 128 ? 6 : 4); }
constexpr int kGemmThreads = 384;    // producer warpgroup (one active thread) + 2 consumer warpgroups

struct GemmArgs {
  const float* bias;   // [N] or NULL
  void* C;             // [M, ldc] bf16 or f32
  int M, N, K, ldc;
  int relu, out_f32;
  const __nv_bfloat16* mask;   // optional [M, ldm] saved post-ReLU activation: C *= (mask > 0)  (ReLU backward)
  int ldm;
  // split-K (few output tiles, long K — the actor's fc layer at small batch): blockIdx.z owns kb_per_split k-blocks
  // and dumps its raw fp32 accumulator tile to partial[z][row][col]; gemm_splitk_reduce_kernel finishes the epilogue
  float* partial;              // NULL: no split
  int kb_per_split, ldp, mpad;
};

__device__ __forceinline__ bool bf16_positive(__nv_bfloat16 h) { return __bfloat162float(h) > 0.f; }

template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap map_a,
                                                                      const __grid_constant__ CUtensorMap map_b,
                                                                      const GemmArgs g) {
  constexpr int A_STAGE = kGemmBM * kGemmBK * 2;     // 16 KB
  constexpr int B_STAGE = BN * kGemmBK * 2;
  constexpr int kGemmStages = gemm_stages(BN);
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  // SWIZZLE_128B atoms need 1024-byte alignment: align by hand (the launch reserves the slack)
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  unsigned char* sA = smem;                                     // [stages][128 rows][128 B]
  unsigned char* sB = smem + kGemmStages * A_STAGE;             // [stages][BN rows][128 B]
  __shared__ __align__(8) unsigned long long full_bar[kGemmStages], empty_bar[kGemmStages];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kGemmBM, n0 = blockIdx.y * BN;
  const int num_kb_all = (g.K + kGemmBK - 1) / kGemmBK;
  const int kb0 = g.partial ? (int)blockIdx.z * g.kb_per_split : 0;
  const int num_kb = g.partial ? min(g.kb_per_split, num_kb_all - kb0) : num_kb_all;     // this CTA's k-blocks

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < kGemmStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);          // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();            // chain kernel (launch_chain): A comes from the previous kernel of the stream
  pdl_trigger();

  if (warp < 4) {
    // ===== TMA producer =====
    if (warp == 0 && lane == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % kGemmStages;
        const uint32_t ph = (kb / kGemmStages) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1u);                                  // slot free (first pass: immediately)
        mbar_arrive_expect_tx(&full_bar[s], A_STAGE + B_STAGE);
        tma_load_2d(sA + s * A_STAGE, &map_a, (kb0 + kb) * kGemmBK, m0, &full_bar[s]);
        tma_load_2d(sB + s * B_STAGE, &map_b, (kb0 + kb) * kGemmBK, n0, &full_bar[s]);
      }
    }
    return;
  }
  // ===== consumers: warpgroup c owns rows [64c, 64c + 64) of the tile =====
  const int c = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127;
  float d[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  const uint32_t a_lo0 = gmma_lo(sA) + (uint32_t)(c * 64 * 128 >> 4), b_lo0 = gmma_lo(sB);
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % kGemmStages;
    mbar_wait(&full_bar[s], (kb / kGemmStages) & 1);                      // TMA bytes have landed
    wgmma_fence();
    const uint32_t a_lo = a_lo0 + (uint32_t)(s * (A_STAGE >> 4)), b_lo = b_lo0 + (uint32_t)(s * (B_STAGE >> 4));
#pragma unroll
    for (int k = 0; k < kGemmBK / 16; ++k)      // 16 bf16 = 32 bytes along K inside the swizzle atom: +2 units
      wgmma_bf16<BN>(d, gmma_desc(kGmmaHiSw128, a_lo + 2 * k), gmma_desc(kGmmaHiSw128, b_lo + 2 * k), (kb | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();                                                      // k-block kb-1 has retired: free its stage
    if (kb > 0 && t == 0) mbar_arrive(&empty_bar[(kb - 1) % kGemmStages]);
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  const int rbase = m0 + 64 * c;
  if (g.partial) {
    // raw accumulator dump (padded tile grid: no bounds), finished by gemm_splitk_reduce_kernel
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int row = rbase + gmma_row(t, i), col = n0 + gmma_col(t, i);
      *reinterpret_cast<float2*>(g.partial + ((size_t)blockIdx.z * g.mpad + row) * g.ldp + col) = make_float2(d[i], d[i + 1]);
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const int row = rbase + gmma_row(t, i), col = n0 + gmma_col(t, i);
    if (row >= g.M || col >= g.N) continue;
    const bool two = col + 1 < g.N;
    float v0 = d[i] + (g.bias ? g.bias[col] : 0.f), v1 = d[i + 1] + ((g.bias && two) ? g.bias[col + 1] : 0.f);
    if (g.relu) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
    if (g.mask) {
      const __nv_bfloat16* mrow = g.mask + (size_t)row * g.ldm + col;
      if (!bf16_positive(mrow[0])) v0 = 0.f;
      if (two && !bf16_positive(mrow[1])) v1 = 0.f;
    }
    if (g.out_f32) {
      float* dst = reinterpret_cast<float*>(g.C) + (size_t)row * g.ldc + col;
      if (two && (g.ldc & 1) == 0) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
      else {
        dst[0] = v0;
        if (two) dst[1] = v1;
      }
    } else {
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(g.C) + (size_t)row * g.ldc + col;
      if (two && (g.ldc & 1) == 0) *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
      else {
        dst[0] = __float2bfloat16(v0);
        if (two) dst[1] = __float2bfloat16(v1);
      }
    }
  }
}

// C[row, col] = act(sum_z partial[z][row][col] + bias[col]) in split order (deterministic)
__global__ void __launch_bounds__(256) gemm_splitk_reduce_kernel(const float* __restrict__ partial, int splits, int mpad,
                                                                 int ldp, const GemmArgs g) {
  pdl_wait();            // chain kernel (launch_chain)
  pdl_trigger();
  const int n4 = (g.N + 3) >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)g.M * n4) return;
  const int row = (int)(idx / n4), col = (int)(idx - (long long)row * n4) * 4;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int z = 0; z < splits; ++z) {
    const float4 p = *reinterpret_cast<const float4*>(partial + ((size_t)z * mpad + row) * ldp + col);
    a.x += p.x, a.y += p.y, a.z += p.z, a.w += p.w;
  }
  float v[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (col + i >= g.N) break;
    float x = v[i] + (g.bias ? g.bias[col + i] : 0.f);
    x = g.relu ? fmaxf(x, 0.f) : x;
    if (g.out_f32) reinterpret_cast<float*>(g.C)[(size_t)row * g.ldc + col + i] = x;
    else reinterpret_cast<__nv_bfloat16*>(g.C)[(size_t)row * g.ldc + col + i] = __float2bfloat16(x);
  }
}

// Hidden layer + small heads of the actor step in one pass (examples/IMPALA/atari_model.py policy head after the fc
// layer): a warp owns one row.  H[row, :] = relu(sum_z partial[z][row][:] + bias) (split-K reduce; or, with
// partial == NULL, H is read as written by the GEMM epilogue), rounded to bf16 and stored; then
// out2[row, n] = b2[n] + sum_c bf16(H[row, c]) * W2[n, c] for the N2 <= 32 head rows — fp32, fixed order (16-column
// lane partials, xor-shuffle tree), so the per-step chain has one launch instead of reduce + a tensor-core GEMM that
// is all prologue at N2 = 18.
struct HeadsArgs {
  const __nv_bfloat16* W2;   // [N2, N] bf16
  const float* b2;           // [N2] or NULL
  float* out2;               // [M, ldo2]
  int N2, ldo2;
};
constexpr int kHeadsMaxN = 1024, kHeadsMaxN2 = 32;

__global__ void __launch_bounds__(256) fc_reduce_heads_kernel(const float* __restrict__ partial, int splits, int mpad, int ldp,
                                                              const float* __restrict__ bias, __nv_bfloat16* __restrict__ H,
                                                              int ldh, int M, int N, int relu, const HeadsArgs hd) {
  extern __shared__ __align__(16) unsigned char heads_smem[];
  __nv_bfloat16* sW = reinterpret_cast<__nv_bfloat16*>(heads_smem);          // [N2][N]
  for (int i = threadIdx.x; i < hd.N2 * N / 8; i += blockDim.x)            // head weights: written by the operand refresh
    reinterpret_cast<uint4*>(sW)[i] = __ldg(reinterpret_cast<const uint4*>(hd.W2) + i);
  pdl_wait();            // chain kernel (launch_chain)
  pdl_trigger();
  __syncthreads();
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int nchunk = N >> 7;                                               // 128 columns per pass: 4 per lane
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < M; row += gridDim.x * wpb) {
    float acc[kHeadsMaxN2];
#pragma unroll
    for (int n = 0; n < kHeadsMaxN2; ++n) acc[n] = 0.f;
    for (int j = 0; j < nchunk; ++j) {
      const int col = j * 128 + lane * 4;
      float hv[4];
      if (partial) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int z = 0; z < splits; ++z) {
          const float4 p = *reinterpret_cast<const float4*>(partial + ((size_t)z * mpad + row) * ldp + col);
          a.x += p.x, a.y += p.y, a.z += p.z, a.w += p.w;
        }
        const float4 b4 = bias ? *reinterpret_cast<const float4*>(bias + col) : make_float4(0.f, 0.f, 0.f, 0.f);
        hv[0] = a.x + b4.x, hv[1] = a.y + b4.y, hv[2] = a.z + b4.z, hv[3] = a.w + b4.w;
        if (relu) {
#pragma unroll
          for (int i = 0; i < 4; ++i) hv[i] = fmaxf(hv[i], 0.f);
        }
        __nv_bfloat162 lo = __floats2bfloat162_rn(hv[0], hv[1]), hi = __floats2bfloat162_rn(hv[2], hv[3]);
        *reinterpret_cast<uint2*>(H + (size_t)row * ldh + col) =
            make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
        hv[0] = __low2float(lo), hv[1] = __high2float(lo), hv[2] = __low2float(hi), hv[3] = __high2float(hi);
      } else {
        const uint2 u = *reinterpret_cast<const uint2*>(H + (size_t)row * ldh + col);
        const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&u.x), hi = *reinterpret_cast<const __nv_bfloat162*>(&u.y);
        hv[0] = __low2float(lo), hv[1] = __high2float(lo), hv[2] = __low2float(hi), hv[3] = __high2float(hi);
      }
#pragma unroll
      for (int n = 0; n < kHeadsMaxN2; ++n) {
        if (n < hd.N2) {
          const uint2 w = *reinterpret_cast<const uint2*>(sW + (size_t)n * N + col);
          const __nv_bfloat162 wl = *reinterpret_cast<const __nv_bfloat162*>(&w.x), wh = *reinterpret_cast<const __nv_bfloat162*>(&w.y);
          acc[n] = fmaf(hv[0], __low2float(wl), acc[n]);
          acc[n] = fmaf(hv[1], __high2float(wl), acc[n]);
          acc[n] = fmaf(hv[2], __low2float(wh), acc[n]);
          acc[n] = fmaf(hv[3], __high2float(wh), acc[n]);
        }
      }
    }
#pragma unroll
    for (int n = 0; n < kHeadsMaxN2; ++n) {
      if (n < hd.N2) {
        float v = acc[n];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) hd.out2[(size_t)row * hd.ldo2 + n] = v + (hd.b2 ? hd.b2[n] : 0.f);
      }
    }
  }
}

// The head alone, when H already exists (after the GEMM epilogue or the plain split-K reduce): out2 = H . W2^T + b2 with
// warp-level mma.sync.m16n8k16 (bf16 x bf16 -> f32).  N2 <= 24 columns are a sliver of a wgmma tile — that kernel
// would spend its time on barrier setup and the TMA ring for 8 k-blocks — while here a 16-row tile is
// four warps, each reducing a quarter of K straight from global memory (fragments are 4-byte loads in the operands'
// native row-major layouts), then one shared-memory pass adds the four partial tiles in a fixed order.
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                               uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

constexpr int kHeadsMmaNT = 3;       // n-tiles of 8 head rows: N2 <= 24

__global__ void __launch_bounds__(128) heads_mma_kernel(const __nv_bfloat16* __restrict__ H, int ldh, int M, int N,
                                                        const HeadsArgs hd) {
  __shared__ float red[4][16][kHeadsMmaNT * 8];
  pdl_wait();            // chain kernel (launch_chain)
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tig = lane & 3;
  const int row0 = blockIdx.x * 16;
  const int kper = N >> 2, kb = warp * kper;                       // this warp's quarter of the reduction
  const __nv_bfloat16* h0 = H + (size_t)min(row0 + g, M - 1) * ldh + tig * 2;
  const __nv_bfloat16* h1 = H + (size_t)min(row0 + g + 8, M - 1) * ldh + tig * 2;
  const __nv_bfloat16* wr[kHeadsMmaNT];
  bool wok[kHeadsMmaNT];
#pragma unroll
  for (int nt = 0; nt < kHeadsMmaNT; ++nt) {
    wok[nt] = nt * 8 + g < hd.N2;
    wr[nt] = hd.W2 + (size_t)min(nt * 8 + g, hd.N2 - 1) * N + tig * 2;
  }
  float c[kHeadsMmaNT][4];
#pragma unroll
  for (int nt = 0; nt < kHeadsMmaNT; ++nt) c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;
#pragma unroll 4
  for (int k0 = kb; k0 < kb + kper; k0 += 16) {
    const uint32_t a0 = *reinterpret_cast<const uint32_t*>(h0 + k0), a1 = *reinterpret_cast<const uint32_t*>(h1 + k0);
    const uint32_t a2 = *reinterpret_cast<const uint32_t*>(h0 + k0 + 8), a3 = *reinterpret_cast<const uint32_t*>(h1 + k0 + 8);
#pragma unroll
    for (int nt = 0; nt < kHeadsMmaNT; ++nt) {
      uint32_t b0 = __ldg(reinterpret_cast<const uint32_t*>(wr[nt] + k0)), b1 = __ldg(reinterpret_cast<const uint32_t*>(wr[nt] + k0 + 8));
      if (!wok[nt]) b0 = b1 = 0u;
      mma_bf16_16816(c[nt], a0, a1, a2, a3, b0, b1);
    }
  }
#pragma unroll
  for (int nt = 0; nt < kHeadsMmaNT; ++nt) {
    red[warp][g][nt * 8 + tig * 2] = c[nt][0], red[warp][g][nt * 8 + tig * 2 + 1] = c[nt][1];
    red[warp][g + 8][nt * 8 + tig * 2] = c[nt][2], red[warp][g + 8][nt * 8 + tig * 2 + 1] = c[nt][3];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 16 * kHeadsMmaNT * 8; i += 128) {
    const int r = i / (kHeadsMmaNT * 8), n = i - r * (kHeadsMmaNT * 8), row = row0 + r;
    if (row < M && n < hd.N2)
      hd.out2[(size_t)row * hd.ldo2 + n] = ((red[0][r][n] + red[1][r][n]) + (red[2][r][n] + red[3][r][n])) + (hd.b2 ? hd.b2[n] : 0.f);
  }
}

// rank-2 bf16 tensor map {K (contiguous), rows}, box {64, box_rows}, SWIZZLE_128B
static int make_tensor_map_bf16_sw128(CUtensorMap* map, const void* base, uint64_t K, uint64_t rows, uint64_t pitch_bytes,
                                      uint32_t box_rows) {
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
  const cuuint64_t gdim[2] = {K, rows};
  const cuuint64_t gstride[1] = {pitch_bytes};
  const cuuint32_t box[2] = {(cuuint32_t)kGemmBK, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS
             ? 0
             : -2;
}

template <int BN>
static int launch_gemm(const CUtensorMap& ma, const CUtensorMap& mb, const GemmArgs& g, int splits, cudaStream_t st) {
  const size_t smem = (size_t)gemm_stages(BN) * (kGemmBM * kGemmBK * 2 + BN * kGemmBK * 2) + 1024;
  RL_SMEM_OPTIN(gemm_bf16_tn_kernel<BN>);
  dim3 grid((g.M + kGemmBM - 1) / kGemmBM, (g.N + BN - 1) / BN, splits);
  launch_chain(gemm_bf16_tn_kernel<BN>, grid, dim3(kGemmThreads), smem, st, ma, mb, g);
  return 0;
}

}  // namespace rl

using namespace rl;

static int gemm_launch(const void* A, const void* B, const float* bias, void* C, int M, int N, int K, int lda, int ldb,
                       int ldc, int relu, int out_f32, const void* mask, int ldm, void* workspace, size_t workspace_bytes,
                       rl_stream_t stream, const HeadsArgs* heads = nullptr);

// The 2 x 2 cluster + TMA multicast form of the B200 build is not part of the sm_90a kernels; 0 is the only setting.
extern "C" int rl_debug_set_gemm_cluster(int enable) {
  RL_CHECK_ARG(enable == 0, "gemm cluster form: not built for sm_90a (only 0 is accepted)");
  return RL_OK;
}
static int g_heads_mma = 1;      // 1: mma.sync head kernel after the plain reduce; 0: warp-per-row CUDA-core kernel(s)

extern "C" int rl_gemm_bf16_tn(const void* A, const void* B, const float* bias, void* C, int M, int N, int K, int lda,
                               int ldb, int ldc, int relu, int out_f32, rl_stream_t stream) {
  return gemm_launch(A, B, bias, C, M, N, K, lda, ldb, ldc, relu, out_f32, nullptr, 0, nullptr, 0, stream);
}

extern "C" int rl_gemm_bf16_tn_splitk(const void* A, const void* B, const float* bias, void* C, int M, int N, int K,
                                      int lda, int ldb, int ldc, int relu, int out_f32, void* workspace,
                                      size_t workspace_bytes, rl_stream_t stream) {
  RL_CHECK_ARG(!workspace || aligned16(workspace), "gemm_bf16_tn_splitk: workspace must be 16-byte aligned");
  return gemm_launch(A, B, bias, C, M, N, K, lda, ldb, ldc, relu, out_f32, nullptr, 0, workspace, workspace_bytes, stream);
}

extern "C" int rl_debug_set_heads_mma(int enable) {
  g_heads_mma = enable ? 1 : 0;
  return RL_OK;
}

extern "C" int rl_gemm_bf16_tn_heads(const void* A, const void* B, const float* bias, void* H, int M, int N, int K, int lda,
                                     int ldb, int ldh, int relu, const void* W2, const float* b2, int N2, float* out2,
                                     int ldo2, void* workspace, size_t workspace_bytes, rl_stream_t stream) {
  RL_CHECK_ARG(W2 && out2 && N2 >= 1 && N2 <= kHeadsMaxN2 && ldo2 >= N2, "gemm_bf16_tn_heads: 1 <= N2 <= 32 heads required");
  RL_CHECK_ARG(N % 128 == 0 && N <= kHeadsMaxN && ldh % 4 == 0 && (size_t)N2 * N * 2 <= 48 * 1024 && aligned16(W2) &&
                   (!bias || aligned16(bias)),
               "gemm_bf16_tn_heads: N must be a multiple of 128 (<= 1024), N2*N*2 <= 48 KB, ldh % 4 == 0");
  RL_CHECK_ARG(!workspace || aligned16(workspace), "gemm_bf16_tn_heads: workspace must be 16-byte aligned");
  HeadsArgs hd;
  hd.W2 = (const __nv_bfloat16*)W2, hd.b2 = b2, hd.out2 = out2, hd.N2 = N2, hd.ldo2 = ldo2;
  return gemm_launch(A, B, bias, H, M, N, K, lda, ldb, ldh, relu, 0, nullptr, 0, workspace, workspace_bytes, stream, &hd);
}

extern "C" int rl_gemm_bf16_tn_masked(const void* A, const void* B, void* C, const void* mask, int M, int N, int K,
                                      int lda, int ldb, int ldc, int ldm, int out_f32, rl_stream_t stream) {
  RL_CHECK_ARG(mask && ldm >= N, "gemm_bf16_tn_masked: mask required, ldm >= N");
  return gemm_launch(A, B, nullptr, C, M, N, K, lda, ldb, ldc, 0, out_f32, mask, ldm, nullptr, 0, stream);
}

static int device_sms() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return effective_sms(sms);
}

static int launch_heads(const float* partial, int splits, int mpad, int ldp, const float* bias, void* H, int ldh, int M,
                        int N, int relu, const HeadsArgs& hd, cudaStream_t st) {
  if (!partial && g_heads_mma && hd.N2 <= 8 * kHeadsMmaNT && N % 64 == 0 && ldh % 2 == 0)
    return launch_chain(heads_mma_kernel, dim3((unsigned)((M + 15) / 16)), dim3(128), 0, st, (const __nv_bfloat16*)H, ldh, M, N,
                        hd) == cudaSuccess
               ? 0
               : -1;
  const size_t smem = (size_t)hd.N2 * N * 2;
  int blocks = (M + 7) / 8;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  return launch_chain(fc_reduce_heads_kernel, dim3((unsigned)blocks), dim3(256), smem, st, partial, splits, mpad, ldp, bias,
                      (__nv_bfloat16*)H, ldh, M, N, relu, hd) == cudaSuccess
             ? 0
             : -1;
}

static int gemm_launch(const void* A, const void* B, const float* bias, void* C, int M, int N, int K, int lda, int ldb,
                       int ldc, int relu, int out_f32, const void* mask, int ldm, void* workspace, size_t workspace_bytes,
                       rl_stream_t stream, const HeadsArgs* heads) {
  RL_CHECK_ARG(A && B && C && M > 0 && N > 0 && K > 0, "gemm_bf16_tn: bad argument");
  RL_CHECK_ARG(aligned16(A) && aligned16(B) && aligned16(C), "gemm_bf16_tn: pointers must be 16-byte aligned");
  RL_CHECK_ARG(lda >= K && ldb >= K && ldc >= N && (lda % 8) == 0 && (ldb % 8) == 0,
               "gemm_bf16_tn: lda/ldb must be >= K and multiples of 8 elements (TMA row pitch)");
  int BN = N > 128 ? 256 : (N > 64 ? 128 : (N > 32 ? 64 : 32));
  // small problems: prefer narrower tiles until the grid covers about two thirds of the SMs, but keep N >= 64 so
  // that each wgmma instruction still carries enough tensor-core work per shared-memory operand read
  const int sms = device_sms();
  const long long mt = (M + kGemmBM - 1) / kGemmBM;
  while (BN > 64 && mt * ((N + BN - 1) / BN) < (2 * sms) / 3) BN >>= 1;
  alignas(64) CUtensorMap ma, mb;
  if (make_tensor_map_bf16_sw128(&ma, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, kGemmBM) ||
      make_tensor_map_bf16_sw128(&mb, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, (uint32_t)BN)) {
    set_error("gemm_bf16_tn: cuTensorMapEncodeTiled failed");
    return RL_ERR_CUDA;
  }
  GemmArgs g;
  g.bias = bias, g.C = C, g.M = M, g.N = N, g.K = K, g.ldc = ldc, g.relu = relu, g.out_f32 = out_f32;
  g.mask = (const __nv_bfloat16*)mask, g.ldm = ldm;
  g.partial = nullptr, g.kb_per_split = 0, g.ldp = 0, g.mpad = 0;
  // split-K: fewer output tiles than half the SMs and a long reduction (one CTA would walk >= 16 k-blocks alone)
  const int nt = (N + BN - 1) / BN, num_kb = (K + kGemmBK - 1) / kGemmBK;
  int splits = 1;
  if (workspace && !mask && mt * nt * 2 <= sms && num_kb >= 16) {
    int want = (int)(sms / (mt * nt));
    if (want > num_kb / 8) want = num_kb / 8;
    if (want > 8) want = 8;
    const int per = (num_kb + want - 1) / want;
    want = (num_kb + per - 1) / per;                                  // no empty split
    const size_t need = (size_t)want * (size_t)(mt * kGemmBM) * (size_t)(nt * BN) * sizeof(float);
    if (want > 1 && need <= workspace_bytes) {
      splits = want;
      g.partial = reinterpret_cast<float*>(workspace), g.kb_per_split = per, g.ldp = nt * BN, g.mpad = (int)mt * kGemmBM;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  switch (BN) {
    case 256: launch_gemm<256>(ma, mb, g, splits, st); break;
    case 128: launch_gemm<128>(ma, mb, g, splits, st); break;
    case 64: launch_gemm<64>(ma, mb, g, splits, st); break;
    default: launch_gemm<32>(ma, mb, g, splits, st); break;
  }
  if (splits > 1) {
    if (heads && !(g_heads_mma && heads->N2 <= 8 * kHeadsMmaNT && N % 64 == 0)) {
      // split-K reduce, bias, ReLU, bf16 H and the heads in ONE warp-per-row kernel
      if (launch_heads(g.partial, splits, g.mpad, g.ldp, bias, C, ldc, M, N, relu, *heads, st)) {
        set_error("gemm_bf16_tn_heads: heads launch failed");
        return RL_ERR_CUDA;
      }
      RL_CHECK_LAUNCH("rl_gemm_bf16_tn_heads");
      return RL_OK;
    }
    const long long items = (long long)M * ((N + 3) / 4);
    launch_chain(gemm_splitk_reduce_kernel, dim3((unsigned)((items + 255) / 256)), dim3(256), 0, st,
                 (const float*)g.partial, splits, g.mpad, g.ldp, g);
  }
  RL_CHECK_LAUNCH("rl_gemm_bf16_tn");
  if (heads && launch_heads(nullptr, 0, 0, 0, nullptr, C, ldc, M, N, 0, *heads, st)) {
    set_error("gemm_bf16_tn_heads: heads launch failed");
    return RL_ERR_CUDA;
  }
  return RL_OK;
}
