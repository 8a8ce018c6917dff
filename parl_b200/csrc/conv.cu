// K6 (convolutions) — NHWC bf16 convolution forward as an implicit GEMM on the Hopper tensor cores:
//   out[n,oh,ow,:] = relu( sum_{r,s,c} in[n, oh*stride-pad+r, ow*stride-pad+s, c] * W[:, (r,s,c)] + bias )
// for the three conv layers of the Atari actor-critic (a13: benchmark/torch/a2c/atari_model.py:26-44; conv1
// in its space-to-depth form, see rl_obs_stack_gather out_dtype 3).  GEMM view: M = N*Hout*Wout output
// pixels, N = Cout (32 / 64), K = KH*KW*Cin ordered (r, s, c) so that one 128-byte k-block is 1 or 2 filter taps.
//
// sm_90a structure (persistent CTAs, one per SM, tiles of 128 output pixels):
//   warps 0-3      : producers — thread i gathers row i of the 128 x 64 A k-block straight from the NHWC input with
//                    16-byte cp.async (zero-fill outside the image), writing the SWIZZLE_128B K-major layout by hand;
//                    a kStages-deep ring, completion published per stage through "full" mbarriers
//   warpgroups 1-2 : weights [Cout, K] stay RESIDENT in shared memory (one TMA load per CTA); warpgroup c issues
//                    wgmma m64nCout for rows [64c, 64c + 64) of each tile, then bias + ReLU, bf16, NHWC store
//                    straight from its accumulator registers
#include <cuda_bf16.h>

#include "common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace rl {

__device__ __forceinline__ void cp_async16_zfill(uint32_t smem_dst, const void* gsrc, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes) : "memory");
}

constexpr int kCvBM = 128;
constexpr int kCvStages = 6;
constexpr int kCvLag = 3;            // cp.async groups in flight per producer thread before publishing a stage
constexpr int kCvThreads = 384;      // 4 producer warps + 2 consumer warpgroups

struct ConvArgs {
  const __nv_bfloat16* in;   // [N, Hin, Win, Cin]
  const float* bias;         // [Cout]
  __nv_bfloat16* out;        // [N, Hout, Wout, Cout]
  int N, Hin, Win, Cin, KH, KW, stride, pad, Hout, Wout;
  int M, num_kb, num_tiles, relu;
};

template <int COUT, int CIN>
__global__ void __launch_bounds__(kCvThreads, 1) conv_igemm_fwd_kernel(const __grid_constant__ CUtensorMap map_w,
                                                                       const ConvArgs g) {
  constexpr int A_STAGE = kCvBM * 128;          // 16 KB: 128 rows x 64 bf16
  constexpr int W_KB = COUT * 128;              // bytes of one weight k-block
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  unsigned char* sW = smem;                                    // [num_kb][COUT][128 B]
  unsigned char* sA = smem + ((g.num_kb * W_KB + 1023) & ~1023);   // [stages][128][128 B]
  __shared__ __align__(8) unsigned long long full_bar[kCvStages], empty_bar[kCvStages], w_bar;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_w);
    for (int s = 0; s < kCvStages; ++s) {
      mbar_init(&full_bar[s], 128);              // every producer thread arrives
      mbar_init(&empty_bar[s], 2);               // one arrival per consumer warpgroup
    }
    mbar_init(&w_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int HWo = g.Hout * g.Wout;

  if (threadIdx.x < 128) {
    // ===================== producers: implicit-GEMM gather of the A operand =====================
    const int row = threadIdx.x;                                   // 0..127
    const uint32_t row_smem = (uint32_t)row * 128u;
    const uint32_t sw = (uint32_t)(row & 7);
    uint32_t it = 0;                                               // global k-block counter (ring position)
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      const int m = tile * kCvBM + row;
      const bool mok = m < g.M;
      int n = 0, oh = 0, ow = 0;
      if (mok) {
        n = m / HWo;
        const int rem = m - n * HWo;
        oh = rem / g.Wout;
        ow = rem - oh * g.Wout;
      }
      const int ih0 = oh * g.stride - g.pad, iw0 = ow * g.stride - g.pad;
      const __nv_bfloat16* in_n = g.in + (size_t)n * g.Hin * g.Win * g.Cin;
      for (int kb = 0; kb < g.num_kb; ++kb, ++it) {
        const uint32_t s = it % kCvStages;
        const uint32_t ph = (it / kCvStages) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        const uint32_t stage_base = smem_u32(sA + s * A_STAGE) + row_smem;
        // one k-block = 64 K-elements = 64/CIN filter taps of CIN channels each (K ordered (r, s, c))
        constexpr int TAPS = 64 / CIN, CPT = CIN / 8;              // taps per k-block, 16-byte chunks per tap
#pragma unroll
        for (int tt = 0; tt < TAPS; ++tt) {
          const int tap = kb * TAPS + tt;
          const int r = tap / g.KW;
          const int sx = tap - r * g.KW;
          const int ih = ih0 + r, iw = iw0 + sx;
          const bool ok = mok && ih >= 0 && ih < g.Hin && iw >= 0 && iw < g.Win;
          const __nv_bfloat16* src = ok ? in_n + ((size_t)ih * g.Win + iw) * CIN : g.in;
#pragma unroll
          for (int cc = 0; cc < CPT; ++cc) {
            const uint32_t j = (uint32_t)(tt * CPT + cc);
            cp_async16_zfill(stage_base + ((j ^ sw) << 4), src + (ok ? cc * 8 : 0), ok ? 16u : 0u);
          }
        }
        cp_async_commit();
        if (it >= kCvLag) {
          cp_async_wait<kCvLag>();                                 // k-block (it - kCvLag) has landed
          fence_proxy_async_smem();                                // make it visible to the tensor-core proxy
          mbar_arrive(&full_bar[(it - kCvLag) % kCvStages]);
        }
      }
    }
    // drain: publish the last kCvLag k-blocks
    cp_async_wait<0>();
    fence_proxy_async_smem();
    for (uint32_t d = (it >= (uint32_t)kCvLag ? it - kCvLag : 0u); d < it; ++d) mbar_arrive(&full_bar[d % kCvStages]);
    return;
  }
  // ===================== consumers: weights (once), wgmma, epilogue =====================
  const int c = (threadIdx.x >> 7) - 1, t = threadIdx.x & 127;
  if (threadIdx.x == 128) {
    mbar_arrive_expect_tx(&w_bar, (uint32_t)(g.num_kb * W_KB));
    for (int kb = 0; kb < g.num_kb; ++kb) tma_load_2d(sW + kb * W_KB, &map_w, kb * 64, 0, &w_bar);
  }
  mbar_wait(&w_bar, 0);
  const uint32_t a_lo0 = gmma_lo(sA) + (uint32_t)(c * 64 * 128 >> 4), w_lo0 = gmma_lo(sW);
  float bias_r[COUT / 2];                      // bias of the column of each accumulator element
#pragma unroll
  for (int i = 0; i < COUT / 2; ++i) bias_r[i] = __ldg(g.bias + gmma_col(t, i));
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
    float d[COUT / 2];
#pragma unroll
    for (int i = 0; i < COUT / 2; ++i) d[i] = 0.f;
    for (int kb = 0; kb < g.num_kb; ++kb, ++it) {
      const uint32_t s = it % kCvStages;
      mbar_wait(&full_bar[s], (it / kCvStages) & 1u);
      wgmma_fence();
      const uint32_t a_lo = a_lo0 + s * (uint32_t)(A_STAGE >> 4), w_lo = w_lo0 + (uint32_t)(kb * (W_KB >> 4));
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_bf16<COUT>(d, gmma_desc(kGmmaHiSw128, a_lo + 2 * k), gmma_desc(kGmmaHiSw128, w_lo + 2 * k), (kb | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if (t == 0) mbar_arrive(&empty_bar[s]);
    }
    wgmma_fence_regs(d);
#pragma unroll
    for (int i = 0; i < COUT / 2; i += 2) {
      const int m = tile * kCvBM + 64 * c + gmma_row(t, i), col = gmma_col(t, i);
      if (m < g.M) {
        float x0 = d[i] + bias_r[i], x1 = d[i + 1] + bias_r[i + 1];
        if (g.relu) x0 = fmaxf(x0, 0.f), x1 = fmaxf(x1, 0.f);
        *reinterpret_cast<__nv_bfloat162*>(g.out + (size_t)m * COUT + col) = __floats2bfloat162_rn(x0, x1);
      }
    }
  }
}

static int make_weight_map(CUtensorMap* map, const void* w, int K, int Cout) {
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
  const cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)Cout};
  const cuuint64_t gstride[1] = {(cuuint64_t)K * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)Cout};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), gdim, gstride, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS
             ? 0
             : -2;
}

template <int COUT, int CIN>
static void launch_conv(const CUtensorMap& mw, const ConvArgs& g, int sms, cudaStream_t st) {
  const size_t smem = (size_t)((g.num_kb * COUT * 128 + 1023) & ~1023) + (size_t)kCvStages * kCvBM * 128 + 1024;
  RL_SMEM_OPTIN(conv_igemm_fwd_kernel<COUT, CIN>);
  const int grid = g.num_tiles < sms ? g.num_tiles : sms;
  conv_igemm_fwd_kernel<COUT, CIN><<<grid, kCvThreads, smem, st>>>(mw, g);
}

}  // namespace rl

using namespace rl;

extern "C" int rl_conv2d_nhwc_bf16_fwd(const void* in, const void* weight_krsc, const float* bias, void* out, int N,
                                       int Hin, int Win, int Cin, int Cout, int KH, int KW, int stride, int pad,
                                       int relu, rl_stream_t stream) {
  RL_CHECK_ARG(in && weight_krsc && bias && out && N > 0, "conv2d_nhwc_bf16_fwd: bad argument");
  RL_CHECK_ARG(aligned16(in) && aligned16(weight_krsc) && aligned16(out), "conv2d_nhwc_bf16_fwd: 16-byte alignment required");
  RL_CHECK_ARG(Cout == 32 || Cout == 64, "conv2d_nhwc_bf16_fwd: Cout must be 32 or 64 (got %d)", Cout);
  RL_CHECK_ARG(Cin == 32 || Cin == 64, "conv2d_nhwc_bf16_fwd: Cin must be 32 or 64 (got %d)", Cin);
  const int K = KH * KW * Cin;
  RL_CHECK_ARG(K % 64 == 0, "conv2d_nhwc_bf16_fwd: KH*KW*Cin = %d must be a multiple of 64", K);
  ConvArgs g;
  g.in = (const __nv_bfloat16*)in, g.bias = bias, g.out = (__nv_bfloat16*)out;
  g.N = N, g.Hin = Hin, g.Win = Win, g.Cin = Cin, g.KH = KH, g.KW = KW, g.stride = stride, g.pad = pad;
  g.Hout = (Hin + 2 * pad - KH) / stride + 1, g.Wout = (Win + 2 * pad - KW) / stride + 1;
  RL_CHECK_ARG(g.Hout > 0 && g.Wout > 0, "conv2d_nhwc_bf16_fwd: empty output");
  const long long M = (long long)N * g.Hout * g.Wout;
  RL_CHECK_ARG(M < (1LL << 31), "conv2d_nhwc_bf16_fwd: too many output pixels");
  g.M = (int)M, g.num_kb = K / 64, g.num_tiles = (int)((M + kCvBM - 1) / kCvBM), g.relu = relu;
  RL_CHECK_ARG((size_t)g.num_kb * Cout * 128 + (size_t)kCvStages * kCvBM * 128 + 2048 <= 227 * 1024,
               "conv2d_nhwc_bf16_fwd: weights do not fit in shared memory");
  alignas(64) CUtensorMap mw;
  if (make_weight_map(&mw, weight_krsc, K, Cout)) {
    set_error("conv2d_nhwc_bf16_fwd: cuTensorMapEncodeTiled failed");
    return RL_ERR_CUDA;
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (Cout == 32 && Cin == 64) launch_conv<32, 64>(mw, g, sms, st);
  else if (Cout == 32) launch_conv<32, 32>(mw, g, sms, st);
  else if (Cin == 64) launch_conv<64, 64>(mw, g, sms, st);
  else launch_conv<64, 32>(mw, g, sms, st);
  RL_CHECK_LAUNCH("rl_conv2d_nhwc_bf16_fwd");
  return RL_OK;
}
