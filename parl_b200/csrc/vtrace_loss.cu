// K1 — fused IMPALA loss: log-softmax + entropy + KL + V-trace backward scan +
// policy-gradient/value/entropy loss and its gradient, ONE launch.
//
// Reference arithmetic being replaced (PaddlePaddle/PARL):
//   parl/algorithms/paddle/impala/vtrace.py:99-139   V-trace recurrences
//   parl/algorithms/paddle/impala/impala.py:25-79    VTraceLoss (SUM reductions)
//   parl/algorithms/paddle/impala/impala.py:119-132  log-prob = sum(log_softmax * onehot)
//   parl/algorithms/paddle/impala/impala.py:148-208  row dropping / bootstrap / KL
//
// Layout in HBM: logits [T,B,A] f32, per-step scalars [T,B].  Two kernels:
//
//  * vtrace_loss_v8_kernel (default where eligible: time-major, TMA-aligned, T <= 64, B % 4 == 0, even A <= 18 — the
//    C3 learner batch): a CTA owns 4 adjacent env columns for ALL T rows, fetched as two half-tiles in time that are
//    all in flight from the first instruction; one element per thread per half with its logits register-resident
//    as packed pairs; in-warp shuffle suffix scan composed across warps after one block sync per half.
//  * vtrace_loss_kernel (v4, every other shape and the env-major layout; rl_debug_set_vtrace_path(4) forces it):
//    same CTA shape, chunks of <= 56 rows staged by 2-D TMA tensor maps (cp.async for env-major / unaligned shapes),
//    array-free two-sweep softmax, scan on warp 0, gradient tile written in place and TMA-stored.
//  Both: deterministic loss reduction (CTA partials -> last CTA, fp64).  Earlier designs (v5 warp-autonomous, v6
//  warp-per-8-row-chunk with 32 registers) were measured slower and removed: DESIGN.md section 4.
// Algorithmic traffic: (12A+17) bytes per kept (t,b) element (SURVEY.md 8d).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"
#include "tma.cuh"

namespace rl {

constexpr int kBW = 4;     // env columns per CTA
constexpr int kNT = 224;   // threads per CTA: one (t,b) element per thread, TC <= kNT / kBW = 56 rows per chunk

struct VtraceLossArgs {
  const float* tl;
  const float* bl;
  const void* actions;
  const float* rewards;
  const uint8_t* dones;
  const float* values;
  float* d_logits;
  float* d_values;
  float* vs_out;
  float* pg_out;
  float* losses;
  float* partials;     // [grid, 4]
  unsigned* ticket;    // zero on entry, zero on exit
  int T, B, A, TC;
  int act64, vec;
  float gamma, clip_rho, clip_pg, vf_coeff, ent_coeff;
};

// All index arithmetic is 32-bit (the host rejects T*B*A >= 2^31) and division-free:
// element i of a chunk is (t_local, b_local) = (i >> 2, i & 3) for both layouts.
template <bool EM>
__device__ __forceinline__ int gidx(int t, int b, int T, int B) {
  return EM ? b * T + t : t * B + b;
}
template <bool EM>
__device__ __forceinline__ int sidx(int tl, int bl, int TC) {
  return EM ? bl * TC + tl : tl * kBW + bl;
}

// global <-> shared tile copy, one segment per warp iteration, lanes stride the segment.
//   TM: nt row segments of nb*A floats (smem stride kBW*A);  EM: nb column segments of nt*A floats (stride TC*A).
template <bool EM, bool TO_SMEM>
__device__ __forceinline__ void copy_tile(float* s, const float* gsrc, float* gdst, int A, int T, int B, int TC,
                                          int t0, int nt, int b0, int nb, bool vec) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nseg = EM ? nb : nt;
  const int seglen = (EM ? nt : nb) * A;           // floats
  const int sstride = (EM ? TC : kBW) * A;
  const int gstride = (EM ? T : B) * A;            // floats between consecutive segments in global memory
  int goff = (EM ? (b0 * T + t0) : (t0 * B + b0)) * A + warp * gstride;
  float* sp = s + warp * sstride;
  for (int sg = warp; sg < nseg; sg += kNT / 32, goff += (kNT / 32) * gstride, sp += (kNT / 32) * sstride) {
    if (vec) {
      for (int k = lane * 4; k < seglen; k += 128) {
        if (TO_SMEM) cp_async16(sp + k, gsrc + goff + k);
        else *reinterpret_cast<float4*>(gdst + goff + k) = *reinterpret_cast<const float4*>(sp + k);
      }
    } else {
      for (int k = lane; k < seglen; k += 32) {
        if (TO_SMEM) cp_async4(sp + k, gsrc + goff + k);
        else gdst[goff + k] = sp[k];
      }
    }
  }
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kL2E = 1.4426950408889634f;   // log2(e)
constexpr float kLN2 = 0.6931471805599453f;   // ln(2)

// Per-element softmax statistics in TWO array-free sweeps over the shared-memory rows (registers hold only
// running scalars, so 7 CTAs x 7 warps stay resident per SM):
//   sweep 1: m = max_j x_j, my = max_j y_j                                   (x target, y behaviour logits)
//   sweep 2: with xs_j = (x_j - m) log2e, e_j = 2^xs_j:  S = sum e_j, W = sum e_j xs_j, Y = sum e_j y_j,
//            Sy = sum 2^((y_j - my) log2e)
// from which  log2 p_j = xs_j - log2 S,  sum_j p_j log2 p_j = W/S - log2 S,  sum_j p_j y_j = Y/S.
// The tiles are left untouched; phase C recomputes p_j from x_j (one FFMA + MUFU.EX2 each).
struct SoftmaxStats {
  float nm;      // -m * log2e
  float l2S;     // log2 sum_j 2^xs_j
  float inv;     // 1 / S
  float la;      // log pi(a)      (natural log)
  float lma;     // log mu(a)
  float H;       // entropy of pi  (natural log)
  float KL;      // KL(pi || mu)
};

template <int A_>
__device__ __forceinline__ SoftmaxStats softmax_stats(const float* __restrict__ st, const float* __restrict__ sb, int A,
                                                      int act) {
  SoftmaxStats r;
  float m, my;
  if constexpr (A_ > 0 && (A_ & 1) == 0) {
    float2 a = *reinterpret_cast<const float2*>(st);
    float2 b = *reinterpret_cast<const float2*>(sb);
    m = fmaxf(a.x, a.y), my = fmaxf(b.x, b.y);
#pragma unroll 4
    for (int j = 2; j < A_; j += 2) {
      a = *reinterpret_cast<const float2*>(st + j);
      b = *reinterpret_cast<const float2*>(sb + j);
      m = fmaxf(m, fmaxf(a.x, a.y));
      my = fmaxf(my, fmaxf(b.x, b.y));
    }
  } else {
    m = st[0], my = sb[0];
    for (int j = 1; j < A; ++j) m = fmaxf(m, st[j]), my = fmaxf(my, sb[j]);
  }
  const float nm = -m * kL2E, nmy = -my * kL2E;
  float S0 = 0.f, S1 = 0.f, W0 = 0.f, W1 = 0.f, Y0 = 0.f, Y1 = 0.f, Sy0 = 0.f, Sy1 = 0.f;
  if constexpr (A_ > 0 && (A_ & 1) == 0) {
#pragma unroll 3
    for (int j = 0; j < A_; j += 2) {
      const float2 a = *reinterpret_cast<const float2*>(st + j);
      const float2 b = *reinterpret_cast<const float2*>(sb + j);
      const float xs0 = fmaf(a.x, kL2E, nm), xs1 = fmaf(a.y, kL2E, nm);
      const float e0 = ex2_approx(xs0), e1 = ex2_approx(xs1);
      S0 += e0, S1 += e1;
      W0 = fmaf(e0, xs0, W0), W1 = fmaf(e1, xs1, W1);
      Y0 = fmaf(e0, b.x, Y0), Y1 = fmaf(e1, b.y, Y1);
      Sy0 += ex2_approx(fmaf(b.x, kL2E, nmy));
      Sy1 += ex2_approx(fmaf(b.y, kL2E, nmy));
    }
  } else {
    for (int j = 0; j < A; ++j) {
      const float xs0 = fmaf(st[j], kL2E, nm);
      const float e0 = ex2_approx(xs0);
      S0 += e0;
      W0 = fmaf(e0, xs0, W0);
      Y0 = fmaf(e0, sb[j], Y0);
      Sy0 += ex2_approx(fmaf(sb[j], kL2E, nmy));
    }
  }
  const float S = S0 + S1, W = W0 + W1, Y = Y0 + Y1, Sy = Sy0 + Sy1;
  const float l2S = lg2_approx(S);
  const float inv = __fdividef(1.0f, S);
  const float logSy = lg2_approx(Sy) * kLN2;
  // explicit fma / rounding: every template instance must give the same bits (TMA and cp.async tile paths agree)
  const float Hn = fmaf(W, inv, -l2S) * kLN2;          // sum_j p_j log p_j
  r.nm = nm, r.l2S = l2S, r.inv = inv;
  r.H = -Hn;
  r.KL = __fadd_rn(__fadd_rn(fmaf(-Y, inv, Hn), my), logSy);   // sum_j p_j (log p_j - log q_j)
  r.la = (fmaf(st[act], kL2E, nm) - l2S) * kLN2;
  r.lma = sb[act] - my - logSy;
  return r;
}

// Shared-memory carve-up (bytes): [tile_tl | pad to 128][tile_bl | pad to 128][s_acc][s_kc]
__host__ __device__ inline int tile_bytes_padded(int TC, int A) { return (TC * kBW * A * 4 + 127) & ~127; }

template <int A_, bool EM, bool TMA>
__global__ void __launch_bounds__(kNT, 7) vtrace_loss_kernel(const VtraceLossArgs p,
                                                            const __grid_constant__ CUtensorMap map_tl,
                                                            const __grid_constant__ CUtensorMap map_bl,
                                                            const __grid_constant__ CUtensorMap map_dl) {
  static_assert(!(TMA && EM), "the TMA tile path is time-major only");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int A = A_ > 0 ? A_ : p.A;
  const int T = p.T, B = p.B, TC = p.TC;
  const int tile_pad = tile_bytes_padded(TC, A);
  float* s_tl = reinterpret_cast<float*>(smem_raw);
  float* s_bl = reinterpret_cast<float*>(smem_raw + tile_pad);
  float* s_acc = reinterpret_cast<float*>(smem_raw + 2 * tile_pad);   // delta, then acc = vs - V
  float* s_kc = s_acc + TC * kBW;                                     // gamma_t * min(rho, 1)
  __shared__ float s_carry[kBW];        // acc at the first row of the chunk processed before (later in time)
  __shared__ float s_red[4][kNT / 32];
  __shared__ bool s_last;
  __shared__ __align__(8) unsigned long long s_mbar;
  uint32_t mbar_phase = 0;
  const int tid = threadIdx.x;
  if (TMA) {
    if (tid == 0) {
      tma_prefetch_desc(&map_tl);
      tma_prefetch_desc(&map_bl);
      tma_prefetch_desc(&map_dl);
      mbar_init(&s_mbar, 1);
      fence_mbar_init();
    }
  }
  if (tid < kBW) s_carry[tid] = 0.f;
  __syncthreads();

  const int b0 = blockIdx.x * kBW;
  const int nb = min(kBW, B - b0);
  // this thread's element of every chunk: (t_local, b_local) = (tid >> 2, tid & 3)
  const int tl_ = tid >> 2, bl_ = tid & 3;
  const int si = sidx<EM>(tl_, bl_, TC);
  float sum_pi = 0.f, sum_vf = 0.f, sum_ent = 0.f, sum_kl = 0.f;
  float acc_carry = 0.f;

  const int nchunks = (T + TC - 1) / TC;
  for (int c = nchunks - 1; c >= 0; --c) {
    const int t0 = c * TC;
    const int nt = min(TC, T - t0);
    const bool vec = p.vec && (((EM ? nt : nb) * A) & 3) == 0;
    if (TMA) {
      // one elected thread: two 2-D TMA tile loads (box = TC rows x kBW*A floats; rows/columns past the
      // tensor edge are zero-filled by the hardware), completion signalled on the mbarrier
      if (tid == 0) {
        mbar_arrive_expect_tx(&s_mbar, 2u * (uint32_t)(TC * kBW * A * 4));
        tma_load_2d(s_tl, &map_tl, b0 * A, t0, &s_mbar);
        tma_load_2d(s_bl, &map_bl, b0 * A, t0, &s_mbar);
      }
    } else {
      copy_tile<EM, true>(s_tl, p.tl, nullptr, A, T, B, TC, t0, nt, b0, nb, vec);
      copy_tile<EM, true>(s_bl, p.bl, nullptr, A, T, B, TC, t0, nt, b0, nb, vec);
      cp_async_commit();
    }

    // ---- per-element scalars straight from global (overlaps the tile copy) ----
    const bool valid = tl_ < nt && bl_ < nb;
    const int t = t0 + tl_;
    const bool loss_row = valid && t < T - 1;
    const int g = gidx<EM>(t, b0 + bl_, T, B);
    int act = 0;
    float e_r = 0.f, e_v = 0.f, e_vn = 0.f, e_g = 0.f;
    if (valid) {
      act = p.act64 ? (int)reinterpret_cast<const long long*>(p.actions)[g] : reinterpret_cast<const int*>(p.actions)[g];
      e_r = p.rewards[g];
      e_v = p.values[g];
      e_g = p.dones[g] ? 0.0f : p.gamma;                  // impala.py:59  (~dones) * discount
      if (t + 1 < T) e_vn = p.values[g + (EM ? 1 : B)];
    }
    if (TMA) {
      mbar_wait(&s_mbar, mbar_phase);
      mbar_phase ^= 1u;
    } else {
      cp_async_wait<0>();
      __syncthreads();
    }

    // ---- phase A: softmax / entropy / KL / rho / delta (element-private, tiles read-only) ----
    SoftmaxStats ss;
    float e_rpg = 0.f;
    ss.nm = 0.f, ss.l2S = 0.f, ss.inv = 0.f, ss.la = 0.f, ss.lma = 0.f, ss.H = 0.f, ss.KL = 0.f;
    if (valid) {
      ss = softmax_stats<A_>(s_tl + si * A, s_bl + si * A, A, act);
      sum_kl += ss.KL;                                    // impala.py:160-162: every row
      if (loss_row) {
        const float rho = expf(ss.la - ss.lma);           // vtrace.py:101-103
        const float rhoc = p.clip_rho >= 0.f ? fminf(rho, p.clip_rho) : rho;
        const float cs = fminf(rho, 1.0f);                // :109
        e_rpg = p.clip_pg >= 0.f ? fminf(rho, p.clip_pg) : rho;
        // deltas = clipped_rhos * (rewards + discounts * values_t_plus_1 - values)   :115
        const float td = __fsub_rn(__fadd_rn(e_r, __fmul_rn(e_g, e_vn)), e_v);
        s_acc[si] = __fmul_rn(rhoc, td);
        s_kc[si] = __fmul_rn(e_g, cs);
        sum_ent += ss.H;
      }
    }
    __syncthreads();

    // ---- phase B: backward-in-time scan acc_t = delta_t + k_t * acc_{t+1} as a warp-shuffle segmented prefix:
    //      warp 0 = 4 columns x 8 time segments; each lane composes the affine maps of its rows, a 3-step
    //      shuffle suffix-scan combines the segments (k_t = 0 at episode cuts makes the prefix segmented),
    //      then each lane replays its rows with the incoming accumulator.
    if (tid < 32) {
      const int col = tid & 3, seg = tid >> 2;                 // lane = seg*4 + col
      const int nrows = min(nt, T - 1 - t0);                   // loss rows of this chunk (bootstrap row skipped)
      const int per = (nrows + 7) >> 3;
      const int lo = min(seg * per, nrows), hi = min(lo + per, nrows);     // this lane's rows [lo, hi)
      const int step = EM ? 1 : kBW;
      const bool colok = col < nb;
      float D = 0.f, K = 1.f;
      if (colok) {
        int sj = sidx<EM>(hi - 1, col, TC);
        for (int q = hi - 1; q >= lo; --q, sj -= step) {
          const float k = s_kc[sj];
          D = fmaf(k, D, s_acc[sj]);
          K *= k;
        }
      }
      // inclusive suffix scan over segments (later time = higher seg): F_seg o F_{seg+off}
#pragma unroll
      for (int off = 1; off < 8; off <<= 1) {
        const float Dn = __shfl_down_sync(0xffffffffu, D, off * 4);
        const float Kn = __shfl_down_sync(0xffffffffu, K, off * 4);
        if (seg + off < 8) {
          D = fmaf(K, Dn, D);
          K *= Kn;
        }
      }
      // accumulator entering this lane's segment = composite of all later segments applied to the carry
      const float Dx = __shfl_down_sync(0xffffffffu, D, 4), Kx = __shfl_down_sync(0xffffffffu, K, 4);
      const float carry_in = __shfl_sync(0xffffffffu, acc_carry, col);       // lanes 0..3 hold the column carries
      float acc = seg < 7 ? fmaf(Kx, carry_in, Dx) : carry_in;
      if (colok) {
        int sj = sidx<EM>(hi - 1, col, TC);
        for (int q = hi - 1; q >= lo; --q, sj -= step) {
          acc = fmaf(s_kc[sj], acc, s_acc[sj]);
          s_acc[sj] = acc;
        }
      }
      // lanes 0..3 (segment 0) end on row 0 of the chunk: that is the carry for the next (earlier) chunk
      if (seg == 0) acc_carry = acc;
    }
    __syncthreads();

    // ---- phase C: advantages, losses, gradient tile (written over the target-logit tile) ----
    if (valid) {
      float* pt = s_tl + si * A;
      if (loss_row) {
        const float acc_n = (t + 1 == T - 1) ? 0.f : (tl_ + 1 < nt ? s_acc[sidx<EM>(tl_ + 1, bl_, TC)] : s_carry[bl_]);
        const float vs = __fadd_rn(s_acc[si], e_v);                    // vtrace.py:125
        const float vs_n = __fadd_rn(acc_n, e_vn);                     // :128-129 (bootstrap at the end)
        const float adv = __fmul_rn(e_rpg, __fsub_rn(__fadd_rn(e_r, __fmul_rn(e_g, vs_n)), e_v));   // :136-137
        const float dv = e_v - vs;
        // explicit fma: the rounding must not depend on how the compiler contracts each template instance
        sum_pi = fmaf(-ss.la, adv, sum_pi);                             // impala.py:67-68
        sum_vf = fmaf(0.5f * dv, dv, sum_vf);                           // :71-72
        p.d_values[g] = p.vf_coeff * dv;
        if (p.vs_out) p.vs_out[t * B + b0 + bl_] = vs;
        if (p.pg_out) p.pg_out[t * B + b0 + bl_] = adv;
        // dL/dz_j = p_j (adv - c_e (H + log p_j)) - adv [j == a],  log p_j = ln2 (xs_j - log2 S)
        const float ce2 = p.ent_coeff * kLN2;
        const float c0 = fmaf(ce2, ss.l2S, adv - p.ent_coeff * ss.H) * ss.inv;   // folded with 1/S
        const float c1 = -ce2 * ss.inv;
        if constexpr (A_ > 0 && (A_ & 1) == 0) {
#pragma unroll 3
          for (int j = 0; j < A_; j += 2) {
            const float2 a = *reinterpret_cast<const float2*>(pt + j);
            const float xs0 = fmaf(a.x, kL2E, ss.nm), xs1 = fmaf(a.y, kL2E, ss.nm);
            const float d0 = ex2_approx(xs0) * fmaf(c1, xs0, c0), d1 = ex2_approx(xs1) * fmaf(c1, xs1, c0);
            *reinterpret_cast<float2*>(pt + j) = make_float2(d0, d1);
          }
        } else {
          for (int j = 0; j < A; ++j) {
            const float xs0 = fmaf(pt[j], kL2E, ss.nm);
            pt[j] = ex2_approx(xs0) * fmaf(c1, xs0, c0);
          }
        }
        pt[act] -= adv;
      } else {
        p.d_values[g] = 0.f;                                            // bootstrap row: no gradient
        for (int j = 0; j < A; ++j) pt[j] = 0.f;
      }
    }
    if (TMA) {
      fence_proxy_async_smem();          // generic-proxy writes of the gradient tile -> visible to the TMA engine
      __syncthreads();
      if (tid < nb) s_carry[tid] = acc_carry;
      if (tid == 0) {
        tma_store_2d(&map_dl, b0 * A, t0, s_tl);
        tma_store_commit();
        tma_store_wait_read();           // smem tile may be overwritten / the CTA may exit afterwards
      }
      if (c > 0) __syncthreads();
    } else {
      __syncthreads();
      if (tid < nb) s_carry[tid] = acc_carry;
      copy_tile<EM, false>(s_tl, nullptr, p.d_logits, A, T, B, TC, t0, nt, b0, nb, vec);
      if (c > 0) __syncthreads();
    }
  }

  // ---- loss reduction: warp -> CTA -> (last CTA) grid, fixed order, fp64 at the end ----
  float sums[4] = {sum_pi, sum_vf, sum_ent, sum_kl};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float w = warp_sum(sums[q]);
    if ((tid & 31) == 0) s_red[q][tid >> 5] = w;
  }
  __syncthreads();
  if (tid < 4) {
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < kNT / 32; ++w) a += s_red[tid][w];
    p.partials[blockIdx.x * 4 + tid] = a;
    __threadfence();
  }
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(p.ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (s_last) {
    __threadfence();
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    {
      // all loads of a pass in flight at once (a loop of dependent L2 round trips is microseconds of single-CTA tail)
      const float4* parts = reinterpret_cast<const float4*>(p.partials);
      const int n = (int)gridDim.x;
      for (int base = 0; base < n; base += kNT * 4) {
        float4 q[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = base + u * kNT + tid;
          q[u] = i < n ? __ldcg(parts + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          acc[0] += (double)q[u].x, acc[1] += (double)q[u].y, acc[2] += (double)q[u].z, acc[3] += (double)q[u].w;
      }
    }
    __shared__ double s_dred[4][kNT / 32];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      double v = acc[q];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((tid & 31) == 0) s_dred[q][tid >> 5] = v;
    }
    __syncthreads();
    if (tid == 0) {
      double r[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        r[q] = 0.0;
        for (int w = 0; w < kNT / 32; ++w) r[q] += s_dred[q][w];
      }
      const float pi = (float)r[0], vf = (float)r[1], ent = (float)r[2];
      p.losses[0] = pi + vf * p.vf_coeff + ent * p.ent_coeff;      // impala.py:78-79
      p.losses[1] = pi;
      p.losses[2] = vf;
      p.losses[3] = ent;
      p.losses[4] = (float)(r[3] / ((double)T * (double)B));
      *p.ticket = 0u;
    }
  }
}

// ---------------------------------------------------------------------------
// a1: plain V-trace on log-probs (exact reference op order; exp in fp64 so the
// float result is correctly rounded).  One lane per env column, coalesced over b.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) vtrace_returns_kernel(const float* __restrict__ blp, const float* __restrict__ tlp,
                                                            const float* __restrict__ disc, const float* __restrict__ rew,
                                                            const float* __restrict__ val, const float* __restrict__ boot,
                                                            int T, int B, float clip_rho, float clip_pg,
                                                            float* __restrict__ vs, float* __restrict__ pg) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float acc = 0.f;
  float v_next = boot[b];
  float vs_next = boot[b];
  for (int t = T - 1; t >= 0; --t) {
    const long long g = (long long)t * B + b;
    const float rho = (float)exp((double)__fsub_rn(tlp[g], blp[g]));
    const float rhoc = clip_rho >= 0.f ? fminf(rho, clip_rho) : rho;
    const float rhopg = clip_pg >= 0.f ? fminf(rho, clip_pg) : rho;
    const float cs = fminf(rho, 1.0f);
    const float d = disc[g], r = rew[g], v = val[g];
    const float delta = __fmul_rn(rhoc, __fsub_rn(__fadd_rn(r, __fmul_rn(d, v_next)), v));
    acc = __fadd_rn(delta, __fmul_rn(__fmul_rn(d, cs), acc));
    const float vs_t = __fadd_rn(acc, v);
    pg[g] = __fmul_rn(rhopg, __fsub_rn(__fadd_rn(r, __fmul_rn(d, vs_next)), v));
    vs[g] = vs_t;
    vs_next = vs_t;
    v_next = v;
  }
}

// ---------------------------------------------------------------------------
// v8 (default for time-major TMA shapes with T <= 64, B % 4 == 0, even A <= 18): the K1 of the C3 learner batch.
//
// v4 spends three shared-memory sweeps with loop overhead, 3 block syncs per tile and a scan on warp 0 only per
// element, and its CTAs load, then compute, then store in lock-step.  v8 keeps the CTA shape "4 env columns x all T
// rows" (the scan never leaves the CTA; 7 CTAs resident per SM, so the B/4 = 1024 CTAs of B = 4096 are 1.1 waves on
// the 132 SMs of an H100) and changes what happens inside it:
//   * the tile is fetched as TWO half-tiles in time (later half first: it heads the backward recurrence), each with
//     its own mbarrier; all four TMA loads are in flight from the first instruction, so the second half streams in
//     while the first is being computed, and its gradient rows leave by TMA while the second half is computed;
//   * 4 warps = one (t,b) element per thread per half; the element's 2A logits are read from shared memory ONCE
//     into registers as 64-bit pairs (stride-18-word LDS.64: conflict-free), all arithmetic on packed pairs
//     (fma2/add2/mul2), exponentials kept in registers for the gradient (no second MUFU pass, no re-read);
//   * the recurrence acc_t = delta_t + k_t acc_{t+1} is a 3-step shuffle suffix scan of affine maps inside each warp
//     (8 rows), composed across the 4 warps after ONE block sync per half, carry between the halves in shared memory;
//   * loss partials: one float4 per CTA, last CTA (ticket) reduces them in fixed order in fp64, overlapped with
//     the drain of the gradient stores.
// ---------------------------------------------------------------------------
typedef unsigned long long u64;
__device__ __forceinline__ u64 pk2(float lo, float hi) {
  u64 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void upk2(u64 v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
// sm_90 has no packed f32x2 arithmetic: each pair op is two scalar round-to-nearest ops (same results)
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
  float a0, a1, b0, b1, c0, c1;
  upk2(a, a0, a1), upk2(b, b0, b1), upk2(c, c0, c1);
  return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1), upk2(b, b0, b1);
  return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1), upk2(b, b0, b1);
  return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
// mbarrier wait with a hardware suspend-time hint (the warp sleeps instead of spinning on the LSU)
__device__ __forceinline__ void mbar_wait_suspend(void* mbar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT_S:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      "@p bra LAB_DONE_S;\n"
      "bra LAB_WAIT_S;\n"
      "LAB_DONE_S:\n"
      "}\n" ::"r"(smem_u32(mbar)),
      "r"(parity), "r"(0x000f4240)
      : "memory");
}

constexpr int kV8Warps = 4;                // 128 threads: 32 rows x 4 columns per pass
constexpr int kV8Rows = 32;                // rows of the later (first processed) pass
constexpr int kV8MaxT = 64;

struct V8Maps {                            // [0] = box of the earlier rows [0, T-R1), [1] = box of the later rows [T-R1, T)
  CUtensorMap tl[2], bl[2], dl[2];
  CUtensorMap act, rew, val, dval;         // per-step scalars [T, B]: box = all T rows x 4 columns (16 bytes)
};

template <int A_>
__global__ void __launch_bounds__(kV8Warps * 32, 7)     // 7 CTAs x 4 warps per SM: B/4 CTAs = one wave at B = 4096
    vtrace_loss_v8_kernel(const VtraceLossArgs p, const __grid_constant__ V8Maps maps) {
  static_assert(A_ >= 2 && (A_ & 1) == 0, "v8 needs an even compile-time A");
  constexpr int CW = 4, NW = kV8Warps, NP = A_ / 2;
  constexpr int kRowBytes = CW * A_ * 4;
  constexpr uint32_t FULL = 0xffffffffu;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ __align__(8) u64 s_bar[2];
  __shared__ float2 s_comp[2][NW][CW];
  __shared__ float s_carry[CW];
  __shared__ float s_red[4][NW];
  __shared__ double s_dred[4][NW];
  __shared__ int s_last;
  const int T = p.T, B = p.B;
  const int R1 = min(T, kV8Rows), R0 = T - R1;           // pass 1 = rows [R0, T) (first), pass 0 = rows [0, R0)
  // shared memory: logits tiles [R1 later rows | R0 earlier rows] x [CW*A] floats (R1 * kRowBytes is a multiple of
  // 128 when R0 > 0, so both TMA destinations are 128-byte aligned), then the scalar tiles [T][CW] in row order
  const int tile_pad = (T * kRowBytes + 127) & ~127;
  const int sc_pad = (T * CW * 4 + 127) & ~127;
  unsigned char* s_x = smem_raw;                         // target logits, overwritten by the gradient
  unsigned char* s_y = smem_raw + tile_pad;              // behaviour logits
  const int* s_act = reinterpret_cast<const int*>(smem_raw + 2 * tile_pad);
  float* s_rew = reinterpret_cast<float*>(smem_raw + 2 * tile_pad + sc_pad);      // rewards, overwritten by d_values
  const float* s_val = reinterpret_cast<const float*>(smem_raw + 2 * tile_pad + 2 * sc_pad);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b0 = blockIdx.x * CW;

  // Every input of the CTA arrives by TMA (no per-thread global loads on the critical path: 16-byte rows of the
  // [T, B] scalar arrays fetched by LDG cost one L1 miss entry each and were what the warps waited for).
  if (tid == 0) {
    tma_prefetch_desc(&maps.tl[1]);
    tma_prefetch_desc(&maps.bl[1]);
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    fence_mbar_init();
  }
  // Programmatic dependent launch (when the launch carries the attribute; no-ops otherwise): the prologue above ran
  // while the predecessor in the stream was still draining; nothing it produced has been touched yet.
  pdl_trigger();
  pdl_wait();
  __syncthreads();                                       // barrier initialisation visible to every waiter / issuer
  // one elected lane per warp issues its share of the seven loads (a single thread needs ~0.4 us for all of them);
  // the transaction bytes are posted by warp 0 — a complete_tx that lands first only drives the count negative, the
  // phase cannot complete before the pending arrival
  if (lane == 0) {
    if (warp == 0) {
      mbar_arrive_expect_tx(&s_bar[1], 2u * (uint32_t)(R1 * kRowBytes) + 3u * (uint32_t)(T * CW * 4));
      if (R0 > 0) mbar_arrive_expect_tx(&s_bar[0], 2u * (uint32_t)(R0 * kRowBytes));
      tma_load_2d(s_x, &maps.tl[1], b0 * A_, R0, &s_bar[1]);            // later rows first: they head the recurrence
    } else if (warp == 1) {
      tma_load_2d(s_y, &maps.bl[1], b0 * A_, R0, &s_bar[1]);
    } else if (warp == 2) {
      tma_load_2d(const_cast<int*>(s_act), &maps.act, b0, 0, &s_bar[1]);
      tma_load_2d(s_rew, &maps.rew, b0, 0, &s_bar[1]);
      tma_load_2d(const_cast<float*>(s_val), &maps.val, b0, 0, &s_bar[1]);
    } else if (R0 > 0) {
      tma_load_2d(s_x + R1 * kRowBytes, &maps.tl[0], b0 * A_, 0, &s_bar[0]);
      tma_load_2d(s_y + R1 * kRowBytes, &maps.bl[0], b0 * A_, 0, &s_bar[0]);
    }
  }
  // ---- this thread's element of each pass: (row r of the pass, column c).  Rows past the pass's last row are
  //      CLAMPED onto it (valid memory, throw-away arithmetic) so that the hot path is branch-free; warps that hold
  //      no row at all skip the arithmetic and contribute identity maps.
  const int r = tid >> 2, c = tid & 3;
  // done flags: the 4 columns of a row are one aligned 32-bit word; lane c == 0 of each row fetches it
  uint32_t dn1 = 0, dn0 = 0;
  if (c == 0) {
    dn1 = *reinterpret_cast<const uint32_t*>(p.dones + (size_t)(R0 + min(r, R1 - 1)) * B + b0);
    if (R0 > 0) dn0 = *reinterpret_cast<const uint32_t*>(p.dones + (size_t)min(r, R0 - 1) * B + b0);
  }

  float sum_pi = 0.f, sum_vf = 0.f, sum_ent = 0.f, sum_kl = 0.f;
  const int h_last = R0 > 0 ? 0 : 1;
#pragma unroll 1
  for (int h = 1; h >= h_last; --h) {
    const int nrows = h ? R1 : R0;
    float D = 0.f, K = 1.f;                              // identity map: rows that do not exist
    float l2S = 0.f, inv = 0.f, H = 0.f, la = 0.f, rpg = 0.f;
    float er = 0.f, ev = 0.f, eg = 0.f, evn = 0.f;
    int act = 0;
    u64 X[NP], E[NP];
#pragma unroll
    for (int j = 0; j < NP; ++j) X[j] = 0ull, E[j] = 0ull;
    const bool warp_on = warp * 8 < nrows;               // warp-uniform
    const int rc = min(r, nrows - 1);
    const int t = (h ? R0 : 0) + rc;
    const bool valid = r < nrows;
    const bool loss = valid && t < T - 1;
    const int soff = ((h ? 0 : R1) + rc) * kRowBytes + c * (A_ * 4);
    float* px = reinterpret_cast<float*>(s_x + soff);
    const float* py = reinterpret_cast<const float*>(s_y + soff);
    if (warp_on) {
      if (h) mbar_wait_suspend(&s_bar[1], 0);
      else mbar_wait_suspend(&s_bar[0], 0);
      // ---- scalars of the element (shared memory; the done word comes from the row's first lane)
      const uint32_t dw = __shfl_sync(FULL, h ? dn1 : dn0, lane & ~3);
      act = s_act[t * CW + c];
      er = s_rew[t * CW + c];
      ev = s_val[t * CW + c];
      evn = s_val[min(t + 1, T - 1) * CW + c];
      eg = ((dw >> (8 * c)) & 0xffu) ? 0.0f : p.gamma;       // impala.py:59  (~dones) * discount
      // ---- phase A: one read of the 2A logits, maxima, then (packed pairs) xs = (x - m) log2e, e = 2^xs,
      //      S = sum e, W = sum e xs, Y = sum e y, Sy = sum 2^((y - my) log2e)
      u64 Y[NP];
#pragma unroll
      for (int j = 0; j < NP; ++j) {
        X[j] = *reinterpret_cast<const u64*>(px + 2 * j);
        Y[j] = *reinterpret_cast<const u64*>(py + 2 * j);
      }
      const float x_act = px[act], y_act = py[act];
      float m, my;
      {
        float a0, a1, c0_, c1_;
        upk2(X[0], a0, a1);
        upk2(Y[0], c0_, c1_);
        m = fmaxf(a0, a1), my = fmaxf(c0_, c1_);
#pragma unroll
        for (int j = 1; j < NP; ++j) {
          upk2(X[j], a0, a1);
          upk2(Y[j], c0_, c1_);
          m = max3(m, a0, a1);
          my = max3(my, c0_, c1_);
        }
      }
      const float nm = -m * kL2E, nmy = -my * kL2E;
      const u64 cL = pk2(kL2E, kL2E), cnm = pk2(nm, nm), cnmy = pk2(nmy, nmy);
      u64 S2 = pk2(0.f, 0.f), W2 = S2, Y2 = S2, Sy2 = S2;
#pragma unroll
      for (int j = 0; j < NP; ++j) {
        const u64 xs = fma2(X[j], cL, cnm);
        const u64 ys = fma2(Y[j], cL, cnmy);
        float a0, a1, c0_, c1_;
        upk2(xs, a0, a1);
        upk2(ys, c0_, c1_);
        const u64 e = pk2(ex2_approx(a0), ex2_approx(a1));
        const u64 ey = pk2(ex2_approx(c0_), ex2_approx(c1_));
        S2 = add2(S2, e);
        W2 = fma2(e, xs, W2);
        Y2 = fma2(e, Y[j], Y2);
        Sy2 = add2(Sy2, ey);
        X[j] = xs;
        E[j] = e;
      }
      float s0, s1, w0, w1, y0, y1, q0, q1;
      upk2(S2, s0, s1);
      upk2(W2, w0, w1);
      upk2(Y2, y0, y1);
      upk2(Sy2, q0, q1);
      const float S = s0 + s1, Wt = w0 + w1, Yt = y0 + y1, Sy = q0 + q1;
      l2S = lg2_approx(S);
      inv = __fdividef(1.0f, S);
      const float logSy = lg2_approx(Sy) * kLN2;
      const float Hn = (Wt * inv - l2S) * kLN2;            // sum_j p_j log p_j
      H = -Hn;
      sum_kl += valid ? Hn - Yt * inv + my + logSy : 0.f;  // impala.py:160-162: every row
      la = (fmaf(x_act, kL2E, nm) - l2S) * kLN2;
      const float lma = y_act - my - logSy;
      const float rho = ex2_approx((la - lma) * kL2E);     // vtrace.py:101-103
      const float rhoc = p.clip_rho >= 0.f ? fminf(rho, p.clip_rho) : rho;
      rpg = p.clip_pg >= 0.f ? fminf(rho, p.clip_pg) : rho;
      // deltas = clipped_rhos * (rewards + discounts * values_t_plus_1 - values)   :115 ; k = discount * min(rho, 1)  :109
      D = loss ? __fmul_rn(rhoc, __fsub_rn(__fadd_rn(er, __fmul_rn(eg, evn)), ev)) : 0.f;
      K = loss ? __fmul_rn(eg, fminf(rho, 1.0f)) : (valid ? 0.f : 1.f);
      sum_ent += loss ? H : 0.f;
      // ---- phase B: suffix scan of the affine maps acc -> D + K acc over the warp's 8 rows (later time = higher lane)
#pragma unroll
      for (int off = CW; off < 32; off <<= 1) {
        const float Dn = __shfl_down_sync(FULL, D, off);
        const float Kn = __shfl_down_sync(FULL, K, off);
        const bool in = lane + off < 32;
        D = in ? fmaf(K, Dn, D) : D;
        K = in ? K * Kn : K;
      }
    }
    if (lane < CW) s_comp[h][warp][lane] = make_float2(D, K);          // the warp's 8 rows as one map, per column
    __syncthreads();
    if (h == 0 && tid == 0) {                              // the later rows' gradient is complete: send it
      tma_store_2d(&maps.dl[1], b0 * A_, R0, s_x);
      tma_store_commit();
    }
    // accumulator entering this warp's rows = later warps' maps applied to the later pass's carry, latest first
    float cin = h ? 0.f : s_carry[c];
    for (int w2 = NW - 1; w2 > warp; --w2) {
      const float2 m2 = s_comp[h][w2][c];
      cin = fmaf(m2.y, cin, m2.x);
    }
    const float acc = fmaf(K, cin, D);
    float acc_n = __shfl_down_sync(FULL, acc, CW);
    acc_n = lane >= 32 - CW ? cin : acc_n;
    if (h == 1 && tid < CW) s_carry[tid] = acc;            // acc at the first row of the later pass
    // ---- phase C: advantages, losses, gradient row in place of the target logits
    const float vs = __fadd_rn(acc, ev);                               // vtrace.py:125
    const float vs_n = __fadd_rn(acc_n, evn);                          // :128-129 (bootstrap at the end)
    const float adv = loss ? __fmul_rn(rpg, __fsub_rn(__fadd_rn(er, __fmul_rn(eg, vs_n)), ev)) : 0.f;   // :136-137
    const float dv = loss ? ev - vs : 0.f;
    sum_pi -= la * adv;                                                 // impala.py:67-68
    sum_vf = fmaf(0.5f * dv, dv, sum_vf);                               // :71-72
    if (valid) {
      s_rew[t * CW + c] = p.vf_coeff * dv;                              // d_values tile (the reward was consumed above)
      if (loss) {
        if (p.vs_out) p.vs_out[t * B + b0 + c] = vs;
        if (p.pg_out) p.pg_out[t * B + b0 + c] = adv;
      }
      // dL/dz_j = p_j (adv - c_e (H + log p_j)) - adv [j == a],  log p_j = ln2 (xs_j - log2 S); all 0 on the last row
      const float ce2 = loss ? p.ent_coeff * kLN2 : 0.f;
      const float c0 = fmaf(ce2, l2S, adv - (loss ? p.ent_coeff * H : 0.f)) * inv;   // folded with 1/S
      const float c1 = -ce2 * inv;
      const u64 c02 = pk2(c0, c0), c12 = pk2(c1, c1);
#pragma unroll
      for (int j = 0; j < NP; ++j) *reinterpret_cast<u64*>(px + 2 * j) = mul2(E[j], fma2(c12, X[j], c02));
      px[act] -= adv;
    }
    fence_proxy_async_smem();            // generic-proxy writes of the gradient rows -> visible to the TMA engine
  }

  // ---- loss reduction: warp -> CTA -> (last CTA) grid, fixed order, fp64 at the end
  sum_pi = warp_sum(sum_pi), sum_vf = warp_sum(sum_vf), sum_ent = warp_sum(sum_ent), sum_kl = warp_sum(sum_kl);
  if (lane == 0) s_red[0][warp] = sum_pi, s_red[1][warp] = sum_vf, s_red[2][warp] = sum_ent, s_red[3][warp] = sum_kl;
  __syncthreads();
  // thread 0: gradient stores, the CTA's partial (one float4), the ticket.  The CTA that draws the last ticket reduces
  // all partials (L2-resident) with EVERY load in flight at once: 8 independent float4 loads per thread, so the
  // single-CTA tail is one L2 round trip instead of a loop of dependent ones.
  if (tid == 0) {
    if (R0 > 0) tma_store_2d(&maps.dl[0], b0 * A_, 0, s_x + R1 * kRowBytes);
    else tma_store_2d(&maps.dl[1], b0 * A_, 0, s_x);
    tma_store_2d(&maps.dval, b0, 0, s_rew);
    tma_store_commit();
    float4 part;
    part.x = (s_red[0][0] + s_red[0][1]) + (s_red[0][2] + s_red[0][3]);
    part.y = (s_red[1][0] + s_red[1][1]) + (s_red[1][2] + s_red[1][3]);
    part.z = (s_red[2][0] + s_red[2][1]) + (s_red[2][2] + s_red[2][3]);
    part.w = (s_red[3][0] + s_red[3][1]) + (s_red[3][2] + s_red[3][3]);
    reinterpret_cast<float4*>(p.partials)[blockIdx.x] = part;
    // release: the partial is visible to whoever observes the incremented ticket (acquire side below)
    unsigned ticket;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(p.ticket) : "memory");
    s_last = ticket == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last) {
    // acquire: thread 0's acq_rel atomic observed every other CTA's release; the block barrier above extends that
    // order to the whole CTA, and the loads below go to L2 (ld.cg), so no further fence is needed
    const int n = (int)gridDim.x;
    const float4* parts = reinterpret_cast<const float4*>(p.partials);
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    for (int base = 0; base < n; base += NW * 32 * 8) {
      float4 q[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = base + u * (NW * 32) + tid;
        q[u] = i < n ? __ldcg(parts + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) a0 += (double)q[u].x, a1 += (double)q[u].y, a2 += (double)q[u].z, a3 += (double)q[u].w;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 += __shfl_xor_sync(FULL, a0, o);
      a1 += __shfl_xor_sync(FULL, a1, o);
      a2 += __shfl_xor_sync(FULL, a2, o);
      a3 += __shfl_xor_sync(FULL, a3, o);
    }
    if (lane == 0) s_dred[0][warp] = a0, s_dred[1][warp] = a1, s_dred[2][warp] = a2, s_dred[3][warp] = a3;
    __syncthreads();
    if (tid == 0) {
      double rr[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) rr[q] = (s_dred[q][0] + s_dred[q][1]) + (s_dred[q][2] + s_dred[q][3]);
      const float pi = (float)rr[0], vf = (float)rr[1], ent = (float)rr[2];
      p.losses[0] = pi + vf * p.vf_coeff + ent * p.ent_coeff;      // impala.py:78-79
      p.losses[1] = pi;
      p.losses[2] = vf;
      p.losses[3] = ent;
      p.losses[4] = (float)(rr[3] / ((double)T * (double)B));
      *p.ticket = 0u;
    }
  }
  if (tid == 0) tma_store_wait_read();   // the shared-memory rows must outlive the bulk reads
}

static int g_vtrace_path = 0;    // rl_debug_set_vtrace_path: 0 = default (v8 where eligible, else v4), 4 = v4 always,
                                 // 8 = v8 without / 9 = v8 with programmatic dependent launch
constexpr bool kK1PdlDefault = false;
static bool k1_pdl() { return g_vtrace_path == 9 || (g_vtrace_path == 0 && kK1PdlDefault); }
// L2 promotion of the logits tensor maps: 1 = 128 B (default), 2 = 256 B (mode 10), 0 = none (mode 11)
static int k1_l2_promo() { return g_vtrace_path == 10 ? 2 : (g_vtrace_path == 11 ? 0 : 1); }

template <int A_>
static bool try_launch_v8(const VtraceLossArgs& a, const float* tl, const float* bl, float* dl, cudaStream_t st) {
  if constexpr (A_ >= 2 && (A_ & 1) == 0 && A_ <= 18) {
    constexpr int CW = 4;
    const int T = a.T, B = a.B;
    if (B % CW != 0 || T > kV8MaxT || T < 2 || a.act64) return false;
    if (!aligned16(a.actions) || !aligned16(a.rewards) || !aligned16(a.values) || !aligned16(a.d_values)) return false;
    if ((reinterpret_cast<uintptr_t>(a.dones) & 3u) != 0) return false;
    const int R1 = T < kV8Rows ? T : kV8Rows, R0 = T - R1;
    alignas(64) V8Maps maps;
    const char* err = nullptr;
    const uint64_t pitch = (uint64_t)B * A_ * sizeof(float);
    CUtensorMap* dst[3] = {maps.tl, maps.bl, maps.dl};
    const float* bases[3] = {tl, bl, dl};
    for (int i = 0; i < 3; ++i) {
      if (cached_tensor_map_2d_f32(&dst[i][1], bases[i], (uint64_t)B * A_, (uint64_t)T, pitch, CW * A_, R1, &err, false,
                                   k1_l2_promo()))
        return false;
      if (cached_tensor_map_2d_f32(&dst[i][0], bases[i], (uint64_t)B * A_, (uint64_t)T, pitch, CW * A_, R0 > 0 ? R0 : R1, &err,
                                   false, k1_l2_promo()))
        return false;
    }
    const uint64_t spitch = (uint64_t)B * 4;
    if (cached_tensor_map_2d_f32(&maps.act, a.actions, (uint64_t)B, (uint64_t)T, spitch, CW, T, &err, true) ||
        cached_tensor_map_2d_f32(&maps.rew, a.rewards, (uint64_t)B, (uint64_t)T, spitch, CW, T, &err) ||
        cached_tensor_map_2d_f32(&maps.val, a.values, (uint64_t)B, (uint64_t)T, spitch, CW, T, &err) ||
        cached_tensor_map_2d_f32(&maps.dval, a.d_values, (uint64_t)B, (uint64_t)T, spitch, CW, T, &err))
      return false;
    const size_t tile = ((size_t)T * CW * A_ * 4 + 127) & ~(size_t)127;
    const size_t sc = ((size_t)T * CW * 4 + 127) & ~(size_t)127;
    static bool attr_done = false;
    if (!attr_done) {
      RL_SMEM_OPTIN(vtrace_loss_v8_kernel<A_>);
      cudaFuncSetAttribute(vtrace_loss_v8_kernel<A_>, cudaFuncAttributePreferredSharedMemoryCarveout,
                           cudaSharedmemCarveoutMaxShared);
      attr_done = true;
    }
    // programmatic dependent launch: the CTAs may become resident (barrier init, descriptor prefetch) while the
    // predecessor in the stream drains; griddepcontrol.wait orders every global access behind its completion
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(B / CW), cfg.blockDim = dim3(kV8Warps * 32), cfg.dynamicSmemBytes = 2 * tile + 3 * sc, cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = k1_pdl() ? 1 : 0;
    cfg.attrs = attr, cfg.numAttrs = 1;
    if (cudaLaunchKernelEx(&cfg, vtrace_loss_v8_kernel<A_>, a, maps) != cudaSuccess) return false;
    return true;
  }
  return false;
}

template <int A_>
static int launch_vtrace_loss(const VtraceLossArgs& a, int layout, bool tma, const CUtensorMap* maps, int grid,
                              size_t smem, cudaStream_t st) {
  if (layout == RL_LAYOUT_ENV_MAJOR) {
    RL_SMEM_OPTIN(vtrace_loss_kernel<A_, true, false>);
    vtrace_loss_kernel<A_, true, false><<<grid, kNT, smem, st>>>(a, maps[0], maps[1], maps[2]);
  } else if (tma) {
    RL_SMEM_OPTIN(vtrace_loss_kernel<A_, false, true>);
    cudaFuncSetAttribute(vtrace_loss_kernel<A_, false, true>, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    vtrace_loss_kernel<A_, false, true><<<grid, kNT, smem, st>>>(a, maps[0], maps[1], maps[2]);
  } else {
    RL_SMEM_OPTIN(vtrace_loss_kernel<A_, false, false>);
    vtrace_loss_kernel<A_, false, false><<<grid, kNT, smem, st>>>(a, maps[0], maps[1], maps[2]);
  }
  return 0;
}

}  // namespace rl

static bool g_disable_tma = false;
// Test / triage hook: force the cp.async tile path (1) or allow the TMA path (0).
extern "C" int rl_debug_set_tma(int disable) {
  g_disable_tma = disable != 0;
  return RL_OK;
}

// Triage hook: 0 = default (v8 where eligible, else v4), 4 = the general v4 kernel always, 8 / 9 = v8 without / with
// programmatic dependent launch.
extern "C" int rl_debug_set_vtrace_path(int mode) {
  if (mode != 0 && mode != 4 && (mode < 8 || mode > 11)) {
    rl::set_error("rl_debug_set_vtrace_path: mode %d not in {0, 4, 8, 9, 10, 11}", mode);
    return RL_ERR_BAD_ARG;
  }
  rl::g_vtrace_path = mode;
  return RL_OK;
}

extern "C" size_t rl_loss_workspace_bytes(int n_cols) {
  const size_t grid = (size_t)(n_cols > 0 ? n_cols : 1);   // >= any kernel's CTA count
  return 256 + grid * 8 * sizeof(float);
}

extern "C" int rl_vtrace_from_importance_weights(const float* blp, const float* tlp, const float* discounts,
                                                 const float* rewards, const float* values, const float* bootstrap,
                                                 int T, int B, float clip_rho, float clip_pg, float* vs, float* pg,
                                                 rl_stream_t stream) {
  RL_CHECK_ARG(blp && tlp && discounts && rewards && values && bootstrap && vs && pg, "vtrace: null pointer");
  RL_CHECK_ARG(T > 0 && B > 0, "vtrace: T=%d B=%d must be positive", T, B);
  rl::vtrace_returns_kernel<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(blp, tlp, discounts, rewards, values,
                                                                                bootstrap, T, B, clip_rho, clip_pg, vs, pg);
  RL_CHECK_LAUNCH("rl_vtrace_from_importance_weights");
  return RL_OK;
}

extern "C" int rl_vtrace_loss_fwd_bwd(const float* target_logits, const float* behaviour_logits, const void* actions,
                                      int actions_i64, const float* rewards, const uint8_t* dones, const float* values,
                                      int T, int B, int A, int layout, float gamma, float clip_rho, float clip_pg,
                                      float vf_coeff, float ent_coeff, float* losses, float* d_logits, float* d_values,
                                      float* vs_out, float* pg_adv_out, void* workspace, size_t workspace_bytes,
                                      rl_stream_t stream) {
  using namespace rl;
  RL_CHECK_ARG(target_logits && behaviour_logits && actions && rewards && dones && values && losses && d_logits &&
                   d_values && workspace,
               "vtrace_loss: null pointer");
  RL_CHECK_ARG(T >= 2 && B >= 1 && A >= 1 && A <= 1024, "vtrace_loss: bad shape T=%d B=%d A=%d (need T>=2)", T, B, A);
  RL_CHECK_ARG(layout == RL_LAYOUT_TIME_MAJOR || layout == RL_LAYOUT_ENV_MAJOR, "vtrace_loss: bad layout %d", layout);
  RL_CHECK_ARG((long long)T * B * A < (1LL << 31), "vtrace_loss: T*B*A must be < 2^31 (32-bit indexing)");
  const int grid = (B + kBW - 1) / kBW;
  if (workspace_bytes < rl_loss_workspace_bytes(B)) {
    set_error("vtrace_loss: workspace too small (%zu < %zu)", workspace_bytes, rl_loss_workspace_bytes(B));
    return RL_ERR_WORKSPACE;
  }
  // chunk of rows staged per pass: as many as fit ~30.5 KB (7 CTAs/SM), one element per thread
  const size_t row_bytes = (size_t)kBW * (2 * A + 2) * sizeof(float);
  int TC = (int)(30500 / row_bytes);
  TC = TC < 1 ? 1 : TC;
  if (TC > kNT / kBW) TC = kNT / kBW;               // one (t,b) element per thread
  if (TC >= T) TC = T; else TC &= ~3;                 // multi-chunk: keep chunk starts 16-byte aligned
  if (TC < 1) TC = 1;
  const size_t smem = 2 * (size_t)tile_bytes_padded(TC, A) + (size_t)TC * kBW * 2 * sizeof(float);
  RL_CHECK_ARG(smem <= 200 * 1024, "vtrace_loss: A=%d too large for the shared-memory tile", A);
  VtraceLossArgs a;
  a.tl = target_logits, a.bl = behaviour_logits, a.actions = actions, a.rewards = rewards, a.dones = dones;
  a.values = values, a.d_logits = d_logits, a.d_values = d_values, a.vs_out = vs_out, a.pg_out = pg_adv_out;
  a.losses = losses;
  a.ticket = reinterpret_cast<unsigned*>(workspace);
  a.partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  a.T = T, a.B = B, a.A = A, a.TC = TC, a.act64 = actions_i64;
  a.gamma = gamma, a.clip_rho = clip_rho, a.clip_pg = clip_pg, a.vf_coeff = vf_coeff, a.ent_coeff = ent_coeff;
  const bool ptr_ok = aligned16(target_logits) && aligned16(behaviour_logits) && aligned16(d_logits);
  if (layout == RL_LAYOUT_TIME_MAJOR) {
    a.vec = ptr_ok && (((long long)B * A) % 4 == 0) && ((kBW * A) % 4 == 0);
  } else {
    a.vec = ptr_ok && (((long long)T * A) % 4 == 0) && (((long long)TC * A) % 4 == 0);
  }
  // TMA tile paths: time-major, 16-byte aligned bases, row pitch a multiple of 16 bytes, box <= 256 elements
  bool tma = layout == RL_LAYOUT_TIME_MAJOR && ptr_ok && (((long long)B * A) % 4 == 0) && kBW * A <= 256 && TC <= 256 &&
             !g_disable_tma;
  cudaStream_t st = (cudaStream_t)stream;
  bool done = false;
  if (tma && g_vtrace_path != 4) {
    switch (A) {
#define RL_CASE(N) case N: done = try_launch_v8<N>(a, target_logits, behaviour_logits, d_logits, st); break;
      RL_CASE(2) RL_CASE(4) RL_CASE(6) RL_CASE(8) RL_CASE(10) RL_CASE(12) RL_CASE(14) RL_CASE(16) RL_CASE(18)
#undef RL_CASE
      default: break;
    }
  }
  if (!done) {
    alignas(64) CUtensorMap maps[3];
    memset(maps, 0, sizeof(maps));
    if (tma) {
      const char* err = nullptr;
      const uint64_t pitch = (uint64_t)B * A * sizeof(float);
      if (cached_tensor_map_2d_f32(&maps[0], target_logits, (uint64_t)B * A, (uint64_t)T, pitch, kBW * A, TC, &err) ||
          cached_tensor_map_2d_f32(&maps[1], behaviour_logits, (uint64_t)B * A, (uint64_t)T, pitch, kBW * A, TC, &err) ||
          cached_tensor_map_2d_f32(&maps[2], d_logits, (uint64_t)B * A, (uint64_t)T, pitch, kBW * A, TC, &err)) {
        tma = false;                       // fall back to the cp.async tile path
      }
    }
    switch (A) {
#define RL_CASE(N) case N: launch_vtrace_loss<N>(a, layout, tma, maps, grid, smem, st); break;
      RL_CASE(2) RL_CASE(3) RL_CASE(4) RL_CASE(5) RL_CASE(6) RL_CASE(7) RL_CASE(8) RL_CASE(9) RL_CASE(10) RL_CASE(12)
      RL_CASE(14) RL_CASE(16) RL_CASE(18)
#undef RL_CASE
      default: launch_vtrace_loss<0>(a, layout, tma, maps, grid, smem, st); break;
    }
  }
  RL_CHECK_LAUNCH("rl_vtrace_loss_fwd_bwd");
  return RL_OK;
}
