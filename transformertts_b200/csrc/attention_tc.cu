// Fused variable-length self-attention on wgmma (flash-style, never materialises the (B,H,T,T) tensors):
//   per CTA one (batch row, head, 128-query tile); two consumer warpgroups own 64 query rows each, one producer warp streams
//   64-key tiles of K and V through a two-stage TMA ring.  Per key tile and warpgroup:
//     S = Q K^T  (wgmma, fp32 accumulators in registers)  ->  online softmax on the accumulator fragment (a row lives in the
//     four lanes of a quad; exp2 domain, keys >= kv_len masked)  ->  P (bf16 hi/lo or fp16) re-packed in registers as the
//     A operand of  O += P V  (wgmma; V is read MN-major straight from the QKV buffer, no transposed copy)  ->  O rescaled
//     in registers only when a row maximum moved.
// Replaces model/layers.py:123-129,138-147 (split/merge heads) and :176-195 (ScaledDotProductAttention) of the
// reference, which materialise logits / softmax / dropout tensors of shape (B,H,T,T) in fp32.
//
// Masking semantics: the reference adds mask*(-1e9) to the logits of padded KEYS (layers.py:186-187); after the
// fp32 add every such logit equals -1e9 and its softmax weight underflows to exactly 0 whenever the row has at least
// one valid key, so skipping those keys is exact.  Rows of padded QUERIES are zeroed by the caller's row mask
// (layers.py:229,262), so they are not computed here (written as zeros).
#include <cstdlib>
#include <cuda_fp16.h>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"
#include "wgmma_sm90.cuh"

namespace ttsb {

constexpr int ATT_BQ = 128;
constexpr int ATT_BKV = 64;
constexpr int ATT_STAGES = 2;
// warps 0-7: two softmax / MMA warpgroups (query rows [64*wg, +64)), warp 8: TMA producer (warps 9-11 idle: the producer
// warpgroup hands its registers to the others with setmaxnreg)
constexpr int ATT_THREADS = 384;

// single MUFU.EX2 (no denormal fix-up code: p < 2^-126 flushes to 0, far below bf16/fp16 resolution of P)
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct MhaKParams {
  int B, T, H;
  int Tk;            // key/value rows (== T for self-attention)
  int causal;        // keys > query index are masked
  int full_queries;  // 0: query rows >= kv_len[b] are written as zeros
  int q_col0, k_col0, v_col0;
  const int* kv_len;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  int ld_out;
  float scale_log2;  // log2(e)/sqrt(dh)
};

template <int DH, bool kSplit>
struct MhaCfg {
  static constexpr int kPlanes = kSplit ? 2 : 1;
  static constexpr int Q_BYTES = ATT_BQ * DH * 2;    // DH/64 panels of [128 x 64]
  static constexpr int K_BYTES = ATT_BKV * DH * 2;   // DH/64 panels of [64 x 64]
  static constexpr int V_BYTES = DH * ATT_BKV * 2;   // DH/64 boxes of [64 keys x 64 dh] (MN-major B operand)
  static constexpr int OFF_Q = 0;
  // stage s holds K_j and V_j of every key tile j with j % ATT_STAGES == s: [K planes][V planes]
  static constexpr int STAGE_BYTES = kPlanes * (K_BYTES + V_BYTES);
  static constexpr int OFF_KV = OFF_Q + kPlanes * Q_BYTES;
  static constexpr int OFF_BAR = OFF_KV + ATT_STAGES * STAGE_BYTES;
  static constexpr int kSmemBytes = OFF_BAR + 128 + 1024;
};

// O (+)= P V for one 16-key slice: A = P in registers, B = V (MN-major)
template <int DH, bool kF16>
__device__ __forceinline__ void mma_pv(float (&o)[DH / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (kF16) {
    if constexpr (DH == 64) wgmma_rs_m64n64_f16<1>(o, a, db, 1);
    else if constexpr (DH == 128) wgmma_rs_m64n128_f16<1>(o, a, db, 1);
    else if constexpr (DH == 192) wgmma_rs_m64n192_f16<1>(o, a, db, 1);
    else wgmma_rs_m64n256_f16<1>(o, a, db, 1);
  } else {
    if constexpr (DH == 64) wgmma_rs_m64n64_bf16<1>(o, a, db, 1);
    else if constexpr (DH == 128) wgmma_rs_m64n128_bf16<1>(o, a, db, 1);
    else if constexpr (DH == 192) wgmma_rs_m64n192_bf16<1>(o, a, db, 1);
    else wgmma_rs_m64n256_bf16<1>(o, a, db, 1);
  }
}

template <int DH, bool kSplit, bool kF16>
__global__ void __launch_bounds__(ATT_THREADS, 1)
mha_tc_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
              const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl, const MhaKParams p) {
  using Cfg = MhaCfg<DH, kSplit>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* bar_q = bars + 0;
  uint64_t* kv_full = bars + 1;                 // [ATT_STAGES]
  uint64_t* kv_empty = kv_full + ATT_STAGES;    // [ATT_STAGES], one arrival per consumer warp

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * ATT_BQ;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  int len = __ldg(p.kv_len + b);
  len = len < 0 ? 0 : (len > p.Tk ? p.Tk : len);

  if (len == 0 || (!p.full_queries && q0 >= len)) {
    // whole query tile is padding (or no key at all): defined (zero) output, no tensor work
    for (int i = threadIdx.x; i < ATT_BQ * (DH / 8); i += blockDim.x) {
      const int t = q0 + i / (DH / 8);
      if (t < p.T) {
        const size_t o = ((size_t)b * p.T + t) * p.ld_out + h * DH + (i % (DH / 8)) * 8;
        st_global_v4(p.out_hi + o, 0, 0, 0, 0);
        if (p.out_lo) st_global_v4(p.out_lo + o, 0, 0, 0, 0);
      }
    }
    return;
  }
  int n_kv = (len + ATT_BKV - 1) / ATT_BKV;
  if (p.causal) n_kv = min(n_kv, (q0 + ATT_BQ + ATT_BKV - 1) / ATT_BKV);  // key tiles beyond the last query row are all masked

  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    for (int s = 0; s < ATT_STAGES; ++s) {
      mbar_init(kv_full + s, 1);
      mbar_init(kv_empty + s, 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  uint8_t* sQ = smem + Cfg::OFF_Q;

  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (warp == 8) {
      // ===================== TMA producer: warp-uniform control flow, one elected lane issues =====================
      const bool leader = elect_one();
      if (leader) {
        mbar_arrive_expect_tx(bar_q, Cfg::kPlanes * Cfg::Q_BYTES);
        for (int pn = 0; pn < DH / 64; ++pn) {
          tma_load_3d(&tmQh, bar_q, sQ + pn * (ATT_BQ * 128), p.q_col0 + h * DH + pn * 64, q0, b);
          if (kSplit) tma_load_3d(&tmQl, bar_q, sQ + Cfg::Q_BYTES + pn * (ATT_BQ * 128), p.q_col0 + h * DH + pn * 64, q0, b);
        }
      }
      // K_j and V_j are [64 keys x 64 columns] boxes of the same buffer, at the K resp. V columns
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % ATT_STAGES;
        mbar_wait(kv_empty + s, ((j / ATT_STAGES) & 1) ^ 1);
        uint8_t* dst = smem + Cfg::OFF_KV + s * Cfg::STAGE_BYTES;
        if (leader) {
          mbar_arrive_expect_tx(kv_full + s, Cfg::STAGE_BYTES);
          for (int pn = 0; pn < DH / 64; ++pn) {
            tma_load_3d(&tmKh, kv_full + s, dst + pn * (ATT_BKV * 128), p.k_col0 + h * DH + pn * 64, j * ATT_BKV, b);
            tma_load_3d(&tmKh, kv_full + s, dst + Cfg::kPlanes * Cfg::K_BYTES + pn * (ATT_BKV * 128), p.v_col0 + h * DH + pn * 64,
                        j * ATT_BKV, b);
            if (kSplit) {
              tma_load_3d(&tmKl, kv_full + s, dst + Cfg::K_BYTES + pn * (ATT_BKV * 128), p.k_col0 + h * DH + pn * 64, j * ATT_BKV, b);
              tma_load_3d(&tmKl, kv_full + s, dst + 2 * Cfg::K_BYTES + Cfg::V_BYTES + pn * (ATT_BKV * 128),
                          p.v_col0 + h * DH + pn * 64, j * ATT_BKV, b);
            }
          }
        }
      }
    }
  } else {
    // ===================== softmax / MMA warpgroups =====================
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int wq = warp & 3;
    const int r0 = wg * 64 + 16 * wq + (lane >> 2);          // this thread's rows r0 and r0 + 8 of the tile
    const int tq[2] = {q0 + r0, q0 + r0 + 8};
    const int cq = 2 * (lane & 3);                            // its columns 8i + cq + {0, 1} of every accumulator
    float o[DH / 2];
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait(bar_q, 0);
    const uint32_t sq = smem_u32(sQ) + wg * (64 * 128);
    for (int j = 0; j < n_kv; ++j) {
      const int st = j % ATT_STAGES;
      mbar_wait(kv_full + st, (j / ATT_STAGES) & 1);
      const uint32_t sk = smem_u32(smem + Cfg::OFF_KV + st * Cfg::STAGE_BYTES);
      const uint32_t sv = sk + Cfg::kPlanes * Cfg::K_BYTES;
      // ---- S = Q K_j^T (raw scores: the running max is kept in raw units, the softmax scale is folded into one FFMA per
      //      element: p = exp2(s * scale_log2 - m * scale_log2))
      float s[32];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DH / 16; ++kk) {
        const uint64_t da = make_smem_desc_sw128(sq + (kk / 4) * (ATT_BQ * 128)) + 2 * (kk % 4);
        const uint64_t db = make_smem_desc_sw128(sk + (kk / 4) * (ATT_BKV * 128)) + 2 * (kk % 4);
        if (kF16) wgmma_ss_m64n64_f16<0, 0>(s, da, db, kk != 0);
        else wgmma_ss_m64n64_bf16<0, 0>(s, da, db, kk != 0);
      }
      if (kSplit) {
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) {
          const uint64_t da_lo = make_smem_desc_sw128(sq + Cfg::Q_BYTES + (kk / 4) * (ATT_BQ * 128)) + 2 * (kk % 4);
          const uint64_t da_hi = make_smem_desc_sw128(sq + (kk / 4) * (ATT_BQ * 128)) + 2 * (kk % 4);
          const uint64_t db_hi = make_smem_desc_sw128(sk + (kk / 4) * (ATT_BKV * 128)) + 2 * (kk % 4);
          const uint64_t db_lo = make_smem_desc_sw128(sk + Cfg::K_BYTES + (kk / 4) * (ATT_BKV * 128)) + 2 * (kk % 4);
          wgmma_ss_m64n64_bf16<0, 0>(s, da_lo, db_hi, 1);
          wgmma_ss_m64n64_bf16<0, 0>(s, da_hi, db_lo, 1);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      // ---- masks: padded keys (only the last key tile can hold them) and the look-ahead mask
      const int k0 = j * ATT_BKV + cq;
      if ((j + 1) * ATT_BKV > len) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (k0 + 8 * (i >> 2) + (i & 1) >= len) s[i] = -INFINITY;
      }
      if (p.causal && (j + 1) * ATT_BKV - 1 > q0) {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (k0 + 8 * (i >> 2) + (i & 1) > tq[(i >> 1) & 1]) s[i] = -INFINITY;
      }
      float alpha[2];
      float psum[2] = {0.f, 0.f};
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * rr], s[4 * i + 2 * rr + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        // lazy running max: the reference point only moves when the row max grew by more than 2^8 (in exponent units), so
        // P stays <= 256 (exact range for fp16/bf16, fp32 accumulation) and the O rescale below becomes rare.  l and O
        // use the same reference, so the final O / l is unchanged.
        const float m_cand = fmaxf(m[rr], mx);
        const bool grow = (m_cand - m[rr]) * p.scale_log2 > 8.f;        // first tile: m = -inf -> true
        const float m_new = grow ? m_cand : m[rr];
        alpha[rr] = grow ? fast_exp2((m[rr] - m_new) * p.scale_log2) : 1.f;  // first tile: exp2(-inf) = 0
        const float neg_m = -m_new * p.scale_log2;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s[4 * i + 2 * rr] = fast_exp2(fmaf(s[4 * i + 2 * rr], p.scale_log2, neg_m));
          s[4 * i + 2 * rr + 1] = fast_exp2(fmaf(s[4 * i + 2 * rr + 1], p.scale_log2, neg_m));
          psum[rr] += s[4 * i + 2 * rr] + s[4 * i + 2 * rr + 1];
        }
        l[rr] = l[rr] * alpha[rr] + psum[rr];   // partial sum over this thread's columns; the quad is summed at the end
        m[rr] = m_new;
      }
      if (__any_sync(0xffffffffu, alpha[0] != 1.f || alpha[1] != 1.f)) {
#pragma unroll
        for (int i = 0; i < DH / 8; ++i) {
          o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
          o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
        }
      }
      // ---- P as the A operand: the fragment of keys [16kk, 16kk + 16) is s[8kk .. 8kk + 8) re-packed pairwise
      uint32_t phi[4][4], plo[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float x0 = s[8 * kk + 2 * i], x1 = s[8 * kk + 2 * i + 1];
          if (kF16) {
            const __half2 hh = __floats2half2_rn(x0, x1);
            phi[kk][i] = *reinterpret_cast<const uint32_t*>(&hh);
          } else {
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(x0, h0, l0);
            split_bf16(x1, h1, l1);
            phi[kk][i] = pack_bf16(h0, h1);
            plo[kk][i] = pack_bf16(l0, l1);
          }
        }
      }
      // ---- O += P V_j
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < ATT_BKV / 16; ++kk) {
        const uint64_t dv = make_smem_desc_mn_sw128(sv, ATT_BKV * 128) + 128 * kk;   // 16 keys = 2048 B
        mma_pv<DH, kF16>(o, phi[kk], dv);
        if (kSplit) {
          const uint64_t dv_lo = make_smem_desc_mn_sw128(sv + Cfg::V_BYTES, ATT_BKV * 128) + 128 * kk;
          mma_pv<DH, kF16>(o, plo[kk], dv);
          mma_pv<DH, kF16>(o, phi[kk], dv_lo);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(kv_empty + st);
    }
    // ---- epilogue: O / l -> bf16 hi/lo at columns [h*DH, (h+1)*DH)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      l[rr] += __shfl_xor_sync(0xffffffffu, l[rr], 1);
      l[rr] += __shfl_xor_sync(0xffffffffu, l[rr], 2);
    }
    const float inv[2] = {l[0] > 0.f ? 1.f / l[0] : 0.f, l[1] > 0.f ? 1.f / l[1] : 0.f};
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      if (tq[rr] < p.T) {
        // the tile holding kv_len also computed its padded query rows as full rows: those are written as (+0) zeros
        const bool pad = !p.full_queries && tq[rr] >= len;
        const size_t ob = ((size_t)b * p.T + tq[rr]) * p.ld_out + h * DH + cq;
#pragma unroll
        for (int i = 0; i < DH / 8; ++i) {
          __nv_bfloat16 h0, l0, h1, l1;
          split_bf16(pad ? 0.f : o[4 * i + 2 * rr] * inv[rr], h0, l0);
          split_bf16(pad ? 0.f : o[4 * i + 2 * rr + 1] * inv[rr], h1, l1);
          *reinterpret_cast<uint32_t*>(p.out_hi + ob + 8 * i) = pack_bf16(h0, h1);
          if (p.out_lo) *reinterpret_cast<uint32_t*>(p.out_lo + ob + 8 * i) = pack_bf16(l0, l1);
        }
      }
    }
  }
  __syncthreads();
}

// ----------------------------------------------------------------------------------------------------
// SIMT bring-up kernel (one block per (b,h,query)); also produces the reference-exact attention weights
// of one batch row on request (padded keys get logit -1e9 exactly as layers.py:186-187).
// ----------------------------------------------------------------------------------------------------
struct MhaSimtPtrs {
  const __nv_bfloat16* qk_hi;
  const __nv_bfloat16* qk_lo;
  int ld_qk;
  const __nv_bfloat16* kv_hi;  // == qk_hi for self-attention
  const __nv_bfloat16* kv_lo;
  int ld_kv;
  int dh;
  int f16;           // operands hold IEEE fp16 bit patterns
  float scale;       // 1/sqrt(dh)
  float* weights;    // (H,T,Tk), (B,H,T,Tk) with weights_all, or null
  int weights_b;
  int weights_all;
  int weights_only;  // 1: only fill weights (for batch row weights_b, or every row with weights_all)
};

__device__ __forceinline__ float ld_split(const __nv_bfloat16* hi, const __nv_bfloat16* lo, size_t i, int f16 = 0) {
  if (f16) return __half2float(reinterpret_cast<const __half*>(hi)[i]);
  float v = __bfloat162float(hi[i]);
  if (lo) v += __bfloat162float(lo[i]);
  return v;
}

__global__ void mha_simt_kernel(const MhaKParams p, const MhaSimtPtrs q) {
  const int tq = blockIdx.x, h = blockIdx.y;
  const int b = (q.weights_only && !q.weights_all) ? q.weights_b : blockIdx.z;
  extern __shared__ float sm[];  // Tk logits + dh query + scratch
  float* logit = sm;
  float* qv = sm + p.Tk;
  __shared__ float red[32];
  const int len = min(max(p.kv_len[b], 0), p.Tk);
  const size_t qrow = ((size_t)b * p.T + tq) * q.ld_qk;
  for (int c = threadIdx.x; c < q.dh; c += blockDim.x) qv[c] = ld_split(q.qk_hi, q.qk_lo, qrow + p.q_col0 + h * q.dh + c, q.f16);
  __syncthreads();
  for (int tk = threadIdx.x; tk < p.Tk; tk += blockDim.x) {
    const size_t krow = ((size_t)b * p.Tk + tk) * q.ld_kv + p.k_col0 + h * q.dh;
    float acc = 0.f;
    for (int c = 0; c < q.dh; ++c) acc = fmaf(qv[c], ld_split(q.kv_hi, q.kv_lo, krow + c, q.f16), acc);
    acc = acc * q.scale;
    // reference: logits += mask * -1e9 with mask = max(padding, look-ahead) in {0,1} (models.py:136-138, layers.py:186-187)
    if (tk >= len || (p.causal && tk > tq)) acc += -1e9f;
    logit[tk] = acc;
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int tk = threadIdx.x; tk < p.Tk; tk += blockDim.x) mx = fmaxf(mx, logit[tk]);
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int tk = threadIdx.x; tk < p.Tk; tk += blockDim.x) {
    const float e = expf(logit[tk] - mx);
    logit[tk] = e;
    sum += e;
  }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) sum += red[w];
  const float inv = 1.f / sum;
  if (q.weights && (q.weights_all || b == q.weights_b)) {
    float* wrow = q.weights + (((size_t)(q.weights_all ? b : 0) * p.H + h) * p.T + tq) * p.Tk;
    for (int tk = threadIdx.x; tk < p.Tk; tk += blockDim.x) wrow[tk] = logit[tk] * inv;
  }
  if (q.weights_only) return;
  const bool pad = !p.full_queries && tq >= len;   // padded query row: zeros (its weights above are still the reference's)
  for (int c = threadIdx.x; c < q.dh; c += blockDim.x) {
    const size_t vcol = (size_t)p.v_col0 + h * q.dh + c;
    float acc = 0.f;
    if (!pad)
      for (int tk = 0; tk < p.Tk; ++tk)
        acc = fmaf(logit[tk], ld_split(q.kv_hi, q.kv_lo, ((size_t)b * p.Tk + tk) * q.ld_kv + vcol, q.f16), acc);
    acc *= inv;
    __nv_bfloat16 hi, lo;
    split_bf16(acc, hi, lo);
    const size_t o = ((size_t)b * p.T + tq) * p.ld_out + h * q.dh + c;
    p.out_hi[o] = hi;
    if (p.out_lo) p.out_lo[o] = lo;
  }
}

// ----------------------------------------------------------------------------------------------------
// Attention weights as a model output (reference-exact fp32: logits + mask * -1e9, softmax; layers.py:176-195).
// Block = 32 queries of one (batch row, head); key tiles of 32 rows are staged through shared memory as fp32
// (hi + lo recombined), lane = key, each warp owns 4 queries.  Three light passes over the (L2-resident) output row:
// logits + running max, exp + sum, scale.  Row stride DH + 4 floats keeps the 128-bit shared loads conflict-free.
// ----------------------------------------------------------------------------------------------------
constexpr int AW_Q = 32;   // queries per block
constexpr int AW_K = 32;   // keys per staged tile

__global__ void __launch_bounds__(256) mha_weights_kernel(const MhaKParams p, const MhaSimtPtrs q) {
  extern __shared__ float aw_sm[];
  const int dh = q.dh;
  const int kst = dh + 4;
  float* Qs = aw_sm;                 // [AW_Q][dh]
  float* Ks = aw_sm + AW_Q * dh;     // [AW_K][dh + 4]
  const int q0 = blockIdx.x * AW_Q, h = blockIdx.y;
  const int b = q.weights_all ? blockIdx.z : q.weights_b;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int len = min(max(p.kv_len[b], 0), p.Tk);
  for (int i = threadIdx.x; i < AW_Q * dh; i += blockDim.x) {
    const int r = i / dh, c = i - r * dh;
    const int tq = q0 + r;
    Qs[i] = tq < p.T ? ld_split(q.qk_hi, q.qk_lo, ((size_t)b * p.T + tq) * q.ld_qk + p.q_col0 + h * dh + c, q.f16) : 0.f;
  }
  float* wbase = q.weights + ((size_t)(q.weights_all ? b : 0) * p.H + h) * (size_t)p.T * p.Tk;
  float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  const int n_tiles = (p.Tk + AW_K - 1) / AW_K;
  for (int kt = 0; kt < n_tiles; ++kt) {
    __syncthreads();  // Qs ready (first tile) / previous tile consumed
    for (int i = threadIdx.x; i < AW_K * dh; i += blockDim.x) {
      const int r = i / dh, c = i - r * dh;
      const int tk = kt * AW_K + r;
      Ks[r * kst + c] = tk < p.Tk ? ld_split(q.kv_hi, q.kv_lo, ((size_t)b * p.Tk + tk) * q.ld_kv + p.k_col0 + h * dh + c, q.f16) : 0.f;
    }
    __syncthreads();
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const float4* krow = reinterpret_cast<const float4*>(Ks + lane * kst);
#pragma unroll 2
    for (int c4 = 0; c4 < dh / 4; ++c4) {
      const float4 kv = krow[c4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 qv = reinterpret_cast<const float4*>(Qs + (warp * 4 + i) * dh)[c4];
        acc[i] = fmaf(qv.x, kv.x, acc[i]);
        acc[i] = fmaf(qv.y, kv.y, acc[i]);
        acc[i] = fmaf(qv.z, kv.z, acc[i]);
        acc[i] = fmaf(qv.w, kv.w, acc[i]);
      }
    }
    const int tk = kt * AW_K + lane;
    if (tk < p.Tk) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int tq = q0 + warp * 4 + i;
        if (tq < p.T) {
          float l = acc[i] * q.scale;
          if (tk >= len || (p.causal && tk > tq)) l += -1e9f;  // mask = max(padding, look-ahead) in {0,1}, times -1e9
          wbase[(size_t)tq * p.Tk + tk] = l;
          mx[i] = fmaxf(mx[i], l);
        }
      }
    }
  }
  // every lane re-reads only what it wrote itself: no fence needed
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int tq = q0 + warp * 4 + i;
    if (tq >= p.T) continue;   // warp-uniform
    float m = mx[i];
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float* wrow = wbase + (size_t)tq * p.Tk;
    float sum = 0.f;
    for (int tk = lane; tk < p.Tk; tk += 32) {
      const float e = expf(wrow[tk] - m);
      wrow[tk] = e;
      sum += e;
    }
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.f / sum;
    for (int tk = lane; tk < p.Tk; tk += 32) wrow[tk] *= inv;
  }
}

template <int DH, bool kSplit, bool kF16>
static int launch_tc(const ttsb_mha_args* a, const MhaKParams& p, cudaStream_t stream) {
  using Cfg = MhaCfg<DH, kSplit>;
  CUtensorMap tmQ[2], tmK[2];
  const bool cross = a->kv_hi != nullptr;
  const int Tk = cross ? a->Tk : a->T;
  const int ld_kv = cross ? a->ld_kv : a->ld_qk;
  for (int hl = 0; hl < 2; ++hl) {
    const void* qk = hl == 0 ? a->qk_hi : (kSplit ? a->qk_lo : a->qk_hi);
    const void* kv = cross ? (hl == 0 ? a->kv_hi : (kSplit ? a->kv_lo : a->kv_hi)) : qk;
    int rc = make_tmap_bf16_3d(&tmQ[hl], qk, (uint64_t)a->ld_qk, a->T, a->B, a->ld_qk, (uint64_t)a->ld_qk * a->T, 64, ATT_BQ);
    if (rc) return rc;
    rc = make_tmap_bf16_3d(&tmK[hl], kv, (uint64_t)ld_kv, Tk, a->B, ld_kv, (uint64_t)ld_kv * Tk, 64, ATT_BKV);
    if (rc) return rc;
  }
  static PerDevice<bool> attr_set;
  if (!attr_set.get()) {
    TTSB_CUDA_OK(cudaFuncSetAttribute(mha_tc_kernel<DH, kSplit, kF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set.get() = true;
  }
  dim3 grid((a->T + ATT_BQ - 1) / ATT_BQ, a->H, a->B);
  mha_tc_kernel<DH, kSplit, kF16><<<grid, ATT_THREADS, Cfg::kSmemBytes, stream>>>(tmQ[0], tmQ[1], tmK[0], tmK[1], p);
  count_launch();
  return check_cuda(cudaGetLastError(), "mha_tc_kernel launch");
}

}  // namespace ttsb

using namespace ttsb;

extern "C" int ttsb_mha_fwd(const ttsb_mha_args* a, void* stream_v) {
  if (!a) { set_last_error("ttsb_mha_fwd: args is NULL"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->B <= 0 || a->T <= 0 || a->H <= 0) { set_last_error("ttsb_mha_fwd: B,T,H must be positive"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (!a->qk_hi || !a->kv_len || !a->out_hi) { set_last_error("ttsb_mha_fwd: NULL tensor"); return TTSB_ERR_INVALID_ARGUMENT; }
  const bool split = a->precision == TTSB_PREC_BF16X3;
  const bool f16 = a->precision == TTSB_PREC_FP16;
  if (split && (!a->qk_lo || !a->out_lo)) { set_last_error("ttsb_mha_fwd: bf16x3 needs the lo planes"); return TTSB_ERR_INVALID_ARGUMENT; }
  const bool cross = a->kv_hi != nullptr;
  if (cross && (a->Tk <= 0 || a->ld_kv % 8 || (split && !a->kv_lo))) {
    set_last_error("ttsb_mha_fwd: cross-attention needs Tk > 0, ld_kv %% 8 == 0 and (bf16x3) the kv lo plane");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (cross && !a->full_queries) { set_last_error("ttsb_mha_fwd: cross-attention computes every query row (set full_queries = 1)"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->causal && cross) { set_last_error("ttsb_mha_fwd: the look-ahead mask applies to self-attention only"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->ld_qk % 8 || a->ld_out % 16 || a->q_col0 % 8 || a->k_col0 % 8 || a->v_col0 % 8) {
    set_last_error("ttsb_mha_fwd: leading dimensions / column offsets must be multiples of 8");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  // H*dh columns from each offset must lie inside their row: past ld the tensor maps read zeros and the SIMT kernel the
  // next row, both without an error
  const int64_t hd = (int64_t)a->H * a->dh;
  const int ld_k = cross ? a->ld_kv : a->ld_qk;
  if (a->dh <= 0 || a->q_col0 < 0 || a->k_col0 < 0 || a->v_col0 < 0 || a->q_col0 + hd > a->ld_qk || a->k_col0 + hd > ld_k ||
      a->v_col0 + hd > ld_k || hd > a->ld_out) {
    set_last_error("ttsb_mha_fwd: need dh > 0, column offsets >= 0, q_col0 + H*dh <= ld_qk, k_col0 / v_col0 + H*dh <= %s and H*dh <= ld_out",
                   cross ? "ld_kv" : "ld_qk");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  // checked before anything is launched: a refused call writes nothing
  if (a->weights_out && !a->weights_all && (a->weights_batch_index < 0 || a->weights_batch_index >= a->B)) {
    set_last_error("ttsb_mha_fwd: weights_batch_index out of range");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MhaKParams p{};
  p.B = a->B; p.T = a->T; p.H = a->H;
  p.Tk = cross ? a->Tk : a->T;
  p.causal = a->causal ? 1 : 0;
  p.full_queries = a->full_queries ? 1 : 0;
  p.q_col0 = a->q_col0; p.k_col0 = a->k_col0; p.v_col0 = a->v_col0; p.kv_len = a->kv_len;
  p.out_hi = static_cast<__nv_bfloat16*>(a->out_hi);
  p.out_lo = static_cast<__nv_bfloat16*>(a->out_lo);  // optional second plane of the OUTPUT (consumer may be bf16x3)
  p.ld_out = a->ld_out;
  p.scale_log2 = 1.4426950408889634f / sqrtf((float)a->dh);

  MhaSimtPtrs q{};
  q.qk_hi = static_cast<const __nv_bfloat16*>(a->qk_hi);
  q.qk_lo = split ? static_cast<const __nv_bfloat16*>(a->qk_lo) : nullptr;
  q.ld_qk = a->ld_qk;
  q.kv_hi = cross ? static_cast<const __nv_bfloat16*>(a->kv_hi) : q.qk_hi;
  q.kv_lo = cross ? (split ? static_cast<const __nv_bfloat16*>(a->kv_lo) : nullptr) : q.qk_lo;
  q.ld_kv = cross ? a->ld_kv : a->ld_qk;
  q.dh = a->dh;
  q.scale = 1.f / sqrtf((float)a->dh);
  q.f16 = f16 ? 1 : 0;
  q.weights = a->weights_out;
  q.weights_b = a->weights_batch_index;
  q.weights_all = a->weights_all ? 1 : 0;
  const size_t simt_smem = (size_t)(p.Tk + a->dh) * sizeof(float);
  const bool need_simt = a->impl == TTSB_IMPL_SIMT;  // the weights-only pass has its own tiled kernel (any Tk)
  if (need_simt && simt_smem > 200 * 1024) { set_last_error("ttsb_mha_fwd: Tk too large for the weights / SIMT kernel"); return TTSB_ERR_UNSUPPORTED; }
  if (need_simt && simt_smem > 48 * 1024) {
    static PerDevice<size_t> simt_attr_pd;
    size_t& simt_attr = simt_attr_pd.get();
    if (simt_smem > simt_attr) {
      TTSB_CUDA_OK(cudaFuncSetAttribute(mha_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)simt_smem));
      simt_attr = simt_smem;
    }
  }

  if (a->impl == TTSB_IMPL_SIMT) {
    q.weights_only = 0;
    mha_simt_kernel<<<dim3(a->T, a->H, a->B), 128, simt_smem, stream>>>(p, q);
    count_launch();
    return check_cuda(cudaGetLastError(), "mha_simt_kernel launch");
  }
  int rc;
#define TTSB_MHA_DISPATCH(DH_)                                                                                      \
  (split ? launch_tc<DH_, true, false>(a, p, stream) : (f16 ? launch_tc<DH_, false, true>(a, p, stream) : launch_tc<DH_, false, false>(a, p, stream)))
#define TTSB_MHA_DISPATCH1(DH_) (f16 ? launch_tc<DH_, false, true>(a, p, stream) : launch_tc<DH_, false, false>(a, p, stream))
  if (a->dh == 128) rc = TTSB_MHA_DISPATCH(128);
  else if (a->dh == 64) rc = TTSB_MHA_DISPATCH(64);
  else if (a->dh == 192 && !split) rc = TTSB_MHA_DISPATCH1(192);
  else if (a->dh == 256 && !split) rc = TTSB_MHA_DISPATCH1(256);
  else { set_last_error("ttsb_mha_fwd: head_dim %d not supported by the tensor-core kernel (64, 128; 192, 256 in single-pass modes)", a->dh); return TTSB_ERR_UNSUPPORTED; }
#undef TTSB_MHA_DISPATCH
#undef TTSB_MHA_DISPATCH1
  if (rc) return rc;
  if (a->weights_out) {
    q.weights_only = 1;
    const size_t aw_smem = (size_t)(AW_Q * a->dh + AW_K * (a->dh + 4)) * sizeof(float);
    static PerDevice<size_t> aw_attr_pd;
    size_t& aw_attr = aw_attr_pd.get();
    if (aw_smem > 48 * 1024 && aw_smem > aw_attr) {
      TTSB_CUDA_OK(cudaFuncSetAttribute(mha_weights_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)aw_smem));
      aw_attr = aw_smem;
    }
    mha_weights_kernel<<<dim3((a->T + AW_Q - 1) / AW_Q, a->H, a->weights_all ? a->B : 1), 256, aw_smem, stream>>>(p, q);
    count_launch();
    return check_cuda(cudaGetLastError(), "mha weights kernel launch");
  }
  return 0;
}
