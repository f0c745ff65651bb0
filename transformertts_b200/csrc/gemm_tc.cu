// Tensor-core GEMM family for the ForwardTransformer blocks (Dense / concat-projection / Conv1D 'same') on the pipeline of
// gemm_pipeline.cuh: the producer reads activations through 3-D maps over (C,T,B) (OOB rows = 'same' zero padding), and
// the thread-per-row epilogue fuses bias / ReLU / residual / LayerNorm / row mask and writes fp32 + bf16 hi/lo (or fp16)
// copies for the next GEMM / the attention kernel.
//
// Replaces, in the reference (TF2/Keras ops): model/layers.py:134-136,149 (q/k/v + concat projection),
// :93-94 (FFN), :19-26,36-40 (Conv1D stack + residual LayerNorm), :498-524 (predictor convs), model/models.py:422.
//
// Precision modes: TTSB_PREC_BF16 (one product) and TTSB_PREC_BF16X3 (A_hi*W_hi + A_lo*W_hi + A_hi*W_lo), the
// latter gives fp32-class products (needed for the 1e-3 mel parity gate) at 3x the tensor-core work.
#include <cuda_fp16.h>

#include "../../include/ttsb.h"
#include "gemm_pipeline.cuh"

namespace ttsb {

struct GemmKParams {
  int B, T, N, block_n, n_tiles, tiles_per_row, num_tiles;
  int tile_begin;  // this launch covers work items [tile_begin, num_tiles)
  int num_seg;
  int seg_src[4], seg_shift[4], seg_kblocks[4];
  const float* bias;
  int relu;
  const float* residual;
  int ld_res;
  const __nv_bfloat16* res_hi;  // LayerNorm epilogue: residual = hi + lo (bf16 pair) when `residual` is NULL
  const __nv_bfloat16* res_lo;
  const float* gamma;
  const float* beta;
  float eps;
  const int* row_len;
  float* out_f32;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  int ld_out;
  float* out_preln;  // optional fp32 (B,T,ld_out): the pre-LayerNorm value (saved for the backward pass)
  float drop_pre_p, drop_post_p;  // training dropout: on the GEMM output before the residual add / on the LayerNorm output
  uint32_t drop_pre_site, drop_post_site, drop_seed;
  int h16;  // 1: out_hi receives IEEE fp16 instead of bf16 (single plane; operands of the fp16 attention)
  int staged;  // 1: 16-bit outputs go through shared memory and TMA tile stores (plain epilogue, block_n % 64 == 0)
};

// kPair: the LayerNorm GEMMs run as a cluster of two CTAs that split the N (row) dimension of one 128-row tile in halves
// (twice as many work items -> no wave-quantisation tail, small-M encoder GEMMs fill the chip) and exchange per-row
// (mean, M2) through distributed shared memory before normalising.
constexpr int PAIR_MAX_BN = 192;
template <bool kSplit, bool kPair>
struct GemmCfg {
  static constexpr int kStages = kSplit ? 2 : 4;
  static constexpr int kBTile = kPair ? PAIR_MAX_BN * GEMM_BK * 2 : B_TILE_BYTES;
  static constexpr int kStageBytes = (kSplit ? 2 : 1) * (A_TILE_BYTES + kBTile);
  using Ring = GemmRing<kStages, kStageBytes>;
  static constexpr int kMaxBn = kPair ? PAIR_MAX_BN : GEMM_MAX_BN;
  static constexpr int kPitch = acc_pitch(kMaxBn);
  // the plain (non-LayerNorm) epilogue stages two planes; pair mode is LayerNorm-only
  static constexpr int kStageOutOffset = stage_out_offset(kMaxBn);
  static_assert(img_bytes(kMaxBn) <= Ring::kBytes && (kPair || kStageOutOffset + STAGE_OUT_BYTES <= Ring::kBytes), "image must fit the ring");
  static constexpr int kRedOffset = Ring::kBytes + GEMM_RING_BAR_BYTES;  // [2][2][128] floats of intra-CTA exchange
  static constexpr int kXchgOffset = kRedOffset + 2048;         // pair mode: [2 slots][128] float2 written by the peer CTA
  static constexpr int kXbarOffset = kXchgOffset + 2048;        // pair mode: 2 mbarriers
  static constexpr int kSmemBytes = kXbarOffset + 64 + 1024;    // + alignment slack
};

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_to_peer(uint32_t saddr, uint32_t peer) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(peer));
  return r;
}
__device__ __forceinline__ void st_cluster_v2(uint32_t addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(addr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0, spins = 0;
  while (!ok) {
    asm volatile(
        "{\n.reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (!ok && ++spins == 0x10000000u) asm volatile("trap;");
  }
}

// ----------------------------------------------------------------------------------------------------
// Epilogue for one 128 x block_n accumulator tile (image rows in shared memory).  8 epilogue warps: warp (quarter, half)
// owns rows [32*quarter, +32) (thread = one output row) and the lower / upper half of the tile's 16-column chunks, so
// two warps per SM sub-partition interleave and hide each other's latencies.  Per-column vectors (bias, gamma, beta) are read
// as warp-uniform float4 loads (buffers are padded to n_pad by the host).
// ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ldg16(const float* __restrict__ p, float (&v)[16]) {
  const float4* q = reinterpret_cast<const float4*>(p);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 f = __ldg(q + j);
    v[4 * j] = f.x; v[4 * j + 1] = f.y; v[4 * j + 2] = f.z; v[4 * j + 3] = f.w;
  }
}

__device__ __forceinline__ void store_chunk(const GemmKParams& p, size_t orow, int col0, const float (&y)[16]) {
  const size_t o = orow * (size_t)p.ld_out + col0;
  if (p.out_f32) {
    st_global_v8f(p.out_f32 + o, y);
    st_global_v8f(p.out_f32 + o + 8, y + 8);
  }
  if (p.out_hi) {
    uint32_t h[8], l[8];
    if (p.h16) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half2 hh = __floats2half2_rn(y[2 * j], y[2 * j + 1]);
        h[j] = *reinterpret_cast<const uint32_t*>(&hh);
      }
    } else {
      pack_hi_lo(y, h, l, p.out_lo != nullptr);
    }
    st_global_v8(p.out_hi + o, h);
    if (p.out_lo && !p.h16) st_global_v8(p.out_lo + o, l);
  }
}

__device__ __forceinline__ void apply_dropout16(float (&y)[16], float p, uint32_t seed, uint32_t site, uint64_t elem0) {
  const uint32_t t16 = dropout_thresh(p) >> 16;
  const float ks = 1.f / (1.f - p);
  // elem0 is a multiple of 16 (ld_out % 16 == 0 for dropout outputs): the eight pair indices share their high word and the
  // low word cannot wrap, so the 64-bit part of the hash is done once per chunk (exact for any tensor size)
  const uint64_t pair0 = elem0 >> 1;
  const uint32_t hterm = dropout_hterm(seed, site, (uint32_t)(pair0 >> 32));
  const uint32_t x0 = (uint32_t)pair0 * DROPOUT_C1;
#pragma unroll
  for (int j = 0; j < 16; j += 2) {
    const uint32_t h = dropout_mix((x0 + (uint32_t)(j >> 1) * DROPOUT_C1) ^ hterm);
    y[j] = (h & 0xffffu) >= t16 ? y[j] * ks : 0.f;
    y[j + 1] = (h >> 16) >= t16 ? y[j + 1] * ks : 0.f;
  }
}

// exchange of per-row partial sums between the two warps that share a lane quarter
__device__ __forceinline__ float pair_sum(float part, float* red, int half, int row, int quarter) {
  red[half * GEMM_BM + row] = part;
  quarter_sync(quarter);
  return part + red[(half ^ 1) * GEMM_BM + row];
}

struct PairCtx {
  int active;          // 1: this tile's LayerNorm statistics are combined with the peer CTA's half of the row
  uint32_t peer_slot;  // shared::cluster address of the peer's exchange slot array for this tile parity
  uint32_t peer_bar;   // shared::cluster address of the peer's exchange mbarrier for this tile parity
  float2* my_slot;     // where the peer writes its (mean, M2)
  uint64_t* my_bar;
  uint32_t parity;
};

template <bool kLN>
__device__ __forceinline__ void epilogue_tile(const GemmKParams& p, float* arow, int b, int t0, int n0, int row, int half,
                                              int quarter, float* red /* [2][2][128] */,
                                              const PairCtx& px, uint8_t* stage_out, const CUtensorMap* tmOh, const CUtensorMap* tmOl,
                                              uint32_t& slab_ctr) {
  const int t = t0 + row;
  const bool row_ok = t < p.T;
  const bool row_keep = row_ok && (p.row_len == nullptr || t < __ldg(p.row_len + b));
  const size_t orow = (size_t)b * p.T + (row_ok ? t : 0);
  const int ncols = min(p.block_n, p.N - n0);  // logical columns in this tile
  const bool partial = ncols < p.block_n;
  const int nch = p.block_n >> 4;
  const int ch_begin = half ? (nch + 1) >> 1 : 0;
  const int ch_end = half ? nch : (nch + 1) >> 1;
  uint32_t r[16];
  float y[16], aux[16];

  if constexpr (!kLN) {
    if (p.staged) {
      // 16-bit outputs as TMA tile stores (staged_slab_begin / _end); rows >= T and columns >= N are clipped by the tensor map
      const bool issuer = half == 0 && (threadIdx.x & 31) == 0;
      const int lrow = row & 31;
      const bool two = p.out_lo != nullptr && !p.h16;
      uint8_t* box_lo = staged_slab_lo_box(stage_out, quarter);
      uint32_t qa[16], qb[16];
      for (int s0 = 0; s0 < nch; s0 += 4) {   // 64-column slab: this warp handles chunks s0 + 2*half, +1
        const int ca = s0 + 2 * half, cb = ca + 1;
        __syncwarp();
        acc_ld16(arow + (ca << 4), qa);
        acc_ld16(arow + (cb << 4), qb);
        uint8_t* box_hi = staged_slab_begin(stage_out, quarter, issuer, two, slab_ctr);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int c0 = (u ? cb : ca) << 4;
          if (p.bias) ldg16(p.bias + n0 + c0, aux);
#pragma unroll
          for (int j = 0; j < 16; ++j) y[j] = __uint_as_float(u ? qb[j] : qa[j]);
          if (p.bias) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] += aux[j];
          }
          if (p.relu) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = fmaxf(y[j], 0.f);
          }
          if (p.drop_pre_p > 0.f) apply_dropout16(y, p.drop_pre_p, p.drop_seed, p.drop_pre_site, orow * (uint64_t)p.ld_out + n0 + c0);
          if (partial) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = (c0 + j < ncols) ? y[j] : 0.f;
          }
          if (!row_keep) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = 0.f;
          }
          uint32_t h[8], l[8];
          if (p.h16) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const __half2 hh = __floats2half2_rn(y[2 * j], y[2 * j + 1]);
              h[j] = *reinterpret_cast<const uint32_t*>(&hh);
            }
          } else {
            pack_hi_lo(y, h, l, two);
          }
          st_box_chunk(box_hi, lrow, 2 * (2 * half + u), h);
          if (two) st_box_chunk(box_lo, lrow, 2 * (2 * half + u), l);
        }
        staged_slab_end(quarter, issuer, [&] {
          tma_store_3d(tmOh, box_hi, n0 + (s0 << 4), t0 + quarter * 32, b);
          if (two) tma_store_3d(tmOl, box_lo, n0 + (s0 << 4), t0 + quarter * 32, b);
        });
      }
      return;
    }
    // direct stores (fp32 outputs, residual adds, odd tile widths)
    constexpr int IN_FLIGHT = 2;
    uint32_t q[IN_FLIGHT][16];
    for (int g0 = ch_begin; g0 < ch_end; g0 += IN_FLIGHT) {
      __syncwarp();
#pragma unroll
      for (int i = 0; i < IN_FLIGHT; ++i)
        if (g0 + i < ch_end) acc_ld16(arow + ((g0 + i) << 4), q[i]);
#pragma unroll
      for (int i = 0; i < IN_FLIGHT; ++i) {
        if (g0 + i < ch_end) {   // warp-uniform
          const int c0 = (g0 + i) << 4;
          if (p.bias) ldg16(p.bias + n0 + c0, aux);
#pragma unroll
          for (int j = 0; j < 16; ++j) y[j] = __uint_as_float(q[i][j]);
          if (p.bias) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] += aux[j];
          }
          if (p.relu) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = fmaxf(y[j], 0.f);
          }
          if (p.drop_pre_p > 0.f) apply_dropout16(y, p.drop_pre_p, p.drop_seed, p.drop_pre_site, orow * (uint64_t)p.ld_out + n0 + c0);
          if (p.residual && row_ok) {
            ld_global_nc_v8f(p.residual + orow * (size_t)p.ld_res + n0 + c0, aux);
            ld_global_nc_v8f(p.residual + orow * (size_t)p.ld_res + n0 + c0 + 8, aux + 8);
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] += aux[j];
          }
          if (partial) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = (c0 + j < ncols) ? y[j] : 0.f;
          }
          if (!row_keep) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = 0.f;
          }
          if (row_ok) store_chunk(p, orow, n0 + c0, y);
        }
      }
    }
    return;
  } else {

  // ---- LayerNorm epilogue (single N tile), two passes over the accumulator image:
  //   pass 1 builds v = acc + bias (+relu) (+dropout) (+residual), parks it back in the image and accumulates SHIFTED sums
  //          s = sum(v - K), q = sum((v - K)^2) with K = the thread's first value (no cancellation: this is Welford's
  //          statistic for the thread's column range, (mean_h, M2_h) = (K + s/n_h, q - s^2/n_h));
  //   the two warps of a lane quarter (column halves) and, in pair mode, the two CTAs of the cluster combine their
  //   (mean, M2, n) with Chan's parallel formula; pass 2 normalises.  The residual row is fetched one chunk ahead of its
  //   use.
  const float inv_n = 1.f / (float)ncols;
  uint32_t r2[16];
  float res[16], res2[16];
  const bool pair_res = p.residual == nullptr && p.res_hi != nullptr;
  const bool has_res = (p.residual != nullptr || pair_res) && row_ok;
  const float* res_row = (has_res && !pair_res) ? p.residual + orow * (size_t)p.ld_res + n0 : nullptr;
  const __nv_bfloat16* res_row_hi = (has_res && pair_res) ? p.res_hi + orow * (size_t)p.ld_res + n0 : nullptr;
  const __nv_bfloat16* res_row_lo = (has_res && pair_res) ? p.res_lo + orow * (size_t)p.ld_res + n0 : nullptr;
  auto fetch = [&](int ch, uint32_t (&rr)[16], float (&rs)[16]) {
    const int c0 = ch << 4;
    acc_ld16(arow + c0, rr);
    if (has_res) {
      if (pair_res) {
        // 16 columns = 32 bytes of hi + 32 bytes of lo; x = hi + lo (bf16 -> fp32 is a 16-bit shift)
        uint32_t h[8], l[8];
        ld_global_nc_v8(res_row_hi + c0, h);
        ld_global_nc_v8(res_row_lo + c0, l);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          rs[2 * j] = __uint_as_float(h[j] << 16) + __uint_as_float(l[j] << 16);
          rs[2 * j + 1] = __uint_as_float(h[j] & 0xffff0000u) + __uint_as_float(l[j] & 0xffff0000u);
        }
      } else {
        ld_global_nc_v8f(res_row + c0, rs);
        ld_global_nc_v8f(res_row + c0 + 8, rs + 8);
      }
    }
  };
  float s_sh = 0.f, q_sh = 0.f, shiftK = 0.f;
  bool have_k = false;
  auto pass1_chunk = [&](int ch, uint32_t (&rr)[16], float (&rs)[16]) {
    const int c0 = ch << 4;
    if (p.bias) ldg16(p.bias + n0 + c0, aux);
#pragma unroll
    for (int j = 0; j < 16; ++j) y[j] = __uint_as_float(rr[j]);
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 16; ++j) y[j] += aux[j];
    }
    if (p.relu) {
#pragma unroll
      for (int j = 0; j < 16; ++j) y[j] = fmaxf(y[j], 0.f);
    }
    if (p.drop_pre_p > 0.f) apply_dropout16(y, p.drop_pre_p, p.drop_seed, p.drop_pre_site, orow * (uint64_t)p.ld_out + n0 + c0);
    if (has_res) {
#pragma unroll
      for (int j = 0; j < 16; ++j) y[j] += rs[j];
    }
    if (partial) {
#pragma unroll
      for (int j = 0; j < 16; ++j) y[j] = (c0 + j < ncols) ? y[j] : 0.f;
    }
    if (!have_k) { shiftK = y[0]; have_k = true; }   // column c0 of the first chunk is always a logical column when n_h > 0
    if (partial) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float dv = (c0 + j < ncols) ? y[j] - shiftK : 0.f;
        s_sh += dv;
        q_sh = fmaf(dv, dv, q_sh);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float dv = y[j] - shiftK;
        s_sh += dv;
        q_sh = fmaf(dv, dv, q_sh);
      }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) rr[j] = __float_as_uint(y[j]);
    if (p.out_preln && row_ok) {
      float* dst = p.out_preln + orow * (size_t)p.ld_out + n0 + c0;
      st_global_v8f(dst, y);
      st_global_v8f(dst + 8, y + 8);
    }
    acc_st16(arow + c0, rr);
  };
  __syncwarp();
  if (ch_begin < ch_end) fetch(ch_begin, r, res);
  for (int ch = ch_begin; ch < ch_end; ch += 2) {
    if (ch + 1 < ch_end) fetch(ch + 1, r2, res2);
    pass1_chunk(ch, r, res);
    if (ch + 1 < ch_end) {
      if (ch + 2 < ch_end) fetch(ch + 2, r, res);
      pass1_chunk(ch + 1, r2, res2);
    }
  }
  // (mean, M2, n) of this thread's column range, then of the CTA's columns (half 0 is always operand 'a': both warps of
  // the pair evaluate the same expression and get bit-identical statistics)
  const int n_mine = max(0, min(ncols, ch_end << 4) - (ch_begin << 4));
  const float nf = (float)n_mine;
  float mean_h = 0.f, m2_h = 0.f;
  if (n_mine > 0) {
    mean_h = shiftK + s_sh / nf;
    m2_h = fmaxf(q_sh - s_sh * s_sh / nf, 0.f);
  }
  float* red_m2 = red + 2 * GEMM_BM;
  red[half * GEMM_BM + row] = mean_h;
  red_m2[half * GEMM_BM + row] = m2_h;
  quarter_sync(quarter);
  const float mean_o = red[(half ^ 1) * GEMM_BM + row], m2_o = red_m2[(half ^ 1) * GEMM_BM + row];
  const float n_a = half == 0 ? nf : (float)(ncols - n_mine), n_b = (float)ncols - n_a;
  const float mean_a = half == 0 ? mean_h : mean_o, mean_b = half == 0 ? mean_o : mean_h;
  const float m2_a = half == 0 ? m2_h : m2_o, m2_b = half == 0 ? m2_o : m2_h;
  float mean, m2;
  if (n_b > 0.f && n_a > 0.f) {
    const float delta = mean_b - mean_a;
    mean = mean_a + delta * (n_b * inv_n);
    m2 = m2_a + m2_b + delta * delta * (n_a * n_b * inv_n);
  } else {
    mean = n_a > 0.f ? mean_a : mean_b;
    m2 = n_a > 0.f ? m2_a : m2_b;
  }
  float n_total = (float)ncols;
  if (px.active) {
    // combine with the peer CTA's half of the row (Chan et al.): exact two-pass statistics with ONE exchange
    if (half == 0) st_cluster_v2(px.peer_slot + (uint32_t)row * 8u, mean, m2);
    asm volatile("fence.acq_rel.cluster;" ::: "memory");
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive_cluster(px.peer_bar);
    mbar_wait_cluster(px.my_bar, px.parity);
    const float2 pr = px.my_slot[row];
    const float delta = mean - pr.x;
    m2 = m2 + pr.y + delta * delta * (0.5f * (float)ncols);
    mean = 0.5f * (mean + pr.x);
    n_total = 2.f * (float)ncols;
  }
  const float rstd = rsqrtf(m2 / n_total + p.eps);
  auto pass2_chunk = [&](int ch, uint32_t (&rr)[16]) {
    const int c0 = ch << 4;
    float bt[16];
    ldg16(p.gamma + n0 + c0, aux);
    ldg16(p.beta + n0 + c0, bt);
#pragma unroll
    for (int j = 0; j < 16; ++j) y[j] = (__uint_as_float(rr[j]) - mean) * rstd * aux[j] + bt[j];
    if (p.drop_post_p > 0.f) apply_dropout16(y, p.drop_post_p, p.drop_seed, p.drop_post_site, orow * (uint64_t)p.ld_out + n0 + c0);
    if (partial) {
#pragma unroll
      for (int j = 0; j < 16; ++j) y[j] = (c0 + j < ncols) ? y[j] : 0.f;
    }
    if (!row_keep) {
#pragma unroll
      for (int j = 0; j < 16; ++j) y[j] = 0.f;
    }
    if (row_ok) store_chunk(p, orow, n0 + c0, y);
  };
  __syncwarp();
  if (ch_begin < ch_end) acc_ld16(arow + (ch_begin << 4), r);
  for (int ch = ch_begin; ch < ch_end; ch += 2) {
    if (ch + 1 < ch_end) acc_ld16(arow + ((ch + 1) << 4), r2);
    pass2_chunk(ch, r);
    if (ch + 1 < ch_end) {
      if (ch + 2 < ch_end) acc_ld16(arow + ((ch + 2) << 4), r);
      pass2_chunk(ch + 1, r2);
    }
  }
  }  // kLN
}

// ----------------------------------------------------------------------------------------------------
// kernel
// ----------------------------------------------------------------------------------------------------
template <bool kSplit, bool kPair, bool kLN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA0h, const __grid_constant__ CUtensorMap tmA0l,
               const __grid_constant__ CUtensorMap tmA1h, const __grid_constant__ CUtensorMap tmA1l,
               const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
               const __grid_constant__ CUtensorMap tmOh, const __grid_constant__ CUtensorMap tmOl, const GemmKParams p) {
  using Cfg = GemmCfg<kSplit, kPair>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  typename Cfg::Ring ring(smem);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // pair mode: the two CTAs of a cluster work on the same 128-row tile, CTA rank r owns columns [r*block_n, (r+1)*block_n)
  const int cta_rank = kPair ? (int)cluster_ctarank() : 0;
  const int work_id = kPair ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int work_stride = kPair ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  uint64_t* xbar = reinterpret_cast<uint64_t*>(smem + Cfg::kXbarOffset);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA0h);
    tma_prefetch_desc(&tmWh);
    ring.init();
    for (int s = 0; s < 2; ++s)
      if (kPair) mbar_init(xbar + s, GEMM_EPI_WARPS);  // one arrival per epilogue warp of the PEER CTA
    fence_mbar_init();
  }
  __syncthreads();
  if (kPair) cluster_sync_all();  // the peer's exchange barriers are initialised before anyone arrives on them

  const uint32_t stage_tx = (kSplit ? 2u : 1u) * (uint32_t)(A_TILE_BYTES + p.block_n * GEMM_BK * 2);

  if (warp >= GEMM_EPI_WARPS) {
    setmaxnreg_dec<40>();
    if (warp > GEMM_EPI_WARPS) goto done;
    // ===================== TMA producer =====================
    const bool leader = elect_one();
    for (int tile = p.tile_begin + work_id; tile < p.num_tiles; tile += work_stride) {
      const int n_tile = kPair ? cta_rank : tile % p.n_tiles;
      const int m_tile = kPair ? tile : tile / p.n_tiles;
      const int b = m_tile / p.tiles_per_row;
      const int t0 = (m_tile % p.tiles_per_row) * GEMM_BM;
      const int n0 = n_tile * p.block_n;
      ring.wait_image_free();
      int kglob = 0;
      for (int s = 0; s < p.num_seg; ++s) {
        const CUtensorMap* mh = p.seg_src[s] == 0 ? &tmA0h : &tmA1h;
        const CUtensorMap* ml = p.seg_src[s] == 0 ? &tmA0l : &tmA1l;
        for (int kb = 0; kb < p.seg_kblocks[s]; ++kb, ++kglob) {
          ring.produce(leader, stage_tx, [&](uint64_t* bar, uint8_t* st) {
            tma_load_3d(mh, bar, st, kb * GEMM_BK, t0 + p.seg_shift[s], b);
            tma_load_2d(&tmWh, bar, st + A_TILE_BYTES, kglob * GEMM_BK, n0);
            if (kSplit) {
              uint8_t* st2 = st + A_TILE_BYTES + Cfg::kBTile;
              tma_load_3d(ml, bar, st2, kb * GEMM_BK, t0 + p.seg_shift[s], b);
              tma_load_2d(&tmWl, bar, st2 + A_TILE_BYTES, kglob * GEMM_BK, n0);
            }
          });
        }
      }
    }
  } else {
    // ===================== two wgmma warpgroups (rows [64*wg, +64) of the tile), then the epilogue =====================
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int quarter = warp & 3;        // epilogue: rows [32*quarter, +32)
    const int half = warp >> 2;          // epilogue: which half of the tile's column chunks
    float* red_all = reinterpret_cast<float*>(smem + Cfg::kRedOffset);
    float* img = reinterpret_cast<float*>(smem);
    int iter = 0;
    float2* xslots = reinterpret_cast<float2*>(smem + Cfg::kXchgOffset);
    uint32_t slab_ctr = 0;  // staged epilogue: slabs stored so far (selects the staging box of single-plane outputs)
    int total_kb = 0;
    for (int s = 0; s < p.num_seg; ++s) total_kb += p.seg_kblocks[s];
    const int nch = (p.block_n + 63) >> 6;   // n64 products per k step; columns past block_n are computed and ignored
    for (int tile = p.tile_begin + work_id; tile < p.num_tiles; tile += work_stride, ++iter) {
      const int n_tile = kPair ? cta_rank : tile % p.n_tiles;
      const int m_tile = kPair ? tile : tile / p.n_tiles;
      const int b = m_tile / p.tiles_per_row;
      const int t0 = (m_tile % p.tiles_per_row) * GEMM_BM;
      float acc[GEMM_NCH][32];
      ring.mma_tile(total_kb, acc, [&](uint32_t st, int kb) {
        const uint32_t a_hi = st + wg * (64 * 128);
        const uint32_t b_hi = st + A_TILE_BYTES;
#pragma unroll
        for (int kk = 0; kk < GEMM_BK / 16; ++kk) {
          const uint64_t da = make_smem_desc_sw128(a_hi) + 2 * kk;
#pragma unroll
          for (int c = 0; c < GEMM_NCH; ++c)
            if (c < nch) wgmma_ss_m64n64_bf16<0, 0>(acc[c], da, make_smem_desc_sw128(b_hi + c * (64 * 128)) + 2 * kk, (kb | kk) != 0);
        }
        if (kSplit) {
          const uint32_t a_lo = st + A_TILE_BYTES + Cfg::kBTile + wg * (64 * 128);
          const uint32_t b_lo = st + 2 * A_TILE_BYTES + Cfg::kBTile;
#pragma unroll
          for (int kk = 0; kk < GEMM_BK / 16; ++kk) {
            const uint64_t da_lo = make_smem_desc_sw128(a_lo) + 2 * kk, da_hi = make_smem_desc_sw128(a_hi) + 2 * kk;
#pragma unroll
            for (int c = 0; c < GEMM_NCH; ++c) {
              if (c < nch) {
                wgmma_ss_m64n64_bf16<0, 0>(acc[c], da_lo, make_smem_desc_sw128(b_hi + c * (64 * 128)) + 2 * kk, 1);
                wgmma_ss_m64n64_bf16<0, 0>(acc[c], da_hi, make_smem_desc_sw128(b_lo + c * (64 * 128)) + 2 * kk, 1);
              }
            }
          }
        }
      });
      park_tile(img, Cfg::kPitch, wg, nch, acc);
      PairCtx px{};
      if (kPair) {
        const int slot = iter & 1;
        px.active = 1;
        px.my_slot = xslots + slot * GEMM_BM;
        px.my_bar = xbar + slot;
        px.peer_slot = map_to_peer(smem_u32(px.my_slot), (uint32_t)(cta_rank ^ 1));
        px.peer_bar = map_to_peer(smem_u32(px.my_bar), (uint32_t)(cta_rank ^ 1));
        px.parity = (uint32_t)((iter >> 1) & 1);
      }
      const int row = quarter * 32 + lane;
      epilogue_tile<kLN>(p, img + (size_t)row * Cfg::kPitch, b, t0, n_tile * p.block_n, row, half, quarter, red_all, px,
                         smem + Cfg::kStageOutOffset, &tmOh, &tmOl, slab_ctr);
      ring.release_tile(!kLN && p.staged && half == 0 && lane == 0);
    }
    Cfg::Ring::finish(!kLN && p.staged && half == 0 && lane == 0);
  }
done:
  __syncthreads();
  if (kPair) cluster_sync_all();  // keep this CTA's shared memory alive until the peer's last remote write / arrive landed
}

// ----------------------------------------------------------------------------------------------------
// SIMT bring-up kernel: same contract, plain loads, one block per output row.  Not a fast path.
// ----------------------------------------------------------------------------------------------------
struct GemmSimtPtrs {
  const __nv_bfloat16* a_hi[2];
  const __nv_bfloat16* a_lo[2];
  int lda[2];
  const __nv_bfloat16* w_hi;
  const __nv_bfloat16* w_lo;
  int k_total;
};

__global__ void gemm_simt_kernel(const GemmKParams p, const GemmSimtPtrs q) {
  const int row = blockIdx.x;
  const int b = row / p.T, t = row % p.T;
  const int n_alloc = p.n_tiles * p.block_n;
  extern __shared__ float srow[];  // n_alloc values + 2 scratch
  for (int n = threadIdx.x; n < n_alloc; n += blockDim.x) {
    float acc = 0.f;
    if (n < p.N) {
      int koff = 0;
      for (int s = 0; s < p.num_seg; ++s) {
        const int src = p.seg_src[s];
        const int ts = t + p.seg_shift[s];
        const int K = p.seg_kblocks[s] * GEMM_BK;
        if (ts >= 0 && ts < p.T) {
          const __nv_bfloat16* ah = q.a_hi[src] + ((size_t)b * p.T + ts) * q.lda[src];
          const __nv_bfloat16* al = q.a_lo[src] ? q.a_lo[src] + ((size_t)b * p.T + ts) * q.lda[src] : nullptr;
          const __nv_bfloat16* wh = q.w_hi + (size_t)n * q.k_total + koff;
          const __nv_bfloat16* wl = q.w_lo ? q.w_lo + (size_t)n * q.k_total + koff : nullptr;
          for (int k = 0; k < K; ++k) {
            const float a1 = __bfloat162float(ah[k]);
            const float w1 = __bfloat162float(wh[k]);
            acc = fmaf(a1, w1, acc);
            if (al) acc = fmaf(__bfloat162float(al[k]), w1, acc);
            if (wl) acc = fmaf(a1, __bfloat162float(wl[k]), acc);
          }
        }
        koff += K;
      }
      if (p.bias) acc += p.bias[n];
      if (p.relu) acc = fmaxf(acc, 0.f);
      if (p.residual) acc += p.residual[(size_t)row * p.ld_res + n];
    }
    srow[n] = acc;
  }
  __syncthreads();
  const bool keep = p.row_len == nullptr || t < p.row_len[b];
  float mean = 0.f, rstd = 1.f;
  if (p.gamma) {
    float* scratch = srow + n_alloc;
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int n = 0; n < p.N; ++n) s += srow[n];
      const float m = s / p.N;
      float v = 0.f;
      for (int n = 0; n < p.N; ++n) v += (srow[n] - m) * (srow[n] - m);
      scratch[0] = m;
      scratch[1] = rsqrtf(v / p.N + p.eps);
    }
    if (p.out_preln)
      for (int n = threadIdx.x; n < n_alloc; n += blockDim.x) p.out_preln[(size_t)row * p.ld_out + n] = n < p.N ? srow[n] : 0.f;
    __syncthreads();
    mean = scratch[0];
    rstd = scratch[1];
  }
  for (int n = threadIdx.x; n < n_alloc; n += blockDim.x) {
    float v = srow[n];
    if (n < p.N) {
      if (p.gamma) v = (v - mean) * rstd * p.gamma[n] + p.beta[n];
    } else {
      v = 0.f;
    }
    if (!keep) v = 0.f;
    __nv_bfloat16 hi, lo;
    split_bf16(v, hi, lo);
    if (p.h16) hi = __ushort_as_bfloat16(__half_as_ushort(__float2half_rn(v)));  // same 16-bit slot, fp16 payload
    const size_t o = (size_t)row * p.ld_out + n;
    if (p.out_f32) p.out_f32[o] = v;
    if (p.out_hi) p.out_hi[o] = hi;
    if (p.out_lo) p.out_lo[o] = lo;
  }
}

// ----------------------------------------------------------------------------------------------------
// host
// ----------------------------------------------------------------------------------------------------
template <bool kSplit, bool kPair, bool kLN>
static int launch_tc(const CUtensorMap (&tmA)[2][2], const CUtensorMap (&tmW)[2], const CUtensorMap (&tmO)[2], const GemmKParams& q,
                     int work, cudaStream_t stream) {
  return launch_pipeline<gemm_tc_kernel<kSplit, kPair, kLN>>(GemmCfg<kSplit, kPair>::kSmemBytes, work, kPair, stream,
                                                             kPair ? "gemm_tc_kernel<pair> launch" : "gemm_tc_kernel launch", tmA[0][0], tmA[0][1], tmA[1][0],
                                                             tmA[1][1], tmW[0], tmW[1], tmO[0], tmO[1], q);
}

static int validate(const ttsb_gemm_args* a, int* k_total_out) {
  if (!a) { set_last_error("ttsb_linear_fwd: args is NULL"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->B <= 0 || a->T <= 0 || a->N <= 0) { set_last_error("ttsb_linear_fwd: B,T,N must be positive"); return TTSB_ERR_INVALID_ARGUMENT; }
  const bool wide_pair = a->ln_gamma && a->block_n == a->N && a->N % 32 == 0 && a->N / 2 <= PAIR_MAX_BN;  // N up to 384 as a CTA pair
  if (a->block_n < 16 || (a->block_n > GEMM_MAX_BN && !wide_pair) || a->block_n % 16) {
    set_last_error("ttsb_linear_fwd: block_n=%d must be a multiple of 16 in [16,256]", a->block_n);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (a->num_segments < 1 || a->num_segments > 4) { set_last_error("ttsb_linear_fwd: num_segments out of range"); return TTSB_ERR_INVALID_ARGUMENT; }
  int kt = 0;
  for (int s = 0; s < a->num_segments; ++s) {
    if (a->seg_k[s] <= 0 || a->seg_k[s] % GEMM_BK) { set_last_error("ttsb_linear_fwd: seg_k must be a positive multiple of 64"); return TTSB_ERR_INVALID_ARGUMENT; }
    const int src = a->seg_src[s];
    if (src < 0 || src > 1 || !a->a_hi[src]) { set_last_error("ttsb_linear_fwd: bad segment source"); return TTSB_ERR_INVALID_ARGUMENT; }
    if (a->precision == TTSB_PREC_BF16X3 && !a->a_lo[src]) { set_last_error("ttsb_linear_fwd: bf16x3 needs a_lo"); return TTSB_ERR_INVALID_ARGUMENT; }
    if (a->lda[src] % 8 || a->a_col0[src] % 8) { set_last_error("ttsb_linear_fwd: lda/a_col0 must be multiples of 8"); return TTSB_ERR_INVALID_ARGUMENT; }
    kt += a->seg_k[s];
  }
  if (!a->w_hi || (a->precision == TTSB_PREC_BF16X3 && !a->w_lo)) { set_last_error("ttsb_linear_fwd: missing packed weights"); return TTSB_ERR_INVALID_ARGUMENT; }
  const int n_tiles = (a->N + a->block_n - 1) / a->block_n;
  if (a->ld_out < n_tiles * a->block_n || a->ld_out % 8 || ((a->out_hi || a->out_lo) && a->ld_out % 16)) {
    set_last_error("ttsb_linear_fwd: ld_out=%d must be >= %d and a multiple of 8 (16 with 16-bit outputs: 32-byte stores)", a->ld_out,
                   n_tiles * a->block_n);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (a->ln_gamma && (n_tiles != 1 || !a->ln_beta)) { set_last_error("ttsb_linear_fwd: LayerNorm epilogue needs N <= block_n and beta"); return TTSB_ERR_INVALID_ARGUMENT; }
  if ((a->residual && (a->ld_res % 8)) || (!a->residual && a->residual_hi && (a->ld_res % 16))) {
    set_last_error("ttsb_linear_fwd: ld_res must be a multiple of 8 (fp32) / 16 (bf16 pair): 32-byte loads");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (a->precision != TTSB_PREC_BF16 && a->precision != TTSB_PREC_BF16X3) { set_last_error("ttsb_linear_fwd: unknown precision"); return TTSB_ERR_INVALID_ARGUMENT; }
  *k_total_out = kt;
  return 0;
}

}  // namespace ttsb

using namespace ttsb;

extern "C" int ttsb_linear_fwd(const ttsb_gemm_args* a, void* stream_v) {
  int k_total = 0;
  int rc = validate(a, &k_total);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const bool split = a->precision == TTSB_PREC_BF16X3;

  GemmKParams p{};
  p.B = a->B; p.T = a->T; p.N = a->N; p.block_n = a->block_n;
  p.n_tiles = (a->N + a->block_n - 1) / a->block_n;
  p.tiles_per_row = (a->T + GEMM_BM - 1) / GEMM_BM;
  p.num_tiles = a->B * p.tiles_per_row * p.n_tiles;
  // LayerNorm GEMMs whose row splits into two equal halves can run as CTA pairs (see GemmCfg): a pair finishes a 128-row
  // tile in ~0.57 of the single-CTA time, so work is handed out at half-tile granularity.  The schedule with the fewest
  // (weighted) rounds wins: all single-CTA tiles, all pairs, or full waves of single-CTA tiles followed by a pair-mode
  // tail (two launches).
  const bool pair_ok = a->impl != TTSB_IMPL_SIMT && a->ln_gamma != nullptr && p.n_tiles == 1 && a->N == a->block_n &&
                       a->N % 32 == 0 && a->N / 2 <= PAIR_MAX_BN && a->N >= 64;
  const bool single_ok = a->block_n <= GEMM_MAX_BN;
  bool pair = false;
  int hybrid_full = 0;  // > 0: tiles [0, hybrid_full) single-CTA, the rest as pairs
  if (pair_ok) {
    const int t = a->B * p.tiles_per_row, sms = num_sms(), clusters = sms / 2;
    const float kPairCost = 0.57f;
    const float c_single = single_ok ? (float)((t + sms - 1) / sms) : 1e30f;
    const float c_pair = kPairCost * (float)((t + clusters - 1) / clusters);
    const int full = (t / sms) * sms, rem = t - full;
    const float c_hyb = (single_ok && full > 0 && rem > 0) ? (float)(full / sms) + kPairCost * (float)((rem + clusters - 1) / clusters) : 1e30f;
    if (c_hyb < c_single && c_hyb < c_pair) { pair = true; hybrid_full = full; }
    else pair = c_pair < c_single;
  }
  const int num_m_tiles = a->B * p.tiles_per_row;
  p.num_seg = a->num_segments;
  int src_k[2] = {0, 0};
  for (int s = 0; s < a->num_segments; ++s) {
    p.seg_src[s] = a->seg_src[s];
    p.seg_shift[s] = a->seg_shift[s];
    p.seg_kblocks[s] = a->seg_k[s] / GEMM_BK;
    if (a->seg_k[s] > src_k[a->seg_src[s]]) src_k[a->seg_src[s]] = a->seg_k[s];
  }
  p.bias = a->bias; p.relu = a->relu; p.residual = a->residual; p.ld_res = a->ld_res;
  p.res_hi = static_cast<const __nv_bfloat16*>(a->residual_hi);
  p.res_lo = static_cast<const __nv_bfloat16*>(a->residual_lo);
  if (!a->residual && (a->residual_hi || a->residual_lo)) {
    if (!a->residual_hi || !a->residual_lo || !a->ln_gamma || a->impl == TTSB_IMPL_SIMT) {
      set_last_error("ttsb_linear_fwd: a bf16 hi/lo residual needs both planes and the tensor-core LayerNorm epilogue");
      return TTSB_ERR_INVALID_ARGUMENT;
    }
  }
  p.gamma = a->ln_gamma; p.beta = a->ln_beta; p.eps = a->ln_eps; p.row_len = a->row_len;
  p.out_f32 = a->out_f32;
  p.out_hi = static_cast<__nv_bfloat16*>(a->out_hi);
  p.out_lo = split ? static_cast<__nv_bfloat16*>(a->out_lo) : nullptr;
  p.ld_out = a->ld_out;
  p.h16 = a->out_fp16 ? 1 : 0;
  p.out_preln = a->out_preln;
  p.drop_pre_p = a->drop_pre_p; p.drop_post_p = a->drop_post_p;
  p.drop_pre_site = a->drop_pre_site; p.drop_post_site = a->drop_post_site; p.drop_seed = a->drop_seed;
  if (a->drop_pre_p < 0.f || a->drop_pre_p >= 1.f || a->drop_post_p < 0.f || a->drop_post_p >= 1.f) {
    set_last_error("ttsb_linear_fwd: dropout rates must be in [0,1)");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if ((a->drop_pre_p > 0.f || a->drop_post_p > 0.f) && a->impl == TTSB_IMPL_SIMT) {
    set_last_error("ttsb_linear_fwd: dropout is only implemented in the tensor-core kernel");
    return TTSB_ERR_UNSUPPORTED;
  }
  if (p.h16) p.out_lo = nullptr;

  if (a->impl == TTSB_IMPL_SIMT) {
    GemmSimtPtrs q{};
    for (int i = 0; i < 2; ++i) {
      q.a_hi[i] = a->a_hi[i] ? static_cast<const __nv_bfloat16*>(a->a_hi[i]) + a->a_col0[i] : nullptr;
      q.a_lo[i] = (split && a->a_lo[i]) ? static_cast<const __nv_bfloat16*>(a->a_lo[i]) + a->a_col0[i] : nullptr;
      q.lda[i] = a->lda[i];
    }
    q.w_hi = static_cast<const __nv_bfloat16*>(a->w_hi);
    q.w_lo = split ? static_cast<const __nv_bfloat16*>(a->w_lo) : nullptr;
    q.k_total = k_total;
    const int n_alloc = p.n_tiles * p.block_n;
    gemm_simt_kernel<<<a->B * a->T, 256, (n_alloc + 2) * sizeof(float), stream>>>(p, q);
    count_launch();
    return check_cuda(cudaGetLastError(), "gemm_simt_kernel launch");
  }

  // tensor maps: activations as (C, T, B) boxes of (64, 128, 1); weights as (K_total, N_pad) boxes of (64, block_n)
  CUtensorMap tmA[2][2];
  for (int i = 0; i < 2; ++i) {
    const int use = a->a_hi[i] ? i : 0;  // unused slots alias source 0 so the kernel params stay valid
    const int kext = src_k[use] > 0 ? src_k[use] : GEMM_BK;
    for (int h = 0; h < 2; ++h) {
      const void* base = h == 0 ? a->a_hi[use] : (split ? a->a_lo[use] : a->a_hi[use]);
      rc = make_tmap_bf16_3d(&tmA[i][h], static_cast<const __nv_bfloat16*>(base) + a->a_col0[use], kext, a->T, a->B,
                             (uint64_t)a->lda[use], (uint64_t)a->lda[use] * a->T, GEMM_BK, GEMM_BM);
      if (rc) return rc;
    }
  }
  auto launch = [&](bool as_pair, int tile_begin, int tile_end) -> int {
    GemmKParams q = p;
    if (as_pair) {
      q.block_n = a->N / 2;
      q.n_tiles = 1;  // per work item; the two column halves belong to the two CTAs of the cluster
    }
    q.tile_begin = tile_begin;
    q.num_tiles = tile_end;
    const int work = tile_end - tile_begin;
    CUtensorMap tmW[2];
    for (int h = 0; h < 2; ++h) {
      const void* base = h == 0 ? a->w_hi : (split ? a->w_lo : a->w_hi);
      int rc2 = make_tmap_bf16_2d(&tmW[h], base, k_total, as_pair ? a->N : q.n_tiles * q.block_n, (uint64_t)k_total, GEMM_BK, q.block_n);
      if (rc2) return rc2;
    }
    // plain epilogue with 16-bit outputs only: tile stores through shared memory
    CUtensorMap tmO[2] = {tmW[0], tmW[1]};  // placeholders when the staged path is off
    q.staged = 0;
    if (!as_pair && q.gamma == nullptr && q.out_hi != nullptr && q.out_f32 == nullptr && q.out_preln == nullptr &&
        q.residual == nullptr && q.block_n % 64 == 0 && q.ld_out % 8 == 0) {
      const int width = q.n_tiles * q.block_n;
      int rc3 = make_tmap_bf16_3d(&tmO[0], q.out_hi, (uint64_t)width, (uint64_t)a->T, (uint64_t)a->B, (uint64_t)q.ld_out,
                                  (uint64_t)q.ld_out * a->T, 64, 32);
      if (rc3) return rc3;
      if (q.out_lo) {
        rc3 = make_tmap_bf16_3d(&tmO[1], q.out_lo, (uint64_t)width, (uint64_t)a->T, (uint64_t)a->B, (uint64_t)q.ld_out,
                                (uint64_t)q.ld_out * a->T, 64, 32);
        if (rc3) return rc3;
      }
      q.staged = 1;
    }
    // pair mode: a cluster of two CTAs per 128-row tile.  Separate instantiations for the LayerNorm and the plain epilogue:
    // each gets its own register allocation
    if (as_pair) return split ? launch_tc<true, true, true>(tmA, tmW, tmO, q, work, stream) : launch_tc<false, true, true>(tmA, tmW, tmO, q, work, stream);
    if (q.gamma != nullptr)
      return split ? launch_tc<true, false, true>(tmA, tmW, tmO, q, work, stream) : launch_tc<false, false, true>(tmA, tmW, tmO, q, work, stream);
    return split ? launch_tc<true, false, false>(tmA, tmW, tmO, q, work, stream) : launch_tc<false, false, false>(tmA, tmW, tmO, q, work, stream);
  };
  if (pair && hybrid_full > 0) {
    rc = launch(false, 0, hybrid_full);
    if (rc) return rc;
    return launch(true, hybrid_full, num_m_tiles);
  }
  if (pair) return launch(true, 0, num_m_tiles);
  return launch(false, 0, p.num_tiles);
}

TTSB_DEFINE_SALT_SETTER(set_salt_gemm)
