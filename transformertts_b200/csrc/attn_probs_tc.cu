// Attention probabilities of the training step in ONE kernel:  P = softmax(scale * Q K^T + key mask), P_drop = dropout(P)
// (model/layers.py:176-188: scaled_dot_product_attention up to the attention weights, and the Dropout on them at :189-191
// of the MultiHeadAttention call).  The two-kernel path (ttsb_bgemm writing fp32 logits, ttsb_softmax_fwd reading them
// back) moves 4*T*T bytes each way per (batch row, head); here the logits never leave the registers.
//
// A work item is (z = b*H + h, 128 query rows).  A softmax row spans all keys, so the logits are produced TWICE: pass 1
// sweeps the live 64-key tiles and keeps the running row maximum and sum (online rescaling), pass 2 recomputes every tile
// and writes the normalised probabilities.  The extra QK^T is cheap (contraction over dh only) next to the 8*T*T bytes of
// fp32 round trip it replaces.
//
//   warps 0-7  two wgmma warpgroups, each owning 64 query rows of the item: S = Q K^T with fp32 accumulators in
//              registers (a row lives in the four lanes of a quad), softmax / dropout on the fragment, bf16 pairs stored
//              straight from it
//   warp 8     TMA producer: Q tile of the item once (resident), K tiles (64 keys) through a ring (warps 9-11 idle: the
//              producer warpgroup hands its registers to the others with setmaxnreg)
//
// Masks follow ttsb_softmax_fwd with flags == 0: keys >= len[b] get probability exactly 0, query rows >= len[b] are written
// as zeros.  Dropout decisions come from the same stateless hash at the same element index ((z*T + m)*ld + k), so the
// backward pass (MODE 1 below, or the dS epilogue of ttsb_bgemm) regenerates them.
//
// MODE 1 of the same kernel is the backward counterpart (softmax gradient fused into the dP product, what ttsb_bgemm does
// with sm_P set): the MMA is dP = dO V^T (one pass), and dS = scale * P * (dropout(dP) - D) is formed on the fragment with
// the saved P read next to it.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"
#include "wgmma_sm90.cuh"

namespace ttsb {

constexpr int AP_BM = 128;
constexpr int AP_BN = 64;
constexpr int AP_THREADS = 384;
constexpr int AP_QBOX_BYTES = 128 * 64 * 2;         // [128 query rows x 64 k] K-major box
constexpr int AP_KBOX_BYTES = AP_BN * 64 * 2;       // [64 keys x 64 k]
constexpr int AP_MAX_STAGES = 8;
constexpr int AP_BAR_BYTES = 512;
constexpr int AP_MAX_SMEM = 227 * 1024;

struct ApParams {
  int Z, H, T, Tk, dh, kbs, nst;
  int q_col0, k_col0;     // first column of head 0 of Q / K in the (B, T, ld) activation tensor
  int m_tiles, n_tiles;   // query tiles per z, key tiles covering ld_p columns
  int ld_p;
  const int* kv_len;
  float scale_log2e;
  float drop_p;
  uint32_t seed, site;
  int two_outputs;
  __nv_bfloat16* out0;    // MODE 0: P_pre, MODE 1: dS
  __nv_bfloat16* out1;    // MODE 0: P_drop
  // MODE 1 (dS): saved probabilities (Z, T, ld_p), row statistic D (Z*T), plain scale
  const __nv_bfloat16* sm_P;
  const float* sm_D;
  float scale;
};

__device__ __forceinline__ float ap_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t ap_pack(float a, float b) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}

template <int MODE>
__global__ void __launch_bounds__(AP_THREADS, 1)
attn_probs_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const ApParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int q_bytes = p.kbs * AP_QBOX_BYTES;
  const int k_bytes = p.kbs * AP_KBOX_BYTES;
  uint8_t* q_smem = smem;
  uint8_t* k_smem = smem + q_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(k_smem + p.nst * k_bytes);
  uint64_t* q_full = bars;
  uint64_t* q_empty = bars + 1;
  uint64_t* k_full = bars + 2;
  uint64_t* k_empty = k_full + AP_MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 8);
    for (int s = 0; s < AP_MAX_STAGES; ++s) {
      mbar_init(k_full + s, 1);
      mbar_init(k_empty + s, 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int num_items = p.Z * p.m_tiles;

  // 64-key tiles of an item that are produced by MMAs: none when every query row of the tile is padding
  auto live_tiles = [&](int item, int& z, int& m0, int& len) -> int {
    z = item / p.m_tiles;
    m0 = (item % p.m_tiles) * AP_BM;
    len = min(max(__ldg(p.kv_len + z / p.H), 0), p.Tk);
    return m0 < len ? (len + AP_BN - 1) / AP_BN : 0;
  };

  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (warp == 8) {
      // ===================== TMA producer =====================
      const bool leader = elect_one();
      uint32_t jc = 0, qc = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        int z, m0, len;
        const int nkl = live_tiles(item, z, m0, len);
        if (nkl == 0) continue;
        const int b = z / p.H, h = z % p.H;
        mbar_wait_parked(q_empty, (qc & 1) ^ 1);
        if (leader) {
          mbar_arrive_expect_tx(q_full, (uint32_t)q_bytes);
          for (int kb = 0; kb < p.kbs; ++kb) tma_load_3d(&tmQ, q_full, q_smem + kb * AP_QBOX_BYTES, p.q_col0 + h * p.dh + kb * 64, m0, b);
        }
        ++qc;
        for (int job = 0; job < (MODE == 0 ? 2 : 1) * nkl; ++job) {       // probabilities: pass 1, then pass 2
          const int j = job < nkl ? job : job - nkl;
          const int stage = jc % p.nst;
          mbar_wait_parked(k_empty + stage, ((jc / p.nst) & 1) ^ 1);
          if (leader) {
            mbar_arrive_expect_tx(k_full + stage, (uint32_t)k_bytes);
            for (int kb = 0; kb < p.kbs; ++kb)
              tma_load_3d(&tmK, k_full + stage, k_smem + stage * k_bytes + kb * AP_KBOX_BYTES, p.k_col0 + h * p.dh + kb * 64, j * AP_BN, b);
          }
          ++jc;
        }
      }
    }
  } else {
    // ===================== wgmma / softmax warpgroups =====================
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int rloc = wg * 64 + 16 * (warp & 3) + (lane >> 2);   // this thread's rows rloc and rloc + 8 of the item
    const int cq = 2 * (lane & 3);                              // its columns 8i + cq + {0, 1} of every 64-key tile
    const uint32_t thresh16 = dropout_thresh(p.drop_p) >> 16;
    const float ks = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
    const float c = p.scale_log2e;
    const uint32_t hterm = dropout_hterm(p.seed, p.site, 0u);
    uint32_t jc = 0, qc = 0;
    // one 64-key tile of S = Q K^T (MODE 1: dP = dO V^T) for this warpgroup's 64 rows; releases the K stage
    auto produce = [&](float (&s)[32]) {
      const int stage = jc % p.nst;
      mbar_wait_parked(k_full + stage, (jc / p.nst) & 1);
      const uint32_t qs = smem_u32(q_smem) + wg * (64 * 128);
      const uint32_t kst = smem_u32(k_smem + stage * k_bytes);
      wgmma_fence();
      for (int kb = 0; kb < p.kbs; ++kb) {
        const uint64_t a = make_smem_desc_sw128(qs + kb * AP_QBOX_BYTES);
        const uint64_t bd = make_smem_desc_sw128(kst + kb * AP_KBOX_BYTES);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_ss_m64n64_bf16<0, 0>(s, a + 2 * kk, bd + 2 * kk, (kb | kk) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      __syncwarp();
      if (lane == 0) mbar_arrive(k_empty + stage);
      ++jc;
    };

    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      int z, m0, len;
      const int nkl = live_tiles(item, z, m0, len);
      const int m[2] = {m0 + rloc, m0 + rloc + 8};
      const bool live[2] = {m[0] < len, m[1] < len};
      const bool in_t[2] = {m[0] < p.T, m[1] < p.T};
      if (nkl > 0) mbar_wait_parked(q_full, qc & 1);
      // element offset of (row m, column 0) in the (Z, T, ld_p) layout; pair indices fit 32 bits (< 2^33 elements)
      const size_t rowoff[2] = {((size_t)z * p.T + (in_t[0] ? m[0] : 0)) * p.ld_p, ((size_t)z * p.T + (in_t[1] ? m[1] : 0)) * p.ld_p};
      const int n_out = max(p.n_tiles, nkl);   // every produced tile is consumed, also past the last column of the output
      if constexpr (MODE == 1) {
        // ---------------- dS = scale * P * (keep * dP / (1-p) - D), one pass
        const float dsum[2] = {live[0] ? __ldg(p.sm_D + (size_t)z * p.T + m[0]) : 0.f, live[1] ? __ldg(p.sm_D + (size_t)z * p.T + m[1]) : 0.f};
        const float sc = p.scale, sks = p.scale * ks;
        for (int j = 0; j < n_out; ++j) {
          float s[32];
          const bool has_mma = j < nkl;
          if (has_mma) produce(s);
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            if (!in_t[rr]) continue;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int col = j * AP_BN + 8 * i + cq;
              if (col >= p.ld_p) continue;
              float y0 = 0.f, y1 = 0.f;
              if (has_mma && live[rr] && col < len) {
                const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p.sm_P + rowoff[rr] + col));
                const float p0 = __uint_as_float(w << 16), p1 = __uint_as_float(w & 0xffff0000u);
                const uint32_t hsh = dropout_mix((uint32_t)((rowoff[rr] + col) >> 1) * DROPOUT_C1 ^ hterm);
                y0 = fmaf((hsh & 0xffffu) >= thresh16 ? p0 * sks : 0.f, s[4 * i + 2 * rr], -(p0 * sc) * dsum[rr]);
                y1 = fmaf((hsh >> 16) >= thresh16 ? p1 * sks : 0.f, s[4 * i + 2 * rr + 1], -(p1 * sc) * dsum[rr]);
                if (col + 1 >= len) y1 = 0.f;
              }
              *reinterpret_cast<uint32_t*>(p.out0 + rowoff[rr] + col) = ap_pack(y0, y1);
            }
          }
        }
      } else {
        float mx[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
        // ---------------- pass 1: running maximum and sum over the live key tiles
        for (int j = 0; j < nkl; ++j) {
          float s[32];
          produce(s);
          const int n0 = j * AP_BN + cq;
          if (j * AP_BN + AP_BN > len) {
#pragma unroll
            for (int i = 0; i < 32; ++i) s[i] = (n0 + 8 * (i >> 2) + (i & 1) < len) ? s[i] : -INFINITY;
          }
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            float cm = -INFINITY;
#pragma unroll
            for (int i = 0; i < 8; ++i) cm = fmaxf(cm, fmaxf(s[4 * i + 2 * rr], s[4 * i + 2 * rr + 1]));
            cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 1));
            cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 2));   // finite: key j*64 of a live tile is < len
            const float mnew = fmaxf(mx[rr], cm * c);
            const float neg = -mnew;
            float a0 = 0.f, a1 = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              a0 += ap_ex2(fmaf(s[4 * i + 2 * rr], c, neg));
              a1 += ap_ex2(fmaf(s[4 * i + 2 * rr + 1], c, neg));
            }
            l[rr] = fmaf(l[rr], ap_ex2(mx[rr] - mnew), a0 + a1);   // mx = -inf on the first tile: ex2(-inf) = 0
            mx[rr] = mnew;
          }
        }
        float inv[2] = {0.f, 0.f};
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          l[rr] += __shfl_xor_sync(0xffffffffu, l[rr], 1);
          l[rr] += __shfl_xor_sync(0xffffffffu, l[rr], 2);
          inv[rr] = (nkl > 0 && live[rr]) ? 1.f / l[rr] : 0.f;
          mx[rr] = live[rr] ? mx[rr] : INFINITY;      // dead query rows: ex2(x - inf) = 0
        }
        // ---------------- pass 2: recomputed logits -> probabilities (and dropped probabilities) -> bf16 pairs
        for (int j = 0; j < n_out; ++j) {
          float s[32];
          const bool has_mma = j < nkl;
          if (has_mma) produce(s);
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            if (!in_t[rr]) continue;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int col = j * AP_BN + 8 * i + cq;
              if (col >= p.ld_p) continue;
              float p0 = 0.f, p1 = 0.f;
              if (has_mma && col < len) {
                p0 = ap_ex2(fmaf(s[4 * i + 2 * rr], c, -mx[rr])) * inv[rr];
                p1 = col + 1 < len ? ap_ex2(fmaf(s[4 * i + 2 * rr + 1], c, -mx[rr])) * inv[rr] : 0.f;
              }
              *reinterpret_cast<uint32_t*>(p.out0 + rowoff[rr] + col) = ap_pack(p0, p1);
              if (p.two_outputs) {
                const uint32_t hsh = dropout_mix((uint32_t)((rowoff[rr] + col) >> 1) * DROPOUT_C1 ^ hterm);
                const float d0 = (hsh & 0xffffu) >= thresh16 ? p0 * ks : 0.f;
                const float d1 = (hsh >> 16) >= thresh16 ? p1 * ks : 0.f;
                *reinterpret_cast<uint32_t*>(p.out1 + rowoff[rr] + col) = ap_pack(d0, d1);
              }
            }
          }
        }
      }
      if (nkl > 0) {   // every MMA of this warp that reads the Q tile has completed
        __syncwarp();
        if (lane == 0) mbar_arrive(q_empty);
        ++qc;
      }
    }
  }
  __syncthreads();
}

}  // namespace ttsb

using namespace ttsb;

static int ap_ring_stages(int dh) {
  const int kbs = dh / 64;
  const int fixed = 1024 + AP_BAR_BYTES + kbs * AP_QBOX_BYTES;
  const int n = (AP_MAX_SMEM - fixed) / (kbs * AP_KBOX_BYTES);
  return n > AP_MAX_STAGES ? AP_MAX_STAGES : n;
}

extern "C" int ttsb_attn_probs_supported(int dh, int ld_p) {
  return dh > 0 && dh % 64 == 0 && dh <= 192 && ld_p > 0 && ld_p % 8 == 0 && ap_ring_stages(dh) >= 2;
}

// shared launcher: A operand = query-side rows (Q or dO), B operand = key-side rows (K or V)
template <int MODE>
static int ap_launch(const void* a, int ld_a, int a_col0, const void* bmat, int ld_b, int b_col0, int B, int H, int T, int dh, ApParams p,
                     void* out0, void* out1, int ld_p, cudaStream_t stream) {
  p.Z = B * H; p.H = H; p.T = T; p.Tk = T; p.dh = dh; p.kbs = dh / 64;
  p.q_col0 = a_col0; p.k_col0 = b_col0;
  p.m_tiles = (T + AP_BM - 1) / AP_BM;
  p.n_tiles = (ld_p + AP_BN - 1) / AP_BN;
  p.ld_p = ld_p;
  p.nst = ap_ring_stages(dh);
  p.out0 = static_cast<__nv_bfloat16*>(out0);
  p.out1 = static_cast<__nv_bfloat16*>(out1);
  const int smem_bytes = 1024 + AP_BAR_BYTES + p.kbs * AP_QBOX_BYTES + p.nst * p.kbs * AP_KBOX_BYTES;
  CUtensorMap tmQ, tmK;
  int rc = make_tmap_bf16_3d(&tmQ, a, (uint64_t)ld_a, (uint64_t)T, (uint64_t)B, (uint64_t)ld_a, (uint64_t)ld_a * T, 64, AP_BM);
  if (rc) return rc;
  rc = make_tmap_bf16_3d(&tmK, bmat, (uint64_t)ld_b, (uint64_t)T, (uint64_t)B, (uint64_t)ld_b, (uint64_t)ld_b * T, 64, AP_BN);
  if (rc) return rc;
  static PerDevice<bool> attr_set;
  if (!attr_set.get()) {
    TTSB_CUDA_OK(cudaFuncSetAttribute(attn_probs_tc_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, AP_MAX_SMEM));
    attr_set.get() = true;
  }
  const int items = p.Z * p.m_tiles;
  const int grid = items < num_sms() ? items : num_sms();
  attn_probs_tc_kernel<MODE><<<grid, AP_THREADS, smem_bytes, stream>>>(tmQ, tmK, p);
  count_launch();
  return check_cuda(cudaGetLastError(), MODE == 0 ? "attn_probs_tc_kernel<0> launch" : "attn_probs_tc_kernel<1> launch");
}

static bool ap_bad_layout(const void* t, int ld, int col0, int H, int dh) {
  return !t || ld % 8 || col0 % 8 || col0 < 0 || col0 + H * dh > ld || (reinterpret_cast<uintptr_t>(t) & 15);
}

extern "C" int ttsb_attn_probs_fwd(const void* qkv, int ld, int q_col0, int k_col0, int B, int H, int T, int dh,
                                   const int32_t* kv_len, float scale, float drop_p, uint32_t seed, uint32_t site, void* P_pre,
                                   void* P_drop, int ld_p, void* stream_v) {
  if (!qkv || !kv_len || !P_pre || !P_drop || B <= 0 || H <= 0 || T <= 0) {
    set_last_error("ttsb_attn_probs_fwd: NULL tensor or non-positive dimension");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (!ttsb_attn_probs_supported(dh, ld_p) || ld_p < T || (uint64_t)B * H * T * (uint64_t)ld_p >= (1ull << 33) ||
      ap_bad_layout(qkv, ld, q_col0, H, dh) || ap_bad_layout(qkv, ld, k_col0, H, dh) || drop_p < 0.f || drop_p >= 1.f ||
      (reinterpret_cast<uintptr_t>(P_pre) & 15) || (reinterpret_cast<uintptr_t>(P_drop) & 15)) {
    set_last_error("ttsb_attn_probs_fwd: need dh in {64,128,192}, ld_p >= T, ld_p % 8 == 0, < 2^33 probabilities, 16-byte aligned tensors and column offsets");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  ApParams p{};
  p.kv_len = kv_len;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.drop_p = drop_p; p.seed = seed; p.site = site;
  p.two_outputs = (P_drop != P_pre) ? 1 : 0;
  return ap_launch<0>(qkv, ld, q_col0, qkv, ld, k_col0, B, H, T, dh, p, P_pre, P_drop, ld_p, static_cast<cudaStream_t>(stream_v));
}

extern "C" int ttsb_attn_ds_bwd(const void* dO, int ld_do, int do_col0, const void* v, int ld_v, int v_col0, int B, int H, int T, int dh,
                                const int32_t* kv_len, const void* P_pre, const float* D, float scale, float drop_p, uint32_t seed,
                                uint32_t site, void* dS, int ld_p, void* stream_v) {
  if (!dO || !v || !kv_len || !P_pre || !D || !dS || B <= 0 || H <= 0 || T <= 0) {
    set_last_error("ttsb_attn_ds_bwd: NULL tensor or non-positive dimension");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (!ttsb_attn_probs_supported(dh, ld_p) || ld_p < T || (uint64_t)B * H * T * (uint64_t)ld_p >= (1ull << 33) ||
      ap_bad_layout(dO, ld_do, do_col0, H, dh) || ap_bad_layout(v, ld_v, v_col0, H, dh) || drop_p < 0.f || drop_p >= 1.f ||
      (reinterpret_cast<uintptr_t>(P_pre) & 15) || (reinterpret_cast<uintptr_t>(dS) & 15)) {
    set_last_error("ttsb_attn_ds_bwd: need dh in {64,128,192}, ld_p >= T, ld_p % 8 == 0, < 2^33 probabilities, 16-byte aligned tensors and column offsets");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  ApParams p{};
  p.kv_len = kv_len;
  p.scale = scale;
  p.drop_p = drop_p; p.seed = seed; p.site = site;
  p.sm_P = static_cast<const __nv_bfloat16*>(P_pre);
  p.sm_D = D;
  return ap_launch<1>(dO, ld_do, do_col0, v, ld_v, v_col0, B, H, T, dh, p, dS, nullptr, ld_p, static_cast<cudaStream_t>(stream_v));
}

TTSB_DEFINE_SALT_SETTER(set_salt_attn_probs)
