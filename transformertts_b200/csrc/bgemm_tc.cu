// Batched / reduction GEMMs of the training step on wgmma (single-pass bf16, fp32 accumulate in registers), run on the
// pipeline of gemm_pipeline.cuh (4-stage ring, one [128 x 64] A and one [<=256 x 64] B tile per stage):
//
//  mode BATCHED : out[z][m][n] = alpha * sum_k A_z[m][k] * B_z[n][k]        z = (batch row b, head h)
//                 both operands come from activations (per-(b,h) B operand), e.g. S = Q K^T, O = P V, dP = dO V^T,
//                 dQ = dS K, dK = dS^T Q, dV = P^T dO of the attention forward/backward (model/layers.py:176-195 and
//                 its gradient), each operand addressed through a 3-D TMA map with per-head column/row offsets.
//  mode WGRAD   : dW[seg*Cin + c][n] += sum_b sum_t X_seg[b][t + shift_seg][c] * G[b][t][n]
//                 weight gradients of Dense / concat-Dense / Conv1D (k taps = k segments), reduction over all B*T
//                 rows split across CTAs, partial tiles added with fp32 red.global.add (Keras (K,N) layout).
//
// Operand majorness.  wgmma reads an operand either K-major (the contraction index is contiguous in memory: rows of
// 128 B hold 64 k) or MN-major (the M/N index is contiguous: rows of 128 B hold 64 m, one row per k).  Supporting both
// means NO transposed copies are ever made: P^T, dS^T, dO^T, V^T, K^T and the X^T / G^T of the weight gradients are just
// the same row-major tensors read MN-major.  An MN-major tile is fetched as ceil(rows/64) TMA boxes of [64 k x 64 mn]
// (8 KiB each, 128B swizzle) and described to the MMA with LBO = 8192 B (next 64-wide MN block), SBO = 1024 B (next 8 k).
#include <cuda_fp16.h>

#include "../../include/ttsb.h"
#include "gemm_pipeline.cuh"

namespace ttsb {

using BgRing = GemmRing<4, A_TILE_BYTES + B_TILE_BYTES>;
constexpr int BG_PITCH = acc_pitch(GEMM_MAX_BN);
constexpr int BG_STAGE_OUT_OFFSET = stage_out_offset(GEMM_MAX_BN);
static_assert(BG_STAGE_OUT_OFFSET + STAGE_OUT_BYTES <= BgRing::kBytes, "image and staging must fit the ring");
constexpr int BG_SMEM_BYTES = BgRing::kBytes + GEMM_RING_BAR_BYTES + 1024;  // + alignment slack

struct BgOperand {
  int h_col;     // added to coordinate 0 (contiguous dim) per head
  int h_row;     // added to coordinate 1 per head
  int z_batch;   // 1: coordinate 2 = z (b*H + h); 0: coordinate 2 = b
  int mn_major;  // 1: coordinate 0 runs over M/N, coordinate 1 over K
};

struct BgParams {
  int mode;  // 0 batched, 1 wgrad
  // batched
  int Z, H, M, N, K;  // per-z problem: M x N x K
  BgOperand opA, opB;
  float alpha;
  float* out_f32;
  __nv_bfloat16* out_bf16;
  int ld_out;                 // row stride (elements)
  long long out_z_stride;     // stride between z (or b when out_by_b) problems
  int out_h_col;              // column offset per head
  int out_by_b;               // 1: batch index of the output is b (heads side by side in columns)
  int out_cols;               // writable columns of one problem's row (multiple of 16)
  const int* row_len;         // optional [B]: rows m >= len[b] are written as zero
  const int* col_len;         // optional [B]: columns n >= len[b] are written as zero
  // fused softmax backward (see ttsb_bgemm_args): dS = sm_scale * P_pre * (dropout(acc) - D)
  const __nv_bfloat16* sm_P;
  const __nv_bfloat16* sm_Pdrop;  // optional: saved post-dropout probabilities (dropout decision = P_drop != 0)
  const float* sm_D;
  float sm_scale, sm_drop_p;
  uint32_t sm_seed, sm_site;
  int sm_flags;
  const int* sm_len;
  // wgrad
  int B, T, Cin, num_seg, seg_src[4], seg_shift[4], splits, b_per_split;
  float* dw;                  // fp32 (num_seg*Cin, N) accumulated with atomics
  // common
  int block_n, n_tiles, m_tiles, num_tiles;
  int staged;  // 1: bf16 output through shared staging + TMA tile stores (batched mode, block_n % 64 == 0)
};

__global__ void __launch_bounds__(GEMM_THREADS, 1)
bgemm_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO, const BgParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  BgRing ring(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA0);
    tma_prefetch_desc(&tmB);
    ring.init();
    fence_mbar_init();
  }
  __syncthreads();
  const bool a_mn = p.mode == 1 || p.opA.mn_major;
  const bool b_mn = p.mode == 1 || p.opB.mn_major;
  const int b_boxes = (p.block_n + 63) / 64;
  const uint32_t stage_tx = (uint32_t)(A_TILE_BYTES + (b_mn ? b_boxes * MN_BOX_BYTES : p.block_n * GEMM_BK * 2));
  const int t_chunks = (p.T + GEMM_BK - 1) / GEMM_BK;

  // number of k-blocks of a tile (uniform across roles)
  auto tile_kblocks = [&](int tile) -> int {
    if (p.mode == 0) return (p.K + GEMM_BK - 1) / GEMM_BK;
    const int split = tile % p.splits;
    const int b0 = split * p.b_per_split;
    const int nb = min(p.b_per_split, p.B - b0);
    return nb > 0 ? nb * t_chunks : 0;
  };

  if (warp >= GEMM_EPI_WARPS) {
    setmaxnreg_dec<40>();
    if (warp > GEMM_EPI_WARPS) goto done;
    // ===================== TMA producer =====================
    const bool leader = elect_one();
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      if (tile_kblocks(tile) == 0) continue;
      ring.wait_image_free();
      if (p.mode == 0) {
        const int n_tile = tile % p.n_tiles;
        const int m_tile = (tile / p.n_tiles) % p.m_tiles;
        const int z = tile / (p.n_tiles * p.m_tiles);
        const int b = z / p.H, h = z % p.H;
        const int m0 = m_tile * GEMM_BM, n0 = n_tile * p.block_n;
        const int kbs = (p.K + GEMM_BK - 1) / GEMM_BK;
        const int za = p.opA.z_batch ? z : b, zb = p.opB.z_batch ? z : b;
        for (int kb = 0; kb < kbs; ++kb) {
          ring.produce(leader, stage_tx, [&](uint64_t* bar, uint8_t* st) {
            if (a_mn) {
              for (int i = 0; i < GEMM_BM / 64; ++i)
                tma_load_3d(&tmA0, bar, st + i * MN_BOX_BYTES, m0 + 64 * i + h * p.opA.h_col, kb * GEMM_BK + h * p.opA.h_row, za);
            } else {
              tma_load_3d(&tmA0, bar, st, kb * GEMM_BK + h * p.opA.h_col, m0 + h * p.opA.h_row, za);
            }
            if (b_mn) {
              for (int i = 0; i < b_boxes; ++i)
                tma_load_3d(&tmB, bar, st + A_TILE_BYTES + i * MN_BOX_BYTES, n0 + 64 * i + h * p.opB.h_col,
                            kb * GEMM_BK + h * p.opB.h_row, zb);
            } else {
              tma_load_3d(&tmB, bar, st + A_TILE_BYTES, kb * GEMM_BK + h * p.opB.h_col, n0 + h * p.opB.h_row, zb);
            }
          });
        }
      } else {
        int r = tile;
        const int split = r % p.splits; r /= p.splits;
        const int n_tile = r % p.n_tiles; r /= p.n_tiles;
        const int m_tile = r % p.m_tiles; r /= p.m_tiles;
        const int seg = r;
        const CUtensorMap* mA = p.seg_src[seg] == 0 ? &tmA0 : &tmA1;
        const int c0 = m_tile * GEMM_BM, n0 = n_tile * p.block_n;
        const int b0 = split * p.b_per_split;
        const int b1 = min(b0 + p.b_per_split, p.B);
        const int shift = p.seg_shift[seg];
        for (int b = b0; b < b1; ++b) {
          for (int tc = 0; tc < t_chunks; ++tc) {
            ring.produce(leader, stage_tx, [&](uint64_t* bar, uint8_t* st) {
              for (int i = 0; i < GEMM_BM / 64; ++i)
                tma_load_3d(mA, bar, st + i * MN_BOX_BYTES, c0 + 64 * i, tc * GEMM_BK + shift, b);
              for (int i = 0; i < b_boxes; ++i)
                tma_load_3d(&tmB, bar, st + A_TILE_BYTES + i * MN_BOX_BYTES, n0 + 64 * i, tc * GEMM_BK, b);
            });
          }
        }
      }
    }
  } else {
    // ===================== two wgmma warpgroups (rows [64*wg, +64) of the tile), then the epilogue =====================
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int quarter = warp & 3;        // epilogue: rows [32*quarter, +32)
    const int half = warp >> 2;          // epilogue: which half of the tile's column chunks
    const int row = quarter * 32 + lane;
    float* img = reinterpret_cast<float*>(smem);
    float* arow = img + (size_t)row * BG_PITCH;
    const int nch = p.block_n >> 4;
    const int ch_begin = half ? (nch + 1) >> 1 : 0;
    const int ch_end = half ? nch : (nch + 1) >> 1;
    const int nmma = (p.block_n + 63) >> 6;   // n64 products per k step; columns past block_n are computed and ignored
    const uint32_t a_step = a_mn ? (16 * 128) >> 4 : 2;  // descriptor advance per 16 k
    const uint32_t b_step = b_mn ? (16 * 128) >> 4 : 2;
    uint32_t r[16];
    uint32_t slab_ctr = 0;  // staged epilogue: slabs stored so far (selects the staging box)
    // the same 64-row / 64-column block offsets hold for both majornesses: a K-major block is 64 rows of 128 B, an MN-major
    // block one [64 k x 64 mn] TMA box
    auto mma = [&](float (&d)[32], uint64_t da, uint64_t db, uint32_t accum) {
      if (a_mn) {
        if (b_mn) wgmma_ss_m64n64_bf16<1, 1>(d, da, db, accum); else wgmma_ss_m64n64_bf16<1, 0>(d, da, db, accum);
      } else {
        if (b_mn) wgmma_ss_m64n64_bf16<0, 1>(d, da, db, accum); else wgmma_ss_m64n64_bf16<0, 0>(d, da, db, accum);
      }
    };
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int kbs = tile_kblocks(tile);
      if (kbs == 0) continue;
      float acc[GEMM_NCH][32];
      ring.mma_tile(kbs, acc, [&](uint32_t st, int kb) {
        const uint64_t a = a_mn ? make_smem_desc_mn_sw128(st + wg * 8192, MN_BOX_BYTES) : make_smem_desc_sw128(st + wg * 8192);
#pragma unroll
        for (int c = 0; c < GEMM_NCH; ++c) {
          if (c < nmma) {
            const uint32_t bs = st + A_TILE_BYTES + c * 8192;
            const uint64_t bd = b_mn ? make_smem_desc_mn_sw128(bs, MN_BOX_BYTES) : make_smem_desc_sw128(bs);
#pragma unroll
            for (int kk = 0; kk < GEMM_BK / 16; ++kk) mma(acc[c], a + a_step * kk, bd + b_step * kk, (kb | kk) != 0);
          }
        }
      });
      park_tile(img, BG_PITCH, wg, nmma, acc);
      if (p.mode == 0) {
        const int n_tile = tile % p.n_tiles;
        const int m_tile = (tile / p.n_tiles) % p.m_tiles;
        const int z = tile / (p.n_tiles * p.m_tiles);
        const int b = z / p.H, h = z % p.H;
        const int m = m_tile * GEMM_BM + row;
        const int n0 = n_tile * p.block_n;
        const bool row_ok = m < p.M;
        const bool row_keep = row_ok && (p.row_len == nullptr || m < __ldg(p.row_len + b));
        const int clen = p.col_len ? __ldg(p.col_len + b) : p.N;
        const size_t o = (size_t)(p.out_by_b ? b : z) * (size_t)p.out_z_stride + (size_t)(row_ok ? m : 0) * p.ld_out + h * p.out_h_col + n0;
        if (p.staged) {
          // ---- bf16 output as TMA tile stores, one plane (staged_slab_begin / _end).  Rows >= M / columns past the tensor are clipped by
          //      the tensor map.  With sm_P set the value is the fused softmax backward of the row (see below).
          uint8_t* stage_out = smem + BG_STAGE_OUT_OFFSET;
          const bool issuer = half == 0 && lane == 0;
          const int lrow = row & 31;
          const bool sm = p.sm_P != nullptr;
          int len = p.N;
          bool live = row_keep;
          float dsum = 0.f;
          if (sm) {
            len = min(max(__ldg(p.sm_len + b), 0), p.N);
            live = row_ok && ((p.sm_flags & 2) ? len > 0 : m < len);
            if (p.sm_flags & 1) len = min(len, m + 1);
            dsum = live ? __ldg(p.sm_D + (size_t)z * p.M + m) : 0.f;
          }
          const uint32_t thresh = dropout_thresh(p.sm_drop_p);
          const float ks = p.sm_drop_p > 0.f ? 1.f / (1.f - p.sm_drop_p) : 1.f;
          uint32_t qa[16], qb[16];
          // fused softmax backward: the P_pre row segments of the NEXT slab are requested before the current slab is
          // processed: the slab loop is a dependent chain (image load -> math -> shared store -> barrier -> TMA store) with two
          // warps per lane quarter and nothing else to hide a global load behind
          uint4 pn00, pn01, pn10, pn11;   // next slab: [chunk u][16-byte half]
          auto prefetch = [&](int s0n) {
            pn00 = pn01 = pn10 = pn11 = make_uint4(0, 0, 0, 0);
            if (sm && s0n < nch && live) {
              const int ca_n = (s0n + 2 * half) << 4, cb_n = ca_n + 16;
              if (n0 + ca_n < len) {
                const uint4* src = reinterpret_cast<const uint4*>(p.sm_P + o + ca_n);
                pn00 = __ldg(src);
                pn01 = __ldg(src + 1);
              }
              if (n0 + cb_n < len) {
                const uint4* src = reinterpret_cast<const uint4*>(p.sm_P + o + cb_n);
                pn10 = __ldg(src);
                pn11 = __ldg(src + 1);
              }
            }
          };
          prefetch(0);
          for (int s0 = 0; s0 < nch; s0 += 4) {
            const int ca = s0 + 2 * half, cb = ca + 1;
            uint4 pv[2][2], pd[2][2];
            pv[0][0] = pn00; pv[0][1] = pn01; pv[1][0] = pn10; pv[1][1] = pn11;
            prefetch(s0 + 4);
            if (sm) {
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                const int c0 = (u ? cb : ca) << 4;
                pd[u][0] = pd[u][1] = make_uint4(0, 0, 0, 0);
                if (p.sm_Pdrop != nullptr && live && n0 + c0 < len) {
                  const uint4* sd = reinterpret_cast<const uint4*>(p.sm_Pdrop + o + c0);
                  pd[u][0] = __ldg(sd);
                  pd[u][1] = __ldg(sd + 1);
                }
              }
            }
            __syncwarp();
            acc_ld16(arow + (ca << 4), qa);
            acc_ld16(arow + (cb << 4), qb);
            uint8_t* box = staged_slab_begin(stage_out, quarter, issuer, false, slab_ctr);
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int c0 = (u ? cb : ca) << 4;
              float y[16];
              if (sm) {
                // dS[j] = scale * P[j] * (keep[j] * dP[j] / (1-p) - D)  as  fma(a, dP, -(ps * D)),  ps = scale * P,
                // a = keep ? ps / (1-p) : 0; one mask hash per element pair; the key-length test only in the boundary chunk
                const uint32_t* pw = reinterpret_cast<const uint32_t*>(pv[u]);
                const uint16_t* dd = reinterpret_cast<const uint16_t*>(pd[u]);
                const size_t e0 = o + c0;
                const int kbase = n0 + c0;
                const float sks = p.sm_scale * ks;
                // mask hash of pair k of this chunk: mix((x0 + k*C1) ^ hterm) -- the host admits < 2^33 elements in this
                // mode, so the pair index fits 32 bits (no 64-bit index arithmetic per pair)
                const uint32_t hx0 = (uint32_t)(e0 >> 1) * DROPOUT_C1;
                const uint32_t hterm = dropout_hterm(p.sm_seed, p.sm_site, 0u);
                const uint32_t th16 = thresh >> 16;
                if (!live || kbase >= len) {
#pragma unroll
                  for (int j = 0; j < 16; ++j) y[j] = 0.f;
                } else {
#pragma unroll
                  for (int j = 0; j < 16; j += 2) {
                    const float p0 = __uint_as_float(pw[j >> 1] << 16), p1 = __uint_as_float(pw[j >> 1] & 0xffff0000u);
                    bool k0 = true, k1 = true;
                    if (p.sm_drop_p > 0.f) {
                      if (p.sm_Pdrop != nullptr) { k0 = (dd[j] & 0x7fffu) != 0; k1 = (dd[j + 1] & 0x7fffu) != 0; }
                      else {
                        const uint32_t hsh = dropout_mix((hx0 + (uint32_t)(j >> 1) * DROPOUT_C1) ^ hterm);
                        k0 = (hsh & 0xffffu) >= th16;
                        k1 = (hsh >> 16) >= th16;
                      }
                    }
                    const float r0 = __uint_as_float(u ? qb[j] : qa[j]), r1 = __uint_as_float(u ? qb[j + 1] : qa[j + 1]);
                    y[j] = fmaf(k0 ? p0 * sks : 0.f, r0, -(p0 * p.sm_scale) * dsum);
                    y[j + 1] = fmaf(k1 ? p1 * sks : 0.f, r1, -(p1 * p.sm_scale) * dsum);
                  }
                  if (kbase + 16 > len) {   // the chunk that straddles the key length (P is zero there already; keep exact zeros)
#pragma unroll
                    for (int j = 0; j < 16; ++j) y[j] = (kbase + j < len) ? y[j] : 0.f;
                  }
                }
              } else {
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                  const int n = n0 + c0 + j;
                  y[j] = (row_keep && n < clen && n < p.N) ? __uint_as_float(u ? qb[j] : qa[j]) * p.alpha : 0.f;
                }
              }
              uint32_t hh[8];
              pack_hi(y, hh);
              st_box_chunk(box, lrow, 2 * (2 * half + u), hh);
            }
            staged_slab_end(quarter, issuer, [&] {
              if (n0 + (s0 << 4) < p.out_cols)
                tma_store_3d(&tmO, box, h * p.out_h_col + n0 + (s0 << 4), m_tile * GEMM_BM + quarter * 32, p.out_by_b ? b : z);
            });
          }
        } else if (p.sm_P != nullptr) {
          // ---- softmax backward fused into the dP product (see ttsb_bgemm_args): this thread owns query row m of
          //      problem z.  The P_pre row segments of all its chunks are requested before the first accumulator load.
          int len = min(max(__ldg(p.sm_len + b), 0), p.N);
          const bool live = row_ok && ((p.sm_flags & 2) ? len > 0 : m < len);
          if (p.sm_flags & 1) len = min(len, m + 1);
          const float dsum = live ? __ldg(p.sm_D + (size_t)z * p.M + m) : 0.f;
          const uint32_t thresh = dropout_thresh(p.sm_drop_p);
          const float ks = p.sm_drop_p > 0.f ? 1.f / (1.f - p.sm_drop_p) : 1.f;
          // chunks of this thread in groups of four: the P_pre (and P_drop) row segments of a group are requested before
          // its first accumulator load.  The dropout decision is read back from the saved P_drop (kept <=> P_drop != 0 wherever
          // P_pre != 0) when sm_Pdrop is given; otherwise it is regenerated from the hash.
          constexpr int GRP = 4;
          for (int g0 = ch_begin; g0 < ch_end; g0 += GRP) {
            uint4 pv[GRP][2], pd[GRP][2];
#pragma unroll
            for (int i = 0; i < GRP; ++i) {
              const int c0 = (g0 + i) << 4;
              const bool need = g0 + i < ch_end && live && n0 + c0 < len;
              if (need) {
                const uint4* src = reinterpret_cast<const uint4*>(p.sm_P + o + c0);
                pv[i][0] = __ldg(src);
                pv[i][1] = __ldg(src + 1);
              } else {
                pv[i][0] = make_uint4(0, 0, 0, 0);
                pv[i][1] = make_uint4(0, 0, 0, 0);
              }
              if (need && p.sm_Pdrop != nullptr) {
                const uint4* src = reinterpret_cast<const uint4*>(p.sm_Pdrop + o + c0);
                pd[i][0] = __ldg(src);
                pd[i][1] = __ldg(src + 1);
              } else {
                pd[i][0] = make_uint4(0, 0, 0, 0);
                pd[i][1] = make_uint4(0, 0, 0, 0);
              }
            }
#pragma unroll
            for (int i = 0; i < GRP; ++i) {
              const int ch = g0 + i;
              if (ch < ch_end) {   // warp-uniform
                const int c0 = ch << 4;
                __syncwarp();
                acc_ld16(arow + c0, r);
                if (row_ok && n0 + c0 < p.out_cols) {
                  const size_t e0 = o + c0;  // element index in the (Z, M, ld_out) layout shared by P_pre, P_drop, dP and dS
                  uint32_t hh[8];
                  if (live && n0 + c0 < len) {
                    const __nv_bfloat16* pp = reinterpret_cast<const __nv_bfloat16*>(pv[i]);
                    const uint16_t* dd = reinterpret_cast<const uint16_t*>(pd[i]);
                    float y[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                      const int k = n0 + c0 + j;
                      bool keep = true;
                      if (p.sm_drop_p > 0.f) keep = p.sm_Pdrop != nullptr ? (dd[j] & 0x7fffu) != 0 : dropout_keep(p.sm_seed, p.sm_site, e0 + j, thresh);
                      const float g = keep ? __uint_as_float(r[j]) * ks : 0.f;
                      y[j] = k < len ? p.sm_scale * __bfloat162float(pp[j]) * (g - dsum) : 0.f;
                    }
                    pack_hi(y, hh);
                  } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) hh[j] = 0u;
                  }
                  st_global_v8(p.out_bf16 + e0, hh);
                }
              }
            }
          }
        } else
        for (int ch = ch_begin; ch < ch_end; ++ch) {
          const int c0 = ch << 4;
          __syncwarp();
          acc_ld16(arow + c0, r);
          if (row_ok && n0 + c0 < p.out_cols) {  // out_cols (multiple of 16) bounds the writable part of the row
            float y[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const int n = n0 + c0 + j;
              y[j] = (row_keep && n < clen && n < p.N) ? __uint_as_float(r[j]) * p.alpha : 0.f;
            }
            if (p.out_f32) {
              st_global_v8f(p.out_f32 + o + c0, y);
              st_global_v8f(p.out_f32 + o + c0 + 8, y + 8);
            }
            if (p.out_bf16) {
              uint32_t hh[8];
              pack_hi(y, hh);
              st_global_v8(p.out_bf16 + o + c0, hh);
            }
          }
        }
      } else {
        int rr = tile / p.splits;
        const int n_tile = rr % p.n_tiles; rr /= p.n_tiles;
        const int m_tile = rr % p.m_tiles; rr /= p.m_tiles;
        const int seg = rr;
        const int c = m_tile * GEMM_BM + row;
        const int n0 = n_tile * p.block_n;
        const bool row_ok = c < p.Cin;
        float* dst = p.dw + ((size_t)seg * p.Cin + (row_ok ? c : 0)) * p.N + n0;
        for (int ch = ch_begin; ch < ch_end; ++ch) {
          const int c0 = ch << 4;
          __syncwarp();
          acc_ld16(arow + c0, r);
          if (row_ok) {
            if ((p.N & 3) == 0 && n0 + c0 + 16 <= p.N) {   // 16-byte aligned: four vector reductions instead of sixteen scalar ones
#pragma unroll
              for (int j = 0; j < 16; j += 4)
                asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(dst + c0 + j), "f"(__uint_as_float(r[j])),
                             "f"(__uint_as_float(r[j + 1])), "f"(__uint_as_float(r[j + 2])), "f"(__uint_as_float(r[j + 3]))
                             : "memory");
            } else {
#pragma unroll
              for (int j = 0; j < 16; ++j)
                if (n0 + c0 + j < p.N) atomicAdd(dst + c0 + j, __uint_as_float(r[j]));
            }
          }
        }
      }
      ring.release_tile(p.staged && half == 0 && lane == 0);
    }
    BgRing::finish(p.staged && half == 0 && lane == 0);
  }
done:
  __syncthreads();
}

static int pick_block_n(int N) {
  const int n16 = (N + 15) / 16 * 16;
  return n16 < GEMM_MAX_BN ? n16 : GEMM_MAX_BN;
}

}  // namespace ttsb

using namespace ttsb;

extern "C" int ttsb_bgemm(const ttsb_bgemm_args* a, void* stream_v) {
  if (!a) { set_last_error("ttsb_bgemm: args is NULL"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->B <= 0 || a->H <= 0 || a->M <= 0 || a->N <= 0 || a->K <= 0) { set_last_error("ttsb_bgemm: non-positive dimension"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (!a->a || !a->b || (!a->out_f32 && !a->out_bf16)) { set_last_error("ttsb_bgemm: NULL tensor"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->ld_out % 16 || a->out_cols % 16 || a->out_cols <= 0 || a->out_h_col % 16) {
    set_last_error("ttsb_bgemm: ld_out, out_cols and out_h_col must be multiples of 16 (32-byte stores)");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  BgParams p{};
  p.mode = 0;
  p.Z = a->B * a->H; p.H = a->H; p.M = a->M; p.N = a->N; p.K = a->K;
  p.opA = {a->a_h_col, a->a_h_row, a->a_z_batch, a->a_mn_major};
  p.opB = {a->b_h_col, a->b_h_row, a->b_z_batch, a->b_mn_major};
  p.alpha = a->alpha;
  p.out_f32 = a->out_f32;
  p.out_bf16 = static_cast<__nv_bfloat16*>(a->out_bf16);
  p.ld_out = a->ld_out; p.out_z_stride = a->out_batch_stride; p.out_h_col = a->out_h_col; p.out_by_b = a->out_by_b; p.out_cols = a->out_cols;
  p.row_len = a->row_len; p.col_len = a->col_len;
  if (a->sm_P) {
    if (!a->sm_D || !a->sm_len || !a->out_bf16 || a->out_by_b || a->out_h_col || a->out_batch_stride != (long long)a->M * a->ld_out ||
        a->sm_drop_p < 0.f || a->sm_drop_p >= 1.f || (unsigned long long)a->B * a->H * a->M * (unsigned long long)a->ld_out >= (1ull << 33)) {
      set_last_error("ttsb_bgemm: the fused softmax backward needs sm_D, sm_len, out_bf16, the (Z, M, ld_out) output layout and < 2^33 elements");
      return TTSB_ERR_INVALID_ARGUMENT;
    }
    p.sm_P = static_cast<const __nv_bfloat16*>(a->sm_P);
    p.sm_Pdrop = (a->sm_drop_p > 0.f && a->sm_Pdrop) ? static_cast<const __nv_bfloat16*>(a->sm_Pdrop) : nullptr;
    p.sm_D = a->sm_D; p.sm_scale = a->sm_scale; p.sm_drop_p = a->sm_drop_p; p.sm_seed = a->sm_seed; p.sm_site = a->sm_site;
    p.sm_flags = a->sm_flags; p.sm_len = a->sm_len;
    p.out_f32 = nullptr;
  }
  p.block_n = pick_block_n(a->N);
  p.n_tiles = (a->N + p.block_n - 1) / p.block_n;
  p.m_tiles = (a->M + GEMM_BM - 1) / GEMM_BM;
  p.num_tiles = p.Z * p.m_tiles * p.n_tiles;
  p.T = 1;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_bf16_3d(&tmA, a->a, (uint64_t)a->a_dim0, (uint64_t)a->a_dim1, (uint64_t)a->a_dim2, (uint64_t)a->a_stride1,
                             (uint64_t)a->a_stride2, GEMM_BK, a->a_mn_major ? 64 : GEMM_BM);
  if (rc) return rc;
  rc = make_tmap_bf16_3d(&tmB, a->b, (uint64_t)a->b_dim0, (uint64_t)a->b_dim1, (uint64_t)a->b_dim2, (uint64_t)a->b_stride1,
                         (uint64_t)a->b_stride2, GEMM_BK, a->b_mn_major ? 64 : p.block_n);
  if (rc) return rc;
  // bf16-only outputs of a tile width that fills whole 64-column boxes go through shared staging + TMA tile stores
  CUtensorMap tmO = tmB;
  if (p.out_bf16 && !p.out_f32 && p.block_n % 64 == 0 && (reinterpret_cast<uintptr_t>(p.out_bf16) & 15) == 0) {
    const uint64_t cols = p.out_by_b ? (uint64_t)p.H * p.out_h_col : (uint64_t)p.out_cols;
    rc = make_tmap_bf16_3d(&tmO, p.out_bf16, cols, (uint64_t)p.M, (uint64_t)(p.out_by_b ? a->B : p.Z), (uint64_t)p.ld_out,
                           (uint64_t)p.out_z_stride, 64, 32);
    if (rc) return rc;
    p.staged = 1;
  }
  return launch_pipeline<bgemm_tc_kernel>(BG_SMEM_BYTES, p.num_tiles, false, stream, "bgemm_tc_kernel launch", tmA, tmA, tmB, tmO, p);
}

extern "C" int ttsb_wgrad(const ttsb_wgrad_args* a, void* stream_v) {
  if (!a) { set_last_error("ttsb_wgrad: args is NULL"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->B <= 0 || a->T <= 0 || a->Cin <= 0 || a->N <= 0 || a->num_segments < 1 || a->num_segments > 4) {
    set_last_error("ttsb_wgrad: bad dimensions");
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (!a->x[0] || !a->g || !a->dw || a->ldg % 8) { set_last_error("ttsb_wgrad: NULL tensor or ldg not a multiple of 8"); return TTSB_ERR_INVALID_ARGUMENT; }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  BgParams p{};
  p.mode = 1;
  p.B = a->B; p.T = a->T; p.Cin = a->Cin; p.N = a->N; p.num_seg = a->num_segments; p.H = 1;
  for (int s = 0; s < a->num_segments; ++s) {
    p.seg_src[s] = a->seg_src[s];
    p.seg_shift[s] = a->seg_shift[s];
    if (a->seg_src[s] < 0 || a->seg_src[s] > 1 || !a->x[a->seg_src[s]] || a->ldx[a->seg_src[s]] % 8) {
      set_last_error("ttsb_wgrad: bad segment source");
      return TTSB_ERR_INVALID_ARGUMENT;
    }
  }
  p.dw = a->dw;
  p.block_n = pick_block_n(a->N);
  p.n_tiles = (a->N + p.block_n - 1) / p.block_n;
  p.m_tiles = (a->Cin + GEMM_BM - 1) / GEMM_BM;
  const int base_tiles = a->num_segments * p.m_tiles * p.n_tiles;
  int splits = (2 * num_sms() + base_tiles - 1) / base_tiles;
  if (splits > a->B) splits = a->B;
  if (splits < 1) splits = 1;
  p.b_per_split = (a->B + splits - 1) / splits;
  p.splits = (a->B + p.b_per_split - 1) / p.b_per_split;
  p.num_tiles = base_tiles * p.splits;
  CUtensorMap tmA[2], tmB;
  for (int i = 0; i < 2; ++i) {
    const int use = a->x[i] ? i : 0;
    int rc = make_tmap_bf16_3d(&tmA[i], a->x[use], (uint64_t)a->Cin, (uint64_t)a->T, (uint64_t)a->B, (uint64_t)a->ldx[use],
                               (uint64_t)a->ldx[use] * a->T, GEMM_BK, 64);
    if (rc) return rc;
  }
  int rc = make_tmap_bf16_3d(&tmB, a->g, (uint64_t)a->N, (uint64_t)a->T, (uint64_t)a->B, (uint64_t)a->ldg, (uint64_t)a->ldg * a->T, GEMM_BK, 64);
  if (rc) return rc;
  return launch_pipeline<bgemm_tc_kernel>(BG_SMEM_BYTES, p.num_tiles, false, stream, "bgemm_tc_kernel launch", tmA[0], tmA[1], tmB, tmB, p);
}

TTSB_DEFINE_SALT_SETTER(set_salt_bgemm)
