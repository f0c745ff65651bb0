// Bandwidth-bound row kernels of the text->mel path: embedding + LayerNorm + positional encoding, the length
// regulator (durations -> int -> scan -> frame->phoneme indices -> gather, fused with the decoder prologue), the
// predictor heads, pitch embedding, length helpers and the operand preparation (bf16 hi/lo split, weight packing).
// None of these touch tensor cores: they are coalesced, 16-byte vectorised HBM kernels, one warp per row.
#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace ttsb {

constexpr int ROW_MAX_V4 = 4;  // a warp holds one row of up to 32*4*4 = 512 floats in registers

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// LayerNorm (Keras non-fused: biased variance, rsqrt(var+eps)) of a row held as float4 fragments, + scalar*pe, store.
__device__ __forceinline__ void ln_pe_store(float4 (&v)[ROW_MAX_V4], int nv, int d, int lane, const float* gamma,
                                            const float* beta, float eps, const float* pe_row, float scalar, float* out_f32,
                                            __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, float drop_p = 0.f, uint32_t seed = 0,
                                            uint32_t site = 0, uint64_t elem0 = 0) {
  const uint32_t thresh = dropout_thresh(drop_p);
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < ROW_MAX_V4; ++i)
    if (i < nv && (i * 32 + lane) * 4 < d) s += v[i].x + v[i].y + v[i].z + v[i].w;
  const float mean = warp_sum(s) / d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < ROW_MAX_V4; ++i)
    if (i < nv && (i * 32 + lane) * 4 < d) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
      q += a * a + b * b + c * c + e * e;
    }
  const float rstd = rsqrtf(warp_sum(q) / d + eps);
#pragma unroll
  for (int i = 0; i < ROW_MAX_V4; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    if (i < nv && c0 < d) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c0));
      const float4 bt = __ldg(reinterpret_cast<const float4*>(beta + c0));
      const float4 pe = pe_row ? __ldg(reinterpret_cast<const float4*>(pe_row + c0)) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 y;
      y.x = (v[i].x - mean) * rstd * g.x + bt.x + scalar * pe.x;
      y.y = (v[i].y - mean) * rstd * g.y + bt.y + scalar * pe.y;
      y.z = (v[i].z - mean) * rstd * g.z + bt.z + scalar * pe.z;
      y.w = (v[i].w - mean) * rstd * g.w + bt.w + scalar * pe.w;
      if (drop_p > 0.f) {  // keras Dropout after LayerNorm + PE (model/layers.py:301), training only
        y.x = dropout_keep(seed, site, elem0 + c0 + 0, thresh) ? y.x * keep_scale : 0.f;
        y.y = dropout_keep(seed, site, elem0 + c0 + 1, thresh) ? y.y * keep_scale : 0.f;
        y.z = dropout_keep(seed, site, elem0 + c0 + 2, thresh) ? y.z * keep_scale : 0.f;
        y.w = dropout_keep(seed, site, elem0 + c0 + 3, thresh) ? y.w * keep_scale : 0.f;
      }
      if (out_f32) *reinterpret_cast<float4*>(out_f32 + c0) = y;
      if (out_hi) {
        __nv_bfloat16 h0, l0, h1, l1, h2, l2, h3, l3;
        split_bf16(y.x, h0, l0); split_bf16(y.y, h1, l1); split_bf16(y.z, h2, l2); split_bf16(y.w, h3, l3);
        *reinterpret_cast<uint2*>(out_hi + c0) = make_uint2(pack_bf16(h0, h1), pack_bf16(h2, h3));
        if (out_lo) *reinterpret_cast<uint2*>(out_lo + c0) = make_uint2(pack_bf16(l0, l1), pack_bf16(l2, l3));
      }
    }
  }
}

__global__ void embed_ln_pe_kernel(const int* __restrict__ tokens, const float* __restrict__ emb, const float* gamma,
                                   const float* beta, const float* pe, const float* pos_scalar, int rows, int T, int d,
                                   int vocab, float eps, float* out_f32, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo,
                                   float drop_p, uint32_t seed, uint32_t site) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  int tok = __ldg(tokens + row);
  tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);
  const int t = row % T;
  const int nv = (d + 127) / 128;
  float4 v[ROW_MAX_V4];
#pragma unroll
  for (int i = 0; i < ROW_MAX_V4; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    v[i] = (i < nv && c0 < d) ? __ldg(reinterpret_cast<const float4*>(emb + (size_t)tok * d + c0)) : make_float4(0, 0, 0, 0);
  }
  const size_t o = (size_t)row * d;
  ln_pe_store(v, nv, d, lane, gamma, beta, eps, pe + (size_t)t * d, __ldg(pos_scalar), out_f32 ? out_f32 + o : nullptr,
              out_hi ? out_hi + o : nullptr, out_lo ? out_lo + o : nullptr, drop_p, seed, site, (uint64_t)o);
}

__global__ void expand_ln_pe_kernel(const float* __restrict__ x, const int* __restrict__ idx, const float* gamma,
                                    const float* beta, const float* pe, const float* pos_scalar, int B, int Tp, int Tm, int d,
                                    float eps, float* out_f32, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, float drop_p,
                                    uint32_t seed, uint32_t site) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B * Tm) return;
  const int lane = threadIdx.x & 31;
  const int b = row / Tm, t = row % Tm;
  const int src = __ldg(idx + row);
  const int nv = (d + 127) / 128;
  float4 v[ROW_MAX_V4];
#pragma unroll
  for (int i = 0; i < ROW_MAX_V4; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    v[i] = (src >= 0 && i < nv && c0 < d) ? __ldg(reinterpret_cast<const float4*>(x + ((size_t)b * Tp + src) * d + c0))
                                          : make_float4(0, 0, 0, 0);
  }
  const size_t o = (size_t)row * d;
  ln_pe_store(v, nv, d, lane, gamma, beta, eps, pe + (size_t)t * d, __ldg(pos_scalar), out_f32 ? out_f32 + o : nullptr,
              out_hi ? out_hi + o : nullptr, out_lo ? out_lo + o : nullptr, drop_p, seed, site, (uint64_t)o);
}

// Decoder prologue of one row per sentence at a device-side position (cached autoregressive decoding): the PE row is
// pe[pos[b]] instead of the output frame index of expand_ln_pe_kernel.
__global__ void decode_prologue_kernel(const float* __restrict__ x, const int* __restrict__ pos, const float* gamma,
                                       const float* beta, const float* pe, int pe_rows, const float* pos_scalar, int B, int d,
                                       float eps, float* out_f32, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B) return;
  const int lane = threadIdx.x & 31;
  const int t = min(max(__ldg(pos + row), 0), pe_rows - 1);
  const int nv = (d + 127) / 128;
  float4 v[ROW_MAX_V4];
#pragma unroll
  for (int i = 0; i < ROW_MAX_V4; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    v[i] = (i < nv && c0 < d) ? __ldg(reinterpret_cast<const float4*>(x + (size_t)row * d + c0)) : make_float4(0, 0, 0, 0);
  }
  const size_t o = (size_t)row * d;
  ln_pe_store(v, nv, d, lane, gamma, beta, eps, pe + (size_t)t * d, __ldg(pos_scalar), out_f32 ? out_f32 + o : nullptr,
              out_hi ? out_hi + o : nullptr, out_lo ? out_lo + o : nullptr);
}

// Stand-alone LayerNorm + row mask for model dimensions whose row does not fit one 256-column accumulator tile (d = 384):
// the GEMM writes the pre-norm value (acc + bias + residual), this kernel normalises it (model/layers.py:211,40,102).
__global__ void layernorm_fwd_kernel(const float* __restrict__ x, const float* gamma, const float* beta, int rows, int T, int d,
                                     int ld, float eps, const int* __restrict__ row_len, float* out_f32, __nv_bfloat16* out_hi,
                                     __nv_bfloat16* out_lo) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int b = row / T, t = row % T;
  const int nv = (d + 127) / 128;
  const size_t o = (size_t)row * ld;
  if (row_len != nullptr && t >= __ldg(row_len + b)) {
    for (int c0 = lane * 4; c0 < d; c0 += 128) {
      if (out_f32) *reinterpret_cast<float4*>(out_f32 + o + c0) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (out_hi) *reinterpret_cast<uint2*>(out_hi + o + c0) = make_uint2(0u, 0u);
      if (out_lo) *reinterpret_cast<uint2*>(out_lo + o + c0) = make_uint2(0u, 0u);
    }
    return;
  }
  float4 v[ROW_MAX_V4];
#pragma unroll
  for (int i = 0; i < ROW_MAX_V4; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    v[i] = (i < nv && c0 < d) ? __ldg(reinterpret_cast<const float4*>(x + o + c0)) : make_float4(0, 0, 0, 0);
  }
  ln_pe_store(v, nv, d, lane, gamma, beta, eps, nullptr, 0.f, out_f32 ? out_f32 + o : nullptr, out_hi ? out_hi + o : nullptr,
              out_lo ? out_lo + o : nullptr);
}

// Expand (model/layers.py:549-565) as a gather: 16-byte vectorised, one warp per output frame.
__global__ void length_regulate_kernel(const float* __restrict__ x, const int* __restrict__ idx, int B, int Tp, int Tm, int d,
                                       float* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B * Tm) return;
  const int lane = threadIdx.x & 31;
  const int b = row / Tm;
  const int src = __ldg(idx + row);
  const float4* s = reinterpret_cast<const float4*>(x + ((size_t)b * Tp + (src >= 0 ? src : 0)) * d);
  float4* o = reinterpret_cast<float4*>(out + (size_t)row * d);
  for (int c = lane; c < d / 4; c += 32) o[c] = src >= 0 ? __ldg(s + c) : make_float4(0, 0, 0, 0);
}

// durations -> *scalar -> min(max_mask) -> max(min_mask) -> round-half-even -> int32 ; per-row totals
__global__ void durations_to_int_kernel(const float* __restrict__ dur, float scalar, const float* max_mask,
                                        const float* min_mask, int Tp, int* __restrict__ out_int, int* __restrict__ out_len) {
  const int b = blockIdx.x;
  int local = 0, neg = 0;
  for (int i = threadIdx.x; i < Tp; i += blockDim.x) {
    const size_t o = (size_t)b * Tp + i;
    float v = __fmul_rn(dur[o], scalar);
    if (max_mask) v = fminf(v, max_mask[o]);
    if (min_mask) v = fmaxf(v, min_mask[o]);
    const int n = __float2int_rn(v);  // round-half-to-even, as tf.math.round (model/layers.py:551)
    out_int[o] = n;
    local += n;
    neg |= n < 0;
  }
  __shared__ int red[32], red_neg[32];
  for (int o = 16; o; o >>= 1) {
    local += __shfl_xor_sync(0xffffffffu, local, o);
    neg |= __shfl_xor_sync(0xffffffffu, neg, o);
  }
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = local; red_neg[threadIdx.x >> 5] = neg; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0, any_neg = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { s += red[w]; any_neg |= red_neg[w]; }
    // a negative duration has no meaning for the length regulator (the reference's RaggedTensor construction raises):
    // flagged through the row length so that the host needs no second device->host read
    out_len[b] = any_neg ? -1 : s;
  }
}

// int durations (B,Tp) -> frame->phoneme map (B,Tm): inclusive scan in shared memory, then a binary search per frame.
__global__ void expand_indices_kernel(const int* __restrict__ dur, int Tp, int Tm, int* __restrict__ out_idx) {
  extern __shared__ int cum[];  // Tp inclusive sums
  __shared__ int warp_tot[32];
  const int b = blockIdx.x;
  const int per = (Tp + blockDim.x - 1) / blockDim.x;
  const int beg = threadIdx.x * per;
  const int end = min(beg + per, Tp);
  int s = 0;
  for (int i = beg; i < end; ++i) s += max(dur[(size_t)b * Tp + i], 0);
  // block exclusive scan of the per-thread sums
  int incl = s;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int w = lane < (int)(blockDim.x >> 5) ? warp_tot[lane] : 0;
    int wi = w;
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += n;
    }
    warp_tot[lane] = wi - w;  // exclusive
  }
  __syncthreads();
  int run = warp_tot[wid] + incl - s;
  for (int i = beg; i < end; ++i) {
    run += max(dur[(size_t)b * Tp + i], 0);
    cum[i] = run;
  }
  __syncthreads();
  const int total = Tp > 0 ? cum[Tp - 1] : 0;
  for (int t = threadIdx.x; t < Tm; t += blockDim.x) {
    int r = -1;
    if (t < total) {
      int lo = 0, hi = Tp - 1;  // first i with cum[i] > t
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cum[mid] > t) hi = mid; else lo = mid + 1;
      }
      r = lo;
    }
    out_idx[(size_t)b * Tm + t] = r;
  }
}

__global__ void statpred_head_kernel(const float* __restrict__ h, int ldh, int C, const float* __restrict__ w, const float* bias,
                                     int relu, const int* row_len, int rows, int T, float* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
  for (int c = lane; c < C; c += 32) acc = fmaf(h[(size_t)row * ldh + c], __ldg(w + c), acc);
  acc = warp_sum(acc);
  if (lane == 0) {
    acc += __ldg(bias);
    if (relu) acc = fmaxf(acc, 0.f);
    const int b = row / T, t = row % T;
    if (row_len && t >= row_len[b]) acc = 0.f;
    out[row] = acc;
  }
}

__global__ void pitch_embed_add_kernel(const float* __restrict__ x, const float* __restrict__ pitch, const float* __restrict__ w,
                                       const float* __restrict__ bias, int64_t n4, int d4, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int64_t row = i / d4;
  const int c4 = (int)(i % d4);
  const float pv = __ldg(pitch + row);
  const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + i);
  const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + c4);
  const float4 bv = __ldg(reinterpret_cast<const float4*>(bias) + c4);
  float4 y;
  y.x = xv.x + fmaxf(fmaf(pv, wv.x, bv.x), 0.f);
  y.y = xv.y + fmaxf(fmaf(pv, wv.y, bv.y), 0.f);
  y.z = xv.z + fmaxf(fmaf(pv, wv.z, bv.z), 0.f);
  y.w = xv.w + fmaxf(fmaf(pv, wv.w, bv.w), 0.f);
  reinterpret_cast<float4*>(out)[i] = y;
}

// utils/spectrogram_ops.py:8-13, literally: a frame counts iff (#channels != pad) != C*pad
__global__ void mel_lengths_kernel(const float* __restrict__ mel, int T, int C, float pad, int* __restrict__ out) {
  // grid (B, ceil(T / 64)): every block counts 64 frames (8 warps x 8 frames) and adds its count to out[b] (zeroed by the host)
  const int b = blockIdx.x;
  const float sum_tot = (float)C * pad;
  int local = 0;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int t_end = min(T, (int)(blockIdx.y + 1) * 64);
  for (int t = blockIdx.y * 64 + wid; t < t_end; t += nw) {
    int cnt = 0;
    for (int c = lane; c < C; c += 32) cnt += (mel[((size_t)b * T + t) * C + c] != pad) ? 1 : 0;
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0 && (float)cnt != sum_tot) local += 1;
  }
  __shared__ int red[32];
  if (lane == 0) red[wid] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < nw; ++w) s += red[w];
    if (s) atomicAdd(out + b, s);
  }
}

__global__ void phoneme_lengths_kernel(const int* __restrict__ ph, int T, int pad, int* __restrict__ out) {
  const int b = blockIdx.x;
  int local = 0;
  for (int t = threadIdx.x; t < T; t += blockDim.x) local += ph[(size_t)b * T + t] != pad ? 1 : 0;
  __shared__ int red[32];
  for (int o = 16; o; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    out[b] = s;
  }
}

__global__ void split_bf16_kernel(const float* __restrict__ x, int64_t n, __nv_bfloat16* hi, __nv_bfloat16* lo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  __nv_bfloat16 h, l;
  split_bf16(x[i], h, l);
  hi[i] = h;
  if (lo) lo[i] = l;
}

// Keras (K,N) -> packed [n_pad, K] bf16 hi/lo (rows >= N are zero)
__global__ void pack_weight_kernel(const float* __restrict__ w, int K, int N, int n_pad, __nv_bfloat16* hi, __nv_bfloat16* lo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_pad * K) return;
  const int n = (int)(i / K), k = (int)(i % K);
  const float v = n < N ? w[(size_t)k * N + n] : 0.f;
  __nv_bfloat16 h, l;
  split_bf16(v, h, l);
  hi[i] = h;
  if (lo) lo[i] = l;
}

// Batched operand preparation for the training step: every packed bf16 weight (forward and data-gradient layouts), padded
// bias and padded LayerNorm vector is described once (ttsb_pack_desc, device array) and refreshed by ONE launch per step.
//   dst[r][c] = (r < R && c % cb < cb_valid) ? src[r*sr + (c / cb)*s_outer + (c % cb)*s_inner] : 0
__global__ void repack_batched_kernel(const ttsb_pack_desc* __restrict__ descs) {
  // 64x64 tiles staged through shared memory: the load runs along whichever source axis is contiguous (rows for the
  // transposing forward packs of Keras (K,N) kernels, columns otherwise), the store always along destination columns.
  __shared__ float tile[64][65];
  const ttsb_pack_desc d = descs[blockIdx.y];
  const int tiles_c = (d.C_cols + 63) >> 6, tiles_r = (d.R_pad + 63) >> 6;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;   // 256 threads: 64 x 4
  const bool along_r = d.sr == 1 && d.s_inner != 1;
  for (int tl = blockIdx.x; tl < tiles_r * tiles_c; tl += gridDim.x) {
    const int r0 = (tl / tiles_c) << 6, c0 = (tl % tiles_c) << 6;
    if (along_r) {
      const int r = r0 + tx;
#pragma unroll 4
      for (int j = ty; j < 64; j += 4) {
        const int c = c0 + j, blk = c / d.cb, ci = c % d.cb;
        tile[tx][j] = (r < d.R && c < d.C_cols && ci < d.cb_valid)
                          ? d.src[(long long)r * d.sr + (long long)blk * d.s_outer + (long long)ci * d.s_inner] : 0.f;
      }
    } else {
      const int c = c0 + tx, blk = c / d.cb, ci = c % d.cb;
      const bool cok = c < d.C_cols && ci < d.cb_valid;
      const long long coff = (long long)blk * d.s_outer + (long long)ci * d.s_inner;
#pragma unroll 4
      for (int j = ty; j < 64; j += 4) {
        const int r = r0 + j;
        tile[j][tx] = (cok && r < d.R) ? d.src[(long long)r * d.sr + coff] : 0.f;
      }
    }
    __syncthreads();
    const int c = c0 + tx;
    if (c < d.C_cols) {
#pragma unroll 4
      for (int j = ty; j < 64; j += 4) {
        const int r = r0 + j;
        if (r >= d.R_pad) break;
        const long long o = (long long)r * d.dst_ld + c;
        if (d.dst_f32) static_cast<float*>(d.dst)[o] = tile[j][tx];
        else static_cast<__nv_bfloat16*>(d.dst)[o] = __float2bfloat16_rn(tile[j][tx]);
      }
    }
    __syncthreads();
  }
}

static inline int bad(const char* msg) {
  set_last_error("%s", msg);
  return TTSB_ERR_INVALID_ARGUMENT;
}

}  // namespace ttsb

using namespace ttsb;
#define STREAM(s) static_cast<cudaStream_t>(s)

#define LAUNCH_OK(name)  \
  count_launch();        \
  return check_cuda(cudaGetLastError(), name)

extern "C" int ttsb_pack_weight(const float* w_kn, int K, int N, int n_pad, void* w_hi, void* w_lo, void* stream) {
  if (!w_kn || !w_hi || K <= 0 || N <= 0 || n_pad < N) return bad("ttsb_pack_weight: bad arguments");
  const int64_t n = (int64_t)n_pad * K;
  pack_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM(stream)>>>(w_kn, K, N, n_pad, static_cast<__nv_bfloat16*>(w_hi),
                                                                            static_cast<__nv_bfloat16*>(w_lo));
  LAUNCH_OK("pack_weight_kernel");
}

extern "C" int ttsb_repack_batched(const ttsb_pack_desc* descs_device, int n, void* stream) {
  if (!descs_device || n <= 0) return bad("ttsb_repack_batched: bad arguments");
  repack_batched_kernel<<<dim3(48, n), 256, 0, STREAM(stream)>>>(descs_device);
  LAUNCH_OK("repack_batched_kernel");
}

extern "C" int ttsb_split_bf16(const float* x, int64_t n, void* x_hi, void* x_lo, void* stream) {
  if (!x || !x_hi || n < 0) return bad("ttsb_split_bf16: bad arguments");
  if (n == 0) return 0;
  split_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, STREAM(stream)>>>(x, n, static_cast<__nv_bfloat16*>(x_hi),
                                                                           static_cast<__nv_bfloat16*>(x_lo));
  LAUNCH_OK("split_bf16_kernel");
}

extern "C" int ttsb_embed_ln_pe_train_fwd(const int32_t* tokens, const float* emb, const float* gamma, const float* beta,
                                          const float* pe, const float* pos_scalar, int B, int T, int d, int vocab, float eps,
                                          float drop_p, uint32_t seed, uint32_t site, float* out_f32, void* out_hi, void* out_lo,
                                          void* stream) {
  if (!tokens || !emb || !gamma || !beta || !pe || !pos_scalar) return bad("ttsb_embed_ln_pe_fwd: NULL input");
  if (B <= 0 || T <= 0 || d <= 0 || d % 4 || d > 128 * ROW_MAX_V4 || vocab <= 0) return bad("ttsb_embed_ln_pe_fwd: need d % 4 == 0, d <= 512");
  const int rows = B * T;
  embed_ln_pe_kernel<<<(rows + 7) / 8, 256, 0, STREAM(stream)>>>(tokens, emb, gamma, beta, pe, pos_scalar, rows, T, d, vocab, eps,
                                                                out_f32, static_cast<__nv_bfloat16*>(out_hi),
                                                                static_cast<__nv_bfloat16*>(out_lo), drop_p, seed, site);
  LAUNCH_OK("embed_ln_pe_kernel");
}

extern "C" int ttsb_embed_ln_pe_fwd(const int32_t* tokens, const float* emb, const float* gamma, const float* beta,
                                    const float* pe, const float* pos_scalar, int B, int T, int d, int vocab, float eps,
                                    float* out_f32, void* out_hi, void* out_lo, void* stream) {
  return ttsb_embed_ln_pe_train_fwd(tokens, emb, gamma, beta, pe, pos_scalar, B, T, d, vocab, eps, 0.f, 0u, 0u, out_f32, out_hi, out_lo, stream);
}

extern "C" int ttsb_expand_ln_pe_train_fwd(const float* x, const int32_t* idx, const float* gamma, const float* beta, const float* pe,
                                           const float* pos_scalar, int B, int Tp, int Tm, int d, float eps, float drop_p, uint32_t seed,
                                           uint32_t site, float* out_f32, void* out_hi, void* out_lo, void* stream) {
  if (!x || !idx || !gamma || !beta || !pe || !pos_scalar) return bad("ttsb_expand_ln_pe_fwd: NULL input");
  if (B <= 0 || Tp <= 0 || Tm < 0 || d <= 0 || d % 4 || d > 128 * ROW_MAX_V4) return bad("ttsb_expand_ln_pe_fwd: need d % 4 == 0, d <= 512");
  if (Tm == 0) return 0;
  const int rows = B * Tm;
  expand_ln_pe_kernel<<<(rows + 7) / 8, 256, 0, STREAM(stream)>>>(x, idx, gamma, beta, pe, pos_scalar, B, Tp, Tm, d, eps, out_f32,
                                                                 static_cast<__nv_bfloat16*>(out_hi),
                                                                 static_cast<__nv_bfloat16*>(out_lo), drop_p, seed, site);
  LAUNCH_OK("expand_ln_pe_kernel");
}

extern "C" int ttsb_expand_ln_pe_fwd(const float* x, const int32_t* idx, const float* gamma, const float* beta, const float* pe,
                                     const float* pos_scalar, int B, int Tp, int Tm, int d, float eps, float* out_f32, void* out_hi,
                                     void* out_lo, void* stream) {
  return ttsb_expand_ln_pe_train_fwd(x, idx, gamma, beta, pe, pos_scalar, B, Tp, Tm, d, eps, 0.f, 0u, 0u, out_f32, out_hi, out_lo, stream);
}

extern "C" int ttsb_decode_prologue(const float* x, const int32_t* pos, const float* gamma, const float* beta, const float* pe, int pe_rows,
                                    const float* pos_scalar, int B, int d, float eps, float* out_f32, void* out_hi, void* out_lo,
                                    void* stream) {
  if (!x || !pos || !gamma || !beta || !pe || !pos_scalar) return bad("ttsb_decode_prologue: NULL input");
  if (B <= 0 || pe_rows <= 0 || d <= 0 || d % 4 || d > 128 * ROW_MAX_V4) return bad("ttsb_decode_prologue: need B, pe_rows > 0, d % 4 == 0, d <= 512");
  decode_prologue_kernel<<<(B + 7) / 8, 256, 0, STREAM(stream)>>>(x, pos, gamma, beta, pe, pe_rows, pos_scalar, B, d, eps, out_f32,
                                                                  static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo));
  LAUNCH_OK("decode_prologue_kernel");
}

extern "C" int ttsb_layernorm_fwd(const float* x, const float* gamma, const float* beta, int B, int T, int d, int ld, float eps,
                                  const int32_t* row_len, float* out_f32, void* out_hi, void* out_lo, void* stream) {
  if (!x || !gamma || !beta) return bad("ttsb_layernorm_fwd: NULL input");
  if (B <= 0 || T <= 0 || d <= 0 || d % 4 || d > 128 * ROW_MAX_V4 || ld < d || ld % 4) return bad("ttsb_layernorm_fwd: need d % 4 == 0, d <= 512");
  const int rows = B * T;
  layernorm_fwd_kernel<<<(rows + 7) / 8, 256, 0, STREAM(stream)>>>(x, gamma, beta, rows, T, d, ld, eps, row_len, out_f32,
                                                                  static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo));
  LAUNCH_OK("layernorm_fwd_kernel");
}

extern "C" int ttsb_length_regulate_fwd(const float* x, const int32_t* idx, int B, int Tp, int Tm, int d, float* out, void* stream) {
  if (!x || !idx || !out) return bad("ttsb_length_regulate_fwd: NULL input");
  if (B <= 0 || Tp <= 0 || Tm < 0 || d <= 0 || d % 4) return bad("ttsb_length_regulate_fwd: need d % 4 == 0");
  if (Tm == 0) return 0;
  const int rows = B * Tm;
  length_regulate_kernel<<<(rows + 7) / 8, 256, 0, STREAM(stream)>>>(x, idx, B, Tp, Tm, d, out);
  LAUNCH_OK("length_regulate_kernel");
}

extern "C" int ttsb_durations_to_int(const float* dur, float scalar, const float* max_mask, const float* min_mask, int B, int Tp,
                                     int32_t* out_int, int32_t* out_len, void* stream) {
  if (!dur || !out_int || !out_len || B <= 0 || Tp <= 0) return bad("ttsb_durations_to_int: bad arguments");
  durations_to_int_kernel<<<B, 256, 0, STREAM(stream)>>>(dur, scalar, max_mask, min_mask, Tp, out_int, out_len);
  LAUNCH_OK("durations_to_int_kernel");
}

extern "C" int ttsb_expand_indices(const int32_t* dur_int, int B, int Tp, int Tm, int32_t* out_idx, void* stream) {
  if (!dur_int || !out_idx || B <= 0 || Tp <= 0 || Tm < 0) return bad("ttsb_expand_indices: bad arguments");
  if (Tp > 12000) return bad("ttsb_expand_indices: Tp too large for the shared-memory scan");
  if (Tm == 0) return 0;
  expand_indices_kernel<<<B, 1024, Tp * sizeof(int), STREAM(stream)>>>(dur_int, Tp, Tm, out_idx);
  LAUNCH_OK("expand_indices_kernel");
}

extern "C" int ttsb_statpred_head_fwd(const float* h, int ldh, int C, const float* w, const float* bias, int relu,
                                      const int32_t* row_len, int B, int T, float* out, void* stream) {
  if (!h || !w || !bias || !out || B <= 0 || T <= 0 || C <= 0 || ldh < C) return bad("ttsb_statpred_head_fwd: bad arguments");
  const int rows = B * T;
  statpred_head_kernel<<<(rows + 7) / 8, 256, 0, STREAM(stream)>>>(h, ldh, C, w, bias, relu, row_len, rows, T, out);
  LAUNCH_OK("statpred_head_kernel");
}

extern "C" int ttsb_pitch_embed_add_fwd(const float* x, const float* pitch, const float* w, const float* bias, int B, int T, int d,
                                        float* out, void* stream) {
  if (!x || !pitch || !w || !bias || !out || B <= 0 || T <= 0 || d <= 0 || d % 4) return bad("ttsb_pitch_embed_add_fwd: bad arguments");
  const int64_t n4 = (int64_t)B * T * d / 4;
  pitch_embed_add_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, STREAM(stream)>>>(x, pitch, w, bias, n4, d / 4, out);
  LAUNCH_OK("pitch_embed_add_kernel");
}

extern "C" int ttsb_mel_lengths(const float* mel, int B, int T, int C, float padding_value, int32_t* out, void* stream) {
  if (!mel || !out || B <= 0 || T <= 0 || C <= 0) return bad("ttsb_mel_lengths: bad arguments");
  TTSB_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(int32_t) * (size_t)B, STREAM(stream)));
  mel_lengths_kernel<<<dim3(B, (T + 63) / 64), 256, 0, STREAM(stream)>>>(mel, T, C, padding_value, out);
  LAUNCH_OK("mel_lengths_kernel");
}

extern "C" int ttsb_phoneme_lengths(const int32_t* phonemes, int B, int T, int32_t padding, int32_t* out, void* stream) {
  if (!phonemes || !out || B <= 0 || T <= 0) return bad("ttsb_phoneme_lengths: bad arguments");
  phoneme_lengths_kernel<<<B, 256, 0, STREAM(stream)>>>(phonemes, T, padding, out);
  LAUNCH_OK("phoneme_lengths_kernel");
}

TTSB_DEFINE_SALT_SETTER(set_salt_rowops)
