// Cached autoregressive decoding of the Aligner (model/models.py:271-292): single-query attention over a key/value cache and
// the end-of-iteration commit (mel frames, next decoder input, stop decision).
//
// ttsb_decode_attn is flash-decoding: one query row per (sentence, head), so the work is reading K and V once.  A CTA of four
// warps owns a contiguous key range; inside it a key row is read by dh/8 lanes with one 16-byte load each, so a warp covers
// 32*8/dh keys per load.  Logits of the range stay in shared memory (fp32), the softmax is exact over the range, and P V is
// accumulated in fp32 per lane.  When B*H CTAs would leave most of the 132 SMs idle, the keys are split over several CTAs
// that park (max, sum, unnormalised output) in the workspace; the last CTA to arrive (atomic counter) combines them in split
// order and resets the counter, so the result does not depend on which CTA finished last.
#include <cuda_fp16.h>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace ttsb {

constexpr int DA_THREADS = 128;
constexpr int DA_WARPS = DA_THREADS / 32;
constexpr int DA_MAX_SPLIT = 32;     // CTAs per (b, h) at most
constexpr int DA_MAX_CHUNK = 8192;   // keys per CTA at most: the logits of the range live in 32 KB of shared memory
constexpr int DA_UNROLL = 4;         // independent 16-byte loads in flight per lane

struct DecodeAttnParams {
  int B, H, Tk;
  const uint16_t* q;
  int ld_q, q_col0;
  uint16_t* kv;
  int ld_kv, k_col0, v_col0;
  const uint16_t* nkv;  // null: cross mode
  int ld_new, nk_col0, nv_col0;
  const int* pos;
  const int* kv_len;
  const int* done;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  int ld_out;
  float* probs;
  int probs_T;
  int n_split, chunk;
  float scale;
  int* counters;   // [B*H]
  float* partial;  // [B*H][DA_MAX_SPLIT][2 + dh]: max, sum, unnormalised output
};

template <bool F16>
__device__ __forceinline__ void cvt8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t;
    if constexpr (F16) t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
    else t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, w) : v + w;
  }
  __syncthreads();  // red[] may still be read by the previous reduction
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[0];
#pragma unroll
  for (int w = 1; w < DA_WARPS; ++w) v = is_max ? fmaxf(v, red[w]) : v + red[w];
  return v;
}

template <int DH, bool F16>
__global__ void __launch_bounds__(DA_THREADS) decode_attn_kernel(const DecodeAttnParams p) {
  constexpr int G = DH / 8;             // lanes per key row
  constexpr int KPW = 32 / G;           // keys per warp and load
  constexpr int KPB = KPW * DA_WARPS;   // keys per CTA and load
  extern __shared__ float sm_logit[];   // [chunk]
  __shared__ float sm_o[DA_WARPS][DH];
  __shared__ float sm_red[DA_WARPS];
  __shared__ float sm_f[DA_MAX_SPLIT];
  __shared__ int sm_last;
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  if (p.done && __ldg(p.done + b)) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane / G, gl = lane % G;  // key slot inside the warp, 8-column slice of the head
  const bool self = p.nkv != nullptr;
  const int pos = __ldg(p.pos + b);
  const int len = self ? min(max(pos + 1, 1), p.Tk) : min(max(__ldg(p.kv_len + b), 1), p.Tk);
  const int k0 = split * p.chunk;
  const int k1 = min(k0 + p.chunk, len);       // keys attended by this CTA
  const int kend = min(k0 + p.chunk, p.Tk);    // columns of the probability row written by this CTA
  const int n_live = (len + p.chunk - 1) / p.chunk;  // CTAs of (b, h) whose range holds keys at this length (>= 1)
  const int n = max(k1 - k0, 0);
  const size_t kv_row0 = (size_t)b * p.Tk;
  float* prow = p.probs && pos >= 0 && pos < p.probs_T ? p.probs + (((size_t)b * p.H + h) * p.probs_T + pos) * p.Tk : nullptr;
  const uint16_t* new_row = self ? p.nkv + (size_t)b * p.ld_new : nullptr;

  // self mode: the new key / value row goes into the cache (split 0 writes it; no CTA of this launch reads it back from there)
  if (self && split == 0 && pos >= 0 && pos < p.Tk && tid < 2 * G) {
    const int kv_sel = tid / G, c = (tid % G) * 8;
    const uint4 v = *reinterpret_cast<const uint4*>(new_row + (kv_sel ? p.nv_col0 : p.nk_col0) + h * DH + c);
    *reinterpret_cast<uint4*>(p.kv + (kv_row0 + pos) * p.ld_kv + (kv_sel ? p.v_col0 : p.k_col0) + h * DH + c) = v;
  }
  // The split is sized for the capacity Tk (the grid is fixed, e.g. inside a captured step), so while the self-attention cache
  // is short most CTAs hold no key: they write the zero tail of the probability row and leave without taking part in the
  // combine, which then spans the n_live CTAs that do.
  if (split >= n_live) {
    if (prow)
      for (int i = k0 + tid; i < kend; i += DA_THREADS) prow[i] = 0.f;
    return;
  }
  auto load_row = [&](int key, int col0, int ncol0) -> uint4 {
    if (self && key == pos) return *reinterpret_cast<const uint4*>(new_row + ncol0 + h * DH + gl * 8);
    return __ldg(reinterpret_cast<const uint4*>(p.kv + (kv_row0 + key) * p.ld_kv + col0 + h * DH + gl * 8));
  };

  float qf[8];
  cvt8<F16>(__ldg(reinterpret_cast<const uint4*>(p.q + (size_t)b * p.ld_q + p.q_col0 + h * DH + gl * 8)), qf);

  // ---- logits of the key range (loop bounds are warp-uniform: the shuffles see every lane)
  for (int base = k0 + warp * KPW; base < k1; base += KPB * DA_UNROLL) {
    uint4 kr[DA_UNROLL];
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) {
      const int key = base + u * KPB + g;
      kr[u] = key < k1 ? load_row(key, p.k_col0, p.nk_col0) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) {
      float kf[8];
      cvt8<F16>(kr[u], kf);
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(qf[j], kf[j], acc);
#pragma unroll
      for (int o = G / 2; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      const int key = base + u * KPB + g;
      if (gl == 0 && key < k1) sm_logit[key - k0] = acc * p.scale;
    }
  }
  __syncthreads();
  // ---- softmax over the range
  float m = -INFINITY;
  for (int i = tid; i < n; i += DA_THREADS) m = fmaxf(m, sm_logit[i]);
  m = block_reduce(m, sm_red, true);
  float s = 0.f;
  for (int i = tid; i < n; i += DA_THREADS) {
    const float e = expf(sm_logit[i] - m);
    sm_logit[i] = e;
    s += e;
  }
  s = block_reduce(s, sm_red, false);  // its barriers also publish the exponentials
  // ---- P V
  float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int base = k0 + warp * KPW; base < k1; base += KPB * DA_UNROLL) {
    uint4 vr[DA_UNROLL];
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) {
      const int key = base + u * KPB + g;
      vr[u] = key < k1 ? load_row(key, p.v_col0, p.nv_col0) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) {
      const int key = base + u * KPB + g;
      const float pk = key < k1 ? sm_logit[key - k0] : 0.f;
      float vf[8];
      cvt8<F16>(vr[u], vf);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf(pk, vf[j], o[j]);
    }
  }
#pragma unroll
  for (int off = G; off < 32; off <<= 1)
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] += __shfl_xor_sync(0xffffffffu, o[j], off);
  if (g == 0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) sm_o[warp][gl * 8 + j] = o[j];
  }
  __syncthreads();

  const size_t out_row = (size_t)b * p.ld_out + h * DH;
  if (n_live == 1) {
    const float inv = 1.f / s;
    if (prow)
      for (int i = k0 + tid; i < kend; i += DA_THREADS) prow[i] = i < k1 ? sm_logit[i - k0] * inv : 0.f;
    for (int c = tid; c < DH; c += DA_THREADS) {
      float acc = 0.f;
#pragma unroll
      for (int w = 0; w < DA_WARPS; ++w) acc += sm_o[w][c];
      __nv_bfloat16 hi, lo;
      split_bf16(acc * inv, hi, lo);
      p.out_hi[out_row + c] = hi;
      if (p.out_lo) p.out_lo[out_row + c] = lo;
    }
    return;
  }

  // ---- split keys: park the partial result, the last CTA of (b, h) combines
  const int bh = b * p.H + h;
  float* part = p.partial + ((size_t)bh * DA_MAX_SPLIT + split) * (2 + DH);
  if (tid == 0) { part[0] = m; part[1] = s; }
  for (int c = tid; c < DH; c += DA_THREADS) {
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < DA_WARPS; ++w) acc += sm_o[w][c];
    part[2 + c] = acc;
  }
  if (prow)  // unnormalised exponentials; the combining CTA rescales them
    for (int i = k0 + tid; i < kend; i += DA_THREADS) prow[i] = i < k1 ? sm_logit[i - k0] : 0.f;
  __threadfence();
  __syncthreads();
  if (tid == 0) sm_last = atomicAdd(p.counters + bh, 1) == n_live - 1;
  __syncthreads();
  if (!sm_last) return;
  __threadfence();
  const float* parts = p.partial + (size_t)bh * DA_MAX_SPLIT * (2 + DH);
  if (tid == 0) {
    float mx = -INFINITY;
    for (int i = 0; i < n_live; ++i) mx = fmaxf(mx, __ldcg(parts + (size_t)i * (2 + DH)));
    float sum = 0.f;
    for (int i = 0; i < n_live; ++i) {
      const float f = expf(__ldcg(parts + (size_t)i * (2 + DH)) - mx);
      sm_f[i] = f;
      sum += __ldcg(parts + (size_t)i * (2 + DH) + 1) * f;
    }
    const float inv = 1.f / sum;
    for (int i = 0; i < n_live; ++i) sm_f[i] *= inv;
    p.counters[bh] = 0;  // ready for the next launch
  }
  __syncthreads();
  for (int c = tid; c < DH; c += DA_THREADS) {
    float acc = 0.f;
    for (int i = 0; i < n_live; ++i) acc += __ldcg(parts + (size_t)i * (2 + DH) + 2 + c) * sm_f[i];
    __nv_bfloat16 hi, lo;
    split_bf16(acc, hi, lo);
    p.out_hi[out_row + c] = hi;
    if (p.out_lo) p.out_lo[out_row + c] = lo;
  }
  if (prow)
    for (int i = tid; i < len; i += DA_THREADS) prow[i] = __ldcg(prow + i) * sm_f[i / p.chunk];
}

// ---- end of one decode iteration: one warp per sentence, one CTA
__global__ void decode_commit_kernel(const float* __restrict__ post, int ld_post, int B, int r, int mel, int stop_col,
                                     int stop_index, int max_iters, float* mel_out, float* stop_out, __nv_bfloat16* next_hi,
                                     __nv_bfloat16* next_lo, int ld_next, int* pos, int* done, int* n, int* all_done) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int all = 1;
  for (int b = warp; b < B; b += nw) {
    if (done[b]) continue;  // warp-uniform
    const int ps = pos[b];
    const float* src = post + (size_t)b * r * ld_post;
    const size_t f0 = (size_t)b * max_iters * r + (size_t)ps * r;  // first output frame of this iteration
    for (int i = lane; i < r * mel; i += 32) {
      const int j = i / mel, c = i - j * mel;
      mel_out[f0 * mel + i] = src[(size_t)j * ld_post + c];
    }
    if (stop_out)
      for (int i = lane; i < r * 3; i += 32) stop_out[f0 * 3 + i] = src[(size_t)(i / 3) * ld_post + stop_col + i % 3];
    const float* last = src + (size_t)(r - 1) * ld_post;
    for (int c = lane; c < mel; c += 32) {  // models.py:280: the last predicted frame is the next input
      __nv_bfloat16 hi, lo;
      split_bf16(last[c], hi, lo);
      next_hi[(size_t)b * ld_next + c] = hi;
      if (next_lo) next_lo[(size_t)b * ld_next + c] = lo;
    }
    // models.py:287: tf.argmax (the first maximal index) of the last stop distribution
    int am = 0;
    float best = last[stop_col];
    for (int k = 1; k < 3; ++k)
      if (last[stop_col + k] > best) { best = last[stop_col + k]; am = k; }
    const int cnt = ps + 1;
    const bool fin = am == stop_index || cnt >= max_iters;
    __syncwarp();
    if (lane == 0) {
      n[b] = cnt;
      if (fin) done[b] = 1;
      else pos[b] = cnt;
    }
    if (!fin) all = 0;
  }
  all = __syncthreads_and(all);
  if (threadIdx.x == 0) *all_done = all;
}

static int bad(const char* msg) {
  set_last_error("%s", msg);
  return TTSB_ERR_INVALID_ARGUMENT;
}

// keys per CTA: about two CTAs per SM over all (b, h), at least 64 keys per CTA, at most DA_MAX_SPLIT CTAs per (b, h)
static void decode_split(int B, int H, int Tk, int* n_split, int* chunk) {
  const int bh = B * H;
  int want = (2 * num_sms() + bh - 1) / bh;
  want = want < 1 ? 1 : (want > DA_MAX_SPLIT ? DA_MAX_SPLIT : want);
  int c = (Tk + want - 1) / want;
  c = c < 64 ? 64 : (c + 31) / 32 * 32;
  if ((int64_t)c * DA_MAX_SPLIT < Tk) c = (Tk + DA_MAX_SPLIT - 1) / DA_MAX_SPLIT;
  *chunk = c;
  *n_split = (Tk + c - 1) / c;
}

static int64_t counters_bytes(int B, int H) { return ((int64_t)B * H * 4 + 255) / 256 * 256; }

template <int DH>
static int launch_decode_attn(const DecodeAttnParams& p, bool f16, cudaStream_t stream) {
  const dim3 grid(p.n_split, p.H, p.B);
  const size_t smem = (size_t)p.chunk * sizeof(float);
  if (f16) decode_attn_kernel<DH, true><<<grid, DA_THREADS, smem, stream>>>(p);
  else decode_attn_kernel<DH, false><<<grid, DA_THREADS, smem, stream>>>(p);
  count_launch();
  return check_cuda(cudaGetLastError(), "decode_attn_kernel launch");
}

}  // namespace ttsb

using namespace ttsb;

extern "C" int64_t ttsb_decode_attn_workspace_bytes(int B, int H, int dh) {
  if (B <= 0 || H <= 0 || dh <= 0) return 0;
  return counters_bytes(B, H) + (int64_t)B * H * DA_MAX_SPLIT * (2 + dh) * (int64_t)sizeof(float);
}

extern "C" int ttsb_decode_attn(const ttsb_decode_attn_args* a, void* stream) {
  if (!a) return bad("ttsb_decode_attn: args is NULL");
  if (a->B <= 0 || a->H <= 0 || a->Tk <= 0) return bad("ttsb_decode_attn: B, H and Tk must be positive");
  if (a->dh != 64 && a->dh != 128 && a->dh != 256) {
    set_last_error("ttsb_decode_attn: head size %d is not supported (64, 128, 256)", a->dh);
    return TTSB_ERR_UNSUPPORTED;
  }
  if (a->precision != TTSB_PREC_FP16 && a->precision != TTSB_PREC_BF16) {
    set_last_error("ttsb_decode_attn: precision must be TTSB_PREC_FP16 or TTSB_PREC_BF16 (single-pass 16-bit operands)");
    return TTSB_ERR_UNSUPPORTED;
  }
  const bool self = a->new_kv != nullptr;
  if (!a->q || !a->kv || !a->pos || !a->out_hi || !a->workspace || (!self && !a->kv_len))
    return bad("ttsb_decode_attn: NULL tensor (q, kv, pos, out_hi, workspace; kv_len in cross mode)");
  const int hd = a->H * a->dh;
  if (a->ld_q % 8 || a->q_col0 % 8 || a->ld_kv % 8 || a->k_col0 % 8 || a->v_col0 % 8 ||
      (self && (a->ld_new % 8 || a->new_k_col0 % 8 || a->new_v_col0 % 8)))
    return bad("ttsb_decode_attn: leading dimensions and column offsets must be multiples of 8 (16-byte loads)");
  if (a->q_col0 + hd > a->ld_q || a->k_col0 + hd > a->ld_kv || a->v_col0 + hd > a->ld_kv || a->ld_out < hd ||
      (self && (a->new_k_col0 + hd > a->ld_new || a->new_v_col0 + hd > a->ld_new)))
    return bad("ttsb_decode_attn: H*dh columns from a column offset exceed a leading dimension");
  if (a->probs && a->probs_T <= 0) return bad("ttsb_decode_attn: probs_T must be positive with probs");
  if (a->workspace_bytes < ttsb_decode_attn_workspace_bytes(a->B, a->H, a->dh))
    return bad("ttsb_decode_attn: workspace smaller than ttsb_decode_attn_workspace_bytes");
  DecodeAttnParams p{};
  p.B = a->B; p.H = a->H; p.Tk = a->Tk;
  p.q = static_cast<const uint16_t*>(a->q); p.ld_q = a->ld_q; p.q_col0 = a->q_col0;
  p.kv = static_cast<uint16_t*>(a->kv); p.ld_kv = a->ld_kv; p.k_col0 = a->k_col0; p.v_col0 = a->v_col0;
  p.nkv = static_cast<const uint16_t*>(a->new_kv); p.ld_new = a->ld_new; p.nk_col0 = a->new_k_col0; p.nv_col0 = a->new_v_col0;
  p.pos = a->pos; p.kv_len = a->kv_len; p.done = a->done;
  p.out_hi = static_cast<__nv_bfloat16*>(a->out_hi);
  p.out_lo = static_cast<__nv_bfloat16*>(a->out_lo);
  p.ld_out = a->ld_out;
  p.probs = a->probs; p.probs_T = a->probs_T;
  decode_split(a->B, a->H, a->Tk, &p.n_split, &p.chunk);
  if (p.chunk > DA_MAX_CHUNK) {
    set_last_error("ttsb_decode_attn: Tk = %d exceeds %d keys", a->Tk, DA_MAX_CHUNK * DA_MAX_SPLIT);
    return TTSB_ERR_UNSUPPORTED;
  }
  p.scale = 1.f / sqrtf((float)a->dh);
  p.counters = static_cast<int*>(a->workspace);
  p.partial = reinterpret_cast<float*>(static_cast<uint8_t*>(a->workspace) + counters_bytes(a->B, a->H));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool f16 = a->precision == TTSB_PREC_FP16;
  if (a->dh == 64) return launch_decode_attn<64>(p, f16, s);
  if (a->dh == 128) return launch_decode_attn<128>(p, f16, s);
  return launch_decode_attn<256>(p, f16, s);
}

extern "C" int ttsb_decode_commit(const float* post, int ld_post, int B, int r, int mel, int stop_col, int stop_index, int max_iters,
                                  float* mel_out, float* stop_out, void* next_hi, void* next_lo, int ld_next, int32_t* pos,
                                  int32_t* done, int32_t* n, int32_t* all_done, void* stream) {
  if (!post || !mel_out || !next_hi || !pos || !done || !n || !all_done) return bad("ttsb_decode_commit: NULL tensor");
  if (B <= 0 || r <= 0 || mel <= 0 || max_iters <= 0 || stop_index < 0 || stop_index > 2)
    return bad("ttsb_decode_commit: B, r, mel and max_iters must be positive and stop_index in [0, 3)");
  if (stop_col < mel || ld_post < stop_col + 3 || ld_next < mel)
    return bad("ttsb_decode_commit: need stop_col >= mel, ld_post >= stop_col + 3 and ld_next >= mel");
  decode_commit_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(post, ld_post, B, r, mel, stop_col, stop_index, max_iters,
                                                                       mel_out, stop_out, static_cast<__nv_bfloat16*>(next_hi),
                                                                       static_cast<__nv_bfloat16*>(next_lo), ld_next, pos, done, n,
                                                                       all_done);
  count_launch();
  return check_cuda(cudaGetLastError(), "decode_commit_kernel launch");
}
