// The WaveRNN generator's sample-rate recurrence (fatchord/WaveRNN, models/fatchord_version.py: generate), every step of every
// fold of every clip in one persistent cooperative launch, then the fold crossfade (xfade_and_unfold), crop and fade-out.
//
// Rows are the folds of all clips.  The frame-rate conditioning (the MelResNet output's projections and each mel frame's
// projection) comes from ttsb_conv1d_ex_tc; per step a row adds sum_j K[p][j] P[f + j] for the mel and the aux projection of
// its frame (zero past the clip, as fatchord's zero-padded last fold has it).  Because I's only recurrent input is the
// previous sample, I is folded into the GRU1 phase: W_ih1 x = x_prev (W_ih1 I_0) + W_ih1 (conditioning), the second term
// projected at frame rate.
//
// Weight-stationary: CTA b of WR_CTAS owns hidden units [4b, 4b + 4) of both GRUs (their r, z and n rows together, so the
// gates finish in the phase that computes them), of fc1 and of fc2, and ceil(n_classes / WR_CTAS) rows of fc3; those rows
// stay in shared memory for the whole call (fp32 in bf16x3, bf16 in bf16).  Activations and hidden states go through L2
// (fp32, ld.global.cg).  One step is five phases with a grid barrier after each:
//   1. sample x_prev of every row from the previous logits (every CTA, redundantly), GRU1   -> h1, x + h1
//   2. GRU2                                                                                -> h2, x + h1 + h2
//   3. fc1, 4. fc2, 5. fc3                                                                 -> logits
// A warp takes 8 rows at a time, lane = 4 row + k quarter; every dot product is summed in a fixed k order (per lane in k
// order, then lanes 0+1, 2+3, then the pairs), so a row's arithmetic depends on neither the number of rows nor its place.
//
// Random numbers are counter-based (splitmix64 of seed, fold, step, draw), restated in numpy in oracle/wavernn_oracle.py.
#include <cooperative_groups.h>

#include <algorithm>
#include <type_traits>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace cg = cooperative_groups;

namespace ttsb {

constexpr int WR_D = TTSB_WAVERNN_DIMS;   // rnn_dims = fc_dims
constexpr int WR_CTAS = WR_D / 4;         // 128 slices of 4 units
static_assert(WR_CTAS == TTSB_WAVERNN_CTAS, "the header's CTA count");
constexpr int WR_THREADS = 512;
constexpr int WR_WARPS = WR_THREADS / 32;
constexpr int WR_MAX_FC3 = 8;             // fc3 rows per CTA: 1024 classes / 128
// vec offsets (fp32)
constexpr int V_I0 = 0, V_BX = 512, V_U1 = 1024, V_BG1 = 2560, V_BHH1 = 4096, V_BG2 = 5632, V_BHH2 = 7168, V_B3 = 8704,
              V_B4 = 9216, V_B5 = 9728;
// weight rows (each WR_D wide)
constexpr int W_HH1 = 0, W_IH2 = 1536, W_HH2 = 3072, W_FC1 = 4608, W_FC2 = 5120, W_FC3 = 5632;
// conditioning columns
constexpr int C_PX = 0, C_PG1 = 512;                                   // mel projection
constexpr int C_AX = 0, C_AG1 = 512, C_AG2 = 2048, C_A3 = 3584, C_A4 = 4096;   // aux projection
constexpr int SMEM_ROWS = 12 + 12 + 12 + 4 + 4;                         // + fc3 rows

constexpr int WR_SEGS = 6;   // timed segments of a step: sampling, GRU1, GRU2, fc1, fc2, fc3

struct WrParams {
  int R, L, n_taps, hop, nc, ncp, q, mode, cap;
  const int4* rows;        // (clip, fold, first, valid)
  const int32_t* row0;     // per clip: conditioning row of frame 0
  const uint32_t* seeds;   // per clip
  const float* taps;
  const __nv_bfloat16 *mp_hi, *mp_lo, *ax_hi, *ax_lo;
  int ld_mp, ld_ax;
  const float* vec;
  const void* w;
  float *h1, *h2, *x2, *x3, *f1, *f2, *logits, *samples, *capture;
  int64_t* timings;   // NULL, or (WR_CTAS, 2 WR_SEGS): per CTA and segment, ns of work and of the barrier after it
};

__device__ __forceinline__ uint64_t wr_mix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// uniform in [1e-5, 1 - 1e-5] keyed by (seed, fold, step, draw): (23 hash bits + 0.5) 2^-23, clamped
__device__ __forceinline__ float wr_uniform(uint32_t seed, uint32_t fold, uint32_t step, uint32_t draw) {
  uint64_t z = wr_mix(((uint64_t)seed << 32) | fold);
  z = wr_mix(z ^ (((uint64_t)step << 8) | draw));
  const float v = ((float)(uint32_t)(z >> 41) + 0.5f) * 0x1p-23f;
  return fminf(fmaxf(v, 1e-5f), 1.0f - 1e-5f);
}

__device__ __forceinline__ float wr_cond(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int64_t idx) {
  float v = __bfloat162float(hi[idx]);
  if (lo) v += __bfloat162float(lo[idx]);
  return v;
}

__device__ __forceinline__ uint64_t wr_now() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ float wr_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

template <bool kBf16>
__device__ __forceinline__ float4 wr_ldw(const void* sw, int idx) {
  if constexpr (kBf16) {
    const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(sw) + idx);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  } else {
    return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(sw) + idx);
  }
}

template <bool kBf16>
__device__ __forceinline__ float4 wr_lda(const float* p) {
  float4 a = __ldcg(reinterpret_cast<const float4*>(p));
  if constexpr (kBf16) {
    a.x = __bfloat162float(__float2bfloat16_rn(a.x));
    a.y = __bfloat162float(__float2bfloat16_rn(a.y));
    a.z = __bfloat162float(__float2bfloat16_rn(a.z));
    a.w = __bfloat162float(__float2bfloat16_rn(a.w));
  }
  return a;
}

// acc[m] = sum_k W[m0 + m][k] act[r][k] over k in [0, 512) for M (<= kM) smem rows, summed over the 4 lanes of the row
template <bool kBf16, int kM>
__device__ __forceinline__ void wr_matvec(const void* sw, int m0, int M, const float* act, int r, int kq, float (&acc)[kM]) {
#pragma unroll
  for (int m = 0; m < kM; ++m) acc[m] = 0.f;
  const float* a = act + (int64_t)r * WR_D + 4 * kq;
#pragma unroll 4
  for (int i = 0; i < WR_D / 16; ++i) {
    const float4 av = wr_lda<kBf16>(a + 16 * i);
#pragma unroll
    for (int m = 0; m < kM; ++m) {
      if (m < M) {
        const float4 wv = wr_ldw<kBf16>(sw, (m0 + m) * WR_D + 16 * i + 4 * kq);
        acc[m] = fmaf(wv.x, av.x, acc[m]);
        acc[m] = fmaf(wv.y, av.y, acc[m]);
        acc[m] = fmaf(wv.z, av.z, acc[m]);
        acc[m] = fmaf(wv.w, av.w, acc[m]);
      }
    }
  }
#pragma unroll
  for (int m = 0; m < kM; ++m) {
    acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], 1);
    acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], 2);
  }
}

template <int kM>
__device__ __forceinline__ float wr_pick(const float (&acc)[kM], int m) {
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < kM; ++i)
    if (i == m) v = acc[i];
  return v;
}

// the sample of row r drawn from the logits of step `step` (one warp; every lane returns it)
__device__ float wr_sample(const WrParams& p, int r, int step) {
  const int lane = threadIdx.x & 31;
  const int4 row = p.rows[r];
  const uint32_t seed = p.seeds[row.x];
  const float* lg = p.logits + (int64_t)r * p.ncp;
  if (p.mode == TTSB_WAVERNN_MOL) {
    float score = -INFINITY;
    int idx = 1 << 30;
    if (lane < 10) {
      const float u = wr_uniform(seed, (uint32_t)row.y, (uint32_t)step, (uint32_t)lane);
      score = __ldcg(lg + lane) - logf(-logf(u));
      idx = lane;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float s2 = __shfl_xor_sync(0xffffffffu, score, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, idx, o);
      if (s2 > score || (s2 == score && i2 < idx)) { score = s2; idx = i2; }
    }
    const float mu = __ldcg(lg + 10 + idx);
    const float ls = fmaxf(__ldcg(lg + 20 + idx), -32.23619130191664f);   // log(1e-14)
    const float u = wr_uniform(seed, (uint32_t)row.y, (uint32_t)step, 10u);
    const float x = mu + expf(ls) * (logf(u) - logf(1.0f - u));
    return fminf(fmaxf(x, -1.0f), 1.0f);
  }
  // RAW: softmax and the inverse CDF of one uniform; lane l owns classes [l c, (l + 1) c)
  const int c = p.nc / 32;
  float mx = -INFINITY;
  for (int i = 0; i < c; ++i) mx = fmaxf(mx, __ldcg(lg + lane * c + i));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float part = 0.f;
  for (int i = 0; i < c; ++i) part += expf(__ldcg(lg + lane * c + i) - mx);
  float incl = part;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const float total = __shfl_sync(0xffffffffu, incl, 31);
  const float target = wr_uniform(seed, (uint32_t)row.y, (uint32_t)step, 0u) * total;
  const unsigned hit = __ballot_sync(0xffffffffu, incl > target);
  const int owner = hit ? __ffs(hit) - 1 : 31;
  int k = owner * c + c - 1;
  if (lane == owner) {
    float run = incl - part;
    for (int i = 0; i < c; ++i) {
      run += expf(__ldcg(lg + lane * c + i) - mx);
      if (run > target) { k = lane * c + i; break; }
    }
  }
  k = __shfl_sync(0xffffffffu, k, owner);
  return 2.0f * (float)k / (float)(p.nc - 1) - 1.0f;
}

template <bool kBf16>
__global__ void __launch_bounds__(WR_THREADS, 1) wavernn_kernel(const WrParams p) {
  extern __shared__ __align__(16) unsigned char wr_smem[];
  using WT = typename std::conditional<kBf16, __nv_bfloat16, float>::type;
  WT* sw = reinterpret_cast<WT*>(wr_smem);
  const int rows_smem = SMEM_ROWS + p.q;
  float* xs = reinterpret_cast<float*>(wr_smem + (size_t)rows_smem * WR_D * sizeof(WT));
  cg::grid_group grid = cg::this_grid();
  const int b = blockIdx.x, u0 = 4 * b;
  const WT* wg = reinterpret_cast<const WT*>(p.w);

  // this CTA's weight rows: GRU1 hh (12), GRU2 ih (12), GRU2 hh (12), fc1 (4), fc2 (4), fc3 (q); smem row g * 4 + j is gate g of
  // unit u0 + j
  for (int idx = threadIdx.x; idx < rows_smem * WR_D; idx += WR_THREADS) {
    const int m = idx / WR_D, k = idx % WR_D;
    int src = -1;
    if (m < 36) {
      const int mat = m / 12, g = (m % 12) / 4, j = m % 4;
      src = (mat == 0 ? W_HH1 : mat == 1 ? W_IH2 : W_HH2) + g * WR_D + u0 + j;
    } else if (m < 40) {
      src = W_FC1 + u0 + (m - 36);
    } else if (m < 44) {
      src = W_FC2 + u0 + (m - 40);
    } else {
      const int cls = b * p.q + (m - 44);
      if (cls < p.nc) src = W_FC3 + cls;
    }
    sw[idx] = src >= 0 ? wg[(int64_t)src * WR_D + k] : WT(0.f);
  }
  // zero state (buffer 0) of this CTA's units
  for (int idx = threadIdx.x; idx < p.R * 4; idx += WR_THREADS) {
    const int64_t o = (int64_t)(idx / 4) * WR_D + u0 + idx % 4;
    p.h1[o] = 0.f;
    p.h2[o] = 0.f;
  }
  __syncthreads();
  grid.sync();

  // optional phase timers (p.timings): thread 0 charges the time since the last mark to segment `seg`, first up to the CTA's
  // last warp (work), then through the grid barrier that follows it (wait)
  __shared__ unsigned long long s_time[2 * WR_SEGS];
  const bool timed = p.timings != nullptr;
  uint64_t tmark = 0;
  if (timed && threadIdx.x < 2 * WR_SEGS) s_time[threadIdx.x] = 0;
  if (timed && threadIdx.x == 0) tmark = wr_now();
  auto finish = [&](int seg, bool barrier) {
    if (timed) {
      __syncthreads();
      if (threadIdx.x == 0) {
        const uint64_t t = wr_now();
        s_time[2 * seg] += t - tmark;
        tmark = t;
      }
    }
    if (barrier) grid.sync();
    if (timed && threadIdx.x == 0) {
      const uint64_t t = wr_now();
      s_time[2 * seg + 1] += t - tmark;
      tmark = t;
    }
  };

  const int warp = threadIdx.x / 32, lane = threadIdx.x & 31, rr = lane >> 2, kq = lane & 3;
  const int u = u0 + kq;
  const int64_t RD = (int64_t)p.R * WR_D;
  const int groups = (p.R + 7) / 8;
  const int half = p.n_taps / 2;
  const float* vec = p.vec;

  for (int s = 0; s < p.L; ++s) {
    const float* h1o = p.h1 + (s & 1) * RD;
    float* h1n = p.h1 + ((s + 1) & 1) * RD;
    const float* h2o = p.h2 + (s & 1) * RD;
    float* h2n = p.h2 + ((s + 1) & 1) * RD;

    // ---- phase 1: x_prev of every row, then GRU1
    for (int r = warp; r < p.R; r += WR_WARPS) {
      const float x = s == 0 ? 0.f : wr_sample(p, r, s - 1);
      if (lane == 0) {
        xs[r] = x;
        if (b == 0 && s > 0) p.samples[(int64_t)r * p.L + s - 1] = x;
      }
    }
    __syncthreads();
    finish(0, false);
    for (int g8 = warp; g8 < groups; g8 += WR_WARPS) {
      const int r = g8 * 8 + rr, rc = min(r, p.R - 1);
      float acc[12];
      wr_matvec<kBf16, 12>(sw, 0, 12, h1o, rc, kq, acc);
      if (r < p.R) {
        const int4 row = p.rows[r];
        const float xp = xs[r];
        const bool live = s < row.w;
        int64_t base = 0;
        int pp = 0;
        if (live) {
          const int n = row.z + s, f = n / p.hop;
          pp = n - f * p.hop;
          base = (int64_t)p.row0[row.x] + f;
        }
        float gi[3], gh[3];
#pragma unroll
        for (int g = 0; g < 3; ++g) {
          const int col = g * WR_D + u;
          float v = fmaf(xp, vec[V_U1 + col], vec[V_BG1 + col]);
          if (live) {
            float c = wr_cond(p.ax_hi, p.ax_lo, base * p.ld_ax + C_AG1 + col);
            for (int j = 0; j < p.n_taps; ++j)
              c = fmaf(__ldg(p.taps + pp * p.n_taps + j), wr_cond(p.mp_hi, p.mp_lo, (base + j - half) * p.ld_mp + C_PG1 + col), c);
            v += c;
          }
          gi[g] = v;
          gh[g] = wr_pick(acc, g * 4 + kq) + vec[V_BHH1 + col];
        }
        float x = fmaf(xp, vec[V_I0 + u], vec[V_BX + u]);
        if (live) {
          float c = wr_cond(p.ax_hi, p.ax_lo, base * p.ld_ax + C_AX + u);
          for (int j = 0; j < p.n_taps; ++j)
            c = fmaf(__ldg(p.taps + pp * p.n_taps + j), wr_cond(p.mp_hi, p.mp_lo, (base + j - half) * p.ld_mp + C_PX + u), c);
          x += c;
        }
        const float rg = wr_sigmoid(gi[0] + gh[0]), zg = wr_sigmoid(gi[1] + gh[1]);
        const float ng = tanhf(gi[2] + rg * gh[2]);
        const int64_t o = (int64_t)r * WR_D + u;
        const float h = (1.0f - zg) * ng + zg * __ldcg(h1o + o);
        __stcg(h1n + o, h);
        __stcg(p.x2 + o, x + h);
      }
    }
    finish(1, true);

    // ---- phase 2: GRU2 over [x + h1, a2]
    for (int g8 = warp; g8 < groups; g8 += WR_WARPS) {
      const int r = g8 * 8 + rr, rc = min(r, p.R - 1);
      float ai[12], ah[12];
      wr_matvec<kBf16, 12>(sw, 12, 12, p.x2, rc, kq, ai);
      wr_matvec<kBf16, 12>(sw, 24, 12, h2o, rc, kq, ah);
      if (r < p.R) {
        const int4 row = p.rows[r];
        const bool live = s < row.w;
        const int64_t base = live ? (int64_t)p.row0[row.x] + (row.z + s) / p.hop : 0;
        float gi[3], gh[3];
#pragma unroll
        for (int g = 0; g < 3; ++g) {
          const int col = g * WR_D + u;
          float v = wr_pick(ai, g * 4 + kq) + vec[V_BG2 + col];
          if (live) v += wr_cond(p.ax_hi, p.ax_lo, base * p.ld_ax + C_AG2 + col);
          gi[g] = v;
          gh[g] = wr_pick(ah, g * 4 + kq) + vec[V_BHH2 + col];
        }
        const float rg = wr_sigmoid(gi[0] + gh[0]), zg = wr_sigmoid(gi[1] + gh[1]);
        const float ng = tanhf(gi[2] + rg * gh[2]);
        const int64_t o = (int64_t)r * WR_D + u;
        const float h = (1.0f - zg) * ng + zg * __ldcg(h2o + o);
        __stcg(h2n + o, h);
        __stcg(p.x3 + o, __ldcg(p.x2 + o) + h);
      }
    }
    finish(2, true);

    // ---- phases 3 and 4: fc1 over [x, a3], fc2 over [fc1, a4], ReLU
#pragma unroll 1
    for (int layer = 0; layer < 2; ++layer) {
      const float* in = layer == 0 ? p.x3 : p.f1;
      float* out = layer == 0 ? p.f1 : p.f2;
      for (int g8 = warp; g8 < groups; g8 += WR_WARPS) {
        const int r = g8 * 8 + rr, rc = min(r, p.R - 1);
        float acc[4];
        wr_matvec<kBf16, 4>(sw, 36 + 4 * layer, 4, in, rc, kq, acc);
        if (r < p.R) {
          const int4 row = p.rows[r];
          float v = wr_pick(acc, kq) + vec[(layer == 0 ? V_B3 : V_B4) + u];
          if (s < row.w) {
            const int64_t base = (int64_t)p.row0[row.x] + (row.z + s) / p.hop;
            v += wr_cond(p.ax_hi, p.ax_lo, base * p.ld_ax + (layer == 0 ? C_A3 : C_A4) + u);
          }
          __stcg(out + (int64_t)r * WR_D + u, fmaxf(v, 0.f));
        }
      }
      finish(3 + layer, true);
    }

    // ---- phase 5: fc3 -> logits (and the capture)
    const int ncls = min(p.q, p.nc - b * p.q);
    if (ncls > 0) {
      for (int g8 = warp; g8 < groups; g8 += WR_WARPS) {
        const int r = g8 * 8 + rr, rc = min(r, p.R - 1);
        float acc[WR_MAX_FC3];
        wr_matvec<kBf16, WR_MAX_FC3>(sw, 44, ncls, p.f2, rc, kq, acc);
        if (r < p.R) {
          for (int m = kq; m < ncls; m += 4) {
            const int cls = b * p.q + m;
            const float v = wr_pick(acc, m) + vec[V_B5 + cls];
            __stcg(p.logits + (int64_t)r * p.ncp + cls, v);
            if (s < p.cap) p.capture[((int64_t)r * p.cap + s) * p.nc + cls] = v;
          }
        }
      }
    }
    finish(5, true);
  }
  if (timed && threadIdx.x < 2 * WR_SEGS) p.timings[(int64_t)b * 2 * WR_SEGS + threadIdx.x] = (int64_t)s_time[threadIdx.x];
  // the last step's samples
  if (b == 0) {
    for (int r = warp; r < p.R; r += WR_WARPS) {
      const float x = wr_sample(p, r, p.L - 1);
      if (lane == 0) p.samples[(int64_t)r * p.L + p.L - 1] = x;
    }
  }
}

struct WrClip {
  int row0, n_folds, wave_len;
  int64_t out_off;
};

// fatchord's tail of generate(): mu-law decode (RAW), xfade_and_unfold (batched), crop to (T - 1) hop, linear fade-out over
// the last 20 hop samples; in float64
__global__ void wavernn_unfold_kernel(const float* samples, int L, const WrClip* clips, int n_clips, int batched, int target,
                                      int overlap, int hop, int raw, int nc, float* wav) {
  const int c = blockIdx.y;
  if (c >= n_clips) return;
  const WrClip cl = clips[c];
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= cl.wave_len) return;
  const int silence = overlap / 2, fade = overlap - silence;
  const double step = fade > 1 ? 2.0 / (double)(fade - 1) : 0.0;   // np.linspace(-1, 1, fade); a single point is -1
  auto decode = [&](double y) {
    if (!raw) return y;
    const double mu = (double)(nc - 1);
    return (y > 0 ? 1.0 : (y < 0 ? -1.0 : 0.0)) / mu * (pow(1.0 + mu, fabs(y)) - 1.0);
  };
  double y = 0.0;
  if (batched) {
    const int stride = target + overlap;
    for (int i = 0; i < cl.n_folds; ++i) {
      const int k = n - i * stride;
      if (k < 0 || k >= L) continue;
      double v = decode((double)samples[(int64_t)(cl.row0 + i) * L + k]);
      if (k < overlap) {   // fade_in = [zeros(silence), sqrt(0.5 (1 + t))]
        if (k < silence) v *= 0.0;
        else {
          const int t = k - silence;
          const double tt = (t == fade - 1 && fade > 1) ? 1.0 : -1.0 + t * step;
          v *= sqrt(0.5 * (1.0 + tt));
        }
      }
      if (k >= L - overlap) {   // fade_out = [ones(silence), sqrt(0.5 (1 - t))]
        const int t = k - (L - overlap) - silence;
        if (t >= 0) {
          const double tt = (t == fade - 1 && fade > 1) ? 1.0 : -1.0 + t * step;
          v *= sqrt(0.5 * (1.0 - tt));
        }
      }
      y += v;
    }
  } else {
    y = decode((double)samples[(int64_t)cl.row0 * L + n]);
  }
  const int nf = 20 * hop, k = n - (cl.wave_len - nf);
  if (k >= 0) y *= k == nf - 1 ? 0.0 : 1.0 + k * (-1.0 / (double)(nf - 1));
  wav[cl.out_off + n] = (float)y;
}

struct WrLayout {
  int R, L, ncp;
  int64_t o_h1, o_h2, o_x2, o_x3, o_f1, o_f2, o_logits, o_samples, o_rows, o_clips, o_row0, o_seeds, total;
};

static int wr_folds(int64_t total, int target, int overlap) {
  // fold_with_overlap's fold count, in Python's floor division
  const int64_t st = (int64_t)target + overlap;
  const int64_t a = total - overlap;
  int64_t nf = a >= 0 ? a / st : -((-a + st - 1) / st);
  const int64_t ext = nf * st + overlap;
  if (total - ext != 0) nf += 1;
  return (int)nf;
}

static int wr_layout(const char* what, const int32_t* frames, int n_clips, int hop, int batched, int target, int overlap, int nc,
                     WrLayout* ly) {
  if (n_clips < 1 || !frames) { set_last_error("%s: n_clips must be >= 1 with a frames table", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (hop < 1 || hop > 65536) { set_last_error("%s: hop = %d must be in [1, 65536]", what, hop); return TTSB_ERR_INVALID_ARGUMENT; }
  if (nc < 2 || nc > 1024) { set_last_error("%s: n_classes = %d", what, nc); return TTSB_ERR_INVALID_ARGUMENT; }
  if (batched && (target < 1 || overlap < 1)) { set_last_error("%s: target = %d and overlap = %d must be >= 1", what, target, overlap); return TTSB_ERR_INVALID_ARGUMENT; }
  int64_t R = 0, L = batched ? (int64_t)target + 2 * (int64_t)overlap : 0;
  for (int c = 0; c < n_clips; ++c) {
    if (frames[c] < TTSB_WAVERNN_MIN_FRAMES || (int64_t)frames[c] * hop > (1 << 28)) {
      set_last_error("%s: clip %d has %d frames; the generator needs %d .. 2^28 / hop", what, c, frames[c], TTSB_WAVERNN_MIN_FRAMES);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
    const int64_t total = (int64_t)frames[c] * hop;
    if (batched) {
      if (total <= overlap) { set_last_error("%s: clip %d has %lld samples, not more than the overlap %d", what, c, (long long)total, overlap); return TTSB_ERR_INVALID_ARGUMENT; }
      R += wr_folds(total, target, overlap);
    } else {
      R += 1;
      L = total > L ? total : L;
    }
  }
  if (L > (1 << 28) || R > TTSB_WAVERNN_MAX_ROWS) {
    set_last_error("%s: %lld folds of %lld steps; at most %d folds", what, (long long)R, (long long)L, TTSB_WAVERNN_MAX_ROWS);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  ly->R = (int)R;
  ly->L = (int)L;
  ly->ncp = (nc + 31) / 32 * 32;
  int64_t o = 0;
  auto take = [&](int64_t bytes) { const int64_t at = o; o += (bytes + 255) / 256 * 256; return at; };
  const int64_t rd = R * WR_D * 4;
  ly->o_h1 = take(2 * rd);
  ly->o_h2 = take(2 * rd);
  ly->o_x2 = take(rd);
  ly->o_x3 = take(rd);
  ly->o_f1 = take(rd);
  ly->o_f2 = take(rd);
  ly->o_logits = take(R * ly->ncp * 4);
  ly->o_samples = take(R * L * 4);
  ly->o_rows = take(R * 16);
  ly->o_clips = take((int64_t)n_clips * sizeof(WrClip));
  ly->o_row0 = take((int64_t)n_clips * 4);
  ly->o_seeds = take((int64_t)n_clips * 4);
  ly->total = o;
  return 0;
}

template <bool kBf16>
static int wr_smem_bytes(int q, int R) {
  return (SMEM_ROWS + q) * WR_D * (kBf16 ? 2 : 4) + R * 4;
}

template <bool kBf16>
static int wr_launch(const WrParams& p, cudaStream_t stream) {
  const int smem = wr_smem_bytes<kBf16>(p.q, p.R);
  if (check_cuda(cudaFuncSetAttribute(wavernn_kernel<kBf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "wavernn smem attribute")) return TTSB_ERR_CUDA;
  int per_sm = 0;
  if (check_cuda(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wavernn_kernel<kBf16>, WR_THREADS, smem), "wavernn occupancy")) return TTSB_ERR_CUDA;
  int dev = current_device(), coop = 0;
  if (check_cuda(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev), "cooperative attribute")) return TTSB_ERR_CUDA;
  if (!coop || per_sm * num_sms() < WR_CTAS) {
    set_last_error("ttsb_wavernn_generate: %d CTAs of %d bytes of shared memory cannot all be resident (%d per SM on %d SMs%s)", WR_CTAS,
                   smem, per_sm, num_sms(), coop ? "" : ", no cooperative launch");
    return TTSB_ERR_UNSUPPORTED;
  }
  void* args[] = {const_cast<WrParams*>(&p)};
  count_launch();
  return check_cuda(cudaLaunchCooperativeKernel((const void*)wavernn_kernel<kBf16>, dim3(WR_CTAS), dim3(WR_THREADS), args, smem, stream),
                    "wavernn_kernel cooperative launch");
}

struct WrArgs {
  const int32_t* frames;
  const uint32_t* seeds;
  int n_clips;
  int hop;
  int batched;
  int target;
  int overlap;
  int n_rows;
  int n_taps;
  const float* taps;
  const void* melp_hi;
  const void* melp_lo;
  int ld_melp;
  const void* aux_hi;
  const void* aux_lo;
  int ld_aux;
  int cond_halo;
  int64_t cond_rows;
  const float* vec;
  const void* weights;
  int mode;
  int n_classes;
  int precision;
  float* wav_out;
  float* capture;
  int capture_steps;
  float* samples_out;
  int64_t* timings;
  void* workspace;
  int64_t workspace_bytes;
};

static bool wr_aligned(const void* p, int a) { return ((uintptr_t)p % a) == 0; }

}  // namespace ttsb

using namespace ttsb;

extern "C" int64_t ttsb_wavernn_workspace_bytes(const int32_t* frames, int n_clips, int hop, int batched, int target, int overlap,
                                                int n_classes) {
  WrLayout ly;
  if (wr_layout("ttsb_wavernn_workspace_bytes", frames, n_clips, hop, batched, target, overlap, n_classes, &ly)) return -1;
  return ly.total;
}

static int wr_generate(const WrArgs* a, void* stream_v) {
  const char* what = "ttsb_wavernn_generate";
  if (a->precision != TTSB_PREC_BF16 && a->precision != TTSB_PREC_BF16X3) { set_last_error("%s: unknown precision", what); return TTSB_ERR_INVALID_ARGUMENT; }
  const bool split = a->precision == TTSB_PREC_BF16X3;
  if (a->mode == TTSB_WAVERNN_MOL) {
    if (a->n_classes != 30) { set_last_error("%s: MOL takes 30 logits, got n_classes = %d", what, a->n_classes); return TTSB_ERR_INVALID_ARGUMENT; }
  } else if (a->mode == TTSB_WAVERNN_RAW) {
    if (a->n_classes != 256 && a->n_classes != 512 && a->n_classes != 1024) {
      set_last_error("%s: RAW takes 2^bits logits with 8 <= bits <= 10, got n_classes = %d", what, a->n_classes);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
  } else {
    set_last_error("%s: mode = %d is neither TTSB_WAVERNN_MOL nor TTSB_WAVERNN_RAW", what, a->mode);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  WrLayout ly;
  int rc = wr_layout(what, a->frames, a->n_clips, a->hop, a->batched, a->target, a->overlap, a->n_classes, &ly);
  if (rc) return rc;
  if (a->n_rows != ly.R) { set_last_error("%s: n_rows = %d, but the clips make %d folds", what, a->n_rows, ly.R); return TTSB_ERR_INVALID_ARGUMENT; }
  if (!a->seeds) { set_last_error("%s: seeds is NULL", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->n_taps < 1 || a->n_taps > TTSB_WAVERNN_MAX_TAPS || a->n_taps % 2 == 0 || !a->taps || !wr_aligned(a->taps, 4)) {
    set_last_error("%s: n_taps = %d must be odd and in [1, %d], with a 4-byte aligned taps table", what, a->n_taps, TTSB_WAVERNN_MAX_TAPS);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  const int half = a->n_taps / 2;
  if (a->cond_halo < half || a->cond_halo > TTSB_CONV1D_EX_MAX_HALO) {
    set_last_error("%s: cond_halo = %d must cover the %d mel taps on each side and be <= %d", what, a->cond_halo, half, TTSB_CONV1D_EX_MAX_HALO);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  int64_t cond_rows = 0;
  for (int c = 0; c < a->n_clips; ++c) cond_rows += a->frames[c] + 2 * (int64_t)a->cond_halo;
  if (a->cond_rows != cond_rows) {
    set_last_error("%s: cond_rows = %lld, but the clips with cond_halo %d take %lld rows", what, (long long)a->cond_rows, a->cond_halo, (long long)cond_rows);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (!a->melp_hi || !a->aux_hi || (split != (a->melp_lo != nullptr)) || (split != (a->aux_lo != nullptr))) {
    set_last_error("%s: the conditioning needs hi planes, and lo planes exactly in bf16x3", what);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (a->ld_melp < 2048 || a->ld_aux < 4608) {
    set_last_error("%s: ld_melp = %d must be >= 2048 and ld_aux = %d >= 4608", what, a->ld_melp, a->ld_aux);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  const void* bf[4] = {a->melp_hi, a->melp_lo, a->aux_hi, a->aux_lo};
  for (const void* p : bf)
    if (p && !wr_aligned(p, 2)) { set_last_error("%s: conditioning planes must be 2-byte aligned", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (!a->vec || !a->weights || !wr_aligned(a->vec, 16) || !wr_aligned(a->weights, 16)) {
    set_last_error("%s: vec and weights must be 16-byte aligned device buffers", what);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (!a->wav_out || !wr_aligned(a->wav_out, 4)) { set_last_error("%s: wav_out must be a 4-byte aligned device buffer", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->capture_steps < 0 || a->capture_steps > ly.L || (a->capture_steps > 0) != (a->capture != nullptr) ||
      (a->capture && !wr_aligned(a->capture, 4))) {
    set_last_error("%s: capture_steps = %d must be in [0, %d] and given exactly with a 4-byte aligned capture buffer", what, a->capture_steps, ly.L);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (a->timings && !wr_aligned(a->timings, 8)) { set_last_error("%s: timings must be 8-byte aligned", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->samples_out && !wr_aligned(a->samples_out, 4)) { set_last_error("%s: samples_out must be 4-byte aligned", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (!a->workspace || !wr_aligned(a->workspace, 256) || a->workspace_bytes < ly.total) {
    set_last_error("%s: workspace missing, not 256-byte aligned or smaller than ttsb_wavernn_workspace_bytes (%lld)", what, (long long)ly.total);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  const int q = (a->n_classes + WR_CTAS - 1) / WR_CTAS;
  if ((split ? wr_smem_bytes<false>(q, ly.R) : wr_smem_bytes<true>(q, ly.R)) > 227 * 1024 - 2 * WR_SEGS * 8) {   // the timers' static shared memory
    set_last_error("%s: %d folds do not fit the shared memory", what, ly.R);
    return TTSB_ERR_UNSUPPORTED;
  }

  // host tables: rows (clip, fold, first, valid), clips, row0, seeds
  const int R = ly.R, L = ly.L, n = a->n_clips;
  unsigned char* ws = static_cast<unsigned char*>(a->workspace);
  int32_t* hrows = new int32_t[(size_t)R * 4];
  WrClip* hclips = new WrClip[n];
  int32_t* hrow0 = new int32_t[n];
  int64_t cond0 = 0, out_off = 0;
  int r = 0;
  for (int c = 0; c < n; ++c) {
    const int64_t total = (int64_t)a->frames[c] * a->hop;
    const int nf = a->batched ? wr_folds(total, a->target, a->overlap) : 1;
    hclips[c] = WrClip{r, nf, (a->frames[c] - 1) * a->hop, out_off};
    hrow0[c] = (int32_t)(cond0 + a->cond_halo);
    for (int i = 0; i < nf; ++i, ++r) {
      const int64_t first = a->batched ? (int64_t)i * (a->target + a->overlap) : 0;
      const int64_t valid = total - first < L ? total - first : L;
      hrows[4 * r] = c;
      hrows[4 * r + 1] = i;
      hrows[4 * r + 2] = (int32_t)first;
      hrows[4 * r + 3] = (int32_t)(valid > 0 ? valid : 0);
    }
    cond0 += a->frames[c] + 2 * a->cond_halo;
    out_off += (int64_t)(a->frames[c] - 1) * a->hop;
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  rc = check_cuda(cudaMemcpyAsync(ws + ly.o_rows, hrows, (size_t)R * 16, cudaMemcpyHostToDevice, stream), "wavernn rows copy");
  if (!rc) rc = check_cuda(cudaMemcpyAsync(ws + ly.o_clips, hclips, (size_t)n * sizeof(WrClip), cudaMemcpyHostToDevice, stream), "wavernn clips copy");
  if (!rc) rc = check_cuda(cudaMemcpyAsync(ws + ly.o_row0, hrow0, (size_t)n * 4, cudaMemcpyHostToDevice, stream), "wavernn row0 copy");
  if (!rc) rc = check_cuda(cudaMemcpyAsync(ws + ly.o_seeds, a->seeds, (size_t)n * 4, cudaMemcpyHostToDevice, stream), "wavernn seeds copy");
  // copies from pageable host memory return once the runtime has staged the data, so the tables may be freed here
  delete[] hrows;
  delete[] hclips;
  delete[] hrow0;
  if (rc) return rc;

  WrParams p;
  p.R = R;
  p.L = L;
  p.n_taps = a->n_taps;
  p.hop = a->hop;
  p.nc = a->n_classes;
  p.ncp = ly.ncp;
  p.q = q;
  p.mode = a->mode;
  p.cap = a->capture_steps;
  p.rows = reinterpret_cast<const int4*>(ws + ly.o_rows);
  p.row0 = reinterpret_cast<const int32_t*>(ws + ly.o_row0);
  p.seeds = reinterpret_cast<const uint32_t*>(ws + ly.o_seeds);
  p.taps = a->taps;
  p.mp_hi = static_cast<const __nv_bfloat16*>(a->melp_hi);
  p.mp_lo = static_cast<const __nv_bfloat16*>(a->melp_lo);
  p.ax_hi = static_cast<const __nv_bfloat16*>(a->aux_hi);
  p.ax_lo = static_cast<const __nv_bfloat16*>(a->aux_lo);
  p.ld_mp = a->ld_melp;
  p.ld_ax = a->ld_aux;
  p.vec = a->vec;
  p.w = a->weights;
  p.h1 = reinterpret_cast<float*>(ws + ly.o_h1);
  p.h2 = reinterpret_cast<float*>(ws + ly.o_h2);
  p.x2 = reinterpret_cast<float*>(ws + ly.o_x2);
  p.x3 = reinterpret_cast<float*>(ws + ly.o_x3);
  p.f1 = reinterpret_cast<float*>(ws + ly.o_f1);
  p.f2 = reinterpret_cast<float*>(ws + ly.o_f2);
  p.logits = reinterpret_cast<float*>(ws + ly.o_logits);
  p.samples = reinterpret_cast<float*>(ws + ly.o_samples);
  p.capture = a->capture;
  p.timings = a->timings;
  rc = split ? wr_launch<false>(p, stream) : wr_launch<true>(p, stream);
  if (rc) return rc;
  if (a->samples_out)
    if ((rc = check_cuda(cudaMemcpyAsync(a->samples_out, p.samples, (size_t)R * L * 4, cudaMemcpyDeviceToDevice, stream), "wavernn samples copy"))) return rc;
  int64_t max_len = 0;
  for (int c = 0; c < n; ++c) max_len = std::max(max_len, (int64_t)(a->frames[c] - 1) * a->hop);
  dim3 grid((unsigned)((max_len + 255) / 256), (unsigned)n);
  wavernn_unfold_kernel<<<grid, 256, 0, stream>>>(p.samples, L, reinterpret_cast<const WrClip*>(ws + ly.o_clips), n, a->batched, a->target,
                                                  a->overlap, a->hop, a->mode == TTSB_WAVERNN_RAW, a->n_classes, a->wav_out);
  count_launch();
  return check_cuda(cudaGetLastError(), "wavernn_unfold_kernel launch");
}

extern "C" int ttsb_wavernn_generate(const int32_t* frames, const uint32_t* seeds, int n_clips, int hop, int batched, int target, int overlap, int n_rows, int n_taps, const float* taps, const void* melp_hi, const void* melp_lo, int ld_melp, const void* aux_hi, const void* aux_lo, int ld_aux, int cond_halo, int64_t cond_rows, const float* vec, const void* weights, int mode, int n_classes, int precision, float* wav_out, float* capture, int capture_steps, float* samples_out, int64_t* timings, void* workspace, int64_t workspace_bytes, void* stream) {
  const WrArgs a{frames, seeds, n_clips, hop, batched, target, overlap, n_rows, n_taps, taps, melp_hi, melp_lo, ld_melp, aux_hi, aux_lo, ld_aux, cond_halo, cond_rows, vec, weights, mode, n_classes, precision, wav_out, capture, capture_steps, samples_out, timings, workspace, workspace_bytes};
  return wr_generate(&a, stream);
}
