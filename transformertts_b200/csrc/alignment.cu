// Duration extraction from the Aligner's attention maps (reference: utils/alignments.py:58-143, utils/metrics.py:5-70):
// per-head attention scores, best / score-weighted head, shortest monotonic path through (max - attention), durations.
//
// The reference builds a sparse graph (right / down / down-right edges weighted by the target node) and runs
// scipy's Dijkstra.  The graph is a DAG whose edge weight depends on the target only, so the same distances come out of
// the dynamic programme dist[i][j] = w[i][j] + min(dist[i][j-1], dist[i-1][j], dist[i-1][j-1]); cells of one anti-diagonal
// are independent, so one block sweeps the (mel_len-2) x (phon_len-2) matrix of a batch row diagonal by diagonal in float64
// (what scipy accumulates in), keeps three diagonals in shared memory, stores one predecessor byte per cell and walks the
// path back.  Identical to the reference whenever no two predecessor distances tie exactly.
#include <cuda_runtime.h>

#include <cstdint>

#include "ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace ttsb {

__device__ __forceinline__ float wsumf(float v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// scores[(b*H + h)*3 + {0,1,2}] = jumpiness, peakiness, 3 / diagonality (utils/metrics.py:5-44), lengths already "- 1"
__global__ void attention_scores_kernel(const float* __restrict__ att, int H, int Tq, int Tk, const int* __restrict__ q_len,
                                        const int* __restrict__ k_len, int r, float* __restrict__ scores) {
  extern __shared__ int amax_idx[];  // [Tq]
  __shared__ float red[2][32];
  const int bh = blockIdx.x, b = bh / H;
  const int ml = q_len[b], pl = k_len[b];
  const int max_m = min(max(ml, 0), Tq), max_n = min(max(pl, 0), Tk);
  const float* a = att + (size_t)bh * Tq * Tk;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float peak = 0.f, diag = 0.f;
  for (int q = wid; q < Tq; q += nw) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    float dsum = 0.f;
    const double jq = max_m > 0 ? (double)q / (double)max_m : 0.0;
    for (int k = lane; k < Tk; k += 32) {
      const float v = a[(size_t)q * Tk + k];
      if (v > best) { best = v; bi = k; }   // first maximum within this lane's strided scan
      if (q < max_m && k < max_n) dsum += v * (float)fabs((double)k / (double)max_n - jq);
    }
    for (int o = 16; o; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }   // argmax = smallest index among the maxima
    }
    dsum = wsumf(dsum);
    if (lane == 0) {
      amax_idx[q] = bi;
      if (q < ml) peak += best;   // mask = arange(Tq) < mel_len
      diag += dsum;
    }
  }
  if (lane == 0) { red[0][wid] = peak; red[1][wid] = diag; }
  __syncthreads();
  int loc = 0;
  for (int q = 1 + threadIdx.x; q < Tq; q += blockDim.x) {
    const int d = abs(amax_idx[q] - amax_idx[q - 1]);
    if (d <= r && q < ml) loc += 1;
  }
  for (int o = 16; o; o >>= 1) loc += __shfl_xor_sync(0xffffffffu, loc, o);
  __shared__ int redi[32];
  if (lane == 0) redi[wid] = loc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float p = 0.f, d = 0.f;
    int l = 0;
    for (int w = 0; w < nw; ++w) { p += red[0][w]; d += red[1][w]; l += redi[w]; }
    scores[bh * 3 + 0] = (float)((double)l / (double)(ml - 1));
    scores[bh * 3 + 1] = p / (float)Tq;     // reduce_mean over the PADDED length
    scores[bh * 3 + 2] = 3.f / d;
  }
}

// one block per batch row: reference matrix = att[b, head, 1:ml, 1:pl] of the best head (or the score-weighted head sum)
__global__ void durations_dp_kernel(const float* __restrict__ att, int H, int Tq, int Tk, const int* __restrict__ q_len,
                                    const int* __restrict__ k_len, const float* __restrict__ scores, int weighted,
                                    uint8_t* __restrict__ pred_all, int32_t* __restrict__ durations) {
  extern __shared__ double dsm[];  // 3 diagonals of Tk doubles + head weights
  const int b = blockIdx.x;
  const int ml = q_len[b], pl = k_len[b];
  const int M = min(ml, Tq) - 1, N = min(pl, Tk) - 1;   // rows 1..ml-1, columns 1..pl-1
  int32_t* dur = durations + (size_t)b * Tk;
  for (int k = threadIdx.x; k < Tk; k += blockDim.x) dur[k] = 0;
  if (M <= 0 || N <= 0) return;
  double* D0 = dsm;
  double* D1 = dsm + Tk;
  double* D2 = dsm + 2 * Tk;
  float* hw = reinterpret_cast<float*>(dsm + 3 * Tk);   // [H] head weights
  __shared__ int best_head;
  __shared__ float red[32];
  if (threadIdx.x == 0) {
    int bh = 0;
    float bs = -INFINITY;
    for (int h = 0; h < H; ++h) {
      const float* s = scores + ((size_t)b * H + h) * 3;
      const float tot = s[2] + s[0] + s[1];   // diag_measure + jumpiness + peakiness (alignments.py:122)
      hw[h] = tot;
      if (tot > bs) { bs = tot; bh = h; }     // np.argmax: first maximum
    }
    best_head = bh;
  }
  __syncthreads();
  const float* abase = att + (size_t)b * H * Tq * Tk;
  auto ref = [&](int i, int j) -> float {   // element (i, j) of the cropped reference matrix, float32 like numpy
    const size_t off = (size_t)(i + 1) * Tk + (j + 1);
    if (!weighted) return abase[(size_t)best_head * Tq * Tk + off];
    float acc = 0.f;
    for (int h = 0; h < H; ++h) acc = __fadd_rn(acc, __fmul_rn(abase[(size_t)h * Tq * Tk + off], hw[h]));
    return acc;
  };
  // attn_max over the cropped matrix
  float mx = -INFINITY;
  for (int e = threadIdx.x; e < M * N; e += blockDim.x) mx = fmaxf(mx, ref(e / N, e % N));
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
  uint8_t* pred = pred_all + (size_t)b * Tq * Tk;
  const double INF = 1e300;
  for (int d = 0; d < M + N - 1; ++d) {
    const int j_lo = max(0, d - M + 1), j_hi = min(d, N - 1);
    for (int j = j_lo + threadIdx.x; j <= j_hi; j += blockDim.x) {
      const int i = d - j;
      double best = INF;
      uint8_t code = 0;
      if (d == 0) {
        best = 0.0;   // the start node costs nothing
      } else {
        if (j > 0 && D1[j - 1] < best) { best = D1[j - 1]; code = 0; }            // left  (i, j-1)
        if (i > 0 && D1[j] < best) { best = D1[j]; code = 1; }                    // up    (i-1, j)
        if (i > 0 && j > 0 && D2[j - 1] < best) { best = D2[j - 1]; code = 2; }   // diag  (i-1, j-1)
        best += (double)__fsub_rn(mx, ref(i, j));   // path_probs = attn_max - attention (float32), summed in float64
      }
      D0[j] = best;
      pred[(size_t)i * N + j] = code;
    }
    __syncthreads();
    double* t = D2; D2 = D1; D1 = D0; D0 = t;   // rotate: the diagonal just written becomes d-1
  }
  if (threadIdx.x == 0) {
    int i = M - 1, j = N - 1, last_row = -1;
    while (true) {
      if (i != last_row) { dur[j] += 1; last_row = i; }   // walking back, the first visit of a row is its right-most column
      if (i == 0 && j == 0) break;
      const uint8_t c = pred[(size_t)i * N + j];
      if (c == 0) --j; else if (c == 1) --i; else { --i; --j; }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Per-character pitch (extract_durations.py:108-115 of the reference, batched): the mean of the voiced (!= 0), < 400 Hz
// (after de-normalisation) frame pitches under each character.  The mean is bit-exact with np.mean: the kept values are
// summed in numpy's pairwise order (numpy/core/src/umath/loops_utils.h.src, pairwise_sum_DOUBLE) and divided by their
// count.  That order depends on the count n of kept values only:
//   n < 8:        sequential from 0.0;
//   8 <= n <= 128: eight strided accumulators ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the n % 8 tail sequentially;
//   n > 128:      sum(first n2) + sum(rest), n2 = n/2 rounded down to a multiple of 8.
// A segment is a handful of frames, so one thread walks one character's frames; the tree of the n > 128 case is evaluated
// with an explicit stack, consuming the kept values left to right.
// ---------------------------------------------------------------------------------------------------------------------
struct KeptPitch {   // the kept frame values of one segment, in order
  const double* p;
  int i;
  double mean, std;
  __device__ __forceinline__ static bool keep(double v, double mean, double std) {
    // numpy evaluates values * std + mean as two rounded operations: no FMA contraction
    return v != 0.0 && __dadd_rn(__dmul_rn(v, std), mean) < 400.0;
  }
  __device__ __forceinline__ double next() {
    while (true) {
      const double v = p[i++];
      if (keep(v, mean, std)) return v;
    }
  }
};

__device__ double pairwise_leaf(KeptPitch& src, int n) {   // n <= 128
  if (n < 8) {
    double s = 0.0;
    for (int k = 0; k < n; ++k) s = __dadd_rn(s, src.next());
    return s;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = src.next();
  int k = 8;
  for (; k < n - (n % 8); k += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], src.next());
  }
  double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; k < n; ++k) s = __dadd_rn(s, src.next());
  return s;
}

__device__ double pairwise_sum(KeptPitch& src, int n) {
  int right_n[32];      // pending right halves; depth <= log2(n / 128) + 1 < 32 for any int n
  double left[32];
  bool left_done[32];
  int sp = 0;
  while (true) {
    while (n > 128) {
      int n2 = n / 2;
      n2 -= n2 % 8;
      right_n[sp] = n - n2;
      left_done[sp] = false;
      ++sp;
      n = n2;
    }
    double s = pairwise_leaf(src, n);
    while (sp > 0 && left_done[sp - 1]) {   // both halves done: fold into the parent
      --sp;
      s = __dadd_rn(left[sp], s);
    }
    if (sp == 0) return s;
    left[sp - 1] = s;                       // left half done: descend into the right half
    left_done[sp - 1] = true;
    n = right_n[sp - 1];
  }
}

// one block per batch row: exclusive prefix sum of the durations in shared memory, then one thread per character
__global__ void pitch_per_char_kernel(const double* __restrict__ pitch, int Tm, const int32_t* __restrict__ pitch_len,
                                      const int32_t* __restrict__ durations, int Tp, const int32_t* __restrict__ n_chars,
                                      double pitch_mean, double pitch_std, double* __restrict__ out) {
  extern __shared__ int cum[];   // [Tp + 1]
  const int b = blockIdx.x;
  const int32_t* dur = durations + (size_t)b * Tp;
  if (threadIdx.x < 32) {        // warp 0: 32 contiguous chunks, warp scan of the chunk sums
    const int lane = threadIdx.x;
    const int chunk = (Tp + 31) / 32;
    const int lo = min(lane * chunk, Tp), hi = min(lo + chunk, Tp);
    int s = 0;
    for (int i = lo; i < hi; ++i) s += dur[i];
    int incl = s;
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    int run = incl - s;
    for (int i = lo; i < hi; ++i) {
      cum[i] = run;
      run += dur[i];
    }
    if (lane == 31) cum[Tp] = incl;
  }
  __syncthreads();
  const int L = min(max(pitch_len[b], 0), Tm);
  const int nc = min(max(n_chars[b], 0), Tp);
  const double* row = pitch + (size_t)b * Tm;
  for (int c = threadIdx.x; c < Tp; c += blockDim.x) {
    double v = 0.0;
    if (c < nc) {
      const int lo = min(cum[c], L), hi = min(cum[c + 1], L);   // pitch[a:b] clipped at the pitch length, as numpy slices
      int n = 0;
      for (int f = lo; f < hi; ++f) n += KeptPitch::keep(row[f], pitch_mean, pitch_std);
      if (n > 0) {
        KeptPitch src{row, lo, pitch_mean, pitch_std};
        v = pairwise_sum(src, n) / (double)n;
      }
    }
    out[(size_t)b * Tp + c] = v;
  }
}

static inline int bad(const char* msg) {
  set_last_error("%s", msg);
  return TTSB_ERR_INVALID_ARGUMENT;
}

}  // namespace ttsb

using namespace ttsb;

extern "C" int ttsb_attention_scores(const float* att, int B, int H, int Tq, int Tk, const int32_t* mel_len, const int32_t* phon_len,
                                     int r, float* scores, void* stream) {
  if (!att || !mel_len || !phon_len || !scores || B <= 0 || H <= 0 || Tq <= 1 || Tk <= 0 || (size_t)Tq * sizeof(int) > 160 * 1024)
    return bad("ttsb_attention_scores: bad arguments");
  const size_t sm = (size_t)Tq * sizeof(int);
  if (sm > 48 * 1024) {
    static PerDevice<size_t> attr_pd;
    size_t& attr = attr_pd.get();
    if (sm > attr) {
      TTSB_CUDA_OK(cudaFuncSetAttribute(attention_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
      attr = sm;
    }
  }
  attention_scores_kernel<<<B * H, 256, sm, static_cast<cudaStream_t>(stream)>>>(att, H, Tq, Tk, mel_len, phon_len, r, scores);
  count_launch();
  return check_cuda(cudaGetLastError(), "attention_scores_kernel");
}

extern "C" int ttsb_durations_from_attention(const float* att, int B, int H, int Tq, int Tk, const int32_t* mel_len,
                                             const int32_t* phon_len, const float* scores, int weighted, uint8_t* scratch,
                                             int32_t* durations, void* stream) {
  if (!att || !mel_len || !phon_len || !scores || !scratch || !durations || B <= 0 || H <= 0 || Tq <= 0 || Tk <= 0)
    return bad("ttsb_durations_from_attention: bad arguments");
  const size_t sm = 3 * (size_t)Tk * sizeof(double) + (size_t)H * sizeof(float) + 16;
  if (sm > 160 * 1024) return bad("ttsb_durations_from_attention: Tk too large");
  if (sm > 48 * 1024) {
    static PerDevice<size_t> attr_pd;
    size_t& attr = attr_pd.get();
    if (sm > attr) {
      TTSB_CUDA_OK(cudaFuncSetAttribute(durations_dp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
      attr = sm;
    }
  }
  durations_dp_kernel<<<B, 256, sm, static_cast<cudaStream_t>(stream)>>>(att, H, Tq, Tk, mel_len, phon_len, scores, weighted, scratch,
                                                                         durations);
  count_launch();
  return check_cuda(cudaGetLastError(), "durations_dp_kernel");
}

extern "C" int ttsb_pitch_per_char(const double* pitch, int B, int Tm, const int32_t* pitch_len, const int32_t* durations, int Tp,
                                   const int32_t* n_chars, double pitch_mean, double pitch_std, double* out, void* stream) {
  if (!pitch || !pitch_len || !durations || !n_chars || !out || B <= 0 || Tm <= 0 || Tp <= 0)
    return bad("ttsb_pitch_per_char: bad arguments");
  const size_t sm = ((size_t)Tp + 1) * sizeof(int);
  if (sm > 48 * 1024) return bad("ttsb_pitch_per_char: Tp too large");
  pitch_per_char_kernel<<<B, 128, sm, static_cast<cudaStream_t>(stream)>>>(pitch, Tm, pitch_len, durations, Tp, n_chars, pitch_mean,
                                                                           pitch_std, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "pitch_per_char_kernel");
}
