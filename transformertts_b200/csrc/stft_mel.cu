// STFT (n_fft 1024, hop 256, periodic Hann, reflect padding) -> magnitude -> banded mel filterbank -> log, fused.
// Replaces data/audio.py:81-92 (librosa.stft + librosa.feature.melspectrogram(S=|D|)) and the normalisers
// (data/audio.py:209-231).  HBM-bound by design: the audio is read once (neighbouring frames hit L1/L2) and only the
// (frames, 80) log-mel is written; the 513-bin spectrum never leaves the SM.
//
// One warp transforms TWO consecutive real frames as one 1024-point complex FFT (frame A -> real, frame B -> imag):
// 1024 = 32 x 32 Cooley-Tukey, both 32-point passes fully in registers (one column per lane), one shared-memory
// transpose in between, twiddles from a table in shared memory.  The two spectra are separated with
// X_A[k] = (Z[k] + conj Z[N-k])/2, X_B[k] = (Z[k] - conj Z[N-k])/(2i).
#include <math.h>
#include <stdlib.h>

#include <vector>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "fft32.cuh"
#include "ttsb_host.h"

namespace ttsb {

constexpr int NFFT = 1024;
constexpr int HOP = 256;
constexpr int NBINS = 513;
constexpr int STFT_WARPS = 8;
constexpr int MAX_MELS = 128;

__device__ float g_tw_re[NFFT];   // cos(2 pi i / 1024)
__device__ float g_tw_im[NFFT];   // -sin(2 pi i / 1024)
__device__ float g_window[NFFT];  // periodic Hann
// The filterbank's band structure, computed on the host from the caller's band table for each call and passed by value:
// row m has non-zero weights at bins [lo[m], lo[m] + len[m]) only; the packed (v2) table keeps them at off[m] ..
// off[m] + len[m] - 1 (`taps` weights in all); kmax = 1 + the highest bin any row reads.
struct MelBands {
  int lo[MAX_MELS], len[MAX_MELS], off[MAX_MELS];
  int kmax;
  int taps;   // off[n_mels - 1] + len[n_mels - 1]: weights in the packed table
};

__device__ __forceinline__ float sample_reflect(const float* __restrict__ clip, int n, int i) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return __ldg(clip + i);
}

struct StftSmem {
  float tw_re[NFFT];
  float tw_im[NFFT];
  float buf_re[STFT_WARPS][32 * 33];
  float buf_im[STFT_WARPS][32 * 33];
  float mag[STFT_WARPS][2][NBINS + 7];
};

__global__ void __launch_bounds__(STFT_WARPS * 32, 2)
stft_mel_kernel(const float* __restrict__ wav, int n_samples, int n_frames, int pairs_per_clip, const float* __restrict__ basis,
                const __grid_constant__ MelBands bands, int n_mels, int normalizer, float* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  StftSmem& sm = *reinterpret_cast<StftSmem*>(smem_raw);
  for (int i = threadIdx.x; i < NFFT; i += blockDim.x) {
    sm.tw_re[i] = g_tw_re[i];
    sm.tw_im[i] = g_tw_im[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int clip = blockIdx.y;
  const int pair = blockIdx.x * STFT_WARPS + warp;
  if (pair >= pairs_per_clip) return;
  const float* x = wav + (size_t)clip * n_samples;
  const int fA = 2 * pair, fB = 2 * pair + 1;
  const bool hasB = fB < n_frames;
  float* bre = sm.buf_re[warp];
  float* bim = sm.buf_im[warp];

  // ---- pass 1: lane n2 transforms x[32*n1 + n2], n1 = 0..31
  float re[32], im[32];
  const int sA = fA * HOP - NFFT / 2, sB = fB * HOP - NFFT / 2;
  const bool interior = sA >= 0 && (hasB ? sB : sA) + NFFT <= n_samples;
#pragma unroll
  for (int n1 = 0; n1 < 32; ++n1) {
    const int i = 32 * n1 + lane;
    const float w = g_window[i];
    float a, b;
    if (interior) {
      a = __ldg(x + sA + i);
      b = hasB ? __ldg(x + sB + i) : 0.f;
    } else {
      a = sample_reflect(x, n_samples, sA + i);
      b = hasB ? sample_reflect(x, n_samples, sB + i) : 0.f;
    }
    re[n1] = a * w;
    im[n1] = b * w;
  }
  fft32(re, im);
  // ---- twiddle by W_1024^(n2*k1) and transpose through shared memory: slot i holds k1 = bitrev5(i)
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int k1 = bitrev5(i);
    const int tw = (lane * k1) & (NFFT - 1);
    const float c = sm.tw_re[tw], s = sm.tw_im[tw];
    bre[k1 * 33 + lane] = re[i] * c - im[i] * s;
    bim[k1 * 33 + lane] = re[i] * s + im[i] * c;
  }
  __syncwarp();
  // ---- pass 2: lane k1 transforms over n2
#pragma unroll
  for (int n2 = 0; n2 < 32; ++n2) {
    re[n2] = bre[lane * 33 + n2];
    im[n2] = bim[lane * 33 + n2];
  }
  __syncwarp();
  fft32(re, im);
  // Z[k1 + 32*k2] with k2 = bitrev5(i) -> shared (aliases the transpose buffer; 1024 <= 32*33)
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int k = lane + 32 * bitrev5(i);
    bre[k] = re[i];
    bim[k] = im[i];
  }
  __syncwarp();
  // ---- separate the two real spectra, magnitudes
  float* magA = sm.mag[warp][0];
  float* magB = sm.mag[warp][1];
  for (int k = lane; k < NBINS; k += 32) {
    const int k2 = (NFFT - k) & (NFFT - 1);
    const float z1r = bre[k], z1i = bim[k], z2r = bre[k2], z2i = bim[k2];
    const float ar = 0.5f * (z1r + z2r), ai = 0.5f * (z1i - z2i);
    const float br = 0.5f * (z1i + z2i), bi = -0.5f * (z1r - z2r);
    magA[k] = sqrtf(ar * ar + ai * ai);
    magB[k] = sqrtf(br * br + bi * bi);
  }
  __syncwarp();
  // ---- banded mel filterbank + normaliser
  for (int m = lane; m < n_mels; m += 32) {
    const int lo = bands.lo[m], hi = lo + bands.len[m];
    float accA = 0.f, accB = 0.f;
    for (int k = lo; k < hi; ++k) {
      const float wgt = __ldg(basis + (size_t)m * NBINS + k);
      accA = fmaf(wgt, magA[k], accA);
      accB = fmaf(wgt, magB[k], accB);
    }
    float ya, yb;
    if (normalizer == 0) {
      ya = logf(fmaxf(accA, 1e-5f));
      yb = logf(fmaxf(accB, 1e-5f));
    } else {
      ya = 20.f * log10f(fmaxf(accA, 1e-5f));
      yb = 20.f * log10f(fmaxf(accB, 1e-5f));
      ya = fminf(fmaxf((ya + 100.f) / 100.f, 0.f), 1.f) * 8.f - 4.f;
      yb = fminf(fmaxf((yb + 100.f) / 100.f, 0.f), 1.f) * 8.f - 4.f;
    }
    out[((size_t)clip * n_frames + fA) * n_mels + m] = ya;
    if (hasB) out[((size_t)clip * n_frames + fB) * n_mels + m] = yb;
  }
}

// ----------------------------------------------------------------------------------------------------
// Version 2 of the fused kernel (the one ttsb_stft_mel_log launches; the kernel above runs band tables wider than the packed
// filterbank holds, and every basis under TTSB_STFT_V1=1 for A/B runs).
// Version 1 waits on global loads of samples, window, filter weights and band bounds with nothing to hide them behind, and
// its mel loop has shared-memory bank conflicts.  Changes:
//   * persistent warps; the samples of the NEXT frame pair are requested into the (dead) FFT registers before the
//     magnitude / mel phase of the current pair, so their latency is hidden behind ~500 instructions of other work;
//   * window, twiddles (as (cos, -sin) pairs), packed filter weights and band bounds live in shared memory;
//   * complex values cross shared memory as 8-byte (re, im) pairs (half the load / store instructions);
//   * only the bins below the highest non-zero filter tap are separated (372 of 513 at f_max = 8 kHz), magnitudes with
//     x * rsqrt(x) instead of the IEEE sqrt sequence;
//   * the filterbank is stored banded and packed (727 weights), a lane owns bands m, m+32, m+64.  Each block gathers the
//     packed weights from the rows of the call's own basis, at the bands the host computed from the call's band table: no
//     table outlives a launch, so a basis rewritten in place or a new basis at a freed address is read as it stands.
// ----------------------------------------------------------------------------------------------------
constexpr int V2_WARPS = 8;
constexpr int MAX_TAPS = 2048;          // packed non-zero filter weights (a triangular basis has < 2 * 513)

struct StftSmem2 {
  float2 tw[NFFT];                       // (cos, -sin)(2 pi i / 1024)
  float window[NFFT];
  float mel_w[MAX_TAPS];
  int mel_lo[MAX_MELS], mel_len[MAX_MELS], mel_off[MAX_MELS];
  float2 buf[V2_WARPS][32 * 33];         // per-warp transpose / spectrum buffer; later (|X_A|, |X_B|) per bin, in place
};

// samples of frame pair `pair` of one clip x (n_samples, n_frames) into the FFT registers, reflect-padded at the clip's edges
__device__ __forceinline__ void load_clip_pair(const float* __restrict__ x, int n_samples, int n_frames, int pair, int lane,
                                               float (&re)[32], float (&im)[32]) {
  const int fA = 2 * pair, fB = fA + 1;
  const bool hasB = fB < n_frames;
  const int sA = fA * HOP - NFFT / 2, sB = fB * HOP - NFFT / 2;
  if (sA >= 0 && (hasB ? sB : sA) + NFFT <= n_samples) {
#pragma unroll
    for (int n1 = 0; n1 < 32; ++n1) {
      re[n1] = __ldg(x + sA + 32 * n1 + lane);
      im[n1] = hasB ? __ldg(x + sB + 32 * n1 + lane) : 0.f;
    }
  } else {
#pragma unroll
    for (int n1 = 0; n1 < 32; ++n1) {
      re[n1] = sample_reflect(x, n_samples, sA + 32 * n1 + lane);
      im[n1] = hasB ? sample_reflect(x, n_samples, sB + 32 * n1 + lane) : 0.f;
    }
  }
}

__device__ __forceinline__ void load_pair(const float* __restrict__ wav, int n_samples, int n_frames, int pairs_per_clip, int item,
                                          int lane, float (&re)[32], float (&im)[32]) {
  const int clip = item / pairs_per_clip, pair = item - clip * pairs_per_clip;
  load_clip_pair(wav + (size_t)clip * n_samples, n_samples, n_frames, pair, lane, re, im);
}

// shared-memory tables of the v2 kernels; the packed filterbank is gathered from the rows of the call's own basis
__device__ __forceinline__ void load_v2_tables(StftSmem2& sm, const float* __restrict__ basis, const MelBands& bands, int n_mels) {
  for (int i = threadIdx.x; i < NFFT; i += blockDim.x) {
    sm.tw[i] = make_float2(g_tw_re[i], g_tw_im[i]);
    sm.window[i] = g_window[i];
  }
  for (int i = threadIdx.x; i < MAX_MELS; i += blockDim.x) {
    sm.mel_lo[i] = bands.lo[i];
    sm.mel_len[i] = i < n_mels ? bands.len[i] : 0;
    sm.mel_off[i] = bands.off[i];
  }
  __syncthreads();
  // one independent load per packed weight: weight i belongs to the last row m with off[m] <= i (rows are packed in order)
  for (int i = threadIdx.x; i < bands.taps; i += blockDim.x) {
    int m = 0;
    for (int step = MAX_MELS / 2; step > 0; step >>= 1)
      if (m + step < n_mels && sm.mel_off[m + step] <= i) m += step;
    sm.mel_w[i] = __ldg(basis + (size_t)m * NBINS + sm.mel_lo[m] + (i - sm.mel_off[m]));
  }
  __syncthreads();
}

// One frame pair, samples already in re / im: window, 1024-point complex FFT, spectra, mel filterbank, normaliser; rows outA and
// (when outB is not NULL) outB of the output.  `prefetch` runs as soon as the FFT registers are dead (the v2 kernels request the
// next pair's samples there).
template <class Prefetch>
__device__ __forceinline__ void mel_pair(const StftSmem2& sm, float2* buf, int lane, int kmax, int n_mels, int normalizer,
                                         float (&re)[32], float (&im)[32], float* __restrict__ outA, float* __restrict__ outB,
                                         Prefetch prefetch) {
  // ---- window, pass 1 (lane n2 transforms over n1)
#pragma unroll
  for (int n1 = 0; n1 < 32; ++n1) {
    const float w = sm.window[32 * n1 + lane];
    re[n1] *= w;
    im[n1] *= w;
  }
  fft32(re, im);
  // ---- twiddle by W_1024^(n2*k1) and transpose through shared memory: slot i holds k1 = bitrev5(i)
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int k1 = bitrev5(i);
    const float2 t = sm.tw[(lane * k1) & (NFFT - 1)];
    buf[k1 * 33 + lane] = make_float2(re[i] * t.x - im[i] * t.y, re[i] * t.y + im[i] * t.x);
  }
  __syncwarp();
  // ---- pass 2 (lane k1 transforms over n2)
#pragma unroll
  for (int n2 = 0; n2 < 32; ++n2) {
    const float2 v = buf[lane * 33 + n2];
    re[n2] = v.x;
    im[n2] = v.y;
  }
  __syncwarp();
  fft32(re, im);
#pragma unroll
  for (int i = 0; i < 32; ++i) buf[lane + 32 * bitrev5(i)] = make_float2(re[i], im[i]);   // Z[k1 + 32 k2], natural order
  __syncwarp();
  // ---- the FFT registers are dead
  prefetch();
  // ---- separate the two real spectra (bins below the highest filter tap); the magnitudes (|X_A[k]|, |X_B[k]|) replace
  //      Z[k] in place: bin k is only ever read together with bin N-k > 512 by the lane that owns k
  for (int k = lane; k < kmax; k += 32) {
    const float2 z1 = buf[k], z2 = buf[(NFFT - k) & (NFFT - 1)];
    const float ar = z1.x + z2.x, ai = z1.y - z2.y;      // 2 X_A[k]
    const float br = z1.y + z2.y, bi = z1.x - z2.x;      // 2 X_B[k] (up to a rotation by -i: same magnitude)
    const float pa = ar * ar + ai * ai, pb = br * br + bi * bi;
    buf[k] = make_float2(pa > 0.f ? 0.5f * pa * rsqrtf(pa) : 0.f, pb > 0.f ? 0.5f * pb * rsqrtf(pb) : 0.f);
  }
  __syncwarp();
  // ---- banded mel filterbank + normaliser: lane owns bands lane, lane + 32, lane + 64, ...
  for (int m = lane; m < n_mels; m += 32) {
    const int lo = sm.mel_lo[m], len = sm.mel_len[m];
    const float* w = sm.mel_w + sm.mel_off[m];
    float accA = 0.f, accB = 0.f;
    for (int i = 0; i < len; ++i) {
      const float wgt = w[i];
      const float2 mg = buf[lo + i];
      accA = fmaf(wgt, mg.x, accA);
      accB = fmaf(wgt, mg.y, accB);
    }
    float ya, yb;
    if (normalizer == 0) {
      ya = logf(fmaxf(accA, 1e-5f));
      yb = logf(fmaxf(accB, 1e-5f));
    } else {
      ya = 20.f * log10f(fmaxf(accA, 1e-5f));
      yb = 20.f * log10f(fmaxf(accB, 1e-5f));
      ya = fminf(fmaxf((ya + 100.f) / 100.f, 0.f), 1.f) * 8.f - 4.f;
      yb = fminf(fmaxf((yb + 100.f) / 100.f, 0.f), 1.f) * 8.f - 4.f;
    }
    outA[m] = ya;
    if (outB) outB[m] = yb;
  }
  __syncwarp();   // buf / mag are rewritten by the next iteration
}

__global__ void __launch_bounds__(V2_WARPS * 32, 2)
stft_mel_v2_kernel(const float* __restrict__ wav, int n_samples, int n_frames, int pairs_per_clip, int n_items,
                   const float* __restrict__ basis, const __grid_constant__ MelBands bands, int n_mels, int normalizer,
                   float* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  StftSmem2& sm = *reinterpret_cast<StftSmem2*>(smem_raw);
  load_v2_tables(sm, basis, bands, n_mels);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kmax = bands.kmax;
  const int gw = blockIdx.x * V2_WARPS + warp, nw = gridDim.x * V2_WARPS;
  float2* buf = sm.buf[warp];
  float re[32], im[32];
  int item = gw;
  if (item < n_items) load_pair(wav, n_samples, n_frames, pairs_per_clip, item, lane, re, im);
  for (; item < n_items; item += nw) {
    const int clip = item / pairs_per_clip, pair = item - clip * pairs_per_clip;
    const int fA = 2 * pair, fB = fA + 1;
    float* outA = out + ((size_t)clip * n_frames + fA) * n_mels;
    mel_pair(sm, buf, lane, kmax, n_mels, normalizer, re, im, outA, fB < n_frames ? outA + n_mels : nullptr, [&] {
      if (item + nw < n_items) load_pair(wav, n_samples, n_frames, pairs_per_clip, item + nw, lane, re, im);
    });
  }
}

// ---- packed ragged batch (ttsb_stft_mel_log_batch).  The clip table (uploaded by the entry point) holds three (n_clips + 1)
// prefix arrays: so[c] first sample, fo[c] first output frame, po[c] first frame PAIR of clip c.  A pair never spans two clips.
__device__ __forceinline__ void load_batch_pair(const float* __restrict__ wav, const int32_t* __restrict__ tab, int n_clips, int item,
                                                int lane, float (&re)[32], float (&im)[32]) {
  const int32_t* so = tab;
  const int32_t* fo = tab + (n_clips + 1);
  const int32_t* po = tab + 2 * (n_clips + 1);
  const int c = find_clip(po, n_clips, item);
  const int s0 = __ldg(so + c);
  load_clip_pair(wav + s0, __ldg(so + c + 1) - s0, __ldg(fo + c + 1) - __ldg(fo + c), item - __ldg(po + c), lane, re, im);
}

__global__ void __launch_bounds__(V2_WARPS * 32, 2)
stft_mel_batch_kernel(const float* __restrict__ wav, const int32_t* __restrict__ tab, int n_clips, int n_items,
                      const float* __restrict__ basis, const __grid_constant__ MelBands bands, int n_mels, int normalizer,
                      float* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  StftSmem2& sm = *reinterpret_cast<StftSmem2*>(smem_raw);
  load_v2_tables(sm, basis, bands, n_mels);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kmax = bands.kmax;
  const int gw = blockIdx.x * V2_WARPS + warp, nw = gridDim.x * V2_WARPS;
  float2* buf = sm.buf[warp];
  const int32_t* fo = tab + (n_clips + 1);
  const int32_t* po = tab + 2 * (n_clips + 1);
  float re[32], im[32];
  int item = gw;
  if (item < n_items) load_batch_pair(wav, tab, n_clips, item, lane, re, im);
  for (; item < n_items; item += nw) {
    const int c = find_clip(po, n_clips, item);
    const int fA = 2 * (item - __ldg(po + c));
    const int T = __ldg(fo + c + 1) - __ldg(fo + c);
    float* outA = out + ((size_t)__ldg(fo + c) + fA) * n_mels;
    mel_pair(sm, buf, lane, kmax, n_mels, normalizer, re, im, outA, fA + 1 < T ? outA + n_mels : nullptr, [&] {
      if (item + nw < n_items) load_batch_pair(wav, tab, n_clips, item + nw, lane, re, im);
    });
  }
}

static int init_tables() {
  static PerDevice<bool> done_pd;  // __constant__ tables and function attributes are per device
  bool& done = done_pd.get();
  if (done) return 0;
  static float tr[NFFT], ti[NFFT], win[NFFT];
  for (int i = 0; i < NFFT; ++i) {
    const double a = 2.0 * M_PI * (double)i / (double)NFFT;
    tr[i] = (float)cos(a);
    ti[i] = (float)(-sin(a));
    win[i] = (float)(0.5 - 0.5 * cos(a));
  }
  TTSB_CUDA_OK(cudaMemcpyToSymbol(g_tw_re, tr, sizeof(tr)));
  TTSB_CUDA_OK(cudaMemcpyToSymbol(g_tw_im, ti, sizeof(ti)));
  TTSB_CUDA_OK(cudaMemcpyToSymbol(g_window, win, sizeof(win)));
  TTSB_CUDA_OK(cudaFuncSetAttribute(stft_mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(StftSmem)));
  TTSB_CUDA_OK(cudaFuncSetAttribute(stft_mel_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(StftSmem2)));
  TTSB_CUDA_OK(cudaFuncSetAttribute(stft_mel_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(StftSmem2)));
  done = true;
  return 0;
}

// lo / len / off / kmax of the caller's band table (n_mels, 2) int32 in host memory: band[2m], band[2m+1] = first / past-last
// non-zero bin of row m.  Returns 0, or TTSB_ERR_INVALID_ARGUMENT for a row outside 0 <= first <= past-last <= 513.  *packed = 0
// when the rows hold more weights than the packed table of the v2 kernels (MAX_TAPS).
static int mel_bands(const char* who, const int32_t* band, int n_mels, MelBands* b, bool* packed) {
  *b = MelBands{};
  int off = 0;
  for (int m = 0; m < n_mels; ++m) {
    const int lo = band[2 * m], hi = band[2 * m + 1];
    if (lo < 0 || hi < lo || hi > NBINS) {
      set_last_error("%s: band row %d is [%d, %d); need 0 <= band[2m] <= band[2m+1] <= 513", who, m, lo, hi);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
    b->lo[m] = lo;
    b->len[m] = hi - lo;
    b->off[m] = off;
    b->kmax = max(b->kmax, hi);
    off += hi - lo;
  }
  b->taps = off;
  *packed = off <= MAX_TAPS;
  return 0;
}

}  // namespace ttsb

using namespace ttsb;

extern "C" int ttsb_stft_mel_log(const float* wav, int n_clips, int n_samples, const float* mel_basis, const int32_t* band,
                                 int n_mels, int normalizer, float* out, void* stream_v) {
  if (!wav || !mel_basis || !band || !out) { set_last_error("ttsb_stft_mel_log: NULL tensor"); return TTSB_ERR_INVALID_ARGUMENT; }
  if (n_clips <= 0) { set_last_error("ttsb_stft_mel_log: n_clips %d; need n_clips >= 1", n_clips); return TTSB_ERR_INVALID_ARGUMENT; }
  if (n_samples <= NFFT / 2) {
    set_last_error("ttsb_stft_mel_log: n_samples %d; need n_samples > 512", n_samples);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (n_mels <= 0 || n_mels > MAX_MELS) { set_last_error("ttsb_stft_mel_log: n_mels %d; need 0 < n_mels <= 128", n_mels); return TTSB_ERR_INVALID_ARGUMENT; }
  if (normalizer != 0 && normalizer != 1) {
    set_last_error("ttsb_stft_mel_log: normalizer %d; need normalizer in {0,1}", normalizer);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  MelBands bands;
  bool packed;
  int rc = mel_bands("ttsb_stft_mel_log", band, n_mels, &bands, &packed);
  if (rc) return rc;
  rc = init_tables();
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int n_frames = 1 + n_samples / HOP;
  const int pairs = (n_frames + 1) / 2;
  static const bool use_v1 = getenv("TTSB_STFT_V1") != nullptr;
  if (!use_v1 && packed) {
    const int n_items = pairs * n_clips;
    const int grid2 = min((n_items + V2_WARPS - 1) / V2_WARPS, 2 * num_sms());
    stft_mel_v2_kernel<<<grid2, V2_WARPS * 32, sizeof(StftSmem2), stream>>>(wav, n_samples, n_frames, pairs, n_items, mel_basis, bands,
                                                                            n_mels, normalizer, out);
    count_launch();
    return check_cuda(cudaGetLastError(), "stft_mel_v2_kernel launch");
  }
  dim3 grid((pairs + STFT_WARPS - 1) / STFT_WARPS, n_clips);
  stft_mel_kernel<<<grid, STFT_WARPS * 32, sizeof(StftSmem), stream>>>(wav, n_samples, n_frames, pairs, mel_basis, bands, n_mels,
                                                                        normalizer, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "stft_mel_kernel launch");
}

static int mel_batch_bad(const char* fmt, long long a = 0, long long b = 0) {
  set_last_error(fmt, a, b);
  return TTSB_ERR_INVALID_ARGUMENT;
}

extern "C" int64_t ttsb_stft_mel_log_batch_workspace_bytes(int n_clips) {
  if (n_clips < 1) {
    set_last_error("ttsb_stft_mel_log_batch_workspace_bytes: n_clips < 1");
    return -1;
  }
  return 3 * (int64_t)(n_clips + 1) * (int64_t)sizeof(int32_t);
}

extern "C" int ttsb_stft_mel_log_batch(const float* wav, const int32_t* sample_offsets, const int32_t* frame_offsets, int n_clips,
                                       const float* mel_basis, const int32_t* band, int n_mels, int normalizer, void* workspace,
                                       int64_t workspace_bytes, float* out, void* stream_v) {
  if (!wav || !sample_offsets || !frame_offsets || !mel_basis || !band || !workspace || !out)
    return mel_batch_bad("ttsb_stft_mel_log_batch: NULL pointer");
  if (n_clips < 1) return mel_batch_bad("ttsb_stft_mel_log_batch: n_clips %lld; need n_clips >= 1", n_clips);
  if (n_mels <= 0 || n_mels > MAX_MELS) return mel_batch_bad("ttsb_stft_mel_log_batch: n_mels %lld; need 0 < n_mels <= 128", n_mels);
  if (normalizer != 0 && normalizer != 1)
    return mel_batch_bad("ttsb_stft_mel_log_batch: normalizer %lld; need normalizer in {0,1}", normalizer);
  if (workspace_bytes < ttsb_stft_mel_log_batch_workspace_bytes(n_clips))
    return mel_batch_bad("ttsb_stft_mel_log_batch: workspace too small (ttsb_stft_mel_log_batch_workspace_bytes)");
  if (reinterpret_cast<uintptr_t>(workspace) % 4 != 0) return mel_batch_bad("ttsb_stft_mel_log_batch: workspace must be 4-byte aligned");
  if (sample_offsets[0] != 0 || frame_offsets[0] != 0) return mel_batch_bad("ttsb_stft_mel_log_batch: offsets must start at 0");
  std::vector<int32_t> tab(3 * (size_t)(n_clips + 1));
  int32_t* so = tab.data();
  int32_t* fo = so + (n_clips + 1);
  int32_t* po = fo + (n_clips + 1);
  long long p = 0;
  for (int c = 0; c < n_clips; ++c) {
    const long long L = (long long)sample_offsets[c + 1] - sample_offsets[c];
    if (L <= NFFT / 2) return mel_batch_bad("ttsb_stft_mel_log_batch: clip %lld has %lld samples; need more than 512", c, L);
    const long long T = 1 + L / HOP;
    if ((long long)frame_offsets[c + 1] - frame_offsets[c] != T)
      return mel_batch_bad("ttsb_stft_mel_log_batch: frame_offsets give clip %lld %lld frames; its samples give 1 + L/256", c,
                           (long long)frame_offsets[c + 1] - frame_offsets[c]);
    p += (T + 1) / 2;
    if (p > INT32_MAX) return mel_batch_bad("ttsb_stft_mel_log_batch: too many frames");
    so[c + 1] = sample_offsets[c + 1];
    fo[c + 1] = frame_offsets[c + 1];
    po[c + 1] = (int32_t)p;
  }
  MelBands bands;
  bool packed;
  int rc = mel_bands("ttsb_stft_mel_log_batch", band, n_mels, &bands, &packed);
  if (rc) return rc;
  if (!packed) {
    set_last_error("ttsb_stft_mel_log_batch: the band table spans more mel weights than the packed filterbank holds (%d)", MAX_TAPS);
    return TTSB_ERR_UNSUPPORTED;
  }
  rc = init_tables();
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  TTSB_CUDA_OK(cudaMemcpyAsync(workspace, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  const int n_items = (int)p;
  const int grid = min((n_items + V2_WARPS - 1) / V2_WARPS, 2 * num_sms());
  stft_mel_batch_kernel<<<grid, V2_WARPS * 32, sizeof(StftSmem2), stream>>>(wav, static_cast<const int32_t*>(workspace), n_clips, n_items,
                                                                             mel_basis, bands, n_mels, normalizer, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "stft_mel_batch_kernel launch");
}
