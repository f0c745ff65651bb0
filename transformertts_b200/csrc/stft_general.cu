// The STFT family at any supported configuration: n_fft a power of two in [256, 4096], 1 <= hop <= win_length <= n_fft, win_length >= 2,
// periodic Hann of win_length centred in n_fft (librosa's pad_center), centred frames with reflect padding.  The kernels of the
// reference configuration (1024 / 256 / 1024: stft_mel.cu, griffin_lim.cu) stay as they are; these serve every other one.
//
//   ttsb_stft_mel_log_ragged   : STFT -> magnitude -> banded mel filterbank -> normaliser of a packed ragged batch
//   ttsb_stft_complex_ragged   : librosa.stft of a packed ragged batch -> complex64 (frames, n_fft/2 + 1)
//   ttsb_istft_ragged          : librosa.istft of a packed ragged batch (window-sum-square normalisation, centre trim)
//   ttsb_griffinlim_ragged     : the Griffin-Lim loop of ttsb_griffinlim_batch (phase update fused into the iSTFT's spectrum
//                                load -> per-clip overlap-add -> per-clip complex STFT)
//   ttsb_mel_to_linear_ex      : ttsb_mel_to_linear's projected-gradient NNLS at n_fft/2 + 1 bins
//
// One CTA transforms TWO real frames of one clip as one n_fft-point complex FFT (frame A -> real part, frame B -> imaginary part;
// the inverse packs two Hermitian spectra the same way).  The FFT is an in-place radix-2 decimation-in-time transform in shared
// memory: the windowed samples are stored at bit-reversed positions, then log2(n_fft) butterfly passes, one __syncthreads each.
// The twiddles W_N^j (j < N/2) and the window are computed in float64 on the host, rounded once and uploaded into the workspace
// with the clip table (one copy per call).  A frame pair never spans two clips, reflect padding happens at each clip's own edges
// and the overlap-add stays inside a clip, so a clip's output does not depend, bit for bit, on the batch around it.
#include <math.h>

#include <vector>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace ttsb {
namespace sg {

constexpr int MIN_NFFT = 256;
constexpr int MAX_NFFT = 4096;
constexpr int THREADS = 256;
constexpr int MAX_MELS = 128;

// what every kernel needs to know of the configuration; tw and win point into the workspace
struct Cfg {
  int n_fft, log2n, hop, n_bins;
  const float2* tw;   // (cos, -sin)(2 pi j / n_fft), j < n_fft / 2
  const float* win;   // periodic Hann(win_length) centred in n_fft, zero outside
};

__device__ __forceinline__ float sample_reflect(const float* __restrict__ x, int n, int i) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return __ldg(x + i);
}

__device__ __forceinline__ int bitrev(int i, int log2n) { return (int)(__brev((unsigned)i) >> (32 - log2n)); }

// In-place forward FFT of z (natural order out) whose input was stored at bit-reversed positions; ends with __syncthreads.
__device__ __forceinline__ void block_fft(float2* z, const Cfg& cfg) {
  const int half_n = cfg.n_fft >> 1;
  for (int s = 1; s <= cfg.log2n; ++s) {
    const int half = 1 << (s - 1);
    const int tstep = cfg.n_fft >> s;                  // W_{2 half}^j = W_N^{j N / (2 half)}
    for (int b = threadIdx.x; b < half_n; b += blockDim.x) {
      const int j = b & (half - 1);
      const int i0 = ((b >> (s - 1)) << s) + j, i1 = i0 + half;
      const float2 w = __ldg(cfg.tw + j * tstep);
      const float2 u = z[i0], v = z[i1];
      const float tr = v.x * w.x - v.y * w.y, ti = v.x * w.y + v.y * w.x;
      z[i0] = make_float2(u.x + tr, u.y + ti);
      z[i1] = make_float2(u.x - tr, u.y - ti);
    }
    __syncthreads();
  }
}

// windowed samples of frames lA and lA + 1 (if hasB) of a clip x of L samples -> z at bit-reversed positions, then the FFT
__device__ __forceinline__ void stft_pair(const float* __restrict__ x, int L, int lA, bool hasB, const Cfg& cfg, float2* z) {
  const int sA = lA * cfg.hop - cfg.n_fft / 2, sB = sA + cfg.hop;
  for (int n = threadIdx.x; n < cfg.n_fft; n += blockDim.x) {
    const float w = __ldg(cfg.win + n);
    const float a = sample_reflect(x, L, sA + n) * w;
    const float b = hasB ? sample_reflect(x, L, sB + n) * w : 0.f;
    z[bitrev(n, cfg.log2n)] = make_float2(a, b);
  }
  __syncthreads();
  block_fft(z, cfg);
}

// Clip tables (int32 prefix arrays of n_clips + 1 entries each, built and checked on the host):
//   analysis  (log-mel, complex STFT): so first sample, fo first frame, po first frame pair of clip c
//   synthesis (iSTFT, Griffin-Lim)    : fo first frame, po first frame pair, wo first output sample of clip c
struct Clip {
  int c, first_frame, frames;
};
__device__ __forceinline__ Clip clip_of_pair(const int32_t* __restrict__ fo, const int32_t* __restrict__ po, int n_clips, int pair) {
  Clip k;
  k.c = find_clip(po, n_clips, pair);
  k.first_frame = __ldg(fo + k.c);
  k.frames = __ldg(fo + k.c + 1) - k.first_frame;
  return k;
}

// ---- log-mel of a packed ragged batch: one CTA per frame pair
__global__ void __launch_bounds__(THREADS)
stft_mel_ragged_kernel(const float* __restrict__ wav, const int32_t* __restrict__ tab, int n_clips, Cfg cfg,
                       const float* __restrict__ basis, const int32_t* __restrict__ band, int n_mels, int normalizer,
                       float* __restrict__ out) {
  extern __shared__ float2 smem[];
  float2* z = smem;                      // n_fft
  float2* mag = smem + cfg.n_fft;        // (|X_A[k]|, |X_B[k]|), n_bins
  const int32_t* so = tab;
  const int32_t* fo = tab + (n_clips + 1);
  const int32_t* po = tab + 2 * (n_clips + 1);
  const int pair = blockIdx.x;
  const Clip k = clip_of_pair(fo, po, n_clips, pair);
  const int lA = 2 * (pair - __ldg(po + k.c));
  const bool hasB = lA + 1 < k.frames;
  const int s0 = __ldg(so + k.c);
  stft_pair(wav + s0, __ldg(so + k.c + 1) - s0, lA, hasB, cfg, z);
  // separate the two real spectra: X_A[k] = (Z[k] + conj Z[N-k]) / 2, X_B[k] = (Z[k] - conj Z[N-k]) / (2i)
  for (int b = threadIdx.x; b < cfg.n_bins; b += blockDim.x) {
    const float2 z1 = z[b], z2 = z[(cfg.n_fft - b) & (cfg.n_fft - 1)];
    const float ar = z1.x + z2.x, ai = z1.y - z2.y;
    const float br = z1.y + z2.y, bi = z1.x - z2.x;
    mag[b] = make_float2(0.5f * sqrtf(ar * ar + ai * ai), 0.5f * sqrtf(br * br + bi * bi));
  }
  __syncthreads();
  // banded mel filterbank (row m of the dense basis is non-zero on [band lo, hi), clamped to the row) + normaliser
  float* outA = out + ((size_t)k.first_frame + lA) * n_mels;
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    const int lo = max(__ldg(band + 2 * m), 0), hi = min(__ldg(band + 2 * m + 1), cfg.n_bins);
    const float* w = basis + (size_t)m * cfg.n_bins;
    float accA = 0.f, accB = 0.f;
    for (int b = lo; b < hi; ++b) {
      const float wgt = __ldg(w + b);
      const float2 mg = mag[b];
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
    if (hasB) outA[n_mels + m] = yb;
  }
}

// ---- complex STFT of the clips of an analysis table (so, fo, po) -> out (frames, n_bins)
__device__ __forceinline__ void stft_complex_pair(const float* __restrict__ wav, const int32_t* __restrict__ so,
                                                  const int32_t* __restrict__ fo, const int32_t* __restrict__ po, int n_clips,
                                                  const Cfg& cfg, float2* __restrict__ out, float2* z) {
  const int pair = blockIdx.x;
  const Clip k = clip_of_pair(fo, po, n_clips, pair);
  const int lA = 2 * (pair - __ldg(po + k.c));
  const bool hasB = lA + 1 < k.frames;
  const int s0 = __ldg(so + k.c);
  stft_pair(wav + s0, __ldg(so + k.c + 1) - s0, lA, hasB, cfg, z);
  float2* A = out + ((size_t)k.first_frame + lA) * cfg.n_bins;
  for (int b = threadIdx.x; b < cfg.n_bins; b += blockDim.x) {
    const float2 z1 = z[b], z2 = z[(cfg.n_fft - b) & (cfg.n_fft - 1)];
    A[b] = make_float2(0.5f * (z1.x + z2.x), 0.5f * (z1.y - z2.y));
    if (hasB) A[cfg.n_bins + b] = make_float2(0.5f * (z1.y + z2.y), -0.5f * (z1.x - z2.x));
  }
}

__global__ void __launch_bounds__(THREADS)
stft_complex_ragged_kernel(const float* __restrict__ wav, const int32_t* __restrict__ tab, int n_clips, Cfg cfg, float2* __restrict__ out) {
  extern __shared__ float2 smem[];
  stft_complex_pair(wav, tab, tab + (n_clips + 1), tab + 2 * (n_clips + 1), n_clips, cfg, out, smem);
}

// Griffin-Lim re-analysis: the waveform's clip c starts at wo[c] and has wo[c + 1] - wo[c] samples
__global__ void __launch_bounds__(THREADS)
stft_complex_synth_kernel(const float* __restrict__ wav, const int32_t* __restrict__ tab, int n_clips, Cfg cfg, float2* __restrict__ out) {
  extern __shared__ float2 smem[];
  stft_complex_pair(wav, tab + 2 * (n_clips + 1), tab, tab + (n_clips + 1), n_clips, cfg, out, smem);
}

// ---- phase update of "fast" Griffin-Lim for one bin (as griffin_lim.cu's gl_project): a = r - alpha t; S a / (|a| + 1e-16)
struct ProjLoad {
  const float2* __restrict__ spec;      // non-NULL: a stored spectrum (ttsb_istft_ragged)
  const float2* __restrict__ rebuilt;   // latest re-analysis of the waveform
  const float2* __restrict__ tprev;     // the one before (NULL on the first update)
  const float* __restrict__ S;          // target magnitudes
  const float2* __restrict__ init;      // non-NULL: first pass, S * init_angles
  float alpha;
  __device__ __forceinline__ float2 operator()(size_t i) const {
    if (spec != nullptr) return __ldg(spec + i);
    const float s = __ldg(S + i);
    if (init != nullptr) {
      const float2 a = __ldg(init + i);
      return make_float2(s * a.x, s * a.y);
    }
    float2 a = __ldg(rebuilt + i);
    if (tprev != nullptr) {
      const float2 t = __ldg(tprev + i);
      a.x = a.x - alpha * t.x;
      a.y = a.y - alpha * t.y;
    }
    const float mag = sqrtf(a.x * a.x + a.y * a.y) + 1e-16f;
    return make_float2(s * (a.x / mag), s * (a.y / mag));
  }
};

// ---- irfft * window of two spectra of one clip -> time frames (frames, n_fft); table: synthesis (fo, po, wo)
__global__ void __launch_bounds__(THREADS)
istft_frames_ragged_kernel(ProjLoad load, const int32_t* __restrict__ tab, int n_clips, Cfg cfg, float* __restrict__ frames) {
  extern __shared__ float2 smem[];
  float2* z = smem;
  const int32_t* fo = tab;
  const int32_t* po = tab + (n_clips + 1);
  const int pair = blockIdx.x;
  const Clip k = clip_of_pair(fo, po, n_clips, pair);
  const int fA = k.first_frame + 2 * (pair - __ldg(po + k.c));
  if (fA >= k.first_frame + k.frames) return;
  const bool hasB = fA + 1 < k.first_frame + k.frames;
  const int N = cfg.n_fft, nyq = N / 2;
  const size_t A = (size_t)fA * cfg.n_bins, B = A + cfg.n_bins;
  // conj(Z)[k], Z = A_full + i B_full, with the Hermitian extension X_full[k] = conj(X[N - k]) for k > N/2 and the imaginary
  // parts of the DC and Nyquist bins dropped (as numpy's irfft does)
  for (int b = threadIdx.x; b < N; b += blockDim.x) {
    const int kk = b <= nyq ? b : N - b;
    float2 a = load(A + kk);
    float2 c = hasB ? load(B + kk) : make_float2(0.f, 0.f);
    if (kk == 0 || kk == nyq) { a.y = 0.f; c.y = 0.f; }
    if (b > nyq) { a.y = -a.y; c.y = -c.y; }
    z[bitrev(b, cfg.log2n)] = make_float2(a.x - c.y, -(a.y + c.x));
  }
  __syncthreads();
  block_fft(z, cfg);
  // z[n] = conj(FFT(conj Z))[n] / N: frame A = Re / N, frame B = -Im / N
  const float inv_n = 1.f / N;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const float w = __ldg(cfg.win + n) * inv_n;
    frames[(size_t)fA * N + n] = z[n].x * w;
    if (hasB) frames[((size_t)fA + 1) * N + n] = -z[n].y * w;
  }
}

// ---- overlap-add + window-sum-square normalisation + centre trim, per clip: out[n] of the packed waveform
__global__ void overlap_add_ragged_kernel(const float* __restrict__ frames, const int32_t* __restrict__ tab, int n_clips, Cfg cfg,
                                          int n_out, float* __restrict__ out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_out) return;
  const int32_t* fo = tab;
  const int32_t* wo = tab + 2 * (n_clips + 1);
  const int c = find_clip(wo, n_clips, n);
  const int f0 = __ldg(fo + c), T = __ldg(fo + c + 1) - f0;
  const float* fr = frames + (size_t)f0 * cfg.n_fft;
  const int s = n - __ldg(wo + c) + cfg.n_fft / 2;   // position in the clip's untrimmed signal
  const int f_hi = min(s / cfg.hop, T - 1);
  const int f_lo = max((s - (cfg.n_fft - 1) + cfg.hop - 1) / cfg.hop, 0);
  float acc = 0.f, wss = 0.f;
  for (int f = f_lo; f <= f_hi; ++f) {
    const int i = s - f * cfg.hop;
    acc += __ldg(fr + (size_t)f * cfg.n_fft + i);
    const float w = __ldg(cfg.win + i);
    wss = fmaf(w, w, wss);
  }
  out[n] = wss > 1.17549435e-38f ? acc / wss : acc;
}

// ---- mel amplitudes (T, n_mels) -> linear magnitudes (T, n_bins): ttsb_mel_to_linear's solver, x and y in dynamic shared memory
__global__ void __launch_bounds__(256)
mel_to_linear_ex_kernel(const float* __restrict__ mel, int n_mels, int n_bins, const float* __restrict__ basis,
                        const float* __restrict__ pinv, const int* __restrict__ band, const int* __restrict__ bin_mels, float step,
                        int n_iter, float* __restrict__ out) {
  extern __shared__ float nnls_smem[];
  float* x = nnls_smem;
  float* y = x + n_bins;
  __shared__ float r[MAX_MELS], m[MAX_MELS];
  const int t = blockIdx.x;
  for (int i = threadIdx.x; i < n_mels; i += blockDim.x) m[i] = mel[(size_t)t * n_mels + i];
  __syncthreads();
  for (int k = threadIdx.x; k < n_bins; k += blockDim.x) {   // clipped least-squares start: max(pinv(A) m, 0)
    float acc = 0.f;
    for (int j = 0; j < n_mels; ++j) acc = fmaf(__ldg(pinv + (size_t)k * n_mels + j), m[j], acc);
    x[k] = y[k] = fmaxf(acc, 0.f);
  }
  __syncthreads();
  float tk = 1.f;
  for (int it = 0; it < n_iter; ++it) {
    for (int j = threadIdx.x; j < n_mels; j += blockDim.x) {       // r = A y - m
      float acc = 0.f;
      for (int k = band[2 * j]; k < band[2 * j + 1]; ++k) acc = fmaf(__ldg(basis + (size_t)j * n_bins + k), y[k], acc);
      r[j] = acc - m[j];
    }
    __syncthreads();
    const float tn = 0.5f * (1.f + sqrtf(1.f + 4.f * tk * tk));
    const float beta = (tk - 1.f) / tn;
    for (int k = threadIdx.x; k < n_bins; k += blockDim.x) {        // x+ = max(y - step A^T r, 0); FISTA extrapolation
      float g = 0.f;
      for (int j = bin_mels[2 * k]; j < bin_mels[2 * k + 1]; ++j) g = fmaf(__ldg(basis + (size_t)j * n_bins + k), r[j], g);
      const float xn = fmaxf(y[k] - step * g, 0.f);
      y[k] = xn + beta * (xn - x[k]);
      x[k] = xn;
    }
    tk = tn;
    __syncthreads();
  }
  for (int k = threadIdx.x; k < n_bins; k += blockDim.x) out[(size_t)t * n_bins + k] = x[k];
}

// ---------------------------------------------------------------------------------------------------- host side
int64_t align256(int64_t b) { return (b + 255) & ~int64_t(255); }

bool config_ok(int n_fft, int hop, int win) {
  return n_fft >= MIN_NFFT && n_fft <= MAX_NFFT && (n_fft & (n_fft - 1)) == 0 && win >= 2 && win <= n_fft && hop >= 1 && hop <= win;
}

int bad_config(const char* who, int n_fft, int hop, int win) {
  set_last_error("%s: unsupported STFT configuration n_fft %d, hop %d, win_length %d; need n_fft a power of two in [256, 4096] and "
                 "1 <= hop <= win_length <= n_fft, 2 <= win_length", who, n_fft, hop, win);
  return TTSB_ERR_INVALID_ARGUMENT;
}

int bad(const char* fmt, long long a = 0, long long b = 0, long long c = 0) {
  set_last_error(fmt, a, b, c);
  return TTSB_ERR_INVALID_ARGUMENT;
}

// Workspace: [twiddles (n_fft/2 float2) | window (n_fft float) | clip table (3 (n_clips + 1) int32) | per-op regions]
struct Layout {
  int64_t tw, win, table, extra, total;
};
Layout layout(int n_fft, int n_clips, int64_t extra_bytes) {
  Layout l;
  l.tw = 0;
  l.win = align256((int64_t)(n_fft / 2) * 8);
  l.table = l.win + align256((int64_t)n_fft * 4);
  l.extra = l.table + align256(3 * ((int64_t)n_clips + 1) * 4);
  l.total = l.extra + align256(extra_bytes);
  return l;
}

// host image of the twiddle / window / table regions; uploaded with one copy
struct HostTables {
  std::vector<unsigned char> bytes;
  int32_t* table;
  HostTables(const Layout& l, int n_fft, int win_length) : bytes((size_t)l.extra, 0) {
    float2* tw = reinterpret_cast<float2*>(bytes.data() + l.tw);
    for (int j = 0; j < n_fft / 2; ++j) {
      const double a = 2.0 * M_PI * (double)j / (double)n_fft;
      tw[j] = make_float2((float)cos(a), (float)(-sin(a)));
    }
    float* win = reinterpret_cast<float*>(bytes.data() + l.win);
    const int lpad = (n_fft - win_length) / 2;
    for (int i = 0; i < win_length; ++i) win[lpad + i] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * (double)i / (double)win_length));
    table = reinterpret_cast<int32_t*>(bytes.data() + l.table);
  }
};

Cfg make_cfg(void* workspace, const Layout& l, int n_fft, int hop) {
  Cfg c;
  c.n_fft = n_fft;
  c.log2n = 0;
  while ((1 << c.log2n) < n_fft) ++c.log2n;
  c.hop = hop;
  c.n_bins = n_fft / 2 + 1;
  c.tw = reinterpret_cast<const float2*>(static_cast<char*>(workspace) + l.tw);
  c.win = reinterpret_cast<const float*>(static_cast<char*>(workspace) + l.win);
  return c;
}

int upload(void* workspace, const HostTables& h, cudaStream_t stream) {
  TTSB_CUDA_OK(cudaMemcpyAsync(workspace, h.bytes.data(), h.bytes.size(), cudaMemcpyHostToDevice, stream));
  return 0;
}

int set_smem(const void* kernel, int bytes) {
  TTSB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return 0;
}

int fft_smem(int n_fft) { return n_fft * (int)sizeof(float2); }

// Analysis table (so, fo, po) from host sample offsets; frame_offsets (optional) must give every clip 1 + L / hop frames.
// Returns the number of frame pairs, or -1 after set_last_error.
long long analysis_table(const char* who, const int32_t* sample_offsets, const int32_t* frame_offsets, int n_clips, int n_fft, int hop,
                         int32_t* tab) {
  int32_t* so = tab;
  int32_t* fo = so + (n_clips + 1);
  int32_t* po = fo + (n_clips + 1);
  if (sample_offsets[0] != 0 || (frame_offsets && frame_offsets[0] != 0)) {
    set_last_error("%s: offsets must start at 0", who);
    return -1;
  }
  long long f = 0, p = 0;
  so[0] = fo[0] = po[0] = 0;
  for (int c = 0; c < n_clips; ++c) {
    const long long L = (long long)sample_offsets[c + 1] - sample_offsets[c];
    if (L <= n_fft / 2) {
      set_last_error("%s: clip %d has %lld samples; reflect padding at n_fft %d needs more than %d", who, c, L, n_fft, n_fft / 2);
      return -1;
    }
    const long long T = 1 + L / hop;
    if (frame_offsets && (long long)frame_offsets[c + 1] - frame_offsets[c] != T) {
      set_last_error("%s: frame_offsets give clip %d %lld frames; its %lld samples give 1 + L / hop = %lld", who, c,
                     (long long)frame_offsets[c + 1] - frame_offsets[c], L, T);
      return -1;
    }
    f += T;
    p += (T + 1) / 2;
    if (f > INT32_MAX / MAX_NFFT) {
      set_last_error("%s: more than %d frames in one call", who, INT32_MAX / MAX_NFFT);
      return -1;
    }
    so[c + 1] = sample_offsets[c + 1];
    fo[c + 1] = (int32_t)f;
    po[c + 1] = (int32_t)p;
  }
  return p;
}

// Synthesis table (fo, po, wo) from host frame offsets; every clip needs at least min_frames frames.  Returns the number of frame
// pairs, or -1 after set_last_error.
long long synthesis_table(const char* who, const int32_t* frame_offsets, int n_clips, int hop, int min_frames, int32_t* tab) {
  int32_t* fo = tab;
  int32_t* po = fo + (n_clips + 1);
  int32_t* wo = po + (n_clips + 1);
  if (frame_offsets[0] != 0) {
    set_last_error("%s: frame offsets must start at 0", who);
    return -1;
  }
  long long p = 0, w = 0;
  fo[0] = po[0] = wo[0] = 0;
  for (int c = 0; c < n_clips; ++c) {
    const long long T = (long long)frame_offsets[c + 1] - frame_offsets[c];
    if (T < min_frames) {
      set_last_error("%s: clip %d has %lld frames; need at least %d", who, c, T, min_frames);
      return -1;
    }
    p += (T + 1) / 2;
    w += (long long)hop * (T - 1);
    if (frame_offsets[c + 1] > INT32_MAX / MAX_NFFT || w > INT32_MAX) {
      set_last_error("%s: more than %d frames or 2^31 samples in one call", who, INT32_MAX / MAX_NFFT);
      return -1;
    }
    fo[c + 1] = frame_offsets[c + 1];
    po[c + 1] = (int32_t)p;
    wo[c + 1] = (int32_t)w;
  }
  return p;
}

}  // namespace sg
}  // namespace ttsb

using namespace ttsb;
using namespace ttsb::sg;

// ---- log-mel
extern "C" int64_t ttsb_stft_mel_log_ragged_workspace_bytes(int n_clips, int n_fft) {
  if (n_clips < 1 || n_fft < MIN_NFFT || n_fft > MAX_NFFT) {
    set_last_error("ttsb_stft_mel_log_ragged_workspace_bytes: need n_clips >= 1, n_fft in [256, 4096]");
    return -1;
  }
  return layout(n_fft, n_clips, 0).total;
}

extern "C" int ttsb_stft_mel_log_ragged(const float* wav, const int32_t* sample_offsets, const int32_t* frame_offsets, int n_clips,
                                        int n_fft, int hop_length, int win_length, const float* mel_basis, const int32_t* band, int n_mels,
                                        int normalizer, void* workspace, int64_t workspace_bytes, float* out, void* stream_v) {
  const char* who = "ttsb_stft_mel_log_ragged";
  if (!wav || !sample_offsets || !frame_offsets || !mel_basis || !band || !workspace || !out)
    return bad("ttsb_stft_mel_log_ragged: NULL pointer");
  if (!config_ok(n_fft, hop_length, win_length)) return bad_config(who, n_fft, hop_length, win_length);
  if (n_clips < 1 || n_mels < 1 || n_mels > MAX_MELS || (normalizer != 0 && normalizer != 1))
    return bad("ttsb_stft_mel_log_ragged: need n_clips >= 1, 0 < n_mels <= 128, normalizer in {0,1}");
  const Layout l = layout(n_fft, n_clips, 0);
  if (workspace_bytes < l.total) return bad("ttsb_stft_mel_log_ragged: workspace too small (ttsb_stft_mel_log_ragged_workspace_bytes)");
  if (reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return bad("ttsb_stft_mel_log_ragged: workspace must be 256-byte aligned");
  HostTables h(l, n_fft, win_length);
  const long long pairs = analysis_table(who, sample_offsets, frame_offsets, n_clips, n_fft, hop_length, h.table);
  if (pairs < 0) return TTSB_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int smem = fft_smem(n_fft) + (n_fft / 2 + 1) * (int)sizeof(float2);
  int rc = set_smem((const void*)stft_mel_ragged_kernel, smem);
  if (rc) return rc;
  rc = upload(workspace, h, stream);
  if (rc) return rc;
  stft_mel_ragged_kernel<<<(unsigned)pairs, THREADS, smem, stream>>>(wav, reinterpret_cast<const int32_t*>(static_cast<char*>(workspace) + l.table),
                                                                   n_clips, make_cfg(workspace, l, n_fft, hop_length), mel_basis, band,
                                                                   n_mels, normalizer, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "stft_mel_ragged_kernel launch");
}

// ---- complex STFT
extern "C" int64_t ttsb_stft_complex_ragged_workspace_bytes(int n_clips, int n_fft) {
  if (n_clips < 1 || n_fft < MIN_NFFT || n_fft > MAX_NFFT) {
    set_last_error("ttsb_stft_complex_ragged_workspace_bytes: need n_clips >= 1, n_fft in [256, 4096]");
    return -1;
  }
  return layout(n_fft, n_clips, 0).total;
}

extern "C" int ttsb_stft_complex_ragged(const float* wav, const int32_t* sample_offsets, int n_clips, int n_fft, int hop_length,
                                        int win_length, void* workspace, int64_t workspace_bytes, float* spec_out, void* stream_v) {
  const char* who = "ttsb_stft_complex_ragged";
  if (!wav || !sample_offsets || !workspace || !spec_out) return bad("ttsb_stft_complex_ragged: NULL pointer");
  if (!config_ok(n_fft, hop_length, win_length)) return bad_config(who, n_fft, hop_length, win_length);
  if (n_clips < 1) return bad("ttsb_stft_complex_ragged: n_clips < 1");
  const Layout l = layout(n_fft, n_clips, 0);
  if (workspace_bytes < l.total) return bad("ttsb_stft_complex_ragged: workspace too small (ttsb_stft_complex_ragged_workspace_bytes)");
  if (reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return bad("ttsb_stft_complex_ragged: workspace must be 256-byte aligned");
  HostTables h(l, n_fft, win_length);
  const long long pairs = analysis_table(who, sample_offsets, nullptr, n_clips, n_fft, hop_length, h.table);
  if (pairs < 0) return TTSB_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  int rc = set_smem((const void*)stft_complex_ragged_kernel, fft_smem(n_fft));
  if (rc) return rc;
  rc = upload(workspace, h, stream);
  if (rc) return rc;
  stft_complex_ragged_kernel<<<(unsigned)pairs, THREADS, fft_smem(n_fft), stream>>>(
      wav, reinterpret_cast<const int32_t*>(static_cast<char*>(workspace) + l.table), n_clips, make_cfg(workspace, l, n_fft, hop_length),
      reinterpret_cast<float2*>(spec_out));
  count_launch();
  return check_cuda(cudaGetLastError(), "stft_complex_ragged_kernel launch");
}

// ---- iSTFT and Griffin-Lim: the extra region holds the time frames (F, n_fft) and, for Griffin-Lim, two spectra (F, n_bins)
namespace {
int64_t frames_bytes(int F, int n_fft) { return align256((int64_t)F * n_fft * 4); }
int64_t spec_bytes(int F, int n_fft) { return align256((int64_t)F * (n_fft / 2 + 1) * 8); }
bool synth_shape_ok(int F, int n_clips, int n_fft) {
  return n_clips >= 1 && F >= 2 * (int64_t)n_clips && n_fft >= MIN_NFFT && n_fft <= MAX_NFFT && F <= INT32_MAX / MAX_NFFT;
}

// launches of one iSTFT: frames from `load`, then the per-clip overlap-add
void istft_launch(const ProjLoad& load, const int32_t* tab, int n_clips, const Cfg& cfg, long long pairs, float* frames, int n_out,
                  float* wav_out, cudaStream_t stream) {
  istft_frames_ragged_kernel<<<(unsigned)pairs, THREADS, fft_smem(cfg.n_fft), stream>>>(load, tab, n_clips, cfg, frames);
  count_launch();
  overlap_add_ragged_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, stream>>>(frames, tab, n_clips, cfg, n_out, wav_out);
  count_launch();
}
}  // namespace

extern "C" int64_t ttsb_istft_ragged_workspace_bytes(int total_frames, int n_clips, int n_fft) {
  if (!synth_shape_ok(total_frames, n_clips, n_fft)) {
    set_last_error("ttsb_istft_ragged_workspace_bytes: need n_clips >= 1, 2 n_clips <= total_frames <= %d, n_fft in [256, 4096]",
                   INT32_MAX / MAX_NFFT);
    return -1;
  }
  return layout(n_fft, n_clips, frames_bytes(total_frames, n_fft)).total;
}

extern "C" int ttsb_istft_ragged(const float* spec, const int32_t* frame_offsets, int n_clips, int n_fft, int hop_length, int win_length,
                                 void* workspace, int64_t workspace_bytes, float* wav_out, void* stream_v) {
  const char* who = "ttsb_istft_ragged";
  if (!spec || !frame_offsets || !workspace || !wav_out) return bad("ttsb_istft_ragged: NULL pointer");
  if (!config_ok(n_fft, hop_length, win_length)) return bad_config(who, n_fft, hop_length, win_length);
  if (n_clips < 1) return bad("ttsb_istft_ragged: n_clips < 1");
  const int F = frame_offsets[n_clips];
  if (!synth_shape_ok(F, n_clips, n_fft))
    return bad("ttsb_istft_ragged: need 2 n_clips <= total frames <= %lld (got %lld frames)", INT32_MAX / MAX_NFFT, F);
  const Layout l = layout(n_fft, n_clips, frames_bytes(F, n_fft));
  if (workspace_bytes < l.total) return bad("ttsb_istft_ragged: workspace too small (ttsb_istft_ragged_workspace_bytes)");
  if (reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return bad("ttsb_istft_ragged: workspace must be 256-byte aligned");
  HostTables h(l, n_fft, win_length);
  const long long pairs = synthesis_table(who, frame_offsets, n_clips, hop_length, 2, h.table);
  if (pairs < 0) return TTSB_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  int rc = set_smem((const void*)istft_frames_ragged_kernel, fft_smem(n_fft));
  if (rc) return rc;
  rc = upload(workspace, h, stream);
  if (rc) return rc;
  char* ws = static_cast<char*>(workspace);
  ProjLoad load{reinterpret_cast<const float2*>(spec), nullptr, nullptr, nullptr, nullptr, 0.f};
  istft_launch(load, reinterpret_cast<const int32_t*>(ws + l.table), n_clips, make_cfg(workspace, l, n_fft, hop_length), pairs,
               reinterpret_cast<float*>(ws + l.extra), h.table[3 * (n_clips + 1) - 1], wav_out, stream);
  return check_cuda(cudaGetLastError(), "istft ragged kernels launch");
}

extern "C" int64_t ttsb_griffinlim_ragged_workspace_bytes(int total_frames, int n_clips, int n_fft) {
  if (!synth_shape_ok(total_frames, n_clips, n_fft)) {
    set_last_error("ttsb_griffinlim_ragged_workspace_bytes: need n_clips >= 1, 2 n_clips <= total_frames <= %d, n_fft in [256, 4096]",
                   INT32_MAX / MAX_NFFT);
    return -1;
  }
  return layout(n_fft, n_clips, frames_bytes(total_frames, n_fft) + 2 * spec_bytes(total_frames, n_fft)).total;
}

extern "C" int ttsb_griffinlim_ragged(const float* magnitude, const float* init_angles, const int32_t* frame_offsets, int n_clips,
                                      int n_fft, int hop_length, int win_length, int n_iter, float momentum, void* workspace,
                                      int64_t workspace_bytes, float* wav_out, void* stream_v) {
  const char* who = "ttsb_griffinlim_ragged";
  if (!magnitude || !init_angles || !frame_offsets || !workspace || !wav_out) return bad("ttsb_griffinlim_ragged: NULL pointer");
  if (!config_ok(n_fft, hop_length, win_length)) return bad_config(who, n_fft, hop_length, win_length);
  if (n_clips < 1) return bad("ttsb_griffinlim_ragged: n_clips < 1");
  if (n_iter < 0) return bad("ttsb_griffinlim_ragged: n_iter < 0");
  if (!(momentum >= 0.f) || isinf(momentum)) return bad("ttsb_griffinlim_ragged: momentum must be finite and >= 0");
  const int F = frame_offsets[n_clips];
  if (!synth_shape_ok(F, n_clips, n_fft))
    return bad("ttsb_griffinlim_ragged: need 2 n_clips <= total frames <= %lld (got %lld frames)", INT32_MAX / MAX_NFFT, F);
  const int64_t fb = frames_bytes(F, n_fft), sb = spec_bytes(F, n_fft);
  const Layout l = layout(n_fft, n_clips, fb + 2 * sb);
  if (workspace_bytes < l.total) return bad("ttsb_griffinlim_ragged: workspace too small (ttsb_griffinlim_ragged_workspace_bytes)");
  if (reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return bad("ttsb_griffinlim_ragged: workspace must be 256-byte aligned");
  // the re-analysis of a clip's hop (T - 1) samples gives T frames only when that is more than n_fft / 2 samples
  const int min_frames = n_fft / 2 / hop_length + 2;
  HostTables h(l, n_fft, win_length);
  const long long pairs = synthesis_table(who, frame_offsets, n_clips, hop_length, min_frames, h.table);
  if (pairs < 0) return TTSB_ERR_INVALID_ARGUMENT;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  int rc = set_smem((const void*)istft_frames_ragged_kernel, fft_smem(n_fft));
  if (!rc) rc = set_smem((const void*)stft_complex_synth_kernel, fft_smem(n_fft));
  if (rc) return rc;
  rc = upload(workspace, h, stream);
  if (rc) return rc;
  char* ws = static_cast<char*>(workspace);
  const int32_t* tab = reinterpret_cast<const int32_t*>(ws + l.table);
  const Cfg cfg = make_cfg(workspace, l, n_fft, hop_length);
  float* frames = reinterpret_cast<float*>(ws + l.extra);
  float2* spec[2] = {reinterpret_cast<float2*>(ws + l.extra + fb), reinterpret_cast<float2*>(ws + l.extra + fb + sb)};
  const int n_out = h.table[3 * (n_clips + 1) - 1];
  // librosa's loop: project, iSTFT, re-analyse; n_iter times, then one last projection + iSTFT
  ProjLoad load{nullptr, nullptr, nullptr, magnitude, reinterpret_cast<const float2*>(init_angles), momentum / (1.f + momentum)};
  for (int it = 0;; ++it) {
    istft_launch(load, tab, n_clips, cfg, pairs, frames, n_out, wav_out, stream);
    if (it == n_iter) break;
    float2* next = load.rebuilt == spec[0] ? spec[1] : spec[0];   // the buffer not holding the latest re-analysis
    stft_complex_synth_kernel<<<(unsigned)pairs, THREADS, fft_smem(n_fft), stream>>>(wav_out, tab, n_clips, cfg, next);
    count_launch();
    load.tprev = load.rebuilt;
    load.rebuilt = next;
    load.init = nullptr;
  }
  return check_cuda(cudaGetLastError(), "griffinlim ragged kernels launch");
}

extern "C" int ttsb_mel_to_linear_ex(const float* mel_amp, int n_frames, int n_mels, int n_bins, const float* mel_basis,
                                     const float* basis_pinv, const int32_t* band, const int32_t* bin_mels, float step, int n_iter,
                                     float* out, void* stream_v) {
  if (!mel_amp || !mel_basis || !basis_pinv || !band || !bin_mels || !out) return bad("ttsb_mel_to_linear_ex: NULL pointer");
  if (n_frames <= 0 || n_mels <= 0 || n_mels > MAX_MELS || n_bins < MIN_NFFT / 2 + 1 || n_bins > MAX_NFFT / 2 + 1 || n_iter < 0 ||
      !(step > 0.f))
    return bad("ttsb_mel_to_linear_ex: need n_frames > 0, 0 < n_mels <= 128, 129 <= n_bins <= 2049, n_iter >= 0, step > 0");
  const int smem = 2 * n_bins * (int)sizeof(float);
  mel_to_linear_ex_kernel<<<n_frames, 256, smem, static_cast<cudaStream_t>(stream_v)>>>(mel_amp, n_mels, n_bins, mel_basis, basis_pinv,
                                                                                         band, bin_mels, step, n_iter, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "mel_to_linear_ex_kernel launch");
}
