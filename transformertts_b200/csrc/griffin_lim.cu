// mel -> waveform on the GPU (SURVEY 8f row 4; reference: Audio.reconstruct_waveform, data/audio.py:94-110 =
// librosa.feature.inverse.mel_to_stft(power=1) + librosa.griffinlim(n_iter=32, momentum 0.99), librosa 0.7.1).
//
//   ttsb_mel_to_linear       : per frame, min_x>=0 ||A x - m||^2 for the (n_mels x 513) mel basis A -- started, like librosa's
//                              nnls, from the clipped least-squares solution max(pinv(A) m, 0); solved with a fixed number
//                              of FISTA projected-gradient steps (step 1/||A||_2^2) instead of scipy's L-BFGS-B: one block
//                              per frame, everything in shared memory, deterministic (oracle/audio_oracle.py restates both
//                              solvers; they agree to ~0.4 % in x on speech-like input, see tests/test_oracle.py)
//   ttsb_stft_complex        : librosa.stft (reflect padding, periodic Hann) -> complex64 (T, 513)
//   ttsb_istft               : librosa.istft (irfft, window, overlap-add, window-sum-square normalisation, centre trim)
//   ttsb_griffinlim_update   : angles = rebuilt - momentum/(1+momentum) * previous; angles /= |angles| + 1e-16; next = S * angles
//   ttsb_griffinlim_batch    : the whole Griffin-Lim loop for a packed ragged batch of clips, one launch per stage and iteration
//                              (phase update fused into the iSTFT's load -> per-clip overlap-add -> per-clip complex STFT)
//
// FFTs: one warp transforms TWO real frames at once as one 1024-point complex FFT (32 x 32 Cooley-Tukey, both 32-point
// passes in registers, one shared-memory transpose) -- forward: frame A -> real part, frame B -> imaginary part, spectra
// separated by symmetry; inverse: Z = A_full + i B_full (Hermitian extensions), ifft(Z) = conj(fft(conj Z)) / N, frame A =
// real part, frame B = imaginary part.  These kernels are latency-bound small work (a 10 s utterance is 862 frames x 33
// passes); the throughput-critical STFT is the fused log-mel kernel in stft_mel.cu.
#include <math.h>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "fft32.cuh"
#include "ttsb_host.h"

namespace ttsb {
namespace gl {

constexpr int NFFT = 1024;
constexpr int HOP = 256;
constexpr int NBINS = 513;
constexpr int WARPS = 4;

__device__ float g_tw_re[NFFT];   // cos(2 pi i / 1024)
__device__ float g_tw_im[NFFT];   // -sin(2 pi i / 1024)
__device__ float g_window[NFFT];  // periodic Hann

// Forward 1024-point complex FFT by one warp.  In: lane n2 holds z[32*n1 + n2] in (re[n1], im[n1]).  Out: Z[k] in natural
// order in bre[k], bim[k] (shared, >= 32*33 floats each, private to the warp).
__device__ __forceinline__ void warp_fft1024(float (&re)[32], float (&im)[32], float* bre, float* bim, int lane) {
  fft32(re, im);
#pragma unroll
  for (int i = 0; i < 32; ++i) {   // twiddle by W_1024^(n2*k1), k1 = bitrev5(i), and transpose through shared memory
    const int k1 = bitrev5(i);
    const int tw = (lane * k1) & (NFFT - 1);
    const float c = g_tw_re[tw], s = g_tw_im[tw];
    bre[k1 * 33 + lane] = re[i] * c - im[i] * s;
    bim[k1 * 33 + lane] = re[i] * s + im[i] * c;
  }
  __syncwarp();
#pragma unroll
  for (int n2 = 0; n2 < 32; ++n2) {
    re[n2] = bre[lane * 33 + n2];
    im[n2] = bim[lane * 33 + n2];
  }
  __syncwarp();
  fft32(re, im);
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int k = lane + 32 * bitrev5(i);
    bre[k] = re[i];
    bim[k] = im[i];
  }
  __syncwarp();
}

// x[i] of a signal of n samples with reflect padding (i in [-(n-1), 2(n-1)]).  CLAMP: the batched path reads lengths from a
// device table; for a malformed table the index is clamped into [0, n) and an empty signal reads 0, so no access leaves the clip.
template <bool CLAMP>
__device__ __forceinline__ float sample_reflect(const float* __restrict__ x, int n, int i) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  if (CLAMP) {
    if (n <= 0) return 0.f;
    i = min(max(i, 0), n - 1);
  }
  return __ldg(x + i);
}

// The per-frame-pair bodies below are shared by the single-clip kernels and the packed-batch kernels, so both compute the same
// bits for the same pair of frames.  A pair is always two frames of ONE clip: the two real frames share one complex FFT, and the
// rounding of each depends on the other, so pairing across a clip boundary would make a clip's waveform depend on its neighbour.

// ---- stft of frames lA (and lA + 1 if hasB) of a signal of L samples -> rows fA (and fA + 1) of out, 513 complex bins each
template <bool CLAMP>
__device__ __forceinline__ void stft_pair(const float* __restrict__ wav, int L, int lA, bool hasB, float2* __restrict__ out, int fA,
                                          float* bre, float* bim, int lane) {
  const int fB = fA + 1;
  float re[32], im[32];
  const int sA = lA * HOP - NFFT / 2, sB = sA + HOP;
#pragma unroll
  for (int n1 = 0; n1 < 32; ++n1) {
    const int i = 32 * n1 + lane;
    const float w = g_window[i];
    re[n1] = sample_reflect<CLAMP>(wav, L, sA + i) * w;
    im[n1] = hasB ? sample_reflect<CLAMP>(wav, L, sB + i) * w : 0.f;
  }
  warp_fft1024(re, im, bre, bim, lane);
  for (int k = lane; k < NBINS; k += 32) {
    const int k2 = (NFFT - k) & (NFFT - 1);
    const float z1r = bre[k], z1i = bim[k], z2r = bre[k2], z2i = bim[k2];
    out[(size_t)fA * NBINS + k] = make_float2(0.5f * (z1r + z2r), 0.5f * (z1i - z2i));
    if (hasB) out[(size_t)fB * NBINS + k] = make_float2(0.5f * (z1i + z2i), -0.5f * (z1r - z2r));
  }
}

// ---- irfft * window of spectra fA and fA + 1 (if hasB; as read by `load`) -> time frames fA / fA + 1 of `frames` (1024 each)
template <class Load>
__device__ __forceinline__ void istft_pair(const Load& load, int fA, bool hasB, float* __restrict__ frames, float* bre, float* bim,
                                           int lane) {
  const int fB = fA + 1;
  const size_t A = (size_t)fA * NBINS, B = (size_t)fB * NBINS;
  // conj(Z)[k], Z = A_full + i B_full, with the Hermitian extension X_full[k] = conj(X[1024 - k]) for k > 512 and the
  // imaginary parts of the DC and Nyquist bins dropped (as numpy's irfft does)
  float re[32], im[32];
#pragma unroll
  for (int n1 = 0; n1 < 32; ++n1) {
    const int k = 32 * n1 + lane;
    const int kk = k <= 512 ? k : NFFT - k;
    float2 a = load(A + kk);
    float2 b = hasB ? load(B + kk) : make_float2(0.f, 0.f);
    if (kk == 0 || kk == 512) { a.y = 0.f; b.y = 0.f; }
    if (k > 512) { a.y = -a.y; b.y = -b.y; }
    // Z = (a.x - b.y) + i (a.y + b.x);  conj(Z) = (a.x - b.y) - i (a.y + b.x)
    re[n1] = a.x - b.y;
    im[n1] = -(a.y + b.x);
  }
  warp_fft1024(re, im, bre, bim, lane);
  // z[n] = conj(FFT(conj Z))[n] / N:  frame A = Re z = bre / N,  frame B = Im z = -bim / N
  const float inv_n = 1.f / NFFT;
  for (int n = lane; n < NFFT; n += 32) {
    const float w = g_window[n] * inv_n;
    frames[(size_t)fA * NFFT + n] = bre[n] * w;
    if (hasB) frames[(size_t)fB * NFFT + n] = -bim[n] * w;
  }
}

// ---- overlap-add + window-sum-square normalisation + centre trim of T frames: output sample n, n in [0, 256 (T - 1))
__device__ __forceinline__ float overlap_add_sample(const float* __restrict__ frames, int T, int n) {
  const int s = n + NFFT / 2;                       // position in the untrimmed signal
  const int f_hi = min(s / HOP, T - 1);
  const int f_lo = max((s - (NFFT - 1) + HOP - 1) / HOP, 0);
  float acc = 0.f, wss = 0.f;
  for (int f = f_lo; f <= f_hi; ++f) {
    const int i = s - f * HOP;
    acc += __ldg(frames + (size_t)f * NFFT + i);
    const float w = g_window[i];
    wss = fmaf(w, w, wss);
  }
  return wss > 1.17549435e-38f ? acc / wss : acc;
}

// ---- phase update of "fast" Griffin-Lim for one bin: a = r - alpha t (no t on the first update); S a / (|a| + 1e-16)
__device__ __forceinline__ float2 gl_project(float2 r, const float2* __restrict__ tprev, size_t i, float s, float alpha) {
  float2 a = r;
  if (tprev != nullptr) {
    const float2 t = tprev[i];
    a.x = r.x - alpha * t.x;
    a.y = r.y - alpha * t.y;
  }
  const float mag = sqrtf(a.x * a.x + a.y * a.y) + 1e-16f;
  return make_float2(s * (a.x / mag), s * (a.y / mag));
}

// spectrum loaders of istft_pair: a stored spectrum, or the Griffin-Lim projection computed on the fly (never stored)
struct SpecLoad {
  const float2* __restrict__ spec;
  __device__ __forceinline__ float2 operator()(size_t i) const { return __ldg(spec + i); }
};
struct GlProjLoad {
  const float2* __restrict__ rebuilt;   // latest re-analysis of the waveform
  const float2* __restrict__ tprev;     // the one before (NULL on the first update)
  const float* __restrict__ S;          // target magnitudes
  const float2* __restrict__ init;      // non-NULL: first pass, S * init_angles
  float alpha;
  __device__ __forceinline__ float2 operator()(size_t i) const {
    const float s = __ldg(S + i);
    if (init != nullptr) {
      const float2 a = __ldg(init + i);
      return make_float2(s * a.x, s * a.y);
    }
    return gl_project(__ldg(rebuilt + i), tprev, i, s, alpha);
  }
};

// ---- wav (L) -> complex spectrum (T, 513), T = 1 + L / 256
__global__ void __launch_bounds__(WARPS * 32)
stft_complex_kernel(const float* __restrict__ wav, int L, int T, float2* __restrict__ out) {
  __shared__ float sre[WARPS][32 * 33], sim[WARPS][32 * 33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pair = blockIdx.x * WARPS + warp;
  const int fA = 2 * pair, fB = fA + 1;
  if (fA >= T) return;
  stft_pair<false>(wav, L, fA, fB < T, out, fA, sre[warp], sim[warp], lane);
}

// ---- complex spectrum (T, 513) -> windowed time frames (T, 1024): irfft * window
__global__ void __launch_bounds__(WARPS * 32)
istft_frames_kernel(const float2* __restrict__ spec, int T, float* __restrict__ frames) {
  __shared__ float sre[WARPS][32 * 33], sim[WARPS][32 * 33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pair = blockIdx.x * WARPS + warp;
  const int fA = 2 * pair, fB = fA + 1;
  if (fA >= T) return;
  istft_pair(SpecLoad{spec}, fA, fB < T, frames, sre[warp], sim[warp], lane);
}

// ---- overlap-add + window-sum-square normalisation + centre trim: out[n], n in [0, 256 (T - 1))
__global__ void overlap_add_kernel(const float* __restrict__ frames, int T, int n_out, float* __restrict__ out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_out) return;
  out[n] = overlap_add_sample(frames, T, n);
}

// ---- phase update of "fast" Griffin-Lim
__global__ void gl_update_kernel(const float2* __restrict__ rebuilt, const float2* __restrict__ tprev, const float* __restrict__ S,
                                 float alpha, int64_t n, float2* __restrict__ proj) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  proj[i] = gl_project(rebuilt[i], tprev, (size_t)i, S[i], alpha);
}

// ---- packed ragged batch (ttsb_griffinlim_batch).  The clip table in the workspace holds three (n_clips + 1) prefix arrays,
// derived once per call from the caller's frame offsets and clamped so that every index formed from them stays inside the buffers
// total_frames / n_clips size:
//   fo[c]: first frame of clip c      (monotone, fo[0] = 0, fo[n] = F)
//   po[c]: first frame PAIR of clip c (a clip of T frames has (T + 1) / 2 pairs; sum <= (F + n) / 2)
//   wo[c]: first output sample        (clip c has 256 (T_c - 1) samples, clamped to the 256 (F - n) of wav_out)
__global__ void gl_batch_table_kernel(const int32_t* __restrict__ off, int n_clips, int F, int32_t* __restrict__ tab) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int32_t* fo = tab;
  int32_t* po = tab + (n_clips + 1);
  int32_t* wo = tab + 2 * (n_clips + 1);
  const int n_wav = HOP * (F - n_clips);
  int f = 0, p = 0, w = 0;
  fo[0] = po[0] = wo[0] = 0;
  for (int c = 0; c < n_clips; ++c) {
    const int e = c + 1 == n_clips ? F : min(max(off[c + 1], f), F);
    const int T = e - f;
    p += (T + 1) / 2;
    w = min(w + HOP * max(T - 1, 0), n_wav);
    f = e;
    fo[c + 1] = f;
    po[c + 1] = p;
    wo[c + 1] = w;
  }
}

__global__ void __launch_bounds__(WARPS * 32)
istft_frames_batch_kernel(GlProjLoad load, const int32_t* __restrict__ tab, int n_clips, float* __restrict__ frames) {
  __shared__ float sre[WARPS][32 * 33], sim[WARPS][32 * 33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pair = blockIdx.x * WARPS + warp;
  const int32_t* fo = tab;
  const int32_t* po = tab + (n_clips + 1);
  if (pair >= __ldg(po + n_clips)) return;
  const int c = find_clip(po, n_clips, pair);
  const int fA = __ldg(fo + c) + 2 * (pair - __ldg(po + c)), end = __ldg(fo + c + 1);
  if (fA >= end) return;
  istft_pair(load, fA, fA + 1 < end, frames, sre[warp], sim[warp], lane);
}

__global__ void overlap_add_batch_kernel(const float* __restrict__ frames, const int32_t* __restrict__ tab, int n_clips, int n_out,
                                         float* __restrict__ out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_out) return;
  const int32_t* fo = tab;
  const int32_t* wo = tab + 2 * (n_clips + 1);
  if (n >= __ldg(wo + n_clips)) {   // only reached with a malformed offset table
    out[n] = 0.f;
    return;
  }
  const int c = find_clip(wo, n_clips, n);
  const int f0 = __ldg(fo + c);
  out[n] = overlap_add_sample(frames + (size_t)f0 * NFFT, __ldg(fo + c + 1) - f0, n - __ldg(wo + c));
}

__global__ void __launch_bounds__(WARPS * 32)
stft_complex_batch_kernel(const float* __restrict__ wav, const int32_t* __restrict__ tab, int n_clips, float2* __restrict__ out) {
  __shared__ float sre[WARPS][32 * 33], sim[WARPS][32 * 33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pair = blockIdx.x * WARPS + warp;
  const int32_t* fo = tab;
  const int32_t* po = tab + (n_clips + 1);
  const int32_t* wo = tab + 2 * (n_clips + 1);
  if (pair >= __ldg(po + n_clips)) return;
  const int c = find_clip(po, n_clips, pair);
  const int f0 = __ldg(fo + c), T = __ldg(fo + c + 1) - f0;
  const int lA = 2 * (pair - __ldg(po + c));
  if (lA >= T) return;
  const int w0 = __ldg(wo + c);
  stft_pair<true>(wav + w0, __ldg(wo + c + 1) - w0, lA, lA + 1 < T, out, f0 + lA, sre[warp], sim[warp], lane);
}

// ---- mel amplitudes (T, n_mels) -> linear magnitudes (T, 513): non-negative least squares per frame
constexpr int NNLS_MAX_MELS = 128;
__global__ void __launch_bounds__(256)
mel_to_linear_kernel(const float* __restrict__ mel, int n_mels, const float* __restrict__ basis, const float* __restrict__ pinv,
                     const int* __restrict__ band, const int* __restrict__ bin_mels, float step, int n_iter, float* __restrict__ out) {
  __shared__ float x[NBINS], y[NBINS], r[NNLS_MAX_MELS], m[NNLS_MAX_MELS];
  const int t = blockIdx.x;
  for (int i = threadIdx.x; i < n_mels; i += blockDim.x) m[i] = mel[(size_t)t * n_mels + i];
  __syncthreads();
  for (int k = threadIdx.x; k < NBINS; k += blockDim.x) {   // clipped least-squares start: max(pinv(A) m, 0)
    float acc = 0.f;
    for (int j = 0; j < n_mels; ++j) acc = fmaf(__ldg(pinv + (size_t)k * n_mels + j), m[j], acc);
    x[k] = y[k] = fmaxf(acc, 0.f);
  }
  __syncthreads();
  float tk = 1.f;
  for (int it = 0; it < n_iter; ++it) {
    for (int j = threadIdx.x; j < n_mels; j += blockDim.x) {       // r = A y - m  (row j of A is non-zero on [band lo, hi))
      float acc = 0.f;
      for (int k = band[2 * j]; k < band[2 * j + 1]; ++k) acc = fmaf(__ldg(basis + (size_t)j * NBINS + k), y[k], acc);
      r[j] = acc - m[j];
    }
    __syncthreads();
    const float tn = 0.5f * (1.f + sqrtf(1.f + 4.f * tk * tk));
    const float beta = (tk - 1.f) / tn;
    for (int k = threadIdx.x; k < NBINS; k += blockDim.x) {        // x+ = max(y - step A^T r, 0); FISTA extrapolation
      float g = 0.f;
      for (int j = bin_mels[2 * k]; j < bin_mels[2 * k + 1]; ++j) g = fmaf(__ldg(basis + (size_t)j * NBINS + k), r[j], g);
      const float xn = fmaxf(y[k] - step * g, 0.f);
      y[k] = xn + beta * (xn - x[k]);
      x[k] = xn;
    }
    tk = tn;
    __syncthreads();
  }
  for (int k = threadIdx.x; k < NBINS; k += blockDim.x) out[(size_t)t * NBINS + k] = x[k];
}

static int init_tables() {
  static PerDevice<bool> done_pd;
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
  done = true;
  return 0;
}

}  // namespace gl
}  // namespace ttsb

using namespace ttsb;

static int gl_bad(const char* msg) {
  set_last_error("%s", msg);
  return TTSB_ERR_INVALID_ARGUMENT;
}

extern "C" int ttsb_stft_complex(const float* wav, int n_samples, float* spec_out, void* stream_v) {
  if (!wav || !spec_out || n_samples <= gl::NFFT / 2) return gl_bad("ttsb_stft_complex: need n_samples > 512");
  int rc = gl::init_tables();
  if (rc) return rc;
  const int T = 1 + n_samples / gl::HOP, pairs = (T + 1) / 2;
  gl::stft_complex_kernel<<<(pairs + gl::WARPS - 1) / gl::WARPS, gl::WARPS * 32, 0, static_cast<cudaStream_t>(stream_v)>>>(
      wav, n_samples, T, reinterpret_cast<float2*>(spec_out));
  count_launch();
  return check_cuda(cudaGetLastError(), "stft_complex_kernel launch");
}

extern "C" int64_t ttsb_istft_workspace_bytes(int n_frames) { return (int64_t)n_frames * gl::NFFT * (int64_t)sizeof(float); }

extern "C" int ttsb_istft(const float* spec, int n_frames, void* workspace, int64_t workspace_bytes, float* wav_out, void* stream_v) {
  if (!spec || !workspace || !wav_out || n_frames < 2) return gl_bad("ttsb_istft: NULL tensor or fewer than 2 frames");
  if (workspace_bytes < ttsb_istft_workspace_bytes(n_frames)) return gl_bad("ttsb_istft: workspace too small (ttsb_istft_workspace_bytes)");
  int rc = gl::init_tables();
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int pairs = (n_frames + 1) / 2;
  float* frames = static_cast<float*>(workspace);
  gl::istft_frames_kernel<<<(pairs + gl::WARPS - 1) / gl::WARPS, gl::WARPS * 32, 0, stream>>>(reinterpret_cast<const float2*>(spec), n_frames, frames);
  count_launch();
  const int n_out = gl::HOP * (n_frames - 1);
  gl::overlap_add_kernel<<<(n_out + 255) / 256, 256, 0, stream>>>(frames, n_frames, n_out, wav_out);
  count_launch();
  return check_cuda(cudaGetLastError(), "istft kernels launch");
}

extern "C" int ttsb_griffinlim_update(const float* rebuilt, const float* previous, const float* magnitude, float momentum, int64_t n,
                                      float* projected_out, void* stream_v) {
  if (!rebuilt || !magnitude || !projected_out || n <= 0) return gl_bad("ttsb_griffinlim_update: bad arguments");
  const float alpha = momentum / (1.f + momentum);
  gl::gl_update_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_v)>>>(
      reinterpret_cast<const float2*>(rebuilt), reinterpret_cast<const float2*>(previous), magnitude, alpha, n,
      reinterpret_cast<float2*>(projected_out));
  count_launch();
  return check_cuda(cudaGetLastError(), "gl_update_kernel launch");
}

// ---- Griffin-Lim over a packed ragged batch.  Workspace: the time frames (F, 1024) fp32, two complex spectra (F, 513) that
// rotate as rebuilt / previous, and the clip table; each region starts on a 256-byte boundary.
namespace {
constexpr int GL_BATCH_MAX_FRAMES = INT32_MAX / gl::NFFT;   // keeps every sample index of the packed buffers in int
int64_t align256(int64_t b) { return (b + 255) & ~int64_t(255); }
struct GlBatchLayout {
  int64_t frames, spec, table, total;
};
GlBatchLayout gl_batch_layout(int F, int n_clips) {
  GlBatchLayout l;
  l.frames = 0;
  l.spec = align256((int64_t)F * gl::NFFT * (int64_t)sizeof(float));
  const int64_t spec_bytes = align256((int64_t)F * gl::NBINS * (int64_t)sizeof(float2));
  l.table = l.spec + 2 * spec_bytes;
  l.total = l.table + align256(3 * (int64_t)(n_clips + 1) * (int64_t)sizeof(int32_t));
  return l;
}
bool gl_batch_shape_ok(int F, int n_clips) { return n_clips >= 1 && F >= 4 * (int64_t)n_clips && F <= GL_BATCH_MAX_FRAMES; }
}  // namespace

extern "C" int64_t ttsb_griffinlim_batch_workspace_bytes(int total_frames, int n_clips) {
  if (!gl_batch_shape_ok(total_frames, n_clips)) {
    set_last_error("ttsb_griffinlim_batch_workspace_bytes: need n_clips >= 1 and 4 * n_clips <= total_frames <= %d", GL_BATCH_MAX_FRAMES);
    return -1;
  }
  return gl_batch_layout(total_frames, n_clips).total;
}

extern "C" int ttsb_griffinlim_batch(const float* magnitude, const float* init_angles, const int32_t* frame_offsets, int n_clips,
                                     int total_frames, int n_iter, float momentum, void* workspace, int64_t workspace_bytes,
                                     float* wav_out, void* stream_v) {
  if (!magnitude || !init_angles || !frame_offsets || !workspace || !wav_out)
    return gl_bad("ttsb_griffinlim_batch: NULL tensor");
  if (!gl_batch_shape_ok(total_frames, n_clips)) {
    set_last_error("ttsb_griffinlim_batch: need n_clips >= 1 and 4 * n_clips <= total_frames <= %d (got n_clips %d, total_frames %d)",
                   GL_BATCH_MAX_FRAMES, n_clips, total_frames);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (n_iter < 0) return gl_bad("ttsb_griffinlim_batch: n_iter < 0");
  if (!(momentum >= 0.f) || isinf(momentum)) return gl_bad("ttsb_griffinlim_batch: momentum must be finite and >= 0");
  const GlBatchLayout lay = gl_batch_layout(total_frames, n_clips);
  if (workspace_bytes < lay.total) return gl_bad("ttsb_griffinlim_batch: workspace too small (ttsb_griffinlim_batch_workspace_bytes)");
  if (reinterpret_cast<uintptr_t>(workspace) % 16 != 0) return gl_bad("ttsb_griffinlim_batch: workspace must be 16-byte aligned");
  int rc = gl::init_tables();
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  char* ws = static_cast<char*>(workspace);
  float* frames = reinterpret_cast<float*>(ws + lay.frames);
  float2* spec[2] = {reinterpret_cast<float2*>(ws + lay.spec), reinterpret_cast<float2*>(ws + lay.spec + (lay.table - lay.spec) / 2)};
  int32_t* tab = reinterpret_cast<int32_t*>(ws + lay.table);
  const int F = total_frames, n_out = gl::HOP * (F - n_clips);
  const int max_pairs = (F + n_clips) / 2;
  const unsigned pair_blocks = (unsigned)((max_pairs + gl::WARPS - 1) / gl::WARPS);
  const unsigned ola_blocks = (unsigned)((n_out + 255) / 256);

  gl::gl_batch_table_kernel<<<1, 1, 0, stream>>>(frame_offsets, n_clips, F, tab);
  count_launch();
  // librosa's loop (and Audio.griffinlim_device's): project, iSTFT, re-analyse; n_iter times, then one last projection + iSTFT
  gl::GlProjLoad load{nullptr, nullptr, magnitude, reinterpret_cast<const float2*>(init_angles), momentum / (1.f + momentum)};
  for (int it = 0;; ++it) {
    gl::istft_frames_batch_kernel<<<pair_blocks, gl::WARPS * 32, 0, stream>>>(load, tab, n_clips, frames);
    count_launch();
    gl::overlap_add_batch_kernel<<<ola_blocks, 256, 0, stream>>>(frames, tab, n_clips, n_out, wav_out);
    count_launch();
    if (it == n_iter) break;
    float2* next = load.rebuilt == spec[0] ? spec[1] : spec[0];   // the buffer not holding the latest re-analysis
    gl::stft_complex_batch_kernel<<<pair_blocks, gl::WARPS * 32, 0, stream>>>(wav_out, tab, n_clips, next);
    count_launch();
    load.tprev = load.rebuilt;
    load.rebuilt = next;
    load.init = nullptr;
  }
  return check_cuda(cudaGetLastError(), "griffinlim batch kernels launch");
}

extern "C" int ttsb_mel_to_linear(const float* mel_amp, int n_frames, int n_mels, const float* mel_basis, const float* basis_pinv,
                                  const int32_t* band, const int32_t* bin_mels, float step, int n_iter, float* out, void* stream_v) {
  if (!mel_amp || !mel_basis || !basis_pinv || !band || !bin_mels || !out || n_frames <= 0 || n_mels <= 0 || n_mels > gl::NNLS_MAX_MELS ||
      n_iter < 0 || !(step > 0.f))
    return gl_bad("ttsb_mel_to_linear: bad arguments (n_mels <= 128, step > 0)");
  gl::mel_to_linear_kernel<<<n_frames, 256, 0, static_cast<cudaStream_t>(stream_v)>>>(mel_amp, n_mels, mel_basis, basis_pinv, band, bin_mels,
                                                                                      step, n_iter, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "mel_to_linear_kernel launch");
}
