// WORLD's spectral envelope (CheapTrick) of a packed ragged batch of clips at the DIO / StoneMask frames of
// ttsb_pitch_dio_stonemask, and SPTK's mel-cepstrum of it (pysptk's sp2mc as a matrix W from the host): what pyworld.cheaptrick
// and pysptk.sp2mc compute for the WORLD mel-cepstral distortion of evaluate_tts.py --mcep.  tests/world_mcep_oracle.py
// restates both in numpy; DESIGN.md section 15 lists the readings of WORLD's C++ below.
//
// CheapTrick, one CTA per frame (clip-local frame i at t = i frame_period / 1000), float64, every transform in shared memory:
//   f0 <= 3 fs / (n - 3) (unvoiced included) -> 500 Hz;  half = round(1.5 fs / f0), origin = round(t fs + 0.001);
//   w_k = 0.5 cos(pi (k / 1.5 / fs) f0) + 0.5 for k = -half .. half, divided by sqrt(sum w^2);
//   v_k = x[clamp(origin + k, 0, L - 1)] w_k + 1e-12 randn(frame, k + half, 0);  v -= w sum(v) / sum(w);  zero-padded to n;
//   P = |FFT(v)|^2 on bins 0 .. n/2; DC correction: bins below f0 get the spectrum mirrored about f0 added (interp1Q);
//   linear smoothing over width 2 f0 / 3: cumulative sum (sequential, as WORLD's) of the spectrum mirrored by `boundary` bins
//   at each end, read at f -+ width / 2 by interp1Q, difference / width;  + |randn(frame, bin, 1)| eps;
//   cepstrum of log P (mirrored to n, forward FFT, real part) times the smoothing lifter sin(pi f0 q) / (pi f0 q) and the
//   compensation lifter (1 - 2 q1) + 2 q1 cos(2 pi q f0), q = i / fs, divided by n; inverse FFT; exp.
// WORLD draws its safeguard noise from one generator that runs through the whole call; here every draw is WORLD's randn (the sum
// of 12 uniforms of 28 bits, minus 6) of uniforms hashed by splitmix64 from (clip-local frame, index, site), integer arithmetic
// the restatement repeats bit for bit, so a frame's envelope depends on neither the earlier frames nor the batch.
// Sums are reduced in a fixed order (per-thread strided partials, a butterfly in each warp, the warps in order), so the result
// does not depend on the batch either.
//
// The file builds with -fmad=false, as the other WORLD restatement (pitch.cu): every product and sum is rounded on its own.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace ttsb {
namespace {

constexpr int CT_THREADS = 256;
constexpr int MC_THREADS = 128;
constexpr double CT_SAFE_GUARD = 1e-12;             // world::kMySafeGuardMinimum
constexpr double CT_EPS = 2.220446049250313e-16;    // world::kEps
constexpr double CT_DEFAULT_F0 = 500.0;             // world::kDefaultF0
constexpr int CT_MIN_FFT = 256, CT_MAX_FFT = 4096;

struct CtParams {
  int fs, n, log2n, n_clips;
  double frame_period, q1;
  double f0_floor;    // 3 fs / (n - 3): at or below it a frame takes 500 Hz
  double f0_max;      // fs / 4: above it (and for NaN) a frame's envelope is NaN
};

__device__ __forceinline__ int ct_round(double x) { return x > 0 ? (int)(x + 0.5) : (int)(x - 0.5); }

__device__ __forceinline__ uint64_t ct_mix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// WORLD's randn: 12 uniforms of 28 bits summed, / 2^28, - 6 (exact).  Key z = mix(frame << 32 | site << 16 | index); hash r of
// z ^ r (r = 0 .. 5) gives two uniforms, its bits 36..63 and 4..31.
__device__ __forceinline__ double ct_randn(uint32_t frame, uint32_t index, uint32_t site) {
  const uint64_t z = ct_mix(((uint64_t)frame << 32) | ((uint64_t)site << 16) | index);
  uint64_t s = 0;
#pragma unroll
  for (uint64_t r = 0; r < 6; ++r) {
    const uint64_t h = ct_mix(z ^ r);
    s += (h >> 36) + ((h >> 4) & 0xFFFFFFFull);
  }
  return (double)s / 268435456.0 - 6.0;
}

// The sum of every thread's v: a butterfly within each warp (every lane gets the same bits), then the warps in order.
__device__ double ct_block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < CT_THREADS / 32; ++w) s += red[w];
  return s;
}

// In-place inclusive cumulative sum of a[0 .. m) in WORLD's order, one addition after the other, by thread 0 (the loads of 8
// values go ahead of their additions).  The smoothing takes the difference of two partial sums that can be ~1e10 times larger
// than it, so any other order moves the envelope by far more than its other roundings do.
__device__ void ct_cumsum(double* a, int m) {
  if (threadIdx.x == 0) {
    double s = 0.0;
    int i = 0;
    for (; i + 8 <= m; i += 8) {
      double v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = a[i + j];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s += v[j];
        a[i + j] = s;
      }
    }
    for (; i < m; ++i) {
      s += a[i];
      a[i] = s;
    }
  }
  __syncthreads();
}

// In-place radix-2 FFT of n = 2^log2n points: bit reversal, then log2n stages of butterflies.  tw[m] = exp(-2 pi i m / n) for
// m < n / 2; the inverse transform conjugates the twiddles and does not scale.
__device__ void ct_fft(double2* a, int n, int log2n, const double2* __restrict__ tw, bool inverse) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int j = (int)(__brev((unsigned)i) >> (32 - log2n));
    if (i < j) {
      const double2 t = a[i];
      a[i] = a[j];
      a[j] = t;
    }
  }
  __syncthreads();
  for (int half = 1, stride = n >> 1; half < n; half <<= 1, stride >>= 1) {
    for (int t = threadIdx.x; t < n / 2; t += blockDim.x) {
      const int j = t & (half - 1);
      const int i0 = ((t - j) << 1) + j, i1 = i0 + half;
      double2 w = __ldg(tw + j * stride);
      if (inverse) w.y = -w.y;
      const double2 u = a[i0], v = a[i1];
      const double vr = v.x * w.x - v.y * w.y, vi = v.x * w.y + v.y * w.x;
      a[i0] = make_double2(u.x + vr, u.y + vi);
      a[i1] = make_double2(u.x - vr, u.y - vi);
    }
    __syncthreads();
  }
}

// WORLD's interp1Q on a uniform axis x0 + k dx: y[b] + (y[b + 1] - y[b]) frac, b = int((xi - x0) / dx), the step past the
// last point taken as 0
__device__ __forceinline__ double ct_interp1q(const double* y, int m, double x0, double dx, double xi) {
  const int b = (int)((xi - x0) / dx);
  const double fr = (xi - x0) / dx - b;
  const double dy = b < m - 1 ? y[b + 1] - y[b] : 0.0;
  return y[b] + dy * fr;
}

// Shared memory: n complex doubles (the transforms), the power spectrum (n/2 + 1) and the mirrored spectrum's cumulative sum.
__host__ __device__ __forceinline__ int ct_seg_len(int n) { return n / 2 + 2 * (n / 6 + 2) + 1; }
__host__ __device__ __forceinline__ size_t ct_smem_bytes(int n) {
  return (size_t)n * sizeof(double2) + (size_t)(n / 2 + 1 + ct_seg_len(n)) * sizeof(double);
}

__global__ void __launch_bounds__(CT_THREADS)
cheaptrick_kernel(const float* __restrict__ wav, const int32_t* __restrict__ so, const int32_t* __restrict__ fo,
                  const double* __restrict__ f0_in, const double2* __restrict__ tw, CtParams p, double* __restrict__ out) {
  extern __shared__ double2 ct_sm[];
  __shared__ double red[CT_THREADS / 32];
  double2* buf = ct_sm;
  double* spec = reinterpret_cast<double*>(buf + p.n);
  double* seg = spec + p.n / 2 + 1;
  const int n = p.n, nh = n / 2;
  const int g = blockIdx.x;
  const int c = find_clip(fo, p.n_clips, g);
  const int frame = g - __ldg(fo + c);
  const int s0 = __ldg(so + c), L = __ldg(so + c + 1) - s0;
  double* env = out + (size_t)g * (nh + 1);
  double f0 = __ldg(f0_in + g);
  if (f0 <= p.f0_floor) f0 = CT_DEFAULT_F0;
  if (!(f0 <= p.f0_max)) {   // NaN, or so high that the smoothing would read past the spectrum
    for (int i = threadIdx.x; i <= nh; i += blockDim.x) env[i] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  const double fs = (double)p.fs;

  // ---- the F0-adaptive window (imaginary parts) and its norm
  const int half = ct_round(1.5 * fs / f0);
  const int nw = 2 * half + 1;
  double acc = 0.0;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    double w = 0.0;
    if (k < nw) {
      const double pos = (double)(k - half) / 1.5 / fs;
      w = 0.5 * cos(M_PI * pos * f0) + 0.5;
    }
    buf[k] = make_double2(0.0, w);
    acc += w * w;
  }
  const double norm = sqrt(ct_block_sum(acc, red));
  // ---- windowed waveform with the safeguard noise, then the DC removal
  const double t = (double)frame * p.frame_period / 1000.0;
  const int origin = ct_round(t * fs + 0.001);
  double sv = 0.0, sw = 0.0;
  for (int k = threadIdx.x; k < nw; k += blockDim.x) {
    const double w = buf[k].y / norm;
    const int idx = min(L - 1, max(0, origin + k - half));
    const double v = (double)__ldg(wav + s0 + idx) * w + ct_randn((uint32_t)frame, (uint32_t)k, 0) * CT_SAFE_GUARD;
    buf[k] = make_double2(v, w);
    sv += v;
    sw += w;
  }
  const double tot_v = ct_block_sum(sv, red);
  const double coef = tot_v / ct_block_sum(sw, red);
  for (int k = threadIdx.x; k < nw; k += blockDim.x) {
    const double2 b = buf[k];
    buf[k] = make_double2(b.x - b.y * coef, 0.0);
  }
  __syncthreads();

  // ---- power spectrum
  ct_fft(buf, n, p.log2n, tw, false);
  for (int i = threadIdx.x; i <= nh; i += blockDim.x) spec[i] = buf[i].x * buf[i].x + buf[i].y * buf[i].y;
  __syncthreads();

  // ---- DC correction: interp1Q(f0, -fs / n, spec, ul + 1, i fs / n) added to bins i < ul - 1
  const int ul = 2 + (int)(f0 * n / fs);
  {
    const double dx = -fs / n;
    for (int i = threadIdx.x; i < ul - 1; i += blockDim.x) seg[i] = ct_interp1q(spec, ul + 1, f0, dx, (double)i * fs / n);
    __syncthreads();
    for (int i = threadIdx.x; i < ul - 1; i += blockDim.x) spec[i] = spec[i] + seg[i];
    __syncthreads();
  }

  // ---- linear smoothing over width 2 f0 / 3: the cumulative sum of the mirrored spectrum times fs / n
  const double width = f0 * 2.0 / 3.0;
  const int bd = (int)(width * n / fs) + 1;
  const int m = nh + 2 * bd + 1;
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const double v = i < bd ? spec[bd - i] : (i < nh + bd ? spec[i - bd] : spec[nh - (i - (nh + bd))]);
    seg[i] = v * fs / n;
  }
  __syncthreads();
  ct_cumsum(seg, m);
  // ---- interpolated at f -+ width / 2, plus the infinitesimal noise; the log, mirrored to n points
  {
    const double x0 = -(bd - 0.5) * fs / n, dx = fs / n;
    for (int i = threadIdx.x; i <= nh; i += blockDim.x) {
      const double f_lo = (double)i / n * fs - width / 2.0;
      const double f_hi = f_lo + width;
      const double lo = ct_interp1q(seg, m, x0, dx, f_lo), hi = ct_interp1q(seg, m, x0, dx, f_hi);
      const double v = (hi - lo) / width + fabs(ct_randn((uint32_t)frame, (uint32_t)i, 1)) * CT_EPS;
      const double lv = log(v);
      buf[i] = make_double2(lv, 0.0);
      if (i > 0 && i < nh) buf[n - i] = make_double2(lv, 0.0);
    }
  }
  __syncthreads();

  // ---- smoothing with recovery: the cepstrum, both lifters, back to the log spectrum
  ct_fft(buf, n, p.log2n, tw, false);
  for (int i = threadIdx.x; i <= nh; i += blockDim.x) {
    double sl = 1.0, cl = (1.0 - 2.0 * p.q1) + 2.0 * p.q1;
    if (i > 0) {
      const double q = (double)i / fs;
      sl = sin(M_PI * f0 * q) / (M_PI * f0 * q);
      cl = (1.0 - 2.0 * p.q1) + 2.0 * p.q1 * cos(2.0 * M_PI * q * f0);
    }
    const double v = buf[i].x * sl * cl / n;
    buf[i] = make_double2(v, 0.0);
    if (i > 0 && i < nh) buf[n - i] = make_double2(v, 0.0);
  }
  __syncthreads();
  ct_fft(buf, n, p.log2n, tw, true);
  for (int i = threadIdx.x; i <= nh; i += blockDim.x) env[i] = exp(buf[i].x);
}

// mc[f][k] = sum_j W[k][j] log(sp[f][j]), one CTA per frame: warp w takes k = w, w + 4, ...; lane l sums j = l, l + 32, ... in
// order, then a butterfly over the lanes
__global__ void __launch_bounds__(MC_THREADS)
sp2mc_kernel(const double* __restrict__ sp, int nb, const double* __restrict__ W, int n_coef, double* __restrict__ mc) {
  extern __shared__ double mc_sm[];
  const size_t f = blockIdx.x;
  for (int j = threadIdx.x; j < nb; j += blockDim.x) mc_sm[j] = log(__ldg(sp + f * nb + j));
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x >> 5; k < n_coef; k += MC_THREADS / 32) {
    const double* w = W + (size_t)k * nb;
    double s = 0.0;
    for (int j = lane; j < nb; j += 32) s += __ldg(w + j) * mc_sm[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) mc[f * n_coef + k] = s;
  }
}

int ws_bad(const char* fmt, long long a = 0, long long b = 0) {
  set_last_error(fmt, a, b);
  return TTSB_ERR_INVALID_ARGUMENT;
}

int ct_log2(int n) {
  int l = 0;
  while ((1 << l) < n) ++l;
  return l;
}

bool ct_fft_size_ok(int n) { return n >= CT_MIN_FFT && n <= CT_MAX_FFT && (n & (n - 1)) == 0; }

size_t ct_align16(size_t x) { return (x + 15) & ~(size_t)15; }

struct CtPlan {
  CtParams p;
  int64_t frames = 0;
  size_t off_fo = 0, off_tw = 0;
  int64_t bytes = 0;
};

// Checks the scalars and the host offset tables and lays out the workspace: sample offsets, frame offsets, twiddles.
int ct_plan(const int32_t* so, const int32_t* fo, int n_clips, int fs, double frame_period, double q1, int fft_size, CtPlan& pl) {
  if (!so || !fo) return ws_bad("ttsb_cheaptrick: NULL offset table");
  if (n_clips < 1) return ws_bad("ttsb_cheaptrick: n_clips %lld < 1", n_clips);
  if (fs < 8000 || fs > 192000) return ws_bad("ttsb_cheaptrick: fs %lld outside [8000, 192000]", fs);
  if (!(frame_period > 0) || !isfinite(frame_period)) return ws_bad("ttsb_cheaptrick: frame_period must be finite and > 0");
  if (!isfinite(q1)) return ws_bad("ttsb_cheaptrick: q1 must be finite");
  if (!ct_fft_size_ok(fft_size))
    return ws_bad("ttsb_cheaptrick: fft_size %lld is not a power of two in [256, 4096]", fft_size);
  // the default F0's window (2 round(1.5 fs / 500) + 1 samples) must fit the transform, i.e. 3 fs / (n - 3) < 500 Hz
  if (2 * (int)(1.5 * fs / CT_DEFAULT_F0 + 0.5) + 1 > fft_size - 2)
    return ws_bad("ttsb_cheaptrick: fft_size %lld is too short at fs %lld (its F0 floor 3 fs / (fft_size - 3) must be below "
                  "500 Hz)", fft_size, fs);
  if (so[0] != 0 || fo[0] != 0) return ws_bad("ttsb_cheaptrick: offset tables must start at 0");
  for (int c = 0; c < n_clips; ++c) {
    const long long L = (long long)so[c + 1] - so[c];
    if (L < 1) return ws_bad("ttsb_cheaptrick: clip %lld has %lld samples", c, L);
    const long long nf = (long long)(int)(1000.0 * (double)L / fs / frame_period) + 1;
    if ((long long)fo[c + 1] - fo[c] != nf)
      return ws_bad("ttsb_cheaptrick: f0_offsets give clip %lld %lld frames; WORLD's frame count differs", c,
                    (long long)fo[c + 1] - fo[c]);
  }
  pl.frames = fo[n_clips];
  CtParams& p = pl.p;
  p.fs = fs;
  p.n = fft_size;
  p.log2n = ct_log2(fft_size);
  p.n_clips = n_clips;
  p.frame_period = frame_period;
  p.q1 = q1;
  p.f0_floor = 3.0 * fs / (fft_size - 3.0);
  p.f0_max = fs / 4.0;
  pl.off_fo = ct_align16((size_t)(n_clips + 1) * sizeof(int32_t));
  pl.off_tw = ct_align16(pl.off_fo + (size_t)(n_clips + 1) * sizeof(int32_t));
  pl.bytes = (int64_t)(pl.off_tw + (size_t)(fft_size / 2) * sizeof(double2));
  return 0;
}

}  // namespace
}  // namespace ttsb

using namespace ttsb;

extern "C" int64_t ttsb_cheaptrick_workspace_bytes(const int32_t* sample_offsets, const int32_t* f0_offsets, int n_clips, int fs,
                                                   double frame_period_ms, int fft_size) {
  CtPlan pl;
  if (ct_plan(sample_offsets, f0_offsets, n_clips, fs, frame_period_ms, 0.0, fft_size, pl)) return -1;
  return pl.bytes;
}

extern "C" int ttsb_cheaptrick(const float* wav, const int32_t* sample_offsets, int n_clips, int fs, double frame_period_ms,
                               const double* f0, const int32_t* f0_offsets, double q1, int fft_size, void* workspace,
                               int64_t workspace_bytes, double* envelope_out, void* stream_v) {
  if (!wav || !f0 || !workspace || !envelope_out) return ws_bad("ttsb_cheaptrick: NULL pointer");
  CtPlan pl;
  if (int rc = ct_plan(sample_offsets, f0_offsets, n_clips, fs, frame_period_ms, q1, fft_size, pl)) return rc;
  if (workspace_bytes < pl.bytes)
    return ws_bad("ttsb_cheaptrick: workspace holds %lld bytes, needs %lld (ttsb_cheaptrick_workspace_bytes)", workspace_bytes, pl.bytes);
  if (reinterpret_cast<uintptr_t>(workspace) % 16 != 0) return ws_bad("ttsb_cheaptrick: workspace must be 16-byte aligned");
  // host image of the workspace: both offset tables and the twiddles exp(-2 pi i m / n), one copy
  std::vector<uint8_t> host((size_t)pl.bytes, 0);
  memcpy(host.data(), sample_offsets, (size_t)(n_clips + 1) * sizeof(int32_t));
  memcpy(host.data() + pl.off_fo, f0_offsets, (size_t)(n_clips + 1) * sizeof(int32_t));
  double2* tw = reinterpret_cast<double2*>(host.data() + pl.off_tw);
  for (int m = 0; m < fft_size / 2; ++m) {
    const double a = 2.0 * M_PI * m / fft_size;
    tw[m] = make_double2(cos(a), -sin(a));
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  TTSB_CUDA_OK(cudaMemcpyAsync(ws, host.data(), host.size(), cudaMemcpyHostToDevice, stream));
  const size_t sm = ct_smem_bytes(fft_size);
  if (sm > 48 * 1024) {
    static PerDevice<size_t> attr_pd;
    size_t& attr = attr_pd.get();
    if (sm > attr) {
      TTSB_CUDA_OK(cudaFuncSetAttribute(cheaptrick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
      attr = sm;
    }
  }
  cheaptrick_kernel<<<(unsigned)pl.frames, CT_THREADS, sm, stream>>>(
      wav, reinterpret_cast<const int32_t*>(ws), reinterpret_cast<const int32_t*>(ws + pl.off_fo), f0,
      reinterpret_cast<const double2*>(ws + pl.off_tw), pl.p, envelope_out);
  count_launch();
  return check_cuda(cudaGetLastError(), "cheaptrick_kernel launch");
}

extern "C" int ttsb_sp2mc(const double* envelope, int n_frames, int fft_size, const double* matrix, int order, double* mc_out,
                          void* stream_v) {
  if (!envelope || !matrix || !mc_out) return ws_bad("ttsb_sp2mc: NULL pointer");
  if (n_frames < 1) return ws_bad("ttsb_sp2mc: n_frames %lld < 1", n_frames);
  if (!ct_fft_size_ok(fft_size)) return ws_bad("ttsb_sp2mc: fft_size %lld is not a power of two in [256, 4096]", fft_size);
  if (order < 1 || order >= fft_size / 2) return ws_bad("ttsb_sp2mc: need 1 <= order < fft_size / 2, got order %lld", order);
  const int nb = fft_size / 2 + 1;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  sp2mc_kernel<<<(unsigned)n_frames, MC_THREADS, (size_t)nb * sizeof(double), stream>>>(envelope, nb, matrix, order + 1, mc_out);
  count_launch();
  return check_cuda(cudaGetLastError(), "sp2mc_kernel launch");
}
