// Leading and trailing silence of a packed ragged batch of clips (ttsb_trim_silence_bounds): librosa.effects.trim(y, top_db,
// frame_length=256, hop_length=64) as the reference's Audio.trim_audio_silence calls it (reference: data/audio.py:164-169).
//
// Per clip of L samples (librosa 0.7.1's trim -> feature.rms(center=True) ** 2 -> power_to_db(ref=np.max, amin=1e-10)):
//   x: the clip reflect-padded by 128 samples on each side (np.pad 'reflect', repeated for clips shorter than 129 samples);
//   frame t = 0 .. L / 64 covers x[64 t .. 64 t + 255];  p_t = (((x0^2 + x1^2) + x2^2) + ... + x255^2) / 256 in float64;
//   db_t = 10 log10(max(1e-10, p_t)) - 10 log10(max(1e-10, max_t p_t));  frame t is non-silent iff db_t > -top_db;
//   [start, end) = [64 f, min(L, 64 (l + 1))) for the first and last non-silent frames f and l, [0, 0) when there is none.
// A float32 sample's square is exact in float64, so p_t rounds only in the 255 additions, taken in sample order; the file is
// built with -fmad=false, so nothing contracts.  The clip's maximum (the bit pattern of a non-negative double orders as the
// double does) and its first and last non-silent frames are integer atomics, whose result does not depend on their order:
// a clip's bounds do not depend on the other clips of the batch or its position in it.
//
// Three launches per batch whatever the number of clips: frame powers and clip maxima, the dB test, the bounds.
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace ttsb {
namespace {

constexpr int TRIM_FRAME = 256;     // librosa.effects.trim's frame_length as the reference passes it
constexpr int TRIM_HOP = 64;        // and its hop_length
constexpr int TRIM_PAD = TRIM_FRAME / 2;
constexpr int TRIM_THREADS = 256;
constexpr double TRIM_AMIN = 1e-10;

struct TrimState {                  // per clip; the host writes the initial values
  unsigned long long max_bits;      // bit pattern of max_t p_t (0: +0.0)
  unsigned int first;               // first non-silent frame (UINT_MAX: none yet)
  int last;                         // last non-silent frame (-1: none yet)
};

__device__ __forceinline__ int trim_find(const int32_t* __restrict__ off, int n, int x) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(off + mid) <= x) lo = mid; else hi = mid;
  }
  return lo;
}

// np.pad(y, 128, 'reflect') index: period 2 (L - 1) reflection about the first and last samples; a 1-sample clip repeats itself
__device__ __forceinline__ int trim_reflect(int i, int L) {
  if (L == 1) return 0;
  const int P = 2 * (L - 1);
  i %= P;
  if (i < 0) i += P;
  return i >= L ? P - i : i;
}

// Combines v with the values of the following lanes of the same clip: lanes of one clip are consecutive, so after the five
// steps the first lane of each clip's run holds the combination over the run.
template <typename T, typename Op>
__device__ __forceinline__ T trim_segment_reduce(T v, int c, Op op) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T w = __shfl_down_sync(0xffffffffu, v, o);
    const int cw = __shfl_down_sync(0xffffffffu, c, o);
    if (lane + o < 32 && cw == c) v = op(v, w);
  }
  return v;
}

__device__ __forceinline__ bool trim_run_head(int c) {
  const int up = __shfl_up_sync(0xffffffffu, c, 1);
  return c >= 0 && ((threadIdx.x & 31) == 0 || up != c);
}

// p_t of every frame of the batch, and each clip's maximum
__global__ void __launch_bounds__(TRIM_THREADS)
trim_power_kernel(const float* __restrict__ wav, const int32_t* __restrict__ sample_off, const int32_t* __restrict__ frame_off,
                  int n_clips, int total_frames, double* __restrict__ power, TrimState* __restrict__ state) {
  // the loop bound is uniform across a warp: every lane takes part in the shuffles
  for (long long base = (long long)blockIdx.x * blockDim.x; base < total_frames; base += (long long)gridDim.x * blockDim.x) {
    const int g = (int)base + (int)threadIdx.x;
    int c = -1;
    unsigned long long bits = 0;
    if (g < total_frames) {
      c = trim_find(frame_off, n_clips, g);
      const int s0 = __ldg(sample_off + c), L = __ldg(sample_off + c + 1) - s0;
      const int i0 = (g - __ldg(frame_off + c)) * TRIM_HOP - TRIM_PAD;
      const float* x = wav + s0;
      double acc = 0.0;
      if (i0 >= 0 && i0 + TRIM_FRAME <= L) {
        for (int k = 0; k < TRIM_FRAME; ++k) {
          const double v = (double)__ldg(x + i0 + k);
          acc = acc + v * v;
        }
      } else {
        for (int k = 0; k < TRIM_FRAME; ++k) {
          const double v = (double)__ldg(x + trim_reflect(i0 + k, L));
          acc = acc + v * v;
        }
      }
      const double p = acc / (double)TRIM_FRAME;
      power[g] = p;
      bits = (unsigned long long)__double_as_longlong(p);
    }
    bits = trim_segment_reduce(bits, c, [](unsigned long long a, unsigned long long b) { return a > b ? a : b; });
    if (trim_run_head(c)) atomicMax(&state[c].max_bits, bits);
  }
}

// the dB test of every frame against its clip's maximum; each clip's first and last non-silent frame
__global__ void __launch_bounds__(TRIM_THREADS)
trim_test_kernel(const int32_t* __restrict__ frame_off, int n_clips, int total_frames, const double* __restrict__ power,
                 double top_db, TrimState* __restrict__ state) {
  for (long long base = (long long)blockIdx.x * blockDim.x; base < total_frames; base += (long long)gridDim.x * blockDim.x) {
    const int g = (int)base + (int)threadIdx.x;
    int c = -1, first = INT_MAX, last = -1;
    if (g < total_frames) {
      c = trim_find(frame_off, n_clips, g);
      const double ref = __longlong_as_double((long long)state[c].max_bits);
      const double db = 10.0 * log10(fmax(TRIM_AMIN, power[g])) - 10.0 * log10(fmax(TRIM_AMIN, ref));
      if (db > -top_db) first = last = g - __ldg(frame_off + c);
    }
    first = trim_segment_reduce(first, c, [](int a, int b) { return a < b ? a : b; });
    last = trim_segment_reduce(last, c, [](int a, int b) { return a > b ? a : b; });
    if (trim_run_head(c)) {
      if (first != INT_MAX) atomicMin(&state[c].first, (unsigned int)first);
      if (last >= 0) atomicMax(&state[c].last, last);
    }
  }
}

__global__ void trim_bounds_kernel(const int32_t* __restrict__ sample_off, int n_clips, const TrimState* __restrict__ state,
                                   int32_t* __restrict__ bounds) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n_clips; c += gridDim.x * blockDim.x) {
    const int L = sample_off[c + 1] - sample_off[c];
    const TrimState s = state[c];
    int start = 0, end = 0;
    if (s.last >= 0) {
      start = (int)s.first * TRIM_HOP;
      const long long past = (long long)(s.last + 1) * TRIM_HOP;
      end = past < L ? (int)past : L;
    }
    bounds[2 * c] = start;
    bounds[2 * c + 1] = end;
  }
}

int trim_bad(const char* fmt, long long a = 0, long long b = 0) {
  set_last_error(fmt, a, b);
  return TTSB_ERR_INVALID_ARGUMENT;
}

size_t trim_align16(size_t x) { return (x + 15) & ~(size_t)15; }

struct TrimPlan {
  std::vector<int32_t> frame_off;
  size_t off_samples = 0, off_frames = 0, off_power = 0;
  int64_t bytes = 0;
};

// Checks the offsets and lays out the workspace: clip states, sample offsets, frame offsets, frame powers.
int trim_plan(const int32_t* sample_offsets, int n_clips, TrimPlan& p) {
  if (!sample_offsets) return trim_bad("ttsb_trim_silence: NULL sample_offsets");
  if (n_clips < 1) return trim_bad("ttsb_trim_silence: n_clips %lld < 1", n_clips);
  if (sample_offsets[0] != 0) return trim_bad("ttsb_trim_silence: sample_offsets must start at 0, got %lld", sample_offsets[0]);
  p.frame_off.assign(1, 0);
  long long frames = 0;
  for (int c = 0; c < n_clips; ++c) {
    const long long L = (long long)sample_offsets[c + 1] - sample_offsets[c];
    if (L < 0) return trim_bad("ttsb_trim_silence: sample_offsets decrease at clip %lld", c);
    if (L == 0) return trim_bad("ttsb_trim_silence: clip %lld is empty", c);
    frames += 1 + L / TRIM_HOP;
    if (frames > INT32_MAX) return trim_bad("ttsb_trim_silence: too many frames");
    p.frame_off.push_back((int32_t)frames);
  }
  p.off_samples = trim_align16((size_t)n_clips * sizeof(TrimState));
  p.off_frames = trim_align16(p.off_samples + (size_t)(n_clips + 1) * sizeof(int32_t));
  p.off_power = trim_align16(p.off_frames + (size_t)(n_clips + 1) * sizeof(int32_t));
  p.bytes = (int64_t)(p.off_power + (size_t)frames * sizeof(double));
  return 0;
}

}  // namespace
}  // namespace ttsb

using namespace ttsb;

extern "C" int64_t ttsb_trim_silence_workspace_bytes(const int32_t* sample_offsets, int n_clips) {
  TrimPlan p;
  if (trim_plan(sample_offsets, n_clips, p)) return -1;
  return p.bytes;
}

extern "C" int ttsb_trim_silence_bounds(const float* wav, const int32_t* sample_offsets, int n_clips, double top_db, void* workspace,
                                        int64_t workspace_bytes, int32_t* bounds, void* stream_v) {
  if (!wav || !workspace || !bounds) return trim_bad("ttsb_trim_silence: NULL pointer");
  TrimPlan p;
  int rc = trim_plan(sample_offsets, n_clips, p);
  if (rc) return rc;
  if (!isfinite(top_db) || top_db <= 0.0) {
    set_last_error("ttsb_trim_silence: top_db must be finite and > 0, got %g", top_db);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (workspace_bytes < p.bytes) return trim_bad("ttsb_trim_silence: workspace too small (%lld bytes, need %lld)", workspace_bytes, p.bytes);
  if (reinterpret_cast<uintptr_t>(workspace) % 16 != 0) return trim_bad("ttsb_trim_silence: workspace must be 16-byte aligned");
  // host image of the workspace up to the frame powers: initial clip states and both offset tables, one copy
  std::vector<uint8_t> host(p.off_power, 0);
  TrimState* st = reinterpret_cast<TrimState*>(host.data());
  for (int c = 0; c < n_clips; ++c) st[c] = TrimState{0ull, 0xffffffffu, -1};
  memcpy(host.data() + p.off_samples, sample_offsets, (size_t)(n_clips + 1) * sizeof(int32_t));
  memcpy(host.data() + p.off_frames, p.frame_off.data(), p.frame_off.size() * sizeof(int32_t));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  TTSB_CUDA_OK(cudaMemcpyAsync(ws, host.data(), host.size(), cudaMemcpyHostToDevice, stream));
  TrimState* state = reinterpret_cast<TrimState*>(ws);
  const int32_t* so = reinterpret_cast<const int32_t*>(ws + p.off_samples);
  const int32_t* fo = reinterpret_cast<const int32_t*>(ws + p.off_frames);
  double* power = reinterpret_cast<double*>(ws + p.off_power);
  const int total = p.frame_off.back();
  const int grid = (int)std::min(((long long)total + TRIM_THREADS - 1) / TRIM_THREADS, (long long)16 * num_sms());
  trim_power_kernel<<<grid, TRIM_THREADS, 0, stream>>>(wav, so, fo, n_clips, total, power, state);
  count_launch();
  rc = check_cuda(cudaGetLastError(), "trim_power_kernel launch");
  if (rc) return rc;
  trim_test_kernel<<<grid, TRIM_THREADS, 0, stream>>>(fo, n_clips, total, power, top_db, state);
  count_launch();
  rc = check_cuda(cudaGetLastError(), "trim_test_kernel launch");
  if (rc) return rc;
  trim_bounds_kernel<<<(n_clips + 255) / 256, 256, 0, stream>>>(so, n_clips, state, bounds);
  count_launch();
  return check_cuda(cudaGetLastError(), "trim_bounds_kernel launch");
}
