// Band-limited resampling of a packed ragged batch of clips (ttsb_resample_batch): resampy's `kaiser_best` interpolator as
// librosa.load(path, sr=...) reaches it (reference: data/audio.py:126-130), every clip from its own source rate to one target rate.
//
// Per output sample t of a clip of L samples (resampy's resample_f, single channel):
//   r_t: the time register, r_0 = 0, r_{t+1} = fl(r_t + 1/ratio) in float64;
//   m = trunc(r_t), frac = scale (r_t - m), off = trunc(512 frac), eta = 512 frac - off;
//   left wing  i < min(m + 1, (nwin - off) / step):      acc += (h'[off + i step] + eta D'[off + i step]) x[m - i]
//   right wing k < min(L - m - 1, (nwin - off2) / step):  the same from frac2 = scale - frac with x[m + 1 + k];
// every operation in float64 in that order, the accumulator rounded to float32 after each tap (resampy adds into a float32
// array).  The file is built with -fmad=false and spells the products and sums as __d*_rn as well: no contraction.
//
// The time register is a serial float64 recurrence, but it is exactly piecewise linear: while r stays in one binade [2^e, 2^e+1)
// with ulp u, r + inc rounds to r + d with the constant d = round(inc / u) u (inc's bits below u are not exactly half an ulp,
// or, when they are, r / u is even and d is the even one of the two neighbours).  The host walks the recurrence binade by
// binade, emitting segments (t0, r0, d) with r_t = r0 + (t - t0) d exact for every t of the segment, and takes each step near a
// binade's top, and the odd tie step, with a genuine float64 addition.  3 M output samples at the common rate pairs (8 to 96 kHz
// to 16, 22.05, 24 or 44.1 kHz) take 23-24 segments, so the kernel computes any r_t in O(log) without a serial prologue,
// bit-identical to the recurrence.
//
// The interpolation table h' (h scaled by ratio when downsampling) and its differences D' are rebuilt on the device for each
// distinct (ratio, step) of the batch, reordered by filter phase: row `off` holds (h'[off + i step], D'[off + i step]) for
// i = 0, 1, ... as double2, so a thread's taps read consecutive 16-byte entries instead of one 32-byte sector each.
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

constexpr int RS_NUM_TABLE = 512;       // resampy's kaiser_best: 2^9 table entries per zero crossing
constexpr int RS_THREADS = 256;
constexpr int RS_MAX_WINDOW = 1 << 22;

struct RsClip {
  long long in0;    // first input sample of the clip in wav
  int L;            // input samples
  int n_out;        // computed output samples int(L ratio); the clip's remaining output samples (ceil - int) are zero
  int copy;         // 1: source rate == target rate, the output is the input
  int step;         // int(scale 512)
  int row;          // row length of the clip's phase-ordered table
  int seg0;         // first segment of the clip's time register
  int n_seg;
  int pad_;
  long long table;  // first double2 of the clip's table
  double scale;     // min(1, ratio)
};

struct RsSeg {
  double r0, d;     // r_t = r0 + (t - t0) d, exact
  long long t0;
  long long pad_;
};

struct RsTable {    // one per distinct (ratio, step)
  double mul;       // ratio when downsampling, 1 otherwise
  int scaled;       // h' = h * ratio (resampy scales only when ratio < 1)
  int step, row;
  long long base;   // first double2
};

__device__ __forceinline__ int rs_find(const int32_t* __restrict__ tab, int n, int x) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(tab + mid) <= x) lo = mid; else hi = mid;
  }
  return lo;
}

// table k, entry (off, i) = (h'[j], h'[j+1] - h'[j]) with j = off + i step (zeros past the window; never read)
__global__ void resample_table_kernel(const double* __restrict__ h, int nwin, const RsTable* __restrict__ tabs, double2* __restrict__ out) {
  const RsTable tb = tabs[blockIdx.y];
  const int n = (tb.step + 1) * tb.row;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
    const int off = e / tb.row, i = e - off * tb.row;
    const long long j = off + (long long)i * tb.step;
    double2 v = make_double2(0.0, 0.0);
    if (j < nwin) {
      const double a = tb.scaled ? __dmul_rn(__ldg(h + j), tb.mul) : __ldg(h + j);
      v.x = a;
      if (j + 1 < nwin) v.y = __dsub_rn(tb.scaled ? __dmul_rn(__ldg(h + j + 1), tb.mul) : __ldg(h + j + 1), a);
    }
    out[tb.base + e] = v;
  }
}

__device__ __forceinline__ float rs_wing(const double2* __restrict__ row, int n, double eta, const float* __restrict__ x, int dir,
                                         float acc) {
  for (int i = 0; i < n; ++i) {
    const double2 hd = row[i];
    const double w = __dadd_rn(hd.x, __dmul_rn(eta, hd.y));
    acc = __double2float_rn(__dadd_rn((double)acc, __dmul_rn(w, (double)__ldg(x + dir * i))));
  }
  return acc;
}

__global__ void __launch_bounds__(RS_THREADS)
resample_kernel(const float* __restrict__ wav, const int32_t* __restrict__ out_off, const RsClip* __restrict__ clips,
                const RsSeg* __restrict__ segs, const double2* __restrict__ tables, int n_clips, int total, int nwin,
                float* __restrict__ out) {
  // 64-bit loop index: total may be up to INT32_MAX, and o + grid stride must not wrap
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += (long long)gridDim.x * blockDim.x) {
    const int c = rs_find(out_off, n_clips, (int)o);
    const RsClip& cl = clips[c];
    const int t = (int)o - __ldg(out_off + c);
    const float* x = wav + cl.in0;
    if (cl.copy) { out[o] = __ldg(x + t); continue; }
    if (t >= cl.n_out) { out[o] = 0.f; continue; }
    int lo = cl.seg0, hi = cl.seg0 + cl.n_seg;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (segs[mid].t0 <= t) lo = mid; else hi = mid;
    }
    const RsSeg sg = segs[lo];
    const double r = __dadd_rn(sg.r0, __dmul_rn((double)(t - sg.t0), sg.d));
    const double scale = cl.scale;
    const int step = cl.step, L = cl.L;
    const double2* tab = tables + cl.table;
    const int m = (int)r;
    const double frac = __dmul_rn(scale, __dsub_rn(r, (double)m));
    double idx = __dmul_rn(frac, (double)RS_NUM_TABLE);
    int off = (int)idx;
    double eta = __dsub_rn(idx, (double)off);
    float acc = rs_wing(tab + (size_t)off * cl.row, min(m + 1, (nwin - off) / step), eta, x + m, -1, 0.f);
    const double frac2 = __dsub_rn(scale, frac);
    idx = __dmul_rn(frac2, (double)RS_NUM_TABLE);
    off = (int)idx;
    eta = __dsub_rn(idx, (double)off);
    acc = rs_wing(tab + (size_t)off * cl.row, min(L - m - 1, (nwin - off) / step), eta, x + m + 1, 1, acc);
    out[o] = acc;
  }
}

// Segments of r_0 .. r_{n_out - 1} (see the file's header).  Every double operation here is exact except the r + inc steps,
// which are the recurrence's own.
void plan_register(double inc, long long n_out, std::vector<RsSeg>& segs) {
  segs.push_back({0.0, 0.0, 0, 0});
  long long t = 1;
  double r = inc;
  while (t < n_out) {
    int e;
    frexp(r, &e);                                   // r in [2^(e-1), 2^e): ulp 2^(e-53)
    const double u = ldexp(1.0, e - 53);
    const double qf = inc / u;                      // r >= inc, so u >= ulp(inc) and inc / u < 2^53
    const long long q = (long long)qf;
    const double f = qf - (double)q;
    const long long N = (long long)(r / u);         // in [2^52, 2^53)
    long long step = f < 0.5 ? q : f > 0.5 ? q + 1 : (q % 2 == 0 ? q : q + 1);
    if (f == 0.5 && N % 2 != 0) step = 0;           // the first tie step from an odd N rounds the other way: take it for real
    long long K = 0;                                // closed-form steps: every exact sum stays below 2^53 u
    if (step > 0) {
      const long long room = (1LL << 53) - 2 - N - step;
      if (room >= 0) K = room / step + 1;
    }
    if (K > n_out - 1 - t) K = n_out - 1 - t;
    const double d = (double)step * u;
    segs.push_back({r, d, t, 0});
    r = r + (double)K * d;
    t += K + 1;
    r = r + inc;
  }
}

struct RsPlan {
  std::vector<RsClip> clips;
  std::vector<RsSeg> segs;
  std::vector<RsTable> tables;
  std::vector<int32_t> out_off;
  long long table_entries = 0;
  int64_t bytes = 0;
  size_t off_clips = 0, off_segs = 0, off_tabs = 0, off_out = 0;
};

int rs_bad(const char* fmt, long long a = 0, long long b = 0, long long c = 0, long long d = 0) {
  set_last_error(fmt, a, b, c, d);
  return TTSB_ERR_INVALID_ARGUMENT;
}

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// Checks the host tables and lays out the workspace.  out_offsets may be NULL (the workspace query).
int make_plan(const int32_t* sample_offsets, const int32_t* src_rates, int n_clips, int dst_rate, int n_window,
              const int32_t* out_offsets, RsPlan& p) {
  if (!sample_offsets || !src_rates) return rs_bad("ttsb_resample_batch: NULL offset or rate table");
  if (n_clips < 1) return rs_bad("ttsb_resample_batch: n_clips < 1");
  if (dst_rate <= 0) return rs_bad("ttsb_resample_batch: target rate %lld <= 0", dst_rate);
  if (n_window < 2 || n_window > RS_MAX_WINDOW) return rs_bad("ttsb_resample_batch: n_window %lld outside [2, %lld]", n_window, RS_MAX_WINDOW);
  if (sample_offsets[0] != 0) return rs_bad("ttsb_resample_batch: sample_offsets must start at 0");
  if (out_offsets && out_offsets[0] != 0) return rs_bad("ttsb_resample_batch: out_offsets must start at 0");
  long long out_total = 0;
  p.out_off.assign(1, 0);
  for (int c = 0; c < n_clips; ++c) {
    const long long L = (long long)sample_offsets[c + 1] - sample_offsets[c];
    if (L < 0) return rs_bad("ttsb_resample_batch: sample_offsets decrease at clip %lld", c);
    const int sr = src_rates[c];
    if (sr <= 0) return rs_bad("ttsb_resample_batch: clip %lld has source rate %lld <= 0", c, sr);
    RsClip cl{};
    cl.in0 = sample_offsets[c];
    cl.L = (int)L;
    long long n_total;
    if (sr == dst_rate) {
      cl.copy = 1;
      n_total = L;
    } else {
      const double ratio = (double)dst_rate / (double)sr;
      const long long n_out = (long long)((double)L * ratio);
      if (n_out < 1)
        return rs_bad("ttsb_resample_batch: clip %lld has %lld samples at %lld Hz: too short to resample (no output sample)", c, L, sr);
      n_total = (long long)ceil((double)L * ratio);
      const double scale = ratio < 1.0 ? ratio : 1.0;
      const int step = (int)(scale * RS_NUM_TABLE);
      if (step < 1) return rs_bad("ttsb_resample_batch: clip %lld: ratio %lld / %lld is below 1/512", c, dst_rate, sr);
      cl.n_out = (int)n_out;
      cl.scale = scale;
      cl.step = step;
      cl.row = n_window / step + 1;
      const double mul = ratio < 1.0 ? ratio : 1.0;
      int k = 0;
      while (k < (int)p.tables.size() && !(p.tables[k].mul == mul && p.tables[k].step == step)) ++k;
      if (k == (int)p.tables.size()) {
        p.tables.push_back({mul, ratio < 1.0 ? 1 : 0, step, cl.row, p.table_entries});
        p.table_entries += (long long)(step + 1) * cl.row;
      }
      cl.table = p.tables[k].base;
      cl.seg0 = (int)p.segs.size();
      plan_register(1.0 / ratio, n_out, p.segs);
      cl.n_seg = (int)p.segs.size() - cl.seg0;
    }
    if (out_offsets && (long long)out_offsets[c + 1] - out_offsets[c] != n_total)
      return rs_bad("ttsb_resample_batch: out_offsets give clip %lld %lld samples; ceil(L * dst_rate / src_rate) is %lld", c,
                    (long long)out_offsets[c + 1] - out_offsets[c], n_total);
    out_total += n_total;
    if (out_total > INT32_MAX || (long long)sample_offsets[c + 1] > INT32_MAX) return rs_bad("ttsb_resample_batch: too many samples");
    p.out_off.push_back((int32_t)out_total);
    p.clips.push_back(cl);
  }
  p.off_tabs = 0;
  p.off_clips = align16(p.off_tabs + (size_t)p.table_entries * sizeof(double2));
  p.off_segs = align16(p.off_clips + p.clips.size() * sizeof(RsClip));
  p.off_out = align16(p.off_segs + p.segs.size() * sizeof(RsSeg));
  const size_t off_desc = align16(p.off_out + p.out_off.size() * sizeof(int32_t));
  p.bytes = (int64_t)align16(off_desc + p.tables.size() * sizeof(RsTable));
  return 0;
}

}  // namespace
}  // namespace ttsb

using namespace ttsb;

extern "C" int64_t ttsb_resample_batch_workspace_bytes(const int32_t* sample_offsets, const int32_t* src_rates, int n_clips,
                                                       int dst_rate, int n_window) {
  RsPlan p;
  if (make_plan(sample_offsets, src_rates, n_clips, dst_rate, n_window, nullptr, p)) return -1;
  return p.bytes;
}

extern "C" int ttsb_resample_batch(const float* wav, const int32_t* sample_offsets, const int32_t* src_rates, int n_clips, int dst_rate,
                                   const double* half_window, int n_window, const int32_t* out_offsets, void* workspace,
                                   int64_t workspace_bytes, float* out, void* stream_v) {
  if (!wav || !half_window || !out_offsets || !workspace || !out) return rs_bad("ttsb_resample_batch: NULL pointer");
  RsPlan p;
  int rc = make_plan(sample_offsets, src_rates, n_clips, dst_rate, n_window, out_offsets, p);
  if (rc) return rc;
  if (workspace_bytes < p.bytes) return rs_bad("ttsb_resample_batch: workspace too small (%lld bytes, need %lld)", workspace_bytes, p.bytes);
  if (reinterpret_cast<uintptr_t>(workspace) % 16 != 0) return rs_bad("ttsb_resample_batch: workspace must be 16-byte aligned");
  const size_t off_desc = align16(p.off_out + p.out_off.size() * sizeof(int32_t));
  std::vector<uint8_t> host((size_t)p.bytes - p.off_clips);
  uint8_t* h0 = host.data() - p.off_clips;        // host image of the workspace from off_clips on
  memcpy(h0 + p.off_clips, p.clips.data(), p.clips.size() * sizeof(RsClip));
  memcpy(h0 + p.off_segs, p.segs.data(), p.segs.size() * sizeof(RsSeg));
  memcpy(h0 + p.off_out, p.out_off.data(), p.out_off.size() * sizeof(int32_t));
  memcpy(h0 + off_desc, p.tables.data(), p.tables.size() * sizeof(RsTable));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  TTSB_CUDA_OK(cudaMemcpyAsync(ws + p.off_clips, host.data(), host.size(), cudaMemcpyHostToDevice, stream));
  double2* tables = reinterpret_cast<double2*>(ws + p.off_tabs);
  if (!p.tables.empty()) {
    int most = 0;
    for (const RsTable& t : p.tables) most = std::max(most, (t.step + 1) * t.row);
    dim3 grid((most + 255) / 256, (unsigned)p.tables.size());
    resample_table_kernel<<<grid, 256, 0, stream>>>(half_window, n_window, reinterpret_cast<const RsTable*>(ws + off_desc), tables);
    count_launch();
    rc = check_cuda(cudaGetLastError(), "resample_table_kernel launch");
    if (rc) return rc;
  }
  const int total = p.out_off.back();
  if (total == 0) return 0;
  const int grid = (int)std::min(((long long)total + RS_THREADS - 1) / RS_THREADS, (long long)64 * num_sms());
  resample_kernel<<<grid, RS_THREADS, 0, stream>>>(wav, reinterpret_cast<const int32_t*>(ws + p.off_out),
                                                   reinterpret_cast<const RsClip*>(ws + p.off_clips),
                                                   reinterpret_cast<const RsSeg*>(ws + p.off_segs), tables, n_clips, total, n_window, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "resample_kernel launch");
}
