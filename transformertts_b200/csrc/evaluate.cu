// Objective scoring of synthesised mels (evaluate_tts.py; no reference counterpart): mel-cepstral distortion after dynamic time
// warping, for a packed ragged batch of (x, y) pairs of log-mel sequences.
//
// The definition (include/ttsb.h, tests/evaluation_oracle.py restates it in float64 numpy):
//   c_k[t]  = sum_m D[k][m] x[t][m], k = 1..K, D the orthonormal DCT-II of the M log-mel bins (c0, the energy, is left out);
//   d(i, j) = kappa sqrt(2 sum_k (c_k[i] - c'_k[j])^2), kappa = 10 / ln 10 from the host;
//   C[i][j] = d(i, j) + min(C[i-1][j-1], C[i-1][j], C[i][j-1]), C[0][0] = d(0, 0); the path length L rides along with C.
// Every product and sum is rounded on its own (explicit __dmul_rn / __dadd_rn, and the file builds with -fmad=false), sums run
// in the order the definition gives, and sqrt is IEEE, so the result is the float64 restatement's bit for bit.
//
// Two kernels: mcd_cepstra_kernel writes the cepstra of every frame of both sides, k-major, into the workspace (so the
// threads of one anti-diagonal, whose frames are consecutive, read consecutive addresses); mcd_dtw_kernel runs one CTA per
// pair over the anti-diagonals of its cost matrix, indexed along the pair's shorter side, with three rolling diagonals of
// (C, L) in shared memory.  No atomics and no cross-pair state: a pair's result does not depend on the batch.
//
// ttsb_mcd_dtw_path runs the same sweep (mcd_dtw_kernel<true>; ttsb_mcd_dtw is the <false> instantiation, whose code the
// flag leaves as it was) and also records the predecessor each cell took, as two bit-planes per 32 cells of a diagonal:
// word 2w has bit l set when cell 32w + l took (i - 1, j), word 2w + 1 when it took (i, j - 1), neither for the diagonal.
// Each warp writes its two words from __ballot_sync, so no atomics and no byte-sized stores.  Diagonal d of a pair holds
// 2 ceil(n_d / 32) words (n_d its cells) after those of diagonals 0 .. d - 1, from the pair's offset in the workspace.
// After the last diagonal, thread 0 of the CTA walks back from (Tx - 1, Ty - 1) and writes the path from entry L - 1 down.
//
// ttsb_mcd_dtw_ceps(_path) score cepstra the caller computed (the WORLD mel-cepstra of world_sp.cu): mcd_ceps_copy_kernel
// copies columns first .. first + K - 1 of the frame-major float64 rows into the same k-major workspace, and the same
// mcd_dtw_kernel<false / true> sweeps it.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <vector>

#include "ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace ttsb {

constexpr int DTW_THREADS = 256;
constexpr size_t DTW_CELL_BYTES = sizeof(double) + sizeof(int32_t);   // one (C, L) entry of a diagonal

// ceps[(k - 1) F + f] = c_k of frame f, f < Fx from x, else frame f - Fx of y; dct (K, M) holds the rows k = 1..K
__global__ void mcd_cepstra_kernel(const float* __restrict__ x, int64_t Fx, const float* __restrict__ y, int64_t F, int M,
                                   const double* __restrict__ dct, int K, double* __restrict__ ceps) {
  const int64_t n = F * K;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(e / F);
    const int64_t f = e - (int64_t)k * F;
    const float* row = f < Fx ? x + f * M : y + (f - Fx) * M;
    const double* d = dct + (size_t)k * M;
    double acc = 0.0;
    for (int m = 0; m < M; ++m) acc = __dadd_rn(acc, __dmul_rn(__ldg(d + m), (double)__ldg(row + m)));
    ceps[e] = acc;
  }
}

// ceps[k F + f] = column first + k of row f of x (f < Fx), else of row f - Fx of y; rows of ld doubles
__global__ void mcd_ceps_copy_kernel(const double* __restrict__ x, int64_t Fx, const double* __restrict__ y, int64_t F, int ld,
                                     int first, int K, double* __restrict__ ceps) {
  const int64_t n = F * K;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(e / F);
    const int64_t f = e - (int64_t)k * F;
    ceps[e] = f < Fx ? __ldg(x + f * ld + first + k) : __ldg(y + (f - Fx) * ld + first + k);
  }
}

__device__ __forceinline__ double frame_distance(const double* __restrict__ ceps, int64_t F, int K, int64_t fa, int64_t fb,
                                                 double kappa) {
  double s = 0.0;
  for (int k = 0; k < K; ++k) {
    const double t = __dsub_rn(__ldg(ceps + (int64_t)k * F + fa), __ldg(ceps + (int64_t)k * F + fb));
    s = __dadd_rn(s, __dmul_rn(t, t));
  }
  return __dmul_rn(kappa, __dsqrt_rn(__dmul_rn(2.0, s)));
}

__device__ __forceinline__ int dtw_diag_len(int d, int Nu, int Nv) { return min(d, Nu - 1) - max(0, d - Nv + 1) + 1; }

// tab: x frame offsets (n_pairs + 1), then y frame offsets (n_pairs + 1), both as indices into the cepstra (y after x).
// kPath: bit_off (n_pairs) is each pair's first word of choice bits in `bits`; pair p's path starts at int2 entry
// x0 + (y0 - tab[n_pairs + 1]) - p of path_out, i.e. after the Tx + Ty - 1 entries of every earlier pair.
template <bool kPath>
__global__ void __launch_bounds__(DTW_THREADS)
mcd_dtw_kernel(const double* __restrict__ ceps, int64_t F, int K, const int32_t* __restrict__ tab, int n_pairs, double kappa,
               double* __restrict__ cost_out, int32_t* __restrict__ len_out, uint32_t* __restrict__ bits,
               const int64_t* __restrict__ bit_off, int2* __restrict__ path_out) {
  extern __shared__ double dtw_sm[];
  const int p = blockIdx.x;
  const int64_t x0 = tab[p], y0 = tab[n_pairs + 1 + p];
  const int Tx = tab[p + 1] - tab[p], Ty = tab[n_pairs + 2 + p] - tab[n_pairs + 1 + p];
  // u runs along the shorter side, v = d - u along the longer one; (i, j) = swapped ? (v, u) : (u, v)
  const bool swapped = Tx > Ty;
  const int Nu = swapped ? Ty : Tx, Nv = swapped ? Tx : Ty;
  const int64_t u0 = swapped ? y0 : x0, v0 = swapped ? x0 : y0;
  double* C0 = dtw_sm;   // diagonal d, d - 1, d - 2
  double* C1 = C0 + Nu;
  double* C2 = C1 + Nu;
  int32_t* L0 = reinterpret_cast<int32_t*>(C2 + Nu);
  int32_t* L1 = L0 + Nu;
  int32_t* L2 = L1 + Nu;
  uint32_t* wd = kPath ? bits + bit_off[p] : nullptr;   // the words of diagonal d
  for (int d = 0; d < Nu + Nv - 1; ++d) {
    const int u_lo = max(0, d - Nv + 1), u_hi = min(d, Nu - 1);
    for (int u = u_lo + threadIdx.x; u <= u_hi; u += blockDim.x) {
      const int v = d - u;
      const double dist = frame_distance(ceps, F, K, u0 + u, v0 + v, kappa);
      double best = 0.0;
      int32_t len = 0;
      int choice = 0;   // 0: (i - 1, j - 1), 1: (i - 1, j), 2: (i, j - 1)
      if (d > 0) {
        // the predecessors on diagonal d - 1: (u - 1, v) and (u, v - 1); which one is (i - 1, j) depends on the orientation
        const bool has_a = u > 0, has_b = v > 0;
        const bool i_up_is_a = !swapped;               // (i - 1, j) = (u - 1, v) unless swapped
        const bool has_up = i_up_is_a ? has_a : has_b, has_left = i_up_is_a ? has_b : has_a;
        const int up_idx = i_up_is_a ? u - 1 : u, left_idx = i_up_is_a ? u : u - 1;
        best = INFINITY;
        if (has_a && has_b) { best = C2[u - 1]; len = L2[u - 1]; }                                     // (i - 1, j - 1)
        if (has_up && C1[up_idx] < best) { best = C1[up_idx]; len = L1[up_idx]; choice = 1; }          // (i - 1, j)
        if (has_left && C1[left_idx] < best) { best = C1[left_idx]; len = L1[left_idx]; choice = 2; }  // (i, j - 1)
      }
      const double c = __dadd_rn(dist, best);
      C0[u] = c;
      L0[u] = len + 1;
      if (d == Nu + Nv - 2) {   // the one cell of the last diagonal: (Tx - 1, Ty - 1)
        cost_out[p] = c;
        len_out[p] = len + 1;
      }
      if constexpr (kPath) {
        // the lanes of this warp with a cell on the diagonal are a prefix of it, and all of them are here
        const int lane = threadIdx.x & 31, c0 = u - lane - u_lo;   // c0: the warp's first cell, a multiple of 32
        const int n = min(32, u_hi - u_lo - c0 + 1);
        const unsigned mask = n == 32 ? 0xffffffffu : (1u << n) - 1u;
        const unsigned up = __ballot_sync(mask, choice == 1), left = __ballot_sync(mask, choice == 2);
        if (lane == 0) reinterpret_cast<uint2*>(wd)[c0 >> 5] = make_uint2(up, left);
      }
    }
    __syncthreads();
    double* tc = C2; C2 = C1; C1 = C0; C0 = tc;
    int32_t* tl = L2; L2 = L1; L1 = L0; L0 = tl;
    if constexpr (kPath) { if (d < Nu + Nv - 2) wd += 2 * ((dtw_diag_len(d, Nu, Nv) + 31) >> 5); }
  }
  if constexpr (kPath) {
    // the traceback: the choice bits of every diagonal and len_out[p] were written before the last __syncthreads
    if (threadIdx.x != 0) return;
    int2* out = path_out + (x0 + (y0 - tab[n_pairs + 1]) - p);
    int i = Tx - 1, j = Ty - 1, d = Nu + Nv - 2;
    for (int k = len_out[p] - 1; k >= 0; --k) {
      out[k] = make_int2(i, j);
      if (d == 0) break;
      const int c = (swapped ? j : i) - max(0, d - Nv + 1);
      const uint2 w = reinterpret_cast<const uint2*>(wd)[c >> 5];
      const int choice = (w.x >> (c & 31)) & 1u ? 1 : (w.y >> (c & 31)) & 1u ? 2 : 0;
      i -= choice != 2;
      j -= choice != 1;
      for (int back = choice == 0 ? 2 : 1; back > 0; --back) {
        --d;
        wd -= 2 * ((dtw_diag_len(d, Nu, Nv) + 31) >> 5);
      }
    }
  }
}

struct McdPlan {
  int64_t fx, frames;   // x frames, x + y frames
  int max_short;        // the longest shorter side of any pair: the diagonal length the shared memory must hold
  int64_t ceps_bytes, bytes;
  std::vector<int64_t> bit_off;   // with the path: each pair's first word of choice bits, then the total
};

// the words of choice bits of a Tx x Ty pair: 2 ceil(n_d / 32) for each anti-diagonal d of n_d cells
static int64_t path_bit_words(int64_t tx, int64_t ty) {
  const int64_t nu = tx < ty ? tx : ty, nv = tx < ty ? ty : tx;
  int64_t words = 0;
  for (int64_t d = 0; d < nu + nv - 1; ++d) {
    const int64_t n = (d < nu - 1 ? d : nu - 1) - (d - nv + 1 > 0 ? d - nv + 1 : 0) + 1;
    words += 2 * ((n + 31) / 32);
  }
  return words;
}

// checks the pair tables and n_ceps (and, with the path, the cell limit); 0, or TTSB_ERR_INVALID_ARGUMENT with the error text
// set.  Workspace: the cepstra, the pair table, and with the path the bit offsets (int64, n_pairs) and the choice bits.
static int mcd_plan(const char* fn, const int32_t* xo, const int32_t* yo, int n_pairs, int n_ceps, bool path, McdPlan* pl) {
  if (!xo || !yo) { set_last_error("%s: NULL offset table", fn); return TTSB_ERR_INVALID_ARGUMENT; }
  if (n_pairs < 1) { set_last_error("%s: need n_pairs >= 1, got %d", fn, n_pairs); return TTSB_ERR_INVALID_ARGUMENT; }
  if (n_ceps < 1) { set_last_error("%s: need n_ceps >= 1, got %d", fn, n_ceps); return TTSB_ERR_INVALID_ARGUMENT; }
  if (xo[0] != 0 || yo[0] != 0) { set_last_error("%s: offsets must start at 0", fn); return TTSB_ERR_INVALID_ARGUMENT; }
  pl->max_short = 0;
  for (int p = 0; p < n_pairs; ++p) {
    const long long tx = (long long)xo[p + 1] - xo[p], ty = (long long)yo[p + 1] - yo[p];
    if (tx < 1 || ty < 1) {
      set_last_error("%s: pair %d has %lld x frames and %lld y frames; every sequence needs at least 1", fn, p, tx, ty);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
    const long long s = tx < ty ? tx : ty;
    if (s > TTSB_MCD_DTW_MAX_FRAMES) {
      set_last_error("%s: pair %d is %lld x %lld frames; the shorter side may have at most %d frames (the shared-memory "
                     "diagonals of one pair hold that many; about 47 s at hop 256)", fn, p, tx, ty, TTSB_MCD_DTW_MAX_FRAMES);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
    if (path && tx * ty > TTSB_MCD_DTW_PATH_MAX_CELLS) {
      set_last_error("%s: pair %d is %lld x %lld frames, %lld cells; the path variant takes at most %d cells per pair (2 bits "
                     "of workspace each)", fn, p, tx, ty, tx * ty, TTSB_MCD_DTW_PATH_MAX_CELLS);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
    pl->max_short = (int)(s > pl->max_short ? s : pl->max_short);
  }
  pl->fx = xo[n_pairs];
  pl->frames = pl->fx + yo[n_pairs];
  if (pl->frames > INT32_MAX) { set_last_error("%s: more than 2^31 - 1 frames in all", fn); return TTSB_ERR_INVALID_ARGUMENT; }
  pl->ceps_bytes = pl->frames * n_ceps * (int64_t)sizeof(double);
  pl->bytes = pl->ceps_bytes + 2 * ((int64_t)n_pairs + 1) * (int64_t)sizeof(int32_t);
  if (path) {
    pl->bit_off.assign((size_t)n_pairs + 1, 0);
    for (int p = 0; p < n_pairs; ++p)
      pl->bit_off[p + 1] = pl->bit_off[p] + path_bit_words((int64_t)xo[p + 1] - xo[p], (int64_t)yo[p + 1] - yo[p]);
    pl->bytes += (int64_t)n_pairs * (int64_t)sizeof(int64_t) + pl->bit_off[n_pairs] * (int64_t)sizeof(uint32_t);
  }
  return 0;
}

// Checks the workspace, uploads the pair table (and the path's bit offsets), lets `fill` write the k-major cepstra into the
// workspace and sweeps them with mcd_dtw_kernel<kPath>.
template <bool kPath, typename Fill>
static int mcd_dtw_launch(const char* fn, const McdPlan& pl, const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps,
                          double kappa, void* workspace, int64_t workspace_bytes, double* cost_out, int32_t* path_len_out,
                          int32_t* path_out, void* stream_v, Fill fill) {
  if (workspace_bytes < pl.bytes) {
    set_last_error("%s: workspace holds %lld bytes, needs %lld (%s_workspace_bytes)", fn, (long long)workspace_bytes,
                   (long long)pl.bytes, fn);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (reinterpret_cast<uintptr_t>(workspace) % 8 != 0) {
    set_last_error("%s: workspace must be 8-byte aligned", fn);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  std::vector<int32_t> tab(2 * ((size_t)n_pairs + 1));
  for (int p = 0; p <= n_pairs; ++p) {
    tab[p] = x_offsets[p];
    tab[n_pairs + 1 + p] = (int32_t)(pl.fx + y_offsets[p]);   // y frames follow the x frames in the cepstra
  }
  const size_t sm = 3 * (size_t)pl.max_short * DTW_CELL_BYTES;
  {
    static PerDevice<size_t> attr_pd;   // one per instantiation
    size_t& attr = attr_pd.get();
    if (sm > 48 * 1024 && sm > attr) {
      TTSB_CUDA_OK(cudaFuncSetAttribute(mcd_dtw_kernel<kPath>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
      attr = sm;
    }
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  double* ceps = static_cast<double*>(workspace);
  int32_t* tab_dev = reinterpret_cast<int32_t*>(static_cast<uint8_t*>(workspace) + pl.ceps_bytes);
  TTSB_CUDA_OK(cudaMemcpyAsync(tab_dev, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  int64_t* bit_off = nullptr;
  uint32_t* bits = nullptr;
  if (kPath) {   // after the pair table, which ends 8-byte aligned; the bit offsets are even, so each pair's words are too
    bit_off = reinterpret_cast<int64_t*>(tab_dev + tab.size());
    bits = reinterpret_cast<uint32_t*>(bit_off + n_pairs);
    TTSB_CUDA_OK(cudaMemcpyAsync(bit_off, pl.bit_off.data(), (size_t)n_pairs * sizeof(int64_t), cudaMemcpyHostToDevice, stream));
  }
  const int64_t n = pl.frames * n_ceps;
  const int grid = (int)std::min<int64_t>((n + 255) / 256, 8 * (int64_t)num_sms());
  if (int rc = fill(ceps, grid, stream)) return rc;
  mcd_dtw_kernel<kPath><<<n_pairs, DTW_THREADS, sm, stream>>>(ceps, pl.frames, n_ceps, tab_dev, n_pairs, kappa, cost_out, path_len_out,
                                                              bits, bit_off, reinterpret_cast<int2*>(path_out));
  count_launch();
  return check_cuda(cudaGetLastError(), "mcd_dtw_kernel");
}

template <bool kPath>
static int mcd_dtw_run(const char* fn, const float* x, const int32_t* x_offsets, const float* y, const int32_t* y_offsets, int n_pairs,
                       int n_mels, const double* dct, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes, double* cost_out,
                       int32_t* path_len_out, int32_t* path_out, void* stream_v) {
  if (!x || !y || !dct || !workspace || !cost_out || !path_len_out || (kPath && !path_out)) {
    set_last_error("%s: NULL pointer", fn);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (n_mels < 2 || n_ceps < 1 || n_ceps >= n_mels) {
    set_last_error("%s: need 1 <= n_ceps < n_mels (c0 is left out), got n_ceps %d, n_mels %d", fn, n_ceps, n_mels);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (!std::isfinite(kappa) || kappa <= 0.0) {
    set_last_error("%s: kappa must be finite and positive", fn);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  McdPlan pl;
  if (int rc = mcd_plan(fn, x_offsets, y_offsets, n_pairs, n_ceps, kPath, &pl)) return rc;
  return mcd_dtw_launch<kPath>(fn, pl, x_offsets, y_offsets, n_pairs, n_ceps, kappa, workspace, workspace_bytes, cost_out, path_len_out,
                               path_out, stream_v, [&](double* ceps, int grid, cudaStream_t stream) {
                                 mcd_cepstra_kernel<<<grid, 256, 0, stream>>>(x, pl.fx, y, pl.frames, n_mels, dct, n_ceps, ceps);
                                 count_launch();
                                 return check_cuda(cudaGetLastError(), "mcd_cepstra_kernel");
                               });
}

template <bool kPath>
static int mcd_dtw_ceps_run(const char* fn, const double* x, const int32_t* x_offsets, const double* y, const int32_t* y_offsets,
                            int n_pairs, int ld, int first, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes,
                            double* cost_out, int32_t* path_len_out, int32_t* path_out, void* stream_v) {
  if (!x || !y || !workspace || !cost_out || !path_len_out || (kPath && !path_out)) {
    set_last_error("%s: NULL pointer", fn);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (n_ceps < 1 || first < 0 || (int64_t)first + n_ceps > ld) {
    set_last_error("%s: need n_ceps >= 1, first >= 0 and first + n_ceps <= ld, got first %d, n_ceps %d, ld %d", fn, first, n_ceps, ld);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (!std::isfinite(kappa) || kappa <= 0.0) {
    set_last_error("%s: kappa must be finite and positive", fn);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  McdPlan pl;
  if (int rc = mcd_plan(fn, x_offsets, y_offsets, n_pairs, n_ceps, kPath, &pl)) return rc;
  return mcd_dtw_launch<kPath>(fn, pl, x_offsets, y_offsets, n_pairs, n_ceps, kappa, workspace, workspace_bytes, cost_out, path_len_out,
                               path_out, stream_v, [&](double* ceps, int grid, cudaStream_t stream) {
                                 mcd_ceps_copy_kernel<<<grid, 256, 0, stream>>>(x, pl.fx, y, pl.frames, ld, first, n_ceps, ceps);
                                 count_launch();
                                 return check_cuda(cudaGetLastError(), "mcd_ceps_copy_kernel");
                               });
}

}  // namespace ttsb

using namespace ttsb;

extern "C" int64_t ttsb_mcd_dtw_workspace_bytes(const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps) {
  McdPlan pl;
  if (mcd_plan("ttsb_mcd_dtw_workspace_bytes", x_offsets, y_offsets, n_pairs, n_ceps, false, &pl)) return -1;
  return pl.bytes;
}

extern "C" int ttsb_mcd_dtw(const float* x, const int32_t* x_offsets, const float* y, const int32_t* y_offsets, int n_pairs, int n_mels,
                            const double* dct, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes, double* cost_out,
                            int32_t* path_len_out, void* stream_v) {
  return mcd_dtw_run<false>("ttsb_mcd_dtw", x, x_offsets, y, y_offsets, n_pairs, n_mels, dct, n_ceps, kappa, workspace, workspace_bytes,
                            cost_out, path_len_out, nullptr, stream_v);
}

extern "C" int64_t ttsb_mcd_dtw_path_workspace_bytes(const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps) {
  McdPlan pl;
  if (mcd_plan("ttsb_mcd_dtw_path_workspace_bytes", x_offsets, y_offsets, n_pairs, n_ceps, true, &pl)) return -1;
  return pl.bytes;
}

extern "C" int ttsb_mcd_dtw_path(const float* x, const int32_t* x_offsets, const float* y, const int32_t* y_offsets, int n_pairs,
                                 int n_mels, const double* dct, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes,
                                 double* cost_out, int32_t* path_len_out, int32_t* path_out, void* stream_v) {
  return mcd_dtw_run<true>("ttsb_mcd_dtw_path", x, x_offsets, y, y_offsets, n_pairs, n_mels, dct, n_ceps, kappa, workspace,
                           workspace_bytes, cost_out, path_len_out, path_out, stream_v);
}

extern "C" int64_t ttsb_mcd_dtw_ceps_workspace_bytes(const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps) {
  McdPlan pl;
  if (mcd_plan("ttsb_mcd_dtw_ceps_workspace_bytes", x_offsets, y_offsets, n_pairs, n_ceps, false, &pl)) return -1;
  return pl.bytes;
}

extern "C" int ttsb_mcd_dtw_ceps(const double* x, const int32_t* x_offsets, const double* y, const int32_t* y_offsets, int n_pairs, int ld,
                                 int first, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes, double* cost_out,
                                 int32_t* path_len_out, void* stream_v) {
  return mcd_dtw_ceps_run<false>("ttsb_mcd_dtw_ceps", x, x_offsets, y, y_offsets, n_pairs, ld, first, n_ceps, kappa, workspace,
                                 workspace_bytes, cost_out, path_len_out, nullptr, stream_v);
}

extern "C" int64_t ttsb_mcd_dtw_ceps_path_workspace_bytes(const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps) {
  McdPlan pl;
  if (mcd_plan("ttsb_mcd_dtw_ceps_path_workspace_bytes", x_offsets, y_offsets, n_pairs, n_ceps, true, &pl)) return -1;
  return pl.bytes;
}

extern "C" int ttsb_mcd_dtw_ceps_path(const double* x, const int32_t* x_offsets, const double* y, const int32_t* y_offsets, int n_pairs,
                                      int ld, int first, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes,
                                      double* cost_out, int32_t* path_len_out, int32_t* path_out, void* stream_v) {
  return mcd_dtw_ceps_run<true>("ttsb_mcd_dtw_ceps_path", x, x_offsets, y, y_offsets, n_pairs, ld, first, n_ceps, kappa, workspace,
                                workspace_bytes, cost_out, path_len_out, path_out, stream_v);
}
