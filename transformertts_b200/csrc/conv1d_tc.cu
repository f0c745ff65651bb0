// Ragged-batch Conv1D on the pipeline of gemm_pipeline.cuh, for the MelGAN and HiFi-GAN generators: dilated convs, the
// ResStack's shortcut + 1x1 conv as one two-source product, transposed convs phrased over their input rows, and the input
// convs.  Clips are packed channels-last with `halo` rows on each side (include/ttsb.h), so a tap is a row shift of a 2-D TMA
// load and a 128-row tile may span several clips.  The epilogue (one thread per row) maps the row to its clip, skips halo
// rows, adds the bias, an optional residual and the multi-receptive-field sum, writes y and LeakyReLU(y) as bf16 hi/lo planes
// and mirrors the rows next to each clip edge into the halos the next conv reads.  ttsb_conv1d_ex_tc takes the halo (up to 64
// rows), up to 16 taps and the slope per call; ttsb_conv1d_out_tanh_ex (ttsb_conv1d_out_clamp_ex for BigVGAN v2) is the
// generators' N = 1 output layer, and ttsb_snake_aa_ex BigVGAN's anti-aliased Snake activation on the same layout.
#include <vector>

#include "../../include/ttsb.h"
#include "gemm_pipeline.cuh"

namespace ttsb {

struct ConvKParams {
  int rows;  // GEMM rows: every row of the packed input layout, halos included
  int N, block_n, n_tiles, num_tiles;
  int num_taps;
  int tap_src[TTSB_CONV1D_EX_MAX_TAPS], tap_shift[TTSB_CONV1D_EX_MAX_TAPS];
  int kblocks[2];
  int n_clips;
  const int32_t* tab;  // device: region start rows [n_clips + 1], then the clip_offsets prefix sums [n_clips + 1]
  int up, halo_mode, ld_out;
  int halo;
  float slope;
  const float* bias;
  const __nv_bfloat16* res_hi;  // residual planes, output layout
  const __nv_bfloat16* res_lo;
  float* sum;                   // fp32 multi-receptive-field sum, output layout
  int sum_mode;
  float sum_div;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  __nv_bfloat16* act_hi;
  __nv_bfloat16* act_lo;
};

template <bool kSplit>
struct ConvCfg {
  using Stage = KMajorStage<kSplit, B_TILE_BYTES>;
  using Ring = typename Stage::Ring;
  static constexpr int kPitch = acc_pitch(GEMM_MAX_BN);
  static_assert(img_bytes(GEMM_MAX_BN) <= Ring::kBytes, "image must fit the ring");
  static constexpr int kSmemBytes = Ring::kBytes + GEMM_RING_BAR_BYTES + 1024;  // + alignment slack
};

// 16 columns of output row orow: y (and LeakyReLU(y)) as bf16 hi/lo, or zeros
__device__ __forceinline__ void conv_store16(const ConvKParams& p, size_t orow, int col, const float (&y)[16], bool zero, float slope) {
  const size_t o = orow * (size_t)p.ld_out + col;
  uint32_t h[8], l[8];
  float v[16];
  if (p.out_hi) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = zero ? 0.f : y[j];
    pack_hi_lo(v, h, l, p.out_lo != nullptr);
    st_global_v8(p.out_hi + o, h);
    if (p.out_lo) st_global_v8(p.out_lo + o, l);
  }
  if (p.act_hi) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = zero ? 0.f : (y[j] > 0.f ? y[j] : slope * y[j]);
    pack_hi_lo(v, h, l, p.act_lo != nullptr);
    st_global_v8(p.act_hi + o, h);
    if (p.act_lo) st_global_v8(p.act_lo + o, l);
  }
}

// residual (hi + lo) and multi-receptive-field sum steps on 16 columns of output row orow
__device__ __forceinline__ void conv_res_sum16(const ConvKParams& p, size_t orow, int col, float (&y)[16]) {
  const size_t o = orow * (size_t)p.ld_out + col;
  if (p.res_hi) {
    uint32_t h[8], l[8];
    ld_global_nc_v8(p.res_hi + o, h);
    if (p.res_lo) ld_global_nc_v8(p.res_lo + o, l);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float r0 = __uint_as_float(h[k] << 16), r1 = __uint_as_float(h[k] & 0xffff0000u);
      if (p.res_lo) { r0 += __uint_as_float(l[k] << 16); r1 += __uint_as_float(l[k] & 0xffff0000u); }
      y[2 * k] += r0;
      y[2 * k + 1] += r1;
    }
  }
  if (p.sum_mode == TTSB_CONV1D_SUM_WRITE) {
    st_global_v8f(p.sum + o, y);
    st_global_v8f(p.sum + o + 8, y + 8);
  } else if (p.sum_mode != TTSB_CONV1D_SUM_NONE) {  // torch's order: sum = sum + y; the last add is followed by / nk
    float s[16];
#pragma unroll
    for (int k = 0; k < 16; k += 4) *reinterpret_cast<float4*>(s + k) = *reinterpret_cast<const float4*>(p.sum + o + k);
#pragma unroll
    for (int k = 0; k < 16; ++k) s[k] += y[k];
    if (p.sum_mode == TTSB_CONV1D_SUM_ADD) {
      st_global_v8f(p.sum + o, s);
      st_global_v8f(p.sum + o + 8, s + 8);
    } else {
#pragma unroll
      for (int k = 0; k < 16; ++k) y[k] = s[k] / p.sum_div;
    }
  }
}

__device__ __forceinline__ void conv_epilogue(const ConvKParams& p, const float* arow, int g, int n0, int half) {
  if (g >= p.rows) return;
  const int H = p.halo;
  const float slope = p.slope;
  const int32_t* reg = p.tab;
  const int32_t* off = p.tab + p.n_clips + 1;
  const int c = find_clip(reg, p.n_clips, g);
  const int off_c = __ldg(off + c);
  const int L = __ldg(off + c + 1) - off_c;
  const int j = g - __ldg(reg + c) - H;
  if (j < 0 || j >= L) return;  // a halo row: written only by the mirror stores of the rows it copies
  const int Lo = L * p.up;
  const long long base = (long long)off_c * p.up + (long long)(2 * c + 1) * H;  // output row of clip position 0
  const int nch = p.block_n >> 4;
  const int ch_begin = half ? (nch + 1) >> 1 : 0;
  const int ch_end = half ? nch : (nch + 1) >> 1;
  uint32_t q[16];
  float y[16], bs[16];
  for (int ch = ch_begin; ch < ch_end; ++ch) {
    const int col = n0 + (ch << 4);
    acc_ld16(arow + (ch << 4), q);
#pragma unroll
    for (int k = 0; k < 16; ++k) y[k] = __uint_as_float(q[k]);
    if (p.bias) {
      ldg16(p.bias + col, bs);
#pragma unroll
      for (int k = 0; k < 16; ++k) y[k] += bs[k];
    }
    const int phase = col / p.ld_out, cc = col - phase * p.ld_out;
    const int pos = j * p.up + phase;  // position in the output clip
    conv_res_sum16(p, (size_t)(base + pos), cc, y);
    conv_store16(p, (size_t)(base + pos), cc, y, false, slope);
    if (p.halo_mode == TTSB_HALO_REFLECT) {
      if (pos >= 1 && pos <= H) conv_store16(p, (size_t)(base - pos), cc, y, false, slope);
      if (pos >= Lo - 1 - H && pos <= Lo - 2) conv_store16(p, (size_t)(base + 2 * (Lo - 1) - pos), cc, y, false, slope);
    } else if (p.halo_mode == TTSB_HALO_ZERO) {
      if (pos < H) conv_store16(p, (size_t)(base - 1 - pos), cc, y, true, slope);
      if (pos >= Lo - H) conv_store16(p, (size_t)(base + 2 * Lo - 1 - pos), cc, y, true, slope);
    }
  }
}

// tensor maps: A[src][hi/lo] (ld_in[src], rows) boxes (64, 128); W[hi/lo] (K_total, N) boxes (64, block_n).  kNch: block_n / 64
// (the wgmma width)
template <bool kSplit, int kNch>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
conv1d_tc_kernel(const __grid_constant__ CUtensorMap tmA0h, const __grid_constant__ CUtensorMap tmA0l,
                 const __grid_constant__ CUtensorMap tmA1h, const __grid_constant__ CUtensorMap tmA1l,
                 const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const ConvKParams p) {
  using Cfg = ConvCfg<kSplit>;
  static_assert(kNch >= 1 && kNch <= GEMM_NCH, "tile width");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  typename Cfg::Ring ring(smem);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA0h);
    tma_prefetch_desc(&tmWh);
    ring.init();
    fence_mbar_init();
  }
  __syncthreads();

  const uint32_t stage_tx = Cfg::Stage::tx_bytes(p.block_n);
  if (warp >= GEMM_EPI_WARPS) {
    setmaxnreg_dec<40>();
    if (warp > GEMM_EPI_WARPS) goto done;
    // ===================== TMA producer =====================
    const bool leader = elect_one();
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int m0 = (tile / p.n_tiles) * GEMM_BM;
      const int n0 = (tile % p.n_tiles) * p.block_n;
      ring.wait_image_free();
      int kglob = 0;
      for (int s = 0; s < p.num_taps; ++s) {
        const int src = p.tap_src[s];
        const CUtensorMap* mh = src == 0 ? &tmA0h : &tmA1h;
        const CUtensorMap* ml = src == 0 ? &tmA0l : &tmA1l;
        for (int kb = 0; kb < p.kblocks[src]; ++kb, ++kglob) {
          Cfg::Stage::produce(ring, leader, stage_tx, mh, ml, &tmWh, &tmWl, kglob, n0, [&](const CUtensorMap* m, uint64_t* bar, uint8_t* dst) {
            tma_load_2d(m, bar, dst, kb * GEMM_BK, m0 + p.tap_shift[s]);   // rows outside the buffer load as zeros
          });
        }
      }
    }
  } else {
    // ===================== two wgmma warpgroups, then the epilogue =====================
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int quarter = warp & 3;
    const int half = warp >> 2;
    float* img = reinterpret_cast<float*>(smem);
    int total_kb = 0;
    for (int s = 0; s < p.num_taps; ++s) total_kb += p.kblocks[p.tap_src[s]];
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int m0 = (tile / p.n_tiles) * GEMM_BM;
      const int n0 = (tile % p.n_tiles) * p.block_n;
      Cfg::Stage::template mma_park_tile<kNch>(ring, total_kb, img, Cfg::kPitch, wg);
      const int row = quarter * 32 + lane;
      __syncwarp();
      conv_epilogue(p, img + (size_t)row * Cfg::kPitch, m0 + row, n0, half);
      ring.release_tile(false);
    }
  }
done:
  __syncthreads();
}

// one thread per output sample: tanh(bias + 7-tap dot product over the padded channels), fixed summation order; the 3 rows of
// padding on each side are the clip's halo rows (reflected for MelGAN, zeros for HiFi-GAN).  kClamp: clamp(., -1, 1) instead of
// tanh (BigVGAN v2's output layer)
template <bool kClamp>
__global__ void __launch_bounds__(256)
conv1d_out_tanh_kernel(const __nv_bfloat16* __restrict__ in_hi, const __nv_bfloat16* __restrict__ in_lo, int ld_in, int channels, int halo,
                       const int32_t* __restrict__ tab, int n_clips, int drop_tail, const float* __restrict__ weight, float bias,
                       int total, float* __restrict__ wav_out) {
  extern __shared__ float sw[];  // (7, channels)
  for (int i = threadIdx.x; i < 7 * channels; i += blockDim.x) sw[i] = weight[i];
  __syncthreads();
  const int32_t* off = tab + n_clips + 1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = find_clip(off, n_clips, i);
    const int off_c = __ldg(off + c);
    const int j = i - off_c;
    if (j >= __ldg(off + c + 1) - off_c - drop_tail) continue;
    const size_t row = (size_t)__ldg(tab + c) + halo + j;
    float acc = bias;
    for (int k = 0; k < 7; ++k) {
      const __nv_bfloat16* h = in_hi + (row + k - 3) * (size_t)ld_in;
      const __nv_bfloat16* l = in_lo ? in_lo + (row + k - 3) * (size_t)ld_in : nullptr;
      for (int ch = 0; ch < channels; ++ch) {
        float x = __bfloat162float(h[ch]);
        if (l) x += __bfloat162float(l[ch]);
        acc = fmaf(x, sw[k * channels + ch], acc);
      }
    }
    wav_out[off_c - (size_t)c * drop_tail + j] = kClamp ? fminf(fmaxf(acc, -1.f), 1.f) : tanhf(acc);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// BigVGAN's anti-aliased periodic activation (Activation1d), per clip and channel, over the same ragged layout:
//   u[m] = 2 sum_i x[clamp(i - 5, 0, L - 1)] h_up[m + 15 - 2i]        m in [0, 2L), the six i with the tap in [0, 12)
//   s[m] = u[m] + inv_beta sin^2(alpha u[m])
//   y[t] = sum_j h_down[j] s[clamp(2t + j - 5, 0, 2L - 1)]             t in [0, L)
// A CTA takes SAA_ROWS rows of the packed layout (which may span clips) and 32 columns, one per lane.  It stages the input
// rows [r0 - 6, r0 + SAA_ROWS + 6) in shared memory as fp32, computes both phases of s for the rows [r0 - 3, r0 + SAA_ROWS
// + 3) and then the outputs; every index is clamped to the row's own clip, found in the uploaded clip table, so no clip
// reads another's rows or the halos.  Each value is computed by one thread in a fixed order: a clip's output does not
// depend on the tiling or the batch.
constexpr int SAA_ROWS = 64;
constexpr int SAA_THREADS = 256;
constexpr int SAA_XPAD = 6;  // s rows r0 - 3 .. need x rows 3 further out
constexpr int SAA_SPAD = 3;  // output row t reads s at positions 2t - 5 .. 2t + 6: rows t - 3 .. t + 3
constexpr int SAA_XROWS = SAA_ROWS + 2 * SAA_XPAD;
constexpr int SAA_SROWS = SAA_ROWS + 2 * SAA_SPAD;

struct SnakeAAParams {
  const __nv_bfloat16* in_hi;
  const __nv_bfloat16* in_lo;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  int ld, channels, halo, rows, n_clips;
  const int32_t* tab;  // region start rows [n_clips + 1], then the clip_offsets prefix sums [n_clips + 1]
  const float* alpha;
  const float* inv_beta;
  float h_up[12];
  float h_down[12];
};

__global__ void __launch_bounds__(SAA_THREADS)
snake_aa_kernel(const __grid_constant__ SnakeAAParams p) {
  __shared__ float xs[SAA_XROWS][32];
  __shared__ float ss[SAA_SROWS][2][32];
  __shared__ int2 meta[SAA_XROWS];  // per staged row: (row of its clip's position 0, L), L = 0 for a halo row or outside
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * SAA_ROWS;
  const int col = blockIdx.y * 32 + lane;
  const bool any_live = blockIdx.y * 32 < p.channels;  // CTA-uniform: all 32 columns are padding otherwise
  const bool live = col < p.channels;
  const int32_t* off = p.tab + p.n_clips + 1;
  for (int k = threadIdx.x; k < SAA_XROWS; k += SAA_THREADS) {
    const int g = r0 - SAA_XPAD + k;
    int2 m = make_int2(0, 0);
    if (g >= 0 && g < p.rows) {
      const int c = find_clip(p.tab, p.n_clips, g);
      const int base = __ldg(p.tab + c) + p.halo;
      const int L = __ldg(off + c + 1) - __ldg(off + c);
      if (g >= base && g < base + L) m = make_int2(base, L);
    }
    meta[k] = m;
  }
  __syncthreads();
  if (any_live) {
    for (int k = warp; k < SAA_XROWS; k += SAA_THREADS / 32) {
      float v = 0.f;
      if (live && meta[k].y) {
        const size_t o = (size_t)(r0 - SAA_XPAD + k) * p.ld + col;
        v = __bfloat162float(p.in_hi[o]);
        if (p.in_lo) v += __bfloat162float(p.in_lo[o]);
      }
      xs[k][lane] = v;
    }
    __syncthreads();
    const float a = live ? __ldg(p.alpha + col) : 0.f;
    const float ib = live ? __ldg(p.inv_beta + col) : 0.f;
    for (int k = warp; k < SAA_SROWS; k += SAA_THREADS / 32) {
      const int2 m = meta[k + SAA_XPAD - SAA_SPAD];
      if (!live || !m.y) continue;
      const int pos = r0 - SAA_SPAD + k - m.x;  // position in the clip
      const int xb = m.x - (r0 - SAA_XPAD);      // staged row of the clip's position 0
#pragma unroll
      for (int ph = 0; ph < 2; ++ph) {
        // m = 2 pos + ph: i = pos + 2 + ph + q (q = 0..5) reads x[pos - 3 + ph + q] with tap 11 - ph - 2q
        float acc = 0.f;
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const int i = min(max(pos - 3 + ph + q, 0), m.y - 1);
          acc = fmaf(xs[xb + i][lane], p.h_up[11 - ph - 2 * q], acc);
        }
        const float u = 2.f * acc;
        const float sn = sinf(a * u);
        ss[k][ph][lane] = fmaf(ib, sn * sn, u);
      }
    }
    __syncthreads();
  }
  if (col >= p.ld) return;
  for (int k = warp; k < SAA_ROWS; k += SAA_THREADS / 32) {
    const int2 m = meta[k + SAA_XPAD];
    if (!m.y) continue;  // a halo row (or past the end): never written
    float y = 0.f;
    if (live) {
      const int t = r0 + k - m.x;
      const int sb = m.x - (r0 - SAA_SPAD);  // s row of the clip's position 0
#pragma unroll
      for (int j = 0; j < 12; ++j) {
        const int mm = min(max(2 * t + j - 5, 0), 2 * m.y - 1);
        y = fmaf(p.h_down[j], ss[sb + (mm >> 1)][mm & 1][lane], y);
      }
    }
    const size_t o = (size_t)(r0 + k) * p.ld + col;
    const __nv_bfloat16 hi = __float2bfloat16_rn(y);
    p.out_hi[o] = hi;
    if (p.out_lo) p.out_lo[o] = __float2bfloat16_rn(y - __bfloat162float(hi));
  }
}

// checks the host offset table and fills tab (region starts, prefix sums); min_out_len: the least up * L_c; *rows: input
// rows, *out_rows: output rows of the layout; 0 on success
static int conv_table(const char* what, const int32_t* clip_offsets, int n_clips, int up, int halo, int min_out_len, std::vector<int32_t>& tab,
                      long long* rows, long long* out_rows) {
  if (!clip_offsets) { set_last_error("%s: clip_offsets is NULL", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (n_clips < 1) { set_last_error("%s: n_clips must be >= 1", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (clip_offsets[0] != 0) { set_last_error("%s: clip_offsets[0] must be 0", what); return TTSB_ERR_INVALID_ARGUMENT; }
  tab.assign(2 * (size_t)(n_clips + 1), 0);
  for (int c = 0; c < n_clips; ++c) {
    const long long L = (long long)clip_offsets[c + 1] - clip_offsets[c];
    if (L < 1) { set_last_error("%s: clip_offsets must be increasing (clip %d has %lld rows)", what, c, L); return TTSB_ERR_INVALID_ARGUMENT; }
    if (L * up < min_out_len) {
      set_last_error("%s: clip %d has %lld output rows; this halo mode needs at least %d", what, c, L * up, min_out_len);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
  }
  const long long total = (long long)clip_offsets[n_clips] * up + 2LL * halo * n_clips;
  if (total > INT32_MAX || (long long)clip_offsets[n_clips] + 2LL * halo * n_clips > INT32_MAX) {
    set_last_error("%s: too many rows", what);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  for (int c = 0; c <= n_clips; ++c) {
    tab[c] = clip_offsets[c] + 2 * halo * c;
    tab[n_clips + 1 + c] = clip_offsets[c];
  }
  *rows = (long long)clip_offsets[n_clips] + 2LL * halo * n_clips;
  *out_rows = total;
  return 0;
}

static int check_workspace(const char* what, const void* ws, int64_t bytes, int n_clips) {
  if (!ws || bytes < 2 * (int64_t)(n_clips + 1) * 4 || reinterpret_cast<uintptr_t>(ws) % 4) {
    set_last_error("%s: workspace missing, too small (ttsb_conv1d_workspace_bytes) or not 4-byte aligned", what);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  return 0;
}

// launches the instantiation whose wgmma width kNch * 64 is p.block_n
template <bool kSplit, int kNch = 1>
static int conv_launch_tc(const CUtensorMap (&tmA)[2][2], const CUtensorMap (&tmW)[2], const ConvKParams& p, cudaStream_t stream) {
  if constexpr (kNch < GEMM_NCH) {
    if (p.block_n > kNch * 64) return conv_launch_tc<kSplit, kNch + 1>(tmA, tmW, p, stream);
  }
  return launch_pipeline<conv1d_tc_kernel<kSplit, kNch>>(ConvCfg<kSplit>::kSmemBytes, p.num_tiles, false, stream, "conv1d_tc_kernel launch",
                                                         tmA[0][0], tmA[0][1], tmA[1][0], tmA[1][1], tmW[0], tmW[1], p);
}

// the host side of ttsb_conv1d_ex_tc: every refusal before any CUDA call
static int conv1d_launch(const char* what, const ttsb_conv1d_ex_args* a, void* stream_v) {
  if (a->precision != TTSB_PREC_BF16 && a->precision != TTSB_PREC_BF16X3) { set_last_error("%s: unknown precision", what); return TTSB_ERR_INVALID_ARGUMENT; }
  const bool split = a->precision == TTSB_PREC_BF16X3;
  const int H = a->halo;
  if (H < 0 || H > TTSB_CONV1D_EX_MAX_HALO) { set_last_error("%s: halo = %d must be in [0, %d]", what, H, TTSB_CONV1D_EX_MAX_HALO); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->num_taps < 1 || a->num_taps > TTSB_CONV1D_EX_MAX_TAPS) { set_last_error("%s: num_taps must be in [1, %d]", what, TTSB_CONV1D_EX_MAX_TAPS); return TTSB_ERR_INVALID_ARGUMENT; }
  int k_total = 0;
  for (int s = 0; s < a->num_taps; ++s) {
    const int src = a->tap_src[s];
    if (src < 0 || src > 1 || !a->in_hi[src] || (split && !a->in_lo[src])) {
      set_last_error("%s: tap %d reads source %d, which is missing (bf16x3 needs in_lo too)", what, s, src);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
    if (a->ld_in[src] < GEMM_BK || a->ld_in[src] % GEMM_BK) { set_last_error("%s: ld_in[%d] = %d must be a positive multiple of 64", what, src, a->ld_in[src]); return TTSB_ERR_INVALID_ARGUMENT; }
    if (a->tap_shift[s] < -H || a->tap_shift[s] > H) { set_last_error("%s: |tap_shift| must be <= %d (the halo)", what, H); return TTSB_ERR_INVALID_ARGUMENT; }
    k_total += a->ld_in[src];
  }
  if (!a->w_hi || (split && !a->w_lo)) { set_last_error("%s: missing packed weights", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->N < 64 || a->N % 64 || (a->N > GEMM_MAX_BN && a->N % GEMM_MAX_BN)) { set_last_error("%s: N = %d must be a multiple of 64, at most 256 or a multiple of 256", what, a->N); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->up < 1 || a->N % a->up || a->N / a->up != a->ld_out || a->ld_out % 16) { set_last_error("%s: need N = up * ld_out with ld_out a multiple of 16", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->halo_mode < TTSB_HALO_NONE || a->halo_mode > TTSB_HALO_ZERO) { set_last_error("%s: unknown halo_mode", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (!(a->slope == a->slope) || a->slope < 0.f || a->slope > 1.f) { set_last_error("%s: slope must be in [0, 1]", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->res_hi && split != (a->res_lo != nullptr)) { set_last_error("%s: the residual needs res_lo in bf16x3 and only there", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (!a->res_hi && a->res_lo) { set_last_error("%s: res_lo without res_hi", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->res_hi && (a->res_hi == a->out_hi || a->res_hi == a->act_hi)) { set_last_error("%s: the residual must not alias an output", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if ((reinterpret_cast<uintptr_t>(a->res_hi) | reinterpret_cast<uintptr_t>(a->res_lo) | reinterpret_cast<uintptr_t>(a->sum)) % 16) {
    set_last_error("%s: res_hi, res_lo and sum must be 16-byte aligned", what);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (a->sum_mode < TTSB_CONV1D_SUM_NONE || a->sum_mode > TTSB_CONV1D_SUM_FINISH) { set_last_error("%s: unknown sum_mode", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if ((a->sum_mode != TTSB_CONV1D_SUM_NONE) != (a->sum != nullptr)) { set_last_error("%s: sum must be given exactly when sum_mode is not NONE", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (a->sum_mode == TTSB_CONV1D_SUM_FINISH && !(a->sum_div >= 1.f && a->sum_div < 1e6f)) { set_last_error("%s: sum_div must be in [1, 1e6)", what); return TTSB_ERR_INVALID_ARGUMENT; }
  const bool stores = a->sum_mode == TTSB_CONV1D_SUM_WRITE || a->sum_mode == TTSB_CONV1D_SUM_ADD;
  if (!a->out_hi && !a->act_hi && !stores) { set_last_error("%s: no output", what); return TTSB_ERR_INVALID_ARGUMENT; }
  const int min_len = a->halo_mode == TTSB_HALO_REFLECT ? H + 1 : (a->halo_mode == TTSB_HALO_ZERO ? H : 1);
  std::vector<int32_t> tab;
  long long rows = 0, out_rows = 0;
  int rc = conv_table(what, a->clip_offsets, a->n_clips, a->up, H, min_len, tab, &rows, &out_rows);
  if (rc) return rc;
  if (a->out_rows != out_rows) {
    set_last_error("%s: out_rows = %lld, but the output layout of these clips has %lld rows (residual, sum and outputs all have that shape)",
                   what, (long long)a->out_rows, out_rows);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  rc = check_workspace(what, a->workspace, a->workspace_bytes, a->n_clips);
  if (rc) return rc;
  // last of the argument checks: the planes the epilogue writes (16-byte vector stores; in bf16 the lo planes are ignored)
  const void* outs[4] = {a->out_hi, split && a->out_hi ? a->out_lo : nullptr, a->act_hi, split && a->act_hi ? a->act_lo : nullptr};
  if ((reinterpret_cast<uintptr_t>(outs[0]) | reinterpret_cast<uintptr_t>(outs[1]) | reinterpret_cast<uintptr_t>(outs[2]) |
       reinterpret_cast<uintptr_t>(outs[3]) | reinterpret_cast<uintptr_t>(a->bias)) % 16) {
    set_last_error("%s: out_hi, out_lo, act_hi, act_lo and bias must be 16-byte aligned", what);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  for (const void* o : outs) {
    if (!o) continue;
    if (o == a->res_hi || o == a->res_lo) { set_last_error("%s: the residual must not alias an output", what); return TTSB_ERR_INVALID_ARGUMENT; }
    // other tiles' taps still read the rows this tile's epilogue and mirror stores write: a conv cannot run in place
    for (int s = 0; s < a->num_taps; ++s) {
      const int src = a->tap_src[s];
      if (o == a->in_hi[src] || (split && o == a->in_lo[src])) {
        set_last_error("%s: an output plane aliases an input plane of source %d (no in-place conv)", what, src);
        return TTSB_ERR_INVALID_ARGUMENT;
      }
    }
  }

  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  ConvKParams p{};
  p.rows = (int)rows;
  p.N = a->N;
  p.block_n = a->N < GEMM_MAX_BN ? a->N : GEMM_MAX_BN;
  p.n_tiles = a->N / p.block_n;
  p.num_tiles = (int)((rows + GEMM_BM - 1) / GEMM_BM) * p.n_tiles;
  p.num_taps = a->num_taps;
  for (int s = 0; s < a->num_taps; ++s) { p.tap_src[s] = a->tap_src[s]; p.tap_shift[s] = a->tap_shift[s]; }
  for (int i = 0; i < 2; ++i) p.kblocks[i] = a->in_hi[i] ? a->ld_in[i] / GEMM_BK : 0;
  p.n_clips = a->n_clips;
  p.tab = static_cast<const int32_t*>(a->workspace);
  p.up = a->up;
  p.halo_mode = a->halo_mode;
  p.ld_out = a->ld_out;
  p.halo = H;
  p.slope = a->slope;
  p.bias = a->bias;
  p.res_hi = static_cast<const __nv_bfloat16*>(a->res_hi);
  p.res_lo = static_cast<const __nv_bfloat16*>(a->res_lo);
  p.sum = a->sum;
  p.sum_mode = a->sum_mode;
  p.sum_div = a->sum_div;
  p.out_hi = static_cast<__nv_bfloat16*>(a->out_hi);
  p.out_lo = split && a->out_hi ? static_cast<__nv_bfloat16*>(a->out_lo) : nullptr;
  p.act_hi = static_cast<__nv_bfloat16*>(a->act_hi);
  p.act_lo = split && a->act_hi ? static_cast<__nv_bfloat16*>(a->act_lo) : nullptr;

  CUtensorMap tmA[2][2], tmW[2];
  for (int i = 0; i < 2; ++i) {
    const int use = a->in_hi[i] ? i : (a->in_hi[0] ? 0 : 1);  // an unused slot aliases the other source
    for (int h = 0; h < 2; ++h) {
      const void* base = (h == 1 && split) ? a->in_lo[use] : a->in_hi[use];
      rc = make_tmap_bf16_2d(&tmA[i][h], base, (uint64_t)a->ld_in[use], (uint64_t)rows, (uint64_t)a->ld_in[use], GEMM_BK, GEMM_BM);
      if (rc) return rc;
    }
  }
  for (int h = 0; h < 2; ++h) {
    rc = make_tmap_bf16_2d(&tmW[h], (h == 1 && split) ? a->w_lo : a->w_hi, (uint64_t)k_total, (uint64_t)a->N, (uint64_t)k_total, GEMM_BK, p.block_n);
    if (rc) return rc;
  }
  TTSB_CUDA_OK(cudaMemcpyAsync(a->workspace, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  return split ? conv_launch_tc<true>(tmA, tmW, p, stream) : conv_launch_tc<false>(tmA, tmW, p, stream);
}

template <bool kClamp>
static int out_tanh_launch(const char* what, const void* in_hi, const void* in_lo, int ld_in, int channels, int halo,
                           const int32_t* clip_offsets, int n_clips, int drop_tail, const float* weight, float bias, void* workspace,
                           int64_t workspace_bytes, float* wav_out, void* stream_v) {
  if (!in_hi || !weight || !wav_out) { set_last_error("%s: NULL pointer", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (channels < 1 || ld_in < channels || ld_in > 256 || ld_in % 8) { set_last_error("%s: need 1 <= channels <= ld_in <= 256, ld_in %% 8 == 0", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (drop_tail < 0) { set_last_error("%s: drop_tail < 0", what); return TTSB_ERR_INVALID_ARGUMENT; }
  std::vector<int32_t> tab;
  long long rows = 0, out_rows = 0;
  // the 3-row padding lies in the halos, so any clip that outlasts drop_tail works
  int rc = conv_table(what, clip_offsets, n_clips, 1, halo, drop_tail + 1, tab, &rows, &out_rows);
  if (rc) return rc;
  rc = check_workspace(what, workspace, workspace_bytes, n_clips);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  TTSB_CUDA_OK(cudaMemcpyAsync(workspace, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  const int total = clip_offsets[n_clips];
  const int grid = min((total + 255) / 256, 8 * num_sms());
  conv1d_out_tanh_kernel<kClamp><<<grid, 256, 7 * channels * sizeof(float), stream>>>(
      static_cast<const __nv_bfloat16*>(in_hi), static_cast<const __nv_bfloat16*>(in_lo), ld_in, channels, halo,
      static_cast<const int32_t*>(workspace), n_clips, drop_tail, weight, bias, total, wav_out);
  count_launch();
  return check_cuda(cudaGetLastError(), "conv1d_out_tanh_kernel launch");
}

static int snake_aa_launch(const void* in_hi, const void* in_lo, void* out_hi, void* out_lo, int ld, int channels, int halo,
                           const int32_t* clip_offsets, int n_clips, const float* alpha, const float* inv_beta, const float* h_up,
                           const float* h_down, int precision, void* workspace, int64_t workspace_bytes, void* stream_v) {
  const char* what = "ttsb_snake_aa_ex";
  if (precision != TTSB_PREC_BF16 && precision != TTSB_PREC_BF16X3) { set_last_error("%s: unknown precision", what); return TTSB_ERR_INVALID_ARGUMENT; }
  const bool split = precision == TTSB_PREC_BF16X3;
  if (!in_hi || !out_hi || (split && (!in_lo || !out_lo))) {
    set_last_error("%s: in_hi or out_hi is NULL, or in_lo or out_lo in bf16x3", what);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  if (!alpha || !inv_beta || !h_up || !h_down) { set_last_error("%s: alpha, inv_beta, h_up or h_down is NULL", what); return TTSB_ERR_INVALID_ARGUMENT; }
  if (ld < 8 || ld % 8) { set_last_error("%s: ld = %d must be a positive multiple of 8", what, ld); return TTSB_ERR_INVALID_ARGUMENT; }
  if (channels < 1 || channels > ld) { set_last_error("%s: channels = %d must be in [1, ld = %d]", what, channels, ld); return TTSB_ERR_INVALID_ARGUMENT; }
  if (halo < 0 || halo > TTSB_CONV1D_EX_MAX_HALO) { set_last_error("%s: halo = %d must be in [0, %d]", what, halo, TTSB_CONV1D_EX_MAX_HALO); return TTSB_ERR_INVALID_ARGUMENT; }
  const void* planes[4] = {in_hi, split ? in_lo : nullptr, out_hi, split ? out_lo : nullptr};
  if ((reinterpret_cast<uintptr_t>(planes[0]) | reinterpret_cast<uintptr_t>(planes[1]) | reinterpret_cast<uintptr_t>(planes[2]) |
       reinterpret_cast<uintptr_t>(planes[3])) % 16 || (reinterpret_cast<uintptr_t>(alpha) | reinterpret_cast<uintptr_t>(inv_beta)) % 4) {
    set_last_error("%s: in_hi, in_lo, out_hi and out_lo must be 16-byte aligned, alpha and inv_beta 4-byte aligned", what);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  for (int o = 2; o < 4; ++o)
    if (planes[o] && (planes[o] == planes[0] || planes[o] == planes[1] || (o == 3 && planes[3] == planes[2]))) {
      set_last_error("%s: an output plane aliases an input plane or the other output plane (no in-place activation)", what);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
  std::vector<int32_t> tab;
  long long rows = 0, out_rows = 0;
  int rc = conv_table(what, clip_offsets, n_clips, 1, halo, 1, tab, &rows, &out_rows);
  if (rc) return rc;
  rc = check_workspace(what, workspace, workspace_bytes, n_clips);
  if (rc) return rc;

  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  SnakeAAParams p{};
  p.in_hi = static_cast<const __nv_bfloat16*>(in_hi);
  p.in_lo = split ? static_cast<const __nv_bfloat16*>(in_lo) : nullptr;
  p.out_hi = static_cast<__nv_bfloat16*>(out_hi);
  p.out_lo = split ? static_cast<__nv_bfloat16*>(out_lo) : nullptr;
  p.ld = ld;
  p.channels = channels;
  p.halo = halo;
  p.rows = (int)rows;
  p.n_clips = n_clips;
  p.tab = static_cast<const int32_t*>(workspace);
  p.alpha = alpha;
  p.inv_beta = inv_beta;
  for (int j = 0; j < 12; ++j) { p.h_up[j] = h_up[j]; p.h_down[j] = h_down[j]; }
  TTSB_CUDA_OK(cudaMemcpyAsync(workspace, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  const dim3 grid((unsigned)((rows + SAA_ROWS - 1) / SAA_ROWS), (unsigned)((ld + 31) / 32));
  snake_aa_kernel<<<grid, SAA_THREADS, 0, stream>>>(p);
  count_launch();
  return check_cuda(cudaGetLastError(), "snake_aa_kernel launch");
}

}  // namespace ttsb

using namespace ttsb;

extern "C" int64_t ttsb_conv1d_workspace_bytes(int n_clips) {
  if (n_clips < 1) {
    set_last_error("ttsb_conv1d_workspace_bytes: n_clips < 1");
    return -1;
  }
  return 2 * (int64_t)(n_clips + 1) * (int64_t)sizeof(int32_t);
}

extern "C" int ttsb_conv1d_ex_tc(const ttsb_conv1d_ex_args* a, void* stream_v) {
  if (!a) { set_last_error("ttsb_conv1d_ex_tc: args is NULL"); return TTSB_ERR_INVALID_ARGUMENT; }
  return conv1d_launch("ttsb_conv1d_ex_tc", a, stream_v);
}

extern "C" int ttsb_conv1d_out_tanh_ex(const void* in_hi, const void* in_lo, int ld_in, int channels, int halo, const int32_t* clip_offsets,
                                       int n_clips, int drop_tail, const float* weight, float bias, void* workspace, int64_t workspace_bytes,
                                       float* wav_out, void* stream_v) {
  if (halo < 3 || halo > TTSB_CONV1D_EX_MAX_HALO) {
    set_last_error("ttsb_conv1d_out_tanh_ex: halo = %d must be in [3, %d]", halo, TTSB_CONV1D_EX_MAX_HALO);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  return out_tanh_launch<false>("ttsb_conv1d_out_tanh_ex", in_hi, in_lo, ld_in, channels, halo, clip_offsets, n_clips, drop_tail, weight,
                                bias, workspace, workspace_bytes, wav_out, stream_v);
}

extern "C" int ttsb_conv1d_out_clamp_ex(const void* in_hi, const void* in_lo, int ld_in, int channels, int halo, const int32_t* clip_offsets,
                                        int n_clips, int drop_tail, const float* weight, float bias, void* workspace, int64_t workspace_bytes,
                                        float* wav_out, void* stream_v) {
  if (halo < 3 || halo > TTSB_CONV1D_EX_MAX_HALO) {
    set_last_error("ttsb_conv1d_out_clamp_ex: halo = %d must be in [3, %d]", halo, TTSB_CONV1D_EX_MAX_HALO);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  return out_tanh_launch<true>("ttsb_conv1d_out_clamp_ex", in_hi, in_lo, ld_in, channels, halo, clip_offsets, n_clips, drop_tail, weight,
                               bias, workspace, workspace_bytes, wav_out, stream_v);
}

extern "C" int ttsb_snake_aa_ex(const void* in_hi, const void* in_lo, void* out_hi, void* out_lo, int ld, int channels, int halo,
                                const int32_t* clip_offsets, int n_clips, const float* alpha, const float* inv_beta, const float* h_up,
                                const float* h_down, int precision, void* workspace, int64_t workspace_bytes, void* stream_v) {
  return snake_aa_launch(in_hi, in_lo, out_hi, out_lo, ld, channels, halo, clip_offsets, n_clips, alpha, inv_beta, h_up, h_down, precision,
                         workspace, workspace_bytes, stream_v);
}
