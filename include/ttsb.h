/*
 * ttsb.h -- C ABI of libttsb.so, the H100 (sm_90a) kernels behind the ForwardTransformer text->mel hot path
 * of as-ideas/TransformerTTS.
 *
 * The reference has no FFI/plugin interface: its boundary is the Python API (model/models.py:344-642,
 * data/audio.py:88-92).  The host-side mirror of that API lives in transformertts_b200/ and binds these entry
 * points with ctypes (transformertts_b200/lib.py); INTEGRATION.md shows the stub a maintainer of the reference
 * would add.  Each entry point names the reference lines it replaces.
 *
 * Conventions
 *   - every function returns 0 on success, a negative TTSB_ERR_* otherwise; ttsb_last_error() gives the text
 *     (thread-local);
 *   - all pointers are CALLER-OWNED DEVICE pointers unless the name ends in _host; nothing is allocated inside;
 *   - `stream` is a cudaStream_t passed as void*; all work is stream-ordered, no hidden synchronisation;
 *   - activations are row-major (B, T, C) channels-last as in Keras; "hi/lo" pairs are the bf16 split of an fp32
 *     tensor (x ~= hi + lo) used by the 3-pass bf16 tensor-core mode; lo pointers may be NULL in single-pass mode;
 *   - packed weights are bf16 [N_pad, K] (K contiguous), produced from the Keras (K, N) / (k, Cin, Cout) layout by
 *     ttsb_pack_weight.
 */
#ifndef TTSB_H_
#define TTSB_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TTSB_OK 0
#define TTSB_ERR_INVALID_ARGUMENT (-1)
#define TTSB_ERR_CUDA (-2)
#define TTSB_ERR_UNSUPPORTED (-3)

#define TTSB_ABI_VERSION 5

/* precision of the tensor-core products */
#define TTSB_PREC_BF16 0   /* single bf16 pass, fp32 accumulate */
#define TTSB_PREC_BF16X3 1 /* hi*hi + lo*hi + hi*lo, fp32 accumulate (fp32-class accuracy) */
#define TTSB_PREC_FP16 2   /* ttsb_mha_fwd only: single IEEE fp16 pass (11-bit mantissa), q/k/vT hold fp16 */

/* implementation selector (debug): the tensor-core (wgmma/TMA) kernels -- TTSB_IMPL named "tcgen05" for API stability -- or the plain SIMT CUDA kernels kept for bring-up */
#define TTSB_IMPL_TCGEN05 0
#define TTSB_IMPL_SIMT 1

const char* ttsb_last_error(void);
int ttsb_abi_version(void);
/* number of kernels this library has launched since load / since the last reset (bench.py "gpu_launches") */
int64_t ttsb_launch_count(void);
void ttsb_reset_launch_count(void);
/* a host that replays a captured CUDA graph of N library launches adds N per replay, so the counter keeps meaning
 * "kernels of this library that ran" */
void ttsb_add_launch_count(int64_t n);

/* Dropout decisions are a stateless hash of (seed, site, element index); `seed` is a by-value argument of every kernel that
 * draws them.  The 32-bit word *salt_dev (DEVICE memory) is XORed into that seed by all kernels launched afterwards on the
 * stream (stream-ordered device-to-device copies into the library's constant memory; 0 after load).  A host that replays a
 * captured training step puts this call at the head of the capture and rewrites *salt_dev before every replay, which gives
 * each step its own masks although the captured `seed` arguments never change. */
int ttsb_set_dropout_salt(const uint32_t* salt_dev, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Weight / activation preparation
 * ------------------------------------------------------------------------------------------------------- */
/* Keras kernel (K, N) fp32 (Conv1D (k, Cin, Cout) is the same memory with K = k*Cin) -> packed bf16 hi/lo
 * [n_pad, K], rows >= N zero.  w_lo may be NULL. */
int ttsb_pack_weight(const float* w_kn, int K, int N, int n_pad, void* w_hi, void* w_lo, void* stream);
/* Batched refresh of packed operands (training: the weights change every step).  One descriptor per destination block:
 *   dst[r][c] = (r < R && c % cb < cb_valid) ? src[r*sr + (c / cb)*s_outer + (c % cb)*s_inner] : 0,   r < R_pad, c < C_cols
 * which covers the forward packing (K,N)->[N_pad,K], the data-gradient packings of Dense ((K,N)->[K_pad,N_pad]) and Conv1D
 * ((k,Cin,Cout)->[Cin_pad, k*Cout_pad]) and zero-padded fp32 vectors (bias, LayerNorm gamma/beta).  The descriptor array
 * lives in DEVICE memory (built once); one launch refreshes everything. */
typedef struct ttsb_pack_desc {
  const float* src;
  void* dst;
  int R, R_pad, C_cols;
  int cb, cb_valid;
  long long sr, s_outer, s_inner;
  int dst_ld;
  int dst_f32; /* 1: destination is fp32, 0: bf16 */
} ttsb_pack_desc;
int ttsb_repack_batched(const ttsb_pack_desc* descs_device, int n, void* stream);
/* fp32 [n] -> bf16 hi (and lo when non-NULL) */
int ttsb_split_bf16(const float* x, int64_t n, void* x_hi, void* x_lo, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Encoder prologue: Embedding + LayerNorm + scalar*PE   (model/models.py:522, model/layers.py:299-300)
 * tokens int32 (B,T); emb (vocab,d); pe (max_pos,d) fp32; pos_scalar device scalar.
 * ------------------------------------------------------------------------------------------------------- */
int ttsb_embed_ln_pe_fwd(const int32_t* tokens, const float* emb, const float* gamma, const float* beta,
                         const float* pe, const float* pos_scalar, int B, int T, int d, int vocab, float eps,
                         float* out_f32, void* out_hi, void* out_lo, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Tensor-core GEMM family:  Dense, dual-input Dense (concat projection) and Conv1D(k, 'same')
 *   (model/layers.py:134-136,149 MHA projections; :93-94 FFN; :19-26 Conv1D; model/models.py:422 mel Dense)
 *
 *   out[b,t,:] = epilogue( bias + sum_s  A_{src[s]}[b, t + shift[s], :] @ W[koff_s : koff_s + K_s, :] )
 *
 * Segments: a Dense has one segment (shift 0); the concat projection has two sources; a k-tap 'same' conv has k
 * segments over the same source with shifts -(k-1)/2 ... ; rows outside [0,T) read as zero.
 * Epilogue (in this order): +bias, relu?, +residual?, LayerNorm over the first ln_n columns?, zero rows t >= row_len[b]?.
 * ------------------------------------------------------------------------------------------------------- */
typedef struct ttsb_gemm_args {
  int B, T;                 /* rows = B*T */
  int N;                    /* logical output columns */
  int block_n;              /* N tile (multiple of 16, <= 256); packed W has n_tiles*block_n rows */
  int num_segments;         /* 1..4 */
  int seg_src[4];           /* 0 or 1: which A source */
  int seg_shift[4];         /* time shift of the source rows */
  int seg_k[4];             /* K of the segment (multiple of 64) */
  const void* a_hi[2];      /* bf16 (B,T,lda) sources */
  const void* a_lo[2];      /* NULL in TTSB_PREC_BF16 */
  int lda[2];               /* row stride in elements */
  int a_col0[2];            /* first column of the source inside its row */
  const void* w_hi;         /* packed bf16 [n_tiles*block_n, K_total] */
  const void* w_lo;
  const float* bias;        /* [n_tiles*block_n] (zero padded past N) or NULL */
  int relu;
  const float* residual;    /* fp32 (B,T,ld_res) or NULL */
  int ld_res;
  const float* ln_gamma;    /* LayerNorm params [block_n] (padded) or NULL */
  const float* ln_beta;
  float ln_eps;
  const int32_t* row_len;   /* [B] valid lengths or NULL */
  float* out_f32;           /* any of the three may be NULL */
  void* out_hi;
  void* out_lo;
  int ld_out;               /* row stride of all outputs, >= n_tiles*block_n, multiple of 8 (16 with 16-bit outputs) */
  int out_fp16;             /* 1: out_hi receives IEEE fp16 (single plane) instead of bf16 hi/lo */
  float* out_preln;         /* optional fp32 (B,T,ld_out): value before the LayerNorm (saved for the backward pass) */
  /* training dropout (keras semantics, stateless mask from (seed, site, element index)): drop_pre on the GEMM output
   * after bias/ReLU and before the residual add; drop_post on the LayerNorm output */
  float drop_pre_p, drop_post_p;
  uint32_t drop_pre_site, drop_post_site, drop_seed;
  int precision;            /* TTSB_PREC_* */
  int impl;                 /* TTSB_IMPL_* */
  /* residual given as a bf16 hi/lo pair instead of fp32 (residual == NULL): value = hi + lo, row stride ld_res.  In
   * bf16x3 inference the activation pair IS the residual stream (16 mantissa bits), so the LayerNorm GEMMs neither write
   * nor re-read an fp32 copy of every activation (LayerNorm epilogue only). */
  const void* residual_hi;
  const void* residual_lo;
} ttsb_gemm_args;

int ttsb_linear_fwd(const ttsb_gemm_args* args, void* stream);

/* Stand-alone LayerNorm (+ row mask) over rows of fp32 x (B,T,ld)[:, :, :d]  (model/layers.py:27,96,207: epsilon 1e-6).
 * Used when a row is wider than one 256-column accumulator tile (model dimension 384): the GEMM then writes the
 * pre-norm value and this kernel produces the fp32 + bf16 hi/lo activation triple. */
int ttsb_layernorm_fwd(const float* x, const float* gamma, const float* beta, int B, int T, int d, int ld, float eps,
                       const int32_t* row_len, float* out_f32, void* out_hi, void* out_lo, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused variable-length attention  (model/layers.py:138-147 split/merge heads, :176-195 scaled dot product)
 *   self-attention (kv_hi == NULL): q,k,v are columns q_col0 + h*dh / k_col0 + h*dh / v_col0 + h*dh of ONE buffer
 *     (B,T,ld_qk), the QKV GEMM output; Tk = T.
 *   cross-attention (kv_hi != NULL; model/layers.py:315-327 CrossAttentionResnorm): q from (B,T,ld_qk) at q_col0,
 *     k and v from a second buffer (B,Tk,ld_kv) at k_col0 / v_col0 (the K|V GEMM of the encoder output).
 *   out: bf16 hi (and lo when out_lo != NULL) (B,T,ld_out), head h at columns h*dh.
 *   The H*dh columns from each column offset (>= 0) must lie inside their row (ld_qk, ld_kv, ld_out); a call that breaks
 *   this, or names a weights_batch_index outside [0, B), returns TTSB_ERR_INVALID_ARGUMENT and writes nothing.
 *   Masking follows the reference's additive -1e9 masks: keys t >= kv_len[b] (padding mask, transformer_utils.py:24-32)
 *   and, with causal = 1, keys t > query index (look-ahead mask, transformer_utils.py:35-37; the Aligner passes
 *   max(padding, look-ahead), models.py:136-138).
 *   full_queries = 0: query rows >= kv_len[b] are written as zeros (ForwardTransformer blocks multiply them by the
 *   mask right after, layers.py:228-230); 1: every query row is computed from the unmasked keys as the reference does
 *   (Aligner decoder blocks never re-mask their rows).
 *   precision TTSB_PREC_FP16: the buffers hold IEEE fp16 (written by ttsb_linear_fwd with out_fp16 = 1), one
 *   tensor-core pass.  Head dims 64, 128 (all precisions), 192, 256 (single-pass precisions).
 * ------------------------------------------------------------------------------------------------------- */
typedef struct ttsb_mha_args {
  int B, T, H, dh;
  const void* qk_hi;
  const void* qk_lo;
  int ld_qk, q_col0, k_col0, v_col0;
  const int32_t* kv_len; /* [B] */
  void* out_hi;
  void* out_lo;
  int ld_out;
  /* optional: materialised softmax weights, reference-exact fp32 (logits + mask * -1e9, softmax).
   * weights_all = 0: ONE batch row, (H,T,Tk) (the ForwardTransformer's callers read item 0 only);
   * weights_all = 1: every row, (B,H,T,Tk) (the Aligner's cross-attention is a model output, models.py:150-153) */
  float* weights_out;
  int weights_batch_index;
  int precision;
  int impl;
  /* ---- ABI 2 ---- */
  const void* kv_hi;     /* NULL: self-attention */
  const void* kv_lo;
  int ld_kv, Tk;
  int causal;
  int full_queries;
  int weights_all;
} ttsb_mha_args;

int ttsb_mha_fwd(const ttsb_mha_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Cached autoregressive decoding of the Aligner  (model/models.py:271-292 Aligner.predict, a batch of sentences at a time)
 *   The decoder is causal, so one iteration computes ONE new decoder row per sentence: each self-attention block keeps the
 *   keys / values of the rows already decoded in a cache, and every position lives in device memory (pos[b] = index of the
 *   row being decoded), so one captured step replays for every iteration.
 *
 * ttsb_decode_attn: one query row per (sentence b, head h); logits scaled by 1/sqrt(dh), fp32 softmax, as ttsb_mha_fwd.
 *   q: 16-bit (B, ld_q), head h at columns q_col0 + h*dh.
 *   self mode (new_kv != NULL): the new row's key and value (new_kv (B, ld_new), head h at new_k_col0 / new_v_col0 + h*dh: the
 *     QKV GEMM output) are copied bit for bit into the cache kv (B, Tk, ld_kv) at row pos[b] (columns k_col0 / v_col0 + h*dh),
 *     and the query attends over keys 0..pos[b] (look-ahead mask); kv_len is not read.  pos[b] < Tk.
 *   cross mode (new_kv == NULL): attends over the keys < kv_len[b] (padding mask, kv_len[b] >= 1) of kv, which is not written.
 *   Masked keys get probability exactly 0, as the reference's additive -1e9 mask gives after the fp32 softmax.
 *   out: bf16 hi (and lo when non-NULL) (B, ld_out), head h at columns h*dh: the attention operand of the concat projection.
 *   probs (optional): the fp32 probability row of (b, h), written at (b, h, pos[b], :) of a (B, H, probs_T, Tk) buffer.
 *   done (optional, [B]): rows with done[b] != 0 are skipped; nothing is read or written for them.
 *   precision: TTSB_PREC_FP16 (q / kv hold IEEE fp16) or TTSB_PREC_BF16.  dh in {64, 128, 256}; leading dimensions and
 *   column offsets are multiples of 8 (16-byte loads).
 *   Keys are split across the warps of a CTA and, when B*H is small against the SM count, across CTAs sized for Tk; the CTAs
 *   whose range holds keys at the row's current length park partial results, and the last of them to finish combines them in
 *   a fixed order (deterministic).  workspace: at least ttsb_decode_attn_workspace_bytes(B, H, dh) bytes of device memory.
 *   It starts with B*H counter words, which must be zero before the first call and which every call leaves at zero; the
 *   partial results follow at an offset that depends on B*H and keep whatever the last call wrote there.  So calls may share
 *   one workspace (stream-ordered) only when they have the same B and H; calls with another B or H need their own.
 * ttsb_decode_prologue: the decoder prologue (model/layers.py:406-410) for one row per sentence at a device-side position:
 *   out[b] = LayerNorm(x[b]) + pos_scalar * pe[pos[b]]  (x fp32 (B, d); pe (pe_rows, d) is the table whose row t is position
 *   t*r; positions are clamped to [0, pe_rows)); writes the fp32 + bf16 hi/lo triple (B, d).  d % 4 == 0, d <= 512.
 * ttsb_decode_commit: the end of one iteration (model/models.py:280-289), one CTA, for every row b with done[b] == 0:
 *   post fp32 (B*r, ld_post) is the step's postnet output (frame j of row b at row b*r + j; mel in columns [0, mel), the
 *   three stop logits from column stop_col);
 *   mel_out[b, pos[b]*r + j, :] = frame j  (mel_out fp32 (B, max_iters*r, mel)); stop_out (optional, fp32 (B, max_iters*r, 3))
 *   the same for the stop logits;
 *   next_hi / next_lo (B, ld_next) bf16, columns [0, mel) = frame r-1 split into hi/lo: the next input (next_lo may be NULL);
 *   n[b] = pos[b] + 1; done[b] = 1 when the first arg-max of the last stop row is stop_index or n[b] == max_iters, else
 *   pos[b] += 1;  *all_done = 1 when every row is done, else 0.
 * ------------------------------------------------------------------------------------------------------- */
typedef struct ttsb_decode_attn_args {
  int B, H, dh;
  const void* q;
  int ld_q, q_col0;
  void* kv;
  int ld_kv, Tk, k_col0, v_col0;
  const void* new_kv;         /* NULL: cross mode */
  int ld_new, new_k_col0, new_v_col0;
  const int32_t* pos;         /* [B] */
  const int32_t* kv_len;      /* [B], cross mode */
  const int32_t* done;        /* [B] or NULL */
  void* out_hi;
  void* out_lo;
  int ld_out;
  float* probs;               /* or NULL */
  int probs_T;
  int precision;
  void* workspace;
  int64_t workspace_bytes;
} ttsb_decode_attn_args;

int64_t ttsb_decode_attn_workspace_bytes(int B, int H, int dh);
int ttsb_decode_attn(const ttsb_decode_attn_args* args, void* stream);
int ttsb_decode_prologue(const float* x, const int32_t* pos, const float* gamma, const float* beta, const float* pe, int pe_rows,
                         const float* pos_scalar, int B, int d, float eps, float* out_f32, void* out_hi, void* out_lo,
                         void* stream);
int ttsb_decode_commit(const float* post, int ld_post, int B, int r, int mel, int stop_col, int stop_index, int max_iters,
                       float* mel_out, float* stop_out, void* next_hi, void* next_lo, int ld_next, int32_t* pos, int32_t* done,
                       int32_t* n, int32_t* all_done, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Training-step GEMMs (single-pass bf16, fp32 accumulate) -- gradients of the layers above
 *
 * ttsb_bgemm: per-(batch row b, head h) products  out_z[m][n] = alpha * sum_k A_z[m][k] * B_z[n][k]  where both operands
 *   are activations: S = Q K^T, O = P V, dP = dO V^T, dQ = dS K, dK = dS^T Q, dV = P^T dO (model/layers.py:179-193 and
 *   its gradient).  Each operand is a bf16 tensor described as (dim0 contiguous, dim1 rows, dim2 batches) with element
 *   strides.  K-major operand (x_mn_major = 0): dim0 is the contraction axis, dim1 the M (or N) axis; MN-major operand
 *   (x_mn_major = 1): dim0 is the M (or N) axis, dim1 the contraction axis -- so a transposed operand (P^T, dS^T, dO^T,
 *   V^T, K^T) is the SAME tensor read MN-major and no transposed copies exist.  The tile origin of problem z = (b,h) is
 *   (c0 + h*h_col, c1 + h*h_row, z_batch ? z : b).
 *   The contraction runs in k blocks of 64 and relies on the tensor map's zero fill past its extent for the tail
 *   [K, round_up(K, 64)).  So when K % 64 != 0 each operand's contraction axis (dim0 if K-major, dim1 if MN-major) must
 *   have extent exactly K, and with H > 1 no per-head offset along it (h_col if K-major, h_row if MN-major) -- otherwise
 *   the tail would be the next head's data; such a call returns TTSB_ERR_INVALID_ARGUMENT.  Head sizes 64, 128, 192, 256
 *   and every T / Tk of the attention products satisfy this; several heads of size 32 or 96 do not.
 * ttsb_wgrad: weight gradients  dW[seg*Cin + c][n] += sum_{b,t} X_seg[b][t + shift_seg][c] * G[b][t][n]  for Dense
 *   (1 segment), concat-Dense (2 sources) and Conv1D (k segments with the tap shifts); X and G are the row-major bf16
 *   activations / output gradients (B, T, ld) read MN-major; dW is fp32 in the Keras (K, N) layout and is ACCUMULATED
 *   into.
 * ------------------------------------------------------------------------------------------------------- */
typedef struct ttsb_bgemm_args {
  int B, H, M, N, K;
  const void* a;
  long long a_dim0, a_dim1, a_dim2, a_stride1, a_stride2;
  int a_h_col, a_h_row, a_z_batch, a_mn_major;
  const void* b;
  long long b_dim0, b_dim1, b_dim2, b_stride1, b_stride2;
  int b_h_col, b_h_row, b_z_batch, b_mn_major;
  float alpha;
  float* out_f32;            /* either or both */
  void* out_bf16;
  int ld_out;                /* row stride (elements), multiple of 16 */
  long long out_batch_stride;/* elements between consecutive z (or b when out_by_b) */
  int out_h_col;             /* column offset per head */
  int out_by_b;              /* 1: output batch index is b (heads side by side in the columns) */
  int out_cols;              /* writable columns per row of one problem (multiple of 16); columns >= N are written 0 */
  const int32_t* row_len;    /* optional [B]: rows m >= row_len[b] are written as zeros */
  const int32_t* col_len;    /* optional [B]: columns n >= col_len[b] are written as zeros */
  /* ---- ABI 2: fused softmax backward.  With sm_P != NULL the product is dP = dO V^T of an attention backward and the
   * epilogue writes dS = sm_scale * P_pre * (dropout(dP) - D) (bf16, out_bf16) instead of dP, with the masking rules and
   * dropout hash of ttsb_softmax_bwd: sm_P = P_pre bf16 in the OUTPUT layout (requires out_by_b = 0, out_h_col = 0,
   * out_batch_stride = M * ld_out), sm_D fp32 [B*H*M] = rowsum(P_drop * dP) = dO . O per (row, head)
   * (ttsb_rowdot_heads), sm_len = key lengths [B], sm_flags as ttsb_softmax_bwd. */
  const void* sm_P;
  const float* sm_D;
  float sm_scale, sm_drop_p;
  uint32_t sm_seed, sm_site;
  int sm_flags;
  const int32_t* sm_len;
  const void* sm_Pdrop;      /* optional: the saved post-dropout probabilities (same layout); the dropout decision is then
                              * read back from it (kept <=> P_drop != 0 where P_pre != 0) instead of re-hashed */
} ttsb_bgemm_args;

int ttsb_bgemm(const ttsb_bgemm_args* args, void* stream);

typedef struct ttsb_wgrad_args {
  int B, T, Cin, N;
  int num_segments;          /* 1..4 */
  int seg_src[4];            /* which x source */
  int seg_shift[4];          /* time shift of the source rows (conv taps); rows outside [0,T) read as zero */
  const void* x[2];          /* bf16 (B, T, ldx[i]); the first Cin columns are used */
  int ldx[2];
  const void* g;             /* bf16 (B, T, ldg); the first N columns are used */
  int ldg;
  float* dw;                 /* fp32 (num_segments*Cin, N), accumulated */
} ttsb_wgrad_args;

int ttsb_wgrad(const ttsb_wgrad_args* args, void* stream);

/* out[(b*H + h)*T + t] = sum_c x[b,t,h*dh+c] * y[b,t,h*dh+c]  (bf16 (B,T,ld) inputs, fp32 out): the row statistic
 * D = dO . O of the attention backward (equals rowsum(P_drop * dP), so dP never has to be materialised). */
int ttsb_rowdot_heads(const void* x_bf16, const void* y_bf16, int B, int T, int H, int dh, int ld, float* out, void* stream);

/* Row softmax of materialised, pre-scaled scores S fp32 (B*H, T, ld) with key masking (model/layers.py:186-192) and
 * attention dropout: P_pre = softmax, P_drop = dropout(P_pre) (pass the same pointer twice when drop_p == 0). */
/* flags: bit 0 = look-ahead mask (keys > query index masked, transformer_utils.py:35-37); bit 1 = every query row is live
 * (Aligner blocks); without it query rows >= kv_len[b] are written as zeros (they are masked downstream). */
int ttsb_softmax_fwd(const float* S, int B, int H, int T, int Tk, int ld, const int32_t* kv_len, float drop_p,
                     uint32_t seed, uint32_t site, int flags, void* P_pre, void* P_drop, void* stream);
/* The two calls above (logits GEMM + ttsb_softmax_fwd) fused for self-attention with flags == 0: P_pre = softmax(scale *
 * Q K^T) over keys < kv_len[b], P_drop = dropout(P_pre), both bf16 (B*H, T, ld_p); the logits stay in tensor memory.
 * qkv is a bf16 (B, T, ld) activation tensor holding head h of Q at columns q_col0 + h*dh and of K at k_col0 + h*dh.
 * Needs dh in {64, 128, 192} and fewer than 2^33 probabilities (ttsb_attn_probs_supported; otherwise use the two calls
 * above); pass P_drop == P_pre when drop_p == 0.
 * Same dropout element index as ttsb_softmax_fwd: (z*T + t)*ld_p + key. */
int ttsb_attn_probs_supported(int dh, int ld_p);
int ttsb_attn_probs_fwd(const void* qkv, int ld, int q_col0, int k_col0, int B, int H, int T, int dh, const int32_t* kv_len,
                        float scale, float drop_p, uint32_t seed, uint32_t site, void* P_pre, void* P_drop, int ld_p,
                        void* stream);
/* Backward counterpart (the same kernel, one pass): dS = scale * P_pre * (dropout(dO V^T) - D) bf16 (B*H, T, ld_p), the
 * softmax gradient of model/layers.py:186-192 fused into the dP product -- what ttsb_bgemm does with sm_P set, with sixteen
 * epilogue warps and no fp32 dP in HBM.  dO bf16 (B, T, ld_do) holds head h at columns do_col0 + h*dh, v bf16 (B, T, ld_v)
 * at v_col0 + h*dh; D fp32 (B*H*T) from ttsb_rowdot_heads; keys >= kv_len[b] and query rows >= kv_len[b] give zeros. */
int ttsb_attn_ds_bwd(const void* dO, int ld_do, int do_col0, const void* v, int ld_v, int v_col0, int B, int H, int T, int dh,
                     const int32_t* kv_len, const void* P_pre, const float* D, float scale, float drop_p, uint32_t seed,
                     uint32_t site, void* dS, int ld_p, void* stream);
int ttsb_softmax_bwd(const void* P_pre, const float* dP, int B, int H, int T, int Tk, int ld, const int32_t* kv_len,
                     float scale, float drop_p, uint32_t seed, uint32_t site, int flags, void* dS, void* stream);
/* LayerNorm backward from the saved pre-norm values u (keras LayerNormalization, model/layers.py:27,96,207,295,508). */
int ttsb_layernorm_bwd(const float* dz, const float* u, const float* gamma, int B, int T, int C, int ld, float eps,
                       const int32_t* row_len, int relu_mask, float pre_drop_p, uint32_t pre_site, float post_drop_p,
                       uint32_t post_site, uint32_t seed, float* du, void* g_bf16, float* dgamma, float* dbeta, float* dbias,
                       void* stream);
/* column sums of bf16 (rows, ld)[:, :C] accumulated into fp32 out[C] (bias gradients) */
int ttsb_colsum_bf16(const void* x, int64_t rows, int C, int ld, float* out, void* stream);
/* three adjacent column segments of width seg -> three outputs (the q / k / v bias gradients from the (rows, 3d) buffer) */
int ttsb_colsum_bf16_x3(const void* x, int64_t rows, int seg, int ld, float* out0, float* out1, float* out2, void* stream);
int ttsb_relu_bwd(void* dy_bf16, const void* h_bf16, int64_t n, void* stream);
/* ttsb_relu_bwd plus the bias gradient of the layer that produced h, in the same pass: colsum[c] += sum_rows (masked dy)
 * (dy, h bf16 (rows, C) contiguous). */
int ttsb_relu_bwd_colsum(void* dy, const void* h, int64_t rows, int C, float* colsum, void* stream);
/* fp32 (rows, C) -> bf16 (rows, ld_out >= C) with zero padding columns */
int ttsb_cast_bf16_pad(const float* x, int64_t rows, int C, void* out_bf16, int ld_out, void* stream);
/* mean |pred - target| over ALL elements of pred[:, :Tt] (utils/losses.py:41-49 as called with mask=None), added to
 * *loss_out; grad = weight * sign(pred - target) / numel (zero for rows >= Tt). */
int ttsb_mae_loss(const float* pred, int B, int Tp, int Tt, int C, const float* target_f32, const int32_t* target_i32,
                  float weight, float* loss_out, float* grad, void* stream);
/* Duration extraction from the Aligner's attention maps (utils/alignments.py:103-143; the producer of the durations the
 * ForwardTransformer trains on).  Lengths are the reference's "mel_lengths(mels) - 1" / "phoneme_lengths(phonemes) - 1".
 * ttsb_attention_scores: utils/metrics.py:5-44 -> scores (B,H,3) = jumpiness, peakiness, 3 / diagonality.
 * ttsb_durations_from_attention: reference matrix = att[b, best head, 1:mel_len, 1:phon_len] (or the score-weighted sum of
 *   the heads), shortest monotonic path through (max - attention) (utils/alignments.py:58-91: scipy Dijkstra; here the
 *   equivalent anti-diagonal dynamic programme in float64), durations int32 (B,Tk) (zero beyond phon_len - 1).
 *   scratch: B*Tq*Tk bytes. */
int ttsb_attention_scores(const float* att, int B, int H, int Tq, int Tk, const int32_t* mel_len, const int32_t* phon_len, int r,
                          float* scores, void* stream);
int ttsb_durations_from_attention(const float* att, int B, int H, int Tq, int Tk, const int32_t* mel_len, const int32_t* phon_len,
                                  const float* scores, int weighted, uint8_t* scratch, int32_t* durations, void* stream);
/* Per-character pitch (extract_durations.py:108-115, batched): character c < n_chars[b] covers frames [cum[c], cum[c+1]) of
 * the exclusive prefix sum of durations (B,Tp) (non-negative), clipped at pitch_len[b] <= Tm.  A frame value v of pitch
 * (B,Tm) is kept iff v != 0 and v*pitch_std + pitch_mean < 400 (two rounded float64 operations); out (B,Tp) float64 is the
 * mean of the kept values, bit-exact with np.mean (numpy's pairwise summation order), or 0 when none is kept.
 * Characters >= n_chars[b] are 0.  Tp <= 12287. */
int ttsb_pitch_per_char(const double* pitch, int B, int Tm, const int32_t* pitch_len, const int32_t* durations, int Tp,
                        const int32_t* n_chars, double pitch_mean, double pitch_std, double* out, void* stream);

/* Aligner losses (SURVEY 8(f) row 1).
 * ttsb_scaled_ce_loss: utils/losses.py:4-21 new_scaled_crossentropy -- sparse softmax CE of logits (B,Tp,ld)[:, :Tt, :C] against
 *   int targets (B,Tt); sample weight (target != 0) + (target == index) * (scaling - 1); Keras SUM_OVER_BATCH_SIZE
 *   (sum / (B*Tt)); added to *loss_out.
 * ttsb_diag_loss: utils/metrics.py:47-70 batch_diagonal_mask + models.py:189-205 -- mean over (b,h) of
 *   sum_{q<q_len, k<k_len} att[b,h,q,k] * |k/k_len - q/q_len|, divided by 10; added to *loss_out. */
int ttsb_scaled_ce_loss(const float* logits, int B, int Tp, int Tt, int C, int ld, const int32_t* targets, int index,
                        float scaling, float* loss_out, float grad_weight, float* grad /* optional (B,Tp,ld_grad) */, int ld_grad,
                        void* stream);
/* training form of ttsb_diag_loss on the post-dropout probabilities P (bf16, (B*H,Tq,ld)): *loss_out += loss_scale * loss,
 * dP (fp32, same layout, optional) += grad_scale * d loss / d P */
int ttsb_diag_loss_train(const void* P_bf16, int B, int H, int Tq, int Tk, int ld, const int32_t* q_len, const int32_t* k_len,
                         float loss_scale, float* loss_out, float grad_scale, float* dP, void* stream);
int ttsb_diag_loss(const float* att, int B, int H, int Tq, int Tk, const int32_t* q_len, const int32_t* k_len,
                   float* loss_out, void* stream);
/* Expand backward: dx[b,i,:] = sum of dm[b,t,:] over t in [s_i, s_i + max(dur_i, 0)) clipped to [0, Tm), s_i the exclusive
 * prefix sum of the non-negative durations (fp32, d multiple of 4, Tp <= 12000) */
int ttsb_expand_bwd(const float* dm, const int32_t* dur_int, int B, int Tp, int Tm, int d, float* dx, void* stream);
int ttsb_embedding_bwd(const float* dx, const int32_t* tokens, int B, int T, int d, int vocab, float* demb, void* stream);
/* d(pos_encoding_scalar) = sum dropout(g) * PE[t]; (drop_p, seed, site) regenerate the prologue dropout mask */
int ttsb_pe_scalar_bwd(const float* g, const float* pe, int B, int T, int d, float drop_p, uint32_t seed, uint32_t site,
                       float* dscalar, void* stream);
/* training variants of the two stack prologues: keras Dropout after LayerNorm + PE (model/layers.py:301) */
int ttsb_embed_ln_pe_train_fwd(const int32_t* tokens, const float* emb, const float* gamma, const float* beta,
                               const float* pe, const float* pos_scalar, int B, int T, int d, int vocab, float eps,
                               float drop_p, uint32_t seed, uint32_t site, float* out_f32, void* out_hi, void* out_lo,
                               void* stream);
int ttsb_expand_ln_pe_train_fwd(const float* x, const int32_t* idx, const float* gamma, const float* beta, const float* pe,
                                const float* pos_scalar, int B, int Tp, int Tm, int d, float eps, float drop_p, uint32_t seed,
                                uint32_t site, float* out_f32, void* out_hi, void* out_lo, void* stream);
int ttsb_pitch_embed_bwd(const float* g, const float* pitch, const float* w, const float* bias, int B, int T, int d,
                         float* dw, float* db, void* stream);
int ttsb_statpred_head_bwd(const float* gout, const float* out, const float* h, int ldh, int C, const float* w, int relu,
                           const int32_t* row_len, int B, int T, float* dh, float* dw, float* db, void* stream);
/* Keras/TF-2.2 Adam (utils/training_config_manager.py:102-106): theta -= lr_t * m / (sqrt(v) + eps) with
 * lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t) computed by the caller; grad is multiplied by grad_scale first. */
int ttsb_adam_tf_step(float* param, const float* grad, float* m, float* v, int64_t n, float lr_t, float beta1, float beta2,
                      float eps, float grad_scale, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * StatPredictor head  Dense(C->1, relu|linear) * mask   (model/layers.py:479-485)
 *   h fp32 (B,T,ldh) -> out fp32 (B,T)
 * ------------------------------------------------------------------------------------------------------- */
int ttsb_statpred_head_fwd(const float* h, int ldh, int C, const float* w, const float* bias, int relu,
                           const int32_t* row_len, int B, int T, float* out, void* stream);

/* x + relu(pitch*w + b)  (model/models.py:527-531; Dense(1->d, relu)) -> fp32 (B,T,d) */
int ttsb_pitch_embed_add_fwd(const float* x, const float* pitch, const float* w, const float* bias, int B, int T,
                             int d, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Length regulator  (model/models.py:532-540, model/layers.py:549-565)
 * ------------------------------------------------------------------------------------------------------- */
/* durations (B,Tp) fp32 * scalar -> min(max_mask) -> max(min_mask) -> round-half-even -> int32.
 * max_mask / min_mask may be NULL.  Also writes per-row totals to out_len[B]; a row that holds a negative duration gets
 * out_len = -1 (the reference's ragged-tensor construction raises on it; the host checks this one array). */
int ttsb_durations_to_int(const float* dur, float scalar, const float* max_mask, const float* min_mask, int B, int Tp,
                          int32_t* out_int, int32_t* out_len, void* stream);
/* int durations (B,Tp) -> frame->phoneme index map (B,Tm) (-1 at padded frames); row totals must be <= Tm */
int ttsb_expand_indices(const int32_t* dur_int, int B, int Tp, int Tm, int32_t* out_idx, void* stream);
/* out[b,t,:] = idx[b,t] >= 0 ? x[b, idx[b,t], :] : 0     (Expand; fp32, d multiple of 4) */
int ttsb_length_regulate_fwd(const float* x, const int32_t* idx, int B, int Tp, int Tm, int d, float* out, void* stream);
/* fused Expand + decoder prologue LN + scalar*PE (model/layers.py:299-300): writes fp32 + bf16 hi/lo */
int ttsb_expand_ln_pe_fwd(const float* x, const int32_t* idx, const float* gamma, const float* beta, const float* pe,
                          const float* pos_scalar, int B, int Tp, int Tm, int d, float eps, float* out_f32, void* out_hi,
                          void* out_lo, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * utils/spectrogram_ops.py:8-17
 * ------------------------------------------------------------------------------------------------------- */
int ttsb_mel_lengths(const float* mel, int B, int T, int C, float padding_value, int32_t* out, void* stream);
int ttsb_phoneme_lengths(const int32_t* phonemes, int B, int T, int32_t padding, int32_t* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * STFT -> mel filterbank -> log   (data/audio.py:72-92, 209-231)
 *   wav fp32 (n_clips, n_samples); out fp32 (n_clips, n_frames, n_mels), n_frames = 1 + n_samples/hop.
 *   n_fft must be 1024 (the reference's config), hop 256, window = periodic Hann(1024), reflect padding.
 *   mel_basis fp32 (n_mels, 513) dense on the device; band int32 (n_mels, 2) in HOST memory: band[2m], band[2m+1] = first /
 *   past-last bin of row m that may hold a non-zero weight (0 <= first <= past-last <= 513; an empty row is (0, 0)).  Only
 *   the weights inside each row's band are read, from mel_basis itself on every call: nothing is kept between calls, so a
 *   basis rewritten in place is used as it now stands.  normalizer 0 = MelGAN log(clip 1e-5), 1 = WaveRNN.  Bad arguments
 *   give TTSB_ERR_INVALID_ARGUMENT before any CUDA call, with the argument named in ttsb_last_error().  The entry point never
 *   waits for the device (it may be captured in a CUDA graph once the library has run one call on that device).  A band table
 *   spanning more than 2048 weights runs a slower kernel that reads the basis from global memory.
 * ------------------------------------------------------------------------------------------------------- */
int ttsb_stft_mel_log(const float* wav, int n_clips, int n_samples, const float* mel_basis, const int32_t* band, int n_mels,
                      int normalizer, float* out, void* stream);
/* The same for a packed ragged batch of clips (create_training_data.py:41-47 over a corpus).  Clip c owns samples
 *   sample_offsets[c] .. sample_offsets[c+1] - 1 of wav and output frames frame_offsets[c] .. frame_offsets[c+1] - 1 of out
 *   (fp32 (total_frames, n_mels)), with frame_offsets[c+1] - frame_offsets[c] = 1 + L_c/256.  Both offset tables are int32
 *   (n_clips + 1) in HOST memory, starting at 0; every clip needs L_c > 512.  The entry point checks them and copies a clip
 *   table into `workspace` (ttsb_stft_mel_log_batch_workspace_bytes(n_clips) bytes of device memory, 4-byte aligned) before
 *   its one launch; a malformed table is refused with TTSB_ERR_INVALID_ARGUMENT before any CUDA call.  Reflect padding happens
 *   at each clip's own edges and a frame pair never spans two clips, so clip c's mel is bit-identical to ttsb_stft_mel_log on
 *   that clip alone, wherever it sits in the batch.  mel_basis and band as for ttsb_stft_mel_log; a band table spanning more
 *   than 2048 weights gives TTSB_ERR_UNSUPPORTED. */
int64_t ttsb_stft_mel_log_batch_workspace_bytes(int n_clips);   /* -1 for n_clips < 1 */
int ttsb_stft_mel_log_batch(const float* wav, const int32_t* sample_offsets, const int32_t* frame_offsets, int n_clips,
                            const float* mel_basis, const int32_t* band, int n_mels, int normalizer, void* workspace,
                            int64_t workspace_bytes, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * f0 by WORLD's DIO + StoneMask  (Audio.extract_pitch, data/audio.py:146-151: pw.dio(y, fs, frame_period) then pw.stonemask;
 * speed 1, float64 arithmetic; oracle/pitch_oracle.py restates the algorithm)
 *   wav: fp32 clips packed end to end, clip c at samples sample_offsets[c] .. sample_offsets[c+1] - 1 (int32 (n_clips + 1), HOST
 *   memory, from 0).  Clip c has WORLD's int(1000.0 L_c / fs / frame_period_ms) + 1 frames (computed in double in that order);
 *   f0_offsets (int32 (n_clips + 1), HOST memory) must hold their prefix sums, and f0_out (fp64 (f0_offsets[n_clips]), device)
 *   receives the refined f0 of every frame in Hz, 0 where unvoiced.  pyworld's defaults are f0_floor 71, f0_ceil 800,
 *   channels_in_octave 2, allowed_range 0.1.  A clip with no more frames than DIO's voice_range_minimum (3 at the reference's
 *   settings) is refused: WORLD's FixF0Contour returns nothing defined there.
 *   workspace: ttsb_pitch_workspace_bytes(...) bytes of device memory, 256-byte aligned (about 190 bytes per sample).  Malformed
 *   offsets or scalars give TTSB_ERR_INVALID_ARGUMENT before any CUDA call.  A clip's f0 does not depend, bit for bit, on the
 *   other clips of the batch or its position in it. */
int64_t ttsb_pitch_workspace_bytes(const int32_t* sample_offsets, int n_clips, int fs, double frame_period_ms, double f0_floor,
                                   double f0_ceil, double channels_in_octave);   /* -1 for invalid arguments */
int ttsb_pitch_dio_stonemask(const float* wav, const int32_t* sample_offsets, int n_clips, int fs, double frame_period_ms,
                             double f0_floor, double f0_ceil, double channels_in_octave, double allowed_range,
                             const int32_t* f0_offsets, double* f0_out, void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Resampling  (Audio.resample_ragged_device; data/audio.py:126-130: librosa.load(path, sr=...) -> librosa.resample(res_type=
 * 'kaiser_best') -> resampy.resample(filter='kaiser_best') + fix_length; tests/resample_oracle.py restates the algorithm)
 *   wav: fp32 clips packed end to end, clip c at samples sample_offsets[c] .. sample_offsets[c+1] - 1, sampled at src_rates[c]
 *   Hz (sample_offsets int32 (n_clips + 1) and src_rates int32 (n_clips), both in HOST memory; mixed rates share one launch).
 *   half_window: the interpolation filter's half window, float64 (n_window) in device memory, 512 entries per zero crossing
 *   (resampy's kaiser_best: n_window 32769).  Clip c becomes ceil(L_c ratio_c) samples at dst_rate, ratio_c = (double) dst_rate /
 *   src_rates[c]: int(L_c ratio_c) computed samples then zeros; a clip already at dst_rate is copied unchanged.  out_offsets (int32
 *   (n_clips + 1), HOST memory, from 0) must hold the prefix sums of those lengths; out: fp32 (out_offsets[n_clips]) on the device.
 *   Every sample follows resampy's resample_f in float64 without contraction, the accumulator rounded to float32 after each tap,
 *   and the float64 time register r_{t+1} = r_t + 1/ratio is reproduced bit for bit (see csrc/resample.cu), so clip c's output
 *   does not depend on the other clips or its position in the batch.
 *   workspace: ttsb_resample_batch_workspace_bytes(...) bytes of device memory, 16-byte aligned (about 530 KB per distinct
 *   downsampling ratio, plus the clip and time-register tables).  Offsets that do not start at 0 or decrease, a rate <= 0,
 *   out_offsets that disagree with ceil(L ratio), a clip with int(L ratio) < 1 and a short workspace give
 *   TTSB_ERR_INVALID_ARGUMENT before any CUDA call. */
int64_t ttsb_resample_batch_workspace_bytes(const int32_t* sample_offsets, const int32_t* src_rates, int n_clips, int dst_rate,
                                            int n_window);   /* -1 for invalid arguments */
int ttsb_resample_batch(const float* wav, const int32_t* sample_offsets, const int32_t* src_rates, int n_clips, int dst_rate,
                        const double* half_window, int n_window, const int32_t* out_offsets, void* workspace, int64_t workspace_bytes,
                        float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Silence trimming  (Audio.trim_silence_bounds_device; data/audio.py:164-169: librosa.effects.trim(y, top_db, frame_length=256,
 * hop_length=64); tests/trim_oracle.py restates the algorithm)
 *   wav: fp32 clips packed end to end, clip c at samples sample_offsets[c] .. sample_offsets[c+1] - 1 (int32 (n_clips + 1), HOST
 *   memory, from 0; every clip at least one sample).  Per clip of L samples: x is the clip reflect-padded by 128 samples on each
 *   side as np.pad(y, 128, 'reflect') pads it (repeated reflection below 129 samples, a 1-sample clip repeated); frame
 *   t = 0 .. L / 64 has the power p_t = (sum of x[64 t + k]^2, k = 0 .. 255, added in k order) / 256 in float64; frame t is
 *   non-silent iff 10 log10(max(1e-10, p_t)) - 10 log10(max(1e-10, max_t p_t)) > -top_db, in float64.  bounds: int32
 *   (n_clips, 2) in device memory receives [start, end) = [64 f, min(L, 64 (l + 1))) relative to the clip for its first and last
 *   non-silent frames f and l ([0, 0) if there is none, which top_db > 0 rules out).  A clip's bounds do not depend on the other
 *   clips or its position in the batch.  Three launches whatever the number of clips.
 *   workspace: ttsb_trim_silence_workspace_bytes(...) bytes of device memory, 16-byte aligned (8 bytes per frame plus 24 per
 *   clip).  Offsets that do not start at 0 or decrease, an empty clip, a top_db that is not finite or <= 0 and a short workspace
 *   give TTSB_ERR_INVALID_ARGUMENT before any CUDA call. */
int64_t ttsb_trim_silence_workspace_bytes(const int32_t* sample_offsets, int n_clips);   /* -1 for invalid arguments */
int ttsb_trim_silence_bounds(const float* wav, const int32_t* sample_offsets, int n_clips, double top_db, void* workspace,
                             int64_t workspace_bytes, int32_t* bounds, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * FLAC decoding  (Audio.read_flac_batch; data/audio.py:126-130: librosa.load(path) reads a .flac file through libsndfile;
 * RFC 9639; tests/flac_oracle.py restates the format as an encoder and a plain decoder)
 *   data: the frame bytes of every file (each file's bytes after its metadata blocks) concatenated in device memory; file f is
 *   data[byte_offsets[f] .. byte_offsets[f+1]) (int64 (n_files + 1), HOST memory, from 0, at most 2^31 - 1 bytes per file).
 *   stream_info: int64 (n_files, TTSB_FLAC_INFO_FIELDS) in HOST memory, each file's STREAMINFO as (channels, bits_per_sample,
 *   sample_rate, min_block_size, max_block_size, total_samples).  Supported: 1 to 8 channels, 4 to 24 bits per sample, block sizes
 *   16 <= min <= max <= 65535 (the last frame may be shorter), fixed and variable blocking, every frame-header code form.
 *   mono_out: fp32 (sum of total_samples) on the device; file f's samples start at the sum of the totals of files < f and are what
 *   libsndfile's float read gives (sample x 2^-(bits_per_sample - 1), exact) averaged over the channels as np.mean(y, axis=1) does
 *   on float32 ((x0 + x1) + x2 ... for up to 7 channels, pairwise for 8, then an IEEE division).  pcm_out (optional, NULL for
 *   none): int32 on the device, file f's samples interleaved (sample i channel c at P_f + i channels_f + c, P_f the sum of
 *   total_samples x channels of files < f).  status_out: int32 (n_files, 2) on the device, (TTSB_FLAC_OK, frames) or (reason,
 *   index of the frame where decoding stopped) per file; a file that fails gets zeros in its outputs and the others decode
 *   normally.  The MD5 signature of STREAMINFO is not checked (libsndfile does not check it either).  Five launches whatever the
 *   number of files; a file's output does not depend on the other files of the call.
 *   workspace: ttsb_flac_decode_workspace_bytes(...) bytes of device memory, 16-byte aligned (about 2.4 bytes per frame byte, 24 per
 *   frame and 4 per sample and channel).  NULL pointers, offsets that do not start at 0 or decrease, n_files outside [1, 65535],
 *   a stream of 25 to 32 bits (refused by name) or outside the supported set, an unknown (0) total and a short workspace give
 *   TTSB_ERR_INVALID_ARGUMENT before any CUDA call. */
#define TTSB_FLAC_INFO_FIELDS 6
#define TTSB_FLAC_OK 0
#define TTSB_FLAC_NO_SYNC 1         /* no valid frame header (sync, codes, CRC-8) where a frame must start */
#define TTSB_FLAC_BAD_FRAME 2       /* a reserved or invalid subframe, LPC or residual code, or non-zero padding */
#define TTSB_FLAC_TRUNCATED 3       /* the data ends inside a frame or before STREAMINFO's total */
#define TTSB_FLAC_CRC 4             /* the frame's CRC-16 (polynomial 0x8005) does not match */
#define TTSB_FLAC_NUMBER 5          /* the coded frame or sample number is not the expected one */
#define TTSB_FLAC_MISMATCH 6        /* block size, rate, channels or depth disagree with STREAMINFO */
#define TTSB_FLAC_TOTAL 7           /* the frames hold more samples than STREAMINFO's total */
int64_t ttsb_flac_decode_workspace_bytes(const int64_t* byte_offsets, const int64_t* stream_info, int n_files);  /* -1: invalid */
int ttsb_flac_decode_batch(const uint8_t* data, const int64_t* byte_offsets, const int64_t* stream_info, int n_files,
                           float* mono_out, int32_t* pcm_out, int32_t* status_out, void* workspace, int64_t workspace_bytes,
                           void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Spectral envelope by WORLD's CheapTrick  (Audio.spectral_envelope_device; pyworld.cheaptrick(x, f0, t, fs, q1=-0.15,
 * f0_floor=71); tests/world_mcep_oracle.py restates the algorithm; the readings of WORLD's C++ are in DESIGN.md section 9)
 *   wav: fp32 clips packed end to end, clip c at samples sample_offsets[c] .. sample_offsets[c+1] - 1 (int32 (n_clips + 1), HOST
 *   memory, from 0).  The frames are those of ttsb_pitch_dio_stonemask: clip c has int(1000.0 L_c / fs / frame_period_ms) + 1
 *   frames at t_i = i frame_period_ms / 1000, f0_offsets (int32 (n_clips + 1), HOST memory) their prefix sums and f0 (fp64, device)
 *   the F0 of every frame in Hz (0: unvoiced).  fft_size: a power of two in [256, 4096] whose F0 floor 3 fs / (fft_size - 3) is
 *   below 500 Hz; pyworld's is 2^(1 + int(log2(3 fs / f0_floor + 1))): 1024 at 16 to 24 kHz and 2048 at 44.1 and 48 kHz for
 *   f0_floor 71.  A frame whose F0 is at or below that floor takes 500 Hz (WORLD's default); a frame whose F0 is above fs / 4 or
 *   NaN gets an envelope of NaN.  envelope_out (fp64 (f0_offsets[n_clips], fft_size / 2 + 1), device) receives the power spectral
 *   envelope of every frame, bins 0 .. fft_size / 2.  Float64 throughout, without FMA contraction.  WORLD's safeguard noise (1e-12
 *   randn per windowed sample, |randn| eps per bin) is drawn from a counter-based hash keyed by (clip-local frame, sample or bin,
 *   site) instead of WORLD's sequential generator, so a clip's envelope does not depend, bit for bit, on the other clips or its
 *   position in the batch.  One CTA per frame.
 *   workspace: ttsb_cheaptrick_workspace_bytes(...) bytes of device memory, 16-byte aligned (the offset tables and fft_size / 2
 *   twiddles).  NULL pointers, malformed offsets, an empty clip, f0_offsets that disagree with WORLD's frame count, fs outside
 *   [8000, 192000], a frame_period_ms or q1 that is not finite (or <= 0), an fft_size out of range and a short workspace give
 *   TTSB_ERR_INVALID_ARGUMENT before any CUDA call. */
int64_t ttsb_cheaptrick_workspace_bytes(const int32_t* sample_offsets, const int32_t* f0_offsets, int n_clips, int fs,
                                        double frame_period_ms, int fft_size);   /* -1 for invalid arguments */
int ttsb_cheaptrick(const float* wav, const int32_t* sample_offsets, int n_clips, int fs, double frame_period_ms, const double* f0,
                    const int32_t* f0_offsets, double q1, int fft_size, void* workspace, int64_t workspace_bytes, double* envelope_out,
                    void* stream);

/* Mel-cepstrum of power spectral envelopes  (Audio.world_mcep_batch; pysptk.sp2mc(sp, order, alpha))
 *   envelope: fp64 (n_frames, fft_size / 2 + 1) on the device, fft_size a power of two in [256, 4096]; matrix: fp64 (order + 1,
 *   fft_size / 2 + 1) on the device, the linear map of sp2mc (irfft of log sp, c0 halved, SPTK's freqt to order at alpha) that
 *   utils/evaluation.py's sp2mc_matrix builds on the host.  mc_out (fp64 (n_frames, order + 1), device) receives
 *   mc[f][k] = sum_j matrix[k][j] log(envelope[f][j]), summed in a fixed order, so a frame's result does not depend on the
 *   others.  One CTA per frame, no workspace.  NULL pointers, n_frames < 1, an fft_size out of range and an order outside
 *   [1, fft_size / 2) give TTSB_ERR_INVALID_ARGUMENT before any CUDA call. */
int ttsb_sp2mc(const double* envelope, int n_frames, int fft_size, const double* matrix, int order, double* mc_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * mel -> waveform  (Audio.reconstruct_waveform, data/audio.py:94-110: librosa mel_to_stft(power=1) + griffinlim(32, momentum .99))
 *   n_fft 1024, hop 256, periodic Hann, centred frames with reflect padding (the reference configuration).
 * ------------------------------------------------------------------------------------------------------- */
/* mel amplitudes (n_frames, n_mels) -> non-negative linear magnitudes (n_frames, 513): per frame min_{x>=0} |A x - m|^2 for the
 * mel basis A (n_mels, 513), from the start max(pinv(A) m, 0) that librosa's nnls uses, with n_iter FISTA steps of size `step`
 * (1 / |A|_2^2).  band[2*j], band[2*j+1] = first / past-last non-zero bin of basis row j; bin_mels[2*k], [2*k+1] = first /
 * past-last mel row that is non-zero at bin k.  basis_pinv is (513, n_mels). */
int ttsb_mel_to_linear(const float* mel_amp, int n_frames, int n_mels, const float* mel_basis, const float* basis_pinv,
                       const int32_t* band, const int32_t* bin_mels, float step, int n_iter, float* out, void* stream);
/* librosa.stft: wav (n_samples) -> complex64 (1 + n_samples/256, 513) as interleaved (re, im) floats */
int ttsb_stft_complex(const float* wav, int n_samples, float* spec_out, void* stream);
/* librosa.istft: complex64 (n_frames, 513) -> wav (256 * (n_frames - 1)).  workspace: ttsb_istft_workspace_bytes(n_frames) bytes
 * of device memory (the windowed time frames before the overlap-add). */
int64_t ttsb_istft_workspace_bytes(int n_frames);
int ttsb_istft(const float* spec, int n_frames, void* workspace, int64_t workspace_bytes, float* wav_out, void* stream);
/* one phase update of fast Griffin-Lim over n complex bins: a = rebuilt - momentum/(1+momentum) * previous (previous may be
 * NULL: first iteration); a /= |a| + 1e-16; projected_out = magnitude * a.  rebuilt / previous / projected_out are complex64. */
int ttsb_griffinlim_update(const float* rebuilt, const float* previous, const float* magnitude, float momentum, int64_t n,
                           float* projected_out, void* stream);
/* Griffin-Lim for a packed ragged batch of clips: librosa.griffinlim (0.7.1, "fast", momentum) of every clip, n_iter iterations
 * plus the final iSTFT, with a number of launches that does not depend on n_clips (1 + 3 n_iter + 2).
 *   Clip c owns frames frame_offsets[c] .. frame_offsets[c+1] - 1 of the packed arrays (frame_offsets: int32 (n_clips + 1) in
 *   device memory, frame_offsets[0] = 0, frame_offsets[n_clips] = total_frames, every clip >= 4 frames -- the host checks this;
 *   a malformed table gives wrong numbers, never an access outside the buffers).  Its waveform has 256 (T_c - 1) samples and
 *   starts at sample 256 (frame_offsets[c] - c) of wav_out, so wav_out holds 256 (total_frames - n_clips) fp32 samples.
 *   magnitude fp32 (total_frames, 513); init_angles complex64 (total_frames, 513) of unit modulus.
 *   Each clip is transformed on its own: reflect padding at the clip's own edges, no overlap-add across clips, and a clip's
 *   waveform does not depend, bit for bit, on the other clips of the batch or its position in it.
 *   workspace: ttsb_griffinlim_batch_workspace_bytes(total_frames, n_clips) bytes of device memory, 16-byte aligned.
 *   Needs n_clips >= 1, 4 n_clips <= total_frames <= 2097151, n_iter >= 0, momentum finite and >= 0. */
int64_t ttsb_griffinlim_batch_workspace_bytes(int total_frames, int n_clips);   /* -1 for an invalid shape */
int ttsb_griffinlim_batch(const float* magnitude, const float* init_angles, const int32_t* frame_offsets, int n_clips,
                          int total_frames, int n_iter, float momentum, void* workspace, int64_t workspace_bytes,
                          float* wav_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * The STFT family at any supported configuration  (Audio at settings other than n_fft 1024 / hop 256 / win 1024, e.g. the
 * reference's config/data_config_wavernn.yaml: n_fft 2048, hop 275, win 1100)
 *   n_fft a power of two in [256, 4096], 1 <= hop_length <= win_length <= n_fft, win_length >= 2 (a periodic Hann of one sample
 *   would be 0, where librosa's window is [1]); window = periodic Hann(win_length) centred in
 *   n_fft (librosa's pad_center), centred frames with reflect padding; n_bins = n_fft / 2 + 1.  A clip of L samples has
 *   1 + L / hop frames and needs L > n_fft / 2.  Offset tables are int32 (n_clips + 1) in HOST memory, from 0; the entry points
 *   check them and the configuration and give TTSB_ERR_INVALID_ARGUMENT before any CUDA call, then copy the twiddles, the
 *   window (both computed in float64 and rounded once) and a clip table into `workspace` (device memory, 256-byte aligned, of
 *   the size the matching _workspace_bytes query returns; -1 there for invalid arguments).  Frame pairs never span two clips,
 *   reflect padding happens at each clip's own edges and the overlap-add stays inside a clip, so a clip's output is
 *   bit-identical wherever it sits in the batch.
 * ------------------------------------------------------------------------------------------------------- */
/* log-mel of a packed ragged batch, as ttsb_stft_mel_log_batch: mel_basis fp32 (n_mels, n_bins) dense, band int32 (n_mels, 2) on
 *   the device (as ttsb_mel_to_linear's: band[2m], band[2m+1] = first / past-last non-zero bin of row m; bounds outside [0, n_bins]
 *   are clamped), out fp32 (frame_offsets[n_clips], n_mels), frame_offsets[c+1] - frame_offsets[c] = 1 + L_c / hop_length. */
int64_t ttsb_stft_mel_log_ragged_workspace_bytes(int n_clips, int n_fft);
int ttsb_stft_mel_log_ragged(const float* wav, const int32_t* sample_offsets, const int32_t* frame_offsets, int n_clips, int n_fft,
                             int hop_length, int win_length, const float* mel_basis, const int32_t* band, int n_mels, int normalizer,
                             void* workspace, int64_t workspace_bytes, float* out, void* stream);
/* ttsb_mel_to_linear at n_bins = n_fft / 2 + 1 in [129, 2049] bins: mel_basis (n_mels, n_bins), basis_pinv (n_bins, n_mels),
 *   bin_mels (n_bins, 2), out (n_frames, n_bins). */
int ttsb_mel_to_linear_ex(const float* mel_amp, int n_frames, int n_mels, int n_bins, const float* mel_basis, const float* basis_pinv,
                          const int32_t* band, const int32_t* bin_mels, float step, int n_iter, float* out, void* stream);
/* librosa.stft of every clip of a packed batch: wav (sample_offsets[n_clips]) -> complex64 (sum of 1 + L_c / hop, n_bins) as
 *   interleaved (re, im) floats, clip c's frames after those of clips 0 .. c-1. */
int64_t ttsb_stft_complex_ragged_workspace_bytes(int n_clips, int n_fft);
int ttsb_stft_complex_ragged(const float* wav, const int32_t* sample_offsets, int n_clips, int n_fft, int hop_length, int win_length,
                             void* workspace, int64_t workspace_bytes, float* spec_out, void* stream);
/* librosa.istft of every clip of a packed batch: complex64 (total_frames, n_bins), clip c in frames frame_offsets[c] ..
 *   frame_offsets[c+1] - 1 (>= 2 frames) -> wav_out fp32 (hop (total_frames - n_clips)), clip c's hop (T_c - 1) samples from
 *   sample hop (frame_offsets[c] - c).  Window-sum-square normalisation and centre trim per clip. */
int64_t ttsb_istft_ragged_workspace_bytes(int total_frames, int n_clips, int n_fft);
int ttsb_istft_ragged(const float* spec, const int32_t* frame_offsets, int n_clips, int n_fft, int hop_length, int win_length,
                      void* workspace, int64_t workspace_bytes, float* wav_out, void* stream);
/* ttsb_griffinlim_batch at this configuration (1 + 3 n_iter + 2 launches): magnitude fp32 and init_angles complex64
 *   (total_frames, n_bins), wav_out as ttsb_istft_ragged.  Every clip needs T_c >= n_fft / 2 / hop + 2 frames, so that its
 *   hop (T_c - 1) samples are more than n_fft / 2 (4 at 1024 / 256, 5 at 2048 / 275); n_iter >= 0, momentum finite and >= 0. */
int64_t ttsb_griffinlim_ragged_workspace_bytes(int total_frames, int n_clips, int n_fft);
int ttsb_griffinlim_ragged(const float* magnitude, const float* init_angles, const int32_t* frame_offsets, int n_clips, int n_fft,
                           int hop_length, int win_length, int n_iter, float momentum, void* workspace, int64_t workspace_bytes,
                           float* wav_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Mel-cepstral distortion after dynamic time warping, and its warping path  (evaluate_tts.py, --f0 for the path; no reference
 * counterpart; tests/evaluation_oracle.py restates the definition in float64, tests/dtw_path_oracle.py the path)
 *   A packed ragged batch of n_pairs pairs of fp32 log-mel sequences (frames, n_mels) on the device: pair p compares frames
 *   x_offsets[p] .. x_offsets[p+1] - 1 of x with frames y_offsets[p] .. y_offsets[p+1] - 1 of y (both tables int32
 *   (n_pairs + 1) in HOST memory, from 0, every sequence >= 1 frame).  With K = n_ceps (1 <= K < n_mels):
 *     cepstra   c_k[t] = sum_m dct[k-1][m] x[t][m], k = 1..K, summed in float64 in increasing m; dct fp64 (K, n_mels) on the
 *               device, rows 1..K of the orthonormal DCT-II (c0, the energy, is left out);
 *     distance  d(i, j) = kappa sqrt(2 sum_k (c_k[i] - c'_k[j])^2), summed in increasing k; kappa = 10 / ln 10 from the host;
 *     DTW       steps (1,1), (1,0), (0,1): C[0][0] = d(0,0), C[i][j] = d(i,j) + min(C[i-1][j-1], C[i-1][j], C[i][j-1]),
 *               ties to the diagonal unless another predecessor is strictly smaller, then (i-1, j) before (i, j-1); the
 *               path length L (cells on the path) is that of the chosen predecessor + 1.
 *   Outputs (device): cost_out fp64 (n_pairs) = C[Tx-1][Ty-1], path_len_out int32 (n_pairs) = L[Tx-1][Ty-1]; the pair's MCD is
 *   cost / L.  Every product and sum is rounded on its own (no FMA contraction), so the result equals the float64 restatement
 *   bit for bit and does not depend on the other pairs or the pair's position.  min(Tx, Ty) may be at most
 *   TTSB_MCD_DTW_MAX_FRAMES: one CTA per pair keeps three anti-diagonals of (C, L) in shared memory.
 *   workspace: ttsb_mcd_dtw_workspace_bytes(...) bytes of device memory, 8-byte aligned (the cepstra of every frame and the
 *   pair table).  NULL pointers, malformed offsets, an empty sequence, K out of range, a pair past the frame limit, kappa not
 *   finite and positive and a short workspace give TTSB_ERR_INVALID_ARGUMENT before any CUDA call.
 * ------------------------------------------------------------------------------------------------------- */
#define TTSB_MCD_DTW_MAX_FRAMES 4096
int64_t ttsb_mcd_dtw_workspace_bytes(const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps); /* -1: invalid */
int ttsb_mcd_dtw(const float* x, const int32_t* x_offsets, const float* y, const int32_t* y_offsets, int n_pairs, int n_mels,
                 const double* dct, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes, double* cost_out,
                 int32_t* path_len_out, void* stream);
/* ttsb_mcd_dtw_path: ttsb_mcd_dtw with the same arguments, definition and outputs (cost_out and path_len_out equal
 *   ttsb_mcd_dtw's bit for bit), which also writes each pair's warping path, for frame-level scores along it (the F0 scores of
 *   evaluate_tts.py --f0).
 *   path_out (device) int32 (i, j) pairs: pair p's path starts at entry P_p = sum_{q<p} (Tx_q + Ty_q - 1), the longest a path of
 *   the earlier pairs can be, and runs from (0, 0) to (Tx-1, Ty-1); its first path_len_out[p] entries are written.  Each step
 *   goes to the predecessor the DTW recursion chose, under its tie rule (diagonal, then (i-1, j), then (i, j-1)), so consecutive
 *   entries differ by (1,1), (1,0) or (0,1).  A pair's path does not depend on the other pairs or its position.
 *   The sweep keeps 2 bits per cell of the predecessor it took in the workspace (ttsb_mcd_dtw_path_workspace_bytes(...) bytes,
 *   8-byte aligned); a pair may have at most TTSB_MCD_DTW_PATH_MAX_CELLS cells (Tx * Ty; 4 MiB of bits, e.g. 4096 x 4096 or
 *   1,200 x 13,981), and min(Tx, Ty) is at most TTSB_MCD_DTW_MAX_FRAMES as above.  Everything ttsb_mcd_dtw refuses, a NULL
 *   path_out and a pair past the cell limit give TTSB_ERR_INVALID_ARGUMENT before any CUDA call. */
#define TTSB_MCD_DTW_PATH_MAX_CELLS 16777216
int64_t ttsb_mcd_dtw_path_workspace_bytes(const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps); /* -1: invalid */
int ttsb_mcd_dtw_path(const float* x, const int32_t* x_offsets, const float* y, const int32_t* y_offsets, int n_pairs, int n_mels,
                      const double* dct, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes, double* cost_out,
                      int32_t* path_len_out, int32_t* path_out, void* stream);
/* ttsb_mcd_dtw_ceps, ttsb_mcd_dtw_ceps_path: ttsb_mcd_dtw and ttsb_mcd_dtw_path over cepstra the caller computed (the WORLD
 *   mel-cepstra of evaluate_tts.py --mcep).  x and y are frame-major fp64 (frames, ld) on the device, pair p's frames given by
 *   x_offsets / y_offsets as above; c_k of a frame is its column first + k - 1, k = 1..K = n_ceps (first >= 0, first + K <= ld).
 *   The columns are copied into the workspace ttsb_mcd_dtw reads, and the same kernels sweep them: distance, DTW, tie rule,
 *   frame and cell limits, outputs and path are those of ttsb_mcd_dtw / ttsb_mcd_dtw_path, bit for bit for the same cepstra.
 *   workspace: ttsb_mcd_dtw_ceps_workspace_bytes(...) / ttsb_mcd_dtw_ceps_path_workspace_bytes(...) bytes (the same sizes as
 *   ttsb_mcd_dtw's and ttsb_mcd_dtw_path's), 8-byte aligned.  What those refuse, and first or K out of range, give
 *   TTSB_ERR_INVALID_ARGUMENT before any CUDA call. */
int64_t ttsb_mcd_dtw_ceps_workspace_bytes(const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps); /* -1: invalid */
int ttsb_mcd_dtw_ceps(const double* x, const int32_t* x_offsets, const double* y, const int32_t* y_offsets, int n_pairs, int ld,
                      int first, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes, double* cost_out,
                      int32_t* path_len_out, void* stream);
int64_t ttsb_mcd_dtw_ceps_path_workspace_bytes(const int32_t* x_offsets, const int32_t* y_offsets, int n_pairs, int n_ceps); /* -1 */
int ttsb_mcd_dtw_ceps_path(const double* x, const int32_t* x_offsets, const double* y, const int32_t* y_offsets, int n_pairs, int ld,
                           int first, int n_ceps, double kappa, void* workspace, int64_t workspace_bytes, double* cost_out,
                           int32_t* path_len_out, int32_t* path_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Ragged-batch Conv1D on the tensor cores (the MelGAN and HiFi-GAN generators, transformertts_b200/model/melgan.py and
 * hifigan.py).
 * Layout: a packed ragged batch of n_clips clips, channels-last 16-bit (rows, ld).  Clip c has L_c rows, given as the int32
 * prefix sums clip_offsets[0..n_clips] (HOST memory, clip_offsets[0] = 0), framed by `halo` rows on each side (0..
 * TTSB_CONV1D_EX_MAX_HALO, for the inputs and the outputs alike): its rows are clip_offsets[c] + (2c + 1) halo + [0, L_c), and
 * the buffer holds clip_offsets[n_clips] + 2 halo n_clips rows.  Each call computes, for every clip row t in [0, L_c),
 *   y[c, t, :] = bias + sum_s  in_{tap_src[s]}[c, t + tap_shift[s], :] @ W[koff_s : koff_s + ld_in[tap_src[s]], :]  (+ residual)
 * (up to TTSB_CONV1D_EX_MAX_TAPS taps with |tap_shift| <= halo, so a tap reads the clip's own halos; koff_s = the ld_in of the
 * earlier taps).  W is the (K_total, N) matrix packed by ttsb_pack_weight (n_pad = N); ld_in[src] is a multiple of 64 and every
 * input column is read.  With up > 1 (a transposed conv phrased over its input rows), column n of y[c, t] is channel n % ld_out
 * of output row t up + n / ld_out: the outputs use the same layout with up L_c rows per clip, and N = up ld_out.
 *   res_hi/lo  optional residual in the output layout (ld_out columns, res_lo only in bf16x3): y = bias + conv + (res_hi + res_lo).
 *              Neither plane may be an output plane.
 *   sum        optional fp32 plane in the output layout, for the multi-receptive-field average of HiFi-GAN's resblocks, in torch's
 *              order (xs = rb_0(x); xs += rb_1(x); ...; x = xs / nk), after the residual:
 *                TTSB_CONV1D_SUM_WRITE  sum = y                 (resblock 0)
 *                TTSB_CONV1D_SUM_ADD    sum = sum + y           (the middle resblocks)
 *                TTSB_CONV1D_SUM_FINISH y = (sum + y) / sum_div (the last one; then out / act are written from this y)
 *              WRITE and ADD count as an output, so out and act may both be NULL.
 *   out_rows   rows of the output layout, sum up L_c + 2 halo n_clips: the shape of the outputs, the residual and the sum.
 * Outputs (bf16; the lo planes only in bf16x3; any may be NULL): out_hi/out_lo = y, act_hi/act_lo = LeakyReLU_slope(y), slope
 * in [0, 1].  The conv does not run in place: no output plane may be an input plane a tap reads (in_hi, and in bf16x3 in_lo,
 * of its source), since other tiles' taps still load the rows a tile writes.
 * halo_mode: TTSB_HALO_NONE leaves the outputs' halos alone; TTSB_HALO_REFLECT writes output row L-1+k of a clip as a copy of
 * row L-1-k and row -k as a copy of row k (k = 1..halo, needs up L_c > halo); TTSB_HALO_ZERO writes zeros there (needs
 * up L_c >= halo).  A halo row is written only by the store of the row it mirrors, never by a computed row.  So with
 * TTSB_HALO_NONE and zero-initialised planes the halos stay zero, which is every zero-padded conv's padding, and clips of any
 * length >= 1 work.
 * N is a multiple of 64, and at most 256 or a multiple of 256; ld_out (= N / up) is a multiple of 16; res_hi, res_lo, sum,
 * bias and the output planes the call writes (in bf16 the lo planes are not) are 16-byte aligned.  No atomics: a clip's output is bit-identical wherever it sits in the batch.  workspace:
 * ttsb_conv1d_workspace_bytes(n_clips) bytes of device memory, 4-byte aligned; the entry points copy the clip table there.
 * Malformed offsets, clips too short for the halo mode, a short workspace, misaligned or aliased planes and any inconsistent
 * halo, taps, slope, residual, sum or out_rows give TTSB_ERR_INVALID_ARGUMENT before any CUDA call.
 * ------------------------------------------------------------------------------------------------------- */
#define TTSB_HALO_NONE 0
#define TTSB_HALO_REFLECT 1
#define TTSB_HALO_ZERO 2
#define TTSB_CONV1D_EX_MAX_TAPS 16
#define TTSB_CONV1D_EX_MAX_HALO 64
#define TTSB_CONV1D_SUM_NONE 0
#define TTSB_CONV1D_SUM_WRITE 1
#define TTSB_CONV1D_SUM_ADD 2
#define TTSB_CONV1D_SUM_FINISH 3
typedef struct ttsb_conv1d_ex_args {
  int n_clips;
  const int32_t* clip_offsets; /* HOST, int32 (n_clips + 1) */
  int halo;
  int num_taps;
  int tap_src[TTSB_CONV1D_EX_MAX_TAPS];
  int tap_shift[TTSB_CONV1D_EX_MAX_TAPS];
  const void* in_hi[2];
  const void* in_lo[2];
  int ld_in[2];
  const void* w_hi;
  const void* w_lo;
  const float* bias; /* fp32 (N), or NULL */
  int N;
  int up;
  const void* res_hi; /* or NULL */
  const void* res_lo;
  float* sum; /* fp32 (out_rows, ld_out), or NULL */
  int sum_mode;
  float sum_div;
  void* out_hi;
  void* out_lo;
  void* act_hi;
  void* act_lo;
  int ld_out;
  int64_t out_rows;
  float slope;
  int halo_mode;
  int precision; /* TTSB_PREC_BF16 or TTSB_PREC_BF16X3 */
  void* workspace;
  int64_t workspace_bytes;
} ttsb_conv1d_ex_args;
int64_t ttsb_conv1d_workspace_bytes(int n_clips); /* -1 for n_clips < 1 */
int ttsb_conv1d_ex_tc(const ttsb_conv1d_ex_args* a, void* stream);
/* The generators' output layer: wav = tanh(bias + sum_{k=-3..3} in[t + k, :channels] . weight[k + 3, :]) for every clip row t
 * in [0, L_c - drop_tail), in = hi (+ lo) planes in the layout above with `halo` rows (3..TTSB_CONV1D_EX_MAX_HALO) and ld_in
 * columns; the halos hold the padding (reflected for MelGAN, zeros for HiFi-GAN).  Clip c's samples go to
 * wav_out[clip_offsets[c] - c drop_tail ...].  weight: fp32 (7, channels) on the device, channels <= ld_in <= 256, every
 * L_c > drop_tail >= 0. */
int ttsb_conv1d_out_tanh_ex(const void* in_hi, const void* in_lo, int ld_in, int channels, int halo, const int32_t* clip_offsets,
                            int n_clips, int drop_tail, const float* weight, float bias, void* workspace, int64_t workspace_bytes,
                            float* wav_out, void* stream);
/* The same output layer with clamp(., -1, 1) in place of tanh (BigVGAN v2, use_tanh_at_final = false; pass bias 0 for a
 * conv_post without bias).  Same arguments and refusals. */
int ttsb_conv1d_out_clamp_ex(const void* in_hi, const void* in_lo, int ld_in, int channels, int halo, const int32_t* clip_offsets,
                             int n_clips, int drop_tail, const float* weight, float bias, void* workspace, int64_t workspace_bytes,
                             float* wav_out, void* stream);
/* BigVGAN's anti-aliased periodic activation (Activation1d: UpSample1d, Snake / SnakeBeta, DownSample1d; model/bigvgan.py), one
 * launch for a packed ragged batch.  in = hi (+ lo in bf16x3) planes in the layout above (`halo` rows, 0..
 * TTSB_CONV1D_EX_MAX_HALO, ld columns, the first `channels` live); out = separate planes of the same layout.  Per clip c of
 * L_c >= 1 rows and live channel ch, with x the clip's rows:
 *   u[m] = 2 sum_i x[clamp(i - 5, 0, L - 1)] h_up[m + 15 - 2i]      m in [0, 2L), over the six i with 0 <= m + 15 - 2i <= 11
 *   s[m] = u[m] + inv_beta[ch] sin^2(alpha[ch] u[m])
 *   out[t] = sum_j h_down[j] s[clamp(2t + j - 5, 0, 2L - 1)]         t in [0, L), j = 0..11
 * (F.pad(x, (5, 5), 'replicate'), 2 conv_transpose1d(stride 2), [15 : -15]; then F.pad(s, (5, 6), 'replicate'), conv1d(stride
 * 2)).  fp32 arithmetic with full-range sinf, in a fixed order without atomics: a clip's output is bit-identical wherever it
 * sits in the batch.  Columns [channels, ld) of clip rows are written as 0; halo rows are never written (zero-initialised
 * planes keep the next conv's zero padding).  alpha, inv_beta: fp32 (channels) on the device; h_up, h_down: 12 fp32 taps each
 * in HOST memory.  ld is a multiple of 8, the planes are 16-byte aligned and no output plane is an input plane.  workspace:
 * ttsb_conv1d_workspace_bytes(n_clips) bytes.  NULL or misaligned planes, malformed offsets, channels > ld, aliased planes
 * and a short workspace give TTSB_ERR_INVALID_ARGUMENT before any CUDA call. */
int ttsb_snake_aa_ex(const void* in_hi, const void* in_lo, void* out_hi, void* out_lo, int ld, int channels, int halo,
                     const int32_t* clip_offsets, int n_clips, const float* alpha, const float* inv_beta, const float* h_up,
                     const float* h_down, int precision, void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * WaveRNN generator (fatchord/WaveRNN, transformertts_b200/model/wavernn.py): the sample-rate recurrence of every fold of
 * every clip in one persistent cooperative launch, then the fold crossfade, crop to (T_c - 1) hop samples and the fade-out
 * over the last 20 hop samples (csrc/wavernn.cu).  rnn_dims = fc_dims = TTSB_WAVERNN_DIMS; aux parts of 32 columns.
 * Folds: batched, clip c of T_c frames is cut as fatchord's fold_with_overlap cuts T_c hop samples (fold length target +
 *   2 overlap, stride target + overlap, the last fold zero-padded); otherwise one fold per clip runs max_c T_c hop steps.
 *   n_rows is the caller's fold count, checked against that rule.  Clip c's folds use seeds[c] (host uint32) and draw
 *   uniforms keyed by (seeds[c], fold index, step, draw): 11 per step in MOL, 1 in RAW, as oracle/wavernn_oracle.py states.
 * Conditioning, bf16 hi (+ lo in bf16x3) planes in the ragged layout of ttsb_conv1d_ex_tc (frames as rows, cond_halo rows on
 *   each side of every clip, cond_rows in all; the halo rows of melp are zero):
 *   melp (ld_melp >= 2048): per mel frame, columns [0, 512) its projection onto I's mel columns, [512, 2048) onto W_ih1 I_mel.
 *   aux (ld_aux >= 4608): per frame, [0, 512) a1 onto I, [512, 2048) a1 onto W_ih1 I, [2048, 3584) a2 onto rnn2's input
 *   weights, [3584, 4096) a3 onto fc1, [4096, 4608) a4 onto fc2 (no biases).
 *   Sample n of a clip (frame f = n / hop, phase p = n % hop) adds aux[f] + sum_j taps[p][j] melp[f + j - n_taps / 2];
 *   samples past T_c hop add nothing (the biases stay).
 * taps: device fp32 (hop, n_taps), n_taps odd <= TTSB_WAVERNN_MAX_TAPS <= 2 cond_halo + 1.
 * vec: device fp32, [0, 512) I's x_prev column, [512, 1024) I's bias, [1024, 2560) W_ih1 I_0, [2560, 4096) W_ih1 b_I + b_ih1,
 *   [4096, 5632) b_hh1, [5632, 7168) b_ih2, [7168, 8704) b_hh2, [8704, 9216) fc1 bias, [9216, 9728) fc2 bias, then fc3's.
 * weights: device, (5632 + n_classes) rows of 512, row-major, fp32 in TTSB_PREC_BF16X3 (fp32 products) and bf16 in
 *   TTSB_PREC_BF16 (bf16 products of bf16-rounded activations, fp32 sums): rows [0, 1536) W_hh1, [1536, 3072) rnn2's
 *   W_ih[:, :512], [3072, 4608) W_hh2, [4608, 5120) fc1[:, :512], [5120, 5632) fc2[:, :512], then fc3.
 * mode TTSB_WAVERNN_MOL (n_classes 30) or TTSB_WAVERNN_RAW (n_classes 2^bits, 8 <= bits <= 10; mu-law decoded).
 * wav_out: device fp32, sum_c (T_c - 1) hop samples, clip after clip.  Every T_c >= TTSB_WAVERNN_MIN_FRAMES.
 * capture: NULL, or device fp32 (n_rows, capture_steps, n_classes): the logits of each fold's first capture_steps steps.
 * samples_out: NULL, or device fp32 (n_rows, steps): each fold's samples before the crossfade.
 * timings: NULL, or device int64 (TTSB_WAVERNN_CTAS, 12): per CTA, for the six segments of a step (sampling, GRU1, GRU2, fc1,
 *   fc2, fc3), the nanoseconds summed over all steps from the segment's start to its last warp finishing, then through the
 *   grid barrier after it (%globaltimer; the timed run adds a CTA barrier per segment).
 * workspace: ttsb_wavernn_workspace_bytes(...) bytes, 256-byte aligned.  A row's arithmetic does not depend on the other
 * rows, its place or the grid, so a clip's waveform is bit-identical in any batch.  Bad arguments give
 * TTSB_ERR_INVALID_ARGUMENT before any CUDA call; a device that cannot hold the grid resident gives TTSB_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------------------- */
#define TTSB_WAVERNN_DIMS 512
#define TTSB_WAVERNN_MOL 0
#define TTSB_WAVERNN_RAW 1
#define TTSB_WAVERNN_MAX_TAPS 7
#define TTSB_WAVERNN_MIN_FRAMES 21
#define TTSB_WAVERNN_MAX_ROWS 8192
#define TTSB_WAVERNN_CTAS 128
int64_t ttsb_wavernn_workspace_bytes(const int32_t* frames, int n_clips, int hop, int batched, int target, int overlap,
                                     int n_classes); /* -1: invalid */
int ttsb_wavernn_generate(const int32_t* frames /* HOST (n_clips) */, const uint32_t* seeds /* HOST (n_clips) */, int n_clips, int hop,
                          int batched, int target, int overlap, int n_rows, int n_taps, const float* taps, const void* melp_hi,
                          const void* melp_lo, int ld_melp, const void* aux_hi, const void* aux_lo, int ld_aux, int cond_halo,
                          int64_t cond_rows, const float* vec, const void* weights, int mode, int n_classes, int precision,
                          float* wav_out, float* capture, int capture_steps, float* samples_out, int64_t* timings,
                          void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Data-parallel gradient exchange (BASELINE.json: "NCCL allreduce over NVLink on gradient buckets only"; the reference has
 * no distributed code).  One communicator per process / GPU.  NCCL is loaded at run time (libnccl.so.2 of the host
 * process, or $TTSB_NCCL_LIB); without it these return TTSB_ERR_UNSUPPORTED.
 *   ttsb_dp_unique_id       : rank 0 fills a 128-byte id that the host distributes to all ranks (any side channel)
 *   ttsb_dp_init            : collective; binds to the calling thread's current CUDA device
 *   ttsb_dp_allreduce_bucket: in-place SUM of buf[0:count] (fp32, device) across ranks, enqueued on `stream`; the 1/N
 *                             factor is applied by ttsb_adam_tf_step(grad_scale).  Call it as soon as a contiguous slice of
 *                             the flat gradient buffer is final, on a second stream, to overlap it with the remaining
 *                             backward kernels.
 * ------------------------------------------------------------------------------------------------------- */
typedef struct ttsb_dp_comm ttsb_dp_comm;
int ttsb_dp_unique_id(void* id_out_128_bytes);
int ttsb_dp_init(const void* unique_id_128_bytes, int rank, int world, ttsb_dp_comm** out);
int ttsb_dp_allreduce_bucket(ttsb_dp_comm* comm, float* buf, int64_t count, void* stream);
int ttsb_dp_destroy(ttsb_dp_comm* comm);

#ifdef __cplusplus
}
#endif
#endif /* TTSB_H_ */
