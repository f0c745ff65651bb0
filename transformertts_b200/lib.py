"""ctypes binding of libttsb.so (include/ttsb.h).  There is no CPU fallback: if the library is missing or a call
fails, a TtsbError is raised."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional

import torch

PREC_BF16 = 0
PREC_BF16X3 = 1
PREC_FP16 = 2
IMPL_TCGEN05 = 0
IMPL_SIMT = 1

# TTSB_LIB selects another build of the same library (for example a debug build)
_LIB_PATH = Path(os.environ.get('TTSB_LIB') or Path(__file__).resolve().parent / 'libttsb.so')
_lib = None

EXPORTS = [
    'ttsb_last_error', 'ttsb_abi_version', 'ttsb_launch_count', 'ttsb_reset_launch_count', 'ttsb_add_launch_count', 'ttsb_set_dropout_salt', 'ttsb_pack_weight',
    'ttsb_repack_batched',
    'ttsb_split_bf16', 'ttsb_embed_ln_pe_fwd', 'ttsb_linear_fwd', 'ttsb_layernorm_fwd', 'ttsb_mha_fwd', 'ttsb_statpred_head_fwd',
    'ttsb_pitch_embed_add_fwd', 'ttsb_durations_to_int', 'ttsb_expand_indices', 'ttsb_length_regulate_fwd',
    'ttsb_expand_ln_pe_fwd', 'ttsb_mel_lengths', 'ttsb_phoneme_lengths', 'ttsb_stft_mel_log',
    'ttsb_bgemm', 'ttsb_wgrad', 'ttsb_rowdot_heads', 'ttsb_softmax_fwd', 'ttsb_attn_probs_supported', 'ttsb_attn_probs_fwd', 'ttsb_attn_ds_bwd', 'ttsb_softmax_bwd', 'ttsb_layernorm_bwd',
    'ttsb_relu_bwd', 'ttsb_relu_bwd_colsum', 'ttsb_colsum_bf16', 'ttsb_colsum_bf16_x3', 'ttsb_cast_bf16_pad', 'ttsb_mae_loss', 'ttsb_scaled_ce_loss', 'ttsb_diag_loss', 'ttsb_diag_loss_train', 'ttsb_attention_scores', 'ttsb_durations_from_attention', 'ttsb_pitch_per_char', 'ttsb_expand_bwd', 'ttsb_embedding_bwd', 'ttsb_pe_scalar_bwd',
    'ttsb_pitch_embed_bwd', 'ttsb_statpred_head_bwd', 'ttsb_adam_tf_step', 'ttsb_embed_ln_pe_train_fwd',
    'ttsb_expand_ln_pe_train_fwd', 'ttsb_mel_to_linear', 'ttsb_stft_complex', 'ttsb_istft_workspace_bytes', 'ttsb_istft', 'ttsb_griffinlim_update',
    'ttsb_griffinlim_batch_workspace_bytes', 'ttsb_griffinlim_batch',
    'ttsb_dp_unique_id', 'ttsb_dp_init', 'ttsb_dp_allreduce_bucket', 'ttsb_dp_destroy',
    'ttsb_decode_attn_workspace_bytes', 'ttsb_decode_attn', 'ttsb_decode_prologue', 'ttsb_decode_commit',
]


class TtsbError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int), ('T', C.c_int), ('N', C.c_int), ('block_n', C.c_int), ('num_segments', C.c_int),
        ('seg_src', C.c_int * 4), ('seg_shift', C.c_int * 4), ('seg_k', C.c_int * 4),
        ('a_hi', C.c_void_p * 2), ('a_lo', C.c_void_p * 2), ('lda', C.c_int * 2), ('a_col0', C.c_int * 2),
        ('w_hi', C.c_void_p), ('w_lo', C.c_void_p), ('bias', C.c_void_p), ('relu', C.c_int),
        ('residual', C.c_void_p), ('ld_res', C.c_int), ('ln_gamma', C.c_void_p), ('ln_beta', C.c_void_p),
        ('ln_eps', C.c_float), ('row_len', C.c_void_p), ('out_f32', C.c_void_p), ('out_hi', C.c_void_p),
        ('out_lo', C.c_void_p), ('ld_out', C.c_int), ('out_fp16', C.c_int), ('out_preln', C.c_void_p),
        ('drop_pre_p', C.c_float), ('drop_post_p', C.c_float), ('drop_pre_site', C.c_uint32), ('drop_post_site', C.c_uint32),
        ('drop_seed', C.c_uint32), ('precision', C.c_int), ('impl', C.c_int),
        ('residual_hi', C.c_void_p), ('residual_lo', C.c_void_p),
    ]


class PackDesc(C.Structure):
    _fields_ = [
        ('src', C.c_void_p), ('dst', C.c_void_p), ('R', C.c_int), ('R_pad', C.c_int), ('C_cols', C.c_int),
        ('cb', C.c_int), ('cb_valid', C.c_int), ('sr', C.c_longlong), ('s_outer', C.c_longlong), ('s_inner', C.c_longlong),
        ('dst_ld', C.c_int), ('dst_f32', C.c_int),
    ]


class BgemmArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int), ('H', C.c_int), ('M', C.c_int), ('N', C.c_int), ('K', C.c_int),
        ('a', C.c_void_p), ('a_dim0', C.c_longlong), ('a_dim1', C.c_longlong), ('a_dim2', C.c_longlong),
        ('a_stride1', C.c_longlong), ('a_stride2', C.c_longlong), ('a_h_col', C.c_int), ('a_h_row', C.c_int), ('a_z_batch', C.c_int), ('a_mn_major', C.c_int),
        ('b', C.c_void_p), ('b_dim0', C.c_longlong), ('b_dim1', C.c_longlong), ('b_dim2', C.c_longlong),
        ('b_stride1', C.c_longlong), ('b_stride2', C.c_longlong), ('b_h_col', C.c_int), ('b_h_row', C.c_int), ('b_z_batch', C.c_int), ('b_mn_major', C.c_int),
        ('alpha', C.c_float), ('out_f32', C.c_void_p), ('out_bf16', C.c_void_p), ('ld_out', C.c_int),
        ('out_batch_stride', C.c_longlong), ('out_h_col', C.c_int), ('out_by_b', C.c_int), ('out_cols', C.c_int),
        ('row_len', C.c_void_p), ('col_len', C.c_void_p),
        ('sm_P', C.c_void_p), ('sm_D', C.c_void_p), ('sm_scale', C.c_float), ('sm_drop_p', C.c_float),
        ('sm_seed', C.c_uint32), ('sm_site', C.c_uint32), ('sm_flags', C.c_int), ('sm_len', C.c_void_p), ('sm_Pdrop', C.c_void_p),
    ]


class WgradArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int), ('T', C.c_int), ('Cin', C.c_int), ('N', C.c_int), ('num_segments', C.c_int),
        ('seg_src', C.c_int * 4), ('seg_shift', C.c_int * 4), ('x', C.c_void_p * 2), ('ldx', C.c_int * 2),
        ('g', C.c_void_p), ('ldg', C.c_int), ('dw', C.c_void_p),
    ]


class MhaArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int), ('T', C.c_int), ('H', C.c_int), ('dh', C.c_int),
        ('qk_hi', C.c_void_p), ('qk_lo', C.c_void_p), ('ld_qk', C.c_int), ('q_col0', C.c_int), ('k_col0', C.c_int),
        ('v_col0', C.c_int), ('kv_len', C.c_void_p),
        ('out_hi', C.c_void_p), ('out_lo', C.c_void_p), ('ld_out', C.c_int),
        ('weights_out', C.c_void_p), ('weights_batch_index', C.c_int), ('precision', C.c_int), ('impl', C.c_int),
        ('kv_hi', C.c_void_p), ('kv_lo', C.c_void_p), ('ld_kv', C.c_int), ('Tk', C.c_int), ('causal', C.c_int),
        ('full_queries', C.c_int), ('weights_all', C.c_int),
    ]


class DecodeAttnArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int), ('H', C.c_int), ('dh', C.c_int), ('q', C.c_void_p), ('ld_q', C.c_int), ('q_col0', C.c_int),
        ('kv', C.c_void_p), ('ld_kv', C.c_int), ('Tk', C.c_int), ('k_col0', C.c_int), ('v_col0', C.c_int),
        ('new_kv', C.c_void_p), ('ld_new', C.c_int), ('new_k_col0', C.c_int), ('new_v_col0', C.c_int),
        ('pos', C.c_void_p), ('kv_len', C.c_void_p), ('done', C.c_void_p), ('out_hi', C.c_void_p), ('out_lo', C.c_void_p),
        ('ld_out', C.c_int), ('probs', C.c_void_p), ('probs_T', C.c_int), ('precision', C.c_int),
        ('workspace', C.c_void_p), ('workspace_bytes', C.c_int64),
    ]


def library_path() -> Path:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load libttsb.so (built in-tree by transformertts_b200.build).  Raises TtsbError when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise TtsbError(f'{_LIB_PATH} not found -- run `python -m transformertts_b200.build` (no CPU fallback exists)')
    lib = C.CDLL(str(_LIB_PATH))
    lib.ttsb_last_error.restype = C.c_char_p
    lib.ttsb_launch_count.restype = C.c_int64
    lib.ttsb_reset_launch_count.restype = None
    lib.ttsb_add_launch_count.restype = None
    lib.ttsb_add_launch_count.argtypes = [C.c_int64]
    lib.ttsb_istft_workspace_bytes.restype = C.c_int64
    lib.ttsb_griffinlim_batch_workspace_bytes.restype = C.c_int64
    lib.ttsb_decode_attn_workspace_bytes.restype = C.c_int64
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise TtsbError(f'libttsb.so does not export {name}')
    _lib = lib
    return lib


def _check(rc: int, what: str):
    if rc != 0:
        raise TtsbError(f'{what} failed ({rc}): {load().ttsb_last_error().decode()}')


_last_dev = -1  # device index of the last tensor handed to ptr(): checked against the current device by _stream()


def ptr(t: Optional[torch.Tensor]):
    global _last_dev
    if t is None:
        return None
    if not t.is_cuda:
        raise TtsbError('libttsb expects CUDA tensors')
    _last_dev = t.device.index
    return C.c_void_p(t.data_ptr())


def _stream():
    """Current stream of the current device.  Kernels launch on the CURRENT device, so the tensors must live there: the
    model classes enter `torch.cuda.device(model.device)` around every public call; raw users of this module get an error
    instead of a launch on device 0 against device-1 pointers."""
    cur = _get_device()
    if _last_dev >= 0 and _last_dev != cur:
        raise TtsbError(f'tensor lives on cuda:{_last_dev} but the current device is cuda:{cur}; '
                        f'wrap the call in torch.cuda.device({_last_dev})')
    return C.c_void_p(_get_raw_stream(cur))


# torch.cuda.current_stream() builds a Stream object through several python layers (~5 us); a training step makes ~400
# launches, so the raw C entry points are used when this torch build has them
_get_device = getattr(torch._C, '_cuda_getDevice', None) or torch.cuda.current_device
_get_raw_stream = getattr(torch._C, '_cuda_getCurrentRawStream', None) or (lambda dev: torch.cuda.current_stream(dev).cuda_stream)


def launch_count() -> int:
    return int(load().ttsb_launch_count())


def reset_launch_count():
    load().ttsb_reset_launch_count()


def add_launch_count(n: int):
    load().ttsb_add_launch_count(int(n))


def set_dropout_salt(salt_dev: torch.Tensor):
    """salt_dev: int32/uint32 CUDA tensor with one element (see include/ttsb.h)."""
    _check(load().ttsb_set_dropout_salt(ptr(salt_dev), _stream()), 'ttsb_set_dropout_salt')


# ------------------------------------------------------------------------------------------------------------
# thin typed wrappers (shapes are taken from the tensors; all tensors must be contiguous)
# ------------------------------------------------------------------------------------------------------------
def pack_weight(w_kn: torch.Tensor, n_pad: int, split: bool):
    """Keras (K,N) fp32 kernel (Conv1D (k,Cin,Cout) is reshaped to (k*Cin, Cout)) -> bf16 hi/lo [n_pad, K]."""
    w2 = w_kn.reshape(-1, w_kn.shape[-1]).contiguous().float()
    K, N = w2.shape
    hi = torch.empty((n_pad, K), dtype=torch.bfloat16, device=w2.device)
    lo = torch.empty_like(hi) if split else None
    _check(load().ttsb_pack_weight(ptr(w2), K, N, n_pad, ptr(hi), ptr(lo), _stream()), 'ttsb_pack_weight')
    return hi, lo


def upload_pack_descs(descs, device) -> torch.Tensor:
    """ctypes PackDesc list -> device byte tensor (kept alive by the caller)."""
    arr = (PackDesc * len(descs))(*descs)
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
    return host.to(device)


def repack_batched(descs_dev: torch.Tensor, n: int):
    _check(load().ttsb_repack_batched(ptr(descs_dev), n, _stream()), 'ttsb_repack_batched')


def split_bf16(x: torch.Tensor, split: bool):
    x = x.contiguous().float()
    hi = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi) if split else None
    _check(load().ttsb_split_bf16(ptr(x), C.c_int64(x.numel()), ptr(hi), ptr(lo), _stream()), 'ttsb_split_bf16')
    return hi, lo


def linear_fwd(args: GemmArgs):
    _check(load().ttsb_linear_fwd(C.byref(args), _stream()), 'ttsb_linear_fwd')


def layernorm_fwd(x, gamma, beta, d, eps, row_len, out_f32, out_hi, out_lo):
    B, T, ld = x.shape
    _check(load().ttsb_layernorm_fwd(ptr(x), ptr(gamma), ptr(beta), B, T, d, ld, C.c_float(eps), ptr(row_len), ptr(out_f32),
                                     ptr(out_hi), ptr(out_lo), _stream()), 'ttsb_layernorm_fwd')


def mha_fwd(args: MhaArgs):
    _check(load().ttsb_mha_fwd(C.byref(args), _stream()), 'ttsb_mha_fwd')


def embed_ln_pe_fwd(tokens, emb, gamma, beta, pe, pos_scalar, eps, out_f32, out_hi, out_lo, drop=(0.0, 0, 0)):
    B, T = tokens.shape
    vocab, d = emb.shape
    _check(load().ttsb_embed_ln_pe_train_fwd(ptr(tokens), ptr(emb), ptr(gamma), ptr(beta), ptr(pe), ptr(pos_scalar), B, T, d,
                                             vocab, C.c_float(eps), C.c_float(drop[0]), C.c_uint32(drop[1]), C.c_uint32(drop[2]),
                                             ptr(out_f32), ptr(out_hi), ptr(out_lo), _stream()), 'ttsb_embed_ln_pe_fwd')


def expand_ln_pe_fwd(x, idx, gamma, beta, pe, pos_scalar, eps, out_f32, out_hi, out_lo, drop=(0.0, 0, 0)):
    B, Tp, d = x.shape
    Tm = idx.shape[1]
    _check(load().ttsb_expand_ln_pe_train_fwd(ptr(x), ptr(idx), ptr(gamma), ptr(beta), ptr(pe), ptr(pos_scalar), B, Tp, Tm, d,
                                              C.c_float(eps), C.c_float(drop[0]), C.c_uint32(drop[1]), C.c_uint32(drop[2]),
                                              ptr(out_f32), ptr(out_hi), ptr(out_lo), _stream()), 'ttsb_expand_ln_pe_fwd')


def length_regulate_fwd(x, idx, out):
    B, Tp, d = x.shape
    Tm = idx.shape[1]
    _check(load().ttsb_length_regulate_fwd(ptr(x), ptr(idx), B, Tp, Tm, d, ptr(out), _stream()), 'ttsb_length_regulate_fwd')


def durations_to_int(dur, scalar, max_mask, min_mask, out_int, out_len):
    B, Tp = dur.shape
    _check(load().ttsb_durations_to_int(ptr(dur), C.c_float(scalar), ptr(max_mask), ptr(min_mask), B, Tp, ptr(out_int),
                                        ptr(out_len), _stream()), 'ttsb_durations_to_int')


def expand_indices(dur_int, Tm, out_idx):
    B, Tp = dur_int.shape
    _check(load().ttsb_expand_indices(ptr(dur_int), B, Tp, Tm, ptr(out_idx), _stream()), 'ttsb_expand_indices')


def statpred_head_fwd(h, C_in, w, bias, relu, row_len, out):
    B, T, ldh = h.shape
    _check(load().ttsb_statpred_head_fwd(ptr(h), ldh, C_in, ptr(w), ptr(bias), int(relu), ptr(row_len), B, T, ptr(out),
                                         _stream()), 'ttsb_statpred_head_fwd')


def pitch_embed_add_fwd(x, pitch, w, bias, out):
    B, T, d = x.shape
    _check(load().ttsb_pitch_embed_add_fwd(ptr(x), ptr(pitch), ptr(w), ptr(bias), B, T, d, ptr(out), _stream()),
           'ttsb_pitch_embed_add_fwd')


def mel_lengths(mel, padding_value, out):
    B, T, Cc = mel.shape
    _check(load().ttsb_mel_lengths(ptr(mel), B, T, Cc, C.c_float(padding_value), ptr(out), _stream()), 'ttsb_mel_lengths')


def phoneme_lengths(ph, padding, out):
    B, T = ph.shape
    _check(load().ttsb_phoneme_lengths(ptr(ph), B, T, int(padding), ptr(out), _stream()), 'ttsb_phoneme_lengths')


def stft_mel_log(wav, mel_basis, normalizer, out):
    n_clips, n_samples = wav.shape
    n_mels = mel_basis.shape[0]
    _check(load().ttsb_stft_mel_log(ptr(wav), n_clips, n_samples, ptr(mel_basis), n_mels, int(normalizer), ptr(out),
                                    _stream()), 'ttsb_stft_mel_log')


# ------------------------------------------------------------------------------------------------------------
# training-step kernels
# ------------------------------------------------------------------------------------------------------------
def bgemm(args: BgemmArgs):
    _check(load().ttsb_bgemm(C.byref(args), _stream()), 'ttsb_bgemm')


def rowdot_heads(x, y, H, dh, out):
    B, T, ld = x.shape
    _check(load().ttsb_rowdot_heads(ptr(x), ptr(y), B, T, H, dh, ld, ptr(out), _stream()), 'ttsb_rowdot_heads')


def wgrad(args: WgradArgs):
    _check(load().ttsb_wgrad(C.byref(args), _stream()), 'ttsb_wgrad')


SOFTMAX_CAUSAL, SOFTMAX_FULL_QUERIES = 1, 2


def softmax_fwd(S, B, H, T, Tk, ld, kv_len, drop_p, seed, site, P_pre, P_drop, flags=0):
    _check(load().ttsb_softmax_fwd(ptr(S), B, H, T, Tk, ld, ptr(kv_len), C.c_float(drop_p), C.c_uint32(seed), C.c_uint32(site),
                                   int(flags), ptr(P_pre), ptr(P_drop), _stream()), 'ttsb_softmax_fwd')


def attn_probs_supported(dh: int, ld_p: int) -> bool:
    return bool(load().ttsb_attn_probs_supported(int(dh), int(ld_p)))


def attn_probs_fwd(qkv, ld, q_col0, k_col0, B, H, T, dh, kv_len, scale, drop_p, seed, site, P_pre, P_drop, ld_p):
    """P_pre = softmax(scale * Q K^T), P_drop = dropout(P_pre) in one kernel (include/ttsb.h: ttsb_attn_probs_fwd)."""
    _check(load().ttsb_attn_probs_fwd(ptr(qkv), ld, q_col0, k_col0, B, H, T, dh, ptr(kv_len), C.c_float(scale), C.c_float(drop_p),
                                      C.c_uint32(seed), C.c_uint32(site), ptr(P_pre), ptr(P_drop), ld_p, _stream()),
           'ttsb_attn_probs_fwd')


def attn_ds_bwd(dO, ld_do, do_col0, v, ld_v, v_col0, B, H, T, dh, kv_len, P_pre, D, scale, drop_p, seed, site, dS, ld_p):
    """dS = scale * P_pre * (dropout(dO V^T) - D) in one kernel (include/ttsb.h: ttsb_attn_ds_bwd)."""
    _check(load().ttsb_attn_ds_bwd(ptr(dO), ld_do, do_col0, ptr(v), ld_v, v_col0, B, H, T, dh, ptr(kv_len), ptr(P_pre), ptr(D),
                                   C.c_float(scale), C.c_float(drop_p), C.c_uint32(seed), C.c_uint32(site), ptr(dS), ld_p, _stream()),
           'ttsb_attn_ds_bwd')


def softmax_bwd(P_pre, dP, B, H, T, Tk, ld, kv_len, scale, drop_p, seed, site, dS, flags=0):
    _check(load().ttsb_softmax_bwd(ptr(P_pre), ptr(dP), B, H, T, Tk, ld, ptr(kv_len), C.c_float(scale), C.c_float(drop_p),
                                   C.c_uint32(seed), C.c_uint32(site), int(flags), ptr(dS), _stream()), 'ttsb_softmax_bwd')


def layernorm_bwd(dz, u, gamma, B, T, Cc, ld, eps, row_len, relu_mask, du, g_bf16, dgamma, dbeta, pre_drop=(0.0, 0),
                  post_drop=(0.0, 0), seed=0, dbias=None):
    _check(load().ttsb_layernorm_bwd(ptr(dz), ptr(u), ptr(gamma), B, T, Cc, ld, C.c_float(eps), ptr(row_len), int(relu_mask),
                                     C.c_float(pre_drop[0]), C.c_uint32(pre_drop[1]), C.c_float(post_drop[0]),
                                     C.c_uint32(post_drop[1]), C.c_uint32(seed), ptr(du), ptr(g_bf16), ptr(dgamma), ptr(dbeta),
                                     ptr(dbias), _stream()), 'ttsb_layernorm_bwd')


def colsum_bf16(x, rows, Cc, ld, out):
    _check(load().ttsb_colsum_bf16(ptr(x), C.c_int64(rows), Cc, ld, ptr(out), _stream()), 'ttsb_colsum_bf16')


def relu_bwd(dy, h):
    _check(load().ttsb_relu_bwd(ptr(dy), ptr(h), C.c_int64(dy.numel()), _stream()), 'ttsb_relu_bwd')


def relu_bwd_colsum(dy, h, colsum):
    """dy *= (h > 0) in place and colsum += column sums of the result (the bias gradient of the layer that produced h)."""
    Cc = dy.shape[-1]
    _check(load().ttsb_relu_bwd_colsum(ptr(dy), ptr(h), C.c_int64(dy.numel() // Cc), Cc, ptr(colsum), _stream()), 'ttsb_relu_bwd_colsum')


def colsum_bf16_x3(x, rows, seg, ld, out0, out1, out2):
    _check(load().ttsb_colsum_bf16_x3(ptr(x), C.c_int64(rows), seg, ld, ptr(out0), ptr(out1), ptr(out2), _stream()), 'ttsb_colsum_bf16_x3')


def cast_bf16_pad(x, rows, Cc, out, ld_out):
    _check(load().ttsb_cast_bf16_pad(ptr(x), C.c_int64(rows), Cc, ptr(out), ld_out, _stream()), 'ttsb_cast_bf16_pad')


def mae_loss(pred, B, Tp, Tt, Cc, target, weight, loss_out, grad):
    tf = ptr(target) if target.dtype == torch.float32 else None
    ti = ptr(target) if target.dtype == torch.int32 else None
    _check(load().ttsb_mae_loss(ptr(pred), B, Tp, Tt, Cc, tf, ti, C.c_float(weight), ptr(loss_out), ptr(grad), _stream()),
           'ttsb_mae_loss')


def scaled_ce_loss(logits, Tt, Cc, targets, index, scaling, loss_out, grad_weight=1.0, grad=None):
    B, Tp, ld = logits.shape
    _check(load().ttsb_scaled_ce_loss(ptr(logits), B, Tp, Tt, Cc, ld, ptr(targets), int(index), C.c_float(scaling), ptr(loss_out),
                                      C.c_float(grad_weight), ptr(grad), grad.shape[-1] if grad is not None else 0, _stream()),
           'ttsb_scaled_ce_loss')


def diag_loss_train(P_bf16, B, H, Tq, Tk, ld, q_len, k_len, loss_scale, loss_out, grad_scale, dP):
    _check(load().ttsb_diag_loss_train(ptr(P_bf16), B, H, Tq, Tk, ld, ptr(q_len), ptr(k_len), C.c_float(loss_scale), ptr(loss_out),
                                       C.c_float(grad_scale), ptr(dP), _stream()), 'ttsb_diag_loss_train')


def attention_scores(att, mel_len, phon_len, r, scores):
    B, H, Tq, Tk = att.shape
    _check(load().ttsb_attention_scores(ptr(att), B, H, Tq, Tk, ptr(mel_len), ptr(phon_len), int(r), ptr(scores), _stream()),
           'ttsb_attention_scores')


def durations_from_attention(att, mel_len, phon_len, scores, weighted, scratch, durations):
    B, H, Tq, Tk = att.shape
    _check(load().ttsb_durations_from_attention(ptr(att), B, H, Tq, Tk, ptr(mel_len), ptr(phon_len), ptr(scores), int(bool(weighted)),
                                                ptr(scratch), ptr(durations), _stream()), 'ttsb_durations_from_attention')


def pitch_per_char(pitch, pitch_len, durations, n_chars, pitch_mean, pitch_std, out):
    B, Tm = pitch.shape
    Tp = durations.shape[1]
    _check(load().ttsb_pitch_per_char(ptr(pitch), B, Tm, ptr(pitch_len), ptr(durations), Tp, ptr(n_chars), C.c_double(pitch_mean),
                                      C.c_double(pitch_std), ptr(out), _stream()), 'ttsb_pitch_per_char')


def diag_loss(att, q_len, k_len, loss_out):
    B, H, Tq, Tk = att.shape
    _check(load().ttsb_diag_loss(ptr(att), B, H, Tq, Tk, ptr(q_len), ptr(k_len), ptr(loss_out), _stream()), 'ttsb_diag_loss')


def expand_bwd(dm, dur_int, dx):
    B, Tm, d = dm.shape
    Tp = dur_int.shape[1]
    _check(load().ttsb_expand_bwd(ptr(dm), ptr(dur_int), B, Tp, Tm, d, ptr(dx), _stream()), 'ttsb_expand_bwd')


def embedding_bwd(dx, tokens, demb):
    B, T, d = dx.shape
    _check(load().ttsb_embedding_bwd(ptr(dx), ptr(tokens), B, T, d, demb.shape[0], ptr(demb), _stream()), 'ttsb_embedding_bwd')


def pe_scalar_bwd(g, pe, dscalar, drop=(0.0, 0, 0)):
    B, T, d = g.shape
    _check(load().ttsb_pe_scalar_bwd(ptr(g), ptr(pe), B, T, d, C.c_float(drop[0]), C.c_uint32(drop[1]), C.c_uint32(drop[2]),
                                     ptr(dscalar), _stream()), 'ttsb_pe_scalar_bwd')


def pitch_embed_bwd(g, pitch, w, bias, dw, db):
    B, T, d = g.shape
    _check(load().ttsb_pitch_embed_bwd(ptr(g), ptr(pitch), ptr(w), ptr(bias), B, T, d, ptr(dw), ptr(db), _stream()),
           'ttsb_pitch_embed_bwd')


def statpred_head_bwd(gout, out, h, C_in, w, relu, row_len, dh, dw, db):
    B, T, ldh = h.shape
    _check(load().ttsb_statpred_head_bwd(ptr(gout), ptr(out), ptr(h), ldh, C_in, ptr(w), int(relu), ptr(row_len), B, T, ptr(dh),
                                         ptr(dw), ptr(db), _stream()), 'ttsb_statpred_head_bwd')


def adam_tf_step(param, grad, m, v, lr_t, beta1, beta2, eps, grad_scale=1.0):
    _check(load().ttsb_adam_tf_step(ptr(param), ptr(grad), ptr(m), ptr(v), C.c_int64(param.numel()), C.c_float(lr_t),
                                    C.c_float(beta1), C.c_float(beta2), C.c_float(eps), C.c_float(grad_scale), _stream()),
           'ttsb_adam_tf_step')


# ------------------------------------------------------------------------------------------------------------
# data-parallel gradient exchange (NCCL behind the C ABI)
# ------------------------------------------------------------------------------------------------------------
def dp_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    _check(load().ttsb_dp_unique_id(buf), 'ttsb_dp_unique_id')
    return buf.raw


def dp_init(unique_id: bytes, rank: int, world: int):
    comm = C.c_void_p()
    _check(load().ttsb_dp_init(C.c_char_p(unique_id), int(rank), int(world), C.byref(comm)), 'ttsb_dp_init')
    return comm


def dp_allreduce_bucket(comm, buf: torch.Tensor, stream: int):
    """In-place sum of the contiguous fp32 CUDA tensor `buf` across ranks on the raw stream handle `stream`."""
    _check(load().ttsb_dp_allreduce_bucket(comm, ptr(buf), C.c_int64(buf.numel()), C.c_void_p(stream)), 'ttsb_dp_allreduce_bucket')


def dp_destroy(comm):
    _check(load().ttsb_dp_destroy(comm), 'ttsb_dp_destroy')


# ------------------------------------------------------------------------------------------------------------
# mel -> waveform (Griffin-Lim)
# ------------------------------------------------------------------------------------------------------------
def mel_to_linear(mel_amp, basis, pinv, band, bin_mels, step, n_iter, out):
    T, n_mels = mel_amp.shape
    _check(load().ttsb_mel_to_linear(ptr(mel_amp), T, n_mels, ptr(basis), ptr(pinv), ptr(band), ptr(bin_mels), C.c_float(step), int(n_iter),
                                     ptr(out), _stream()), 'ttsb_mel_to_linear')


def stft_complex(wav, spec_out):
    _check(load().ttsb_stft_complex(ptr(wav), wav.numel(), ptr(spec_out), _stream()), 'ttsb_stft_complex')


def istft(spec, workspace, wav_out):
    T = spec.shape[0]
    _check(load().ttsb_istft(ptr(spec), T, ptr(workspace), C.c_int64(workspace.numel() * workspace.element_size()), ptr(wav_out), _stream()),
           'ttsb_istft')


def istft_workspace_bytes(n_frames: int) -> int:
    return int(load().ttsb_istft_workspace_bytes(int(n_frames)))


def griffinlim_update(rebuilt, previous, magnitude, momentum, projected_out):
    _check(load().ttsb_griffinlim_update(ptr(rebuilt), ptr(previous), ptr(magnitude), C.c_float(momentum), C.c_int64(magnitude.numel()),
                                         ptr(projected_out), _stream()), 'ttsb_griffinlim_update')


def griffinlim_batch_workspace_bytes(total_frames: int, n_clips: int) -> int:
    n = int(load().ttsb_griffinlim_batch_workspace_bytes(int(total_frames), int(n_clips)))
    if n < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return n


def griffinlim_batch(magnitude, init_angles, frame_offsets, n_iter, momentum, workspace, wav_out):
    """Griffin-Lim of every clip of a packed batch (include/ttsb.h: ttsb_griffinlim_batch).  magnitude fp32 (F, 513),
    init_angles complex64 (F, 513), frame_offsets int32 (n_clips + 1) on the device, wav_out fp32 (256 (F - n_clips))."""
    F = magnitude.shape[0]
    _check(load().ttsb_griffinlim_batch(ptr(magnitude), ptr(init_angles), ptr(frame_offsets), frame_offsets.numel() - 1, F, int(n_iter),
                                        C.c_float(momentum), ptr(workspace), C.c_int64(workspace.numel() * workspace.element_size()),
                                        ptr(wav_out), _stream()), 'ttsb_griffinlim_batch')


# ------------------------------------------------------------------------------------------------------------
# cached autoregressive decoding (Aligner.predict_batch)
# ------------------------------------------------------------------------------------------------------------
def decode_attn_workspace_bytes(B: int, H: int, dh: int) -> int:
    return int(load().ttsb_decode_attn_workspace_bytes(int(B), int(H), int(dh)))


def decode_attn(args: DecodeAttnArgs):
    _check(load().ttsb_decode_attn(C.byref(args), _stream()), 'ttsb_decode_attn')


def decode_prologue(x, pos, gamma, beta, pe, pos_scalar, eps, out_f32, out_hi, out_lo):
    """out[b] = LayerNorm(x[b]) + pos_scalar * pe[pos[b]]; x fp32 (B, d)."""
    d = x.shape[-1]
    B = x.numel() // d
    _check(load().ttsb_decode_prologue(ptr(x), ptr(pos), ptr(gamma), ptr(beta), ptr(pe), pe.shape[0], ptr(pos_scalar), B, d,
                                       C.c_float(eps), ptr(out_f32), ptr(out_hi), ptr(out_lo), _stream()), 'ttsb_decode_prologue')


def decode_commit(post, B, r, mel, stop_col, stop_index, max_iters, mel_out, stop_out, next_hi, next_lo, pos, done, n, all_done):
    """End of one decode iteration (include/ttsb.h: ttsb_decode_commit); post fp32 (B*r, ld_post), next_hi / next_lo (B, ld_next)."""
    _check(load().ttsb_decode_commit(ptr(post), post.shape[-1], int(B), int(r), int(mel), int(stop_col), int(stop_index), int(max_iters),
                                     ptr(mel_out), ptr(stop_out), ptr(next_hi), ptr(next_lo), next_hi.shape[-1], ptr(pos), ptr(done),
                                     ptr(n), ptr(all_done), _stream()), 'ttsb_decode_commit')
