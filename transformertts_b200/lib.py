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
    'ttsb_stft_mel_log_batch_workspace_bytes', 'ttsb_stft_mel_log_batch', 'ttsb_pitch_workspace_bytes', 'ttsb_pitch_dio_stonemask',
    'ttsb_dp_unique_id', 'ttsb_dp_init', 'ttsb_dp_allreduce_bucket', 'ttsb_dp_destroy',
    'ttsb_decode_attn_workspace_bytes', 'ttsb_decode_attn', 'ttsb_decode_prologue', 'ttsb_decode_commit',
    'ttsb_conv1d_workspace_bytes', 'ttsb_conv1d_ex_tc', 'ttsb_conv1d_out_tanh_ex', 'ttsb_conv1d_out_clamp_ex', 'ttsb_snake_aa_ex',
    'ttsb_resample_batch_workspace_bytes', 'ttsb_resample_batch',
    'ttsb_mcd_dtw_workspace_bytes', 'ttsb_mcd_dtw', 'ttsb_mcd_dtw_path_workspace_bytes', 'ttsb_mcd_dtw_path',
    'ttsb_stft_mel_log_ragged_workspace_bytes', 'ttsb_stft_mel_log_ragged', 'ttsb_mel_to_linear_ex',
    'ttsb_stft_complex_ragged_workspace_bytes', 'ttsb_stft_complex_ragged', 'ttsb_istft_ragged_workspace_bytes', 'ttsb_istft_ragged',
    'ttsb_griffinlim_ragged_workspace_bytes', 'ttsb_griffinlim_ragged',
    'ttsb_wavernn_workspace_bytes', 'ttsb_wavernn_generate',
    'ttsb_trim_silence_workspace_bytes', 'ttsb_trim_silence_bounds',
    'ttsb_cheaptrick_workspace_bytes', 'ttsb_cheaptrick', 'ttsb_sp2mc',
    'ttsb_mcd_dtw_ceps_workspace_bytes', 'ttsb_mcd_dtw_ceps', 'ttsb_mcd_dtw_ceps_path_workspace_bytes', 'ttsb_mcd_dtw_ceps_path',
    'ttsb_flac_decode_workspace_bytes', 'ttsb_flac_decode_batch',
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


# include/ttsb.h: TTSB_FLAC_* (index = status code)
FLAC_STATUS = ('ok', 'no valid frame header where a frame must start', 'a reserved or invalid subframe or residual code',
               'the data ends inside a frame or before the STREAMINFO total', 'CRC-16 mismatch',
               'unexpected frame or sample number', 'frame header disagrees with STREAMINFO',
               'the frames hold more samples than the STREAMINFO total')


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
    lib.ttsb_stft_mel_log_batch_workspace_bytes.restype = C.c_int64
    lib.ttsb_pitch_workspace_bytes.restype = C.c_int64
    lib.ttsb_conv1d_workspace_bytes.restype = C.c_int64
    for name in ('ttsb_conv1d_out_tanh_ex', 'ttsb_conv1d_out_clamp_ex'):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                       C.c_float, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.ttsb_snake_aa_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    lib.ttsb_pitch_workspace_bytes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double]
    lib.ttsb_pitch_dio_stonemask.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
                                             C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.ttsb_resample_batch_workspace_bytes.restype = C.c_int64
    lib.ttsb_resample_batch_workspace_bytes.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.ttsb_resample_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.ttsb_mcd_dtw_workspace_bytes.restype = C.c_int64
    lib.ttsb_mcd_dtw_workspace_bytes.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.ttsb_mcd_dtw.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_double,
                                 C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ttsb_mcd_dtw_path_workspace_bytes.restype = C.c_int64
    lib.ttsb_mcd_dtw_path_workspace_bytes.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.ttsb_mcd_dtw_path.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_double,
                                      C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    for name in ('ttsb_stft_mel_log_ragged_workspace_bytes', 'ttsb_stft_complex_ragged_workspace_bytes',
                 'ttsb_istft_ragged_workspace_bytes', 'ttsb_griffinlim_ragged_workspace_bytes'):
        getattr(lib, name).restype = C.c_int64
    lib.ttsb_stft_mel_log_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                             C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.ttsb_mel_to_linear_ex.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                                          C.c_int, C.c_void_p, C.c_void_p]
    lib.ttsb_stft_complex_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p,
                                             C.c_void_p]
    lib.ttsb_istft_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.c_void_p]
    lib.ttsb_griffinlim_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                           C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.ttsb_wavernn_workspace_bytes.restype = C.c_int64
    lib.ttsb_wavernn_workspace_bytes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.ttsb_wavernn_generate.argtypes = [t for _, t in WAVERNN_PARAMS] + [C.c_void_p]
    lib.ttsb_trim_silence_workspace_bytes.restype = C.c_int64
    lib.ttsb_trim_silence_workspace_bytes.argtypes = [C.c_void_p, C.c_int]
    lib.ttsb_trim_silence_bounds.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.ttsb_cheaptrick_workspace_bytes.restype = C.c_int64
    lib.ttsb_cheaptrick_workspace_bytes.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_int]
    lib.ttsb_cheaptrick.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_double, C.c_int,
                                    C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.ttsb_sp2mc.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    for name in ('ttsb_mcd_dtw_ceps_workspace_bytes', 'ttsb_mcd_dtw_ceps_path_workspace_bytes'):
        getattr(lib, name).restype = C.c_int64
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.ttsb_mcd_dtw_ceps.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double,
                                      C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ttsb_mcd_dtw_ceps_path.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                           C.c_double, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ttsb_flac_decode_workspace_bytes.restype = C.c_int64
    lib.ttsb_flac_decode_workspace_bytes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.ttsb_flac_decode_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_int64, C.c_void_p]
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


def _host_band(band, n_mels: int):
    """int32 (n_mels, 2) band table in host memory (numpy or a CPU tensor) -> (the array, a pointer to its data, valid for as long
    as the array lives)."""
    import numpy as np
    if torch.is_tensor(band):
        if band.is_cuda:
            raise TtsbError('band must be a host table (numpy or a CPU tensor); a device tensor would cost a synchronisation')
        band = band.numpy()
    a = np.ascontiguousarray(band, dtype=np.int32)
    if a.shape != (n_mels, 2):
        raise TtsbError(f'band must be ({n_mels}, 2), got {a.shape}')
    return a, C.c_void_p(a.ctypes.data)


def stft_mel_log(wav, mel_basis, band, normalizer, out):
    """Log-mel of equal-length clips (include/ttsb.h: ttsb_stft_mel_log).  wav fp32 (n_clips, n_samples), mel_basis fp32
    (n_mels, 513) and out fp32 (n_clips, 1 + n_samples // 256, n_mels) on the device; band int32 (n_mels, 2) in host memory."""
    n_clips, n_samples = wav.shape
    n_mels = mel_basis.shape[0]
    keep, bp = _host_band(band, n_mels)
    _check(load().ttsb_stft_mel_log(ptr(wav), n_clips, n_samples, ptr(mel_basis), bp, n_mels, int(normalizer), ptr(out),
                                    _stream()), 'ttsb_stft_mel_log')


def _host_offsets(offsets):
    """int32 (n + 1) offset table in host memory -> (ctypes array, n)."""
    import numpy as np
    a = np.ascontiguousarray(np.asarray(offsets.cpu() if torch.is_tensor(offsets) else offsets, dtype=np.int64))
    if a.ndim != 1 or len(a) < 2 or a.min() < 0 or a.max() > 2**31 - 1:
        raise TtsbError(f'offset table must be 1-D, at least 2 entries, within int32; got shape {a.shape}')
    return (C.c_int32 * len(a))(*a.tolist()), len(a) - 1


def stft_mel_log_batch(wav, sample_offsets, frame_offsets, mel_basis, band, normalizer, out):
    """Log-mel of a packed ragged batch (include/ttsb.h: ttsb_stft_mel_log_batch).  wav fp32 (total_samples,) and out fp32
    (total_frames, n_mels) on the device; the offset tables (n_clips + 1) and band int32 (n_mels, 2) are host tables."""
    so, n = _host_offsets(sample_offsets)
    fo, n_f = _host_offsets(frame_offsets)
    if n_f != n:
        raise TtsbError(f'{n} clips in sample_offsets, {n_f} in frame_offsets')
    nb = int(load().ttsb_stft_mel_log_batch_workspace_bytes(n))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    keep, bp = _host_band(band, mel_basis.shape[0])
    ws = torch.empty(nb, dtype=torch.uint8, device=wav.device)
    _check(load().ttsb_stft_mel_log_batch(ptr(wav), so, fo, n, ptr(mel_basis), bp, mel_basis.shape[0], int(normalizer), ptr(ws),
                                          C.c_int64(nb), ptr(out), _stream()), 'ttsb_stft_mel_log_batch')


def pitch_workspace_bytes(sample_offsets, fs, frame_period_ms, f0_floor=71.0, f0_ceil=800.0, channels_in_octave=2.0) -> int:
    so, n = _host_offsets(sample_offsets)
    nb = int(load().ttsb_pitch_workspace_bytes(so, n, int(fs), float(frame_period_ms), float(f0_floor), float(f0_ceil),
                                               float(channels_in_octave)))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return nb


def pitch_dio_stonemask(wav, sample_offsets, fs, frame_period_ms, f0_offsets, f0_out, workspace, f0_floor=71.0, f0_ceil=800.0,
                        channels_in_octave=2.0, allowed_range=0.1):
    """f0 of a packed ragged batch by DIO + StoneMask (include/ttsb.h: ttsb_pitch_dio_stonemask).  wav fp32 and f0_out fp64 on
    the device; the offset tables are host sequences; workspace: pitch_workspace_bytes(...) bytes on the device."""
    so, n = _host_offsets(sample_offsets)
    fo, n_f = _host_offsets(f0_offsets)
    if n_f != n:
        raise TtsbError(f'{n} clips in sample_offsets, {n_f} in f0_offsets')
    _check(load().ttsb_pitch_dio_stonemask(ptr(wav), so, n, int(fs), float(frame_period_ms), float(f0_floor), float(f0_ceil),
                                           float(channels_in_octave), float(allowed_range), fo, ptr(f0_out), ptr(workspace),
                                           C.c_int64(workspace.numel() * workspace.element_size()), _stream()), 'ttsb_pitch_dio_stonemask')


def _host_rates(rates, n: int):
    import numpy as np
    a = np.asarray(rates.cpu() if torch.is_tensor(rates) else rates, dtype=np.int64).reshape(-1)
    if len(a) != n or (len(a) and (a.min() < -2**31 or a.max() > 2**31 - 1)):
        raise TtsbError(f'{len(a)} source rates for {n} clips (int32 each)')
    return (C.c_int32 * n)(*a.tolist())


def resample_batch_workspace_bytes(sample_offsets, src_rates, dst_rate: int, n_window: int) -> int:
    so, n = _host_offsets(sample_offsets)
    nb = int(load().ttsb_resample_batch_workspace_bytes(so, _host_rates(src_rates, n), n, int(dst_rate), int(n_window)))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return nb


def resample_batch(wav, sample_offsets, src_rates, dst_rate, half_window, out_offsets, out):
    """Resample every clip of a packed ragged batch to dst_rate (include/ttsb.h: ttsb_resample_batch).  wav fp32, half_window
    fp64 and out fp32 on the device; the offset tables (n_clips + 1) and src_rates (n_clips) are host sequences."""
    so, n = _host_offsets(sample_offsets)
    oo, n_o = _host_offsets(out_offsets)
    if n_o != n:
        raise TtsbError(f'{n} clips in sample_offsets, {n_o} in out_offsets')
    rates = _host_rates(src_rates, n)
    nb = resample_batch_workspace_bytes(sample_offsets, src_rates, dst_rate, half_window.numel())
    ws = torch.empty(nb, dtype=torch.uint8, device=wav.device)
    _check(load().ttsb_resample_batch(ptr(wav), so, rates, n, int(dst_rate), ptr(half_window), half_window.numel(), oo, ptr(ws),
                                      C.c_int64(nb), ptr(out), _stream()), 'ttsb_resample_batch')


def trim_silence_workspace_bytes(sample_offsets) -> int:
    so, n = _host_offsets(sample_offsets)
    nb = int(load().ttsb_trim_silence_workspace_bytes(so, n))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return nb


def trim_silence_bounds(wav, sample_offsets, top_db: float, bounds):
    """[start, end) of the non-silent part of every clip of a packed ragged batch (include/ttsb.h: ttsb_trim_silence_bounds).
    wav fp32 and bounds int32 (n_clips, 2) on the device; sample_offsets (n_clips + 1) is a host sequence."""
    so, n = _host_offsets(sample_offsets)
    nb = trim_silence_workspace_bytes(sample_offsets)
    ws = torch.empty(nb, dtype=torch.uint8, device=wav.device)
    _check(load().ttsb_trim_silence_bounds(ptr(wav), so, n, float(top_db), ptr(ws), C.c_int64(nb), ptr(bounds), _stream()),
           'ttsb_trim_silence_bounds')


def _flac_tables(byte_offsets, infos):
    import numpy as np
    bo = np.ascontiguousarray(np.asarray(byte_offsets, dtype=np.int64))
    n = len(infos)
    if bo.ndim != 1 or len(bo) != n + 1:
        raise TtsbError(f'{len(bo)} byte offsets for {n} files (need n_files + 1)')
    info = np.asarray(infos, dtype=np.int64).reshape(-1)
    if len(info) != 6 * n:
        raise TtsbError(f'stream info must hold 6 values per file (include/ttsb.h: TTSB_FLAC_INFO_FIELDS), got {len(info)} for {n}')
    return (C.c_int64 * len(bo))(*bo.tolist()), (C.c_int64 * len(info))(*info.tolist()), n


def flac_decode_workspace_bytes(byte_offsets, infos) -> int:
    """infos: per file (channels, bits_per_sample, sample_rate, min_block_size, max_block_size, total_samples)."""
    bo, table, n = _flac_tables(byte_offsets, infos)
    nb = int(load().ttsb_flac_decode_workspace_bytes(bo, table, n))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return nb


def flac_decode_batch(data, byte_offsets, infos, mono_out, status_out, pcm_out=None):
    """Decode the frame bytes of every file of a packed batch of FLAC streams (include/ttsb.h: ttsb_flac_decode_batch).  data uint8,
    mono_out fp32, status_out int32 (n_files, 2) and pcm_out int32 (optional) on the device; byte_offsets (n_files + 1) and infos
    (flac_decode_workspace_bytes) are host sequences."""
    bo, table, n = _flac_tables(byte_offsets, infos)
    nb = flac_decode_workspace_bytes(byte_offsets, infos)
    ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=mono_out.device)
    _check(load().ttsb_flac_decode_batch(ptr(data) if data.numel() else None, bo, table, n, ptr(mono_out), ptr(pcm_out),
                                         ptr(status_out), ptr(ws), C.c_int64(nb), _stream()), 'ttsb_flac_decode_batch')


# the longest shorter side of a pair ttsb_mcd_dtw takes (include/ttsb.h: TTSB_MCD_DTW_MAX_FRAMES)
MCD_DTW_MAX_FRAMES = 4096


def mcd_dtw_workspace_bytes(x_offsets, y_offsets, n_ceps: int) -> int:
    xo, n = _host_offsets(x_offsets)
    yo, n_y = _host_offsets(y_offsets)
    if n_y != n:
        raise TtsbError(f'{n} pairs in x_offsets, {n_y} in y_offsets')
    nb = int(load().ttsb_mcd_dtw_workspace_bytes(xo, yo, n, int(n_ceps)))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return nb


def mcd_dtw(x, x_offsets, y, y_offsets, dct, kappa, cost_out, path_len_out):
    """DTW cost and path length of every pair of a packed ragged batch of log-mel sequences (include/ttsb.h: ttsb_mcd_dtw).
    x, y fp32 (frames, n_mels), dct fp64 (n_ceps, n_mels), cost_out fp64 (n_pairs,) and path_len_out int32 (n_pairs,) on the
    device; the offset tables (n_pairs + 1) are host sequences."""
    xo, n = _host_offsets(x_offsets)
    yo, n_y = _host_offsets(y_offsets)
    if n_y != n:
        raise TtsbError(f'{n} pairs in x_offsets, {n_y} in y_offsets')
    n_ceps, n_mels = dct.shape
    nb = mcd_dtw_workspace_bytes(x_offsets, y_offsets, n_ceps)
    ws = torch.empty(nb, dtype=torch.uint8, device=x.device)
    _check(load().ttsb_mcd_dtw(ptr(x), xo, ptr(y), yo, n, int(n_mels), ptr(dct), int(n_ceps), float(kappa), ptr(ws), C.c_int64(nb),
                               ptr(cost_out), ptr(path_len_out), _stream()), 'ttsb_mcd_dtw')


# the most cells (Tx * Ty) of a pair ttsb_mcd_dtw_path takes (include/ttsb.h: TTSB_MCD_DTW_PATH_MAX_CELLS)
MCD_DTW_PATH_MAX_CELLS = 16777216


def mcd_dtw_path_workspace_bytes(x_offsets, y_offsets, n_ceps: int) -> int:
    xo, n = _host_offsets(x_offsets)
    yo, n_y = _host_offsets(y_offsets)
    if n_y != n:
        raise TtsbError(f'{n} pairs in x_offsets, {n_y} in y_offsets')
    nb = int(load().ttsb_mcd_dtw_path_workspace_bytes(xo, yo, n, int(n_ceps)))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return nb


def mcd_dtw_path(x, x_offsets, y, y_offsets, dct, kappa, cost_out, path_len_out, path_out):
    """mcd_dtw that also writes each pair's warping path (include/ttsb.h: ttsb_mcd_dtw_path): path_out int32 (sum of
    Tx + Ty - 1, 2) on the device, pair p's path from row sum_{q<p} (Tx_q + Ty_q - 1)."""
    xo, n = _host_offsets(x_offsets)
    yo, n_y = _host_offsets(y_offsets)
    if n_y != n:
        raise TtsbError(f'{n} pairs in x_offsets, {n_y} in y_offsets')
    n_ceps, n_mels = dct.shape
    nb = mcd_dtw_path_workspace_bytes(x_offsets, y_offsets, n_ceps)
    ws = torch.empty(nb, dtype=torch.uint8, device=x.device)
    _check(load().ttsb_mcd_dtw_path(ptr(x), xo, ptr(y), yo, n, int(n_mels), ptr(dct), int(n_ceps), float(kappa), ptr(ws), C.c_int64(nb),
                                    ptr(cost_out), ptr(path_len_out), ptr(path_out), _stream()), 'ttsb_mcd_dtw_path')


def cheaptrick_workspace_bytes(sample_offsets, f0_offsets, fs: int, frame_period_ms: float, fft_size: int) -> int:
    so, n = _host_offsets(sample_offsets)
    fo, n_f = _host_offsets(f0_offsets)
    if n_f != n:
        raise TtsbError(f'{n} clips in sample_offsets, {n_f} in f0_offsets')
    nb = int(load().ttsb_cheaptrick_workspace_bytes(so, fo, n, int(fs), float(frame_period_ms), int(fft_size)))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return nb


def cheaptrick(wav, sample_offsets, fs, frame_period_ms, f0, f0_offsets, q1, fft_size, envelope_out):
    """WORLD's CheapTrick spectral envelope of every frame of a packed ragged batch (include/ttsb.h: ttsb_cheaptrick).  wav fp32,
    f0 fp64 (frames,) and envelope_out fp64 (frames, fft_size / 2 + 1) on the device; the offset tables are host sequences."""
    so, n = _host_offsets(sample_offsets)
    fo, _ = _host_offsets(f0_offsets)
    nb = cheaptrick_workspace_bytes(sample_offsets, f0_offsets, fs, frame_period_ms, fft_size)
    ws = torch.empty(nb, dtype=torch.uint8, device=wav.device)
    _check(load().ttsb_cheaptrick(ptr(wav), so, n, int(fs), float(frame_period_ms), ptr(f0), fo, float(q1), int(fft_size), ptr(ws),
                                  C.c_int64(nb), ptr(envelope_out), _stream()), 'ttsb_cheaptrick')


def sp2mc(envelope, matrix, mc_out):
    """mc = matrix . log(envelope) per frame (include/ttsb.h: ttsb_sp2mc).  envelope fp64 (frames, fft_size / 2 + 1), matrix fp64
    (order + 1, fft_size / 2 + 1) and mc_out fp64 (frames, order + 1) on the device."""
    n_frames, nb = envelope.shape
    if matrix.dim() != 2 or matrix.shape[1] != nb or tuple(mc_out.shape) != (n_frames, matrix.shape[0]):
        raise TtsbError(f'envelope {tuple(envelope.shape)}, matrix {tuple(matrix.shape)} and mc_out {tuple(mc_out.shape)}: need '
                        f'(frames, bins), (order + 1, bins) and (frames, order + 1)')
    _check(load().ttsb_sp2mc(ptr(envelope), int(n_frames), 2 * (nb - 1), ptr(matrix), int(matrix.shape[0]) - 1, ptr(mc_out), _stream()),
           'ttsb_sp2mc')


def mcd_dtw_ceps_workspace_bytes(x_offsets, y_offsets, n_ceps: int, path: bool = False) -> int:
    xo, n = _host_offsets(x_offsets)
    yo, n_y = _host_offsets(y_offsets)
    if n_y != n:
        raise TtsbError(f'{n} pairs in x_offsets, {n_y} in y_offsets')
    fn = load().ttsb_mcd_dtw_ceps_path_workspace_bytes if path else load().ttsb_mcd_dtw_ceps_workspace_bytes
    nb = int(fn(xo, yo, n, int(n_ceps)))
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return nb


def mcd_dtw_ceps(x, x_offsets, y, y_offsets, first: int, n_ceps: int, kappa, cost_out, path_len_out, path_out=None):
    """ttsb_mcd_dtw_ceps (ttsb_mcd_dtw_ceps_path when path_out is given) over caller-given cepstra: x, y fp64 (frames, ld) on the
    device, columns first .. first + n_ceps - 1 scored; cost_out, path_len_out and path_out as mcd_dtw / mcd_dtw_path take them."""
    xo, n = _host_offsets(x_offsets)
    yo, n_y = _host_offsets(y_offsets)
    if n_y != n:
        raise TtsbError(f'{n} pairs in x_offsets, {n_y} in y_offsets')
    if x.dim() != 2 or y.dim() != 2 or x.shape[1] != y.shape[1]:
        raise TtsbError(f'x {tuple(x.shape)} and y {tuple(y.shape)}: need two (frames, ld) arrays of the same ld')
    nb = mcd_dtw_ceps_workspace_bytes(x_offsets, y_offsets, n_ceps, path=path_out is not None)
    ws = torch.empty(nb, dtype=torch.uint8, device=x.device)
    head = (ptr(x), xo, ptr(y), yo, n, int(x.shape[1]), int(first), int(n_ceps), float(kappa), ptr(ws), C.c_int64(nb), ptr(cost_out),
            ptr(path_len_out))
    if path_out is None:
        _check(load().ttsb_mcd_dtw_ceps(*head, _stream()), 'ttsb_mcd_dtw_ceps')
    else:
        _check(load().ttsb_mcd_dtw_ceps_path(*head, ptr(path_out), _stream()), 'ttsb_mcd_dtw_ceps_path')


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
# the STFT family at any supported (n_fft, hop, win_length) (csrc/stft_general.cu); offset tables are host sequences
# ------------------------------------------------------------------------------------------------------------
def _workspace(nb: int, device) -> torch.Tensor:
    if nb < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return torch.empty(nb, dtype=torch.uint8, device=device)


def stft_mel_log_ragged(wav, sample_offsets, frame_offsets, n_fft, hop_length, win_length, mel_basis, band, normalizer, out):
    """Log-mel of a packed ragged batch (include/ttsb.h: ttsb_stft_mel_log_ragged).  wav fp32 (total_samples,), mel_basis fp32
    (n_mels, n_fft/2 + 1), its row bounds band int32 (n_mels, 2) and out fp32 (total_frames, n_mels) on the device."""
    so, n = _host_offsets(sample_offsets)
    fo, n_f = _host_offsets(frame_offsets)
    if n_f != n:
        raise TtsbError(f'{n} clips in sample_offsets, {n_f} in frame_offsets')
    n_mels = mel_basis.shape[0]
    if tuple(band.shape) != (n_mels, 2) or band.dtype != torch.int32:
        raise TtsbError(f'band must be int32 ({n_mels}, 2), got {band.dtype} {tuple(band.shape)}')
    ws = _workspace(int(load().ttsb_stft_mel_log_ragged_workspace_bytes(n, int(n_fft))), wav.device)
    _check(load().ttsb_stft_mel_log_ragged(ptr(wav), so, fo, n, int(n_fft), int(hop_length), int(win_length), ptr(mel_basis), ptr(band), n_mels,
                                           int(normalizer), ptr(ws), ws.numel(), ptr(out), _stream()), 'ttsb_stft_mel_log_ragged')


def mel_to_linear_ex(mel_amp, basis, pinv, band, bin_mels, step, n_iter, out):
    """ttsb_mel_to_linear at basis.shape[1] = n_fft/2 + 1 bins (include/ttsb.h: ttsb_mel_to_linear_ex)."""
    T, n_mels = mel_amp.shape
    _check(load().ttsb_mel_to_linear_ex(ptr(mel_amp), T, n_mels, basis.shape[1], ptr(basis), ptr(pinv), ptr(band), ptr(bin_mels),
                                        float(step), int(n_iter), ptr(out), _stream()), 'ttsb_mel_to_linear_ex')


def stft_complex_ragged(wav, sample_offsets, n_fft, hop_length, win_length, spec_out):
    """librosa.stft of every clip of a packed batch (include/ttsb.h: ttsb_stft_complex_ragged) -> spec_out fp32
    (total_frames, n_fft/2 + 1, 2), clip c with 1 + L_c // hop frames."""
    so, n = _host_offsets(sample_offsets)
    ws = _workspace(int(load().ttsb_stft_complex_ragged_workspace_bytes(n, int(n_fft))), wav.device)
    _check(load().ttsb_stft_complex_ragged(ptr(wav), so, n, int(n_fft), int(hop_length), int(win_length), ptr(ws), ws.numel(),
                                           ptr(spec_out), _stream()), 'ttsb_stft_complex_ragged')


def istft_ragged(spec, frame_offsets, n_fft, hop_length, win_length, wav_out):
    """librosa.istft of every clip of a packed batch (include/ttsb.h: ttsb_istft_ragged): spec fp32 (total_frames, n_fft/2 + 1, 2)
    -> wav_out fp32 (hop (total_frames - n_clips)), clip c at sample hop (frame_offsets[c] - c)."""
    fo, n = _host_offsets(frame_offsets)
    ws = _workspace(int(load().ttsb_istft_ragged_workspace_bytes(spec.shape[0], n, int(n_fft))), spec.device)
    _check(load().ttsb_istft_ragged(ptr(spec), fo, n, int(n_fft), int(hop_length), int(win_length), ptr(ws), ws.numel(), ptr(wav_out),
                                    _stream()), 'ttsb_istft_ragged')


def griffinlim_ragged(magnitude, init_angles, frame_offsets, n_fft, hop_length, win_length, n_iter, momentum, wav_out):
    """Griffin-Lim of every clip of a packed batch (include/ttsb.h: ttsb_griffinlim_ragged).  magnitude fp32 (F, n_fft/2 + 1),
    init_angles complex64 (F, n_fft/2 + 1) and wav_out fp32 (hop (F - n_clips)) on the device."""
    fo, n = _host_offsets(frame_offsets)
    ws = _workspace(int(load().ttsb_griffinlim_ragged_workspace_bytes(magnitude.shape[0], n, int(n_fft))), magnitude.device)
    _check(load().ttsb_griffinlim_ragged(ptr(magnitude), ptr(init_angles), fo, n, int(n_fft), int(hop_length), int(win_length),
                                         int(n_iter), float(momentum), ptr(ws), ws.numel(), ptr(wav_out), _stream()),
           'ttsb_griffinlim_ragged')


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


# ------------------------------------------------------------------------------------------------------------
# ragged-batch Conv1D (the MelGAN and HiFi-GAN generators)
# ------------------------------------------------------------------------------------------------------------
# MelGAN's halo rows on each side of a clip (model/melgan.py): the largest tap shift of its convs, that of the ResStacks'
# dilation-9 convs.  Not a header constant: every call passes its halo (HiFi-GAN's depends on the config).
CONV1D_HALO = 9
HALO_NONE, HALO_REFLECT, HALO_ZERO = 0, 1, 2
CONV1D_EX_MAX_TAPS = 16
CONV1D_EX_MAX_HALO = 64
SUM_NONE, SUM_WRITE, SUM_ADD, SUM_FINISH = 0, 1, 2, 3


def conv1d_workspace_bytes(n_clips: int) -> int:
    n = int(load().ttsb_conv1d_workspace_bytes(int(n_clips)))
    if n < 0:
        raise TtsbError(load().ttsb_last_error().decode())
    return n


class Conv1dExArgs(C.Structure):
    _fields_ = [
        ('n_clips', C.c_int), ('clip_offsets', C.c_void_p), ('halo', C.c_int), ('num_taps', C.c_int),
        ('tap_src', C.c_int * CONV1D_EX_MAX_TAPS), ('tap_shift', C.c_int * CONV1D_EX_MAX_TAPS),
        ('in_hi', C.c_void_p * 2), ('in_lo', C.c_void_p * 2), ('ld_in', C.c_int * 2),
        ('w_hi', C.c_void_p), ('w_lo', C.c_void_p), ('bias', C.c_void_p), ('N', C.c_int), ('up', C.c_int),
        ('res_hi', C.c_void_p), ('res_lo', C.c_void_p), ('sum', C.c_void_p), ('sum_mode', C.c_int), ('sum_div', C.c_float),
        ('out_hi', C.c_void_p), ('out_lo', C.c_void_p), ('act_hi', C.c_void_p), ('act_lo', C.c_void_p), ('ld_out', C.c_int),
        ('out_rows', C.c_int64), ('slope', C.c_float), ('halo_mode', C.c_int), ('precision', C.c_int),
        ('workspace', C.c_void_p), ('workspace_bytes', C.c_int64),
    ]


def conv1d_ex_tc(args: Conv1dExArgs):
    """One ragged-batch conv (include/ttsb.h: ttsb_conv1d_ex_tc).  args.clip_offsets points at a host int32 table."""
    _check(load().ttsb_conv1d_ex_tc(C.byref(args), _stream()), 'ttsb_conv1d_ex_tc')


def conv1d_out_tanh_ex(in_hi, in_lo, channels, halo, clip_offsets, drop_tail, weight, bias, workspace, wav_out):
    """The generators' output layer over a layout of `halo` rows (include/ttsb.h: ttsb_conv1d_out_tanh_ex); clip_offsets: host
    sequence (n_clips + 1)."""
    co, n = _host_offsets(clip_offsets)
    _check(load().ttsb_conv1d_out_tanh_ex(ptr(in_hi), ptr(in_lo), in_hi.shape[-1], int(channels), int(halo), co, n, int(drop_tail),
                                          ptr(weight), C.c_float(bias), ptr(workspace),
                                          C.c_int64(workspace.numel() * workspace.element_size()), ptr(wav_out), _stream()),
           'ttsb_conv1d_out_tanh_ex')


def conv1d_out_clamp_ex(in_hi, in_lo, channels, halo, clip_offsets, drop_tail, weight, bias, workspace, wav_out):
    """conv1d_out_tanh_ex with clamp(., -1, 1) in place of tanh (include/ttsb.h: ttsb_conv1d_out_clamp_ex)."""
    co, n = _host_offsets(clip_offsets)
    _check(load().ttsb_conv1d_out_clamp_ex(ptr(in_hi), ptr(in_lo), in_hi.shape[-1], int(channels), int(halo), co, n, int(drop_tail),
                                           ptr(weight), C.c_float(bias), ptr(workspace),
                                           C.c_int64(workspace.numel() * workspace.element_size()), ptr(wav_out), _stream()),
           'ttsb_conv1d_out_clamp_ex')


def snake_aa_ex(src, dst, channels, halo, clip_offsets, alpha, inv_beta, h_up, h_down, workspace):
    """BigVGAN's anti-aliased Snake activation over a packed ragged layout (include/ttsb.h: ttsb_snake_aa_ex).  src / dst:
    (hi, lo) planes, lo None in bf16; clip_offsets: host sequence (n_clips + 1); alpha / inv_beta: fp32 (channels) device
    tensors; h_up / h_down: 12 host taps each."""
    co, n = _host_offsets(clip_offsets)
    split = src[1] is not None
    up = (C.c_float * 12)(*[float(v) for v in h_up])
    down = (C.c_float * 12)(*[float(v) for v in h_down])
    _check(load().ttsb_snake_aa_ex(ptr(src[0]), ptr(src[1]), ptr(dst[0]), ptr(dst[1]), src[0].shape[-1], int(channels), int(halo), co, n,
                                   ptr(alpha), ptr(inv_beta), C.cast(up, C.c_void_p), C.cast(down, C.c_void_p),
                                   PREC_BF16X3 if split else PREC_BF16, ptr(workspace),
                                   C.c_int64(workspace.numel() * workspace.element_size()), _stream()),
           'ttsb_snake_aa_ex')


# ------------------------------------------------------------------------------------------------------------
# WaveRNN generator (include/ttsb.h: ttsb_wavernn_generate)
# ------------------------------------------------------------------------------------------------------------
WAVERNN_DIMS = 512
WAVERNN_MOL, WAVERNN_RAW = 0, 1
WAVERNN_MAX_TAPS = 7
WAVERNN_MIN_FRAMES = 21
WAVERNN_CTAS = 128
WAVERNN_SEGMENTS = ('sampling', 'gru1', 'gru2', 'fc1', 'fc2', 'fc3')   # the timed segments of a step


# ttsb_wavernn_generate's parameters in order (the stream follows)
WAVERNN_PARAMS = (
    ('frames', C.c_void_p), ('seeds', C.c_void_p), ('n_clips', C.c_int), ('hop', C.c_int), ('batched', C.c_int), ('target', C.c_int),
    ('overlap', C.c_int), ('n_rows', C.c_int), ('n_taps', C.c_int), ('taps', C.c_void_p), ('melp_hi', C.c_void_p),
    ('melp_lo', C.c_void_p), ('ld_melp', C.c_int), ('aux_hi', C.c_void_p), ('aux_lo', C.c_void_p), ('ld_aux', C.c_int),
    ('cond_halo', C.c_int), ('cond_rows', C.c_int64), ('vec', C.c_void_p), ('weights', C.c_void_p), ('mode', C.c_int),
    ('n_classes', C.c_int), ('precision', C.c_int), ('wav_out', C.c_void_p), ('capture', C.c_void_p), ('capture_steps', C.c_int),
    ('samples_out', C.c_void_p), ('timings', C.c_void_p), ('workspace', C.c_void_p), ('workspace_bytes', C.c_int64),
)


def wavernn_workspace_bytes(frames, hop: int, batched: bool, target: int, overlap: int, n_classes: int) -> int:
    tab = (C.c_int32 * len(frames))(*[int(f) for f in frames])
    n = int(load().ttsb_wavernn_workspace_bytes(C.cast(tab, C.c_void_p), len(frames), int(hop), int(bool(batched)), int(target),
                                                int(overlap), int(n_classes)))
    if n < 0:
        raise TtsbError(f'ttsb_wavernn_workspace_bytes: {load().ttsb_last_error().decode()}')
    return n


def wavernn_generate_rc(stream=None, **kw) -> int:
    """ttsb_wavernn_generate with the parameters of WAVERNN_PARAMS by name (missing ones NULL / 0) -> its return code."""
    unknown = set(kw) - {n for n, _ in WAVERNN_PARAMS}
    if unknown:
        raise TypeError(f'ttsb_wavernn_generate has no parameter {sorted(unknown)[0]}')
    return int(load().ttsb_wavernn_generate(*[kw.get(n, None if t is C.c_void_p else 0) for n, t in WAVERNN_PARAMS], stream))


def wavernn_generate(**kw):
    """One WaveRNN generation (include/ttsb.h: ttsb_wavernn_generate); frames / seeds point at host tables."""
    _check(wavernn_generate_rc(_stream(), **kw), 'ttsb_wavernn_generate')
