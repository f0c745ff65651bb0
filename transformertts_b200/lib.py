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
    """Load libttsb.so (built in-tree by transformertts_b200.build) and declare the C signature of every entry point
    (SIGNATURES).  Raises TtsbError when the library or one of its entry points is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise TtsbError(f'{_LIB_PATH} not found -- run `python -m transformertts_b200.build` (no CPU fallback exists)')
    lib = C.CDLL(str(_LIB_PATH))
    for name, (restype, argtypes) in SIGNATURES.items():
        if not hasattr(lib, name):
            raise TtsbError(f'libttsb.so does not export {name}')
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def _check(rc: int, what: str):
    if rc != 0:
        raise TtsbError(f'{what} failed ({rc}): {load().ttsb_last_error().decode()}')


def _call(name: str, *args):
    """Entry point `name` with `args` and the current stream; raises TtsbError on a nonzero return code."""
    _check(getattr(load(), name)(*args, _stream()), name)


def _workspace_size(name: str, *args) -> int:
    """The byte count the workspace query `name` returns; raises TtsbError when it refuses the arguments (a negative size)."""
    nb = getattr(load(), name)(*args)
    if nb < 0:
        raise TtsbError(f'{name} failed ({nb}): {load().ttsb_last_error().decode()}')
    return nb


def _workspace(nb: int, device) -> torch.Tensor:
    return torch.empty(nb, dtype=torch.uint8, device=device)


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
    return load().ttsb_launch_count()


def reset_launch_count():
    load().ttsb_reset_launch_count()


def add_launch_count(n: int):
    load().ttsb_add_launch_count(n)


def set_dropout_salt(salt_dev: torch.Tensor):
    """salt_dev: int32/uint32 CUDA tensor with one element (see include/ttsb.h)."""
    _call('ttsb_set_dropout_salt', ptr(salt_dev))


# ------------------------------------------------------------------------------------------------------------
# thin typed wrappers (shapes are taken from the tensors; all tensors must be contiguous)
# ------------------------------------------------------------------------------------------------------------
def pack_weight(w_kn: torch.Tensor, n_pad: int, split: bool):
    """Keras (K,N) fp32 kernel (Conv1D (k,Cin,Cout) is reshaped to (k*Cin, Cout)) -> bf16 hi/lo [n_pad, K]."""
    w2 = w_kn.reshape(-1, w_kn.shape[-1]).contiguous().float()
    K, N = w2.shape
    hi = torch.empty((n_pad, K), dtype=torch.bfloat16, device=w2.device)
    lo = torch.empty_like(hi) if split else None
    _call('ttsb_pack_weight', ptr(w2), K, N, n_pad, ptr(hi), ptr(lo))
    return hi, lo


def upload_pack_descs(descs, device) -> torch.Tensor:
    """ctypes PackDesc list -> device byte tensor (kept alive by the caller)."""
    arr = (PackDesc * len(descs))(*descs)
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
    return host.to(device)


def repack_batched(descs_dev: torch.Tensor, n: int):
    _call('ttsb_repack_batched', ptr(descs_dev), n)


def split_bf16(x: torch.Tensor, split: bool):
    x = x.contiguous().float()
    hi = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi) if split else None
    _call('ttsb_split_bf16', ptr(x), x.numel(), ptr(hi), ptr(lo))
    return hi, lo


def linear_fwd(args: GemmArgs):
    _call('ttsb_linear_fwd', C.byref(args))


def layernorm_fwd(x, gamma, beta, d, eps, row_len, out_f32, out_hi, out_lo):
    B, T, ld = x.shape
    _call('ttsb_layernorm_fwd', ptr(x), ptr(gamma), ptr(beta), B, T, d, ld, eps, ptr(row_len), ptr(out_f32), ptr(out_hi), ptr(out_lo))


def mha_fwd(args: MhaArgs):
    _call('ttsb_mha_fwd', C.byref(args))


def embed_ln_pe_fwd(tokens, emb, gamma, beta, pe, pos_scalar, eps, out_f32, out_hi, out_lo, drop=(0.0, 0, 0)):
    B, T = tokens.shape
    vocab, d = emb.shape
    _call('ttsb_embed_ln_pe_train_fwd', ptr(tokens), ptr(emb), ptr(gamma), ptr(beta), ptr(pe), ptr(pos_scalar), B, T, d, vocab, eps,
          drop[0], drop[1], drop[2], ptr(out_f32), ptr(out_hi), ptr(out_lo))


def expand_ln_pe_fwd(x, idx, gamma, beta, pe, pos_scalar, eps, out_f32, out_hi, out_lo, drop=(0.0, 0, 0)):
    B, Tp, d = x.shape
    Tm = idx.shape[1]
    _call('ttsb_expand_ln_pe_train_fwd', ptr(x), ptr(idx), ptr(gamma), ptr(beta), ptr(pe), ptr(pos_scalar), B, Tp, Tm, d, eps, drop[0],
          drop[1], drop[2], ptr(out_f32), ptr(out_hi), ptr(out_lo))


def length_regulate_fwd(x, idx, out):
    B, Tp, d = x.shape
    Tm = idx.shape[1]
    _call('ttsb_length_regulate_fwd', ptr(x), ptr(idx), B, Tp, Tm, d, ptr(out))


def durations_to_int(dur, scalar, max_mask, min_mask, out_int, out_len):
    B, Tp = dur.shape
    _call('ttsb_durations_to_int', ptr(dur), scalar, ptr(max_mask), ptr(min_mask), B, Tp, ptr(out_int), ptr(out_len))


def expand_indices(dur_int, Tm, out_idx):
    B, Tp = dur_int.shape
    _call('ttsb_expand_indices', ptr(dur_int), B, Tp, Tm, ptr(out_idx))


def statpred_head_fwd(h, C_in, w, bias, relu, row_len, out):
    B, T, ldh = h.shape
    _call('ttsb_statpred_head_fwd', ptr(h), ldh, C_in, ptr(w), ptr(bias), relu, ptr(row_len), B, T, ptr(out))


def pitch_embed_add_fwd(x, pitch, w, bias, out):
    B, T, d = x.shape
    _call('ttsb_pitch_embed_add_fwd', ptr(x), ptr(pitch), ptr(w), ptr(bias), B, T, d, ptr(out))


def mel_lengths(mel, padding_value, out):
    B, T, Cc = mel.shape
    _call('ttsb_mel_lengths', ptr(mel), B, T, Cc, padding_value, ptr(out))


def phoneme_lengths(ph, padding, out):
    B, T = ph.shape
    _call('ttsb_phoneme_lengths', ptr(ph), B, T, padding, ptr(out))


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
    _call('ttsb_stft_mel_log', ptr(wav), n_clips, n_samples, ptr(mel_basis), bp, n_mels, normalizer, ptr(out))


def _host_offsets(offsets):
    """int32 (n + 1) offset table in host memory -> (ctypes array, n)."""
    import numpy as np
    a = np.ascontiguousarray(np.asarray(offsets.cpu() if torch.is_tensor(offsets) else offsets, dtype=np.int64))
    if a.ndim != 1 or len(a) < 2 or a.min() < 0 or a.max() > 2**31 - 1:
        raise TtsbError(f'offset table must be 1-D, at least 2 entries, within int32; got shape {a.shape}')
    return (C.c_int32 * len(a))(*a.tolist()), len(a) - 1


def _offset_pair(unit: str = 'clips', **tables):
    """Two host offset tables over the same clips (or pairs), given by name -> (ctypes array, ctypes array, n).  Refuses
    tables that describe different numbers of them."""
    (name_a, a), (name_b, b) = tables.items()
    a, n = _host_offsets(a)
    b, n_b = _host_offsets(b)
    if n_b != n:
        raise TtsbError(f'{n} {unit} in {name_a}, {n_b} in {name_b}')
    return a, b, n


def stft_mel_log_batch(wav, sample_offsets, frame_offsets, mel_basis, band, normalizer, out):
    """Log-mel of a packed ragged batch (include/ttsb.h: ttsb_stft_mel_log_batch).  wav fp32 (total_samples,) and out fp32
    (total_frames, n_mels) on the device; the offset tables (n_clips + 1) and band int32 (n_mels, 2) are host tables."""
    so, fo, n = _offset_pair(sample_offsets=sample_offsets, frame_offsets=frame_offsets)
    nb = _workspace_size('ttsb_stft_mel_log_batch_workspace_bytes', n)
    keep, bp = _host_band(band, mel_basis.shape[0])
    ws = _workspace(nb, wav.device)
    _call('ttsb_stft_mel_log_batch', ptr(wav), so, fo, n, ptr(mel_basis), bp, mel_basis.shape[0], normalizer, ptr(ws), nb, ptr(out))


def pitch_workspace_bytes(sample_offsets, fs, frame_period_ms, f0_floor=71.0, f0_ceil=800.0, channels_in_octave=2.0) -> int:
    so, n = _host_offsets(sample_offsets)
    return _workspace_size('ttsb_pitch_workspace_bytes', so, n, fs, frame_period_ms, f0_floor, f0_ceil, channels_in_octave)


def pitch_dio_stonemask(wav, sample_offsets, fs, frame_period_ms, f0_offsets, f0_out, workspace, f0_floor=71.0, f0_ceil=800.0,
                        channels_in_octave=2.0, allowed_range=0.1):
    """f0 of a packed ragged batch by DIO + StoneMask (include/ttsb.h: ttsb_pitch_dio_stonemask).  wav fp32 and f0_out fp64 on
    the device; the offset tables are host sequences; workspace: pitch_workspace_bytes(...) bytes on the device."""
    so, fo, n = _offset_pair(sample_offsets=sample_offsets, f0_offsets=f0_offsets)
    _call('ttsb_pitch_dio_stonemask', ptr(wav), so, n, fs, frame_period_ms, f0_floor, f0_ceil, channels_in_octave, allowed_range, fo,
          ptr(f0_out), ptr(workspace), workspace.nbytes)


def _host_rates(rates, n: int):
    import numpy as np
    a = np.asarray(rates.cpu() if torch.is_tensor(rates) else rates, dtype=np.int64).reshape(-1)
    if len(a) != n or (len(a) and (a.min() < -2**31 or a.max() > 2**31 - 1)):
        raise TtsbError(f'{len(a)} source rates for {n} clips (int32 each)')
    return (C.c_int32 * n)(*a.tolist())


def resample_batch_workspace_bytes(sample_offsets, src_rates, dst_rate: int, n_window: int) -> int:
    so, n = _host_offsets(sample_offsets)
    return _workspace_size('ttsb_resample_batch_workspace_bytes', so, _host_rates(src_rates, n), n, dst_rate, n_window)


def resample_batch(wav, sample_offsets, src_rates, dst_rate, half_window, out_offsets, out):
    """Resample every clip of a packed ragged batch to dst_rate (include/ttsb.h: ttsb_resample_batch).  wav fp32, half_window
    fp64 and out fp32 on the device; the offset tables (n_clips + 1) and src_rates (n_clips) are host sequences."""
    so, oo, n = _offset_pair(sample_offsets=sample_offsets, out_offsets=out_offsets)
    rates = _host_rates(src_rates, n)
    nb = resample_batch_workspace_bytes(sample_offsets, src_rates, dst_rate, half_window.numel())
    ws = _workspace(nb, wav.device)
    _call('ttsb_resample_batch', ptr(wav), so, rates, n, dst_rate, ptr(half_window), half_window.numel(), oo, ptr(ws), nb, ptr(out))


def trim_silence_workspace_bytes(sample_offsets) -> int:
    so, n = _host_offsets(sample_offsets)
    return _workspace_size('ttsb_trim_silence_workspace_bytes', so, n)


def trim_silence_bounds(wav, sample_offsets, top_db: float, bounds):
    """[start, end) of the non-silent part of every clip of a packed ragged batch (include/ttsb.h: ttsb_trim_silence_bounds).
    wav fp32 and bounds int32 (n_clips, 2) on the device; sample_offsets (n_clips + 1) is a host sequence."""
    so, n = _host_offsets(sample_offsets)
    nb = trim_silence_workspace_bytes(sample_offsets)
    ws = _workspace(nb, wav.device)
    _call('ttsb_trim_silence_bounds', ptr(wav), so, n, top_db, ptr(ws), nb, ptr(bounds))


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
    return _workspace_size('ttsb_flac_decode_workspace_bytes', bo, table, n)


def flac_decode_batch(data, byte_offsets, infos, mono_out, status_out, pcm_out=None):
    """Decode the frame bytes of every file of a packed batch of FLAC streams (include/ttsb.h: ttsb_flac_decode_batch).  data uint8,
    mono_out fp32, status_out int32 (n_files, 2) and pcm_out int32 (optional) on the device; byte_offsets (n_files + 1) and infos
    (flac_decode_workspace_bytes) are host sequences."""
    bo, table, n = _flac_tables(byte_offsets, infos)
    nb = flac_decode_workspace_bytes(byte_offsets, infos)
    ws = _workspace(max(nb, 16), mono_out.device)
    _call('ttsb_flac_decode_batch', ptr(data) if data.numel() else None, bo, table, n, ptr(mono_out), ptr(pcm_out), ptr(status_out),
          ptr(ws), nb)


# the longest shorter side of a pair ttsb_mcd_dtw takes (include/ttsb.h: TTSB_MCD_DTW_MAX_FRAMES)
MCD_DTW_MAX_FRAMES = 4096


def mcd_dtw_workspace_bytes(x_offsets, y_offsets, n_ceps: int) -> int:
    xo, yo, n = _offset_pair('pairs', x_offsets=x_offsets, y_offsets=y_offsets)
    return _workspace_size('ttsb_mcd_dtw_workspace_bytes', xo, yo, n, n_ceps)


def mcd_dtw(x, x_offsets, y, y_offsets, dct, kappa, cost_out, path_len_out):
    """DTW cost and path length of every pair of a packed ragged batch of log-mel sequences (include/ttsb.h: ttsb_mcd_dtw).
    x, y fp32 (frames, n_mels), dct fp64 (n_ceps, n_mels), cost_out fp64 (n_pairs,) and path_len_out int32 (n_pairs,) on the
    device; the offset tables (n_pairs + 1) are host sequences."""
    xo, yo, n = _offset_pair('pairs', x_offsets=x_offsets, y_offsets=y_offsets)
    n_ceps, n_mels = dct.shape
    nb = mcd_dtw_workspace_bytes(x_offsets, y_offsets, n_ceps)
    ws = _workspace(nb, x.device)
    _call('ttsb_mcd_dtw', ptr(x), xo, ptr(y), yo, n, n_mels, ptr(dct), n_ceps, kappa, ptr(ws), nb, ptr(cost_out), ptr(path_len_out))


# the most cells (Tx * Ty) of a pair ttsb_mcd_dtw_path takes (include/ttsb.h: TTSB_MCD_DTW_PATH_MAX_CELLS)
MCD_DTW_PATH_MAX_CELLS = 16777216


def mcd_dtw_path_workspace_bytes(x_offsets, y_offsets, n_ceps: int) -> int:
    xo, yo, n = _offset_pair('pairs', x_offsets=x_offsets, y_offsets=y_offsets)
    return _workspace_size('ttsb_mcd_dtw_path_workspace_bytes', xo, yo, n, n_ceps)


def mcd_dtw_path(x, x_offsets, y, y_offsets, dct, kappa, cost_out, path_len_out, path_out):
    """mcd_dtw that also writes each pair's warping path (include/ttsb.h: ttsb_mcd_dtw_path): path_out int32 (sum of
    Tx + Ty - 1, 2) on the device, pair p's path from row sum_{q<p} (Tx_q + Ty_q - 1)."""
    xo, yo, n = _offset_pair('pairs', x_offsets=x_offsets, y_offsets=y_offsets)
    n_ceps, n_mels = dct.shape
    nb = mcd_dtw_path_workspace_bytes(x_offsets, y_offsets, n_ceps)
    ws = _workspace(nb, x.device)
    _call('ttsb_mcd_dtw_path', ptr(x), xo, ptr(y), yo, n, n_mels, ptr(dct), n_ceps, kappa, ptr(ws), nb, ptr(cost_out),
          ptr(path_len_out), ptr(path_out))


def cheaptrick_workspace_bytes(sample_offsets, f0_offsets, fs: int, frame_period_ms: float, fft_size: int) -> int:
    so, fo, n = _offset_pair(sample_offsets=sample_offsets, f0_offsets=f0_offsets)
    return _workspace_size('ttsb_cheaptrick_workspace_bytes', so, fo, n, fs, frame_period_ms, fft_size)


def cheaptrick(wav, sample_offsets, fs, frame_period_ms, f0, f0_offsets, q1, fft_size, envelope_out):
    """WORLD's CheapTrick spectral envelope of every frame of a packed ragged batch (include/ttsb.h: ttsb_cheaptrick).  wav fp32,
    f0 fp64 (frames,) and envelope_out fp64 (frames, fft_size / 2 + 1) on the device; the offset tables are host sequences."""
    so, n = _host_offsets(sample_offsets)
    fo, _ = _host_offsets(f0_offsets)
    nb = cheaptrick_workspace_bytes(sample_offsets, f0_offsets, fs, frame_period_ms, fft_size)
    ws = _workspace(nb, wav.device)
    _call('ttsb_cheaptrick', ptr(wav), so, n, fs, frame_period_ms, ptr(f0), fo, q1, fft_size, ptr(ws), nb, ptr(envelope_out))


def sp2mc(envelope, matrix, mc_out):
    """mc = matrix . log(envelope) per frame (include/ttsb.h: ttsb_sp2mc).  envelope fp64 (frames, fft_size / 2 + 1), matrix fp64
    (order + 1, fft_size / 2 + 1) and mc_out fp64 (frames, order + 1) on the device."""
    n_frames, nb = envelope.shape
    if matrix.dim() != 2 or matrix.shape[1] != nb or tuple(mc_out.shape) != (n_frames, matrix.shape[0]):
        raise TtsbError(f'envelope {tuple(envelope.shape)}, matrix {tuple(matrix.shape)} and mc_out {tuple(mc_out.shape)}: need '
                        f'(frames, bins), (order + 1, bins) and (frames, order + 1)')
    _call('ttsb_sp2mc', ptr(envelope), n_frames, 2 * (nb - 1), ptr(matrix), matrix.shape[0] - 1, ptr(mc_out))


def mcd_dtw_ceps_workspace_bytes(x_offsets, y_offsets, n_ceps: int, path: bool = False) -> int:
    xo, yo, n = _offset_pair('pairs', x_offsets=x_offsets, y_offsets=y_offsets)
    name = 'ttsb_mcd_dtw_ceps_path_workspace_bytes' if path else 'ttsb_mcd_dtw_ceps_workspace_bytes'
    return _workspace_size(name, xo, yo, n, n_ceps)


def mcd_dtw_ceps(x, x_offsets, y, y_offsets, first: int, n_ceps: int, kappa, cost_out, path_len_out, path_out=None):
    """ttsb_mcd_dtw_ceps (ttsb_mcd_dtw_ceps_path when path_out is given) over caller-given cepstra: x, y fp64 (frames, ld) on the
    device, columns first .. first + n_ceps - 1 scored; cost_out, path_len_out and path_out as mcd_dtw / mcd_dtw_path take them."""
    xo, yo, n = _offset_pair('pairs', x_offsets=x_offsets, y_offsets=y_offsets)
    if x.dim() != 2 or y.dim() != 2 or x.shape[1] != y.shape[1]:
        raise TtsbError(f'x {tuple(x.shape)} and y {tuple(y.shape)}: need two (frames, ld) arrays of the same ld')
    nb = mcd_dtw_ceps_workspace_bytes(x_offsets, y_offsets, n_ceps, path=path_out is not None)
    ws = _workspace(nb, x.device)
    head = (ptr(x), xo, ptr(y), yo, n, x.shape[1], first, n_ceps, kappa, ptr(ws), nb, ptr(cost_out), ptr(path_len_out))
    if path_out is None:
        _call('ttsb_mcd_dtw_ceps', *head)
    else:
        _call('ttsb_mcd_dtw_ceps_path', *head, ptr(path_out))


# ------------------------------------------------------------------------------------------------------------
# training-step kernels
# ------------------------------------------------------------------------------------------------------------
def bgemm(args: BgemmArgs):
    _call('ttsb_bgemm', C.byref(args))


def rowdot_heads(x, y, H, dh, out):
    B, T, ld = x.shape
    _call('ttsb_rowdot_heads', ptr(x), ptr(y), B, T, H, dh, ld, ptr(out))


def wgrad(args: WgradArgs):
    _call('ttsb_wgrad', C.byref(args))


SOFTMAX_CAUSAL, SOFTMAX_FULL_QUERIES = 1, 2


def softmax_fwd(S, B, H, T, Tk, ld, kv_len, drop_p, seed, site, P_pre, P_drop, flags=0):
    _call('ttsb_softmax_fwd', ptr(S), B, H, T, Tk, ld, ptr(kv_len), drop_p, seed, site, flags, ptr(P_pre), ptr(P_drop))


def attn_probs_supported(dh: int, ld_p: int) -> bool:
    return bool(load().ttsb_attn_probs_supported(dh, ld_p))


def attn_probs_fwd(qkv, ld, q_col0, k_col0, B, H, T, dh, kv_len, scale, drop_p, seed, site, P_pre, P_drop, ld_p):
    """P_pre = softmax(scale * Q K^T), P_drop = dropout(P_pre) in one kernel (include/ttsb.h: ttsb_attn_probs_fwd)."""
    _call('ttsb_attn_probs_fwd', ptr(qkv), ld, q_col0, k_col0, B, H, T, dh, ptr(kv_len), scale, drop_p, seed, site, ptr(P_pre),
          ptr(P_drop), ld_p)


def attn_ds_bwd(dO, ld_do, do_col0, v, ld_v, v_col0, B, H, T, dh, kv_len, P_pre, D, scale, drop_p, seed, site, dS, ld_p):
    """dS = scale * P_pre * (dropout(dO V^T) - D) in one kernel (include/ttsb.h: ttsb_attn_ds_bwd)."""
    _call('ttsb_attn_ds_bwd', ptr(dO), ld_do, do_col0, ptr(v), ld_v, v_col0, B, H, T, dh, ptr(kv_len), ptr(P_pre), ptr(D), scale,
          drop_p, seed, site, ptr(dS), ld_p)


def softmax_bwd(P_pre, dP, B, H, T, Tk, ld, kv_len, scale, drop_p, seed, site, dS, flags=0):
    _call('ttsb_softmax_bwd', ptr(P_pre), ptr(dP), B, H, T, Tk, ld, ptr(kv_len), scale, drop_p, seed, site, flags, ptr(dS))


def layernorm_bwd(dz, u, gamma, B, T, Cc, ld, eps, row_len, relu_mask, du, g_bf16, dgamma, dbeta, pre_drop=(0.0, 0),
                  post_drop=(0.0, 0), seed=0, dbias=None):
    _call('ttsb_layernorm_bwd', ptr(dz), ptr(u), ptr(gamma), B, T, Cc, ld, eps, ptr(row_len), relu_mask, pre_drop[0], pre_drop[1],
          post_drop[0], post_drop[1], seed, ptr(du), ptr(g_bf16), ptr(dgamma), ptr(dbeta), ptr(dbias))


def colsum_bf16(x, rows, Cc, ld, out):
    _call('ttsb_colsum_bf16', ptr(x), rows, Cc, ld, ptr(out))


def relu_bwd(dy, h):
    _call('ttsb_relu_bwd', ptr(dy), ptr(h), dy.numel())


def relu_bwd_colsum(dy, h, colsum):
    """dy *= (h > 0) in place and colsum += column sums of the result (the bias gradient of the layer that produced h)."""
    Cc = dy.shape[-1]
    _call('ttsb_relu_bwd_colsum', ptr(dy), ptr(h), dy.numel() // Cc, Cc, ptr(colsum))


def colsum_bf16_x3(x, rows, seg, ld, out0, out1, out2):
    _call('ttsb_colsum_bf16_x3', ptr(x), rows, seg, ld, ptr(out0), ptr(out1), ptr(out2))


def cast_bf16_pad(x, rows, Cc, out, ld_out):
    _call('ttsb_cast_bf16_pad', ptr(x), rows, Cc, ptr(out), ld_out)


def mae_loss(pred, B, Tp, Tt, Cc, target, weight, loss_out, grad):
    tf = ptr(target) if target.dtype == torch.float32 else None
    ti = ptr(target) if target.dtype == torch.int32 else None
    _call('ttsb_mae_loss', ptr(pred), B, Tp, Tt, Cc, tf, ti, weight, ptr(loss_out), ptr(grad))


def scaled_ce_loss(logits, Tt, Cc, targets, index, scaling, loss_out, grad_weight=1.0, grad=None):
    B, Tp, ld = logits.shape
    _call('ttsb_scaled_ce_loss', ptr(logits), B, Tp, Tt, Cc, ld, ptr(targets), index, scaling, ptr(loss_out), grad_weight, ptr(grad),
          grad.shape[-1] if grad is not None else 0)


def diag_loss_train(P_bf16, B, H, Tq, Tk, ld, q_len, k_len, loss_scale, loss_out, grad_scale, dP):
    _call('ttsb_diag_loss_train', ptr(P_bf16), B, H, Tq, Tk, ld, ptr(q_len), ptr(k_len), loss_scale, ptr(loss_out), grad_scale, ptr(dP))


def attention_scores(att, mel_len, phon_len, r, scores):
    B, H, Tq, Tk = att.shape
    _call('ttsb_attention_scores', ptr(att), B, H, Tq, Tk, ptr(mel_len), ptr(phon_len), r, ptr(scores))


def durations_from_attention(att, mel_len, phon_len, scores, weighted, scratch, durations):
    B, H, Tq, Tk = att.shape
    _call('ttsb_durations_from_attention', ptr(att), B, H, Tq, Tk, ptr(mel_len), ptr(phon_len), ptr(scores), int(bool(weighted)),
          ptr(scratch), ptr(durations))


def pitch_per_char(pitch, pitch_len, durations, n_chars, pitch_mean, pitch_std, out):
    B, Tm = pitch.shape
    Tp = durations.shape[1]
    _call('ttsb_pitch_per_char', ptr(pitch), B, Tm, ptr(pitch_len), ptr(durations), Tp, ptr(n_chars), pitch_mean, pitch_std, ptr(out))


def diag_loss(att, q_len, k_len, loss_out):
    B, H, Tq, Tk = att.shape
    _call('ttsb_diag_loss', ptr(att), B, H, Tq, Tk, ptr(q_len), ptr(k_len), ptr(loss_out))


def expand_bwd(dm, dur_int, dx):
    B, Tm, d = dm.shape
    Tp = dur_int.shape[1]
    _call('ttsb_expand_bwd', ptr(dm), ptr(dur_int), B, Tp, Tm, d, ptr(dx))


def embedding_bwd(dx, tokens, demb):
    B, T, d = dx.shape
    _call('ttsb_embedding_bwd', ptr(dx), ptr(tokens), B, T, d, demb.shape[0], ptr(demb))


def pe_scalar_bwd(g, pe, dscalar, drop=(0.0, 0, 0)):
    B, T, d = g.shape
    _call('ttsb_pe_scalar_bwd', ptr(g), ptr(pe), B, T, d, drop[0], drop[1], drop[2], ptr(dscalar))


def pitch_embed_bwd(g, pitch, w, bias, dw, db):
    B, T, d = g.shape
    _call('ttsb_pitch_embed_bwd', ptr(g), ptr(pitch), ptr(w), ptr(bias), B, T, d, ptr(dw), ptr(db))


def statpred_head_bwd(gout, out, h, C_in, w, relu, row_len, dh, dw, db):
    B, T, ldh = h.shape
    _call('ttsb_statpred_head_bwd', ptr(gout), ptr(out), ptr(h), ldh, C_in, ptr(w), relu, ptr(row_len), B, T, ptr(dh), ptr(dw), ptr(db))


def adam_tf_step(param, grad, m, v, lr_t, beta1, beta2, eps, grad_scale=1.0):
    _call('ttsb_adam_tf_step', ptr(param), ptr(grad), ptr(m), ptr(v), param.numel(), lr_t, beta1, beta2, eps, grad_scale)


# ------------------------------------------------------------------------------------------------------------
# data-parallel gradient exchange (NCCL behind the C ABI)
# ------------------------------------------------------------------------------------------------------------
def dp_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    _check(load().ttsb_dp_unique_id(buf), 'ttsb_dp_unique_id')
    return buf.raw


def dp_init(unique_id: bytes, rank: int, world: int):
    comm = C.c_void_p()
    _check(load().ttsb_dp_init(unique_id, rank, world, C.byref(comm)), 'ttsb_dp_init')
    return comm


def dp_allreduce_bucket(comm, buf: torch.Tensor, stream: int):
    """In-place sum of the contiguous fp32 CUDA tensor `buf` across ranks on the raw stream handle `stream`."""
    _check(load().ttsb_dp_allreduce_bucket(comm, ptr(buf), buf.numel(), stream), 'ttsb_dp_allreduce_bucket')


def dp_destroy(comm):
    _check(load().ttsb_dp_destroy(comm), 'ttsb_dp_destroy')


# ------------------------------------------------------------------------------------------------------------
# mel -> waveform (Griffin-Lim)
# ------------------------------------------------------------------------------------------------------------
def mel_to_linear(mel_amp, basis, pinv, band, bin_mels, step, n_iter, out):
    T, n_mels = mel_amp.shape
    _call('ttsb_mel_to_linear', ptr(mel_amp), T, n_mels, ptr(basis), ptr(pinv), ptr(band), ptr(bin_mels), step, n_iter, ptr(out))


def stft_complex(wav, spec_out):
    _call('ttsb_stft_complex', ptr(wav), wav.numel(), ptr(spec_out))


def istft(spec, workspace, wav_out):
    T = spec.shape[0]
    _call('ttsb_istft', ptr(spec), T, ptr(workspace), workspace.nbytes, ptr(wav_out))


def istft_workspace_bytes(n_frames: int) -> int:
    return _workspace_size('ttsb_istft_workspace_bytes', n_frames)


def griffinlim_update(rebuilt, previous, magnitude, momentum, projected_out):
    _call('ttsb_griffinlim_update', ptr(rebuilt), ptr(previous), ptr(magnitude), momentum, magnitude.numel(), ptr(projected_out))


def griffinlim_batch_workspace_bytes(total_frames: int, n_clips: int) -> int:
    return _workspace_size('ttsb_griffinlim_batch_workspace_bytes', total_frames, n_clips)


def griffinlim_batch(magnitude, init_angles, frame_offsets, n_iter, momentum, workspace, wav_out):
    """Griffin-Lim of every clip of a packed batch (include/ttsb.h: ttsb_griffinlim_batch).  magnitude fp32 (F, 513),
    init_angles complex64 (F, 513), frame_offsets int32 (n_clips + 1) on the device, wav_out fp32 (256 (F - n_clips))."""
    F = magnitude.shape[0]
    _call('ttsb_griffinlim_batch', ptr(magnitude), ptr(init_angles), ptr(frame_offsets), frame_offsets.numel() - 1, F, n_iter, momentum,
          ptr(workspace), workspace.nbytes, ptr(wav_out))


# ------------------------------------------------------------------------------------------------------------
# the STFT family at any supported (n_fft, hop, win_length) (csrc/stft_general.cu); offset tables are host sequences
# ------------------------------------------------------------------------------------------------------------
def stft_mel_log_ragged(wav, sample_offsets, frame_offsets, n_fft, hop_length, win_length, mel_basis, band, normalizer, out):
    """Log-mel of a packed ragged batch (include/ttsb.h: ttsb_stft_mel_log_ragged).  wav fp32 (total_samples,), mel_basis fp32
    (n_mels, n_fft/2 + 1), its row bounds band int32 (n_mels, 2) and out fp32 (total_frames, n_mels) on the device."""
    so, fo, n = _offset_pair(sample_offsets=sample_offsets, frame_offsets=frame_offsets)
    n_mels = mel_basis.shape[0]
    if tuple(band.shape) != (n_mels, 2) or band.dtype != torch.int32:
        raise TtsbError(f'band must be int32 ({n_mels}, 2), got {band.dtype} {tuple(band.shape)}')
    ws = _workspace(_workspace_size('ttsb_stft_mel_log_ragged_workspace_bytes', n, n_fft), wav.device)
    _call('ttsb_stft_mel_log_ragged', ptr(wav), so, fo, n, n_fft, hop_length, win_length, ptr(mel_basis), ptr(band), n_mels, normalizer,
          ptr(ws), ws.numel(), ptr(out))


def mel_to_linear_ex(mel_amp, basis, pinv, band, bin_mels, step, n_iter, out):
    """ttsb_mel_to_linear at basis.shape[1] = n_fft/2 + 1 bins (include/ttsb.h: ttsb_mel_to_linear_ex)."""
    T, n_mels = mel_amp.shape
    _call('ttsb_mel_to_linear_ex', ptr(mel_amp), T, n_mels, basis.shape[1], ptr(basis), ptr(pinv), ptr(band), ptr(bin_mels), step, n_iter,
          ptr(out))


def stft_complex_ragged(wav, sample_offsets, n_fft, hop_length, win_length, spec_out):
    """librosa.stft of every clip of a packed batch (include/ttsb.h: ttsb_stft_complex_ragged) -> spec_out fp32
    (total_frames, n_fft/2 + 1, 2), clip c with 1 + L_c // hop frames."""
    so, n = _host_offsets(sample_offsets)
    ws = _workspace(_workspace_size('ttsb_stft_complex_ragged_workspace_bytes', n, n_fft), wav.device)
    _call('ttsb_stft_complex_ragged', ptr(wav), so, n, n_fft, hop_length, win_length, ptr(ws), ws.numel(), ptr(spec_out))


def istft_ragged(spec, frame_offsets, n_fft, hop_length, win_length, wav_out):
    """librosa.istft of every clip of a packed batch (include/ttsb.h: ttsb_istft_ragged): spec fp32 (total_frames, n_fft/2 + 1, 2)
    -> wav_out fp32 (hop (total_frames - n_clips)), clip c at sample hop (frame_offsets[c] - c)."""
    fo, n = _host_offsets(frame_offsets)
    ws = _workspace(_workspace_size('ttsb_istft_ragged_workspace_bytes', spec.shape[0], n, n_fft), spec.device)
    _call('ttsb_istft_ragged', ptr(spec), fo, n, n_fft, hop_length, win_length, ptr(ws), ws.numel(), ptr(wav_out))


def griffinlim_ragged(magnitude, init_angles, frame_offsets, n_fft, hop_length, win_length, n_iter, momentum, wav_out):
    """Griffin-Lim of every clip of a packed batch (include/ttsb.h: ttsb_griffinlim_ragged).  magnitude fp32 (F, n_fft/2 + 1),
    init_angles complex64 (F, n_fft/2 + 1) and wav_out fp32 (hop (F - n_clips)) on the device."""
    fo, n = _host_offsets(frame_offsets)
    ws = _workspace(_workspace_size('ttsb_griffinlim_ragged_workspace_bytes', magnitude.shape[0], n, n_fft), magnitude.device)
    _call('ttsb_griffinlim_ragged', ptr(magnitude), ptr(init_angles), fo, n, n_fft, hop_length, win_length, n_iter, momentum, ptr(ws),
          ws.numel(), ptr(wav_out))


# ------------------------------------------------------------------------------------------------------------
# cached autoregressive decoding (Aligner.predict_batch)
# ------------------------------------------------------------------------------------------------------------
def decode_attn_workspace_bytes(B: int, H: int, dh: int) -> int:
    return _workspace_size('ttsb_decode_attn_workspace_bytes', B, H, dh)


def decode_attn(args: DecodeAttnArgs):
    _call('ttsb_decode_attn', C.byref(args))


def decode_prologue(x, pos, gamma, beta, pe, pos_scalar, eps, out_f32, out_hi, out_lo):
    """out[b] = LayerNorm(x[b]) + pos_scalar * pe[pos[b]]; x fp32 (B, d)."""
    d = x.shape[-1]
    B = x.numel() // d
    _call('ttsb_decode_prologue', ptr(x), ptr(pos), ptr(gamma), ptr(beta), ptr(pe), pe.shape[0], ptr(pos_scalar), B, d, eps, ptr(out_f32),
          ptr(out_hi), ptr(out_lo))


def decode_commit(post, B, r, mel, stop_col, stop_index, max_iters, mel_out, stop_out, next_hi, next_lo, pos, done, n, all_done):
    """End of one decode iteration (include/ttsb.h: ttsb_decode_commit); post fp32 (B*r, ld_post), next_hi / next_lo (B, ld_next)."""
    _call('ttsb_decode_commit', ptr(post), post.shape[-1], B, r, mel, stop_col, stop_index, max_iters, ptr(mel_out), ptr(stop_out),
          ptr(next_hi), ptr(next_lo), next_hi.shape[-1], ptr(pos), ptr(done), ptr(n), ptr(all_done))


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
    return _workspace_size('ttsb_conv1d_workspace_bytes', n_clips)


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
    _call('ttsb_conv1d_ex_tc', C.byref(args))


def conv1d_out_tanh_ex(in_hi, in_lo, channels, halo, clip_offsets, drop_tail, weight, bias, workspace, wav_out):
    """The generators' output layer over a layout of `halo` rows (include/ttsb.h: ttsb_conv1d_out_tanh_ex); clip_offsets: host
    sequence (n_clips + 1)."""
    co, n = _host_offsets(clip_offsets)
    _call('ttsb_conv1d_out_tanh_ex', ptr(in_hi), ptr(in_lo), in_hi.shape[-1], channels, halo, co, n, drop_tail, ptr(weight), bias,
          ptr(workspace), workspace.nbytes, ptr(wav_out))


def conv1d_out_clamp_ex(in_hi, in_lo, channels, halo, clip_offsets, drop_tail, weight, bias, workspace, wav_out):
    """conv1d_out_tanh_ex with clamp(., -1, 1) in place of tanh (include/ttsb.h: ttsb_conv1d_out_clamp_ex)."""
    co, n = _host_offsets(clip_offsets)
    _call('ttsb_conv1d_out_clamp_ex', ptr(in_hi), ptr(in_lo), in_hi.shape[-1], channels, halo, co, n, drop_tail, ptr(weight), bias,
          ptr(workspace), workspace.nbytes, ptr(wav_out))


def snake_aa_ex(src, dst, channels, halo, clip_offsets, alpha, inv_beta, h_up, h_down, workspace):
    """BigVGAN's anti-aliased Snake activation over a packed ragged layout (include/ttsb.h: ttsb_snake_aa_ex).  src / dst:
    (hi, lo) planes, lo None in bf16; clip_offsets: host sequence (n_clips + 1); alpha / inv_beta: fp32 (channels) device
    tensors; h_up / h_down: 12 host taps each."""
    co, n = _host_offsets(clip_offsets)
    split = src[1] is not None
    up = (C.c_float * 12)(*[float(v) for v in h_up])
    down = (C.c_float * 12)(*[float(v) for v in h_down])
    _call('ttsb_snake_aa_ex', ptr(src[0]), ptr(src[1]), ptr(dst[0]), ptr(dst[1]), src[0].shape[-1], channels, halo, co, n, ptr(alpha),
          ptr(inv_beta), C.cast(up, C.c_void_p), C.cast(down, C.c_void_p), PREC_BF16X3 if split else PREC_BF16, ptr(workspace),
          workspace.nbytes)


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
    return _workspace_size('ttsb_wavernn_workspace_bytes', C.cast(tab, C.c_void_p), len(frames), hop, int(bool(batched)), target,
                           overlap, n_classes)


def wavernn_generate_rc(stream=None, **kw) -> int:
    """ttsb_wavernn_generate with the parameters of WAVERNN_PARAMS by name (missing ones NULL / 0) -> its return code."""
    unknown = set(kw) - {n for n, _ in WAVERNN_PARAMS}
    if unknown:
        raise TypeError(f'ttsb_wavernn_generate has no parameter {sorted(unknown)[0]}')
    return load().ttsb_wavernn_generate(*[kw.get(n, None if t is C.c_void_p else 0) for n, t in WAVERNN_PARAMS], stream)


def wavernn_generate(**kw):
    """One WaveRNN generation (include/ttsb.h: ttsb_wavernn_generate); frames / seeds point at host tables."""
    _check(wavernn_generate_rc(_stream(), **kw), 'ttsb_wavernn_generate')


# ------------------------------------------------------------------------------------------------------------
# The C signature of every entry point of include/ttsb.h, in the header's order: name -> (restype, argtypes).  load() declares
# them all, so ctypes checks each call's argument count and converts every argument to its C type, or refuses it.  Pointers
# are c_void_p, except the argument structs passed by reference, which take only their own mirror; tests/test_abi.py checks
# every row against the header.
# ------------------------------------------------------------------------------------------------------------
_P, _I, _I64, _U32, _F, _D = C.c_void_p, C.c_int, C.c_int64, C.c_uint32, C.c_float, C.c_double
SIGNATURES = {
    'ttsb_last_error': (C.c_char_p, []),
    'ttsb_abi_version': (_I, []),
    'ttsb_launch_count': (_I64, []),
    'ttsb_reset_launch_count': (None, []),
    'ttsb_add_launch_count': (None, [_I64]),
    'ttsb_set_dropout_salt': (_I, [_P, _P]),
    'ttsb_pack_weight': (_I, [_P, _I, _I, _I, _P, _P, _P]),
    'ttsb_repack_batched': (_I, [_P, _I, _P]),
    'ttsb_split_bf16': (_I, [_P, _I64, _P, _P, _P]),
    'ttsb_embed_ln_pe_fwd': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P, _P, _P, _P]),
    'ttsb_linear_fwd': (_I, [C.POINTER(GemmArgs), _P]),
    'ttsb_layernorm_fwd': (_I, [_P, _P, _P, _I, _I, _I, _I, _F, _P, _P, _P, _P, _P]),
    'ttsb_mha_fwd': (_I, [C.POINTER(MhaArgs), _P]),
    'ttsb_decode_attn_workspace_bytes': (_I64, [_I, _I, _I]),
    'ttsb_decode_attn': (_I, [C.POINTER(DecodeAttnArgs), _P]),
    'ttsb_decode_prologue': (_I, [_P, _P, _P, _P, _P, _I, _P, _I, _I, _F, _P, _P, _P, _P]),
    'ttsb_decode_commit': (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _P, _P, _P, _P, _P]),
    'ttsb_bgemm': (_I, [C.POINTER(BgemmArgs), _P]),
    'ttsb_wgrad': (_I, [C.POINTER(WgradArgs), _P]),
    'ttsb_rowdot_heads': (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    'ttsb_softmax_fwd': (_I, [_P, _I, _I, _I, _I, _I, _P, _F, _U32, _U32, _I, _P, _P, _P]),
    'ttsb_attn_probs_supported': (_I, [_I, _I]),
    'ttsb_attn_probs_fwd': (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _P, _F, _F, _U32, _U32, _P, _P, _I, _P]),
    'ttsb_attn_ds_bwd': (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _F, _F, _U32, _U32, _P, _I, _P]),
    'ttsb_softmax_bwd': (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _F, _F, _U32, _U32, _I, _P, _P]),
    'ttsb_layernorm_bwd': (_I, [_P, _P, _P, _I, _I, _I, _I, _F, _P, _I, _F, _U32, _F, _U32, _U32, _P, _P, _P, _P, _P, _P]),
    'ttsb_colsum_bf16': (_I, [_P, _I64, _I, _I, _P, _P]),
    'ttsb_colsum_bf16_x3': (_I, [_P, _I64, _I, _I, _P, _P, _P, _P]),
    'ttsb_relu_bwd': (_I, [_P, _P, _I64, _P]),
    'ttsb_relu_bwd_colsum': (_I, [_P, _P, _I64, _I, _P, _P]),
    'ttsb_cast_bf16_pad': (_I, [_P, _I64, _I, _P, _I, _P]),
    'ttsb_mae_loss': (_I, [_P, _I, _I, _I, _I, _P, _P, _F, _P, _P, _P]),
    'ttsb_attention_scores': (_I, [_P, _I, _I, _I, _I, _P, _P, _I, _P, _P]),
    'ttsb_durations_from_attention': (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _I, _P, _P, _P]),
    'ttsb_pitch_per_char': (_I, [_P, _I, _I, _P, _P, _I, _P, _D, _D, _P, _P]),
    'ttsb_scaled_ce_loss': (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _F, _P, _F, _P, _I, _P]),
    'ttsb_diag_loss_train': (_I, [_P, _I, _I, _I, _I, _I, _P, _P, _F, _P, _F, _P, _P]),
    'ttsb_diag_loss': (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P]),
    'ttsb_expand_bwd': (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    'ttsb_embedding_bwd': (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    'ttsb_pe_scalar_bwd': (_I, [_P, _P, _I, _I, _I, _F, _U32, _U32, _P, _P]),
    'ttsb_embed_ln_pe_train_fwd': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _F, _U32, _U32, _P, _P, _P, _P]),
    'ttsb_expand_ln_pe_train_fwd': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _F, _U32, _U32, _P, _P, _P, _P]),
    'ttsb_pitch_embed_bwd': (_I, [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P]),
    'ttsb_statpred_head_bwd': (_I, [_P, _P, _P, _I, _I, _P, _I, _P, _I, _I, _P, _P, _P, _P]),
    'ttsb_adam_tf_step': (_I, [_P, _P, _P, _P, _I64, _F, _F, _F, _F, _F, _P]),
    'ttsb_statpred_head_fwd': (_I, [_P, _I, _I, _P, _P, _I, _P, _I, _I, _P, _P]),
    'ttsb_pitch_embed_add_fwd': (_I, [_P, _P, _P, _P, _I, _I, _I, _P, _P]),
    'ttsb_durations_to_int': (_I, [_P, _F, _P, _P, _I, _I, _P, _P, _P]),
    'ttsb_expand_indices': (_I, [_P, _I, _I, _I, _P, _P]),
    'ttsb_length_regulate_fwd': (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    'ttsb_expand_ln_pe_fwd': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P, _P, _P, _P]),
    'ttsb_mel_lengths': (_I, [_P, _I, _I, _I, _F, _P, _P]),
    'ttsb_phoneme_lengths': (_I, [_P, _I, _I, _I, _P, _P]),
    'ttsb_stft_mel_log': (_I, [_P, _I, _I, _P, _P, _I, _I, _P, _P]),
    'ttsb_stft_mel_log_batch_workspace_bytes': (_I64, [_I]),
    'ttsb_stft_mel_log_batch': (_I, [_P, _P, _P, _I, _P, _P, _I, _I, _P, _I64, _P, _P]),
    'ttsb_pitch_workspace_bytes': (_I64, [_P, _I, _I, _D, _D, _D, _D]),
    'ttsb_pitch_dio_stonemask': (_I, [_P, _P, _I, _I, _D, _D, _D, _D, _D, _P, _P, _P, _I64, _P]),
    'ttsb_resample_batch_workspace_bytes': (_I64, [_P, _P, _I, _I, _I]),
    'ttsb_resample_batch': (_I, [_P, _P, _P, _I, _I, _P, _I, _P, _P, _I64, _P, _P]),
    'ttsb_trim_silence_workspace_bytes': (_I64, [_P, _I]),
    'ttsb_trim_silence_bounds': (_I, [_P, _P, _I, _D, _P, _I64, _P, _P]),
    'ttsb_flac_decode_workspace_bytes': (_I64, [_P, _P, _I]),
    'ttsb_flac_decode_batch': (_I, [_P, _P, _P, _I, _P, _P, _P, _P, _I64, _P]),
    'ttsb_cheaptrick_workspace_bytes': (_I64, [_P, _P, _I, _I, _D, _I]),
    'ttsb_cheaptrick': (_I, [_P, _P, _I, _I, _D, _P, _P, _D, _I, _P, _I64, _P, _P]),
    'ttsb_sp2mc': (_I, [_P, _I, _I, _P, _I, _P, _P]),
    'ttsb_mel_to_linear': (_I, [_P, _I, _I, _P, _P, _P, _P, _F, _I, _P, _P]),
    'ttsb_stft_complex': (_I, [_P, _I, _P, _P]),
    'ttsb_istft_workspace_bytes': (_I64, [_I]),
    'ttsb_istft': (_I, [_P, _I, _P, _I64, _P, _P]),
    'ttsb_griffinlim_update': (_I, [_P, _P, _P, _F, _I64, _P, _P]),
    'ttsb_griffinlim_batch_workspace_bytes': (_I64, [_I, _I]),
    'ttsb_griffinlim_batch': (_I, [_P, _P, _P, _I, _I, _I, _F, _P, _I64, _P, _P]),
    'ttsb_stft_mel_log_ragged_workspace_bytes': (_I64, [_I, _I]),
    'ttsb_stft_mel_log_ragged': (_I, [_P, _P, _P, _I, _I, _I, _I, _P, _P, _I, _I, _P, _I64, _P, _P]),
    'ttsb_mel_to_linear_ex': (_I, [_P, _I, _I, _I, _P, _P, _P, _P, _F, _I, _P, _P]),
    'ttsb_stft_complex_ragged_workspace_bytes': (_I64, [_I, _I]),
    'ttsb_stft_complex_ragged': (_I, [_P, _P, _I, _I, _I, _I, _P, _I64, _P, _P]),
    'ttsb_istft_ragged_workspace_bytes': (_I64, [_I, _I, _I]),
    'ttsb_istft_ragged': (_I, [_P, _P, _I, _I, _I, _I, _P, _I64, _P, _P]),
    'ttsb_griffinlim_ragged_workspace_bytes': (_I64, [_I, _I, _I]),
    'ttsb_griffinlim_ragged': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P, _I64, _P, _P]),
    'ttsb_mcd_dtw_workspace_bytes': (_I64, [_P, _P, _I, _I]),
    'ttsb_mcd_dtw': (_I, [_P, _P, _P, _P, _I, _I, _P, _I, _D, _P, _I64, _P, _P, _P]),
    'ttsb_mcd_dtw_path_workspace_bytes': (_I64, [_P, _P, _I, _I]),
    'ttsb_mcd_dtw_path': (_I, [_P, _P, _P, _P, _I, _I, _P, _I, _D, _P, _I64, _P, _P, _P, _P]),
    'ttsb_mcd_dtw_ceps_workspace_bytes': (_I64, [_P, _P, _I, _I]),
    'ttsb_mcd_dtw_ceps': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _D, _P, _I64, _P, _P, _P]),
    'ttsb_mcd_dtw_ceps_path_workspace_bytes': (_I64, [_P, _P, _I, _I]),
    'ttsb_mcd_dtw_ceps_path': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _D, _P, _I64, _P, _P, _P, _P]),
    'ttsb_conv1d_workspace_bytes': (_I64, [_I]),
    'ttsb_conv1d_ex_tc': (_I, [C.POINTER(Conv1dExArgs), _P]),
    'ttsb_conv1d_out_tanh_ex': (_I, [_P, _P, _I, _I, _I, _P, _I, _I, _P, _F, _P, _I64, _P, _P]),
    'ttsb_conv1d_out_clamp_ex': (_I, [_P, _P, _I, _I, _I, _P, _I, _I, _P, _F, _P, _I64, _P, _P]),
    'ttsb_snake_aa_ex': (_I, [_P, _P, _P, _P, _I, _I, _I, _P, _I, _P, _P, _P, _P, _I, _P, _I64, _P]),
    'ttsb_wavernn_workspace_bytes': (_I64, [_P, _I, _I, _I, _I, _I, _I]),
    'ttsb_wavernn_generate': (_I, [t for _, t in WAVERNN_PARAMS] + [_P]),
    'ttsb_dp_unique_id': (_I, [_P]),
    'ttsb_dp_init': (_I, [_P, _I, _I, _P]),
    'ttsb_dp_allreduce_bucket': (_I, [_P, _P, _I64, _P]),
    'ttsb_dp_destroy': (_I, [_P]),
}
# the exported names alone, in the header's order
EXPORTS = tuple(SIGNATURES)
