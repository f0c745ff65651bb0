"""Helpers shared by the GPU parity tests: drive single kernels of libttsb.so through the C ABI."""
from __future__ import annotations

import numpy as np
import torch

from transformertts_b200 import lib
from transformertts_b200.model.models import _PackedLinear, _round_up

DEV = 'cuda:0'
# what the columns of a source buffer outside [a_col0, a_col0 + C) hold: a GEMM that reads them is far off its reference
WIDE_SOURCE_FILL = 3.0e4


def split_or_none(x: torch.Tensor, split: bool):
    return lib.split_bf16(x, split)


# ----------------------------------------------------------------------------------------------------------
# the stateless dropout mask of csrc/ttsb_common.cuh (dropout_hterm, dropout_mix, dropout_keep, dropout_thresh) in numpy
# uint32 arithmetic: element idx of (seed, site) is kept when its 16-bit half of the hash of pair idx >> 1 is >= thresh >> 16
# ----------------------------------------------------------------------------------------------------------
DROPOUT_C1 = 0x9E3779B1


def _u32(x):
    """uint32 array (at least 1-D, so products wrap silently as in C)."""
    return np.atleast_1d(np.asarray(x, dtype=np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def dropout_thresh(p: float) -> int:
    return int(float(np.float32(p)) * 4294967296.0) if p > 0 else 0


def dropout_hterm(seed: int, site: int, pair_hi, salt: int = 0):
    s = _u32(seed ^ salt)
    return (_u32(pair_hi) * np.uint32(0x85EBCA77)) ^ (s * np.uint32(0xC2B2AE3D)) ^ (_u32(site) * np.uint32(0x27D4EB2F))


def dropout_mix(x):
    x = _u32(x)
    x = x ^ (x >> np.uint32(16))
    x = x * np.uint32(0x7FEB352D)
    x = x ^ (x >> np.uint32(15))
    x = x * np.uint32(0x846CA68B)
    return x ^ (x >> np.uint32(16))


def dropout_keep(seed: int, site: int, idx, p: float, salt: int = 0) -> np.ndarray:
    """Keep decisions of the elements `idx` (any integer array) at rate p."""
    idx = np.asarray(idx, dtype=np.uint64)
    pair = idx >> np.uint64(1)
    h = dropout_mix((_u32(pair & np.uint64(0xFFFFFFFF)) * np.uint32(DROPOUT_C1)) ^ dropout_hterm(seed, site, pair >> np.uint64(32), salt))
    half = np.where((idx & np.uint64(1)) != 0, h >> np.uint32(16), h & np.uint32(0xFFFF))
    return half >= np.uint32(dropout_thresh(p) >> 16)


def dropout_mask(B: int, T: int, N: int, ld: int, seed: int, site: int, p: float, salt: int = 0) -> np.ndarray:
    """(B,T,N) keep mask of a (B,T,ld) tensor whose element (b,t,n) is drawn at index (b*T + t)*ld + n."""
    idx = (np.arange(B * T, dtype=np.uint64)[:, None] * np.uint64(ld) + np.arange(N, dtype=np.uint64)[None, :]).reshape(B, T, N)
    return dropout_keep(seed, site, idx, p, salt)


def dropout_scale(p: float) -> float:
    """1/(1-p) as the kernels compute it, in fp32."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


def _poison16(shape):
    """16-bit buffer of all-ones bit patterns: NaN read as bf16 and as fp16."""
    t = torch.empty(shape, device=DEV, dtype=torch.bfloat16)
    t.view(torch.int16).fill_(-1)
    return t


def run_gemm(x_list, w_kn, bias, seg_src, seg_shift, seg_k, *, precision='bf16x3', impl='tcgen05', relu=False,
             residual=None, ln=None, row_len=None, block_n=None, single_tile=False, out_fp16=False, outputs=None, ld_out=None,
             lda=None, a_col0=None, residual_pair=None, out_preln=False, dropout=None, dropout_post=None, seed=0):
    """x_list: fp32 (B,T,C) sources (on GPU).  Returns dict with requested outputs.

    outputs: any subset of 'f32', 'hi', 'lo' (default: all three, 'lo' only in bf16x3); with out_fp16 'hi' holds fp16.
    ld_out: row stride of the outputs (default n_pad).  lda / a_col0: per source, the source is placed at column a_col0 of
    a buffer with lda columns whose other columns hold WIDE_SOURCE_FILL.  residual_pair: bf16 (hi, lo) residual.
    out_preln: also return the pre-LayerNorm value.  dropout / dropout_post: (p, site) of drop_pre / drop_post.
    Every output starts as NaN; out['launches'] is the number of kernel launches of the call."""
    split = precision == 'bf16x3'
    B, T, _ = x_list[0].shape
    pl = _PackedLinear(w_kn, bias, seg_k, split, single_tile=single_tile, block_n=block_n)
    a = lib.GemmArgs()
    a.B, a.T, a.N, a.block_n = B, T, pl.N, pl.block_n
    a.num_segments = len(seg_k)
    keep = []
    for s in range(len(seg_k)):
        a.seg_src[s], a.seg_shift[s], a.seg_k[s] = seg_src[s], seg_shift[s], seg_k[s]
    for i, x in enumerate(x_list):
        C = x.shape[-1]
        ld = lda[i] if lda is not None else C
        c0 = a_col0[i] if a_col0 is not None else 0
        if ld != C or c0 != 0:
            assert c0 + C <= ld
            buf = torch.full((B, T, ld), WIDE_SOURCE_FILL, device=x.device)
            buf[..., c0:c0 + C] = x
            x = buf
        hi, lo = lib.split_bf16(x, split)
        keep += [hi, lo]
        a.a_hi[i] = hi.data_ptr()
        a.a_lo[i] = lo.data_ptr() if lo is not None else None
        a.lda[i] = ld
        a.a_col0[i] = c0
    a.w_hi = pl.w_hi.data_ptr()
    a.w_lo = pl.w_lo.data_ptr() if pl.w_lo is not None else None
    a.bias = pl.bias.data_ptr() if pl.bias is not None else None
    a.relu = int(relu)
    if residual is not None:
        a.residual = residual.data_ptr()
        a.ld_res = residual.shape[-1]
    if residual_pair is not None:
        a.residual_hi, a.residual_lo = residual_pair[0].data_ptr(), residual_pair[1].data_ptr()
        a.ld_res = residual_pair[0].shape[-1]
    if ln is not None:
        from transformertts_b200.model.models import _pad_vec
        g_pad, b_pad = _pad_vec(ln[0], pl.n_pad), _pad_vec(ln[1], pl.n_pad)
        keep += [g_pad, b_pad]
        a.ln_gamma, a.ln_beta, a.ln_eps = g_pad.data_ptr(), b_pad.data_ptr(), 1e-6
    if row_len is not None:
        a.row_len = row_len.data_ptr()
    if outputs is None:
        outputs = ('f32', 'hi', 'lo')
    ld = ld_out or pl.n_pad
    out = {}
    # poison the outputs so unwritten elements are visible
    out_f32 = torch.full((B, T, ld), float('nan'), device=DEV) if 'f32' in outputs else None
    out_hi = _poison16((B, T, ld)) if 'hi' in outputs else None
    out_lo = _poison16((B, T, ld)) if 'lo' in outputs and split else None
    preln = torch.full((B, T, ld), float('nan'), device=DEV) if out_preln else None
    a.out_f32 = out_f32.data_ptr() if out_f32 is not None else None
    a.out_hi = out_hi.data_ptr() if out_hi is not None else None
    a.out_lo = out_lo.data_ptr() if out_lo is not None else None
    a.out_preln = preln.data_ptr() if preln is not None else None
    a.ld_out = ld
    a.out_fp16 = int(out_fp16)
    if dropout is not None:
        a.drop_pre_p, a.drop_pre_site = dropout
    if dropout_post is not None:
        a.drop_post_p, a.drop_post_site = dropout_post
    a.drop_seed = seed
    a.precision = lib.PREC_BF16X3 if split else lib.PREC_BF16
    a.impl = lib.IMPL_SIMT if impl == 'simt' else lib.IMPL_TCGEN05
    lib.reset_launch_count()
    lib.linear_fwd(a)
    out['launches'] = lib.launch_count()
    torch.cuda.synchronize()
    out['f32'] = out_f32
    out['hi'] = out_hi
    out['lo'] = out_lo
    out['preln'] = preln
    out['n_pad'] = pl.n_pad
    return out


def ref_gemm(x_list, w_kn, bias, seg_src, seg_shift, seg_k, *, precision, relu=False, residual=None, ln=None, row_len=None,
             residual_pair=None, dropout=None, dropout_post=None, seed=0, salt=0, ld_out=None, device='cpu', return_preln=False):
    """float64 reference of the same contract (on `device`).  In 'bf16' mode the operands are first rounded to bf16 (that is
    the kernel's arithmetic); in 'bf16x3' mode the fp32 operands are used as they are.  residual_pair adds
    float(hi) + float(lo); dropout / dropout_post = (p, site) apply the restated masks, drawn at (b*T + t)*ld_out + n, as
    keep * x * fp32(1/(1-p)).  return_preln: also return the value before the LayerNorm (not row-masked)."""
    dev = torch.device(device)
    xs = [x.detach().to(dev).double() if precision == 'bf16x3' else x.detach().to(dev).bfloat16().double() for x in x_list]
    w = w_kn.detach().to(dev).reshape(-1, w_kn.shape[-1])
    w = w.double() if precision == 'bf16x3' else w.bfloat16().double()
    B, T, _ = xs[0].shape
    N = w.shape[1]
    acc = torch.zeros(B, T, N, dtype=torch.float64, device=dev)
    koff = 0
    for s, k in enumerate(seg_k):
        x = xs[seg_src[s]]
        sh = seg_shift[s]
        lo, hi = max(0, -sh), min(T, T - sh)
        if hi > lo:
            acc[:, lo:hi] += x[:, lo + sh:hi + sh, :k] @ w[koff:koff + k]
        koff += k
    if bias is not None:
        acc += bias.detach().to(dev).double()
    if relu:
        acc = torch.relu(acc)

    def drop(v, spec):
        p, site = spec
        keep = torch.from_numpy(dropout_mask(B, T, N, ld_out, seed, site, p, salt)).to(dev)
        return v * keep * dropout_scale(p)

    if dropout is not None:
        acc = drop(acc, dropout)
    if residual is not None:
        acc += residual.detach().to(dev).double()[..., :N]
    if residual_pair is not None:
        acc += residual_pair[0].detach().to(dev).double()[..., :N] + residual_pair[1].detach().to(dev).double()[..., :N]
    preln = acc
    if ln is not None:
        g, b = ln[0].detach().to(dev).double(), ln[1].detach().to(dev).double()
        mean = acc.mean(-1, keepdim=True)
        var = ((acc - mean) ** 2).mean(-1, keepdim=True)
        acc = (acc - mean) * torch.rsqrt(var + 1e-6) * g + b
    if dropout_post is not None:
        acc = drop(acc, dropout_post)
    if row_len is not None:
        keep = torch.arange(T, device=dev)[None, :] < row_len.detach().to(dev)[:, None]
        acc = acc * keep[..., None]
    return (acc, preln) if return_preln else acc


def _to16(x, precision, split):
    if precision == 'fp16':
        return x.contiguous().half(), None
    return lib.split_bf16(x, split)


def run_mha(q, k, v, kv_len, H, *, precision='bf16x3', impl='tcgen05', weights_b=None):
    """q,k,v fp32 (B,T,d) on GPU -> attention output fp32 (B,T,d) (hi+lo recombined)."""
    split = precision == 'bf16x3'
    B, T, d = q.shape
    dh = d // H
    qk = torch.cat([q, k, v], dim=-1).contiguous()
    qk_hi, qk_lo = _to16(qk, precision, split)
    out_hi = torch.full((B, T, d), float('nan'), device=DEV, dtype=torch.bfloat16)
    out_lo = torch.full((B, T, d), float('nan'), device=DEV, dtype=torch.bfloat16)
    m = lib.MhaArgs()
    m.B, m.T, m.H, m.dh = B, T, H, dh
    m.qk_hi = qk_hi.data_ptr()
    m.qk_lo = qk_lo.data_ptr() if split else None
    m.ld_qk, m.q_col0, m.k_col0, m.v_col0 = 3 * d, 0, d, 2 * d
    m.kv_len = kv_len.data_ptr()
    m.out_hi = out_hi.data_ptr()
    m.out_lo = out_lo.data_ptr()
    m.ld_out = d
    wts = None
    if weights_b is not None:
        wts = torch.full((H, T, T), float('nan'), device=DEV)
        m.weights_out = wts.data_ptr()
        m.weights_batch_index = weights_b
    m.precision = {'bf16x3': lib.PREC_BF16X3, 'bf16': lib.PREC_BF16, 'fp16': lib.PREC_FP16}[precision]
    m.impl = lib.IMPL_SIMT if impl == 'simt' else lib.IMPL_TCGEN05
    lib.mha_fwd(m)
    torch.cuda.synchronize()
    out = out_hi.float() + out_lo.float()
    return out, wts


def ref_mha(q, k, v, kv_len, H, precision):
    """float64 CPU attention with the reference's additive -1e9 key mask (model/layers.py:176-195)."""
    cast = {'bf16x3': lambda t: t.detach().cpu().double(), 'bf16': lambda t: t.detach().cpu().bfloat16().double(),
            'fp16': lambda t: t.detach().cpu().half().double()}[precision]
    q, k, v = cast(q), cast(k), cast(v)
    B, T, d = q.shape
    dh = d // H
    sp = lambda t: t.reshape(B, T, H, dh).permute(0, 2, 1, 3)
    logits = sp(q) @ sp(k).transpose(-1, -2) / (dh ** 0.5)
    mask = (torch.arange(T)[None, :] >= kv_len.cpu()[:, None]).double()[:, None, None, :]
    logits = (logits.float() + (mask * -1e9).float()).double()  # fp32 add as in the reference
    w = torch.softmax(logits, -1)
    out = (w @ sp(v)).permute(0, 2, 1, 3).reshape(B, T, d)
    return out, w


def operand16(t: torch.Tensor, precision: str) -> torch.Tensor:
    """float64 (CPU) value of what the attention kernels read for fp32 `t`: the fp16 or bf16 rounding, or in bf16x3 the sum
    hi + lo of its split (hi = bf16(t), lo = bf16(t - hi), both round to nearest, as ttsb_split_bf16 computes them)."""
    t = t.detach().cpu().float()
    if precision == 'fp16':
        return t.half().double()
    hi = t.bfloat16()
    if precision == 'bf16':
        return hi.double()
    return hi.double() + (t - hi.float()).bfloat16().double()


def _place(B, T, ld, parts):
    """fp32 (B, T, ld) buffer holding each (tensor, column offset) of `parts`; every other column is NaN."""
    buf = torch.full((B, T, ld), float('nan'), device=DEV)
    taken = torch.zeros(ld, dtype=torch.bool)
    for x, c0 in parts:
        C = x.shape[-1]
        assert 0 <= c0 and c0 + C <= ld and not taken[c0:c0 + C].any()
        taken[c0:c0 + C] = True
        buf[..., c0:c0 + C] = x
    return buf


def run_mha_general(q, kv_k, kv_v, kv_len, H, *, precision='fp16', impl='tcgen05', causal=False, cross=False, full_queries=True,
                    weights_all=False, weights_b=None, ld_qk=None, ld_kv=None, cols=None, out=None):
    """General form of ttsb_mha_fwd: q fp32 (B,T,d); k,v fp32 (B,Tk,d).  cross=True keeps k|v in a second buffer.

    Layout: q, k and v sit at column offsets cols = (q_col0, k_col0, v_col0) of a (B,T,ld_qk) buffer (self-attention), or q at
    q_col0 of (B,T,ld_qk) and k, v at k_col0 / v_col0 of (B,Tk,ld_kv) (cross); columns outside them hold NaN.  Defaults:
    (0, d, 2d) and ld_qk = 3d, or (0, 0, d), ld_qk = d and ld_kv = 2d.  out: the caller's (out_hi, out_lo or None) 16-bit
    buffers of shape (rows >= B*T, ld_out), written through the ABI as they are (out_lo None passes NULL); by default both
    planes are (B*T, d) and NaN.  weights_b: the weights of that batch row, (H,T,Tk); weights_all: (B,H,T,Tk); NaN before.
    Returns (hi + lo of columns [0, d) of the first B*T rows as (B,T,d), weights)."""
    split = precision == 'bf16x3'
    B, T, d = q.shape
    Tk = kv_k.shape[1]
    dh = d // H
    m = lib.MhaArgs()
    m.B, m.T, m.H, m.dh = B, T, H, dh
    keep = []
    if cross:
        q_col0, k_col0, v_col0 = cols or (0, 0, d)
        qb_hi, qb_lo = _to16(_place(B, T, ld_qk or d, [(q, q_col0)]), precision, split)
        kv_hi, kv_lo = _to16(_place(B, Tk, ld_kv or 2 * d, [(kv_k, k_col0), (kv_v, v_col0)]), precision, split)
        keep += [qb_hi, qb_lo, kv_hi, kv_lo]
        m.qk_hi = qb_hi.data_ptr()
        m.qk_lo = qb_lo.data_ptr() if split else None
        m.ld_qk, m.q_col0 = qb_hi.shape[-1], q_col0
        m.kv_hi = kv_hi.data_ptr()
        m.kv_lo = kv_lo.data_ptr() if split else None
        m.ld_kv, m.Tk, m.k_col0, m.v_col0 = kv_hi.shape[-1], Tk, k_col0, v_col0
    else:
        assert Tk == T
        q_col0, k_col0, v_col0 = cols or (0, d, 2 * d)
        qk_hi, qk_lo = _to16(_place(B, T, ld_qk or 3 * d, [(q, q_col0), (kv_k, k_col0), (kv_v, v_col0)]), precision, split)
        keep += [qk_hi, qk_lo]
        m.qk_hi = qk_hi.data_ptr()
        m.qk_lo = qk_lo.data_ptr() if split else None
        m.ld_qk, m.q_col0, m.k_col0, m.v_col0 = qk_hi.shape[-1], q_col0, k_col0, v_col0
    m.kv_len = kv_len.data_ptr()
    if out is None:
        out = (_poison16((B * T, d)), _poison16((B * T, d)))
    out_hi, out_lo = out
    m.out_hi = out_hi.data_ptr()
    m.out_lo = out_lo.data_ptr() if out_lo is not None else None
    m.ld_out = out_hi.shape[-1]
    m.causal = int(causal)
    m.full_queries = int(full_queries)
    wts = None
    if weights_all:
        wts = torch.full((B, H, T, Tk), float('nan'), device=DEV)
        m.weights_out = wts.data_ptr()
        m.weights_all = 1
    elif weights_b is not None:
        wts = torch.full((H, T, Tk), float('nan'), device=DEV)
        m.weights_out = wts.data_ptr()
        m.weights_batch_index = weights_b
    m.precision = {'bf16x3': lib.PREC_BF16X3, 'bf16': lib.PREC_BF16, 'fp16': lib.PREC_FP16}[precision]
    m.impl = lib.IMPL_SIMT if impl == 'simt' else lib.IMPL_TCGEN05
    lib.mha_fwd(m)
    torch.cuda.synchronize()
    res = out_hi[:B * T].float() + (out_lo[:B * T].float() if out_lo is not None else 0)
    return res.reshape(B, T, -1)[..., :d], wts


def ref_mha_general(q, k, v, kv_len, H, precision, causal=False, full_queries=True):
    """float64 CPU attention on the operands the kernel reads (operand16); additive -1e9 mask = max(key padding, look-ahead)
    (models.py:136-138, layers.py:186-187).  full_queries=False: query rows >= kv_len[b] of the output are zero."""
    q, k, v = (operand16(t, precision) for t in (q, k, v))
    B, T, d = q.shape
    Tk = k.shape[1]
    dh = d // H
    sp = lambda t: t.reshape(B, t.shape[1], H, dh).permute(0, 2, 1, 3)
    logits = sp(q) @ sp(k).transpose(-1, -2) / (dh ** 0.5)
    mask = (torch.arange(Tk)[None, :] >= kv_len.cpu()[:, None]).double()[:, None, None, :].expand(B, 1, T, Tk)
    if causal:
        look = (torch.arange(Tk)[None, :] > torch.arange(T)[:, None]).double()[None, None]
        mask = torch.maximum(mask, look)
    logits = (logits.float() + (mask * -1e9).float()).double()
    w = torch.softmax(logits, -1)
    out = (w @ sp(v)).permute(0, 2, 1, 3).reshape(B, T, d)
    if not full_queries:
        out = out.masked_fill((torch.arange(T)[None, :] >= kv_len.cpu()[:, None])[..., None], 0.0)
    return out, w


# ----------------------------------------------------------------------------------------------------------
# ttsb_bgemm evaluated literally from its argument description (include/ttsb.h: ttsb_bgemm_args), in float64 on the host
# ----------------------------------------------------------------------------------------------------------
def bgemm_operand(x, dims, strides, off, B: int, H: int, n_mn: int, K: int) -> np.ndarray:
    """float64 (B*H, n_mn, K) operand of every problem z = (b, h), read element by element as the tensor map addresses it:
    x is the whole bf16 buffer, off = (h_col, h_row, z_batch, pointer offset in elements[, mn_major]) as TrainEngine._bgemm
    takes it.  Coordinates outside (dim0, dim1, dim2) read as zero (the TMA fill); NaN inside them stays NaN."""
    flat = x.detach().cpu().double().reshape(-1).numpy()
    h_col, h_row, z_batch, ptr_off = off[:4]
    mn_major = off[4] if len(off) > 4 else 0
    z = np.arange(B * H)
    b, h = z // H, z % H
    i_mn, i_k = np.arange(n_mn)[None, :, None], np.arange(K)[None, None, :]
    c0 = (i_mn if mn_major else i_k) + (h * h_col)[:, None, None]
    c1 = (i_k if mn_major else i_mn) + (h * h_row)[:, None, None]
    c2 = (z if z_batch else b)[:, None, None]
    c0, c1, c2 = np.broadcast_arrays(c0, c1, c2)
    inside = (c0 < dims[0]) & (c1 < dims[1]) & (c2 < dims[2])
    idx = ptr_off + c0 + c1 * strides[0] + c2 * strides[1]
    out = np.zeros(c0.shape)
    out[inside] = flat[idx[inside]]
    return out


def ref_bgemm(B, H, M, N, K, a, a_dims, a_strides, a_off, b, b_dims, b_strides, b_off):
    """(sum_k A_z[m][k] * B_z[n][k], sum_k |A_z[m][k] * B_z[n][k]|), each float64 (B*H, M, N), alpha not applied."""
    A = bgemm_operand(a, a_dims, a_strides, a_off, B, H, M, K)
    Bm = bgemm_operand(b, b_dims, b_strides, b_off, B, H, N, K)
    return A @ Bm.transpose(0, 2, 1), np.abs(A) @ np.abs(Bm).transpose(0, 2, 1)


def bgemm_out_index(B, H, M, out_cols, ld_out, out_batch_stride, out_h_col=0, out_by_b=0, out_ptr_off=0) -> np.ndarray:
    """int64 (B*H, M, out_cols): the element of the output buffer that holds column n of row m of problem z."""
    z = np.arange(B * H)
    batch = (z // H if out_by_b else z)[:, None, None]
    return (out_ptr_off + batch * out_batch_stride + np.arange(M)[None, :, None] * ld_out + ((z % H) * out_h_col)[:, None, None]
            + np.arange(out_cols)[None, None, :])
