"""Training step of the ForwardTransformer (reference: ForwardTransformer._train_step, model/models.py:464-482;
losses utils/losses.py:41-70 with weights [1,1,3] models.py:485; Adam utils/training_config_manager.py:102-106).

The forward pass is run in single-pass bf16 tensor-core mode (BASELINE.json configs[2]: "bf16") and keeps what the
backward needs; the backward is hand-written: every gradient GEMM runs on the wgmma tensor-core kernels (data gradients through the forward
GEMM kernel with re-packed weights, weight gradients and the attention gradients through ttsb_wgrad / ttsb_bgemm),
everything else through the row kernels of csrc/train_ops.cu.  Parameters, gradients and Adam moments live in flat
fp32 buffers so that Adam is one launch and data-parallel all-reduce works on contiguous buckets.
"""
from __future__ import annotations

import contextlib
import math
from typing import Dict

import torch

from .. import lib
from .models import (LN_EPS, _capture_graphs, _fill_inputs, _lru_get, _lru_make_room, _pad_vec, _PackedLinear, _qkv_block_n, _replay,
                     _round_up, _static_inputs)
from .transformer_utils import mask_from_lengths


def check_head_sizes(stacks) -> None:
    """The attention products of the training step contract over the head's columns in 64-wide k blocks (ttsb_bgemm,
    include/ttsb.h): a head size that is not a multiple of 64 would add the next head's columns to this head's scores, so
    only a block with a single head (whose columns end where the tensor ends) may have one, as a multiple of 16."""
    for name, st in stacks.items():
        for i, H in enumerate(st['heads']):
            dh = int(st['d']) // int(H)
            if dh % 64 != 0 and (int(H) != 1 or dh % 16 != 0):
                raise ValueError(
                    f"{name} block {i}: {H} heads at model dimension {st['d']} give a head size of {dh}, which the training step "
                    f'does not support (inference does).  Head sizes that train: multiples of 64 (64, 128, 192, 256), or a '
                    f'multiple of 16 in a block with a single head; choose {name}_num_heads accordingly.')


class Adam:
    """Optimizer state in the reference's terms: lr (assignable), iterations, Keras hyper-parameters."""

    def __init__(self, learning_rate: float, beta_1: float = 0.9, beta_2: float = 0.98, epsilon: float = 1e-9):
        self.lr = float(learning_rate)
        self.beta_1, self.beta_2, self.epsilon = beta_1, beta_2, epsilon
        self.iterations = 0
        self.m = None
        self.v = None


class TrainEngine:
    def __init__(self, model):
        check_head_sizes(model._stacks)
        self.model = model
        self.dev = model.device
        names = list(model._param_shapes().keys())
        sizes = [model.weights[n].numel() for n in names]
        padded = [_round_up(sz, 8) for sz in sizes]  # every parameter starts 32-byte aligned (kernels use float4 loads)
        self.names = names
        total = sum(padded)
        self.flat_w = torch.zeros(total, dtype=torch.float32, device=self.dev)
        self.flat_g = torch.zeros(total, dtype=torch.float32, device=self.dev)
        off = 0
        self.g: Dict[str, torch.Tensor] = {}
        self.offsets: Dict[str, tuple] = {}
        for n, sz, psz in zip(names, sizes, padded):
            self.offsets[n] = (off, psz)
            shape = model.weights[n].shape
            self.flat_w[off:off + sz].copy_(model.weights[n].reshape(-1))
            model.weights[n] = self.flat_w[off:off + sz].view(shape)  # parameters become views of the flat buffer
            self.g[n] = self.flat_g[off:off + sz].view(shape)
            off += psz
        dec = [self.offsets[n] for n in names if n.startswith('decoder.')]
        self.decoder_range = (dec[0][0], dec[-1][0] + dec[-1][1])  # contiguous slice of the flat buffers
        model._packed = None
        self.P = None
        self.world = 1
        self.base_seed = 1234
        self.seed = 1234
        self.rank = 0
        self.drop_sites = 0
        self._salt_dev = None
        self._graphs = {}
        self._graph_pool = None
        self._loss_scratch = torch.zeros(1, dtype=torch.float32, device=self.dev)   # loss word of the diagonal-loss gradient

    # ------------------------------------------------------------------------------------------------
    # packed operands for the step (weights change every step)
    # ------------------------------------------------------------------------------------------------
    def _pack(self):
        """Every packed operand of the step is allocated once, with one ttsb_pack_desc per destination block that describes
        how to refresh it from the flat fp32 parameters; every step then repacks them in a single kernel launch."""
        if self.P is None:
            self.P, self._descs = {}, []
            self._build_packs()
            self._n_descs = len(self._descs)
            self._descs_dev = lib.upload_pack_descs(self._descs, self.dev)
        lib.repack_batched(self._descs_dev, self._n_descs)
        return self.P

    def _desc(self, src, dst_ptr, R, R_pad, C_cols, cb, cb_valid, sr, s_outer, s_inner, dst_ld, f32=0):
        d_ = lib.PackDesc()
        d_.src, d_.dst = src.data_ptr() if torch.is_tensor(src) else src, dst_ptr
        d_.R, d_.R_pad, d_.C_cols, d_.cb, d_.cb_valid = R, R_pad, C_cols, cb, cb_valid
        d_.sr, d_.s_outer, d_.s_inner, d_.dst_ld, d_.dst_f32 = sr, s_outer, s_inner, dst_ld, f32
        self._descs.append(d_)

    def _vec(self, src, dst, n_valid):  # zero-padded fp32 vector copy
        self._desc(src, dst.data_ptr(), 1, 1, dst.numel(), dst.numel(), n_valid, 0, 0, 1, dst.numel(), f32=1)

    def _fwd(self, key, parts, K, seg_k, single=False, block_n=None, k_valid=None):
        """parts: [(w (Kv,Ni) view, b (Ni))] concatenated along N (q|k|v) -- forward packing [N_pad, K]; rows k_valid..K of
        the contraction are zero (the Aligner feeds its 80 mel channels as a 128-wide K block)."""
        kv = K if k_valid is None else k_valid
        N = sum(w.shape[-1] for w, _ in parts)
        pl = _PackedLinear.empty(K, N, seg_k, self.dev, single_tile=single, block_n=block_n)
        if kv != K:
            pl.w_hi.zero_()
        row = 0
        for i, (w, b) in enumerate(parts):
            Ni = w.shape[-1]
            last = i == len(parts) - 1
            self._desc(w, pl.w_hi.data_ptr() + 2 * row * K, Ni, (pl.n_pad - row) if last else Ni, K, K, kv, 1, 0, Ni, K)
            self._desc(b, pl.bias.data_ptr() + 4 * row, 1, 1, (pl.n_pad - row) if last else Ni, pl.n_pad, Ni, 0, 0, 1, pl.n_pad, f32=1)
            row += Ni
        self.P[key] = pl

    def _dgrad_dense(self, key, parts, K):
        """parts: [w (K,Ni)] concatenated along N -- data-gradient packing [K_pad, N_pad] (contraction over N)."""
        N = sum(w.shape[-1] for w in parts)
        npad = _round_up(N, 64)
        pl = _PackedLinear.empty(npad, K, [npad], self.dev, bias=False)
        col = 0
        for i, w in enumerate(parts):
            Ni = w.shape[-1]
            last = i == len(parts) - 1
            width = (npad - col) if last else Ni
            self._desc(w, pl.w_hi.data_ptr() + 2 * col, K, pl.n_pad, width, width, Ni, Ni, 0, 1, npad)
            col += Ni
        self.P[key] = pl

    def _dgrad_conv(self, key, w):
        k, cin, cout = w.shape
        cpad = _round_up(cout, 64)
        pl = _PackedLinear.empty(k * cpad, cin, [cpad] * k, self.dev, bias=False)
        self._desc(w, pl.w_hi.data_ptr(), cin, pl.n_pad, k * cpad, cpad, cout, cout, cin * cout, 1, k * cpad)
        self.P[key] = pl

    def _pack_attention(self, pre, d):
        """Self-attention sub-block: q|k|v as one GEMM and its data gradient, then the output projection."""
        W = self.model.weights
        qkv = [(W[pre + n + '.w'], W[pre + n + '.b']) for n in ('wq', 'wk', 'wv')]
        self._fwd(pre + 'qkv', qkv, d, [d], block_n=_qkv_block_n(d))
        self._dgrad_dense(pre + 'qkv.d', [w for w, _ in qkv], d)
        self._pack_wo(pre, d)

    def _pack_wo(self, pre, d):
        """Output projection on concat([x, attn]) and its data gradients towards x and attn."""
        W = self.model.weights
        self._fwd(pre + 'wo', [(W[pre + 'wo.w'], W[pre + 'wo.b'])], 2 * d, [d, d], single=True)
        self._dgrad_dense(pre + 'wo.dx', [W[pre + 'wo.w'][:d]], d)
        self._dgrad_dense(pre + 'wo.da', [W[pre + 'wo.w'][d:]], d)

    def _pack_ffn(self, pre, d, F):
        W = self.model.weights
        self._fwd(pre + 'ffn1', [(W[pre + 'ffn1.w'], W[pre + 'ffn1.b'])], d, [d])
        self._fwd(pre + 'ffn2', [(W[pre + 'ffn2.w'], W[pre + 'ffn2.b'])], F, [F], single=True)
        self._dgrad_dense(pre + 'ffn1.d', [W[pre + 'ffn1.w']], d)
        self._dgrad_dense(pre + 'ffn2.d', [W[pre + 'ffn2.w']], F)

    def _build_packs(self):
        m = self.model
        W, P, dev = m.weights, self.P, self.dev
        for name, st in m._stacks.items():
            d = st['d']
            for i, _ in enumerate(st['heads']):
                pre = f'{name}.b{i}.'
                self._pack_attention(pre, d)
                if i < st['n_dense']:
                    self._pack_ffn(pre, d, int(st['ffn']))
                else:
                    cin = d
                    n = len(st['filters'])
                    kk = int(st['kernel'])
                    for j, f in enumerate(st['filters']):
                        w = W[pre + f'conv{j}.w']
                        self._fwd(pre + f'conv{j}', [(w.view(kk * cin, f), W[pre + f'conv{j}.b'])], kk * cin, [cin] * kk,
                                  single=(j == n - 1))
                        self._dgrad_conv(pre + f'conv{j}.d', w)
                        cin = f
        d_enc = m._stacks['encoder']['d']
        for name, filt, k in (('dur_pred', m.config['duration_conv_filters'], m.config['duration_kernel_size']),
                              ('pitch_pred', m.config['pitch_conv_filters'], m.config['pitch_kernel_size'])):
            cin = d_enc
            kk = int(k)
            for j, f in enumerate(filt):
                f = int(f)
                bn = _round_up(f, 64)  # 226 -> 256 columns so the next contraction is a multiple of 64
                w = W[f'{name}.conv{j}.w']
                self._fwd(f'{name}.conv{j}', [(w.view(kk * cin, f), W[f'{name}.conv{j}.b'])], kk * cin, [cin] * kk, single=True,
                          block_n=bn)
                g_pad = torch.zeros(bn, dtype=torch.float32, device=dev)
                b_pad = torch.zeros(bn, dtype=torch.float32, device=dev)
                self._vec(W[f'{name}.ln{j}.gamma'], g_pad, f)
                self._vec(W[f'{name}.ln{j}.beta'], b_pad, f)
                P[f'{name}.ln{j}'] = (g_pad, b_pad)
                self._dgrad_conv(f'{name}.conv{j}.d', w)
                cin = f
        dd = m._stacks['decoder']['d']
        self._fwd('out', [(W['out.w'], W['out.b'])], dd, [dd])
        self._dgrad_dense('out.d', [W['out.w']], dd)
        for name, st in m._stacks.items():
            P[f'{name}.pe'] = m._prepare_pe(name)

    # ------------------------------------------------------------------------------------------------
    # small helpers
    # ------------------------------------------------------------------------------------------------
    def _bf(self, *shape):
        return torch.empty(shape, dtype=torch.bfloat16, device=self.dev)

    def _f32(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.dev)

    def _wgrad(self, xs, g, ldg, B, T, Cin, N, segs, dw):
        """xs: [(bf16 (B,T,ld) tensor, ld)] sources; segs: [(source index, time shift)]; g: bf16 (B,T,ldg) output gradient."""
        a = lib.WgradArgs()
        a.B, a.T, a.Cin, a.N = B, T, Cin, N
        a.num_segments = len(segs)
        for s_, (src, shift) in enumerate(segs):
            a.seg_src[s_], a.seg_shift[s_] = src, shift
        for i, (x, ld) in enumerate(xs):
            a.x[i] = x.data_ptr()
            a.ldx[i] = ld
        a.g = g.data_ptr()
        a.ldg = ldg
        a.dw = dw.data_ptr()
        lib.wgrad(a)

    def _bgemm(self, B, H, M, N, K, a, a_dims, a_strides, a_off, b, b_dims, b_strides, b_off, alpha=1.0, out_f32=None, out_bf16=None,
               ld_out=0, out_batch_stride=0, out_h_col=0, out_by_b=0, out_cols=0, out_ptr_off=0, row_len=None, col_len=None,
               softmax_bwd=None):
        g = lib.BgemmArgs()
        g.B, g.H, g.M, g.N, g.K = B, H, M, N, K
        g.a = a.data_ptr() + 2 * a_off[3]
        g.a_dim0, g.a_dim1, g.a_dim2 = a_dims
        g.a_stride1, g.a_stride2 = a_strides
        g.a_h_col, g.a_h_row, g.a_z_batch = a_off[:3]
        g.a_mn_major = a_off[4] if len(a_off) > 4 else 0
        g.b = b.data_ptr() + 2 * b_off[3]
        g.b_dim0, g.b_dim1, g.b_dim2 = b_dims
        g.b_stride1, g.b_stride2 = b_strides
        g.b_h_col, g.b_h_row, g.b_z_batch = b_off[:3]
        g.b_mn_major = b_off[4] if len(b_off) > 4 else 0
        g.alpha = alpha
        if out_f32 is not None:
            g.out_f32 = out_f32.data_ptr() + 4 * out_ptr_off
        if out_bf16 is not None:
            g.out_bf16 = out_bf16.data_ptr() + 2 * out_ptr_off
        g.ld_out, g.out_batch_stride, g.out_h_col, g.out_by_b, g.out_cols = ld_out, out_batch_stride, out_h_col, out_by_b, out_cols
        g.row_len = row_len.data_ptr() if row_len is not None else None
        g.col_len = col_len.data_ptr() if col_len is not None else None
        if softmax_bwd is not None:  # (P_pre, D, scale, drop_p, seed, site, flags, key lengths): epilogue writes dS, not dP
            P_pre, D, scale, drop_p, seed, site, flags, lens = softmax_bwd[:8]
            g.sm_P, g.sm_D, g.sm_len = P_pre.data_ptr(), D.data_ptr(), lens.data_ptr()
            if len(softmax_bwd) > 8 and softmax_bwd[8] is not None and drop_p > 0:
                g.sm_Pdrop = softmax_bwd[8].data_ptr()
            g.sm_scale, g.sm_drop_p, g.sm_seed, g.sm_site, g.sm_flags = scale, drop_p, seed, site, flags
        lib.bgemm(g)

    # ------------------------------------------------------------------------------------------------
    # attention core on saved probabilities (self: q,k,v in one buffer; cross: q buffer + k|v buffer)
    # ------------------------------------------------------------------------------------------------
    @staticmethod
    def _fused_probs(qb, kb, flags, dh, ldp):
        """Self-attention without softmax flags runs on attn_probs_tc.cu where that kernel takes the head size; otherwise the
        fp32 logits are materialised by a batched GEMM and the softmax kernels."""
        return kb is qb and flags == 0 and lib.attn_probs_supported(dh, ldp)

    def _attn_fwd(self, B, H, dh, T, Tk, qb, q_ld, q_col, kb, k_ld, k_col, v_col, lens, flags=0):
        d = H * dh
        ldp = _round_up(Tk, 16)
        Z = B * H
        scale = 1.0 / math.sqrt(dh)
        rate = self.drop_rate
        P_pre = self._bf(Z, T, ldp)
        P_drop = self._bf(Z, T, ldp) if rate > 0 else P_pre
        site = self._site()
        if self._fused_probs(qb, kb, flags, dh, ldp):
            # logits, softmax and attention dropout in one kernel: the (Z, T, T) fp32 logits never reach HBM
            lib.attn_probs_fwd(qb, q_ld, q_col, k_col, B, H, T, dh, lens, scale, rate, self.seed, site, P_pre, P_drop, ldp)
        else:
            S = self._f32(Z, T, ldp)
            self._bgemm(B, H, T, Tk, dh, qb, (d, T, B), (q_ld, q_ld * T), (dh, 0, 0, q_col), kb, (d, Tk, B), (k_ld, k_ld * Tk),
                        (dh, 0, 0, k_col), alpha=scale, out_f32=S, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp)
            lib.softmax_fwd(S, B, H, T, Tk, ldp, lens, rate, self.seed, site, P_pre, P_drop, flags=flags)
            del S
        out = self._bf(B, T, d)
        # O = P V: V is read MN-major straight from its buffer (columns v_col + h*dh), no transposed copy
        self._bgemm(B, H, T, dh, Tk, P_drop, (Tk, T, Z), (ldp, T * ldp), (0, 0, 1, 0), kb, (d, Tk, B), (k_ld, k_ld * Tk),
                    (dh, 0, 0, v_col, 1), out_bf16=out, ld_out=d, out_batch_stride=T * d, out_h_col=dh, out_by_b=1, out_cols=dh)
        return out, dict(P_pre=P_pre, P_drop=P_drop, ldp=ldp, site=site, flags=flags, out=out)

    def _attn_bwd(self, c, B, H, dh, T, Tk, dout, qb, q_ld, q_col, kb, k_ld, k_col, v_col, lens, dq_buf, dq_ld, dq_col, dkv_buf,
                  dkv_ld, dk_col, dv_col, diag=None):
        """dout: bf16 (B,T,d) gradient of the attention output.  Writes dQ into dq_buf[:, :, dq_col:], dK / dV into
        dkv_buf[:, :, dk_col:] / [dv_col:] (bf16).  diag = (grad_scale, q_len, k_len) adds the gradient of the diagonal loss
        on the post-dropout probabilities to dP."""
        d = H * dh
        ldp, site, flags = c['ldp'], c['site'], c['flags']
        Z = B * H
        scale = 1.0 / math.sqrt(dh)
        rate = self.drop_rate
        dS = self._bf(Z, T, ldp)
        if diag is not None:
            dP = self._f32(Z, T, ldp)
            self._bgemm(B, H, T, Tk, dh, dout, (d, T, B), (d, d * T), (dh, 0, 0, 0), kb, (d, Tk, B), (k_ld, k_ld * Tk), (dh, 0, 0, v_col),
                        out_f32=dP, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp)
            lib.diag_loss_train(c['P_drop'], B, H, T, Tk, ldp, diag[1], diag[2], 0.0, self._loss_scratch, diag[0], dP)
            lib.softmax_bwd(c['P_pre'], dP, B, H, T, Tk, ldp, lens, scale, rate, self.seed, site, dS, flags=flags)
            del dP
        else:
            # dS straight out of the dP = dO V^T product: rowsum(P_drop * dP) = dO . O per (row, head), so the fp32 dP
            # matrix (Z*T*Tk*4 bytes) is never written or re-read
            D = self._f32(Z * T)
            lib.rowdot_heads(dout, c['out'], H, dh, D)
            if self._fused_probs(qb, kb, flags, dh, ldp):
                # sixteen-warp epilogue twin of the forward probability kernel (dropout decisions re-drawn from the hash)
                lib.attn_ds_bwd(dout, d, 0, kb, k_ld, v_col, B, H, T, dh, lens, c['P_pre'], D, scale, rate, self.seed, site, dS, ldp)
            else:   # dropout decisions read back from the saved P_drop
                self._bgemm(B, H, T, Tk, dh, dout, (d, T, B), (d, d * T), (dh, 0, 0, 0), kb, (d, Tk, B), (k_ld, k_ld * Tk),
                            (dh, 0, 0, v_col), out_bf16=dS, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp,
                            softmax_bwd=(c['P_pre'], D, scale, rate, self.seed, site, flags, lens, c['P_drop']))
        # dQ = dS K : A = dS (K-major over keys), B = K read MN-major
        self._bgemm(B, H, T, dh, Tk, dS, (Tk, T, Z), (ldp, T * ldp), (0, 0, 1, 0), kb, (d, Tk, B), (k_ld, k_ld * Tk),
                    (dh, 0, 0, k_col, 1), out_bf16=dq_buf, ld_out=dq_ld, out_batch_stride=T * dq_ld, out_h_col=dh, out_by_b=1,
                    out_cols=dh, out_ptr_off=dq_col)
        # dK = dS^T Q : A = dS read MN-major (= dS^T), B = Q read MN-major
        self._bgemm(B, H, Tk, dh, T, dS, (Tk, T, Z), (ldp, T * ldp), (0, 0, 1, 0, 1), qb, (d, T, B), (q_ld, q_ld * T),
                    (dh, 0, 0, q_col, 1), out_bf16=dkv_buf, ld_out=dkv_ld, out_batch_stride=Tk * dkv_ld, out_h_col=dh, out_by_b=1,
                    out_cols=dh, out_ptr_off=dk_col)
        # dV = P^T dO : A = P_drop read MN-major, B = dO read MN-major
        self._bgemm(B, H, Tk, dh, T, c['P_drop'], (Tk, T, Z), (ldp, T * ldp), (0, 0, 1, 0, 1), dout, (d, T, B), (d, d * T),
                    (dh, 0, 0, 0, 1), out_bf16=dkv_buf, ld_out=dkv_ld, out_batch_stride=Tk * dkv_ld, out_h_col=dh, out_by_b=1,
                    out_cols=dh, out_ptr_off=dv_col)

    # ------------------------------------------------------------------------------------------------
    # one self-attention block: forward (saving) and backward
    # ------------------------------------------------------------------------------------------------
    def _block_fwd(self, name, i, x_f, x_bf, lens, B, T):
        m, P, W = self.model, self.P, self.model.weights
        st = m._stacks[name]
        d, H = st['d'], st['heads'][i]
        dh = d // H
        pre = f'{name}.b{i}.'
        rate = self.drop_rate
        c = {'x_f': x_f, 'x_bf': x_bf, 'T': T}
        qkv = self._bf(B, T, 3 * d)
        m._gemm(P[pre + 'qkv'], B, T, [(x_bf, None, d, 0)], [0], [0], out_hi=qkv, ld_out=3 * d)
        attn, c_sa = self._attn_fwd(B, H, dh, T, T, qkv, 3 * d, 0, qkv, 3 * d, d, 2 * d, lens)
        y_f, y_bf, u1 = self._f32(B, T, d), self._bf(B, T, d), self._f32(B, T, d)
        site_o = self._site()
        m._gemm(P[pre + 'wo'], B, T, [(x_bf, None, d, 0), (attn, None, d, 0)], [0, 1], [0, 0], residual=x_f,
                ln=(W[pre + 'ln1.gamma'], W[pre + 'ln1.beta']), row_len=lens, out_f32=y_f, out_hi=y_bf, out_preln=u1,
                dropout=(rate, site_o))
        z_f, z_bf, u2 = self._f32(B, T, d), self._bf(B, T, d), self._f32(B, T, d)
        site_c = self._site()
        if i < st['n_dense']:
            F = int(st['ffn'])
            h = self._bf(B, T, F)
            m._gemm(P[pre + 'ffn1'], B, T, [(y_bf, None, d, 0)], [0], [0], relu=True, out_hi=h, ld_out=F)
            m._gemm(P[pre + 'ffn2'], B, T, [(h, None, F, 0)], [0], [0], residual=y_f, ln=(W[pre + 'ln2.gamma'], W[pre + 'ln2.beta']),
                    row_len=lens, out_f32=z_f, out_hi=z_bf, out_preln=u2, dropout=(rate, site_c))
            hs = [h]
        else:
            k = int(st['kernel'])
            shifts = m._conv_shifts(k)
            hs = []
            cur, ld = y_bf, d
            n = len(st['filters'])
            for j in range(n - 1):
                f = st['filters'][j]
                h = self._bf(B, T, f)
                m._gemm(P[pre + f'conv{j}'], B, T, [(cur, None, ld, 0)], [0] * k, shifts, relu=True, out_hi=h, ld_out=f)
                hs.append(h)
                cur, ld = h, f
            m._gemm(P[pre + f'conv{n - 1}'], B, T, [(cur, None, ld, 0)], [0] * k, shifts, residual=y_f,
                    ln=(W[pre + 'ln2.gamma'], W[pre + 'ln2.beta']), row_len=lens, out_f32=z_f, out_hi=z_bf, out_preln=u2,
                    dropout=(rate, site_c))
        c.update(qkv=qkv, sa=c_sa, attn=attn, y_f=y_f, y_bf=y_bf, u1=u1, u2=u2, hs=hs, sites=(site_o, site_c))
        return z_f, z_bf, c

    def _block_bwd(self, name, i, c, dz, lens, B, diag=None):
        """diag: see _attn_bwd."""
        m, P, W, G = self.model, self.P, self.model.weights, self.g
        st = m._stacks[name]
        d, H = st['d'], st['heads'][i]
        dh = d // H
        T = c['T']
        pre = f'{name}.b{i}.'
        rate = self.drop_rate
        site_o, site_c = c['sites']
        # ---- LayerNorm 2 (+ row mask) ; the branch gradient carries the branch dropout mask
        du2, g2 = self._f32(B, T, d), self._bf(B, T, d)
        last_b = G[pre + ('ffn2.b' if i < st['n_dense'] else f"conv{len(st['filters']) - 1}.b")]
        lib.layernorm_bwd(dz, c['u2'], W[pre + 'ln2.gamma'], B, T, d, d, LN_EPS, lens, False, du2, g2, G[pre + 'ln2.gamma'],
                          G[pre + 'ln2.beta'], pre_drop=(rate, site_c), seed=self.seed, dbias=last_b)
        if i < st['n_dense']:
            F = int(st['ffn'])
            h = c['hs'][0]
            self._wgrad([(h, F)], g2, d, B, T, F, d, [(0, 0)], G[pre + 'ffn2.w'])
            dh_ = self._bf(B, T, F)
            m._gemm(P[pre + 'ffn2.d'], B, T, [(g2, None, d, 0)], [0], [0], out_hi=dh_, ld_out=F)
            lib.relu_bwd_colsum(dh_, h, G[pre + 'ffn1.b'])     # ReLU mask + the bias gradient in one pass
            self._wgrad([(c['y_bf'], d)], dh_, F, B, T, d, F, [(0, 0)], G[pre + 'ffn1.w'])
            dy = self._f32(B, T, d)
            m._gemm(P[pre + 'ffn1.d'], B, T, [(dh_, None, F, 0)], [0], [0], residual=du2, out_f32=dy, ld_out=d)
        else:
            k = int(st['kernel'])
            shifts = m._conv_shifts(k)
            dshifts = [-s for s in shifts]
            n = len(st['filters'])
            inputs = [c['y_bf']] + c['hs']  # input of conv j
            in_dims = [d] + list(st['filters'][:-1])
            g_cur, g_dim = g2, d
            for j in range(n - 1, -1, -1):
                cin = in_dims[j]
                # bias gradients: the last conv's comes out of the LayerNorm backward kernel, the others out of the ReLU-mask pass
                self._wgrad([(inputs[j], cin)], g_cur, g_cur.shape[-1], B, T, cin, g_dim, [(0, s_) for s_ in shifts], G[pre + f'conv{j}.w'])
                kpad = _round_up(g_dim, 64)
                assert g_cur.shape[-1] == kpad, 'gradient operand must be padded to the packed contraction width'
                if j > 0:
                    dx_ = self._bf(B, T, cin)
                    m._gemm(P[pre + f'conv{j}.d'], B, T, [(g_cur, None, kpad, 0)], [0] * k, dshifts, out_hi=dx_, ld_out=cin)
                    lib.relu_bwd_colsum(dx_, inputs[j], G[pre + f'conv{j - 1}.b'])
                    g_cur, g_dim = dx_, cin
                else:
                    dy = self._f32(B, T, d)
                    m._gemm(P[pre + 'conv0.d'], B, T, [(g_cur, None, kpad, 0)], [0] * k, dshifts, residual=du2, out_f32=dy, ld_out=d)
        # ---- LayerNorm 1
        du1, g1 = self._f32(B, T, d), self._bf(B, T, d)
        lib.layernorm_bwd(dy, c['u1'], W[pre + 'ln1.gamma'], B, T, d, d, LN_EPS, lens, False, du1, g1, G[pre + 'ln1.gamma'],
                          G[pre + 'ln1.beta'], pre_drop=(rate, site_o), seed=self.seed, dbias=G[pre + 'wo.b'])
        self._wgrad([(c['x_bf'], d), (c['attn'], d)], g1, d, B, T, d, d, [(0, 0), (1, 0)], G[pre + 'wo.w'])
        dattn = self._bf(B, T, d)
        m._gemm(P[pre + 'wo.da'], B, T, [(g1, None, d, 0)], [0], [0], out_hi=dattn, ld_out=d)
        dx_acc = self._f32(B, T, d)
        m._gemm(P[pre + 'wo.dx'], B, T, [(g1, None, d, 0)], [0], [0], residual=du1, out_f32=dx_acc, ld_out=d)
        # ---- attention backward on the saved probabilities
        qkv = c['qkv']
        dqkv = self._bf(B, T, 3 * d)
        self._attn_bwd(c['sa'], B, H, dh, T, T, dattn, qkv, 3 * d, 0, qkv, 3 * d, d, 2 * d, lens, dqkv, 3 * d, 0, dqkv, 3 * d, d, 2 * d,
                       diag=diag)
        # ---- q/k/v projections
        # the three Dense layers own separate (d,d) kernels and biases but share the (B,T,3d) gradient buffer: one column-sum
        # launch with three outputs, one weight-gradient GEMM of width 3d into a scratch matrix, three strided adds
        lib.colsum_bf16_x3(dqkv, B * T, d, 3 * d, G[pre + 'wq.b'], G[pre + 'wk.b'], G[pre + 'wv.b'])
        dw_qkv = torch.zeros((d, 3 * d), dtype=torch.float32, device=self.dev)
        self._wgrad([(c['x_bf'], d)], dqkv, 3 * d, B, T, d, 3 * d, [(0, 0)], dw_qkv)
        for n_, nm in enumerate(('wq', 'wk', 'wv')):
            G[pre + nm + '.w'].add_(dw_qkv[:, n_ * d:(n_ + 1) * d])
        dx = self._f32(B, T, d)
        m._gemm(P[pre + 'qkv.d'], B, T, [(dqkv, None, 3 * d, 0)], [0], [0], residual=dx_acc, out_f32=dx, ld_out=d)
        return dx

    def _tmp_zero(self, n):
        return torch.zeros(n, dtype=torch.float32, device=self.dev)

    def _site(self):
        self.drop_sites += 1
        return self.drop_sites

    # ------------------------------------------------------------------------------------------------
    # predictors
    # ------------------------------------------------------------------------------------------------
    def _pred_fwd(self, name, x_bf, lens, B, T, relu_head):
        m, P, W = self.model, self.P, self.model.weights
        filt = m.config['duration_conv_filters' if name == 'dur_pred' else 'pitch_conv_filters']
        k = int(m.config['duration_kernel_size' if name == 'dur_pred' else 'pitch_kernel_size'])
        shifts = m._conv_shifts(k)
        rate = float(m.config.get('predictors_dropout', 0.0)) if self.use_dropout else 0.0
        cur, ld = x_bf, x_bf.shape[-1]
        us, outs, sites = [], [], []
        h_f = None
        for j, f in enumerate(filt):
            pl = P[f'{name}.conv{j}']
            h_f, o_bf, u = self._f32(B, T, pl.n_pad), self._bf(B, T, pl.n_pad), self._f32(B, T, pl.n_pad)
            site = self._site()
            m._gemm(pl, B, T, [(cur, None, ld, 0)], [0] * k, shifts, relu=True, ln=P[f'{name}.ln{j}'], out_f32=h_f, out_hi=o_bf,
                    out_preln=u, dropout_post=(rate, site))
            us.append(u)
            outs.append(o_bf)
            sites.append(site)
            cur, ld = o_bf, pl.n_pad
        out = self._f32(B, T)
        lib.statpred_head_fwd(h_f, int(filt[-1]), W[f'{name}.out.w'].reshape(-1), W[f'{name}.out.b'], relu_head, lens, out)
        return out, dict(us=us, outs=outs, h_f=h_f, x_bf=x_bf, sites=sites, rate=rate, out=out, relu=relu_head)

    def _pred_bwd(self, name, c, gout, lens, B, T, dx_acc):
        """Returns the accumulated encoder-output gradient (fp32)."""
        m, P, W, G = self.model, self.P, self.model.weights, self.g
        filt = [int(f) for f in m.config['duration_conv_filters' if name == 'dur_pred' else 'pitch_conv_filters']]
        k = int(m.config['duration_kernel_size' if name == 'dur_pred' else 'pitch_kernel_size'])
        shifts = m._conv_shifts(k)
        dshifts = [-s for s in shifts]
        d_enc = m._stacks['encoder']['d']
        ldh = c['h_f'].shape[-1]
        dh = self._f32(B, T, ldh)
        lib.statpred_head_bwd(gout, c['out'], c['h_f'], filt[-1], W[f'{name}.out.w'].reshape(-1), c['relu'], lens, dh,
                              G[f'{name}.out.w'].view(-1), G[f'{name}.out.b'])
        dz = dh
        n = len(filt)
        for j in range(n - 1, -1, -1):
            C = filt[j]
            ld = c['us'][j].shape[-1]
            gam = _pad_vec(W[f'{name}.ln{j}.gamma'], ld)
            dg, db = self._tmp_zero(ld), self._tmp_zero(ld)
            g_bf = self._bf(B, T, ld)
            lib.layernorm_bwd(dz, c['us'][j], gam, B, T, C, ld, LN_EPS, None, True, None, g_bf, dg, db,
                              post_drop=(c['rate'], c['sites'][j]), seed=self.seed, dbias=G[f'{name}.conv{j}.b'])
            G[f'{name}.ln{j}.gamma'].add_(dg[:C])
            G[f'{name}.ln{j}.beta'].add_(db[:C])
            cin = d_enc if j == 0 else filt[j - 1]
            src = c['x_bf'] if j == 0 else c['outs'][j - 1]
            self._wgrad([(src, src.shape[-1])], g_bf, ld, B, T, cin, C, [(0, s_) for s_ in shifts], G[f'{name}.conv{j}.w'])
            if j > 0:
                ldn = c['us'][j - 1].shape[-1]
                dz = self._f32(B, T, ldn)
                m._gemm(P[f'{name}.conv{j}.d'], B, T, [(g_bf, None, ld, 0)], [0] * k, dshifts, out_f32=dz, ld_out=ldn)
            else:
                out = self._f32(B, T, d_enc)
                m._gemm(P[f'{name}.conv0.d'], B, T, [(g_bf, None, ld, 0)], [0] * k, dshifts, residual=dx_acc, out_f32=out, ld_out=d_enc)
                return out

    # ------------------------------------------------------------------------------------------------
    # full step
    # ------------------------------------------------------------------------------------------------
    def forward_backward(self, phonemes, mel_tgt, dur_tgt, pitch_tgt, training=True, sync=None):
        """Eager step: forward (+ backward when training).  `sync.bucket_ready` is called as soon as the decoder gradients
        are final (the data-parallel all-reduce of that bucket then overlaps the encoder backward)."""
        self._set_salt(0)
        with self._step_state(self.model.step, training):
            gen = self._fb_gen(phonemes, mel_tgt, dur_tgt, pitch_tgt, training)
            out = next(gen)                 # forward (+ decoder backward)
            if training:
                if sync is not None:        # decoder gradients are final: start their all-reduce under the encoder backward
                    sync.bucket_ready(*self.decoder_range)
                next(gen, None)             # encoder-side backward
            else:
                gen.close()
            return out

    def _seed(self, iteration: int) -> int:
        """Dropout seed of the step at `iteration` (per rank)."""
        return (self.base_seed * 2654435761 + iteration * 40503 + self.rank * 97) & 0x7fffffff

    @contextlib.contextmanager
    def _step_state(self, iteration: int, training: bool):
        """While a step is issued: its dropout rate and seed, and the model's GEMMs in single-pass bf16."""
        m = self.model
        self.use_dropout = training and m.train_dropout
        self.drop_rate = float(m.config.get('dropout_rate', 0.0)) if self.use_dropout else 0.0
        self.seed = m._drop_seed = self._seed(iteration)
        saved_precision = m.precision
        m.precision = 'bf16'
        try:
            yield
        finally:
            m.precision = saved_precision

    def _set_salt(self, value: int):
        """Device-resident word XORed into every dropout seed (include/ttsb.h: ttsb_set_dropout_salt): 0 in eager steps,
        a per-step value under CUDA-graph replay (the captured seed arguments are frozen)."""
        if self._salt_dev is None:
            self._salt_dev = torch.zeros(1, dtype=torch.int32, device=self.dev)
            self._salt_host = torch.zeros(1, dtype=torch.int32).pin_memory()
            self._salt_value = 0
            self._salt_applied = 0      # what the library's constant memory currently holds
        if value == 0 and self._salt_applied == 0:
            return
        self._salt_host[0] = value
        self._salt_dev.copy_(self._salt_host, non_blocking=True)
        if value == 0:                  # eager path after graphed steps: reset the library state once
            lib.set_dropout_salt(self._salt_dev)
            self._salt_applied = 0

    def _fb_gen(self, phonemes, mel_tgt, dur_tgt, pitch_tgt, training=True, Tm_hint=None):
        """The step as a generator: yields the output dictionary after the forward pass + decoder backward (decoder
        gradients final), finishes with the encoder-side backward.  The caller holds the _step_state."""
        m, W, G = self.model, self.model.weights, self.g
        dev = self.dev
        self.drop_sites = 0
        P = self._pack()
        x = torch.as_tensor(phonemes).to(device=dev, dtype=torch.int32).contiguous()
        mel_tgt = torch.as_tensor(mel_tgt).to(device=dev, dtype=torch.float32).contiguous()
        dur_tgt = torch.as_tensor(dur_tgt).to(device=dev, dtype=torch.int32).contiguous()
        pitch_tgt = torch.as_tensor(pitch_tgt).to(device=dev, dtype=torch.float32).contiguous()
        B, Tp = x.shape
        d = m._stacks['encoder']['d']
        enc_len = torch.empty((B,), dtype=torch.int32, device=dev)
        lib.phoneme_lengths(x, 0, enc_len)
        h_f, h_bf, enc_ctx = self._encoder_fwd(x, enc_len)
        dur_out, dur_ctx = self._pred_fwd('dur_pred', h_bf, enc_len, B, Tp, True)
        pit_out, pit_ctx = self._pred_fwd('pitch_pred', h_bf, enc_len, B, Tp, False)
        h_pe = self._f32(B, Tp, d)
        pw = W['pitch_embed.w'].reshape(-1)
        lib.pitch_embed_add_fwd(h_f, pitch_tgt, pw, W['pitch_embed.b'], h_pe)
        dur_int = torch.empty((B, Tp), dtype=torch.int32, device=dev)
        dec_len = torch.empty((B,), dtype=torch.int32, device=dev)
        lib.durations_to_int(dur_tgt.float(), 1.0, None, None, dur_int, dec_len)
        mel_len = mel_tgt.shape[1]
        # decoder length = longest expanded row, but never shorter than the target: a data-parallel shard (or a batch
        # padded to a bucket length) may hold only rows shorter than the padded target of the GLOBAL batch, which the
        # reference would have processed at the global length (extra frames are padding rows, masked like any other)
        Tm = Tm_hint if Tm_hint is not None else max(int(dec_len.max().item()), mel_len)
        idx = torch.empty((B, Tm), dtype=torch.int32, device=dev)
        lib.expand_indices(dur_int, Tm, idx)
        dd = m._stacks['decoder']['d']
        expanded = self._f32(B, Tm, dd)
        lib.length_regulate_fwd(h_pe, idx, expanded)
        m_f, m_bf = self._f32(B, Tm, dd), self._bf(B, Tm, dd)
        site_d = self._site()
        lib.expand_ln_pe_fwd(h_pe, idx, W['decoder.ln.gamma'], W['decoder.ln.beta'], P['decoder.pe'],
                             W['decoder.pos_scalar'].reshape(1), LN_EPS, m_f, m_bf, None, drop=(self.drop_rate, self.seed, site_d))
        dec_ctx = []
        for i in range(len(m._stacks['decoder']['heads'])):
            m_f, m_bf, c = self._block_fwd('decoder', i, m_f, m_bf, dec_len, B, Tm)
            dec_ctx.append(c)
        mel = self._f32(B, Tm, m.mel_channels)
        m._gemm(P['out'], B, Tm, [(m_bf, None, dd, 0)], [0], [0], out_f32=mel, ld_out=m.mel_channels)
        # ---- losses (utils/losses.py:41-70, weights [1,1,3]) and their gradients
        losses = torch.zeros(3, dtype=torch.float32, device=dev)
        wts = m.loss_weights
        dmel = self._f32(B, Tm, m.mel_channels)
        ddur, dpit = self._f32(B, Tp), self._f32(B, Tp)
        lib.mae_loss(mel, B, Tm, mel_len, m.mel_channels, mel_tgt, wts[0], losses[0:1], dmel)
        lib.mae_loss(dur_out, B, Tp, Tp, 1, dur_tgt, wts[1], losses[1:2], ddur)
        lib.mae_loss(pit_out, B, Tp, Tp, 1, pitch_tgt, wts[2], losses[2:3], dpit)
        out = {'mel': mel, 'duration': dur_out[..., None], 'pitch': pit_out[..., None],
               'expanded_mask': mask_from_lengths(dec_len, Tm), 'encoder_attention': {}, 'decoder_attention': {},
               'losses': {'mel': losses[0], 'duration': losses[1], 'pitch': losses[2]},
               'loss': wts[0] * losses[0] + wts[1] * losses[1] + wts[2] * losses[2], 'mel_lengths': dec_len}
        if not training:
            yield out
            return
        # =============================== backward ===============================
        self.flat_g.zero_()
        C = m.mel_channels
        kpad = _round_up(C, 64)
        g = self._bf(B, Tm, kpad)
        lib.cast_bf16_pad(dmel, B * Tm, C, g, kpad)
        lib.colsum_bf16(g, B * Tm, C, kpad, G['out.b'])
        self._wgrad([(m_bf, dd)], g, kpad, B, Tm, dd, C, [(0, 0)], G['out.w'])
        dz = self._f32(B, Tm, dd)
        m._gemm(P['out.d'], B, Tm, [(g, None, kpad, 0)], [0], [0], out_f32=dz, ld_out=dd)
        for i in range(len(dec_ctx) - 1, -1, -1):
            dz = self._block_bwd('decoder', i, dec_ctx[i], dz, dec_len, B)
            dec_ctx[i] = None
        d_exp = self._prologue_bwd('decoder', dz, expanded, dec_len, B, Tm, site_d)
        yield out             # decoder gradients are final
        dh_pe = self._f32(B, Tp, d)
        lib.expand_bwd(d_exp, dur_int, dh_pe)
        lib.pitch_embed_bwd(dh_pe, pitch_tgt, pw, W['pitch_embed.b'], G['pitch_embed.w'].view(-1), G['pitch_embed.b'])
        # predictors read the encoder output; their input gradient is accumulated onto dh_pe
        acc = self._pred_bwd('dur_pred', dur_ctx, ddur, enc_len, B, Tp, dh_pe)
        acc = self._pred_bwd('pitch_pred', pit_ctx, dpit, enc_len, B, Tp, acc)
        self._encoder_bwd(enc_ctx, acc)

    # ------------------------------------------------------------------------------------------------
    # encoder: embedding, LayerNorm, PE and the self-attention blocks (both engines)
    # ------------------------------------------------------------------------------------------------
    def _encoder_fwd(self, x, enc_len):
        m, W = self.model, self.model.weights
        B, Tp = x.shape
        d = m._stacks['encoder']['d']
        # the embedding rows are kept as the LayerNorm input for the backward pass
        e_rows = self._f32(1, B * Tp, d)
        lib.length_regulate_fwd(W['embedding'].view(1, -1, d), x.view(1, -1), e_rows)
        h_f, h_bf = self._f32(B, Tp, d), self._bf(B, Tp, d)
        site = self._site()
        lib.embed_ln_pe_fwd(x, W['embedding'], W['encoder.ln.gamma'], W['encoder.ln.beta'], self.P['encoder.pe'],
                            W['encoder.pos_scalar'].reshape(1), LN_EPS, h_f, h_bf, None, drop=(self.drop_rate, self.seed, site))
        blocks = []
        for i in range(len(m._stacks['encoder']['heads'])):
            h_f, h_bf, c = self._block_fwd('encoder', i, h_f, h_bf, enc_len, B, Tp)
            blocks.append(c)
        return h_f, h_bf, dict(x=x, lens=enc_len, e_rows=e_rows.view(B, Tp, d), site=site, blocks=blocks)

    def _encoder_bwd(self, ctx, dz, diag=None):
        """dz: fp32 gradient of the encoder output; diag: see _attn_bwd (diagonal loss on the encoder maps)."""
        blocks, lens, (B, Tp, _) = ctx['blocks'], ctx['lens'], ctx['e_rows'].shape
        for i in range(len(blocks) - 1, -1, -1):
            dz = self._block_bwd('encoder', i, blocks[i], dz, lens, B, diag=diag)
            blocks[i] = None
        de = self._prologue_bwd('encoder', dz, ctx['e_rows'], lens, B, Tp, ctx['site'])
        lib.embedding_bwd(de, ctx['x'], self.g['embedding'])

    # ------------------------------------------------------------------------------------------------
    # the step as CUDA graphs, Adam launched eagerly
    # ------------------------------------------------------------------------------------------------
    def step_graphed(self, phonemes, mel_tgt, dur_tgt, pitch_tgt, sync=None):
        """Replays the step captured for this input shape (captures it on first use) as two graphs: forward + decoder
        backward | encoder-side backward.  ~400 launches, each with host-side tensor-map encoding, become two graph
        launches: the eager step is host-launch bound (tools/step_cpu_time.py)."""
        m = self.model
        ins = [torch.as_tensor(t) for t in (phonemes, mel_tgt, dur_tgt, pitch_tgt)]
        B, Tp = ins[0].shape
        mel_len = ins[1].shape[1]
        Tm = max(int(ins[2].sum(1).max()), mel_len)          # host sync only if the durations live on the device
        key = (B, Tp, mel_len, Tm, bool(m.train_dropout), float(m.config.get('dropout_rate', 0.0)))

        def capture(static):
            with self._step_state(0, True):      # the seed is frozen in the graph; the salt varies per step
                self._set_salt(1)
                gen = self._fb_gen(*static, training=True, Tm_hint=Tm)

                def forward():
                    lib.set_dropout_salt(self._salt_dev)
                    return next(gen)
                return _capture_graphs(self, self.dev, lambda: list(self._fb_gen(*static, training=True, Tm_hint=Tm)),
                                       forward, lambda: next(gen, None))
        return self._replay_step(key, ins, (torch.int32, torch.float32, torch.int32, torch.float32), capture, sync)

    def _replay_step(self, key, inputs, dtypes, capture, sync=None):
        """Replays the graphs of `key` in self._graphs, captured on first use by `capture(static inputs)` -> [(graph, output)]
        (the first graph's output is the step's output dictionary).  Per-step state that the captured kernel arguments
        cannot carry lives in device memory: the dropout salt (see _set_salt); Adam's scalars are not captured (one eager
        launch).  Outputs are views of static buffers, valid until the next step of the same shape (loss / losses are
        copied out)."""
        ent = _lru_get(self._graphs, key)
        if ent is None:
            _lru_make_room(self._graphs, 4)
            static = _static_inputs(self.dev, inputs, dtypes)
            captured = capture(static)
            ent = self._graphs[key] = {'ins': static, 'graphs': [g for g, _ in captured], 'out': captured[0][1]}
        else:
            _fill_inputs(ent['ins'], inputs)
        self._set_salt(((self.model.step + 1) * 40503 + 12345) & 0x7fffffff)
        self._salt_applied = 1
        first, *rest = ent['graphs']
        _replay(first)
        if sync is not None:      # decoder gradients are final
            sync.bucket_ready(*self.decoder_range)
        for g in rest:
            _replay(g)
        out = dict(ent['out'])
        out['loss'] = out['loss'].clone()
        out['losses'] = {k: v.clone() for k, v in out['losses'].items()}
        return out

    def _prologue_bwd(self, name, g, u, lens, B, T, site):
        m, W, G = self.model, self.model.weights, self.g
        d = m._stacks[name]['d']
        lib.pe_scalar_bwd(g, self.P[f'{name}.pe'], G[f'{name}.pos_scalar'].view(1), drop=(self.drop_rate, self.seed, site))
        du = self._f32(B, T, d)
        lib.layernorm_bwd(g, u.contiguous(), W[f'{name}.ln.gamma'], B, T, d, d, LN_EPS, None, False, du, None,
                          G[f'{name}.ln.gamma'], G[f'{name}.ln.beta'], post_drop=(self.drop_rate, site), seed=self.seed)
        return du

    # ------------------------------------------------------------------------------------------------
    def apply_adam(self, opt: Adam, grad_scale: float = 1.0):
        if opt.m is None:
            opt.m = torch.zeros_like(self.flat_w)
            opt.v = torch.zeros_like(self.flat_w)
        opt.iterations += 1
        t = opt.iterations
        lr_t = opt.lr * math.sqrt(1.0 - opt.beta_2 ** t) / (1.0 - opt.beta_1 ** t)
        lib.adam_tf_step(self.flat_w, self.flat_g, opt.m, opt.v, lr_t, opt.beta_1, opt.beta_2, opt.epsilon, grad_scale)
        self.model._packed = None
