"""Training step of the Aligner (reference: model/models.py:168-216 ``_gta_forward`` + ``_train_step``): teacher-forced
forward in single-pass bf16 with saved activations, hand-written backward, Keras-form Adam -- on the same kernels as the
ForwardTransformer engine (training.py), whose packing, encoder, attention core and graph replay it shares; this file
adds the CrossAttentionDenseBlock (layers.py:330-349), DecoderPrenet, FinalProj / Postnet and the Aligner losses.

Differences to the ForwardTransformer blocks that matter for the backward pass:
  * decoder rows are never re-masked (no ``row_len`` in the LayerNorm GEMMs / LayerNorm backward);
  * decoder self-attention uses the look-ahead + padding mask and keeps every query row (softmax flags);
  * cross-attention reads K|V from a second GEMM over the encoder output; its gradient flows back into the encoder
    output from every decoder block (accumulated through the residual input of the data-gradient GEMM);
  * the diagonal loss (models.py:186-207) is taken on the post-dropout attention probabilities and adds a term to dP.
"""
from __future__ import annotations

import torch

from .. import lib
from .models import LN_EPS, _capture_graphs, _PackedLinear, _qkv_block_n, _round_up
from .training import TrainEngine
from .transformer_utils import mask_from_lengths

FULLQ = lib.SOFTMAX_FULL_QUERIES
CAUSAL = lib.SOFTMAX_CAUSAL


class AlignerTrainEngine(TrainEngine):
    # ------------------------------------------------------------------------------------------------
    # packed operands
    # ------------------------------------------------------------------------------------------------
    def _build_packs(self):
        m = self.model
        W = m.weights
        enc, dec = m._stacks['encoder'], m._stacks['decoder']
        d_enc, d, mel = enc['d'], dec['d'], m.mel_channels
        for i, _ in enumerate(enc['heads']):
            self._pack_attention(f'encoder.b{i}.', d_enc)
            self._pack_ffn(f'encoder.b{i}.', d_enc, int(enc['ffn']))
        kmel = _round_up(mel, 64)
        pd = int(m.config['decoder_prenet_dimension'])
        self._fwd('prenet.d1', [(W['prenet.d1.w'], W['prenet.d1.b'])], kmel, [kmel], k_valid=mel)
        self._fwd('prenet.d2', [(W['prenet.d2.w'], W['prenet.d2.b'])], pd, [pd])
        self._dgrad_dense('prenet.d2.d', [W['prenet.d2.w']], pd)
        for i, _ in enumerate(dec['heads']):
            pre = f'decoder.b{i}.'
            self._pack_attention(pre + 'sa.', d)
            c = pre + 'ca.'
            self._fwd(c + 'q', [(W[c + 'wq.w'], W[c + 'wq.b'])], d, [d])
            self._dgrad_dense(c + 'q.d', [W[c + 'wq.w']], d)
            kv = [(W[c + 'wk.w'], W[c + 'wk.b']), (W[c + 'wv.w'], W[c + 'wv.b'])]
            self._fwd(c + 'kv', kv, d_enc, [d_enc], block_n=_qkv_block_n(d))
            self._dgrad_dense(c + 'kv.d', [w for w, _ in kv], d_enc)
            self._pack_wo(c, d)
            self._pack_ffn(pre, d, int(dec['ffn']))
        # FinalProj[:, :, :r*mel] per reduction factor (models.py:146); Postnet: mel | stop heads in one GEMM
        self._fp = {}
        for r in range(1, m.max_r + 1):
            N = r * mel
            w, b = W['final_proj.w'][:, :N], W['final_proj.b'][:N]
            pl = _PackedLinear.empty(d, N, [d], self.dev)
            self._desc(w, pl.w_hi.data_ptr(), N, pl.n_pad, d, d, d, 1, 0, W['final_proj.w'].shape[1], d)
            self._desc(b, pl.bias.data_ptr(), 1, 1, pl.n_pad, pl.n_pad, N, 0, 0, 1, pl.n_pad, f32=1)
            npad = _round_up(N, 64)
            pd_ = _PackedLinear.empty(npad, d, [npad], self.dev, bias=False)
            self._desc(w, pd_.w_hi.data_ptr(), d, pd_.n_pad, npad, npad, N, W['final_proj.w'].shape[1], 0, 1, npad)
            self._fp[r] = (pl, pd_)
        post = [(W['postnet.mel.w'], W['postnet.mel.b']), (W['postnet.stop.w'], W['postnet.stop.b'])]
        self._fwd('postnet', post, kmel, [kmel], k_valid=mel)
        self._dgrad_dense('postnet.d', [w for w, _ in post], mel)
        self.P['encoder.pe'] = m._prepare_pe('encoder')

    # ------------------------------------------------------------------------------------------------
    # CrossAttentionDenseBlock
    # ------------------------------------------------------------------------------------------------
    def _cadb_fwd(self, i, x_f, x_bf, enc_bf, enc_len, dec_len, B, T, Tp):
        m, P, W = self.model, self.P, self.model.weights
        dec, d_enc = m._stacks['decoder'], m._stacks['encoder']['d']
        d, H = dec['d'], dec['heads'][i]
        dh = d // H
        pre = f'decoder.b{i}.'
        rate = self.drop_rate
        c = {'x_f': x_f, 'x_bf': x_bf}
        # ---- self-attention (look-ahead + padding mask), residual, LayerNorm
        qkv = self._bf(B, T, 3 * d)
        m._gemm(P[pre + 'sa.qkv'], B, T, [(x_bf, None, d, 0)], [0], [0], out_hi=qkv, ld_out=3 * d)
        attn, c_sa = self._attn_fwd(B, H, dh, T, T, qkv, 3 * d, 0, qkv, 3 * d, d, 2 * d, dec_len, CAUSAL | FULLQ)
        y_f, y_bf, u1 = self._f32(B, T, d), self._bf(B, T, d), self._f32(B, T, d)
        site_o = self._site()
        m._gemm(P[pre + 'sa.wo'], B, T, [(x_bf, None, d, 0), (attn, None, d, 0)], [0, 1], [0, 0], residual=x_f,
                ln=(W[pre + 'sa.ln.gamma'], W[pre + 'sa.ln.beta']), out_f32=y_f, out_hi=y_bf, out_preln=u1, dropout=(rate, site_o))
        # ---- cross-attention onto the encoder output
        qb = self._bf(B, T, d)
        kvb = self._bf(B, Tp, 2 * d)
        m._gemm(P[pre + 'ca.q'], B, T, [(y_bf, None, d, 0)], [0], [0], out_hi=qb, ld_out=d)
        m._gemm(P[pre + 'ca.kv'], B, Tp, [(enc_bf, None, d_enc, 0)], [0], [0], out_hi=kvb, ld_out=2 * d)
        ca, c_ca = self._attn_fwd(B, H, dh, T, Tp, qb, d, 0, kvb, 2 * d, 0, d, enc_len, FULLQ)
        z_f, z_bf, u2 = self._f32(B, T, d), self._bf(B, T, d), self._f32(B, T, d)
        site_c = self._site()
        m._gemm(P[pre + 'ca.wo'], B, T, [(y_bf, None, d, 0), (ca, None, d, 0)], [0, 1], [0, 0], residual=y_f,
                ln=(W[pre + 'ca.ln.gamma'], W[pre + 'ca.ln.beta']), out_f32=z_f, out_hi=z_bf, out_preln=u2, dropout=(rate, site_c))
        # ---- feed-forward
        F = int(dec['ffn'])
        h = self._bf(B, T, F)
        m._gemm(P[pre + 'ffn1'], B, T, [(z_bf, None, d, 0)], [0], [0], relu=True, out_hi=h, ld_out=F)
        o_f, o_bf, u3 = self._f32(B, T, d), self._bf(B, T, d), self._f32(B, T, d)
        site_f = self._site()
        m._gemm(P[pre + 'ffn2'], B, T, [(h, None, F, 0)], [0], [0], residual=z_f, ln=(W[pre + 'ln2.gamma'], W[pre + 'ln2.beta']),
                out_f32=o_f, out_hi=o_bf, out_preln=u3, dropout=(rate, site_f))
        c.update(qkv=qkv, attn=attn, sa=c_sa, y_bf=y_bf, u1=u1, qb=qb, kvb=kvb, ca=ca, cac=c_ca, z_bf=z_bf, u2=u2, h=h, u3=u3,
                 sites=(site_o, site_c, site_f))
        return o_f, o_bf, c

    def _cadb_bwd(self, i, c, do, enc_bf, enc_len, dec_len, d_enc_acc, B, T, Tp, diag):
        m, P, W, G = self.model, self.P, self.model.weights, self.g
        dec, d_enc = m._stacks['decoder'], m._stacks['encoder']['d']
        d, H = dec['d'], dec['heads'][i]
        dh = d // H
        pre = f'decoder.b{i}.'
        rate = self.drop_rate
        site_o, site_c, site_f = c['sites']
        F = int(dec['ffn'])
        # ---- FFNResNorm
        du3, g3 = self._f32(B, T, d), self._bf(B, T, d)
        lib.layernorm_bwd(do, c['u3'], W[pre + 'ln2.gamma'], B, T, d, d, LN_EPS, None, False, du3, g3, G[pre + 'ln2.gamma'],
                          G[pre + 'ln2.beta'], pre_drop=(rate, site_f), seed=self.seed, dbias=G[pre + 'ffn2.b'])
        h = c['h']
        self._wgrad([(h, F)], g3, d, B, T, F, d, [(0, 0)], G[pre + 'ffn2.w'])
        dh_ = self._bf(B, T, F)
        m._gemm(P[pre + 'ffn2.d'], B, T, [(g3, None, d, 0)], [0], [0], out_hi=dh_, ld_out=F)
        lib.relu_bwd(dh_, h)
        lib.colsum_bf16(dh_, B * T, F, F, G[pre + 'ffn1.b'])
        self._wgrad([(c['z_bf'], d)], dh_, F, B, T, d, F, [(0, 0)], G[pre + 'ffn1.w'])
        dz = self._f32(B, T, d)
        m._gemm(P[pre + 'ffn1.d'], B, T, [(dh_, None, F, 0)], [0], [0], residual=du3, out_f32=dz, ld_out=d)
        # ---- CrossAttentionResnorm
        du2, g2 = self._f32(B, T, d), self._bf(B, T, d)
        lib.layernorm_bwd(dz, c['u2'], W[pre + 'ca.ln.gamma'], B, T, d, d, LN_EPS, None, False, du2, g2, G[pre + 'ca.ln.gamma'],
                          G[pre + 'ca.ln.beta'], pre_drop=(rate, site_c), seed=self.seed, dbias=G[pre + 'ca.wo.b'])
        self._wgrad([(c['y_bf'], d), (c['ca'], d)], g2, d, B, T, d, d, [(0, 0), (1, 0)], G[pre + 'ca.wo.w'])
        dca = self._bf(B, T, d)
        m._gemm(P[pre + 'ca.wo.da'], B, T, [(g2, None, d, 0)], [0], [0], out_hi=dca, ld_out=d)
        dy_acc = self._f32(B, T, d)
        m._gemm(P[pre + 'ca.wo.dx'], B, T, [(g2, None, d, 0)], [0], [0], residual=du2, out_f32=dy_acc, ld_out=d)
        dq = self._bf(B, T, d)
        dkv = self._bf(B, Tp, 2 * d)
        self._attn_bwd(c['cac'], B, H, dh, T, Tp, dca, c['qb'], d, 0, c['kvb'], 2 * d, 0, d, enc_len, dq, d, 0, dkv, 2 * d, 0, d,
                       diag=diag)
        lib.colsum_bf16(dq, B * T, d, d, G[pre + 'ca.wq.b'])
        self._wgrad([(c['y_bf'], d)], dq, d, B, T, d, d, [(0, 0)], G[pre + 'ca.wq.w'])
        dy = self._f32(B, T, d)
        m._gemm(P[pre + 'ca.q.d'], B, T, [(dq, None, d, 0)], [0], [0], residual=dy_acc, out_f32=dy, ld_out=d)
        for n_, nm in enumerate(('wk', 'wv')):
            gs = dkv[..., n_ * d:]
            lib.colsum_bf16(gs, B * Tp, d, 2 * d, G[pre + 'ca.' + nm + '.b'])
            self._wgrad([(enc_bf, d_enc)], gs, 2 * d, B, Tp, d_enc, d, [(0, 0)], G[pre + 'ca.' + nm + '.w'])
        d_enc_new = self._f32(B, Tp, d_enc)
        m._gemm(P[pre + 'ca.kv.d'], B, Tp, [(dkv, None, 2 * d, 0)], [0], [0], residual=d_enc_acc, out_f32=d_enc_new, ld_out=d_enc)
        # ---- SelfAttentionResNorm
        du1, g1 = self._f32(B, T, d), self._bf(B, T, d)
        lib.layernorm_bwd(dy, c['u1'], W[pre + 'sa.ln.gamma'], B, T, d, d, LN_EPS, None, False, du1, g1, G[pre + 'sa.ln.gamma'],
                          G[pre + 'sa.ln.beta'], pre_drop=(rate, site_o), seed=self.seed, dbias=G[pre + 'sa.wo.b'])
        self._wgrad([(c['x_bf'], d), (c['attn'], d)], g1, d, B, T, d, d, [(0, 0), (1, 0)], G[pre + 'sa.wo.w'])
        dattn = self._bf(B, T, d)
        m._gemm(P[pre + 'sa.wo.da'], B, T, [(g1, None, d, 0)], [0], [0], out_hi=dattn, ld_out=d)
        dx_acc = self._f32(B, T, d)
        m._gemm(P[pre + 'sa.wo.dx'], B, T, [(g1, None, d, 0)], [0], [0], residual=du1, out_f32=dx_acc, ld_out=d)
        qkv = c['qkv']
        dqkv = self._bf(B, T, 3 * d)
        self._attn_bwd(c['sa'], B, H, dh, T, T, dattn, qkv, 3 * d, 0, qkv, 3 * d, d, 2 * d, dec_len, dqkv, 3 * d, 0, dqkv, 3 * d, d, 2 * d)
        for n_, nm in enumerate(('wq', 'wk', 'wv')):
            gs = dqkv[..., n_ * d:]
            lib.colsum_bf16(gs, B * T, d, 3 * d, G[pre + 'sa.' + nm + '.b'])
            self._wgrad([(c['x_bf'], d)], gs, 3 * d, B, T, d, d, [(0, 0)], G[pre + 'sa.' + nm + '.w'])
        dx = self._f32(B, T, d)
        m._gemm(P[pre + 'sa.qkv.d'], B, T, [(dqkv, None, 3 * d, 0)], [0], [0], residual=dx_acc, out_f32=dx, ld_out=d)
        return dx, d_enc_new

    # ------------------------------------------------------------------------------------------------
    # full step
    # ------------------------------------------------------------------------------------------------
    def step_graphed(self, inp, tar, stop_prob):
        """forward + backward of the teacher-forced step as ONE CUDA graph per input shape (single process; with a gradient
        all-reduce in the middle the eager path is used).  Per-step dropout masks come from the device-resident salt
        (TrainEngine._set_salt); Adam stays an eager launch."""
        m = self.model
        ins = [torch.as_tensor(t) for t in (inp, tar, stop_prob)]
        key = (tuple(ins[0].shape), tuple(ins[1].shape), int(m.r), m.force_encoder_diagonal, m.force_decoder_diagonal,
               bool(m.train_dropout))

        def capture(static):
            def step():
                lib.set_dropout_salt(self._salt_dev)
                return self.forward_backward(*static, training=True)
            self._set_salt(1)
            return _capture_graphs(self, self.dev, lambda: self.forward_backward(*static, training=True), step)
        return self._replay_step(key, ins, (torch.int32, torch.float32, torch.int32), capture)

    def forward_backward(self, inp, tar, stop_prob, training=True, sync=None):
        m, W, G = self.model, self.model.weights, self.g
        dev = self.dev
        self.drop_sites = 0
        with self._step_state(m.step, training):
            prenet_rate = float(m.config.get('decoder_prenet_dropout', 0.0)) if self.use_dropout else 0.0
            P = self._pack()
            r = int(m.r)
            mel = m.mel_channels
            kmel = _round_up(mel, 64)
            x = torch.as_tensor(inp).to(device=dev, dtype=torch.int32).contiguous()
            tar = torch.as_tensor(tar).to(device=dev, dtype=torch.float32)
            stop = torch.as_tensor(stop_prob).to(device=dev, dtype=torch.int32)
            tar_inp, tar_real, tar_stop = tar[:, :-1], tar[:, 1:].contiguous(), stop[:, 1:].contiguous()
            mel_len = tar_inp.shape[1]
            tgt = tar_inp[:, 0::r, :].contiguous()
            B, Tp = x.shape
            T = tgt.shape[1]
            d_enc, d = m._stacks['encoder']['d'], m._stacks['decoder']['d']
            enc_len = torch.empty((B,), dtype=torch.int32, device=dev)
            lib.phoneme_lengths(x, 0, enc_len)
            dec_len = torch.empty((B,), dtype=torch.int32, device=dev)
            lib.mel_lengths(tgt, 0.0, dec_len)
            _, enc_bf, enc_ctx = self._encoder_fwd(x, enc_len)
            # ---- decoder prenet (layers.py:420-443): relu Dense -> dropout -> relu Dense -> dropout
            t_pad = self._bf(B, T, kmel)
            lib.cast_bf16_pad(tgt, B * T, mel, t_pad, kmel)
            pdim = int(m.config['decoder_prenet_dimension'])
            h1 = self._bf(B, T, pdim)
            site_p1 = self._site()
            m._gemm(P['prenet.d1'], B, T, [(t_pad, None, kmel, 0)], [0], [0], relu=True, out_hi=h1, ld_out=pdim, dropout=(prenet_rate, site_p1))
            pre_out, h2 = self._f32(B, T, d), self._bf(B, T, d)
            site_p2 = self._site()
            m._gemm(P['prenet.d2'], B, T, [(h1, None, pdim, 0)], [0], [0], relu=True, out_f32=pre_out, out_hi=h2, ld_out=d,
                    dropout=(prenet_rate, site_p2))
            # ---- CrossAttentionBlocks prologue: LN(inputs) + scalar * PE[:, :T*r:r] -> dropout
            P['decoder.pe'] = m._decoder_pe(r)
            idx = torch.arange(T, dtype=torch.int32, device=dev)[None, :].expand(B, T).contiguous()
            x_f, x_bf = self._f32(B, T, d), self._bf(B, T, d)
            site_d = self._site()
            lib.expand_ln_pe_fwd(pre_out, idx, W['decoder.ln.gamma'], W['decoder.ln.beta'], P['decoder.pe'],
                                 W['decoder.pos_scalar'].reshape(1), LN_EPS, x_f, x_bf, None, drop=(self.drop_rate, self.seed, site_d))
            dec_ctx = []
            n_dec = len(m._stacks['decoder']['heads'])
            for i in range(n_dec):
                x_f, x_bf, c = self._cadb_fwd(i, x_f, x_bf, enc_bf, enc_len, dec_len, B, T, Tp)
                dec_ctx.append(c)
            # ---- FinalProj[:, :, :r*mel] -> (B, T*r, mel) -> Postnet
            fp, fp_d = self._fp[r]
            n_fp = r * mel
            lin = self._f32(B, T, n_fp)
            m._gemm(fp, B, T, [(x_bf, None, d, 0)], [0], [0], out_f32=lin, ld_out=n_fp)
            Tr = T * r
            linear = lin.view(B, Tr, mel)
            l_pad = self._bf(B, Tr, kmel)
            lib.cast_bf16_pad(linear, B * Tr, mel, l_pad, kmel)
            pn = P['postnet']
            post = self._f32(B, Tr, pn.n_pad)
            m._gemm(pn, B, Tr, [(l_pad, None, kmel, 0)], [0], [0], out_f32=post)
            mel_out = post[..., :mel].contiguous()
            stop_out = post[..., mel:mel + 3].contiguous()
            # ---- losses (models.py:179-207; loss weights [1, 1])
            wts = m.loss_weights
            losses = torch.zeros(3, dtype=torch.float32, device=dev)
            dmel = self._f32(B, Tr, mel)
            dstop = self._f32(B, Tr, 3)
            lib.mae_loss(mel_out, B, Tr, mel_len, mel, tar_real, wts[0], losses[0:1], dmel)
            lib.scaled_ce_loss(stop_out, mel_len, 3, tar_stop, m.stop_prob_index, m.stop_scaling, losses[1:2], wts[1], dstop)
            enc_blocks = enc_ctx['blocks']
            n_maps = (n_dec if m.force_decoder_diagonal else 0) + (len(enc_blocks) if m.force_encoder_diagonal else 0)
            norm = 1.0 + n_maps
            if m.force_decoder_diagonal:
                for i, c in enumerate(dec_ctx):
                    H = m._stacks['decoder']['heads'][i]
                    lib.diag_loss_train(c['cac']['P_drop'], B, H, T, Tp, c['cac']['ldp'], dec_len, enc_len, 1.0 / norm, losses[2:3], 0.0, None)
            if m.force_encoder_diagonal:
                for i, c in enumerate(enc_blocks):
                    H = m._stacks['encoder']['heads'][i]
                    lib.diag_loss_train(c['sa']['P_drop'], B, H, Tp, Tp, c['sa']['ldp'], enc_len, enc_len, 1.0 / norm, losses[2:3], 0.0, None)
            out = {'mel': mel_out, 'stop_prob': stop_out, 'linear': linear, 'decoder_output': x_f,
                   'mel_mask': mask_from_lengths(dec_len, T), 'text_mask': mask_from_lengths(enc_len, Tp),
                   'mel_lengths': dec_len, 'text_lengths': enc_len, 'decoder_attention': {}, 'encoder_attention': {},
                   'losses': {'mel': losses[0], 'stop_prob': losses[1], 'diag_loss': losses[2]},
                   'loss': wts[0] * losses[0] + wts[1] * losses[1] + losses[2]}
            if not training:
                return out
            # =============================== backward ===============================
            self.flat_g.zero_()
            g_post = self._bf(B, Tr, kmel)   # columns 0..79: d mel, 80..82: d stop logits, rest zero
            gp32 = torch.zeros((B, Tr, kmel), dtype=torch.float32, device=dev)
            gp32[..., :mel] = dmel
            gp32[..., mel:mel + 3] = dstop
            lib.cast_bf16_pad(gp32, B * Tr, kmel, g_post, kmel)
            lib.colsum_bf16(g_post, B * Tr, mel, kmel, G['postnet.mel.b'])
            lib.colsum_bf16(g_post[..., mel:], B * Tr, 3, kmel, G['postnet.stop.b'])
            self._wgrad([(l_pad, kmel)], g_post, kmel, B, Tr, mel, mel, [(0, 0)], G['postnet.mel.w'])
            self._wgrad([(l_pad, kmel)], g_post[..., mel:], kmel, B, Tr, mel, 3, [(0, 0)], G['postnet.stop.w'])
            dlin = self._f32(B, Tr, mel)
            m._gemm(P['postnet.d'], B, Tr, [(g_post, None, kmel, 0)], [0], [0], out_f32=dlin, ld_out=mel)
            # FinalProj: (B, T*r, mel) gradient is the (B, T, r*mel) gradient of the sliced Dense output
            nfp_pad = _round_up(n_fp, 64)
            g_fp = self._bf(B, T, nfp_pad)
            lib.cast_bf16_pad(dlin.view(B * T, n_fp), B * T, n_fp, g_fp, nfp_pad)
            db = torch.zeros(_round_up(n_fp, 8), dtype=torch.float32, device=dev)
            lib.colsum_bf16(g_fp, B * T, n_fp, nfp_pad, db)
            G['final_proj.b'][:n_fp].add_(db[:n_fp])
            dw = torch.zeros((d, n_fp), dtype=torch.float32, device=dev)
            self._wgrad([(x_bf, d)], g_fp, nfp_pad, B, T, d, n_fp, [(0, 0)], dw)
            G['final_proj.w'][:, :n_fp].add_(dw)
            dz = self._f32(B, T, d)
            m._gemm(fp_d, B, T, [(g_fp, None, nfp_pad, 0)], [0], [0], out_f32=dz, ld_out=d)
            # decoder blocks
            d_enc_acc = None
            diag = (1.0 / norm, dec_len, enc_len) if m.force_decoder_diagonal else None
            for i in range(n_dec - 1, -1, -1):
                dz, d_enc_acc = self._cadb_bwd(i, dec_ctx[i], dz, enc_bf, enc_len, dec_len, d_enc_acc, B, T, Tp, diag)
                dec_ctx[i] = None
            d_pre = self._prologue_bwd('decoder', dz, pre_out, None, B, T, site_d)
            # prenet: relu + dropout gradients from the saved (post-dropout) outputs, then the two Dense layers
            keep = 1.0 / (1.0 - prenet_rate) if prenet_rate > 0 else 1.0
            g2 = self._bf(B, T, d)
            lib.cast_bf16_pad(d_pre, B * T, d, g2, d)
            lib.relu_bwd(g2, h2)
            if keep != 1.0:
                g2.mul_(keep)
            lib.colsum_bf16(g2, B * T, d, d, G['prenet.d2.b'])
            self._wgrad([(h1, pdim)], g2, d, B, T, pdim, d, [(0, 0)], G['prenet.d2.w'])
            g1 = self._bf(B, T, pdim)
            m._gemm(P['prenet.d2.d'], B, T, [(g2, None, d, 0)], [0], [0], out_hi=g1, ld_out=pdim)
            lib.relu_bwd(g1, h1)
            if keep != 1.0:
                g1.mul_(keep)
            lib.colsum_bf16(g1, B * T, pdim, pdim, G['prenet.d1.b'])
            self._wgrad([(t_pad, kmel)], g1, pdim, B, T, mel, pdim, [(0, 0)], G['prenet.d1.w'])
            if sync is not None:
                sync.bucket_ready(*self.decoder_range)
            # encoder (the encoder maps' diagonal loss adds to dP inside the block backward)
            self._encoder_bwd(enc_ctx, d_enc_acc, diag=(1.0 / norm, enc_len, enc_len) if m.force_encoder_diagonal else None)
            return out
