"""Aligner: host-side mirror of the reference's teacher-forced encoder-decoder (model/models.py:15-341) -- the model
that produces the attention maps durations are extracted from (SURVEY.md section 8(f), next row #1).

Built here: the teacher-forced forward (``call`` / ``_forward`` / ``_forward_encoder`` / ``_forward_decoder``) and the
validation step with its losses (``_val_step`` = ``_gta_forward(training=False)``, models.py:168-220), every layer
through libttsb.so; ``_train_step`` (teacher-forced forward with dropout in single-pass bf16, hand-written backward,
Keras-form Adam) lives in aligner_training.py; ``predict`` is the reference's autoregressive loop over the same decoder call.

Parameter names (flat dict, Keras layouts):
  embedding; encoder.* exactly as ForwardTransformer dense blocks (models.py docstring);
  prenet.d1.{w,b}, prenet.d2.{w,b}                                  (DecoderPrenet, layers.py:420-443)
  decoder.ln.{gamma,beta}, decoder.pos_scalar                       (CrossAttentionBlocks, layers.py:381-417)
  decoder.b{i}.sa.{wq,wk,wv,wo}.{w,b}, decoder.b{i}.sa.ln.{gamma,beta}   (SelfAttentionResNorm, layers.py:198-211)
  decoder.b{i}.ca.{wq,wk,wv,wo}.{w,b}, decoder.b{i}.ca.ln.{gamma,beta}   (CrossAttentionResnorm, layers.py:315-327)
  decoder.b{i}.ffn1.{w,b}, decoder.b{i}.ffn2.{w,b}, decoder.b{i}.ln2.{gamma,beta}  (FFNResNorm, layers.py:82-102)
  final_proj.{w,b}  (d, mel*max_r);  postnet.stop.{w,b} (mel,3);  postnet.mel.{w,b} (mel,mel)   (layers.py:446-460)
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from .. import lib
from .models import (LN_EPS, ForwardTransformer, _capture_graphs, _fill_inputs, _lru_get, _lru_make_room, _on_device, _PackedLinear,
                     _qkv_block_n, _replay, _round_up, _static_inputs)
from .transformer_utils import mask_from_lengths, positional_encoding

ALIGNER_VOCAB = 129  # 126 symbols + pad + start + end (reference: data/text/tokenizer.py:17-26 with add_start_end=True)
# predict_batch: decode steps issued between two host reads of the "all rows done" word (finished rows stay frozen, so the
# result does not depend on it; it only bounds the steps run after the last row has stopped)
_DECODE_SYNC_EVERY = 8
_DECODE_GRAPH_CACHE = 2   # captured decode steps kept per model (each holds its caches and map buffers)


class Aligner(ForwardTransformer):
    def __init__(self,
                 encoder_model_dimension: int,
                 decoder_model_dimension: int,
                 encoder_num_heads: list,
                 decoder_num_heads: list,
                 encoder_max_position_encoding: int,
                 decoder_max_position_encoding: int,
                 encoder_prenet_dimension: int,
                 decoder_prenet_dimension: int,
                 dropout_rate: float,
                 mel_start_value: float,
                 mel_end_value: float,
                 mel_channels: int,
                 phoneme_language: str = 'en-us',
                 with_stress: bool = True,
                 decoder_prenet_dropout: float = 0.1,
                 model_breathing: bool = False,
                 encoder_feed_forward_dimension: int = None,
                 decoder_feed_forward_dimension: int = None,
                 max_r: int = 10,
                 debug=False,
                 **kwargs):
        loc = dict(locals())
        self.config = {k: v for k, v in loc.items() if k not in ('self', 'kwargs', '__class__')}
        self.config.update(kwargs)
        if int(encoder_prenet_dimension) != int(encoder_model_dimension):
            raise ValueError('the embedding (encoder prenet) feeds the encoder blocks directly: dimensions must match '
                             '(reference: model/models.py:53-65)')
        # cuda_graphs / train_graphs replay the teacher-forced validation step / training step as CUDA graphs per input shape
        # (the steps are ~90 / ~430 dependent launches of small kernels: host-launch bound when issued eagerly)
        self._init_runtime(mel_channels, debug, kwargs)
        self.vocab_size = int(kwargs.get('vocab_size', ALIGNER_VOCAB))
        self.return_attention_weights = True      # attention maps are model outputs (models.py:150-153, 297)
        self._val_graphs = {}
        self._decode_graphs = {}
        self.decode_stats = None   # predict_batch: {'steps', 'host_reads'} of the last call
        self.max_r = int(max_r)
        self.r = int(max_r)                        # models.py:46 -- starts at max_r, lowered by the schedule via set_constants
        self.stop_prob_index = 2
        self.force_encoder_diagonal = False
        self.force_decoder_diagonal = False
        self.stop_scaling = float(kwargs.get('stop_loss_scaling', 8.0))
        self.start_vec = torch.full((1, self.mel_channels), float(mel_start_value))
        self.end_vec = torch.full((1, self.mel_channels), float(mel_end_value))
        self._stacks = {
            'encoder': dict(d=int(encoder_model_dimension), heads=list(encoder_num_heads), n_dense=len(encoder_num_heads),
                            ffn=encoder_feed_forward_dimension, filters=[], kernel=None, max_pos=int(encoder_max_position_encoding)),
            'decoder': dict(d=int(decoder_model_dimension), heads=list(decoder_num_heads), n_dense=len(decoder_num_heads),
                            ffn=decoder_feed_forward_dimension, filters=[], kernel=None, max_pos=int(decoder_max_position_encoding)),
        }
        self.loss_weights = [1., 1.]
        self._init_weights(seed=int(kwargs.get('seed', 42)))

    # ------------------------------------------------------------------------------------------------
    def _param_shapes(self) -> Dict[str, tuple]:
        c = self.config
        enc, dec = self._stacks['encoder'], self._stacks['decoder']
        d_enc, d_dec, mel = enc['d'], dec['d'], self.mel_channels
        sh = {'embedding': (self.vocab_size, d_enc)}

        def mha(pre, d_q, d_kv, d):
            sh[pre + 'wq.w'], sh[pre + 'wq.b'] = (d_q, d), (d,)
            sh[pre + 'wk.w'], sh[pre + 'wk.b'] = (d_kv, d), (d,)
            sh[pre + 'wv.w'], sh[pre + 'wv.b'] = (d_kv, d), (d,)
            sh[pre + 'wo.w'], sh[pre + 'wo.b'] = (d_q + d, d), (d,)

        def ln(pre, n):
            sh[pre + '.gamma'], sh[pre + '.beta'] = (n,), (n,)

        def lin(pre, fin, fout):
            sh[pre + '.w'], sh[pre + '.b'] = (fin, fout), (fout,)

        ln('encoder.ln', d_enc)
        sh['encoder.pos_scalar'] = ()
        for i, _ in enumerate(enc['heads']):
            pre = f'encoder.b{i}.'
            mha(pre, d_enc, d_enc, d_enc)
            ln(pre + 'ln1', d_enc)
            lin(pre + 'ffn1', d_enc, int(enc['ffn']))
            lin(pre + 'ffn2', int(enc['ffn']), d_enc)
            ln(pre + 'ln2', d_enc)
        lin('prenet.d1', mel, int(c['decoder_prenet_dimension']))
        lin('prenet.d2', int(c['decoder_prenet_dimension']), d_dec)
        ln('decoder.ln', d_dec)
        sh['decoder.pos_scalar'] = ()
        for i, _ in enumerate(dec['heads']):
            pre = f'decoder.b{i}.'
            mha(pre + 'sa.', d_dec, d_dec, d_dec)
            ln(pre + 'sa.ln', d_dec)
            mha(pre + 'ca.', d_dec, d_enc, d_dec)
            ln(pre + 'ca.ln', d_dec)
            lin(pre + 'ffn1', d_dec, int(dec['ffn']))
            lin(pre + 'ffn2', int(dec['ffn']), d_dec)
            ln(pre + 'ln2', d_dec)
        lin('final_proj', d_dec, mel * self.max_r)
        lin('postnet.stop', mel, 3)
        lin('postnet.mel', mel, mel)
        return sh

    # ------------------------------------------------------------------------------------------------
    def _prepare(self):
        if self._packed is not None and self._packed['precision'] == self.precision:
            return self._packed
        lib.load()
        W, sp = self.weights, self._split
        P = {'precision': self.precision}
        enc, dec = self._stacks['encoder'], self._stacks['decoder']
        d_enc, d_dec, mel = enc['d'], dec['d'], self.mel_channels
        if d_enc % 64 or d_dec % 64 or int(enc['ffn']) % 64 or int(dec['ffn']) % 64 or int(self.config['decoder_prenet_dimension']) % 64:
            raise lib.TtsbError('Aligner: model / feed-forward / prenet dimensions must be multiples of 64 (GEMM K blocks)')
        P['encoder.pe'] = self._prepare_pe('encoder')
        for i, _ in enumerate(enc['heads']):
            self._pack_attention(P, f'encoder.b{i}.', d_enc)
            self._pack_ffn(P, f'encoder.b{i}.', d_enc, int(enc['ffn']))
        # K = mel_channels (80) is padded with zero rows to one 128-wide K block pair
        self._mel_k = _round_up(mel, 64)

        def pad_rows(w):
            out = torch.zeros((self._mel_k, w.shape[1]), dtype=w.dtype, device=w.device)
            out[:w.shape[0]] = w
            return out

        P['prenet.d1'] = _PackedLinear(pad_rows(W['prenet.d1.w']), W['prenet.d1.b'], [self._mel_k], sp)
        P['prenet.d2'] = _PackedLinear(W['prenet.d2.w'], W['prenet.d2.b'], [int(self.config['decoder_prenet_dimension'])], sp)
        for i, _ in enumerate(dec['heads']):
            pre = f'decoder.b{i}.'
            self._pack_attention(P, pre + 'sa.', d_dec)
            c = pre + 'ca.'
            P[c + 'q'] = _PackedLinear(W[c + 'wq.w'], W[c + 'wq.b'], [d_dec], sp)
            P[c + 'kv'] = _PackedLinear(torch.cat([W[c + 'wk.w'], W[c + 'wv.w']], dim=1), torch.cat([W[c + 'wk.b'], W[c + 'wv.b']]),
                                        [d_enc], sp, block_n=_qkv_block_n(d_dec))
            P[c + 'wo'] = _PackedLinear(W[c + 'wo.w'], W[c + 'wo.b'], [d_dec, d_dec], sp, single_tile=True)
            self._pack_ffn(P, pre, d_dec, int(dec['ffn']))
        # Postnet: mel (80) and stop (3) heads share one GEMM over the padded linear frames
        w_post = pad_rows(torch.cat([W['postnet.mel.w'], W['postnet.stop.w']], dim=1))
        P['postnet'] = _PackedLinear(w_post, torch.cat([W['postnet.mel.b'], W['postnet.stop.b']]), [self._mel_k], sp)
        self._packed = P
        self._final_proj = {}
        self._pe_r = {}
        return P

    def _final_proj_r(self, r: int) -> _PackedLinear:
        """Dense(mel*max_r) followed by [:, :, :r*mel] (models.py:146): only the first r*mel output columns are computed."""
        if r not in self._final_proj:
            n = r * self.mel_channels
            self._final_proj[r] = _PackedLinear(self.weights['final_proj.w'][:, :n].contiguous(), self.weights['final_proj.b'][:n].contiguous(),
                                                [self._stacks['decoder']['d']], self._split)
        return self._final_proj[r]

    def _final_proj_frames_r(self, r: int) -> _PackedLinear:
        """The first r*mel columns of FinalProj with every frame padded to _mel_k columns (zero weights and bias): the GEMM
        output, viewed as (rows*r, _mel_k), is the zero-padded postnet input of the cached decode step."""
        key = ('frames', r)
        if key not in self._final_proj:
            mel, k, d = self.mel_channels, self._mel_k, self._stacks['decoder']['d']
            w = torch.zeros((d, r, k), dtype=torch.float32, device=self.device)
            b = torch.zeros((r, k), dtype=torch.float32, device=self.device)
            w[:, :, :mel] = self.weights['final_proj.w'][:, :r * mel].reshape(d, r, mel)
            b[:, :mel] = self.weights['final_proj.b'][:r * mel].reshape(r, mel)
            self._final_proj[key] = _PackedLinear(w.reshape(d, r * k), b.reshape(-1), [d], self._split)
        return self._final_proj[key]

    def _decoder_pe(self, r: int) -> torch.Tensor:
        """pos_encoding[:, :T*r:r] (layers.py:409) as a dense table so row t of the table is position t*r."""
        if not hasattr(self, '_pe_r'):
            self._pe_r = {}
        if r not in self._pe_r:
            st = self._stacks['decoder']
            self._pe_r[r] = positional_encoding(st['max_pos'], st['d'])[0][::r].to(self.device).contiguous()
        return self._pe_r[r]

    # ------------------------------------------------------------------------------------------------
    def _cadb(self, P, i: int, x, enc, enc_len, dec_len, B: int, T: int, Tp: int):
        """CrossAttentionDenseBlock (layers.py:330-349): no row masks inside the block; every query row is computed."""
        W = self.weights
        dec, d_enc = self._stacks['decoder'], self._stacks['encoder']['d']
        d, H = dec['d'], dec['heads'][i]
        dh = d // H
        pre = f'decoder.b{i}.'
        if self.attention_precision == 'bf16x3':
            raise lib.TtsbError("Aligner attention runs in the single-pass modes ('fp16' / 'bf16'): head dim 256 needs them")
        f16 = self.attention_precision == 'fp16'
        adt = torch.float16 if f16 else torch.bfloat16
        x_f, x_hi, x_lo = x
        # ---- masked (look-ahead + padding) self-attention, residual, LayerNorm
        qkv = P[pre + 'sa.qkv']
        qk = torch.empty((B, T, qkv.n_pad), dtype=adt, device=self.device)
        self._gemm(qkv, B, T, [(x_hi, x_lo, d, 0)], [0], [0], out_hi=qk, out_fp16=f16)
        (a_hi, a_lo), _ = self._mha(B, T, H, dh, qk, qkv.n_pad, (0, d, 2 * d), dec_len, causal=True, full_queries=True)
        y = self._act(B, T, d)
        self._gemm(P[pre + 'sa.wo'], B, T, [(x_hi, x_lo, d, 0), (a_hi, a_lo, d, 0)], [0, 1], [0, 0], residual=x_f,
                   ln=(W[pre + 'sa.ln.gamma'], W[pre + 'sa.ln.beta']), out_f32=y[0], out_hi=y[1], out_lo=y[2])
        # ---- cross-attention onto the encoder output (keys masked by the encoder padding mask), residual, LayerNorm
        pq, pkv = P[pre + 'ca.q'], P[pre + 'ca.kv']
        qb = torch.empty((B, T, pq.n_pad), dtype=adt, device=self.device)
        kvb = torch.empty((B, Tp, pkv.n_pad), dtype=adt, device=self.device)
        self._gemm(pq, B, T, [(y[1], y[2], d, 0)], [0], [0], out_hi=qb, out_fp16=f16)
        self._gemm(pkv, B, Tp, [(enc[1], enc[2], d_enc, 0)], [0], [0], out_hi=kvb, out_fp16=f16)
        (c_hi, c_lo), wts = self._mha(B, T, H, dh, qb, pq.n_pad, (0, 0, d), enc_len, kv=kvb, ld_kv=pkv.n_pad, Tk=Tp,
                                      full_queries=True, maps='all')
        z = self._act(B, T, d)
        self._gemm(P[pre + 'ca.wo'], B, T, [(y[1], y[2], d, 0), (c_hi, c_lo, d, 0)], [0, 1], [0, 0], residual=y[0],
                   ln=(W[pre + 'ca.ln.gamma'], W[pre + 'ca.ln.beta']), out_f32=z[0], out_hi=z[1], out_lo=z[2])
        # ---- feed-forward, residual, LayerNorm
        f1 = P[pre + 'ffn1']
        _, h_hi, h_lo = self._act(B, T, f1.n_pad, f32=False)
        self._gemm(f1, B, T, [(z[1], z[2], d, 0)], [0], [0], relu=True, out_hi=h_hi, out_lo=h_lo)
        o = self._act(B, T, d)
        self._gemm(P[pre + 'ffn2'], B, T, [(h_hi, h_lo, f1.n_pad, 0)], [0], [0], residual=z[0],
                   ln=(W[pre + 'ln2.gamma'], W[pre + 'ln2.beta']), out_f32=o[0], out_hi=o[1], out_lo=o[2])
        return o, wts

    # ------------------------------------------------------------------------------------------------
    # reference API
    # ------------------------------------------------------------------------------------------------
    def _call_encoder(self, inputs, training=False):
        """models.py:127-133 -> (encoder output triple, padding mask, attention weights, lengths)."""
        if training:
            raise lib.TtsbError('Aligner.call runs the inference path (training=False); dropout + backward live in train_step (aligner_training.AlignerTrainEngine)')
        P, W, dev = self._prepare(), self.weights, self.device
        x = torch.as_tensor(inputs).to(device=dev, dtype=torch.int32).contiguous()
        if x.dim() != 2:
            raise ValueError('input tokens must have shape (batch, length)')
        B, Tp = x.shape
        d = self._stacks['encoder']['d']
        enc_len = torch.empty((B,), dtype=torch.int32, device=dev)
        lib.phoneme_lengths(x, 0, enc_len)
        h = self._act(B, Tp, d)
        lib.embed_ln_pe_fwd(x, W['embedding'], W['encoder.ln.gamma'], W['encoder.ln.beta'], P['encoder.pe'],
                            W['encoder.pos_scalar'].reshape(1), LN_EPS, h[0], h[1], h[2])
        attn = {}
        for i in range(len(self._stacks['encoder']['heads'])):
            h = self._block(P, 'encoder', i, h, enc_len, B, Tp, attn, f'Encoder_DenseBlock{i + 1}_SelfAttention', maps='all')
        return h, mask_from_lengths(enc_len, Tp), attn, enc_len

    def _call_decoder(self, encoder_output, targets, encoder_padding_mask, training=False, enc_len=None):
        """models.py:135-154.  encoder_output: the activation triple returned by _call_encoder."""
        if training:
            raise lib.TtsbError('Aligner.call runs the inference path (training=False); dropout + backward live in train_step (aligner_training.AlignerTrainEngine)')
        P, W, dev = self._prepare(), self.weights, self.device
        tgt = torch.as_tensor(targets).to(device=dev, dtype=torch.float32).contiguous()
        B, T, mel = tgt.shape
        if mel != self.mel_channels:
            raise ValueError(f'targets must have {self.mel_channels} channels')
        r = int(self.r)
        dec = self._stacks['decoder']
        d = dec['d']
        Tp = encoder_output[0].shape[1]
        if enc_len is None:
            enc_len = (1.0 - encoder_padding_mask[:, 0, 0, :]).sum(dim=1).to(torch.int32).contiguous()
        if T * r > dec['max_pos']:
            raise ValueError('target length * r exceeds decoder_max_position_encoding')
        # value-derived mel padding mask (transformer_utils.py:29-32) as per-row lengths (batches are padded at the end)
        dec_len = torch.empty((B,), dtype=torch.int32, device=dev)
        lib.mel_lengths(tgt, 0.0, dec_len)
        # ---- DecoderPrenet (layers.py:420-443): relu Dense -> relu Dense
        k = self._mel_k
        padded = torch.zeros((B, T, k), dtype=torch.float32, device=dev)
        padded[..., :mel] = tgt
        t_hi, t_lo = lib.split_bf16(padded, self._split)
        p1 = P['prenet.d1']
        _, h_hi, h_lo = self._act(B, T, p1.n_pad, f32=False)
        self._gemm(p1, B, T, [(t_hi, t_lo, k, 0)], [0], [0], relu=True, out_hi=h_hi, out_lo=h_lo)
        pre_out = torch.empty((B, T, d), dtype=torch.float32, device=dev)
        self._gemm(P['prenet.d2'], B, T, [(h_hi, h_lo, p1.n_pad, 0)], [0], [0], relu=True, out_f32=pre_out)
        # ---- CrossAttentionBlocks prologue (layers.py:406-410): LN(inputs) + scalar * PE[:, :T*r:r]
        idx = torch.arange(T, dtype=torch.int32, device=dev)[None, :].expand(B, T).contiguous()
        x = self._act(B, T, d)
        lib.expand_ln_pe_fwd(pre_out, idx, W['decoder.ln.gamma'], W['decoder.ln.beta'], self._decoder_pe(r),
                             W['decoder.pos_scalar'].reshape(1), LN_EPS, x[0], x[1], x[2])
        attn = {}
        n = len(dec['heads'])
        for i in range(n):
            x, wts = self._cadb(P, i, x, encoder_output, enc_len, dec_len, B, T, Tp)
            key = 'Decoder_LastBlock_CrossAttention' if i == n - 1 else f'Decoder_DenseBlock{i + 1}_CrossAttention'
            attn[key] = wts
        # ---- FinalProj[:, :, :r*mel] -> (B, T*r, mel) -> Postnet (models.py:146-150)
        fp = self._final_proj_r(r)
        lin = torch.empty((B, T, r * mel), dtype=torch.float32, device=dev)
        self._gemm(fp, B, T, [(x[1], x[2], d, 0)], [0], [0], out_f32=lin, ld_out=r * mel)
        linear = lin.view(B, T * r, mel)
        lpad = torch.zeros((B, T * r, k), dtype=torch.float32, device=dev)
        lpad[..., :mel] = linear
        l_hi, l_lo = lib.split_bf16(lpad, self._split)
        pn = P['postnet']
        post = torch.empty((B, T * r, pn.n_pad), dtype=torch.float32, device=dev)
        self._gemm(pn, B, T * r, [(l_hi, l_lo, k, 0)], [0], [0], out_f32=post)
        return {'mel': post[..., :mel].contiguous(), 'stop_prob': post[..., mel:mel + 3].contiguous(),
                'decoder_attention': attn, 'decoder_output': x[0], 'linear': linear,
                'mel_mask': mask_from_lengths(dec_len, T), 'mel_lengths': dec_len}

    @_on_device
    def call(self, inputs, targets, training=False):
        """models.py:294-298."""
        enc, padding_mask, enc_attn, enc_len = self._call_encoder(inputs, training)
        out = self._call_decoder(enc, targets, padding_mask, training, enc_len=enc_len)
        out.update({'encoder_attention': enc_attn, 'text_mask': padding_mask, 'text_lengths': enc_len,
                    'encoder_output': enc[0]})
        return out

    __call__ = call

    def _forward(self, inp, output):
        return self.call(inp, output, training=False)

    @_on_device
    def _forward_encoder(self, inputs):
        enc, mask, attn, _ = self._call_encoder(inputs, training=False)
        return enc, mask, attn

    @_on_device
    def _forward_decoder(self, encoder_output, targets, encoder_padding_mask):
        return self._call_decoder(encoder_output, targets, encoder_padding_mask, training=False)

    @_on_device
    def _gta_forward(self, inp, tar, stop_prob, training=False):
        """models.py:168-210 (forward + losses).  Returns (model_out, None): there is no tape here."""
        tar = torch.as_tensor(tar).to(device=self.device, dtype=torch.float32)
        stop = torch.as_tensor(stop_prob).to(device=self.device, dtype=torch.int32)
        tar_inp, tar_real, tar_stop = tar[:, :-1], tar[:, 1:].contiguous(), stop[:, 1:].contiguous()
        mel_len = tar_inp.shape[1]
        tar_mel = tar_inp[:, 0::self.r, :].contiguous()
        out = self.call(inp, tar_mel, training=training)
        dev = self.device
        B = tar.shape[0]
        l_mel = torch.zeros((1,), dtype=torch.float32, device=dev)
        l_stop = torch.zeros((1,), dtype=torch.float32, device=dev)
        lib.mae_loss(out['mel'], B, out['mel'].shape[1], mel_len, self.mel_channels, tar_real, 1.0, l_mel, None)
        lib.scaled_ce_loss(out['stop_prob'], mel_len, 3, tar_stop, self.stop_prob_index, self.stop_scaling, l_stop)
        d_loss = torch.zeros((1,), dtype=torch.float32, device=dev)
        norm = 1.0
        if self.force_decoder_diagonal:
            for w in out['decoder_attention'].values():
                lib.diag_loss(w, out['mel_lengths'], out['text_lengths'], d_loss)
            norm += len(out['decoder_attention'])
        if self.force_encoder_diagonal:
            for w in out['encoder_attention'].values():
                lib.diag_loss(w, out['text_lengths'], out['text_lengths'], d_loss)
            norm += len(out['encoder_attention'])
        d_loss = d_loss / norm
        loss = self.loss_weights[0] * l_mel + self.loss_weights[1] * l_stop + d_loss
        out.update({'loss': loss[0], 'losses': {'mel': l_mel[0], 'stop_prob': l_stop[0], 'diag_loss': d_loss[0]}})
        return out, None

    def _val_step(self, inp, tar, stop_prob):
        if self.cuda_graphs:
            return self._val_step_graphed(inp, tar, stop_prob)
        return self._gta_forward(inp, tar, stop_prob, training=False)[0]

    @_on_device
    def _val_step_graphed(self, inp, tar, stop_prob):
        """The validation step captured once per (shapes, r, diagonal flags) and replayed; outputs are copied out of the
        graph's static buffers."""
        inp, tar, stop_prob = torch.as_tensor(inp), torch.as_tensor(tar), torch.as_tensor(stop_prob)
        self._prepare()
        key = (tuple(inp.shape), tuple(tar.shape), self.r, self.force_encoder_diagonal, self.force_decoder_diagonal, id(self._packed))
        ent = _lru_get(self._val_graphs, key)
        if ent is None:
            _lru_make_room(self._val_graphs, 4)
            ins = _static_inputs(self.device, (inp, tar, stop_prob), (torch.int32, torch.float32, torch.int32))
            [(g, (out, _))] = _capture_graphs(self, self.device, lambda: self._gta_forward(*ins), lambda: self._gta_forward(*ins))
            ent = self._val_graphs[key] = {'ins': ins, 'g': g, 'out': out}
        else:
            _fill_inputs(ent['ins'], (inp, tar, stop_prob))
        _replay(ent['g'])

        def cp(v):
            if torch.is_tensor(v):
                return v.clone()
            if isinstance(v, dict):
                return {k: cp(x) for k, x in v.items()}
            return v
        return cp(ent['out'])

    val_step = _val_step

    def _get_engine(self):
        if self._engine is None:
            from .aligner_training import AlignerTrainEngine
            self._engine = AlignerTrainEngine(self)
        return self._engine

    @_on_device
    def _train_step(self, inp, tar, stop_prob, data_parallel: bool = False):
        """models.py:212-216: teacher-forced forward (dropout on, single-pass bf16), hand-written backward, Adam.
        The returned dictionary has the losses and outputs; attention maps are not materialised in fp32 on this path."""
        if self.optimizer is None:
            self._compile(self.stop_scaling)
        eng = self._get_engine()
        sync = None
        if data_parallel:
            from ..utils.data_parallel import make_grad_sync
            sync = make_grad_sync(eng.flat_g)
        if self.train_graphs and sync is None:
            out = eng.step_graphed(inp, tar, stop_prob)
        else:
            out = eng.forward_backward(inp, tar, stop_prob, training=True, sync=sync)
        scale = sync.finish() if sync is not None else 1.0
        eng.apply_adam(self.optimizer, grad_scale=scale)
        return out

    train_step = _train_step

    def predict(self, inp, max_length=1000, encode=True, verbose=True):
        """models.py:271-292: autoregressive decoding of one token row.  As in the reference the encoder runs once and the
        decoder is re-run on the whole prefix every iteration; the prefix grows by the last predicted frame, the returned mel
        by the last r frames, and decoding stops when the arg-max of the last stop distribution is `stop_prob_index`.
        One host read per iteration (the stop decision), as `int(tf.argmax(...))` is in the reference."""
        if encode:
            inp = self.encode_text(inp)
        return self._predict_tokens(inp, max_length, verbose)

    @_on_device
    def _predict_tokens(self, inp, max_length, verbose):
        dev = self.device
        inp = torch.as_tensor(inp).to(device=dev, dtype=torch.int32).reshape(1, -1)
        output = self.start_vec.to(device=dev, dtype=torch.float32).reshape(1, 1, self.mel_channels)
        output_concat = output.clone()
        out_dict = {}
        enc, padding_mask, enc_attn, enc_len = self._call_encoder(inp, training=False)
        r = int(self.r)
        for _ in range(int(max_length // r) + 1):
            mo = self._call_decoder(enc, output, padding_mask, training=False, enc_len=enc_len)
            output = torch.cat([output, mo['mel'][:1, -1:, :]], dim=-2)
            output_concat = torch.cat([output_concat, mo['mel'][:1, -r:, :]], dim=-2)
            out_dict = {'mel': output_concat[0, 1:, :], 'decoder_attention': mo['decoder_attention'], 'encoder_attention': enc_attn}
            if int(torch.argmax(mo['stop_prob'][:, -1], dim=-1)) == self.stop_prob_index:
                if verbose:
                    print('Stopping')
                break
        return out_dict

    # ------------------------------------------------------------------------------------------------
    # cached autoregressive decoding of a batch of sentences
    # ------------------------------------------------------------------------------------------------
    def predict_batch(self, inputs, max_length=1000, verbose=False) -> List[dict]:
        """`predict` (models.py:271-292) for a batch of token rows, with a key/value cache instead of the re-run of the decoder
        over the whole prefix.  inputs: a list of 1-D token-id sequences, or a (B, Tp) array padded with 0 at the end.

        Returns one dict per row in the shape `predict` returns for that row alone: 'mel' (n_b*r, mel_channels),
        'decoder_attention' {key: (1, H, n_b, Tp_b)}, 'encoder_attention' {key: (1, H, Tp_b, Tp_b)}, plus 'stop_prob'
        (n_b*r, 3), the stop logits.  n_b is the first iteration whose last stop distribution has its arg-max at
        `stop_prob_index`, or max_length // r + 1; Tp_b is the row's token count.

        The decoder is causal and its rows do not depend on later ones, so each iteration decodes one row per sentence: the
        encoder and every block's cross-attention K|V run once, each self-attention block appends the new row's K and V to its
        cache, and the step reads its positions from device memory.  One difference from the re-run is left out on purpose:
        the reference masks a decoder key whose input frame sums to exactly 0 in every channel (transformer_utils.py:29-32);
        a predicted frame does that with probability zero, and the cached decode never masks one.  With `cuda_graphs` the
        step is captured once per (B, Tp, max_length, r, precisions) and replayed; the host reads one "all rows done" word
        every few steps."""
        r = int(self.r)
        max_iters = int(max_length) // r + 1
        if max_iters * r > self._stacks['decoder']['max_pos']:
            raise ValueError('target length * r exceeds decoder_max_position_encoding')
        return self._predict_batch(self._token_batch(inputs), max_iters, r, verbose)

    @staticmethod
    def _token_batch(inputs) -> torch.Tensor:
        if torch.is_tensor(inputs) or isinstance(inputs, np.ndarray):
            tokens = torch.as_tensor(inputs).to(torch.int32)
            if tokens.dim() != 2:
                raise ValueError('inputs must be a list of token sequences or a (batch, length) array')
        else:
            rows = [torch.as_tensor(np.asarray(row)).reshape(-1).to(torch.int32) for row in inputs]
            if not rows:
                raise ValueError('inputs is empty')
            tokens = torch.zeros((len(rows), max(len(row) for row in rows)), dtype=torch.int32)
            for b, row in enumerate(rows):
                tokens[b, :len(row)] = row
        nz = tokens.cpu() != 0
        if tokens.shape[0] == 0 or tokens.shape[1] == 0 or not bool(nz[:, 0].all()):
            raise ValueError('every row needs at least one token')
        if bool((nz[:, 1:] & ~nz[:, :-1]).any()):
            raise ValueError('pad id 0 inside a sequence: batches must be padded at the end')
        return tokens

    @_on_device
    def _predict_batch(self, tokens, max_iters: int, r: int, verbose: bool) -> List[dict]:
        P = self._prepare()
        B, Tp = tokens.shape
        enc, _, enc_attn, enc_len = self._call_encoder(tokens, training=False)
        if self.cuda_graphs and self.impl != 'simt':
            key = (B, Tp, max_iters, r, self.precision, self.attention_precision, id(P))
            ent = _lru_get(self._decode_graphs, key)
            if ent is None:
                _lru_make_room(self._decode_graphs, _DECODE_GRAPH_CACHE)
                st = self._decode_state(P, B, Tp, max_iters, r)
                self._decode_prefill(P, st, enc, enc_len)   # the capture's warm-up step runs on a valid state
                [(g, _)] = _capture_graphs(self, self.device, lambda: self._decode_step(P, st), lambda: self._decode_step(P, st))
                ent = self._decode_graphs[key] = {'st': st, 'g': g, 'P': P}
            st = ent['st']

            def step():
                _replay(ent['g'])
        else:
            st = self._decode_state(P, B, Tp, max_iters, r)

            def step():
                self._decode_step(P, st)
        self._decode_prefill(P, st, enc, enc_len)
        flag = torch.empty((1,), dtype=torch.int32, pin_memory=True)
        steps = reads = 0
        while steps < max_iters:
            for _ in range(min(_DECODE_SYNC_EVERY, max_iters - steps)):
                step()
                steps += 1
            if steps == max_iters:   # every row is done at the iteration cap
                break
            flag.copy_(st['all_done'], non_blocking=True)
            torch.cuda.current_stream().synchronize()
            reads += 1
            if int(flag[0]):
                break
        lens = torch.stack([st['n'], enc_len]).cpu()
        reads += 1
        self.decode_stats = {'steps': steps, 'host_reads': reads}
        n_dec = len(self._stacks['decoder']['heads'])
        out = []
        for b in range(B):
            nb, tb = int(lens[0, b]), int(lens[1, b])
            if verbose and nb < max_iters:
                print(f'row {b}: stopping after {nb} iterations')
            out.append({
                'mel': st['mel'][b, :nb * r].clone(),
                'stop_prob': st['stop'][b, :nb * r].clone(),
                'decoder_attention': {('Decoder_LastBlock_CrossAttention' if i == n_dec - 1 else f'Decoder_DenseBlock{i + 1}_CrossAttention'):
                                      st['maps'][i][b:b + 1, :, :nb, :tb].clone() for i in range(n_dec)},
                'encoder_attention': {k: w[b:b + 1, :, :tb, :tb].clone() for k, w in enc_attn.items()},
            })
        return out

    def _decode_state(self, P, B: int, Tp: int, max_iters: int, r: int) -> dict:
        """Device buffers of one batch decode: caches, maps and outputs for the whole call plus the step's activations."""
        if self.attention_precision == 'bf16x3':
            raise lib.TtsbError("Aligner attention runs in the single-pass modes ('fp16' / 'bf16'): head dim 256 needs them")
        dev, dec = self.device, self._stacks['decoder']
        d, mel, k = dec['d'], self.mel_channels, self._mel_k
        adt = torch.float16 if self.attention_precision == 'fp16' else torch.bfloat16
        i32 = dict(dtype=torch.int32, device=dev)
        fp = self._final_proj_frames_r(r)
        start = torch.zeros((B, k), dtype=torch.float32, device=dev)
        start[:, :mel] = self.start_vec.to(dev)
        start_hi, start_lo = lib.split_bf16(start, self._split)
        return {
            'B': B, 'Tp': Tp, 'r': r, 'max_iters': max_iters, 'fp': fp, 'pe': self._decoder_pe(r),
            'pos': torch.zeros((B,), **i32), 'done': torch.zeros((B,), **i32), 'n': torch.zeros((B,), **i32),
            'all_done': torch.zeros((1,), **i32), 'enc_len': torch.zeros((B,), **i32),
            'start': (start_hi, start_lo), 'in': (torch.empty_like(start_hi), torch.empty_like(start_lo) if start_lo is not None else None),
            # ttsb_decode_attn's workspace layout depends on the head count: one per head count of the stack (A5: 4 and 1)
            'workspace': {H: torch.zeros((lib.decode_attn_workspace_bytes(B, H, d // H),), dtype=torch.uint8, device=dev)
                          for H in set(dec['heads'])},
            'cache': [torch.empty((B, max_iters, 2 * d), dtype=adt, device=dev) for _ in dec['heads']],
            'kv': [torch.empty((B, Tp, P[f'decoder.b{i}.ca.kv'].n_pad), dtype=adt, device=dev) for i in range(len(dec['heads']))],
            'maps': [torch.empty((B, H, max_iters, Tp), dtype=torch.float32, device=dev) for H in dec['heads']],
            'mel': torch.empty((B, max_iters * r, mel), dtype=torch.float32, device=dev),
            'stop': torch.empty((B, max_iters * r, 3), dtype=torch.float32, device=dev),
            # one step's activations: rows = sentences
            'h1': self._act(1, B, P['prenet.d1'].n_pad, f32=False), 'pre': torch.empty((B, d), dtype=torch.float32, device=dev),
            'x': self._act(1, B, d), 'y': self._act(1, B, d), 'z': self._act(1, B, d), 'o': [self._act(1, B, d), self._act(1, B, d)],
            'qkv': torch.empty((B, P['decoder.b0.sa.qkv'].n_pad), dtype=adt, device=dev),
            'q': torch.empty((B, P['decoder.b0.ca.q'].n_pad), dtype=adt, device=dev),
            'att': self._act(1, B, d, f32=False), 'h': self._act(1, B, P['decoder.b0.ffn1'].n_pad, f32=False),
            'lin': self._act(1, B, fp.n_pad, f32=False),
            'post': torch.empty((B * r, P['postnet'].n_pad), dtype=torch.float32, device=dev),
        }

    def _decode_prefill(self, P, st, enc, enc_len):
        """Once per call: every block's cross-attention K|V of the encoder output, the start frame as every row's first input,
        positions and flags at zero."""
        d_enc = self._stacks['encoder']['d']
        f16 = self.attention_precision == 'fp16'
        for i, kv in enumerate(st['kv']):
            self._gemm(P[f'decoder.b{i}.ca.kv'], st['B'], st['Tp'], [(enc[1], enc[2], d_enc, 0)], [0], [0], out_hi=kv, out_fp16=f16)
        st['enc_len'].copy_(enc_len)
        for t in ('pos', 'done', 'n', 'all_done'):
            st[t].zero_()
        for dst, src in zip(st['in'], st['start']):
            if dst is not None:
                dst.copy_(src)

    def _decode_attn(self, st, H, dh, q, ld_q, kv, ld_kv, Tk, new=False, probs=None):
        """ttsb_decode_attn: self mode (`new`: K and V of the new row at columns d / 2d of q, cached at (0, d) of kv) or
        cross mode over the encoder K|V (keys < enc_len)."""
        d = H * dh
        a = lib.DecodeAttnArgs()
        a.B, a.H, a.dh = st['B'], H, dh
        a.q, a.ld_q, a.q_col0 = q.data_ptr(), ld_q, 0
        a.kv, a.ld_kv, a.Tk, a.k_col0, a.v_col0 = kv.data_ptr(), ld_kv, Tk, 0, d
        if new:
            a.new_kv, a.ld_new, a.new_k_col0, a.new_v_col0 = q.data_ptr(), ld_q, d, 2 * d
        else:
            a.kv_len = st['enc_len'].data_ptr()
        a.pos, a.done = st['pos'].data_ptr(), st['done'].data_ptr()
        _, at_hi, at_lo = st['att']
        a.out_hi = at_hi.data_ptr()
        a.out_lo = at_lo.data_ptr() if at_lo is not None else None
        a.ld_out = d
        if probs is not None:
            a.probs, a.probs_T = probs.data_ptr(), probs.shape[2]
        a.precision = lib.PREC_FP16 if self.attention_precision == 'fp16' else lib.PREC_BF16
        ws = st['workspace'][H]
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        lib.decode_attn(a)

    def _decode_step(self, P, st):
        """One iteration for every row: prenet, prologue at pos[b], the blocks with cached self-attention, FinalProj, postnet,
        commit.  Every GEMM takes the B rows as one sequence (a Dense has no time shift), so they share 128-row tiles."""
        W = self.weights
        dec = self._stacks['decoder']
        d, B, r, k = dec['d'], st['B'], st['r'], self._mel_k
        f16 = self.attention_precision == 'fp16'
        in_hi, in_lo = st['in']
        _, h_hi, h_lo = st['h1']
        self._gemm(P['prenet.d1'], 1, B, [(in_hi, in_lo, k, 0)], [0], [0], relu=True, out_hi=h_hi, out_lo=h_lo)
        self._gemm(P['prenet.d2'], 1, B, [(h_hi, h_lo, P['prenet.d1'].n_pad, 0)], [0], [0], relu=True, out_f32=st['pre'])
        x = st['x']
        lib.decode_prologue(st['pre'], st['pos'], W['decoder.ln.gamma'], W['decoder.ln.beta'], st['pe'], W['decoder.pos_scalar'].reshape(1),
                            LN_EPS, x[0], x[1], x[2])
        _, a_hi, a_lo = st['att']
        for i, H in enumerate(dec['heads']):
            pre = f'decoder.b{i}.'
            qkv = P[pre + 'sa.qkv']
            self._gemm(qkv, 1, B, [(x[1], x[2], d, 0)], [0], [0], out_hi=st['qkv'], out_fp16=f16)
            self._decode_attn(st, H, d // H, st['qkv'], qkv.n_pad, st['cache'][i], 2 * d, st['max_iters'], new=True)
            y = st['y']
            self._gemm(P[pre + 'sa.wo'], 1, B, [(x[1], x[2], d, 0), (a_hi, a_lo, d, 0)], [0, 1], [0, 0], residual=x[0],
                       ln=(W[pre + 'sa.ln.gamma'], W[pre + 'sa.ln.beta']), out_f32=y[0], out_hi=y[1], out_lo=y[2])
            pq, pkv = P[pre + 'ca.q'], P[pre + 'ca.kv']
            self._gemm(pq, 1, B, [(y[1], y[2], d, 0)], [0], [0], out_hi=st['q'], out_fp16=f16)
            self._decode_attn(st, H, d // H, st['q'], pq.n_pad, st['kv'][i], pkv.n_pad, st['Tp'], probs=st['maps'][i])
            z = st['z']
            self._gemm(P[pre + 'ca.wo'], 1, B, [(y[1], y[2], d, 0), (a_hi, a_lo, d, 0)], [0, 1], [0, 0], residual=y[0],
                       ln=(W[pre + 'ca.ln.gamma'], W[pre + 'ca.ln.beta']), out_f32=z[0], out_hi=z[1], out_lo=z[2])
            f1 = P[pre + 'ffn1']
            _, f_hi, f_lo = st['h']
            self._gemm(f1, 1, B, [(z[1], z[2], d, 0)], [0], [0], relu=True, out_hi=f_hi, out_lo=f_lo)
            o = st['o'][i % 2]
            self._gemm(P[pre + 'ffn2'], 1, B, [(f_hi, f_lo, f1.n_pad, 0)], [0], [0], residual=z[0],
                       ln=(W[pre + 'ln2.gamma'], W[pre + 'ln2.beta']), out_f32=o[0], out_hi=o[1], out_lo=o[2])
            x = o
        # FinalProj[:, :r*mel] with frames padded to k columns = the postnet's input rows (models.py:146-150)
        fp = st['fp']
        _, l_hi, l_lo = st['lin']
        self._gemm(fp, 1, B, [(x[1], x[2], d, 0)], [0], [0], out_hi=l_hi, out_lo=l_lo)
        pn = P['postnet']
        self._gemm(pn, 1, B * r, [(l_hi, l_lo, k, 0)], [0], [0], out_f32=st['post'])
        mel = self.mel_channels
        lib.decode_commit(st['post'], B, r, mel, mel, self.stop_prob_index, st['max_iters'], st['mel'], st['stop'], in_hi, in_lo,
                          st['pos'], st['done'], st['n'], st['all_done'])

    def _compile(self, stop_scaling=None, optimizer=None):
        """models.py:222-227.  stop_scaling None keeps the model's (``stop_loss_scaling`` of its config, default 8), so that
        restoring optimizer state from a checkpoint does not reset it."""
        from .training import Adam
        self.loss_weights = [1., 1.]
        if stop_scaling is not None:
            self.stop_scaling = float(stop_scaling)
        self.optimizer = optimizer if optimizer is not None else Adam(1.0e-4)

    def align(self, text, mel, mels_have_start_end_vectors: bool = False, phonemize: bool = False, encode_phonemes: bool = False,
              plot: bool = True):
        """models.py:247-269 -> (last-block cross-attention (N, heads, T, phonemes), model output of ``call``).
        text: token ids (N, Tp) or (Tp,); mel: (N, T, mel) or (T, mel) without the start vector, or with start and end vectors
        when ``mels_have_start_end_vectors`` (the end vector is then dropped, as the teacher-forced input drops it).  The
        input is prepended with the start vector, sliced [:, 0::r] and run through ``call(training=False)``.  ``plot`` is
        accepted for the reference's signature and ignored."""
        if phonemize:
            raise NotImplementedError('phonemization needs the espeak phonemizer, which is outside the built path; '
                                      'pass token ids')
        if encode_phonemes:   # phoneme string -> ids with start / end tokens (the Aligner's tokenizer)
            from ..data.text import Tokenizer
            text = Tokenizer(add_start_end=True, model_breathing=bool(self.config.get('model_breathing', False)))(text)
        text = torch.as_tensor(text).to(torch.int32)
        if text.dim() < 2:
            text = text[None]
        mel = torch.as_tensor(mel).to(device=self.device, dtype=torch.float32)
        if mel.dim() < 3:
            mel = mel[None]
        if self.r != 1:
            print('WARNING: reduction factor != 1.')
        if mels_have_start_end_vectors:
            tar_inp = mel[:, :-1]
        else:
            start = self.start_vec.to(device=self.device, dtype=torch.float32)[None].expand(mel.shape[0], 1, self.mel_channels)
            tar_inp = torch.cat([start, mel], dim=1)
        model_out = self.call(text, tar_inp[:, 0::self.r].contiguous(), training=False)
        return model_out['decoder_attention']['Decoder_LastBlock_CrossAttention'], model_out

    def _set_r(self, r):
        self.r = int(r)

    def set_constants(self, learning_rate: float = None, reduction_factor: float = None, decoder_prenet_dropout: float = None,
                      force_encoder_diagonal: bool = None, force_decoder_diagonal: bool = None):
        """models.py:300-312."""
        if learning_rate is not None and self.optimizer is not None:
            self.optimizer.lr = float(learning_rate)
        if reduction_factor is not None:
            self._set_r(reduction_factor)
        if force_encoder_diagonal is not None:
            self.force_encoder_diagonal = bool(force_encoder_diagonal)
        if force_decoder_diagonal is not None:
            self.force_decoder_diagonal = bool(force_decoder_diagonal)

    @classmethod
    def from_config(cls, config: dict, max_r: int = 10):
        """models.py:320-341."""
        keys = ('encoder_model_dimension', 'decoder_model_dimension', 'encoder_num_heads', 'decoder_num_heads',
                'encoder_max_position_encoding', 'decoder_max_position_encoding', 'encoder_prenet_dimension',
                'decoder_prenet_dimension', 'dropout_rate', 'mel_start_value', 'mel_end_value', 'mel_channels',
                'phoneme_language', 'with_stress', 'decoder_prenet_dropout', 'model_breathing',
                'encoder_feed_forward_dimension', 'decoder_feed_forward_dimension')
        kw = {k: config[k] for k in keys if k in config}
        extra = {k: config[k] for k in ('vocab_size', 'precision', 'attention_precision', 'impl', 'device', 'seed', 'stop_loss_scaling', 'train_dropout') if k in config}
        return cls(max_r=int(config.get('max_r', max_r)), debug=config.get('debug', False), **kw, **extra)
