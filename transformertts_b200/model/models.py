"""ForwardTransformer: host-side mirror of the reference's text->mel model (model/models.py:344-642) over torch CUDA
tensors, executing every layer through libttsb.so (hand-written sm_90a kernels, include/ttsb.h).

Same constructor arguments, methods and output dictionary as the reference class; tensors are torch.Tensor instead of
tf.Tensor.  There is no CPU / eager-PyTorch fallback: without the CUDA library the model raises TtsbError.

Parameter names (flat dict, Keras layouts -- Dense (in,out), Conv1D (k,in,out)):
  embedding; {encoder,decoder}.ln.{gamma,beta}; {..}.pos_scalar;
  {..}.b{i}.{wq,wk,wv,wo}.{w,b}; {..}.b{i}.ln1.{gamma,beta}; dense block: ffn1/ffn2.{w,b}; conv block: conv{j}.{w,b};
  {..}.b{i}.ln2.{gamma,beta}; {dur_pred,pitch_pred}.conv{j}.{w,b} / .ln{j}.{gamma,beta} / .out.{w,b};
  pitch_embed.{w,b}; out.{w,b}
"""
from __future__ import annotations

import math
from pathlib import Path
from typing import Dict, List, Optional

import numpy as np
import torch

from .. import lib
from .transformer_utils import mask_from_lengths, positional_encoding

def _on_device(fn):
    """Run a public method with the model's device as the current CUDA device (libttsb launches on the current device)."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *a, **k):
        with torch.cuda.device(self.device):
            return fn(self, *a, **k)
    return wrapped


LN_EPS = 1e-6  # reference: model/layers.py:27,96,207,295,508
DEFAULT_VOCAB = 127  # 126 phoneme/punctuation symbols + pad id 0 (reference: data/text/tokenizer.py:17-20)


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def _pick_block_n(N: int, need_single_tile: bool) -> int:
    n16 = _round_up(N, 16)
    if n16 <= 256:
        return n16
    if need_single_tile and N <= 384 and N % 32 == 0:
        return N  # LayerNorm GEMM run as a CTA pair, each CTA owning N/2 <= 192 columns (csrc/gemm_tc.cu, kPair)
    # wider / odd rows: several N tiles; a LayerNorm epilogue then runs as a separate row kernel
    for bn in range(256, 15, -16):
        if n16 % bn == 0:
            return bn
    return 256


class _PackedLinear:
    """One GEMM of the family in include/ttsb.h: packed bf16 weights + bias + static shape info."""

    def __init__(self, w_kn: torch.Tensor, bias: Optional[torch.Tensor], seg_k: List[int], split: bool, single_tile: bool = False,
                 block_n: Optional[int] = None):
        K, N = w_kn.reshape(-1, w_kn.shape[-1]).shape
        self._tile(K, N, seg_k, single_tile, block_n)
        self.w_hi, self.w_lo = lib.pack_weight(w_kn, self.n_pad, split)
        self.bias = None
        if bias is not None:  # the epilogue reads whole 16-column chunks: pad to n_pad
            self.bias = torch.zeros(self.n_pad, dtype=torch.float32, device=bias.device)
            self.bias[:N] = bias.float()

    @classmethod
    def empty(cls, K: int, N: int, seg_k: List[int], device, single_tile: bool = False, block_n: Optional[int] = None,
              bias: bool = True) -> '_PackedLinear':
        """Buffers allocated but not filled (the training engine refreshes them every step with one batched launch,
        lib.repack_batched)."""
        pl = cls.__new__(cls)
        pl._tile(K, N, seg_k, single_tile, block_n)
        pl.w_hi = torch.empty((pl.n_pad, K), dtype=torch.bfloat16, device=device)
        pl.w_lo = None
        pl.bias = torch.zeros(pl.n_pad, dtype=torch.float32, device=device) if bias else None
        return pl

    def _tile(self, K, N, seg_k, single_tile, block_n):
        assert sum(seg_k) == K, (seg_k, K)
        self.N, self.K, self.seg_k = N, K, seg_k
        self.block_n = block_n or _pick_block_n(N, single_tile)
        self.n_tiles = (N + self.block_n - 1) // self.block_n
        self.n_pad = self.n_tiles * self.block_n


def _qkv_block_n(d: int) -> int:
    """N tile of a projection onto q|k|v (or k|v): one head-aligned tile of width d, or two of d/2."""
    return d if d <= 256 else d // 2


# ---- CUDA graphs: per-shape caches (least recently used evicted first) whose graphs share one private memory pool
def _capture_graphs(owner, device, warmup, *stages):
    """Runs `warmup()` eagerly on a side stream (one-time function attributes, packs, allocator), then captures each stage
    as one CUDA graph in `owner._graph_pool` (created on first use).  Returns [(graph, stage output)];
    graph.ttsb_launches is the number of library kernels inside it (added to the launch count per replay)."""
    side = torch.cuda.Stream(device=device)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        warmup()
    torch.cuda.current_stream().wait_stream(side)
    if owner._graph_pool is None:
        owner._graph_pool = torch.cuda.graph_pool_handle()
    captured = []
    n0 = lib.launch_count()
    for fn in stages:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=owner._graph_pool):
            out = fn()
        n1 = lib.launch_count()
        g.ttsb_launches, n0 = n1 - n0, n1
        captured.append((g, out))
    return captured


def _replay(g):
    g.replay()
    lib.add_launch_count(g.ttsb_launches)


def _lru_get(cache: dict, key):
    """The cached entry (now the most recently used), or None."""
    ent = cache.pop(key, None)
    if ent is not None:
        cache[key] = ent
    return ent


def _lru_make_room(cache: dict, limit: int):
    while len(cache) >= limit:
        cache.pop(next(iter(cache)))


def _static_inputs(device, tensors, dtypes):
    """Device copies of a step's inputs for a graph to read; _fill_inputs refreshes them before each replay."""
    return [t.to(device=device, dtype=dt).contiguous().clone() for t, dt in zip(tensors, dtypes)]


def _fill_inputs(static, tensors):
    for dst, src in zip(static, tensors):
        dst.copy_(src, non_blocking=True)


def _pad_vec(v: torch.Tensor, n: int) -> torch.Tensor:
    if v.numel() == n:
        return v.contiguous()
    out = torch.zeros(n, dtype=v.dtype, device=v.device)
    out[:v.numel()] = v
    return out


class ForwardTransformer:
    def __init__(self,
                 encoder_model_dimension: int,
                 decoder_model_dimension: int,
                 dropout_rate: float,
                 decoder_num_heads: list,
                 encoder_num_heads: list,
                 encoder_max_position_encoding: int,
                 decoder_max_position_encoding: int,
                 encoder_dense_blocks: int,
                 decoder_dense_blocks: int,
                 duration_conv_filters: list,
                 pitch_conv_filters: list,
                 duration_kernel_size: int,
                 pitch_kernel_size: int,
                 predictors_dropout: float,
                 mel_channels: int,
                 phoneme_language: str = 'en-us',
                 with_stress: bool = True,
                 model_breathing: bool = False,
                 transposed_attn_convs: bool = True,
                 encoder_attention_conv_filters: list = None,
                 decoder_attention_conv_filters: list = None,
                 encoder_attention_conv_kernel: int = None,
                 decoder_attention_conv_kernel: int = None,
                 encoder_feed_forward_dimension: int = None,
                 decoder_feed_forward_dimension: int = None,
                 debug=False,
                 **kwargs):
        # same config bookkeeping as the reference (model/models.py:453-462): ctor args + extra yaml keys
        loc = dict(locals())
        self.config = {k: v for k, v in loc.items() if k not in ('self', 'kwargs', '__class__')}
        self.config.update(kwargs)
        if encoder_model_dimension != decoder_model_dimension:
            raise ValueError('Expand feeds the encoder output to the decoder: model dimensions must match')
        self._init_runtime(mel_channels, debug, kwargs)
        # reference tokenizer: 126 symbols + pad, one more id when model_breathing adds the breathing token (tokenizer.py:28-33)
        self.vocab_size = int(kwargs.get('vocab_size', DEFAULT_VOCAB + (1 if model_breathing else 0)))
        self.loss_weights = [1., 1., 3.]
        self._stacks = {}
        for name in ('encoder', 'decoder'):
            d = int(self.config[f'{name}_model_dimension'])
            heads = list(self.config[f'{name}_num_heads'])
            n_dense = int(self.config[f'{name}_dense_blocks'])
            self._stacks[name] = dict(
                d=d, heads=heads, n_dense=n_dense, ffn=self.config.get(f'{name}_feed_forward_dimension'),
                filters=[int(f) for f in (self.config.get(f'{name}_attention_conv_filters') or [])],
                kernel=self.config.get(f'{name}_attention_conv_kernel'),
                max_pos=int(self.config[f'{name}_max_position_encoding']))
        self._init_weights(seed=int(kwargs.get('seed', 42)))

    def _init_runtime(self, mel_channels, debug, kwargs):
        """Constructor state shared with the Aligner: device, numerics, CUDA-graph caches, optimizer and engine slots."""
        self.mel_channels = int(mel_channels)
        self.alphabet = kwargs.get('alphabet')
        self.device = torch.device(kwargs.get('device', 'cuda:0'))
        # numerics of the tensor-core products: 'bf16x3' meets the 1e-3 mel parity gate, 'bf16' is the fast mode
        self.precision = kwargs.get('precision', 'bf16x3')
        self.impl = kwargs.get('impl', 'tcgen05')
        # attention products: single-pass IEEE fp16 keeps the mel error below the 1e-3 gate (smoke() measures 4.3e-4) at a third
        # of the tensor work of bf16x3; 'bf16' / 'bf16x3' remain selectable
        self.attention_precision = kwargs.get('attention_precision', 'fp16' if self.precision == 'bf16x3' else 'bf16')
        self.return_attention_weights = bool(kwargs.get('return_attention_weights', False))
        # inference: capture the step as CUDA graphs per input shape and replay them (see call())
        self.cuda_graphs = bool(kwargs.get('cuda_graphs', False))
        self.max_cached_graphs = int(kwargs.get('max_cached_graphs', 8))
        self._enc_graphs = {}
        self._graph_pool = None
        self._len_host = None
        self.debug = debug
        self.weights: Dict[str, torch.Tensor] = {}
        self._packed = None
        self._prof = None  # bench.py: {tag: [(start_event, end_event, flops)]} for tagged GEMM launches
        self.optimizer = None
        self.train_dropout = bool(kwargs.get('train_dropout', True))  # False: deterministic training step (parity tests)
        # training: replay the step as CUDA graphs per input shape (training.TrainEngine.step_graphed)
        self.train_graphs = bool(kwargs.get('train_graphs', False))
        self._engine = None
        self._drop_seed = 0

    # ------------------------------------------------------------------------------------------------
    # parameters
    # ------------------------------------------------------------------------------------------------
    def _param_shapes(self) -> Dict[str, tuple]:
        c = self.config
        shapes = {}
        d_enc = self._stacks['encoder']['d']
        shapes['embedding'] = (self.vocab_size, d_enc)
        for name, st in self._stacks.items():
            d = st['d']
            shapes[f'{name}.ln.gamma'] = (d,)
            shapes[f'{name}.ln.beta'] = (d,)
            shapes[f'{name}.pos_scalar'] = ()
            for i, _ in enumerate(st['heads']):
                pre = f'{name}.b{i}.'
                for w in ('wq', 'wk', 'wv'):
                    shapes[pre + w + '.w'] = (d, d)
                    shapes[pre + w + '.b'] = (d,)
                shapes[pre + 'wo.w'] = (2 * d, d)
                shapes[pre + 'wo.b'] = (d,)
                shapes[pre + 'ln1.gamma'] = (d,)
                shapes[pre + 'ln1.beta'] = (d,)
                if i < st['n_dense']:
                    F = int(st['ffn'])
                    shapes[pre + 'ffn1.w'] = (d, F)
                    shapes[pre + 'ffn1.b'] = (F,)
                    shapes[pre + 'ffn2.w'] = (F, d)
                    shapes[pre + 'ffn2.b'] = (d,)
                else:
                    cin = d
                    for j, f in enumerate(st['filters']):
                        shapes[pre + f'conv{j}.w'] = (int(st['kernel']), cin, f)
                        shapes[pre + f'conv{j}.b'] = (f,)
                        cin = f
                shapes[pre + 'ln2.gamma'] = (d,)
                shapes[pre + 'ln2.beta'] = (d,)
        for name, filt, k in (('dur_pred', c['duration_conv_filters'], c['duration_kernel_size']),
                              ('pitch_pred', c['pitch_conv_filters'], c['pitch_kernel_size'])):
            cin = d_enc
            for j, f in enumerate(filt):
                shapes[f'{name}.conv{j}.w'] = (int(k), cin, int(f))
                shapes[f'{name}.conv{j}.b'] = (int(f),)
                shapes[f'{name}.ln{j}.gamma'] = (int(f),)
                shapes[f'{name}.ln{j}.beta'] = (int(f),)
                cin = int(f)
            shapes[f'{name}.out.w'] = (cin, 1)
            shapes[f'{name}.out.b'] = (1,)
        shapes['pitch_embed.w'] = (1, d_enc)
        shapes['pitch_embed.b'] = (d_enc,)
        shapes['out.w'] = (self._stacks['decoder']['d'], self.mel_channels)
        shapes['out.b'] = (self.mel_channels,)
        return shapes

    def _init_weights(self, seed: int):
        """Keras defaults the reference relies on: glorot_uniform kernels, zero biases, LayerNorm (1,0),
        Embedding uniform(-0.05, 0.05), pos_encoding_scalar 1.0 (model/layers.py:282)."""
        g = torch.Generator(device='cpu').manual_seed(seed)
        w = {}
        for name, shape in self._param_shapes().items():
            if name == 'embedding':
                t = (torch.rand(shape, generator=g) * 2 - 1) * 0.05
            elif name.endswith('.gamma') or name.endswith('pos_scalar'):
                t = torch.ones(shape)
            elif name.endswith('.beta') or name.endswith('.b'):
                t = torch.zeros(shape)
            else:  # kernels
                if len(shape) == 3:
                    fan_in, fan_out = shape[0] * shape[1], shape[0] * shape[2]
                else:
                    fan_in, fan_out = shape
                lim = math.sqrt(6.0 / (fan_in + fan_out))
                t = (torch.rand(shape, generator=g) * 2 - 1) * lim
            w[name] = t
        self.set_weights(w)

    def set_weights(self, weights: Dict[str, torch.Tensor]):
        shapes = self._param_shapes()
        missing = set(shapes) - set(weights)
        if missing:
            raise KeyError(f'missing parameters: {sorted(missing)[:5]} ...')
        for name, shape in shapes.items():
            t = torch.as_tensor(weights[name]).detach().to(torch.float32)
            if tuple(t.shape) != tuple(shape):
                raise ValueError(f'{name}: expected shape {shape}, got {tuple(t.shape)}')
            if self._engine is not None:  # parameters are views of the flat training buffer: update in place
                self.weights[name].copy_(t.to(self.device))
            else:
                self.weights[name] = t.to(self.device).contiguous()
        self._packed = None
        self._enc_graphs = {}  # captured graphs hold the old packed operands

    def get_weights(self) -> Dict[str, torch.Tensor]:
        return {k: v.detach().clone() for k, v in self.weights.items()}

    @property
    def trainable_variables(self) -> List[torch.Tensor]:
        return [self.weights[k] for k in self._param_shapes()]

    @_on_device
    def build_model_weights(self) -> None:
        """Reference builds Keras variables with a dummy call (model/models.py:597-598); here they exist already."""
        self._prepare()

    # ------------------------------------------------------------------------------------------------
    # operand preparation (packed bf16 weights, PE tables)
    # ------------------------------------------------------------------------------------------------
    @property
    def _split(self) -> bool:
        return self.precision == 'bf16x3'

    @property
    def _prec(self) -> int:
        return lib.PREC_BF16X3 if self._split else lib.PREC_BF16

    @property
    def _impl(self) -> int:
        return lib.IMPL_SIMT if self.impl == 'simt' else lib.IMPL_TCGEN05

    def _prepare(self):
        if self._packed is not None and self._packed['precision'] == self.precision:  # weights are packed per GEMM precision
            return self._packed
        lib.load()
        W = self.weights
        sp = self._split
        P = {'precision': self.precision}
        self._enc_graphs = {}  # captured graphs read the previous packed operands
        for name, st in self._stacks.items():
            d = st['d']
            P[f'{name}.pe'] = self._prepare_pe(name)
            for i, _ in enumerate(st['heads']):
                pre = f'{name}.b{i}.'
                self._pack_attention(P, pre, d)
                if i < st['n_dense']:
                    self._pack_ffn(P, pre, d, int(st['ffn']))
                else:
                    cin = d
                    nconv = len(st['filters'])
                    for j, f in enumerate(st['filters']):
                        P[pre + f'conv{j}'] = _PackedLinear(W[pre + f'conv{j}.w'], W[pre + f'conv{j}.b'],
                                                            [cin] * int(st['kernel']), sp, single_tile=(j == nconv - 1))
                        cin = f
        d_enc = self._stacks['encoder']['d']
        for name, filt, k in (('dur_pred', self.config['duration_conv_filters'], self.config['duration_kernel_size']),
                              ('pitch_pred', self.config['pitch_conv_filters'], self.config['pitch_kernel_size'])):
            cin = d_enc
            for j, f in enumerate(filt):
                pl = _PackedLinear(W[f'{name}.conv{j}.w'], W[f'{name}.conv{j}.b'], [cin] * int(k), sp, single_tile=True)
                P[f'{name}.conv{j}'] = pl
                P[f'{name}.ln{j}'] = (_pad_vec(W[f'{name}.ln{j}.gamma'], pl.n_pad), _pad_vec(W[f'{name}.ln{j}.beta'], pl.n_pad))
                cin = int(f)
        P['out'] = _PackedLinear(W['out.w'], W['out.b'], [self._stacks['decoder']['d']], sp)
        P['pitch_embed.w'] = W['pitch_embed.w'].reshape(-1).contiguous()
        self._packed = P
        return P

    def _pack_attention(self, P, pre: str, d: int):
        """Self-attention sub-block: q|k|v as one GEMM, output projection on concat([x, attn])."""
        W, sp = self.weights, self._split
        wqkv = torch.cat([W[pre + 'wq.w'], W[pre + 'wk.w'], W[pre + 'wv.w']], dim=1)
        bqkv = torch.cat([W[pre + 'wq.b'], W[pre + 'wk.b'], W[pre + 'wv.b']])
        P[pre + 'qkv'] = _PackedLinear(wqkv, bqkv, [d], sp, block_n=_qkv_block_n(d))
        P[pre + 'wo'] = _PackedLinear(W[pre + 'wo.w'], W[pre + 'wo.b'], [d, d], sp, single_tile=True)

    def _pack_ffn(self, P, pre: str, d: int, F: int):
        W, sp = self.weights, self._split
        P[pre + 'ffn1'] = _PackedLinear(W[pre + 'ffn1.w'], W[pre + 'ffn1.b'], [d], sp)
        P[pre + 'ffn2'] = _PackedLinear(W[pre + 'ffn2.w'], W[pre + 'ffn2.b'], [F], sp, single_tile=True)

    def _prepare_pe(self, name: str) -> torch.Tensor:
        st = self._stacks[name]
        key = f'_pe_{name}'
        if not hasattr(self, key):
            setattr(self, key, positional_encoding(st['max_pos'], st['d'])[0].to(self.device).contiguous())
        return getattr(self, key)

    # ------------------------------------------------------------------------------------------------
    # kernels
    # ------------------------------------------------------------------------------------------------
    def _act(self, B, T, C, f32=True):
        """Allocate an activation triple (fp32, bf16 hi, bf16 lo)."""
        dev = self.device
        f = torch.empty((B, T, C), dtype=torch.float32, device=dev) if f32 else None
        hi = torch.empty((B, T, C), dtype=torch.bfloat16, device=dev)
        lo = torch.empty((B, T, C), dtype=torch.bfloat16, device=dev) if self._split else None
        return f, hi, lo

    def _gemm(self, pl: _PackedLinear, B, T, srcs, seg_src, seg_shift, relu=False, residual=None, ln=None, row_len=None,
              out_f32=None, out_hi=None, out_lo=None, ld_out=None, tag=None, out_fp16=False, out_preln=None,
              dropout=None, dropout_post=None, residual_pair=None):
        prof = self._prof
        if prof is not None and tag is not None:
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
        a = lib.GemmArgs()
        a.B, a.T, a.N, a.block_n = B, T, pl.N, pl.block_n
        a.num_segments = len(pl.seg_k)
        for s, k in enumerate(pl.seg_k):
            a.seg_src[s] = seg_src[s]
            a.seg_shift[s] = seg_shift[s]
            a.seg_k[s] = k
        for i, (hi, lo, ld, col0) in enumerate(srcs):
            a.a_hi[i] = hi.data_ptr()
            a.a_lo[i] = lo.data_ptr() if lo is not None else None
            a.lda[i] = ld
            a.a_col0[i] = col0
        a.w_hi = pl.w_hi.data_ptr()
        a.w_lo = pl.w_lo.data_ptr() if pl.w_lo is not None else None
        a.bias = pl.bias.data_ptr() if pl.bias is not None else None
        a.relu = int(relu)
        if residual is not None:
            a.residual = residual.data_ptr()
            a.ld_res = residual.shape[-1]
        elif residual_pair is not None:   # the bf16 hi/lo activation pair is the residual stream (bf16x3 inference)
            a.residual_hi = residual_pair[0].data_ptr()
            a.residual_lo = residual_pair[1].data_ptr()
            a.ld_res = residual_pair[0].shape[-1]
        unfused_ln = None
        if ln is not None and pl.n_tiles > 1:
            # the row does not fit one accumulator tile: GEMM writes the pre-norm value, LayerNorm runs as a row kernel
            if dropout_post is not None and dropout_post[0] > 0:
                raise lib.TtsbError('post-LayerNorm dropout needs the fused epilogue (N <= 256)')
            unfused_ln = (ln, row_len, out_f32, out_hi, out_lo)
            if out_preln is None:
                out_preln = torch.empty((B, T, pl.n_pad), dtype=torch.float32, device=self.device)
            out_f32, out_hi, out_lo, row_len, ln = out_preln, None, None, None, None
            a.out_f32 = out_f32.data_ptr()
            a.out_hi = None
            a.out_lo = None
            a.row_len = None
            out_preln = None
        if ln is not None:
            ln = (_pad_vec(ln[0], pl.n_pad), _pad_vec(ln[1], pl.n_pad))
            a.ln_gamma = ln[0].data_ptr()
            a.ln_beta = ln[1].data_ptr()
            a.ln_eps = LN_EPS
        a.row_len = row_len.data_ptr() if row_len is not None else None
        a.out_f32 = out_f32.data_ptr() if out_f32 is not None else None
        a.out_hi = out_hi.data_ptr() if out_hi is not None else None
        a.out_lo = out_lo.data_ptr() if out_lo is not None else None
        a.ld_out = ld_out if ld_out is not None else pl.n_pad
        a.out_fp16 = int(out_fp16)
        a.out_preln = out_preln.data_ptr() if out_preln is not None else None
        if dropout is not None and dropout[0] > 0:
            a.drop_pre_p, a.drop_pre_site = dropout[0], dropout[1]
        if dropout_post is not None and dropout_post[0] > 0:
            a.drop_post_p, a.drop_post_site = dropout_post[0], dropout_post[1]
        a.drop_seed = self._drop_seed
        a.precision = self._prec
        a.impl = self._impl
        lib.linear_fwd(a)
        if unfused_ln is not None:
            (g_, b_), rl, of, oh, ol = unfused_ln
            lib.layernorm_fwd(out_f32, g_, b_, pl.N, LN_EPS, rl, of, oh, ol if self._split else None)
        if prof is not None and tag is not None:
            e1.record()
            prof.setdefault(tag, []).append((e0, e1, 2.0 * B * T * pl.K * pl.N))

    def _pair_stream(self, name: str) -> bool:
        """bf16x3 + tensor-core kernels + LayerNorm fused in the GEMM epilogue (row fits one accumulator tile or a CTA pair): the hi/lo
        pair is the residual stream and no fp32 activation plane is kept between blocks."""
        d = self._stacks[name]['d']
        return self._split and self.impl != 'simt' and _pick_block_n(d, True) >= d

    def _conv_shifts(self, k: int) -> List[int]:
        return [j - (k - 1) // 2 for j in range(k)]

    def _mha(self, B, T, H, dh, qk, ld_qk, cols, lens, qk_lo=None, kv=None, ld_kv=0, Tk=None, causal=False,
             full_queries=False, maps=None):
        """Fused attention (include/ttsb.h: ttsb_mha_fwd).  qk holds Q at column cols[0] and, without a separate `kv` buffer,
        K / V at cols[1] / cols[2]; with `kv` (Tk rows, leading dimension ld_kv) K and V are read from there.  maps: None,
        'first' (the probabilities of batch row 0) or 'all' (every row) -> returned fp32 (B or 1, H, T, Tk)."""
        d = H * dh
        _, at_hi, at_lo = self._act(B, T, d, f32=False)
        m = lib.MhaArgs()
        m.B, m.T, m.H, m.dh = B, T, H, dh
        m.qk_hi = qk.data_ptr()
        m.qk_lo = qk_lo.data_ptr() if qk_lo is not None else None
        m.ld_qk, (m.q_col0, m.k_col0, m.v_col0) = ld_qk, cols
        if kv is not None:
            m.kv_hi = kv.data_ptr()
            m.ld_kv, m.Tk = ld_kv, Tk
        m.kv_len = lens.data_ptr()
        m.out_hi = at_hi.data_ptr()
        m.out_lo = at_lo.data_ptr() if at_lo is not None else None
        m.ld_out = d
        m.causal, m.full_queries = int(causal), int(full_queries)
        wts = None
        if maps is not None:
            wts = torch.empty((B if maps == 'all' else 1, H, T, Tk or T), dtype=torch.float32, device=self.device)
            m.weights_out = wts.data_ptr()
            m.weights_batch_index = 0
            m.weights_all = int(maps == 'all')
        m.precision = {'fp16': lib.PREC_FP16, 'bf16': lib.PREC_BF16, 'bf16x3': lib.PREC_BF16X3}[self.attention_precision]
        m.impl = self._impl
        lib.mha_fwd(m)
        return (at_hi, at_lo), wts

    def _block(self, P, name: str, i: int, x, lens, B: int, T: int, attn_out: Optional[dict], key: str, need_f32: bool = True,
               maps: str = 'first'):
        """One SelfAttentionDenseBlock / SelfAttentionConvBlock (reference: model/layers.py:214-264).  With
        `return_attention_weights` the probabilities (`maps` rows, see _mha) are stored in attn_out[key].

        In bf16x3 mode the hi/lo pair of an activation carries 16 mantissa bits and serves as the residual stream itself:
        the LayerNorm GEMMs then write no fp32 copy (x[0] / the returned z[0] are None unless `need_f32`) -- 4 instead of
        8 bytes stored per element by the epilogue that bounds those GEMMs."""
        st = self._stacks[name]
        d, H = st['d'], st['heads'][i]
        dh = d // H
        pre = f'{name}.b{i}.'
        W = self.weights
        x_f, x_hi, x_lo = x
        dev = self.device
        # --- q,k,v projections: one GEMM into one (B,T,3d) buffer (the attention kernel reads V MN-major from it)
        qkv = P[pre + 'qkv']
        ap = self.attention_precision
        att_split = ap == 'bf16x3'
        if att_split and not self._split:
            raise lib.TtsbError("attention_precision='bf16x3' needs precision='bf16x3'")
        qk_hi = torch.empty((B, T, qkv.n_pad), dtype=torch.float16 if ap == 'fp16' else torch.bfloat16, device=dev)
        qk_lo = torch.empty_like(qk_hi) if att_split else None
        self._gemm(qkv, B, T, [(x_hi, x_lo, d, 0)], [0], [0], out_hi=qk_hi, out_lo=qk_lo, out_fp16=(ap == 'fp16'))
        # --- fused attention
        (at_hi, at_lo), wts = self._mha(B, T, H, dh, qk_hi, qkv.n_pad, (0, d, 2 * d), lens, qk_lo=qk_lo,
                                        maps=maps if attn_out is not None and self.return_attention_weights else None)
        if attn_out is not None:
            attn_out[key] = wts
        # --- output projection on concat([x, attn]) + residual + LayerNorm + row mask
        pair_stream = self._pair_stream(name)
        y = self._act(B, T, d, f32=not pair_stream)

        def res(t):  # residual operand of a LayerNorm GEMM: fp32 plane if it exists, else the hi/lo pair
            return dict(residual=t[0]) if t[0] is not None else dict(residual_pair=(t[1], t[2]))

        self._gemm(P[pre + 'wo'], B, T, [(x_hi, x_lo, d, 0), (at_hi, at_lo, d, 0)], [0, 1], [0, 0], **res(x),
                   ln=(W[pre + 'ln1.gamma'], W[pre + 'ln1.beta']), row_len=lens, out_f32=y[0], out_hi=y[1], out_lo=y[2])
        z = self._act(B, T, d, f32=need_f32 or not pair_stream)
        if i < st['n_dense']:
            F = int(st['ffn'])
            _, h_hi, h_lo = self._act(B, T, P[pre + 'ffn1'].n_pad, f32=False)
            self._gemm(P[pre + 'ffn1'], B, T, [(y[1], y[2], d, 0)], [0], [0], relu=True, out_hi=h_hi, out_lo=h_lo)
            self._gemm(P[pre + 'ffn2'], B, T, [(h_hi, h_lo, P[pre + 'ffn1'].n_pad, 0)], [0], [0], **res(y),
                       ln=(W[pre + 'ln2.gamma'], W[pre + 'ln2.beta']), row_len=lens, out_f32=z[0], out_hi=z[1], out_lo=z[2])
        else:
            k = int(st['kernel'])
            shifts = self._conv_shifts(k)
            h_hi, h_lo, ld = y[1], y[2], d
            n = len(st['filters'])
            for j in range(n - 1):
                pl = P[pre + f'conv{j}']
                _, o_hi, o_lo = self._act(B, T, pl.n_pad, f32=False)
                self._gemm(pl, B, T, [(h_hi, h_lo, ld, 0)], [0] * k, shifts, relu=True, out_hi=o_hi, out_lo=o_lo,
                           tag=f'{name}.conv{j}')
                h_hi, h_lo, ld = o_hi, o_lo, pl.n_pad
            self._gemm(P[pre + f'conv{n - 1}'], B, T, [(h_hi, h_lo, ld, 0)], [0] * k, shifts, **res(y),
                       ln=(W[pre + 'ln2.gamma'], W[pre + 'ln2.beta']), row_len=lens, out_f32=z[0], out_hi=z[1], out_lo=z[2],
                       tag=f'{name}.conv{n - 1}')
        return z

    def _stat_predictor(self, P, name: str, x, lens, B: int, T: int, relu_head: bool):
        """StatPredictor (reference: model/layers.py:463-524).  The input is already zero at padded rows."""
        W = self.weights
        filt = self.config['duration_conv_filters' if name == 'dur_pred' else 'pitch_conv_filters']
        k = int(self.config['duration_kernel_size' if name == 'dur_pred' else 'pitch_kernel_size'])
        shifts = self._conv_shifts(k)
        _, h_hi, h_lo = x
        ld = x[1].shape[-1]
        h_f = None
        for j, f in enumerate(filt):
            pl = P[f'{name}.conv{j}']
            h_f, o_hi, o_lo = self._act(B, T, pl.n_pad)
            self._gemm(pl, B, T, [(h_hi, h_lo, ld, 0)], [0] * k, shifts, relu=True,
                       ln=P[f'{name}.ln{j}'], out_f32=h_f, out_hi=o_hi, out_lo=o_lo)
            h_hi, h_lo, ld = o_hi, o_lo, pl.n_pad
        out = torch.empty((B, T), dtype=torch.float32, device=self.device)
        lib.statpred_head_fwd(h_f, int(filt[-1]), W[f'{name}.out.w'].reshape(-1).contiguous(), W[f'{name}.out.b'], relu_head, lens, out)
        return out

    # ------------------------------------------------------------------------------------------------
    # reference API
    # ------------------------------------------------------------------------------------------------
    # ---- the two halves of call(): everything up to the integer durations, and the length regulator + decoder.  The
    # output length Tm = max_b sum_i durations[b,i] is data dependent (as in the reference), so the host reads the row
    # totals once between the two (one device->host copy + sync per call; it also carries the negative-duration flag).
    def _stage_encoder(self, P, x, tgt_dur, tgt_pitch, scalar: float, mx, mn):
        W = self.weights
        dev = self.device
        B, Tp = x.shape
        d = self._stacks['encoder']['d']
        enc_len = torch.empty((B,), dtype=torch.int32, device=dev)
        lib.phoneme_lengths(x, 0, enc_len)
        pair_stream = self._pair_stream('encoder')
        h = self._act(B, Tp, d, f32=not pair_stream)
        lib.embed_ln_pe_fwd(x, W['embedding'], W['encoder.ln.gamma'], W['encoder.ln.beta'], P['encoder.pe'],
                            W['encoder.pos_scalar'].reshape(1), LN_EPS, h[0], h[1], h[2])
        enc_attn = {}
        n_enc = len(self._stacks['encoder']['heads'])
        for i in range(n_enc):   # the pitch embedding below reads the fp32 plane of the last block
            h = self._block(P, 'encoder', i, h, enc_len, B, Tp, enc_attn, self._attn_key('encoder', i), need_f32=(i == n_enc - 1))
        durations = self._stat_predictor(P, 'dur_pred', h, enc_len, B, Tp, relu_head=True)
        pitch = self._stat_predictor(P, 'pitch_pred', h, enc_len, B, Tp, relu_head=False)
        src_pitch = tgt_pitch if tgt_pitch is not None else pitch
        h_pe = torch.empty((B, Tp, d), dtype=torch.float32, device=dev)
        lib.pitch_embed_add_fwd(h[0], src_pitch, P['pitch_embed.w'], W['pitch_embed.b'], h_pe)
        use_dur = tgt_dur if tgt_dur is not None else durations
        dur_int = torch.empty((B, Tp), dtype=torch.int32, device=dev)
        dec_len = torch.empty((B,), dtype=torch.int32, device=dev)
        lib.durations_to_int(use_dur, scalar, mx, mn, dur_int, dec_len)
        return {'h_pe': h_pe, 'durations': durations, 'pitch': pitch, 'dur_int': dur_int, 'dec_len': dec_len,
                'encoder_attention': enc_attn}

    def _stage_decoder(self, P, st, B: int, Tm: int):
        W = self.weights
        dev = self.device
        dd = self._stacks['decoder']['d']
        dec_attn = {}
        idx = torch.empty((B, Tm), dtype=torch.int32, device=dev)
        lib.expand_indices(st['dur_int'], Tm, idx)
        m = self._act(B, Tm, dd, f32=not self._pair_stream('decoder'))
        lib.expand_ln_pe_fwd(st['h_pe'], idx, W['decoder.ln.gamma'], W['decoder.ln.beta'], P['decoder.pe'],
                             W['decoder.pos_scalar'].reshape(1), LN_EPS, m[0], m[1], m[2])
        for i in range(len(self._stacks['decoder']['heads'])):
            m = self._block(P, 'decoder', i, m, st['dec_len'], B, Tm, dec_attn, self._attn_key('decoder', i), need_f32=False)
        mel = torch.empty((B, Tm, self.mel_channels), dtype=torch.float32, device=dev)
        self._gemm(P['out'], B, Tm, [(m[1], m[2], dd, 0)], [0], [0], out_f32=mel, ld_out=self.mel_channels)
        return mel, dec_attn

    def _read_lengths(self, dec_len: torch.Tensor) -> int:
        """Row totals -> host (pinned, one sync): returns Tm; raises on a negative duration (flagged as length -1)."""
        B = dec_len.shape[0]
        if self._len_host is None or self._len_host.numel() < B:
            self._len_host = torch.empty((max(B, 64),), dtype=torch.int32).pin_memory()
        hb = self._len_host[:B]
        hb.copy_(dec_len, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        if int(hb.min()) < 0:
            raise ValueError('negative duration')
        return int(hb.max())

    @_on_device
    def call(self, x, target_durations=None, target_pitch=None, training=False, durations_scalar=1.,
             max_durations_mask=None, min_durations_mask=None):
        """reference: model/models.py:518-550.  x int (B,Tp) with trailing pad id 0; targets (B,Tp,1) or (B,Tp).

        With ``cuda_graphs=True`` (constructor keyword) the two halves are captured once per input shape as CUDA graphs
        and replayed: ~85 dependent launches become two graph launches (the step is otherwise partly host-launch bound)."""
        if training:
            raise lib.TtsbError('training=True goes through train_step (dropout + backward); call() is inference-only')
        P = self._prepare()
        dev = self.device
        x = torch.as_tensor(x)
        if x.dim() != 2:
            raise ValueError('input tokens must have shape (batch, length)')
        B, Tp = x.shape

        def prep(t, dtype):
            return None if t is None else torch.as_tensor(t).reshape(B, Tp)

        tgt_dur, tgt_pitch = prep(target_durations, torch.float32), prep(target_pitch, torch.float32)
        mx, mn = prep(max_durations_mask, torch.float32), prep(min_durations_mask, torch.float32)
        scalar = 1.0 if tgt_dur is not None else float(durations_scalar)
        use_graphs = self.cuda_graphs and not self.return_attention_weights and self._prof is None and self.impl != 'simt'
        if use_graphs:
            return self._call_graphed(P, x, tgt_dur, tgt_pitch, scalar, mx, mn)

        def dev_t(t, dtype):
            return None if t is None else t.to(device=dev, dtype=dtype).contiguous()

        st = self._stage_encoder(P, dev_t(x, torch.int32), dev_t(tgt_dur, torch.float32), dev_t(tgt_pitch, torch.float32), scalar,
                                 dev_t(mx, torch.float32), dev_t(mn, torch.float32))
        Tm = self._read_lengths(st['dec_len'])
        if Tm == 0:
            mel, dec_attn = torch.zeros((B, 0, self.mel_channels), dtype=torch.float32, device=dev), {}
        else:
            mel, dec_attn = self._stage_decoder(P, st, B, Tm)
        return self._outputs(st, mel, dec_attn, Tm)

    def _outputs(self, st, mel, dec_attn, Tm, clone: bool = False):
        c = (lambda t: t.clone()) if clone else (lambda t: t)
        dec_len = c(st['dec_len'])
        return {'mel': c(mel),
                'duration': c(st['durations'])[..., None],
                'pitch': c(st['pitch'])[..., None],
                'expanded_mask': mask_from_lengths(dec_len, Tm),
                'encoder_attention': st['encoder_attention'],
                'decoder_attention': dec_attn,
                'int_durations': c(st['dur_int']),
                'mel_lengths': dec_len}

    # ---- CUDA-graph replay of the two halves (static input / output buffers live in one private memory pool)
    def _capture(self, fn):
        [(g, out)] = _capture_graphs(self, self.device, fn, fn)
        return g, out

    def _call_graphed(self, P, x, tgt_dur, tgt_pitch, scalar, mx, mn):
        dev = self.device
        B, Tp = x.shape
        key = (B, Tp, tgt_dur is not None, tgt_pitch is not None, mx is not None, mn is not None, scalar, self.precision,
               self.attention_precision, id(P))
        ent = _lru_get(self._enc_graphs, key)
        if ent is None:
            _lru_make_room(self._enc_graphs, self.max_cached_graphs)
            f32 = lambda t: None if t is None else torch.empty((B, Tp), dtype=torch.float32, device=dev)  # noqa: E731
            ins = {'x': torch.empty((B, Tp), dtype=torch.int32, device=dev), 'dur': f32(tgt_dur), 'pitch': f32(tgt_pitch),
                   'mx': f32(mx), 'mn': f32(mn)}
            self._fill(ins, x, tgt_dur, tgt_pitch, mx, mn)
            g, st = self._capture(lambda: self._stage_encoder(P, ins['x'], ins['dur'], ins['pitch'], scalar, ins['mx'], ins['mn']))
            ent = {'ins': ins, 'graph': g, 'st': st, 'dec': {}}
            self._enc_graphs[key] = ent
        else:
            self._fill(ent['ins'], x, tgt_dur, tgt_pitch, mx, mn)
        _replay(ent['graph'])
        st = ent['st']
        Tm = self._read_lengths(st['dec_len'])
        if Tm == 0:
            return self._outputs(st, torch.zeros((B, 0, self.mel_channels), dtype=torch.float32, device=dev), {}, 0, clone=True)
        dec = _lru_get(ent['dec'], Tm)
        if dec is None:
            _lru_make_room(ent['dec'], self.max_cached_graphs)
            g, (mel, dec_attn) = self._capture(lambda: self._stage_decoder(P, st, B, Tm))
            dec = {'graph': g, 'mel': mel}
            ent['dec'][Tm] = dec
        _replay(dec['graph'])
        # outputs are copied out of the graph's static buffers (20 MB of mel at C2), so a result stays valid
        # across later calls exactly as in eager mode
        return self._outputs(st, dec['mel'], {}, Tm, clone=True)

    @staticmethod
    def _fill(ins, x, tgt_dur, tgt_pitch, mx, mn):
        for dst, src in ((ins['x'], x), (ins['dur'], tgt_dur), (ins['pitch'], tgt_pitch), (ins['mx'], mx), (ins['mn'], mn)):
            if dst is not None:
                dst.copy_(src, non_blocking=True)

    __call__ = call

    def _attn_key(self, name: str, i: int) -> str:
        n_dense = self._stacks[name]['n_dense']
        cname = name.capitalize()
        if i < n_dense:
            return f'{cname}_DenseBlock{i + 1}_SelfAttention'
        return f'{cname}_ConvBlock{i - n_dense + 1}_SelfAttention'

    def forward(self, input_sequence, durations_scalar):
        """reference: model/models.py:509-512."""
        return self.call(input_sequence, target_durations=None, target_pitch=None, training=False,
                         durations_scalar=durations_scalar, max_durations_mask=None, min_durations_mask=None)

    def encode_text(self, text):
        tp = getattr(self, 'text_pipeline', None)
        if tp is None:
            raise NotImplementedError('text encoding needs the espeak phonemizer, which is outside the built path; '
                                      'pass token ids with encode=False or attach a text_pipeline')
        return tp(text)

    def _duration_mask(self, encoded: np.ndarray, table: Optional[dict], default: float) -> torch.Tensor:
        """reference: model/models.py:579-595 (per-phoneme max / min duration)."""
        mask = np.full(encoded.shape, default, dtype=np.float32)
        if table is not None:
            tok = self.text_pipeline.tokenizer
            for sym, val in table.items():
                mask[encoded == tok(sym)[0]] = val
        return torch.from_numpy(mask)

    def predict(self, inp, encode=True, speed_regulator=1., phoneme_max_duration=None, phoneme_min_duration=None,
                max_durations_mask=None, min_durations_mask=None, phoneme_durations=None, phoneme_pitch=None):
        """reference: model/models.py:559-577 (passed max/min masks are overwritten by the per-phoneme ones, as there)."""
        if encode:
            inp = self.encode_text(inp)
        inp = torch.as_tensor(np.asarray(inp) if not torch.is_tensor(inp) else inp)
        if inp.dim() < 2:
            inp = inp[None]
        inp = inp.to(torch.int32)
        host = inp.cpu().numpy()
        nz = host != 0
        if (nz[:, 1:] & ~nz[:, :-1]).any():
            raise ValueError('pad id 0 inside a sequence: batches must be padded at the end')
        duration_scalar = float(np.float32(1. / speed_regulator))
        max_mask = self._duration_mask(host, phoneme_max_duration, float('inf'))
        min_mask = self._duration_mask(host, phoneme_min_duration, 0.0)
        out = self.call(inp, target_durations=phoneme_durations, target_pitch=phoneme_pitch, training=False,
                        durations_scalar=duration_scalar, max_durations_mask=max_mask, min_durations_mask=min_mask)
        out['mel'] = out['mel'].squeeze()
        return out

    # ------------------------------------------------------------------------------------------------
    # persistence (reference: model/models.py:600-638 -- config.yaml + weights file in one directory)
    # ------------------------------------------------------------------------------------------------
    def save_model(self, path: str, with_optimizer: bool = True):
        """reference: model/models.py:600-619 (config.yaml with `step` + weights in one directory).  Besides the weights
        the optimizer state is written (Adam moments, iterations, learning rate, dropout seed base), which is what the
        reference's tf.train.Checkpoint(step, optimizer, net) holds (train_tts.py:121-131): a directory written here is
        enough to resume training bit-for-bit."""
        import yaml
        path = Path(path)
        path.mkdir(parents=True, exist_ok=True)
        cfg = {k: v for k, v in self.config.items() if k != 'device'}
        if self.alphabet is not None:
            cfg['alphabet'] = self.alphabet
        cfg['step'] = self.step
        with open(path / 'config.yaml', 'w') as f:
            yaml.safe_dump(cfg, f)
        torch.save({k: v.detach().cpu() for k, v in self.weights.items()}, path / 'model_weights.pt')
        from .hdf5_weights import save_keras_hdf5
        save_keras_hdf5(self, path / 'model_weights.hdf5')
        if with_optimizer and self.optimizer is not None:
            torch.save(self.optimizer_state(), path / 'optimizer.pt')

    def optimizer_state(self) -> dict:
        """Adam state keyed by parameter name (independent of the flat-buffer layout)."""
        opt = self.optimizer
        state = {'iterations': int(opt.iterations), 'lr': float(opt.lr), 'beta_1': opt.beta_1, 'beta_2': opt.beta_2,
                 'epsilon': opt.epsilon, 'm': {}, 'v': {}}
        if self._engine is not None:
            state['base_seed'] = int(self._engine.base_seed)
        if opt.m is not None:
            eng = self._get_engine()
            for name in eng.names:
                off, _ = eng.offsets[name]
                n = self.weights[name].numel()
                state['m'][name] = opt.m[off:off + n].view(self.weights[name].shape).detach().cpu().clone()
                state['v'][name] = opt.v[off:off + n].view(self.weights[name].shape).detach().cpu().clone()
        return state

    def load_optimizer_state(self, state: dict):
        from .training import Adam
        if self.optimizer is None:
            self._compile(optimizer=Adam(state['lr'], beta_1=state['beta_1'], beta_2=state['beta_2'], epsilon=state['epsilon']))
        opt = self.optimizer
        opt.lr, opt.iterations = float(state['lr']), int(state['iterations'])
        opt.beta_1, opt.beta_2, opt.epsilon = state['beta_1'], state['beta_2'], state['epsilon']
        eng = self._get_engine()
        if 'base_seed' in state:
            eng.base_seed = int(state['base_seed'])
        if state['m']:
            opt.m = torch.zeros_like(eng.flat_w)
            opt.v = torch.zeros_like(eng.flat_w)
            for name in eng.names:
                off, _ = eng.offsets[name]
                n = self.weights[name].numel()
                opt.m[off:off + n].copy_(state['m'][name].reshape(-1))
                opt.v[off:off + n].copy_(state['v'][name].reshape(-1))

    @classmethod
    def load_model(cls, path, **overrides):
        """reference: model/models.py:621-638.  ``overrides`` (e.g. device=..., precision=...) update the stored config.
        Weights come from model_weights.pt, or from a Keras model_weights.hdf5 written by the reference; when the
        directory holds optimizer.pt (see save_model) the optimizer state and `step` are restored as well."""
        import yaml
        path = Path(path)
        with open(path / 'config.yaml', 'r') as f:
            config = yaml.safe_load(f)
        config.pop('step', None)
        config.update(overrides)
        model = cls.from_config(config)
        if (path / 'model_weights.pt').exists():
            model.set_weights(torch.load(path / 'model_weights.pt', map_location='cpu'))
        else:
            from .hdf5_weights import load_keras_hdf5
            model.set_weights(load_keras_hdf5(model, path / 'model_weights.hdf5'))
        if (path / 'optimizer.pt').exists():
            model.load_optimizer_state(torch.load(path / 'optimizer.pt', map_location='cpu'))
        return model

    @classmethod
    def from_config(cls, config: dict, custom_objects=None):
        return cls(**config)

    # ------------------------------------------------------------------------------------------------
    # training (reference: model/models.py:464-507)
    # ------------------------------------------------------------------------------------------------
    def _compile(self, optimizer=None, learning_rate: float = 1.0e-4):
        """reference: model/models.py:484-490 + utils/training_config_manager.py:102-106 (Adam b1 .9, b2 .98, eps 1e-9)."""
        from .training import Adam
        self.loss_weights = [1., 1., 3.]
        self.optimizer = optimizer if optimizer is not None else Adam(learning_rate)

    def _get_engine(self):
        if self._engine is None:
            from .training import TrainEngine
            self._engine = TrainEngine(self)
        return self._engine

    @_on_device
    def train_step(self, input_sequence, target_sequence, target_durations, target_pitch, data_parallel: bool = False):
        """reference: model/models.py:464-482.  data_parallel=True: this process holds one shard of the batch; gradients
        are summed over the default torch.distributed group (bucketed, overlapped with the backward pass) and scaled 1/N."""
        if self.optimizer is None:
            self._compile()
        eng = self._get_engine()
        sync = None
        if data_parallel:
            from ..utils.data_parallel import make_grad_sync
            sync = make_grad_sync(eng.flat_g)
        if self.train_graphs:
            out = eng.step_graphed(input_sequence, target_sequence, target_durations, target_pitch, sync=sync)
        else:
            out = eng.forward_backward(input_sequence, target_sequence, target_durations, target_pitch, training=True, sync=sync)
        scale = sync.finish() if sync is not None else 1.0
        eng.apply_adam(self.optimizer, grad_scale=scale)
        return out

    @_on_device
    def val_step(self, input_sequence, target_sequence, target_durations, target_pitch):
        """reference: model/models.py:492-507."""
        return self._get_engine().forward_backward(input_sequence, target_sequence, target_durations, target_pitch, training=False)

    @property
    def step(self) -> int:
        return int(self.optimizer.iterations) if self.optimizer is not None else 0

    def set_constants(self, learning_rate: float = None, **kwargs):
        if learning_rate is not None and self.optimizer is not None:
            self.optimizer.lr = float(learning_rate)
