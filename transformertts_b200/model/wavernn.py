"""WaveRNN generator (fatchord/WaveRNN, the vocoder the reference's ``data_config_wavernn.yaml`` section is made for) on the
GPU, a ragged batch of clips per call.

Everything that is not recurrent runs at frame rate through ``ttsb_conv1d_ex_tc`` on melgan.py's packed layout (zero halos):
the MelResNet (conv_in with BatchNorm folded and ReLU, the ResBlocks with their residual, conv_out), then one product that
projects each frame's four aux parts onto I, W_ih1 I, rnn2's input weights, fc1 and fc2, and one that projects each mel
frame onto I's mel columns and W_ih1 I.  The mel path of the upsample network is linear and reaches at most `half` frames,
so m_up[hop f + p] = sum_j K[p, j] m[f + j - half] exactly, with K extracted in float64 (composite_taps); the
recurrence adds sum_j K[p, j] P[f + j - half] of the projected frames instead of materialising m_up.

The recurrence itself, every step of every fold of every clip, is one persistent cooperative launch of
``ttsb_wavernn_generate`` (csrc/wavernn.cu), which also crossfades the folds, crops and fades out.

Seeds are per clip (``seeds[c]``, default c), so a clip's audio does not depend on its batch; fatchord draws from torch's
unseeded global RNG.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from transformertts_b200 import lib
from transformertts_b200.model.melgan import _Conv, _cols, conv_taps, layout_rows, pack_clips, run_conv

N_MELS = 80
MEL_COLS = 128            # the 80 mel channels padded to two k blocks
DIMS = lib.WAVERNN_DIMS
MIN_FRAMES = lib.WAVERNN_MIN_FRAMES
TARGET, OVERLAP = 11_000, 550
BN_EPS = 1e-5
MELP_COLS, AUX_COLS = 2048, 4608
_BN = ('weight', 'bias', 'running_mean', 'running_var', 'num_batches_tracked')


def _key(sd, k):
    if k not in sd:
        raise KeyError(f'WaveRNN checkpoint: missing key {k}')
    return tuple(sd[k].shape)


def infer_hparams(sd) -> dict:
    """Every hyper-parameter of a fatchord state dict, from its shapes: pad, res_blocks, compute / res_out dims, upsample
    factors, rnn / fc dims, mode and bits."""
    cin = _key(sd, 'upsample.resnet.conv_in.weight')
    if len(cin) != 3 or cin[2] % 2 == 0:
        raise ValueError(f'WaveRNN checkpoint: upsample.resnet.conv_in.weight has shape {cin}, expected (compute, feat, 2 pad + 1)')
    res_blocks = 0
    while f'upsample.resnet.layers.{res_blocks}.conv1.weight' in sd:
        res_blocks += 1
    factors = []
    while f'upsample.up_layers.{2 * len(factors) + 1}.weight' in sd:
        w = tuple(sd[f'upsample.up_layers.{2 * len(factors) + 1}.weight'].shape)
        if len(w) != 4 or w[:3] != (1, 1, 1) or w[3] < 3 or w[3] % 2 == 0:
            raise ValueError(f'WaveRNN checkpoint: upsample.up_layers.{2 * len(factors) + 1}.weight has shape {w}, expected (1, 1, 1, 2 s + 1)')
        factors.append((w[3] - 1) // 2)
    if not factors:
        raise KeyError('WaveRNN checkpoint: missing key upsample.up_layers.1.weight')
    n_classes = _key(sd, 'fc3.weight')[0]
    bits = None
    if n_classes != 30:
        bits = int(round(np.log2(n_classes))) if n_classes > 0 else 0
        if 2 ** bits != n_classes:
            raise ValueError(f'WaveRNN checkpoint: fc3 has {n_classes} rows, neither 30 (MOL) nor 2^bits (RAW)')
    return dict(pad=(cin[2] - 1) // 2, feat_dims=cin[1], compute_dims=cin[0], res_blocks=res_blocks,
                res_out_dims=_key(sd, 'upsample.resnet.conv_out.weight')[0], upsample_factors=tuple(factors),
                rnn_dims=_key(sd, 'rnn1.weight_hh_l0')[1], fc_dims=_key(sd, 'fc1.weight')[0], mode='MOL' if bits is None else 'RAW',
                bits=bits, n_classes=n_classes)


def expected_keys(h: dict) -> Dict[str, tuple]:
    """fatchord's state-dict keys and shapes for hyper-parameters h (model.save writes the bare state dict)."""
    C, F, R, A, D, Fc = h['compute_dims'], h['feat_dims'], h['res_out_dims'], h['res_out_dims'] // 4, h['rnn_dims'], h['fc_dims']
    keys = {'upsample.resnet.conv_in.weight': (C, F, 2 * h['pad'] + 1)}
    bn = lambda p: {f'{p}.{n}': (() if n == 'num_batches_tracked' else (C,)) for n in _BN}   # noqa: E731
    keys.update(bn('upsample.resnet.batch_norm'))
    for i in range(h['res_blocks']):
        p = f'upsample.resnet.layers.{i}'
        keys[f'{p}.conv1.weight'] = keys[f'{p}.conv2.weight'] = (C, C, 1)
        keys.update(bn(f'{p}.batch_norm1'))
        keys.update(bn(f'{p}.batch_norm2'))
    keys['upsample.resnet.conv_out.weight'] = (R, C, 1)
    keys['upsample.resnet.conv_out.bias'] = (R,)
    for i, s in enumerate(h['upsample_factors']):
        keys[f'upsample.up_layers.{2 * i + 1}.weight'] = (1, 1, 1, 2 * s + 1)
    keys['I.weight'], keys['I.bias'] = (D, F + A + 1), (D,)
    for n, cin in (('rnn1', D), ('rnn2', D + A)):
        keys[f'{n}.weight_ih_l0'], keys[f'{n}.weight_hh_l0'] = (3 * D, cin), (3 * D, D)
        keys[f'{n}.bias_ih_l0'] = keys[f'{n}.bias_hh_l0'] = (3 * D,)
    keys['fc1.weight'], keys['fc1.bias'] = (Fc, D + A), (Fc,)
    keys['fc2.weight'], keys['fc2.bias'] = (Fc, Fc + A), (Fc,)
    keys['fc3.weight'], keys['fc3.bias'] = (h['n_classes'], Fc), (h['n_classes'],)
    keys['step'] = (1,)
    return keys


def check_hparams(h: dict):
    """Refuses hyper-parameters this implementation does not run (ValueError naming the reason)."""
    if h['rnn_dims'] != DIMS or h['fc_dims'] != DIMS:
        raise ValueError(f"WaveRNN: rnn_dims = {h['rnn_dims']} and fc_dims = {h['fc_dims']}; the kernel runs {DIMS} only")
    if h['feat_dims'] != N_MELS:
        raise ValueError(f"WaveRNN: feat_dims = {h['feat_dims']}; the vocoder takes {N_MELS} mels")
    for name in ('compute_dims', 'res_out_dims'):
        c = h[name]
        if c < 64 or c % 64 or (c > 256 and c % 256):
            raise ValueError(f'WaveRNN: {name} = {c} must be a multiple of 64, at most 256 or a multiple of 256')
    if h['res_out_dims'] % 4:
        raise ValueError(f"WaveRNN: res_out_dims = {h['res_out_dims']} must split into four aux parts")
    if h['mode'] == 'RAW' and not 8 <= h['bits'] <= 10:
        raise ValueError(f"WaveRNN: RAW with bits = {h['bits']}; 8 <= bits <= 10 are supported")
    half = reach_frames(h['upsample_factors'])
    if 2 * half + 1 > lib.WAVERNN_MAX_TAPS:
        raise ValueError(f"WaveRNN: upsample factors {h['upsample_factors']} reach {half} frames; at most {lib.WAVERNN_MAX_TAPS // 2}")
    if h['pad'] < half:
        raise ValueError(f"WaveRNN: pad = {h['pad']} is less than the {half} frames the upsample factors {h['upsample_factors']} reach")
    if 2 * h['pad'] + 1 > lib.CONV1D_EX_MAX_TAPS:
        raise ValueError(f"WaveRNN: pad = {h['pad']} gives a conv_in of {2 * h['pad'] + 1} taps; at most {lib.CONV1D_EX_MAX_TAPS}")


def composite_taps(up_weights, factors, half):
    """The upsample network's mel path as a per-phase filter: m_up[hop f + p] = sum_j K[p, j] m[f + j - half] for j in
    [0, 2 half], K (hop, 2 half + 1) in float64, from unit impulses through the stretch / conv chain (up_weights: the
    (2 s + 1)-wide conv kernels).  Exact when the chain reaches at most `half` frames (reach_frames) and the mel is padded
    with at least that many zero frames."""
    hop = int(np.prod(factors))
    n = 4 * half + 1                    # frames: the output frame in the centre, 2 half frames of zeros on each side
    centre = n // 2
    K = np.zeros((hop, 2 * half + 1))
    for j in range(2 * half + 1):
        m = torch.zeros(1, 1, 1, n, dtype=torch.float64)
        m[..., centre + j - half] = 1.0
        for s, w in zip(factors, up_weights):
            m = m.repeat_interleave(s, dim=-1)
            m = F.conv2d(m, torch.as_tensor(w, dtype=torch.float64).reshape(1, 1, 1, 2 * s + 1), padding=(0, s))
        K[:, j] = m[0, 0, 0, centre * hop:(centre + 1) * hop].numpy()
    return K


def reach_frames(factors) -> int:
    """Frames on each side that an upsampled sample depends on: stage i's conv spans s_i samples at rate s_1 .. s_i."""
    reach, rate = 0.0, 1
    for s in factors:
        rate *= s
        reach += s / rate
    return int(math.ceil(reach - 1e-9))


def fold_bn(w: np.ndarray, sd, prefix: str):
    """A bias-free conv followed by eval-mode BatchNorm -> (weight, bias), in float64."""
    g = lambda n: sd[f'{prefix}.{n}'].detach().cpu().double().numpy()   # noqa: E731
    scale = g('weight') / np.sqrt(g('running_var') + BN_EPS)
    return w * scale[:, None, None], g('bias') - g('running_mean') * scale


def fold_count(total: int, target: int, overlap: int) -> int:
    """fold_with_overlap's number of folds for a sequence of `total` samples."""
    n = (total - overlap) // (target + overlap)
    if total - (n * (overlap + target) + overlap) != 0:
        n += 1
    return n


def fold_rows(frames: Sequence[int], hop: int, batched: bool, target: int, overlap: int):
    """-> ([(clip, fold, first sample, valid samples)], steps per fold): the rows the kernel runs."""
    L = target + 2 * overlap if batched else max(frames) * hop
    rows = []
    for c, T in enumerate(frames):
        total = T * hop
        for i in range(fold_count(total, target, overlap) if batched else 1):
            first = i * (target + overlap) if batched else 0
            rows.append((c, i, first, max(0, min(L, total - first))))
    return rows, L


def crossfade_gains(L: int, overlap: int) -> np.ndarray:
    """The gain xfade_and_unfold applies to each sample of a fold of length L."""
    silence, fade = overlap // 2, overlap - overlap // 2
    t = np.linspace(-1, 1, fade)
    g = np.ones(L)
    g[:overlap] *= np.concatenate([np.zeros(silence), np.sqrt(0.5 * (1 + t))])
    g[L - overlap:] *= np.concatenate([np.ones(silence), np.sqrt(0.5 * (1 - t))])
    return g


class WaveRNNGenerator:
    """fatchord's WaveRNN generator, vocoding ragged batches on the GPU.

    precision: 'bf16x3' (fp32-class: fp32 products in the recurrence, hi/lo split operands in the convs) or 'bf16' (single
    bf16 products everywhere, fp32 sums and states)."""

    def __init__(self, device=None, precision: str = 'bf16x3'):
        if precision not in ('bf16x3', 'bf16'):
            raise ValueError(f"precision must be 'bf16x3' or 'bf16', got {precision!r}")
        self.device = torch.device(device if device is not None else 'cuda')
        self.precision = precision
        self.split = precision == 'bf16x3'
        self.h: Optional[dict] = None

    @classmethod
    def from_checkpoint(cls, path, device=None, precision: str = 'bf16x3') -> 'WaveRNNGenerator':
        g = cls(device=device, precision=precision)
        g.load_state_dict(torch.load(path, map_location='cpu', weights_only=True))
        return g

    @property
    def hop(self) -> int:
        return int(np.prod(self.h['upsample_factors']))

    @staticmethod
    def check_state_dict(sd) -> dict:
        """Checks a bare fatchord state dict against the shapes its own hyper-parameters imply -> those hyper-parameters."""
        if not isinstance(sd, dict):
            raise TypeError(f'expected a state dict, got {type(sd).__name__}')
        h = infer_hparams(sd)
        want = expected_keys(h)
        missing = [k for k in want if k not in sd]
        if missing:
            raise KeyError(f'WaveRNN checkpoint: missing key {missing[0]}' + (f' (and {len(missing) - 1} more)' if len(missing) > 1 else ''))
        extra = [k for k in sd if k not in want]
        if extra:
            raise KeyError(f'WaveRNN checkpoint: unexpected key {extra[0]}' + (f' (and {len(extra) - 1} more)' if len(extra) > 1 else ''))
        for k, shape in want.items():
            if tuple(sd[k].shape) != tuple(shape) and not (k.endswith('num_batches_tracked') and sd[k].numel() == 1):
                raise ValueError(f'WaveRNN checkpoint: {k} has shape {tuple(sd[k].shape)}, expected {tuple(shape)}')
        check_hparams(h)
        return h

    def load_state_dict(self, sd) -> 'WaveRNNGenerator':
        h = self.check_state_dict(sd)
        f = lambda k: sd[k].detach().cpu().double().numpy()   # noqa: E731
        dev, split = self.device, self.split
        pad, C, Ro, A = h['pad'], h['compute_dims'], h['res_out_dims'], h['res_out_dims'] // 4
        self.halo = max(lib.CONV1D_HALO, pad)
        self.half = reach_frames(h['upsample_factors'])
        K = composite_taps([f(f'upsample.up_layers.{2 * i + 1}.weight') for i in range(len(h['upsample_factors']))],
                           h['upsample_factors'], self.half)
        Iw, Ib = f('I.weight'), f('I.bias')
        I0, Im, Ia = Iw[:, 0], Iw[:, 1:1 + N_MELS], Iw[:, 1 + N_MELS:]
        Wih1, bih1, Wih2 = f('rnn1.weight_ih_l0'), f('rnn1.bias_ih_l0'), f('rnn2.weight_ih_l0')
        fc1, fc2, fc3 = f('fc1.weight'), f('fc2.weight'), f('fc3.weight')
        convs = {}
        with torch.cuda.device(dev):
            w, b = fold_bn(f('upsample.resnet.conv_in.weight'), sd, 'upsample.resnet.batch_norm')
            convs['in'] = _Conv(conv_taps(w, 1, MEL_COLS, C), b, [(0, s) for s in range(-pad, pad + 1)], split, dev)
            for i in range(h['res_blocks']):
                p = f'upsample.resnet.layers.{i}'
                for j in (1, 2):
                    w, b = fold_bn(f(f'{p}.conv{j}.weight'), sd, f'{p}.batch_norm{j}')
                    convs[f'res{i}.{j}'] = _Conv(conv_taps(w, 1, C, C), b, [(0, 0)], split, dev)
            convs['out'] = _Conv(conv_taps(f('upsample.resnet.conv_out.weight'), 1, C, Ro), f('upsample.resnet.conv_out.bias'),
                                 [(0, 0)], split, dev)
            # frame-rate projections (no biases: past a clip the conditioning is zero and the biases stay)
            ma = np.zeros((_cols(Ro), AUX_COLS))
            ma[0:A, 0:512] = Ia.T
            ma[0:A, 512:2048] = (Wih1 @ Ia).T
            ma[A:2 * A, 2048:3584] = Wih2[:, DIMS:].T
            ma[2 * A:3 * A, 3584:4096] = fc1[:, DIMS:].T
            ma[3 * A:4 * A, 4096:4608] = fc2[:, DIMS:].T
            convs['auxp'] = _Conv(ma, np.zeros(AUX_COLS), [(0, 0)], split, dev)
            mm = np.zeros((MEL_COLS, MELP_COLS))
            mm[:N_MELS, 0:512] = Im.T
            mm[:N_MELS, 512:2048] = (Wih1 @ Im).T
            convs['melp'] = _Conv(mm, np.zeros(MELP_COLS), [(0, 0)], split, dev)
            vec = np.concatenate([I0, Ib, Wih1 @ I0, Wih1 @ Ib + bih1, f('rnn1.bias_hh_l0'), f('rnn2.bias_ih_l0'), f('rnn2.bias_hh_l0'),
                                  f('fc1.bias'), f('fc2.bias'), f('fc3.bias')])
            self._vec = torch.from_numpy(vec.astype(np.float32)).to(dev)
            wmat = np.concatenate([f('rnn1.weight_hh_l0'), Wih2[:, :DIMS], f('rnn2.weight_hh_l0'), fc1[:, :DIMS], fc2[:, :DIMS], fc3])
            wt = torch.from_numpy(wmat.astype(np.float32)).to(dev)
            self._w = wt.contiguous() if split else wt.to(torch.bfloat16).contiguous()
            self._taps = torch.from_numpy(np.ascontiguousarray(K, dtype=np.float32)).to(dev)
        self._convs = convs
        self.h = h
        return self

    # ---------------------------------------------------------------------------------------------------- forward
    def _planes(self, rows: int, cols: int):
        """Zeroed hi (and lo) planes: halo rows are never written, so they keep the zero padding."""
        hi = torch.zeros((rows, cols), dtype=torch.bfloat16, device=self.device)
        return hi, (torch.zeros_like(hi) if self.split else None)

    def _run(self, name, counts, src, **kw):
        run_conv(self._convs[name], counts, [src], 1, self.split, rows_halo=self.halo, **kw)

    def conditioning(self, fmels: Sequence[np.ndarray]):
        """fatchord-space mels (80, T_c) -> (aux (rows, cols(res_out)), melp planes, auxp planes) in the packed layout."""
        h, H, ws = self.h, self.halo, None
        counts = [m.shape[1] for m in fmels]
        rows = layout_rows(counts, halo=H)
        C, Ro = h['compute_dims'], h['res_out_dims']
        x = pack_clips([np.asarray(m, dtype=np.float32).T for m in fmels], MEL_COLS, lib.HALO_ZERO, halo=H)
        ws = torch.empty(lib.conv1d_workspace_bytes(len(fmels)), dtype=torch.uint8, device=self.device)
        src = lib.split_bf16(torch.from_numpy(x).to(self.device), self.split)
        a, b, t = self._planes(rows, C), self._planes(rows, C), self._planes(rows, C)
        self._run('in', counts, src, act=a, slope=0.0, ws=ws)
        for i in range(h['res_blocks']):
            self._run(f'res{i}.1', counts, a, act=t, slope=0.0, ws=ws)
            self._run(f'res{i}.2', counts, t, res=a, out=b, ws=ws)
            a, b = b, a
        aux = self._planes(rows, _cols(Ro))
        self._run('out', counts, a, out=aux, ws=ws)
        auxp, melp = self._planes(rows, AUX_COLS), self._planes(rows, MELP_COLS)
        self._run('auxp', counts, aux, out=auxp, ws=ws)
        self._run('melp', counts, src, out=melp, ws=ws)
        return aux, melp, auxp

    def _generate(self, fmels, seeds, batched, target, overlap, capture_steps=0, keep_samples=False, timings=None):
        """-> (packed waveform, captured logits (rows, capture_steps, n_classes) or None, per-fold samples (rows, steps) or None).
        timings: None, or a device int64 (lib.WAVERNN_CTAS, 2 len(lib.WAVERNN_SEGMENTS)) tensor that receives the kernel's phase
        timers (include/ttsb.h: ttsb_wavernn_generate)."""
        if self.h is None:
            raise RuntimeError('WaveRNNGenerator: no weights loaded (from_checkpoint / load_state_dict)')
        if not fmels:
            raise ValueError('vocode_batch: no mels')
        for c, m in enumerate(fmels):
            if m.ndim != 2 or m.shape[0] != N_MELS:
                raise ValueError(f'mel {c} has shape {m.shape}; the vocoder needs ({N_MELS}, T)')
            if m.shape[1] < MIN_FRAMES:
                raise ValueError(f'mel {c} has {m.shape[1]} frames; WaveRNN generation needs at least {MIN_FRAMES} (its fade-out '
                                 f'spans the last 20 hops)')
        if batched and (target < 1 or overlap < 1):
            raise ValueError(f'target = {target} and overlap = {overlap} must be >= 1')
        frames = [m.shape[1] for m in fmels]
        seeds = list(range(len(fmels))) if seeds is None else [int(s) for s in seeds]
        if len(seeds) != len(fmels):
            raise ValueError(f'{len(seeds)} seeds for {len(fmels)} mels')
        hop, h = self.hop, self.h
        rows, L = fold_rows(frames, hop, batched, target, overlap)
        with torch.cuda.device(self.device):
            _, melp, auxp = self.conditioning(fmels)
            ws = torch.empty(lib.wavernn_workspace_bytes(frames, hop, batched, target, overlap, h['n_classes']), dtype=torch.uint8,
                             device=self.device)
            wav = torch.empty(sum((T - 1) * hop for T in frames), dtype=torch.float32, device=self.device)
            cap = torch.empty((len(rows), capture_steps, h['n_classes']), dtype=torch.float32, device=self.device) if capture_steps else None
            samples = torch.empty((len(rows), L), dtype=torch.float32, device=self.device) if keep_samples else None
            ftab = (lib.C.c_int32 * len(frames))(*frames)
            stab = (lib.C.c_uint32 * len(seeds))(*[s & 0xFFFFFFFF for s in seeds])
            lib.wavernn_generate(
                frames=lib.C.cast(ftab, lib.C.c_void_p), seeds=lib.C.cast(stab, lib.C.c_void_p), n_clips=len(frames), hop=hop,
                batched=int(bool(batched)), target=int(target), overlap=int(overlap), n_rows=len(rows), n_taps=self._taps.shape[1],
                taps=lib.ptr(self._taps), melp_hi=lib.ptr(melp[0]), melp_lo=lib.ptr(melp[1]), ld_melp=MELP_COLS,
                aux_hi=lib.ptr(auxp[0]), aux_lo=lib.ptr(auxp[1]), ld_aux=AUX_COLS, cond_halo=self.halo, cond_rows=melp[0].shape[0],
                vec=lib.ptr(self._vec), weights=lib.ptr(self._w), mode=lib.WAVERNN_MOL if h['mode'] == 'MOL' else lib.WAVERNN_RAW,
                n_classes=h['n_classes'], precision=lib.PREC_BF16X3 if self.split else lib.PREC_BF16, wav_out=lib.ptr(wav),
                capture=lib.ptr(cap), capture_steps=int(capture_steps), samples_out=lib.ptr(samples), timings=lib.ptr(timings),
                workspace=lib.ptr(ws), workspace_bytes=ws.numel())
        return wav, cap, samples

    def vocode_device(self, mels: Sequence[np.ndarray], seeds=None, batched: bool = True, target: int = TARGET,
                      overlap: int = OVERLAP) -> torch.Tensor:
        """vocode_batch, leaving the packed float32 waveform ((T_c - 1) hop samples per clip, clip after clip) on the device."""
        fm = [(np.asarray(m, dtype=np.float32) + np.float32(4.0)) / np.float32(8.0) for m in mels]
        return self._generate(fm, seeds, batched, target, overlap)[0]

    def vocode_batch(self, mels: Sequence[np.ndarray], seeds=None, batched: bool = True, target: int = TARGET,
                     overlap: int = OVERLAP) -> List[np.ndarray]:
        """This project's WaveRNN-normalised mels (80, T_c) (clip((dB + 100) / 100, 0, 1) 8 - 4) -> float32 waveforms of
        (T_c - 1) hop samples, what fatchord's generate() gives for fatchord's normalize() of the same mel, clip c drawn
        with seeds[c] (default c)."""
        wav = self.vocode_device(mels, seeds, batched, target, overlap).cpu().numpy()
        off = np.concatenate([[0], np.cumsum([(np.asarray(m).shape[1] - 1) * self.hop for m in mels])])
        return [wav[off[c]:off[c + 1]] for c in range(len(mels))]

    def generate(self, mel, batched: bool = True, target: int = TARGET, overlap: int = OVERLAP, seed: int = 0) -> np.ndarray:
        """fatchord's generate() for one (1, 80, T) mel in fatchord's input space, without save_path -> float32 waveform."""
        m = torch.as_tensor(mel).detach().cpu().float()
        if m.ndim == 3:
            if m.shape[0] != 1:
                raise ValueError(f'generate takes one mel, got a batch of {m.shape[0]}')
            m = m[0]
        return self._generate([m.numpy()], [seed], batched, target, overlap)[0].cpu().numpy()

