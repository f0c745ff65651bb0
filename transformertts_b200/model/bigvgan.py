"""BigVGAN generator (NVIDIA/BigVGAN, Lee et al., ICLR 2023: the 22.05 kHz, hop-256 configs and any config of the same form)
on the GPU, a packed ragged batch of clips per call.

Every conv is one ``ttsb_conv1d_ex_tc`` launch over all clips, on melgan.py's packed layout with ``halo`` rows on each side of
every clip (the largest tap shift of the config: 25 rows for the published ones), and every anti-aliased Snake activation is
one ``ttsb_snake_aa_ex`` launch (2x Kaiser-sinc upsampling, SnakeBeta, low-pass and 2x decimation, each clip's replicate
padding at its own edges).  Every conv pads with zeros and neither kernel writes a halo row, so the planes are
zero-initialised and the halos stay zero; a clip of any length >= 1 frame works.  Per call: the split of the input mel,
conv_pre, then per stage the transposed conv (as melgan.py phrases it, no activation before it) and the AMPBlock1s (per
dilation: activation, conv, activation, conv + residual), activation_post and conv_post (``ttsb_conv1d_out_tanh_ex``, or
``ttsb_conv1d_out_clamp_ex`` for the v2 final layer).  The multi-receptive-field average is the conv epilogue's fp32 sum
plane, in torch's order, as in hifigan.py.

Channel counts are carried in columns the conv kernel takes (``stage_cols``): at least 64, a multiple of 64, at most 256 or
a multiple of 256, also as u times the width for the transposed conv into the stage.  The 1536-channel config's 384, 192
and 96 channels become 512, 256 and 128 columns whose extra weights are zero; the activation writes those columns as 0.

The state-dict key layout is the published module tree; it is kept in KEYS below, the one place to correct it against a
released checkpoint (none was available to check it against).
"""
from __future__ import annotations

import json
from pathlib import Path
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from transformertts_b200 import lib
from transformertts_b200.model.melgan import (_Conv, conv_taps, fold_weight_norm, layout_rows, pack_clips, ragged_offsets, run_conv,
                                              transposed_taps)

HOP = 256
MEL_COLS = 128            # conv_pre's num_mels channels padded to two k blocks
MAX_WAV_VALUE = 32767.0   # BigVGAN's inference scale
FILTER_TAPS = 12          # the Kaiser-sinc filters of UpSample1d / DownSample1d (ratio 2)
ARCH_KEYS = ('resblock', 'upsample_rates', 'upsample_kernel_sizes', 'upsample_initial_channel', 'resblock_kernel_sizes',
             'resblock_dilation_sizes', 'activation', 'snake_logscale')
DEFAULTS = {'num_mels': 80, 'use_tanh_at_final': True, 'use_bias_at_final': True}   # v1's final layer when absent
AUDIO_KEYS = ('sampling_rate', 'num_mels', 'hop_size', 'fmax')
_AMP = dict(resblock='1', resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
            activation='snakebeta', snake_logscale=True, num_mels=80, sampling_rate=22050, hop_size=256, fmax=8000)
PRESETS = {
    'base': dict(_AMP, upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512),
    'bigvgan': dict(_AMP, upsample_rates=[4, 4, 2, 2, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4, 4, 4], upsample_initial_channel=1536),
}

# The published state-dict layout (NVIDIA/BigVGAN bigvgan.py, activations.py, alias_free_activation/torch/*.py).  Convs carry
# weight_g / weight_v (or weight after remove_weight_norm) and bias; an activation prefix carries the rest.
KEYS = {
    'conv_pre': 'conv_pre',
    'up': 'ups.{i}.0',                                # each ups[i] is a one-element ModuleList
    'convs1': 'resblocks.{n}.convs1.{m}',
    'convs2': 'resblocks.{n}.convs2.{m}',
    'block_act': 'resblocks.{n}.activations.{k}',     # Activation1d k of AMPBlock1 n: a1 = [0::2], a2 = [1::2]
    'post_act': 'activation_post',
    'conv_post': 'conv_post',
    'alpha': '{act}.act.alpha',
    'beta': '{act}.act.beta',                         # SnakeBeta only
    'up_filter': '{act}.upsample.filter',
    'down_filter': '{act}.downsample.lowpass.filter',
}


def load_config(config) -> dict:
    """A preset name ('base' | 'bigvgan'), the path of a BigVGAN config.json, or a dict -> the checked config: the
    generator's keys, with use_tanh_at_final / use_bias_at_final / num_mels defaulted, and under 'audio' whichever of
    sampling_rate, num_mels, hop_size and fmax it gives."""
    if isinstance(config, (str, Path)) and str(config).lower() in PRESETS:
        h = dict(PRESETS[str(config).lower()])
    elif isinstance(config, (str, Path)):
        with open(config, 'r') as f:
            h = json.load(f)
    elif isinstance(config, dict):
        h = dict(config)
    else:
        raise TypeError(f'config must be a preset name, a path or a dict, got {type(config).__name__}')
    missing = [k for k in ARCH_KEYS if k not in h]
    if missing:
        raise ValueError(f'BigVGAN config: missing key {missing[0]}')
    out = {k: h[k] for k in ARCH_KEYS}
    out.update({k: h.get(k, v) for k, v in DEFAULTS.items()})
    out['audio'] = dict(h['audio']) if isinstance(h.get('audio'), dict) else {k: h[k] for k in AUDIO_KEYS if k in h}
    out['resblock'] = str(out['resblock'])
    check_config(out)
    return out


def stage_cols(h: dict) -> List[int]:
    """Columns of the activation of stage 0 (conv_pre's output) .. n (the last upsampling stage's): the least width >= the
    channel count that is a multiple of 64, at most 256 or a multiple of 256, and (for stages after the first) gives a
    transposed conv of u times that many columns of the same form."""
    def ok(n):
        return n % 64 == 0 and (n <= 256 or n % 256 == 0)
    c0, rates, out = h['upsample_initial_channel'], h['upsample_rates'], []
    for i in range(len(rates) + 1):
        w = max(64, -(-(c0 // 2 ** i) // 64) * 64)
        while not (ok(w) and (i == 0 or ok(rates[i - 1] * w))):
            w += 64
        out.append(w)
    return out


def check_config(h: dict):
    """Refuses a config this implementation does not run (ValueError naming the reason)."""
    if h['resblock'] != '1':
        raise ValueError(f"BigVGAN config: resblock {h['resblock']!r} is not supported; only '1' (AMPBlock1, which every published "
                         f"checkpoint uses)")
    if h['activation'] not in ('snake', 'snakebeta'):
        raise ValueError(f"BigVGAN config: activation must be 'snake' or 'snakebeta', got {h['activation']!r}")
    nm = h['num_mels']
    if not isinstance(nm, int) or not 1 <= nm <= MEL_COLS:
        raise ValueError(f'BigVGAN config: num_mels = {nm!r} must be an integer in [1, {MEL_COLS}]')
    rates, kernels = list(h['upsample_rates']), list(h['upsample_kernel_sizes'])
    if not rates or len(rates) != len(kernels):
        raise ValueError('BigVGAN config: upsample_rates and upsample_kernel_sizes must be non-empty and of equal length')
    if int(np.prod(rates)) != HOP:
        raise ValueError(f'BigVGAN config: the upsample rates multiply to {int(np.prod(rates))}, not the hop of {HOP}')
    for u, k in zip(rates, kernels):
        if u % 2 or k != 2 * u:
            raise ValueError(f'BigVGAN config: upsample kernel {k} with rate {u}; only kernel = 2 rate with an even rate is supported')
    ks, ds = list(h['resblock_kernel_sizes']), list(h['resblock_dilation_sizes'])
    if not ks or len(ks) != len(ds):
        raise ValueError('BigVGAN config: resblock_kernel_sizes and resblock_dilation_sizes must be non-empty and of equal length')
    for k, d in zip(ks, ds):
        if k % 2 == 0 or k < 1 or k > lib.CONV1D_EX_MAX_TAPS:
            raise ValueError(f'BigVGAN config: resblock kernel {k} must be odd and at most {lib.CONV1D_EX_MAX_TAPS}')
        if len(d) < 1 or min(d) < 1:
            raise ValueError(f'BigVGAN config: AMPBlock1 takes dilations >= 1, got {list(d)}')
    if halo_rows(h) > lib.CONV1D_EX_MAX_HALO:
        raise ValueError(f'BigVGAN config: a tap shift of {halo_rows(h)} rows exceeds {lib.CONV1D_EX_MAX_HALO}')
    c0 = h['upsample_initial_channel']
    for i in range(len(rates) + 1):
        if c0 // 2 ** i < 1 or (c0 // 2 ** i) * 2 ** i != c0:
            raise ValueError(f'BigVGAN config: stage {i} has {c0} / 2^{i} channels, which is not a positive integer')
    if stage_cols(h)[-1] > 256:
        raise ValueError('BigVGAN config: conv_post takes at most 256 channels')


def check_audio(h: dict, sampling_rate, mel_channels, hop_length, f_max):
    """Refuses (ValueError naming the key) a config whose sampling_rate, num_mels, hop_size or fmax differs from the given
    audio settings; keys the config does not give are not checked.  fmax / f_max None mean sampling_rate / 2."""
    a = h['audio']
    mine = {'sampling_rate': sampling_rate, 'num_mels': mel_channels, 'hop_size': hop_length}
    for k, v in mine.items():
        if k in a and float(a[k]) != float(v):
            raise ValueError(f'BigVGAN config: {k} = {a[k]} differs from the audio settings ({v})')
    if 'fmax' in a:
        want = sampling_rate / 2 if f_max is None else f_max
        got = a.get('sampling_rate', sampling_rate) / 2 if a['fmax'] is None else a['fmax']
        if float(got) != float(want):
            raise ValueError(f"BigVGAN config: fmax = {a['fmax']} differs from the audio settings (f_max {f_max})")


def halo_rows(h: dict) -> int:
    """Halo rows of the packed layout: the largest tap shift of any conv (conv_pre / conv_post: 3)."""
    return max([3] + [d * (k - 1) // 2 for k, ds in zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes']) for d in ds])


def _blocks(h: dict):
    """[(stage i, resblock index n, kernel k, dilations)] in execution order."""
    nk = len(h['resblock_kernel_sizes'])
    return [(i, i * nk + j, k, d) for i in range(len(h['upsample_rates']))
            for j, (k, d) in enumerate(zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes']))]


def layer_shapes(h: dict) -> Dict[str, tuple]:
    """conv name -> (kind, weight shape): kind 'conv' (Cout, Cin, k) or 'convT' (Cin, Cout, k)."""
    c0 = h['upsample_initial_channel']
    out = {KEYS['conv_pre']: ('conv', (c0, h['num_mels'], 7))}
    for i, k in enumerate(h['upsample_kernel_sizes']):
        out[KEYS['up'].format(i=i)] = ('convT', (c0 // 2 ** i, c0 // 2 ** (i + 1), k))
    for i, n, k, dil in _blocks(h):
        ch = c0 // 2 ** (i + 1)
        for m in range(len(dil)):
            out[KEYS['convs1'].format(n=n, m=m)] = ('conv', (ch, ch, k))
            out[KEYS['convs2'].format(n=n, m=m)] = ('conv', (ch, ch, k))
    out[KEYS['conv_post']] = ('conv', (1, c0 // 2 ** len(h['upsample_rates']), 7))
    return out


def activation_prefixes(h: dict) -> Dict[str, int]:
    """Activation1d prefix -> its channel count, in the state dict's order."""
    c0, out = h['upsample_initial_channel'], {}
    for i, n, _, dil in _blocks(h):
        for k in range(2 * len(dil)):
            out[KEYS['block_act'].format(n=n, k=k)] = c0 // 2 ** (i + 1)
    out[KEYS['post_act']] = c0 // 2 ** len(h['upsample_rates'])
    return out


def expected_keys(h: dict, weight_norm: bool = True) -> Dict[str, tuple]:
    """The checkpoint's state-dict keys and shapes (weight_g / weight_v form, or the plain `weight` remove_weight_norm
    leaves), filter buffers included."""
    keys = {}
    for name, (kind, shape) in layer_shapes(h).items():
        if name != KEYS['conv_post'] or h['use_bias_at_final']:
            keys[f'{name}.bias'] = (shape[1] if kind == 'convT' else shape[0],)
        if weight_norm:
            keys[f'{name}.weight_g'] = (shape[0], 1, 1)
            keys[f'{name}.weight_v'] = shape
        else:
            keys[f'{name}.weight'] = shape
    for act, ch in activation_prefixes(h).items():
        keys[KEYS['alpha'].format(act=act)] = (ch,)
        if h['activation'] == 'snakebeta':
            keys[KEYS['beta'].format(act=act)] = (ch,)
        keys[KEYS['up_filter'].format(act=act)] = (1, 1, FILTER_TAPS)
        keys[KEYS['down_filter'].format(act=act)] = (1, 1, FILTER_TAPS)
    return keys


def launches_per_call(h: dict) -> int:
    """Library launches of one vocode call: the mel split, conv_pre, per stage the transposed conv and per dilation of every
    AMPBlock1 two activations and two convs, activation_post, conv_post."""
    return 4 + len(h['upsample_rates']) * (1 + 4 * sum(len(d) for d in h['resblock_dilation_sizes']))


def snake_params(h: dict, alpha: np.ndarray, beta: Optional[np.ndarray]):
    """Checkpoint alpha (and beta) -> float64 (alpha, inv_beta) as the kernel takes them: exp under snake_logscale, then
    1 / (beta + 1e-9); Snake is the case beta = alpha."""
    a = np.exp(alpha) if h['snake_logscale'] else np.asarray(alpha, dtype=np.float64)
    if beta is None:
        return a, 1.0 / (a + 1e-9)
    b = np.exp(beta) if h['snake_logscale'] else np.asarray(beta, dtype=np.float64)
    return a, 1.0 / (b + 1e-9)


def _padded(b: np.ndarray, cols: int, reps: int = 1) -> np.ndarray:
    out = np.zeros(reps * cols)
    for r in range(reps):
        out[r * cols:r * cols + len(b)] = b
    return out


class _Act:
    """One Activation1d: per-channel fp32 alpha and inv_beta on the device, the two 12-tap filters on the host."""

    def __init__(self, channels: int, alpha: np.ndarray, inv_beta: np.ndarray, h_up: np.ndarray, h_down: np.ndarray, device):
        self.channels = channels
        self.alpha = torch.from_numpy(np.ascontiguousarray(alpha, dtype=np.float32)).to(device)
        self.inv_beta = torch.from_numpy(np.ascontiguousarray(inv_beta, dtype=np.float32)).to(device)
        self.h_up = [float(v) for v in np.asarray(h_up, dtype=np.float32).reshape(-1)]
        self.h_down = [float(v) for v in np.asarray(h_down, dtype=np.float32).reshape(-1)]


class BigVGANGenerator:
    """The BigVGAN generator of NVIDIA/BigVGAN, vocoding ragged batches on the GPU.

    config: a preset name ('base' | 'bigvgan'), the path of its config.json or a dict.
    precision: 'bf16x3' (hi/lo split operands, fp32-class products) or 'bf16' (one bf16 product per conv)."""

    def __init__(self, config='base', device=None, precision: str = 'bf16x3'):
        if precision not in ('bf16x3', 'bf16'):
            raise ValueError(f"precision must be 'bf16x3' or 'bf16', got {precision!r}")
        self.h = load_config(config)
        self.halo = halo_rows(self.h)
        self.cols = stage_cols(self.h)
        self.device = torch.device(device if device is not None else 'cuda')
        self.precision = precision
        self.split = precision == 'bf16x3'
        self._convs: Optional[dict] = None
        self._acts: Optional[dict] = None

    @property
    def num_mels(self) -> int:
        return self.h['num_mels']

    # ---------------------------------------------------------------------------------------------------- loading
    @classmethod
    def from_checkpoint(cls, path, config=None, device=None, precision: str = 'bf16x3') -> 'BigVGANGenerator':
        """config None: the config.json beside the checkpoint, as BigVGAN's inference reads it."""
        if config is None:
            config = Path(path).parent / 'config.json'
            if not config.exists():
                raise FileNotFoundError(f'{config} not found: pass the generator config (a config.json path or base / bigvgan)')
        g = cls(config=config, device=device, precision=precision)
        g.load_state_dict(torch.load(path, map_location='cpu', weights_only=True))
        return g

    def fold_state_dict(self, sd) -> Dict[str, np.ndarray]:
        """Checks a checkpoint (``{'generator': sd}`` or a bare state dict, weight-normed or folded) against the config and
        returns float64 arrays: {conv name: weight, conv name + '.bias': bias (zeros for a conv_post without bias),
        activation prefix + '.alpha' / '.inv_beta' / '.h_up' / '.h_down'}."""
        if isinstance(sd, dict) and 'generator' in sd:
            sd = sd['generator']
        if not isinstance(sd, dict):
            raise TypeError(f'expected a state dict, got {type(sd).__name__}')
        keys = set(sd)
        normed, plain = expected_keys(self.h, True), expected_keys(self.h, False)
        want = normed if any(k.endswith('.weight_g') or k.endswith('.weight_v') for k in keys) else plain
        missing = sorted(set(want) - keys)
        if missing:
            raise KeyError(f'BigVGAN checkpoint: missing key {missing[0]}' + (f' (and {len(missing) - 1} more)' if len(missing) > 1 else ''))
        extra = sorted(keys - set(want))
        if extra:
            raise KeyError(f'BigVGAN checkpoint: unexpected key {extra[0]}' + (f' (and {len(extra) - 1} more)' if len(extra) > 1 else ''))
        for k, shape in want.items():
            if tuple(sd[k].shape) != tuple(shape):
                raise ValueError(f'BigVGAN checkpoint: {k} has shape {tuple(sd[k].shape)}, expected {tuple(shape)}')
        f64 = {k: sd[k].detach().cpu().double().numpy() for k in want}
        out = {}
        for name, (kind, shape) in layer_shapes(self.h).items():
            out[name] = fold_weight_norm(f64[f'{name}.weight_g'], f64[f'{name}.weight_v']) if want is normed else f64[f'{name}.weight']
            out[name + '.bias'] = f64.get(f'{name}.bias', np.zeros(shape[1] if kind == 'convT' else shape[0]))
        for act in activation_prefixes(self.h):
            beta = f64[KEYS['beta'].format(act=act)] if self.h['activation'] == 'snakebeta' else None
            out[act + '.alpha'], out[act + '.inv_beta'] = snake_params(self.h, f64[KEYS['alpha'].format(act=act)], beta)
            out[act + '.h_up'] = f64[KEYS['up_filter'].format(act=act)].reshape(-1)
            out[act + '.h_down'] = f64[KEYS['down_filter'].format(act=act)].reshape(-1)
        return out

    def load_state_dict(self, sd) -> 'BigVGANGenerator':
        w = self.fold_state_dict(sd)
        h, dev, split, cols = self.h, self.device, self.split, self.cols
        convs, acts = {}, {}
        with torch.cuda.device(dev):
            name = KEYS['conv_pre']
            convs[name] = _Conv(conv_taps(w[name], 1, MEL_COLS, cols[0]), _padded(w[name + '.bias'], cols[0]),
                                [(0, s) for s in range(-3, 4)], split, dev)
            for i, u in enumerate(h['upsample_rates']):
                name = KEYS['up'].format(i=i)
                convs[name] = _Conv(transposed_taps(w[name], u, cols[i], cols[i + 1]), _padded(w[name + '.bias'], cols[i + 1], u),
                                    [(0, -1), (0, 0), (0, 1)], split, dev)
            for i, n, k, dil in _blocks(h):
                cc = cols[i + 1]
                for m, d in enumerate(dil):
                    for key, dd in ((KEYS['convs1'].format(n=n, m=m), d), (KEYS['convs2'].format(n=n, m=m), 1)):
                        convs[key] = _Conv(conv_taps(w[key], dd, cc, cc), _padded(w[key + '.bias'], cc),
                                           [(0, (s - (k - 1) // 2) * dd) for s in range(k)], split, dev)
            for act, ch in activation_prefixes(h).items():
                acts[act] = _Act(ch, w[act + '.alpha'], w[act + '.inv_beta'], w[act + '.h_up'], w[act + '.h_down'], dev)
            name = KEYS['conv_post']
            self._post_w = torch.from_numpy(np.ascontiguousarray(w[name][0].T, dtype=np.float32)).to(dev)   # (7, C_last)
            self._post_b = float(w[name + '.bias'][0])
        self._convs, self._acts = convs, acts
        return self

    # ---------------------------------------------------------------------------------------------------- forward
    def _planes(self, rows: int, cols: int):
        """Zeroed hi (and lo) planes: halo rows are never written, so they keep the zero padding."""
        hi = torch.zeros((rows, cols), dtype=torch.bfloat16, device=self.device)
        return hi, (torch.zeros_like(hi) if self.split else None)

    def _conv(self, name, counts, src, up=1, **kw):
        run_conv(self._convs[name], counts, [src], up, self.split, rows_halo=self.halo, **kw)

    def _act(self, name, offsets, src, dst, ws):
        a = self._acts[name]
        lib.snake_aa_ex(src, dst, a.channels, self.halo, offsets, a.alpha, a.inv_beta, a.h_up, a.h_down, ws)

    def vocode_device(self, mels: Sequence[np.ndarray]) -> torch.Tensor:
        """vocode_batch, leaving the packed float32 waveform (256 sum T_c samples, clip after clip) on the device."""
        if self._convs is None:
            raise RuntimeError('BigVGANGenerator: no weights loaded (from_checkpoint / load_state_dict)')
        ms = [np.asarray(m, dtype=np.float32) for m in mels]
        if not ms:
            raise ValueError('vocode_batch: no mels')
        nm = self.num_mels
        for c, m in enumerate(ms):
            if m.ndim != 2 or m.shape[0] != nm or m.shape[1] < 1:
                raise ValueError(f'mel {c} has shape {m.shape}; the vocoder needs ({nm}, T) with T >= 1 frames')
        h, H, cols = self.h, self.halo, self.cols
        counts = [m.shape[1] for m in ms]
        x = pack_clips([m.T for m in ms], MEL_COLS, lib.HALO_ZERO, halo=H)
        with torch.cuda.device(self.device):
            ws = torch.empty(lib.conv1d_workspace_bytes(len(ms)), dtype=torch.uint8, device=self.device)
            src = lib.split_bf16(torch.from_numpy(x).to(self.device), self.split)
            cur = self._planes(layout_rows(counts, halo=H), cols[0])
            self._conv(KEYS['conv_pre'], counts, src, out=cur, ws=ws)
            nk = len(h['resblock_kernel_sizes'])
            for i, u in enumerate(h['upsample_rates']):
                counts_in, counts = counts, [c * u for c in counts]
                rows, cc, off = layout_rows(counts, halo=H), cols[i + 1], ragged_offsets(counts)
                x_st = self._planes(rows, cc)
                self._conv(KEYS['up'].format(i=i), counts_in, cur, u, out=x_st, ws=ws)
                t1, t2, pair = self._planes(rows, cc), self._planes(rows, cc), [self._planes(rows, cc) for _ in range(2)]
                cur = self._planes(rows, cc)         # the stage's output: the AMPBlocks' average
                total = torch.empty((rows, cc), dtype=torch.float32, device=self.device) if nk > 1 else None
                for j, (_, n, _, dil) in enumerate(_blocks(h)[i * nk:(i + 1) * nk]):
                    xin = x_st
                    for m in range(len(dil)):
                        self._act(KEYS['block_act'].format(n=n, k=2 * m), off, xin, t1, ws)
                        self._conv(KEYS['convs1'].format(n=n, m=m), counts, t1, out=t2, ws=ws)
                        self._act(KEYS['block_act'].format(n=n, k=2 * m + 1), off, t2, t1, ws)
                        name = KEYS['convs2'].format(n=n, m=m)
                        if m + 1 < len(dil):            # x = xt + x, kept for the next dilation
                            nxt = pair[m % 2]
                            self._conv(name, counts, t1, res=xin, out=nxt, ws=ws)
                            xin = nxt
                        elif nk == 1:
                            self._conv(name, counts, t1, res=xin, out=cur, ws=ws)
                        else:                            # the block's output goes to the sum
                            mode = lib.SUM_WRITE if j == 0 else (lib.SUM_FINISH if j == nk - 1 else lib.SUM_ADD)
                            self._conv(name, counts, t1, res=xin, sum_plane=total, sum_mode=mode, sum_div=float(nk),
                                       out=cur if mode == lib.SUM_FINISH else None, ws=ws)
                del x_st, t2, pair, total
            self._act(KEYS['post_act'], off, cur, t1, ws)
            wav = torch.empty(HOP * sum(m.shape[1] for m in ms), dtype=torch.float32, device=self.device)
            out_layer = lib.conv1d_out_tanh_ex if h['use_tanh_at_final'] else lib.conv1d_out_clamp_ex
            out_layer(t1[0], t1[1], self._acts[KEYS['post_act']].channels, H, off, 0, self._post_w, self._post_b, ws, wav)
        return wav

    def vocode_batch(self, mels: Sequence[np.ndarray]) -> List[np.ndarray]:
        """Log-mels (num_mels, T_c) (ln(max(S, 1e-5)), the MelGAN normaliser's) -> float32 waveforms of 256 T_c samples: what the
        generator computes per clip, before the int16 conversion."""
        wav = self.vocode_device(mels).cpu().numpy()
        off = ragged_offsets([np.asarray(m).shape[1] for m in mels], HOP)
        return [wav[off[c]:off[c + 1]] for c in range(len(mels))]

    def inference(self, mel) -> torch.Tensor:
        """BigVGAN's inference for one (1, num_mels, T) or (num_mels, T) mel: (wav * MAX_WAV_VALUE).astype(int16), 256 T samples
        on the CPU."""
        m = torch.as_tensor(mel).detach().cpu().float()
        if m.ndim == 3:
            if m.shape[0] != 1:
                raise ValueError(f'inference takes one mel, got a batch of {m.shape[0]}')
            m = m[0]
        wav = self.vocode_batch([m.numpy()])[0]
        return torch.from_numpy((wav * np.float32(MAX_WAV_VALUE)).astype(np.int16))


def conv_flops(h: dict, frames: int) -> Dict[str, float]:
    """Multiply-add FLOPs (2 per MAC) of the convs for `frames` mel frames: 'useful' over the config's channels, 'issued' over
    the padded columns the kernel runs (stage_cols, conv_pre's MEL_COLS)."""
    cols, c0, rates = stage_cols(h), h['upsample_initial_channel'], h['upsample_rates']
    useful = 2.0 * frames * 7 * h['num_mels'] * c0
    issued = 2.0 * frames * 7 * MEL_COLS * cols[0]
    T = frames
    for i, (u, k) in enumerate(zip(rates, h['upsample_kernel_sizes'])):
        cin, cout = c0 // 2 ** i, c0 // 2 ** (i + 1)
        useful += 2.0 * T * cin * cout * k                  # each input row meets k taps of cout outputs (spread over u rows)
        issued += 2.0 * T * 3 * cols[i] * u * cols[i + 1]
        T *= u
        for kk, dil in zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes']):
            useful += 2.0 * T * 2 * len(dil) * kk * cout * cout
            issued += 2.0 * T * 2 * len(dil) * kk * cols[i + 1] * cols[i + 1]
    cl = c0 // 2 ** len(rates)
    useful += 2.0 * T * 7 * cl
    issued += 2.0 * T * 7 * cl
    return {'useful': useful, 'issued': issued}


def activation_bytes(h: dict, frames: int, split: bool) -> float:
    """Bytes one vocode call's activation launches read and write at their least (each live and padded column of every clip row
    read once per plane and written once per plane)."""
    cols, rates, T, total = stage_cols(h), h['upsample_rates'], frames, 0.0
    planes = 2 if split else 1
    for i, u in enumerate(rates):
        T *= u
        n_act = 2 * sum(len(d) for d in h['resblock_dilation_sizes']) + (1 if i == len(rates) - 1 else 0)
        total += n_act * T * cols[i + 1] * 2 * planes * 2
    return total

