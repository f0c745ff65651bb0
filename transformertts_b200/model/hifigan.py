"""HiFi-GAN generator (jik876/hifi-gan, the V1 / V2 / V3 configs and any config of the same form) on the GPU, a packed ragged
batch of clips per call.

Every conv is one ``ttsb_conv1d_ex_tc`` launch over all clips (csrc/conv1d_tc.cu), on melgan.py's packed layout with
``halo`` rows on each side of every clip: the largest tap shift of the config (25 rows for V1 / V2, 36 for V3).  Every
HiFi-GAN conv pads with zeros, so the activation planes are zero-initialised and stored without halo writes: the halos stay
zero, and a clip of any length >= 1 frame works.  Per call: the split of the input mel, conv_pre, then per stage the
transposed conv (as melgan.py phrases it) and the resblock convs, then conv_post (``ttsb_conv1d_out_tanh_ex``).  The
epilogues apply LeakyReLU (0.1, and 0.01 before conv_post), the resblocks' identity residual and the multi-receptive-field
average: the last conv of resblock 0 writes an fp32 sum plane, the others add to it in torch's order, and the last add is
divided by the number of resblocks and written as the next stage's activation.

Channel counts below 64 are padded to 64 columns (the tensor-core k block), as in melgan.py.
"""
from __future__ import annotations

import json
from pathlib import Path
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from transformertts_b200 import lib
from transformertts_b200.model.melgan import (_Conv, _cols, conv_taps, fold_weight_norm, layout_rows, pack_clips, ragged_offsets,
                                              run_conv, transposed_taps)

HOP = 256
N_MELS = 80
MEL_COLS = 128            # conv_pre's 80 channels padded to two k blocks
MAX_WAV_VALUE = 32768.0
SLOPE = 0.1               # models.py's LRELU_SLOPE
POST_SLOPE = 0.01         # torch's default, before conv_post
CONFIG_KEYS = ('resblock', 'upsample_rates', 'upsample_kernel_sizes', 'upsample_initial_channel', 'resblock_kernel_sizes',
               'resblock_dilation_sizes')
PRESETS = {
    'v1': dict(resblock='1', upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512,
               resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]]),
    'v2': dict(resblock='1', upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=128,
               resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]]),
    'v3': dict(resblock='2', upsample_rates=[8, 8, 4], upsample_kernel_sizes=[16, 16, 8], upsample_initial_channel=256,
               resblock_kernel_sizes=[3, 5, 7], resblock_dilation_sizes=[[1, 2], [2, 6], [3, 12]]),
}


def load_config(config) -> dict:
    """A preset name ('v1' | 'v2' | 'v3'), the path of a jik876 config.json, or a dict -> the checked config (the generator's
    keys only)."""
    if isinstance(config, (str, Path)) and str(config).lower() in PRESETS:
        h = dict(PRESETS[str(config).lower()])
    elif isinstance(config, (str, Path)):
        with open(config, 'r') as f:
            h = json.load(f)
    elif isinstance(config, dict):
        h = dict(config)
    else:
        raise TypeError(f'config must be a preset name, a path or a dict, got {type(config).__name__}')
    missing = [k for k in CONFIG_KEYS if k not in h]
    if missing:
        raise ValueError(f'HiFi-GAN config: missing key {missing[0]}')
    h = {k: h[k] for k in CONFIG_KEYS}
    h['resblock'] = str(h['resblock'])
    check_config(h)
    return h


def check_config(h: dict):
    """Refuses a config this implementation does not run (ValueError naming the reason)."""
    if h['resblock'] not in ('1', '2'):
        raise ValueError(f"HiFi-GAN config: resblock must be '1' or '2', got {h['resblock']!r}")
    rates, kernels = list(h['upsample_rates']), list(h['upsample_kernel_sizes'])
    if not rates or len(rates) != len(kernels):
        raise ValueError('HiFi-GAN config: upsample_rates and upsample_kernel_sizes must be non-empty and of equal length')
    if int(np.prod(rates)) != HOP:
        raise ValueError(f'HiFi-GAN config: the upsample rates multiply to {int(np.prod(rates))}, not the hop of {HOP}')
    for u, k in zip(rates, kernels):
        if u % 2 or k != 2 * u:
            raise ValueError(f'HiFi-GAN config: upsample kernel {k} with rate {u}; only kernel = 2 rate with an even rate is supported')
    ks, ds = list(h['resblock_kernel_sizes']), list(h['resblock_dilation_sizes'])
    if not ks or len(ks) != len(ds):
        raise ValueError('HiFi-GAN config: resblock_kernel_sizes and resblock_dilation_sizes must be non-empty and of equal length')
    n_dil = 3 if h['resblock'] == '1' else 2    # models.py's ResBlock1 / ResBlock2 use that many dilations
    for k, d in zip(ks, ds):
        if k % 2 == 0 or k < 1 or k > lib.CONV1D_EX_MAX_TAPS:
            raise ValueError(f'HiFi-GAN config: resblock kernel {k} must be odd and at most {lib.CONV1D_EX_MAX_TAPS}')
        if len(d) != n_dil or min(d) < 1:
            raise ValueError(f"HiFi-GAN config: resblock {h['resblock']} takes {n_dil} dilations >= 1, got {list(d)}")
    if halo_rows(h) > lib.CONV1D_EX_MAX_HALO:
        raise ValueError(f'HiFi-GAN config: a tap shift of {halo_rows(h)} rows exceeds {lib.CONV1D_EX_MAX_HALO}')
    c0 = h['upsample_initial_channel']
    for i in range(len(rates) + 1):
        c = c0 // 2 ** i
        if c < 1 or c * 2 ** i != c0 or (c > 64 and c % 64):
            raise ValueError(f'HiFi-GAN config: stage {i} has {c0} / 2^{i} channels; each must be an integer, <= 64 or a multiple of 64')
        if i > 0:
            n = rates[i - 1] * _cols(c)
            if n > 256 and n % 256:
                raise ValueError(f'HiFi-GAN config: upsample {i - 1} gives {n} columns, neither <= 256 nor a multiple of 256')
    if c0 // 2 ** len(rates) > 256:
        raise ValueError('HiFi-GAN config: conv_post takes at most 256 channels')


def halo_rows(h: dict) -> int:
    """Halo rows of the packed layout: the largest tap shift of any conv (conv_pre / conv_post: 3)."""
    return max([3] + [d * (k - 1) // 2 for k, ds in zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes']) for d in ds])


def _resblock_convs(h: dict, n: int, dil) -> List[tuple]:
    """[(name, dilation)] of resblock n, in execution order."""
    if h['resblock'] == '1':
        return [c for m, d in enumerate(dil) for c in ((f'resblocks.{n}.convs1.{m}', d), (f'resblocks.{n}.convs2.{m}', 1))]
    return [(f'resblocks.{n}.convs.{m}', d) for m, d in enumerate(dil)]


def layer_shapes(h: dict) -> Dict[str, tuple]:
    """conv name -> (kind, weight shape): kind 'conv' (Cout, Cin, k) or 'convT' (Cin, Cout, k)."""
    c0, nk = h['upsample_initial_channel'], len(h['resblock_kernel_sizes'])
    out = {'conv_pre': ('conv', (c0, N_MELS, 7))}
    for i, k in enumerate(h['upsample_kernel_sizes']):
        out[f'ups.{i}'] = ('convT', (c0 // 2 ** i, c0 // 2 ** (i + 1), k))
    for i in range(len(h['upsample_rates'])):
        ch = c0 // 2 ** (i + 1)
        for j, (k, dil) in enumerate(zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes'])):
            for name, _ in _resblock_convs(h, i * nk + j, dil):
                out[name] = ('conv', (ch, ch, k))
    out['conv_post'] = ('conv', (1, c0 // 2 ** len(h['upsample_rates']), 7))
    return out


def expected_keys(h: dict, weight_norm: bool = True) -> Dict[str, tuple]:
    """The checkpoint's state-dict keys and shapes (weight_g / weight_v form, or the plain `weight` remove_weight_norm leaves)."""
    keys = {}
    for name, (kind, shape) in layer_shapes(h).items():
        keys[f'{name}.bias'] = (shape[1] if kind == 'convT' else shape[0],)
        if weight_norm:
            keys[f'{name}.weight_g'] = (shape[0], 1, 1)
            keys[f'{name}.weight_v'] = shape
        else:
            keys[f'{name}.weight'] = shape
    return keys


def launches_per_call(h: dict) -> int:
    """Library launches of one vocode call: the mel split, conv_pre, per stage the transposed conv and every resblock conv,
    conv_post."""
    per_block = 6 if h['resblock'] == '1' else 2
    return 3 + len(h['upsample_rates']) * (1 + per_block * len(h['resblock_kernel_sizes']))


def _padded(b: np.ndarray, cols: int, reps: int = 1) -> np.ndarray:
    out = np.zeros(reps * cols)
    for r in range(reps):
        out[r * cols:r * cols + len(b)] = b
    return out


class HiFiGANGenerator:
    """The HiFi-GAN generator of jik876/hifi-gan, vocoding ragged batches on the GPU.

    config: a preset name ('v1' | 'v2' | 'v3'), the path of its config.json or a dict.
    precision: 'bf16x3' (hi/lo split operands, fp32-class products) or 'bf16' (one bf16 product per conv)."""

    def __init__(self, config='v1', device=None, precision: str = 'bf16x3'):
        if precision not in ('bf16x3', 'bf16'):
            raise ValueError(f"precision must be 'bf16x3' or 'bf16', got {precision!r}")
        self.h = load_config(config)
        self.halo = halo_rows(self.h)
        self.device = torch.device(device if device is not None else 'cuda')
        self.precision = precision
        self.split = precision == 'bf16x3'
        self._convs: Optional[dict] = None

    # ---------------------------------------------------------------------------------------------------- loading
    @classmethod
    def from_checkpoint(cls, path, config=None, device=None, precision: str = 'bf16x3') -> 'HiFiGANGenerator':
        """config None: the config.json beside the checkpoint, as jik876's inference.py reads it."""
        if config is None:
            config = Path(path).parent / 'config.json'
            if not config.exists():
                raise FileNotFoundError(f'{config} not found: pass the generator config (a config.json path or v1 / v2 / v3)')
        g = cls(config=config, device=device, precision=precision)
        g.load_state_dict(torch.load(path, map_location='cpu', weights_only=True))
        return g

    def fold_state_dict(self, sd) -> Dict[str, np.ndarray]:
        """Checks a checkpoint (``{'generator': sd}`` or a bare state dict, weight-normed or folded) against the config and
        returns {conv name: float64 weight, conv name + '.bias': float64 bias}."""
        if isinstance(sd, dict) and 'generator' in sd:
            sd = sd['generator']
        if not isinstance(sd, dict):
            raise TypeError(f'expected a state dict, got {type(sd).__name__}')
        keys = set(sd)
        normed, plain = expected_keys(self.h, True), expected_keys(self.h, False)
        want = normed if any(k.endswith('.weight_g') or k.endswith('.weight_v') for k in keys) else plain
        missing = sorted(set(want) - keys)
        if missing:
            raise KeyError(f'HiFi-GAN checkpoint: missing key {missing[0]}' + (f' (and {len(missing) - 1} more)' if len(missing) > 1 else ''))
        extra = sorted(keys - set(want))
        if extra:
            raise KeyError(f'HiFi-GAN checkpoint: unexpected key {extra[0]}' + (f' (and {len(extra) - 1} more)' if len(extra) > 1 else ''))
        for k, shape in want.items():
            if tuple(sd[k].shape) != tuple(shape):
                raise ValueError(f'HiFi-GAN checkpoint: {k} has shape {tuple(sd[k].shape)}, expected {tuple(shape)}')
        f64 = {k: sd[k].detach().cpu().double().numpy() for k in want}
        out = {}
        for name in layer_shapes(self.h):
            out[name] = fold_weight_norm(f64[f'{name}.weight_g'], f64[f'{name}.weight_v']) if want is normed else f64[f'{name}.weight']
            out[name + '.bias'] = f64[f'{name}.bias']
        return out

    def load_state_dict(self, sd) -> 'HiFiGANGenerator':
        w = self.fold_state_dict(sd)
        h, dev, split = self.h, self.device, self.split
        c0, nk = h['upsample_initial_channel'], len(h['resblock_kernel_sizes'])
        convs = {}
        with torch.cuda.device(dev):
            cc = _cols(c0)
            convs['conv_pre'] = _Conv(conv_taps(w['conv_pre'], 1, MEL_COLS, cc), _padded(w['conv_pre.bias'], cc),
                                      [(0, s) for s in range(-3, 4)], split, dev)
            for i, u in enumerate(h['upsample_rates']):
                ci, cc = _cols(c0 // 2 ** i), _cols(c0 // 2 ** (i + 1))
                convs[f'ups.{i}'] = _Conv(transposed_taps(w[f'ups.{i}'], u, ci, cc), _padded(w[f'ups.{i}.bias'], cc, u),
                                          [(0, -1), (0, 0), (0, 1)], split, dev)
                for j, (k, dil) in enumerate(zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes'])):
                    for name, d in _resblock_convs(h, i * nk + j, dil):
                        convs[name] = _Conv(conv_taps(w[name], d, cc, cc), _padded(w[name + '.bias'], cc),
                                            [(0, (s - (k - 1) // 2) * d) for s in range(k)], split, dev)
            self._post_w = torch.from_numpy(np.ascontiguousarray(w['conv_post'][0].T, dtype=np.float32)).to(dev)   # (7, C_last)
            self._post_b = float(w['conv_post.bias'][0])
        self._convs = convs
        return self

    # ---------------------------------------------------------------------------------------------------- forward
    def _planes(self, rows: int, cols: int):
        """Zeroed hi (and lo) planes: halo rows are never written, so they keep the zero padding."""
        hi = torch.zeros((rows, cols), dtype=torch.bfloat16, device=self.device)
        return hi, (torch.zeros_like(hi) if self.split else None)

    def _run(self, name, counts, src, up=1, **kw):
        run_conv(self._convs[name], counts, [src], up, self.split, rows_halo=self.halo, **kw)

    def vocode_device(self, mels: Sequence[np.ndarray]) -> torch.Tensor:
        """vocode_batch, leaving the packed float32 waveform (256 sum T_c samples, clip after clip) on the device."""
        if self._convs is None:
            raise RuntimeError('HiFiGANGenerator: no weights loaded (from_checkpoint / load_state_dict)')
        ms = [np.asarray(m, dtype=np.float32) for m in mels]
        if not ms:
            raise ValueError('vocode_batch: no mels')
        for c, m in enumerate(ms):
            if m.ndim != 2 or m.shape[0] != N_MELS or m.shape[1] < 1:
                raise ValueError(f'mel {c} has shape {m.shape}; the vocoder needs ({N_MELS}, T) with T >= 1 frames')
        h, H = self.h, self.halo
        c0, nk = h['upsample_initial_channel'], len(h['resblock_kernel_sizes'])
        counts = [m.shape[1] for m in ms]
        x = pack_clips([m.T for m in ms], MEL_COLS, lib.HALO_ZERO, halo=H)
        with torch.cuda.device(self.device):
            ws = torch.empty(lib.conv1d_workspace_bytes(len(ms)), dtype=torch.uint8, device=self.device)
            src = lib.split_bf16(torch.from_numpy(x).to(self.device), self.split)
            act = self._planes(layout_rows(counts, halo=H), _cols(c0))
            self._run('conv_pre', counts, src, act=act, slope=SLOPE, ws=ws)
            n_stages = len(h['upsample_rates'])
            for i, u in enumerate(h['upsample_rates']):
                counts_in, counts = counts, [c * u for c in counts]
                rows, cc = layout_rows(counts, halo=H), _cols(c0 // 2 ** (i + 1))
                x_st, a_st = self._planes(rows, cc), self._planes(rows, cc)
                self._run(f'ups.{i}', counts_in, act, u, out=x_st, act=a_st, slope=SLOPE, ws=ws)
                t, pair = self._planes(rows, cc), [(self._planes(rows, cc), self._planes(rows, cc)) for _ in range(2)]
                act = self._planes(rows, cc)        # the stage's output: LeakyReLU of the resblock average
                total = torch.empty((rows, cc), dtype=torch.float32, device=self.device) if nk > 1 else None
                final_slope = SLOPE if i < n_stages - 1 else POST_SLOPE
                for j, dil in enumerate(h['resblock_dilation_sizes']):
                    names = _resblock_convs(h, i * nk + j, dil)
                    xin, ain = x_st, a_st
                    step = 2 if h['resblock'] == '1' else 1
                    for m in range(0, len(names), step):
                        if step == 2:                        # ResBlock1: xt = c1(lrelu(x)) into t, then c2 reads lrelu(xt)
                            self._run(names[m][0], counts, ain, act=t, slope=SLOPE, ws=ws)
                            branch = t
                        else:
                            branch = ain
                        name = names[m + step - 1][0]
                        if m + step < len(names):            # x = branch conv + x, kept for the next pair
                            nxt = pair[(m // step) % 2]
                            self._run(name, counts, branch, res=xin, out=nxt[0], act=nxt[1], slope=SLOPE, ws=ws)
                            xin, ain = nxt
                        elif nk == 1:
                            self._run(name, counts, branch, res=xin, act=act, slope=final_slope, ws=ws)
                        else:                                # the resblock's output goes to the sum
                            mode = lib.SUM_WRITE if j == 0 else (lib.SUM_FINISH if j == nk - 1 else lib.SUM_ADD)
                            fin = mode == lib.SUM_FINISH
                            self._run(name, counts, branch, res=xin, sum_plane=total, sum_mode=mode, sum_div=float(nk),
                                      act=act if fin else None, slope=final_slope, ws=ws)
                del x_st, a_st, t, pair, total
            wav = torch.empty(HOP * sum(m.shape[1] for m in ms), dtype=torch.float32, device=self.device)
            lib.conv1d_out_tanh_ex(act[0], act[1], c0 // 2 ** n_stages, H, ragged_offsets(counts), 0, self._post_w, self._post_b, ws, wav)
        return wav

    def vocode_batch(self, mels: Sequence[np.ndarray]) -> List[np.ndarray]:
        """Log-mels (80, T_c) (the MelGAN normaliser's ln(max(S, 1e-5))) -> float32 waveforms of 256 T_c samples: what the
        generator computes per clip, before inference.py's int16 conversion."""
        wav = self.vocode_device(mels).cpu().numpy()
        off = ragged_offsets([np.asarray(m).shape[1] for m in mels], HOP)
        return [wav[off[c]:off[c + 1]] for c in range(len(mels))]

    def inference(self, mel) -> torch.Tensor:
        """jik876's inference.py for one (1, 80, T) or (80, T) mel: (wav * 32768).astype(int16), 256 T samples on the CPU."""
        m = torch.as_tensor(mel).detach().cpu().float()
        if m.ndim == 3:
            if m.shape[0] != 1:
                raise ValueError(f'inference takes one mel, got a batch of {m.shape[0]}')
            m = m[0]
        wav = self.vocode_batch([m.numpy()])[0]
        return torch.from_numpy((wav * np.float32(MAX_WAV_VALUE)).astype(np.int16))
