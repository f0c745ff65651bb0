"""Float64 CPU restatement of the BigVGAN generator (NVIDIA/BigVGAN ``bigvgan.py``, Lee et al., ICLR 2023; inference only), built
op by op from its published layer list.  No checkpoint or code of that repository was available, so the state-dict keys and
shapes, the filter construction and the v2 final-layer flags below are pinned to that description, not to a downloaded file.

    conv_pre        Conv1d(num_mels -> C0, 7, padding 3)
    stage i         x = ups.i.0(x) (ConvTranspose1d(C0/2^i -> C0/2^(i+1), k_i, u_i, padding (k_i - u_i)/2); no activation
                    before it); x = (resblocks[i nk](x) + ... + resblocks[i nk + nk - 1](x)) / nk
    AMPBlock1       for each m: xt = activations[2m](x); xt = convs1.m(xt); xt = activations[2m + 1](xt); xt = convs2.m(xt);
                    x = xt + x   (convs1.m: kernel k, dilation d_m, padding d_m (k - 1) / 2; convs2.m: dilation 1)
    activation_post Activation1d, then conv_post Conv1d(C_last -> 1, 7, padding 3, bias = use_bias_at_final), then tanh
                    (use_tanh_at_final, the default) or clamp(-1, 1)

Activation1d is upsample -> act -> downsample:
    UpSample1d      F.pad(x, (5, 5), 'replicate'); 2 conv_transpose1d(x, filter, stride 2, groups C); [..., 15:-15]
    Snake(Beta)     x + 1 / (beta + 1e-9) sin^2(alpha x), alpha = exp(alpha) (and beta = exp(beta)) under snake_logscale;
                    Snake has no beta: 1 / (alpha + 1e-9)
    DownSample1d    lowpass: F.pad(x, (5, 6), 'replicate'); conv1d(x, filter, stride 2, groups C)
with both filters kaiser_sinc_filter1d(0.25, 0.3, 12), registered as buffers (so they are in the state dict).

Folded parameter counts (weights, biases, alpha and beta; the filter buffers are not parameters) at 80 mels with the v1
final layer: base 13,943,361 and bigvgan 112,199,473, the paper's 14 M and 112 M.

``init_state_dict(h, seed)`` draws a seeded state dict whose activations stay O(1) and whose waveform has a standard deviation
of about 0.1-0.3 on log-mels, as hifigan_oracle.py does.
"""
from __future__ import annotations

import math
import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.melgan_oracle import make_mels  # noqa: F401  (the same MelGAN-normalised log-mels, any n_mels)

HOP = 256
MAX_WAV_VALUE = 32768.0
_AMP = dict(resblock='1', resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
            activation='snakebeta', snake_logscale=True, num_mels=80)
CONFIGS = {
    'base': dict(_AMP, upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512),
    'bigvgan': dict(_AMP, upsample_rates=[4, 4, 2, 2, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4, 4, 4], upsample_initial_channel=1536),
}
N_PARAMS = {'base': 13_943_361, 'bigvgan': 112_199_473}   # after folding the weight norm, 80 mels, v1 final layer


def kaiser_sinc_filter1d(cutoff: float, half_width: float, kernel_size: int, dtype=torch.float64) -> torch.Tensor:
    """BigVGAN's Kaiser-windowed sinc low-pass, (1, 1, kernel_size), normalised to sum 1."""
    even = kernel_size % 2 == 0
    half_size = kernel_size // 2
    delta_f = 4 * half_width
    A = 2.285 * (half_size - 1) * math.pi * delta_f + 7.95
    if A > 50.0:
        beta = 0.1102 * (A - 8.7)
    elif A >= 21.0:
        beta = 0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0)
    else:
        beta = 0.0
    window = torch.kaiser_window(kernel_size, periodic=False, beta=beta, dtype=dtype)
    time = (torch.arange(-half_size, half_size, dtype=dtype) + 0.5) if even else (torch.arange(kernel_size, dtype=dtype) - half_size)
    if cutoff == 0:
        filt = torch.zeros_like(time)
    else:
        filt = 2 * cutoff * window * torch.sinc(2 * cutoff * time)
        filt = filt / filt.sum()
    return filt.view(1, 1, kernel_size)


def _wn(m: nn.Module) -> nn.Module:
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return torch.nn.utils.weight_norm(m)


def get_padding(k: int, d: int = 1) -> int:
    return d * (k - 1) // 2


class Snake(nn.Module):
    def __init__(self, ch: int, alpha_logscale: bool):
        super().__init__()
        self.alpha_logscale = alpha_logscale
        self.alpha = nn.Parameter(torch.zeros(ch) if alpha_logscale else torch.ones(ch))

    def forward(self, x):
        a = self.alpha[None, :, None]
        if self.alpha_logscale:
            a = torch.exp(a)
        return x + 1.0 / (a + 1e-9) * torch.pow(torch.sin(x * a), 2)


class SnakeBeta(nn.Module):
    def __init__(self, ch: int, alpha_logscale: bool):
        super().__init__()
        self.alpha_logscale = alpha_logscale
        self.alpha = nn.Parameter(torch.zeros(ch) if alpha_logscale else torch.ones(ch))
        self.beta = nn.Parameter(torch.zeros(ch) if alpha_logscale else torch.ones(ch))

    def forward(self, x):
        a, b = self.alpha[None, :, None], self.beta[None, :, None]
        if self.alpha_logscale:
            a, b = torch.exp(a), torch.exp(b)
        return x + 1.0 / (b + 1e-9) * torch.pow(torch.sin(x * a), 2)


class UpSample1d(nn.Module):
    def __init__(self, ratio: int = 2, kernel_size: int = 12):
        super().__init__()
        self.ratio, self.stride, self.kernel_size = ratio, ratio, kernel_size
        self.pad = kernel_size // ratio - 1
        self.pad_left = self.pad * self.stride + (kernel_size - self.stride) // 2
        self.pad_right = self.pad * self.stride + (kernel_size - self.stride + 1) // 2
        self.register_buffer('filter', kaiser_sinc_filter1d(0.5 / ratio, 0.6 / ratio, kernel_size))

    def forward(self, x):
        C = x.shape[1]
        x = F.pad(x, (self.pad, self.pad), mode='replicate')
        x = self.ratio * F.conv_transpose1d(x, self.filter.expand(C, -1, -1), stride=self.stride, groups=C)
        return x[..., self.pad_left:-self.pad_right]


class LowPassFilter1d(nn.Module):
    def __init__(self, cutoff: float = 0.5, half_width: float = 0.6, stride: int = 1, kernel_size: int = 12):
        super().__init__()
        even = kernel_size % 2 == 0
        self.pad_left = kernel_size // 2 - int(even)
        self.pad_right = kernel_size // 2
        self.stride = stride
        self.register_buffer('filter', kaiser_sinc_filter1d(cutoff, half_width, kernel_size))

    def forward(self, x):
        C = x.shape[1]
        x = F.pad(x, (self.pad_left, self.pad_right), mode='replicate')
        return F.conv1d(x, self.filter.expand(C, -1, -1), stride=self.stride, groups=C)


class DownSample1d(nn.Module):
    def __init__(self, ratio: int = 2, kernel_size: int = 12):
        super().__init__()
        self.lowpass = LowPassFilter1d(cutoff=0.5 / ratio, half_width=0.6 / ratio, stride=ratio, kernel_size=kernel_size)

    def forward(self, x):
        return self.lowpass(x)


class Activation1d(nn.Module):
    def __init__(self, activation: nn.Module):
        super().__init__()
        self.act = activation
        self.upsample = UpSample1d(2, 12)
        self.downsample = DownSample1d(2, 12)

    def forward(self, x):
        return self.downsample(self.act(self.upsample(x)))


def _act(h: dict, ch: int) -> nn.Module:
    cls = Snake if h['activation'] == 'snake' else SnakeBeta
    return Activation1d(cls(ch, alpha_logscale=bool(h['snake_logscale'])))


class AMPBlock1(nn.Module):
    def __init__(self, h: dict, ch: int, k: int, dilation):
        super().__init__()
        self.convs1 = nn.ModuleList([_wn(nn.Conv1d(ch, ch, k, 1, dilation=d, padding=get_padding(k, d))) for d in dilation])
        self.convs2 = nn.ModuleList([_wn(nn.Conv1d(ch, ch, k, 1, dilation=1, padding=get_padding(k, 1))) for _ in dilation])
        self.activations = nn.ModuleList([_act(h, ch) for _ in range(2 * len(dilation))])

    def forward(self, x):
        acts1, acts2 = self.activations[::2], self.activations[1::2]
        for c1, c2, a1, a2 in zip(self.convs1, self.convs2, acts1, acts2):
            xt = c2(a2(c1(a1(x))))
            x = xt + x
        return x


class Generator(nn.Module):
    def __init__(self, h: dict):
        super().__init__()
        self.num_kernels = len(h['resblock_kernel_sizes'])
        self.num_upsamples = len(h['upsample_rates'])
        c0 = h['upsample_initial_channel']
        self.conv_pre = _wn(nn.Conv1d(h['num_mels'], c0, 7, 1, padding=3))
        self.ups = nn.ModuleList([nn.ModuleList([_wn(nn.ConvTranspose1d(c0 // 2 ** i, c0 // 2 ** (i + 1), k, u, padding=(k - u) // 2))])
                                  for i, (u, k) in enumerate(zip(h['upsample_rates'], h['upsample_kernel_sizes']))])
        self.resblocks = nn.ModuleList()
        ch = c0
        for i in range(len(self.ups)):
            ch = c0 // 2 ** (i + 1)
            for k, d in zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes']):
                self.resblocks.append(AMPBlock1(h, ch, k, d))
        self.activation_post = _act(h, ch)
        self.use_bias_at_final = bool(h.get('use_bias_at_final', True))
        self.use_tanh_at_final = bool(h.get('use_tanh_at_final', True))
        self.conv_post = _wn(nn.Conv1d(ch, 1, 7, 1, padding=3, bias=self.use_bias_at_final))

    def forward(self, x):
        x = self.conv_pre(x)
        for i in range(self.num_upsamples):
            for up in self.ups[i]:
                x = up(x)
            xs = None
            for j in range(self.num_kernels):
                y = self.resblocks[i * self.num_kernels + j](x)
                xs = y if xs is None else xs + y
            x = xs / self.num_kernels
        x = self.conv_post(self.activation_post(x))
        return torch.tanh(x) if self.use_tanh_at_final else torch.clamp(x, min=-1.0, max=1.0)


def config(h, **overrides) -> dict:
    """A preset name ('base' | 'bigvgan') or a config dict -> the config dict, with `overrides` applied."""
    return dict(CONFIGS[h.lower()] if isinstance(h, str) else h, **overrides)


def build(h, state_dict=None, dtype=torch.float64) -> Generator:
    """Generator of config `h` in `dtype` on the CPU, loaded with `state_dict` (weight_g / weight_v form) when given."""
    g = Generator(config(h)).to(dtype)
    if state_dict is not None:
        g.load_state_dict(state_dict)
    return g.eval()


def n_params(h) -> int:
    """Parameters of the folded generator, counted from the layer list (weights, biases, alpha and beta)."""
    h = config(h)
    c0, ks = h["upsample_initial_channel"], h["resblock_kernel_sizes"]
    per_act = 2 if h['activation'] == 'snakebeta' else 1
    n = c0 * h['num_mels'] * 7 + c0
    ch = c0
    for i, k in enumerate(h['upsample_kernel_sizes']):
        cin, ch = c0 // 2 ** i, c0 // 2 ** (i + 1)
        n += cin * ch * k + ch
        for kk, dil in zip(ks, h['resblock_dilation_sizes']):
            n += 2 * len(dil) * (ch * ch * kk + ch) + 2 * len(dil) * per_act * ch
    n += per_act * ch + ch * 7 + (1 if h.get('use_bias_at_final', True) else 0)
    return n


def _gain(name: str, m: nn.Module) -> float:
    """Row-norm gain of each weight-normed conv: the residual streams keep a variance of about 1 and the waveform a std of
    about 0.2."""
    if name == 'conv_pre':
        return 0.25                       # log-mels are around -6: this brings the first activations to O(1)
    if name == 'conv_post':
        return 0.13
    if isinstance(m, nn.ConvTranspose1d):
        cin, cout, k = m.weight_v.shape
        return (cout * k / 2 / cin) ** 0.5
    if '.convs2.' in name:
        return 0.4                        # the branch added to the residual stream
    return 1.0


def init_state_dict(h, seed: int = 0) -> dict:
    """Seeded float64 state dict (weight_g / weight_v form, the published keys and filter buffers) with O(1) activations and a
    waveform std of about 0.1-0.3.  alpha and beta are drawn around their initial values (log scale: exp(+-0.5))."""
    h = config(h)
    gen = torch.Generator().manual_seed(seed)
    g = Generator(h).to(torch.float64)
    for name, m in g.named_modules():
        if isinstance(m, (nn.Conv1d, nn.ConvTranspose1d)):
            m.weight_v.data.copy_(torch.randn(m.weight_v.shape, generator=gen, dtype=torch.float64))
            m.weight_g.data.fill_(_gain(name, m))
            m.weight_g.data.mul_(1.0 + 0.1 * torch.randn(m.weight_g.shape, generator=gen, dtype=torch.float64))
            if m.bias is not None:
                m.bias.data.copy_(0.05 * torch.randn(m.bias.shape, generator=gen, dtype=torch.float64))
        elif isinstance(m, (Snake, SnakeBeta)):
            for p in ([m.alpha, m.beta] if isinstance(m, SnakeBeta) else [m.alpha]):
                r = 0.5 * torch.randn(p.shape, generator=gen, dtype=torch.float64)
                p.data.copy_(r if m.alpha_logscale else torch.exp(r))
    return {k: v.detach().clone() for k, v in g.state_dict().items()}
