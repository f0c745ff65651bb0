"""Float64 CPU restatement of the HiFi-GAN generator (jik876/hifi-gan ``models.py``, inference only), written from its published
layer list; no checkpoint of that repository was available, so the state-dict keys and shapes below are pinned to that
specification, not to a downloaded file.  Folded parameter counts: V1 13,926,017, V2 925,985, V3 1,462,273 (the paper's
13.92 M, 0.92 M and 1.46 M).

    conv_pre  Conv1d(80 -> C0, 7, padding 3)
    stage i   x = leaky_relu(x, 0.1); x = ups.i(x) (ConvTranspose1d(C0/2^i -> C0/2^(i+1), k_i, u_i, padding (k_i - u_i)/2));
              x = (resblocks[i nk](x) + ... + resblocks[i nk + nk - 1](x)) / nk
    ResBlock1 for each m: xt = convs2.m(leaky_relu(convs1.m(leaky_relu(x, 0.1)), 0.1)); x = xt + x
              (convs1.m: kernel k, dilation d_m, padding d_m (k - 1) / 2; convs2.m: kernel k, dilation 1, padding (k - 1) / 2)
    ResBlock2 for each m: x = convs.m(leaky_relu(x, 0.1)) + x
    conv_post leaky_relu(x) (slope 0.01), Conv1d(C_last -> 1, 7, padding 3), tanh

The input is the log-mel ``ln(max(S, 1e-5))`` (the project's MelGAN normaliser); T frames give 256 T samples with no pad
frames, and jik876's ``inference.py`` converts with ``(wav * 32768).astype(int16)``.

``init_state_dict(config, seed)`` draws a seeded state dict whose activations stay O(1) and whose waveform has a standard
deviation of about 0.1-0.3 on log-mels (torch's default initialisation would hide errors behind tiny values).
"""
from __future__ import annotations

import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.melgan_oracle import make_mels  # noqa: F401  (the same MelGAN-normalised log-mels)

LRELU_SLOPE = 0.1
MAX_WAV_VALUE = 32768.0
HOP = 256
N_MELS = 80

CONFIGS = {
    'v1': dict(resblock='1', upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512,
               resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]]),
    'v2': dict(resblock='1', upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=128,
               resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]]),
    'v3': dict(resblock='2', upsample_rates=[8, 8, 4], upsample_kernel_sizes=[16, 16, 8], upsample_initial_channel=256,
               resblock_kernel_sizes=[3, 5, 7], resblock_dilation_sizes=[[1, 2], [2, 6], [3, 12]]),
}
N_PARAMS = {'v1': 13_926_017, 'v2': 925_985, 'v3': 1_462_273}   # after folding the weight norm


def _wn(m: nn.Module) -> nn.Module:
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return torch.nn.utils.weight_norm(m)


def get_padding(k: int, d: int = 1) -> int:
    return d * (k - 1) // 2


class ResBlock1(nn.Module):
    def __init__(self, ch: int, k: int, dilation):
        super().__init__()
        self.convs1 = nn.ModuleList([_wn(nn.Conv1d(ch, ch, k, 1, dilation=d, padding=get_padding(k, d))) for d in dilation])
        self.convs2 = nn.ModuleList([_wn(nn.Conv1d(ch, ch, k, 1, dilation=1, padding=get_padding(k, 1))) for _ in dilation])

    def forward(self, x):
        for c1, c2 in zip(self.convs1, self.convs2):
            xt = c2(F.leaky_relu(c1(F.leaky_relu(x, LRELU_SLOPE)), LRELU_SLOPE))
            x = xt + x
        return x


class ResBlock2(nn.Module):
    def __init__(self, ch: int, k: int, dilation):
        super().__init__()
        self.convs = nn.ModuleList([_wn(nn.Conv1d(ch, ch, k, 1, dilation=d, padding=get_padding(k, d))) for d in dilation])

    def forward(self, x):
        for c in self.convs:
            x = c(F.leaky_relu(x, LRELU_SLOPE)) + x
        return x


class Generator(nn.Module):
    def __init__(self, h: dict):
        super().__init__()
        self.num_kernels = len(h['resblock_kernel_sizes'])
        self.num_upsamples = len(h['upsample_rates'])
        c0 = h['upsample_initial_channel']
        self.conv_pre = _wn(nn.Conv1d(N_MELS, c0, 7, 1, padding=3))
        block = ResBlock1 if str(h['resblock']) == '1' else ResBlock2
        self.ups = nn.ModuleList([_wn(nn.ConvTranspose1d(c0 // 2 ** i, c0 // 2 ** (i + 1), k, u, padding=(k - u) // 2))
                                  for i, (u, k) in enumerate(zip(h['upsample_rates'], h['upsample_kernel_sizes']))])
        self.resblocks = nn.ModuleList()
        ch = c0
        for i in range(len(self.ups)):
            ch = c0 // 2 ** (i + 1)
            for k, d in zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes']):
                self.resblocks.append(block(ch, k, d))
        self.conv_post = _wn(nn.Conv1d(ch, 1, 7, 1, padding=3))

    def forward(self, x):
        x = self.conv_pre(x)
        for i in range(self.num_upsamples):
            x = self.ups[i](F.leaky_relu(x, LRELU_SLOPE))
            xs = None
            for j in range(self.num_kernels):
                y = self.resblocks[i * self.num_kernels + j](x)
                xs = y if xs is None else xs + y
            x = xs / self.num_kernels
        return torch.tanh(self.conv_post(F.leaky_relu(x)))


def config(h) -> dict:
    """A preset name ('v1' | 'v2' | 'v3') or a config dict -> the config dict."""
    return dict(CONFIGS[h.lower()]) if isinstance(h, str) else dict(h)


def build(h, state_dict=None, dtype=torch.float64) -> Generator:
    """Generator of config `h` in `dtype` on the CPU, loaded with `state_dict` (weight_g / weight_v form) when given."""
    g = Generator(config(h)).to(dtype)
    if state_dict is not None:
        g.load_state_dict(state_dict)
    return g.eval()


def inference(g: Generator, mel):
    """jik876's inference.py for one (80, T) mel: the int16 waveform of 256 T samples."""
    with torch.no_grad():
        y = g(torch.as_tensor(mel, dtype=next(g.parameters()).dtype)[None]).squeeze()
    return (y * MAX_WAV_VALUE).numpy().astype('int16')


def _gain(name: str, m: nn.Module, h: dict) -> float:
    """Row-norm gain of each weight-normed conv: the residual streams keep a variance of about 1 and the waveform a std of
    about 0.2."""
    if name == 'conv_pre':
        return 0.25                       # log-mels are around -6: this brings the first activations to O(1)
    if name == 'conv_post':
        return 0.3
    if isinstance(m, nn.ConvTranspose1d):
        cin, cout, k = m.weight_v.shape
        return (cout * k / 2 / cin) ** 0.5 * 1.4     # per input channel: an output row sums cin * 2 of its k taps
    if '.convs2.' in name or str(h['resblock']) == '2':
        return 0.6                        # the branch added to the residual stream
    return 1.4


def init_state_dict(h, seed: int = 0) -> dict:
    """Seeded float64 state dict (weight_g / weight_v form) with O(1) activations and a waveform std of about 0.1-0.3."""
    h = config(h)
    gen = torch.Generator().manual_seed(seed)
    g = Generator(h).to(torch.float64)
    for name, m in g.named_modules():
        if isinstance(m, (nn.Conv1d, nn.ConvTranspose1d)):
            m.weight_v.data.copy_(torch.randn(m.weight_v.shape, generator=gen, dtype=torch.float64))
            m.weight_g.data.fill_(_gain(name, m, h))
            m.weight_g.data.mul_(1.0 + 0.1 * torch.randn(m.weight_g.shape, generator=gen, dtype=torch.float64))
            m.bias.data.copy_(0.05 * torch.randn(m.bias.shape, generator=gen, dtype=torch.float64))
    return {k: v.detach().clone() for k, v in g.state_dict().items()}
