"""Float64 CPU restatement of the MelGAN generator (seungwonpark/melgan, the vocoder the reference's synthesis notebook loads
with torch.hub), written from its published layer list; no checkpoint of that repository was available, so the state-dict
keys and shapes below are pinned to that specification, not to a downloaded file.

    forward(mel) = generator((mel + 5) / 5)            mel: (B, 80, T), MelGAN-normalised log-mel
    inference(mel): 10 frames of -11.5129 appended, forward, the last 2560 samples dropped, * 32768, clamped, .short()

``init_state_dict(seed)`` draws a seeded state dict whose activations stay O(1) and whose waveform has a standard deviation
of about 0.3 on log-mels (torch's default initialisation gives about 0.005, which would hide errors behind tiny values).
"""
from __future__ import annotations

import warnings

import torch
import torch.nn as nn

MAX_WAV_VALUE = 32768.0
HOP = 256
PAD_FRAMES = 10
PAD_VALUE = -11.5129
N_PARAMS = 4_266_050
N_TENSORS = 126


def _wn(m: nn.Module) -> nn.Module:
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return torch.nn.utils.weight_norm(m)


class ResStack(nn.Module):
    def __init__(self, channel: int):
        super().__init__()
        self.blocks = nn.ModuleList([
            nn.Sequential(nn.LeakyReLU(0.2), nn.ReflectionPad1d(3 ** i), _wn(nn.Conv1d(channel, channel, kernel_size=3, dilation=3 ** i)),
                          nn.LeakyReLU(0.2), _wn(nn.Conv1d(channel, channel, kernel_size=1)))
            for i in range(3)])
        self.shortcuts = nn.ModuleList([_wn(nn.Conv1d(channel, channel, kernel_size=1)) for _ in range(3)])

    def forward(self, x):
        for block, shortcut in zip(self.blocks, self.shortcuts):
            x = shortcut(x) + block(x)
        return x


class Generator(nn.Module):
    def __init__(self, mel_channel: int = 80):
        super().__init__()
        self.mel_channel = mel_channel
        self.generator = nn.Sequential(
            nn.ReflectionPad1d(3), _wn(nn.Conv1d(mel_channel, 512, kernel_size=7, stride=1)), nn.LeakyReLU(0.2),
            _wn(nn.ConvTranspose1d(512, 256, kernel_size=16, stride=8, padding=4)), ResStack(256), nn.LeakyReLU(0.2),
            _wn(nn.ConvTranspose1d(256, 128, kernel_size=16, stride=8, padding=4)), ResStack(128), nn.LeakyReLU(0.2),
            _wn(nn.ConvTranspose1d(128, 64, kernel_size=4, stride=2, padding=1)), ResStack(64), nn.LeakyReLU(0.2),
            _wn(nn.ConvTranspose1d(64, 32, kernel_size=4, stride=2, padding=1)), ResStack(32), nn.LeakyReLU(0.2),
            nn.ReflectionPad1d(3), _wn(nn.Conv1d(32, 1, kernel_size=7, stride=1)), nn.Tanh(),
        )

    def forward(self, mel):
        return self.generator((mel + 5.0) / 5.0)

    def inference(self, mel):
        if mel.ndim == 2:
            mel = mel.unsqueeze(0)
        pad = torch.full((1, self.mel_channel, PAD_FRAMES), PAD_VALUE, dtype=mel.dtype, device=mel.device)
        audio = self.forward(torch.cat((mel, pad), dim=2)).squeeze()
        audio = audio[:-(HOP * PAD_FRAMES)]
        audio = MAX_WAV_VALUE * audio
        return audio.clamp(min=-MAX_WAV_VALUE, max=MAX_WAV_VALUE - 1).short()


def build(state_dict=None, dtype=torch.float64) -> Generator:
    """Generator in `dtype` on the CPU, loaded with `state_dict` (weight_g / weight_v form) when given."""
    g = Generator().to(dtype)
    if state_dict is not None:
        g.load_state_dict(state_dict)
    return g.eval()


def _gains(name: str, module: nn.Module) -> float:
    """Row-norm gain of each weight-normed conv, chosen so that the residual stream keeps a variance of about 1."""
    if isinstance(module, nn.ConvTranspose1d):
        cin, cout, k = module.weight_v.shape
        return (cout * k / 2 / cin) ** 0.5 * 1.4     # per input channel: an output row sums cin * 2 of its k taps
    if name.endswith('.0') and 'shortcuts' in name:
        return 0.55
    if module.kernel_size[0] == 1:
        return 0.75
    if module.out_channels == 1:
        return 3.0
    return 1.4


def init_state_dict(seed: int = 0) -> dict:
    """Seeded float64 state dict (weight_g / weight_v form) with O(1) activations and a waveform std of about 0.3."""
    gen = torch.Generator().manual_seed(seed)
    g = Generator().to(torch.float64)
    for name, m in g.named_modules():
        if isinstance(m, (nn.Conv1d, nn.ConvTranspose1d)):
            v = torch.randn(m.weight_v.shape, generator=gen, dtype=torch.float64)
            m.weight_v.data.copy_(v)
            m.weight_g.data.fill_(_gains(name, m))
            m.weight_g.data.mul_(1.0 + 0.1 * torch.randn(m.weight_g.shape, generator=gen, dtype=torch.float64))
            m.bias.data.copy_(0.05 * torch.randn(m.bias.shape, generator=gen, dtype=torch.float64))
    return {k: v.detach().clone() for k, v in g.state_dict().items()}


def make_mels(counts, n_mels: int = 80, seed: int = 0):
    """Seeded speech-like MelGAN-normalised log-mels (n_mels, T_c): smooth in time and frequency, in [-11.5, 1.5]."""
    import numpy as np
    rng = np.random.default_rng(seed)
    out = []
    for T in counts:
        f = np.linspace(0, 1, n_mels)[:, None]
        t = np.arange(T)[None, :]
        base = -4.0 - 4.0 * f + 2.5 * np.sin(0.21 * t + 6 * f + rng.uniform(0, 6)) * np.exp(-2 * f)
        m = base + 0.6 * rng.standard_normal((n_mels, T))
        out.append(np.clip(m, -11.5129, 1.5).astype(np.float32))
    return out
