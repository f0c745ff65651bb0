"""Float64 torch restatement of fatchord/WaveRNN's generator: ``models/fatchord_version.py`` (MelResNet, Stretch2d,
UpsampleNetwork, WaveRNN.generate, fold_with_overlap, xfade_and_unfold), ``utils/distribution.py``
(sample_from_discretized_mix_logistic), ``utils/dsp.py`` (decode_mu_law) and the generation defaults of ``hparams.py``,
written from the published code; no checkpoint of that repository was available, so the state-dict keys and shapes below
are pinned to that code, not to a downloaded file.

Two deliberate differences from the published code, both about where randomness comes from:
  * every uniform is drawn from ``uniform(seed, fold, step, draw)``, a stateless counter-based generator that the GPU kernel
    (csrc/wavernn.cu) computes bit for bit, instead of torch's global RNG.  MOL draws 11 per step (10 Gumbel, 1 logistic),
    RAW one.
  * RAW's categorical draw is the inverse CDF of that one uniform: the first class whose cumulative probability exceeds it.

``replay`` runs the recurrence teacher-forced on given samples (the GPU's), so that logits and draws can be compared step by
step without the chaos of a free-running sampler.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

# hparams.py: voc_* generation defaults and the WaveRNN audio section
HOP = 275
UPSAMPLE_FACTORS = (5, 5, 11)
RNN_DIMS = FC_DIMS = 512
COMPUTE_DIMS = RES_OUT_DIMS = 128
RES_BLOCKS = 10
PAD = 2
FEAT_DIMS = 80
BITS = 9
TARGET = 11_000
OVERLAP = 550
MIN_FRAMES = 21                 # generate()'s 20-hop fade-out needs (T - 1) hop >= 20 hop
LOG_SCALE_MIN = math.log(1e-14)
N_PARAMS_MOL = 4_233_675        # trainable parameters at the defaults, MOL
N_PARAMS_RAW9 = 4_480_941       # the same with 9-bit RAW


# ------------------------------------------------------------------------------------------------------------ the model
class ResBlock(nn.Module):
    def __init__(self, dims):
        super().__init__()
        self.conv1 = nn.Conv1d(dims, dims, kernel_size=1, bias=False)
        self.conv2 = nn.Conv1d(dims, dims, kernel_size=1, bias=False)
        self.batch_norm1 = nn.BatchNorm1d(dims)
        self.batch_norm2 = nn.BatchNorm1d(dims)

    def forward(self, x):
        residual = x
        x = F.relu(self.batch_norm1(self.conv1(x)))
        x = self.batch_norm2(self.conv2(x))
        return x + residual


class MelResNet(nn.Module):
    def __init__(self, res_blocks, in_dims, compute_dims, res_out_dims, pad):
        super().__init__()
        k_size = pad * 2 + 1
        self.conv_in = nn.Conv1d(in_dims, compute_dims, kernel_size=k_size, bias=False)
        self.batch_norm = nn.BatchNorm1d(compute_dims)
        self.layers = nn.ModuleList([ResBlock(compute_dims) for _ in range(res_blocks)])
        self.conv_out = nn.Conv1d(compute_dims, res_out_dims, kernel_size=1)

    def forward(self, x):
        x = F.relu(self.batch_norm(self.conv_in(x)))
        for f in self.layers:
            x = f(x)
        return self.conv_out(x)


class Stretch2d(nn.Module):
    def __init__(self, x_scale, y_scale):
        super().__init__()
        self.x_scale, self.y_scale = x_scale, y_scale

    def forward(self, x):
        b, c, h, w = x.size()
        x = x.unsqueeze(-1).unsqueeze(3)
        x = x.repeat(1, 1, 1, self.y_scale, 1, self.x_scale)
        return x.view(b, c, h * self.y_scale, w * self.x_scale)


class UpsampleNetwork(nn.Module):
    def __init__(self, feat_dims, upsample_scales, compute_dims, res_blocks, res_out_dims, pad):
        super().__init__()
        total_scale = int(np.prod(upsample_scales))
        self.indent = pad * total_scale
        self.resnet = MelResNet(res_blocks, feat_dims, compute_dims, res_out_dims, pad)
        self.resnet_stretch = Stretch2d(total_scale, 1)
        self.up_layers = nn.ModuleList()
        for scale in upsample_scales:
            k_size = (1, scale * 2 + 1)
            conv = nn.Conv2d(1, 1, kernel_size=k_size, padding=(0, scale), bias=False)
            conv.weight.data.fill_(1. / k_size[1])
            self.up_layers.append(Stretch2d(scale, 1))
            self.up_layers.append(conv)

    def forward(self, m):
        aux = self.resnet(m).unsqueeze(1)
        aux = self.resnet_stretch(aux).squeeze(1)
        m = m.unsqueeze(1)
        for f in self.up_layers:
            m = f(m)
        m = m.squeeze(1)[:, :, self.indent:-self.indent]
        return m.transpose(1, 2), aux.transpose(1, 2)


class WaveRNN(nn.Module):
    def __init__(self, rnn_dims=RNN_DIMS, fc_dims=FC_DIMS, bits=BITS, pad=PAD, upsample_factors=UPSAMPLE_FACTORS,
                 feat_dims=FEAT_DIMS, compute_dims=COMPUTE_DIMS, res_out_dims=RES_OUT_DIMS, res_blocks=RES_BLOCKS,
                 hop_length=HOP, mode='MOL'):
        super().__init__()
        self.mode = mode
        self.pad = pad
        self.n_classes = 2 ** bits if mode == 'RAW' else 30
        self.rnn_dims = rnn_dims
        self.aux_dims = res_out_dims // 4
        self.hop_length = hop_length
        self.upsample = UpsampleNetwork(feat_dims, upsample_factors, compute_dims, res_blocks, res_out_dims, pad)
        self.I = nn.Linear(feat_dims + self.aux_dims + 1, rnn_dims)
        self.rnn1 = nn.GRU(rnn_dims, rnn_dims, batch_first=True)
        self.rnn2 = nn.GRU(rnn_dims + self.aux_dims, rnn_dims, batch_first=True)
        self.fc1 = nn.Linear(rnn_dims + self.aux_dims, fc_dims)
        self.fc2 = nn.Linear(fc_dims + self.aux_dims, fc_dims)
        self.fc3 = nn.Linear(fc_dims, self.n_classes)
        self.step = nn.Parameter(torch.zeros(1).long(), requires_grad=False)

    def num_params(self):
        return sum(p.numel() for p in self.parameters() if p.requires_grad)

    def conditioning(self, mel):
        """(1, 80, T) fatchord-space mel -> m_up (T hop, 80), aux (T hop, res_out_dims): generate()'s upsampling."""
        mels = F.pad(mel.transpose(1, 2), (0, 0, self.pad, self.pad)).transpose(1, 2)   # pad_tensor(side='both')
        m_up, aux = self.upsample(mels)
        return m_up[0], aux[0]

    def _cells(self):
        c1 = nn.GRUCell(self.rnn1.input_size, self.rnn_dims).to(self.fc3.weight)
        c2 = nn.GRUCell(self.rnn2.input_size, self.rnn_dims).to(self.fc3.weight)
        for cell, gru in ((c1, self.rnn1), (c2, self.rnn2)):
            cell.weight_ih.data, cell.weight_hh.data = gru.weight_ih_l0.data, gru.weight_hh_l0.data
            cell.bias_ih.data, cell.bias_hh.data = gru.bias_ih_l0.data, gru.bias_hh_l0.data
        return c1, c2

    def step_logits(self, cells, x, m_t, a_t, h1, h2):
        """One step of generate()'s loop for a batch of rows -> (logits, h1, h2)."""
        a1, a2, a3, a4 = torch.split(a_t, self.aux_dims, dim=1)
        x = self.I(torch.cat([x, m_t, a1], dim=1))
        h1 = cells[0](x, h1)
        x = x + h1
        h2 = cells[1](torch.cat([x, a2], dim=1), h2)
        x = x + h2
        x = F.relu(self.fc1(torch.cat([x, a3], dim=1)))
        x = F.relu(self.fc2(torch.cat([x, a4], dim=1)))
        return self.fc3(x), h1, h2

    @torch.no_grad()
    def generate(self, mels, batched=True, target=TARGET, overlap=OVERLAP, seed=0):
        """fatchord's generate(mels (1, 80, T), save_path=None, batched, target, overlap, mu_law=hp.mu_law) with the uniforms
        of ``uniform(seed, fold, step, draw)`` -> float64 numpy waveform of (T - 1) hop samples."""
        wave_len = (mels.size(-1) - 1) * self.hop_length
        m_up, aux = self.conditioning(mels)
        m_up, aux = m_up[None], aux[None]
        if batched:
            m_up = fold_with_overlap(m_up, target, overlap)
            aux = fold_with_overlap(aux, target, overlap)
        b, L, _ = m_up.shape
        cells = self._cells()
        dev, dt = self.fc3.weight.device, self.fc3.weight.dtype
        h1 = torch.zeros(b, self.rnn_dims, device=dev, dtype=dt)
        h2 = torch.zeros_like(h1)
        x = torch.zeros(b, 1, device=dev, dtype=dt)
        out = []
        for i in range(L):
            logits, h1, h2 = self.step_logits(cells, x, m_up[:, i], aux[:, i], h1, h2)
            u = uniforms(seed, np.arange(b), i, 11 if self.mode == 'MOL' else 1)
            s = np.array([self.sample(lg, uu)[0] for lg, uu in zip(logits.cpu().numpy(), u)])
            out.append(s)
            x = torch.from_numpy(s).to(dev, dt)[:, None]
        output = np.stack(out, 1).astype(np.float64)
        if self.mode == 'RAW':
            output = decode_mu_law(output, self.n_classes, False)
        output = xfade_and_unfold(output, target, overlap) if batched else output[0]
        fade_out = np.linspace(1, 0, 20 * self.hop_length)
        output = output[:wave_len]
        output[-20 * self.hop_length:] *= fade_out
        return output

    def sample(self, logits, u):
        """One row's draw from float64 logits with uniforms u -> (sample, margin): the margin is the gap between the two best
        Gumbel scores (MOL) or the distance of the uniform from the edges of the chosen class's CDF interval (RAW)."""
        logits = np.asarray(logits, dtype=np.float64)
        if self.mode == 'MOL':
            return sample_mol(logits, u)
        return sample_raw(logits, u[0])


def sample_mol(y, u):
    """sample_from_discretized_mix_logistic for one row of 30 logits, uniforms u[0..10]."""
    nr = 10
    scores = y[:nr] - np.log(-np.log(u[:nr]))
    order = np.argsort(-scores, kind='stable')
    k = int(order[0])
    margin = float(scores[order[0]] - scores[order[1]])
    mu = y[nr + k]
    ls = max(y[2 * nr + k], LOG_SCALE_MIN)
    x = mu + np.exp(ls) * (np.log(u[nr]) - np.log(1. - u[nr]))
    return float(np.clip(x, -1., 1.)), margin


def sample_raw(y, u):
    """softmax, then the first class whose cumulative probability exceeds u, mapped to 2 k / (n - 1) - 1."""
    p = np.exp(y - y.max())
    cdf = np.cumsum(p / p.sum())
    k = int(min(np.searchsorted(cdf, u, side='right'), len(y) - 1))
    margin = float(min(u - (cdf[k - 1] if k > 0 else 0.0), cdf[k] - u if k < len(y) - 1 else 1.0))
    return 2. * k / (len(y) - 1.) - 1., margin


def decode_mu_law(y, mu, from_labels=True):
    if from_labels:
        y = 2 * y / (2 ** math.log2(mu) - 1.) - 1.      # label_2_float(y, log2(mu))
    mu = mu - 1
    return np.sign(y) / mu * ((1 + mu) ** np.abs(y) - 1)


# ------------------------------------------------------------------------------------------------------------ folds
def pad_tensor(x, pad, side='both'):
    b, t, c = x.size()
    total = t + 2 * pad if side == 'both' else t + pad
    padded = torch.zeros(b, total, c, dtype=x.dtype, device=x.device)
    if side == 'before' or side == 'both':
        padded[:, pad:pad + t, :] = x
    elif side == 'after':
        padded[:, :t, :] = x
    return padded


def fold_with_overlap(x, target, overlap):
    """fatchord's fold_with_overlap, literally."""
    _, total_len, features = x.size()
    num_folds = (total_len - overlap) // (target + overlap)
    extended_len = num_folds * (overlap + target) + overlap
    remaining = total_len - extended_len
    if remaining != 0:
        num_folds += 1
        padding = target + 2 * overlap - remaining
        x = pad_tensor(x, padding, side='after')
    folded = torch.zeros(num_folds, target + 2 * overlap, features, dtype=x.dtype, device=x.device)
    for i in range(num_folds):
        start = i * (target + overlap)
        end = start + target + 2 * overlap
        folded[i] = x[:, start:end, :]
    return folded


def xfade_and_unfold(y, target, overlap):
    """fatchord's xfade_and_unfold, literally (y: (num_folds, length) float64, modified in place)."""
    num_folds, length = y.shape
    target = length - 2 * overlap
    total_len = num_folds * (target + overlap) + overlap
    silence_len = overlap // 2
    fade_len = overlap - silence_len
    silence = np.zeros((silence_len), dtype=np.float64)
    linear = np.ones((silence_len), dtype=np.float64)
    t = np.linspace(-1, 1, fade_len, dtype=np.float64)
    fade_in = np.sqrt(0.5 * (1 + t))
    fade_out = np.sqrt(0.5 * (1 - t))
    fade_in = np.concatenate([silence, fade_in])
    fade_out = np.concatenate([linear, fade_out])
    y[:, :overlap] *= fade_in
    y[:, -overlap:] *= fade_out
    unfolded = np.zeros((total_len), dtype=np.float64)
    for i in range(num_folds):
        start = i * (target + overlap)
        end = start + target + 2 * overlap
        unfolded[start:end] += y[i]
    return unfolded


# ------------------------------------------------------------------------------------------------------------ randomness
_M64 = (1 << 64) - 1


def _mix(x):
    with np.errstate(over='ignore'):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def uniforms(seed, fold, step, n_draws):
    """(len(fold), n_draws) float32 uniforms in [1e-5, 1 - 1e-5] keyed by (seed, fold, step, draw), as csrc/wavernn.cu draws
    them: splitmix64 of seed << 32 | fold, xor step << 8 | draw, splitmix64 again; (top 23 bits + 0.5) 2^-23, clamped."""
    fold = np.atleast_1d(np.asarray(fold, dtype=np.uint64))
    seed = np.broadcast_to(np.asarray(seed, dtype=np.uint64), fold.shape)
    z = _mix((seed << np.uint64(32)) | fold)[:, None]
    d = (np.uint64(step) << np.uint64(8)) | np.arange(n_draws, dtype=np.uint64)[None, :]
    z = _mix(z ^ d)
    v = ((z >> np.uint64(41)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    return np.minimum(np.maximum(v, np.float32(1e-5)), np.float32(1) - np.float32(1e-5))


# ------------------------------------------------------------------------------------------------------------ helpers
def init_state_dict(seed: int = 0, mode: str = 'MOL', bits: int = BITS, **dims) -> dict:
    """Seeded float64 state dict of fatchord's keys whose activations stay O(1): weights N(0, 1 / fan_in) scaled so the
    GRUs neither saturate nor die, BatchNorm statistics away from identity, random up-layer kernels, and output layers
    whose samples wander over [-1, 1]."""
    gen = torch.Generator().manual_seed(seed)
    net = WaveRNN(bits=bits, mode=mode, **dims).to(torch.float64)
    sd = {}
    for k, v in net.state_dict().items():
        if k == 'step':
            sd[k] = torch.zeros(1, dtype=torch.long)
            continue
        r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)   # noqa: E731
        if k.endswith('running_mean'):
            t = 0.1 * r(v.shape)
        elif k.endswith('running_var'):
            t = 1.0 + 0.3 * torch.rand(v.shape, generator=gen, dtype=torch.float64)
        elif k.endswith('num_batches_tracked'):
            t = torch.zeros_like(v)
        elif 'batch_norm' in k and k.endswith('weight'):
            t = 1.0 + 0.1 * r(v.shape)
        elif 'batch_norm' in k and k.endswith('bias'):
            t = 0.05 * r(v.shape)
        elif 'up_layers' in k:
            t = (1.0 + 0.5 * r(v.shape)) / v.shape[-1]
        elif v.ndim >= 2:
            fan_in = int(np.prod(v.shape[1:]))
            gain = 0.5 if 'layers.' in k else 1.0
            t = gain * r(v.shape) / math.sqrt(fan_in)
        else:
            t = 0.1 * r(v.shape)
        sd[k] = t
    return sd


def build(sd, device='cpu') -> WaveRNN:
    """WaveRNN in float64 (eval mode) sized from the state dict's own shapes (load_state_dict then checks every key)."""
    cin = tuple(sd['upsample.resnet.conv_in.weight'].shape)            # (compute, feat, 2 pad + 1)
    factors, i = [], 1
    while f'upsample.up_layers.{i}.weight' in sd:
        factors.append((sd[f'upsample.up_layers.{i}.weight'].shape[-1] - 1) // 2)
        i += 2
    res_blocks = 0
    while f'upsample.resnet.layers.{res_blocks}.conv1.weight' in sd:
        res_blocks += 1
    n_classes = sd['fc3.weight'].shape[0]
    mode = 'MOL' if n_classes == 30 else 'RAW'
    net = WaveRNN(rnn_dims=sd['rnn1.weight_hh_l0'].shape[1], fc_dims=sd['fc1.weight'].shape[0],
                  bits=int(round(math.log2(n_classes))) if mode == 'RAW' else BITS, pad=(cin[2] - 1) // 2,
                  upsample_factors=tuple(factors), feat_dims=cin[1], compute_dims=cin[0],
                  res_out_dims=sd['upsample.resnet.conv_out.weight'].shape[0], res_blocks=res_blocks,
                  hop_length=int(np.prod(factors)), mode=mode).to(torch.float64)
    net.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    return net.to(device).eval()


def make_mels(lengths, seed: int = 0, n_mels: int = 80):
    """Seeded speech-like WaveRNN-normalised log-mels (n_mels, T_c) in [-4, 4] (this project's normaliser)."""
    rng = np.random.default_rng(seed)
    out = []
    for T in lengths:
        f = np.linspace(0, 1, n_mels)[:, None]
        t = np.arange(T)[None, :]
        base = 0.5 - 2.5 * f + 1.8 * np.sin(0.19 * t + 5 * f + rng.uniform(0, 6)) * np.exp(-1.5 * f)
        out.append(np.clip(base + 0.5 * rng.standard_normal((n_mels, T)), -4.0, 4.0).astype(np.float32))
    return out


def to_fatchord(mel):
    """This project's WaveRNN normaliser (clip((dB + 100) / 100, 0, 1) 8 - 4) -> fatchord's normalize(): (mel + 4) / 8."""
    return (np.asarray(mel, dtype=np.float64) + 4.0) / 8.0


@torch.no_grad()
def replay(net: WaveRNN, mels, samples, seeds, batched=True, target=TARGET, overlap=OVERLAP, capture_steps=None, steps=None):
    """Teacher-forced float64 run on given samples.  mels: this project's normalised (80, T_c); samples: (R, L) the GPU's
    per-fold samples (row order: clip after clip, fold after fold).  Step s of row r feeds samples[r, s - 1] back.
    steps: replay only the first `steps` steps of every fold.
    -> dict(logits (R, capture_steps, n_classes), draws (R, L), margins (R, L))."""
    dev, dt = net.fc3.weight.device, net.fc3.weight.dtype
    m_rows, a_rows, keys = [], [], []
    for c, mel in enumerate(mels):
        m_up, aux = net.conditioning(torch.from_numpy(to_fatchord(mel))[None].to(dev, dt))
        m_up, aux = m_up[None], aux[None]
        if batched:
            m_up, aux = fold_with_overlap(m_up, target, overlap), fold_with_overlap(aux, target, overlap)
        m_rows.append(m_up)
        a_rows.append(aux)
        keys += [(seeds[c], i) for i in range(m_up.shape[0])]
    L = max(m.shape[1] for m in m_rows)
    m_all = torch.cat([F.pad(m, (0, 0, 0, L - m.shape[1])) for m in m_rows])
    a_all = torch.cat([F.pad(a, (0, 0, 0, L - a.shape[1])) for a in a_rows])
    L = L if steps is None else steps
    R = m_all.shape[0]
    samples = np.asarray(samples, dtype=np.float64)
    assert samples.shape == (R, L), (samples.shape, (R, L))
    cap = L if capture_steps is None else capture_steps
    cells = net._cells()
    h1 = torch.zeros(R, net.rnn_dims, device=dev, dtype=dt)
    h2 = torch.zeros_like(h1)
    x = torch.zeros(R, 1, device=dev, dtype=dt)
    seeds_r = np.array([k[0] for k in keys], dtype=np.uint64)
    folds_r = np.array([k[1] for k in keys], dtype=np.uint64)
    nd = 11 if net.mode == 'MOL' else 1
    logits_out = np.zeros((R, cap, net.n_classes))
    draws, margins = np.zeros((R, L)), np.zeros((R, L))
    for s in range(L):
        logits, h1, h2 = net.step_logits(cells, x, m_all[:, s], a_all[:, s], h1, h2)
        lg = logits.cpu().numpy()
        if s < cap:
            logits_out[:, s] = lg
        u = uniforms(seeds_r, folds_r, s, nd).astype(np.float64)
        for r in range(R):
            draws[r, s], margins[r, s] = net.sample(lg[r], u[r])
        x = torch.from_numpy(samples[:, s]).to(dev, dt)[:, None]
    return dict(logits=logits_out, draws=draws, margins=margins)
