"""MelGAN generator (the vocoder of the reference's synthesis notebook: seungwonpark/melgan via torch.hub) on the GPU, a
packed ragged batch of clips per call.

Every conv of the generator is one ``ttsb_conv1d_ex_tc`` launch over all clips (csrc/conv1d_tc.cu): clips are packed
channels-last with ``lib.CONV1D_HALO`` halo rows on each side, which hold each clip's own reflect (or zero) padding, so a tap
is a row shift and no clip sees another.  Per call: the input conv, then per upsampling stage the transposed conv plus two
products per ResStack block (the dilated conv; the shortcut and the block's 1x1 conv as one two-source product), then the
output layer: 30 conv launches (31 with the split of the input mel) whatever the number of clips.  LeakyReLU is applied in the epilogues.

Channel counts below 64 are padded to 64 columns (the tensor-core k block): the 32-channel stage, a quarter of the generator's
FLOPs, runs 4x its useful products.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from transformertts_b200 import lib

HOP = 256
PAD_FRAMES = 10           # inference(): frames of PAD_VALUE appended to every mel
PAD_VALUE = -11.5129      # ln(1e-5), the MelGAN normaliser's floor
MAX_WAV_VALUE = 32768.0
MIN_FRAMES = 4
N_MELS = 80
MEL_COLS = 128            # the input conv's 80 channels padded to two k blocks
# (transposed conv, ResStack, Cin, Cout, kernel, stride)
STAGES = [('generator.3', 'generator.4', 512, 256, 16, 8), ('generator.6', 'generator.7', 256, 128, 16, 8),
          ('generator.9', 'generator.10', 128, 64, 4, 2), ('generator.12', 'generator.13', 64, 32, 4, 2)]
IN_CONV, OUT_CONV = 'generator.1', 'generator.16'


def _cols(c: int) -> int:
    """Column count of a c-channel activation: at least one 64-wide k block."""
    return max(64, c)


def layer_shapes() -> Dict[str, tuple]:
    """conv name -> (kind, weight shape): kind 'conv' (Cout, Cin, k) or 'convT' (Cin, Cout, k)."""
    out = {IN_CONV: ('conv', (512, N_MELS, 7))}
    for tname, rname, cin, cout, k, _ in STAGES:
        out[tname] = ('convT', (cin, cout, k))
        for i in range(3):
            out[f'{rname}.blocks.{i}.2'] = ('conv', (cout, cout, 3))
            out[f'{rname}.blocks.{i}.4'] = ('conv', (cout, cout, 1))
            out[f'{rname}.shortcuts.{i}'] = ('conv', (cout, cout, 1))
    out[OUT_CONV] = ('conv', (1, 32, 7))
    return out


def expected_keys(weight_norm: bool = True) -> Dict[str, tuple]:
    """The checkpoint's state-dict keys and shapes (weight_g / weight_v form, or the plain `weight` remove_weight_norm leaves)."""
    keys = {}
    for name, (kind, shape) in layer_shapes().items():
        keys[f'{name}.bias'] = (shape[1] if kind == 'convT' else shape[0],)
        if weight_norm:
            keys[f'{name}.weight_g'] = (shape[0], 1, 1)
            keys[f'{name}.weight_v'] = shape
        else:
            keys[f'{name}.weight'] = shape
    return keys


def fold_weight_norm(g: np.ndarray, v: np.ndarray) -> np.ndarray:
    """torch.nn.utils.weight_norm (dim=0) in float64: w = g v / ||v||, the norm taken over every dim but the first."""
    v = np.asarray(v, dtype=np.float64)
    norm = np.sqrt((v.reshape(v.shape[0], -1) ** 2).sum(axis=1)).reshape((-1,) + (1,) * (v.ndim - 1))
    return np.asarray(g, dtype=np.float64).reshape(norm.shape) * v / norm


def conv_taps(w: np.ndarray, dilation: int, cin_cols: int, cout_cols: int) -> np.ndarray:
    """Conv1d weight (Cout, Cin, k), 'same' padding of dilation (k - 1) / 2 -> (k cin_cols, cout_cols): tap s (row shift
    (s - (k - 1) / 2) dilation) in rows [s cin_cols, + Cin)."""
    cout, cin, k = w.shape
    m = np.zeros((k * cin_cols, cout_cols))
    for s in range(k):
        m[s * cin_cols:s * cin_cols + cin, :cout] = w[:, :, s].T
    return m


def transposed_taps(w: np.ndarray, u: int, cin_cols: int, cout_cols: int) -> np.ndarray:
    """ConvTranspose1d weight (Cin, Cout, 2u), stride u, padding u/2 -> the (3 cin_cols, u cout_cols) matrix of an ordinary
    conv over the input rows: output row t u + r (column block r) = sum over row shifts d in (-1, 0, 1) of
    x[t + d] @ W[:, :, r + u/2 - d u] (taps outside [0, 2u) are zero).  Input rows outside the clip are zero."""
    cin, cout, k = w.shape
    assert k == 2 * u and u % 2 == 0
    m = np.zeros((3 * cin_cols, u * cout_cols))
    for ti, d in enumerate((-1, 0, 1)):
        for r in range(u):
            j = r + u // 2 - d * u
            if 0 <= j < k:
                m[ti * cin_cols:ti * cin_cols + cin, r * cout_cols:r * cout_cols + cout] = w[:, :, j]
    return m


def halo_source_rows(L: int, halo: int, mode: int) -> np.ndarray:
    """Source row (in [0, L)) of each row -halo .. L - 1 + halo of a padded clip, -1 for a zero row: the rule the conv
    epilogue's mirror stores follow.  mode: lib.HALO_REFLECT (torch's 'reflect') or lib.HALO_ZERO."""
    i = np.arange(-halo, L + halo)
    if mode == lib.HALO_ZERO:
        return np.where((i >= 0) & (i < L), i, -1)
    if L <= halo:
        raise ValueError(f'a reflect halo of {halo} rows needs more than {halo} rows; the clip has {L}')
    return np.where(i < 0, -i, np.where(i >= L, 2 * (L - 1) - i, i))


def ragged_offsets(counts: Sequence[int], rate: int = 1) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(np.asarray(counts, dtype=np.int64) * rate)]).astype(np.int64)


def layout_rows(counts: Sequence[int], rate: int = 1, halo: int = lib.CONV1D_HALO) -> int:
    """Rows of the packed layout of clips with counts[c] * rate rows each and `halo` rows on each side."""
    return int(np.sum(counts) * rate) + 2 * halo * len(counts)


def pack_clips(clips: Sequence[np.ndarray], cols: int, mode: int, halo: int = lib.CONV1D_HALO) -> np.ndarray:
    """Host packing of (L_c, C) clips into the halo layout (rows, cols) float32, halos filled by `mode`."""
    H = halo
    out = np.zeros((layout_rows([len(x) for x in clips], halo=H), cols), dtype=np.float32)
    r = 0
    for x in clips:
        L, Cc = x.shape
        src = halo_source_rows(L, H, mode)
        block = np.where((src >= 0)[:, None], x[np.maximum(src, 0)], 0.0)
        out[r:r + L + 2 * H, :Cc] = block
        r += L + 2 * H
    return out


def unpack_clips(buf: np.ndarray, counts: Sequence[int], channels: int, halo: int = lib.CONV1D_HALO) -> List[np.ndarray]:
    """The clip rows (L_c, channels) of a packed layout."""
    H, r, out = halo, 0, []
    for L in counts:
        out.append(buf[r + H:r + H + L, :channels])
        r += L + 2 * H
    return out


class _Conv:
    """One packed product: weights (bf16 hi/lo, [N, K]), fp32 bias (N) and the tap table."""

    def __init__(self, mat: np.ndarray, bias: np.ndarray, taps, split: bool, device):
        self.N = mat.shape[1]
        self.taps = taps       # [(source, row shift)]
        w = torch.from_numpy(np.ascontiguousarray(mat, dtype=np.float32)).to(device)
        self.w_hi, self.w_lo = lib.pack_weight(w, self.N, split)
        self.bias = torch.from_numpy(np.ascontiguousarray(bias, dtype=np.float32)).to(device)


def run_conv(conv: _Conv, counts_in, srcs, up: int, split: bool, out=None, act=None, halo=lib.HALO_NONE, ws=None,
             rows_halo: int = lib.CONV1D_HALO, slope: float = 0.2, res=None, sum_plane=None, sum_mode: int = lib.SUM_NONE, sum_div: float = 1.0):
    """One ttsb_conv1d_ex_tc launch: srcs = [(hi, lo)] per source, out / act / res = (hi, lo) planes or None, over a layout of
    `rows_halo` halo rows; act is LeakyReLU_slope; sum_plane is fp32 in the output layout.  The defaults are MelGAN's."""
    a = lib.Conv1dExArgs()
    off = ragged_offsets(counts_in)
    tab = (lib.C.c_int32 * len(off))(*off.tolist())
    a.n_clips = len(counts_in)
    a.clip_offsets = lib.C.cast(tab, lib.C.c_void_p)
    a.halo = rows_halo
    a.num_taps = len(conv.taps)
    for s, (src, shift) in enumerate(conv.taps):
        a.tap_src[s], a.tap_shift[s] = src, shift
    for i, (hi, lo) in enumerate(srcs):
        a.in_hi[i], a.in_lo[i], a.ld_in[i] = lib.ptr(hi), lib.ptr(lo), hi.shape[1]
    a.w_hi, a.w_lo, a.bias = lib.ptr(conv.w_hi), lib.ptr(conv.w_lo), lib.ptr(conv.bias)
    a.N, a.up, a.ld_out = conv.N, up, conv.N // up
    if out is not None:
        a.out_hi, a.out_lo = lib.ptr(out[0]), lib.ptr(out[1])
    if act is not None:
        a.act_hi, a.act_lo = lib.ptr(act[0]), lib.ptr(act[1])
    a.halo_mode = halo
    a.precision = lib.PREC_BF16X3 if split else lib.PREC_BF16
    a.workspace, a.workspace_bytes = lib.ptr(ws), ws.numel()
    a.slope = slope
    if res is not None:
        a.res_hi, a.res_lo = lib.ptr(res[0]), lib.ptr(res[1])
    if sum_plane is not None:
        a.sum = lib.ptr(sum_plane)
    a.sum_mode, a.sum_div = sum_mode, sum_div
    a.out_rows = layout_rows([c * up for c in counts_in], halo=rows_halo)
    lib.conv1d_ex_tc(a)


class MelGANGenerator:
    """The MelGAN generator of seungwonpark/melgan, vocoding ragged batches on the GPU.

    precision: 'bf16x3' (hi/lo split operands, fp32-class products) or 'bf16' (one bf16 product per conv)."""

    def __init__(self, device=None, precision: str = 'bf16x3'):
        if precision not in ('bf16x3', 'bf16'):
            raise ValueError(f"precision must be 'bf16x3' or 'bf16', got {precision!r}")
        self.device = torch.device(device if device is not None else 'cuda')
        self.precision = precision
        self.split = precision == 'bf16x3'
        self._convs: Optional[dict] = None

    # ---------------------------------------------------------------------------------------------------- loading
    @classmethod
    def from_checkpoint(cls, path, device=None, precision: str = 'bf16x3') -> 'MelGANGenerator':
        g = cls(device=device, precision=precision)
        g.load_state_dict(torch.load(path, map_location='cpu', weights_only=True))
        return g

    @staticmethod
    def fold_state_dict(sd) -> Dict[str, np.ndarray]:
        """Checks a checkpoint (``{'model_g': sd, ...}`` or a bare state dict, weight-normed or folded) against the
        specification and returns {conv name: float64 weight, conv name + '.bias': float64 bias}."""
        if isinstance(sd, dict) and 'model_g' in sd:
            sd = sd['model_g']
        if not isinstance(sd, dict):
            raise TypeError(f'expected a state dict, got {type(sd).__name__}')
        keys = set(sd)
        normed = expected_keys(True)
        plain = expected_keys(False)
        want = normed if any(k.endswith('.weight_g') or k.endswith('.weight_v') for k in keys) else plain
        missing = sorted(set(want) - keys)
        if missing:
            raise KeyError(f'MelGAN checkpoint: missing key {missing[0]}' + (f' (and {len(missing) - 1} more)' if len(missing) > 1 else ''))
        extra = sorted(keys - set(want))
        if extra:
            raise KeyError(f'MelGAN checkpoint: unexpected key {extra[0]}' + (f' (and {len(extra) - 1} more)' if len(extra) > 1 else ''))
        for k, shape in want.items():
            if tuple(sd[k].shape) != tuple(shape):
                raise ValueError(f'MelGAN checkpoint: {k} has shape {tuple(sd[k].shape)}, expected {tuple(shape)}')
        f64 = {k: sd[k].detach().cpu().double().numpy() for k in want}
        out = {}
        for name in layer_shapes():
            out[name] = fold_weight_norm(f64[f'{name}.weight_g'], f64[f'{name}.weight_v']) if want is normed else f64[f'{name}.weight']
            out[name + '.bias'] = f64[f'{name}.bias']
        return out

    def load_state_dict(self, sd) -> 'MelGANGenerator':
        w = self.fold_state_dict(sd)
        dev, split = self.device, self.split
        convs = {}
        with torch.cuda.device(dev):
            convs['in'] = _Conv(conv_taps(w[IN_CONV], 1, MEL_COLS, 512), w[IN_CONV + '.bias'], [(0, s) for s in range(-3, 4)], split, dev)
            for si, (tname, rname, cin, cout, k, u) in enumerate(STAGES):
                cc = _cols(cout)
                bias = np.zeros(u * cc)
                for r in range(u):
                    bias[r * cc:r * cc + cout] = w[tname + '.bias']
                convs[f'up{si}'] = _Conv(transposed_taps(w[tname], u, _cols(cin), cc), bias, [(0, -1), (0, 0), (0, 1)], split, dev)
                for i in range(3):
                    d = 3 ** i
                    b = np.zeros(cc)
                    b[:cout] = w[f'{rname}.blocks.{i}.2.bias']
                    convs[f'dil{si}.{i}'] = _Conv(conv_taps(w[f'{rname}.blocks.{i}.2'], d, cc, cc), b, [(0, -d), (0, 0), (0, d)], split, dev)
                    m = np.concatenate([conv_taps(w[f'{rname}.shortcuts.{i}'], 1, cc, cc), conv_taps(w[f'{rname}.blocks.{i}.4'], 1, cc, cc)])
                    b = np.zeros(cc)
                    b[:cout] = w[f'{rname}.shortcuts.{i}.bias'] + w[f'{rname}.blocks.{i}.4.bias']
                    convs[f'mix{si}.{i}'] = _Conv(m, b, [(0, 0), (1, 0)], split, dev)
            self._out_w = torch.from_numpy(np.ascontiguousarray(w[OUT_CONV][0].T, dtype=np.float32)).to(dev)   # (7, 32)
            self._out_b = float(w[OUT_CONV + '.bias'][0])
        self._convs = convs
        return self

    # ---------------------------------------------------------------------------------------------------- forward
    def _planes(self, rows: int, cols: int):
        hi = torch.empty((rows, cols), dtype=torch.bfloat16, device=self.device)
        return hi, (torch.empty_like(hi) if self.split else None)

    def _run(self, conv: _Conv, counts_in, srcs, up: int, out=None, act=None, halo=lib.HALO_NONE, ws=None):
        """One conv launch: srcs = [(hi, lo)] per source, out / act = (hi, lo) planes or None."""
        run_conv(conv, counts_in, srcs, up, self.split, out=out, act=act, halo=halo, ws=ws)

    def vocode_device(self, mels: Sequence[np.ndarray]) -> torch.Tensor:
        """vocode_batch, leaving the packed float32 waveform (256 sum T_c samples, clip after clip) on the device."""
        if self._convs is None:
            raise RuntimeError('MelGANGenerator: no weights loaded (from_checkpoint / load_state_dict)')
        ms = [np.asarray(m, dtype=np.float32) for m in mels]
        if not ms:
            raise ValueError('vocode_batch: no mels')
        for c, m in enumerate(ms):
            if m.ndim != 2 or m.shape[0] != N_MELS or m.shape[1] < MIN_FRAMES:
                raise ValueError(f'mel {c} has shape {m.shape}; the vocoder needs ({N_MELS}, T) with T >= {MIN_FRAMES} frames')
        frames = [m.shape[1] + PAD_FRAMES for m in ms]
        pad = np.full((PAD_FRAMES, N_MELS), PAD_VALUE, dtype=np.float32)
        x = pack_clips([(np.concatenate([m.T, pad]) + 5.0) / 5.0 for m in ms], MEL_COLS, lib.HALO_REFLECT)
        cv = self._convs
        with torch.cuda.device(self.device):
            ws = torch.empty(lib.conv1d_workspace_bytes(len(ms)), dtype=torch.uint8, device=self.device)
            src = lib.split_bf16(torch.from_numpy(x).to(self.device), self.split)
            act = self._planes(layout_rows(frames), 512)
            self._run(cv['in'], frames, [src], 1, act=act, halo=lib.HALO_ZERO, ws=ws)
            counts = frames
            for si, (_, _, _, cout, _, u) in enumerate(STAGES):
                last = si == len(STAGES) - 1
                counts_out = [c * u for c in counts]
                rows, cc = layout_rows(counts_out), _cols(cout)
                xa, xb, a_new, h = self._planes(rows, cc), self._planes(rows, cc), self._planes(rows, cc), self._planes(rows, cc)
                self._run(cv[f'up{si}'], counts, [act], u, out=xa, act=a_new, halo=lib.HALO_REFLECT, ws=ws)
                act = a_new
                for i in range(3):
                    self._run(cv[f'dil{si}.{i}'], counts_out, [act], 1, act=h, ws=ws)
                    final = i == 2
                    halo = lib.HALO_REFLECT if (not final or last) else lib.HALO_ZERO
                    self._run(cv[f'mix{si}.{i}'], counts_out, [xa, h], 1, out=None if final else xb, act=act, halo=halo, ws=ws)
                    xa, xb = xb, xa
                counts = counts_out
            wav = torch.empty(HOP * sum(m.shape[1] for m in ms), dtype=torch.float32, device=self.device)
            lib.conv1d_out_tanh_ex(act[0], act[1], 32, lib.CONV1D_HALO, ragged_offsets(counts), HOP * PAD_FRAMES, self._out_w,
                                   self._out_b, ws, wav)
        return wav

    def vocode_batch(self, mels: Sequence[np.ndarray]) -> List[np.ndarray]:
        """Normalised mels (n_mels, T_c), as Audio.reconstruct_waveform_batch takes them -> float32 waveforms of 256 T_c samples:
        what the generator's inference() computes per clip, before its int16 conversion."""
        wav = self.vocode_device(mels).cpu().numpy()
        off = ragged_offsets([np.asarray(m).shape[1] for m in mels], HOP)
        return [wav[off[c]:off[c + 1]] for c in range(len(mels))]

    def inference(self, mel) -> torch.Tensor:
        """seungwonpark/melgan's Generator.inference: (1, 80, T) or (80, T) mel -> int16 waveform (256 T) on the CPU."""
        m = torch.as_tensor(mel).detach().cpu().float()
        if m.ndim == 3:
            if m.shape[0] != 1:
                raise ValueError(f'inference takes one mel, got a batch of {m.shape[0]}')
            m = m[0]
        wav = torch.from_numpy(self.vocode_batch([m.numpy()])[0]).double()
        return (MAX_WAV_VALUE * wav).clamp(min=-MAX_WAV_VALUE, max=MAX_WAV_VALUE - 1).short()
