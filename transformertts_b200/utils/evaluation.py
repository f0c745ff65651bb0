"""Objective scores of a trained ForwardTransformer against held-out recordings (evaluate_tts.py, train_tts.py --evaluate; the
reference has no counterpart: it shows validation predictions in TensorBoard).

* MCD-DTW: mel-cepstral distortion after dynamic time warping, on the GPU (``ttsb_mcd_dtw``).  The cepstra are the orthonormal
  DCT-II of the natural-log mels (the MelGAN normaliser's ln(max(S, 1e-5)); WaveRNN-normalised mels are mapped back to it by
  ``natural_log_mels``), coefficients 1..K with c0 (the energy) left out;
  the frame distance is 10 / ln 10 * sqrt(2 sum_k (c_k - c'_k)^2) dB and a line's MCD is the DTW path cost over the path
  length.  This is not the all-pass warped mel-cepstrum of SPTK / WORLD, so the numbers are not comparable to MCD figures in
  papers that use those; they rank models and vocoders of this project against each other (``mcep=True`` below gives the
  comparable one).
* Duration errors of the integer durations against the Aligner's durations: mean absolute error in frames per phoneme, the
  rate of exact matches and the ratio of predicted to recorded frames.
* Pitch RMSE over the phonemes whose target pitch is not 0 (unvoiced), in normalised units and, with ``pitch_stats.pkl``, in Hz.
* F0 of vocoded audio (``f0=True``): the WORLD F0 (DIO + StoneMask on the GPU) of the vocoded waveforms against the recorded
  frame pitch, frame by frame along the MCD-DTW warping path (``ttsb_mcd_dtw_path``): gross pitch error (GPE), voicing
  decision error (VDE), F0 frame error (FFE) and the F0 RMSE in cents (``f0_scores``).
* WORLD mel-cepstral distortion of vocoded audio (``mcep=True``): the MCD that published TTS and vocoder work reports.  Both
  the vocoded waveforms and the recordings go through DIO + StoneMask, CheapTrick and pysptk's sp2mc (``Audio.world_mcep_batch``,
  order 24 at ``mcep_alpha(fs)`` by default); mc_1..mc_order are DTW-aligned and scored by 10 / ln 10 sqrt(2 sum_k dmc_k^2) per
  path step (``mcep_mcd_dtw``, ``ttsb_mcd_dtw_ceps``).  Its numbers are comparable to those of pyworld + pysptk pipelines (WORLD's
  safeguard noise is drawn differently, see DESIGN.md section 7).

Corpus values are means over lines."""
from __future__ import annotations

import json
import math
import pickle
from dataclasses import dataclass
from pathlib import Path
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from .. import lib

KAPPA = 10.0 / math.log(10.0)   # dB per neper-like unit of the cepstral distance: 10 / ln 10
DEFAULT_N_CEPS = 24


def dct_matrix(n_mels: int, n_ceps: int) -> np.ndarray:
    """Rows k = 1..n_ceps of the orthonormal DCT-II of n_mels points: D[k][m] = sqrt(2 / M) cos(pi k (2m + 1) / (2M))."""
    m = np.arange(n_mels, dtype=np.float64)[None, :]
    k = np.arange(1, n_ceps + 1, dtype=np.float64)[:, None]
    return np.sqrt(2.0 / n_mels) * np.cos(np.pi * k * (2 * m + 1) / (2 * n_mels))


def check_normalizer(config: dict, what: str = 'model'):
    """MCD here is defined on natural-log mels; the WaveRNN normaliser's mels are scaled differently."""
    normalizer = config.get('normalizer')
    if normalizer != 'MelGAN':
        raise ValueError(f'MCD is computed from the MelGAN normaliser\'s natural-log mels (ln(max(S, 1e-5))); this {what}\'s '
                         f'normalizer is {normalizer!r}, whose cepstra would not be comparable')


LN10_OVER_20 = math.log(10.0) / 20.0


def _wavernn_to_natural_log(m: torch.Tensor) -> torch.Tensor:
    return ((m + 4.0) / 8.0 * 100.0 - 100.0) * LN10_OVER_20


def natural_log_mels(config: dict, what: str = 'model') -> Callable[[torch.Tensor], torch.Tensor]:
    """The map from this config's normalised mels to the natural-log mels ln(max(S, 1e-5)) MCD is defined on: the identity for
    the MelGAN normaliser; for WaveRNN's clip((20 log10 max(S, 1e-5) + 100) / 100, 0, 1) * 8 - 4, whose -100 dB floor is the
    same 1e-5, ln S = ((y + 4) / 8 * 100 - 100) ln 10 / 20, exact below 0 dB (the WaveRNN normaliser clips louder bins to 0 dB).
    Any other normaliser is refused (check_normalizer)."""
    normalizer = config.get('normalizer')
    if normalizer == 'WaveRNN':
        return _wavernn_to_natural_log
    check_normalizer(config, what)
    return lambda m: m


def _offsets(counts) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(np.asarray(counts, dtype=np.int64))])


def mcd_dtw_packed(x: torch.Tensor, x_offsets, y: torch.Tensor, y_offsets, n_ceps: int = DEFAULT_N_CEPS):
    """ttsb_mcd_dtw on packed fp32 log-mels (frames, n_mels) on one device, host offset tables (n_pairs + 1).
    -> (cost float64 (n_pairs,), path_len int32 (n_pairs,), mcd = cost / path_len), numpy arrays."""
    n_mels = x.shape[1]
    if y.shape[1] != n_mels or x.device != y.device:
        raise ValueError(f'x {tuple(x.shape)} on {x.device} and y {tuple(y.shape)} on {y.device}: need the same n_mels and device')
    n = len(x_offsets) - 1
    with torch.cuda.device(x.device):
        dct = torch.from_numpy(dct_matrix(n_mels, n_ceps)).to(x.device)
        cost = torch.empty(n, dtype=torch.float64, device=x.device)
        path_len = torch.empty(n, dtype=torch.int32, device=x.device)
        lib.mcd_dtw(x.contiguous(), x_offsets, y.contiguous(), y_offsets, dct, KAPPA, cost, path_len)
        cost, path_len = cost.cpu().numpy(), path_len.cpu().numpy()
    return cost, path_len, cost / path_len


MCD_DTW_PATH_BUDGET = 1 << 30   # bytes of ttsb_mcd_dtw_path workspace per call (cepstra and 2 bits per DTW cell)


def mcd_dtw_paths(mels_a: Sequence, mels_b: Sequence, n_ceps: int = DEFAULT_N_CEPS, workspace_budget: int = MCD_DTW_PATH_BUDGET):
    """mcd_dtw with the warping paths (``ttsb_mcd_dtw_path``): -> (cost, path_len, mcd, paths), the first three as mcd_dtw
    returns them (bit for bit) and paths[i] int32 (path_len[i], 2), the (i, j) frame pairs of line i's optimal path from (0, 0)
    to (Tx - 1, Ty - 1).  The pairs are split into calls whose workspaces hold at most `workspace_budget` bytes (a pair larger
    than that runs alone); a pair's result does not depend on the others, so the split changes nothing."""
    if len(mels_a) != len(mels_b) or len(mels_a) == 0:
        raise ValueError(f'need two non-empty lists of the same length, got {len(mels_a)} and {len(mels_b)}')
    device = next((m.device for m in list(mels_a) + list(mels_b) if torch.is_tensor(m) and m.is_cuda),
                  torch.device('cuda', torch.cuda.current_device()))
    lens = [(int(np.shape(a)[0]), int(np.shape(b)[0])) for a, b in zip(mels_a, mels_b)]
    groups, size = [[]], 0
    for i, (tx, ty) in enumerate(lens):
        # a pair's workspace alone bounds its share of a batch's (the batch shares one pair table)
        nb = lib.mcd_dtw_path_workspace_bytes([0, tx], [0, ty], n_ceps) if tx > 0 and ty > 0 else 0
        if groups[-1] and size + nb > workspace_budget:
            groups.append([])
            size = 0
        groups[-1].append(i)
        size += nb
    n = len(lens)
    cost, path_len, paths = np.empty(n), np.empty(n, dtype=np.int32), [None] * n
    for g in groups:
        x, xo = _pack([mels_a[i] for i in g], device)
        y, yo = _pack([mels_b[i] for i in g], device)
        n_mels = x.shape[1]
        if y.shape[1] != n_mels:
            raise ValueError(f'x {tuple(x.shape)} and y {tuple(y.shape)}: need the same n_mels')
        starts = np.concatenate([[0], np.cumsum([lens[i][0] + lens[i][1] - 1 for i in g])])
        with torch.cuda.device(device):
            dct = torch.from_numpy(dct_matrix(n_mels, n_ceps)).to(device)
            c = torch.empty(len(g), dtype=torch.float64, device=device)
            ln = torch.empty(len(g), dtype=torch.int32, device=device)
            path = torch.empty((int(starts[-1]), 2), dtype=torch.int32, device=device)
            lib.mcd_dtw_path(x, xo, y, yo, dct, KAPPA, c, ln, path)
            c, ln, path = c.cpu().numpy(), ln.cpu().numpy(), path.cpu().numpy()
        for r, i in enumerate(g):
            cost[i], path_len[i] = c[r], ln[r]
            paths[i] = path[starts[r]:starts[r] + ln[r]].copy()
    return cost, path_len, cost / path_len, paths


def mcep_alpha(fs: int) -> float:
    """pysptk.util.mcepalpha(fs): the all-pass constant alpha on the grid 0, 0.001, .. 0.999 whose frequency warping
    arctan((1 - a^2) sin w / ((1 + a^2) cos w - 2a)) (mod pi) is closest in mean square to the mel scale 1000 / ln 2 ln(1 + f /
    1000), both normalised to end at 1, over 1000 points up to fs / 2 (0.41 at 16 kHz, 0.455 at 22.05 kHz, 0.544 at 44.1 kHz)."""
    n = 1000
    f = (fs / 2.0) / n * np.arange(n)
    mel = 1000.0 / np.log(2) * np.log(1 + f / 1000.0)
    mel = mel / mel[-1]
    omega = np.pi / n * np.arange(n)
    alphas = np.arange(0.0, 1.0, 0.001)
    a = alphas[:, None]
    with np.errstate(divide='ignore', invalid='ignore'):
        warp = np.arctan((1 - a * a) * np.sin(omega) / ((1 + a * a) * np.cos(omega) - 2 * a))
    warp = np.where(warp < 0, warp + np.pi, warp)
    warp = warp / warp[:, -1:]
    return float(alphas[int(np.argmin(np.sum((mel - warp) ** 2, axis=1) / n))])


def sp2mc_matrix(fft_size: int, order: int, alpha: float) -> np.ndarray:
    """pysptk.sp2mc as a matrix: sp2mc(sp, order, alpha) = W @ log(sp) for a power spectrum sp of fft_size / 2 + 1 bins, W float64
    (order + 1, fft_size / 2 + 1).  Built by running sp2mc's linear steps on the unit vectors: c = irfft(e_j), c[0] /= 2, then
    SPTK's freqt recursion over all fft_size coefficients of c (g_0 = c_i + a d_0, g_1 = (1 - a^2) d_0 + a d_1,
    g_k = d_{k-1} + a (d_k - g_{k-1}), for i = fft_size - 1 .. 0)."""
    nb = fft_size // 2 + 1
    c = np.fft.irfft(np.eye(nb), n=fft_size, axis=0)      # (fft_size, nb): column j is irfft(e_j)
    c[0] /= 2.0
    b = 1.0 - alpha * alpha
    g = np.zeros((order + 1, nb))
    for i in range(fft_size - 1, -1, -1):
        d = g.copy()
        g[0] = c[i] + alpha * d[0]
        if order >= 1:
            g[1] = b * d[0] + alpha * d[1]
        for k in range(2, order + 1):
            g[k] = d[k - 1] + alpha * (d[k] - g[k - 1])
    return g


def mcep_mcd_dtw(mceps_a: Sequence, mceps_b: Sequence, order: int):
    """MCD-DTW of mel-cepstra mceps_a[i] against mceps_b[i] (float64 (T, >= order + 1), tensors or arrays) on coefficients
    1..order (``ttsb_mcd_dtw_ceps``; mc_0, the energy, is left out) -> (cost, path_len, mcd) numpy arrays as mcd_dtw returns them."""
    if len(mceps_a) != len(mceps_b) or len(mceps_a) == 0:
        raise ValueError(f'need two non-empty lists of the same length, got {len(mceps_a)} and {len(mceps_b)}')
    device = next((m.device for m in list(mceps_a) + list(mceps_b) if torch.is_tensor(m) and m.is_cuda),
                  torch.device('cuda', torch.cuda.current_device()))

    def pack(ms):
        ts = [torch.as_tensor(m).to(device=device, dtype=torch.float64) for m in ms]
        for i, t in enumerate(ts):
            if t.dim() != 2 or t.shape[0] < 1 or t.shape[1] < order + 1:
                raise ValueError(f'mel-cepstrum {i} has shape {tuple(t.shape)}; expected (T, >= {order + 1}) with T >= 1')
        return torch.cat(ts).contiguous(), _offsets([t.shape[0] for t in ts])
    x, xo = pack(mceps_a)
    y, yo = pack(mceps_b)
    if x.shape[1] != y.shape[1]:
        raise ValueError(f'mel-cepstra of {x.shape[1]} and {y.shape[1]} coefficients')
    n = len(xo) - 1
    with torch.cuda.device(device):
        cost = torch.empty(n, dtype=torch.float64, device=device)
        path_len = torch.empty(n, dtype=torch.int32, device=device)
        lib.mcd_dtw_ceps(x, xo, y, yo, 1, order, KAPPA, cost, path_len)
        cost, path_len = cost.cpu().numpy(), path_len.cpu().numpy()
    return cost, path_len, cost / path_len


def f0_scores(f0_a_hz, f0_b_hz, path) -> dict:
    """Pitch and voicing of contour a against contour b (Hz, 0 = unvoiced; voiced means f0 > 0) over the steps (i, j) of a
    warping path, float64.  A step counts when i < len(a) and j < len(b) (a WORLD contour can be a frame shorter than the mel the
    path aligns); f0_steps is their number.  VDE: voicing mismatches / steps; GPE: steps voiced on both sides with
    |f_a / f_b - 1| > 0.2 / steps voiced on both sides; FFE: (gross errors + voicing mismatches) / steps; f0_rmse_cents:
    sqrt(mean((1200 log2(f_a / f_b))^2)) over the steps voiced on both sides.  A score with an empty denominator is None."""
    a, b = np.asarray(f0_a_hz, dtype=np.float64).reshape(-1), np.asarray(f0_b_hz, dtype=np.float64).reshape(-1)
    path = np.asarray(path, dtype=np.int64).reshape(-1, 2)
    scored = path[(path[:, 0] < len(a)) & (path[:, 1] < len(b))]
    fa, fb = a[scored[:, 0]], b[scored[:, 1]]
    va, vb = fa > 0.0, fb > 0.0
    both = va & vb
    n, n_both, flips = len(scored), int(both.sum()), int((va != vb).sum())
    ratio = fa[both] / fb[both]
    gross = int((np.abs(ratio - 1.0) > 0.2).sum())
    cents = 1200.0 * np.log2(ratio)
    return {'gpe': gross / n_both if n_both else None, 'vde': flips / n if n else None, 'ffe': (gross + flips) / n if n else None,
            'f0_rmse_cents': float(np.sqrt(np.mean(cents * cents))) if n_both else None, 'f0_steps': n}


def _pack(mels, device) -> tuple:
    ts = [torch.as_tensor(m).to(device=device, dtype=torch.float32) for m in mels]
    for i, t in enumerate(ts):
        if t.dim() != 2 or t.shape[0] < 1:
            raise ValueError(f'mel {i} has shape {tuple(t.shape)}; expected (T, n_mels) with T >= 1')
    return torch.cat(ts).contiguous(), _offsets([t.shape[0] for t in ts])


def mcd_dtw(mels_a: Sequence, mels_b: Sequence, n_ceps: int = DEFAULT_N_CEPS):
    """MCD-DTW of mels_a[i] against mels_b[i] for every i: lists of (T, n_mels) natural-log mels (tensors or arrays; on the
    device of the first CUDA tensor, else the current CUDA device).  -> (cost, path_len, mcd) numpy arrays, one entry per pair;
    mcd in dB per path step."""
    if len(mels_a) != len(mels_b) or len(mels_a) == 0:
        raise ValueError(f'need two non-empty lists of the same length, got {len(mels_a)} and {len(mels_b)}')
    device = next((m.device for m in list(mels_a) + list(mels_b) if torch.is_tensor(m) and m.is_cuda),
                  torch.device('cuda', torch.cuda.current_device()))
    x, xo = _pack(mels_a, device)
    y, yo = _pack(mels_b, device)
    return mcd_dtw_packed(x, xo, y, yo, n_ceps)


# ----------------------------------------------------------------------------------------------------------------------
# the validation split and the scores of one model
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class ValidationSet:
    """The validation lines as train_tts.py reads them: phoneme strings, recorded mels (T, n_mels), the Aligner's integer
    durations and per-phoneme pitch (normalised; 0 = unvoiced), and (pitch_mean, pitch_std) in Hz when known."""
    names: List[str]
    phonemes: List[str]
    mels: List[np.ndarray]
    durations: List[np.ndarray]
    pitch: List[np.ndarray]
    pitch_stats: Optional[tuple] = None
    frame_pitch: Optional[List[np.ndarray]] = None   # recorded F0 per mel frame in Hz (0 = unvoiced), float64
    recordings: Optional[List[np.ndarray]] = None    # the waveforms the mels were computed from, float32 at the data's rate


def load_recordings(cm, names: Sequence[str], mels: Sequence[np.ndarray]) -> List[np.ndarray]:
    """The waveform of every line, rebuilt from ``wav_directory`` as create_training_data.py built the one its mel came from
    (Audio.load_wavs at the config's audio settings: read_wav or the GPU FLAC decoder, GPU resampling of an off-rate file, volume normalisation,
    trim_silence when configured, the pad to the hop).  A line whose rebuilt waveform does not give its stored mel's frame count
    (1 + L // hop_length) is refused with ValueError; a missing wav_directory or file raises FileNotFoundError."""
    from ..data.audio import Audio
    from ..data.datasets import scan_recordings
    if cm.wav_directory is None:
        raise FileNotFoundError('the recordings are read from the wav_directory of the paths settings, and the config has none')
    wav_paths = scan_recordings(cm.wav_directory)
    missing = [n for n in names if n not in wav_paths]
    if missing:
        raise FileNotFoundError(f'no recording {missing[0]}.wav or .flac below {cm.wav_directory}'
                                + (f' (and {len(missing) - 1} more)' if len(missing) > 1 else ''))
    audio = Audio.from_config(cm.config)
    wavs = audio.load_wavs([wav_paths[n] for n in names])
    for n, w, m in zip(names, wavs, mels):
        frames = 1 + len(w) // audio.hop_length
        if frames != m.shape[0]:
            raise ValueError(f'line {n}: the recording rebuilt from {wav_paths[n]} gives {frames} mel frames, its stored mel has '
                             f'{m.shape[0]}; the mel was not computed from this file at these audio settings')
    return wavs


def load_validation_set(cm, frame_pitch: bool = False, recordings: bool = False) -> ValidationSet:
    """The config's validation split (``valid_metadata``, ``mels``, ``durations`` and ``char_pitch`` of a
    TrainingConfigManager), plus ``pitch_stats.pkl`` when the data directory has one.  With frame_pitch, also the recorded
    frame F0 ``pitch.<audio>/<name>.npy`` in Hz: create_training_data.py stores it normalised, so it is de-normalised with
    ``pitch_stats.pkl`` (p std + mean where p != 0); a missing file or missing statistics raise FileNotFoundError.  With
    recordings, also each line's waveform (load_recordings)."""
    from ..data.datasets import DataReader
    reader = DataReader(cm.valid_metadata_path, is_processed=True)
    names = list(reader.text_dict)
    if not names:
        raise ValueError(f'no validation lines in {cm.valid_metadata_path}')
    stats = None
    if (cm.data_dir / 'pitch_stats.pkl').exists():
        with open(cm.data_dir / 'pitch_stats.pkl', 'rb') as f:
            st = pickle.load(f)
        stats = (float(st['pitch_mean']), float(st['pitch_std']))
    frames = None
    if frame_pitch:
        if stats is None:
            raise FileNotFoundError(f'{cm.data_dir / "pitch_stats.pkl"} not found: the frame pitch is stored normalised and needs '
                                    f'its statistics')
        missing = [cm.pitch_dir / f'{n}.npy' for n in names if not (cm.pitch_dir / f'{n}.npy').exists()]
        if missing:
            raise FileNotFoundError(f'no frame pitch {missing[0]}' + (f' (and {len(missing) - 1} more)' if len(missing) > 1 else ''))
        frames = []
        for n in names:
            p = np.load(cm.pitch_dir / f'{n}.npy').astype(np.float64).reshape(-1)
            frames.append(np.where(p != 0.0, p * stats[1] + stats[0], 0.0))
    mels = [np.load(cm.mel_dir / f'{n}.npy').astype(np.float32) for n in names]
    return ValidationSet(
        names=names, phonemes=[reader.text_dict[n] for n in names], mels=mels,
        durations=[np.load(cm.duration_dir / f'{n}.npy').astype(np.int64) for n in names],
        pitch=[np.load(cm.pitch_per_char / f'{n}.npy').astype(np.float32).reshape(-1) for n in names], pitch_stats=stats,
        frame_pitch=frames, recordings=load_recordings(cm, names, mels) if recordings else None)


def tokenize(model, phonemes: Sequence[str]) -> List[List[int]]:
    """The lines' token ids, with the tokenizer predict_tts.py builds for the model."""
    from ..data.text import Tokenizer
    tok = Tokenizer(add_start_end=False, model_breathing=bool(model.config.get('model_breathing', False)), alphabet=model.alphabet)
    return [tok(p) for p in phonemes]


def duration_scores(pred: np.ndarray, target: np.ndarray) -> dict:
    pred, target = np.asarray(pred, dtype=np.int64), np.asarray(target, dtype=np.int64)
    if pred.shape != target.shape:
        raise ValueError(f'{pred.shape[0]} predicted durations for {target.shape[0]} target durations')
    return {'duration_mae': float(np.abs(pred - target).mean()), 'duration_exact': float((pred == target).mean()),
            'frame_ratio': float(pred.sum() / target.sum()) if target.sum() > 0 else None}


def pitch_scores(pred: np.ndarray, target: np.ndarray, stats: Optional[tuple]) -> dict:
    pred, target = np.asarray(pred, dtype=np.float64).reshape(-1), np.asarray(target, dtype=np.float64).reshape(-1)
    voiced = target != 0.0
    if not voiced.any():
        return {'pitch_rmse': None, 'pitch_rmse_hz': None}
    err = pred[voiced] - target[voiced]
    out = {'pitch_rmse': float(np.sqrt(np.mean(err * err))), 'pitch_rmse_hz': None}
    if stats is not None:
        mean, std = stats
        hz = (pred[voiced] * std + mean) - (target[voiced] * std + mean)
        out['pitch_rmse_hz'] = float(np.sqrt(np.mean(hz * hz)))
    return out


def _mcd_fields(prefix: str, pred_mels: list, ref_mels: list, n_ceps: int, to_ln=lambda m: m, with_paths: bool = False) -> tuple:
    """({prefix}mcd / dtw_cost / path_len per line, the mels mapped to natural-log mels by to_ln, paths): None for a line whose
    prediction has no frame.  paths[i] is line i's warping path with with_paths (mcd_dtw_paths, the same scores), else None."""
    rows = [{f'{prefix}mcd': None, f'{prefix}dtw_cost': None, f'{prefix}path_len': None} for _ in pred_mels]
    paths = [None] * len(pred_mels)
    keep = [i for i, m in enumerate(pred_mels) if m.shape[0] > 0]
    if keep:
        a = [to_ln(torch.as_tensor(pred_mels[i])) for i in keep]
        b = [to_ln(torch.as_tensor(ref_mels[i])) for i in keep]
        if with_paths:
            cost, path_len, mcd, kept_paths = mcd_dtw_paths(a, b, n_ceps)
            for r, i in enumerate(keep):
                paths[i] = kept_paths[r]
        else:
            cost, path_len, mcd = mcd_dtw(a, b, n_ceps)
        for r, i in enumerate(keep):
            rows[i] = {f'{prefix}mcd': float(mcd[r]), f'{prefix}dtw_cost': float(cost[r]), f'{prefix}path_len': int(path_len[r])}
    return rows, paths


F0_KEYS = ('gpe', 'vde', 'ffe', 'f0_rmse_cents', 'f0_steps')
F0_FLOOR = 71.0                    # pyworld's default f0_floor, which Audio.extract_pitch_device runs DIO with
PITCH_CHUNK_SAMPLES = 1 << 24      # samples per DIO call (its workspace takes about 190 bytes per sample)


def _dio_takes(audio, n_samples: int) -> bool:
    """Whether ttsb_pitch_dio_stonemask takes a clip of n_samples: it needs more WORLD frames than DIO's voice_range_minimum."""
    fp = audio.hop_length / audio.sampling_rate * 1000
    return int(audio._pitch_frames([n_samples])[0]) > int(0.5 + 1000.0 / fp / F0_FLOOR) * 2 + 1


def _f0_fields(prefix: str, audio, wavs: list, paths: list, frame_pitch: list) -> List[dict]:
    """{prefix}gpe / vde / ffe / f0_rmse_cents / f0_steps per line: the F0 of wavs[i] against the recorded frame_pitch[i] along
    paths[i] (f0_scores); None for a line without a path or too short for DIO."""
    rows = [{prefix + k: None for k in F0_KEYS} for _ in wavs]
    keep = [i for i, (w, p) in enumerate(zip(wavs, paths)) if p is not None and _dio_takes(audio, len(w))]
    chunks, samples = [[]], 0
    for i in keep:
        if chunks[-1] and samples + len(wavs[i]) > PITCH_CHUNK_SAMPLES:
            chunks.append([])
            samples = 0
        chunks[-1].append(i)
        samples += len(wavs[i])
    for chunk in chunks:
        if chunk:   # a clip's F0 does not depend on the other clips of the batch
            for i, f0 in zip(chunk, audio.extract_pitch_batch([wavs[i] for i in chunk])):
                rows[i] = {prefix + k: v for k, v in f0_scores(f0, frame_pitch[i], paths[i]).items()}
    return rows


MCEP_KEYS = ('mcep_mcd', 'mcep_dtw_cost', 'mcep_path_len')


def _mcep_fields(prefix: str, audio, wavs: list, rec_mceps: list, order: int, alpha: float) -> List[dict]:
    """{prefix}mcep_mcd / mcep_dtw_cost / mcep_path_len per line: the WORLD mel-cepstra of wavs[i] against rec_mceps[i]
    (mcep_mcd_dtw over mc_1..mc_order); None for a line without a waveform, or whose waveform or recording is too short for DIO."""
    rows = [{prefix + k: None for k in MCEP_KEYS} for _ in wavs]
    keep = [i for i, (w, r) in enumerate(zip(wavs, rec_mceps)) if w is not None and r is not None and _dio_takes(audio, len(w))]
    if keep:
        mceps = audio.world_mcep_batch([wavs[i] for i in keep], order=order, alpha=alpha)
        cost, path_len, mcd = mcep_mcd_dtw(mceps, [rec_mceps[i] for i in keep], order)
        for r, i in enumerate(keep):
            rows[i] = {prefix + 'mcep_mcd': float(mcd[r]), prefix + 'mcep_dtw_cost': float(cost[r]),
                       prefix + 'mcep_path_len': int(path_len[r])}
    return rows


def _resynthesis_mels(audio, wavs: List[np.ndarray]) -> List[torch.Tensor]:
    """Log-mels of vocoded waveforms through the ragged front end (Audio.mel_spectrogram_ragged_device)."""
    for i, w in enumerate(wavs):
        if len(w) < audio.min_mel_samples:
            raise ValueError(f'line {i}: the vocoder gave {len(w)} samples; the log-mel front end needs at least {audio.min_mel_samples}')
    packed = torch.from_numpy(np.ascontiguousarray(np.concatenate(wavs), dtype=np.float32)).to(audio.device)
    mel, fo = audio.mel_spectrogram_ragged_device(packed, _offsets([len(w) for w in wavs]))
    return [mel[int(fo[i]):int(fo[i + 1])] for i in range(len(wavs))]


def _means(lines: List[dict]) -> dict:
    """Per key, the mean over the lines that have a value (None when none has)."""
    out = {}
    for key in lines[0]:
        if key != 'name':
            vals = [ln[key] for ln in lines if ln[key] is not None]
            out[key] = float(np.mean(vals)) if vals else None
    return out


def evaluate_model(model, vs: ValidationSet, n_ceps: int = DEFAULT_N_CEPS, teacher_forced: bool = True,
                   vocode: Optional[Callable[[List[np.ndarray]], List[np.ndarray]]] = None, audio=None, batch_size: int = 64,
                   f0: bool = False, mcep: bool = False, mcep_order: int = DEFAULT_N_CEPS, mcep_alpha: Optional[float] = None) -> dict:
    """Scores of `model` on `vs`: {'lines': [one dict per line], 'mean': {means over lines}}.

    Free-running (``predict_batch`` of the phonemes alone): MCD-DTW against the recorded mel, duration and pitch errors.  With
    teacher_forced, also ``predict_batch`` with the target durations and pitch, scored by MCD-DTW (tf_*).  With vocode (a
    function from a list of (T, n_mels) mels to waveforms) and audio (the model's Audio), the free-running mels and the recorded
    mels are vocoded, their log-mels re-extracted on the GPU and each scored against the recorded mel (vocoded_* and
    copy_synthesis_*; the latter is the vocoder's own floor).  With f0 (needs vocode and vs.frame_pitch), also the F0 scores of
    both sets of waveforms against the recorded frame pitch along the same MCD-DTW paths (vocoded_gpe ... and
    copy_synthesis_gpe ..., see f0_scores), with the F0 of Audio.extract_pitch_batch at WORLD's settings of the training data.
    With mcep (needs vocode and vs.recordings), also the WORLD mel-cepstral distortion of both sets of waveforms against the
    recordings (vocoded_mcep_mcd / _dtw_cost / _path_len and copy_synthesis_mcep_*): Audio.world_mcep_batch at mcep_order and
    mcep_alpha (None: mcep_alpha(fs)) on each side, mcep_mcd_dtw over mc_1..mc_order."""
    if f0 and (vocode is None or vs.frame_pitch is None):
        raise ValueError('the F0 scores need a vocoder and the recorded frame pitch (load_validation_set(cm, frame_pitch=True))')
    if mcep and (vocode is None or vs.recordings is None):
        raise ValueError('the WORLD MCD needs a vocoder and the recordings (load_validation_set(cm, recordings=True))')
    to_ln = natural_log_mels(model.config)
    tokens = tokenize(model, vs.phonemes)
    outs = model.predict_batch(tokens, encode=False, phoneme_max_duration=None, batch_size=batch_size)
    pred_mels = [o['mel'] for o in outs]
    lines = [{'name': n, 'frames_predicted': int(o['mel_lengths']), 'frames_recorded': int(m.shape[0])}
             for n, o, m in zip(vs.names, outs, vs.mels)]
    for i, row in enumerate(_mcd_fields('', pred_mels, vs.mels, n_ceps, to_ln)[0]):
        lines[i].update(row)
        lines[i].update(duration_scores(outs[i]['int_durations'].cpu().numpy(), vs.durations[i]))
        lines[i].update(pitch_scores(outs[i]['pitch'].cpu().numpy(), vs.pitch[i], vs.pitch_stats))
    if teacher_forced:
        tf = model.predict_batch(tokens, encode=False, phoneme_max_duration=None, phoneme_durations=vs.durations,
                                 phoneme_pitch=vs.pitch, batch_size=batch_size)
        for i, row in enumerate(_mcd_fields('teacher_forced_', [o['mel'] for o in tf], vs.mels, n_ceps, to_ln)[0]):
            lines[i].update(row)
    if vocode is not None:
        if audio is None:
            raise ValueError('vocoding needs the Audio front end of the model')
        kept = [i for i, m in enumerate(pred_mels) if m.shape[0] > 0]
        vocoded = [torch.empty(0)] * len(pred_mels)   # a line without frames has nothing to vocode: its score stays None
        vocoded_wavs = [None] * len(pred_mels)
        if kept:
            wavs = vocode([pred_mels[i].cpu().numpy() for i in kept])
            for i, w, m in zip(kept, wavs, _resynthesis_mels(audio, wavs)):
                vocoded[i], vocoded_wavs[i] = m, w
        copy_wavs = vocode(vs.mels)
        copy = _resynthesis_mels(audio, copy_wavs)
        rows, paths = _mcd_fields('vocoded_', vocoded, vs.mels, n_ceps, to_ln, with_paths=f0)
        crows, cpaths = _mcd_fields('copy_synthesis_', copy, vs.mels, n_ceps, to_ln, with_paths=f0)
        for i, (row, crow) in enumerate(zip(rows, crows)):
            lines[i].update(row)
            lines[i].update(crow)
        if f0:
            for prefix, wavs, ps in (('vocoded_', vocoded_wavs, paths), ('copy_synthesis_', copy_wavs, cpaths)):
                for i, row in enumerate(_f0_fields(prefix, audio, wavs, ps, vs.frame_pitch)):
                    lines[i].update(row)
        if mcep:
            rec = [None] * len(vs.recordings)
            kept = [i for i, w in enumerate(vs.recordings) if _dio_takes(audio, len(w))]
            if kept:
                for i, mc in zip(kept, audio.world_mcep_batch([vs.recordings[i] for i in kept], order=mcep_order, alpha=mcep_alpha)):
                    rec[i] = mc
            for prefix, wavs in (('vocoded_', vocoded_wavs), ('copy_synthesis_', copy_wavs)):
                for i, row in enumerate(_mcep_fields(prefix, audio, wavs, rec, mcep_order, mcep_alpha)):
                    lines[i].update(row)
    return {'lines': lines, 'mean': _means(lines)}


def summary_line(label: str, result: dict) -> str:
    m = result['mean']

    def f(key, fmt='.3f'):
        v = m.get(key)
        return 'n/a' if v is None else format(v, fmt)
    s = (f'{label}: MCD-DTW {f("mcd")} dB'
         + (f' (teacher-forced {f("teacher_forced_mcd")})' if 'teacher_forced_mcd' in m else '')
         + f' | duration MAE {f("duration_mae")} frames, exact {f("duration_exact")}, frame ratio {f("frame_ratio")}'
         + f' | pitch RMSE {f("pitch_rmse")}' + (f' ({f("pitch_rmse_hz", ".2f")} Hz)' if m.get('pitch_rmse_hz') is not None else ''))
    if 'vocoded_mcd' in m:
        s += f' | vocoded MCD {f("vocoded_mcd")}, copy synthesis {f("copy_synthesis_mcd")}'
    if 'vocoded_mcep_mcd' in m:
        s += f' | WORLD MCD vocoded {f("vocoded_mcep_mcd")}, copy synthesis {f("copy_synthesis_mcep_mcd")}'
    for label, p in (('vocoded', 'vocoded_'), ('copy synthesis', 'copy_synthesis_')):
        if f'{p}gpe' in m:
            s += (f' | {label} GPE {f(p + "gpe")}, VDE {f(p + "vde")}, FFE {f(p + "ffe")}, '
                  f'F0 RMSE {f(p + "f0_rmse_cents", ".1f")} cents')
    return s


def write_json(obj, path: Path):
    path = Path(path)
    path.parent.mkdir(parents=True, exist_ok=True)
    with open(path, 'w') as f:
        json.dump(obj, f, indent=1)
