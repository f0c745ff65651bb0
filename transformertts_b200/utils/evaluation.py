"""Objective scores of a trained ForwardTransformer against held-out recordings (evaluate_tts.py, train_tts.py --evaluate; the
reference has no counterpart: it shows validation predictions in TensorBoard).

* MCD-DTW: mel-cepstral distortion after dynamic time warping, on the GPU (``ttsb_mcd_dtw``).  The cepstra are the orthonormal
  DCT-II of the natural-log mels (the MelGAN normaliser's ln(max(S, 1e-5)); WaveRNN-normalised mels are mapped back to it by
  ``natural_log_mels``), coefficients 1..K with c0 (the energy) left out;
  the frame distance is 10 / ln 10 * sqrt(2 sum_k (c_k - c'_k)^2) dB and a line's MCD is the DTW path cost over the path
  length.  This is not the all-pass warped mel-cepstrum of SPTK / WORLD, so the numbers are not comparable to MCD figures in
  papers that use those; they rank models and vocoders of this project against each other.
* Duration errors of the integer durations against the Aligner's durations: mean absolute error in frames per phoneme, the
  rate of exact matches and the ratio of predicted to recorded frames.
* Pitch RMSE over the phonemes whose target pitch is not 0 (unvoiced), in normalised units and, with ``pitch_stats.pkl``, in Hz.

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


def load_validation_set(cm) -> ValidationSet:
    """The config's validation split (``valid_metadata``, ``mels``, ``durations`` and ``char_pitch`` of a
    TrainingConfigManager), plus ``pitch_stats.pkl`` when the data directory has one."""
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
    return ValidationSet(
        names=names, phonemes=[reader.text_dict[n] for n in names],
        mels=[np.load(cm.mel_dir / f'{n}.npy').astype(np.float32) for n in names],
        durations=[np.load(cm.duration_dir / f'{n}.npy').astype(np.int64) for n in names],
        pitch=[np.load(cm.pitch_per_char / f'{n}.npy').astype(np.float32).reshape(-1) for n in names], pitch_stats=stats)


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


def _mcd_fields(prefix: str, pred_mels: list, ref_mels: list, n_ceps: int, to_ln=lambda m: m) -> List[dict]:
    """{prefix}mcd / dtw_cost / path_len per line, the mels mapped to natural-log mels by to_ln; None for a line whose prediction
    has no frame."""
    rows = [{f'{prefix}mcd': None, f'{prefix}dtw_cost': None, f'{prefix}path_len': None} for _ in pred_mels]
    keep = [i for i, m in enumerate(pred_mels) if m.shape[0] > 0]
    if keep:
        cost, path_len, mcd = mcd_dtw([to_ln(torch.as_tensor(pred_mels[i])) for i in keep],
                                      [to_ln(torch.as_tensor(ref_mels[i])) for i in keep], n_ceps)
        for r, i in enumerate(keep):
            rows[i] = {f'{prefix}mcd': float(mcd[r]), f'{prefix}dtw_cost': float(cost[r]), f'{prefix}path_len': int(path_len[r])}
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
                   vocode: Optional[Callable[[List[np.ndarray]], List[np.ndarray]]] = None, audio=None, batch_size: int = 64) -> dict:
    """Scores of `model` on `vs`: {'lines': [one dict per line], 'mean': {means over lines}}.

    Free-running (``predict_batch`` of the phonemes alone): MCD-DTW against the recorded mel, duration and pitch errors.  With
    teacher_forced, also ``predict_batch`` with the target durations and pitch, scored by MCD-DTW (tf_*).  With vocode (a
    function from a list of (T, n_mels) mels to waveforms) and audio (the model's Audio), the free-running mels and the recorded
    mels are vocoded, their log-mels re-extracted on the GPU and each scored against the recorded mel (vocoded_* and
    copy_synthesis_*; the latter is the vocoder's own floor)."""
    to_ln = natural_log_mels(model.config)
    tokens = tokenize(model, vs.phonemes)
    outs = model.predict_batch(tokens, encode=False, phoneme_max_duration=None, batch_size=batch_size)
    pred_mels = [o['mel'] for o in outs]
    lines = [{'name': n, 'frames_predicted': int(o['mel_lengths']), 'frames_recorded': int(m.shape[0])}
             for n, o, m in zip(vs.names, outs, vs.mels)]
    for i, row in enumerate(_mcd_fields('', pred_mels, vs.mels, n_ceps, to_ln)):
        lines[i].update(row)
        lines[i].update(duration_scores(outs[i]['int_durations'].cpu().numpy(), vs.durations[i]))
        lines[i].update(pitch_scores(outs[i]['pitch'].cpu().numpy(), vs.pitch[i], vs.pitch_stats))
    if teacher_forced:
        tf = model.predict_batch(tokens, encode=False, phoneme_max_duration=None, phoneme_durations=vs.durations,
                                 phoneme_pitch=vs.pitch, batch_size=batch_size)
        for i, row in enumerate(_mcd_fields('teacher_forced_', [o['mel'] for o in tf], vs.mels, n_ceps, to_ln)):
            lines[i].update(row)
    if vocode is not None:
        if audio is None:
            raise ValueError('vocoding needs the Audio front end of the model')
        kept = [i for i, m in enumerate(pred_mels) if m.shape[0] > 0]
        vocoded = [torch.empty(0)] * len(pred_mels)   # a line without frames has nothing to vocode: its score stays None
        if kept:
            for i, m in zip(kept, _resynthesis_mels(audio, vocode([pred_mels[i].cpu().numpy() for i in kept]))):
                vocoded[i] = m
        copy = _resynthesis_mels(audio, vocode(vs.mels))
        for i, (row, crow) in enumerate(zip(_mcd_fields('vocoded_', vocoded, vs.mels, n_ceps, to_ln),
                                            _mcd_fields('copy_synthesis_', copy, vs.mels, n_ceps, to_ln))):
            lines[i].update(row)
            lines[i].update(crow)
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
    return s


def write_json(obj, path: Path):
    path = Path(path)
    path.parent.mkdir(parents=True, exist_ok=True)
    with open(path, 'w') as f:
        json.dump(obj, f, indent=1)
