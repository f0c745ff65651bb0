"""Duration extraction from the Aligner's attention maps, mirroring the reference's ``utils/alignments.py`` (same function
names and argument meaning).  The attention scores (utils/metrics.py:5-44) and the shortest-monotonic-path search
(utils/alignments.py:58-91, scipy Dijkstra in the reference) run on the GPU: ``ttsb_attention_scores`` and
``ttsb_durations_from_attention`` (anti-diagonal dynamic programme in float64, csrc/alignment.cu).  The per-character
pitch of extract_durations.py:108-115 runs there too (``ttsb_pitch_per_char``), on the durations still on the device."""
from __future__ import annotations

from typing import List, Tuple

import numpy as np
import torch

from .. import lib
from .spectrogram_ops import mel_lengths, phoneme_lengths


def duration_to_alignment_matrix(durations) -> np.ndarray:
    """utils/alignments.py:94-100: (phonemes, frames) 0/1 matrix with durations[i] ones in row i, one after the other."""
    durations = np.asarray(durations).astype(int)
    starts = np.cumsum(np.append([0], durations[:-1]))
    tot = int(np.sum(durations))
    out = np.zeros((len(durations), tot))
    for i, (s, d) in enumerate(zip(starts, durations)):
        out[i, s:s + d] = 1.0
    return out


def attention_score(att: torch.Tensor, mel_len: torch.Tensor, phon_len: torch.Tensor, r: int = 1):
    """utils/metrics.py:5-24 -> (loc_score, peak_score, 3 / diag_score), each (N, heads) float32 on the GPU."""
    att = att.to(dtype=torch.float32).contiguous()
    B, H = att.shape[:2]
    scores = torch.empty((B, H, 3), dtype=torch.float32, device=att.device)
    lib.attention_scores(att, mel_len.to(device=att.device, dtype=torch.int32).contiguous(),
                         phon_len.to(device=att.device, dtype=torch.int32).contiguous(), r, scores)
    return scores[..., 0], scores[..., 1], scores[..., 2]


def durations_from_alignment_device(batch_alignments, mels, phonemes, weighted: bool = False):
    """The device half of ``get_durations_from_alignment``: -> (durations (N, phonemes) int32, mel_len, phon_len, scores
    (N, heads, 3)), all on the GPU.  Row b holds ``phon_len[b] - 1`` durations followed by zeros; lengths are the reference's
    ``mel_lengths - 1`` / ``phoneme_lengths - 1``."""
    att = torch.as_tensor(batch_alignments)
    if not att.is_cuda:
        att = att.cuda()
    att = att.to(torch.float32).contiguous()
    dev = att.device
    B, H, Tq, Tk = att.shape
    mel_len = (mel_lengths(torch.as_tensor(mels).to(dev), padding_value=0.) - 1).to(torch.int32).contiguous()
    phon_len = (phoneme_lengths(torch.as_tensor(phonemes).to(dev)) - 1).to(torch.int32).contiguous()
    scores = torch.empty((B, H, 3), dtype=torch.float32, device=dev)
    lib.attention_scores(att, mel_len, phon_len, 1, scores)
    durations = torch.empty((B, Tk), dtype=torch.int32, device=dev)
    scratch = torch.empty((B, Tq * Tk), dtype=torch.uint8, device=dev)
    lib.durations_from_attention(att, mel_len, phon_len, scores, weighted, scratch, durations)
    return durations, mel_len, phon_len, scores


def durations_to_host(durations: torch.Tensor, mel_len: torch.Tensor, phon_len: torch.Tensor) -> List[np.ndarray]:
    """Per-utterance int32 durations of ``durations_from_alignment_device``, with the reference's sum assertion."""
    d_host = durations.cpu().numpy()
    ml, pl = mel_len.cpu().numpy(), phon_len.cpu().numpy()
    out = []
    for b in range(d_host.shape[0]):
        d = d_host[b, :max(int(pl[b]) - 1, 0)].copy()
        if int(d.sum()) != int(ml[b]) - 1:   # same assertion as the reference (alignments.py:136)
            raise AssertionError(f'{int(d.sum())} vs {int(ml[b]) - 1}')
        out.append(d)
    return out


def pitch_per_char_batch(pitch, pitch_len, durations, n_chars, mean: float, std: float) -> torch.Tensor:
    """Per-character pitch of a batch on the GPU (``ttsb_pitch_per_char``; reference: extract_durations.py:108-115, one
    utterance at a time there).  pitch (B, Tm) float64 frame pitch, zero-padded; pitch_len (B,) its lengths; durations (B, Tp)
    int; n_chars (B,) the characters to fill, ``min(mel_len, len(durations))`` as the reference loops.  Returns (B, Tp)
    float64 on the device, bit-exact with ``datasets.pitch_per_char`` row by row (zeros from n_chars on).

    The work is a few comparisons and additions per frame: what this saves over the reference's per-file CPU pool is the
    round trip of the durations through the disk, not arithmetic time."""
    dev = torch.device('cuda', torch.cuda.current_device())
    if torch.is_tensor(durations) and durations.is_cuda:
        dev = durations.device
    pitch = torch.as_tensor(pitch).to(device=dev, dtype=torch.float64).contiguous()
    durations = torch.as_tensor(durations).to(device=dev, dtype=torch.int32).contiguous()
    pitch_len = torch.as_tensor(pitch_len).to(device=dev, dtype=torch.int32).contiguous()
    n_chars = torch.as_tensor(n_chars).to(device=dev, dtype=torch.int32).contiguous()
    if pitch.dim() != 2 or durations.dim() != 2 or pitch.shape[0] != durations.shape[0]:
        raise ValueError('pitch must be (B, Tm) and durations (B, Tp) with the same B')
    if pitch.shape[1] == 0:   # no frames at all: every character is unvoiced
        pitch = torch.zeros((pitch.shape[0], 1), dtype=torch.float64, device=dev)
    out = torch.empty(durations.shape, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        lib.pitch_per_char(pitch, pitch_len, durations, n_chars, float(mean), float(std), out)
    return out


def get_durations_from_alignment(batch_alignments, mels, phonemes, weighted: bool = False) -> Tuple[List[np.ndarray], None, torch.Tensor,
                                                                                                 torch.Tensor, torch.Tensor]:
    """utils/alignments.py:103-143.  batch_alignments: (N, heads, mel, phonemes) attention weights of the last decoder block
    (``Decoder_LastBlock_CrossAttention``); mels with start/end vectors, phonemes with start/end tokens.
    Returns (durations [list of int32 arrays of length phon_len - 1], None, jumpiness, peakiness, diag_measure); the second
    element is the reference's plotting matrix (best attention + binary alignment), which is not produced here.

    Ties: the reference runs scipy's Dijkstra on an explicit graph; the CUDA kernel runs the equivalent dynamic programme over
    anti-diagonals and breaks EXACT cost ties in a fixed order (left, up, diagonal), scipy by heap-pop order.  On generic
    attention maps the shortest path is unique and the durations are bit-identical (tests); on plateaus of exactly equal cost
    (saturated / all-zero attention regions) the two may pick different, equally short paths."""
    durations, mel_len, phon_len, scores = durations_from_alignment_device(batch_alignments, mels, phonemes, weighted)
    return durations_to_host(durations, mel_len, phon_len), None, scores[..., 0], scores[..., 1], scores[..., 2]
