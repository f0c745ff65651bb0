#!/usr/bin/env python
"""Duration and per-character pitch extraction with a trained Aligner: the reference's ``extract_durations.py``, the step
between ``train_aligner.py`` and ``train_tts.py``.

    python extract_durations.py --config config/training_config.yaml [--best] [--autoregressive_weights DIR]
                                [--skip_char_pitch] [--skip_durations]

For every utterance of the phonemized metadata (``phonemized_metadata.*.txt``), in the config's mel-length buckets:
teacher-forced ``val_step`` at r=1 -> last-block cross-attention -> durations (shortest monotonic path through the attention
of the best head or, by default, the score-weighted heads) -> per-character pitch: the mean voiced frame pitch under each
character's frames (frame pitch from ``pitch.*/<name>.npy``, float64, de-normalised with ``pitch_stats.pkl`` for the
400 Hz cut).  Both run on the GPU; the durations stay on the device for the pitch pass.  Output: ``durations.*/<name>.npy``
(int32, one entry per phoneme, summing to the mel frame count) and ``char_pitch.*/<name>.npy`` (float64), the layout
``train_tts.py`` reads.  ``--skip_durations`` reads existing durations and recomputes only the pitch.

The pitch pass is a few operations per frame: the run time is reading and writing the per-utterance files.
"""
from __future__ import annotations

import argparse
import pickle
import time

import numpy as np
import torch

from transformertts_b200.utils.training_config_manager import TrainingConfigManager

LAST_LAYER_KEY = 'Decoder_LastBlock_CrossAttention'


def load_pitch_batch(cm, names):
    """Frame pitch of the named utterances, zero-padded to (B, max length) float64, and the lengths."""
    rows = [np.asarray(np.load((cm.pitch_dir / n).with_suffix('.npy').as_posix()), dtype=np.float64).reshape(-1) for n in names]
    lens = np.array([len(p) for p in rows], dtype=np.int32)
    out = np.zeros((len(rows), max(1, int(lens.max()) if len(rows) else 1)), dtype=np.float64)
    for i, p in enumerate(rows):
        out[i, :len(p)] = p
    return out, lens


def save_char_pitch(cm, names, char_pitch, n_phonemes):
    for i, name in enumerate(names):
        np.save((cm.pitch_per_char / name).with_suffix('.npy').as_posix(), char_pitch[i, :n_phonemes[i]].copy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', dest='config', type=str, required=True)
    ap.add_argument('--best', dest='best', action='store_true', help='Use best head instead of weighted average of heads.')
    ap.add_argument('--autoregressive_weights', type=str, default=None, help='Explicit path to autoregressive model weights.')
    ap.add_argument('--skip_char_pitch', dest='skip_char_pitch', action='store_true')
    ap.add_argument('--skip_durations', dest='skip_durations', action='store_true')
    args = ap.parse_args()
    weighted = not args.best
    print(f'DurationExtraction{"_weighted" if weighted else "_best"}')
    from transformertts_b200.data import datasets as ds
    from transformertts_b200.data.text import Tokenizer
    from transformertts_b200.utils.alignments import durations_from_alignment_device, durations_to_host, pitch_per_char_batch

    cm = TrainingConfigManager(args.config, aligner=True)
    cfg = cm.config
    device = torch.device('cuda', torch.cuda.current_device())
    for d in (cm.duration_dir, cm.pitch_per_char):
        d.mkdir(parents=True, exist_ok=True)
    want_pitch = not args.skip_char_pitch
    if want_pitch:
        with open(cm.data_dir / 'pitch_stats.pkl', 'rb') as f:
            stats = pickle.load(f)
        mean, std = float(stats['pitch_mean']), float(stats['pitch_std'])
    n_utt, t0 = 0, time.perf_counter()
    if not args.skip_durations:
        model = cm.load_model(args.autoregressive_weights, device=str(device))
        if model.r != 1:
            print(f"ERROR: model's reduction factor is greater than 1, check config. (r={model.r}")
        prep = ds.AlignerPreprocessor.from_config(cm, Tokenizer(add_start_end=True, model_breathing=bool(cfg.get('model_breathing', False))))
        dataset = ds.AlignerDataset.from_config(cm, prep, kind='phonemized').get_dataset(
            bucket_batch_sizes=cfg['bucket_batch_sizes'], bucket_boundaries=cfg['bucket_boundaries'], shuffle=False, drop_remainder=False)
        print(f'Extracting attention from layer {LAST_LAYER_KEY}')
        for c, b in enumerate(dataset.all_batches()):
            tokens, mel, stop = b['tokens'].to(device), b['mel'].to(device), b['stop_prob'].to(device)
            out = model.val_step(tokens, mel, stop)
            att = out['decoder_attention'][LAST_LAYER_KEY]
            dur_dev, mel_len, phon_len, scores = durations_from_alignment_device(att, mel, tokens, weighted=weighted)
            names = b['name']
            n_phon = (b['tokens'] != 0).sum(1).numpy() - 2      # start / end tokens excluded
            if want_pitch:
                # the reference loops over min(mel frames, len(durations)) characters (extract_durations.py:111)
                mel_frames = (b['stop_prob'] != 0).sum(1).numpy() - 2
                pitch, plen = load_pitch_batch(cm, names)
                char_pitch = pitch_per_char_batch(pitch, plen, dur_dev, np.minimum(mel_frames, n_phon), mean, std)
            durations = durations_to_host(dur_dev, mel_len, phon_len)
            for i, name in enumerate(names):
                np.save((cm.duration_dir / name).with_suffix('.npy').as_posix(), durations[i])
            if want_pitch:
                save_char_pitch(cm, names, char_pitch.cpu().numpy(), n_phon)
            s = scores.mean(0).tolist()
            print(f'batch {c}: {len(names)} utterances  jumpiness / peakiness / diagonality per head: '
                  + '  '.join(f'h{h} {v[0]:.4f} {v[1]:.4f} {v[2]:.4f}' for h, v in enumerate(s)), flush=True)
            n_utt += len(names)
    elif want_pitch:
        names_all = ds.DataReader.from_config(cm, kind='phonemized').filenames
        print(f'\nComputing phoneme-wise pitch')
        print(f'{len(names_all)} items found in {cm.phonemized_metadata_path}.')
        for k in range(0, len(names_all), 64):
            names = names_all[k:k + 64]
            durs = [np.load((cm.duration_dir / n).with_suffix('.npy').as_posix()) for n in names]
            mel_frames = np.array([np.load((cm.mel_dir / n).with_suffix('.npy').as_posix(), mmap_mode='r').shape[0] for n in names])
            n_phon = np.array([len(d) for d in durs])
            dur_pad = np.zeros((len(names), max(1, int(n_phon.max()))), dtype=np.int32)
            for i, d in enumerate(durs):
                dur_pad[i, :len(d)] = d
            pitch, plen = load_pitch_batch(cm, names)
            char_pitch = pitch_per_char_batch(pitch, plen, dur_pad, np.minimum(mel_frames, n_phon), mean, std)
            save_char_pitch(cm, names, char_pitch.cpu().numpy(), n_phon)
            n_utt += len(names)
    dt = time.perf_counter() - t0
    print(f'{n_utt} utterances in {dt:.1f} s ({n_utt / max(dt, 1e-9):.1f} utterances/s)')
    print('Done.')


if __name__ == '__main__':
    main()
