#!/usr/bin/env python
"""Time the WORLD mel-cepstra (ttsb_cheaptrick + ttsb_sp2mc) and evaluate_tts.py --mcep on the GPU.

    python tools/mcep_bench.py [--lines 100 1000] [--iters 5] [--eval_lines 100] [--out result.json]

* ttsb_cheaptrick and ttsb_sp2mc on validation-sized batches: `--lines` clips of 200-1,200 frames at 22050 Hz / hop 256 (cut from
  seeded speech-like clips), their DIO / StoneMask F0 computed once beforehand, CUDA events around `--iters` calls of each after
  a warm-up, alternating the two; the envelopes of the batch are checked against those of its first clip alone.
* evaluate_tts.py --vocoder griffinlim: the wall time of one run (a fresh process) with --mcep and one without, on a temporary
  data directory of `--eval_lines` validation lines whose recordings are wavs of 200-1,200 frames and whose mels come from them,
  scored with a seeded LJ256 model.
The card's name and power limit are read in the same run and printed with the numbers."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
import time
import wave
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / 'tools'))

from eval_bench import card  # noqa: E402

FS, HOP = 22050, 256


def _clips(n: int, seed: int) -> list:
    """n clips of 200-1,200 frames, cut from 16 seeded speech-like clips of 15 s (generating each one is slow)."""
    from oracle import pitch_oracle as po
    rng = np.random.default_rng(seed)
    base = [po.speech_like_clip(15.0, seed=seed * 100 + i) for i in range(16)]
    out = []
    for t in rng.integers(200, 1201, n):
        b = base[int(rng.integers(len(base)))]
        L = int(t) * HOP - 1
        s = int(rng.integers(0, len(b) - L))
        out.append(b[s:s + L].copy())
    return out


def time_kernels(n_lines: int, iters: int) -> dict:
    from transformertts_b200 import lib
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.utils import evaluation as ev
    audio = Audio(sampling_rate=FS, n_fft=1024, mel_channels=80, hop_length=HOP, win_length=1024, f_min=0, f_max=8000,
                  normalizer='MelGAN')
    clips = _clips(n_lines, n_lines)
    wav, so = audio._pack(clips)
    fo = np.concatenate([[0], np.cumsum(audio._pitch_frames(np.diff(so)))])
    f0 = torch.empty(int(fo[-1]), dtype=torch.float64, device='cuda')
    start = 0
    while start < len(clips):   # the F0 a chunk at a time (DIO's workspace is about 190 bytes per sample); not timed
        stop = start
        while stop < len(clips) and so[stop + 1] - so[start] <= ev.PITCH_CHUNK_SAMPLES:
            stop += 1
        stop = max(stop, start + 1)
        f, _ = audio.extract_pitch_device(wav[int(so[start]):int(so[stop])], so[start:stop + 1] - so[start])
        f0[int(fo[start]):int(fo[stop])] = f
        start = stop
    n = audio.cheaptrick_fft_size
    env = torch.empty((int(fo[-1]), n // 2 + 1), dtype=torch.float64, device='cuda')
    W = torch.from_numpy(ev.sp2mc_matrix(n, 24, ev.mcep_alpha(FS))).cuda()
    mc = torch.empty((int(fo[-1]), 25), dtype=torch.float64, device='cuda')
    fp = HOP / FS * 1000
    calls = {'cheaptrick': lambda: lib.cheaptrick(wav, so, FS, fp, f0, fo, -0.15, n, env),
             'sp2mc': lambda: lib.sp2mc(env, W, mc)}
    for call in calls.values():
        call()
    torch.cuda.synchronize()
    alone, _ = audio.spectral_envelope_device(wav[:int(so[1])], so[:2], f0[:int(fo[1])], fo[:2])
    if not torch.equal(alone, env[:int(fo[1])]):
        raise SystemExit('the first clip\'s envelope differs alone and in the batch')
    ms = {k: [] for k in calls}
    for _ in range(3):   # alternate the two, so drift on a shared machine falls on both
        for name, call in calls.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                call()
            e.record()
            e.synchronize()
            ms[name].append(s.elapsed_time(e) / iters)
    best = {k: min(v) for k, v in ms.items()}
    return {'lines': n_lines, 'frames': int(fo[-1]), 'samples': int(so[-1]), 'fft_size': n,
            'ms_per_call': {k: round(v, 3) for k, v in best.items()},
            'ms_per_call_all': {k: [round(t, 3) for t in v] for k, v in ms.items()},
            'us_per_frame': {k: round(1000 * v / int(fo[-1]), 4) for k, v in best.items()}}


def _write_wav(path, y):
    pcm = np.clip(np.rint(np.asarray(y, np.float64) * 32767), -32768, 32767).astype('<i2')
    with wave.open(str(path), 'wb') as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(FS)
        f.writeframes(pcm.tobytes())


def time_evaluate_tts_mcep(n_lines: int) -> dict:
    import yaml
    from oracle import forward_oracle as fo
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.data.text import ALL_PHONEMES
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    rng = np.random.default_rng(4)
    letters = [c for c in ALL_PHONEMES if c.isalpha()][:30] + [' ']
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
        raw['paths'].update(log_directory=str(tmp / 'logs'), train_data_directory=str(tmp / 'data'), wav_directory=str(tmp / 'wavs'))
        (tmp / 'cfg.yaml').write_text(yaml.safe_dump(raw))
        cm = TrainingConfigManager(str(tmp / 'cfg.yaml'))
        for d in (cm.mel_dir, cm.duration_dir, cm.pitch_per_char, cm.wav_directory):
            d.mkdir(parents=True, exist_ok=True)
        names = [f'w{i:04d}' for i in range(n_lines)]
        for name, y in zip(names, _clips(n_lines, 7)):
            _write_wav(cm.wav_directory / f'{name}.wav', y)
        audio = Audio.from_config(cm.config)
        mels = audio.mel_spectrogram_ragged(audio.load_wavs([cm.wav_directory / f'{n}.wav' for n in names]))
        rows, frames = [], 0
        for name, mel in zip(names, mels):
            n_ph = int(rng.integers(len(mel) // 8, len(mel) // 5))
            np.save(cm.mel_dir / f'{name}.npy', mel)
            np.save(cm.duration_dir / f'{name}.npy', np.bincount(rng.integers(0, n_ph, len(mel)), minlength=n_ph).astype(np.int32))
            np.save(cm.pitch_per_char / f'{name}.npy', rng.normal(0, 1, n_ph).astype(np.float32))
            rows.append(f'{name}|' + ''.join(rng.choice(letters, n_ph)) + '\n')
            frames += len(mel)
        cm.valid_metadata_path.write_text(''.join(rows), encoding='utf-8')
        cfg = dict(fo.CONFIGS['LJ256'], sampling_rate=FS, n_fft=1024, hop_length=HOP, win_length=1024, f_min=0, f_max=8000,
                   normalizer='MelGAN')
        p = fo.init_params(cfg, seed=7)
        p['dur_pred.out.b'] = torch.tensor([5.0])    # about 5 frames per phoneme, as the recorded lines have
        model = ForwardTransformer(**cfg)
        model.set_weights(p)
        model.save_model(tmp / 'model', with_optimizer=False)
        out = {'lines': n_lines, 'recorded_frames': frames}
        for key, extra in (('wall_s_mcep', ['--mcep']), ('wall_s_without_mcep', [])):
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, str(ROOT / 'evaluate_tts.py'), '--config', str(tmp / 'cfg.yaml'), '-p', str(tmp / 'model'),
                                '--vocoder', 'griffinlim', '-o', str(tmp / key)] + extra, capture_output=True, text=True, cwd=str(ROOT))
            out[key] = round(time.perf_counter() - t0, 2)
            if r.returncode != 0:
                raise SystemExit(r.stdout[-2000:] + r.stderr[-3000:])
            summary = [ln for ln in r.stdout.splitlines() if 'MCD-DTW' in ln]
            out['summary' + key[len('wall_s'):]] = summary[0] if summary else None
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lines', type=int, nargs='+', default=[100, 1000])
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--eval_lines', type=int, default=100)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to measure')
    res = dict(card(), world_mcep=[time_kernels(n, args.iters) for n in args.lines])
    if args.eval_lines:
        res['evaluate_tts_griffinlim'] = time_evaluate_tts_mcep(args.eval_lines)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
