"""The log-mel front end and batched Griffin-Lim at the reference STFT configuration (n_fft 1024 / hop 256 / win 1024, the fused
kernels) and at the reference's WaveRNN configuration (n_fft 2048 / hop 275 / win 1100, csrc/stft_general.cu).

    python tools/stft_config_bench.py [--minutes 10] [--seconds 3] [--out DIR]

Workloads, the same seeded audio at both configurations:
  * log-mel: Audio.mel_spectrogram_ragged_device over a corpus of 1-10 s clips (`--minutes` of audio at 22050 Hz) packed in one
    device buffer, in batches of create_training_data.BATCH_SAMPLES samples; output stays on the device.
  * Griffin-Lim: Audio.griffinlim_batch_device, 32 iterations, over 64 ragged clips of 1-10 s (magnitudes of the clips' own
    STFT, seeded phases).
Each arm is warmed up once, then timed with CUDA events over as many passes as fill at least `--seconds` (at least 3 passes).  A
pass includes what every call does on the host: the clip table is built and uploaded from pageable memory, which waits for the
copy.  Prints one JSON line with audio seconds processed per second, milliseconds per pass and the pass count for every arm, and
the card name and power limit read in the same run."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import audio_oracle as ao  # noqa: E402
from transformertts_b200.data.audio import Audio  # noqa: E402

FS = 22050
CONFIGS = {'reference_1024_256_1024': dict(n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000, normalizer='MelGAN'),
           'wavernn_2048_275_1100': dict(n_fft=2048, hop_length=275, win_length=1100, f_min=40, f_max=None, normalizer='WaveRNN')}


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def lengths(n: int, seed: int):
    return [int(x) for x in np.random.default_rng(seed).integers(FS, 10 * FS, n)]


def timed(fn, seconds: float) -> tuple:
    """(ms per call, calls): one warm-up call, one call to size the window, then CUDA events around enough calls to fill
    `seconds` (at least 3)"""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    reps = max(3, int(np.ceil(seconds * 1e3 / max(start.elapsed_time(end), 1e-3))))
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps, reps


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument('--minutes', type=float, default=10.0)
    p.add_argument('--seconds', type=float, default=3.0)
    p.add_argument('--out', default=None)
    args = p.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('stft_config_bench.py measures the GPU kernels and needs a CUDA device')
    from create_training_data import BATCH_SAMPLES
    lens, total = [], 0
    rng = np.random.default_rng(5)
    while total < args.minutes * 60 * FS:
        lens.append(int(rng.integers(FS, 10 * FS)))
        total += lens[-1]
    wav = torch.from_numpy((0.1 * rng.standard_normal(total)).astype(np.float32)).cuda()
    so = np.concatenate([[0], np.cumsum(lens)])
    batches, start = [], 0
    for c in range(1, len(lens) + 1):       # clips [start, c) while they fit in one batch
        if c == len(lens) or so[c + 1] - so[start] > BATCH_SAMPLES:
            batches.append((wav[so[start]:so[c]], so[start:c + 1] - so[start]))
            start = c
    gl_lens = lengths(64, 7)
    result = dict(card=card(), corpus_clips=len(lens), corpus_seconds=total / FS, gl_clips=64, gl_seconds=sum(gl_lens) / FS,
                  gl_iterations=32)
    for name, cfg in CONFIGS.items():
        a = Audio(sampling_rate=FS, mel_channels=80, device='cuda:0', **cfg)
        ms, reps = timed(lambda: [a.mel_spectrogram_ragged_device(w, o) for w, o in batches], args.seconds)
        result[f'{name}_logmel_ms'], result[f'{name}_logmel_passes'] = ms, reps
        result[f'{name}_logmel_audio_s_per_s'] = total / FS / (ms / 1e3)
        clips = [ao.make_clips(1, L, seed=i)[0] for i, L in enumerate(gl_lens)]
        S = [np.abs(ao.stft(y, a.n_fft, a.hop_length, a.win_length)).T for y in clips]
        fo = np.concatenate([[0], np.cumsum([len(s) for s in S])])
        S = torch.from_numpy(np.ascontiguousarray(np.concatenate(S), dtype=np.float32)).cuda()
        g = torch.Generator(device='cpu').manual_seed(3)
        phase = 2 * np.pi * torch.rand(tuple(S.shape), generator=g, dtype=torch.float64)
        init = torch.polar(torch.ones_like(phase), phase).to(torch.complex64).cuda()
        ms, reps = timed(lambda: a.griffinlim_batch_device(S, fo, n_iter=32, init_angles=init), args.seconds)
        result[f'{name}_griffinlim_ms'], result[f'{name}_griffinlim_passes'] = ms, reps
        result[f'{name}_griffinlim_audio_s_per_s'] = sum(gl_lens) / FS / (ms / 1e3)
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'stft_config_bench.json').write_text(line + '\n')


if __name__ == '__main__':
    main()
