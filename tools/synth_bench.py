"""Mel -> waveform for a file's worth of utterances: the per-clip `Audio.reconstruct_waveform` loop against one
`Audio.reconstruct_waveform_batch` call.

    python tools/synth_bench.py [--clips 64] [--reps 3] [--n-iter 32] [--out DIR]

Workload: `--clips` seeded ragged clips of 2-10 s (T_c uniform in 173..862 frames, LJSpeech-like lengths); their mels come
from the CUDA front end (Audio.mel_spectrogram).  Both paths use the same phase seeds (clip c: seed c), so their outputs are
comparable clip by clip.  Both are run once before timing; a timing is the host clock around whole calls followed by
torch.cuda.synchronize(), averaged over `--reps` calls.  Prints one JSON line: seconds per call of each path, library launches
per call, the largest |difference| between the two paths' waveforms, and the card name and power limit read in the same run.
`griffinlim_only_*` times the Griffin-Lim loop alone (griffinlim_device per clip against one griffinlim_batch_device call) with
the magnitudes and initial phases already on the device: the whole calls also draw the phases on the host.
`--out` also writes it to DIR/synth_bench.json."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle import audio_oracle as ao  # noqa: E402
from transformertts_b200 import lib  # noqa: E402
from transformertts_b200.data.audio import Audio  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def timed(fn, reps):
    """Run fn once (warm-up), then `reps` times; seconds per call, library launches per call, last result."""
    out = fn()
    torch.cuda.synchronize()
    lib.reset_launch_count()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps, lib.launch_count() / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clips', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--n-iter', type=int, default=32)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    audio = Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                  normalizer='MelGAN')
    lengths = np.random.default_rng(2024).integers(173, 863, size=args.clips)
    mels = [audio.mel_spectrogram(ao.make_clips(1, 256 * (int(T) - 1), seed=500 + c)[0]).T for c, T in enumerate(lengths)]

    def per_clip():
        return [audio.reconstruct_waveform(m, n_iter=args.n_iter, seed=c) for c, m in enumerate(mels)]

    def batched():
        return audio.reconstruct_waveform_batch(mels, n_iter=args.n_iter, seed=0)

    t_loop, l_loop, w_loop = timed(per_clip, args.reps)
    t_batch, l_batch, w_batch = timed(batched, args.reps)
    diff = max(float(np.abs(a - b).max()) for a, b in zip(w_loop, w_batch))

    # the Griffin-Lim loop alone: magnitudes and initial phases already on the device (both calls above also draw the phases
    # on the host, from the CPU generator, and copy them over)
    counts = [m.shape[1] for m in mels]
    off = np.concatenate([[0], np.cumsum(counts)])
    amp = np.concatenate([np.exp(m).T.astype(np.float32) for m in mels])
    S = audio.mel_to_linear_device(torch.from_numpy(np.ascontiguousarray(amp)).cuda())
    init = torch.cat([torch.polar(torch.ones(t, 513, dtype=torch.float64), 2 * np.pi * torch.rand(t, 513, dtype=torch.float64))
                      for t in counts]).to(torch.complex64).cuda()
    S_c = [S[off[c]:off[c + 1]] for c in range(len(mels))]
    init_c = [init[off[c]:off[c + 1]] for c in range(len(mels))]
    t_gl_loop, _, _ = timed(lambda: [audio.griffinlim_device(s, n_iter=args.n_iter, init_angles=i) for s, i in zip(S_c, init_c)], args.reps)
    t_gl_batch, _, _ = timed(lambda: audio.griffinlim_batch_device(S, off, n_iter=args.n_iter, init_angles=init), args.reps)

    res = dict(workload='reconstruct_waveform', clips=args.clips, frames=int(lengths.sum()), min_frames=int(lengths.min()),
               max_frames=int(lengths.max()), n_iter=args.n_iter, reps=args.reps, per_clip_s=round(t_loop, 5),
               batch_s=round(t_batch, 5), speedup=round(t_loop / t_batch, 2), per_clip_launches=l_loop, batch_launches=l_batch,
               max_abs_diff=diff, griffinlim_only_per_clip_s=round(t_gl_loop, 5), griffinlim_only_batch_s=round(t_gl_batch, 5),
               griffinlim_only_speedup=round(t_gl_loop / t_gl_batch, 2), audio_s=round(float(256 * (lengths - 1).sum() / 22050), 1),
               card=card())
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'synth_bench.json').write_text(line + '\n')


if __name__ == '__main__':
    main()
