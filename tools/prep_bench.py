"""Training-data preparation throughput: log-mel + DIO/StoneMask pitch on the GPU, create_training_data.py end to end, and the numpy
restatement of WORLD on the host cores.

    python tools/prep_bench.py [--minutes 20] [--reps 3] [--cpu-clips 8] [--source-rate HZ] [--trim] [--out DIR]

Workload: seeded speech-like clips of 1-10 s (oracle/pitch_oracle.py speech_like_clip) until `--minutes` of audio, synthesised at
`--source-rate` (default: the configured 22050 Hz).
  * gpu: Audio.mel_spectrogram_ragged_device + Audio.extract_pitch_device on the packed corpus in batches of
    create_training_data.BATCH_SAMPLES, upload and download included (at another source rate, each batch is first resampled on
    the device by Audio.resample_ragged_device); host clock around the calls, ending in a device synchronise; one warm-up pass,
    then the mean of `--reps` passes.
  * resample (another source rate only): Audio.resample_ragged_device alone on each packed batch, timed with CUDA events over
    `--reps` passes after a warm-up; output samples/s and filter taps/s (taps counted from the clip lengths and resampy's
    per-sample wing lengths), and tests/resample_oracle.py (numpy, one core) on the first `--cpu-clips` clips beside it.
  * script: create_training_data.py run once as a subprocess on the same clips written as 16-bit WAV into a temporary directory
    (file reading, resampling, .npy writing, the phonemized metadata and the Python start-up included).
  * trim (`--trim` only): Audio.trim_silence_bounds_device (ttsb_trim_silence_bounds at top_db 60) alone on each packed batch,
    timed with CUDA events over `--reps` passes after a warm-up, beside the log-mel and pitch calls timed the same way on the same
    batches.  With `--trim` the script arm runs with `trim_silence: true, trim_silence_top_db: 60` as well (the clips then carry
    0-2 s of leading and trailing silence, tests/trim_oracle.py padded_speech).
  * cpu: oracle/pitch_oracle.extract_pitch (numpy restatement, not pyworld) on the first `--cpu-clips` clips with a process pool
    over all host cores, scaled to audio seconds per second.
Prints one JSON line with audio seconds processed per second for each arm, the FP64 operation count of the pitch filters derived
from the shapes, and the card name and power limit read in the same run.  `--out` also writes it to DIR/prep_bench.json."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

import numpy as np
import torch
import yaml

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import pitch_oracle as po  # noqa: E402
sys.path.insert(0, str(ROOT / 'tests'))
import resample_oracle as ro  # noqa: E402  (the numpy restatement of resampling kept with the tests)
import trim_oracle as to  # noqa: E402
from transformertts_b200.data.audio import Audio  # noqa: E402

FS, HOP = 22050, 256


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def corpus(minutes: float, sr: int = FS, silence: bool = False):
    clips, total, i = [], 0, 0
    rng = np.random.default_rng(11)
    while total < minutes * 60 * sr:
        if silence:
            x = to.padded_speech(1, 7000 + i, fs=float(sr), min_s=1.0, max_s=10.0)[0]
        else:
            x = po.speech_like_clip(float(rng.uniform(1.0, 10.0)), 7000 + i, fs=float(sr))
        clips.append(po.pad_for_hop(x) if sr == FS else x)
        total += len(x)
        i += 1
    return clips


def fp64_filter_ops(n_samples: int) -> int:
    """FP64 operations of the low-cut and band filters (2 per tap and sample)."""
    bounds = po.boundary_f0s()
    taps = 2 * po.matlab_round(FS / 50.0) + 1 + sum(4 * h for h in po.band_half_lengths(FS, bounds))
    return 2 * taps * n_samples


def batch_bounds(clips, budget):
    i, out = 0, []
    while i < len(clips):
        j, n = i, 0
        while j < len(clips) and n < budget:
            n += len(clips[j])
            j += 1
        out.append((i, j))
        i = j
    return out


def gpu_pass(audio, clips, budget, sr=FS):
    for i, j in batch_bounds(clips, budget):
        wav, so = audio._pack(clips[i:j])
        if sr != FS:
            wav, so = audio.resample_ragged_device(wav, so, [sr] * (j - i))
        mel, _ = audio.mel_spectrogram_ragged_device(wav, so)
        f0, _ = audio.extract_pitch_device(wav, so)
        mel.cpu(), f0.cpu()
    torch.cuda.synchronize()


def resample_taps(lengths, sr) -> int:
    """Filter taps of resampy's loop over clips of `lengths` samples from sr to FS (left + right wing per output sample; the
    time register taken as t / ratio, which moves a wing's length by at most one tap at a few samples)."""
    ratio = FS / sr
    scale = min(1.0, ratio)
    step, nwin = int(scale * 512), 512 * 64 + 1
    taps = 0
    for L in lengths:
        r = np.arange(int(L * ratio)) / ratio
        m = r.astype(np.int64)
        frac = scale * (r - m)
        off, off2 = (frac * 512).astype(np.int64), ((scale - frac) * 512).astype(np.int64)
        taps += int(np.minimum(m + 1, (nwin - off) // step).sum() + np.maximum(np.minimum(L - m - 1, (nwin - off2) // step), 0).sum())
    return taps


def resample_arm(audio, clips, budget, sr, reps):
    """Audio.resample_ragged_device alone on each packed batch (uploaded beforehand), CUDA events around the calls."""
    packed = []
    for i, j in batch_bounds(clips, budget):
        wav, so = audio._pack(clips[i:j])
        packed.append((wav, so, [sr] * (j - i)))
    n_out = sum(int(audio.resample_ragged_device(*p)[1][-1]) for p in packed)   # warm-up
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        for p in packed:
            audio.resample_ragged_device(*p)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / 1000 / reps, n_out


def trim_arm(audio, clips, budget, reps):
    """ttsb_trim_silence_bounds alone, then log-mel and pitch alone, on each packed batch (uploaded beforehand); CUDA events
    around each set of calls -> (trim seconds, mel + pitch seconds) per pass."""
    packed = [audio._pack(clips[i:j]) for i, j in batch_bounds(clips, budget)]

    def timed(fn):
        for p in packed:                     # warm-up
            fn(*p)
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(reps):
            for p in packed:
                fn(*p)
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / 1000 / reps

    t_trim = timed(audio.trim_silence_bounds_device)
    t_mel_pitch = timed(lambda wav, so: (audio.mel_spectrogram_ragged_device(wav, so), audio.extract_pitch_device(wav, so)))
    return t_trim, t_mel_pitch


def write_wav(path, x, sr):
    """16-bit PCM at sr, scaled and clipped as Audio.save_wav writes it."""
    import wave
    pcm = np.clip(np.rint(np.asarray(x, np.float32) * np.float32(32767)), -32768, 32767).astype('<i2')
    with wave.open(str(path), 'wb') as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(int(sr))
        f.writeframes(pcm.tobytes())


def _oracle_pitch(x):
    return po.extract_pitch(x, FS, HOP)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--minutes', type=float, default=20.0)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--cpu-clips', type=int, default=8)
    ap.add_argument('--source-rate', type=int, default=FS)
    ap.add_argument('--trim', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('prep_bench needs a CUDA device')
    import create_training_data as ctd
    sr = args.source_rate
    if args.trim and sr != FS:
        raise SystemExit('--trim times the trim at the configured rate; leave --source-rate at its default')
    clips = corpus(args.minutes, sr, silence=args.trim)
    seconds = sum(len(c) for c in clips) / sr
    audio = Audio(sampling_rate=FS, n_fft=1024, mel_channels=80, hop_length=HOP, win_length=1024, f_min=0, f_max=8000,
                  normalizer='MelGAN', trim_silence_top_db=60)
    gpu_pass(audio, clips, ctd.BATCH_SAMPLES, sr)
    t0 = time.perf_counter()
    for _ in range(args.reps):
        gpu_pass(audio, clips, ctd.BATCH_SAMPLES, sr)
    t_gpu = (time.perf_counter() - t0) / args.reps

    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        (tmp / 'wavs').mkdir()
        lines = []
        for i, x in enumerate(clips):
            write_wav(tmp / 'wavs' / f'C{i:05d}.wav', x, sr)
            lines.append(f'C{i:05d}|text|hɛloʊ wɜld\n')
        (tmp / 'metadata.csv').write_text(''.join(lines), encoding='utf-8')
        cfg = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
        cfg['paths'].update(log_directory=str(tmp / 'logs'), train_data_directory=str(tmp / 'data'),
                            metadata_path=str(tmp / 'metadata.csv'), wav_directory=str(tmp / 'wavs'))
        cfg['training_data_settings'].update(n_test=10)
        if args.trim:
            cfg['audio_settings'].update(trim_silence=True, trim_silence_top_db=60)
        (tmp / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, str(ROOT / 'create_training_data.py'), '--config', str(tmp / 'cfg.yaml')], capture_output=True,
                           text=True, cwd=tmp)
        t_script = time.perf_counter() - t0
        if r.returncode != 0:
            raise SystemExit(r.stdout[-2000:] + r.stderr[-2000:])

    rs = {}
    if args.trim:
        t_trim, t_mel_pitch = trim_arm(audio, clips, ctd.BATCH_SAMPLES, args.reps)
        rs.update(trim_silence=True, trim_gpu_seconds=round(t_trim, 6), trim_gpu_audio_s_per_s=round(seconds / t_trim, 1),
                  mel_pitch_gpu_seconds_same_batches=round(t_mel_pitch, 5),
                  trim_fraction_of_mel_pitch=round(t_trim / t_mel_pitch, 5))
    if sr != FS:
        t_rs, n_out = resample_arm(audio, clips, ctd.BATCH_SAMPLES, sr, args.reps)
        taps = resample_taps([len(c) for c in clips], sr)
        t0 = time.perf_counter()
        resampled = [ro.resample(x, sr, FS) for x in clips[:args.cpu_clips]]
        t_rs_cpu = time.perf_counter() - t0
        rs = {'source_rate': sr, 'resample_gpu_seconds': round(t_rs, 5), 'resample_output_samples': n_out,
              'resample_gpu_output_samples_per_s': round(n_out / t_rs), 'resample_taps': taps,
              'resample_gpu_taps_per_s': round(taps / t_rs), 'resample_gpu_audio_s_per_s': round(seconds / t_rs, 1),
              'resample_cpu_numpy_one_core_audio_s_per_s': round(sum(len(x) for x in clips[:args.cpu_clips]) / sr / t_rs_cpu, 2)}
    sub = clips[:args.cpu_clips] if sr == FS else resampled      # the pitch restatement runs at the configured rate
    workers = os.cpu_count() or 1
    t0 = time.perf_counter()
    with ProcessPoolExecutor(max_workers=workers) as ex:
        list(ex.map(_oracle_pitch, sub))
    t_cpu = time.perf_counter() - t0
    sub_seconds = sum(len(c) for c in sub) / FS
    n = sum(len(c) for c in clips) if sr == FS else rs['resample_output_samples']
    res = {
        'card': card(), 'audio_seconds': round(seconds, 1), 'clips': len(clips),
        'gpu_mel_pitch_audio_s_per_s': round(seconds / t_gpu, 1), 'gpu_seconds': round(t_gpu, 4),
        'script_end_to_end_audio_s_per_s': round(seconds / t_script, 1), 'script_seconds': round(t_script, 2),
        'cpu_numpy_restatement_not_pyworld_audio_s_per_s': round(sub_seconds / t_cpu, 2), 'cpu_workers': workers,
        'cpu_subset_audio_seconds': round(sub_seconds, 1),
        'pitch_filter_fp64_gflop': round(fp64_filter_ops(n) / 1e9, 2),
        'pitch_filter_fp64_tflop_s_whole_gpu_pass': round(fp64_filter_ops(n) / t_gpu / 1e12, 3),
        **rs,
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'prep_bench.json').write_text(line + '\n')


if __name__ == '__main__':
    main()
