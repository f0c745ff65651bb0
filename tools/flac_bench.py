#!/usr/bin/env python
"""FLAC decoding on the GPU: decode rate of ttsb_flac_decode_batch and the create_training_data.py loader on a corpus stored as
FLAC against the same corpus as WAV.

    python tools/flac_bench.py [--files 1000] [--out DIR]

The seeded corpus (tests/flac_oracle.py, libFLAC-like settings: block 4096, LPC order 8, mid/side per frame, PADDING,
VORBIS_COMMENT and SEEKTABLE) has files of 2 to 10 s, half 48 kHz stereo 24-bit (VCTK / Hi-Fi TTS-like) and half 22050 Hz mono
16-bit (LJSpeech-like).  It is written to a temporary directory.  Printed, with the card name and power limit read in the same
run: the decode time from CUDA events (the compressed upload excluded) as seconds of audio per second, and the loader time
(read, decode or read_wav, resample to 22050 Hz, preprocess) of the FLAC corpus and of the WAV corpus.
"""
from __future__ import annotations

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

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / 'tests')]


def _make(args):
    import flac_oracle as fo
    i, d = args
    rng = np.random.default_rng(10_000 + i)
    rate, C, bps = (48000, 2, 24) if i % 2 == 0 else (22050, 1, 16)
    n = int(rng.uniform(2.0, 10.0) * rate)
    x = fo.speech_like(n, C, bps, rate, 20_000 + i)
    (Path(d) / 'flac' / f'f{i:04d}.flac').write_bytes(fo.encode(x, rate, bps))
    fo.write_wav(Path(d) / 'wav' / f'f{i:04d}.wav', x, rate, bps)
    return n / rate


def _card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--files', type=int, default=1000)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', type=str, default=None, help='directory for a JSON copy of the result')
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('flac_bench needs a CUDA device')
    import create_training_data as ctd
    from transformertts_b200 import lib
    from transformertts_b200.build import build
    from transformertts_b200.data.audio import Audio, FlacStream
    build(verbose=False)
    card = _card()
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / 'flac').mkdir()
        (Path(d) / 'wav').mkdir()
        t0 = time.time()
        with ProcessPoolExecutor(max_workers=max(1, min(32, os.cpu_count() or 1))) as pool:
            seconds = sum(pool.map(_make, [(i, d) for i in range(args.files)], chunksize=4))
        build_s = time.time() - t0
        flacs = sorted((Path(d) / 'flac').glob('*.flac'))
        wavs = sorted((Path(d) / 'wav').glob('*.wav'))
        flac_bytes = sum(p.stat().st_size for p in flacs)
        streams = [FlacStream.read(p) for p in flacs]
        dev = torch.device('cuda:0')
        frames = [st.data[st.frame_offset:] for st in streams]
        bo = np.concatenate([[0], np.cumsum([len(b) for b in frames])]).astype(np.int64)
        info = [st.stream_info() for st in streams]
        totals = np.array([st.total_samples for st in streams])
        data = torch.from_numpy(np.frombuffer(b''.join(frames), np.uint8).copy()).to(dev)
        mono = torch.empty(int(totals.sum()), dtype=torch.float32, device=dev)
        status = torch.empty((len(streams), 2), dtype=torch.int32, device=dev)
        lib.flac_decode_batch(data, bo, info, mono, status)                  # warm-up
        torch.cuda.synchronize()
        assert not status[:, 0].any().item(), 'a bench file failed to decode'
        times = []
        for _ in range(args.repeats):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            lib.flac_decode_batch(data, bo, info, mono, status)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b) / 1e3)
        del data, mono, status
        audio = Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                      normalizer='MelGAN', norm_wav=True, target_dBFS=-30, int16_max=32767)

        def loader(paths):
            torch.cuda.synchronize()
            t = time.time()
            n = 0
            for raw in ctd.batches(paths, ctd.BATCH_SAMPLES, ctd.wav_loader(audio), ctd.loaded_samples(audio)):
                n += sum(len(y) for _, y in ctd.finish_batch(audio, raw, {}))
            torch.cuda.synchronize()
            return time.time() - t, n
        loader(flacs[:8])
        loader(wavs[:8])
        flac_s, n_flac = loader(flacs)
        wav_s, n_wav = loader(wavs)
        assert n_flac == n_wav
    res = dict(card=card, files=args.files, audio_seconds=round(seconds, 1), flac_mbytes=round(flac_bytes / 1e6, 1),
               corpus_build_s=round(build_s, 1), decode_s=[round(t, 5) for t in times],
               decode_audio_s_per_s=round(seconds / min(times)), loader_flac_s=round(flac_s, 2), loader_wav_s=round(wav_s, 2))
    print(json.dumps(res))
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'flac_bench.json').write_text(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
