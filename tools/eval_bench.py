#!/usr/bin/env python
"""Time ttsb_mcd_dtw and evaluate_tts.py on the GPU.

    python tools/eval_bench.py [--pairs 100 1000] [--iters 20] [--lines 100] [--out result.json]

* ttsb_mcd_dtw: seeded pairs of 200-1,200 frames (80 mels, K = 24), CUDA events around `--iters` calls after a warm-up, per
  batch size.  The cells (sum of Tx * Ty) are reported with the time, since the work of the DTW sweep is proportional to them.
* evaluate_tts.py: the wall time of one run (a fresh process, as a user starts it) on a temporary data directory of `--lines`
  validation lines with recorded mels of 200-1,200 frames, scored with a seeded LJ256 model, free-running and teacher-forced.
The card's name and power limit are read in the same run and printed with the numbers."""
from __future__ import annotations

import argparse
import json
import pickle
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card() -> dict:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ['unknown, unknown'])[0].split(', ')
    return {'gpu': name, 'power_limit': power}


def _mels(n, rng):
    return [np.clip(rng.normal(-5, 2, (int(t), 80)), -11.5, 2).astype(np.float32) for t in rng.integers(200, 1201, n)]


def time_kernel(n_pairs: int, iters: int) -> dict:
    from transformertts_b200 import lib
    from transformertts_b200.utils import evaluation as ev
    rng = np.random.default_rng(n_pairs)
    a = [torch.from_numpy(m).cuda() for m in _mels(n_pairs, rng)]
    b = [torch.from_numpy(m).cuda() for m in _mels(n_pairs, rng)]
    x, xo = ev._pack(a, a[0].device)
    y, yo = ev._pack(b, a[0].device)
    dct = torch.from_numpy(ev.dct_matrix(80, ev.DEFAULT_N_CEPS)).cuda()
    cost = torch.empty(n_pairs, dtype=torch.float64, device='cuda')
    path_len = torch.empty(n_pairs, dtype=torch.int32, device='cuda')

    def call():   # one ttsb_mcd_dtw: argument checks, the pair-table upload, the cepstra and the DTW kernels
        lib.mcd_dtw(x, xo, y, yo, dct, ev.KAPPA, cost, path_len)
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        call()
    end.record()
    end.synchronize()
    ms = start.elapsed_time(end) / iters
    cells = int(sum(int(p.shape[0]) * int(q.shape[0]) for p, q in zip(a, b)))
    return {'pairs': n_pairs, 'ms_per_call': round(ms, 3), 'cells': cells, 'gcells_per_s': round(cells / ms / 1e6, 3)}


def time_evaluate_tts(n_lines: int) -> dict:
    import yaml
    from oracle import forward_oracle as fo
    from transformertts_b200.data.text import ALL_PHONEMES
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    rng = np.random.default_rng(3)
    letters = [c for c in ALL_PHONEMES if c.isalpha()][:30] + [' ']
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
        raw['paths'].update(log_directory=str(tmp / 'logs'), train_data_directory=str(tmp / 'data'))
        (tmp / 'cfg.yaml').write_text(yaml.safe_dump(raw))
        cm = TrainingConfigManager(str(tmp / 'cfg.yaml'))
        for d in (cm.mel_dir, cm.duration_dir, cm.pitch_per_char):
            d.mkdir(parents=True, exist_ok=True)
        rows, frames = [], 0
        for i, mel in enumerate(_mels(n_lines, rng)):
            n_ph = int(rng.integers(len(mel) // 8, len(mel) // 5))
            name = f'e{i:04d}'
            np.save(cm.mel_dir / f'{name}.npy', mel)
            np.save(cm.duration_dir / f'{name}.npy', np.bincount(rng.integers(0, n_ph, len(mel)), minlength=n_ph).astype(np.int32))
            np.save(cm.pitch_per_char / f'{name}.npy', rng.normal(0, 1, n_ph).astype(np.float32))
            rows.append(f'{name}|' + ''.join(rng.choice(letters, n_ph)) + '\n')
            frames += len(mel)
        cm.valid_metadata_path.write_text(''.join(rows), encoding='utf-8')
        with open(cm.data_dir / 'pitch_stats.pkl', 'wb') as f:
            pickle.dump({'pitch_mean': 205.7, 'pitch_std': 41.3}, f)
        cfg = dict(fo.CONFIGS['LJ256'], sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                   normalizer='MelGAN')
        p = fo.init_params(cfg, seed=7)
        p['dur_pred.out.b'] = torch.tensor([5.0])    # about 5 frames per phoneme, as the recorded lines have
        model = ForwardTransformer(**cfg)
        model.set_weights(p)
        model.save_model(tmp / 'model', with_optimizer=False)
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, str(ROOT / 'evaluate_tts.py'), '--config', str(tmp / 'cfg.yaml'), '-p', str(tmp / 'model')],
                           capture_output=True, text=True, cwd=str(ROOT))
        wall = time.perf_counter() - t0
        if r.returncode != 0:
            raise SystemExit(r.stdout[-2000:] + r.stderr[-3000:])
        summary = [ln for ln in r.stdout.splitlines() if 'MCD-DTW' in ln]
        return {'lines': n_lines, 'recorded_frames': frames, 'wall_s': round(wall, 2), 'summary': summary[0] if summary else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, nargs='+', default=[100, 1000])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--lines', type=int, default=100)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to measure')
    res = dict(card(), mcd_dtw=[time_kernel(n, args.iters) for n in args.pairs])
    if args.lines:
        res['evaluate_tts'] = time_evaluate_tts(args.lines)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
