#!/usr/bin/env python
"""Time ttsb_mcd_dtw_path against ttsb_mcd_dtw, and evaluate_tts.py --f0, on the GPU.

    python tools/dtw_path_bench.py [--pairs 100 1000] [--iters 20] [--lines 100] [--out result.json]

* ttsb_mcd_dtw and ttsb_mcd_dtw_path on the seeded pairs of 200-1,200 frames of tools/eval_bench.py (80 mels, K = 24), CUDA
  events around `--iters` calls of each after a warm-up, alternating the two, per batch size: the difference is the cost of
  recording each cell's choice and tracing the paths back.  The path variant's outputs are checked against ttsb_mcd_dtw's.
* evaluate_tts.py --vocoder griffinlim --f0: the wall time of one run (a fresh process) on a temporary data directory of
  `--lines` validation lines with recorded mels of 200-1,200 frames and their frame pitch, scored with a seeded LJ256 model, and
  the same run without --f0.
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
sys.path.insert(0, str(ROOT / 'tools'))

from eval_bench import _mels, card  # noqa: E402


def time_kernels(n_pairs: int, iters: int) -> dict:
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
    cost_p, len_p = torch.empty_like(cost), torch.empty_like(path_len)
    entries = int(sum(int(p.shape[0]) + int(q.shape[0]) - 1 for p, q in zip(a, b)))
    path = torch.empty((entries, 2), dtype=torch.int32, device='cuda')
    calls = {'mcd_dtw': lambda: lib.mcd_dtw(x, xo, y, yo, dct, ev.KAPPA, cost, path_len),
             'mcd_dtw_path': lambda: lib.mcd_dtw_path(x, xo, y, yo, dct, ev.KAPPA, cost_p, len_p, path)}
    for call in calls.values():
        for _ in range(3):
            call()
    torch.cuda.synchronize()
    if not (torch.equal(cost, cost_p) and torch.equal(path_len, len_p)):
        raise SystemExit('ttsb_mcd_dtw_path disagrees with ttsb_mcd_dtw')
    ms = {k: [] for k in calls}
    for _ in range(3):   # alternate the two, so drift on a shared machine falls on both
        for name, call in calls.items():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(iters):
                call()
            end.record()
            end.synchronize()
            ms[name].append(start.elapsed_time(end) / iters)
    cells = int(sum(int(p.shape[0]) * int(q.shape[0]) for p, q in zip(a, b)))
    best = {k: min(v) for k, v in ms.items()}
    return {'pairs': n_pairs, 'cells': cells, 'path_entries': entries,
            'ms_per_call': {k: round(v, 3) for k, v in best.items()},
            'ms_per_call_all': {k: [round(t, 3) for t in v] for k, v in ms.items()},
            'path_over_plain': round(best['mcd_dtw_path'] / best['mcd_dtw'], 3),
            'workspace_bytes': {'mcd_dtw': lib.mcd_dtw_workspace_bytes(xo, yo, ev.DEFAULT_N_CEPS),
                                'mcd_dtw_path': lib.mcd_dtw_path_workspace_bytes(xo, yo, ev.DEFAULT_N_CEPS)}}


def time_evaluate_tts_f0(n_lines: int) -> dict:
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
        for d in (cm.mel_dir, cm.duration_dir, cm.pitch_per_char, cm.pitch_dir):
            d.mkdir(parents=True, exist_ok=True)
        rows, frames = [], 0
        for i, mel in enumerate(_mels(n_lines, rng)):
            n_ph = int(rng.integers(len(mel) // 8, len(mel) // 5))
            name = f'e{i:04d}'
            np.save(cm.mel_dir / f'{name}.npy', mel)
            np.save(cm.duration_dir / f'{name}.npy', np.bincount(rng.integers(0, n_ph, len(mel)), minlength=n_ph).astype(np.int32))
            np.save(cm.pitch_per_char / f'{name}.npy', rng.normal(0, 1, n_ph).astype(np.float32))
            p = rng.normal(0, 1, len(mel))
            p[rng.random(len(mel)) < 0.3] = 0.0
            np.save(cm.pitch_dir / f'{name}.npy', p)
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
        out = {'lines': n_lines, 'recorded_frames': frames}
        for key, extra in (('wall_s_f0', ['--f0']), ('wall_s_without_f0', [])):
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
    ap.add_argument('--pairs', type=int, nargs='+', default=[100, 1000])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--lines', type=int, default=100)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: nothing to measure')
    res = dict(card(), dtw=[time_kernels(n, args.iters) for n in args.pairs])
    if args.lines:
        res['evaluate_tts_griffinlim'] = time_evaluate_tts_f0(args.lines)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + '\n')


if __name__ == '__main__':
    main()
