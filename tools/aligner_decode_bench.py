"""Autoregressive Aligner decoding on the GPU: the reference-faithful `Aligner.predict` (the whole decoder re-run on the whole
prefix every iteration, one sentence per call) against the cached batch decode `Aligner.predict_batch`, eager and as a
replayed CUDA-graph step.

    python tools/aligner_decode_bench.py [--reps N] [--max-length 800] [--out DIR]
    python tools/aligner_decode_bench.py --profile [--out DIR]    # device time of one decode step per kernel (torch.profiler)

Set-up: the shipped aligner_settings (A5), seeded weights, stop-head bias (6, 0, -6) so every row runs to max_length (800 =
the C5 frame count), 130 tokens per row (C5), r = 1 and r = 10.  Every shape is run once before it is timed; a timing is the
host clock around whole calls, which end in a device synchronise (the final host read of the row lengths).  Per-step figures
of predict_batch divide the whole call, encoder and cross-attention K|V prefill included, by the steps run.  Prints one JSON
line per measurement and the largest |mel difference| between predict and predict_batch at B = 1; `--out` also writes them
to DIR/aligner_decode_bench.json.

--profile runs instead one eager predict_batch call (r = 1, max_length 100, B = 1 and 16, after a warm-up call) under
torch.profiler and prints, per kernel, launches per step, mean µs per launch and the share of the call's device time.  It is a
run of its own because tracing slows the host."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle import aligner_oracle as alo  # noqa: E402
from transformertts_b200 import lib  # noqa: E402
from transformertts_b200.model.aligner import Aligner  # noqa: E402

TP = 130


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def timed(fn, reps):
    """Run fn once (warm-up of every shape), then `reps` times; seconds per call, library launches per call, last result."""
    out = fn()
    torch.cuda.synchronize()
    lib.reset_launch_count()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps, lib.launch_count() / reps, out


def profile_split(models, tok, out_dir):
    from torch.profiler import ProfilerActivity, profile
    m = models[False]
    m.set_constants(reduction_factor=1)
    rows = []
    for B in (1, 16):
        m.predict_batch(tok[:B], max_length=100)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.predict_batch(tok[:B], max_length=100)
            torch.cuda.synchronize()
        steps = m.decode_stats['steps']
        evs = [(e.key, e.count, e.self_device_time_total) for e in prof.key_averages()]
        evs = [e for e in evs if e[2] > 0]
        total = sum(t for _, _, t in evs)
        for name, count, t in sorted(evs, key=lambda e: -e[2])[:8]:
            rows.append({'B': B, 'kernel': name[:90], 'launches_per_step': count / steps, 'us_per_launch': t / count,
                         'share_of_device_time': t / total})
            print(json.dumps(rows[-1]), flush=True)
    if out_dir:
        Path(out_dir).mkdir(parents=True, exist_ok=True)
        (Path(out_dir) / 'aligner_decode_profile.json').write_text(json.dumps(rows, indent=1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--predict-reps', type=int, default=1)
    ap.add_argument('--max-length', type=int, default=800)
    ap.add_argument('--out', default=None)
    ap.add_argument('--profile', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('aligner_decode_bench needs a CUDA device')
    cfg = alo.ALIGNER_CONFIGS['A5']
    params = alo.init_aligner_params(cfg, seed=7)
    params['postnet.stop.b'] = torch.tensor((6.0, 0.0, -6.0))
    tok, _, _ = alo.make_aligner_inputs(cfg, 16, TP, 8, seed=500, ragged=False)
    models = {}
    for graphs in (False, True):
        models[graphs] = Aligner.from_config(dict(cfg), max_r=cfg['max_r'])
        models[graphs].cuda_graphs = graphs
        models[graphs].set_weights(params)
    gpu = card()
    print(json.dumps({'card': gpu}), flush=True)
    if args.profile:
        return profile_split(models, tok, args.out)
    results = []

    def report(rec):
        rec['card'] = gpu
        results.append(rec)
        print(json.dumps(rec), flush=True)

    for r in (1, 10):
        iters = args.max_length // r + 1
        frames = iters * r
        for m in models.values():
            m.set_constants(reduction_factor=r)
        m = models[False]
        sec, launches, ref = timed(lambda: m.predict(tok[0], max_length=args.max_length, encode=False, verbose=False), args.predict_reps)
        report({'what': 'predict', 'r': r, 'B': 1, 'graphs': False, 'iterations': iters, 's_per_call': sec, 'frames_per_s': frames / sec,
                'us_per_iteration': 1e6 * sec / iters, 'launches_per_iteration': launches / iters, 'host_reads_per_call': iters})
        for B in (1, 16):
            for graphs in (False, True):
                m = models[graphs]
                sec, launches, out = timed(lambda: m.predict_batch(tok[:B], max_length=args.max_length), args.reps)
                st = m.decode_stats
                assert all(o['mel'].shape[0] == frames for o in out)
                rec = {'what': 'predict_batch', 'r': r, 'B': B, 'graphs': graphs, 'iterations': st['steps'], 's_per_call': sec,
                       'frames_per_s': B * frames / sec, 'us_per_step': 1e6 * sec / st['steps'],
                       'launches_per_step': launches / st['steps'], 'host_reads_per_call': st['host_reads']}
                if B == 1:
                    rec['max_abs_mel_diff_vs_predict'] = float((out[0]['mel'].cpu() - ref['mel'].float().cpu()).abs().max())
                report(rec)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'aligner_decode_bench.json').write_text(json.dumps(results, indent=1))


if __name__ == '__main__':
    main()
