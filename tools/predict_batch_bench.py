"""Lines per second of text -> mel: ForwardTransformer.predict one line per call against predict_batch.

    python tools/predict_batch_bench.py [--lines 256] [--batch-size 64] [--out result.json]
    python tools/predict_batch_bench.py --ln-gemm [--libs LIB_A LIB_B --rounds 3]

Lines mode: seeded LJ256 weights (oracle.forward_oracle.init_params, seed 7, duration bias 6 so that a phoneme lasts a few
frames, as a trained model's do) and 256 seeded phoneme lines of 20-180 tokens.  The per-line loop and predict_batch each
run eager and with cuda_graphs=True: one untimed pass over all lines (module loads, allocator, graph captures), then timed
passes, each ending in a device synchronise.  Reports lines/s and mel frames/s, with the card's name and power limit read
by nvidia-smi in the same run.

--ln-gemm: CUDA-event time of the fused LayerNorm GEMMs at the C2 shape (64 rows of 1024 frames, d = 256): the decoder's
output projection (K = 512) and the last conv of a conv block (K = 3 x 1024), bf16x3 and bf16.  With --libs the
measurement runs in a fresh process per library (TTSB_LIB), alternating the libraries for --rounds rounds.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card() -> dict:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(',')]
    return {'gpu': name, 'power_limit': power}


def make_lines(n: int, seed: int):
    import numpy as np

    from oracle import forward_oracle as fo
    g = np.random.default_rng(seed)
    return [g.integers(1, fo.VOCAB_SIZE, size=int(k)).astype(np.int32) for k in g.integers(20, 181, size=n)]


def make_model(cuda_graphs: bool):
    import torch

    from oracle import forward_oracle as fo
    from transformertts_b200.model.models import ForwardTransformer
    p = fo.init_params(fo.CONFIGS['LJ256'], seed=7)
    p['dur_pred.out.b'] = torch.tensor([6.0])
    m = ForwardTransformer(**fo.CONFIGS['LJ256'], cuda_graphs=cuda_graphs, max_cached_graphs=64)
    m.set_weights(p)
    return m


def lines_mode(args) -> dict:
    import torch
    lines = make_lines(args.lines, seed=11)
    res = dict(card(), lines=len(lines), tokens=int(sum(len(t) for t in lines)), batch_size=args.batch_size)
    for graphs in (False, True):
        m = make_model(graphs)
        runs = {'predict_loop': lambda: [m.predict(t, encode=False) for t in lines],
                'predict_batch': lambda: m.predict_batch(lines, batch_size=args.batch_size)}
        for name, fn in runs.items():
            out = fn()                                   # untimed pass
            frames = sum(int(o['mel_lengths'][0]) if name == 'predict_loop' else o['mel_lengths'] for o in out)
            del out
            torch.cuda.synchronize()
            times = []
            for _ in range(args.passes):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
            best = min(times)
            key = f"{name}{'_graphs' if graphs else '_eager'}"
            res[key] = {'s_per_pass': [round(t, 4) for t in times], 'lines_per_s': round(len(lines) / best, 1),
                        'mel_frames_per_s': round(frames / best), 'mel_frames': frames}
            print(key, res[key], file=sys.stderr, flush=True)
    return res


def ln_gemm_mode(args) -> dict:
    import torch

    from transformertts_b200.model.models import ForwardTransformer, _PackedLinear
    from oracle import forward_oracle as fo
    B, T, N = 64, 1024, 256
    res = dict(card(), lib=os.environ.get('TTSB_LIB', 'default'), shape=f'B={B} T={T} N={N}')
    g = torch.Generator(device='cpu').manual_seed(0)
    for precision in ('bf16x3', 'bf16'):
        m = ForwardTransformer(**fo.CONFIGS['LJ256'], precision=precision)
        m._prepare()
        for name, K in (('wo', 512), ('conv_last', 3 * 1024)):
            x = torch.randn(B, T, K // (3 if name == 'conv_last' else 1), generator=g).cuda() * 0.5
            Kx = x.shape[-1]
            pl = _PackedLinear((torch.randn(K, N, generator=g) / K ** 0.5).cuda(), torch.zeros(N).cuda(), [Kx] * (K // Kx),
                               m._split, single_tile=True)
            hi = x.to(torch.bfloat16)
            lo = (x - hi.float()).to(torch.bfloat16) if m._split else None
            r = torch.randn(B, T, N, generator=g).cuda()
            rh = r.to(torch.bfloat16)
            ln = (torch.ones(N).cuda(), torch.zeros(N).cuda())
            lens = torch.full((B,), T, dtype=torch.int32, device='cuda')
            out = [torch.empty((B, T, N), dtype=torch.bfloat16, device='cuda') for _ in range(2)]
            kw = dict(residual_pair=(rh, (r - rh.float()).to(torch.bfloat16))) if m._split else dict(residual=r)
            shifts = [0] if K == Kx else [-1, 0, 1]

            def run():
                m._gemm(pl, B, T, [(hi, lo, Kx, 0)], [0] * len(shifts), shifts, ln=ln, row_len=lens, out_hi=out[0],
                        out_lo=out[1] if m._split else None, **kw)
            for _ in range(10):
                run()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.reps
            res[f'{precision}_{name}_us'] = round(1e3 * ms, 2)
            res[f'{precision}_{name}_tflops'] = round(2.0 * B * T * K * N / (ms * 1e-3) / 1e12, 1)
    return res


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument('--lines', type=int, default=256)
    ap.add_argument('--batch-size', type=int, default=64)
    ap.add_argument('--passes', type=int, default=3)
    ap.add_argument('--ln-gemm', action='store_true')
    ap.add_argument('--libs', nargs='+', default=None)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=200)
    ap.add_argument('--out', default=None)
    args = ap.parse_args(argv)
    if args.ln_gemm and args.libs:
        results = []
        for _ in range(args.rounds):
            for lib in args.libs:
                env = dict(os.environ, TTSB_LIB=str(Path(lib).resolve()))
                r = subprocess.run([sys.executable, __file__, '--ln-gemm', '--reps', str(args.reps)], env=env, capture_output=True,
                                   text=True, check=True)
                results.append(json.loads(r.stdout.strip().splitlines()[-1]))
        res = {'rounds': results}
    else:
        res = ln_gemm_mode(args) if args.ln_gemm else lines_mode(args)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + '\n')
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
