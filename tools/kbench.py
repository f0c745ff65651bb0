"""Kernel micro-benchmarks through the C ABI (CUDA events on the current stream, after warm-up).

    python tools/kbench.py mha  [--B 64 --T 1000 --H 2 --dh 128 --precision fp16]

Prints one JSON line per case, for A/B measurements of a single kernel; the benchmark of record is bench.py.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transformertts_b200 import lib  # noqa: E402


def _time(fn, iters=30, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_mha(a):
    dev = torch.device('cuda:0')
    B, T, H, dh = a.B, a.T, a.H, a.dh
    d = H * dh
    split = a.precision == 'bf16x3'
    g = torch.Generator(device='cpu').manual_seed(1)
    qk = torch.randn(B, T, 3 * d, generator=g).to(dev)
    if a.precision == 'fp16':
        qk_hi, qk_lo = qk.half(), None
    else:
        qk_hi, qk_lo = lib.split_bf16(qk, split)
    kv_len = torch.full((B,), T, dtype=torch.int32, device=dev)
    out_hi = torch.empty(B, T, d, device=dev, dtype=torch.bfloat16)
    out_lo = torch.empty(B, T, d, device=dev, dtype=torch.bfloat16)
    m = lib.MhaArgs()
    m.B, m.T, m.H, m.dh = B, T, H, dh
    m.qk_hi = qk_hi.data_ptr()
    m.qk_lo = qk_lo.data_ptr() if split else None
    m.ld_qk, m.q_col0, m.k_col0, m.v_col0 = 3 * d, 0, d, 2 * d
    m.kv_len = kv_len.data_ptr()
    m.out_hi = out_hi.data_ptr()
    m.out_lo = out_lo.data_ptr()
    m.ld_out = d
    m.precision = {'bf16x3': lib.PREC_BF16X3, 'bf16': lib.PREC_BF16, 'fp16': lib.PREC_FP16}[a.precision]
    m.impl = lib.IMPL_TCGEN05
    ms = _time(lambda: lib.mha_fwd(m))
    flops = 4.0 * B * H * T * T * dh
    print(json.dumps({'kernel': 'mha_tc', 'B': B, 'T': T, 'H': H, 'dh': dh, 'precision': a.precision,
                      'us': round(ms * 1e3, 2),
                      'algorithmic_tflops': round(flops / ms / 1e9, 1)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('what', choices=['mha'])
    ap.add_argument('--B', type=int, default=64)
    ap.add_argument('--T', type=int, default=1000)
    ap.add_argument('--H', type=int, default=2)
    ap.add_argument('--dh', type=int, default=128)
    ap.add_argument('--precision', default='fp16')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('kbench needs a GPU')
    bench_mha(a)


if __name__ == '__main__':
    main()
