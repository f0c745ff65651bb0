"""Times ttsb_linear_fwd (csrc/gemm_tc.cu) at the shapes of the C2 step, with CUDA events after a warm-up.

    python tools/gemm_bench.py [--precision bf16x3 bf16] [--iters 20] [--windows 5]
    TTSB_LIB=<other libttsb.so> python tools/gemm_bench.py      # the same cases against another build

Cases, at the decoder's 64 x 1000 rows and at the encoder's 64 x 128:
  qkv    256 -> 768, one fp16 plane (the operands of the fp16 attention), three 256-wide tiles
  conv0  3 row-shifted segments of 256 -> 1024, ReLU, bf16 hi/lo planes (hi only in bf16), four 256-wide tiles
  conv1  3 x 1024 -> 256 with residual and LayerNorm (f32 + 16-bit planes): the image epilogue, as a control
  wo     two sources 256 | 256 -> 256 with residual and LayerNorm: a second control
Prints the card's name, power limit and top SM clock, then one JSON line per case: the median time of `--windows`
windows of `--iters` launches each, the algorithmic TFLOP/s (2·M·K·N) and the TFLOP/s of tensor products (three per
multiply-add in bf16x3).  Needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transformertts_b200 import lib  # noqa: E402
from transformertts_b200.model.models import _PackedLinear, _pad_vec  # noqa: E402

# name: (source widths, segments (src, shift, k), N, epilogue)
CASES = {
    'qkv': ([256], [(0, 0, 256)], 768, 'fp16'),
    'conv0': ([256], [(0, -1, 256), (0, 0, 256), (0, 1, 256)], 1024, 'relu_hilo'),
    'conv1': ([1024], [(0, -1, 1024), (0, 0, 1024), (0, 1, 1024)], 256, 'ln'),
    'wo': ([256, 256], [(0, 0, 256), (1, 0, 256)], 256, 'ln'),
}
ROWS = {'decoder': (64, 1000), 'encoder': (64, 128)}


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(',')]
    return {'card': name, 'power_limit': power, 'max_sm_clock': clock}


def make_case(name, B, T, precision, g, dev):
    widths, segs, N, epi = CASES[name]
    split = precision == 'bf16x3'
    K = sum(k for _, _, k in segs)
    keep = []
    a = lib.GemmArgs()
    pl = _PackedLinear(torch.randn(K, N, generator=g).to(dev) / K ** 0.5, torch.randn(N, generator=g).to(dev), [k for _, _, k in segs],
                       split, single_tile=epi == 'ln')
    keep.append(pl)
    a.B, a.T, a.N, a.block_n = B, T, pl.N, pl.block_n
    a.num_segments = len(segs)
    for s, (src, shift, k) in enumerate(segs):
        a.seg_src[s], a.seg_shift[s], a.seg_k[s] = src, shift, k
    for i, C in enumerate(widths):
        hi, lo = lib.split_bf16(torch.randn(B, T, C, generator=g).to(dev), split)
        keep += [hi, lo]
        a.a_hi[i] = hi.data_ptr()
        a.a_lo[i] = lo.data_ptr() if lo is not None else None
        a.lda[i] = C
    a.w_hi = pl.w_hi.data_ptr()
    a.w_lo = pl.w_lo.data_ptr() if pl.w_lo is not None else None
    a.bias = pl.bias.data_ptr()
    a.ld_out = pl.n_pad
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    keep.append(lens)
    a.row_len = lens.data_ptr()

    def plane(dtype):
        t = torch.empty(B, T, pl.n_pad, dtype=dtype, device=dev)
        keep.append(t)
        return t.data_ptr()

    if epi == 'fp16':
        a.out_fp16 = 1
        a.out_hi = plane(torch.float16)
    else:
        a.out_hi = plane(torch.bfloat16)
        a.out_lo = plane(torch.bfloat16) if split else None
    if epi == 'relu_hilo':
        a.relu = 1
    if epi == 'ln':
        res = torch.randn(B, T, pl.n_pad, generator=g).to(dev)
        gamma, beta = _pad_vec(torch.ones(N, device=dev), pl.n_pad), _pad_vec(torch.zeros(N, device=dev), pl.n_pad)
        keep += [res, gamma, beta]
        a.residual, a.ld_res = res.data_ptr(), pl.n_pad
        a.ln_gamma, a.ln_beta, a.ln_eps = gamma.data_ptr(), beta.data_ptr(), 1e-6
        a.out_f32 = plane(torch.float32)
    a.precision = lib.PREC_BF16X3 if split else lib.PREC_BF16
    a.impl = lib.IMPL_TCGEN05
    return a, keep, 2.0 * B * T * K * N, pl.block_n


def time_us(fn, iters, windows, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3 / iters)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--precision', nargs='+', default=['bf16x3', 'bf16'], choices=['bf16x3', 'bf16'])
    ap.add_argument('--cases', nargs='+', default=list(CASES), choices=list(CASES))
    ap.add_argument('--rows', nargs='+', default=list(ROWS), choices=list(ROWS))
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--windows', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('gemm_bench.py needs a CUDA device')
    dev = torch.device('cuda:0')
    print(json.dumps({**card(), 'lib': str(lib.library_path())}), flush=True)
    g = torch.Generator().manual_seed(1)
    for precision in args.precision:
        for rows in args.rows:
            B, T = ROWS[rows]
            for name in args.cases:
                a, keep, flops, block_n = make_case(name, B, T, precision, g, dev)
                ts = time_us(lambda: lib.linear_fwd(a), args.iters, args.windows)
                us = statistics.median(ts)
                tflops = flops / us * 1e-6
                print(json.dumps({'case': name, 'rows': rows, 'B': B, 'T': T, 'precision': precision, 'block_n': block_n,
                                  'us': round(us, 2), 'us_range': [round(min(ts), 2), round(max(ts), 2)],
                                  'algorithmic_tflops': round(tflops, 1),
                                  'product_tflops': round(tflops * (3 if precision == 'bf16x3' else 1), 1)}), flush=True)
                del keep


if __name__ == '__main__':
    main()
