"""Mel -> waveform with the MelGAN or HiFi-GAN generator for a file's worth of utterances.

    python tools/vocoder_bench.py [--clips 64] [--reps 3] [--out DIR]
    python tools/vocoder_bench.py --vocoder hifigan [--config v1|v2|v3] [--clips 64] [--reps 3] [--out DIR]
    python tools/vocoder_bench.py --vocoder bigvgan [--config base|bigvgan] [--clips 64] [--reps 3] [--out DIR]
    python tools/vocoder_bench.py --vocoder wavernn [--clips 64] [--reps 3] [--out DIR]

Workload: that of tools/synth_bench.py -- `--clips` seeded ragged clips of 2-10 s (T_c uniform in 173..862 frames), mels from
the CUDA front end (Audio.mel_spectrogram) -- and a seeded generator checkpoint (oracle/melgan_oracle.py, seed 0).  Paths:
  notebook   the generator as a torch module in fp32 on the GPU (cuDNN, TF32 off), one clip per call with its 10-frame pad,
             as the reference's synthesis notebook runs it
  bf16x3     MelGANGenerator.vocode_batch, all clips in one call, parity mode
  bf16       the same in fast mode
  griffinlim Audio.reconstruct_waveform_batch (32 iterations), for context
Every path runs once before timing; a timing is the host clock around whole calls followed by torch.cuda.synchronize(),
averaged over `--reps` calls.  FLOPs are counted from the layer shapes (multiply-adds x 2, the useful products only: the
zero-padded columns of the 32-channel stage are not counted).  Prints one JSON line: seconds per call, seconds of audio per
second, library launches per call, achieved TFLOP/s, the largest |difference| of each vocode_batch mode from the notebook
path, and the card name and power limit read in the same run.  `--out` also writes it to DIR/vocoder_bench.json.

With `--vocoder hifigan` the same clips go through a seeded HiFi-GAN generator of `--config` (oracle/hifigan_oracle.py,
seed 0), without pad frames.  Paths: `module`, jik876's generator as a torch module in fp32 on the GPU (cuDNN, TF32 off), one
clip per call as its inference.py runs it; `bf16x3` and `bf16`, HiFiGANGenerator.vocode_batch with all clips in one call.
FLOPs count the useful products of every conv (a transposed conv's output row sums 2 of its k taps per input channel).

With `--vocoder bigvgan` the same clips go through a seeded BigVGAN generator of `--config` (oracle/bigvgan_oracle.py, seed
0, v1 final layer).  Paths: `module`, the oracle's layers as a torch module in fp32 on the GPU (cuDNN, TF32 off), one clip per
call; `bf16x3` and `bf16`, BigVGANGenerator.vocode_batch with all clips in one call.  Also reported: the convs' FLOPs over the
config's channels (useful) and over the padded columns the kernel runs (issued), and, from one more call of each mode under
torch.profiler, the share of GPU time spent in the activation kernel and the bytes per second it achieves at the least
traffic it needs (every column of every clip row read and written once per plane), against the H100 SXM's 3.35 TB/s.

With `--vocoder wavernn` the workload is `--clips` seeded ragged clips of 1-10 s (T_c uniform in 81..802 frames at hop 275,
22050 Hz) of WaveRNN-normalised mels (oracle/wavernn_oracle.make_mels), then one 10 s clip alone, through a seeded MOL
generator at fatchord's defaults (target 11000, overlap 550, batched).  Paths: `torch`, fatchord's generate() loop (I, two
GRU cells, fc1-fc3, the MOL draw) as a torch fp32 module on the GPU, eager, TF32 off, over the same folds as one batch (the
folds of every clip together: fatchord runs one clip per call, which would only be slower); `bf16x3` and `bf16`,
WaveRNNGenerator.vocode_batch.  Reported: seconds per call (each path `--reps` calls after one untimed), audio seconds per second, microseconds per step (call time over
target + 2 overlap steps), library launches, GFLOP per second of audio from the shapes (the recurrence: 2 x 3.83 M
multiply-adds per sample, as the generator computes every sample of every fold), and from one more call with the kernel's
phase timers the µs per step of each segment (sampling, GRU1, GRU2, fc1, fc2, fc3): work and the grid barrier after it."""
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
from oracle import bigvgan_oracle as bo  # noqa: E402
from oracle import hifigan_oracle as ho  # noqa: E402
from oracle import melgan_oracle as mo  # noqa: E402
from oracle import wavernn_oracle as wo  # noqa: E402
from transformertts_b200 import lib  # noqa: E402
from transformertts_b200.data.audio import Audio  # noqa: E402
from transformertts_b200.model import bigvgan as bg  # noqa: E402
from transformertts_b200.model import hifigan as hg  # noqa: E402
from transformertts_b200.model import melgan as mg  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def timed(fn, reps):
    out = fn()
    torch.cuda.synchronize()
    lib.reset_launch_count()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps, lib.launch_count() / reps, out


def generator_flops(frames) -> float:
    """FLOPs of one forward over clips of frames[c] frames (10-frame pad included), from the layer shapes."""
    total = 0.0
    for L in frames:
        total += 2.0 * L * 512 * 80 * 7
        rows = L
        for _, _, cin, cout, _, u in mg.STAGES:
            rows *= u
            total += 2.0 * rows * cout * cin * 2          # each output row of a transposed conv sums 2 of its k taps per input channel
            total += 3 * 2.0 * rows * cout * cout * 5     # per ResStack block: 3-tap conv + two 1x1 convs
        total += 2.0 * rows * 32 * 7
    return total


def hifigan_flops(h: dict, frames) -> float:
    """FLOPs of one HiFi-GAN forward over clips of frames[c] frames, from the layer shapes."""
    shapes = hg.layer_shapes(h)
    rates = h['upsample_rates']
    total = 0.0
    for L in frames:
        total += 2.0 * L * int(np.prod(shapes['conv_pre'][1]))
        rows = L
        for i, u in enumerate(rates):
            cin, cout, _ = shapes[f'ups.{i}'][1]
            rows *= u
            total += 2.0 * rows * cout * cin * 2
            ch = cout
            total += sum(2.0 * rows * int(np.prod(s)) for n, (_, s) in shapes.items() if n.startswith('resblocks.') and s[0] == ch)
        total += 2.0 * rows * int(np.prod(shapes['conv_post'][1]))
    return total


def hifigan_main(args, mels, lengths):
    h = hg.load_config(args.config)
    sd = ho.init_state_dict(h, seed=0)
    module = ho.build(h, sd, dtype=torch.float32).cuda()

    def per_clip():
        with torch.no_grad():
            return [module(torch.from_numpy(m).cuda()[None])[0, 0].cpu().numpy() for m in mels]

    res = dict(workload='hifigan_vocode', config=args.config, clips=args.clips, frames=int(lengths.sum()), min_frames=int(lengths.min()),
               max_frames=int(lengths.max()), reps=args.reps, audio_s=round(float(256 * lengths.sum() / 22050), 1))
    flops = hifigan_flops(h, [int(T) for T in lengths])
    res['gflop_per_call'] = round(flops / 1e9, 1)
    res['gflop_per_audio_s'] = round(flops / 1e9 / res['audio_s'], 2)
    t, launches, w_ref = timed(per_clip, args.reps)
    res.update(module_s=round(t, 5), module_audio_s_per_s=round(res['audio_s'] / t, 1), module_tflops=round(flops / t / 1e12, 2))
    del module
    for prec in ('bf16x3', 'bf16'):
        g = hg.HiFiGANGenerator(h, device='cuda', precision=prec).load_state_dict(sd)
        t, launches, w = timed(lambda: g.vocode_batch(mels), args.reps)
        res.update({f'{prec}_s': round(t, 5), f'{prec}_audio_s_per_s': round(res['audio_s'] / t, 1), f'{prec}_launches': launches,
                    f'{prec}_tflops': round(flops / t / 1e12, 2),
                    f'{prec}_max_abs_diff_vs_module': float(max(np.abs(a - b).max() for a, b in zip(w, w_ref)))})
        del g
        torch.cuda.empty_cache()
    return res


def kernel_share(fn, name):
    """One call under torch.profiler -> (GPU seconds of the kernels whose name contains `name`, GPU seconds of all kernels)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    mine = total = 0.0
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None)
        if t is None:
            t = e.cuda_time_total
        if e.key.startswith('Memcpy') or e.key.startswith('Memset'):
            continue
        total += t
        if name in e.key:
            mine += t
    return mine / 1e6, total / 1e6


def bigvgan_main(args, mels, lengths):
    h = bg.load_config(args.config)
    sd = bo.init_state_dict(h, seed=0)
    module = bo.build(h, sd, dtype=torch.float32).cuda()

    def per_clip():
        with torch.no_grad():
            return [module(torch.from_numpy(m).cuda()[None])[0, 0].cpu().numpy() for m in mels]

    frames = int(lengths.sum())
    res = dict(workload='bigvgan_vocode', config=args.config, clips=args.clips, frames=frames, min_frames=int(lengths.min()),
               max_frames=int(lengths.max()), reps=args.reps, audio_s=round(float(256 * frames / 22050), 1),
               stage_cols=bg.stage_cols(h))
    fl = bg.conv_flops(h, frames)
    res.update(conv_gflop_useful=round(fl['useful'] / 1e9, 1), conv_gflop_issued=round(fl['issued'] / 1e9, 1),
               conv_useful_fraction=round(fl['useful'] / fl['issued'], 3))
    t, _, w_ref = timed(per_clip, args.reps)
    res.update(module_s=round(t, 4), module_audio_s_per_s=round(res['audio_s'] / t, 1))
    del module
    torch.cuda.empty_cache()
    for prec in ('bf16x3', 'bf16'):
        g = bg.BigVGANGenerator(h, device='cuda', precision=prec).load_state_dict(sd)
        t, launches, w = timed(lambda: g.vocode_batch(mels), args.reps)
        act_s, gpu_s = kernel_share(lambda: g.vocode_device(mels), 'snake_aa_kernel')
        act_bytes = bg.activation_bytes(h, frames, prec == 'bf16x3')
        res.update({f'{prec}_s': round(t, 4), f'{prec}_audio_s_per_s': round(res['audio_s'] / t, 1), f'{prec}_launches': launches,
                    f'{prec}_conv_tflops_useful': round(fl['useful'] / t / 1e12, 2),
                    f'{prec}_gpu_s': round(gpu_s, 4), f'{prec}_activation_s': round(act_s, 4),
                    f'{prec}_activation_share': round(act_s / gpu_s, 3),
                    f'{prec}_activation_tb_per_s': round(act_bytes / act_s / 1e12, 2),
                    f'{prec}_activation_of_3p35_tb_per_s': round(act_bytes / act_s / 3.35e12, 3),
                    f'{prec}_max_abs_diff_vs_module': float(max(np.abs(a - b).max() for a, b in zip(w, w_ref)))})
        del g
        torch.cuda.empty_cache()
    return res


def wavernn_torch_loop(net, fmels, target, overlap):
    """fatchord's generate() loop in torch on the GPU, the folds of all clips as one batch (before the crossfade)."""
    ms, auxs = [], []
    with torch.no_grad():
        for m in fmels:
            m_up, aux = net.conditioning(torch.from_numpy(m).cuda()[None])
            ms.append(wo.fold_with_overlap(m_up[None], target, overlap))
            auxs.append(wo.fold_with_overlap(aux[None], target, overlap))
        m_up, aux = torch.cat(ms), torch.cat(auxs)
        cells = net._cells()
        R, L = m_up.shape[:2]
        h1 = torch.zeros(R, 512, device='cuda')
        h2 = torch.zeros_like(h1)
        x = torch.zeros(R, 1, device='cuda')
        out = []
        for i in range(L):
            logits, h1, h2 = net.step_logits(cells, x, m_up[:, i], aux[:, i], h1, h2)
            u = torch.empty(R, 10, device='cuda').uniform_(1e-5, 1 - 1e-5)
            k = (logits[:, :10] - torch.log(-torch.log(u))).argmax(1, keepdim=True)
            mu, ls = logits[:, 10:20].gather(1, k), logits[:, 20:30].gather(1, k).clamp(min=wo.LOG_SCALE_MIN)
            u = torch.empty_like(mu).uniform_(1e-5, 1 - 1e-5)
            x = (mu + torch.exp(ls) * (torch.log(u) - torch.log(1. - u))).clamp(-1, 1)
            out.append(x)
        return torch.cat(out, 1).cpu()


def wavernn_phases(g, fm, steps):
    """One more call with the kernel's phase timers on (a separate run: the timers add a CTA barrier per segment) -> per
    segment of a step, µs per step: work (mean and slowest CTA, to the CTA's last warp) and the grid barrier after it (mean)."""
    tim = torch.zeros((lib.WAVERNN_CTAS, 2 * len(lib.WAVERNN_SEGMENTS)), dtype=torch.int64, device='cuda')
    g._generate(fm, None, True, wo.TARGET, wo.OVERLAP, timings=tim)
    t = tim.cpu().numpy().astype(np.float64) / 1e3 / steps
    out = {seg: dict(work=round(float(t[:, 2 * i].mean()), 1), work_max=round(float(t[:, 2 * i].max()), 1),
                     barrier=round(float(t[:, 2 * i + 1].mean()), 1)) for i, seg in enumerate(lib.WAVERNN_SEGMENTS)}
    out['total'] = round(float(t.sum(1).mean()), 1)
    return out


def wavernn_main(args):
    rng = np.random.default_rng(2024)
    sets = {'batch': [int(T) for T in rng.integers(81, 803, size=args.clips)], 'single': [802]}
    sd = wo.init_state_dict(seed=0)
    net = wo.build(sd).float().cuda()
    from transformertts_b200.model import wavernn as wrn
    res = dict(workload='wavernn_vocode', target=wo.TARGET, overlap=wo.OVERLAP, reps=args.reps)
    steps = wo.TARGET + 2 * wo.OVERLAP
    macs = 3.83e6   # I (rank-1 x_prev column and conditioning), rnn1, rnn2, fc1-fc3 per sample: 2 x 3.83 M FLOP
    for name, lengths in sets.items():
        mels = wo.make_mels(lengths, seed=7)
        fm = [wo.to_fatchord(m).astype(np.float32) for m in mels]
        rows, _ = wrn.fold_rows(lengths, 275, True, wo.TARGET, wo.OVERLAP)
        audio_s = 275 * (sum(lengths) - len(lengths)) / 22050
        r = dict(clips=len(lengths), frames=sum(lengths), folds=len(rows), audio_s=round(audio_s, 1),
                 gflop_per_audio_s=round(2 * macs * len(rows) * steps / 1e9 / audio_s, 1))
        t, _, _ = timed(lambda: wavernn_torch_loop(net, fm, wo.TARGET, wo.OVERLAP), args.reps)
        r.update(torch_s=round(t, 3), torch_audio_s_per_s=round(audio_s / t, 1), torch_us_per_step=round(t / steps * 1e6, 1))
        for prec in ('bf16x3', 'bf16'):
            g = wrn.WaveRNNGenerator(device='cuda', precision=prec).load_state_dict(sd)
            t, launches, _ = timed(lambda: g.vocode_batch(mels), args.reps)
            r.update({f'{prec}_s': round(t, 3), f'{prec}_audio_s_per_s': round(audio_s / t, 1),
                      f'{prec}_us_per_step': round(t / steps * 1e6, 1), f'{prec}_launches': launches,
                      f'{prec}_tflops': round(2 * macs * len(rows) * steps / t / 1e12, 2)})
            r[f'{prec}_phases_us_per_step'] = wavernn_phases(g, fm, steps)
            del g
        res[name] = r
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clips', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--vocoder', choices=('melgan', 'hifigan', 'bigvgan', 'wavernn'), default='melgan')
    ap.add_argument('--config', default=None, help='HiFi-GAN config: v1 (default) / v2 / v3 or a config.json path; BigVGAN config: '
                                                   'base (default) / bigvgan or a config.json path')
    args = ap.parse_args()
    if args.config is None:
        args.config = 'base' if args.vocoder == 'bigvgan' else 'v1'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    if args.vocoder == 'wavernn':
        return report(wavernn_main(args), args)
    audio = Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                  normalizer='MelGAN')
    lengths = np.random.default_rng(2024).integers(173, 863, size=args.clips)
    mels = [audio.mel_spectrogram(ao.make_clips(1, 256 * (int(T) - 1), seed=500 + c)[0]).T for c, T in enumerate(lengths)]
    if args.vocoder == 'hifigan':
        return report(hifigan_main(args, mels, lengths), args)
    if args.vocoder == 'bigvgan':
        return report(bigvgan_main(args, mels, lengths), args)
    sd = mo.init_state_dict(seed=0)
    module = mo.build(sd, dtype=torch.float32).cuda()
    pad = torch.full((1, 80, mo.PAD_FRAMES), mo.PAD_VALUE, device='cuda')

    def notebook():
        with torch.no_grad():
            return [module(torch.cat([torch.from_numpy(m).cuda()[None], pad], 2))[0, 0, :-mo.HOP * mo.PAD_FRAMES].cpu().numpy() for m in mels]

    res = dict(workload='melgan_vocode', clips=args.clips, frames=int(lengths.sum()), min_frames=int(lengths.min()),
               max_frames=int(lengths.max()), reps=args.reps, audio_s=round(float(256 * lengths.sum() / 22050), 1))
    flops = generator_flops([int(T) + mo.PAD_FRAMES for T in lengths])
    res['gflop_per_call'] = round(flops / 1e9, 1)
    res['gflop_per_audio_s'] = round(flops / 1e9 / res['audio_s'], 2)
    t, launches, w_ref = timed(notebook, args.reps)
    res.update(notebook_s=round(t, 5), notebook_audio_s_per_s=round(res['audio_s'] / t, 1), notebook_tflops=round(flops / t / 1e12, 2))
    for prec in ('bf16x3', 'bf16'):
        g = mg.MelGANGenerator(device='cuda', precision=prec).load_state_dict(sd)
        t, launches, w = timed(lambda: g.vocode_batch(mels), args.reps)
        res.update({f'{prec}_s': round(t, 5), f'{prec}_audio_s_per_s': round(res['audio_s'] / t, 1), f'{prec}_launches': launches,
                    f'{prec}_tflops': round(flops / t / 1e12, 2),
                    f'{prec}_max_abs_diff_vs_notebook': float(max(np.abs(a - b).max() for a, b in zip(w, w_ref)))})
        del g
    t, launches, _ = timed(lambda: audio.reconstruct_waveform_batch(mels, seed=0), args.reps)
    res.update(griffinlim_s=round(t, 5), griffinlim_audio_s_per_s=round(res['audio_s'] / t, 1), griffinlim_launches=launches)
    report(res, args)


def report(res, args):
    res['card'] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'vocoder_bench.json').write_text(line + '\n')


if __name__ == '__main__':
    main()
