"""Helpers of tools/ab_lib.sh, which compares two builds of libttsb.so on one GPU.

    TTSB_LIB=<lib> python tools/ab_compare.py vocode DIR    # vocode_batch waveforms of MelGAN and HiFi-GAN V1 -> DIR/*.npy
    python tools/ab_compare.py compare DIR_A DIR_B          # every array of DIR_A against DIR_B, element by element
    python tools/ab_compare.py summary OUT                  # range of each arm's bench.py results in OUT

`vocode` runs the seeded 64-clip workload of tools/vocoder_bench.py (same clip lengths, clips and generator checkpoints) in
bf16x3 and bf16.  `compare` reports, per array, how many elements differ in their bits and the largest |difference|; it
exits with 1 if any array differs or is missing on one side."""
import json
import statistics
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def vocode(out: Path) -> None:
    import torch

    from oracle import audio_oracle as ao
    from oracle import hifigan_oracle as ho
    from oracle import melgan_oracle as mo
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.model import hifigan as hg
    from transformertts_b200.model import melgan as mg

    out.mkdir(parents=True, exist_ok=True)
    audio = Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                  normalizer='MelGAN')
    lengths = np.random.default_rng(2024).integers(173, 863, size=64)
    mels = [audio.mel_spectrogram(ao.make_clips(1, 256 * (int(T) - 1), seed=500 + c)[0]).T for c, T in enumerate(lengths)]
    h = hg.load_config('v1')
    for prec in ('bf16x3', 'bf16'):
        gens = {'melgan': mg.MelGANGenerator(device='cuda', precision=prec).load_state_dict(mo.init_state_dict(seed=0)),
                'hifigan_v1': hg.HiFiGANGenerator(h, device='cuda', precision=prec).load_state_dict(ho.init_state_dict(h, seed=0))}
        for name, g in gens.items():
            wav = g.vocode_batch(mels)
            np.save(out / f'{name}_{prec}.npy', np.concatenate([np.asarray(w, dtype=np.float32).ravel() for w in wav]))
        del gens
        torch.cuda.empty_cache()


def compare(a: Path, b: Path) -> int:
    names = sorted({p.name for p in a.glob('*.npy')} | {p.name for p in b.glob('*.npy')})
    bad = 0
    for n in names:
        if not (a / n).exists() or not (b / n).exists():
            print(f'{n}: only in {a if (a / n).exists() else b}')
            bad += 1
            continue
        x, y = np.load(a / n), np.load(b / n)
        if x.shape != y.shape or x.dtype != y.dtype:
            print(f'{n}: shape/dtype {x.shape} {x.dtype} vs {y.shape} {y.dtype}')
            bad += 1
            continue
        xb, yb = x.view(np.uint8).reshape(x.size, -1), y.view(np.uint8).reshape(y.size, -1)
        ndiff = int((xb != yb).any(axis=1).sum()) if x.size else 0
        dmax = float(np.nanmax(np.abs(x.astype(np.float64) - y.astype(np.float64)))) if ndiff else 0.0
        print(f'{n}: {x.size} elements, {ndiff} differ, max |diff| {dmax:.3g}')
        bad += ndiff > 0
    print(f'{len(names)} arrays, {bad} differ')
    return 1 if bad else 0


def summary(out: Path) -> None:
    def rng(v):
        v = [x for x in v if x is not None]
        return {'min': min(v), 'median': statistics.median(v), 'max': max(v), 'n': len(v)} if v else None

    res = {'card': (out / 'card.txt').read_text().strip() if (out / 'card.txt').exists() else None}
    for arm in ('A', 'B'):
        recs = [json.loads(l) for l in (out / f'infer_{arm}.jsonl').read_text().splitlines() if l.startswith('{')]
        r = {'value': rng([x['value'] for x in recs]),
             'ms_per_step': rng([x['ms_per_step'] for x in recs]),
             'roofline_achieved_tflops': rng([x['roofline']['achieved'] for x in recs]),
             'conv_share_of_step': rng([x['roofline']['share_of_step'] for x in recs]),
             'fast_mode_value': rng([(x.get('fast_mode') or {}).get('value') for x in recs])}
        for mode in ('train', 'aligner'):
            p = out / f'{mode}_{arm}.jsonl'
            if p.exists():
                r[mode] = rng([json.loads(l)['value'] for l in p.read_text().splitlines() if l.startswith('{')])
        res[arm] = r
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    cmd = sys.argv[1] if len(sys.argv) > 1 else ''
    if cmd == 'vocode' and len(sys.argv) == 3:
        vocode(Path(sys.argv[2]))
    elif cmd == 'compare' and len(sys.argv) == 4:
        sys.exit(compare(Path(sys.argv[2]), Path(sys.argv[3])))
    elif cmd == 'summary' and len(sys.argv) == 3:
        summary(Path(sys.argv[2]))
    else:
        sys.exit(__doc__)
