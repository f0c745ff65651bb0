#!/usr/bin/env python
"""Objective scores of ForwardTransformer checkpoints on the validation split (no reference counterpart).

    python evaluate_tts.py --config CFG -p MODEL_DIR [-o OUTDIR]
    python evaluate_tts.py --config CFG -p WEIGHTS_DIR --weights_glob 'step_*'          # every checkpoint, in step order
    python evaluate_tts.py --config CFG -p MODEL_DIR --vocoder melgan --vocoder_checkpoint melgan.pt
    python evaluate_tts.py --config CFG -p MODEL_DIR --vocoder hifigan --vocoder_checkpoint g_02500000 [--vocoder_config v1]
    python evaluate_tts.py --config CFG -p MODEL_DIR --vocoder bigvgan --vocoder_checkpoint bigvgan_generator.pt [--vocoder_config base]
    python evaluate_tts.py --config CFG -p MODEL_DIR --vocoder wavernn --vocoder_checkpoint latest_weights.pyt
    python evaluate_tts.py --config CFG -p MODEL_DIR --vocoder melgan --vocoder_checkpoint melgan.pt --f0    # + pitch / voicing
    python evaluate_tts.py --config CFG -p MODEL_DIR --vocoder melgan --vocoder_checkpoint melgan.pt --mcep  # + WORLD MCD

The validation split is read as train_tts.py reads it (``valid_metadata``, ``mels``, ``durations`` and ``char_pitch`` of the
config's data directory; ``pitch_stats.pkl`` for pitch errors in Hz when it exists).  For every checkpoint:

* free running (``predict_batch`` of the phonemes alone): MCD-DTW against the recorded mel, duration MAE in frames per phoneme,
  the exact-match rate and the ratio of predicted to recorded frames, pitch RMSE over the phonemes with a target pitch != 0;
* teacher forced (``predict_batch`` with the target durations and pitch): MCD-DTW;
* with ``--vocoder``: the free-running mels and the recorded mels (copy synthesis: the vocoder's own floor) are vocoded, their
  log-mels re-extracted on the GPU and scored against the recorded mel;
* with ``--f0`` (needs ``--vocoder`` and the recorded frame pitch ``pitch.<audio>/<name>.npy`` with ``pitch_stats.pkl``): the
  WORLD F0 of both sets of waveforms (DIO + StoneMask on the GPU, at the frame period of the training data) against the
  recorded frame pitch along each line's MCD-DTW warping path: gross pitch error (GPE, |f / f_ref - 1| > 20 %), voicing
  decision error (VDE), F0 frame error (FFE) and the F0 RMSE in cents;
* with ``--mcep`` (needs ``--vocoder`` and the recordings under the config's ``wav_directory``, rebuilt as
  create_training_data.py prepared them): the WORLD mel-cepstral distortion of both sets of waveforms against the recordings,
  the MCD published work reports: CheapTrick envelopes at the DIO / StoneMask F0, pysptk's sp2mc to ``--mcep_order`` (24) at
  ``--mcep_alpha`` (default: pysptk's mcepalpha of the sampling rate, 0.455 at 22050 Hz), DTW over mc_1..mc_order.

The plain MCD is the DCT of the 80-bin natural-log mel (coefficients 1..24), not the SPTK / WORLD mel-cepstrum: compare its
numbers with each other; ``--mcep`` gives the one comparable to papers (see transformertts_b200/utils/evaluation.py).  Per-line
and corpus-mean values go to
``<OUTDIR>/evaluation.json`` (default OUTDIR: MODEL_DIR), one entry per checkpoint; one summary line per checkpoint is printed.
"""
from __future__ import annotations

import re
from argparse import ArgumentParser
from pathlib import Path


def parse_args(argv=None):
    parser = ArgumentParser()
    parser.add_argument('--config', required=True, type=str)
    parser.add_argument('--path', '-p', dest='path', required=True, type=str)
    parser.add_argument('--weights_glob', default=None, type=str, help="checkpoint directories under --path, e.g. 'step_*'")
    parser.add_argument('--outdir', '-o', dest='outdir', default=None, type=str)
    parser.add_argument('--n_ceps', default=24, type=int)
    parser.add_argument('--vocoder', default=None, choices=('griffinlim', 'melgan', 'hifigan', 'bigvgan', 'wavernn'))
    parser.add_argument('--vocoder_checkpoint', default=None, type=str)
    parser.add_argument('--vocoder_config', default=None, type=str,
                        help='HiFi-GAN config (a config.json path or v1 / v2 / v3) or BigVGAN config (a config.json path or base / bigvgan); '
                             'default: the config.json beside the checkpoint')
    parser.add_argument('--f0', action='store_true',
                        help='also score the F0 and voicing of the vocoded audio against the recorded frame pitch (needs --vocoder)')
    parser.add_argument('--mcep', action='store_true',
                        help='also score the WORLD mel-cepstral distortion of the vocoded audio against the recordings (needs --vocoder '
                             'and wav_directory)')
    parser.add_argument('--mcep_order', default=24, type=int)
    parser.add_argument('--mcep_alpha', default=None, type=float, help='all-pass constant (default: mcepalpha of the sampling rate)')
    args = parser.parse_args(argv)
    if args.f0 and args.vocoder is None:
        parser.error('--f0 scores vocoded audio: it needs --vocoder')
    if args.mcep and args.vocoder is None:
        parser.error('--mcep scores vocoded audio: it needs --vocoder')
    if (args.mcep_alpha is not None or args.mcep_order != 24) and not args.mcep:
        parser.error('--mcep_order and --mcep_alpha apply to --mcep only')
    if args.mcep and args.mcep_order < 1:
        parser.error(f'--mcep_order must be at least 1, got {args.mcep_order}')
    if args.mcep_alpha is not None and not abs(args.mcep_alpha) < 1:
        parser.error(f'--mcep_alpha must be in (-1, 1), got {args.mcep_alpha}')
    if args.vocoder in ('melgan', 'hifigan', 'bigvgan', 'wavernn') and args.vocoder_checkpoint is None:
        parser.error(f'--vocoder {args.vocoder} needs --vocoder_checkpoint PATH')
    if args.vocoder_config is not None and args.vocoder not in ('hifigan', 'bigvgan'):
        parser.error('--vocoder_config applies to --vocoder hifigan and bigvgan only')
    return args


def checkpoints(path: Path, pattern):
    """The model directories to score: `path` itself, or its sub-directories matching `pattern` in step order."""
    if pattern is None:
        return [path]
    found = [p for p in path.glob(pattern) if (p / 'config.yaml').exists()]
    if not found:
        raise SystemExit(f'no checkpoint directory matches {path / pattern}')
    step = lambda p: int(m.group(1)) if (m := re.search(r'(\d+)$', p.name)) else -1
    return sorted(found, key=lambda p: (step(p), p.name))


def main(argv=None):
    args = parse_args(argv)
    import yaml
    from predict_tts import VOCODE_CHUNK, load_vocoder, vocode_chunk
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils import evaluation as ev
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager

    cm = TrainingConfigManager(args.config)
    ev.natural_log_mels(cm.config, 'config')
    if args.mcep and cm.wav_directory is None:
        raise SystemExit('--mcep scores against the recordings: the config\'s paths settings need a wav_directory')
    vs = ev.load_validation_set(cm, frame_pitch=args.f0, recordings=args.mcep)
    mcep_alpha = None
    if args.mcep:
        mcep_alpha = args.mcep_alpha if args.mcep_alpha is not None else ev.mcep_alpha(int(cm.config['sampling_rate']))
    root = Path(args.path)
    results = []
    vocoder = None
    for ckpt in checkpoints(root, args.weights_glob):
        model = ForwardTransformer.load_model(ckpt)
        with open(ckpt / 'config.yaml') as f:
            step = yaml.safe_load(f).get('step', model.step)
        ev.natural_log_mels(model.config)
        audio = vocode = None
        if args.vocoder is not None:
            audio = Audio.from_config(model.config)
            if vocoder is None:
                vocoder = load_vocoder(args.vocoder, args.vocoder_checkpoint, args.vocoder_config, model)

            def vocode(mels, audio=audio):
                wavs = []
                for start in range(0, len(mels), VOCODE_CHUNK):
                    part = [m.T for m in mels[start:start + VOCODE_CHUNK]]
                    wavs.extend(vocode_chunk(vocoder, audio, part, start))
                return wavs
        res = ev.evaluate_model(model, vs, n_ceps=args.n_ceps, vocode=vocode, audio=audio, f0=args.f0, mcep=args.mcep,
                                mcep_order=args.mcep_order, mcep_alpha=mcep_alpha)
        res = dict(checkpoint=str(ckpt), step=int(step), **res)
        results.append(res)
        print(ev.summary_line(f'{ckpt.name} (step {step})', res), flush=True)
    out = Path(args.outdir) if args.outdir is not None else root
    summary = {'config': str(args.config), 'n_ceps': args.n_ceps, 'vocoder': args.vocoder, 'lines': len(vs.names)}
    if args.mcep:
        summary.update(mcep_order=args.mcep_order, mcep_alpha=mcep_alpha)
    ev.write_json(dict(summary, checkpoints=results), out / 'evaluation.json')
    print(f'wrote {out / "evaluation.json"}')
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
