#!/usr/bin/env python
"""Text-to-speech from the command line: the reference's ``predict_tts.py``.

    python predict_tts.py -f lines.txt [-p MODEL_DIR | --step 95000] [-o OUTDIR] [-m] [-s] [-v]
    python predict_tts.py -t "phoneme string" ...
    python predict_tts.py -f lines.txt --vocoder melgan --vocoder_checkpoint melgan.pt ...
    python predict_tts.py -f lines.txt --vocoder hifigan --vocoder_checkpoint g_02500000 [--vocoder_config v1|config.json] ...
    python predict_tts.py -f lines.txt --vocoder bigvgan --vocoder_checkpoint bigvgan_generator.pt [--vocoder_config base|bigvgan|config.json] ...
    python predict_tts.py -f lines.txt --vocoder wavernn --vocoder_checkpoint latest_weights.pyt ...

Every input line is tokenised and the lines are turned into mels by ``ForwardTransformer.predict_batch`` (sorted by length,
a padded batch per forward pass; each mel is bit for bit what ``predict`` gives the line alone, which is how the reference
predicts, one line per call).  The mels are vocoded on the GPU with ``Audio.reconstruct_waveform_batch`` (mel inversion + 32 Griffin-Lim iterations), in chunks of
``VOCODE_CHUNK`` lines so that device memory stays bounded however long the file is.  With ``--vocoder melgan`` the chunks
go through a MelGAN generator instead (``MelGANGenerator.vocode_batch``, weights from ``--vocoder_checkpoint``), as the
reference's synthesis notebook does one line at a time; a line of T frames then gives 256 T samples (Griffin-Lim:
256 (T - 1)).  With ``--vocoder hifigan`` they go through a HiFi-GAN generator (``HiFiGANGenerator.vocode_batch``, a
jik876/hifi-gan checkpoint; its config is ``--vocoder_config``, a config.json path or v1 / v2 / v3, by default the
config.json beside the checkpoint), also 256 T samples per line; HiFi-GAN takes the MelGAN normaliser's log-mels, so a
model with another ``normalizer`` is refused.  ``--vocoder bigvgan`` does the same with an NVIDIA/BigVGAN generator
(``BigVGANGenerator.vocode_batch``; config base / bigvgan or a config.json, by default the one beside the checkpoint), which
also refuses a config whose ``sampling_rate``, ``num_mels``, ``hop_size`` or ``fmax`` differs from the model's audio
settings.  With ``--vocoder wavernn`` they go through a fatchord/WaveRNN generator
(``WaveRNNGenerator.vocode_batch``, batched folds of 11000 + 2 550 samples), line i sampled with seed i; its hop is the
product of its upsample factors and must equal the model's, the model must use the ``WaveRNN`` normaliser, a line of T
frames gives 275 (T - 1) samples at hop 275, and a line below 21 frames is refused.  Output:
``<outdir>/outputs/<fname>/<fname>_<data_name>_<git_hash>_<step>.wav``, the concatenation of all lines; with ``--single`` also
``..._<i>.wav`` per line, with ``--store_mel`` ``..._<i>.mel.npy`` (the (T, n_mels) mel of line i).

Differences from the reference:
  * Input lines are phoneme strings in the model's alphabet: the espeak phonemizer is not part of this project.  A symbol
    outside the alphabet raises, as the reference's tokenizer does.  Blank lines are skipped.
  * The Griffin-Lim phase of line i is drawn with seed i (see ``Audio.reconstruct_waveform``), so a run is reproducible; the
    reference draws it from numpy's unseeded global RNG.
  * Config keys that a saved model lacks (``data_name``, ``git_hash``, ``step``) are named ``MISSING`` in the file name.  The
    step is taken from the model directory's config.yaml, else from ``--step`` when the LJSpeech archive is loaded.
  * The .wav files are 16-bit PCM with samples beyond full scale clipped (``Audio.save_wav``).
"""
from __future__ import annotations

from argparse import ArgumentParser
from pathlib import Path

import numpy as np

VOCODE_CHUNK = 16    # lines vocoded per reconstruct_waveform_batch / vocode_batch call
MISSING = 'unknown'  # file-name placeholder for a config key the model does not carry


def parse_args(argv=None):
    parser = ArgumentParser()
    parser.add_argument('--path', '-p', dest='path', default=None, type=str)
    parser.add_argument('--step', dest='step', default='90000', type=str)
    parser.add_argument('--text', '-t', dest='text', default=None, type=str)
    parser.add_argument('--file', '-f', dest='file', default=None, type=str)
    parser.add_argument('--outdir', '-o', dest='outdir', default=None, type=str)
    parser.add_argument('--store_mel', '-m', dest='store_mel', action='store_true')
    parser.add_argument('--verbose', '-v', dest='verbose', action='store_true')
    parser.add_argument('--single', '-s', dest='single', action='store_true')
    parser.add_argument('--vocoder', dest='vocoder', default='griffinlim', choices=('griffinlim', 'melgan', 'hifigan', 'bigvgan', 'wavernn'))
    parser.add_argument('--vocoder_checkpoint', dest='vocoder_checkpoint', default=None, type=str)
    parser.add_argument('--vocoder_config', dest='vocoder_config', default=None, type=str,
                        help='HiFi-GAN config (a config.json path or v1 / v2 / v3) or BigVGAN config (a config.json path or base / bigvgan); '
                             'default: the config.json beside the checkpoint')
    args = parser.parse_args(argv)
    if args.vocoder in ('melgan', 'hifigan', 'bigvgan', 'wavernn') and args.vocoder_checkpoint is None:
        parser.error(f'--vocoder {args.vocoder} needs --vocoder_checkpoint PATH')
    if args.vocoder_config is not None and args.vocoder not in ('hifigan', 'bigvgan'):
        parser.error('--vocoder_config applies to --vocoder hifigan and bigvgan only')
    return args


NO_INPUT_MESSAGE = 'Specify either an input text (-t "some text") or a text input file (-f /path/to/file.txt)'


def read_input(args):
    """-> (fname, lines), or (None, None) when neither --file nor --text is given (reference: predict_tts.py:22-33)."""
    if args.file is not None:
        with open(args.file, 'r') as f:
            text = [line.rstrip('\r\n') for line in f]
        return Path(args.file).stem, [line for line in text if line.strip()]
    if args.text is not None:
        return 'custom_text', [args.text]
    return None, None


def output_names(outdir, fname: str, config: dict, step):
    """-> (directory, file-name stem, path of the combined .wav) as the reference builds them (predict_tts.py:35-44)."""
    data_name = config.get('data_name', MISSING)
    git_hash = config.get('git_hash', MISSING)
    step = config.get('step', MISSING if step is None else step)
    file_name = f'{fname}_{data_name}_{git_hash}_{step}'
    outdir = Path(outdir if outdir is not None else '.') / 'outputs' / f'{fname}'
    return outdir, file_name, (outdir / file_name).with_suffix('.wav')


def line_paths(outdir: Path, file_name: str, i: int):
    """-> (.wav of line i, the path np.save turns into ..._<i>.mel.npy) (reference: predict_tts.py:59-62)."""
    return (outdir / (file_name + f'_{i}')).with_suffix('.wav'), (outdir / (file_name + f'_{i}')).with_suffix('.mel')


def make_tokenizer(model):
    from transformertts_b200.data.text import Tokenizer
    return Tokenizer(add_start_end=False, model_breathing=bool(model.config.get('model_breathing', False)), alphabet=model.alphabet)


def load_model(args):
    """-> (model, config used for the file name, step to name the files with when that config has none)."""
    from transformertts_b200.model.models import ForwardTransformer
    if args.path is not None:
        import yaml
        print(f'Loading model from {args.path}')
        model = ForwardTransformer.load_model(args.path)
        with open(Path(args.path) / 'config.yaml', 'r') as f:
            saved = yaml.safe_load(f)
        config = dict(model.config, **{k: saved[k] for k in ('data_name', 'git_hash', 'step') if k in saved})
        return model, config, model.step
    from transformertts_b200.model.factory import tts_ljspeech
    model = tts_ljspeech(args.step)
    return model, dict(model.config), args.step


def load_vocoder(name: str, checkpoint, config, model):
    """The generator --vocoder names (weights from checkpoint, HiFi-GAN's config from config) on the model's device, or None
    for Griffin-Lim, which Audio.reconstruct_waveform_batch runs.  A generator is refused when the samples it makes per mel frame
    differ from the model's hop_length: its audio would have the wrong length and pitch."""
    if name in ('melgan', 'hifigan', 'bigvgan'):
        from transformertts_b200.model import bigvgan, hifigan, melgan
        upsampling = {'melgan': melgan, 'hifigan': hifigan, 'bigvgan': bigvgan}[name].HOP
        hop = int(model.config['hop_length'])
        if upsampling != hop:
            raise SystemExit(f'--vocoder {name}: the generator upsamples each mel frame to {upsampling} samples, but the audio '
                             f'settings have hop_length {hop}; use --vocoder griffinlim at this hop')
    if name == 'melgan':
        from transformertts_b200.model.melgan import MelGANGenerator
        return MelGANGenerator.from_checkpoint(checkpoint, device=model.device)
    if name in ('hifigan', 'bigvgan'):
        normalizer = model.config.get('normalizer')
        if normalizer != 'MelGAN':
            label = 'HiFi-GAN' if name == 'hifigan' else 'BigVGAN'
            raise SystemExit(f'--vocoder {name} takes the MelGAN normaliser\'s log-mels (ln(max(S, 1e-5))); this model\'s normalizer '
                             f'is {normalizer!r}, whose mels {label} would misread')
    if name == 'hifigan':
        from transformertts_b200.model.hifigan import HiFiGANGenerator
        return HiFiGANGenerator.from_checkpoint(checkpoint, config=config, device=model.device)
    if name == 'bigvgan':
        from transformertts_b200.model.bigvgan import BigVGANGenerator, check_audio, load_config
        if config is None:
            config = Path(checkpoint).parent / 'config.json'
            if not config.exists():
                raise SystemExit(f'--vocoder bigvgan: {config} not found; pass --vocoder_config (a config.json path or base / bigvgan)')
        h = load_config(config)
        c = model.config
        try:
            check_audio(h, c['sampling_rate'], c['mel_channels'], c['hop_length'], c.get('f_max'))
        except ValueError as e:
            raise SystemExit(f'--vocoder bigvgan: {e}')
        return BigVGANGenerator.from_checkpoint(checkpoint, config=h, device=model.device)
    if name == 'wavernn':
        normalizer = model.config.get('normalizer')
        if normalizer != 'WaveRNN':
            raise SystemExit(f'--vocoder wavernn takes the WaveRNN normaliser\'s mels; this model\'s normalizer is {normalizer!r}')
        from transformertts_b200.model.wavernn import WaveRNNGenerator
        g = WaveRNNGenerator.from_checkpoint(checkpoint, device=model.device)
        hop = int(model.config['hop_length'])
        if g.hop != hop:
            raise SystemExit(f'--vocoder wavernn: the generator upsamples each mel frame to {g.hop} samples, but the audio settings '
                             f'have hop_length {hop}')
        return g
    return None


def vocode_chunk(vocoder, audio, mels, start: int):
    """Waveforms of the (n_mels, T) mels of lines start, start + 1, ...: Griffin-Lim (vocoder None) and WaveRNN draw line i
    with seed i."""
    if vocoder is None:
        return audio.reconstruct_waveform_batch(mels, seed=start)
    from transformertts_b200.model.wavernn import MIN_FRAMES, WaveRNNGenerator
    if isinstance(vocoder, WaveRNNGenerator):
        for j, m in enumerate(mels):
            if m.shape[1] < MIN_FRAMES:
                raise ValueError(f'line {start + j} gives a mel of {m.shape[1]} frames; the WaveRNN vocoder needs at least {MIN_FRAMES}')
        return vocoder.vocode_batch(mels, seeds=range(start, start + len(mels)))
    return vocoder.vocode_batch(mels)


def main(argv=None):
    args = parse_args(argv)
    fname, text = read_input(args)
    if text is None:
        print(NO_INPUT_MESSAGE)
        return 0
    model, config, step = load_model(args)
    outdir, file_name, output_path = output_names(args.outdir, fname, config, step)
    outdir.mkdir(exist_ok=True, parents=True)
    from transformertts_b200.data.audio import Audio
    audio = Audio.from_config(model.config)
    tokenizer = make_tokenizer(model)
    vocoder = load_vocoder(args.vocoder, args.vocoder_checkpoint, args.vocoder_config, model)
    print(f'Output wav under {output_path.parent}')
    tokens = []
    for line in text:
        tokens.append(tokenizer(line))
        if args.verbose:
            print(f'Predicting {line}')
            print(f'Tokens: "{tokens[-1]}"')
    outs = model.predict_batch(tokens, encode=False, phoneme_max_duration=None)
    wavs = []
    for start in range(0, len(text), VOCODE_CHUNK):
        mels = []
        for i in range(start, min(start + VOCODE_CHUNK, len(text))):
            mel = outs[i]['mel'].cpu().numpy()                  # (T, n_mels)
            if mel.shape[0] < audio.min_griffinlim_frames:
                raise ValueError(f'line {i} gives a mel of shape {mel.shape}; the vocoder needs at least {audio.min_griffinlim_frames} '
                                 f'frames')
            mels.append(mel)
            if args.store_mel:
                np.save(line_paths(outdir, file_name, i)[1], mel)
        chunk = vocode_chunk(vocoder, audio, [m.T for m in mels], start)
        for j, wav in enumerate(chunk):
            if args.single:
                audio.save_wav(wav, line_paths(outdir, file_name, start + j)[0])
        wavs.extend(chunk)
    audio.save_wav(np.concatenate(wavs), output_path)
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
