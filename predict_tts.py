#!/usr/bin/env python
"""Text-to-speech from the command line: the reference's ``predict_tts.py``.

    python predict_tts.py -f lines.txt [-p MODEL_DIR | --step 95000] [-o OUTDIR] [-m] [-s] [-v]
    python predict_tts.py -t "phoneme string" ...

Every input line is tokenised, turned into a mel by ``ForwardTransformer.predict`` (one line per call, as the reference does)
and vocoded on the GPU with ``Audio.reconstruct_waveform_batch`` (mel inversion + 32 Griffin-Lim iterations), in chunks of
``VOCODE_CHUNK`` lines so that device memory stays bounded however long the file is.  Output:
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

VOCODE_CHUNK = 16    # lines vocoded per reconstruct_waveform_batch call
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
    return parser.parse_args(argv)


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
    print(f'Output wav under {output_path.parent}')
    wavs = []
    for start in range(0, len(text), VOCODE_CHUNK):
        mels = []
        for i in range(start, min(start + VOCODE_CHUNK, len(text))):
            tokens = tokenizer(text[i])
            if args.verbose:
                print(f'Predicting {text[i]}')
                print(f'Tokens: "{tokens}"')
            out = model.predict(tokens, encode=False, phoneme_max_duration=None)
            mel = out['mel'].cpu().numpy()                      # (T, n_mels)
            if mel.ndim != 2 or mel.shape[0] < 4:
                raise ValueError(f'line {i} gives a mel of shape {mel.shape}; the vocoder needs at least 4 frames')
            mels.append(mel)
            if args.store_mel:
                np.save(line_paths(outdir, file_name, i)[1], mel)
        chunk = audio.reconstruct_waveform_batch([m.T for m in mels], seed=start)
        for j, wav in enumerate(chunk):
            if args.single:
                audio.save_wav(wav, line_paths(outdir, file_name, start + j)[0])
        wavs.extend(chunk)
    audio.save_wav(np.concatenate(wavs), output_path)
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
