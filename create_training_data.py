#!/usr/bin/env python
"""Training data from a corpus of wavs: the reference's ``create_training_data.py``.

    python create_training_data.py --config config/training_config.yaml [--skip_mels] [--skip_phonemes]

It reads ``metadata_path`` (LJSpeech ``name|...|text`` lines) and the ``*.wav`` and ``*.flac`` files below ``wav_directory`` (a
name that exists as both is refused), and writes under
``<train_data_directory>.<data_name>/``, as the reference does:
  * ``mels.<audio>/<name>.npy``: log-mel, float32 (T, mel_channels);
  * ``pitch.<audio>/<name>.npy``: per-frame f0 by DIO + StoneMask, float64 (T,), normalised by the corpus statistics;
  * ``pitch_stats.pkl`` ({'pitch_mean', 'pitch_std'}), ``mel_len.pkl`` ({name: T}) and ``under-over_sized_mels.pkl`` (names
    whose mel is longer than ``max_mel_len`` or shorter than ``min_mel_len``);
  * the phonemized, train and valid metadata files (``name|phonemes`` lines), ``n_test`` lines held out by a permutation
    seeded with 42.

The wavs are processed in batches of about ``BATCH_SAMPLES`` samples: a thread pool reads and preprocesses the files ahead of the
GPU, each batch is uploaded once, its log-mels (``ttsb_stft_mel_log_batch``) and pitch (``ttsb_pitch_dio_stonemask``) are
computed on the same packed buffer, and another thread pool writes the ``.npy`` files.

FLAC files are read by the loader threads but decoded on the GPU, every FLAC file of a batch in one ``ttsb_flac_decode_batch``
call; from then on their samples take exactly the path a WAV file's samples take, so a corpus stored as FLAC gives the same
``.npy``, ``.pkl`` and metadata files, byte for byte, as the same corpus stored as WAV.

Wavs at another rate than the audio settings' ``sampling_rate`` are resampled to it as the reference's ``librosa.load(path,
sr=sampling_rate)`` does (resampy's ``kaiser_best`` filter): the off-rate files of a batch go through one
``ttsb_resample_batch`` launch, then through the same ``Audio.preprocess`` (volume normalisation, hop padding) as every other file.
Files already at ``sampling_rate`` take exactly the path they take without resampling.

With ``trim_silence`` set (and ``trim_silence_top_db``), the leading and trailing silence of every file is trimmed as the
reference's ``librosa.effects.trim(y, top_db, frame_length=256, hop_length=64)`` does, after the volume normalisation and before
the hop padding: the files of a batch, at the configured rate and resampled alike, go through one ``ttsb_trim_silence_bounds``
launch, and the loader threads do only the volume normalisation.  The mels, the pitch, ``mel_len.pkl``, the length filter and
the pitch statistics then see the trimmed clips.  Without ``trim_silence`` the script runs exactly as before.

Differences from the reference:
  * Without the ``phonemizer`` package (and espeak), the text column of the metadata is taken to BE phonemes in the model's
    alphabet, as ``predict_tts.py`` does; the script says so when it starts.  With it, the reference's arguments are used.
  * Files are processed in metadata order, so the pitch statistics and the phonemized metadata are in that order; the
    reference's process pool completes them in no fixed order, so its statistics differ in the last bits from run to run.
  * The ``trim_long_silences`` setting is refused (no webrtcvad), and so is ``trim_silence`` without ``trim_silence_top_db``
    (librosa would be called with top_db=None); see ``Audio.preprocess``.
  * A file whose trimmed clip is too short for the log-mel or pitch kernels (fewer than ``n_fft / 2 + 1`` samples, or no more
    WORLD frames than DIO's voice_range_minimum) gets no ``.npy`` files: it is listed in ``under-over_sized_mels.pkl`` with its
    frame count ``1 + L // hop_length`` in ``mel_len.pkl``, and its pitch does not enter the statistics.  The reference computes
    its tiny mel and pitch, and then drops the file by ``min_mel_len`` all the same.
  * Resampling restates resampy's ``kaiser_best`` table from its published parameters rather than reading resampy's precomputed
    file, so it may differ from librosa's result in the last bits of the filter.  A file too short to resample (fewer output
    samples than one) stops the script with its name; the reference's worker would raise inside resampy.
  * ``max_mel_len``, ``min_mel_len`` and ``n_test`` default to the reference's 1200, 80 and 100 when the config lacks them.
  * No TensorBoard summaries.
"""
from __future__ import annotations

import argparse
import pickle
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

BATCH_SAMPLES = 4 * 1024 * 1024          # samples per GPU batch (about 3 minutes at 22050 Hz; ~0.8 GB of pitch workspace)
DEFAULTS = {'max_mel_len': 1200, 'min_mel_len': 80, 'n_test': 100}
ALPHABET = 'ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyzäüößÄÖÜ'   # reference: data/text/symbols.py:10


def config_value(cm, key):
    return cm.config.get(key, DEFAULTS[key])


def text_settings(path) -> dict:
    import yaml
    with open(path, 'rb') as f:
        raw = yaml.safe_load(f)
    return dict(raw.get('text_settings', {}) or {})


def make_phonemizer(config):
    """reference: data/text/tokenizer.py:50-106 through TextToTokens.default(njobs=1); None without the phonemizer package."""
    try:
        from phonemizer.phonemize import phonemize
    except ImportError:
        return None
    import re
    from transformertts_b200.data.text import ALL_PHONEMES
    punctuations = '!,-.:;? \'()'
    ws_re, ws_punct_re = re.compile(r'\s+'), re.compile(f'\\s*([{punctuations}])\\s*')

    def phonemizer(text: str) -> str:
        text = text.replace('-', '—')
        ph = phonemize(text, language=config['phoneme_language'], backend='espeak', strip=True, preserve_punctuation=True,
                       with_stress=config['with_stress'], punctuation_marks=';:,.!?¡¿—…"«»“”', njobs=1,
                       language_switch='remove-flags')
        ph = ph.replace('—', '-')
        ph = ''.join([c for c in ph if c in ALL_PHONEMES])
        ph = re.sub(ws_punct_re, r'\1', re.sub(ws_re, ' ', ph))
        return ph.strip()
    return phonemizer


def batches(paths, budget: int, load, size=len):
    """Consecutive groups of (path, load(path)) whose sizes (`size` of each loaded item: its samples) add up to about `budget`;
    files are read by a thread pool ahead of use."""
    with ThreadPoolExecutor(max_workers=4) as pool:
        batch, n = [], 0
        for path, y in zip(paths, pool.map(load, paths)):
            batch.append((path, y))
            n += size(y)
            if n >= budget:
                yield batch
                batch, n = [], 0
        if batch:
            yield batch


class TooShortToResample(ValueError):
    pass


def wav_loader(audio):
    """path -> Audio.read_for_batch(path): (samples, None) preprocessed as Audio.load_wav does when the file is at the configured
    rate (up to the trim with trim_silence), else the raw mono samples and their rate, to be resampled with the rest of the batch;
    a FLAC file undecoded, to be decoded with the rest of the batch."""
    from transformertts_b200.data import audio as audio_module

    def load(path):
        try:
            return audio.read_for_batch(str(path))
        except audio_module.TooShortToResample as e:
            raise TooShortToResample(f'{path}: {e}') from None
    return load


def loaded_samples(audio):
    """Size of a wav_loader item in the batch budget: its samples at the configured rate, so a batch of resampled files packs
    about as many samples for the mel and pitch kernels as a batch of files already at that rate.  An undecoded FLAC file counts
    its STREAMINFO total (resampled when the file is at another rate)."""
    from transformertts_b200.data.audio import FlacStream, resampled_length

    def size(item):
        y, sr = item
        if isinstance(y, FlacStream):
            return resampled_length(y.total_samples, y.sample_rate, audio.sampling_rate)
        return len(y) if sr is None else resampled_length(len(y), sr, audio.sampling_rate)
    return size


def finish_batch(audio, batch, rates_seen: dict):
    """Audio.finish_batch on the loaded files of a batch (the FLAC ones decoded in one call, the off-rate ones resampled in one
    launch, every one trimmed in one launch with trim_silence) -> batch of (path, samples at the configured rate, preprocessed)."""
    from transformertts_b200.data.audio import FlacStream
    for _, (y, sr) in batch:
        sr = y.sample_rate if isinstance(y, FlacStream) and y.sample_rate != audio.sampling_rate else sr
        if sr is not None:
            rates_seen[sr] = rates_seen.get(sr, 0) + 1
    return list(zip([path for path, _ in batch], audio.finish_batch([item for _, item in batch])))


def too_short(audio, n_samples: int) -> bool:
    """Whether a trimmed clip is too short for the log-mel (reflect padding) or DIO (its contour fix) kernels."""
    from transformertts_b200.utils.evaluation import _dio_takes
    return n_samples < audio.min_mel_samples or not _dio_takes(audio, n_samples)


def process_mels(cm, audio, wav_files, budget: int = BATCH_SAMPLES):
    """reference :39-99 -> (len_dict, remove_files)."""
    cm.mel_dir.mkdir(parents=True, exist_ok=True)
    cm.pitch_dir.mkdir(parents=True, exist_ok=True)
    max_len, min_len = config_value(cm, 'max_mel_len'), config_value(cm, 'min_mel_len')
    len_dict, remove_files, mel_lens, pitches, rates_seen = {}, [], [], {}, {}
    with ThreadPoolExecutor(max_workers=2) as writer:
        for raw in batches(wav_files, budget, wav_loader(audio), loaded_samples(audio)):
            batch = finish_batch(audio, raw, rates_seen)
            short = set()
            if audio.trim_silence:
                short = {c for c, (_, y) in enumerate(batch) if too_short(audio, len(y))}
            kept = [item for c, item in enumerate(batch) if c not in short]
            if kept:
                wav, so = audio._pack([y for _, y in kept])
                mel, fo_mel = audio.mel_spectrogram_ragged_device(wav, so)
                f0, fo_f0 = audio.extract_pitch_device(wav, so)
                mel, f0 = mel.cpu().numpy(), f0.cpu().numpy()
            k = 0       # clip k of the packed batch
            for c, (path, y) in enumerate(batch):
                name = Path(path).stem
                if c in short:
                    len_dict[name] = 1 + len(y) // audio.hop_length
                    remove_files.append(name)
                    continue
                m, p = mel[fo_mel[k]:fo_mel[k + 1]], f0[fo_f0[k]:fo_f0[k + 1]]
                k += 1
                assert m.shape[1] == audio.config['mel_channels'], len(m.shape) == 2
                assert m.shape[0] == p.shape[0], f'{m.shape[0]} == {p.shape[0]} (wav {y.shape})'
                writer.submit(np.save, (cm.mel_dir / name).with_suffix('.npy'), m)
                pitches[(cm.pitch_dir / name).with_suffix('.npy')] = p
                len_dict[name] = m.shape[0]
                if m.shape[0] > max_len or m.shape[0] < min_len:
                    remove_files.append(name)
                else:
                    mel_lens.append(m.shape[0])
        mean, std = pitch_stats(pitches.values())
        with open(cm.data_dir / 'pitch_stats.pkl', 'wb') as f:
            pickle.dump({'pitch_mean': mean, 'pitch_std': std}, f)
        for path, p in pitches.items():
            writer.submit(np.save, path, normalize_pitch(p, mean, std))
    with open(cm.data_dir / 'mel_len.pkl', 'wb') as f:
        pickle.dump(len_dict, f)
    with open(cm.data_dir / 'under-over_sized_mels.pkl', 'wb') as f:
        pickle.dump(remove_files, f)
    if rates_seen:
        print(f"Resampled {sum(rates_seen.values())} file(s) to {audio.sampling_rate} Hz: "
              + ', '.join(f'{n} from {sr} Hz' for sr, n in sorted(rates_seen.items())))
    total_wav_len = np.sum(mel_lens) * audio.config['hop_length']
    print(f"Total duration (hours): {total_wav_len / audio.config['sampling_rate'] / 60. ** 2:.4f}")
    return len_dict, remove_files


def pitch_stats(pitch_vecs):
    """reference :73-77: mean and std of the non-zero frames of every processed file."""
    nonzeros = np.concatenate([v[np.where(v != 0.0)[0]] for v in pitch_vecs])
    return np.mean(nonzeros), np.std(nonzeros)


def normalize_pitch(pitch, mean, std):
    """reference :80-86 (in float64; zeros stay zero)."""
    pitch = pitch.copy()
    zero_idxs = np.where(pitch == 0.0)[0]
    pitch -= mean
    pitch /= std
    pitch[zero_idxs] = 0.0
    return pitch


def process_phonemes(cm, reader, cross_file_ids, phonemizer):
    """reference :101-178; `phonemizer` None: the metadata text is taken as phonemes."""
    with open(cm.data_dir / 'under-over_sized_mels.pkl', 'rb') as f:
        remove_files = pickle.load(f)
    print(f'\nReading metadata from {reader.metadata_path}')
    print(f'\nFound {len(reader.filenames)} lines.')
    filter_metadata = []
    for fname in cross_file_ids:
        item = reader.text_dict[fname]
        non_p = [c for c in item if c in ALPHABET]
        if len(non_p) < 1:
            filter_metadata.append(fname)
    if len(filter_metadata) > 0:
        print(f'Removing {len(filter_metadata)} suspiciously short line(s):')
        for fname in filter_metadata:
            print(f'{fname}: {reader.text_dict[fname]}')
    print(f'\nRemoving {len(remove_files)} line(s) due to mel filtering.')
    remove_files += filter_metadata
    metadata_file_ids = [fname for fname in cross_file_ids if fname not in remove_files]
    metadata_len = len(metadata_file_ids)
    sample_items = np.random.choice(metadata_file_ids, 5)
    test_len = config_value(cm, 'n_test')
    train_len = metadata_len - test_len
    print(f'\nMetadata contains {metadata_len} lines.')
    print(f'\nFiles will be stored under {cm.data_dir}')
    print(f' - all: {cm.phonemized_metadata_path}')
    print(f' - {train_len} training lines: {cm.train_metadata_path}')
    print(f' - {test_len} validation lines: {cm.valid_metadata_path}')
    print('\nMetadata samples:')
    for i in sample_items:
        print(f'{i}:{reader.text_dict[i]}')
    print('\nPHONEMIZING')
    phonemized_data = {}
    for file_id in metadata_file_ids:
        text = reader.text_dict[file_id]
        phonemized_data[file_id] = phonemizer(text) if phonemizer is not None else text
    print('\nPhonemized metadata samples:')
    for i in sample_items:
        print(f'{i}:{phonemized_data[i]}')
    new_metadata = [f'{k}|{v}\n' for k, v in phonemized_data.items()]
    shuffled_metadata = np.random.permutation(new_metadata)
    train_metadata = shuffled_metadata[0:train_len]
    test_metadata = shuffled_metadata[-test_len:]
    with open(cm.phonemized_metadata_path, 'w+', encoding='utf-8') as file:
        file.writelines(new_metadata)
    with open(cm.train_metadata_path, 'w+', encoding='utf-8') as file:
        file.writelines(train_metadata)
    with open(cm.valid_metadata_path, 'w+', encoding='utf-8') as file:
        file.writelines(test_metadata)
    assert metadata_len == len(set(list(phonemized_data.keys()))), \
        f'Length of metadata ({metadata_len}) does not match the length of the phoneme array ({len(set(list(phonemized_data.keys())))}). Check for empty text lines in metadata.'
    assert len(train_metadata) + len(test_metadata) == metadata_len, \
        f'Train and/or validation lengths incorrect. ({len(train_metadata)} + {len(test_metadata)} != {metadata_len})'


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('--config', type=str, required=True)
    parser.add_argument('--skip_phonemes', action='store_true')
    parser.add_argument('--skip_mels', action='store_true')
    args = parser.parse_args(argv)
    for arg in vars(args):
        print('{}: {}'.format(arg, getattr(args, arg)))
    np.random.seed(42)
    phonemizer = None
    if not args.skip_phonemes:
        phonemizer = make_phonemizer(text_settings(args.config))
        if phonemizer is None:
            print('The phonemizer package is not available: the metadata text is taken to be phonemes in the model\'s alphabet.')

    from transformertts_b200.data.datasets import DataReader
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager

    cm = TrainingConfigManager(args.config, aligner=True)
    cm.create_remove_dirs()
    cm.data_dir.mkdir(parents=True, exist_ok=True)
    reader = DataReader.from_config(cm, kind='original', scan_wavs=True)
    print(f'Reading wavs from {reader.wav_directory}')
    print(f'Reading metadata from {reader.metadata_path}')
    print(f'\nFound {len(reader.filenames)} metadata lines.')
    print(f'\nFound {len(reader.wav_paths)} wav files.')
    cross_file_ids = [fid for fid in reader.filenames if fid in reader.wav_paths]
    print(f'\nThere are {len(cross_file_ids)} wav file names that correspond to metadata lines.')

    if not args.skip_mels:
        from transformertts_b200.data.audio import Audio
        print(f'\nMels will be stored under\n{cm.mel_dir}')
        audio = Audio.from_config(cm.config)
        try:
            process_mels(cm, audio, [reader.wav_paths[k] for k in cross_file_ids])
        except TooShortToResample as e:
            raise SystemExit(f'error: {e}') from None

    if not args.skip_phonemes:
        process_phonemes(cm, reader, cross_file_ids, phonemizer)
    print('\nDone')


if __name__ == '__main__':
    main()
