"""CPU tests of the training-data preparation: argument checks of the new entry points without a GPU, Audio.preprocess against a
literal transcription of the reference, DataReader's wav scan, and the metadata half of create_training_data.py against a literal
transcription of reference create_training_data.py:101-178."""
import ctypes as C
import pickle
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import yaml

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def _i32(*v):
    return (C.c_int32 * len(v))(*v)


def test_ragged_mel_refuses_malformed_offsets_and_band_tables_without_gpu(cdll):
    dev = C.c_void_p(256)          # never dereferenced: every check below fails before any CUDA call
    ws = C.c_int64(1 << 20)
    band = _i32(*[0, 513] * 80)
    call = lambda so, fo, n: cdll.ttsb_stft_mel_log_batch(dev, so, fo, n, dev, band, 80, 0, dev, ws, dev, None)
    assert call(_i32(0, 2000, 4000), _i32(0, 8, 17), 2) == -1 and b'frames' in cdll.ttsb_last_error()
    assert call(_i32(0, 500, 4000), _i32(0, 2, 17), 2) == -1 and b'512' in cdll.ttsb_last_error()
    assert call(_i32(5, 2000, 4000), _i32(0, 8, 16), 2) == -1 and b'start at 0' in cdll.ttsb_last_error()
    assert call(_i32(0, 2000), _i32(0, 8), 0) == -1
    # a band table spanning 2049 weights (one more than the packed filterbank holds) is refused before any CUDA call
    wide = _i32(0, 513, 0, 513, 0, 513, 0, 510)
    assert cdll.ttsb_stft_mel_log_batch(dev, _i32(0, 2000, 4000), _i32(0, 8, 16), 2, dev, wide, 4, 0, dev, ws, dev, None) == -3
    assert b'2048' in cdll.ttsb_last_error()
    bad_band = _i32(0, 513, 7, 6)
    assert cdll.ttsb_stft_mel_log_batch(dev, _i32(0, 2000, 4000), _i32(0, 8, 16), 2, dev, bad_band, 2, 0, dev, ws, dev, None) == -1
    assert b'band row 1' in cdll.ttsb_last_error()
    assert cdll.ttsb_stft_mel_log_batch_workspace_bytes(0) == -1


def test_pitch_refuses_malformed_offsets_without_gpu(cdll):
    from transformertts_b200 import lib
    dev = C.c_void_p(256)
    fp = 256 / 22050 * 1000
    call = lambda so, n, fo: lib.load().ttsb_pitch_dio_stonemask(dev, so, n, 22050, fp, 71.0, 800.0, 2.0, 0.1, fo, dev, dev, 1 << 30, None)
    assert call(_i32(0, 700, 3000), 2, _i32(0, 3, 12)) == -1 and b'3 frames' in cdll.ttsb_last_error()
    assert call(_i32(0, 1500, 3000), 2, _i32(0, 6, 13)) == -1 and b'frame count' in cdll.ttsb_last_error()
    assert call(_i32(0, 1500, 1400), 2, _i32(0, 6, 6)) == -1 and b'samples' in cdll.ttsb_last_error()
    assert lib.load().ttsb_pitch_dio_stonemask(dev, _i32(0, 1500), 1, 22050, fp, 71.0, 800.0, 2.0, 0.1, _i32(0, 6), dev, dev, 1024,
                                                None) == -1 and b'workspace' in cdll.ttsb_last_error()
    assert lib.load().ttsb_pitch_workspace_bytes(_i32(0, 1500), 0, 22050, fp, 71.0, 800.0, 2.0) == -1
    assert lib.pitch_workspace_bytes([0, 1500, 4000], 22050, fp) > 0


def test_pitch_workspace_refuses_band_count_band_length_and_short_clips(cdll):
    from oracle import pitch_oracle as po
    fs, fp = 22050, 256 / 22050 * 1000

    def ws(lengths, f0_floor=71.0, channels_in_octave=2.0):
        so = np.concatenate([[0], np.cumsum(lengths)]).tolist()
        return cdll.ttsb_pitch_workspace_bytes(_i32(*so), len(lengths), fs, fp, f0_floor, 800.0, channels_in_octave)

    # 71 .. 800 Hz: 16 bands at 4.5 channels per octave, 17 at 4.6
    assert len(po.boundary_f0s(71.0, 800.0, 4.5)) == 16 and len(po.boundary_f0s(71.0, 800.0, 4.6)) == 17
    assert ws([fs], channels_in_octave=4.5) > 0
    assert ws([fs], channels_in_octave=4.6) == -1 and b'17 bands' in cdll.ttsb_last_error()
    # band 0's low-pass has 4h taps, h = round(fs / (f0_floor sqrt 2) / 2), and must satisfy 2h <= round(fs / 50)
    P = po.matlab_round(fs / 50.0)
    fits = lambda floor: 2 * po.band_half_lengths(fs, po.boundary_f0s(floor, 800.0, 2.0))[0] <= P
    assert fits(36.0) and not fits(35.0)
    assert ws([fs], f0_floor=36.0) > 0
    assert ws([fs], f0_floor=35.0) == -1 and b'band 0 low-pass longer than the low-cut margin' in cdll.ttsb_last_error()
    # a clip of voice_range_minimum frames is refused, one of one frame more is accepted
    vrm = po.voice_range_minimum(fp, 71.0)
    L = next(L for L in range(1, 10 * 256) if po.n_frames(L, fs, fp) > vrm)
    assert po.n_frames(L - 1, fs, fp) == vrm
    assert ws([4000, L]) > 0
    assert ws([4000, L - 1]) == -1 and b'voice_range_minimum' in cdll.ttsb_last_error()


def _ref_normalize_volume(self, wav, increase_only=False, decrease_only=False):
    # reference data/audio.py:154-162, as written
    if increase_only and decrease_only:
        raise ValueError("Both increase only and decrease only are set")
    rms = np.sqrt(np.mean((wav * self.int16_max) ** 2))
    wave_dBFS = 20 * np.log10(rms / self.int16_max)
    dBFS_change = self.target_dBFS - wave_dBFS
    if dBFS_change < 0 and increase_only or dBFS_change > 0 and decrease_only:
        return wav
    return wav * (10 ** (dBFS_change / 20))


def _ref_preprocess(self, y):
    # reference data/audio.py:132-141 without the two trims (refused here)
    if self.norm_wav:
        y = _ref_normalize_volume(self, y, increase_only=True)
    if y.shape[0] % self.hop_length == 0:
        y = np.pad(y, (0, 1))
    return y


def _audio(**kw):
    from transformertts_b200.data.audio import Audio
    return Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                 normalizer='MelGAN', **kw)


@pytest.mark.parametrize('L,scale', [(256 * 40, 0.01), (9001, 0.01), (256 * 12, 0.9), (5000, 0.9)])
def test_preprocess_matches_the_reference_bit_for_bit(L, scale):
    y = (scale * np.random.default_rng(L).standard_normal(L)).astype(np.float32)
    a = _audio(norm_wav=True, target_dBFS=-30, int16_max=(2 ** 15) - 1)
    got, ref = a.preprocess(y), _ref_preprocess(a, y)
    assert got.dtype == ref.dtype and np.array_equal(got, ref)
    b = _audio(norm_wav=False)
    assert np.array_equal(b.preprocess(y), _ref_preprocess(b, y)) and len(b.preprocess(y)) == L + (L % 256 == 0)


def test_preprocess_refuses_trimming_and_load_wav_refuses_other_rates(tmp_path):
    with pytest.raises(NotImplementedError, match='webrtcvad'):
        _audio(trim_long_silences=True).preprocess(np.zeros(1000, np.float32))
    with pytest.raises(NotImplementedError, match='librosa'):
        _audio(trim_silence=True).preprocess(np.zeros(1000, np.float32))
    import scipy.io.wavfile
    scipy.io.wavfile.write(tmp_path / 'a.wav', 16000, np.zeros(1000, np.int16))
    with pytest.raises(ValueError, match='16000'):
        _audio().load_wav(tmp_path / 'a.wav')
    pcm = np.array([[0, 16384], [-32768, 32767]], np.int16)
    scipy.io.wavfile.write(tmp_path / 'b.wav', 22050, pcm)
    y, sr = _audio().load_wav(tmp_path / 'b.wav', preprocess=False)
    assert sr == 22050 and y.dtype == np.float32 and np.array_equal(y, np.mean(pcm.astype(np.float32) / 32768, axis=1))


def test_scan_wavs(tmp_path):
    from transformertts_b200.data.datasets import DataReader
    (tmp_path / 'w' / 'sub').mkdir(parents=True)
    (tmp_path / 'w' / 'a.wav').write_bytes(b'')
    (tmp_path / 'w' / 'sub' / 'b.wav').write_bytes(b'')
    (tmp_path / 'm.csv').write_text('a|x|y\nb|x|y\n')
    r = DataReader(tmp_path / 'm.csv', wav_directory=tmp_path / 'w', scan_wavs=True)
    assert sorted(r.wav_paths) == ['a', 'b'] and r.wav_paths['b'].name == 'b.wav'
    assert not hasattr(DataReader(tmp_path / 'm.csv'), 'wav_paths')
    with pytest.raises(ValueError, match='wav_directory'):
        DataReader(tmp_path / 'm.csv', scan_wavs=True)


def _reference_metadata_half(cm, metadatareader, cross_file_ids, phonemize):
    """reference create_training_data.py:101-178 as written, with p_uimap replaced by an in-order map and the summaries dropped."""
    _alphabet = 'ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyzäüößÄÖÜ'
    remove_files = pickle.load(open(cm.data_dir / 'under-over_sized_mels.pkl', 'rb'))
    phonemized_metadata_path = cm.phonemized_metadata_path
    train_metadata_path = cm.train_metadata_path
    test_metadata_path = cm.valid_metadata_path
    filter_metadata = []
    for fname in cross_file_ids:
        item = metadatareader.text_dict[fname]
        non_p = [c for c in item if c in _alphabet]
        if len(non_p) < 1:
            filter_metadata.append(fname)
    remove_files += filter_metadata
    metadata_file_ids = [fname for fname in cross_file_ids if fname not in remove_files]
    metadata_len = len(metadata_file_ids)
    sample_items = np.random.choice(metadata_file_ids, 5)  # noqa: F841
    test_len = cm.config['n_test']
    train_len = metadata_len - test_len

    def process_phonemes(file_id):
        text = metadatareader.text_dict[file_id]
        return (file_id, phonemize(text))
    phonemized_data = {}
    for (file_id, phonemes) in map(process_phonemes, metadata_file_ids):
        phonemized_data.update({file_id: phonemes})
    new_metadata = [f'{k}|{v}\n' for k, v in phonemized_data.items()]
    shuffled_metadata = np.random.permutation(new_metadata)
    train_metadata = shuffled_metadata[0:train_len]
    test_metadata = shuffled_metadata[-test_len:]
    with open(phonemized_metadata_path, 'w+', encoding='utf-8') as file:
        file.writelines(new_metadata)
    with open(train_metadata_path, 'w+', encoding='utf-8') as file:
        file.writelines(train_metadata)
    with open(test_metadata_path, 'w+', encoding='utf-8') as file:
        file.writelines(test_metadata)


@pytest.mark.parametrize('with_phonemizer', [False, True])
def test_metadata_half_matches_the_reference(tmp_path, monkeypatch, with_phonemizer):
    import create_training_data as ctd
    from transformertts_b200.data.datasets import DataReader
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    wav_dir = tmp_path / 'wavs'
    wav_dir.mkdir()
    rng = np.random.default_rng(1)
    names = [f'LJ{i:03d}' for i in range(30)]
    lines = []
    for i, n in enumerate(names):
        if i != 7:
            (wav_dir / f'{n}.wav').write_bytes(b'')                # LJ007 has no wav
        text = '...' if i == 3 else ''.join(rng.choice(list('abcdefgh ,.'), 12)) + 'x'
        lines.append(f'{n}|raw|{text}\n')
    (tmp_path / 'metadata.csv').write_text(''.join(lines), encoding='utf-8')
    cfg = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    cfg['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'),
                        metadata_path=str(tmp_path / 'metadata.csv'), wav_directory=str(wav_dir))
    cfg['training_data_settings'].update(n_test=5)
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    stub = lambda text, **kw: 'ph:' + text.upper()
    if with_phonemizer:
        pkg, mod = types.ModuleType('phonemizer'), types.ModuleType('phonemizer.phonemize')
        mod.phonemize = stub
        pkg.phonemize = mod
        monkeypatch.setitem(sys.modules, 'phonemizer', pkg)
        monkeypatch.setitem(sys.modules, 'phonemizer.phonemize', mod)
    cm = TrainingConfigManager(tmp_path / 'cfg.yaml', aligner=True)
    cm.data_dir.mkdir(parents=True)
    pickle.dump(['LJ011', 'LJ020'], open(cm.data_dir / 'under-over_sized_mels.pkl', 'wb'))
    ctd.main(['--config', str(tmp_path / 'cfg.yaml'), '--skip_mels'])
    got = [open(p, encoding='utf-8').read() for p in (cm.phonemized_metadata_path, cm.train_metadata_path, cm.valid_metadata_path)]
    reader = DataReader.from_config(cm, kind='original', scan_wavs=True)
    cross = [f for f in reader.filenames if f in reader.wav_paths]
    phon = ctd.make_phonemizer(cm.config) if with_phonemizer else (lambda t: t)
    np.random.seed(42)
    _reference_metadata_half(cm, reader, cross, phon)
    ref = [open(p, encoding='utf-8').read() for p in (cm.phonemized_metadata_path, cm.train_metadata_path, cm.valid_metadata_path)]
    assert got == ref
    kept = [l.split('|')[0] for l in got[0].splitlines()]
    assert 'LJ003' not in kept and 'LJ007' not in kept and 'LJ011' not in kept and len(kept) == 26
    assert len(got[2].splitlines()) == 5 and (not with_phonemizer or got[0].splitlines()[0].split('|')[1].startswith('ph'))
