"""Resampling on the GPU (ttsb_resample_batch through Audio.resample_ragged): bit-identical to the numpy restatement of
librosa.load(sr=...) / resampy kaiser_best (tests/resample_oracle.py) at every common source rate, independent of the batch,
at full batch size, and create_training_data.py end to end on a corpus of mixed rates (reference: data/audio.py:126-130)."""
import pickle
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import yaml

import resample_oracle as ro
from oracle import pitch_oracle as po

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
HOP = 256
RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)


def _audio(sr=22050, **kw):
    from transformertts_b200.data.audio import Audio
    return Audio(sampling_rate=sr, n_fft=1024, mel_channels=80, hop_length=HOP, win_length=1024, f_min=0, f_max=8000,
                 normalizer='MelGAN', **kw)


def _clips(rates, seconds_long=10.0):
    """(samples, rate) for every rate: 3, 47, 1000 and 4801 samples and a long clip, seeded noise plus tones."""
    out = []
    for i, sr in enumerate(rates):
        for j, L in enumerate((3, 47, 1000, 4801, int(seconds_long * sr) + 1)):
            out.append((ro.noisy_tones(L, sr, seed=100 * i + j), sr))
    return out


def _check(got, clips, target):
    for (x, sr), y in zip(clips, got):
        want = ro.resample(x, sr, target)
        assert y.dtype == np.float32 and y.shape == want.shape, (sr, len(x), y.shape, want.shape)
        bad = np.nonzero(y != want)[0]
        assert len(bad) == 0, f'{sr} Hz -> {target} Hz, {len(x)} samples: {len(bad)} samples differ, first at {bad[:5]}'


@pytest.mark.parametrize('target,rates', [(22050, RATES), (24000, (16000, 22050, 44100, 48000))])
def test_bit_identical_to_the_oracle(target, rates):
    audio = _audio(target)
    clips = _clips(rates)
    _check(audio.resample_ragged(clips), clips, target)


def test_ragged_independence():
    audio = _audio()
    clips = _clips(RATES, seconds_long=2.0)
    mixed = audio.resample_ragged(clips)
    rev = audio.resample_ragged(clips[::-1])[::-1]
    alone = [audio.resample_ragged([c])[0] for c in clips]
    by_rate = []
    for sr in RATES:
        by_rate += audio.resample_ragged([c for c in clips if c[1] == sr])
    for a, b, c, d in zip(mixed, rev, alone, by_rate):
        assert np.array_equal(a, b) and np.array_equal(a, c) and np.array_equal(a, d)
    same = [c for c in clips if c[1] == 22050]
    for (x, _), y in zip(same, audio.resample_ragged(same)):
        assert np.array_equal(x, y)                     # a clip already at the target rate comes back unchanged


def test_full_size_batch_against_the_oracle():
    import create_training_data as ctd
    audio = _audio()
    clips = [(ro.noisy_tones(60 * 48000 + 7, 48000, seed=1), 48000), (ro.noisy_tones(20 * 44100, 44100, seed=2), 44100),
             (ro.noisy_tones(10 * 16000 + 1, 16000, seed=3), 16000), (ro.noisy_tones(8 * 48000, 48000, seed=4), 48000),
             (ro.noisy_tones(3 * 22050, 22050, seed=5), 22050)]
    assert sum(len(x) for x, _ in clips) >= ctd.BATCH_SAMPLES
    _check(audio.resample_ragged(clips), clips, 22050)


def _write_wav(path, x, sr):
    import scipy.io.wavfile
    scipy.io.wavfile.write(path, sr, np.clip(np.rint(x * np.float32(32767)), -32768, 32767).astype('<i2'))


def _run(tmp_path, names, texts):
    (tmp_path / 'metadata.csv').write_text(''.join(f'{n}|raw text|{t}\n' for n, t in zip(names, texts)), encoding='utf-8')
    cfg = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    cfg['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'),
                        metadata_path=str(tmp_path / 'metadata.csv'), wav_directory=str(tmp_path / 'wavs'))
    cfg['training_data_settings'].update(n_test=3, min_mel_len=90, max_mel_len=400)
    cfg['audio_settings'] = dict(cfg.get('audio_settings') or {}, norm_wav=True, target_dBFS=-30, int16_max=32767)
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    return subprocess.run([sys.executable, str(ROOT / 'create_training_data.py'), '--config', str(tmp_path / 'cfg.yaml')],
                          cwd=tmp_path, capture_output=True, text=True, timeout=900)


def test_create_training_data_resamples_a_mixed_rate_corpus(tmp_path):
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    wav_dir = tmp_path / 'wavs'
    wav_dir.mkdir()
    rates = [48000, 16000, 22050, 48000, 22050, 16000, 48000, 22050, 48000, 16000]
    rng = np.random.default_rng(0)
    names, texts = [], []
    for i, sr in enumerate(rates):
        x = po.speech_like_clip(float(rng.uniform(1.0, 3.0)), 300 + i, fs=float(sr)) * np.float32(rng.uniform(0.05, 0.8))
        names.append(f'LJ{i:03d}-{sr}')
        texts.append(''.join(rng.choice(list('abdefhijklmnoprstuvwz'), int(rng.integers(5, 30)))))
        _write_wav(wav_dir / f'{names[-1]}.wav', x, sr)
    r = _run(tmp_path, names, texts)
    assert r.returncode == 0, r.stdout + r.stderr
    assert 'Resampled 7 file(s) to 22050 Hz: 3 from 16000 Hz, 4 from 48000 Hz' in r.stdout, r.stdout
    cm = TrainingConfigManager(tmp_path / 'cfg.yaml', aligner=True)
    audio = Audio.from_config(cm.config)
    assert audio.norm_wav
    ref_pitch, mel_len = {}, {}
    for name, sr in zip(names, rates):
        path = wav_dir / f'{name}.wav'
        if sr == 22050:
            y = audio.load_wav(path)[0]                                   # the path a corpus at the configured rate takes
        else:
            x, native = audio.read_wav(path)
            assert native == sr
            y = audio.preprocess(ro.resample(x, sr, 22050))
        mel = np.load(cm.mel_dir / f'{name}.npy')
        assert mel.dtype == np.float32 and np.array_equal(mel, audio.mel_spectrogram(y)), name
        ref_pitch[name] = po.extract_pitch(y, 22050, HOP)
        mel_len[name] = mel.shape[0]
    mean, std = po.pitch_stats(ref_pitch.values())
    stats = pickle.load(open(cm.data_dir / 'pitch_stats.pkl', 'rb'))
    assert abs(stats['pitch_mean'] / mean - 1) < 1e-6 and abs(stats['pitch_std'] / std - 1) < 1e-5
    for name in names:
        p = np.load(cm.pitch_dir / f'{name}.npy')
        ref = po.normalize_pitch(ref_pitch[name], mean, std)
        assert p.dtype == np.float64 and np.array_equal(p == 0, ref == 0) and np.allclose(p, ref, rtol=0, atol=1e-4), name
    assert pickle.load(open(cm.data_dir / 'mel_len.pkl', 'rb')) == mel_len


def test_create_training_data_names_a_file_too_short_to_resample(tmp_path):
    wav_dir = tmp_path / 'wavs'
    wav_dir.mkdir()
    _write_wav(wav_dir / 'LJ000-ok.wav', po.speech_like_clip(1.5, 1, fs=48000.0), 48000)
    _write_wav(wav_dir / 'LJ001-short.wav', np.array([0.1, -0.1], np.float32), 48000)
    r = _run(tmp_path, ['LJ000-ok', 'LJ001-short'], ['abc', 'def'])
    assert r.returncode != 0
    assert 'LJ001-short.wav' in r.stderr and 'too short to resample' in r.stderr, r.stdout + r.stderr
