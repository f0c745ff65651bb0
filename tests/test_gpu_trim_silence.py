"""Silence trimming on the GPU (ttsb_trim_silence_bounds through Audio.trim_silence_ragged / Audio.preprocess): bounds equal to the
float64 restatement of librosa.effects.trim(y, top_db, frame_length=256, hop_length=64) (tests/trim_oracle.py) on ragged
batches and edge clips, independent of the batch, Audio.preprocess bit for bit, and create_training_data.py end to end with
trim_silence on a corpus of mixed rates (reference: data/audio.py:132-141, 164-169)."""
import pickle
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import yaml

import resample_oracle as ro
import trim_oracle as to

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
TOP_DBS = (20, 60, 80)
NORM = dict(norm_wav=True, target_dBFS=-30, int16_max=32767)
WAVERNN = dict(sampling_rate=22050, n_fft=2048, hop_length=275, win_length=1100, f_min=40, f_max=None, normalizer='WaveRNN')
EDGE_LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257)


def _audio(top_db=60, section=None, **kw):
    from transformertts_b200.data.audio import Audio
    s = section or dict(sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000, normalizer='MelGAN')
    return Audio(mel_channels=80, trim_silence_top_db=top_db, **s, **kw)


def _bounds(audio, clips):
    wav, so = audio._pack(clips)
    return [tuple(int(v) for v in b) for b in audio.trim_silence_bounds_device(wav, so).cpu().numpy()]


def _edge_clips():
    """Short clips at every reflection edge, bursts at the first and last samples, all zeros and a quiet burst."""
    out = []
    for L in EDGE_LENGTHS:
        rng = np.random.default_rng(L)
        out.append(rng.standard_normal(L).astype(np.float32))
        y = np.zeros(L, np.float32)
        y[rng.integers(0, L, size=max(1, L // 16))] = rng.standard_normal(max(1, L // 16)).astype(np.float32)
        out.append(y)
        out.append(np.zeros(L, np.float32))
    for L, a, b, amp in ((2560, 1000, 1100, 0.5), (3000, 0, 50, 0.5), (3000, 2950, 3000, 0.5), (2560, 2500, 2560, 0.5),
                         (2560, 1000, 1100, 1e-3), (2561, 0, 2561, 0.25)):
        y = np.zeros(L, np.float32)
        y[a:b] = amp
        out.append(y)
    return out


def _full_batch():
    from create_training_data import BATCH_SAMPLES
    clips, n, seed = [], 0, 0
    while n < BATCH_SAMPLES:
        c = to.padded_speech(1, seed=100 + seed, min_s=1.0, max_s=10.0)[0]
        clips.append(c)
        n += len(c)
        seed += 1
    return clips


def _check(clips, top_db):
    for i, c in enumerate(clips):
        assert to.margin_db(c, top_db) > 1e-6, (i, len(c), top_db)       # no frame is near enough to the threshold to tip
    got = _bounds(_audio(top_db), clips)
    want = [to.bounds64(c, top_db) for c in clips]
    assert got == want, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w][:5]
    return got


def test_bounds_equal_the_float64_oracle():
    speech = to.padded_speech(4, seed=21)
    full = _full_batch()
    assert len(full) > 20 and sum(map(len, full)) >= 4 * 1024 * 1024
    edges = _edge_clips()
    trimmed = 0
    for top_db in TOP_DBS:
        for clips in (speech[:1], speech[1:4], full, edges):
            got = _check(clips, top_db)
            trimmed += sum(g != (0, len(c)) for g, c in zip(got, clips))
    assert trimmed > 3 * len(full)


def test_bounds_and_samples_do_not_depend_on_the_batch():
    audio = _audio(60)
    clips = to.padded_speech(6, seed=33) + [np.zeros(300, np.float32), np.ones(1, np.float32)]
    alone = [audio.trim_silence_ragged([c])[0] for c in clips]
    bounds_alone = [_bounds(audio, [c])[0] for c in clips]
    n = len(clips)
    for shift in range(n):
        order = [(k + shift) % n for k in range(n)]
        batch = [clips[k] for k in order]
        for run in range(2):
            out = audio.trim_silence_ragged(batch)
            assert _bounds(audio, batch) == [bounds_alone[k] for k in order]
            for k, y in zip(order, out):
                assert y.dtype == np.float32 and np.array_equal(y, alone[k]), (shift, run, k)
    assert all(np.array_equal(audio.trim_audio_silence(c), a) for c, a in zip(clips, alone))


@pytest.mark.parametrize('section', ['reference', 'wavernn'])
def test_preprocess_trims_after_normalising_and_before_the_pad(section):
    audio = _audio(60, WAVERNN if section == 'wavernn' else None, trim_silence=True, **NORM)
    hop = audio.hop_length
    clips = to.padded_speech(6, seed=44 if section == 'reference' else 45)
    out = []
    for c in clips:
        y = audio.preprocess(c)
        z = audio.normalize_volume(c, increase_only=True)
        want = to.trim(z, 60)
        want = np.pad(want, (0, 1)) if len(want) % hop == 0 else want
        assert y.dtype == np.float32 and np.array_equal(y, want)
        out.append(y)
    assert sum(len(y) < len(c) for y, c in zip(out, clips)) >= 5
    # a trimmed length that is a multiple of the hop gets its zero sample, as without the trim
    m = int(np.lcm(64, hop)) * max(1, 4096 // int(np.lcm(64, hop)))
    for n in range(m - 300, m + 1):
        c = np.zeros(n + 3000, np.float32)
        c[1000:1000 + n] = 0.25
        a, b = to.bounds64(audio.normalize_volume(c, increase_only=True), 60)
        if (b - a) % hop == 0:
            break
    assert (b - a) % hop == 0 and len(audio.preprocess(c)) == b - a + 1
    mels = audio.mel_spectrogram_ragged(out)
    f0 = audio.extract_pitch_batch(out)
    for y, m, p in zip(out, mels, f0):
        assert m.shape[0] == 1 + len(y) // hop == p.shape[0], (len(y), m.shape, p.shape)


def _write_wav(path, x, sr):
    import scipy.io.wavfile
    scipy.io.wavfile.write(path, sr, np.clip(np.rint(x * np.float32(32767)), -32768, 32767).astype('<i2'))


def test_create_training_data_trims_a_mixed_rate_corpus(tmp_path):
    import create_training_data as ctd
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    wav_dir = tmp_path / 'wavs'
    wav_dir.mkdir()
    rates = [48000, 22050, 22050, 48000, 22050, 48000, 22050, 22050]
    rng = np.random.default_rng(1)
    names, texts = [], []
    for i, sr in enumerate(rates):
        x = to.padded_speech(1, seed=500 + i, fs=float(sr), min_s=1.0, max_s=3.0)[0]
        if i == 6:                                                 # nothing but a click in digital silence
            x = np.zeros(sr, np.float32)
            x[9000:9040] = 0.5
        names.append(f'LJ{i:03d}-{sr}')
        texts.append(''.join(rng.choice(list('abdefhijklmnoprstuvwz'), int(rng.integers(5, 30)))))
        _write_wav(wav_dir / f'{names[-1]}.wav', x, sr)
    (tmp_path / 'metadata.csv').write_text(''.join(f'{n}|raw text|{t}\n' for n, t in zip(names, texts)), encoding='utf-8')
    cfg = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    cfg['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'),
                        metadata_path=str(tmp_path / 'metadata.csv'), wav_directory=str(wav_dir))
    cfg['training_data_settings'].update(n_test=2, min_mel_len=30, max_mel_len=400)
    cfg['audio_settings'] = dict(cfg.get('audio_settings') or {}, trim_silence=True, trim_silence_top_db=60,
                                 trim_long_silences=False, **NORM)
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, str(ROOT / 'create_training_data.py'), '--config', str(tmp_path / 'cfg.yaml')],
                       cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert 'Resampled 3 file(s) to 22050 Hz: 3 from 48000 Hz' in r.stdout, r.stdout
    cm = TrainingConfigManager(tmp_path / 'cfg.yaml', aligner=True)
    audio = Audio.from_config(cm.config)
    assert audio.trim_silence and audio.trim_silence_top_db == 60
    ys, pitches, lens, trimmed = {}, {}, {}, 0
    for name, sr in zip(names, rates):
        x, native = audio.read_wav(wav_dir / f'{name}.wav')
        assert native == sr
        if sr != 22050:
            x = ro.resample(x, sr, 22050)
        z = audio.normalize_volume(x, increase_only=True)
        y = to.trim(z, 60)
        trimmed += len(y) < len(z)
        ys[name] = y = audio.pad_to_hop(y)
        lens[name] = 1 + len(y) // 256
    assert trimmed >= 6
    click = names[6]
    assert len(ys[click]) < audio.min_mel_samples
    assert pickle.load(open(cm.data_dir / 'mel_len.pkl', 'rb')) == lens
    removed = pickle.load(open(cm.data_dir / 'under-over_sized_mels.pkl', 'rb'))
    assert removed == [n for n in names if not 30 <= lens[n] <= 400] and click in removed
    assert not (cm.mel_dir / f'{click}.npy').exists() and not (cm.pitch_dir / f'{click}.npy').exists()
    for name in names:
        if name == click:
            continue
        mel = np.load(cm.mel_dir / f'{name}.npy')
        assert mel.dtype == np.float32 and np.array_equal(mel, audio.mel_spectrogram(ys[name])), name
        pitches[name] = audio.extract_pitch(ys[name])
    mean, std = ctd.pitch_stats(pitches.values())
    stats = pickle.load(open(cm.data_dir / 'pitch_stats.pkl', 'rb'))
    assert stats == {'pitch_mean': mean, 'pitch_std': std}
    for name, p in pitches.items():
        assert np.array_equal(np.load(cm.pitch_dir / f'{name}.npy'), ctd.normalize_pitch(p, mean, std)), name
    kept = [l.split('|')[0] for l in open(cm.phonemized_metadata_path, encoding='utf-8').read().splitlines()]
    assert kept == [n for n in names if n not in removed]
