"""The audio front end and Griffin-Lim at STFT settings other than n_fft 1024 / hop 256 / win 1024 (csrc/stft_general.cu), against
the numpy restatement of librosa 0.7.1 (oracle/audio_oracle.py) and WORLD (oracle/pitch_oracle.py), with the gates the reference
configuration's kernels meet; ragged batches bit for bit against each clip alone; the scripts end to end with the reference's
WaveRNN audio section (22050 Hz, n_fft 2048, hop 275, win 1100, f_min 40, f_max None)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.io.wavfile
import torch
import yaml

from oracle import audio_oracle as ao
from oracle import pitch_oracle as po

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = Path(__file__).resolve().parent.parent

WAVERNN = dict(sampling_rate=22050, n_fft=2048, hop_length=275, win_length=1100, f_min=40, f_max=None, normalizer='WaveRNN')
CONFIGS = {
    'wavernn': WAVERNN,
    '24k': dict(sampling_rate=24000, n_fft=2048, hop_length=300, win_length=1200, f_min=0, f_max=12000, normalizer='MelGAN'),
    '16k_800': dict(sampling_rate=16000, n_fft=1024, hop_length=200, win_length=800, f_min=0, f_max=8000, normalizer='MelGAN'),
    '16k_512': dict(sampling_rate=16000, n_fft=512, hop_length=128, win_length=512, f_min=0, f_max=8000, normalizer='MelGAN'),
    '48k_4096': dict(sampling_rate=48000, n_fft=4096, hop_length=1024, win_length=4096, f_min=0, f_max=None, normalizer='MelGAN',
                     mel_channels=128),
    'reference': dict(sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000, normalizer='MelGAN'),
}


def _audio(name, **kw):
    from transformertts_b200.data.audio import Audio
    settings = {'mel_channels': 80, **CONFIGS[name]}
    settings.update(kw)
    return Audio(**settings)


def _fmax(a):
    return a.f_max


def _lengths(a):
    """the minimum length, multiples of the hop, odd lengths and 10 s"""
    h, n = a.hop_length, a.n_fft
    return [n // 2 + 1, h * 7, h * 13 + 1, n + 101, 12345, 10 * a.sampling_rate]


def _oracle_mel(a, y, normalizer):
    return ao.mel_spectrogram(y, a.sampling_rate, a.n_fft, a.hop_length, a.win_length, a.mel_channels, a.f_min, _fmax(a), normalizer)


def _general_mel(a, clips):
    """log-mels of a list of clips through ttsb_stft_mel_log_ragged (whatever the configuration) -> list of arrays"""
    from transformertts_b200 import lib
    wav, so = a._pack(clips)
    fo = np.concatenate([[0], np.cumsum(a._frames_per_clip(np.diff(so)))])
    out = torch.full((int(fo[-1]), a.mel_channels), float('nan'), device=DEV)
    lib.stft_mel_log_ragged(wav, so, fo, a.n_fft, a.hop_length, a.win_length, a._mel_basis(), a._inverse_tables()['band'],
                            a.normalizer.code, out)
    out = out.cpu().numpy()
    return [out[x:y] for x, y in zip(fo[:-1], fo[1:])]


@pytest.mark.parametrize('name', list(CONFIGS))
@pytest.mark.parametrize('normalizer', ['MelGAN', 'WaveRNN'])
def test_log_mel_matches_oracle(name, normalizer):
    a = _audio(name, normalizer=normalizer)
    clips = [ao.make_clips(1, L, seed=L % 1000)[0] for L in _lengths(a)]
    got = _general_mel(a, clips)
    via_audio = a.mel_spectrogram_ragged(clips)
    for y, g, v in zip(clips, got, via_audio):
        want = _oracle_mel(a, y, normalizer)
        assert g.shape == want.shape == (1 + len(y) // a.hop_length, a.mel_channels)
        assert float(np.abs(g - want).max()) < 1e-3, (len(y), float(np.abs(g - want).max()))
        if name != 'reference':
            assert np.array_equal(v, g)
    if name == 'reference':   # the general kernel against the fused kernel of the reference configuration
        diff = max(float(np.abs(g - v).max()) for g, v in zip(got, via_audio))
        print(f'reference configuration, {normalizer}: largest |general - fused| log-mel difference {diff:.3g}')
        assert diff < 1e-3


@pytest.mark.parametrize('name', ['wavernn', '16k_512', '48k_4096'])
def test_ragged_log_mel_bit_identical_to_each_clip_alone(name):
    a = _audio(name)
    rng = np.random.default_rng(3)
    lens = [a.n_fft // 2 + 1, a.hop_length * 9, a.hop_length * 9 + 1] + [int(x) for x in rng.integers(a.n_fft, 4 * a.sampling_rate, 9)]
    clips = [ao.make_clips(1, L, seed=i)[0] * np.float32(rng.uniform(0.3, 1.0)) for i, L in enumerate(lens)]
    alone = [a.mel_spectrogram(y) for y in clips]
    batch = a.mel_spectrogram_ragged(clips)
    rev = a.mel_spectrogram_ragged(clips[::-1])[::-1]
    again = a.mel_spectrogram_ragged(clips)
    moved = a.mel_spectrogram_ragged([clips[4], clips[0], clips[4]])
    for x, b, r, g in zip(alone, batch, rev, again):
        assert np.array_equal(x, b) and np.array_equal(x, r) and np.array_equal(x, g)
    assert np.array_equal(moved[0], alone[4]) and np.array_equal(moved[2], alone[4]) and np.array_equal(moved[1], alone[0])
    dense = a.mel_spectrogram_batch(np.stack([clips[3], clips[3]]))
    assert np.array_equal(dense[0], alone[3]) and np.array_equal(dense[1], alone[3])


@pytest.mark.parametrize('name', list(CONFIGS))
def test_complex_stft_and_istft(name):
    from transformertts_b200 import lib
    a = _audio(name)
    n, h = a.n_fft, a.hop_length
    clips = [ao.make_clips(1, L, seed=L % 997)[0] for L in (n // 2 + 1 + 3 * h, 5000 + n, 22050)]
    wav, so = a._pack(clips)
    T = [1 + len(y) // h for y in clips]
    fo = np.concatenate([[0], np.cumsum(T)])
    spec = torch.full((int(fo[-1]), n // 2 + 1, 2), float('nan'), device=DEV)
    lib.stft_complex_ragged(wav, so, n, h, a.win_length, spec)
    got = torch.view_as_complex(spec).cpu().numpy()
    Ds = []
    for y, x0, x1 in zip(clips, fo[:-1], fo[1:]):
        D = ao.stft(y, n, h, a.win_length)
        scale = np.abs(D).max()
        assert np.abs(got[x0:x1].T - D).max() < 2e-6 * scale + 1e-5
        D2 = D.copy()
        D2[0] += 0.3j                                  # irfft ignores the imaginary DC / Nyquist parts
        D2[-1] -= 0.7j
        Ds.append(D2)
    packed = torch.view_as_real(torch.from_numpy(np.ascontiguousarray(np.concatenate([D.T for D in Ds]))).to(DEV)).contiguous()
    out = torch.full((h * (int(fo[-1]) - len(clips)),), float('nan'), device=DEV)
    lib.istft_ragged(packed, fo, n, h, a.win_length, out)
    out = out.cpu().numpy()
    for c, (y, D) in enumerate(zip(clips, Ds)):
        w = out[h * (fo[c] - c):h * (fo[c + 1] - c - 1)]
        want = ao.istft(D, h, a.win_length)
        assert w.shape == want.shape and np.abs(w - want).max() < 2e-6, (c, float(np.abs(w - want).max()))
        assert np.abs(w - y[:len(want)]).max() < 5e-6


@pytest.mark.parametrize('name', ['wavernn', '48k_4096'])
def test_mel_inversion_matches_oracle_solver(name):
    a = _audio(name)
    y = ao.make_clips(1, a.sampling_rate, seed=8)[0]
    amp = np.exp(_oracle_mel(a, y, 'MelGAN')).astype(np.float32)                 # (T, n_mels)
    got = a.mel_to_linear_device(torch.from_numpy(amp).to(DEV), n_iter=64).cpu().numpy().T
    want = ao.mel_to_stft(amp.T, sr=a.sampling_rate, n_fft=a.n_fft, fmin=a.f_min, fmax=_fmax(a), solver='pg', n_iter=64)
    assert got.shape == want.shape == (a.n_fft // 2 + 1, amp.shape[0]) and got.min() >= 0
    assert np.linalg.norm(got - want) / np.linalg.norm(want) < 1e-4


@pytest.mark.parametrize('name', list(CONFIGS))
def test_griffinlim_with_shared_initial_phase(name):
    a = _audio(name)
    y = ao.make_clips(1, max(16000, 6 * a.n_fft), seed=9)[0]
    S = ao.mel_to_stft(np.exp(_oracle_mel(a, y, 'MelGAN')).T.astype(np.float32), sr=a.sampling_rate, n_fft=a.n_fft, fmin=a.f_min,
                       fmax=_fmax(a), solver='pg', n_iter=64)
    init = np.exp(2j * np.pi * np.random.default_rng(11).random(S.shape)).astype(np.complex64)
    from transformertts_b200 import lib
    for n_iter, tol in ((0, 5e-6), (32, 5e-3)):
        want = ao.griffinlim(S, n_iter=n_iter, hop_length=a.hop_length, win_length=a.win_length, init_angles=init)
        wav = torch.full((a.hop_length * (S.shape[1] - 1),), float('nan'), device=DEV)
        lib.griffinlim_ragged(torch.from_numpy(np.ascontiguousarray(S.T)).to(DEV), torch.from_numpy(np.ascontiguousarray(init.T)).to(DEV),
                              [0, S.shape[1]], a.n_fft, a.hop_length, a.win_length, n_iter, 0.99, wav)
        got = wav.cpu().numpy()
        assert got.shape == want.shape
        assert np.abs(got - want).max() < tol * max(1.0, np.abs(want).max()), (n_iter, float(np.abs(got - want).max()))
        if name != 'reference':
            via_audio = a.griffinlim_device(torch.from_numpy(np.ascontiguousarray(S.T)).to(DEV), n_iter=n_iter,
                                            init_angles=torch.from_numpy(np.ascontiguousarray(init.T)))
            assert np.array_equal(via_audio.cpu().numpy(), got)
        else:
            fused = a.griffinlim_device(torch.from_numpy(np.ascontiguousarray(S.T)).to(DEV), n_iter=n_iter,
                                        init_angles=torch.from_numpy(np.ascontiguousarray(init.T))).cpu().numpy()
            print(f'reference configuration, {n_iter} iterations: largest |general - fused| sample difference '
                  f'{float(np.abs(fused - got).max()):.3g}')
    e_got = np.linalg.norm(np.abs(ao.stft(got, a.n_fft, a.hop_length, a.win_length)) - S) / np.linalg.norm(S)
    e_want = np.linalg.norm(np.abs(ao.stft(want, a.n_fft, a.hop_length, a.win_length)) - S) / np.linalg.norm(S)
    assert e_got < 1.02 * e_want + 1e-4


@pytest.mark.parametrize('name', ['wavernn', '16k_800', '48k_4096'])
def test_ragged_griffinlim_bit_identical_to_each_clip_alone(name):
    a = _audio(name)
    rng = np.random.default_rng(4)
    m = a.min_griffinlim_frames
    frames = [m, m + 1, 2 * m + 3] + [int(x) for x in rng.integers(m, 120, 5)]
    mels = [_oracle_mel(a, ao.make_clips(1, a.hop_length * (t - 1), seed=i)[0], a.normalizer.__class__.__name__).T
            if a.hop_length * (t - 1) > a.n_fft // 2 else None for i, t in enumerate(frames)]
    mels = [x for x in mels if x is not None]
    alone = [a.reconstruct_waveform(x, n_iter=8, seed=20 + i) for i, x in enumerate(mels)]
    batch = a.reconstruct_waveform_batch(mels, n_iter=8, seed=20)
    rev = a.reconstruct_waveform_batch(mels[::-1], n_iter=8, init_angles=None, seed=None)   # exercise the unseeded path's shapes
    assert [len(w) for w in rev] == [a.hop_length * (x.shape[1] - 1) for x in mels[::-1]]
    again = a.reconstruct_waveform_batch(mels, n_iter=8, seed=20)
    for x, w, b, g in zip(mels, alone, batch, again):
        assert w.shape == (a.hop_length * (x.shape[1] - 1),) and np.isfinite(w).all()
        assert np.array_equal(w, b) and np.array_equal(w, g)
    # the same clip at other positions, with the same phase draw
    init = [np.exp(2j * np.pi * np.random.default_rng(i).random((a.n_fft // 2 + 1, x.shape[1]))).astype(np.complex64)
            for i, x in enumerate(mels)]
    fwd = a.reconstruct_waveform_batch(mels, n_iter=8, init_angles=init)
    bwd = a.reconstruct_waveform_batch(mels[::-1], n_iter=8, init_angles=init[::-1])[::-1]
    for f, b in zip(fwd, bwd):
        assert np.array_equal(f, b)
    with pytest.raises(ValueError, match=f'T >= {m}'):
        a.reconstruct_waveform_batch([mels[0][:, :m - 1]])


def test_pitch_frames_match_mel_frames_and_oracle_at_hop_275():
    a = _audio('wavernn')
    lengths = [L for L in range(1000, 5001) if L % 275 != 0]
    rng = np.random.default_rng(1)
    clips = [(0.1 * rng.standard_normal(L)).astype(np.float32) for L in lengths]
    for i in range(0, len(clips), 1000):
        part = clips[i:i + 1000]
        f0 = a.extract_pitch_batch(part)
        assert [len(f) for f in f0] == [1 + len(x) // 275 for x in part]
        long_enough = [x for x in part if len(x) > a.n_fft // 2]     # the log-mel's reflect padding needs more than 1024 samples
        mel = a.mel_spectrogram_ragged(long_enough)
        assert [len(m) for m in mel] == [1 + len(x) // 275 for x in long_enough]
    fs, hop = 22050, 275
    corpus = po.make_corpus(8, seed=3, min_s=1.0, max_s=6.0)
    corpus = [x if len(x) % hop else np.pad(x, (0, 1)) for x in corpus]
    got = a.extract_pitch_batch(corpus)
    worst = 0.0
    for x, f in zip(corpus, got):
        ref = po.extract_pitch(x, fs, hop)
        assert f.shape == ref.shape == (1 + len(x) // hop,)
        voiced = ref != 0
        assert np.array_equal(f != 0, voiced)
        if voiced.any():
            worst = max(worst, float(np.max(np.abs(f[voiced] / ref[voiced] - 1))))
    assert worst < 1e-6, worst
    assert sum(int((f != 0).sum()) for f in got) > 0.3 * sum(len(f) for f in got)


def _wavernn_section():
    return dict(WAVERNN, mel_channels=80)


def test_create_training_data_with_the_wavernn_audio_section(tmp_path):
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    wav_dir = tmp_path / 'wavs'
    wav_dir.mkdir()
    a = _audio('wavernn')
    clips = po.make_corpus(10, seed=9, min_s=1.0, max_s=3.0)
    names = [f'LJ{i:03d}-{i:04d}' for i in range(len(clips))]
    rng = np.random.default_rng(0)
    phon = sorted(set('abdefhijklmnoprstuvwzæðŋɑɔəɛɪʃʊʌθ'))
    lines = []
    for name, x in zip(names, clips):
        a.save_wav(x, wav_dir / f'{name}.wav')
        lines.append(f"{name}|raw text|{''.join(rng.choice(phon, int(rng.integers(5, 30))))}\n")
    (tmp_path / 'metadata.csv').write_text(''.join(lines), encoding='utf-8')
    cfg = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    cfg['audio_settings'].update(_wavernn_section())
    cfg['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'),
                        metadata_path=str(tmp_path / 'metadata.csv'), wav_directory=str(wav_dir))
    cfg['training_data_settings'].update(n_test=2, min_mel_len=10, max_mel_len=1000)
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, str(ROOT / 'create_training_data.py'), '--config', str(tmp_path / 'cfg.yaml')], cwd=tmp_path,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    cm = TrainingConfigManager(tmp_path / 'cfg.yaml', aligner=True)
    assert cm.config['hop_length'] == 275
    pitches = {}
    for name in names:
        y = a.load_wav(wav_dir / f'{name}.wav')[0]
        mel = np.load(cm.mel_dir / f'{name}.npy')
        assert mel.dtype == np.float32 and np.array_equal(mel, a.mel_spectrogram(y)), name
        pitches[name] = a.extract_pitch(y)
        assert len(pitches[name]) == mel.shape[0]
    mean, std = po.pitch_stats(pitches.values())
    for name in names:
        p, ref = np.load(cm.pitch_dir / f'{name}.npy'), po.normalize_pitch(pitches[name], mean, std)
        assert np.array_equal(p == 0, ref == 0) and np.allclose(p, ref, rtol=0, atol=1e-9), name


def _wavernn_model(tmp_path):
    from oracle import forward_oracle as fo
    from transformertts_b200.model.models import ForwardTransformer
    cfg = dict(fo.CONFIGS['C1'], **_wavernn_section(), data_name='ljspeech')
    p = fo.init_params(cfg, seed=7)
    p['dur_pred.out.b'] = torch.tensor([6.0])
    model = ForwardTransformer(**cfg)
    model.set_weights(p)
    model.save_model(tmp_path / 'model', with_optimizer=False)
    return model


def test_predict_tts_griffinlim_at_hop_275_and_vocoder_hop_refusal(tmp_path):
    _wavernn_model(tmp_path)
    lines = ['həloʊ wɜːld', 'ðɪs ɪz ɐ lɔŋɡɚ tɛst sɛntəns.']
    (tmp_path / 'lines.txt').write_text('\n'.join(lines) + '\n')
    r = subprocess.run([sys.executable, str(ROOT / 'predict_tts.py'), '-p', str(tmp_path / 'model'), '-f', str(tmp_path / 'lines.txt'),
                        '-o', str(tmp_path / 'out'), '-m', '-s'], capture_output=True, text=True, timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    out = tmp_path / 'out' / 'outputs' / 'lines'
    stem = 'lines_ljspeech_unknown_0'
    total = 0
    for i in range(len(lines)):
        mel = np.load(out / f'{stem}_{i}.mel.npy')
        sr, wav = scipy.io.wavfile.read(out / f'{stem}_{i}.wav')
        assert sr == 22050 and len(wav) == 275 * (mel.shape[0] - 1), (len(wav), mel.shape)
        total += len(wav)
    assert len(scipy.io.wavfile.read(out / f'{stem}.wav')[1]) == total
    for voc in ('melgan', 'hifigan'):
        r = subprocess.run([sys.executable, str(ROOT / 'predict_tts.py'), '-p', str(tmp_path / 'model'), '-f', str(tmp_path / 'lines.txt'),
                            '-o', str(tmp_path / 'out2'), '--vocoder', voc, '--vocoder_checkpoint', str(tmp_path / 'missing.pt')],
                           capture_output=True, text=True, timeout=900, cwd=str(ROOT))
        assert r.returncode != 0 and '256' in r.stderr and '275' in r.stderr, r.stderr[-2000:]


def test_evaluate_tts_with_the_wavernn_audio_section(tmp_path):
    """evaluate_tts.py at 22050 / 2048 / 275 / 1100 with the WaveRNN normaliser, Griffin-Lim copy synthesis included: with the
    model's own outputs as targets every error is 0, and the vocoded scores are finite."""
    import json
    import pickle
    from oracle import forward_oracle as fo
    from transformertts_b200.data.text import ALL_PHONEMES
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils import evaluation as ev
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    raw['audio_settings'].update(_wavernn_section())
    raw['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'))
    raw['training_data_settings'].update(bucket_boundaries=[200], bucket_batch_sizes=[2, 2], val_bucket_batch_size=[2, 2])
    cfg_path = tmp_path / 'cfg.yaml'
    cfg_path.write_text(yaml.safe_dump(raw))
    cm = TrainingConfigManager(str(cfg_path))
    cfg = dict(fo.CONFIGS['C1'], **_wavernn_section(), data_name='ljspeech')
    p = fo.init_params(cfg, seed=7)
    p['dur_pred.out.b'] = torch.tensor([3.0])
    model = ForwardTransformer(**cfg)
    model.set_weights(p)
    model.save_model(tmp_path / 'weights' / 'step_0', with_optimizer=False)
    rng = np.random.default_rng(12)
    letters = [c for c in ALL_PHONEMES if c.isalpha()][:30] + [' ']
    lines = {f'w{i:03d}': ''.join(rng.choice(letters, int(rng.integers(8, 24)))) for i in range(6)}
    outs = model.predict_batch(ev.tokenize(model, list(lines.values())), encode=False, phoneme_max_duration=None)
    for d in (cm.data_dir, cm.mel_dir, cm.duration_dir, cm.pitch_per_char):
        d.mkdir(parents=True, exist_ok=True)
    for name, o in zip(lines, outs):
        mel = o['mel'].cpu().numpy()
        np.save(cm.mel_dir / f'{name}.npy', mel.astype(np.float32))
        np.save(cm.duration_dir / f'{name}.npy', o['int_durations'].cpu().numpy().astype(np.int32))
        np.save(cm.pitch_per_char / f'{name}.npy', o['pitch'].cpu().numpy().reshape(-1).astype(np.float32))
    rows = [f'{n}|{ph}\n' for n, ph in lines.items()]
    cm.train_metadata_path.write_text(''.join(rows[:-4]), encoding='utf-8')
    cm.valid_metadata_path.write_text(''.join(rows[-4:]), encoding='utf-8')
    with open(cm.data_dir / 'pitch_stats.pkl', 'wb') as f:
        pickle.dump({'pitch_mean': np.float64(205.7), 'pitch_std': np.float64(41.3)}, f)
    r = subprocess.run([sys.executable, str(ROOT / 'evaluate_tts.py'), '--config', str(cfg_path), '-p', str(tmp_path / 'weights' / 'step_0'),
                        '-o', str(tmp_path / 'out'), '--vocoder', 'griffinlim'], capture_output=True, text=True, timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    res = json.loads((tmp_path / 'out' / 'evaluation.json').read_text())['checkpoints'][0]
    assert [ln['name'] for ln in res['lines']] == list(lines)[-4:]
    for ln in res['lines']:
        assert ln['mcd'] == ln['dtw_cost'] == ln['teacher_forced_mcd'] == 0.0 and ln['path_len'] == ln['frames_recorded'], ln
        assert ln['duration_mae'] == 0.0 and ln['duration_exact'] == 1.0 and ln['pitch_rmse'] == 0.0, ln
        assert np.isfinite(ln['vocoded_mcd']) and np.isfinite(ln['copy_synthesis_mcd']) and ln['copy_synthesis_path_len'] > 0, ln
