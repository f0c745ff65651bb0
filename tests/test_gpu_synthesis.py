"""Batched waveform synthesis on the GPU: ttsb_griffinlim_batch / Audio.griffinlim_batch_device / reconstruct_waveform_batch
against the numpy restatement of librosa 0.7.1 (oracle/audio_oracle.py) and against the single-clip path, clip independence
bit for bit, and predict_tts.py end to end (reference: predict_tts.py, data/audio.py:94-110, 143-144)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.io.wavfile
import torch

from oracle import audio_oracle as ao

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = Path(__file__).resolve().parent.parent
TOL = {0: 5e-6, 4: 2e-4, 32: 5e-3}          # of full scale, as in tests/test_gpu_audio_inverse.py
LENGTHS = (4, 37, 862, 5, 120, 11)         # frames: the shortest allowed, odd and even, a 10 s clip


def _audio():
    from transformertts_b200.data.audio import Audio
    return Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000, normalizer='MelGAN')


def _clip(T, seed):
    """magnitudes (513, T) of a speech-like clip of T frames and a unit-modulus initial phase."""
    y = ao.make_clips(1, 256 * (T - 1), seed=seed)[0]
    S = np.abs(ao.stft(y)).astype(np.float32)
    assert S.shape == (513, T)
    init = np.exp(2j * np.pi * np.random.default_rng(seed + 1000).random(S.shape)).astype(np.complex64)
    return S, init


def _run_batch(a, clips, n_iter):
    """clips: list of (S (513, T), init (513, T)) -> list of float32 waveforms from one griffinlim_batch_device call."""
    S = torch.from_numpy(np.ascontiguousarray(np.concatenate([s.T for s, _ in clips]))).to(DEV)
    init = torch.from_numpy(np.ascontiguousarray(np.concatenate([i.T for _, i in clips])))
    T = [s.shape[1] for s, _ in clips]
    off = np.concatenate([[0], np.cumsum(T)])
    wav = a.griffinlim_batch_device(S, off, n_iter=n_iter, init_angles=init).cpu().numpy()
    assert wav.shape == (256 * (off[-1] - len(T)),)
    starts = 256 * (off[:-1] - np.arange(len(T)))
    return [wav[s:s + 256 * (t - 1)] for s, t in zip(starts, T)]


@pytest.fixture(scope='module')
def clips():
    return [_clip(T, 20 + i) for i, T in enumerate(LENGTHS)]


@pytest.mark.parametrize('n_iter', [0, 4, 32])
def test_batch_matches_oracle(clips, n_iter):
    got = _run_batch(_audio(), clips, n_iter)
    for c, ((S, init), g) in enumerate(zip(clips, got)):
        want = ao.griffinlim(S, n_iter=n_iter, init_angles=init)
        assert g.shape == want.shape, c
        err = np.abs(g - want).max()
        assert err < TOL[n_iter] * max(1.0, np.abs(want).max()), (c, err)
        e_got = np.linalg.norm(np.abs(ao.stft(g)) - S) / np.linalg.norm(S)
        e_want = np.linalg.norm(np.abs(ao.stft(want)) - S) / np.linalg.norm(S)
        assert e_got < 1.02 * e_want + 1e-4, (c, e_got, e_want)


@pytest.mark.parametrize('n_iter', [0, 32])
def test_batch_matches_single_clip_path(clips, n_iter):
    a = _audio()
    got = _run_batch(a, clips, n_iter)
    for c, ((S, init), g) in enumerate(zip(clips, got)):
        one = a.griffinlim_device(torch.from_numpy(np.ascontiguousarray(S.T)).to(DEV), n_iter=n_iter,
                                  init_angles=torch.from_numpy(np.ascontiguousarray(init.T))).cpu().numpy()
        err = np.abs(g - one).max()
        assert err <= (1e-6 if n_iter == 0 else TOL[32]) * max(1.0, np.abs(one).max()), (c, err)
        # the fused projection computes the bits of ttsb_griffinlim_update and the frame pairs are those of the single-clip
        # kernels, so the two paths agree exactly
        assert np.array_equal(g, one), (c, err)


def test_clip_independence_bit_for_bit(clips):
    a = _audio()
    alone = [_run_batch(a, [cl], 32)[0] for cl in clips[:3]]
    together = _run_batch(a, clips[:3], 32)
    moved = _run_batch(a, [clips[2], clips[0], clips[1]], 32)
    others = [_clip(9, 77), _clip(6, 78)]
    neighbours = _run_batch(a, [others[0], clips[1], others[1], clips[0], clips[2]], 32)
    for c in range(3):
        assert np.array_equal(together[c], alone[c]), c
    assert np.array_equal(moved[0], alone[2]) and np.array_equal(moved[1], alone[0]) and np.array_equal(moved[2], alone[1])
    assert np.array_equal(neighbours[1], alone[1]) and np.array_equal(neighbours[3], alone[0]) and np.array_equal(neighbours[4], alone[2])


def _mels(a, lengths, seed):
    return [a.mel_spectrogram(ao.make_clips(1, 256 * (T - 1), seed=seed + i)[0]).T for i, T in enumerate(lengths)]   # (80, T)


def test_reconstruct_waveform_batch_matches_per_clip():
    a = _audio()
    mels = _mels(a, (173, 4, 862, 50, 7), seed=40)
    got = a.reconstruct_waveform_batch(mels, seed=11)
    assert len(got) == len(mels)
    for c, (m, g) in enumerate(zip(mels, got)):
        want = a.reconstruct_waveform(m, seed=11 + c)
        assert g.dtype == np.float32 and g.shape == want.shape == (256 * (m.shape[1] - 1),), c
        err = np.abs(g - want).max()
        assert err < TOL[32] * max(1.0, np.abs(want).max()), (c, err)
    # the mel inversion is per frame: packed frames give the bits of the per-clip call
    amp = [np.ascontiguousarray(np.exp(m).T.astype(np.float32)) for m in mels]
    packed = a.mel_to_linear_device(torch.from_numpy(np.concatenate(amp)).to(DEV)).cpu().numpy()
    single = np.concatenate([a.mel_to_linear_device(torch.from_numpy(x).to(DEV)).cpu().numpy() for x in amp])
    assert np.array_equal(packed, single)
    # explicit phases reproduce reconstruct_waveform's init_angles argument
    init = [np.exp(2j * np.pi * np.random.default_rng(5 + c).random((513, m.shape[1]))).astype(np.complex64) for c, m in enumerate(mels[:2])]
    got = a.reconstruct_waveform_batch(mels[:2], n_iter=4, init_angles=init)
    for c in range(2):
        assert np.array_equal(got[c], a.reconstruct_waveform(mels[c], n_iter=4, init_angles=init[c])), c


def test_launch_count_does_not_depend_on_the_number_of_clips():
    from transformertts_b200 import lib
    a = _audio()
    mels = _mels(a, [20 + 3 * i for i in range(16)], seed=60)
    counts = []
    for batch in (mels[:1], mels):
        a.reconstruct_waveform_batch(batch, n_iter=8, seed=0)
        torch.cuda.synchronize()
        lib.reset_launch_count()
        a.reconstruct_waveform_batch(batch, n_iter=8, seed=0)
        counts.append(lib.launch_count())
    assert counts[0] == counts[1] == 1 + 1 + 3 * 8 + 2, counts     # mel inversion, clip table, 8 x 3 stages, last iSTFT


def test_short_clips_are_refused():
    a = _audio()
    mels = [np.random.default_rng(80 + c).normal(-3, 1, (80, T)).astype(np.float32) for c, T in enumerate((10, 3, 10))]
    with pytest.raises(ValueError, match='mel 1'):
        a.reconstruct_waveform_batch(mels)
    S = torch.ones((12, 513), device=DEV)
    with pytest.raises(ValueError, match='clip 1 has 2 frames'):
        a.griffinlim_batch_device(S, [0, 10, 12])
    with pytest.raises(ValueError, match='frame offsets'):
        a.griffinlim_batch_device(S, [0, 4, 11])
    with pytest.raises(ValueError, match='frame offsets'):
        a.griffinlim_batch_device(S, [1, 6, 12])


def test_predict_tts_end_to_end(tmp_path):
    from oracle import forward_oracle as fo
    from transformertts_b200.model.models import ForwardTransformer
    cfg = dict(fo.CONFIGS['C1'], sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000,
               normalizer='MelGAN', data_name='ljspeech')
    p = fo.init_params(cfg, seed=7)
    p['dur_pred.out.b'] = torch.tensor([6.0])         # about 6 frames per phoneme from the seeded weights
    model = ForwardTransformer(**cfg)
    model.set_weights(p)
    model.save_model(tmp_path / 'model', with_optimizer=False)
    lines = ['həloʊ wɜːld', 'ðɪs ɪz ɐ lɔŋɡɚ tɛst sɛntəns.', 'ɐbɐ']
    (tmp_path / 'lines.txt').write_text('\n'.join(lines) + '\n')
    r = subprocess.run([sys.executable, str(ROOT / 'predict_tts.py'), '-p', str(tmp_path / 'model'), '-f', str(tmp_path / 'lines.txt'),
                        '-o', str(tmp_path / 'out'), '-m', '-s'], capture_output=True, text=True, timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    out = tmp_path / 'out' / 'outputs' / 'lines'
    stem = 'lines_ljspeech_unknown_0'                    # no git hash in a model saved here; step 0
    assert (out / f'{stem}.wav').exists(), sorted(x.name for x in out.iterdir())
    loaded = ForwardTransformer.load_model(tmp_path / 'model')
    from transformertts_b200.data.text import Tokenizer
    tok = Tokenizer(add_start_end=False, model_breathing=False, alphabet=loaded.alphabet)
    mels = []
    for i, line in enumerate(lines):
        mel = loaded.predict(tok(line), encode=False, phoneme_max_duration=None)['mel'].cpu().numpy()
        assert mel.shape[0] >= 4, mel.shape
        assert np.array_equal(np.load(out / f'{stem}_{i}.mel.npy'), mel), i
        mels.append(mel)
    a = _audio()
    wavs = a.reconstruct_waveform_batch([m.T for m in mels], seed=0)
    pcm = []
    for i, w in enumerate(wavs):
        a.save_wav(w, tmp_path / f'want_{i}.wav')
        sr, want = scipy.io.wavfile.read(tmp_path / f'want_{i}.wav')
        sr_got, got = scipy.io.wavfile.read(out / f'{stem}_{i}.wav')
        assert sr_got == sr == 22050 and got.dtype == np.int16 and np.array_equal(got, want), i
        single = a.reconstruct_waveform(mels[i].T, seed=i)
        # the seeded model's waveforms exceed full scale: save_wav clips them, and clipping does not widen a difference
        clipped = np.clip(single, -32768 / 32767, 1.0)
        assert np.abs(got / 32767.0 - clipped).max() < TOL[32] * max(1.0, np.abs(single).max()) + 1.0 / 32767, i
        pcm.append(got)
    _, combined = scipy.io.wavfile.read(out / f'{stem}.wav')
    assert np.array_equal(combined, np.concatenate(pcm))
