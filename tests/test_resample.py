"""CPU tests of resampling to the configured rate (reference: data/audio.py:126-130, librosa.load(sr=...) -> resampy kaiser_best):
the numpy restatement (tests/resample_oracle.py) against a literal scalar transcription of resampy's loop and against known
answers, its output lengths, the argument checks of ttsb_resample_batch without a GPU, and Audio.read_wav."""
import ctypes as C

import numpy as np
import pytest

import resample_oracle as ro

TARGET = 22050


def _literal(x, sr_orig, sr_new, ts):
    """resampy's resample_f for one channel, transcribed statement by statement with Python floats (IEEE float64) and a float32
    output cell, for the output samples `ts` (ascending); the time register runs serially from t = 0."""
    sample_ratio = float(sr_new) / sr_orig
    interp_win = ro.half_window()
    if sample_ratio < 1:
        interp_win = interp_win * sample_ratio
    interp_win = interp_win.tolist()
    interp_delta = [interp_win[j + 1] - interp_win[j] for j in range(len(interp_win) - 1)] + [0.0]
    num_table = 512
    scale = min(1.0, sample_ratio)
    time_increment = 1. / sample_ratio
    index_step = int(scale * num_table)
    time_register = 0.0
    nwin, n_orig = len(interp_win), len(x)
    xs = [float(v) for v in x]
    out, want, t = {}, set(ts), 0
    while t <= ts[-1]:
        if t in want:
            y = np.float32(0.0)
            n = int(time_register)
            frac = scale * (time_register - n)
            index_frac = frac * num_table
            offset = int(index_frac)
            eta = index_frac - offset
            i_max = min(n + 1, (nwin - offset) // index_step)
            for i in range(i_max):
                weight = (interp_win[offset + i * index_step] + eta * interp_delta[offset + i * index_step])
                y = np.float32(float(y) + weight * xs[n - i])
            frac = scale - frac
            index_frac = frac * num_table
            offset = int(index_frac)
            eta = index_frac - offset
            k_max = min(n_orig - n - 1, (nwin - offset) // index_step)
            for k in range(k_max):
                weight = (interp_win[offset + k * index_step] + eta * interp_delta[offset + k * index_step])
                y = np.float32(float(y) + weight * xs[n + k + 1])
            out[t] = y
        time_register += time_increment
        t += 1
    return np.array([out[t] for t in ts], dtype=np.float32)


def test_filter_table():
    h = ro.half_window()
    assert h.dtype == np.float64 and len(h) == 32769
    assert h[0] == 0.9475937167399596 and 1e-8 < h[-1] < 3e-8


@pytest.mark.parametrize('sr', [48000, 44100, 16000])
def test_oracle_equals_a_literal_transcription(sr):
    x = ro.noisy_tones(3 * sr + 17, sr, seed=sr)
    y = ro.resample(x, sr, TARGET)
    n = int(len(x) * TARGET / sr)
    ts = list(range(0, 700)) + list(range(30000, 30600)) + list(range(n - 700, n))   # both clip edges and the middle
    assert np.array_equal(y[ts], _literal(x, sr, TARGET, ts)), sr


def _inner(y):
    return slice(2000, len(y) - 2000)


@pytest.mark.parametrize('sr', [48000, 44100, 24000, 16000])
def test_oracle_known_answers(sr):
    y = ro.resample(ro.tone(1000.0, sr, 2.0), sr, TARGET)
    ideal = 0.5 * np.sin(2 * np.pi * 1000.0 * np.arange(len(y)) / TARGET)
    e = _inner(y)
    assert np.abs(y[e] - ideal[e]).max() < 1e-3
    dc = ro.resample(np.ones(2 * sr, np.float32), sr, TARGET)
    assert np.abs(dc[e] - 1.0).max() < 1e-3


def _level_db(y, amp=0.5):
    e = _inner(y)
    return 20 * np.log10(np.sqrt(np.mean(y[e].astype(np.float64) ** 2)) / (amp / np.sqrt(2)))


def test_oracle_suppresses_tones_above_the_new_nyquist_rate():
    sr = 48000
    assert _level_db(ro.resample(ro.tone(14000.0, sr, 2.0), sr, TARGET)) <= -70
    assert _level_db(ro.resample(ro.tone(11600.0, sr, 2.0), sr, TARGET)) <= -65
    assert _level_db(ro.resample(ro.tone(5000.0, sr, 2.0), sr, TARGET)) > -0.01


def test_oracle_lengths():
    y = ro.resample(np.ones(48001, np.float32), 48000, TARGET)
    assert len(y) == 22051 and y[-1] == 0.0 and y[-2] != 0.0
    assert len(ro.resample(np.ones(3, np.float32), 48000, TARGET)) == 2
    with pytest.raises(ValueError, match='too short'):
        ro.resample(np.ones(2, np.float32), 48000, TARGET)
    x = ro.noisy_tones(1000, TARGET, seed=1)
    same = ro.resample(x, TARGET, TARGET)
    assert same.dtype == np.float32 and np.array_equal(same, x)
    assert len(ro.resample(np.ones(1000, np.float32), 8000, TARGET)) == int(np.ceil(1000 * (TARGET / 8000)))


def test_product_lengths_match_the_oracle():
    from transformertts_b200.data.audio import kaiser_best_half_window, resampled_length
    assert np.array_equal(kaiser_best_half_window(), ro.half_window())
    for L, sr in ((48001, 48000), (3, 48000), (1000, 8000), (12345, 44100), (777, 22050), (5, 16000)):
        assert resampled_length(L, sr, TARGET) == len(ro.resample(np.zeros(L, np.float32), sr, TARGET))
    with pytest.raises(ValueError, match='48000 Hz'):
        resampled_length(2, 48000, TARGET)


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def _i32(*v):
    return (C.c_int32 * len(v))(*v)


def test_resample_refuses_malformed_tables_without_gpu(cdll):
    from transformertts_b200 import lib
    dev = C.c_void_p(256)          # never dereferenced: every check below fails before any CUDA call
    big = C.c_int64(1 << 30)

    def call(so, rates, n, oo, ws=big, dst=TARGET):
        return cdll.ttsb_resample_batch(dev, so, rates, n, dst, dev, 32769, oo, dev, ws, dev, None)

    def err():
        return cdll.ttsb_last_error()

    good_oo = _i32(0, 460, 460 + 1103)        # ceil(1000 * 22050 / 48000), ceil(500 * 22050 / 10000)
    assert call(_i32(5, 1005, 1505), _i32(48000, 10000), 2, good_oo) == -1 and b'start at 0' in err()
    assert call(_i32(0, 1000, 900), _i32(48000, 10000), 2, good_oo) == -1 and b'decrease' in err()
    assert call(_i32(0, 1000, 1500), _i32(48000, 0), 2, good_oo) == -1 and b'rate 0' in err()
    assert call(_i32(0, 1000, 1500), _i32(-8000, 10000), 2, good_oo) == -1 and b'rate -8000' in err()
    assert call(_i32(0, 1000, 1500), _i32(48000, 10000), 2, _i32(0, 459, 459 + 1103)) == -1 and b'ceil' in err()
    assert call(_i32(0, 1000, 1500), _i32(48000, 10000), 2, _i32(1, 461, 461 + 1103)) == -1 and b'start at 0' in err()
    assert call(_i32(0, 1000, 1002), _i32(48000, 48000), 2, _i32(0, 460, 461)) == -1 and b'too short' in err()
    assert call(_i32(0, 1000, 1500), _i32(48000, 10000), 2, good_oo, dst=0) == -1 and b'target rate' in err()
    need = lib.resample_batch_workspace_bytes([0, 1000, 1500], [48000, 10000], TARGET, 32769)
    assert call(_i32(0, 1000, 1500), _i32(48000, 10000), 2, good_oo, ws=C.c_int64(need - 1)) == -1 and b'workspace' in err()
    assert cdll.ttsb_resample_batch(None, _i32(0, 1000), _i32(48000), 1, TARGET, dev, 32769, _i32(0, 460), dev, big, dev, None) == -1
    assert cdll.ttsb_resample_batch_workspace_bytes(_i32(0, 1000), _i32(48000), 0, TARGET, 32769) == -1
    # one phase-ordered table per distinct downsampling ratio (~530 KB each); upsampling shares the unscaled one
    one = lib.resample_batch_workspace_bytes([0, 1000], [48000], TARGET, 32769)
    two = lib.resample_batch_workspace_bytes([0, 1000, 2000], [48000, 44100], TARGET, 32769)
    up = lib.resample_batch_workspace_bytes([0, 1000, 2000], [8000, 16000], TARGET, 32769)
    same = lib.resample_batch_workspace_bytes([0, 1000, 2000], [48000, 48000], TARGET, 32769)
    assert 500_000 < one < same < 600_000 and two > one + 500_000 and 500_000 < up < 700_000
    with pytest.raises(lib.TtsbError, match='too short'):
        lib.resample_batch_workspace_bytes([0, 2], [48000], TARGET, 32769)


def _audio():
    from transformertts_b200.data.audio import Audio
    return Audio(sampling_rate=TARGET, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                 normalizer='MelGAN', norm_wav=True, target_dBFS=-30, int16_max=(2 ** 15) - 1)


def test_read_wav_returns_the_native_rate_and_load_wav_is_unchanged(tmp_path):
    import scipy.io.wavfile
    pcm = (np.random.default_rng(2).standard_normal((3000, 2)) * 3000).astype(np.int16)
    scipy.io.wavfile.write(tmp_path / 'a.wav', 48000, pcm)
    y, sr = _audio().read_wav(tmp_path / 'a.wav')
    assert sr == 48000 and y.dtype == np.float32 and np.array_equal(y, np.mean(pcm.astype(np.float32) / 32768, axis=1))
    with pytest.raises(ValueError, match='48000.*resample'):
        _audio().load_wav(tmp_path / 'a.wav')
    scipy.io.wavfile.write(tmp_path / 'b.wav', TARGET, pcm[:, 0])
    a = _audio()
    y, sr = a.read_wav(tmp_path / 'b.wav')
    assert sr == TARGET and np.array_equal(y, pcm[:, 0].astype(np.float32) / np.float32(32768))
    loaded, sr2 = a.load_wav(tmp_path / 'b.wav')
    assert sr2 == TARGET and loaded.dtype == y.dtype and np.array_equal(loaded, a.preprocess(y))
    assert np.array_equal(a.load_wav(tmp_path / 'b.wav', preprocess=False)[0], y)
