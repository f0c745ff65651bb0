"""CPU tests of the silence trim (reference: data/audio.py:164-169, librosa.effects.trim(y, top_db, frame_length=256,
hop_length=64)): the numpy restatement (tests/trim_oracle.py) against hand-computed answers and a literal np.pad computation, the
argument checks of ttsb_trim_silence_bounds without a GPU, the refused settings, and how often librosa's float32 arithmetic
decides differently from float64 on a seeded corpus."""
import ctypes as C
import math

import numpy as np
import pytest

import trim_oracle as to

EDGE_LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257)


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def _i32(*v):
    return (C.c_int32 * len(v))(*v)


def _audio(**kw):
    from transformertts_b200.data.audio import Audio
    return Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                 normalizer='MelGAN', **kw)


def _burst(L, a, b, amp=0.5):
    y = np.zeros(L, np.float32)
    y[a:b] = amp
    return y


def test_known_answers():
    # a 100-sample burst at [1000, 1100) in digital silence, L = 2560 (a multiple of 64).  Frame t covers samples
    # [64 t - 128, 64 t + 128): frames 14-19 overlap the burst; frame 14 holds 24 burst samples (-6.2 dB against the 100 of
    # frames 15-17), frame 18 76 (-1.2 dB), frame 19 12 (-9.2 dB); every other frame is zero, i.e. 10 log10(1e-10) = -100 dB
    # against -10.1 dB for the loudest.
    y = _burst(2560, 1000, 1100)
    assert to.bounds64(y, 60) == (14 * 64, 20 * 64)
    assert to.bounds64(y, 8) == (14 * 64, 19 * 64)                        # frame 19 (-9.2 dB) is silent at top_db 8
    assert to.bounds64(y, 5) == (15 * 64, 19 * 64)                        # and frame 14 (-6.2 dB) at 5
    # a burst touching the first sample, L = 3000: frame 0 reads it and its reflection, frames 1-2 the burst, frame 3 is zero
    assert to.bounds64(_burst(3000, 0, 50), 60) == (0, 3 * 64)
    # touching the last sample: frames 45 and 46 (the last, 1 + 3000 // 64 = 47 frames) overlap it; end = min(L, 64 * 47)
    assert to.bounds64(_burst(3000, 2950, 3000), 60) == (45 * 64, 3000)
    # L a multiple of 64: the last frame is 40; the burst reaches frames 38-40; end = min(2560, 64 * 41) = 2560
    assert to.bounds64(_burst(2560, 2500, 2560), 60) == (38 * 64, 2560)
    # all zeros: every frame clamps to amin, 0 dB, and the clip is kept whole
    for L in (1, 64, 1000):
        assert to.bounds64(np.zeros(L, np.float32), 60) == (0, L)
    # a quiet burst (amplitude 1e-3: the loudest frame -64.1 dB re 1): the zero frames clamp to -100 dB, which is -35.9 dB
    # relative, non-silent at top_db 60 and silent at 20
    quiet = _burst(2560, 1000, 1100, amp=1e-3)
    assert to.bounds64(quiet, 60) == (0, 2560)
    assert to.bounds64(quiet, 20) == (14 * 64, 20 * 64)
    assert to.bounds32(quiet, 60) == (0, 2560) and to.bounds32(y, 60) == (14 * 64, 20 * 64)


def _literal_bounds(y, top_db):
    """The algorithm written out frame by frame on np.pad's reflect padding, sums in float64 -> (bounds, powers)."""
    x = np.pad(y.astype(np.float64), 128, mode='reflect')
    n = 1 + len(y) // 64
    assert len(x) == len(y) + 256
    p = np.array([np.sum(x[64 * t:64 * t + 256] ** 2) / 256 for t in range(n)])
    db = 10 * np.log10(np.maximum(1e-10, p)) - 10 * np.log10(np.maximum(1e-10, p.max()))
    nz = np.flatnonzero(db > -top_db)
    return (int(64 * nz[0]), int(min(len(y), 64 * (nz[-1] + 1)))), p


@pytest.mark.parametrize('L', EDGE_LENGTHS)
def test_short_clips_against_np_pad(L):
    rng = np.random.default_rng(L)
    for k in range(4):
        y = np.zeros(L, np.float32)
        y[rng.integers(0, L, size=max(1, L // 16))] = rng.standard_normal(max(1, L // 16)).astype(np.float32)
        if k == 0:
            y[:] = rng.standard_normal(L).astype(np.float32)
        for top_db in (3, 20, 60):
            want, p = _literal_bounds(y, top_db)
            assert np.allclose(to.powers64(y), p, rtol=1e-12, atol=0), (L, k)
            assert to.bounds64(y, top_db) == want, (L, k, top_db)
    assert to.bounds64(np.array([0.25], np.float32), 60) == (0, 1)       # one sample, padded with copies of itself


def test_trim_refuses_bad_arguments_without_gpu(cdll):
    dev = C.c_void_p(256)          # never dereferenced: every check below fails before any CUDA call
    ws = C.c_int64(1 << 30)

    def call(so, n, top_db=60.0, nbytes=ws):
        return cdll.ttsb_trim_silence_bounds(dev, so, n, C.c_double(top_db), dev, nbytes, dev, None)

    from transformertts_b200 import lib
    lib.load()
    assert call(_i32(5, 100), 1) == -1 and b'start at 0' in cdll.ttsb_last_error()
    assert call(_i32(0, 100, 50), 2) == -1 and b'decrease at clip 1' in cdll.ttsb_last_error()
    assert call(_i32(0, 100, 100, 300), 3) == -1 and b'clip 1 is empty' in cdll.ttsb_last_error()
    for bad in (0.0, -1.0, math.nan, math.inf, -math.inf):
        assert call(_i32(0, 100), 1, top_db=bad) == -1 and b'top_db' in cdll.ttsb_last_error(), bad
    need = lib.trim_silence_workspace_bytes([0, 100, 1000])
    assert need == cdll.ttsb_trim_silence_workspace_bytes(_i32(0, 100, 1000), 2) > 8 * (1 + 100 // 64 + 1 + 900 // 64)
    assert call(_i32(0, 100, 1000), 2, nbytes=C.c_int64(need - 1)) == -1 and b'workspace too small' in cdll.ttsb_last_error()
    assert cdll.ttsb_trim_silence_bounds(None, _i32(0, 100), 1, C.c_double(60.0), dev, ws, dev, None) == -1
    assert b'NULL' in cdll.ttsb_last_error()
    assert call(_i32(0, 100), 0) == -1
    assert cdll.ttsb_trim_silence_workspace_bytes(_i32(0, 100, 100), 2) == -1
    assert cdll.ttsb_trim_silence_workspace_bytes(_i32(0, 100), 0) == -1


def test_trim_settings_refusals():
    y = np.zeros(1000, np.float32)
    # trim_silence without trim_silence_top_db: librosa.effects.trim would get top_db=None; refused before any GPU work
    for call in (lambda a: a.preprocess(y), lambda a: a.trim_audio_silence(y), lambda a: a.preprocess_before_trim(y)):
        with pytest.raises(NotImplementedError, match=r'librosa\.effects\.trim.*trim_silence_top_db'):
            call(_audio(trim_silence=True))
    # trim_long_silences stays refused, with or without the other trim
    for kw in ({'trim_long_silences': True}, {'trim_long_silences': True, 'trim_silence': True, 'trim_silence_top_db': 60}):
        with pytest.raises(NotImplementedError, match='webrtcvad'):
            _audio(**kw).preprocess(y)
    # without trim_silence, preprocess is volume normalisation and the hop pad, as before
    a = _audio(norm_wav=True, target_dBFS=-30, int16_max=32767, trim_silence=False, trim_silence_top_db=60)
    x = np.random.default_rng(0).standard_normal(512).astype(np.float32) * np.float32(0.01)
    assert np.array_equal(a.preprocess(x), a.pad_to_hop(a.normalize_volume(x, increase_only=True)))
    assert len(a.preprocess(x)) == 513 and len(a.pad_to_hop(x[:300])) == 300


# clips of the seeded corpus (after the reference's volume normalisation) whose float32 bounds differ from the float64 ones
F32_CORPUS_CLIPS = 120
F32_DIFFERENCES = {20: 0, 60: 0, 80: 0}


def test_float32_and_float64_decisions_on_a_seeded_corpus():
    a = _audio(norm_wav=True, target_dBFS=-30, int16_max=32767)
    clips = [a.normalize_volume(c, increase_only=True) for c in to.padded_speech(F32_CORPUS_CLIPS, seed=4)]
    assert all(c.dtype == np.float32 for c in clips)
    counts, trimmed = {}, 0
    for top_db in F32_DIFFERENCES:
        b64 = [to.bounds64(c, top_db) for c in clips]
        counts[top_db] = sum(to.bounds32(c, top_db) != b for c, b in zip(clips, b64))
        trimmed += sum(b != (0, len(c)) for c, b in zip(clips, b64))
    assert counts == F32_DIFFERENCES
    assert trimmed > 2 * F32_CORPUS_CLIPS             # the corpus does exercise the trim
