"""Waveform synthesis without a GPU: argument checks of the batched Griffin-Lim C ABI (every check runs before any CUDA call),
Audio.save_wav (reference: data/audio.py:143-144) and the helpers of predict_tts.py (reference: predict_tts.py)."""
import ctypes as C
import math
import wave

import numpy as np
import pytest
import scipy.io.wavfile

import predict_tts

FAKE = C.c_void_p(0x100000)   # aligned, never dereferenced: validation fails before any launch


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def _audio():
    from transformertts_b200.data.audio import Audio
    return Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000, normalizer='MelGAN')


def _batch(cdll, mag=FAKE, init=FAKE, off=FAKE, n_clips=2, F=12, n_iter=4, momentum=0.99, ws=FAKE, ws_bytes=None, wav=FAKE):
    if ws_bytes is None:
        ws_bytes = max(cdll.ttsb_griffinlim_batch_workspace_bytes(F, n_clips), 0)
    return cdll.ttsb_griffinlim_batch(mag, init, off, n_clips, F, n_iter, C.c_float(momentum), ws, C.c_int64(ws_bytes), wav, None)


def test_griffinlim_batch_argument_validation(cdll):
    for kw in ({'mag': None}, {'init': None}, {'off': None}, {'ws': None}, {'wav': None}):
        assert _batch(cdll, **kw) == -1, kw
        assert b'ttsb_griffinlim_batch: NULL' in cdll.ttsb_last_error()
    for kw in ({'n_clips': 0, 'ws_bytes': 1 << 30}, {'n_clips': -1, 'ws_bytes': 1 << 30}, {'n_clips': 3, 'F': 11, 'ws_bytes': 1 << 30},
               {'F': 0, 'ws_bytes': 1 << 30}):
        assert _batch(cdll, **kw) == -1, kw
        assert b'ttsb_griffinlim_batch: need n_clips >= 1' in cdll.ttsb_last_error()
    assert _batch(cdll, n_iter=-1) == -1
    assert b'ttsb_griffinlim_batch: n_iter' in cdll.ttsb_last_error()
    for m in (-0.5, math.nan, math.inf):
        assert _batch(cdll, momentum=m) == -1, m
        assert b'ttsb_griffinlim_batch: momentum' in cdll.ttsb_last_error()
    need = cdll.ttsb_griffinlim_batch_workspace_bytes(12, 2)
    assert _batch(cdll, ws_bytes=need - 1) == -1
    assert b'ttsb_griffinlim_batch: workspace too small' in cdll.ttsb_last_error()
    assert _batch(cdll, ws=C.c_void_p(0x100004)) == -1
    assert b'ttsb_griffinlim_batch: workspace must be 16-byte aligned' in cdll.ttsb_last_error()


def test_griffinlim_batch_workspace_bytes(cdll):
    from transformertts_b200 import lib
    for F, n in ((0, 0), (12, 0), (7, 2), (-4, 1), (1 << 22, 1)):
        assert cdll.ttsb_griffinlim_batch_workspace_bytes(F, n) == -1, (F, n)
        assert b'ttsb_griffinlim_batch_workspace_bytes' in cdll.ttsb_last_error()
    with pytest.raises(lib.TtsbError, match='ttsb_griffinlim_batch_workspace_bytes'):
        lib.griffinlim_batch_workspace_bytes(7, 2)
    small, big = lib.griffinlim_batch_workspace_bytes(8, 2), lib.griffinlim_batch_workspace_bytes(862, 2)
    # frames (F, 1024) fp32 + two complex spectra (F, 513) + the clip table
    assert small >= 8 * (1024 * 4 + 2 * 513 * 8) and big >= 862 * (1024 * 4 + 2 * 513 * 8) and big > small
    assert lib.griffinlim_batch_workspace_bytes(862, 64) > lib.griffinlim_batch_workspace_bytes(862, 2)


def test_save_wav_writes_pcm16(tmp_path):
    a = _audio()
    y = np.array([0.0, 0.5, -0.5, 1.0, -1.0, 1.5, -1.5, 3e-5, -2e-5, 0.25 / 32767, 0.999999, -1.00002], dtype=np.float32)
    want = np.array([0, 16384, -16384, 32767, -32767, 32767, -32768, 1, -1, 0, 32767, -32768], dtype=np.int16)
    assert np.array_equal(np.clip(np.rint(y * np.float32(32767)), -32768, 32767).astype(np.int16), want)
    path = tmp_path / 'x.wav'
    a.save_wav(y, path)
    sr, got = scipy.io.wavfile.read(path)
    assert sr == 22050 and got.dtype == np.int16 and np.array_equal(got, want)
    with wave.open(str(path), 'rb') as f:
        assert (f.getnchannels(), f.getsampwidth(), f.getframerate(), f.getnframes()) == (1, 2, 22050, len(y))
        assert np.array_equal(np.frombuffer(f.readframes(len(y)), dtype='<i2'), want)
    # a longer signal, written from float64 like the reference's numpy arrays
    z = np.sin(np.linspace(0, 200, 10000)) * 1.2
    a.save_wav(z, tmp_path / 'z.wav')
    _, got = scipy.io.wavfile.read(tmp_path / 'z.wav')
    assert np.array_equal(got, np.clip(np.rint(z.astype(np.float32) * np.float32(32767)), -32768, 32767).astype(np.int16))


def test_predict_tts_output_names(tmp_path):
    cfg = {'data_name': 'ljspeech', 'git_hash': 'bdf06b9', 'step': 95000}
    outdir, stem, combined = predict_tts.output_names(tmp_path, 'lines', cfg, 7)
    assert outdir == tmp_path / 'outputs' / 'lines'
    assert stem == 'lines_ljspeech_bdf06b9_95000'
    assert combined == outdir / 'lines_ljspeech_bdf06b9_95000.wav'
    wav_i, mel_i = predict_tts.line_paths(outdir, stem, 3)
    assert wav_i == outdir / 'lines_ljspeech_bdf06b9_95000_3.wav'
    outdir.mkdir(parents=True)
    np.save(mel_i, np.zeros((2, 2), np.float32))       # what the reference writes with --store_mel
    assert (outdir / 'lines_ljspeech_bdf06b9_95000_3.mel.npy').exists()
    # keys a saved model lacks get the placeholder; the step falls back to the one given
    _, stem, _ = predict_tts.output_names(None, 'custom_text', {'data_name': 'ljspeech'}, 12)
    assert stem == f'custom_text_ljspeech_{predict_tts.MISSING}_12'
    outdir, stem, _ = predict_tts.output_names(None, 'f', {}, None)
    assert stem == f'f_{predict_tts.MISSING}_{predict_tts.MISSING}_{predict_tts.MISSING}' and str(outdir) == 'outputs/f'


def test_predict_tts_reads_lines(tmp_path):
    f = tmp_path / 'my_lines.txt'
    f.write_text('həloʊ wɜːld\n\nðɪs ɪz ɐ tɛst.\r\n')
    fname, lines = predict_tts.read_input(predict_tts.parse_args(['-f', str(f)]))
    assert fname == 'my_lines' and lines == ['həloʊ wɜːld', 'ðɪs ɪz ɐ tɛst.']
    assert predict_tts.read_input(predict_tts.parse_args(['-t', 'ɐ'])) == ('custom_text', ['ɐ'])


def test_predict_tts_tokenises_phonemes():
    from transformertts_b200.data.text import ALL_PHONEMES

    class FakeModel:
        def __init__(self, alphabet, breathing):
            self.alphabet, self.config = alphabet, {'model_breathing': breathing}

    tok = predict_tts.make_tokenizer(FakeModel(None, False))
    ids = tok('həˈloʊ')
    assert ids == [ALL_PHONEMES.index(c) + 1 for c in 'həˈloʊ']           # no start / end tokens
    tok_b = predict_tts.make_tokenizer(FakeModel(None, True))
    assert tok_b('ɐ b')[0] == tok_b.breathing_token_index and len(tok_b('ɐ b')) == 5
    tok_a = predict_tts.make_tokenizer(FakeModel('abc ', False))
    assert tok_a('ab c') == [2, 3, 1, 4]
    with pytest.raises(KeyError):
        tok_a('abd')                                                        # a symbol outside the alphabet raises


def test_predict_tts_without_input_prints_the_usage(capsys):
    assert predict_tts.main([]) == 0
    assert predict_tts.NO_INPUT_MESSAGE in capsys.readouterr().out
