"""CPU tests of the WORLD mel-cepstral distortion: known answers for SPTK's freqt, pysptk's sp2mc and mcepalpha, and WORLD's
CheapTrick as tests/world_mcep_oracle.py restates them (answers that do not depend on the restatement being right), the sp2mc
matrix of utils/evaluation.py against the recursion, and the argument checks of the new entry points without a GPU."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

import world_mcep_oracle as wo

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import pitch_oracle as po   # noqa: E402
from transformertts_b200.utils import evaluation as ev   # noqa: E402

FP = 256 / 22050 * 1000


def _envelope(n, poles=((0.9, 500.0), (0.85, 1500.0), (0.8, 2500.0)), fs=22050.0):
    """|1 / A(e^jw)|^2 of an all-pole filter at the bins 0 .. n / 2, and A's coefficients."""
    a = np.array([1.0])
    for r, f in poles:
        a = np.convolve(a, [1.0, -2 * r * np.cos(2 * np.pi * f / fs), r * r])
    w = 2 * np.pi * np.arange(n // 2 + 1) / n
    A = np.polyval(a[::-1], np.exp(-1j * w))
    return 1.0 / np.abs(A) ** 2, a


def test_alpha_zero_is_the_real_cepstrum():
    sp, _ = _envelope(1024)
    c = np.fft.irfft(np.log(sp))
    c[0] /= 2
    assert np.allclose(wo.sp2mc(sp, 30, 0.0), c[:31], rtol=0, atol=1e-14)
    assert np.allclose(ev.sp2mc_matrix(1024, 30, 0.0) @ np.log(sp), c[:31], rtol=0, atol=1e-13)


def test_freqt_there_and_back():
    c = 0.7 ** np.arange(40) * np.cos(np.arange(40))
    for a in (0.41, 0.554):
        back = wo.freqt(wo.freqt(c, 400, a), 39, -a)
        assert np.abs(back - c).max() < 1e-12, a


def test_sp2mc_matrix_equals_the_recursion():
    rng = np.random.default_rng(1)
    for n, order, alpha in ((1024, 24, 0.455), (2048, 24, 0.554), (512, 10, 0.3)):
        W = ev.sp2mc_matrix(n, order, alpha)
        assert W.shape == (order + 1, n // 2 + 1)
        for _ in range(3):
            sp = np.exp(rng.normal(0, 2, n // 2 + 1))
            want = wo.sp2mc(sp, order, alpha)
            got = W @ np.log(sp)
            assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max(), (n, order)


def test_mel_cepstrum_is_the_cosine_series_over_the_warped_frequency():
    """For a smooth log envelope, log|H(w(b))|^2 = 2 mc_0 + 2 sum_k mc_k cos(k b) over the warped frequency b, so
    mc_k = (1 / pi) int_0^pi log|H(w(b))|^2 cos(k b) db (k >= 1, half that for k = 0), w(b) the inverse all-pass warping;
    integrated by the midpoint rule on a fine grid of b."""
    n, order, alpha = 2048, 40, 0.455
    sp, a = _envelope(n)
    mc = ev.sp2mc_matrix(n, order, alpha) @ np.log(sp)
    b = (np.arange(200000) + 0.5) * np.pi / 200000
    w = b - 2 * np.arctan(alpha * np.sin(b) / (1 + alpha * np.cos(b)))      # the warping at -alpha: w(b)
    logp = -np.log(np.abs(np.polyval(a[::-1], np.exp(-1j * w))) ** 2)
    k = np.arange(order + 1)[:, None]
    direct = (logp[None, :] * np.cos(k * b[None, :])).mean(axis=1)          # (1 / pi) int ... db
    direct[0] /= 2
    assert np.abs(mc - direct).max() < 1e-8, np.abs(mc - direct).max()


def test_mcepalpha_table():
    table = {16000: 0.41, 22050: 0.455, 24000: 0.466, 44100: 0.544, 48000: 0.554}
    for fs, want in table.items():
        assert ev.mcep_alpha(fs) == pytest.approx(want, abs=1e-12), fs
        assert wo.mcepalpha(fs) == pytest.approx(want, abs=1e-12), fs


def test_fft_sizes():
    from transformertts_b200.data.audio import Audio
    for fs, n in ((16000, 1024), (22050, 1024), (24000, 1024), (44100, 2048), (48000, 2048)):
        assert wo.fft_size(fs) == n
        a = Audio(sampling_rate=fs, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=None,
                  normalizer='MelGAN', device='cpu')
        assert a.cheaptrick_fft_size == n


# measured on the restatement: 10 log10(envelope / |H|^2), less its median, stays within 0.048 dB of 0 between 100 Hz and 5 kHz
# (frames 20 to 55); the gate is twice that
PULSE_GATE_DB = 0.1


def test_pulse_train_envelope_follows_the_filter():
    from scipy.signal import lfilter
    fs, period = 22050, 180                     # f0 = 122.5 Hz
    x = np.zeros(fs)
    x[::period] = 1.0
    env_h, a = _envelope(1024)
    y = lfilter([1.0], a, x).astype(np.float32)
    f0 = np.full(wo.n_frames(len(y), fs, FP), fs / period)
    frames = range(20, 60, 7)
    bins = np.arange(513) * fs / 1024
    band = (bins >= 100) & (bins <= 5000)
    for i in frames:
        env = wo.cheaptrick_frame(y, fs, i, FP, float(f0[i]), 1024)
        d = 10 * np.log10(env[band] / env_h[band])
        assert np.abs(d - np.median(d)).max() < PULSE_GATE_DB, (i, np.abs(d - np.median(d)).max())


def test_gain_leaves_mc1_to_mcK_and_silence_stays_finite():
    x = po.speech_like_clip(1.5, seed=5)
    f0 = po.extract_pitch(x, 22050, 256)
    mc = wo.world_mcep(x, 22050, f0, FP)
    mc_loud = wo.world_mcep((x * np.float32(4.0)), 22050, f0, FP)
    assert np.abs(mc_loud[:, 0] - mc[:, 0] - np.log(16.0) / 2).max() < 1e-6
    d = ev.KAPPA * np.sqrt(2 * np.sum((mc_loud[:, 1:] - mc[:, 1:]) ** 2, axis=1))
    assert d.max() < 1e-4, d.max()
    silent = wo.world_mcep(np.zeros(11025, np.float32), 22050, np.zeros(wo.n_frames(11025, 22050, FP)), FP)
    assert np.isfinite(silent).all()


def test_noise_is_an_irwin_hall_normal():
    v = wo.randn(3, np.arange(65536), 0)
    assert abs(v.mean()) < 0.02 and abs(v.std() - 1) < 0.02 and np.abs(v).max() < 6
    assert not np.array_equal(v, wo.randn(3, np.arange(65536), 1)) and not np.array_equal(v, wo.randn(4, np.arange(65536), 0))
    assert np.array_equal(v[:10], wo.randn(3, np.arange(10), 0))


# ---- argument checks without a GPU (fake non-null device pointers: nothing may be launched)
@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def _i32(*v):
    return (C.c_int32 * len(v))(*v)


def test_cheaptrick_refusals(cdll):
    p = C.c_void_p(256)
    so, fo = _i32(0, 22050), _i32(0, 87)
    ws = cdll.ttsb_cheaptrick_workspace_bytes(so, fo, 1, 22050, C.c_double(FP), 1024)
    assert ws > 0

    def call(**kw):
        a = dict(wav=p, so=so, n=1, fs=22050, fp=FP, f0=p, fo=fo, q1=-0.15, fft=1024, ws=p, wsb=ws, out=p)
        a.update(kw)
        return cdll.ttsb_cheaptrick(a['wav'], a['so'], a['n'], a['fs'], C.c_double(a['fp']), a['f0'], a['fo'], C.c_double(a['q1']),
                                    a['fft'], a['ws'], C.c_int64(a['wsb']), a['out'], None)
    for bad, what in (({'wav': None}, b'NULL'), ({'so': None}, b'NULL offset'), ({'n': 0}, b'n_clips'), ({'fs': 4000}, b'fs'),
                      ({'fp': 0.0}, b'frame_period'), ({'q1': float('nan')}, b'q1'), ({'fft': 1000}, b'fft_size'),
                      ({'fft': 8192}, b'fft_size'), ({'fft': 256, 'fs': 48000}, b'too short'),
                      ({'fo': _i32(0, 86)}, b'frame count'), ({'so': _i32(1, 22050)}, b'start at 0'),
                      ({'so': _i32(0, 0), 'fo': _i32(0, 1)}, b'0 samples'), ({'wsb': ws - 1}, b'workspace'),
                      ({'ws': C.c_void_p(264)}, b'aligned')):
        assert call(**bad) == -1, bad
        assert what in cdll.ttsb_last_error(), (bad, cdll.ttsb_last_error())
    assert cdll.ttsb_cheaptrick_workspace_bytes(so, _i32(0, 86), 1, 22050, C.c_double(FP), 1024) == -1


def test_sp2mc_refusals(cdll):
    p = C.c_void_p(256)
    for args, what in (((None, 1, 1024, p, 24, p), b'NULL'), ((p, 0, 1024, p, 24, p), b'n_frames'), ((p, 1, 1000, p, 24, p), b'fft_size'),
                       ((p, 1, 1024, p, 0, p), b'order'), ((p, 1, 1024, p, 512, p), b'order')):
        assert cdll.ttsb_sp2mc(*args, None) == -1, args
        assert what in cdll.ttsb_last_error(), args


def test_mcd_dtw_ceps_refusals(cdll):
    p = C.c_void_p(256)
    xo, yo = _i32(0, 10), _i32(0, 12)
    nb = cdll.ttsb_mcd_dtw_ceps_workspace_bytes(xo, yo, 1, 24)
    assert nb == cdll.ttsb_mcd_dtw_workspace_bytes(xo, yo, 1, 24)
    assert cdll.ttsb_mcd_dtw_ceps_path_workspace_bytes(xo, yo, 1, 24) == cdll.ttsb_mcd_dtw_path_workspace_bytes(xo, yo, 1, 24)
    for path in (False, True):
        fn = cdll.ttsb_mcd_dtw_ceps_path if path else cdll.ttsb_mcd_dtw_ceps
        name = b'ttsb_mcd_dtw_ceps_path' if path else b'ttsb_mcd_dtw_ceps'

        def call(x=p, xo=xo, ld=25, first=1, k=24, kappa=4.34, ws=p, wsb=1 << 20, path_out=p):
            tail = (p, p, path_out) if path else (p, p)
            return fn(x, xo, p, yo, 1, ld, first, k, C.c_double(kappa), ws, C.c_int64(wsb), *tail, None)
        bad_cases = [({'x': None}, b'NULL'), ({'first': -1}, b'first'), ({'first': 2}, b'first + n_ceps'), ({'k': 0}, b'n_ceps'),
                     ({'kappa': 0.0}, b'kappa'), ({'xo': _i32(0, 0)}, b'at least 1'), ({'wsb': 8}, b'workspace'),
                     ({'ws': C.c_void_p(260)}, b'aligned')]
        if path:
            bad_cases.append(({'path_out': None}, b'NULL'))
        for bad, what in bad_cases:
            assert call(**bad) == -1, (path, bad)
            err = cdll.ttsb_last_error()
            assert name in err and what in err, (path, bad, err)
