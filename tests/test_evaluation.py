"""CPU tests of MCD-DTW: the float64 restatement (tests/evaluation_oracle.py) against a plain cell-by-cell loop and known
answers, the host's DCT table and kappa, the duration and pitch scores, and the refusals of ttsb_mcd_dtw, which happen
before any CUDA call."""
import ctypes as C
import math

import numpy as np
import pytest

import evaluation_oracle as eo


def _loop_dtw(dist):
    """The definition, one cell at a time."""
    Tx, Ty = dist.shape
    Cm = [[0.0] * Ty for _ in range(Tx)]
    Lm = [[0] * Ty for _ in range(Tx)]
    for i in range(Tx):
        for j in range(Ty):
            if i == 0 and j == 0:
                Cm[i][j], Lm[i][j] = float(dist[0, 0]), 1
                continue
            best, ln = math.inf, 0
            if i > 0 and j > 0:
                best, ln = Cm[i - 1][j - 1], Lm[i - 1][j - 1]
            if i > 0 and Cm[i - 1][j] < best:
                best, ln = Cm[i - 1][j], Lm[i - 1][j]
            if j > 0 and Cm[i][j - 1] < best:
                best, ln = Cm[i][j - 1], Lm[i][j - 1]
            Cm[i][j], Lm[i][j] = float(dist[i, j]) + best, ln + 1
    return Cm[-1][-1], Lm[-1][-1]


def _loop_cepstra(mel, n_ceps):
    M = mel.shape[1]
    out = np.zeros((mel.shape[0], n_ceps))
    for t in range(mel.shape[0]):
        for k in range(1, n_ceps + 1):
            acc = 0.0
            for m in range(M):
                acc += math.sqrt(2.0 / M) * math.cos(math.pi * k * (2 * m + 1) / (2 * M)) * float(mel[t, m])
            out[t, k - 1] = acc
    return out


@pytest.mark.parametrize('shape', [(1, 1), (1, 7), (7, 1), (5, 9), (12, 12), (17, 6)])
def test_oracle_matches_plain_loop(shape):
    rng = np.random.default_rng(sum(shape))
    a = rng.normal(-5, 2, (shape[0], 16)).astype(np.float32)
    b = rng.normal(-5, 2, (shape[1], 16)).astype(np.float32)
    b[: min(shape) // 2] = a[: min(shape) // 2]            # some exactly equal frames, so some distances tie at 0
    dct = eo.dct_matrix(16, 6)
    ca, cb = eo.cepstra(a, dct), eo.cepstra(b, dct)
    np.testing.assert_allclose(ca, _loop_cepstra(a, 6), rtol=0, atol=1e-12)
    dist = eo.frame_distances(ca, cb)
    for i in range(shape[0]):
        for j in range(shape[1]):
            want = eo.KAPPA * math.sqrt(2 * sum((ca[i, k] - cb[j, k]) ** 2 for k in range(6)))
            assert dist[i, j] == pytest.approx(want, rel=1e-13, abs=1e-13)
    assert eo.dtw(dist) == _loop_dtw(dist)


def test_oracle_tie_rule_on_a_flat_cost_matrix():
    """All distances 0: every predecessor ties, so the path takes the diagonal and then the remaining steps along the long side."""
    for Tx, Ty in ((3, 5), (5, 3), (4, 4), (1, 6)):
        dist = np.zeros((Tx, Ty))
        assert eo.dtw(dist) == _loop_dtw(dist) == (0.0, max(Tx, Ty))


def test_known_answers():
    rng = np.random.default_rng(4)
    mel = rng.normal(-5, 2, (40, 80)).astype(np.float32)
    cost, length, mcd = eo.mcd_dtw(mel, mel)
    assert (cost, length, mcd) == (0.0, 40, 0.0)
    twice = np.repeat(mel, 2, axis=0)                      # every frame repeated twice
    assert eo.mcd_dtw(twice, mel)[:2] == (0.0, 80)
    assert eo.mcd_dtw(mel, twice)[:2] == (0.0, 80)
    # c1 shifted by delta on every frame: the diagonal path, each step costs kappa sqrt(2) |delta|
    c = eo.cepstra(mel, eo.dct_matrix(80, 24))
    for delta in (0.01, -0.25):
        c2 = c.copy()
        c2[:, 0] += delta
        cost, length = eo.dtw(eo.frame_distances(c, c2))
        assert length == 40
        assert abs(cost / length - eo.KAPPA * math.sqrt(2) * abs(delta)) < 1e-12


def test_host_dct_and_kappa_equal_the_oracle():
    from transformertts_b200.utils import evaluation as ev
    for M, K in ((80, 24), (16, 6), (2, 1)):
        D = ev.dct_matrix(M, K)
        assert np.array_equal(D, eo.dct_matrix(M, K))
        full = np.vstack([np.full((1, M), math.sqrt(1.0 / M)), ev.dct_matrix(M, M - 1)])   # with the c0 row: orthonormal
        np.testing.assert_allclose(full @ full.T, np.eye(M), atol=1e-12)
    assert ev.KAPPA == eo.KAPPA == 10.0 / math.log(10.0)


def test_duration_and_pitch_scores():
    from transformertts_b200.utils import evaluation as ev
    d = ev.duration_scores(np.array([3, 0, 5, 2]), np.array([3, 1, 4, 2]))
    assert d == {'duration_mae': 0.5, 'duration_exact': 0.5, 'frame_ratio': 10 / 10}
    p = ev.pitch_scores(np.array([0.5, 1.0, -1.0]), np.array([0.0, 2.0, -1.5]), (200.0, 40.0))
    assert p['pitch_rmse'] == pytest.approx(math.sqrt((1.0 + 0.25) / 2))
    assert p['pitch_rmse_hz'] == pytest.approx(40.0 * math.sqrt((1.0 + 0.25) / 2))
    assert ev.pitch_scores(np.ones(3), np.zeros(3), None) == {'pitch_rmse': None, 'pitch_rmse_hz': None}
    assert ev._means([{'name': 'a', 'x': 1.0, 'y': None}, {'name': 'b', 'x': 3.0, 'y': None}]) == {'x': 2.0, 'y': None}


def test_normalizer_is_checked():
    from transformertts_b200.utils import evaluation as ev
    ev.check_normalizer({'normalizer': 'MelGAN'})
    with pytest.raises(ValueError, match="normalizer is 'WaveRNN'"):
        ev.check_normalizer({'normalizer': 'WaveRNN'})


# ---- refusals through ctypes, without a GPU (fake device pointers: nothing is launched)
@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def _call(cdll, xo, yo, n_mels=80, K=24, ws_bytes=None, kappa=eo.KAPPA, null=False):
    xo_a, yo_a = (C.c_int32 * len(xo))(*xo), (C.c_int32 * len(yo))(*yo)
    p = C.c_void_p(16)
    if ws_bytes is None:
        ws_bytes = 1 << 40
    return cdll.ttsb_mcd_dtw(None if null else p, xo_a, p, yo_a, len(xo) - 1, n_mels, p, K, C.c_double(kappa), p, C.c_int64(ws_bytes), p,
                             p, None)


def _err(cdll):
    return cdll.ttsb_last_error().decode()


def test_refusals_before_any_cuda_call(cdll):
    assert _call(cdll, [0, 5], [0, 6], null=True) == -1 and 'ttsb_mcd_dtw: NULL pointer' in _err(cdll)
    assert _call(cdll, [1, 5], [0, 6]) == -1 and 'offsets must start at 0' in _err(cdll)
    assert _call(cdll, [0, 5, 3], [0, 6, 9]) == -1 and 'pair 1 has -2 x frames' in _err(cdll)
    assert _call(cdll, [0, 5, 5], [0, 6, 9]) == -1 and 'pair 1 has 0 x frames and 3 y frames' in _err(cdll)
    assert _call(cdll, [0, 5], [0, 0]) == -1 and 'at least 1' in _err(cdll)
    assert _call(cdll, [0, 5], [0, 6], K=0) == -1 and 'need 1 <= n_ceps < n_mels' in _err(cdll)
    assert _call(cdll, [0, 5], [0, 6], K=80) == -1 and 'got n_ceps 80, n_mels 80' in _err(cdll)
    assert _call(cdll, [0, 5], [0, 6], kappa=float('nan')) == -1 and 'kappa' in _err(cdll)
    need = (11 * 24) * 8 + 2 * 2 * 4
    assert _call(cdll, [0, 5], [0, 6], ws_bytes=need - 1) == -1
    assert f'workspace holds {need - 1} bytes, needs {need}' in _err(cdll)
    assert _call(cdll, [0, 4097], [0, 5000]) == -1
    assert 'pair 0 is 4097 x 5000 frames; the shorter side may have at most 4096 frames' in _err(cdll)


def test_workspace_query(cdll):
    from transformertts_b200 import lib
    assert lib.MCD_DTW_MAX_FRAMES == 4096
    assert lib.mcd_dtw_workspace_bytes([0, 5, 12], [0, 6, 7], 24) == (19 * 24) * 8 + 2 * 3 * 4
    assert lib.mcd_dtw_workspace_bytes([0, 4096], [0, 9000], 24) == (13096 * 24) * 8 + 2 * 2 * 4
    with pytest.raises(lib.TtsbError, match='at most 4096 frames'):
        lib.mcd_dtw_workspace_bytes([0, 4097], [0, 4097], 24)
    with pytest.raises(lib.TtsbError, match='need n_ceps >= 1'):
        lib.mcd_dtw_workspace_bytes([0, 3], [0, 3], 0)
    with pytest.raises(lib.TtsbError, match='1 pairs in x_offsets, 2 in y_offsets'):
        lib.mcd_dtw_workspace_bytes([0, 3], [0, 3, 4], 24)
