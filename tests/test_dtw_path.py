"""CPU tests of the DTW warping path and the F0 scores along it: the float64 path restatement (tests/dtw_path_oracle.py)
against a plain cell-by-cell loop, evaluation_oracle.dtw and the tie rule; f0_scores on known answers; the frame-pitch loading
of the validation set; and the refusals of ttsb_mcd_dtw_path, which happen before any CUDA call."""
import ctypes as C
import math
import pickle
from types import SimpleNamespace

import numpy as np
import pytest

import dtw_path_oracle as po
import evaluation_oracle as eo


def _loop_path(dist):
    """The definition one cell at a time, with the choice of each cell, then the walk back."""
    Tx, Ty = dist.shape
    Cm = [[0.0] * Ty for _ in range(Tx)]
    Lm = [[0] * Ty for _ in range(Tx)]
    ch = np.zeros((Tx, Ty), dtype=np.int8)
    for i in range(Tx):
        for j in range(Ty):
            if i == 0 and j == 0:
                Cm[i][j], Lm[i][j] = float(dist[0, 0]), 1
                continue
            best, ln, c = math.inf, 0, po.DIAG
            if i > 0 and j > 0:
                best, ln = Cm[i - 1][j - 1], Lm[i - 1][j - 1]
            if i > 0 and Cm[i - 1][j] < best:
                best, ln, c = Cm[i - 1][j], Lm[i - 1][j], po.UP
            if j > 0 and Cm[i][j - 1] < best:
                best, ln, c = Cm[i][j - 1], Lm[i][j - 1], po.LEFT
            Cm[i][j], Lm[i][j], ch[i, j] = float(dist[i, j]) + best, ln + 1, c
    path, i, j = [(Tx - 1, Ty - 1)], Tx - 1, Ty - 1
    while (i, j) != (0, 0):
        di, dj = {po.DIAG: (1, 1), po.UP: (1, 0), po.LEFT: (0, 1)}[int(ch[i, j])]
        i, j = i - di, j - dj
        path.append((i, j))
    return Cm[-1][-1], Lm[-1][-1], path[::-1]


def _dist(shape, seed, palette=False):
    rng = np.random.default_rng(seed)
    a = rng.normal(-5, 2, (shape[0], 16)).astype(np.float32)
    b = rng.normal(-5, 2, (shape[1], 16)).astype(np.float32)
    if palette:   # frames drawn from 3: many exactly tied distances
        pal = a[:1].copy(), b[:1].copy(), rng.normal(-5, 2, (1, 16)).astype(np.float32)
        a = np.concatenate([pal[k] for k in rng.integers(0, 3, shape[0])])
        b = np.concatenate([pal[k] for k in rng.integers(0, 3, shape[1])])
    else:
        b[: min(shape) // 2] = a[: min(shape) // 2]    # some exactly equal frames, so some distances tie at 0
    dct = eo.dct_matrix(16, 6)
    return eo.frame_distances(eo.cepstra(a, dct), eo.cepstra(b, dct))


def _check_path(path, Tx, Ty):
    assert tuple(path[0]) == (0, 0) and tuple(path[-1]) == (Tx - 1, Ty - 1)
    steps = {tuple(s) for s in np.diff(path.astype(np.int64), axis=0)}
    assert steps <= {(1, 1), (1, 0), (0, 1)}


@pytest.mark.parametrize('shape', [(1, 1), (1, 7), (7, 1), (5, 9), (17, 6)])
@pytest.mark.parametrize('palette', [False, True])
def test_restatement_matches_plain_loop(shape, palette):
    dist = _dist(shape, sum(shape), palette)
    cost, length, path = po.dtw_path(dist)
    want_cost, want_len, want_path = _loop_path(dist)
    assert (cost, length) == (want_cost, want_len)
    assert [tuple(p) for p in path] == want_path
    _check_path(path, *shape)


@pytest.mark.parametrize('shape', [(1, 1), (1, 7), (7, 1), (5, 9), (17, 6), (40, 57), (64, 33), (100, 100)])
@pytest.mark.parametrize('palette', [False, True])
def test_path_reproduces_the_mcd_dtw_cost_and_length_bit_for_bit(shape, palette):
    dist = _dist(shape, 3 * sum(shape) + palette, palette)
    cost, length, path = po.dtw_path(dist)
    want_cost, want_len = eo.dtw(dist)
    assert len(path) == length == want_len
    assert np.float64(cost).view(np.uint64) == np.float64(want_cost).view(np.uint64)
    assert np.float64(po.path_sum(dist, path)).view(np.uint64) == np.float64(want_cost).view(np.uint64)
    _check_path(path, *shape)


def test_tie_rule_on_a_flat_cost_matrix():
    """All distances 0: every predecessor ties, so each cell takes the diagonal where it has one; walking back, the path runs
    diagonally until it meets row 0 or column 0, so from (0, 0) it first runs along the longer side."""
    for Tx, Ty in ((3, 5), (5, 3), (4, 4), (1, 6), (6, 1)):
        cost, length, path = po.dtw_path(np.zeros((Tx, Ty)))
        n = abs(Tx - Ty)
        first = [(0, k) for k in range(n + 1)] if Ty >= Tx else [(k, 0) for k in range(n + 1)]
        rest = [(first[-1][0] + k, first[-1][1] + k) for k in range(1, min(Tx, Ty))]
        assert (cost, length) == (0.0, max(Tx, Ty))
        assert [tuple(p) for p in path] == first + rest == _loop_path(np.zeros((Tx, Ty)))[2]


def test_tie_rule_takes_i_minus_1_before_j_minus_1():
    """(1, 1) is expensive: (2, 2)'s predecessors (1, 2) and (2, 1) tie at 0 below the diagonal, and (i - 1, j) wins."""
    dist = np.zeros((3, 3))
    dist[1, 1] = 100.0
    cost, length, path = po.dtw_path(dist)
    assert (cost, length) == (0.0, 4)
    assert [tuple(p) for p in path] == [(0, 0), (0, 1), (1, 2), (2, 2)] == _loop_path(dist)[2]


# ---- f0_scores
def _diag(n):
    return np.stack([np.arange(n), np.arange(n)], axis=1)


def test_f0_scores_known_answers():
    from transformertts_b200.utils.evaluation import f0_scores
    rng = np.random.default_rng(2)
    f = rng.uniform(80, 300, 50)
    f[::7] = 0.0
    assert f0_scores(f, f, _diag(50)) == {'gpe': 0.0, 'vde': 0.0, 'ffe': 0.0, 'f0_rmse_cents': 0.0, 'f0_steps': 50}
    octave = f0_scores(2 * f, f, _diag(50))
    assert octave['gpe'] == 1.0 and octave['f0_rmse_cents'] == pytest.approx(1200.0, rel=1e-12)
    assert octave['vde'] == 0.0 and octave['ffe'] == np.count_nonzero(f) / 50
    flip = f.copy()
    flip[1] = 0.0   # one voiced frame becomes unvoiced
    s = f0_scores(flip, f, _diag(50))
    assert s['vde'] == 1 / 50 and s['ffe'] == 1 / 50 and s['gpe'] == 0.0 and s['f0_rmse_cents'] == 0.0
    z = f0_scores(np.zeros(9), np.zeros(9), _diag(9))
    assert z == {'gpe': None, 'vde': 0.0, 'ffe': 0.0, 'f0_rmse_cents': None, 'f0_steps': 9}
    assert f0_scores(np.zeros(0), f, _diag(5)) == {'gpe': None, 'vde': None, 'ffe': None, 'f0_rmse_cents': None, 'f0_steps': 0}


def test_f0_scores_gross_error_threshold_and_cents():
    from transformertts_b200.utils.evaluation import f0_scores
    b = np.full(4, 100.0)
    a = np.array([119.0, 121.0, 79.0, 100.0])   # 19 %, 21 %, 21 % off and exact
    s = f0_scores(a, b, _diag(4))
    assert s['gpe'] == 0.5 and s['vde'] == 0.0 and s['ffe'] == 0.5
    cents = 1200 * np.log2(a / b)
    assert s['f0_rmse_cents'] == pytest.approx(math.sqrt(np.mean(cents ** 2)), rel=1e-12)


def test_f0_scores_skip_steps_past_a_contour_and_follow_the_path():
    from transformertts_b200.utils.evaluation import f0_scores
    path = np.array([(0, 0), (1, 0), (2, 1), (3, 2), (4, 3)], dtype=np.int32)
    a = np.array([100.0, 100.0, 0.0, 200.0])         # one frame short of the path: step (4, 3) is not scored
    b = np.array([100.0, 150.0, 200.0, 50.0])
    s = f0_scores(a, b, path)
    # scored steps: (0,0) 100/100, (1,0) 100/100, (2,1) unvoiced/150 -> flip, (3,2) 200/200
    assert s['f0_steps'] == 4 and s['vde'] == 0.25 and s['gpe'] == 0.0 and s['ffe'] == 0.25
    s = f0_scores(a, b[:2], path)                     # only the steps with j < 2
    assert s['f0_steps'] == 3 and s['vde'] == 1 / 3 and s['gpe'] == 0.0


# ---- the frame pitch of the validation set
def _cm(tmp_path):
    d = tmp_path / 'data'
    cm = SimpleNamespace(data_dir=d, valid_metadata_path=d / 'valid.txt', mel_dir=d / 'mels', duration_dir=d / 'durations',
                         pitch_per_char=d / 'char_pitch', pitch_dir=d / 'pitch.audio')
    for p in (cm.mel_dir, cm.duration_dir, cm.pitch_per_char, cm.pitch_dir):
        p.mkdir(parents=True)
    cm.valid_metadata_path.write_text('a|ab\nb|abc\n', encoding='utf-8')
    for n, T in (('a', 5), ('b', 7)):
        np.save(cm.mel_dir / f'{n}.npy', np.zeros((T, 80), np.float32))
        np.save(cm.duration_dir / f'{n}.npy', np.ones(len(n), np.int32))
        np.save(cm.pitch_per_char / f'{n}.npy', np.zeros(len(n), np.float32))
    return cm


def test_load_validation_set_denormalises_the_frame_pitch(tmp_path):
    from transformertts_b200.utils import evaluation as ev
    cm = _cm(tmp_path)
    with pytest.raises(FileNotFoundError, match='pitch_stats.pkl'):
        ev.load_validation_set(cm, frame_pitch=True)
    with open(cm.data_dir / 'pitch_stats.pkl', 'wb') as f:
        pickle.dump({'pitch_mean': np.float64(205.7), 'pitch_std': np.float64(41.3)}, f)
    p = {'a': np.array([0.0, 1.0, -0.5, 0.0, 2.0]), 'b': np.array([0.3, 0.0, 0.0, 1.0, -1.0, 0.0, 0.2])}
    np.save(cm.pitch_dir / 'a.npy', p['a'])
    with pytest.raises(FileNotFoundError, match=r'no frame pitch .*b\.npy'):
        ev.load_validation_set(cm, frame_pitch=True)
    np.save(cm.pitch_dir / 'b.npy', p['b'])
    assert ev.load_validation_set(cm).frame_pitch is None
    vs = ev.load_validation_set(cm, frame_pitch=True)
    for n, got in zip(vs.names, vs.frame_pitch):
        assert got.dtype == np.float64
        assert np.array_equal(got, np.where(p[n] != 0, p[n] * 41.3 + 205.7, 0.0)), n


def test_f0_needs_a_vocoder_and_frame_pitch():
    from transformertts_b200.utils import evaluation as ev
    vs = ev.ValidationSet(names=['a'], phonemes=['ab'], mels=[np.zeros((3, 80), np.float32)], durations=[np.ones(2)],
                          pitch=[np.zeros(2)])
    with pytest.raises(ValueError, match='need a vocoder and the recorded frame pitch'):
        ev.evaluate_model(None, vs, f0=True, vocode=lambda mels: mels)


def test_evaluate_tts_f0_needs_a_vocoder(capsys):
    import evaluate_tts
    with pytest.raises(SystemExit):
        evaluate_tts.parse_args(['--config', 'c.yaml', '-p', 'm', '--f0'])
    assert '--f0 scores vocoded audio: it needs --vocoder' in capsys.readouterr().err
    assert evaluate_tts.parse_args(['--config', 'c.yaml', '-p', 'm', '--vocoder', 'griffinlim', '--f0']).f0
    assert not evaluate_tts.parse_args(['--config', 'c.yaml', '-p', 'm']).f0


def test_summary_line_shows_the_f0_scores_only_when_present():
    from transformertts_b200.utils import evaluation as ev
    base = {'mcd': 5.0, 'duration_mae': 1.0, 'duration_exact': 0.5, 'frame_ratio': 1.0, 'pitch_rmse': 0.2,
            'vocoded_mcd': 6.0, 'copy_synthesis_mcd': 3.0}
    plain = ev.summary_line('x', {'mean': base})
    assert 'GPE' not in plain and 'cents' not in plain
    f0 = dict(base, vocoded_gpe=0.125, vocoded_vde=0.25, vocoded_ffe=0.3, vocoded_f0_rmse_cents=80.04, vocoded_f0_steps=100.0,
              copy_synthesis_gpe=0.01, copy_synthesis_vde=0.02, copy_synthesis_ffe=0.03, copy_synthesis_f0_rmse_cents=None,
              copy_synthesis_f0_steps=100.0)
    line = ev.summary_line('x', {'mean': f0})
    assert line.startswith(plain)
    assert ' | vocoded GPE 0.125, VDE 0.250, FFE 0.300, F0 RMSE 80.0 cents' in line
    assert ' | copy synthesis GPE 0.010, VDE 0.020, FFE 0.030, F0 RMSE n/a cents' in line


# ---- refusals through ctypes, without a GPU (fake device pointers: nothing is launched)
@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def _call(cdll, xo, yo, n_mels=80, K=24, ws_bytes=None, kappa=eo.KAPPA, null=None):
    xo_a, yo_a = (C.c_int32 * len(xo))(*xo), (C.c_int32 * len(yo))(*yo)
    args = dict(x=C.c_void_p(16), y=C.c_void_p(16), dct=C.c_void_p(16), ws=C.c_void_p(16), cost=C.c_void_p(16),
                length=C.c_void_p(16), path=C.c_void_p(16))
    if null is not None:
        args[null] = None
    if ws_bytes is None:
        ws_bytes = 1 << 40
    return cdll.ttsb_mcd_dtw_path(args['x'], xo_a, args['y'], yo_a, len(xo) - 1, n_mels, args['dct'], K, C.c_double(kappa), args['ws'],
                                  C.c_int64(ws_bytes), args['cost'], args['length'], args['path'], None)


def _err(cdll):
    return cdll.ttsb_last_error().decode()


def _words(tx, ty):
    """2 ceil(n_d / 32) words of choice bits per anti-diagonal d of n_d cells."""
    return sum(2 * -(-len(range(max(0, d - ty + 1), min(d, tx - 1) + 1)) // 32) for d in range(tx + ty - 1))


def test_refusals_before_any_cuda_call(cdll):
    for null in ('x', 'y', 'dct', 'ws', 'cost', 'length', 'path'):
        assert _call(cdll, [0, 5], [0, 6], null=null) == -1 and 'ttsb_mcd_dtw_path: NULL pointer' in _err(cdll), null
    assert _call(cdll, [1, 5], [0, 6]) == -1 and 'offsets must start at 0' in _err(cdll)
    assert _call(cdll, [0, 5, 5], [0, 6, 9]) == -1 and 'pair 1 has 0 x frames and 3 y frames' in _err(cdll)
    assert _call(cdll, [0, 5], [0, 6], K=80) == -1 and 'got n_ceps 80, n_mels 80' in _err(cdll)
    assert _call(cdll, [0, 5], [0, 6], kappa=-1.0) == -1 and 'kappa' in _err(cdll)
    assert _call(cdll, [0, 4097], [0, 5000]) == -1
    assert 'pair 0 is 4097 x 5000 frames; the shorter side may have at most 4096 frames' in _err(cdll)
    # the cell limit: 4096 x 4096 is exactly 2^24 cells; one more row, or a long pair with a short side, is refused
    assert _call(cdll, [0, 4096], [0, 4097]) == -1
    assert 'pair 0 is 4096 x 4097 frames, 16781312 cells; the path variant takes at most 16777216 cells' in _err(cdll)
    assert _call(cdll, [0, 5, 1205], [0, 6, 15000]) == -1 and 'pair 1 is 1200 x 14994 frames' in _err(cdll)
    need = (11 * 24) * 8 + 2 * 2 * 4 + 8 + 4 * _words(5, 6)
    assert _call(cdll, [0, 5], [0, 6], ws_bytes=need - 1) == -1
    assert f'workspace holds {need - 1} bytes, needs {need} (ttsb_mcd_dtw_path_workspace_bytes)' in _err(cdll)
    # ttsb_mcd_dtw's own workspace is not enough: the choice bits come on top of it
    old = cdll.ttsb_mcd_dtw_workspace_bytes((C.c_int32 * 2)(0, 5), (C.c_int32 * 2)(0, 6), 1, 24)
    assert _call(cdll, [0, 5], [0, 6], ws_bytes=old) == -1 and 'workspace holds' in _err(cdll)


def test_workspace_query(cdll):
    from transformertts_b200 import lib
    assert lib.MCD_DTW_PATH_MAX_CELLS == 4096 * 4096
    assert _words(5, 6) == 20 and _words(33, 1) == 33 * 2 and _words(1, 40) == 40 * 2
    assert lib.mcd_dtw_path_workspace_bytes([0, 5, 12], [0, 6, 7], 24) == (19 * 24) * 8 + 2 * 3 * 4 + 2 * 8 + 4 * (_words(5, 6) + _words(7, 1))
    for tx, ty in ((4096, 4096), (64, 4096), (1200, 13981), (300, 301)):
        want = (tx + ty) * 24 * 8 + 2 * 2 * 4 + 8 + 4 * _words(tx, ty)
        assert lib.mcd_dtw_path_workspace_bytes([0, tx], [0, ty], 24) == want, (tx, ty)
    with pytest.raises(lib.TtsbError, match='at most 16777216 cells'):
        lib.mcd_dtw_path_workspace_bytes([0, 1200], [0, 13982], 24)
    with pytest.raises(lib.TtsbError, match='1 pairs in x_offsets, 2 in y_offsets'):
        lib.mcd_dtw_path_workspace_bytes([0, 3], [0, 3, 4], 24)
