"""ttsb_mcd_dtw_path on the GPU: cost and path length bit-identical to ttsb_mcd_dtw and to the float64 restatement, every path
equal to the restatement's (tests/dtw_path_oracle.py), a pair's path independent of its batch and of the workspace split, the
frame limit, and evaluate_tts.py --f0 end to end against f0_scores on the restated paths."""
import json
import pickle
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import yaml

import dtw_path_oracle as po
import evaluation_oracle as eo

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent

# 1 x 1, a single frame against the longest line and back, max_mel_len squared, and lengths around multiples of 32 (a warp's
# bit-plane word) and 128, with the shorter side on x and on y (the CTA is 256 threads: diagonals of 257+ cells take two passes)
SHAPES = [(1, 1), (1, 1200), (1200, 1), (1200, 1200), (31, 33), (32, 32), (33, 31), (63, 65), (64, 31), (31, 64), (127, 129),
          (128, 128), (129, 127), (255, 257), (256, 200), (200, 256), (257, 513), (513, 257), (97, 384), (384, 97), (700, 1100),
          (1100, 700)]


def _mel(T, rng, palette=None):
    if palette is None:
        return np.clip(rng.normal(-5, 2, (T, 80)), -11.5, 2).astype(np.float32)
    return palette[rng.integers(0, len(palette), T)]


def _pairs(seed):
    rng = np.random.default_rng(seed)
    a, b = [], []
    for tx, ty in SHAPES:
        a.append(_mel(tx, rng))
        b.append(_mel(ty, rng))
    # exactly tied frame distances: sequences drawn from a palette of 3 frames, constant sequences (every distance 0) and a
    # repeated-frame copy
    pal = _mel(3, rng)
    for tx, ty in ((40, 57), (129, 31), (31, 129), (300, 300), (33, 290)):
        a.append(_mel(tx, rng, pal))
        b.append(_mel(ty, rng, pal))
    for tx, ty in ((64, 64), (5, 90), (90, 5), (1, 33), (257, 1)):
        a.append(np.repeat(pal[:1], tx, axis=0))
        b.append(np.repeat(pal[:1], ty, axis=0))
    a.append(_mel(70, rng))
    b.append(np.repeat(a[-1], 2, axis=0)[:129])
    return a, b


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def _restated(x, y, n_ceps=24):
    dct = eo.dct_matrix(x.shape[1], n_ceps)
    return po.dtw_path(eo.frame_distances(eo.cepstra(x, dct), eo.cepstra(y, dct)))


def _cuda(ms):
    return [torch.from_numpy(m).cuda() for m in ms]


def test_paths_equal_the_restatement_and_scores_equal_mcd_dtw():
    from transformertts_b200.utils import evaluation as ev
    a, b = _pairs(seed=31)
    cost0, len0, mcd0 = ev.mcd_dtw(_cuda(a), _cuda(b))
    cost, path_len, mcd, paths = ev.mcd_dtw_paths(_cuda(a), _cuda(b))
    assert np.array_equal(_bits(cost), _bits(cost0)) and np.array_equal(path_len, len0) and np.array_equal(_bits(mcd), _bits(mcd0))
    for i, (x, y) in enumerate(zip(a, b)):
        want_cost, want_len, want_path = _restated(x, y)
        assert _bits(cost[i]) == _bits(want_cost) and path_len[i] == want_len, (i, x.shape, y.shape)
        assert paths[i].dtype == np.int32 and paths[i].shape == (want_len, 2), (i, paths[i].shape, want_len)
        assert np.array_equal(paths[i], want_path), (i, x.shape, y.shape)
    # the known answers: constant sequences follow the diagonal, then the longer side
    assert cost[-6] == 0.0 and path_len[-6] == 64 and np.array_equal(paths[-6], np.stack([np.arange(64)] * 2, axis=1))
    assert [tuple(p) for p in paths[-5][:86]] == [(0, j) for j in range(86)]


def test_a_pair_does_not_depend_on_its_batch_or_the_split():
    from transformertts_b200.utils import evaluation as ev
    rng = np.random.default_rng(22)
    lens = rng.integers(200, 1201, (120, 2))
    a = _cuda([_mel(int(t), rng) for t in lens[:, 0]])
    b = _cuda([_mel(int(t), rng) for t in lens[:, 1]])
    full = ev.mcd_dtw_paths(a, b)
    rev = ev.mcd_dtw_paths(a[::-1], b[::-1])
    split = ev.mcd_dtw_paths(a, b, workspace_budget=3 << 20)   # a few pairs per call
    for other, order in ((rev, slice(None, None, -1)), (split, slice(None))):
        assert np.array_equal(_bits(full[0]), _bits(other[0][order])) and np.array_equal(full[1], other[1][order])
        assert all(np.array_equal(p, q) for p, q in zip(full[3], other[3][order]))
    for i in (0, 61, 119):
        alone = ev.mcd_dtw_paths([a[i]], [b[i]])
        assert _bits(alone[0][0]) == _bits(full[0][i]) and alone[1][0] == full[1][i] and np.array_equal(alone[3][0], full[3][i]), i
    want = _restated(a[61].cpu().numpy(), b[61].cpu().numpy())
    assert _bits(full[0][61]) == _bits(want[0]) and np.array_equal(full[3][61], want[2])


def test_the_frame_limit_and_the_cell_limit():
    from transformertts_b200 import lib
    from transformertts_b200.utils import evaluation as ev
    rng = np.random.default_rng(23)
    a, b = [_mel(4096, rng), _mel(64, rng)], [_mel(64, rng), _mel(4096, rng)]
    cost, path_len, _, paths = ev.mcd_dtw_paths(_cuda(a), _cuda(b))
    cost0, len0, _ = ev.mcd_dtw(_cuda(a), _cuda(b))
    assert np.array_equal(_bits(cost), _bits(cost0)) and np.array_equal(path_len, len0)
    for i in range(2):
        want_cost, want_len, want_path = _restated(a[i], b[i])
        assert _bits(cost[i]) == _bits(want_cost) and np.array_equal(paths[i], want_path), i
    x = torch.zeros((4096, 80), device='cuda')
    with pytest.raises(lib.TtsbError, match='at most 16777216 cells'):
        ev.mcd_dtw_paths([x], [torch.zeros((4097, 80), device='cuda')])


# ---- evaluate_tts.py --f0 end to end
def _model_cfg():
    from oracle import forward_oracle as fo
    return dict(fo.CONFIGS['C1'], sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                normalizer='MelGAN', data_name='ljspeech')


def _phonemes(rng):
    from transformertts_b200.data.text import ALL_PHONEMES
    letters = [c for c in ALL_PHONEMES if c.isalpha()][:30] + [' ']
    return ''.join(rng.choice(letters, int(rng.integers(6, 24))))


def _setup(tmp_path):
    """A seeded model and MelGAN checkpoint, and a data directory of 6 validation lines with frame pitch (normalised, with
    pitch_stats.pkl, as create_training_data.py writes it)."""
    from oracle import forward_oracle as fo
    from oracle import melgan_oracle as mo
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    raw['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'))
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(raw))
    cm = TrainingConfigManager(str(tmp_path / 'cfg.yaml'))
    for d in (cm.data_dir, cm.mel_dir, cm.duration_dir, cm.pitch_per_char, cm.pitch_dir):
        d.mkdir(parents=True, exist_ok=True)
    rng = np.random.default_rng(41)
    lines = {f'f{i:03d}': _phonemes(rng) for i in range(6)}
    for name, ph in lines.items():
        T = int(rng.integers(max(len(ph), 20), 120))
        np.save(cm.mel_dir / f'{name}.npy', _mel(T, rng))
        np.save(cm.duration_dir / f'{name}.npy', np.bincount(rng.integers(0, len(ph), T), minlength=len(ph)).astype(np.int32))
        np.save(cm.pitch_per_char / f'{name}.npy', rng.normal(0, 1, len(ph)).astype(np.float32))
        p = rng.normal(0, 1, T)
        p[rng.random(T) < 0.3] = 0.0
        np.save(cm.pitch_dir / f'{name}.npy', p)
    cm.valid_metadata_path.write_text(''.join(f'{n}|{p}\n' for n, p in lines.items()), encoding='utf-8')
    with open(cm.data_dir / 'pitch_stats.pkl', 'wb') as f:
        pickle.dump({'pitch_mean': np.float64(180.0), 'pitch_std': np.float64(35.0)}, f)
    p = fo.init_params(_model_cfg(), seed=7)
    p['dur_pred.out.b'] = torch.tensor([3.0])
    model = ForwardTransformer(**_model_cfg())
    model.set_weights(p)
    model.save_model(tmp_path / 'model', with_optimizer=False)
    torch.save({'model_g': mo.init_state_dict(seed=11), 'githash': 'seeded'}, tmp_path / 'melgan.pt')
    return cm, lines


def _run(args):
    r = subprocess.run([sys.executable, str(ROOT / 'evaluate_tts.py')] + args, capture_output=True, text=True, timeout=900,
                       cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def test_evaluate_tts_f0_equals_f0_scores_on_the_restated_paths(tmp_path):
    from predict_tts import load_vocoder
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils import evaluation as ev
    cm, lines = _setup(tmp_path)
    common = ['--config', str(tmp_path / 'cfg.yaml'), '-p', str(tmp_path / 'model'), '--vocoder', 'melgan',
              '--vocoder_checkpoint', str(tmp_path / 'melgan.pt')]
    out = _run(common + ['-o', str(tmp_path / 'f0'), '--f0'])
    assert 'vocoded GPE' in out and 'copy synthesis GPE' in out and 'cents' in out
    _run(common + ['-o', str(tmp_path / 'plain')])
    res = json.loads((tmp_path / 'f0' / 'evaluation.json').read_text())['checkpoints'][0]
    plain = json.loads((tmp_path / 'plain' / 'evaluation.json').read_text())['checkpoints'][0]
    f0_keys = {p + k for p in ('vocoded_', 'copy_synthesis_') for k in ev.F0_KEYS}
    # without --f0 there are no F0 keys, and --f0 changes none of the other numbers
    assert not f0_keys & set(plain['mean']) and all(not f0_keys & set(ln) for ln in plain['lines'])
    for ln, pl in zip(res['lines'], plain['lines']):
        assert {k: v for k, v in ln.items() if k not in f0_keys} == pl, ln['name']
    assert {k: v for k, v in res['mean'].items() if k not in f0_keys} == plain['mean']

    # the same waveforms in this process: predict, vocode as evaluate_tts.py does, re-extract mels and F0 on the GPU
    model = ForwardTransformer.load_model(tmp_path / 'model')
    audio = Audio.from_config(model.config)
    vocoder = load_vocoder('melgan', str(tmp_path / 'melgan.pt'), None, model)
    names = list(lines)
    outs = model.predict_batch(ev.tokenize(model, [lines[n] for n in names]), encode=False, phoneme_max_duration=None)
    rec = [np.load(cm.mel_dir / f'{n}.npy') for n in names]
    vs = ev.load_validation_set(cm, frame_pitch=True)
    for prefix, mels in (('vocoded_', [o['mel'].cpu().numpy() for o in outs]), ('copy_synthesis_', rec)):
        wavs = vocoder.vocode_batch([m.T for m in mels])
        re_mels = audio.mel_spectrogram_ragged(wavs)
        f0s = audio.extract_pitch_batch(wavs)
        for i, (ln, n) in enumerate(zip(res['lines'], names)):
            cost, length, path = _restated(re_mels[i], rec[i])
            assert ln[f'{prefix}mcd'] == cost / length and ln[f'{prefix}path_len'] == length, (prefix, n)
            want = ev.f0_scores(f0s[i], vs.frame_pitch[i], path)
            assert {k: ln[prefix + k] for k in ev.F0_KEYS} == want, (prefix, n)
            assert 0 < want['f0_steps'] <= length and want['vde'] is not None, (prefix, n)
    for key in f0_keys:
        vals = [ln[key] for ln in res['lines'] if ln[key] is not None]
        assert res['mean'][key] == (pytest.approx(np.mean(vals), rel=1e-12) if vals else None), key
