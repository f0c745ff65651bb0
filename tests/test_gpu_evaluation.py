"""MCD-DTW on the GPU (ttsb_mcd_dtw) against the float64 restatement bit for bit, its independence of the batch, and
evaluate_tts.py / train_tts.py --evaluate end to end on a small on-disk data directory in the reference's layout."""
import json
import pickle
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import yaml

import evaluation_oracle as eo

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent

# 1 x 1, the longest line against a single frame, max_mel_len squared, and lengths around multiples of 32 and 128 (the CTA
# is 256 threads, so diagonals of 257+ cells take two passes)
SHAPES = [(1, 1), (1, 1200), (1200, 1), (1200, 1200), (31, 33), (32, 32), (33, 31), (63, 65), (127, 129), (128, 128),
          (129, 127), (255, 257), (256, 200), (257, 513), (97, 384), (700, 1100)]


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
    # exactly tied frame distances: sequences drawn from a palette of 3 frames, and constant sequences (every distance 0)
    pal = _mel(3, rng)
    for tx, ty in ((40, 57), (129, 31), (300, 300)):
        a.append(_mel(tx, rng, pal))
        b.append(_mel(ty, rng, pal))
    for tx, ty in ((64, 64), (5, 90), (90, 5)):
        a.append(np.repeat(pal[:1], tx, axis=0))
        b.append(np.repeat(pal[:1], ty, axis=0))
    b[-6] = np.repeat(a[-6], 2, axis=0)[:57]   # a repeated-frame copy
    return a, b


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize('n_ceps', [24, 79])
def test_mcd_dtw_equals_the_oracle_bit_for_bit(n_ceps):
    from transformertts_b200.utils import evaluation as ev
    a, b = _pairs(seed=5 + n_ceps)
    if n_ceps != 24:
        keep = [i for i, (x, y) in enumerate(zip(a, b)) if x.shape[0] * y.shape[0] < 200_000]
        a, b = [a[i] for i in keep], [b[i] for i in keep]
    cost, path_len, mcd = ev.mcd_dtw([torch.from_numpy(x).cuda() for x in a], [torch.from_numpy(y).cuda() for y in b], n_ceps)
    for i, (x, y) in enumerate(zip(a, b)):
        want_cost, want_len, want_mcd = eo.mcd_dtw(x, y, n_ceps)
        assert _bits(cost[i]) == _bits(want_cost), (i, x.shape, y.shape, cost[i], want_cost)
        assert int(path_len[i]) == want_len, (i, x.shape, y.shape, path_len[i], want_len)
        assert mcd[i] == want_mcd
    # the known answers hold on the device too
    assert cost[-3] == 0.0 and path_len[-3] == 64 and path_len[-2] == 90 and path_len[-1] == 90


def test_a_pair_does_not_depend_on_its_batch():
    from transformertts_b200.utils import evaluation as ev
    rng = np.random.default_rng(21)
    lens = rng.integers(200, 1201, (200, 2))
    a = [torch.from_numpy(_mel(int(t), rng)).cuda() for t in lens[:, 0]]
    b = [torch.from_numpy(_mel(int(t), rng)).cuda() for t in lens[:, 1]]
    full = ev.mcd_dtw(a, b)
    again = ev.mcd_dtw(a, b)
    rev = ev.mcd_dtw(a[::-1], b[::-1])
    assert np.array_equal(_bits(full[0]), _bits(again[0])) and np.array_equal(full[1], again[1])
    assert np.array_equal(_bits(full[0]), _bits(rev[0][::-1])) and np.array_equal(full[1], rev[1][::-1])
    for i in (0, 57, 199):
        alone = ev.mcd_dtw([a[i]], [b[i]])
        assert _bits(alone[0][0]) == _bits(full[0][i]) and alone[1][0] == full[1][i], i
    want = eo.mcd_dtw(a[57].cpu().numpy(), b[57].cpu().numpy())
    assert _bits(full[0][57]) == _bits(want[0]) and full[1][57] == want[1]


def test_refused_at_the_frame_limit_and_for_empty_lines():
    from transformertts_b200 import lib
    from transformertts_b200.utils import evaluation as ev
    x = torch.zeros((4097, 80), device='cuda')
    with pytest.raises(lib.TtsbError, match='at most 4096 frames'):
        ev.mcd_dtw([x], [x])
    with pytest.raises(ValueError, match='T >= 1'):
        ev.mcd_dtw([x[:0]], [x])


# ---- evaluate_tts.py / train_tts.py end to end
def _model_cfg():
    from oracle import forward_oracle as fo
    return dict(fo.CONFIGS['C1'], sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                normalizer='MelGAN', data_name='ljspeech')


def _save_model(path: Path, steps=(0,)):
    from oracle import forward_oracle as fo
    from transformertts_b200.model.models import ForwardTransformer
    p = fo.init_params(_model_cfg(), seed=7)
    p['dur_pred.out.b'] = torch.tensor([3.0])       # a few frames per phoneme from the seeded weights
    model = ForwardTransformer(**_model_cfg())
    model.set_weights(p)
    for s in steps:
        model.save_model(path / f'step_{s}', with_optimizer=False)
        cfg = yaml.safe_load((path / f'step_{s}' / 'config.yaml').read_text())
        (path / f'step_{s}' / 'config.yaml').write_text(yaml.safe_dump(dict(cfg, step=s)))
    return model


def _config(tmp_path, **tts):
    raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    raw['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'))
    raw['training_data_settings'].update(bucket_boundaries=[200], bucket_batch_sizes=[2, 2], val_bucket_batch_size=[2, 2])
    raw['tts_settings'].update(tts)
    path = tmp_path / 'cfg.yaml'
    path.write_text(yaml.safe_dump(raw))
    return path


def _phonemes(rng):
    from transformertts_b200.data.text import ALL_PHONEMES
    letters = [c for c in ALL_PHONEMES if c.isalpha()][:30] + [' ']
    return ''.join(rng.choice(letters, int(rng.integers(6, 24))))


def _write_data(cm, lines, targets):
    """lines: {name: phonemes}; targets: {name: (mel (T, 80), durations (Tp,), char pitch (Tp,))}; 4 validation lines."""
    for d in (cm.data_dir, cm.mel_dir, cm.duration_dir, cm.pitch_per_char):
        d.mkdir(parents=True, exist_ok=True)
    for name, (mel, dur, pitch) in targets.items():
        np.save(cm.mel_dir / f'{name}.npy', mel.astype(np.float32))
        np.save(cm.duration_dir / f'{name}.npy', dur.astype(np.int32))
        np.save(cm.pitch_per_char / f'{name}.npy', pitch.astype(np.float32))
    rows = [f'{n}|{p}\n' for n, p in lines.items()]
    cm.train_metadata_path.write_text(''.join(rows[:-4]), encoding='utf-8')
    cm.valid_metadata_path.write_text(''.join(rows[-4:]), encoding='utf-8')
    with open(cm.data_dir / 'pitch_stats.pkl', 'wb') as f:
        pickle.dump({'pitch_mean': np.float64(205.7), 'pitch_std': np.float64(41.3)}, f)
    return list(lines)[-4:]


def _random_targets(lines, seed):
    rng = np.random.default_rng(seed)
    out = {}
    for name, ph in lines.items():
        T = int(rng.integers(len(ph), 90))
        dur = np.bincount(rng.integers(0, len(ph), T), minlength=len(ph))
        pitch = rng.normal(0, 1.2, len(ph))
        pitch[rng.random(len(ph)) < 0.25] = 0.0
        out[name] = (_mel(T, rng), dur, pitch)
    return out


def _run(script, args, timeout=900):
    r = subprocess.run([sys.executable, str(ROOT / script)] + args, capture_output=True, text=True, timeout=timeout, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def test_evaluate_tts_matches_the_oracle_and_runs_melgan_copy_synthesis(tmp_path):
    from oracle import melgan_oracle as mo
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils import evaluation as ev
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    cfg = _config(tmp_path)
    cm = TrainingConfigManager(str(cfg))
    rng = np.random.default_rng(8)
    lines = {f'u{i:03d}': _phonemes(rng) for i in range(8)}
    targets = _random_targets(lines, seed=9)
    valid = _write_data(cm, lines, targets)
    _save_model(tmp_path / 'weights')
    torch.save({'model_g': mo.init_state_dict(seed=11), 'githash': 'seeded'}, tmp_path / 'melgan.pt')
    out = _run('evaluate_tts.py', ['--config', str(cfg), '-p', str(tmp_path / 'weights' / 'step_0'), '-o', str(tmp_path / 'out'),
                                   '--vocoder', 'melgan', '--vocoder_checkpoint', str(tmp_path / 'melgan.pt')])
    assert 'step_0 (step 0): MCD-DTW' in out and 'copy synthesis' in out
    res = json.loads((tmp_path / 'out' / 'evaluation.json').read_text())['checkpoints'][0]
    assert [ln['name'] for ln in res['lines']] == valid
    # the same numbers from the model's predict_batch outputs and the float64 restatement
    model = ForwardTransformer.load_model(tmp_path / 'weights' / 'step_0')
    tokens = ev.tokenize(model, [lines[n] for n in valid])
    free = model.predict_batch(tokens, encode=False, phoneme_max_duration=None)
    forced = model.predict_batch(tokens, encode=False, phoneme_max_duration=None, phoneme_durations=[targets[n][1] for n in valid],
                                 phoneme_pitch=[targets[n][2].astype(np.float32) for n in valid])
    for ln, o, tf, n in zip(res['lines'], free, forced, valid):
        mel, dur, pitch = targets[n]
        cost, length, mcd = eo.mcd_dtw(o['mel'].cpu().numpy(), mel)
        assert (ln['dtw_cost'], ln['path_len'], ln['mcd']) == (cost, length, mcd), n
        assert ln['teacher_forced_mcd'] == eo.mcd_dtw(tf['mel'].cpu().numpy(), mel)[2], n
        pred = o['int_durations'].cpu().numpy()
        assert ln['duration_mae'] == np.abs(pred - dur).mean() and ln['duration_exact'] == (pred == dur).mean(), n
        assert ln['frame_ratio'] == pred.sum() / dur.sum() and ln['frames_predicted'] == o['mel_lengths'], n
        v = pitch.astype(np.float32) != 0
        err = o['pitch'].cpu().numpy().reshape(-1)[v].astype(np.float64) - pitch.astype(np.float32)[v]
        assert ln['pitch_rmse'] == pytest.approx(np.sqrt(np.mean(err ** 2)), rel=1e-12), n
        assert ln['pitch_rmse_hz'] == pytest.approx(41.3 * ln['pitch_rmse'], rel=1e-9), n
        assert np.isfinite(ln['vocoded_mcd']) and np.isfinite(ln['copy_synthesis_mcd']) and ln['copy_synthesis_path_len'] > 0, n
    for key in ('mcd', 'teacher_forced_mcd', 'duration_mae', 'pitch_rmse', 'vocoded_mcd', 'copy_synthesis_mcd'):
        assert res['mean'][key] == pytest.approx(np.mean([ln[key] for ln in res['lines']]), rel=1e-12), key


def test_scores_are_zero_when_the_targets_are_the_models_own_outputs(tmp_path):
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils import evaluation as ev
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    cfg = _config(tmp_path)
    cm = TrainingConfigManager(str(cfg))
    rng = np.random.default_rng(12)
    lines = {f'v{i:03d}': _phonemes(rng) for i in range(7)}
    _save_model(tmp_path / 'weights', steps=(10, 5))
    model = ForwardTransformer.load_model(tmp_path / 'weights' / 'step_5')
    outs = model.predict_batch(ev.tokenize(model, list(lines.values())), encode=False, phoneme_max_duration=None)
    targets = {n: (o['mel'].cpu().numpy(), o['int_durations'].cpu().numpy(), o['pitch'].cpu().numpy().reshape(-1))
               for n, o in zip(lines, outs)}
    valid = _write_data(cm, lines, targets)
    out = _run('evaluate_tts.py', ['--config', str(cfg), '-p', str(tmp_path / 'weights'), '--weights_glob', 'step_*'])
    res = json.loads((tmp_path / 'weights' / 'evaluation.json').read_text())['checkpoints']
    assert [r['step'] for r in res] == [5, 10] and out.count('MCD-DTW 0.000 dB') == 2
    for r in res:
        for ln, n in zip(r['lines'], valid):
            T = targets[n][0].shape[0]
            assert ln['frames_predicted'] == ln['frames_recorded'] == T and ln['path_len'] == T, n
            assert ln['mcd'] == ln['dtw_cost'] == ln['teacher_forced_mcd'] == 0.0 and ln['teacher_forced_path_len'] == T, n
            assert ln['duration_mae'] == 0.0 and ln['duration_exact'] == 1.0 and ln['frame_ratio'] == 1.0, n
            assert ln['pitch_rmse'] == 0.0 and ln['pitch_rmse_hz'] == 0.0, n


def test_train_tts_evaluate_writes_the_scores_at_every_validation(tmp_path):
    from oracle import forward_oracle as fo
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    tts = {k: v for k, v in fo.CONFIGS['C1'].items() if k not in ('mel_channels', 'phoneme_language', 'with_stress', 'model_breathing')}
    cfg = _config(tmp_path, **tts, validation_frequency=2, weights_save_frequency=1000, weights_save_starting_step=1000)
    cm = TrainingConfigManager(str(cfg))
    rng = np.random.default_rng(14)
    lines = {f'w{i:03d}': _phonemes(rng) for i in range(10)}
    valid = _write_data(cm, lines, _random_targets(lines, seed=15))
    out = _run('train_tts.py', ['--config', str(cfg), '--max_steps', '4', '--evaluate'])
    assert 'evaluation at step 2: MCD-DTW' in out and 'evaluation at step 4: MCD-DTW' in out
    for step in (2, 4):
        res = json.loads((cm.log_dir / f'evaluation_step_{step}.json').read_text())
        assert res['step'] == step and [ln['name'] for ln in res['lines']] == valid
        assert 'teacher_forced_mcd' not in res['mean'] and 'duration_mae' in res['mean']
