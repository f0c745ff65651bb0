"""GPU tests of the label-generation pipeline: ttsb_pitch_per_char against the host reference bit for bit, Aligner checkpoint
resume and align(), the train_aligner.py driver (stop / restart, data parallel) and the on-disk chain
train_aligner.py -> extract_durations.py -> train_tts.py."""
import math
import pickle
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import yaml

from oracle import aligner_oracle as alo

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
GOLD = Path(__file__).resolve().parent / 'golden'
SMALL = {k: v for k, v in alo.ALIGNER_CONFIGS['A-small'].items() if k not in ('max_r', 'vocab_size')}


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def _run_batch(rows):
    """rows: [(pitch, durations, mel_len, mean, std)] sharing mean / std -> kernel output per row and the host reference."""
    from transformertts_b200.data.datasets import pitch_per_char
    from transformertts_b200.utils.alignments import pitch_per_char_batch
    B = len(rows)
    Tm = max(1, max(len(r[0]) for r in rows))
    Tp = max(len(r[1]) for r in rows)
    pitch = np.zeros((B, Tm))
    dur = np.zeros((B, Tp), dtype=np.int32)
    for i, (p, d, *_) in enumerate(rows):
        pitch[i, :len(p)], dur[i, :len(d)] = p, d
    plen = [len(r[0]) for r in rows]
    n_chars = [min(r[2], len(r[1])) for r in rows]
    mean, std = rows[0][3], rows[0][4]
    got = pitch_per_char_batch(pitch, plen, torch.from_numpy(dur).cuda(), n_chars, mean, std).cpu().numpy()
    for i, (p, d, mel_len, *_) in enumerate(rows):
        want = pitch_per_char(p, d, mel_len, mean, std)
        assert _bits_equal(got[i, :len(d)], want), (i, np.abs(got[i, :len(d)] - want).max())
        assert not got[i, len(d):].any()


def test_pitch_per_char_kernel_on_golden_cases_bitwise():
    with np.load(GOLD / 'char_pitch.npz') as z:
        n = len({k.split('/')[0] for k in z.files})
        cases = [(z[f'{i}/pitch'], z[f'{i}/durations'], int(z[f'{i}/mel_len']), float(z[f'{i}/stats'][0]), float(z[f'{i}/stats'][1]),
                  z[f'{i}/out']) for i in range(n)]
    from transformertts_b200.utils.alignments import pitch_per_char_batch
    for p, d, ml, mean, std, want in cases:
        _run_batch([(p, d, ml, mean, std)])
        got = pitch_per_char_batch(p[None], [len(p)], d[None], [min(ml, len(d))], mean, std).cpu().numpy()[0]
        assert _bits_equal(got, want)                  # the reference function's own output
    _run_batch([(p, d, ml, cases[0][3], cases[0][4]) for p, d, ml, *_ in cases])   # all cases as one padded batch


def test_pitch_per_char_kernel_random_padded_batches_bitwise():
    rng = np.random.default_rng(5)
    for trial in range(12):
        B = int(rng.integers(1, 17))
        mean, std = float(rng.uniform(100, 260)), float(rng.uniform(15, 90))
        rows = []
        for _ in range(B):
            tp = int(rng.integers(1, 201))
            d = rng.integers(0, 12, tp).astype(np.int32)
            if rng.random() < 0.3:
                d[int(rng.integers(0, tp))] = int(rng.integers(129, 700))   # a segment longer than 128 frames
            tm = int(np.clip(d.sum() + rng.integers(-20, 20), 0, 1200))
            p = rng.normal(0, 1.5, tm)
            p[rng.random(tm) < 0.3] = 0.0
            rows.append((p, d, int(rng.integers(tp // 2, tp + 5)), mean, std))
        _run_batch(rows)


def _cfg(**kw):
    return dict(SMALL, device='cuda:0', **kw)


def test_aligner_resume_in_process_and_hdf5_only_load(tmp_path):
    """N steps, save_model, load_model, M steps == N + M uninterrupted steps (dropout on: the seed base and the step are
    restored); a directory with only model_weights.hdf5 loads the same weights."""
    from transformertts_b200.model.aligner import Aligner
    from transformertts_b200.model.training import Adam
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    batches = [alo.make_aligner_inputs(cfg, 3, 20, 90, seed=600 + i) for i in range(6)]

    def fresh():
        m = Aligner.from_config(_cfg(), max_r=4)
        m.set_weights(p)
        m._compile(optimizer=Adam(1e-4, beta_1=0.9, beta_2=0.98, epsilon=1e-9))
        return m

    def steps(m, bs):
        out = []
        for tok, mel, stop in bs:
            m.set_constants(learning_rate=1e-4 * (1 + m.step), reduction_factor=2 if m.step < 3 else 1,
                            force_decoder_diagonal=m.step < 4, force_encoder_diagonal=m.step < 2)
            out.append(float(m.train_step(tok, mel, stop)['loss']))
        return out

    full = steps(fresh(), batches)
    m = fresh()
    first = steps(m, batches[:3])
    m.save_model(tmp_path / 'ck')
    m2 = Aligner.load_model(tmp_path / 'ck', device='cuda:0')
    w_pt = {k: v.detach().cpu().clone() for k, v in m2.weights.items()}
    assert m2.step == 3 and m2.max_r == 4 and m2.optimizer.m is not None
    assert m2._get_engine().base_seed == m._get_engine().base_seed
    rest = steps(m2, batches[3:])
    for a, b in zip(first + rest, full):
        assert abs(a - b) < 2e-3 * abs(b), (first + rest, full)
    (tmp_path / 'ck' / 'model_weights.pt').unlink()
    m3 = Aligner.load_model(tmp_path / 'ck', device='cuda:0')
    assert m3.step == 3 and set(m3.weights) == set(w_pt)
    for k, v in w_pt.items():
        assert torch.equal(m3.weights[k].cpu(), v), k


@pytest.mark.parametrize('r', [1, 2])
def test_align_equals_call_on_the_teacher_forced_input(r):
    from transformertts_b200.model.aligner import Aligner
    cfg = alo.ALIGNER_CONFIGS['A-small']
    m = Aligner.from_config(_cfg(), max_r=4)
    m.set_weights(alo.init_aligner_params(cfg, seed=7))
    m.set_constants(reduction_factor=r)
    tok, mel, _ = alo.make_aligner_inputs(cfg, 2, 16, 60, seed=9, ragged=False)
    raw = mel[:, 1:-1]                                            # without the start / end vectors
    att, out = m.align(tok, raw)
    tar = torch.cat([torch.full((2, 1, 80), 0.5), raw], dim=1)[:, 0::r].contiguous()
    ref = m.call(tok, tar, training=False)
    assert torch.equal(att, ref['decoder_attention']['Decoder_LastBlock_CrossAttention'])
    assert torch.equal(out['mel'], ref['mel']) and torch.equal(out['stop_prob'], ref['stop_prob'])
    att2, _ = m.align(tok, mel, mels_have_start_end_vectors=True)   # the end vector is dropped, the start vector kept
    assert torch.equal(att2, att)
    att1, _ = m.align(tok[0], raw[0])                               # one unbatched utterance
    assert att1.shape == (1,) + tuple(att.shape[1:]) and float((att1[0] - att[0]).abs().max()) < 1e-5
    with pytest.raises(NotImplementedError):
        m.align('text', raw, phonemize=True)


# ----------------------------------------------------------------------------------------------------------------------
# drivers
# ----------------------------------------------------------------------------------------------------------------------
def _run(script, args, nproc=1, timeout=900):
    cmd = [sys.executable]
    if nproc > 1:
        cmd += ['-m', 'torch.distributed.run', '--nnodes=1', f'--nproc-per-node={nproc}', '--master-addr', '127.0.0.1',
                '--master-port', '29533']
    r = subprocess.run(cmd + [str(ROOT / script)] + args, capture_output=True, text=True, timeout=timeout, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def _losses(stdout):
    return {int(m.group(1)): float(m.group(2)) for m in re.finditer(r'step (\d+)  loss ([0-9.]+)', stdout)}


def _config(tmp_path, **aligner):
    raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    raw['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'))
    raw['training_data_settings'].update(bucket_boundaries=[60, 100], bucket_batch_sizes=[4, 4, 2], val_bucket_batch_size=[2, 2, 2])
    raw['aligner_settings'].update(SMALL)
    raw['aligner_settings'].update(aligner)
    path = tmp_path / 'cfg.yaml'
    path.write_text(yaml.safe_dump(raw))
    return path


def test_train_aligner_stop_and_restart_reproduces_the_loss_curve(tmp_path):
    """r = 4 -> 2 -> 1 and a decoder-diagonal phase ending mid-run: a run stopped at step 5 and restarted continues the
    uninterrupted run's loss curve (weights, Adam state, step, schedules, dropout seeds and batch stream restored)."""
    cfg = _config(tmp_path, reduction_factor_schedule=[[0, 4], [3, 2], [6, 1]], force_encoder_diagonal_steps=2,
                  force_decoder_diagonal_steps=4, validation_frequency=1000, prediction_start_step=1000)
    base = ['--config', str(cfg), '--synthetic', '--batch_size', '2', '--synthetic_shape', '24', '121', '--checkpoint_frequency', '1']
    out_full = _run('train_aligner.py', base + ['--max_steps', '9', '--weights_dir', str(tmp_path / 'a' / 'weights')])
    full = _losses(out_full)
    assert sorted(full) == list(range(1, 10)) and all(math.isfinite(v) for v in full.values())
    assert ' r 4 ' in out_full and ' r 2 ' in out_full and ' r 1 ' in out_full
    out1 = _run('train_aligner.py', base + ['--max_steps', '5', '--weights_dir', str(tmp_path / 'b' / 'weights')])
    assert 'starting training from scratch' in out1
    out2 = _run('train_aligner.py', base + ['--max_steps', '9', '--weights_dir', str(tmp_path / 'b' / 'weights')])
    assert 'resuming training from step 5' in out2 and 'Done.' in out2
    resumed = _losses(out2)
    assert sorted(resumed) == [6, 7, 8, 9]
    for s in (6, 7, 8, 9):
        assert abs(resumed[s] - full[s]) < 2e-3 * abs(full[s]), (s, resumed, full)


def _write_dataset(cm, n=16, seed=3):
    """Mels, frame pitch (normalised, 0 = unvoiced), pitch_stats.pkl and train / valid / phonemized metadata."""
    from transformertts_b200.data.text import ALL_PHONEMES
    rng = np.random.default_rng(seed)
    for d in (cm.data_dir, cm.mel_dir, cm.pitch_dir):
        d.mkdir(parents=True, exist_ok=True)
    letters = [c for c in ALL_PHONEMES if c.isalpha()][:30] + [' ']
    lines = []
    for i in range(n):
        name = f'u{i:03d}'
        T = int(rng.integers(30, 56))
        np.save(cm.mel_dir / f'{name}.npy', np.clip(rng.normal(-5, 2, (T, 80)), -11.5, 2).astype(np.float32))
        p = rng.normal(0, 1.2, T + int(rng.integers(-2, 3)))
        p[rng.random(len(p)) < 0.25] = 0.0
        p[rng.random(len(p)) < 0.05] = 5.5                     # above 400 Hz once de-normalised
        np.save(cm.pitch_dir / f'{name}.npy', p)
        lines.append(f'{name}|' + ''.join(rng.choice(letters, int(rng.integers(6, 20)))) + '\n')
    cm.phonemized_metadata_path.write_text(''.join(lines), encoding='utf-8')
    cm.train_metadata_path.write_text(''.join(lines[:12]), encoding='utf-8')
    cm.valid_metadata_path.write_text(''.join(lines[12:]), encoding='utf-8')
    with open(cm.data_dir / 'pitch_stats.pkl', 'wb') as f:
        pickle.dump({'pitch_mean': np.float64(205.7), 'pitch_std': np.float64(41.3)}, f)
    return [ln.split('|')[0] for ln in lines], {ln.split('|')[0]: ln.split('|')[1].strip('\n') for ln in lines}


def _check_labels(cm, names, phonemes):
    from transformertts_b200.data.datasets import pitch_per_char
    with open(cm.data_dir / 'pitch_stats.pkl', 'rb') as f:
        st = pickle.load(f)
    out = {}
    for name in names:
        d = np.load(cm.duration_dir / f'{name}.npy')
        T = np.load(cm.mel_dir / f'{name}.npy').shape[0]
        assert d.dtype == np.int32 and len(d) == len(phonemes[name]) and int(d.sum()) == T, name
        cp = np.load(cm.pitch_per_char / f'{name}.npy')
        want = pitch_per_char(np.load(cm.pitch_dir / f'{name}.npy'), d, T, float(st['pitch_mean']), float(st['pitch_std']))
        assert _bits_equal(cp, want), name
        out[name] = (d, cp)
    return out


def test_labels_on_disk_from_train_aligner_to_train_tts(tmp_path):
    from transformertts_b200.data import datasets as ds
    from transformertts_b200.data.text import Tokenizer
    from transformertts_b200.utils.alignments import get_durations_from_alignment
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    cfg = _config(tmp_path, reduction_factor_schedule=[[0, 2], [2, 1]], force_encoder_diagonal_steps=1, force_decoder_diagonal_steps=3,
                  validation_frequency=4, prediction_start_step=4, prediction_frequency=4, weights_save_frequency=2)
    cm = TrainingConfigManager(str(cfg), aligner=True)
    names, phonemes = _write_dataset(cm)
    out = _run('train_aligner.py', ['--config', str(cfg), '--max_steps', '4'])
    assert 'validation loss at step 4' in out and 'validation attention peakiness per head' in out
    assert re.search(r'prediction at step 4: \d+ frames', out) and ' r 1 ' in out and 'Done.' in out
    assert (cm.weights_dir / 'step_2' / 'optimizer.pt').exists() and (cm.weights_dir / 'latest' / 'model_weights.hdf5').exists()
    # durations + char pitch
    out = _run('extract_durations.py', ['--config', str(cfg)])
    assert 'utterances/s' in out and 'ERROR' not in out
    labels = _check_labels(cm, names, phonemes)
    # the durations are those of a direct val_step on the same batches
    model = cm.load_model(verbose=False)
    prep = ds.AlignerPreprocessor.from_config(cm, Tokenizer(add_start_end=True, model_breathing=False))
    data = ds.AlignerDataset.from_config(cm, prep, kind='phonemized').get_dataset(
        bucket_batch_sizes=cm.config['bucket_batch_sizes'], bucket_boundaries=cm.config['bucket_boundaries'], shuffle=False,
        drop_remainder=False)
    seen = 0
    for b in data.all_batches():
        o = model.val_step(b['tokens'], b['mel'], b['stop_prob'])
        durs = get_durations_from_alignment(o['decoder_attention']['Decoder_LastBlock_CrossAttention'], b['mel'], b['tokens'],
                                            weighted=True)[0]
        for name, d in zip(b['name'], durs):
            assert np.array_equal(d, labels[name][0]), name
            seen += 1
    assert seen == len(names)
    # pitch only, from the durations on disk
    out = _run('extract_durations.py', ['--config', str(cfg), '--skip_durations'])
    again = _check_labels(cm, names, phonemes)
    assert all(_bits_equal(again[n][1], labels[n][1]) for n in names)
    # best head
    _run('extract_durations.py', ['--config', str(cfg), '--best'])
    _check_labels(cm, names, phonemes)
    # the ForwardTransformer trains on the produced labels
    raw = yaml.safe_load(cfg.read_text())
    raw['tts_settings'].update(validation_frequency=1000, weights_save_frequency=1000)
    cfg.write_text(yaml.safe_dump(raw))
    out = _run('train_tts.py', ['--config', str(cfg), '--max_steps', '2'])
    assert 'Done.' in out and 1 in _losses(out)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_train_aligner_data_parallel_two_ranks(tmp_path):
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    cfg = _config(tmp_path, reduction_factor_schedule=[[0, 2], [2, 1]], validation_frequency=2, prediction_start_step=2,
                  prediction_frequency=1000)
    _write_dataset(TrainingConfigManager(str(cfg), aligner=True))
    out = _run('train_aligner.py', ['--config', str(cfg), '--max_steps', '4'], nproc=2)
    losses = _losses(out)
    assert sorted(losses) == [1, 2, 3, 4] and all(math.isfinite(v) for v in losses.values()) and 'Done.' in out
    assert 'validation loss at step 4' in out
