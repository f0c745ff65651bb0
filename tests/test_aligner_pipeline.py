"""CPU tests of the label-generation pipeline (train_aligner.py -> extract_durations.py): the Aligner branch of the config
manager, the Data API constructors and the per-character pitch, against records of the reference's own code
(tests/golden/make_golden_aligner_pipeline.py), and the C-ABI checks of ttsb_pitch_per_char that need no GPU."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest
import yaml

ROOT = Path(__file__).resolve().parent.parent
GOLD = Path(__file__).resolve().parent / 'golden'


def _golden():
    return json.loads((GOLD / 'aligner_pipeline.json').read_text(encoding='utf-8'))


@pytest.mark.parametrize('variant', ['shipped', 'renamed'])
def test_aligner_config_branch_matches_reference(tmp_path, variant):
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    want = _golden()['configs'][variant]
    path = tmp_path / 'cfg.yaml'
    path.write_text(yaml.safe_dump(want['raw']))
    cm = TrainingConfigManager(str(path), aligner=True)
    assert cm.model_kind == 'aligner'
    for key in ('base_dir', 'log_dir', 'weights_dir', 'data_dir', 'duration_dir', 'pitch_per_char', 'mel_dir', 'pitch_dir',
                'metadata_path', 'train_metadata_path', 'valid_metadata_path', 'phonemized_metadata_path'):
        assert str(getattr(cm, key)) == want[key], key
    assert cm.session_names == want['session_names']
    assert cm.max_r == want['max_r'] and isinstance(cm.max_r, int)
    assert cm.stop_scaling == want['stop_scaling']
    assert sorted(cm.config) == want['keys']
    assert cm.learning_rate == pytest.approx(want['learning_rate'], rel=1e-6)


def test_shipped_config_builds_the_reference_aligner_and_keeps_the_tts_branch(tmp_path):
    from transformertts_b200.model.aligner import Aligner
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.model.training import Adam
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    cfg = str(ROOT / 'config' / 'training_config.yaml')
    cm = TrainingConfigManager(cfg, aligner=True)
    m = cm.get_model(device='cpu')
    assert isinstance(m, Aligner)
    assert m.vocab_size == 129 and m.max_r == 10 and m.r == 10
    assert m._stacks['encoder']['heads'] == [4, 4, 4, 4] and m._stacks['decoder']['heads'] == [4, 4, 4, 4, 1]
    assert m.config['mel_start_value'] == 0.5 and m.config['mel_end_value'] == -0.5
    cm.compile_model(m)
    assert m.stop_scaling == 8.0 and isinstance(m.optimizer, Adam)
    assert (m.optimizer.beta_1, m.optimizer.beta_2, m.optimizer.epsilon) == (0.9, 0.98, 1e-9)
    m.set_constants(learning_rate=3e-5, reduction_factor=2)
    assert m.optimizer.lr == 3e-5 and m.r == 2
    tts = TrainingConfigManager(cfg)
    assert tts.model_kind == 'tts' and tts.base_dir.name == 'tts_swap_conv_dims.alinger_extralayer_layernorm'
    assert 'reduction_factor_schedule' not in tts.config and 'duration_conv_filters' in tts.config
    assert isinstance(tts.get_model(device='cpu'), ForwardTransformer)


def test_aligner_checkpoint_restores_through_the_config_manager(tmp_path):
    """save_model -> TrainingConfigManager.load_model: weights, Adam state, step and the scheduled reduction factor."""
    import torch
    from oracle import aligner_oracle as alo
    from transformertts_b200.model.training import Adam
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    small = {k: v for k, v in alo.ALIGNER_CONFIGS['A-small'].items() if k not in ('max_r', 'vocab_size')}
    raw['aligner_settings'].update(small, reduction_factor_schedule=[[0, 4], [3, 2], [6, 1]], stop_loss_scaling=3)
    raw['paths']['log_directory'] = str(tmp_path / 'logs')
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(raw))
    cm = TrainingConfigManager(str(tmp_path / 'cfg.yaml'), aligner=True)
    m = cm.get_model(device='cpu')
    cm.compile_model(m)
    m.optimizer.iterations = 4
    m.save_model(tmp_path / 'ckpt', with_optimizer=False)
    torch.save({'iterations': 4, 'lr': 2e-5, 'beta_1': 0.9, 'beta_2': 0.98, 'epsilon': 1e-9, 'm': {}, 'v': {}, 'base_seed': 77},
               tmp_path / 'ckpt' / 'optimizer.pt')
    m2 = cm.load_model(str(tmp_path / 'ckpt'), verbose=False, device='cpu')
    assert m2.step == 4 and m2.r == 2 and m2.max_r == 4 and m2.stop_scaling == 3.0
    assert isinstance(m2.optimizer, Adam) and m2.optimizer.lr == 2e-5
    assert all(torch.equal(m2.weights[k], m.weights[k]) for k in m.weights)


def _write_reader_files(tmp_path, meta):
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    raw['paths'].update(wav_directory=str(tmp_path / 'wavs'), metadata_path=str(tmp_path / 'wavs' / 'metadata.csv'),
                        train_data_directory=str(tmp_path / 'tts'), log_directory=str(tmp_path / 'logs'))
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(raw))
    cm = TrainingConfigManager(str(tmp_path / 'cfg.yaml'), aligner=True)
    (tmp_path / 'wavs').mkdir()
    cm.data_dir.mkdir()
    cm.metadata_path.write_text(meta['metadata.csv'], encoding='utf-8')
    for kind, p in (('train', cm.train_metadata_path), ('valid', cm.valid_metadata_path), ('phonemized', cm.phonemized_metadata_path)):
        p.write_text(meta[kind], encoding='utf-8')
    return cm


def test_data_reader_from_config_kinds_match_reference(tmp_path):
    from transformertts_b200.data import datasets as ds
    g = _golden()
    cm = _write_reader_files(tmp_path, g['meta'])
    for kind, want in g['readers'].items():
        r = ds.DataReader.from_config(cm, kind=kind)
        assert str(Path(r.metadata_path).relative_to(tmp_path)) == want['metadata'], kind
        assert r.filenames == want['filenames'], kind
        assert r.text_dict == want['text_dict'], kind
    with pytest.raises(ValueError):
        ds.DataReader.from_config(cm, kind='test')


def test_aligner_dataset_from_config_builds_reference_samples(tmp_path):
    from transformertts_b200.data import datasets as ds
    from transformertts_b200.data.text import Tokenizer
    cm = _write_reader_files(tmp_path, _golden()['meta'])
    cm.mel_dir.mkdir()
    rng = np.random.default_rng(0)
    for i, name in enumerate(ds.DataReader.from_config(cm, kind='phonemized').filenames):
        np.save(cm.mel_dir / f'{name}.npy', rng.normal(-4, 1, (20 + 7 * i, 80)).astype(np.float32))
    tok = Tokenizer(add_start_end=True, model_breathing=False)     # model_breathing: false in the shipped config
    assert tok.vocab_size == 129
    prep = ds.AlignerPreprocessor.from_config(cm, tok)
    data = ds.AlignerDataset.from_config(cm, prep, kind='phonemized')
    assert data.mel_directory == cm.mel_dir
    batches = list(data.get_dataset(bucket_batch_sizes=[4, 4], bucket_boundaries=[1000], shuffle=False, drop_remainder=False,
                                    pin_memory=False).all_batches())
    assert len(batches) == 1
    b = batches[0]
    assert b['name'] == ['LJ001-0001', 'LJ001-0002', 'LJ001-0003', 'LJ001-0004']
    assert b['tokens'][0, 0] == 127 and int(b['tokens'][0, len(tok('pɹˈɪntɪŋ')) - 1]) == 128
    assert float(b['mel'][0, 0, 0]) == 0.5 and float(b['mel'][0, 21, 0]) == -0.5
    assert b['stop_prob'][0, :22].tolist() == [1] * 21 + [2] and int(b['stop_prob'][0, 22:].abs().sum()) == 0


def test_pitch_per_char_equals_reference_function_bitwise():
    """datasets.pitch_per_char (the host reference of the kernel) against the reference's own _pitch_per_char."""
    from transformertts_b200.data.datasets import pitch_per_char
    with np.load(GOLD / 'char_pitch.npz') as z:
        n = len({k.split('/')[0] for k in z.files})
        assert n >= 12
        long_segment = False
        for i in range(n):
            pitch, dur, mel_len, (mean, std), want = (z[f'{i}/pitch'], z[f'{i}/durations'], int(z[f'{i}/mel_len']), z[f'{i}/stats'],
                                                      z[f'{i}/out'])
            got = pitch_per_char(pitch, dur, mel_len, float(mean), float(std))
            assert got.dtype == np.float64 and got.shape == want.shape
            assert np.array_equal(got.view(np.int64), want.view(np.int64)), i
            long_segment |= bool((dur > 128).any())
        assert long_segment


def kernel_order_mean(values: np.ndarray) -> float:
    """The summation order ttsb_pitch_per_char uses (csrc/alignment.cu pairwise_sum), restated: numpy's pairwise sum."""
    def pw(lo, n):
        if n < 8:
            s = 0.0
            for k in range(n):
                s += values[lo + k]
            return s
        if n <= 128:
            r = [values[lo + j] for j in range(8)]
            k = 8
            while k < n - n % 8:
                for j in range(8):
                    r[j] += values[lo + k + j]
                k += 8
            s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            for k in range(k, n):
                s += values[lo + k]
            return s
        n2 = n // 2
        n2 -= n2 % 8
        return pw(lo, n2) + pw(lo + n2, n - n2)
    values = [float(v) for v in values]
    return pw(0, len(values)) / len(values) if values else 0.0


def test_kernel_summation_order_equals_np_mean_bitwise():
    rng = np.random.default_rng(11)
    for n in range(0, 601):
        for _ in range(2):
            a = rng.normal(0, 1, n) * 10.0 ** rng.uniform(-4, 4, n)
            want = np.mean(a) if n > 0 else 0.0
            assert np.float64(kernel_order_mean(a)).view(np.int64) == np.float64(want).view(np.int64), n


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def test_pitch_per_char_abi_validation_without_gpu(cdll):
    from transformertts_b200 import lib
    assert 'ttsb_pitch_per_char' in lib.EXPORTS and hasattr(cdll, 'ttsb_pitch_per_char')
    assert 'ttsb_pitch_per_char(' in (ROOT / 'include' / 'ttsb.h').read_text()
    f = cdll.ttsb_pitch_per_char
    p = C.c_void_p(256)     # never dereferenced: the arguments are refused before any CUDA call
    assert f(None, 1, 10, p, p, 4, p, C.c_double(200.0), C.c_double(50.0), p, None) == -1
    assert b'ttsb_pitch_per_char' in cdll.ttsb_last_error()
    assert f(p, 0, 10, p, p, 4, p, C.c_double(200.0), C.c_double(50.0), p, None) == -1
    assert f(p, 1, 10, p, p, 0, p, C.c_double(200.0), C.c_double(50.0), p, None) == -1
    assert f(p, 1, 10, p, p, 20000, p, C.c_double(200.0), C.c_double(50.0), p, None) == -1
    assert b'Tp too large' in cdll.ttsb_last_error()
