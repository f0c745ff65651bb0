"""Golden records of the REFERENCE'S OWN CODE for tests/test_aligner_pipeline.py (the label-generation pipeline:
train_aligner.py -> extract_durations.py).

    TTS_REFERENCE=<checkout of as-ideas/TransformerTTS> python tests/golden/make_golden_aligner_pipeline.py

  * utils/training_config_manager.py: ``TrainingConfigManager(aligner=True)`` on config/training_config.yaml and on a renamed
    variant (both with the ``wav_directory`` / ``metadata_path`` keys its constructor reads), run on tests/tf_shim: session
    directories, data paths, ``max_r``, ``stop_scaling`` and the flattened keys -> aligner_pipeline.json;
  * data/datasets.py: ``DataReader.from_config`` for the four kinds on small metadata files -> aligner_pipeline.json;
  * extract_durations.py: the nested ``_pitch_per_char`` (taken out of the script by its AST; ``np.float`` is float64, as in
    the numpy the reference was written for) on seeded cases -> char_pitch.npz (inputs and outputs).
"""
import ast
import json
import sys
import tempfile
from pathlib import Path

import numpy as np
import yaml

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(HERE.parent))
import ref_shim  # noqa: E402

# metadata of the Data API comparison: the corpus file (LJSpeech columns) and the processed name|phonemes files
META = {
    'metadata.csv': 'LJ001-0001.wav|Printing, in the only sense|printing in the only sense\nLJ001-0002|really?|really?\n'
                    'LJ001-0003|stop!|stop!\nLJ001-0004|fine.|fine.\n',
    'train': 'LJ001-0001|pɹˈɪntɪŋ\nLJ001-0002|ɹˈiːli?\nLJ001-0004|fˈaɪn.\n',
    'valid': 'LJ001-0003|stˈɑːp!\n',
    'phonemized': 'LJ001-0001|pɹˈɪntɪŋ\nLJ001-0002|ɹˈiːli?\nLJ001-0003|stˈɑːp!\nLJ001-0004|fˈaɪn.\n',
}


def config_variants():
    """(name, raw yaml dict): the shipped config and a renamed one with another schedule / stop scaling."""
    raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    raw['paths'].update(wav_directory='wavs', metadata_path='wavs/metadata.csv')
    other = json.loads(json.dumps(raw))
    other['naming'].update(data_name='ljspeech', aligner_settings_name='aligner_b', text_settings_name='NoStress',
                           audio_settings_name='WaveRNN')
    other['paths'].update(log_directory='runs/x', train_data_directory='data/tts')
    other['aligner_settings']['reduction_factor_schedule'] = [[0, 6], [10, 3], [20, 1]]
    del other['aligner_settings']['stop_loss_scaling']         # the default scaling, 1
    return [('shipped', raw), ('renamed', other)]


def char_pitch_cases():
    """(pitch, durations, mel_len, mean, std) cases of the per-character pitch comparison."""
    rng = np.random.default_rng(2024)
    mean, std = 215.3, 47.9

    def voiced(n, p_unvoiced=0.3, hi=None):
        v = rng.normal(0.0, 1.0, n)
        v[rng.random(n) < p_unvoiced] = 0.0
        if hi is not None:
            v[rng.random(n) < hi] = rng.uniform(4.0, 6.0)   # >= 400 Hz after v * std + mean
        return v

    cases = []
    d = np.array([3, 0, 5, 0, 0, 4, 2], dtype=np.int32)                     # zero-duration characters
    cases.append((voiced(int(d.sum())), d, int(d.sum()), mean, std))
    d = np.array([4, 6, 3, 5], dtype=np.int32)                              # an all-unvoiced segment
    p = voiced(int(d.sum()))
    p[4:10] = 0.0
    cases.append((p, d, 40, mean, std))
    d = rng.integers(1, 9, 20).astype(np.int32)                             # frames >= 400 Hz, including a whole segment
    p = voiced(int(d.sum()), hi=0.25)
    p[:d[0]] = 5.0
    cases.append((p, d, int(d.sum()), mean, std))
    d = rng.integers(2, 7, 15).astype(np.int32)                             # durations running past the pitch length
    cases.append((voiced(int(d.sum()) - 11), d, int(d.sum()), mean, std))
    d = rng.integers(0, 5, 30).astype(np.int32)                             # mel_len < len(durations)
    cases.append((voiced(int(d.sum())), d, 17, mean, std))
    d = np.array([3, 150, 7, 300, 2, 611, 129, 136, 1], dtype=np.int32)     # segments longer than 128 frames
    cases.append((voiced(int(d.sum()), p_unvoiced=0.05), d, int(d.sum()), mean, std))
    for k in range(6):                                                      # generic utterances
        n = int(rng.integers(5, 90))
        d = rng.integers(0, 14, n).astype(np.int32)
        tm = int(d.sum()) + int(rng.integers(-3, 4))
        cases.append((voiced(max(tm, 0), hi=0.05), d, int(rng.integers(n // 2, n + 3)), float(rng.uniform(120, 260)),
                      float(rng.uniform(20, 80))))
    return cases


def reference_pitch_per_char():
    """extract_durations.py's nested _pitch_per_char as a function of (pitch, durations, mel_len, pitch_stats)."""
    tree = ast.parse((ref_shim.REFERENCE / 'extract_durations.py').read_text())
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == '_pitch_per_char')
    code = compile(ast.Module(body=[fn], type_ignores=[]), 'extract_durations.py', 'exec')

    class _Numpy:   # np.float, removed from numpy since, was the builtin float (float64 arrays)
        def __getattr__(self, k):
            return np.float64 if k == 'float' else getattr(np, k)

    def run(pitch, durations, mel_len, pitch_mean, pitch_std):
        ns = {'np': _Numpy(), 'pitch_stats': {'pitch_mean': pitch_mean, 'pitch_std': pitch_std}}
        exec(code, ns)
        return ns['_pitch_per_char'](pitch, durations, mel_len)
    return run


def main():
    ref_shim.activate()
    from utils.training_config_manager import TrainingConfigManager
    from data.datasets import DataReader
    js = {'configs': {}, 'meta': META, 'readers': {}}
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        for name, raw in config_variants():
            path = tmp / f'{name}.yaml'
            path.write_text(yaml.safe_dump(raw))
            cm = TrainingConfigManager(str(path), aligner=True)
            js['configs'][name] = {
                'raw': raw, 'base_dir': str(cm.base_dir), 'log_dir': str(cm.log_dir), 'weights_dir': str(cm.weights_dir),
                'data_dir': str(cm.data_dir), 'duration_dir': str(cm.duration_dir), 'pitch_per_char': str(cm.pitch_per_char),
                'mel_dir': str(cm.mel_dir), 'pitch_dir': str(cm.pitch_dir), 'metadata_path': str(cm.metadata_path),
                'train_metadata_path': str(cm.train_metadata_path), 'valid_metadata_path': str(cm.valid_metadata_path),
                'phonemized_metadata_path': str(cm.phonemized_metadata_path), 'max_r': int(cm.max_r),
                'stop_scaling': float(cm.stop_scaling), 'learning_rate': float(cm.learning_rate), 'keys': sorted(cm.config),
                'session_names': dict(cm.session_names)}
        # DataReader.from_config on metadata files written under tmp (the shipped config's names, paths made absolute)
        raw = json.loads(json.dumps(config_variants()[0][1]))
        raw['paths'].update(wav_directory=str(tmp / 'wavs'), metadata_path=str(tmp / 'wavs' / 'metadata.csv'),
                            train_data_directory=str(tmp / 'tts'), log_directory=str(tmp / 'logs'))
        (tmp / 'reader.yaml').write_text(yaml.safe_dump(raw))
        cm = TrainingConfigManager(str(tmp / 'reader.yaml'), aligner=True)
        (tmp / 'wavs').mkdir()
        cm.data_dir.mkdir()
        cm.metadata_path.write_text(META['metadata.csv'], encoding='utf-8')
        for kind, p in (('train', cm.train_metadata_path), ('valid', cm.valid_metadata_path), ('phonemized', cm.phonemized_metadata_path)):
            p.write_text(META[kind], encoding='utf-8')
        for kind in ('original', 'phonemized', 'train', 'valid'):
            r = DataReader.from_config(cm, kind=kind)
            js['readers'][kind] = {'metadata': str(Path(r.metadata_path).relative_to(tmp)), 'filenames': list(r.filenames),
                                   'text_dict': dict(r.text_dict)}
    (HERE / 'aligner_pipeline.json').write_text(json.dumps(js, indent=1, ensure_ascii=False, sort_keys=True))

    run = reference_pitch_per_char()
    arrays = {}
    for i, (pitch, dur, mel_len, mean, std) in enumerate(char_pitch_cases()):
        out = run(pitch, dur, mel_len, mean, std)
        arrays.update({f'{i}/pitch': pitch, f'{i}/durations': dur, f'{i}/mel_len': np.int64(mel_len),
                       f'{i}/stats': np.array([mean, std]), f'{i}/out': out})
    np.savez_compressed(HERE / 'char_pitch.npz', **arrays)
    print('wrote', HERE / 'aligner_pipeline.json', HERE / 'char_pitch.npz', f'({len(arrays) // 5} pitch cases)')


if __name__ == '__main__':
    main()
