"""Config handling mirroring the reference's ``utils/training_config_manager.py``: the yaml sections are flattened into one
dict (:49-56) -- ``tts_settings`` for the ForwardTransformer, ``aligner_settings`` for the Aligner -- that is splatted into
the model constructor (:94-100), the optimizer is Adam(lr, beta_1 0.9, beta_2 0.98, epsilon 1e-9) (:102-110), the
directory layout of a session (:23-44: ``<log_directory>/<data_name>/<session name>/{logs,weights}`` with the session name
``<tts_settings_name>.<aligner_settings_name>`` or ``<aligner_settings_name>.<text_settings_name>.<audio_settings_name>``,
training data under ``<train_data_directory>.<data_name>/``) and checkpoint restore (:140-160).  Git-hash checks are
outside the hot path."""
from __future__ import annotations

import shutil
from pathlib import Path
from typing import Optional

import numpy as np
import yaml

from ..model.aligner import Aligner
from ..model.models import ForwardTransformer
from ..model.training import Adam
from .scheduling import reduction_schedule

SECTIONS = ('paths', 'naming', 'training_data_settings', 'audio_settings', 'text_settings')


class TrainingConfigManager:
    def __init__(self, config_path: str, aligner: bool = False):
        self.config_path = Path(config_path)
        self.model_kind = 'aligner' if aligner else 'tts'
        self.config = self._load_config()
        c = self.config
        self.learning_rate = float(np.array(c['learning_rate_schedule'])[0, 1])
        self.data_name = str(c.get('data_name', 'data'))
        text_name, audio_name = c.get('text_settings_name', 'text'), c.get('audio_settings_name', 'audio')
        tts_name, aligner_name = c.get('tts_settings_name', 'tts'), c.get('aligner_settings_name', 'aligner')
        self.session_names = {'data': f'{text_name}.{audio_name}'}
        self.session_names['aligner'] = f"{aligner_name}.{self.session_names['data']}"
        self.session_names['tts'] = f'{tts_name}.{aligner_name}'
        self.base_dir = Path(c.get('log_directory', '.')) / self.data_name / self.session_names[self.model_kind]
        self.log_dir = self.base_dir / 'logs'
        self.weights_dir = self.base_dir / 'weights'
        # on-disk training data (reference :31-44)
        self.data_dir = Path(f"{c.get('train_data_directory', 'transformer_tts_data')}.{self.data_name}")
        self.metadata_path = Path(c['metadata_path']) if c.get('metadata_path') else None      # the raw corpus metadata
        self.wav_directory = Path(c['wav_directory']) if c.get('wav_directory') else None
        self.train_metadata_path = self.data_dir / f'train_metadata.{text_name}.txt'
        self.valid_metadata_path = self.data_dir / f'valid_metadata.{text_name}.txt'
        self.phonemized_metadata_path = self.data_dir / f'phonemized_metadata.{text_name}.txt'
        self.mel_dir = self.data_dir / f'mels.{audio_name}'
        self.pitch_dir = self.data_dir / f'pitch.{audio_name}'
        self.duration_dir = self.data_dir / f"durations.{self.session_names['aligner']}"
        self.pitch_per_char = self.data_dir / f"char_pitch.{self.session_names['aligner']}"
        if self.model_kind == 'aligner':
            # reference :45-47
            self.max_r = int(np.array(c['reduction_factor_schedule'])[0, 1])
            self.stop_scaling = float(c.get('stop_loss_scaling', 1.))

    def _load_config(self) -> dict:
        with open(self.config_path, 'rb') as f:
            raw = yaml.safe_load(f)
        flat = {}
        for key in SECTIONS + (f'{self.model_kind}_settings',):
            flat.update(raw.get(key, {}) or {})
        return flat

    def get_model(self, ignore_hash: bool = True, **overrides):
        cfg = dict(self.config)
        cfg.update(overrides)
        if self.model_kind == 'aligner':
            return Aligner.from_config(cfg, max_r=self.max_r)
        return ForwardTransformer.from_config(cfg)

    def compile_model(self, model, beta_1: float = 0.9, beta_2: float = 0.98):
        optimizer = Adam(self.learning_rate, beta_1=beta_1, beta_2=beta_2, epsilon=1e-9)
        if self.model_kind == 'aligner':
            model._compile(stop_scaling=self.stop_scaling, optimizer=optimizer)
        else:
            model._compile(optimizer=optimizer)

    def create_remove_dirs(self, clear_dir: bool = False, clear_logs: bool = False, clear_weights: bool = False):
        """reference :117-138 without the interactive prompt (a flag given on the command line is the confirmation)."""
        self.base_dir.mkdir(exist_ok=True, parents=True)
        if clear_dir or clear_logs:
            shutil.rmtree(self.log_dir, ignore_errors=True)
        if clear_dir or clear_weights:
            shutil.rmtree(self.weights_dir, ignore_errors=True)
        self.log_dir.mkdir(exist_ok=True)
        self.weights_dir.mkdir(exist_ok=True)

    def dump_config(self):
        with open(self.base_dir / 'config.yaml', 'w') as f:
            yaml.safe_dump(dict(self.config, automatic=True), f)

    def latest_checkpoint(self, weights_dir: Optional[Path] = None) -> Optional[Path]:
        """The directory training resumes from: ``weights/latest`` (rewritten every 1000 steps, as the reference's
        CheckpointManager(max_to_keep=1) at train_tts.py:124-125), else the newest ``step_N`` directory that holds optimizer
        state."""
        wd = Path(weights_dir) if weights_dir is not None else self.weights_dir
        if (wd / 'latest' / 'optimizer.pt').exists():
            return wd / 'latest'
        steps = sorted((int(p.name.split('_')[1]), p) for p in wd.glob('step_*') if (p / 'optimizer.pt').exists())
        return steps[-1][1] if steps else None

    def load_model(self, checkpoint_path: str = None, verbose: bool = True, **overrides):
        """reference :140-160: the model of this config with the weights (and optimizer state) of a checkpoint directory.
        An Aligner gets the reduction factor its schedule sets at the restored step."""
        path = Path(checkpoint_path) if checkpoint_path else self.latest_checkpoint()
        if path is None:
            raise FileNotFoundError(f'no checkpoint under {self.weights_dir}')
        cls = Aligner if self.model_kind == 'aligner' else ForwardTransformer
        model = cls.load_model(path, **overrides)
        if model.optimizer is None:
            self.compile_model(model)
        if self.model_kind == 'aligner':
            model.stop_scaling = self.stop_scaling
            model.set_constants(reduction_factor=reduction_schedule(model.step, self.config['reduction_factor_schedule']))
        if verbose:
            print(f'restored weights from {path} at step {model.step}')
        return model
