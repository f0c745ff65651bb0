#!/usr/bin/env python
"""ForwardTransformer training driver with the loop contract of the reference's ``train_tts.py`` (:89-209):

    restore latest checkpoint -> [batch -> lr = piecewise_linear_schedule(step) -> set_constants -> train_step -> losses]
    -> `latest` checkpoint every 1000 steps, `step_N` every weights_save_frequency, validation every validation_frequency

    python train_tts.py --config config/training_config.yaml                       # on-disk training data (see below)
    python train_tts.py --config ... --synthetic [--max_steps N] [--batch_size B]  # seeded LJSpeech-shaped batches
    torchrun --nproc-per-node 8 train_tts.py --config ...                          # data parallel, one process per GPU

Training data: the directory layout the reference's ``create_training_data.py`` / ``extract_durations.py`` write (the
durations and per-character pitch can be produced here with ``train_aligner.py`` + ``extract_durations.py``)
(``<train_data_directory>.<data_name>/`` with ``train_metadata.*.txt`` / ``valid_metadata.*.txt`` (``name|phonemes``),
``mels.*/<name>.npy`` (T,80), ``durations.*/<name>.npy`` int (Tp,), ``char_pitch.*/<name>.npy`` (Tp,)), read by
``transformertts_b200/data/datasets.py`` with the bucket boundaries / batch sizes of the config (yaml :22-24), shuffled with
the reference's seed, assembled in pinned memory and copied to the GPU on a side stream (``PrefetchLoader``).  Under
torchrun every rank takes its row slice of each global batch (bucket batch sizes rounded down to a multiple of the world
size).  TensorBoard logging, audio rendering and the espeak phonemizer are outside the hot path.
"""
from __future__ import annotations

import argparse
import glob
import os
from pathlib import Path

import numpy as np
import torch

from transformertts_b200.utils.data_parallel import init_from_env
from transformertts_b200.utils.scheduling import piecewise_linear_schedule
from transformertts_b200.utils.training_config_manager import TrainingConfigManager


def synthetic_batches(B, Tp, Tm, mel_channels, seed):
    g = torch.Generator().manual_seed(seed)
    while True:
        tok = torch.randint(1, 127, (B, Tp), generator=g, dtype=torch.int32)
        extra = torch.multinomial(torch.ones(B, Tp), Tm - Tp, replacement=True, generator=g)
        dur = torch.ones(B, Tp, dtype=torch.int32)
        dur.scatter_add_(1, extra, torch.ones_like(extra, dtype=torch.int32))
        pitch = torch.randn(B, Tp, generator=g)
        mel = (torch.randn(B, Tm, mel_channels, generator=g) * 2 - 5).clamp(-11.5, 2.0)
        yield {'mel': mel, 'tokens': tok, 'durations': dur, 'pitch': pitch}


def file_batches(pattern):
    files = sorted(glob.glob(pattern))
    if not files:
        raise FileNotFoundError(pattern)
    while True:
        for f in files:
            z = np.load(f)
            yield {'mel': torch.from_numpy(z['mel']), 'tokens': torch.from_numpy(z['phonemes']),
                   'durations': torch.from_numpy(z['durations']), 'pitch': torch.from_numpy(z['pitch'])}


def make_datasets(cm: TrainingConfigManager, cfg: dict, rank: int, world: int, device):
    """reference train_tts.py:100-115: TTSPreprocessor + TTSDataset for 'train' and 'valid', bucketed batches."""
    from transformertts_b200.data import datasets as ds
    from transformertts_b200.data.text import Tokenizer
    tokenizer = Tokenizer(add_start_end=False, model_breathing=bool(cfg.get('model_breathing', False)))
    prep = ds.TTSPreprocessor(int(cfg['mel_channels']), tokenizer)

    def handler(meta, training):
        reader = ds.DataReader(meta, training=training, is_processed=True)
        return ds.TTSDataset(reader, prep, cm.mel_dir, cm.duration_dir, cm.pitch_per_char)

    sizes = list(cfg['bucket_batch_sizes'])
    val_sizes = list(cfg.get('val_bucket_batch_size', sizes))
    if world > 1:
        sizes, val_sizes = ds.round_batch_sizes(sizes, world), ds.round_batch_sizes(val_sizes, world)
    train = handler(cm.train_metadata_path, True).get_dataset(bucket_batch_sizes=sizes, bucket_boundaries=cfg['bucket_boundaries'],
                                                               shuffle=True, drop_remainder=world > 1, rank=rank, world_size=world)
    valid = handler(cm.valid_metadata_path, False).get_dataset(bucket_batch_sizes=val_sizes, bucket_boundaries=cfg['bucket_boundaries'],
                                                               shuffle=False, drop_remainder=True, rank=rank, world_size=world)
    return ds.PrefetchLoader(train, prefetch=4, device=device), valid


def validate(model, valid, device, data_parallel):
    """reference train_tts.py:45-60: mean validation loss over all validation batches (forward only)."""
    tot, n = 0.0, 0
    for b in valid.all_batches():
        out = model.val_step(b['tokens'].to(device), b['mel'].to(device), b['durations'].to(device), b['pitch'].to(device))
        tot += float(out['loss'])
        n += 1
    if data_parallel and n:
        import torch.distributed as dist
        t = torch.tensor([tot, float(n)], device=device)
        dist.all_reduce(t)
        tot, n = float(t[0]), float(t[1])
    return tot / max(n, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', required=True)
    ap.add_argument('--reset_dir', dest='clear_dir', action='store_true', help="deletes everything under this config's folder")
    ap.add_argument('--reset_logs', dest='clear_logs', action='store_true')
    ap.add_argument('--reset_weights', dest='clear_weights', action='store_true', help='start from scratch: delete saved weights')
    ap.add_argument('--synthetic', action='store_true')
    ap.add_argument('--batches', default=None, help='glob of pre-batched .npz files')
    ap.add_argument('--max_steps', type=int, default=None)
    ap.add_argument('--batch_size', type=int, default=32)
    ap.add_argument('--weights_dir', default=None)
    ap.add_argument('--checkpoint_frequency', type=int, default=1000, help="steps between rewrites of weights/latest (reference: 1000)")
    args = ap.parse_args()

    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local_rank)
    device = torch.device('cuda', local_rank)
    rank, world = init_from_env(device=device)
    np.random.seed(42)
    torch.manual_seed(42)

    cm = TrainingConfigManager(args.config)
    cfg = cm.config
    if args.weights_dir:
        cm.weights_dir = Path(args.weights_dir)
        cm.base_dir = cm.weights_dir.parent
        cm.log_dir = cm.base_dir / 'logs'
    if rank == 0:
        cm.create_remove_dirs(clear_dir=args.clear_dir, clear_logs=args.clear_logs, clear_weights=args.clear_weights)
        cm.dump_config()
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
    # ---- model: restore the latest checkpoint (weights + Adam state + step) unless told to start over
    latest = cm.latest_checkpoint()
    if latest is not None:
        model = cm.load_model(str(latest), verbose=False, device=str(device))
        if rank == 0:
            print(f'\nresuming training from step {model.step} ({latest})')
    else:
        model = cm.get_model(device=str(device))
        cm.compile_model(model)
        if rank == 0:
            print('\nstarting training from scratch')
    model._get_engine().rank = rank          # per-rank dropout streams
    # ---- data
    valid = None
    if args.batches:
        data = file_batches(args.batches)
    elif args.synthetic:
        data = synthetic_batches(args.batch_size, 128, 1000, int(cfg.get('mel_channels', 80)), seed=1000 + rank)
        for _ in range(model.step):          # a resumed run continues the batch stream where the killed one stopped
            next(data)
    else:
        data, valid = make_datasets(cm, cfg, rank, world, device)
    max_steps = args.max_steps or int(cfg['max_steps'])
    save_freq, save_start = int(cfg.get('weights_save_frequency', 5000)), int(cfg.get('weights_save_starting_step', 0))
    val_freq = int(cfg.get('validation_frequency', 0) or 0)
    if rank == 0:
        print('\nTRAINING')
    while model.step < max_steps:
        b = next(data)
        lr = piecewise_linear_schedule(model.step, cfg['learning_rate_schedule'])
        model.set_constants(learning_rate=lr)
        out = model.train_step(input_sequence=b['tokens'], target_sequence=b['mel'], target_durations=b['durations'],
                               target_pitch=b['pitch'], data_parallel=world > 1)
        if rank == 0 and (model.step % 10 == 0 or model.step == 1):
            print(f'step {model.step}  loss {float(out["loss"]):.4f}  mel {float(out["losses"]["mel"]):.4f}  '
                  f'duration {float(out["losses"]["duration"]):.4f}  pitch {float(out["losses"]["pitch"]):.4f}  lr {lr:.2e}', flush=True)
        if rank == 0 and model.step % args.checkpoint_frequency == 0:
            model.save_model(cm.weights_dir / 'latest')
        if rank == 0 and model.step % save_freq == 0 and model.step >= save_start:
            model.save_model(cm.weights_dir / f'step_{model.step}')
        if valid is not None and val_freq and model.step % val_freq == 0:
            v = validate(model, valid, device, world > 1)
            if rank == 0:
                print(f'validation loss at step {model.step}: {v:.4f}', flush=True)
    if rank == 0:
        model.save_model(cm.weights_dir / f'step_{model.step}')
        model.save_model(cm.weights_dir / 'latest')
        print('Done.')
    if hasattr(data, 'close'):
        data.close()


if __name__ == '__main__':
    main()
