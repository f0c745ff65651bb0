#!/usr/bin/env python
"""Aligner training driver with the loop contract of the reference's ``train_aligner.py`` (:80-222):

    restore weights/latest -> [batch -> lr = piecewise_linear_schedule(step), r = reduction_schedule(step),
    force_{encoder,decoder}_diagonal = step < force_{encoder,decoder}_diagonal_steps -> set_constants -> train_step]
    -> `latest` checkpoint every --checkpoint_frequency steps, `step_N` every weights_save_frequency, validation (mean
    loss at r=1 plus duration extraction from the last batch) and an autoregressive prediction every
    validation_frequency / prediction_frequency steps once step >= prediction_start_step

    python train_aligner.py --config config/training_config.yaml                       # on-disk training data
    python train_aligner.py --config ... --synthetic [--max_steps N] [--batch_size B]  # seeded batches of random tokens / mels
    torchrun --nproc-per-node 8 train_aligner.py --config ...                          # data parallel, one process per GPU

Training data: ``<train_data_directory>.<data_name>/`` with ``train_metadata.*.txt`` / ``valid_metadata.*.txt``
(``name|phonemes``) and ``mels.*/<name>.npy`` (T, mel_channels), read through ``AlignerDataset`` (start / end vectors and
stop targets added per utterance) with the config's buckets.  The session directory is
``<log_directory>/<data_name>/<aligner_settings_name>.<text_settings_name>.<audio_settings_name>/``, where
``extract_durations.py`` finds the weights.  TensorBoard images and audio and the espeak test sentences are not produced.
"""
from __future__ import annotations

import argparse
import os
from pathlib import Path

import numpy as np
import torch

from transformertts_b200.utils.data_parallel import init_from_env
from transformertts_b200.utils.scheduling import piecewise_linear_schedule, reduction_schedule
from transformertts_b200.utils.training_config_manager import TrainingConfigManager


def synthetic_batches(B, Tp, Tm, mel_channels, start_value, end_value, vocab, seed):
    """Aligner samples as AlignerPreprocessor builds them: start token + random symbols + end token; start vector + mel +
    end vector; stop targets 1, .., 1, 2."""
    g = torch.Generator().manual_seed(seed)
    while True:
        tok = torch.randint(1, vocab - 2, (B, Tp), generator=g, dtype=torch.int32)
        tok[:, 0], tok[:, -1] = vocab - 2, vocab - 1
        mel = (torch.randn(B, Tm, mel_channels, generator=g) * 2 - 5).clamp(-11.5, 2.0)
        mel[:, 0], mel[:, -1] = start_value, end_value
        stop = torch.ones(B, Tm, dtype=torch.int32)
        stop[:, -1] = 2
        yield {'mel': mel, 'tokens': tok, 'stop_prob': stop}


def make_datasets(cm: TrainingConfigManager, cfg: dict, rank: int, world: int, device):
    """reference train_aligner.py:88-105: AlignerPreprocessor + AlignerDataset for 'train' and 'valid', bucketed batches."""
    from transformertts_b200.data import datasets as ds
    from transformertts_b200.data.text import Tokenizer
    prep = ds.AlignerPreprocessor.from_config(cm, Tokenizer(add_start_end=True, model_breathing=bool(cfg.get('model_breathing', False))))
    sizes = list(cfg['bucket_batch_sizes'])
    val_sizes = list(cfg.get('val_bucket_batch_size', sizes))
    if world > 1:
        sizes, val_sizes = ds.round_batch_sizes(sizes, world), ds.round_batch_sizes(val_sizes, world)
    train = ds.AlignerDataset.from_config(cm, prep, kind='train').get_dataset(
        bucket_batch_sizes=sizes, bucket_boundaries=cfg['bucket_boundaries'], shuffle=True, drop_remainder=world > 1, rank=rank,
        world_size=world)
    valid = ds.AlignerDataset.from_config(cm, prep, kind='valid').get_dataset(
        bucket_batch_sizes=val_sizes, bucket_boundaries=cfg['bucket_boundaries'], shuffle=False, drop_remainder=True, rank=rank,
        world_size=world)
    return train, valid


def validate(model, batches, weighted: bool, device, data_parallel: bool):
    """reference train_aligner.py:36-77: mean validation loss at r=1 over all validation batches, then durations from the
    last batch's last-block cross-attention (in the plain and, if configured, the weighted mode; the durations must sum
    to the mel length, as the reference asserts) and its per-head attention scores."""
    from transformertts_b200.utils.alignments import get_durations_from_alignment
    current_r = model.r
    model.set_constants(reduction_factor=1)
    tot, n, out, last = 0.0, 0, None, None
    for b in batches:
        last = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in b.items()}
        out = model.val_step(last['tokens'], last['mel'], last['stop_prob'])
        tot += float(out['loss'])
        n += 1
    if data_parallel:
        import torch.distributed as dist
        t = torch.tensor([tot, float(n)], device=device)
        dist.all_reduce(t)
        tot, n = float(t[0]), int(t[1])
    scores = None
    if out is not None:
        att = out['decoder_attention']['Decoder_LastBlock_CrossAttention']
        for mode in sorted({False, bool(weighted)}):
            _, _, jump, peak, diag = get_durations_from_alignment(att, last['mel'], last['tokens'], weighted=mode)
            scores = (jump.mean(0).tolist(), peak.mean(0).tolist(), diag.mean(0).tolist())
    model.set_constants(reduction_factor=current_r)
    return tot / max(n, 1), scores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', required=True)
    ap.add_argument('--reset_dir', dest='clear_dir', action='store_true', help="deletes everything under this config's folder")
    ap.add_argument('--reset_logs', dest='clear_logs', action='store_true')
    ap.add_argument('--reset_weights', dest='clear_weights', action='store_true', help='start from scratch: delete saved weights')
    ap.add_argument('--synthetic', action='store_true', help='seeded random batches instead of the on-disk training data')
    ap.add_argument('--max_steps', type=int, default=None)
    ap.add_argument('--batch_size', type=int, default=16, help='--synthetic only')
    ap.add_argument('--synthetic_shape', type=int, nargs=2, default=(64, 400), metavar=('TOKENS', 'FRAMES'),
                    help='--synthetic only: tokens and mel frames per sample, start and end included')
    ap.add_argument('--weights_dir', default=None)
    ap.add_argument('--checkpoint_frequency', type=int, default=1000, help='steps between rewrites of weights/latest (reference: 1000)')
    args = ap.parse_args()

    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local_rank)
    device = torch.device('cuda', local_rank)
    rank, world = init_from_env(device=device)
    np.random.seed(42)
    torch.manual_seed(42)

    cm = TrainingConfigManager(args.config, aligner=True)
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
    # ---- model: restore weights/latest (weights + Adam state + step) unless told to start over
    latest = cm.weights_dir / 'latest'
    if (latest / 'optimizer.pt').exists():
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
    mel_channels = int(cfg.get('mel_channels', 80))
    if args.synthetic:
        Tp, Tm = args.synthetic_shape
        synth = dict(Tp=Tp, Tm=Tm, mel_channels=mel_channels, start_value=float(cfg['mel_start_value']),
                     end_value=float(cfg['mel_end_value']), vocab=model.vocab_size)
        data = synthetic_batches(args.batch_size, seed=1000 + rank, **synth)
        for _ in range(model.step):          # a resumed run continues the batch stream where the stopped one ended
            next(data)
        val_gen = synthetic_batches(args.batch_size, seed=7 + rank, **synth)
        val_fixed = [next(val_gen) for _ in range(2)]        # a fixed validation set of two batches

        def valid_batches():
            return iter(val_fixed)
    else:
        from transformertts_b200.data.datasets import PrefetchLoader
        train, valid = make_datasets(cm, cfg, rank, world, device)
        valid_batches = valid.all_batches
        _ = train.next_batch()               # the reference discards the first training batch (train_aligner.py:141)
        data = PrefetchLoader(train, prefetch=4, device=device)
    # the sample the reference predicts from at prediction time: the first validation sample (train_aligner.py:137-139)
    first_val = next(iter(valid_batches()), None)
    val_sample = None if first_val is None else first_val['tokens'][0][first_val['tokens'][0] != 0]
    max_steps = args.max_steps or int(cfg['max_steps'])
    save_freq = int(cfg.get('weights_save_frequency', 5000))
    val_freq = int(cfg.get('validation_frequency', 0) or 0)
    pred_freq = int(cfg.get('prediction_frequency', 0) or 0)
    pred_start = int(cfg.get('prediction_start_step', 0))
    weighted = bool(cfg.get('extract_attention_weighted', False))
    if rank == 0:
        print('\nTRAINING')
        if pred_freq:
            print('note: audio, TensorBoard output and the test sentences (which need espeak) are not produced')
    while model.step < max_steps:
        b = next(data)
        step = model.step
        lr = piecewise_linear_schedule(step, cfg['learning_rate_schedule'])
        r = reduction_schedule(step, cfg['reduction_factor_schedule'])
        model.set_constants(learning_rate=lr, reduction_factor=r,
                            force_encoder_diagonal=step < int(cfg['force_encoder_diagonal_steps']),
                            force_decoder_diagonal=step < int(cfg['force_decoder_diagonal_steps']))
        out = model.train_step(b['tokens'], b['mel'], b['stop_prob'], data_parallel=world > 1)
        if rank == 0:
            ls = out['losses']
            print(f'step {model.step}  loss {float(out["loss"]):.5f}  mel {float(ls["mel"]):.5f}  stop_prob {float(ls["stop_prob"]):.5f}  '
                  f'diag {float(ls["diag_loss"]):.5f}  r {model.r}  lr {lr:.2e}', flush=True)
        if rank == 0 and model.step % args.checkpoint_frequency == 0:
            model.save_model(cm.weights_dir / 'latest')
        if rank == 0 and model.step % save_freq == 0:
            model.save_model(cm.weights_dir / f'step_{model.step}')
        if val_freq and model.step % val_freq == 0 and model.step >= pred_start:
            v, scores = validate(model, valid_batches(), weighted, device, world > 1)
            if rank == 0:
                print(f'validation loss at step {model.step}: {v:.5f}', flush=True)
                if scores is not None:
                    for name, vals in zip(('jumpiness', 'peakiness', 'diagonality'), scores):
                        print(f'  validation attention {name} per head: ' + ' '.join(f'{x:.4f}' for x in vals), flush=True)
        if rank == 0 and val_sample is not None and pred_freq and model.step % pred_freq == 0 and model.step >= pred_start:
            pred = model.predict(val_sample, encode=False, verbose=False)
            print(f'prediction at step {model.step}: {int(pred["mel"].shape[0])} frames', flush=True)
    if rank == 0:
        model.save_model(cm.weights_dir / f'step_{model.step}')
        model.save_model(cm.weights_dir / 'latest')
        print('Done.')
    if hasattr(data, 'close'):
        data.close()


if __name__ == '__main__':
    main()
