"""Golden records of the REFERENCE'S OWN CODE for tests/test_reference_shim.py.

    TTS_REFERENCE=<checkout of as-ideas/TransformerTTS> python tests/golden/make_golden_shim.py

The unmodified reference sources are imported and executed on top of tests/tf_shim (a torch-backed stand-in for the
TensorFlow/Keras primitives) with the oracle's seeded parameters and inputs; what they return is written to
tests/golden/ref_shim.npz (arrays) and tests/golden/ref_shim.json (names, orders, scalars).  Large arrays are stored as a
fixed, seeded sample of their flattened elements (ref_shim.sample_index), so the files stay small.
"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))
import ref_shim  # noqa: E402
from oracle import aligner_oracle as alo  # noqa: E402
from oracle import forward_oracle as fo  # noqa: E402

from ref_shim import CASES, PE_CASES, SPEC_SEED, TOKENIZER_MODES, META_TEXT, LR_SCHED, LR_STEPS, RED_SCHED, RED_STEPS, \
    PRED_SETTINGS, ALIGNER_PRED_CASES  # noqa: E402

ARR, JS = {}, {}


def put(key, t, sample=None):
    a = torch.as_tensor(t).detach().cpu()
    JS['shape/' + key] = list(a.shape)
    a = a.reshape(-1)
    if sample is not None:
        a = a[torch.from_numpy(ref_shim.sample_index(a.numel(), sample, key))]
    ARR[key] = a.numpy().astype(np.float32) if a.dtype in (torch.float64, torch.float32) else a.numpy()


def main():
    ref_shim.activate()
    torch.set_num_threads(4)
    from utils.losses import masked_crossentropy, new_scaled_crossentropy
    targets = np.array([[0, 1, 2]])
    logits = np.array([[[.3, .2, .1], [.3, .2, .1], [.3, .2, .1]]])
    JS['loss/scaled5'] = float(new_scaled_crossentropy(index=2, scaling=5)(targets, logits))
    JS['loss/scaled1'] = float(new_scaled_crossentropy(index=2, scaling=1)(targets, logits))
    JS['loss/masked'] = float(masked_crossentropy(targets, logits))

    from model.layers import Expand
    x = torch.tensor([[[0.54710746, 0.8943467], [0.7140938, 0.97968304], [0.5347662, 0.15213418]]])
    put('expand', Expand(model_dim=2)(x, torch.tensor([[[1.], [3.], [2.]]])))

    for cfg_name, B, Tp, Tm, seed in CASES:
        cfg = fo.CONFIGS[cfg_name]
        p = fo.init_params(cfg, seed=7)
        tok, dur, pit = fo.make_inputs('ragged', B, Tp, Tm, seed=seed)
        durf, pitf = dur[..., None].float(), pit[..., None]
        model = ref_shim.reference_forward_transformer(cfg, p, (tok, durf, pitf))
        with torch.no_grad():
            ref = model.call(tok, target_durations=durf, target_pitch=pitf, training=False)
        k = f'fwd/{cfg_name}/'
        put(k + 'mel', ref['mel'], 1024)
        put(k + 'duration', ref['duration'])
        put(k + 'pitch', ref['pitch'])
        put(k + 'expanded_mask', ref['expanded_mask'])
        for side in ('encoder_attention', 'decoder_attention'):
            JS[k + side] = sorted(ref[side])
            for name in ref[side]:
                put(k + side + '/' + name, ref[side][name], 128)

    cfg = fo.CONFIGS['C1']
    p = dict(fo.init_params(cfg, seed=7))
    p['dur_pred.out.b'] = torch.tensor([3.2])
    tok, dur, pit = fo.make_inputs('ragged', 3, 32, 160, seed=111)
    model = ref_shim.reference_forward_transformer(cfg, p, (tok, dur[..., None].float(), pit[..., None]))
    tokenizer = model.text_pipeline.tokenizer
    sym_a, sym_b = tokenizer.idx_to_token[int(tok[0, 0])], tokenizer.idx_to_token[int(tok[0, 1])]
    JS['pred/id_a'], JS['pred/id_b'] = int(tokenizer(sym_a)[0]), int(tokenizer(sym_b)[0])
    for i, (speed, mx, mn) in enumerate(PRED_SETTINGS):
        with torch.no_grad():
            ref = model.predict(tok, encode=False, speed_regulator=speed, phoneme_max_duration={sym_a: mx} if mx else None,
                                phoneme_min_duration={sym_b: mn} if mn else None)
        put(f'pred/{i}/mel', ref['mel'], 1024)
        put(f'pred/{i}/expanded_mask', ref['expanded_mask'])

    cfg = dict(fo.CONFIGS['C1'], dropout_rate=0.0, predictors_dropout=0.0)
    p = fo.init_params(cfg, seed=7)
    tok, dur, pit = fo.make_inputs('ragged', 3, 24, 150, seed=301)
    mel_tgt = fo.make_mel_targets(dur, 80, seed=302)
    model = ref_shim.reference_forward_transformer(cfg, p, (tok, dur[..., None].float(), pit[..., None]))
    import tensorflow as tf  # the shim
    model._compile(optimizer=tf.keras.optimizers.Adam(1e-4, beta_1=0.9, beta_2=0.98, epsilon=1e-9))
    named = ref_shim.ft_named_parameters(model, cfg)
    out = model.train_step(tok, mel_tgt, dur, pit)
    JS['train/step'] = int(model.step)
    JS['train/loss'] = float(out['loss'])
    for k in ('mel', 'duration', 'pitch'):
        JS['train/losses/' + k] = float(out['losses'][k])
    JS['train/params'] = sorted(named)
    for name, var in named.items():
        put('train/grad/' + name, model.optimizer._slots[id(var)][0] / (1.0 - 0.9), 24)
        put('train/var/' + name, var.detach(), 24)

    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    tok, mel, stop = alo.make_aligner_inputs(cfg, 3, 20, 49, seed=503)
    for r in (1, 2):
        model = ref_shim.reference_aligner(dict(cfg, dropout_rate=0.0, decoder_prenet_dropout=0.0), p, (tok, mel[:, :-1]))
        model._compile(stop_scaling=cfg['stop_loss_scaling'], optimizer=tf.keras.optimizers.Adam(1e-4, beta_1=0.9, beta_2=0.98, epsilon=1e-9))
        model.set_constants(reduction_factor=r, force_decoder_diagonal=True, force_encoder_diagonal=True)
        with torch.no_grad():
            ref = model.val_step(tok, mel, stop)
        k = f'aln/{r}/'
        for n in ('mel', 'stop_prob', 'linear'):
            put(k + n, ref[n], 512)
        for side in ('encoder_attention', 'decoder_attention'):
            JS[k + side] = sorted(ref[side])
            for name in ref[side]:
                put(k + side + '/' + name, ref[side][name], 128)
        JS[k + 'loss'] = float(ref['loss'])
        for n in ('mel', 'stop_prob', 'diag_loss'):
            JS[k + 'losses/' + n] = float(ref['losses'][n])

    from model import transformer_utils as ref_tu
    for n, d in PE_CASES:
        put(f'pe/{n}/{d}', ref_tu.positional_encoding(n, d), 1024)
    seq = torch.tensor([[3, 7, 0, 0], [1, 0, 0, 0]], dtype=torch.int32)
    put('mask/encoder_padding', ref_tu.create_encoder_padding_mask(seq))
    m = torch.zeros(2, 5, 3)
    m[0, :4] = 1.0
    m[1, :2] = -2.0
    put('mask/mel_padding', ref_tu.create_mel_padding_mask(m))
    put('mask/look_ahead', ref_tu.create_look_ahead_mask(7))

    from utils import scheduling as ref_s
    JS['sched/lr'] = [float(ref_s.piecewise_linear_schedule(s, LR_SCHED)) for s in LR_STEPS]
    JS['sched/red'] = [int(ref_s.reduction_schedule(s, RED_SCHED)) for s in RED_STEPS]
    JS['sched/red_below_first'] = int(ref_s.reduction_schedule(5, [[10, 7], [20, 3]]))

    from utils import losses as ref_l
    from utils import spectrogram_ops as ref_ops
    from ref_shim import spec_inputs
    mel, ph, tgt, pred, logits, targets = spec_inputs(SPEC_SEED)
    JS['spec/mel_lengths'] = [int(v) for v in ref_ops.mel_lengths(mel).tolist()]
    JS['spec/phoneme_lengths'] = [int(v) for v in ref_ops.phoneme_lengths(ph).tolist()]
    JS['spec/mae'] = float(ref_l.masked_mean_absolute_error(tgt, pred))
    tot, vals = ref_l.weighted_sum_losses((tgt, tgt), (pred, pred * 2), [ref_l.masked_mean_absolute_error] * 2, [1., 3.])
    JS['spec/weighted_total'] = float(tot)
    JS['spec/weighted_vals'] = [float(v) for v in vals]
    JS['spec/scaled_ce'] = float(ref_l.new_scaled_crossentropy(index=2, scaling=8.0)(targets, logits))

    import tempfile
    from data import metadata_readers as ref_mr
    from data.text.symbols import all_phonemes
    from data.text.tokenizer import Tokenizer as RefTok
    with tempfile.TemporaryDirectory() as td:
        meta = Path(td) / 'metadata.csv'
        meta.write_text(META_TEXT, encoding='utf-8')
        JS['meta/ljspeech'] = ref_mr.ljspeech(str(meta))
        text, up = ref_mr.post_processed_reader(str(meta))
        JS['meta/post_text'], JS['meta/post_up'] = text, up
    JS['tok/all_phonemes'] = list(all_phonemes)
    rng = np.random.default_rng(0)
    for se, br in TOKENIZER_MODES:
        t = RefTok(add_start_end=se, model_breathing=br)
        k = f'tok/{int(se)}{int(br)}/'
        JS[k + 'vocab_size'] = int(t.vocab_size)
        strs = [''.join(rng.choice(all_phonemes, size=int(rng.integers(1, 40)))) for _ in range(20)]
        JS[k + 'strings'] = strs
        JS[k + 'encoded'] = [[int(v) for v in t(s)] for s in strs]
        JS[k + 'decoded'] = [t.decode(t(s)) for s in strs]
    JS['tok/alphabet'] = [int(v) for v in RefTok(alphabet='abc xyz')('a cab')]

    for cfg_name in ('C1', 'LJ256'):
        cfg = fo.CONFIGS[cfg_name]
        p = fo.init_params(cfg, seed=7)
        tok, dur, pit = fo.make_inputs('ragged', 2, 16, 60, seed=5)
        ref = ref_shim.reference_forward_transformer(cfg, p, (tok, dur[..., None].float(), pit[..., None]))
        ident = {id(v): k for k, v in ref_shim.ft_named_parameters(ref, cfg).items()}
        JS[f'order/{cfg_name}'] = [[layer.name, [ident[id(v)] for v in layer.variables if id(v) in ident]] for layer in ref.layers]
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    tok, mel, _ = alo.make_aligner_inputs(cfg, 2, 12, 21, seed=3)
    ref = ref_shim.reference_aligner(cfg, p, (tok, mel[:, :-1]))
    ident = {id(v): k for k, v in ref_shim.aligner_named_parameters(ref, cfg).items()}
    JS['order/aligner'] = [[layer.name, [ident.get(id(v)) for v in layer.variables]] for layer in ref.layers]

    for i, (r, force_long) in enumerate(ALIGNER_PRED_CASES):
        pp = dict(p)
        if force_long:
            pp['postnet.stop.b'] = torch.tensor([6.0, 0.0, -6.0])
        c0 = dict(cfg, dropout_rate=0.0, decoder_prenet_dropout=0.0)
        ref = ref_shim.reference_aligner(c0, pp, (tok, mel[:, :-1]))
        ref._set_r(r)
        with torch.no_grad():
            o_ref = ref.predict(tok[0], max_length=10, encode=False, verbose=False)
        k = f'apred/{i}/'
        JS[k + 'start'] = float(ref.start_vec[0, 0])
        JS[k + 'stop_prob_index'] = int(ref.stop_prob_index)
        put(k + 'mel', o_ref['mel'])
        put(k + 'attention', o_ref['decoder_attention']['Decoder_LastBlock_CrossAttention'])

    np.savez_compressed(HERE / 'ref_shim.npz', **ARR)
    (HERE / 'ref_shim.json').write_text(json.dumps(JS, sort_keys=True) + '\n')


if __name__ == '__main__':
    main()
