"""Pins the oracle to the reference's OWN code.  The unmodified reference sources were executed on top of tests/tf_shim (a
torch-backed stand-in for the TensorFlow/Keras primitives) by tests/golden/make_golden_shim.py, and what they returned is
stored in tests/golden/ref_shim.{npz,json} (large arrays as a fixed, seeded sample of their elements).  These tests
recompute the same cases with oracle/*.py and the host-side mirrors in transformertts_b200/ and compare.
"""
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import ref_shim  # noqa: E402
from ref_shim import expect  # noqa: E402
from oracle import aligner_oracle as alo  # noqa: E402
from oracle import forward_oracle as fo  # noqa: E402

import pytest  # noqa: E402


def _js():
    return ref_shim.golden()[1]


# ----------------------------------------------------------------------------------------------------------------------
# the reference's own known answers (its tests/test_loss.py) and what its loss code returned for them
# ----------------------------------------------------------------------------------------------------------------------
def test_reference_own_loss_test_passes_on_the_shim():
    js = _js()
    # the constants asserted by the reference's tests/test_loss.py, reproduced by its code on the shim ...
    assert js['loss/scaled5'] == pytest.approx(2.3705523014068604, abs=1e-7)
    assert js['loss/scaled1'] == pytest.approx(0.7679619193077087, abs=1e-7)
    assert js['loss/masked'] == pytest.approx(0.7679619193077087, abs=1e-7)
    # ... and by the oracle's restatement
    targets = torch.tensor([[0, 1, 2]])
    logits = torch.tensor([[[.3, .2, .1], [.3, .2, .1], [.3, .2, .1]]], dtype=torch.float64)
    assert float(alo.new_scaled_crossentropy(targets, logits, index=2, scaling=5.0)) == pytest.approx(js['loss/scaled5'], abs=1e-6)
    assert float(alo.new_scaled_crossentropy(targets, logits, index=2, scaling=1.0)) == pytest.approx(js['loss/scaled1'], abs=1e-6)


def test_expand_docstring_example_through_reference_code():
    """model/layers.py:532-542: the reference's Expand layer (ragged-tensor construction) on its own docstring example."""
    x = torch.tensor([[[0.54710746, 0.8943467], [0.7140938, 0.97968304], [0.5347662, 0.15213418]]])
    want = x[0][[0, 1, 1, 1, 2, 2]][None]
    expect('expand', want)
    assert torch.equal(fo.expand(x, torch.tensor([[[1.], [3.], [2.]]])), want)


# ----------------------------------------------------------------------------------------------------------------------
# ForwardTransformer: reference model code vs the oracle
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cfg_name,B,Tp,Tm,seed', ref_shim.CASES)
def test_forward_transformer_call_matches_oracle(cfg_name, B, Tp, Tm, seed):
    cfg = fo.CONFIGS[cfg_name]
    p = fo.init_params(cfg, seed=7)
    tok, dur, pit = fo.make_inputs('ragged', B, Tp, Tm, seed=seed)
    with torch.no_grad():
        got = fo.forward_transformer_call(p, cfg, tok, dur[..., None], pit[..., None])
    k = f'fwd/{cfg_name}/'
    js = _js()
    assert sorted(got['encoder_attention']) == js[k + 'encoder_attention']
    assert sorted(got['decoder_attention']) == js[k + 'decoder_attention']
    expect(k + 'mel', got['mel'], 2e-5)
    expect(k + 'duration', got['duration'], 1e-5)
    expect(k + 'pitch', got['pitch'], 1e-5)
    expect(k + 'expanded_mask', got['expanded_mask'])
    for side in ('encoder_attention', 'decoder_attention'):
        for name in got[side]:
            expect(k + side + '/' + name, got[side][name], 1e-5)


def test_predict_with_predicted_durations_speed_and_duration_masks():
    """model/models.py:559-595: predict() with its speed regulator and per-phoneme max / min duration tables.  Durations are
    predicted (ReLU head, then * 1/speed, min/max masks, round-half-even): the integer durations must be identical."""
    cfg = fo.CONFIGS['C1']
    p = dict(fo.init_params(cfg, seed=7))
    p['dur_pred.out.b'] = torch.tensor([3.2])   # a duration head that produces usable durations
    tok, dur, pit = fo.make_inputs('ragged', 3, 32, 160, seed=111)
    js = _js()
    tok_np = tok.numpy()
    for i, (speed, mx, mn) in enumerate(ref_shim.PRED_SETTINGS):
        mxm = np.full(tok_np.shape, np.inf, dtype=np.float32)
        mnm = np.zeros(tok_np.shape, dtype=np.float32)
        if mx:
            mxm[tok_np == js['pred/id_a']] = mx
        if mn:
            mnm[tok_np == js['pred/id_b']] = mn
        with torch.no_grad():
            got = fo.forward_transformer_call(p, cfg, tok, None, None, durations_scalar=float(np.float32(1. / speed)),
                                              max_durations_mask=torch.from_numpy(mxm), min_durations_mask=torch.from_numpy(mnm))
        assert got['mel'].shape[1] > 0
        expect(f'pred/{i}/mel', got['mel'], 5e-5)
        expect(f'pred/{i}/expanded_mask', got['expanded_mask'])


def test_train_step_of_the_reference_matches_oracle_gradients_and_adam():
    """model/models.py:464-482 run unmodified (GradientTape -> torch autograd, Keras Adam from the shim) with dropout 0:
    loss, the gradients the reference step applied and every parameter after one optimizer step == oracle loss /
    gradients / Keras-form Adam update (at the stored sample of each parameter's elements)."""
    cfg = dict(fo.CONFIGS['C1'], dropout_rate=0.0, predictors_dropout=0.0)
    p = fo.init_params(cfg, seed=7)
    tok, dur, pit = fo.make_inputs('ragged', 3, 24, 150, seed=301)
    mel_tgt = fo.make_mel_targets(dur, 80, seed=302)
    js = _js()
    assert js['train/step'] == 1
    ref_out, ref_g = fo.loss_and_grads(p, cfg, tok, mel_tgt, dur, pit)
    assert abs(js['train/loss'] - float(ref_out['loss'])) < 1e-5
    for k in ('mel', 'duration', 'pitch'):
        assert abs(js['train/losses/' + k] - float(ref_out['losses'][k])) < 1e-5
    assert js['train/params'] == sorted(ref_g)
    gscale = max(float(g.abs().max()) for g in ref_g.values())
    for name in js['train/params']:
        # gradients the reference step applied: after the first Keras-Adam step m = (1 - beta_1) * g
        expect('train/grad/' + name, ref_g[name].double(), 2e-5 * gscale)
        # the applied update, where the gradient is well above fp32 noise (Adam's first step is lr * sign(g): elements
        # whose gradient is analytically zero -- the key biases -- move by +-lr on rounding noise alone, in TF as well)
        w = p[name].clone()
        m, v = torch.zeros_like(w), torch.zeros_like(w)
        fo.adam_tf_step(w, ref_g[name].float(), m, v, 1, 1e-4)
        arrays = ref_shim.golden()[0]
        idx = torch.from_numpy(ref_shim.sample_index(w.numel(), arrays['train/var/' + name].size, 'train/var/' + name))
        var = torch.from_numpy(arrays['train/var/' + name]).double()
        live = ref_g[name].reshape(-1)[idx].double().abs() > 1e-4 * gscale
        if live.any():
            assert float(((w.reshape(-1)[idx].double() - var).abs() * live).max()) < 2e-7, name
            assert float(((var - p[name].reshape(-1)[idx].double()).abs() * live).max()) > 0.9e-4, name


# ----------------------------------------------------------------------------------------------------------------------
# Aligner (SURVEY 8f row 1): reference model code vs the oracle
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('r', [1, 2])
def test_aligner_teacher_forced_step_matches_oracle(r):
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    tok, mel, stop = alo.make_aligner_inputs(cfg, 3, 20, 49, seed=503)
    with torch.no_grad():
        got = alo.gta_forward(p, dict(cfg, dropout_rate=0.0, decoder_prenet_dropout=0.0), tok, mel, stop, r=r,
                              stop_scaling=cfg['stop_loss_scaling'], force_decoder_diagonal=True, force_encoder_diagonal=True)
    k = f'aln/{r}/'
    js = _js()
    for n in ('mel', 'stop_prob', 'linear'):
        expect(k + n, got[n], 5e-5)
    for side in ('encoder_attention', 'decoder_attention'):
        assert sorted(got[side]) == js[k + side]
        for name in got[side]:
            expect(k + side + '/' + name, got[side][name], 1e-5)
    assert abs(float(got['loss']) - js[k + 'loss']) < 2e-5
    for n in ('mel', 'stop_prob', 'diag_loss'):
        assert abs(float(got['losses'][n]) - js[k + 'losses/' + n]) < 2e-5, n


# ----------------------------------------------------------------------------------------------------------------------
# host-side mirrors vs the reference modules they mirror (bit-exact where integers / float64 host maths)
# ----------------------------------------------------------------------------------------------------------------------
def test_positional_encoding_and_masks_bitwise():
    from transformertts_b200.model import transformer_utils as our_tu
    for n, d in ref_shim.PE_CASES:
        expect(f'pe/{n}/{d}', our_tu.positional_encoding(n, d))
        expect(f'pe/{n}/{d}', fo.positional_encoding(n, d))
    seq = torch.tensor([[3, 7, 0, 0], [1, 0, 0, 0]], dtype=torch.int32)
    expect('mask/encoder_padding', fo.create_encoder_padding_mask(seq))
    mel = torch.zeros(2, 5, 3)
    mel[0, :4] = 1.0
    mel[1, :2] = -2.0
    expect('mask/mel_padding', fo.create_mel_padding_mask(mel))
    expect('mask/look_ahead', alo.create_look_ahead_mask(7))


def test_scheduling_bitwise():
    from transformertts_b200.utils import scheduling as our_s
    js = _js()
    assert [our_s.piecewise_linear_schedule(s, ref_shim.LR_SCHED) for s in ref_shim.LR_STEPS] == js['sched/lr']
    assert [our_s.reduction_schedule(s, ref_shim.RED_SCHED) for s in ref_shim.RED_STEPS] == js['sched/red']
    # the reference's quirk: below the first breakpoint it returns the first STEP entry, not the first value
    assert our_s.reduction_schedule(5, [[10, 7], [20, 3]]) == js['sched/red_below_first'] == 10


def test_spectrogram_ops_and_losses():
    js = _js()
    mel, ph, tgt, pred, logits, targets = ref_shim.spec_inputs(ref_shim.SPEC_SEED)
    assert js['spec/mel_lengths'] == [6, 2, 9] and js['spec/phoneme_lengths'] == [3, 1, 5]
    assert abs(js['spec/mae'] - float(fo.masked_mean_absolute_error(tgt, pred))) < 1e-6
    v2 = float(fo.masked_mean_absolute_error(tgt, pred * 2))
    assert abs(js['spec/weighted_vals'][1] - v2) < 1e-6
    assert abs(js['spec/weighted_total'] - (js['spec/mae'] + 3 * v2)) < 1e-5
    assert abs(float(alo.new_scaled_crossentropy(targets, logits, index=2, scaling=8.0)) - js['spec/scaled_ce']) < 1e-6


def test_tokenizer_and_metadata_readers(tmp_path):
    from transformertts_b200.data import datasets as ds
    from transformertts_b200.data.text import Tokenizer
    from transformertts_b200.model.models import DEFAULT_VOCAB
    js = _js()
    assert Tokenizer(add_start_end=False, model_breathing=False).vocab_size == DEFAULT_VOCAB == js['tok/00/vocab_size']
    assert Tokenizer(add_start_end=True, model_breathing=False).vocab_size == alo.ALIGNER_VOCAB == js['tok/10/vocab_size']
    meta = tmp_path / 'metadata.csv'
    meta.write_text(ref_shim.META_TEXT, encoding='utf-8')
    as_json = lambda x: __import__('json').loads(__import__('json').dumps(x))  # noqa: E731  (tuples -> lists, as stored)
    assert as_json(ds.ljspeech(meta)) == js['meta/ljspeech']
    got_text, got_up = ds.post_processed_reader(meta)
    assert as_json(got_text) == js['meta/post_text'] and as_json(got_up) == js['meta/post_up'] and len(got_up) == 20


def test_keras_weight_order_follows_the_reference_constructors():
    """model_weights.hdf5 is matched BY ORDER (transformertts_b200/model/hdf5_weights.py): the order must be the one in
    which the reference's constructors assign layers and variables (Keras: own variables first, then tracked sub-layers in
    assignment order), as walked on the reference classes themselves through the shim's Layer tracking."""
    from transformertts_b200.model import hdf5_weights as hw
    from transformertts_b200.model.models import ForwardTransformer
    js = _js()
    for cfg_name in ('C1', 'LJ256'):
        got = js[f'order/{cfg_name}']
        ours = ForwardTransformer(**fo.CONFIGS[cfg_name], device='cpu')
        want = [(lname, [flat for _, flat in ws]) for lname, ws in hw.keras_layer_order(ours)]
        assert [g[1] for g in got] == [w[1] for w in want]
        # the explicitly named layers keep their names; the two unnamed Dense layers get counter-based names in TF
        assert [g[0] for g in got if g[0][0].isupper() or '_pred' in g[0] or g[0] == 'expand'] == \
            ['Embedding', 'Encoder', 'dur_pred', 'expand', 'pitch_pred', 'Decoder']


def test_tokenizer_mirror_equals_reference_tokenizer():
    from transformertts_b200.data.text import ALL_PHONEMES, Tokenizer
    js = _js()
    assert list(ALL_PHONEMES) == js['tok/all_phonemes']
    for se, br in ref_shim.TOKENIZER_MODES:
        a = Tokenizer(add_start_end=se, model_breathing=br)
        k = f'tok/{int(se)}{int(br)}/'
        assert a.vocab_size == js[k + 'vocab_size']
        for s, enc, dec in zip(js[k + 'strings'], js[k + 'encoded'], js[k + 'decoded']):
            assert list(a(s)) == enc
            assert a.decode(a(s)) == dec
    assert list(Tokenizer(alphabet='abc xyz')('a cab')) == js['tok/alphabet']


def test_keras_weight_order_of_the_aligner():
    from transformertts_b200.model import hdf5_weights as hw
    from transformertts_b200.model.aligner import Aligner
    cfg = alo.ALIGNER_CONFIGS['A-small']
    ours = Aligner.from_config(dict(cfg, device='cpu'), max_r=cfg['max_r'])
    want = [[flat for _, flat in ws] for _, ws in hw.keras_layer_order(ours)]
    got = _js()['order/aligner']
    assert [g[1] for g in got] == want          # includes DecoderPrenet's non-trainable rate variable (None) in last position
    assert [g[0] for g in got] == ['Embedding', 'Encoder', 'DecoderPrenet', 'Decoder', 'FinalProj', 'Postnet']


@pytest.mark.parametrize('r,force_long', ref_shim.ALIGNER_PRED_CASES)
def test_aligner_autoregressive_predict_matches_oracle(r, force_long):
    """Aligner.predict (models.py:271-292, encode=False) of the UNMODIFIED reference against oracle.aligner_predict: same number
    of iterations (stop decision) and the same frames.  force_long biases the stop head so the loop runs to max_length."""
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    if force_long:
        p = dict(p)
        p['postnet.stop.b'] = torch.tensor([6.0, 0.0, -6.0])
    tok, mel, _ = alo.make_aligner_inputs(cfg, 2, 12, 21, seed=3)
    c0 = dict(cfg, dropout_rate=0.0, decoder_prenet_dropout=0.0)
    k = f'apred/{ref_shim.ALIGNER_PRED_CASES.index((r, force_long))}/'
    js = _js()
    o = alo.aligner_predict(p, c0, tok[0], js[k + 'start'], max_length=10, r=r, stop_prob_index=js[k + 'stop_prob_index'])
    if force_long:
        assert o['mel'].shape[0] == (10 // r + 1) * r
    expect(k + 'mel', o['mel'], 1e-5)
    expect(k + 'attention', o['decoder_attention']['Decoder_LastBlock_CrossAttention'], 1e-5)
