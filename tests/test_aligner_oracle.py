"""CPU tests of the Aligner restatement (oracle/aligner_oracle.py): the reference's own known answers for the stop-token
cross entropy (tests/test_loss.py of the reference), the look-ahead mask, an independent torch implementation of the
teacher-forced forward, and the committed golden vectors."""
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import aligner_oracle as alo
from oracle import forward_oracle as fo

GOLD = Path(__file__).parent / 'golden'


def test_scaled_crossentropy_reference_known_answers():
    # reference tests/test_loss.py:12-24
    targets = torch.tensor([[0, 1, 2]])
    logits = torch.tensor([[[.3, .2, .1], [.3, .2, .1], [.3, .2, .1]]])
    assert abs(float(alo.new_scaled_crossentropy(targets, logits, index=2, scaling=5)) - 2.3705523014068604) < 1e-6
    assert abs(float(alo.new_scaled_crossentropy(targets, logits, index=2, scaling=1)) - 0.7679619193077087) < 1e-6


def test_look_ahead_mask_is_strict_upper_triangle():
    m = alo.create_look_ahead_mask(5)
    assert torch.equal(m, torch.triu(torch.ones(5, 5), diagonal=1))


def test_diagonal_mask_values_and_padding():
    m = alo.diagonal_mask(4, 2, (6, 3))
    assert m.shape == (6, 3)
    assert torch.all(m[4:] == 0) and torch.all(m[:, 2:] == 0)
    # |i/max_n - j/max_m| : (j=3, i=0) -> 0.75 ; (j=0, i=1) -> 0.5
    assert abs(float(m[3, 0]) - 0.75) < 1e-7 and abs(float(m[0, 1]) - 0.5) < 1e-7


def _independent_mha(p, pre, q_in, kv, attn_mask_bool, H):
    """stock torch ops only: F.linear + scaled_dot_product_attention with a boolean keep-mask."""
    B, Tq, d = q_in.shape
    dh = d // H
    q = F.linear(q_in, p[pre + 'wq.w'].T, p[pre + 'wq.b']).view(B, Tq, H, dh).transpose(1, 2)
    k = F.linear(kv, p[pre + 'wk.w'].T, p[pre + 'wk.b']).view(B, -1, H, dh).transpose(1, 2)
    v = F.linear(kv, p[pre + 'wv.w'].T, p[pre + 'wv.b']).view(B, -1, H, dh).transpose(1, 2)
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=attn_mask_bool)
    o = o.transpose(1, 2).reshape(B, Tq, d)
    return F.linear(torch.cat([q_in, o], -1), p[pre + 'wo.w'].T, p[pre + 'wo.b'])


def _independent_aligner(p, cfg, tokens, targets, r):
    B, Tp = tokens.shape
    T = targets.shape[1]
    d_enc, d_dec = cfg['encoder_model_dimension'], cfg['decoder_model_dimension']
    key_keep = (tokens != 0)[:, None, None, :]
    x = F.layer_norm(p['embedding'][tokens.long()], (d_enc,), p['encoder.ln.gamma'], p['encoder.ln.beta'], 1e-6)
    x = x + p['encoder.pos_scalar'] * fo.positional_encoding(cfg['encoder_max_position_encoding'], d_enc)[:, :Tp]
    keep_rows = (tokens != 0)[..., None].float()
    for i, H in enumerate(cfg['encoder_num_heads']):
        pre = f'encoder.b{i}.'
        y = F.layer_norm(_independent_mha(p, pre, x, x, key_keep, H) + x, (d_enc,), p[pre + 'ln1.gamma'], p[pre + 'ln1.beta'], 1e-6) * keep_rows
        h = F.linear(F.relu(F.linear(y, p[pre + 'ffn1.w'].T, p[pre + 'ffn1.b'])), p[pre + 'ffn2.w'].T, p[pre + 'ffn2.b'])
        x = F.layer_norm(h + y, (d_enc,), p[pre + 'ln2.gamma'], p[pre + 'ln2.beta'], 1e-6) * keep_rows
    enc = x
    frame_keep = (targets.abs().sum(-1) != 0)
    causal = torch.tril(torch.ones(T, T, dtype=torch.bool))
    self_keep = frame_keep[:, None, None, :] & causal[None, None]
    h = F.relu(F.linear(targets, p['prenet.d1.w'].T, p['prenet.d1.b']))
    h = F.relu(F.linear(h, p['prenet.d2.w'].T, p['prenet.d2.b']))
    x = F.layer_norm(h, (d_dec,), p['decoder.ln.gamma'], p['decoder.ln.beta'], 1e-6)
    x = x + p['decoder.pos_scalar'] * fo.positional_encoding(cfg['decoder_max_position_encoding'], d_dec)[:, :T * r:r]
    for i, H in enumerate(cfg['decoder_num_heads']):
        pre = f'decoder.b{i}.'
        a1 = F.layer_norm(_independent_mha(p, pre + 'sa.', x, x, self_keep, H) + x, (d_dec,), p[pre + 'sa.ln.gamma'], p[pre + 'sa.ln.beta'], 1e-6)
        a2 = F.layer_norm(_independent_mha(p, pre + 'ca.', a1, enc, key_keep, H) + a1, (d_dec,), p[pre + 'ca.ln.gamma'], p[pre + 'ca.ln.beta'], 1e-6)
        f = F.linear(F.relu(F.linear(a2, p[pre + 'ffn1.w'].T, p[pre + 'ffn1.b'])), p[pre + 'ffn2.w'].T, p[pre + 'ffn2.b'])
        x = F.layer_norm(f + a2, (d_dec,), p[pre + 'ln2.gamma'], p[pre + 'ln2.beta'], 1e-6)
    mel = cfg['mel_channels']
    lin = F.linear(x, p['final_proj.w'].T, p['final_proj.b'])[..., :r * mel].reshape(B, T * r, mel)
    return F.linear(lin, p['postnet.mel.w'].T, p['postnet.mel.b']), F.linear(lin, p['postnet.stop.w'].T, p['postnet.stop.b'])


@pytest.mark.parametrize('r', [1, 2])
def test_oracle_matches_independent_torch_implementation(r):
    torch.set_num_threads(4)
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    tokens, mel, _ = alo.make_aligner_inputs(cfg, 3, 20, 48, seed=501)
    tgt = mel[:, 0::r]
    out = alo.aligner_call(p, cfg, tokens, tgt, r=r)
    mel2, stop2 = _independent_aligner(p, cfg, tokens, tgt, r)
    assert (out['mel'] - mel2).abs().max() < 2e-4
    assert (out['stop_prob'] - stop2).abs().max() < 2e-4
    # output contract (models.py:150-153, 297): names and shapes
    assert set(out['decoder_attention']) == {'Decoder_DenseBlock1_CrossAttention', 'Decoder_LastBlock_CrossAttention'}
    assert out['decoder_attention']['Decoder_LastBlock_CrossAttention'].shape == (3, 1, tgt.shape[1], 20)
    assert set(out['encoder_attention']) == {'Encoder_DenseBlock1_SelfAttention', 'Encoder_DenseBlock2_SelfAttention'}
    assert out['mel'].shape == (3, tgt.shape[1] * r, 80) and out['stop_prob'].shape == (3, tgt.shape[1] * r, 3)
    # attention rows are distributions; masked keys get (numerically) zero weight
    w = out['decoder_attention']['Decoder_DenseBlock1_CrossAttention']
    assert (w.sum(-1) - 1).abs().max() < 1e-5
    n1 = int((tokens[1] != 0).sum())
    assert w[1, :, :, n1:].abs().max() < 1e-12


def test_gta_forward_losses_and_diagonal_terms():
    torch.set_num_threads(4)
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    tokens, mel, stop = alo.make_aligner_inputs(cfg, 2, 16, 33, seed=502)
    out = alo.gta_forward(p, cfg, tokens, mel, stop, r=1, stop_scaling=8.0)
    assert abs(float(out['loss']) - float(out['losses']['mel'] + out['losses']['stop_prob'])) < 1e-6
    out_d = alo.gta_forward(p, cfg, tokens, mel, stop, r=1, force_decoder_diagonal=True, force_encoder_diagonal=True)
    d = float(out_d['losses']['diag_loss'])
    assert d > 0
    # norm factor = 1 + number of decoder maps + number of encoder maps (models.py:188-206)
    dec = sum(float((w * alo.batch_diagonal_mask(w, (1 - out_d['mel_mask'][:, 0, 0]).sum(1),
                                                (1 - out_d['text_mask'][:, 0, 0]).sum(1))).sum((-2, -1)).mean()) / 10 for w in out_d['decoder_attention'].values())
    enc = sum(float((w * alo.batch_diagonal_mask(w, (1 - out_d['text_mask'][:, 0, 0]).sum(1), (1 - out_d['text_mask'][:, 0, 0]).sum(1))).sum((-2, -1)).mean()) / 10
              for w in out_d['encoder_attention'].values())
    assert abs(d - (dec + enc) / (1 + 2 + 2)) < 1e-6


def test_golden_aligner_vectors():
    g = np.load(GOLD / 'aligner_small.npz')
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    tokens, mel, stop = alo.make_aligner_inputs(cfg, int(g['B']), int(g['Tp']), int(g['Tm']), seed=int(g['seed']))
    out = alo.gta_forward(p, cfg, tokens, mel, stop, r=1, force_decoder_diagonal=True)
    assert np.abs(out['mel'].numpy() - g['mel']).max() < 1e-4
    assert np.abs(out['stop_prob'].numpy() - g['stop_prob']).max() < 1e-4
    assert np.abs(out['decoder_attention']['Decoder_LastBlock_CrossAttention'].numpy() - g['last_attention']).max() < 1e-5
    assert abs(float(out['loss']) - float(g['loss'])) < 1e-5


def test_duration_path_search_dp_equals_scipy_dijkstra():
    """The reference finds the monotonic path with scipy's Dijkstra on an explicit graph (utils/alignments.py:21-91); the CUDA
    kernel runs the equivalent dynamic programme.  Both restated in oracle/alignment_oracle.py and compared here."""
    from oracle import alignment_oracle as ao
    rng = np.random.default_rng(0)
    shapes = []
    for _ in range(25):
        M = int(rng.integers(5, 50))
        shapes.append((M, int(rng.integers(3, min(M, 20) + 1))))
    # more phonemes than frames (the path moves right inside rows), one row, one column, more columns than the 256 threads
    # of the kernel's anti-diagonal loop
    shapes += [(7, 30), (20, 45), (1, 9), (1, 2), (12, 1), (2, 1), (2, 300), (40, 257)]
    for M, N in shapes:
        logits = rng.normal(0, 1, (M, N)) - 0.3 * N * np.abs(np.arange(M)[:, None] / M - np.arange(N)[None, :] / N)
        a = np.exp(logits)
        a = (a / a.sum(1, keepdims=True)).astype(np.float32)
        d_ref = ao.extract_durations_with_dijkstra(a)
        assert d_ref.sum() == M and np.array_equal(d_ref, ao.durations_by_dynamic_programming(a)), (M, N)
    # M = N = 1: the reference's path walk follows the source's predecessor (-9999) and fails; the DP answers [1]
    with pytest.raises(IndexError):
        ao.extract_durations_with_dijkstra(np.ones((1, 1), np.float32))
    assert ao.durations_by_dynamic_programming(np.ones((1, 1), np.float32)).tolist() == [1]


def test_vectorised_duration_dp_equals_the_loop():
    """tests/test_gpu_duration_edges.py runs the DP over anti-diagonals (the large maps would take minutes as a Python double
    loop): on small maps, random and plateau alike, it equals oracle/alignment_oracle.py's loop bit for bit."""
    from oracle import alignment_oracle as ao
    import test_gpu_duration_edges as gde
    rng = np.random.default_rng(1)
    maps = list(gde.plateau_maps().values())
    for M, N in [(1, 1), (1, 7), (9, 1), (5, 5), (13, 40), (40, 13)]:
        maps.append(gde.diagonal_maps(rng, 1, 1, M, N)[0, 0])
        maps.append(np.round(rng.uniform(0, 1, (M, N)) * 3).astype(np.float32) / 3)   # few levels: many exact ties
    for a in maps:
        assert np.array_equal(gde.dp_durations(a), ao.durations_by_dynamic_programming(a)), a.shape


def test_duration_edge_inputs_tell_wrong_oracles_apart():
    """The exact assertions of tests/test_gpu_duration_edges.py would catch three plausible mistakes: each wrong variant of
    the reference changes the result on at least one of that file's inputs (those that need no GPU-computed scores)."""
    import test_gpu_duration_edges as gde
    cases = {**gde.hand_scored_cases(), **gde.plateau_cases()}
    right = {k: gde.durations_reference(*c) for k, c in cases.items()}

    def changed(**variant):
        return [k for k, c in cases.items() if not np.array_equal(right[k], gde.durations_reference(*c, **variant))]

    assert changed(start=0)                          # cropping from row / column 0 instead of 1
    assert 'tied_heads' in changed(argmax=gde.last_argmax)   # the best head by the last maximum
    assert changed(order='uld')                      # tie order up before left
    # the last maximum also changes the jumpiness of the score inputs (uniform, zero and tied rows)
    for Tq, Tk, H, r in gde.SCORE_SHAPES:
        if Tq > 2000:
            continue
        att, ml, pl = gde.make_score_inputs(Tq, Tk, H, seed=Tq * 7 + Tk)
        right_jump = gde.scores_reference(att, ml, pl, r)[0]
        wrong_jump = gde.scores_reference(att, ml, pl, r, argmax=gde.last_argmax)[0]
        if Tk > 6:
            assert not np.array_equal(right_jump, wrong_jump), (Tq, Tk, H, r)
