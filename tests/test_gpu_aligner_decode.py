"""GPU tests of the cached autoregressive decode (Aligner.predict_batch, csrc/decode.cu).

Every row of a batch decode is checked against the full teacher-forced decoder (Aligner.call) run on that row's own output as
its input, which holds whether or not free-running decoding drifts; against the reference-faithful loop (Aligner.predict);
against single-row decodes; graphed against eager; and the attention kernel against ttsb_mha_fwd and an fp32 reference."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from oracle import aligner_oracle as alo  # noqa: E402
from test_aligner_decode import STOP_BIAS, STOP_ITERS, STOP_MAX_LENGTH, STOP_SEED  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-3       # tests/test_gpu_aligner.py
ATT_TOL = 2e-3
DEV = torch.device('cuda:0')


def _model(cfg, params, cuda_graphs=False):
    from transformertts_b200.model.aligner import Aligner
    m = Aligner.from_config(dict(cfg), max_r=cfg['max_r'])
    m.cuda_graphs = cuda_graphs   # the constructor flag (from_config forwards a fixed set of keys that does not include it)
    m.set_weights(params)
    return m


def _rows(tokens):
    return [t[t != 0] for t in tokens]


def _stop_batch():
    """The committed different-stop inputs (tests/test_aligner_decode.py): three ragged rows that stop after STOP_ITERS."""
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    p['postnet.stop.b'] = torch.tensor(STOP_BIAS)
    tok, _, _ = alo.make_aligner_inputs(cfg, 3, 14, 8, seed=STOP_SEED)
    return cfg, p, tok


def _maxdiff(a, b):
    return float((a.float().cpu() - b.float().cpu()).abs().max())


def _check_against_call(m, rows, outs, r):
    """Test 1: each row's input is the start frame followed by its own output frames mel[r-1::r] without the last; Aligner.call
    on that input must give the row's mel, stop logits and every attention map."""
    assert len(rows) == len(outs)
    start = m.start_vec.to(DEV)
    for row, o in zip(rows, outs):
        n = o['mel'].shape[0] // r
        assert o['mel'].shape == (n * r, m.mel_channels) and o['stop_prob'].shape == (n * r, 3)
        prefix = torch.cat([start, o['mel'][r - 1::r][:-1]])[None]
        ref = m.call(row[None], prefix, training=False)
        assert _maxdiff(o['mel'], ref['mel'][0]) < TOL
        assert _maxdiff(o['stop_prob'], ref['stop_prob'][0]) < TOL
        assert set(o['decoder_attention']) == set(ref['decoder_attention'])
        for k, w in ref['decoder_attention'].items():
            assert o['decoder_attention'][k].shape == w.shape == (1, w.shape[1], n, len(row)), k
            assert _maxdiff(o['decoder_attention'][k], w) < ATT_TOL, k
        for k, w in ref['encoder_attention'].items():
            assert o['encoder_attention'][k].shape == w.shape, k
            assert _maxdiff(o['encoder_attention'][k], w) < ATT_TOL, k


@pytest.mark.parametrize('r,stop_bias,max_length', [(1, None, STOP_MAX_LENGTH), (2, (6.0, 0.0, -6.0), 20), (10, (6.0, 0.0, -6.0), 40)])
def test_rows_match_full_decoder_on_their_own_prefix(r, stop_bias, max_length):
    cfg, p, tok = _stop_batch()
    if stop_bias is not None:   # every row runs to max_length; FinalProj wide enough for r = 10
        cfg = dict(cfg, max_r=10)
        p = alo.init_aligner_params(cfg, seed=7)
        p['postnet.stop.b'] = torch.tensor(stop_bias)
    m = _model(cfg, p)
    m.set_constants(reduction_factor=r)
    rows = _rows(tok)
    outs = m.predict_batch(rows, max_length=max_length)
    want = STOP_ITERS if stop_bias is None else (max_length // r + 1,) * 3
    assert tuple(o['mel'].shape[0] // r for o in outs) == want
    _check_against_call(m, rows, outs, r)


@pytest.mark.parametrize('r,stop_bias', [(1, (6.0, 0.0, -6.0)), (2, (6.0, 0.0, -6.0)), (2, (-6.0, 0.0, 6.0)), (10, (6.0, 0.0, -6.0))])
def test_matches_predict(r, stop_bias):
    """The stop biases of test_aligner_autoregressive_predict (tests/test_gpu_aligner.py) plus r = 10: same length, mel within
    that test's bound."""
    cfg = dict(alo.ALIGNER_CONFIGS['A-small'], max_r=10)
    p = alo.init_aligner_params(cfg, seed=7)
    p['postnet.stop.b'] = torch.tensor(stop_bias)
    tok, _, _ = alo.make_aligner_inputs(cfg, 2, 12, 21, seed=3)
    m = _model(cfg, p)
    m.set_constants(reduction_factor=r)
    ref = m.predict(tok[0], max_length=12, encode=False, verbose=False)
    [got] = m.predict_batch([tok[0]], max_length=12)
    a, b = got['mel'].cpu(), ref['mel'].float().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert float((a - b).abs().max()) < 5e-3 * max(1.0, float(b.abs().max()))
    for k, w in ref['decoder_attention'].items():
        assert got['decoder_attention'][k].shape == w.shape
    for k, w in ref['encoder_attention'].items():
        assert _maxdiff(got['encoder_attention'][k], w) < ATT_TOL


def test_batch_matches_single_rows():
    """A ragged batch whose rows stop at different iterations: every row has its single-row length and outputs (not bit-exact:
    the LayerNorm GEMMs pick single-CTA or CTA-pair tiles by row count)."""
    cfg, p, tok = _stop_batch()
    m = _model(cfg, p)
    m.set_constants(reduction_factor=1)
    rows = _rows(tok)
    outs = m.predict_batch(rows, max_length=STOP_MAX_LENGTH)
    assert tuple(o['mel'].shape[0] for o in outs) == STOP_ITERS
    assert m.decode_stats['steps'] == 8 and m.decode_stats['host_reads'] == 2   # one all-done read after 8 steps, one final
    for row, o in zip(rows, outs):
        [s] = m.predict_batch([row], max_length=STOP_MAX_LENGTH)
        assert s['mel'].shape == o['mel'].shape
        assert _maxdiff(s['mel'], o['mel']) < TOL and _maxdiff(s['stop_prob'], o['stop_prob']) < TOL
        for k, w in s['decoder_attention'].items():
            assert w.shape == o['decoder_attention'][k].shape and _maxdiff(w, o['decoder_attention'][k]) < TOL, k
    # a padded (B, Tp) array gives the same rows as the ragged list
    padded = m.predict_batch(tok, max_length=STOP_MAX_LENGTH)
    for a, b in zip(padded, outs):
        assert torch.equal(a['mel'], b['mel'])


@pytest.mark.parametrize('sync_every', [1, 8])
def test_graphed_equals_eager(sync_every, monkeypatch):
    from transformertts_b200.model import aligner as aligner_mod
    monkeypatch.setattr(aligner_mod, '_DECODE_SYNC_EVERY', sync_every)
    cfg, p, tok = _stop_batch()
    rows = _rows(tok)
    eager, graphed = _model(cfg, p), _model(cfg, p, cuda_graphs=True)
    res = []
    for m in (eager, graphed, graphed):       # the second graphed call replays the cached capture
        m.set_constants(reduction_factor=1)
        res.append(m.predict_batch(rows, max_length=STOP_MAX_LENGTH))
        # the longest row stops after 5 iterations: K = 1 reads after each of 5 steps, K = 8 once after 8; plus the final read
        assert (m.decode_stats['steps'], m.decode_stats['host_reads']) == {1: (5, 6), 8: (8, 2)}[sync_every]
    assert len(graphed._decode_graphs) == 1
    for other in res[1:]:
        for a, b in zip(res[0], other):
            assert torch.equal(a['mel'], b['mel']) and torch.equal(a['stop_prob'], b['stop_prob'])
            for k in a['decoder_attention']:
                assert torch.equal(a['decoder_attention'][k], b['decoder_attention'][k]), k
    assert tuple(o['mel'].shape[0] for o in res[0]) == STOP_ITERS


# ---------------------------------------------------------------------------------------------------------------------
# kernel level
# ---------------------------------------------------------------------------------------------------------------------
def _workspace(B, H, dh):
    from transformertts_b200 import lib
    return torch.zeros((lib.decode_attn_workspace_bytes(B, H, dh),), dtype=torch.uint8, device=DEV)


def _decode_attn(q, ld_q, kv, ld_kv, Tk, pos, H, dh, prec, ws, kv_len=None, new=None, probs=None, done=None):
    from transformertts_b200 import lib
    B, d = pos.shape[0], H * dh
    out_hi = torch.zeros((B, d), dtype=torch.bfloat16, device=DEV)
    out_lo = torch.zeros_like(out_hi)
    a = lib.DecodeAttnArgs()
    a.B, a.H, a.dh = B, H, dh
    a.q, a.ld_q, a.q_col0 = q.data_ptr(), ld_q, 0
    a.kv, a.ld_kv, a.Tk, a.k_col0, a.v_col0 = kv.data_ptr(), ld_kv, Tk, 0, d
    if new is not None:
        a.new_kv, a.ld_new, a.new_k_col0, a.new_v_col0 = new.data_ptr(), new.shape[-1], d, 2 * d
    else:
        a.kv_len = kv_len.data_ptr()
    a.pos = pos.data_ptr()
    a.done = done.data_ptr() if done is not None else None
    a.out_hi, a.out_lo, a.ld_out = out_hi.data_ptr(), out_lo.data_ptr(), d
    if probs is not None:
        a.probs, a.probs_T = probs.data_ptr(), probs.shape[2]
    a.precision = prec
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    lib.decode_attn(a)
    torch.cuda.synchronize()
    return out_hi.float() + out_lo.float()


def _ref_attention(q, k, v, lens, H, dh):
    """fp32: q (B, d), k / v (B, Tk, d), keys < lens[b] -> out (B, d), probs (B, H, Tk)."""
    B, Tk = k.shape[:2]
    qh = q.float().reshape(B, H, 1, dh)
    kh = k.float().reshape(B, Tk, H, dh).permute(0, 2, 1, 3)
    vh = v.float().reshape(B, Tk, H, dh).permute(0, 2, 1, 3)
    logits = (qh @ kh.transpose(-1, -2))[:, :, 0] / dh ** 0.5
    mask = torch.arange(Tk, device=q.device)[None, :] >= lens[:, None]
    logits = logits + mask[:, None, :].float() * -1e9
    w = torch.softmax(logits, -1)
    return (w[:, :, None] @ vh)[:, :, 0].reshape(B, H * dh), w


@pytest.mark.parametrize('dh', [64, 128, 256])
@pytest.mark.parametrize('B,prec', [(3, 'fp16'), (3, 'bf16'), (150, 'fp16')])
def test_decode_attn_cross_mode(dh, B, prec):
    """Against ttsb_mha_fwd on the same buffers (T = 1, cross mode) and an fp32 reference; key lengths 1, lengths that are not a
    multiple of the key split, and the full Tk.  B = 150 runs one CTA per (b, h), B = 3 splits the keys across CTAs."""
    from transformertts_b200 import lib
    g = torch.Generator(device='cpu').manual_seed(dh + B)
    H, Tk = 2, 333
    d = H * dh
    dt = torch.float16 if prec == 'fp16' else torch.bfloat16
    pc = lib.PREC_FP16 if prec == 'fp16' else lib.PREC_BF16
    q = torch.randn((B, d), generator=g).to(DEV, dt)
    kv = torch.randn((B, Tk, 2 * d), generator=g).to(DEV, dt)
    lens = torch.randint(1, Tk + 1, (B,), generator=g, dtype=torch.int32)
    lens[:3] = torch.tensor([1, 200, Tk], dtype=torch.int32)
    lens = lens.to(DEV)
    pos = torch.randint(0, 5, (B,), generator=g, dtype=torch.int32).to(DEV)
    probs = torch.full((B, H, 5, Tk), -1.0, device=DEV)
    ws = _workspace(B, H, dh)
    out = _decode_attn(q, d, kv, 2 * d, Tk, pos, H, dh, pc, ws, kv_len=lens, probs=probs)
    again = _decode_attn(q, d, kv, 2 * d, Tk, pos, H, dh, pc, ws, kv_len=lens)   # the workspace is left ready for reuse
    assert torch.equal(out, again)
    assert int(ws[:B * H * 4].view(torch.int32).count_nonzero()) == 0   # split counters back at zero
    ref_o, ref_w = _ref_attention(q, kv[..., :d], kv[..., d:], lens, H, dh)
    assert float((out - ref_o).abs().max()) < 2e-3 * max(1.0, float(ref_o.abs().max()))
    got_w = probs[torch.arange(B, device=DEV), :, pos.long()]           # (B, H, Tk)
    assert float((got_w - ref_w).abs().max()) < 1e-5
    assert bool((probs.sum(-1) == -Tk).sum() == B * H * 4)               # only row pos[b] was written
    # ttsb_mha_fwd, T = 1 cross mode, over the same buffers
    m = lib.MhaArgs()
    o_hi = torch.zeros((B, 1, d), dtype=torch.bfloat16, device=DEV)
    o_lo = torch.zeros_like(o_hi)
    w_all = torch.empty((B, H, 1, Tk), device=DEV)
    m.B, m.T, m.H, m.dh = B, 1, H, dh
    m.qk_hi, m.ld_qk, m.q_col0, m.k_col0, m.v_col0 = q.data_ptr(), d, 0, 0, d
    m.kv_hi, m.ld_kv, m.Tk = kv.data_ptr(), 2 * d, Tk
    m.kv_len, m.out_hi, m.out_lo, m.ld_out = lens.data_ptr(), o_hi.data_ptr(), o_lo.data_ptr(), d
    m.full_queries, m.weights_out, m.weights_all = 1, w_all.data_ptr(), 1
    m.precision, m.impl = pc, lib.IMPL_TCGEN05
    lib.mha_fwd(m)
    torch.cuda.synchronize()
    assert float((out - (o_hi.float() + o_lo.float())[:, 0]).abs().max()) < 4e-3 * max(1.0, float(ref_o.abs().max()))
    assert float((got_w - w_all[:, :, 0]).abs().max()) < 1e-5


@pytest.mark.parametrize('dh', [64, 128, 256])
def test_decode_attn_self_mode(dh):
    """The new row's K,V land in the cache at pos[b] bit for bit; the query attends over keys 0..pos[b]; rows marked done are
    left alone."""
    from transformertts_b200 import lib
    g = torch.Generator(device='cpu').manual_seed(100 + dh)
    B, H, Tmax = 4, 2, 201
    d = H * dh
    qkv = torch.randn((B, 3 * d), generator=g).to(DEV, torch.float16)
    cache = torch.randn((B, Tmax, 2 * d), generator=g).to(DEV, torch.float16)
    before = cache.clone()
    pos = torch.tensor([0, 7, 130, Tmax - 1], dtype=torch.int32, device=DEV)
    done = torch.tensor([0, 0, 1, 0], dtype=torch.int32, device=DEV)
    probs = torch.zeros((B, H, Tmax, Tmax), device=DEV)
    out = _decode_attn(qkv, 3 * d, cache, 2 * d, Tmax, pos, H, dh, lib.PREC_FP16, _workspace(B, H, dh), new=qkv, probs=probs, done=done)
    expect = before.clone()
    for b in (0, 1, 3):
        expect[b, int(pos[b])] = qkv[b, d:]
    assert torch.equal(cache, expect)                     # bit for bit, and nothing else written (row 2 is done)
    lens = pos + 1
    ref_o, ref_w = _ref_attention(qkv[:, :d], cache[..., :d], cache[..., d:], lens, H, dh)
    live = torch.tensor([0, 1, 3], device=DEV)
    assert float((out[live] - ref_o[live]).abs().max()) < 2e-3 * max(1.0, float(ref_o.abs().max()))
    assert float(out[2].abs().max()) == 0.0
    got_w = probs[torch.arange(B, device=DEV), :, pos.long()]
    assert float((got_w[live] - ref_w[live]).abs().max()) < 1e-5
    assert float(probs[2].abs().max()) == 0.0


def test_shipped_a5_dimensions_graphed():
    """aligner_settings as shipped (d = 256, decoder heads [4, 4, 4, 4, 1]: head sizes 64 and 256) through the graphed path,
    B = 4 ragged rows and max_length = 200, each row against the full decoder on its own prefix."""
    cfg = alo.ALIGNER_CONFIGS['A5']
    p = alo.init_aligner_params(cfg, seed=7)
    p['postnet.stop.b'] = torch.tensor((6.0, 0.0, -6.0))
    tok, _, _ = alo.make_aligner_inputs(cfg, 4, 50, 8, seed=500)
    m = _model(cfg, p, cuda_graphs=True)
    m.set_constants(reduction_factor=1)
    rows = _rows(tok)
    outs = m.predict_batch(rows, max_length=200)
    assert len(m._decode_graphs) == 1
    assert all(o['mel'].shape[0] == 201 for o in outs)
    assert outs[0]['decoder_attention']['Decoder_LastBlock_CrossAttention'].shape == (1, 1, 201, len(rows[0]))
    _check_against_call(m, rows, outs, 1)


def test_decode_attn_workspace_reused_across_steps():
    """One workspace over consecutive self-mode calls of the same B and H, as the decode steps use it: B*H = 80 counters
    (beyond the first 256 bytes), ragged and growing positions, so the number of CTAs that combine changes from call to call.
    Every call matches the fp32 reference and leaves the counters at zero."""
    from transformertts_b200 import lib
    g = torch.Generator(device='cpu').manual_seed(7)
    B, H, dh, Tmax = 20, 4, 64, 300
    d = H * dh
    ws = _workspace(B, H, dh)
    cache = torch.randn((B, Tmax, 2 * d), generator=g).to(DEV, torch.float16)
    start = torch.randint(0, 40, (B,), generator=g, dtype=torch.int32)
    for step in (0, 1, 60, 150, 259):
        pos = (start + step).to(DEV)
        qkv = torch.randn((B, 3 * d), generator=g).to(DEV, torch.float16)
        out = _decode_attn(qkv, 3 * d, cache, 2 * d, Tmax, pos, H, dh, lib.PREC_FP16, ws, new=qkv)
        ref_o, _ = _ref_attention(qkv[:, :d], cache[..., :d], cache[..., d:], pos + 1, H, dh)
        assert float((out - ref_o).abs().max()) < 2e-3 * max(1.0, float(ref_o.abs().max())), step
        assert int(ws[:B * H * 4].view(torch.int32).count_nonzero()) == 0, step


def test_shipped_a5_batch_of_32():
    """A5 (decoder heads [4, 4, 4, 4, 1]) at B = 32: the blocks with four heads and the last block with one use attention
    workspaces of different layouts; every row against the full decoder on its own prefix, graphed and eager alike."""
    cfg = alo.ALIGNER_CONFIGS['A5']
    p = alo.init_aligner_params(cfg, seed=7)
    p['postnet.stop.b'] = torch.tensor((6.0, 0.0, -6.0))
    tok, _, _ = alo.make_aligner_inputs(cfg, 32, 40, 8, seed=501)
    rows = _rows(tok)
    outs = {}
    for graphs in (False, True):
        m = _model(cfg, p, cuda_graphs=graphs)
        m.set_constants(reduction_factor=1)
        outs[graphs] = m.predict_batch(rows, max_length=30)
    assert all(o['mel'].shape[0] == 31 for o in outs[True])
    for a, b in zip(outs[False], outs[True]):
        assert torch.equal(a['mel'], b['mel'])
    _check_against_call(m, rows, outs[True], 1)
