"""CPU tests of the cached autoregressive decode (Aligner.predict_batch): the C-ABI argument checks of its three entry points,
and the causality argument it rests on, checked in float64 on the oracle -- a decode loop that keeps each self-attention
block's keys and values and computes one new row per iteration gives the rows of the reference's loop, which re-runs the
whole decoder on the whole prefix every iteration (oracle/aligner_oracle.py:aligner_predict)."""
import ctypes as C
import math
import re
from pathlib import Path

import pytest
import torch

from oracle import aligner_oracle as alo
from oracle import forward_oracle as fo

ROOT = Path(__file__).resolve().parent.parent

# Inputs of the GPU batch tests (tests/test_gpu_aligner_decode.py) whose rows stop at DIFFERENT iterations: A-small, oracle
# weights of seed 7 with this stop-head bias, the token rows of make_aligner_inputs(A-small, 3, 14, 8, seed=STOP_SEED) at
# r = 1 and max_length = STOP_MAX_LENGTH.  The rows stop after STOP_ITERS iterations, and at every iteration of every row
# the arg-max of the last stop distribution leads the runner-up by at least STOP_MARGIN in logit, so the GPU's rounding
# cannot flip a stop decision.  test_different_stop_constants re-derives all of it.
STOP_BIAS = (0.0, 0.0, -0.55)
STOP_SEED = 9
STOP_MAX_LENGTH = 24
STOP_ITERS = (5, 2, 4)
STOP_MARGIN = 0.05


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


# ---------------------------------------------------------------------------------------------------------------------
# C ABI: argument validation without a GPU (every check runs before any CUDA call)
# ---------------------------------------------------------------------------------------------------------------------
def _attn_args(lib, dh=64, self_mode=True):
    a = lib.DecodeAttnArgs()
    a.B, a.H, a.dh = 2, 4, dh
    fake = C.c_void_p(0x100000)   # never dereferenced: validation fails or passes before any launch
    a.q, a.ld_q, a.q_col0 = fake, 3 * 4 * dh, 0
    a.kv, a.ld_kv, a.Tk, a.k_col0, a.v_col0 = fake, 2 * 4 * dh, 10, 0, 4 * dh
    if self_mode:
        a.new_kv, a.ld_new, a.new_k_col0, a.new_v_col0 = fake, 3 * 4 * dh, 4 * dh, 8 * dh
    else:
        a.kv_len = fake
    a.pos, a.out_hi, a.ld_out = fake, fake, 4 * dh
    a.precision = lib.PREC_FP16
    a.workspace, a.workspace_bytes = fake, 1 << 30
    return a


def test_decode_attn_argument_validation(cdll):
    from transformertts_b200 import lib
    assert cdll.ttsb_decode_attn(None, None) == -1
    assert b'NULL' in cdll.ttsb_last_error()
    a = _attn_args(lib)
    a.q = None
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -1
    assert b'NULL' in cdll.ttsb_last_error()
    a = _attn_args(lib, self_mode=False)
    a.kv_len = None                      # cross mode needs the key lengths
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -1
    a = _attn_args(lib, dh=96)
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -3
    assert b'head size 96' in cdll.ttsb_last_error()
    a = _attn_args(lib)
    a.precision = lib.PREC_BF16X3
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -3
    a = _attn_args(lib)
    a.B = 0
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -1
    a = _attn_args(lib)
    a.ld_kv = 2 * 4 * 64 + 4               # not a multiple of 8
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -1
    a = _attn_args(lib)
    a.v_col0 = 8 * 64                      # V columns run past the row
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -1
    a = _attn_args(lib)
    a.workspace_bytes = cdll.ttsb_decode_attn_workspace_bytes(2, 4, 64) - 1
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -1
    assert b'workspace' in cdll.ttsb_last_error()
    a = _attn_args(lib)
    a.probs, a.probs_T = C.c_void_p(0x100000), 0
    assert cdll.ttsb_decode_attn(C.byref(a), None) == -1
    # the workspace grows with B*H*dh
    assert 0 < lib.decode_attn_workspace_bytes(1, 1, 64) < lib.decode_attn_workspace_bytes(16, 4, 64)
    assert lib.decode_attn_workspace_bytes(0, 4, 64) == 0


def test_decode_prologue_and_commit_argument_validation(cdll):
    fake = C.c_void_p(0x100000)
    eps = C.c_float(1e-6)
    assert cdll.ttsb_decode_prologue(None, fake, fake, fake, fake, 10, fake, 2, 256, eps, fake, fake, fake, None) == -1
    assert b'ttsb_decode_prologue' in cdll.ttsb_last_error()
    assert cdll.ttsb_decode_prologue(fake, fake, fake, fake, fake, 10, fake, 2, 254, eps, fake, fake, fake, None) == -1
    assert cdll.ttsb_decode_prologue(fake, fake, fake, fake, fake, 0, fake, 2, 256, eps, fake, fake, fake, None) == -1
    assert cdll.ttsb_decode_commit(None, 96, 2, 1, 80, 80, 2, 10, fake, None, fake, fake, 128, fake, fake, fake, fake, None) == -1
    assert b'ttsb_decode_commit' in cdll.ttsb_last_error()
    # stop_col inside the mel columns / rows too short for the stop logits / stop_index out of range / next input too narrow
    assert cdll.ttsb_decode_commit(fake, 96, 2, 1, 80, 40, 2, 10, fake, None, fake, fake, 128, fake, fake, fake, fake, None) == -1
    assert cdll.ttsb_decode_commit(fake, 82, 2, 1, 80, 80, 2, 10, fake, None, fake, fake, 128, fake, fake, fake, fake, None) == -1
    assert cdll.ttsb_decode_commit(fake, 96, 2, 1, 80, 80, 3, 10, fake, None, fake, fake, 128, fake, fake, fake, fake, None) == -1
    assert cdll.ttsb_decode_commit(fake, 96, 2, 1, 80, 80, 2, 10, fake, None, fake, fake, 64, fake, fake, fake, fake, None) == -1
    assert cdll.ttsb_decode_commit(fake, 96, 2, 0, 80, 80, 2, 10, fake, None, fake, fake, 128, fake, fake, fake, fake, None) == -1


def test_decode_attn_struct_layout_matches_header():
    from transformertts_b200 import lib
    header = (ROOT / 'include' / 'ttsb.h').read_text()
    body = re.search(r'typedef struct ttsb_decode_attn_args \{(.*?)\} ttsb_decode_attn_args;', header, re.S).group(1)
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    fields = [re.findall(r'([A-Za-z_][A-Za-z0-9_]*)\s*$', part.strip())[0]
              for decl in body.split(';') if decl.strip() for part in decl.split(',')]
    assert fields == [f[0] for f in lib.DecodeAttnArgs._fields_]


def test_predict_batch_rejects_bad_inputs_before_any_gpu_work():
    from transformertts_b200.model.aligner import Aligner
    with pytest.raises(ValueError):
        Aligner._token_batch([[5, 0, 6]])            # pad id inside a row
    with pytest.raises(ValueError):
        Aligner._token_batch(torch.zeros((2,), dtype=torch.int32))
    with pytest.raises(ValueError):
        Aligner._token_batch([[]])
    t = Aligner._token_batch([[3, 4, 5], [7]])
    assert t.tolist() == [[3, 4, 5], [7, 0, 0]] and t.dtype == torch.int32


# ---------------------------------------------------------------------------------------------------------------------
# The causality argument in float64: a cached decode loop equals the reference's re-run loop
# ---------------------------------------------------------------------------------------------------------------------
def _attend(q, k, v, heads, n_valid=None):
    """Scaled dot-product attention of query rows q (1, Tq, d) over keys / values (1, Tk, d) (layers.py:176-195); keys >= n_valid
    get the reference's additive -1e9 mask.  Returns (output (1, Tq, d), weights (1, H, Tq, Tk))."""
    _, Tq, d = q.shape
    Tk, depth = k.shape[1], d // heads

    def split(t):
        return t.reshape(1, -1, heads, depth).permute(0, 2, 1, 3)

    logits = split(q) @ split(k).transpose(-1, -2) / math.sqrt(float(depth))
    if n_valid is not None:
        logits = logits + (torch.arange(Tk) >= n_valid).to(logits.dtype) * fo.NEG_MASK
    w = torch.softmax(logits, dim=-1)
    return (w @ split(v)).permute(0, 2, 1, 3).reshape(1, Tq, d), w


def cached_decode(p, cfg, tok, start_value, max_length, r, stop_prob_index=2):
    """Aligner.predict restated with a key/value cache: the encoder and every cross-attention K|V once, then ONE decoder row
    per iteration -- prenet and prologue of the new frame at position it*r, self-attention of the new row over the cached
    rows 0..it, cross-attention, FFN, FinalProj, postnet -- and the returned rows accumulated."""
    mel_ch = int(cfg['mel_channels'])
    d = int(cfg['decoder_model_dimension'])
    tok = tok.reshape(1, -1)
    padding_mask = fo.create_encoder_padding_mask(tok)
    rate = 0.0
    enc_stack = {'num_heads': list(cfg['encoder_num_heads']), 'dense_blocks': len(cfg['encoder_num_heads']), 'dropout': rate,
                 'pe': fo.positional_encoding(int(cfg['encoder_max_position_encoding']), int(cfg['encoder_model_dimension']))}
    enc, enc_attn = fo.self_attention_blocks(p, 'encoder', enc_stack, p['embedding'][tok.long()], padding_mask, False, None)
    n_tok = int((tok != 0).sum())
    pe = fo.positional_encoding(int(cfg['decoder_max_position_encoding']), d)[0].to(enc.dtype)
    heads = list(cfg['decoder_num_heads'])
    keys = ['Decoder_LastBlock_CrossAttention' if i == len(heads) - 1 else f'Decoder_DenseBlock{i + 1}_CrossAttention'
            for i in range(len(heads))]
    cross_kv = [(fo.dense(enc, p[f'decoder.b{i}.ca.wk.w'], p[f'decoder.b{i}.ca.wk.b']),
                 fo.dense(enc, p[f'decoder.b{i}.ca.wv.w'], p[f'decoder.b{i}.ca.wv.b'])) for i in range(len(heads))]
    cache_k, cache_v = [[] for _ in heads], [[] for _ in heads]
    frame = torch.full((1, 1, mel_ch), float(start_value), dtype=enc.dtype)
    mels, stops, maps = [], [], {k: [] for k in keys}
    for it in range(int(max_length // r) + 1):
        x = alo.decoder_prenet(p, frame, 0.0, False, None)
        x = fo.layer_norm(x, p['decoder.ln.gamma'], p['decoder.ln.beta']) + p['decoder.pos_scalar'] * pe[it * r]
        for i, nh in enumerate(heads):
            pre = f'decoder.b{i}.'
            cache_k[i].append(fo.dense(x, p[pre + 'sa.wk.w'], p[pre + 'sa.wk.b']))
            cache_v[i].append(fo.dense(x, p[pre + 'sa.wv.w'], p[pre + 'sa.wv.b']))
            q = fo.dense(x, p[pre + 'sa.wq.w'], p[pre + 'sa.wq.b'])
            a, _ = _attend(q, torch.cat(cache_k[i], dim=1), torch.cat(cache_v[i], dim=1), nh)
            a1 = fo.layer_norm(fo.dense(torch.cat([x, a], -1), p[pre + 'sa.wo.w'], p[pre + 'sa.wo.b']) + x,
                               p[pre + 'sa.ln.gamma'], p[pre + 'sa.ln.beta'])
            q2 = fo.dense(a1, p[pre + 'ca.wq.w'], p[pre + 'ca.wq.b'])
            c, w = _attend(q2, cross_kv[i][0], cross_kv[i][1], nh, n_valid=n_tok)
            maps[keys[i]].append(w)
            a2 = fo.layer_norm(fo.dense(torch.cat([a1, c], -1), p[pre + 'ca.wo.w'], p[pre + 'ca.wo.b']) + a1,
                               p[pre + 'ca.ln.gamma'], p[pre + 'ca.ln.beta'])
            h = fo.dense(fo.dense(a2, p[pre + 'ffn1.w'], p[pre + 'ffn1.b'], 'relu'), p[pre + 'ffn2.w'], p[pre + 'ffn2.b'])
            x = fo.layer_norm(h + a2, p[pre + 'ln2.gamma'], p[pre + 'ln2.beta'])
        linear = fo.dense(x, p['final_proj.w'], p['final_proj.b'])[:, :, :r * mel_ch].reshape(1, r, mel_ch)
        mel = fo.dense(linear, p['postnet.mel.w'], p['postnet.mel.b'])
        stop = fo.dense(linear, p['postnet.stop.w'], p['postnet.stop.b'])
        mels.append(mel[0])
        stops.append(stop[0])
        frame = mel[:, -1:]
        if int(torch.argmax(stop[0, -1])) == stop_prob_index:
            break
    return {'mel': torch.cat(mels), 'stop_prob': torch.cat(stops), 'decoder_attention': {k: torch.cat(v, dim=2) for k, v in maps.items()},
            'encoder_attention': enc_attn}


@pytest.mark.parametrize('r', [1, 2, 10])
@pytest.mark.parametrize('stop_bias', [(6.0, 0.0, -6.0), (-6.0, 0.0, 6.0)])
def test_cached_decode_equals_reference_loop_fp64(r, stop_bias):
    torch.set_num_threads(4)
    cfg = dict(alo.ALIGNER_CONFIGS['A-small'], max_r=10)   # FinalProj wide enough for r = 10
    p = alo.init_aligner_params(cfg, seed=7, dtype=torch.float64)
    p['postnet.stop.b'] = torch.tensor(stop_bias, dtype=torch.float64)
    tok, _, _ = alo.make_aligner_inputs(cfg, 1, 12, 8, seed=3)
    max_length = {1: 9, 2: 12, 10: 30}[r]
    got = cached_decode(p, cfg, tok[0], 0.5, max_length, r)
    ref = alo.aligner_predict(p, dict(cfg, dropout_rate=0.0, decoder_prenet_dropout=0.0), tok[0], 0.5, max_length=max_length, r=r)
    n_iter = max_length // r + 1 if stop_bias[0] > 0 else 1
    assert got['mel'].shape == ref['mel'].shape == (n_iter * r, 80)
    assert float((got['mel'] - ref['mel']).abs().max()) < 1e-10
    assert float((got['stop_prob'] - ref['stop_prob'][0]).abs().max()) < 1e-10
    assert set(got['decoder_attention']) == set(ref['decoder_attention'])
    for k, w in ref['decoder_attention'].items():
        assert got['decoder_attention'][k].shape == w.shape
        assert float((got['decoder_attention'][k] - w).abs().max()) < 1e-10, k


def test_different_stop_constants():
    """The committed inputs of the GPU batch tests: the rows stop at different iterations, and every stop decision of every
    iteration is clear by STOP_MARGIN in logit (checked on the float32 oracle, which is what the GPU computes)."""
    torch.set_num_threads(4)
    cfg = alo.ALIGNER_CONFIGS['A-small']
    p = alo.init_aligner_params(cfg, seed=7)
    p['postnet.stop.b'] = torch.tensor(STOP_BIAS)
    tok, _, _ = alo.make_aligner_inputs(cfg, 3, 14, 8, seed=STOP_SEED)
    iters = []
    for b in range(3):
        row = tok[b][tok[b] != 0]
        out = cached_decode(p, cfg, row, 0.5, STOP_MAX_LENGTH, 1)
        lead = out['stop_prob'].sort(dim=-1, descending=True).values
        assert float((lead[:, 0] - lead[:, 1]).min()) >= STOP_MARGIN, b
        iters.append(out['mel'].shape[0])
    assert tuple(iters) == STOP_ITERS
    assert len(set(iters)) == 3
