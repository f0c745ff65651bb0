"""ForwardTransformer.predict_batch on the GPU: each line's outputs are bit for bit what predict() gives the line alone, in any
batch, at any batch size and position, eager and with CUDA graphs; the LayerNorm GEMM gives a row the same bits whichever
schedule (single CTA, CTA pair, or the hybrid of both) runs its tile; predict_tts.py end to end."""
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import forward_oracle as fo

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
FIELDS = ('mel', 'duration', 'pitch', 'int_durations')


def _model(cfg_name, precision='bf16x3', dur_bias=3.0, **kw):
    from transformertts_b200.model.models import ForwardTransformer
    cfg = fo.CONFIGS[cfg_name]
    p = fo.init_params(cfg, seed=7)
    p['dur_pred.out.b'] = torch.tensor([dur_bias])     # a few frames per phoneme from the seeded weights
    m = ForwardTransformer(**cfg, precision=precision, **kw)
    m.set_weights(p)
    return m, p


def _lines(lengths, seed):
    g = np.random.default_rng(seed)
    return [g.integers(1, fo.VOCAB_SIZE, size=n).astype(np.int32) for n in lengths]


def _alone(m, line, **kw):
    """predict() of one line, in predict_batch's output shapes."""
    o = m.predict(line, encode=False, **kw)
    T = int(o['mel_lengths'][0])
    return {'mel': o['mel'].reshape(T, m.mel_channels), 'duration': o['duration'][0], 'pitch': o['pitch'][0],
            'int_durations': o['int_durations'][0], 'mel_lengths': T}


def _assert_same(got, want, what):
    assert got['mel_lengths'] == want['mel_lengths'], what
    for f in FIELDS:
        a, b = got[f], want[f]
        assert a.shape == b.shape, (what, f, a.shape, b.shape)
        assert torch.equal(a, b), (what, f, (a.float() - b.float()).abs().max().item())


# ---- the LayerNorm GEMM: the same rows in a pair-mode launch and in single-CTA / hybrid launches
def _ln_gemm(m, N, B, x, w, res, mode, gamma, beta):
    """y = LN(x W + b + res) over B rows of 128 frames, through ForwardTransformer._gemm."""
    from transformertts_b200.model.models import _PackedLinear
    K = x.shape[-1]
    pl = _PackedLinear(w, torch.linspace(-0.1, 0.1, N, device='cuda'), [K], m._split, single_tile=True)
    assert pl.block_n == N
    hi = x[:B].to(torch.bfloat16).contiguous()
    lo = (x[:B] - hi.float()).to(torch.bfloat16).contiguous() if m._split else None
    out = torch.zeros((B, 128, N), dtype=torch.float32, device='cuda')
    kw = {}
    if mode == 'f32':
        kw['residual'] = res[:B].contiguous()
    elif mode == 'pair':
        rh = res[:B].to(torch.bfloat16).contiguous()
        kw['residual_pair'] = (rh, (res[:B] - rh.float()).to(torch.bfloat16).contiguous())
    m._gemm(pl, B, 128, [(hi, lo, K, 0)], [0], [0], ln=(gamma, beta), out_f32=out, **kw)
    return out


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('N', [128, 160, 256])
def test_layernorm_gemm_schedule_invariance(N, precision):
    m, _ = _model('C1', precision)
    m._prepare()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # 128-row tiles: 1 runs as a CTA pair, one full wave of single CTAs runs single, a full wave + 8 runs hybrid
    B_single, B_hybrid = sms, sms + 8
    g = torch.Generator(device='cpu').manual_seed(N)
    K = 192
    x = (torch.randn(B_hybrid, 128, K, generator=g) * 0.5).cuda()
    w = (torch.randn(K, N, generator=g) / K ** 0.5).cuda()
    res = (torch.randn(B_hybrid, 128, N, generator=g) + 3.0).cuda()   # an offset mean: the shifted sums matter
    gamma = (1 + 0.1 * torch.randn(N, generator=g)).cuda()
    beta = (0.1 * torch.randn(N, generator=g)).cuda()
    modes = ['none', 'f32'] + (['pair'] if precision == 'bf16x3' else [])
    for mode in modes:
        big = {B: _ln_gemm(m, N, B, x, w, res, mode, gamma, beta) for B in (B_single, B_hybrid)}
        for b in (0, 1, sms // 2, sms - 1, sms, B_hybrid - 1):
            alone = _ln_gemm(m, N, 1, x[b:b + 1], w, res[b:b + 1], mode, gamma, beta)
            for B, y in big.items():
                if b < B:
                    assert torch.equal(y[b], alone[0]), (mode, B, b, (y[b] - alone[0]).abs().max().item())


# ---- predict_batch against predict()
LENGTHS = [7, 31, 1, 18, 44, 12]


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('cfg', ['C1', 'LJ256', 'LJ256-dense', 'REF384'])
def test_matches_predict(cfg, precision):
    m, _ = _model(cfg, precision)
    lines = _lines(LENGTHS, seed=1)
    got = m.predict_batch(lines)
    assert len(got) == len(lines)
    assert sum(o['mel_lengths'] for o in got) > 0
    for i, line in enumerate(lines):
        _assert_same(got[i], _alone(m, line), (cfg, precision, i))


def test_matches_predict_with_options():
    m, _ = _model('LJ256')
    lines = _lines(LENGTHS, seed=2)
    g = np.random.default_rng(3)
    durs = [g.integers(0, 6, size=len(t)).astype(np.float32) for t in lines]
    pits = [g.standard_normal(len(t)).astype(np.float32) for t in lines]
    got = m.predict_batch(lines, phoneme_durations=durs, phoneme_pitch=pits)
    for i, line in enumerate(lines):      # forced durations and pitch
        _assert_same(got[i], _alone(m, line, phoneme_durations=durs[i][None], phoneme_pitch=pits[i][None]), ('forced', i))
    for speed in (0.9, 1.2):
        got = m.predict_batch(lines, speed_regulator=speed)
        for i, line in enumerate(lines):
            _assert_same(got[i], _alone(m, line, speed_regulator=speed), ('speed', speed, i))
    # per-phoneme max / min duration tables (symbol -> frames), as predict() looks them up through the tokenizer
    m.text_pipeline = SimpleNamespace(tokenizer=lambda s: [int(s)])
    mx, mn = {'5': 1.0, '9': 2.0, '17': 0.5}, {'3': 4.0, '11': 6.0}
    lines = [np.where(np.arange(len(t)) % 3 == 0, np.int32([5, 9, 3, 11, 17][i % 5]), t) for i, t in enumerate(lines)]
    got = m.predict_batch(lines, phoneme_max_duration=mx, phoneme_min_duration=mn)
    for i, line in enumerate(lines):
        _assert_same(got[i], _alone(m, line, phoneme_max_duration=mx, phoneme_min_duration=mn), ('tables', i))


def test_batch_invariance():
    m, _ = _model('LJ256')
    lines = _lines([9, 40, 3, 25, 25, 60, 14, 2], seed=4)
    ref = m.predict_batch(lines, batch_size=1)
    for bs in (3, 64):
        got = m.predict_batch(lines, batch_size=bs)
        for i in range(len(lines)):
            _assert_same(got[i], ref[i], ('batch_size', bs, i))
    # another position in the batch and other neighbours
    order = [5, 0, 7, 2, 6, 1, 3, 4]
    got = m.predict_batch([lines[i] for i in order] + _lines([33, 8], seed=5), batch_size=4)
    for j, i in enumerate(order):
        _assert_same(got[j], ref[i], ('permuted', i))


def test_oracle_parity():
    m, p = _model('LJ256')
    tok, dur, pit = fo.make_inputs('ragged', 5, 40, 200, seed=6)
    lens = (tok != 0).sum(1).tolist()
    lines = [tok[b, :n].numpy() for b, n in enumerate(lens)]
    got = m.predict_batch(lines, phoneme_durations=[dur[b, :n] for b, n in enumerate(lens)],
                          phoneme_pitch=[pit[b, :n] for b, n in enumerate(lens)])
    for b, n in enumerate(lens):
        ref = fo.forward_transformer_call(p, fo.CONFIGS['LJ256'], tok[b:b + 1, :n], dur[b:b + 1, :n, None].float(),
                                          pit[b:b + 1, :n, None])
        assert torch.equal(got[b]['int_durations'].cpu(), dur[b, :n]), b
        err = (got[b]['mel'].cpu() - ref['mel'][0]).abs().max().item()
        assert err < 1e-3, (b, err)


def test_cuda_graphs_match_eager_and_reuse_graphs():
    eager, _ = _model('LJ256')
    graphed, _ = _model('LJ256', cuda_graphs=True)
    g = np.random.default_rng(7)
    # two line sets with the same batch count and the same rounded shapes: Tp <= 48, frames <= 128 per line
    sets = [_lines([40, 3, 17], seed=8), _lines([33, 41, 9], seed=9)]
    durs = [[np.full(len(t), 2.0, np.float32) + g.integers(0, 2, size=len(t)) for t in s] for s in sets]
    counts = []
    for s, d in zip(sets, durs):
        want = eager.predict_batch(s, phoneme_durations=d)
        got = graphed.predict_batch(s, phoneme_durations=d)
        for i in range(len(s)):
            _assert_same(got[i], want[i], ('graphs', i))
        counts.append((len(graphed._enc_graphs), sum(len(e['dec']) for e in graphed._enc_graphs.values())))
    assert counts[0] == counts[1] == (1, 1), counts


def test_edge_lines():
    m, _ = _model('C1')
    lines = _lines([1, 20, 5, 12], seed=10)
    durs = [np.full(len(t), 3.0, np.float32) for t in lines]
    durs[2][:] = 0.0                                      # a line that expands to zero frames
    max_pos = fo.CONFIGS['C1']['decoder_max_position_encoding']
    durs[3][:] = max_pos // len(lines[3])
    durs[3][-1] += max_pos - durs[3].sum()                # a line at the decoder's position-table limit
    for graphs in (False, True):
        m.cuda_graphs = graphs
        got = m.predict_batch(lines, phoneme_durations=durs)
        assert got[2]['mel'].shape == (0, m.mel_channels)
        assert got[3]['mel_lengths'] == max_pos
        assert got[0]['mel'].shape == (3, m.mel_channels)
        for i in (0, 1, 3):
            _assert_same(got[i], _alone(m, lines[i], phoneme_durations=durs[i][None]), ('edge', graphs, i))
    # negative forced durations: the default minimum-duration mask (0) clamps them, in predict() as here
    neg = [d.copy() for d in durs[:2]]
    neg[1][::2] = -4.0
    got = m.predict_batch(lines[:2], phoneme_durations=neg)
    for i in (0, 1):
        _assert_same(got[i], _alone(m, lines[i], phoneme_durations=neg[i][None]), ('negative', i))
    assert int(got[1]['int_durations'].min()) == 0


def test_predict_tts_end_to_end(tmp_path):
    from transformertts_b200.data.text import Tokenizer
    from transformertts_b200.model.models import ForwardTransformer
    cfg = dict(fo.CONFIGS['LJ256'], sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000,
               normalizer='MelGAN', data_name='ljspeech')
    p = fo.init_params(cfg, seed=7)
    p['dur_pred.out.b'] = torch.tensor([6.0])
    model = ForwardTransformer(**cfg)
    model.set_weights(p)
    model.save_model(tmp_path / 'model', with_optimizer=False)
    lines = ['həloʊ wɜːld', 'ðɪs ɪz ɐ lɔŋɡɚ tɛst sɛntəns, ɐ lɔŋɡɚ wɜːld ðɪs ɪz.', 'ɐbɐ', 'tɛst', 'ɪz ɐ həloʊ sɛntəns', 'oʊ']
    (tmp_path / 'lines.txt').write_text('\n'.join(lines) + '\n')
    r = subprocess.run([sys.executable, str(ROOT / 'predict_tts.py'), '-p', str(tmp_path / 'model'), '-f', str(tmp_path / 'lines.txt'),
                        '-o', str(tmp_path / 'out'), '-m'], capture_output=True, text=True, timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    out = tmp_path / 'out' / 'outputs' / 'lines'
    loaded = ForwardTransformer.load_model(tmp_path / 'model')
    tok = Tokenizer(add_start_end=False, model_breathing=False, alphabet=loaded.alphabet)
    for i, line in enumerate(lines):
        mel = loaded.predict(tok(line), encode=False, phoneme_max_duration=None)['mel'].cpu().numpy()
        assert np.array_equal(np.load(out / f'lines_ljspeech_unknown_0_{i}.mel.npy'), mel), i
