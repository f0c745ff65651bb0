"""WaveRNN generator host logic without a GPU: the oracle's layer list, the composite upsampling taps, fold tables, BatchNorm
folding, the counter-based RNG, checkpoint checks, the C ABI's argument validation and the command line."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wavernn_oracle as wo
from transformertts_b200 import lib
from transformertts_b200.model import wavernn as wr


def test_parameter_counts():
    assert wo.WaveRNN(mode='MOL').num_params() == wo.N_PARAMS_MOL == 4_233_675
    assert wo.WaveRNN(mode='RAW', bits=9).num_params() == wo.N_PARAMS_RAW9 == 4_480_941


@pytest.mark.parametrize('factors,pad', [((5, 5, 11), 2), ((4, 4, 16), 2), ((2, 3), 3), ((8, 8, 4), 2)])
def test_composite_taps_equal_the_chain(factors, pad):
    rng = np.random.default_rng(sum(factors))
    half = wr.reach_frames(factors)
    assert half <= pad
    up = wo.UpsampleNetwork(80, factors, 64, 1, 64, pad).double()
    ws = []
    for i, s in enumerate(factors):
        w = torch.from_numpy(rng.standard_normal((1, 1, 1, 2 * s + 1)))
        up.up_layers[2 * i + 1].weight.data.copy_(w)
        ws.append(w.numpy())
    K = wr.composite_taps(ws, factors, half)
    hop = int(np.prod(factors))
    for T in (1, 2, 7, 50):
        m = torch.from_numpy(rng.standard_normal((1, 80, T)))
        mp = F.pad(m, (pad, pad))
        x = mp.unsqueeze(1)
        for f in up.up_layers:
            x = f(x)
        want = x.squeeze(1)[:, :, up.indent:-up.indent][0].detach().numpy()      # (80, T hop)
        mz = np.pad(m[0].numpy(), ((0, 0), (half, half)))
        got = np.zeros_like(want)
        for n in range(T * hop):
            f_, p = divmod(n, hop)
            got[:, n] = mz[:, f_:f_ + 2 * half + 1] @ K[p]
        assert np.abs(got - want).max() < 1e-12


@pytest.mark.parametrize('target,overlap', [(11000, 550), (40, 10), (33, 7), (5, 1)])
@pytest.mark.parametrize('n', [1, 2, 3])
@pytest.mark.parametrize('d', [-1, 0, 1])
def test_fold_tables_match_fatchord(target, overlap, n, d):
    total = n * (target + overlap) + overlap + d
    if total <= overlap:
        pytest.skip('no fold')
    x = torch.arange(1, total + 1, dtype=torch.float64)[None, :, None]
    folded = wo.fold_with_overlap(x, target, overlap)[:, :, 0].numpy()
    hop = 1
    rows, L = wr.fold_rows([total], hop, True, target, overlap)
    assert len(rows) == folded.shape[0] == wr.fold_count(total, target, overlap) and L == folded.shape[1]
    for (c, i, first, valid), row in zip(rows, folded):
        want = np.where(np.arange(L) < valid, first + np.arange(L) + 1, 0)
        assert np.array_equal(row, want)
    y = np.random.default_rng(1).standard_normal(folded.shape)
    want = wo.xfade_and_unfold(y.copy(), target, overlap)
    g = wr.crossfade_gains(L, overlap)
    got = np.zeros_like(want)
    for (_, i, first, _), yy in zip(rows, y):
        got[first:first + L] += yy * g
    assert np.abs(got - want).max() < 1e-15


def test_unbatched_rows():
    rows, L = wr.fold_rows([21, 30], 275, False, 11000, 550)
    assert L == 30 * 275 and rows == [(0, 0, 0, 21 * 275), (1, 0, 0, 30 * 275)]


def test_batchnorm_folding_is_exact():
    sd = wo.init_state_dict(seed=3)
    net = wo.build(sd)
    x = torch.from_numpy(np.random.default_rng(0).standard_normal((1, 80, 9)))
    with torch.no_grad():
        want = net.upsample.resnet.batch_norm(net.upsample.resnet.conv_in(x))[0].numpy()
    w, b = wr.fold_bn(sd['upsample.resnet.conv_in.weight'].numpy(), sd, 'upsample.resnet.batch_norm')
    got = F.conv1d(x, torch.from_numpy(w), torch.from_numpy(b))[0].numpy()
    assert np.abs(got - want).max() < 1e-12


def test_rng_known_answers():
    u = wo.uniforms(0, [0, 1], 0, 11)
    assert u.dtype == np.float32 and u.shape == (2, 11)
    assert np.all(u >= np.float32(1e-5)) and np.all(u <= np.float32(1) - np.float32(1e-5))
    pinned = wo.uniforms(7, [3], 12345, 3)[0]
    assert pinned.tolist() == PINNED_7_3_12345
    big = wo.uniforms(0, np.arange(64), 3, 11)
    assert abs(float(big.mean()) - 0.5) < 0.05
    # keyed by every field
    a = wo.uniforms(1, [2], 3, 4)
    for other in (wo.uniforms(2, [2], 3, 4), wo.uniforms(1, [3], 3, 4), wo.uniforms(1, [2], 4, 4)):
        assert not np.array_equal(a, other)


PINNED_7_3_12345 = [0.6189590096473694, 0.15230685472488403, 0.644137442111969]   # uniforms(seed 7, fold 3, step 12345)


def _sd(**kw):
    return wo.init_state_dict(seed=0, **kw)


def test_checkpoint_refusals_name_the_key():
    sd = _sd()
    wr.WaveRNNGenerator.check_state_dict(sd)
    bad = dict(sd)
    del bad['fc2.bias']
    with pytest.raises(KeyError, match='missing key fc2.bias'):
        wr.WaveRNNGenerator.check_state_dict(bad)
    bad = dict(sd, extra=torch.zeros(1))
    with pytest.raises(KeyError, match='unexpected key extra'):
        wr.WaveRNNGenerator.check_state_dict(bad)
    bad = dict(sd)
    bad['rnn2.bias_hh_l0'] = torch.zeros(7)
    with pytest.raises(ValueError, match='rnn2.bias_hh_l0 has shape'):
        wr.WaveRNNGenerator.check_state_dict(bad)


def test_inferred_hparams():
    h = wr.WaveRNNGenerator.check_state_dict(_sd(mode='RAW', bits=10))
    assert h['mode'] == 'RAW' and h['bits'] == 10 and h['upsample_factors'] == (5, 5, 11) and h['pad'] == 2 and h['res_blocks'] == 10
    h = wr.WaveRNNGenerator.check_state_dict(_sd(pad=3, res_blocks=2, compute_dims=64, res_out_dims=256, upsample_factors=(4, 4, 16)))
    assert (h['pad'], h['res_blocks'], h['compute_dims'], h['res_out_dims'], h['upsample_factors']) == (3, 2, 64, 256, (4, 4, 16))


@pytest.mark.parametrize('kw,match', [(dict(rnn_dims=256), 'rnn_dims'), (dict(fc_dims=384), 'fc_dims'), (dict(mode='RAW', bits=7), 'bits = 7'),
                                      (dict(mode='RAW', bits=11), 'bits = 11'), (dict(compute_dims=96), 'compute_dims'),
                                      (dict(res_out_dims=100), 'res_out_dims'), (dict(pad=1), 'pad = 1'),
                                      (dict(feat_dims=64), 'feat_dims')])
def test_unsupported_dims_are_refused(kw, match):
    with pytest.raises(ValueError, match=match):
        wr.WaveRNNGenerator.check_state_dict(_sd(**kw))


def test_short_clip_refused_by_name():
    g = wr.WaveRNNGenerator(device='cpu')
    g.h = {'upsample_factors': (5, 5, 11), 'n_classes': 30}
    with pytest.raises(ValueError, match='mel 1 has 20 frames'):
        g._generate([np.zeros((80, 21), np.float32), np.zeros((80, 20), np.float32)], None, True, 11000, 550)


# ------------------------------------------------------------------------------------------------------------ the C ABI
def _args(frames=(21, 40)):
    ftab = (C.c_int32 * len(frames))(*frames)
    stab = (C.c_uint32 * len(frames))(*range(len(frames)))
    return dict(frames=C.cast(ftab, C.c_void_p), seeds=C.cast(stab, C.c_void_p), n_clips=len(frames), hop=275, batched=1, target=11000,
                overlap=550, n_rows=len(wr.fold_rows(frames, 275, True, 11000, 550)[0]), n_taps=5, taps=0x1000, melp_hi=0x2000,
                melp_lo=0x3000, ld_melp=2048, aux_hi=0x4000, aux_lo=0x5000, ld_aux=4608, cond_halo=9,
                cond_rows=sum(frames) + 18 * len(frames), vec=0x6000, weights=0x7000, mode=lib.WAVERNN_MOL, n_classes=30,
                precision=lib.PREC_BF16X3, wav_out=0x8000, workspace=0x10000, workspace_bytes=1 << 40, _keep=(ftab, stab))


def _rc(a):
    a = dict(a)
    a.pop('_keep')
    return lib.wavernn_generate_rc(**a)


@pytest.mark.parametrize('field,value,match', [
    ('mode', 5, 'mode'), ('n_classes', 31, 'MOL takes 30'), ('precision', 9, 'precision'), ('n_rows', 3, 'n_rows'),
    ('hop', 0, 'hop'), ('target', 0, 'target'), ('overlap', 0, 'overlap'), ('n_taps', 4, 'n_taps'), ('n_taps', 9, 'n_taps'),
    ('cond_halo', 1, 'cond_halo'), ('cond_rows', 5, 'cond_rows'), ('melp_lo', None, 'lo planes'), ('ld_aux', 4096, 'ld_aux'),
    ('weights', 0x7004, '16-byte'), ('wav_out', None, 'wav_out'), ('capture_steps', 3, 'capture_steps'),
    ('workspace_bytes', 1024, 'workspace'), ('workspace', 0x10004, 'workspace'), ('samples_out', 0x9002, 'samples_out'), ('timings', 0x9004, 'timings')])
def test_abi_validation(field, value, match):
    a = _args()
    a[field] = value
    assert _rc(a) == -1
    assert match in lib.load().ttsb_last_error().decode()


def test_abi_validation_short_clip_and_raw_classes():
    a = _args(frames=(20, 40))
    a['n_rows'] = 2
    assert _rc(a) == -1 and 'clip 0 has 20 frames' in lib.load().ttsb_last_error().decode()
    a = _args()
    a.update(mode=lib.WAVERNN_RAW, n_classes=2048)
    assert _rc(a) == -1 and 'RAW takes 2^bits' in lib.load().ttsb_last_error().decode()
    with pytest.raises(lib.TtsbError):
        lib.wavernn_workspace_bytes([21], 275, True, 11000, 550, 2000)
    assert lib.wavernn_workspace_bytes([21], 275, True, 11000, 550, 30) > 0


# ------------------------------------------------------------------------------------------------------------ command line
def test_cli_parsing():
    import predict_tts
    a = predict_tts.parse_args(['-t', 'x', '--vocoder', 'wavernn', '--vocoder_checkpoint', 'latest_weights.pyt'])
    assert a.vocoder == 'wavernn' and a.vocoder_checkpoint == 'latest_weights.pyt'
    with pytest.raises(SystemExit):
        predict_tts.parse_args(['-t', 'x', '--vocoder', 'wavernn'])
    with pytest.raises(SystemExit):
        predict_tts.parse_args(['-t', 'x', '--vocoder', 'wavernn', '--vocoder_checkpoint', 'a', '--vocoder_config', 'v1'])
    import evaluate_tts
    base = ['--config', 'c.yaml', '-p', 'weights']
    a = evaluate_tts.parse_args(base + ['--vocoder', 'wavernn', '--vocoder_checkpoint', 'latest_weights.pyt'])
    assert a.vocoder == 'wavernn' and a.vocoder_checkpoint == 'latest_weights.pyt'
    with pytest.raises(SystemExit):
        evaluate_tts.parse_args(base + ['--vocoder', 'wavernn'])
    with pytest.raises(SystemExit):
        evaluate_tts.parse_args(base + ['--vocoder', 'wavernn', '--vocoder_checkpoint', 'a', '--vocoder_config', 'v1'])
