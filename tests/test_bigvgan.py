"""CPU tests of the BigVGAN vocoder's host side: the oracle's op-by-op activation against the closed form the kernel computes,
the Kaiser-sinc filter, the parameter counts and key set, the config and checkpoint checks, the C-ABI refusals of
ttsb_snake_aa_ex / ttsb_conv1d_out_clamp_ex, and the scripts' flags and vocoder refusals."""
import ctypes as C
import json
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import bigvgan_oracle as bo
from transformertts_b200 import lib
from transformertts_b200.model import bigvgan as bg

SMALL = dict(bg.PRESETS['base'], upsample_initial_channel=32, resblock_kernel_sizes=[3, 5],
             resblock_dilation_sizes=[[1, 3, 5], [1, 2]])


def closed_form(x, alpha, inv_beta, h_up, h_down):
    """include/ttsb.h's ttsb_snake_aa_ex for one clip x (C, L), written from its index formulas with plain loops."""
    Cc, L = x.shape
    u = np.zeros((Cc, 2 * L))
    for m in range(2 * L):
        for i in range(L + 10):
            tap = m + 15 - 2 * i
            if 0 <= tap <= 11:
                u[:, m] += x[:, min(max(i - 5, 0), L - 1)] * h_up[tap]
    u *= 2.0
    s = u + inv_beta[:, None] * np.sin(alpha[:, None] * u) ** 2
    y = np.zeros((Cc, L))
    for t in range(L):
        for j in range(12):
            y[:, t] += h_down[j] * s[:, min(max(2 * t + j - 5, 0), 2 * L - 1)]
    return y


def test_oracle_activation_matches_the_closed_form():
    rng = np.random.default_rng(1)
    Cc = 6
    act = bo.Activation1d(bo.SnakeBeta(Cc, alpha_logscale=True)).double()
    la, lb = rng.uniform(-3, 3, Cc), rng.uniform(-3, 3, Cc)
    act.act.alpha.data, act.act.beta.data = torch.from_numpy(la), torch.from_numpy(lb)
    alpha, inv_beta = bg.snake_params(dict(snake_logscale=True), la, lb)
    f = act.upsample.filter.reshape(-1).numpy()
    assert np.array_equal(f, act.downsample.lowpass.filter.reshape(-1).numpy())
    lengths = list(range(1, 41)) + [int(n) for n in rng.integers(41, 501, 6)] + [500]
    for L in lengths:
        x = np.clip(8.0 * rng.standard_normal((Cc, L)), -30, 30)
        x[0, 0], x[1, -1] = 30.0, -30.0          # the clamped edges
        with torch.no_grad():
            got = act(torch.from_numpy(x)[None])[0].numpy()
        want = closed_form(x, alpha, inv_beta, f, f)
        assert got.shape == (Cc, L)
        # relative to the output's scale: alpha u reaches ~1000 rad, where one ulp of u moves sin^2 by ~1e-13 absolute
        assert np.abs(got - want).max() < 1e-13 * np.abs(want).max(), L


def test_snake_is_snakebeta_with_beta_alpha():
    rng = np.random.default_rng(2)
    x = torch.from_numpy(rng.standard_normal((1, 4, 9)))
    for log in (True, False):
        a = rng.uniform(-1, 1, 4) if log else np.exp(rng.uniform(-1, 1, 4))
        s = bo.Snake(4, alpha_logscale=log).double()
        s.alpha.data = torch.from_numpy(a)
        alpha, inv_beta = bg.snake_params(dict(snake_logscale=log), a, None)
        want = x.numpy() + inv_beta[None, :, None] * np.sin(alpha[None, :, None] * x.numpy()) ** 2
        with torch.no_grad():
            assert np.abs(s(x).numpy() - want).max() < 1e-14
        b = rng.uniform(-1, 1, 4) if log else np.exp(rng.uniform(-1, 1, 4))
        sb = bo.SnakeBeta(4, alpha_logscale=log).double()
        sb.alpha.data, sb.beta.data = torch.from_numpy(a), torch.from_numpy(b)
        alpha, inv_beta = bg.snake_params(dict(snake_logscale=log), a, b)
        want = x.numpy() + inv_beta[None, :, None] * np.sin(alpha[None, :, None] * x.numpy()) ** 2
        with torch.no_grad():
            assert np.abs(sb(x).numpy() - want).max() < 1e-14


def test_kaiser_sinc_filter():
    f = bo.kaiser_sinc_filter1d(0.25, 0.3, 12)
    assert f.shape == (1, 1, 12) and f.dtype == torch.float64
    f = f.reshape(-1).numpy()
    assert np.abs(f - f[::-1]).max() == 0 and abs(f.sum() - 1) < 1e-15
    A = 2.285 * (6 - 1) * np.pi * (4 * 0.3) + 7.95
    assert 50 < A < 52
    w = np.kaiser(12, 0.1102 * (A - 8.7))
    want = 2 * 0.25 * w * np.sinc(2 * 0.25 * (np.arange(-6, 6) + 0.5))
    assert np.abs(f - want / want.sum()).max() < 1e-15


@pytest.mark.parametrize('v', ['base', 'bigvgan'])
def test_parameter_counts(v):
    n = bo.n_params(v)
    assert n == bo.N_PARAMS[v] and round(n / 1e6) == {'base': 14, 'bigvgan': 112}[v]
    if v == 'base':     # the layer-list count equals the module's (weight norm folded: weight_g is not counted)
        g = bo.Generator(bo.config(v))
        assert sum(p.numel() for k, p in g.named_parameters() if not k.endswith('.weight_g')) == n
    assert bg.PRESETS[v] == dict(bo.CONFIGS[v], sampling_rate=22050, hop_size=256, fmax=8000)


def _folded(h, sd):
    g = bo.build(h, sd)
    for m in g.modules():
        if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
            torch.nn.utils.remove_weight_norm(m)
    return g.state_dict()


@pytest.mark.parametrize('final', ['v1', 'v2'])
@pytest.mark.parametrize('act', ['snakebeta', 'snake'])
def test_oracle_keys_match_the_key_table(final, act):
    h = dict(SMALL, activation=act, num_mels=100)
    if final == 'v2':
        h.update(use_tanh_at_final=False, use_bias_at_final=False)
    c = bg.load_config(h)
    sd = bo.init_state_dict(h, seed=3)
    assert {k: tuple(t.shape) for k, t in sd.items()} == bg.expected_keys(c, True)
    assert {k: tuple(t.shape) for k, t in _folded(h, sd).items()} == bg.expected_keys(c, False)
    assert ('conv_post.bias' in sd) == (final == 'v1')
    assert 'ups.3.0.weight_v' in sd and 'resblocks.7.activations.3.downsample.lowpass.filter' in sd
    assert bo.n_params(h) == sum(t.numel() for k, t in _folded(h, sd).items() if not k.endswith('.filter'))


def test_stage_columns():
    assert bg.stage_cols(bg.load_config('bigvgan')) == [1536, 768, 512, 256, 128, 64, 64]   # 384, 192, 96, 48, 24 padded
    assert bg.stage_cols(bg.load_config('base')) == [512, 256, 128, 64, 64]
    fl = bg.conv_flops(bg.load_config('bigvgan'), 10)
    assert 0.5 < fl['useful'] / fl['issued'] < 0.7
    assert [bg.launches_per_call(bg.load_config(v)) for v in ('base', 'bigvgan')] == [152, 226]
    assert bg.halo_rows(bg.load_config('base')) == 25


def test_config_sources_and_refusals(tmp_path):
    path = tmp_path / 'config.json'
    path.write_text(json.dumps(dict(bo.CONFIGS['base'], batch_size=32, segment_size=8192, sampling_rate=22050, hop_size=256,
                                    fmax=8000, use_cqtd_instead_of_mrd=True)))
    assert bg.load_config(path) == bg.load_config('BASE')
    assert bg.load_config(bg.load_config('bigvgan')) == bg.load_config('bigvgan')
    h = bg.load_config(dict(bo.CONFIGS['base']))
    assert h['use_tanh_at_final'] and h['use_bias_at_final'] and h['audio'] == {'num_mels': 80}
    for bad, text in ((dict(resblock='2'), "resblock '2' is not supported"),
                      (dict(upsample_rates=[8, 8, 2, 4], upsample_kernel_sizes=[16, 16, 4, 8]), 'not the hop of 256'),
                      (dict(upsample_kernel_sizes=[16, 16, 4, 3]), 'kernel = 2 rate'),
                      (dict(upsample_rates=[8, 8, 4, 1], upsample_kernel_sizes=[16, 16, 8, 2]), 'even rate'),
                      (dict(resblock_kernel_sizes=[3, 7, 15], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 10]]), 'exceeds 64'),
                      (dict(num_mels=129), 'num_mels = 129'),
                      (dict(activation='leakyrelu'), "activation must be 'snake' or 'snakebeta'"),
                      (dict(resblock_kernel_sizes=[3, 7, 17]), 'at most 16'),
                      (dict(upsample_rates=[8, 8, 2]), 'equal length')):
        with pytest.raises(ValueError, match=re.escape(text)):
            bg.load_config(dict(bo.CONFIGS['base'], **bad))
    h = dict(bo.CONFIGS['base'])
    del h['snake_logscale']
    with pytest.raises(ValueError, match='missing key snake_logscale'):
        bg.load_config(h)
    with pytest.raises(FileNotFoundError, match='config.json'):
        bg.BigVGANGenerator.from_checkpoint(tmp_path / 'sub' / 'g.pt')


def test_audio_settings_are_checked_by_key():
    h = bg.load_config('base')
    bg.check_audio(h, 22050, 80, 256, 8000)
    for args, key in (((24000, 80, 256, 8000), 'sampling_rate'), ((22050, 100, 256, 8000), 'num_mels'),
                      ((22050, 80, 300, 8000), 'hop_size'), ((22050, 80, 256, None), 'fmax')):
        with pytest.raises(ValueError, match=key):
            bg.check_audio(h, *args)
    h = bg.load_config(dict(bo.CONFIGS['base'], sampling_rate=24000, fmax=None))
    bg.check_audio(h, 24000, 80, 256, None)
    bg.check_audio(h, 24000, 80, 256, 12000)


@pytest.fixture(scope='module')
def small_sd():
    return bo.init_state_dict(SMALL, seed=4)


@pytest.mark.parametrize('wrapped', [False, True])
@pytest.mark.parametrize('normed', [False, True])
def test_checkpoint_loads_in_all_forms(tmp_path, small_sd, wrapped, normed):
    state = small_sd if normed else _folded(SMALL, small_sd)
    torch.save({'generator': state} if wrapped else state, tmp_path / 'g.pt')
    g = bg.BigVGANGenerator(SMALL, device='cpu')
    got = g.fold_state_dict(torch.load(tmp_path / 'g.pt', map_location='cpu', weights_only=True))
    want = g.fold_state_dict(small_sd)
    assert set(got) == set(want)
    for k in want:
        assert np.abs(got[k] - want[k]).max() < 1e-12, k
    w = _folded(SMALL, small_sd)
    for name in bg.layer_shapes(g.h):
        assert np.abs(want[name] - w[name + '.weight'].numpy()).max() < 1e-12, name
    a = 'resblocks.3.activations.2'
    alpha, inv_beta = np.exp(w[a + '.act.alpha'].numpy()), 1 / (np.exp(w[a + '.act.beta'].numpy()) + 1e-9)
    assert np.array_equal(want[a + '.alpha'], alpha) and np.array_equal(want[a + '.inv_beta'], inv_beta)
    assert np.array_equal(want[a + '.h_up'], bo.kaiser_sinc_filter1d(0.25, 0.3, 12).reshape(-1).numpy())


def test_bad_keys_are_refused_by_name(small_sd):
    g = bg.BigVGANGenerator(SMALL, device='cpu')
    bad = dict(small_sd)
    del bad['resblocks.4.convs2.1.weight_v']
    with pytest.raises(KeyError, match=r'missing key resblocks\.4\.convs2\.1\.weight_v'):
        g.fold_state_dict(bad)
    bad = dict(small_sd)
    del bad['activation_post.act.beta']
    with pytest.raises(KeyError, match=r'missing key activation_post\.act\.beta'):
        g.fold_state_dict(bad)
    with pytest.raises(KeyError, match=r'unexpected key resblocks\.9\.convs1\.0\.bias'):
        g.fold_state_dict(dict(small_sd, **{'resblocks.9.convs1.0.bias': torch.zeros(3)}))
    with pytest.raises(ValueError, match=r'ups\.1\.0\.weight_g'):
        g.fold_state_dict(dict(small_sd, **{'ups.1.0.weight_g': torch.zeros(64, 1, 1)}))
    with pytest.raises(ValueError, match=r'resblocks\.2\.activations\.5\.upsample\.filter has shape \(12,\)'):
        g.fold_state_dict(dict(small_sd, **{'resblocks.2.activations.5.upsample.filter': torch.zeros(12)}))
    with pytest.raises(ValueError, match=r'activation_post\.downsample\.lowpass\.filter has shape \(1, 1, 13\)'):
        g.fold_state_dict(dict(small_sd, **{'activation_post.downsample.lowpass.filter': torch.zeros(1, 1, 13)}))
    with pytest.raises(KeyError, match='unexpected key conv_post.bias'):      # a v1 checkpoint against a v2 config
        bg.BigVGANGenerator(dict(SMALL, use_bias_at_final=False), device='cpu').fold_state_dict(small_sd)


def test_vocode_batch_refuses_bad_mels_before_the_gpu():
    g = bg.BigVGANGenerator(dict(bo.CONFIGS['base'], num_mels=100), device='cpu')
    g._convs = {}
    with pytest.raises(ValueError, match='mel 1'):
        g.vocode_device([np.zeros((100, 8), np.float32), np.zeros((100, 0), np.float32)])
    with pytest.raises(ValueError, match=r'mel 0 has shape \(80, 8\)'):
        g.vocode_device([np.zeros((80, 8), np.float32)])


# ---------------------------------------------------------------------------------------------------- the C ABI, no compute
@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build
    build.build(verbose=False)
    return lib.load()


def _snake_args(**kw):
    """Arguments that pass validation; the pointers are aligned dummies (never dereferenced: every call below is refused)."""
    off = (C.c_int32 * 4)(0, 1, 3, 6)
    taps = (C.c_float * 12)()
    a = dict(in_hi=256, in_lo=512, out_hi=768, out_lo=1024, ld=64, channels=24, halo=25, off=off, n=3, alpha=1280, inv_beta=1536,
             h_up=C.cast(taps, C.c_void_p).value, h_down=C.cast(taps, C.c_void_p).value, prec=lib.PREC_BF16X3, ws=2048,
             ws_bytes=32)
    a.update(kw)
    return a, (off, taps)


def _snake_refused(cdll, text, **kw):
    a, keep = _snake_args(**kw)
    rc = cdll.ttsb_snake_aa_ex(a['in_hi'], a['in_lo'], a['out_hi'], a['out_lo'], a['ld'], a['channels'], a['halo'], a['off'], a['n'],
                               a['alpha'], a['inv_beta'], a['h_up'], a['h_down'], a['prec'], a['ws'], C.c_int64(a['ws_bytes']), None)
    err = cdll.ttsb_last_error().decode()
    assert rc == -1 and text in err, err
    del keep


def test_snake_aa_refusals_without_gpu(cdll):
    _snake_refused(cdll, 'unknown precision', prec=7)
    _snake_refused(cdll, 'is NULL', in_hi=None)
    _snake_refused(cdll, 'is NULL', out_lo=None)
    _snake_refused(cdll, 'alpha, inv_beta, h_up or h_down is NULL', inv_beta=None)
    _snake_refused(cdll, 'alpha, inv_beta, h_up or h_down is NULL', h_down=None)
    _snake_refused(cdll, 'ld = 60 must be a positive multiple of 8', ld=60)
    _snake_refused(cdll, 'channels = 65 must be in [1, ld = 64]', channels=65)
    _snake_refused(cdll, 'channels = 0', channels=0)
    _snake_refused(cdll, 'halo = 65', halo=65)
    _snake_refused(cdll, '16-byte aligned', out_hi=776)
    _snake_refused(cdll, '16-byte aligned', in_lo=520)
    _snake_refused(cdll, '4-byte aligned', alpha=1282)
    _snake_refused(cdll, 'aliases an input plane', out_hi=256)
    _snake_refused(cdll, 'aliases an input plane', out_lo=512)
    _snake_refused(cdll, 'aliases an input plane or the other output plane', out_lo=768)
    _snake_refused(cdll, 'n_clips must be >= 1', n=0)
    _snake_refused(cdll, 'increasing', off=(C.c_int32 * 4)(0, 1, 1, 6))
    _snake_refused(cdll, 'clip_offsets[0] must be 0', off=(C.c_int32 * 4)(1, 2, 3, 6))
    _snake_refused(cdll, 'clip_offsets is NULL', off=None)
    _snake_refused(cdll, 'workspace', ws_bytes=31)
    _snake_refused(cdll, 'workspace', ws=None)
    # bf16: the lo planes are not read or written, so NULL lo planes are fine and the refusal comes from elsewhere
    _snake_refused(cdll, 'workspace', prec=lib.PREC_BF16, in_lo=None, out_lo=None, ws_bytes=8)


def test_out_clamp_refusals_without_gpu(cdll):
    off = (C.c_int32 * 4)(0, 1, 3, 6)
    p = C.c_void_p(256)
    f = cdll.ttsb_conv1d_out_clamp_ex
    assert f(p, None, 64, 24, 2, off, 3, 0, p, C.c_float(0), p, C.c_int64(32), p, None) == -1
    assert b'ttsb_conv1d_out_clamp_ex: halo = 2' in cdll.ttsb_last_error()
    assert f(p, None, 64, 65, 25, off, 3, 0, p, C.c_float(0), p, C.c_int64(32), p, None) == -1
    assert b'channels' in cdll.ttsb_last_error()
    assert f(p, None, 512, 24, 25, off, 3, 0, p, C.c_float(0), p, C.c_int64(32), p, None) == -1
    assert b'ld_in <= 256' in cdll.ttsb_last_error()
    assert f(p, None, 64, 24, 25, off, 3, 0, p, C.c_float(0), p, C.c_int64(8), p, None) == -1
    assert b'workspace' in cdll.ttsb_last_error()


# ---------------------------------------------------------------------------------------------------- the scripts
def test_predict_and_evaluate_flags():
    import evaluate_tts
    import predict_tts
    a = predict_tts.parse_args(['-t', 'x', '--vocoder', 'bigvgan', '--vocoder_checkpoint', 'bigvgan_generator.pt'])
    assert a.vocoder == 'bigvgan' and a.vocoder_config is None
    a = predict_tts.parse_args(['-t', 'x', '--vocoder', 'bigvgan', '--vocoder_checkpoint', 'g', '--vocoder_config', 'bigvgan'])
    assert a.vocoder_config == 'bigvgan'
    with pytest.raises(SystemExit):
        predict_tts.parse_args(['-t', 'x', '--vocoder', 'bigvgan'])
    with pytest.raises(SystemExit):
        predict_tts.parse_args(['-t', 'x', '--vocoder', 'wavernn', '--vocoder_checkpoint', 'g', '--vocoder_config', 'base'])
    a = evaluate_tts.parse_args(['--config', 'c', '-p', 'm', '--vocoder', 'bigvgan', '--vocoder_checkpoint', 'g', '--vocoder_config', 'base'])
    assert a.vocoder == 'bigvgan' and a.vocoder_config == 'base'
    with pytest.raises(SystemExit):
        evaluate_tts.parse_args(['--config', 'c', '-p', 'm', '--vocoder', 'bigvgan'])


def _model(**kw):
    cfg = dict(sampling_rate=22050, mel_channels=80, hop_length=256, f_max=8000, normalizer='MelGAN')
    cfg.update(kw)
    return SimpleNamespace(config=cfg, device='cpu')


def test_load_vocoder_refusals(tmp_path):
    from predict_tts import load_vocoder
    ckpt = tmp_path / 'bigvgan_generator.pt'
    with pytest.raises(SystemExit, match='hop_length 275'):
        load_vocoder('bigvgan', ckpt, 'base', _model(hop_length=275))
    with pytest.raises(SystemExit, match="normalizer is 'WaveRNN'"):
        load_vocoder('bigvgan', ckpt, 'base', _model(normalizer='WaveRNN'))
    with pytest.raises(SystemExit, match='config.json not found'):
        load_vocoder('bigvgan', ckpt, None, _model())
    for key, value in (('sampling_rate', 24000), ('num_mels', 100), ('hop_size', 300), ('fmax', 11025)):
        (tmp_path / 'config.json').write_text(json.dumps(dict(bo.CONFIGS['base'], **{key: value})))
        with pytest.raises(SystemExit, match=f'--vocoder bigvgan: BigVGAN config: {key} = {value} differs'):
            load_vocoder('bigvgan', ckpt, None, _model())
    with pytest.raises(SystemExit, match='num_mels = 80 differs'):
        load_vocoder('bigvgan', ckpt, 'bigvgan', _model(mel_channels=100))
