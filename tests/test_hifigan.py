"""CPU tests of the HiFi-GAN vocoder's host side: the oracle's parameter counts and key set, the oracle against an independent
functional composition, the checkpoint loader and config checks, the tap matrices of the dilated convs over zero halos, the
C-ABI refusals of ttsb_conv1d_ex_tc / ttsb_conv1d_out_tanh_ex, and predict_tts's flags."""
import ctypes as C
import json
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import hifigan_oracle as ho
from transformertts_b200 import lib
from transformertts_b200.model import hifigan as hg
from transformertts_b200.model import melgan as mg

SMALL = dict(resblock='1', upsample_rates=[8, 4, 8], upsample_kernel_sizes=[16, 8, 16], upsample_initial_channel=32,
             resblock_kernel_sizes=[3, 5], resblock_dilation_sizes=[[1, 3, 5], [1, 2, 4]])


@pytest.fixture(scope='module')
def sd3():
    return ho.init_state_dict('v3', seed=3)


def _folded(h, sd):
    g = ho.build(h, sd)
    for m in g.modules():
        if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
            torch.nn.utils.remove_weight_norm(m)
    return g.state_dict()


@pytest.mark.parametrize('v', ['v1', 'v2', 'v3'])
def test_oracle_parameter_counts_and_keys(v):
    h = hg.load_config(v)
    g = ho.build(v)
    sd = g.state_dict()
    assert {k: tuple(t.shape) for k, t in sd.items()} == hg.expected_keys(h, True)
    folded = _folded(v, sd)
    assert {k: tuple(t.shape) for k, t in folded.items()} == hg.expected_keys(h, False)
    assert sum(t.numel() for t in folded.values()) == ho.N_PARAMS[v] == {'v1': 13_926_017, 'v2': 925_985, 'v3': 1_462_273}[v]
    assert hg.PRESETS[v] == ho.CONFIGS[v]


def _functional(h, w, mel):
    """The generator as a bare F.conv1d / F.conv_transpose1d composition over folded weights (no nn.Module)."""
    def conv(name, x, d=1):
        k = w[name + '.weight'].shape[2]
        return F.conv1d(x, w[name + '.weight'], w[name + '.bias'], dilation=d, padding=d * (k - 1) // 2)
    nk = len(h['resblock_kernel_sizes'])
    x = conv('conv_pre', mel)
    for i, (u, k) in enumerate(zip(h['upsample_rates'], h['upsample_kernel_sizes'])):
        x = F.conv_transpose1d(F.leaky_relu(x, 0.1), w[f'ups.{i}.weight'], w[f'ups.{i}.bias'], stride=u, padding=(k - u) // 2)
        acc = 0
        for j, dil in enumerate(h['resblock_dilation_sizes']):
            n, xr = i * nk + j, x
            for m, d in enumerate(dil):
                if h['resblock'] == '1':
                    t = conv(f'resblocks.{n}.convs2.{m}', F.leaky_relu(conv(f'resblocks.{n}.convs1.{m}', F.leaky_relu(xr, 0.1), d), 0.1))
                else:
                    t = conv(f'resblocks.{n}.convs.{m}', F.leaky_relu(xr, 0.1), d)
                xr = t + xr
            acc = acc + xr
        x = acc / nk
    return torch.tanh(conv('conv_post', F.leaky_relu(x, 0.01)))


@pytest.mark.parametrize('h', [SMALL, dict(SMALL, resblock='2', resblock_dilation_sizes=[[1, 2], [2, 6]])])
def test_oracle_matches_functional_composition(h):
    sd = ho.init_state_dict(h, seed=4)
    w = _folded(h, sd)
    mel = torch.from_numpy(ho.make_mels([9], seed=5)[0]).double()[None]
    with torch.no_grad():
        want = _functional(hg.load_config(h), w, mel)
        got = ho.build(h, sd)(mel)
    assert got.shape == want.shape == (1, 1, 256 * 9)
    assert (got - want).abs().max().item() < 1e-12


def test_oracle_waveform_is_not_tiny_or_saturated(sd3):
    with torch.no_grad():
        y = ho.build('v3', sd3)(torch.from_numpy(ho.make_mels([40], seed=5)[0]).double()[None])
    assert 0.1 <= float(y.std()) <= 0.35 and float(y.abs().max()) < 0.98


@pytest.mark.parametrize('wrapped', [False, True])
@pytest.mark.parametrize('normed', [False, True])
def test_checkpoint_loads_in_all_forms(tmp_path, sd3, wrapped, normed):
    state = sd3 if normed else _folded('v3', sd3)
    obj = {'generator': state} if wrapped else state
    torch.save(obj, tmp_path / 'g.pt')
    g = hg.HiFiGANGenerator('v3', device='cpu')
    got = g.fold_state_dict(torch.load(tmp_path / 'g.pt', map_location='cpu', weights_only=True))
    want = g.fold_state_dict(sd3)
    assert set(got) == set(want)
    for k in want:
        assert np.abs(got[k] - want[k]).max() < 1e-12, k


def test_weight_norm_folding_matches_torch(sd3):
    w = _folded('v3', sd3)
    g = hg.HiFiGANGenerator('v3', device='cpu')
    got = g.fold_state_dict(sd3)
    for name in hg.layer_shapes(g.h):
        assert np.abs(got[name] - w[name + '.weight'].numpy()).max() < 1e-12, name


def test_bad_keys_are_refused_by_name(sd3):
    g = hg.HiFiGANGenerator('v3', device='cpu')
    bad = dict(sd3)
    del bad['resblocks.4.convs.1.weight_v']
    with pytest.raises(KeyError, match=r'missing key resblocks\.4\.convs\.1\.weight_v'):
        g.fold_state_dict(bad)
    with pytest.raises(KeyError, match=r'unexpected key resblocks\.9\.convs\.0\.bias'):
        g.fold_state_dict(dict(sd3, **{'resblocks.9.convs.0.bias': torch.zeros(3)}))
    with pytest.raises(ValueError, match=r'ups\.1\.weight_g'):
        g.fold_state_dict(dict(sd3, **{'ups.1.weight_g': torch.zeros(64, 1, 1)}))
    with pytest.raises(KeyError, match='missing key'):   # a V1 checkpoint against the V3 config
        g.fold_state_dict(ho.build('v2').state_dict())


def test_config_sources_and_refusals(tmp_path):
    path = tmp_path / 'config.json'
    path.write_text(json.dumps(dict(ho.CONFIGS['v1'], batch_size=16, segment_size=8192, num_mels=80)))
    assert hg.load_config(path) == hg.load_config('V1') == hg.load_config(dict(ho.CONFIGS['v1']))
    for bad, text in ((dict(upsample_kernel_sizes=[16, 16, 4, 3]), 'kernel = 2 rate'),
                      (dict(upsample_rates=[8, 8, 4, 1], upsample_kernel_sizes=[16, 16, 8, 2]), 'even rate'),
                      (dict(upsample_rates=[8, 8, 2]), 'equal length'),
                      (dict(upsample_rates=[8, 8, 2, 4], upsample_kernel_sizes=[16, 16, 4, 8]), 'hop'),
                      (dict(resblock='3'), 'resblock'),
                      (dict(resblock_kernel_sizes=[3, 7, 17]), 'at most 16'),
                      (dict(resblock_dilation_sizes=[[1, 3], [1, 3], [1, 3]]), 'takes 3 dilations'),
                      (dict(resblock_kernel_sizes=[3, 7, 15], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 10]]), 'exceeds 64'),
                      (dict(upsample_initial_channel=96), 'multiple of 64')):
        with pytest.raises(ValueError, match=re.escape(text)):
            hg.load_config(dict(ho.CONFIGS['v1'], **bad))
    h = dict(ho.CONFIGS['v1'])
    del h['resblock']
    with pytest.raises(ValueError, match='missing key resblock'):
        hg.load_config(h)
    with pytest.raises(FileNotFoundError, match='config.json'):
        hg.HiFiGANGenerator.from_checkpoint(tmp_path / 'sub' / 'g.pt')
    assert [hg.halo_rows(hg.load_config(v)) for v in ('v1', 'v2', 'v3')] == [25, 25, 36]
    assert lib.CONV1D_EX_MAX_HALO >= 36 and lib.CONV1D_EX_MAX_TAPS >= 11   # V3's halo, and its 11-tap resblocks
    assert [hg.launches_per_call(hg.load_config(v)) for v in ('v1', 'v2', 'v3')] == [79, 79, 24]


def _apply_taps(x, mat, shifts, cin_cols):
    """float64 reference of the kernel's product: x (rows, Cin) -> (rows, N), tap s reads rows t + shifts[s] (zero outside)."""
    L, cin = x.shape
    out = np.zeros((L, mat.shape[1]))
    for s, d in enumerate(shifts):
        xs = np.zeros((L, cin))
        lo, hi = max(0, -d), min(L, L - d)
        xs[lo:hi] = x[lo + d:hi + d]
        out += xs @ mat[s * cin_cols:s * cin_cols + cin]
    return out


@pytest.mark.parametrize('d', [1, 3, 5, 2, 6, 12])
@pytest.mark.parametrize('k', [3, 7, 11])
def test_tap_matrices_over_zero_halos_match_conv1d(k, d):
    rng = np.random.default_rng(10 * k + d)
    C_, H = 20, d * (k - 1) // 2
    w = rng.standard_normal((C_, C_, k))
    for L in (1, 2, 23):
        x = rng.standard_normal((L, C_)).astype(np.float32).astype(np.float64)   # exact through pack_clips' float32
        want = F.conv1d(torch.from_numpy(x.T)[None], torch.from_numpy(w), dilation=d, padding=H)[0].numpy().T
        xp = mg.pack_clips([x], 32, lib.HALO_ZERO, halo=H).astype(np.float64)[:, :C_]
        assert xp.shape == (L + 2 * H, C_)
        got = _apply_taps(xp, mg.conv_taps(w, d, C_, C_), [(s - (k - 1) // 2) * d for s in range(k)], C_)[H:H + L]
        assert np.abs(got - want).max() < 1e-12, L


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build
    build.build(verbose=False)
    return lib.load()


def _valid_ex(lengths, halo=25, k=11, d=5, up=1):
    """Arguments that pass validation; the pointers are aligned dummies (never dereferenced: every call below is refused)."""
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    tab = (C.c_int32 * len(off))(*off.tolist())
    a = lib.Conv1dExArgs()
    a.n_clips, a.clip_offsets, a.halo, a.num_taps = len(lengths), C.cast(tab, C.c_void_p), halo, k
    for s in range(k):
        a.tap_src[s], a.tap_shift[s] = 0, (s - (k - 1) // 2) * d
    a.in_hi[0] = a.in_lo[0] = a.w_hi = a.w_lo = a.act_hi = a.act_lo = 256
    a.res_hi, a.res_lo, a.out_hi, a.out_lo = 512, 768, 1024, 1280
    a.ld_in[0], a.N, a.up, a.ld_out, a.halo_mode, a.precision = 64, 64 * up, up, 64, lib.HALO_NONE, lib.PREC_BF16X3
    a.slope, a.sum_mode, a.sum_div = 0.1, lib.SUM_NONE, 1.0
    a.out_rows = int(np.sum(lengths)) * up + 2 * halo * len(lengths)
    a.workspace, a.workspace_bytes = 256, 8 * (len(lengths) + 1)
    return a, tab


def _refused(cdll, a, text):
    assert cdll.ttsb_conv1d_ex_tc(C.byref(a), None) == -1
    assert text in cdll.ttsb_last_error().decode(), cdll.ttsb_last_error().decode()


def test_conv1d_ex_refusals_without_gpu(cdll):
    assert cdll.ttsb_conv1d_ex_tc(None, None) == -1 and b'NULL' in cdll.ttsb_last_error()
    a, keep = _valid_ex([1, 2, 3]); a.num_taps = 17; _refused(cdll, a, 'num_taps must be in [1, 16]')
    a, keep = _valid_ex([1, 2, 3]); a.tap_shift[0] = -26; _refused(cdll, a, '|tap_shift| must be <= 25')
    a, keep = _valid_ex([1, 2, 3], halo=65, d=1); _refused(cdll, a, 'halo = 65')
    a, keep = _valid_ex([1, 2, 3]); a.halo = -1; _refused(cdll, a, 'halo = -1')
    a, keep = _valid_ex([1, 2, 3]); a.slope = 1.5; _refused(cdll, a, 'slope')
    a, keep = _valid_ex([1, 2, 3]); a.slope = float('nan'); _refused(cdll, a, 'slope')
    a, keep = _valid_ex([1, 2, 3]); a.res_lo = None; _refused(cdll, a, 'res_lo')
    a, keep = _valid_ex([1, 2, 3]); a.res_hi = None; _refused(cdll, a, 'res_lo without res_hi')
    a, keep = _valid_ex([1, 2, 3]); a.res_hi = 1024; _refused(cdll, a, 'alias')
    a, keep = _valid_ex([1, 2, 3]); a.res_hi = 520; _refused(cdll, a, '16-byte aligned')
    a, keep = _valid_ex([1, 2, 3]); a.sum_mode = 4; a.sum = 2048; _refused(cdll, a, 'unknown sum_mode')
    a, keep = _valid_ex([1, 2, 3]); a.sum_mode = lib.SUM_ADD; _refused(cdll, a, 'sum must be given')
    a, keep = _valid_ex([1, 2, 3]); a.sum = 2048; _refused(cdll, a, 'sum must be given')
    a, keep = _valid_ex([1, 2, 3]); a.sum, a.sum_mode, a.sum_div = 2048, lib.SUM_FINISH, 0.0; _refused(cdll, a, 'sum_div')
    a, keep = _valid_ex([1, 2, 3]); a.out_hi = a.act_hi = None; _refused(cdll, a, 'no output')
    a, keep = _valid_ex([1, 2, 3]); a.out_rows -= 1; _refused(cdll, a, 'out_rows')
    a, keep = _valid_ex([1, 2, 3], up=8); a.out_rows = 6 + 150; _refused(cdll, a, 'out_rows')
    a, keep = _valid_ex([1, 2, 3]); a.workspace_bytes = 16; _refused(cdll, a, 'workspace')
    a, keep = _valid_ex([1, 2, 3]); a.ld_in[0] = 80; _refused(cdll, a, 'ld_in')
    a, keep = _valid_ex([1, 2, 3]); a.in_lo[0] = None; _refused(cdll, a, 'source 0')
    a, keep = _valid_ex([1, 2, 3]); keep[2] = 0; _refused(cdll, a, 'increasing')
    a, keep = _valid_ex([1, 2, 3]); a.halo_mode = lib.HALO_REFLECT; _refused(cdll, a, 'clip 0 has 1 output rows')
    # the output layer over a wide halo
    off = (C.c_int32 * 4)(0, 1, 3, 6)
    p = C.c_void_p(256)
    f = cdll.ttsb_conv1d_out_tanh_ex
    assert f(p, None, 64, 32, 2, off, 3, 0, p, C.c_float(0), p, C.c_int64(32), p, None) == -1
    assert b'halo = 2' in cdll.ttsb_last_error()
    assert f(p, None, 64, 32, 65, off, 3, 0, p, C.c_float(0), p, C.c_int64(32), p, None) == -1
    assert f(p, None, 64, 65, 36, off, 3, 0, p, C.c_float(0), p, C.c_int64(32), p, None) == -1
    assert b'channels' in cdll.ttsb_last_error()
    assert f(p, None, 64, 32, 36, off, 3, 1, p, C.c_float(0), p, C.c_int64(32), p, None) == -1
    assert b'clip 0' in cdll.ttsb_last_error()
    assert f(p, None, 64, 32, 36, off, 3, 0, p, C.c_float(0), p, C.c_int64(8), p, None) == -1
    assert b'workspace' in cdll.ttsb_last_error()


def _valid_ex_apart(lengths):
    """_valid_ex with out, act, residual and input planes at six different (aligned, dummy) addresses."""
    a, keep = _valid_ex(lengths)
    a.act_hi, a.act_lo = 1536, 1792
    return a, keep


def test_conv1d_ex_refuses_misaligned_and_in_place_planes(cdll):
    # the epilogue's 16-byte vector stores and bias loads: a misaligned plane is refused, not faulted on
    aligned = 'out_hi, out_lo, act_hi, act_lo and bias must be 16-byte aligned'
    for field in ('out_hi', 'out_lo', 'act_hi', 'act_lo'):
        a, keep = _valid_ex_apart([1, 2, 3]); setattr(a, field, getattr(a, field) + 8); _refused(cdll, a, aligned)
    a, keep = _valid_ex_apart([1, 2, 3]); a.bias = 2052; _refused(cdll, a, aligned)
    # no in-place conv: an output plane is never a plane a tap reads, and the residual is never an output
    a, keep = _valid_ex_apart([1, 2, 3]); a.out_hi = 256; _refused(cdll, a, 'aliases an input plane of source 0')
    a, keep = _valid_ex_apart([1, 2, 3]); a.in_lo[0] = a.act_lo = 2048; _refused(cdll, a, 'aliases an input plane of source 0')
    a, keep = _valid_ex_apart([1, 2, 3])
    a.in_hi[1], a.in_lo[1], a.ld_in[1], a.tap_src[3] = 2304, 2560, 64, 1
    a.act_hi = 2304; _refused(cdll, a, 'aliases an input plane of source 1')
    a, keep = _valid_ex_apart([1, 2, 3]); a.res_lo = 1280; _refused(cdll, a, 'the residual must not alias an output')
    a, keep = _valid_ex_apart([1, 2, 3]); a.res_lo = 1792; _refused(cdll, a, 'the residual must not alias an output')
    a, keep = _valid_ex_apart([1, 2, 3]); a.res_hi = 1536; _refused(cdll, a, 'the residual must not alias an output')


def test_vocode_batch_refuses_bad_mels_before_the_gpu():
    g = hg.HiFiGANGenerator('v1', device='cpu')
    g._convs = {}   # loading packs on the GPU; the shape check comes first
    with pytest.raises(ValueError, match='mel 1'):
        g.vocode_device([np.zeros((80, 8), np.float32), np.zeros((80, 0), np.float32)])
    with pytest.raises(ValueError, match='mel 0'):
        g.vocode_device([np.zeros((64, 8), np.float32)])


def test_predict_tts_flags():
    import predict_tts
    a = predict_tts.parse_args(['-t', 'x', '--vocoder', 'hifigan', '--vocoder_checkpoint', 'g_02500000'])
    assert a.vocoder == 'hifigan' and a.vocoder_checkpoint == 'g_02500000' and a.vocoder_config is None
    a = predict_tts.parse_args(['-t', 'x', '--vocoder', 'hifigan', '--vocoder_checkpoint', 'g', '--vocoder_config', 'v3'])
    assert a.vocoder_config == 'v3'
    with pytest.raises(SystemExit):
        predict_tts.parse_args(['-t', 'x', '--vocoder', 'hifigan'])
    with pytest.raises(SystemExit):
        predict_tts.parse_args(['-t', 'x', '--vocoder', 'melgan', '--vocoder_checkpoint', 'g', '--vocoder_config', 'v1'])
    a = predict_tts.parse_args(['-t', 'x'])
    assert a.vocoder == 'griffinlim' and a.vocoder_config is None
