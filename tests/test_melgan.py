"""CPU tests of the MelGAN vocoder's host side: the checkpoint specification and loader, weight-norm folding, the transposed-
conv phase layout, the halo rule, the C-ABI refusals of ttsb_conv1d_ex_tc / ttsb_conv1d_out_tanh_ex with MelGAN's
arguments and predict_tts's flags."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import melgan_oracle as mo
from transformertts_b200 import lib
from transformertts_b200.model import melgan as mg


@pytest.fixture(scope='module')
def sd():
    return mo.init_state_dict(seed=3)


def test_oracle_key_set_is_the_checkpoint_pin(sd):
    assert len(sd) == mo.N_TENSORS == 126
    assert sum(v.numel() for v in sd.values()) == mo.N_PARAMS == 4_266_050
    assert {k: tuple(v.shape) for k, v in sd.items()} == mg.expected_keys(True)
    assert len(mg.expected_keys(False)) == 84


def test_oracle_waveform_is_not_tiny_or_saturated(sd):
    g = mo.build(sd)
    with torch.no_grad():
        y = g(torch.from_numpy(mo.make_mels([40], seed=5)[0]).double()[None])
    assert y.shape == (1, 1, 256 * 40)
    assert 0.1 <= float(y.std()) and float(y.abs().max()) < 0.98


def _folded_sd(sd):
    g = mo.build(sd)
    for m in g.modules():
        if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
            torch.nn.utils.remove_weight_norm(m)
    return g.state_dict()


@pytest.mark.parametrize('wrapped', [False, True])
@pytest.mark.parametrize('normed', [False, True])
def test_checkpoint_loads_in_all_forms(tmp_path, sd, wrapped, normed):
    state = sd if normed else _folded_sd(sd)
    obj = {'model_g': state, 'model_d': {}, 'optim_g': {}, 'githash': 'x', 'epoch': 3} if wrapped else state
    path = tmp_path / 'ckpt.pt'
    torch.save(obj, path)
    got = mg.MelGANGenerator.fold_state_dict(torch.load(path, map_location='cpu', weights_only=True))
    want = mg.MelGANGenerator.fold_state_dict(sd)
    assert set(got) == set(want)
    for k in want:
        assert np.abs(got[k] - want[k]).max() < 1e-12, k


def test_bad_keys_are_refused_by_name(sd):
    bad = dict(sd)
    del bad['generator.7.blocks.1.2.weight_v']
    with pytest.raises(KeyError, match=r'generator\.7\.blocks\.1\.2\.weight_v'):
        mg.MelGANGenerator.fold_state_dict(bad)
    bad = dict(sd, **{'generator.99.bias': torch.zeros(3)})
    with pytest.raises(KeyError, match=r'generator\.99\.bias'):
        mg.MelGANGenerator.fold_state_dict(bad)
    bad = dict(sd, **{'generator.12.weight_g': torch.zeros(32, 1, 1)})
    with pytest.raises(ValueError, match=r'generator\.12\.weight_g'):
        mg.MelGANGenerator.fold_state_dict(bad)


def test_weight_norm_folding_matches_torch(sd):
    g = mo.build(sd)
    for name, (kind, _) in mg.layer_shapes().items():
        m = g.get_submodule(name)
        with torch.no_grad():   # the forward pre-hook of weight_norm computes m.weight
            m(torch.zeros((1, m.in_channels, 64), dtype=torch.float64))
        want = m.weight.detach().numpy()
        got = mg.fold_weight_norm(sd[f'{name}.weight_g'].numpy(), sd[f'{name}.weight_v'].numpy())
        assert np.abs(got - want).max() < 1e-12, name
        if kind == 'convT':   # weight (Cin, Cout, k): the norm is per input channel
            assert sd[f'{name}.weight_g'].shape[0] == m.in_channels


def _apply_taps(x, mat, shifts, cin_cols):
    """float64 reference of the kernel's product: x (L, Cin) -> (L, N), tap s reads rows t + shifts[s] (zero outside)."""
    L, cin = x.shape
    out = np.zeros((L, mat.shape[1]))
    for s, d in enumerate(shifts):
        xs = np.zeros((L, cin))
        lo, hi = max(0, -d), min(L, L - d)
        xs[lo:hi] = x[lo + d:hi + d]
        out += xs @ mat[s * cin_cols:s * cin_cols + cin]
    return out


@pytest.mark.parametrize('k,u', [(16, 8), (4, 2)])
def test_transposed_phase_layout_matches_conv_transpose(k, u):
    rng = np.random.default_rng(k)
    cin, cout, L = 24, 16, 13
    w = rng.standard_normal((cin, cout, k))
    x = rng.standard_normal((L, cin))
    want = F.conv_transpose1d(torch.from_numpy(x.T)[None], torch.from_numpy(w), stride=u, padding=u // 2)[0].numpy().T  # (L u, cout)
    mat = mg.transposed_taps(w, u, 32, cout)
    got = _apply_taps(x, mat, (-1, 0, 1), 32).reshape(L * u, cout)
    assert want.shape == (L * u, cout)
    assert np.abs(got - want).max() < 1e-12


@pytest.mark.parametrize('d', [1, 3, 9])
def test_dilated_taps_match_reflect_padded_conv(d):
    rng = np.random.default_rng(d)
    C_, L = 20, 23
    w = rng.standard_normal((C_, C_, 3))
    x = rng.standard_normal((L, C_))
    want = F.conv1d(F.pad(torch.from_numpy(x.T)[None], (d, d), mode='reflect'), torch.from_numpy(w), dilation=d)[0].numpy().T
    src = mg.halo_source_rows(L, lib.CONV1D_HALO, lib.HALO_REFLECT)
    xp = x[src]                      # the clip with its reflect halos, rows -HALO .. L - 1 + HALO
    mat = mg.conv_taps(w, d, C_, C_)
    got = _apply_taps(xp, mat, (-d, 0, d), C_)[lib.CONV1D_HALO:lib.CONV1D_HALO + L]
    assert np.abs(got - want).max() < 1e-12


@pytest.mark.parametrize('pad', [1, 3, 9])
@pytest.mark.parametrize('L', [10, 11, 14, 19, 40])
def test_halo_rule_matches_reflect_pad(pad, L):
    H = lib.CONV1D_HALO
    x = torch.arange(L, dtype=torch.float64)[None, None]
    want = F.pad(x, (pad, pad), mode='reflect')[0, 0].numpy()
    src = mg.halo_source_rows(L, H, lib.HALO_REFLECT)
    assert np.array_equal(src[H - pad:H + L + pad].astype(np.float64), want)
    z = mg.halo_source_rows(L, H, lib.HALO_ZERO)
    assert (z[:H] == -1).all() and (z[H + L:] == -1).all() and np.array_equal(z[H:H + L], np.arange(L))
    with pytest.raises(ValueError):
        mg.halo_source_rows(H, H, lib.HALO_REFLECT)


def test_pack_clips_layout():
    clips = [np.arange(12 * 3, dtype=np.float32).reshape(12, 3), np.ones((10, 3), np.float32)]
    buf = mg.pack_clips(clips, 64, lib.HALO_ZERO)
    assert buf.shape == (22 + 4 * lib.CONV1D_HALO, 64)
    for a, b in zip(mg.unpack_clips(buf, [12, 10], 3), clips):
        assert np.array_equal(a, b)
    assert (buf[:lib.CONV1D_HALO] == 0).all() and (buf[:, 3:] == 0).all()


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build
    build.build(verbose=False)
    return lib.load()


def _valid_args(lengths, ws_bytes=None, up=1, halo=lib.HALO_REFLECT):
    """MelGAN's arguments (9 halo rows, three taps, slope 0.2) that pass validation; the pointers are dummies (never
    dereferenced: every call below is refused)."""
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    tab = (C.c_int32 * len(off))(*off.tolist())
    a = lib.Conv1dExArgs()
    a.n_clips, a.clip_offsets, a.halo, a.num_taps = len(lengths), C.cast(tab, C.c_void_p), lib.CONV1D_HALO, 3
    for s, d in enumerate((-1, 0, 1)):
        a.tap_src[s], a.tap_shift[s] = 0, d
    a.in_hi[0] = a.in_lo[0] = a.w_hi = a.w_lo = a.act_hi = a.act_lo = 256
    a.ld_in[0], a.N, a.up, a.ld_out, a.halo_mode, a.precision = 64, 64 * up, up, 64, halo, lib.PREC_BF16X3
    a.slope, a.sum_mode = 0.2, lib.SUM_NONE
    a.out_rows = mg.layout_rows(lengths, up)
    a.workspace = 256
    a.workspace_bytes = ws_bytes if ws_bytes is not None else 8 * (len(lengths) + 1)
    return a, tab


def _refused(cdll, a, text):
    assert cdll.ttsb_conv1d_ex_tc(C.byref(a), None) == -1
    assert text in cdll.ttsb_last_error().decode(), cdll.ttsb_last_error().decode()


def test_conv1d_refusals_without_gpu(cdll):
    assert cdll.ttsb_conv1d_ex_tc(None, None) == -1 and b'NULL' in cdll.ttsb_last_error()
    assert cdll.ttsb_conv1d_workspace_bytes(0) == -1 and cdll.ttsb_conv1d_workspace_bytes(3) == 32
    a, keep = _valid_args([12, 10]); a.clip_offsets = None; _refused(cdll, a, 'clip_offsets is NULL')
    a, keep = _valid_args([12, 10]); a.in_lo[0] = None; _refused(cdll, a, 'source 0')
    a, keep = _valid_args([12, 10]); a.w_lo = None; _refused(cdll, a, 'weights')
    a, keep = _valid_args([12, 10]); a.act_hi = None; _refused(cdll, a, 'no output')
    a, keep = _valid_args([12, 10]); a.workspace = None; _refused(cdll, a, 'workspace')
    a, keep = _valid_args([12, 10], ws_bytes=16); _refused(cdll, a, 'workspace')
    a, keep = _valid_args([12, 10]); a.tap_shift[0] = -10; _refused(cdll, a, '|tap_shift| must be <= 9')
    a, keep = _valid_args([12, 10]); a.ld_in[0] = 80; _refused(cdll, a, 'ld_in')
    a, keep = _valid_args([12, 10]); a.N = 96; a.ld_out = 96; _refused(cdll, a, 'N = 96')
    a, keep = _valid_args([12, 10]); a.num_taps = 17; _refused(cdll, a, 'num_taps must be in [1, 16]')
    a, keep = _valid_args([12, 10]); a.precision = 2; _refused(cdll, a, 'precision')
    a, keep = _valid_args([12, 12, 9]); _refused(cdll, a, 'clip 2 has 9 output rows')        # reflect halos need 10
    a, keep = _valid_args([2, 3], up=8, halo=lib.HALO_ZERO); a.ld_out = 48; _refused(cdll, a, 'ld_out')
    a, keep = _valid_args([12, 10]); keep[1], keep[2] = 12, 11; _refused(cdll, a, 'increasing')   # non-monotonic
    a, keep = _valid_args([12, 10]); keep[0] = 1; _refused(cdll, a, 'clip_offsets[0]')
    a, keep = _valid_args([12, 10]); a.n_clips = 0; _refused(cdll, a, 'n_clips')
    # the output layer over MelGAN's halo
    off = (C.c_int32 * 3)(0, 3000, 6000)
    p = C.c_void_p(256)
    f = cdll.ttsb_conv1d_out_tanh_ex
    H = lib.CONV1D_HALO
    assert f(None, None, 64, 32, H, off, 2, 2560, p, C.c_float(0), p, C.c_int64(24), p, None) == -1
    assert b'NULL' in cdll.ttsb_last_error()
    assert f(p, None, 64, 32, H, off, 2, 2560, p, C.c_float(0), p, C.c_int64(4), p, None) == -1
    assert b'workspace' in cdll.ttsb_last_error()
    assert f(p, None, 64, 65, H, off, 2, 2560, p, C.c_float(0), p, C.c_int64(24), p, None) == -1
    short = (C.c_int32 * 3)(0, 3000, 5000)
    assert f(p, None, 64, 32, H, short, 2, 2560, p, C.c_float(0), p, C.c_int64(24), p, None) == -1
    assert b'clip 1' in cdll.ttsb_last_error()


def test_vocode_batch_refuses_short_clips_before_the_gpu():
    g = mg.MelGANGenerator(device='cpu')
    g._convs = {}   # loading packs on the GPU; the length check comes first
    with pytest.raises(ValueError, match='mel 1'):
        g.vocode_device([np.zeros((80, 8), np.float32), np.zeros((80, 3), np.float32)])


def test_predict_tts_flags():
    import predict_tts
    a = predict_tts.parse_args(['-t', 'x'])
    assert a.vocoder == 'griffinlim' and a.vocoder_checkpoint is None
    a = predict_tts.parse_args(['-t', 'x', '--vocoder', 'melgan', '--vocoder_checkpoint', 'g.pt'])
    assert a.vocoder == 'melgan' and a.vocoder_checkpoint == 'g.pt'
    with pytest.raises(SystemExit):
        predict_tts.parse_args(['-t', 'x', '--vocoder', 'melgan'])
    with pytest.raises(SystemExit):
        predict_tts.parse_args(['-t', 'x', '--vocoder', 'hifigan'])
