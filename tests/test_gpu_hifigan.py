"""The HiFi-GAN vocoder on the GPU: each conv kind of ttsb_conv1d_ex_tc and ttsb_conv1d_out_tanh_ex against float64 torch
convs, the whole generator (V1, V2, V3) against the float64 oracle (oracle/hifigan_oracle.py), clip independence bit for
bit, inference()'s int16 output, the launch count, and predict_tts.py --vocoder hifigan end to end."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.io.wavfile
import torch
import torch.nn.functional as F

from oracle import hifigan_oracle as ho

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = Path(__file__).resolve().parent.parent
CONV_COUNTS = [1, 2, 3, 37, 800]
FRAMES = (1, 2, 3, 37, 96)
# max |waveform error| against the float64 oracle on the FRAMES batch (seed 21), measured on an H100 80GB HBM3 and noted
# beside each gate; the gates leave about a factor of two
WAVE_TOL = {('v1', 'bf16x3'): 7e-5,   # 3.49e-5
            ('v1', 'bf16'): 3e-2,     # 1.43e-2
            ('v2', 'bf16x3'): 6e-5,   # 3.10e-5
            ('v2', 'bf16'): 3e-2,     # 1.55e-2
            ('v3', 'bf16x3'): 5e-5,   # 2.17e-5
            ('v3', 'bf16'): 2.5e-2}   # 1.10e-2
CONV_TOL = {'bf16x3': 5e-5, 'bf16': 1.5e-2}       # relative to the output's max |value|


def _lrelu(x, slope):
    return np.where(x > 0, x, slope * x)


def _clips(counts, C_, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((L, C_)) for L in counts]


def _dev_planes(x, split):
    from transformertts_b200 import lib
    return lib.split_bf16(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(DEV), split)


def _nan_planes(rows, cols, split):
    hi = torch.full((rows, cols), float('nan'), dtype=torch.bfloat16, device=DEV)
    return hi, (torch.full_like(hi, float('nan')) if split else None)


def _f64(p):
    return p[0].double().cpu().numpy() + (p[1].double().cpu().numpy() if p[1] is not None else 0.0)


def _check_packed(got, want_clips, counts, H, what, prec):
    """Clip rows equal want (to the tolerance); every halo row is still NaN (never written)."""
    from transformertts_b200.model import melgan as mg
    r = 0
    scale = max(1.0, max(np.abs(w).max() for w in want_clips))
    for c, (L, w) in enumerate(zip(counts, want_clips)):
        assert np.isnan(got[r:r + H]).all() and np.isnan(got[r + H + L:r + 2 * H + L]).all(), (what, 'halo written', c)
        g = got[r + H:r + H + L, :w.shape[1]]
        assert np.isfinite(g).all(), (what, c)
        err = np.abs(g - w).max()
        assert err < CONV_TOL[prec] * scale, (what, c, err, scale)
        r += L + 2 * H
    assert r == mg.layout_rows(counts, halo=H)


def _conv64(x, w, b, d):
    """float64 zero-padded 'same' conv of one (L, Cin) clip -> (L, Cout)."""
    k = w.shape[2]
    return F.conv1d(torch.from_numpy(x.T)[None], torch.from_numpy(w), torch.from_numpy(b), dilation=d, padding=d * (k - 1) // 2)[0].numpy().T


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('C_,k,d,H', [(128, 11, 5, 25), (32, 7, 12, 36), (256, 3, 1, 25)])
def test_dilated_residual_and_sum(prec, C_, k, d, H):
    """k-tap dilated conv over zero halos, the identity residual, the three-way MRF sum and its / 3, slopes 0.1 and 0.01,
    clips of 1..800 frames; halo rows are never written."""
    from transformertts_b200 import lib
    from transformertts_b200.model import melgan as mg
    split = prec == 'bf16x3'
    rng = np.random.default_rng(C_ + k)
    cols = max(64, C_)
    counts = CONV_COUNTS
    rows = mg.layout_rows(counts, halo=H)
    ws = torch.empty(lib.conv1d_workspace_bytes(len(counts)), dtype=torch.uint8, device=DEV)
    taps = [(0, (s - (k - 1) // 2) * d) for s in range(k)]

    def packed(clips):
        host = mg.pack_clips([c.astype(np.float32) for c in clips], cols, lib.HALO_ZERO, halo=H).astype(np.float64)
        return host, mg.unpack_clips(host, counts, C_, halo=H)

    xh, xs = packed(_clips(counts, C_, 1))
    rh, rs = packed(_clips(counts, C_, 2))
    src, res = _dev_planes(xh, split), _dev_planes(rh, split)
    ws_ = [rng.standard_normal((C_, C_, k)) / np.sqrt(k * C_) for _ in range(3)]
    bs = [0.1 * rng.standard_normal(C_) for _ in range(3)]
    convs = [mg._Conv(mg.conv_taps(w, d, cols, cols), np.pad(b, (0, cols - C_)), taps, split, torch.device(DEV)) for w, b in zip(ws_, bs)]
    plain = [[_conv64(x, w, b, d) for x in xs] for w, b in zip(ws_, bs)]

    # plain conv, slope 0.1
    out, act = _nan_planes(rows, cols, split), _nan_planes(rows, cols, split)
    mg.run_conv(convs[0], counts, [src], 1, split, out=out, act=act, ws=ws, rows_halo=H, slope=0.1)
    _check_packed(_f64(out), plain[0], counts, H, 'conv out', prec)
    _check_packed(_f64(act), [_lrelu(y, 0.1) for y in plain[0]], counts, H, 'conv act', prec)
    # residual
    out, act = _nan_planes(rows, cols, split), _nan_planes(rows, cols, split)
    mg.run_conv(convs[0], counts, [src], 1, split, out=out, act=act, ws=ws, rows_halo=H, slope=0.1, res=res)
    with_res = [[y + r for y, r in zip(p, rs)] for p in plain]
    _check_packed(_f64(out), with_res[0], counts, H, 'residual out', prec)
    _check_packed(_f64(act), [_lrelu(y, 0.1) for y in with_res[0]], counts, H, 'residual act', prec)
    # MRF sum of three: write, add, finish (/ 3, then LeakyReLU 0.01)
    total = torch.full((rows, cols), float('nan'), dtype=torch.float32, device=DEV)
    out, act = _nan_planes(rows, cols, split), _nan_planes(rows, cols, split)
    for j, mode in enumerate((lib.SUM_WRITE, lib.SUM_ADD, lib.SUM_FINISH)):
        fin = mode == lib.SUM_FINISH
        mg.run_conv(convs[j], counts, [src], 1, split, out=out if fin else None, act=act if fin else None, ws=ws, rows_halo=H,
                    slope=0.01, res=res, sum_plane=total, sum_mode=mode, sum_div=3.0)
    avg = [(a + b + c) / 3 for a, b, c in zip(*with_res)]
    _check_packed(_f64(out), avg, counts, H, 'sum out', prec)
    _check_packed(_f64(act), [_lrelu(y, 0.01) for y in avg], counts, H, 'sum act', prec)


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('C_,H', [(32, 36), (256, 25), (8, 3)])
def test_output_layer_wide_halo(prec, C_, H):
    from transformertts_b200 import lib
    from transformertts_b200.model import melgan as mg
    split = prec == 'bf16x3'
    rng = np.random.default_rng(C_)
    cols = max(64, C_)
    counts = [c * 8 for c in CONV_COUNTS[:4]] + [1, 2, 3]
    x = mg.pack_clips([0.5 * c.astype(np.float32) for c in _clips(counts, C_, 3)], cols, lib.HALO_ZERO, halo=H).astype(np.float64)
    planes = _dev_planes(x, split)
    xs = [c.astype(np.float64) for c in mg.unpack_clips(_f64(planes), counts, C_, halo=H)]
    w = rng.standard_normal((1, C_, 7)) / np.sqrt(7 * C_)
    b = 0.05
    ws = torch.empty(lib.conv1d_workspace_bytes(len(counts)), dtype=torch.uint8, device=DEV)
    wav = torch.full((sum(counts),), float('nan'), dtype=torch.float32, device=DEV)
    lib.conv1d_out_tanh_ex(planes[0], planes[1], C_, H, mg.ragged_offsets(counts), 0,
                           torch.from_numpy(np.ascontiguousarray(w[0].T, dtype=np.float32)).to(DEV), b, ws, wav)
    got = wav.cpu().numpy()
    off = mg.ragged_offsets(counts)
    for c, xc in enumerate(xs):
        want = np.tanh(_conv64(xc, w, np.array([b]), 1)[:, 0])
        assert np.abs(got[off[c]:off[c + 1]] - want).max() < 1e-5, c


# ---------------------------------------------------------------------------------------------------- the whole generator
@pytest.fixture(scope='module')
def sds():
    return {v: ho.init_state_dict(v, seed=21) for v in ('v1', 'v2', 'v3')}


@pytest.fixture(scope='module')
def mels():
    return ho.make_mels(FRAMES, seed=22)


@pytest.fixture(scope='module')
def oracle_wavs(sds, mels):
    out = {}
    for v, sd in sds.items():
        g = ho.build(v, sd)
        with torch.no_grad():
            out[v] = [g(torch.from_numpy(m).double()[None])[0, 0].numpy() for m in mels]
    return out


def _gen(v, sd, prec):
    from transformertts_b200.model.hifigan import HiFiGANGenerator
    return HiFiGANGenerator(v, device=DEV, precision=prec).load_state_dict(sd)


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('v', ['v1', 'v2', 'v3'])
def test_generator_matches_oracle(sds, mels, oracle_wavs, v, prec):
    got = _gen(v, sds[v], prec).vocode_batch(mels)
    errs = []
    for c, (m, g, want) in enumerate(zip(mels, got, oracle_wavs[v])):
        assert g.shape == want.shape == (256 * m.shape[1],), c
        errs.append(float(np.abs(g - want).max()))
    print(f'hifigan {v} {prec}: max |waveform - oracle| per clip {["%.2e" % e for e in errs]}')
    assert max(errs) <= WAVE_TOL[(v, prec)], errs


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_clip_independence_bitwise(sds, mels, prec):
    g = _gen('v2', sds['v2'], prec)
    batch = g.vocode_batch(mels)
    again = g.vocode_batch(mels)
    rev = g.vocode_batch(mels[::-1])[::-1]
    short = ho.make_mels([1 + (i % 5) for i in range(30)], seed=23)
    mixed = g.vocode_batch(short[:15] + list(mels) + short[15:])[15:15 + len(mels)]
    for c, m in enumerate(mels):
        alone = g.vocode_batch([m])[0]
        for other, what in ((again[c], 'second run'), (rev[c], 'reversed'), (mixed[c], 'other neighbours'), (alone, 'alone')):
            assert np.array_equal(batch[c], other), (c, what)


def test_inference_int16(sds, mels, oracle_wavs):
    """inference() is vocode_batch's float waveform * 32768 truncated to int16, as jik876's inference.py converts."""
    g = _gen('v3', sds['v3'], 'bf16x3')
    for m, want in zip(mels[2:4], oracle_wavs['v3'][2:4]):
        got = g.inference(torch.from_numpy(m)[None]).numpy()
        fl = g.vocode_batch([m])[0]
        assert got.dtype == np.int16 and got.shape == (256 * m.shape[1],)
        assert np.array_equal(got, (fl * np.float32(32768.0)).astype(np.int16))
        d = np.abs(got.astype(np.int32) - (want * 32768.0).astype(np.int16).astype(np.int32))
        assert d.max() <= int(np.ceil(32768.0 * WAVE_TOL[('v3', 'bf16x3')])) + 1


@pytest.mark.parametrize('v', ['v1', 'v3'])
def test_launch_count(sds, mels, v):
    from transformertts_b200 import lib
    from transformertts_b200.model.hifigan import launches_per_call
    g = _gen(v, sds[v], 'bf16')
    counts = []
    for batch in ([mels[3]], ho.make_mels([1 + 3 * i for i in range(16)], seed=24)):
        torch.cuda.synchronize()
        lib.reset_launch_count()
        g.vocode_batch(batch)
        counts.append(lib.launch_count())
    assert counts[0] == counts[1] == launches_per_call(g.h) == {'v1': 79, 'v3': 24}[v], counts


def test_predict_tts_hifigan_end_to_end(tmp_path, sds):
    from oracle import forward_oracle as fo
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.model.models import ForwardTransformer
    cfg = dict(fo.CONFIGS['C1'], sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000,
               normalizer='MelGAN', data_name='ljspeech')
    p = fo.init_params(cfg, seed=7)
    p['dur_pred.out.b'] = torch.tensor([6.0])
    model = ForwardTransformer(**cfg)
    model.set_weights(p)
    model.save_model(tmp_path / 'model', with_optimizer=False)
    voc = tmp_path / 'hifigan'
    voc.mkdir()
    torch.save({'generator': sds['v3']}, voc / 'g_00000001')
    (voc / 'config.json').write_text(json.dumps(dict(ho.CONFIGS['v3'], batch_size=16, learning_rate=0.0002, sampling_rate=22050)))
    lines = ['həloʊ wɜːld', 'ðɪs ɪz ɐ lɔŋɡɚ tɛst sɛntəns.', 'ɐbɐ']
    (tmp_path / 'lines.txt').write_text('\n'.join(lines) + '\n')
    r = subprocess.run([sys.executable, str(ROOT / 'predict_tts.py'), '-p', str(tmp_path / 'model'), '-f', str(tmp_path / 'lines.txt'),
                        '-o', str(tmp_path / 'out'), '-m', '-s', '--vocoder', 'hifigan', '--vocoder_checkpoint', str(voc / 'g_00000001')],
                       capture_output=True, text=True, timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    out = tmp_path / 'out' / 'outputs' / 'lines'
    stem = 'lines_ljspeech_unknown_0'
    mels = [np.load(out / f'{stem}_{i}.mel.npy') for i in range(len(lines))]
    wavs = _gen('v3', sds['v3'], 'bf16x3').vocode_batch([m.T for m in mels])
    a = Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000, normalizer='MelGAN')
    pcm = []
    for i, w in enumerate(wavs):
        a.save_wav(w, tmp_path / f'want_{i}.wav')
        _, want = scipy.io.wavfile.read(tmp_path / f'want_{i}.wav')
        sr, got = scipy.io.wavfile.read(out / f'{stem}_{i}.wav')
        assert sr == 22050 and got.dtype == np.int16 and got.shape == (256 * mels[i].shape[0],), i
        assert np.array_equal(got, want), i
        pcm.append(got)
    _, combined = scipy.io.wavfile.read(out / f'{stem}.wav')
    assert np.array_equal(combined, np.concatenate(pcm))
