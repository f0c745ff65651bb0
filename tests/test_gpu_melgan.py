"""The MelGAN vocoder on the GPU: each conv kind of ttsb_conv1d_ex_tc with MelGAN's arguments against float64 torch convs
(halos included), the whole generator against the float64 oracle (oracle/melgan_oracle.py), clip independence bit for bit,
inference()'s int16 output, the launch count, and predict_tts.py --vocoder melgan end to end."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.io.wavfile
import torch
import torch.nn.functional as F

from oracle import melgan_oracle as mo

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = Path(__file__).resolve().parent.parent
FRAMES = (4, 5, 11, 37, 128, 861)
SHORT = [4 + (i % 3) for i in range(40)]          # 128-row tiles straddle clip edges at every stage
# max |waveform error| against the float64 oracle.  Measured on an H100 on the FRAMES batch (seed 11): bf16x3 5.2e-5, bf16
# 2.4e-2; the bf16 gate leaves a factor of two
WAVE_TOL = {'bf16x3': 1e-3, 'bf16': 5e-2}
CONV_TOL = {'bf16x3': 5e-5, 'bf16': 1.5e-2}       # relative to the output's max |value|


@pytest.fixture(scope='module')
def sd():
    return mo.init_state_dict(seed=11)


@pytest.fixture(scope='module')
def gens(sd):
    from transformertts_b200.model.melgan import MelGANGenerator
    return {p: MelGANGenerator(device=DEV, precision=p).load_state_dict(sd) for p in ('bf16x3', 'bf16')}


@pytest.fixture(scope='module')
def oracle(sd):
    return mo.build(sd)


def _oracle_wav(g, mel):
    with torch.no_grad():
        x = torch.cat([torch.from_numpy(mel).double(), torch.full((80, mo.PAD_FRAMES), mo.PAD_VALUE, dtype=torch.float64)], 1)
        return g(x[None])[0, 0, :-mo.HOP * mo.PAD_FRAMES].numpy()


# ---------------------------------------------------------------------------------------------------- one conv at a time
def _run_conv(prec, conv_mat, bias, taps, srcs, counts, up, cout_cols, halo):
    """One ttsb_conv1d_ex_tc call on host-packed float64 sources -> (out, act) packed float64 (rows, cout_cols)."""
    from transformertts_b200 import lib
    from transformertts_b200.model import melgan as mg
    gen = mg.MelGANGenerator(device=DEV, precision=prec)
    conv = mg._Conv(conv_mat, bias, taps, gen.split, torch.device(DEV))
    dev_srcs = [lib.split_bf16(torch.from_numpy(s.astype(np.float32)).to(DEV), gen.split) for s in srcs]
    rows = mg.layout_rows(counts, up)
    out, act = gen._planes(rows, cout_cols), gen._planes(rows, cout_cols)
    for t in out + act:
        if t is not None:
            t.fill_(float('nan'))    # halos that are not written stay NaN
    ws = torch.empty(lib.conv1d_workspace_bytes(len(counts)), dtype=torch.uint8, device=DEV)
    gen._run(conv, counts, dev_srcs, up, out=out, act=act, halo=halo, ws=ws)
    torch.cuda.synchronize()
    f = lambda p: p[0].double().cpu().numpy() + (p[1].double().cpu().numpy() if p[1] is not None else 0.0)  # noqa: E731
    return f(out), f(act)


def _check(prec, got, want_clips, counts_out, cols, halo, what):
    from transformertts_b200.model import melgan as mg
    H = mg.lib.CONV1D_HALO
    want = np.zeros((mg.layout_rows(counts_out), cols))
    r = 0
    for w in want_clips:
        L = len(w)
        src = mg.halo_source_rows(L, H, halo) if halo != mg.lib.HALO_NONE else np.arange(-H, L + H)
        ok = (src >= 0) & (src < L)
        want[r:r + L + 2 * H][ok, :w.shape[1]] = w[src[ok]]
        r += L + 2 * H
    interior = np.zeros(len(want), bool)
    r = 0
    for L in counts_out:
        interior[r + H:r + H + L] = True
        r += L + 2 * H
    rows = interior if halo == mg.lib.HALO_NONE else np.ones(len(want), bool)
    scale = max(1.0, np.abs(want).max())
    err = np.abs(got[rows] - want[rows]).max()
    assert np.isfinite(got[rows]).all(), what
    assert err < CONV_TOL[prec] * scale, (what, err, scale)


def _lrelu(x):
    return np.where(x > 0, x, 0.2 * x)


def _clips(counts, C_, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((L, C_)) for L in counts]


CONV_COUNTS = [L + 10 for L in FRAMES[:5]] + [17] * 3


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('C_', [256, 128, 64, 32])
def test_dilated_and_mix_convs(prec, C_):
    from transformertts_b200 import lib
    from transformertts_b200.model import melgan as mg
    rng = np.random.default_rng(C_)
    cols = max(64, C_)
    counts = CONV_COUNTS
    x = _clips(counts, C_, C_)
    for d in (1, 3, 9):
        w = rng.standard_normal((C_, C_, 3)) / np.sqrt(3 * C_)
        b = 0.1 * rng.standard_normal(C_)
        src = mg.pack_clips([c.astype(np.float32) for c in x], cols, lib.HALO_REFLECT).astype(np.float64)
        xs = [mg.unpack_clips(src, counts, C_)[i].astype(np.float64) for i in range(len(counts))]
        want = [F.conv1d(F.pad(torch.from_numpy(c.T)[None], (d, d), mode='reflect'), torch.from_numpy(w), torch.from_numpy(b), dilation=d)[0].numpy().T
                for c in xs]
        bias = np.zeros(cols); bias[:C_] = b
        out, act = _run_conv(prec, mg.conv_taps(w, d, cols, cols), bias, [(0, -d), (0, 0), (0, d)], [src], counts, 1, cols, lib.HALO_NONE)
        _check(prec, out, want, counts, cols, lib.HALO_NONE, f'dilated d={d} out')
        _check(prec, act, [_lrelu(y) for y in want], counts, cols, lib.HALO_NONE, f'dilated d={d} act')
    # shortcut + 1x1 as one two-source product, reflect halos on both outputs
    ws_, w2 = (rng.standard_normal((C_, C_, 1)) / np.sqrt(C_) for _ in range(2))
    b = 0.1 * rng.standard_normal(C_)
    h = _clips(counts, C_, C_ + 1)
    s0 = mg.pack_clips([c.astype(np.float32) for c in x], cols, lib.HALO_NONE).astype(np.float64)
    s1 = mg.pack_clips([c.astype(np.float32) for c in h], cols, lib.HALO_NONE).astype(np.float64)
    xs, hs = mg.unpack_clips(s0, counts, C_), mg.unpack_clips(s1, counts, C_)
    want = [xi @ ws_[:, :, 0].T + hi @ w2[:, :, 0].T + b for xi, hi in zip(xs, hs)]
    mat = np.concatenate([mg.conv_taps(ws_, 1, cols, cols), mg.conv_taps(w2, 1, cols, cols)])
    bias = np.zeros(cols); bias[:C_] = b
    for halo in (lib.HALO_REFLECT, lib.HALO_ZERO):
        out, act = _run_conv(prec, mat, bias, [(0, 0), (1, 0)], [s0, s1], counts, 1, cols, halo)
        _check(prec, out, want, counts, cols, halo, f'mix halo={halo} out')
        _check(prec, act, [_lrelu(y) for y in want], counts, cols, halo, f'mix halo={halo} act')


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('cin,cout,k,u', [(512, 256, 16, 8), (256, 128, 16, 8), (128, 64, 4, 2), (64, 32, 4, 2)])
def test_transposed_conv(prec, cin, cout, k, u):
    from transformertts_b200 import lib
    from transformertts_b200.model import melgan as mg
    rng = np.random.default_rng(cin)
    cc = max(64, cout)
    counts = CONV_COUNTS if cin > 128 else [c * 8 for c in CONV_COUNTS]
    x = _clips(counts, cin, cin)
    w = rng.standard_normal((cin, cout, k)) / np.sqrt(cin * 2)
    b = 0.1 * rng.standard_normal(cout)
    src = mg.pack_clips([c.astype(np.float32) for c in x], cin, lib.HALO_ZERO).astype(np.float64)
    xs = mg.unpack_clips(src, counts, cin)
    want = [F.conv_transpose1d(torch.from_numpy(c.T)[None], torch.from_numpy(w), torch.from_numpy(b), stride=u, padding=u // 2)[0].numpy().T
            for c in xs]
    bias = np.zeros(u * cc)
    for r in range(u):
        bias[r * cc:r * cc + cout] = b
    out, act = _run_conv(prec, mg.transposed_taps(w, u, cin, cc), bias, [(0, -1), (0, 0), (0, 1)], [src], counts, u, cc, lib.HALO_REFLECT)
    counts_out = [c * u for c in counts]
    _check(prec, out, want, counts_out, cc, lib.HALO_REFLECT, 'convT out')
    _check(prec, act, [_lrelu(y) for y in want], counts_out, cc, lib.HALO_REFLECT, 'convT act')


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_input_conv(prec):
    from transformertts_b200 import lib
    from transformertts_b200.model import melgan as mg
    rng = np.random.default_rng(80)
    counts = CONV_COUNTS + [14] * 20
    x = _clips(counts, 80, 5)
    w = rng.standard_normal((512, 80, 7)) / np.sqrt(7 * 80)
    b = 0.1 * rng.standard_normal(512)
    src = mg.pack_clips([c.astype(np.float32) for c in x], mg.MEL_COLS, lib.HALO_REFLECT).astype(np.float64)
    xs = mg.unpack_clips(src, counts, 80)
    want = [F.conv1d(F.pad(torch.from_numpy(c.T)[None], (3, 3), mode='reflect'), torch.from_numpy(w), torch.from_numpy(b))[0].numpy().T for c in xs]
    out, act = _run_conv(prec, mg.conv_taps(w, 1, mg.MEL_COLS, 512), b, [(0, s) for s in range(-3, 4)], [src], counts, 1, 512, lib.HALO_ZERO)
    _check(prec, out, want, counts, 512, lib.HALO_ZERO, 'input conv out')
    _check(prec, act, [_lrelu(y) for y in want], counts, 512, lib.HALO_ZERO, 'input conv act')


# ---------------------------------------------------------------------------------------------------- the whole generator
@pytest.fixture(scope='module')
def mels():
    return mo.make_mels(FRAMES, seed=12)


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_generator_matches_oracle(gens, oracle, mels, prec):
    got = gens[prec].vocode_batch(mels)
    errs = []
    for c, (m, g) in enumerate(zip(mels, got)):
        want = _oracle_wav(oracle, m)
        assert g.shape == want.shape == (256 * m.shape[1],), c
        errs.append(float(np.abs(g - want).max()))
    print(f'melgan {prec}: max |waveform - oracle| per clip {["%.2e" % e for e in errs]}')
    assert max(errs) <= WAVE_TOL[prec], errs


def test_short_clips_straddling_tiles_match_oracle(gens, oracle):
    ms = mo.make_mels(SHORT, seed=13)
    got = gens['bf16x3'].vocode_batch(ms)
    for c in (0, 1, 2, 17, 39):
        assert np.abs(got[c] - _oracle_wav(oracle, ms[c])).max() <= WAVE_TOL['bf16x3'], c


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_clip_independence_bitwise(gens, mels, prec):
    g = gens[prec]
    batch = g.vocode_batch(mels)
    again = g.vocode_batch(mels)
    rev = g.vocode_batch(mels[::-1])[::-1]
    short = mo.make_mels(SHORT, seed=14)
    mixed = g.vocode_batch(short[:20] + mels + short[20:])[20:20 + len(mels)]
    for c, m in enumerate(mels):
        alone = g.vocode_batch([m])[0]
        for other, what in ((again[c], 'second run'), (rev[c], 'reversed'), (mixed[c], 'other neighbours'), (alone, 'alone')):
            assert np.array_equal(batch[c], other), (c, what)
    s_batch = g.vocode_batch(short)
    for c in (0, 7, 39):
        assert np.array_equal(s_batch[c], g.vocode_batch([short[c]])[0]), c


def test_inference_matches_oracle_int16(gens, oracle, mels):
    """inference() is vocode_batch's float waveform scaled, clamped and truncated exactly; against the oracle's int16 it differs
    by no more than the float error spans (about 5e-5 of full scale: up to 2 LSB)."""
    for m in mels[:4]:
        got = gens['bf16x3'].inference(torch.from_numpy(m)[None]).numpy()
        fl = gens['bf16x3'].vocode_batch([m])[0].astype(np.float64)
        assert np.array_equal(got, np.clip(np.trunc(fl * 32768.0), -32768, 32767).astype(np.int16))
        with torch.no_grad():
            want = oracle.inference(torch.from_numpy(m).double()[None]).numpy()
        assert got.dtype == np.int16 and got.shape == want.shape == (256 * m.shape[1],)
        err = np.abs(fl - _oracle_wav(oracle, m)).max()
        d = np.abs(got.astype(np.int32) - want.astype(np.int32))
        assert err <= WAVE_TOL['bf16x3'] and d.max() <= int(np.ceil(32768.0 * err)), (err, d.max())


def test_launch_count_is_fixed(gens, mels):
    from transformertts_b200 import lib
    counts = []
    for batch in ([mels[2]], mo.make_mels([4 + 3 * i for i in range(16)], seed=15)):
        torch.cuda.synchronize()
        lib.reset_launch_count()
        gens['bf16'].vocode_batch(batch)
        counts.append(lib.launch_count())
    assert counts[0] == counts[1] == 31, counts      # the split of the packed mel + 30 convs


def test_predict_tts_melgan_end_to_end(tmp_path, gens, sd):
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
    torch.save({'model_g': sd, 'githash': 'seeded'}, tmp_path / 'melgan.pt')
    lines = ['həloʊ wɜːld', 'ðɪs ɪz ɐ lɔŋɡɚ tɛst sɛntəns.', 'ɐbɐ']
    (tmp_path / 'lines.txt').write_text('\n'.join(lines) + '\n')
    r = subprocess.run([sys.executable, str(ROOT / 'predict_tts.py'), '-p', str(tmp_path / 'model'), '-f', str(tmp_path / 'lines.txt'),
                        '-o', str(tmp_path / 'out'), '-m', '-s', '--vocoder', 'melgan', '--vocoder_checkpoint', str(tmp_path / 'melgan.pt')],
                       capture_output=True, text=True, timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    out = tmp_path / 'out' / 'outputs' / 'lines'
    stem = 'lines_ljspeech_unknown_0'
    mels = [np.load(out / f'{stem}_{i}.mel.npy') for i in range(len(lines))]
    wavs = gens['bf16x3'].vocode_batch([m.T for m in mels])
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
