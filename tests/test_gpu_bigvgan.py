"""The BigVGAN vocoder on the GPU: ttsb_snake_aa_ex against a float64 restatement of the anti-aliased activation at ragged clip
lengths and every channel width, the clamp output layer, the whole generator (base and bigvgan, v1 and v2 final layers, 80
and 100 mels) against the float64 oracle (oracle/bigvgan_oracle.py), clip independence bit for bit, the launch count, and
predict_tts.py / evaluate_tts.py --vocoder bigvgan end to end."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.io.wavfile
import torch
import torch.nn.functional as F

from oracle import bigvgan_oracle as bo

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = Path(__file__).resolve().parent.parent
ACT_LENGTHS = [1, 2, 3, 5, 6, 7, 11, 12, 13, 63, 64, 65, 127, 128, 129, 1000]
ACT_WIDTHS = [(24, 64), (48, 64), (64, 64), (96, 128), (128, 128), (192, 192), (256, 256), (384, 512), (768, 768), (1536, 1536)]
# max |error| over max |output| against float64 on the same rounded input, measured on an H100 80GB HBM3 over ACT_WIDTHS (the
# largest of the widths noted beside each gate); the gates leave about a factor of two
ACT_TOL = {'bf16x3': 3e-5,    # 1.59e-5
           'bf16': 6e-3}      # 3.09e-3
FRAMES = (1, 2, 3, 17, 40)
# max |waveform error| / max |oracle waveform| on the FRAMES batch (seed 21), measured on an H100 80GB HBM3 and noted beside
# each gate; the gates leave about a factor of two
WAVE_TOL = {('base', 'v1', 80, 'bf16x3'): 1e-4,       # 5.15e-5
            ('base', 'v1', 80, 'bf16'): 4e-2,         # 1.88e-2
            ('base', 'v2', 100, 'bf16x3'): 1e-4,      # 4.82e-5
            ('base', 'v2', 100, 'bf16'): 3e-2,        # 1.54e-2
            ('bigvgan', 'v1', 100, 'bf16x3'): 2e-4,   # 9.97e-5
            ('bigvgan', 'v1', 100, 'bf16'): 5e-2,     # 2.78e-2
            ('bigvgan', 'v2', 80, 'bf16x3'): 2.4e-4,  # 1.19e-4
            ('bigvgan', 'v2', 80, 'bf16'): 5e-2}      # 2.55e-2


def _filters():
    """The published filter, tilted two ways: asymmetric taps catch a reversed tap order, which the symmetric filter hides."""
    f = bo.kaiser_sinc_filter1d(0.25, 0.3, 12).reshape(-1).numpy()
    return (f * (1 + 0.05 * np.arange(12))).astype(np.float32), (f * (1 - 0.03 * np.arange(12))).astype(np.float32)


def closed_form(x, alpha, inv_beta, h_up, h_down):
    """include/ttsb.h's ttsb_snake_aa_ex in float64 for one clip x (L, C)."""
    L = x.shape[0]
    m = np.arange(2 * L)[:, None]
    i = np.arange(L + 10)[None, :]
    tap = m + 15 - 2 * i
    ok = (tap >= 0) & (tap <= 11)
    W = np.where(ok, h_up[np.clip(tap, 0, 11)], 0.0)                     # (2L, L + 10)
    xr = x[np.clip(np.arange(L + 10) - 5, 0, L - 1)]
    u = 2.0 * (W @ xr)
    s = u + inv_beta * np.sin(alpha * u) ** 2
    idx = np.clip(2 * np.arange(L)[:, None] + np.arange(12)[None, :] - 5, 0, 2 * L - 1)
    return np.einsum('tjc,j->tc', s[idx], h_down)


def _f64(p):
    return p[0].double().cpu().numpy() + (p[1].double().cpu().numpy() if p[1] is not None else 0.0)


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('channels,ld', ACT_WIDTHS)
def test_snake_aa_matches_float64(prec, channels, ld):
    from transformertts_b200 import lib
    from transformertts_b200.model import melgan as mg
    split = prec == 'bf16x3'
    rng = np.random.default_rng(channels + ld)
    H = 25
    counts = ACT_LENGTHS
    clips = [np.clip(10.0 * rng.standard_normal((L, channels)), -30, 30) for L in counts]
    clips[3][:, 0] = 30.0
    clips[4][:, -1] = -30.0
    host = mg.pack_clips([c.astype(np.float32) for c in clips], ld, lib.HALO_ZERO, halo=H)
    rows = host.shape[0]
    src = lib.split_bf16(torch.from_numpy(host).to(DEV), split)
    xs = mg.unpack_clips(_f64(src), counts, channels, halo=H)               # the rounded input the kernel reads
    alpha = np.exp(rng.uniform(-3, 3, channels)).astype(np.float32)
    inv_beta = (1.0 / (np.exp(rng.uniform(-3, 3, channels)) + 1e-9)).astype(np.float32)
    h_up, h_down = _filters()
    nan = torch.full((rows, ld), float('nan'), dtype=torch.bfloat16, device=DEV)
    dst = (nan, nan.clone() if split else None)
    ws = torch.empty(lib.conv1d_workspace_bytes(len(counts)), dtype=torch.uint8, device=DEV)
    lib.snake_aa_ex(src, dst, channels, H, mg.ragged_offsets(counts), torch.from_numpy(alpha).to(DEV),
                    torch.from_numpy(inv_beta).to(DEV), h_up, h_down, ws)
    got = _f64(dst)
    wants = [closed_form(x, alpha.astype(np.float64), inv_beta.astype(np.float64), h_up.astype(np.float64), h_down.astype(np.float64))
             for x in xs]
    scale = max(np.abs(w).max() for w in wants)
    r, worst = 0, 0.0
    for c, (L, w) in enumerate(zip(counts, wants)):
        assert np.isnan(got[r:r + H]).all() and np.isnan(got[r + H + L:r + 2 * H + L]).all(), ('halo written', c)
        g = got[r + H:r + H + L]
        assert (g[:, channels:] == 0).all(), ('padded channels not 0', c)
        worst = max(worst, float(np.abs(g[:, :channels] - w).max()) / scale)
        r += L + 2 * H
    print(f'snake_aa {prec} {channels}/{ld}: max |err| / max |out| = {worst:.2e}')
    assert worst < ACT_TOL[prec], worst


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_clamp_output_layer(prec):
    from transformertts_b200 import lib
    from transformertts_b200.model import melgan as mg
    split = prec == 'bf16x3'
    rng = np.random.default_rng(5)
    C_, H, cols = 24, 25, 64
    counts = [1, 2, 3, 37, 800, 4096]
    x = mg.pack_clips([rng.standard_normal((L, C_)).astype(np.float32) for L in counts], cols, lib.HALO_ZERO, halo=H)
    planes = lib.split_bf16(torch.from_numpy(x).to(DEV), split)
    xs = mg.unpack_clips(_f64(planes), counts, C_, halo=H)
    w = 1.5 * rng.standard_normal((1, C_, 7)) / np.sqrt(7 * C_)
    ws = torch.empty(lib.conv1d_workspace_bytes(len(counts)), dtype=torch.uint8, device=DEV)
    wav = torch.full((sum(counts),), float('nan'), dtype=torch.float32, device=DEV)
    lib.conv1d_out_clamp_ex(planes[0], planes[1], C_, H, mg.ragged_offsets(counts), 0,
                            torch.from_numpy(np.ascontiguousarray(w[0].T, dtype=np.float32)).to(DEV), 0.0, ws, wav)
    got = wav.cpu().numpy()
    off = mg.ragged_offsets(counts)
    clamped = 0
    for c, xc in enumerate(xs):
        y = F.conv1d(torch.from_numpy(xc.T)[None], torch.from_numpy(w), padding=3)[0, 0].numpy()
        want = np.clip(y, -1.0, 1.0)
        clamped += int((np.abs(y) > 1).sum())
        assert np.abs(got[off[c]:off[c + 1]] - want).max() < 1e-5, c
    assert clamped > 100     # the clamp is exercised, not only the identity


# ---------------------------------------------------------------------------------------------------- the whole generator
CASES = [('base', 'v1', 80), ('base', 'v2', 100), ('bigvgan', 'v1', 100), ('bigvgan', 'v2', 80)]


def _h(preset, final, n_mels):
    from transformertts_b200.model import bigvgan as bg
    h = dict(bg.PRESETS[preset], num_mels=n_mels)
    if final == 'v2':
        h.update(use_tanh_at_final=False, use_bias_at_final=False)
    return h


@pytest.fixture(scope='module')
def cases():
    out = {}
    for preset, final, n_mels in CASES:
        h = _h(preset, final, n_mels)
        sd = bo.init_state_dict(h, seed=21)
        mels = bo.make_mels(FRAMES, n_mels=n_mels, seed=22)
        g = bo.build(h, sd)
        with torch.no_grad():
            wavs = [g(torch.from_numpy(m).double()[None])[0, 0].numpy() for m in mels]
        out[(preset, final, n_mels)] = (h, sd, mels, wavs)
    return out


def _gen(h, sd, prec):
    from transformertts_b200.model.bigvgan import BigVGANGenerator
    return BigVGANGenerator(h, device=DEV, precision=prec).load_state_dict(sd)


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('case', CASES, ids=['-'.join(map(str, c)) for c in CASES])
def test_generator_matches_oracle(cases, case, prec):
    h, sd, mels, wants = cases[case]
    got = _gen(h, sd, prec).vocode_batch(mels)
    scale = max(float(np.abs(w).max()) for w in wants)
    errs = []
    for c, (m, g, want) in enumerate(zip(mels, got, wants)):
        assert g.shape == want.shape == (256 * m.shape[1],), c
        errs.append(float(np.abs(g - want).max()) / scale)
    print(f'bigvgan {case} {prec}: max |waveform - oracle| / max |oracle| per clip {["%.2e" % e for e in errs]} (scale {scale:.3f})')
    assert max(errs) <= WAVE_TOL[case + (prec,)], errs


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_clip_independence_bitwise(cases, prec):
    h, sd, mels, _ = cases[('base', 'v1', 80)]
    g = _gen(h, sd, prec)
    batch = g.vocode_batch(mels)
    again = g.vocode_batch(mels)
    rev = g.vocode_batch(mels[::-1])[::-1]
    short = bo.make_mels([1 + (i % 5) for i in range(20)], seed=23)
    mixed = g.vocode_batch(short[:10] + list(mels) + short[10:])[10:10 + len(mels)]
    for c, m in enumerate(mels):
        alone = g.vocode_batch([m])[0]
        for other, what in ((again[c], 'second run'), (rev[c], 'reversed'), (mixed[c], 'other neighbours'), (alone, 'alone')):
            assert np.array_equal(batch[c], other), (c, what)


def test_launch_count(cases):
    from transformertts_b200 import lib
    from transformertts_b200.model.bigvgan import launches_per_call
    h, sd, mels, _ = cases[('bigvgan', 'v2', 80)]
    g = _gen(h, sd, 'bf16')
    counts = []
    for batch in ([mels[3]], bo.make_mels([1 + 3 * i for i in range(16)], seed=24)):
        torch.cuda.synchronize()
        lib.reset_launch_count()
        g.vocode_batch(batch)
        counts.append(lib.launch_count())
    assert counts[0] == counts[1] == launches_per_call(g.h) == 226, counts


def _write_checkpoint(d: Path, sd, h):
    d.mkdir()
    torch.save({'generator': sd}, d / 'bigvgan_generator.pt')
    (d / 'config.json').write_text(json.dumps(dict(h, batch_size=32, learning_rate=0.0001, n_fft=1024, win_size=1024, fmin=0)))
    return d / 'bigvgan_generator.pt'


def test_predict_tts_bigvgan_end_to_end(tmp_path, cases):
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
    h, sd, _, _ = cases[('base', 'v1', 80)]
    ckpt = _write_checkpoint(tmp_path / 'bigvgan', sd, h)
    lines = ['həloʊ wɜːld', 'ðɪs ɪz ɐ lɔŋɡɚ tɛst sɛntəns.', 'ɐbɐ']
    (tmp_path / 'lines.txt').write_text('\n'.join(lines) + '\n')
    r = subprocess.run([sys.executable, str(ROOT / 'predict_tts.py'), '-p', str(tmp_path / 'model'), '-f', str(tmp_path / 'lines.txt'),
                        '-o', str(tmp_path / 'out'), '-m', '-s', '--vocoder', 'bigvgan', '--vocoder_checkpoint', str(ckpt)],
                       capture_output=True, text=True, timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    out = tmp_path / 'out' / 'outputs' / 'lines'
    stem = 'lines_ljspeech_unknown_0'
    mels = [np.load(out / f'{stem}_{i}.mel.npy') for i in range(len(lines))]
    wavs = _gen(h, sd, 'bf16x3').vocode_batch([m.T for m in mels])
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


def test_evaluate_tts_bigvgan_leaves_other_scores_unchanged(tmp_path, cases):
    import test_gpu_evaluation as te
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    cfg = te._config(tmp_path)
    cm = TrainingConfigManager(str(cfg))
    rng = np.random.default_rng(8)
    lines = {f'u{i:03d}': te._phonemes(rng) for i in range(8)}
    valid = te._write_data(cm, lines, te._random_targets(lines, seed=9))
    te._save_model(tmp_path / 'weights')
    h, sd, _, _ = cases[('base', 'v2', 100)]
    ckpt = _write_checkpoint(tmp_path / 'bigvgan', sd, dict(h, num_mels=80))
    model_dir = str(tmp_path / 'weights' / 'step_0')
    # the checkpoint's config gives 100 mels against the model's 80: refused by name before any vocoding
    (tmp_path / 'c100.json').write_text(json.dumps(h))
    r = subprocess.run([sys.executable, str(ROOT / 'evaluate_tts.py'), '--config', str(cfg), '-p', model_dir, '-o', str(tmp_path / 'bad'),
                        '--vocoder', 'bigvgan', '--vocoder_checkpoint', str(ckpt), '--vocoder_config', str(tmp_path / 'c100.json')],
                       capture_output=True, text=True, timeout=900, cwd=str(ROOT))
    assert r.returncode != 0 and 'num_mels' in r.stderr, r.stderr[-2000:]
    # an 80-mel generator of the same form scores; every score that does not involve the vocoder is unchanged
    h80 = dict(h, num_mels=80)
    torch.save({'generator': bo.init_state_dict(h80, seed=21)}, ckpt)
    te._run('evaluate_tts.py', ['--config', str(cfg), '-p', model_dir, '-o', str(tmp_path / 'plain')])
    out = te._run('evaluate_tts.py', ['--config', str(cfg), '-p', model_dir, '-o', str(tmp_path / 'voc'), '--vocoder', 'bigvgan',
                                      '--vocoder_checkpoint', str(ckpt)])
    assert 'copy synthesis' in out
    plain = json.loads((tmp_path / 'plain' / 'evaluation.json').read_text())['checkpoints'][0]
    voc = json.loads((tmp_path / 'voc' / 'evaluation.json').read_text())['checkpoints'][0]
    assert [ln['name'] for ln in voc['lines']] == valid
    for a, b in zip(plain['lines'], voc['lines']):
        for k, v in a.items():
            assert b[k] == v, k
        assert np.isfinite(b['vocoded_mcd']) and np.isfinite(b['copy_synthesis_mcd'])
    for k, v in plain['mean'].items():
        assert voc['mean'][k] == v, k
