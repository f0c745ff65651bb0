"""WORLD mel-cepstral distortion on the GPU: ttsb_cheaptrick against the float64 restatement (tests/world_mcep_oracle.py) at
every sampling rate and edge frame, envelopes and mel-cepstra bit-identical in any batch, ttsb_mcd_dtw_ceps(_path) bit for bit
against ttsb_mcd_dtw(_path) on the same cepstra, and evaluate_tts.py --mcep end to end against the restatement."""
import json
import subprocess
import sys
import wave
from pathlib import Path

import numpy as np
import pytest
import torch
import yaml

import evaluation_oracle as eo
import world_mcep_oracle as wo

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import pitch_oracle as po   # noqa: E402

# Against the restatement, measured on an H100 80GB HBM3: log envelopes within 8.5e-13 (natural log, every rate and the F0
# edges), mel-cepstra within 1.8e-15, the end-to-end per-line MCD within 9.0e-15 relative; the gates are 1e-9
LOG_TOL = 1e-9
MCEP_TOL = 1e-9
MCD_REL = 1e-9


def _audio(fs, hop):
    from transformertts_b200.data.audio import Audio
    return Audio(sampling_rate=fs, n_fft=1024, mel_channels=80, hop_length=hop, win_length=1024, f_min=0, f_max=None,
                 normalizer='MelGAN')


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def _envelopes(audio, clips, f0s=None):
    """GPU envelopes of a list of clips at their GPU F0 (or the given F0 contours) -> (list of envelopes, list of F0)."""
    wav, so = audio._pack(clips)
    fo = np.concatenate([[0], np.cumsum(audio._pitch_frames(np.diff(so)))])
    if f0s is None:
        f0, fo = audio.extract_pitch_device(wav, so)
    else:
        f0 = torch.from_numpy(np.concatenate(f0s).astype(np.float64)).cuda()
    env, _ = audio.spectral_envelope_device(wav, so, f0, fo)
    env, f0 = env.cpu().numpy(), f0.cpu().numpy()
    return [env[a:b] for a, b in zip(fo[:-1], fo[1:])], [f0[a:b] for a, b in zip(fo[:-1], fo[1:])]


def _log_err(got, want):
    assert got.shape == want.shape
    both_nan = np.isnan(got) & np.isnan(want)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    return float(np.max(np.abs(np.log(got[~both_nan]) - np.log(want[~both_nan])), initial=0.0))


CASES = [(22050, 256), (16000, 200), (24000, 300), (44100, 512), (48000, 600)]


@pytest.mark.parametrize('fs,hop', CASES)
def test_cheaptrick_equals_the_restatement(fs, hop):
    audio = _audio(fs, hop)
    n = audio.cheaptrick_fft_size
    fp = hop / fs * 1000
    rng = np.random.default_rng(fs)
    secs = [1.0, 10.0, 3.3] if fs == 22050 else [1.2, 2.1]
    clips = [po.speech_like_clip(s, seed=int(rng.integers(1 << 30)), fs=float(fs)) for s in secs]
    clips.append(np.zeros(int(0.5 * fs), np.float32))                      # digital silence
    envs, f0s = _envelopes(audio, clips)
    worst = 0.0
    for c, (x, env, f0) in enumerate(zip(clips, envs, f0s)):
        # both clip edges, unvoiced and voiced frames (every frame of the short clips, a stride through the long one)
        frames = sorted(set(range(0, len(f0), 1 if len(f0) < 300 else 7)) | {len(f0) - 1, len(f0) - 2})
        for i in frames:
            want = wo.cheaptrick_frame(x, fs, i, fp, float(f0[i]), n)
            worst = max(worst, _log_err(env[i], want))
        assert np.isfinite(env).all(), c
        assert (f0 == 0).any(), c
    print(f'MEASURED cheaptrick fs {fs} fft {n}: max |log env - log restated| = {worst:.3e}')
    assert worst < LOG_TOL


def test_cheaptrick_f0_edges():
    """F0 at and just above the floor, unvoiced, at fs / 4 and above it (NaN), and NaN."""
    fs, hop = 22050, 256
    audio = _audio(fs, hop)
    n = audio.cheaptrick_fft_size
    fp = hop / fs * 1000
    x = po.speech_like_clip(1.0, seed=9)
    T = wo.n_frames(len(x), fs, fp)
    floor = 3.0 * fs / (n - 3.0)
    special = [floor, np.nextafter(floor, np.inf), 0.0, -5.0, fs / 4.0, np.nextafter(fs / 4.0, np.inf), np.nan, 71.0, 800.0]
    f0 = np.resize(np.array(special), T)
    envs, _ = _envelopes(audio, [x], [f0])
    worst = 0.0
    for i in range(T):
        want = wo.cheaptrick_frame(x, fs, i, fp, float(f0[i]), n)
        worst = max(worst, _log_err(envs[0][i], want))
    assert np.isnan(envs[0][5]).all() and np.isnan(envs[0][6]).all() and np.isfinite(envs[0][4]).all()
    # at or below the floor the frame takes 500 Hz
    assert np.array_equal(_bits(envs[0][0]), _bits(_envelopes(audio, [x], [np.where(np.arange(T) == 0, 500.0, f0)])[0][0][0]))
    print(f'MEASURED cheaptrick F0 edges: max |log env - log restated| = {worst:.3e}')
    assert worst < LOG_TOL


def test_envelopes_and_mceps_do_not_depend_on_the_batch():
    audio = _audio(22050, 256)
    clips = po.make_corpus(7, seed=3)
    full, _ = _envelopes(audio, clips)
    rev, _ = _envelopes(audio, clips[::-1])
    split = _envelopes(audio, clips[:3])[0] + _envelopes(audio, clips[3:])[0]
    for c in range(len(clips)):
        alone = _envelopes(audio, [clips[c]])[0][0]
        for other in (rev[len(clips) - 1 - c], split[c], alone):
            assert np.array_equal(_bits(full[c]), _bits(other)), c
    mc = audio.world_mcep_batch(clips)
    mc_rev = audio.world_mcep_batch(clips[::-1])
    mc_split = audio.world_mcep_batch(clips[:3]) + audio.world_mcep_batch(clips[3:])
    for c in range(len(clips)):
        assert np.array_equal(_bits(mc[c]), _bits(mc_rev[len(clips) - 1 - c])), c
        assert np.array_equal(_bits(mc[c]), _bits(mc_split[c])), c
        assert np.array_equal(_bits(mc[c]), _bits(audio.world_mcep_batch([clips[c]])[0])), c
    # sp2mc against the restatement on the GPU's own envelopes
    from transformertts_b200.utils import evaluation as ev
    alpha = ev.mcep_alpha(22050)
    worst = max(float(np.abs(mc[c][i] - wo.sp2mc(full[c][i], 24, alpha)).max()) for c in (0, 4) for i in range(0, len(full[c]), 5))
    print(f'MEASURED sp2mc: max |mc - restated| = {worst:.3e}')
    assert worst < MCEP_TOL


def test_mcd_dtw_ceps_equals_mcd_dtw_bit_for_bit():
    from transformertts_b200 import lib
    from transformertts_b200.utils import evaluation as ev
    rng = np.random.default_rng(12)
    lens = [(1, 1), (1, 300), (300, 1), (97, 384), (700, 650), (1200, 1100), (33, 31)]
    a = [np.clip(rng.normal(-5, 2, (tx, 80)), -11.5, 2).astype(np.float32) for tx, _ in lens]
    b = [np.clip(rng.normal(-5, 2, (ty, 80)), -11.5, 2).astype(np.float32) for _, ty in lens]
    dct = eo.dct_matrix(80, 24)
    xo = np.concatenate([[0], np.cumsum([len(m) for m in a])])
    yo = np.concatenate([[0], np.cumsum([len(m) for m in b])])
    x, y = torch.from_numpy(np.concatenate(a)).cuda(), torch.from_numpy(np.concatenate(b)).cuda()
    # the cepstra the existing kernel computes (the restatement's bits), with one extra leading column scored from first = 1
    ca = np.concatenate([eo.cepstra(m, dct) for m in a])
    cb = np.concatenate([eo.cepstra(m, dct) for m in b])
    pad = lambda c: torch.from_numpy(np.concatenate([rng.normal(size=(len(c), 1)), c, rng.normal(size=(len(c), 2))], axis=1)).cuda()
    n = len(lens)
    starts = np.concatenate([[0], np.cumsum([tx + ty - 1 for tx, ty in lens])])
    outs = {}
    for name in ('mel', 'ceps'):
        for path in (False, True):
            cost = torch.empty(n, dtype=torch.float64, device='cuda')
            ln = torch.empty(n, dtype=torch.int32, device='cuda')
            p = torch.full((int(starts[-1]), 2), -1, dtype=torch.int32, device='cuda') if path else None
            dev = torch.from_numpy(dct).cuda()
            if name == 'mel' and not path:
                lib.mcd_dtw(x, xo, y, yo, dev, ev.KAPPA, cost, ln)
            elif name == 'mel':
                lib.mcd_dtw_path(x, xo, y, yo, dev, ev.KAPPA, cost, ln, p)
            else:
                lib.mcd_dtw_ceps(pad(ca), xo, pad(cb), yo, 1, 24, ev.KAPPA, cost, ln, p)
            outs[name, path] = (cost.cpu().numpy(), ln.cpu().numpy(), None if p is None else p.cpu().numpy())
    for path in (False, True):
        m, c = outs['mel', path], outs['ceps', path]
        assert np.array_equal(_bits(m[0]), _bits(c[0])) and np.array_equal(m[1], c[1]), path
        if path:
            for i in range(n):
                L = int(m[1][i])
                assert np.array_equal(m[2][starts[i]:starts[i] + L], c[2][starts[i]:starts[i] + L]), i


# ---- evaluate_tts.py --mcep end to end
def _model_cfg():
    from oracle import forward_oracle as fo
    return dict(fo.CONFIGS['C1'], sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                normalizer='MelGAN', data_name='ljspeech')


def _write_wav(path, y, fs):
    pcm = np.clip(np.rint(np.asarray(y, np.float64) * 32767), -32768, 32767).astype('<i2')
    with wave.open(str(path), 'wb') as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(fs)
        f.writeframes(pcm.tobytes())


def _setup(tmp_path):
    """A seeded model and a data directory of 5 validation lines whose mels come from wavs under wav_directory (one of them at
    44.1 kHz, resampled), with volume normalisation on, as create_training_data.py prepares them."""
    from oracle import forward_oracle as fo
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.data.text import ALL_PHONEMES
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    raw = yaml.safe_load((ROOT / 'config' / 'training_config.yaml').read_text())
    raw['paths'].update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'),
                        wav_directory=str(tmp_path / 'wavs'))
    raw['audio_settings'].update(norm_wav=True, target_dBFS=-30.0, int16_max=32767)
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(raw))
    cm = TrainingConfigManager(str(tmp_path / 'cfg.yaml'))
    for d in (cm.data_dir, cm.mel_dir, cm.duration_dir, cm.pitch_per_char, cm.wav_directory):
        d.mkdir(parents=True, exist_ok=True)
    rng = np.random.default_rng(51)
    letters = [c for c in ALL_PHONEMES if c.isalpha()][:30] + [' ']
    lines = {f'r{i:03d}': ''.join(rng.choice(letters, int(rng.integers(6, 24)))) for i in range(5)}
    paths = []
    for i, name in enumerate(lines):
        fs = 44100 if i == 2 else 22050
        _write_wav(cm.wav_directory / f'{name}.wav', po.speech_like_clip(float(rng.uniform(1.0, 3.0)), seed=600 + i, fs=fs) * 0.5, fs)
        paths.append(cm.wav_directory / f'{name}.wav')
    audio = Audio.from_config(cm.config)
    for name, ph, m in zip(lines, lines.values(), audio.mel_spectrogram_ragged(audio.load_wavs(paths))):
        np.save(cm.mel_dir / f'{name}.npy', m)
        T = m.shape[0]
        np.save(cm.duration_dir / f'{name}.npy', np.bincount(rng.integers(0, len(ph), T), minlength=len(ph)).astype(np.int32))
        np.save(cm.pitch_per_char / f'{name}.npy', rng.normal(0, 1, len(ph)).astype(np.float32))
    cm.valid_metadata_path.write_text(''.join(f'{n}|{p}\n' for n, p in lines.items()), encoding='utf-8')
    p = fo.init_params(_model_cfg(), seed=7)
    p['dur_pred.out.b'] = torch.tensor([3.0])
    model = ForwardTransformer(**_model_cfg())
    model.set_weights(p)
    model.save_model(tmp_path / 'model', with_optimizer=False)
    return cm, lines


def _run(args):
    r = subprocess.run([sys.executable, str(ROOT / 'evaluate_tts.py')] + args, capture_output=True, text=True, timeout=900,
                       cwd=str(ROOT))
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def _restated_mcd(wav, rec, audio, f0_wav, f0_rec, alpha):
    fp = audio.hop_length / audio.sampling_rate * 1000
    ma = np.stack([wo.sp2mc(s, 24, alpha) for s in wo.cheaptrick(wav, audio.sampling_rate, f0_wav, fp)])
    mb = np.stack([wo.sp2mc(s, 24, alpha) for s in wo.cheaptrick(rec, audio.sampling_rate, f0_rec, fp)])
    cost, length = eo.dtw(eo.frame_distances(ma[:, 1:], mb[:, 1:]))
    return cost / length


def test_evaluate_tts_mcep_against_the_restatement(tmp_path):
    from predict_tts import VOCODE_CHUNK, vocode_chunk
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils import evaluation as ev
    cm, lines = _setup(tmp_path)
    common = ['--config', str(tmp_path / 'cfg.yaml'), '-p', str(tmp_path / 'model'), '--vocoder', 'griffinlim']
    out = _run(common + ['-o', str(tmp_path / 'mcep'), '--mcep'])
    assert 'WORLD MCD vocoded' in out
    _run(common + ['-o', str(tmp_path / 'plain')])
    doc = json.loads((tmp_path / 'mcep' / 'evaluation.json').read_text())
    assert doc['mcep_order'] == 24 and doc['mcep_alpha'] == ev.mcep_alpha(22050)
    res = doc['checkpoints'][0]
    plain_doc = json.loads((tmp_path / 'plain' / 'evaluation.json').read_text())
    assert 'mcep_order' not in plain_doc and 'mcep_alpha' not in plain_doc
    plain = plain_doc['checkpoints'][0]
    keys = {p + k for p in ('vocoded_', 'copy_synthesis_') for k in ev.MCEP_KEYS}
    assert not keys & set(plain['mean']) and all(not keys & set(ln) for ln in plain['lines'])
    for ln, pl in zip(res['lines'], plain['lines']):
        assert {k: v for k, v in ln.items() if k not in keys} == pl, ln['name']
    assert {k: v for k, v in res['mean'].items() if k not in keys} == plain['mean']

    # the same waveforms in this process, scored by the restatement at the GPU's F0
    model = ForwardTransformer.load_model(tmp_path / 'model')
    audio = Audio.from_config(model.config)
    vs = ev.load_validation_set(cm, recordings=True)
    outs = model.predict_batch(ev.tokenize(model, vs.phonemes), encode=False, phoneme_max_duration=None)
    alpha = ev.mcep_alpha(22050)
    rec_f0 = audio.extract_pitch_batch(vs.recordings)
    worst = 0.0
    for prefix, mels in (('vocoded_', [o['mel'].cpu().numpy() for o in outs]), ('copy_synthesis_', vs.mels)):
        wavs = []
        for start in range(0, len(mels), VOCODE_CHUNK):
            wavs.extend(vocode_chunk(None, audio, [m.T for m in mels[start:start + VOCODE_CHUNK]], start))
        f0s = audio.extract_pitch_batch(wavs)
        for i, ln in enumerate(res['lines']):
            want = _restated_mcd(wavs[i], vs.recordings[i], audio, f0s[i], rec_f0[i], alpha)
            got = ln[prefix + 'mcep_mcd']
            worst = max(worst, abs(got - want) / want)
            assert got == pytest.approx(want, rel=MCD_REL), (prefix, ln['name'], got, want)
    print(f'MEASURED end to end: max relative MCD difference = {worst:.3e}')
    # the recordings against themselves
    rec_mc = audio.world_mcep_batch(vs.recordings)
    cost, length, mcd = ev.mcep_mcd_dtw(rec_mc, rec_mc, 24)
    assert np.all(mcd == 0.0) and np.array_equal(length, [len(m) for m in rec_mc])


def test_load_validation_set_refuses_a_recording_that_does_not_match_its_mel(tmp_path):
    from transformertts_b200.utils import evaluation as ev
    cm, lines = _setup(tmp_path)
    name = next(iter(lines))
    m = np.load(cm.mel_dir / f'{name}.npy')
    np.save(cm.mel_dir / f'{name}.npy', m[:-1])
    with pytest.raises(ValueError, match=f'line {name}: the recording rebuilt'):
        ev.load_validation_set(cm, recordings=True)
