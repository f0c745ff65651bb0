"""The WaveRNN generator on the GPU against the float64 oracle (oracle/wavernn_oracle.py): the frame-rate conditioning, the
recurrence replayed teacher-forced on the GPU's own samples (logits of every step, every draw), the default fold size, one
fold per clip, per-clip determinism, and predict_tts.py --vocoder wavernn end to end.

Gates are about twice the errors measured on an H100 (DESIGN.md §13 records them)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.io.wavfile
import torch

from oracle import wavernn_oracle as wo
from transformertts_b200.model import wavernn as wr

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent

# precision -> relative conditioning and logits errors, MOL sample error
GATES = {'bf16x3': dict(cond=3e-5, logits=2.5e-5, sample=3e-5), 'bf16': dict(cond=2e-2, logits=1.6e-2, sample=2.5e-2)}
# decisions closer than this to their boundary (Gumbel score gap in MOL, CDF distance in RAW) are excluded from the draw
# check, and may be at most the given share of the steps
MARGIN = {('MOL', 'bf16x3'): 1e-3, ('MOL', 'bf16'): 0.05, ('RAW', 'bf16x3'): 1e-5, ('RAW', 'bf16'): 1e-3}
MAX_EXCLUDED = {('MOL', 'bf16x3'): 0.0025, ('MOL', 'bf16'): 0.09, ('RAW', 'bf16x3'): 0.04}
# bf16 RAW moves the 512-class CDF by more than most class intervals are wide, so nearly every draw is close to a boundary:
# there the draws are gated on how far the GPU's class lands from the oracle's, over every step (share that differ, and the
# 99th percentile and maximum of |k_gpu - k_oracle|)
RAW_BF16_CLASS = dict(differ=0.035, p99=2, max=2)
TGT, OVL = 40, 10


def _gen(mode, precision, seed=0, bits=9):
    sd = wo.init_state_dict(seed=seed, mode=mode, bits=bits)
    return sd, wr.WaveRNNGenerator(precision=precision).load_state_dict(sd)


def _fm(mels):
    return [wo.to_fatchord(m).astype(np.float32) for m in mels]


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
def test_conditioning(precision):
    sd, g = _gen('MOL', precision)
    net = wo.build(sd)
    mels = wo.make_mels([21, 22, 47, 300], seed=1)
    aux, melp, auxp = g.conditioning(_fm(mels))
    torch.cuda.synchronize()
    H = g.halo
    val = lambda p: (p[0].float() + (p[1].float() if p[1] is not None else 0)).cpu().numpy()   # noqa: E731
    aux_g, melp_g, auxp_g = val(aux), val(melp), val(auxp)
    Iw = sd['I.weight'].numpy()
    Wih1 = sd['rnn1.weight_ih_l0'].numpy()
    A = 32
    err = dict(aux=0.0, melp=0.0, auxp=0.0)
    r = 0
    for m in mels:
        T = m.shape[1]
        x = torch.from_numpy(wo.to_fatchord(m))[None]
        with torch.no_grad():
            a = net.upsample.resnet(torch.nn.functional.pad(x, (2, 2)))[0].numpy().T          # (T, 128)
        mm = wo.to_fatchord(m).T
        want_melp = np.concatenate([mm @ Iw[:, 1:81].T, mm @ (Wih1 @ Iw[:, 1:81]).T], 1)
        want_auxp = np.concatenate([a[:, :A] @ Iw[:, 81:].T, a[:, :A] @ (Wih1 @ Iw[:, 81:]).T,
                                    a[:, A:2 * A] @ sd['rnn2.weight_ih_l0'].numpy()[:, 512:].T, a[:, 2 * A:3 * A] @ sd['fc1.weight'].numpy()[:, 512:].T,
                                    a[:, 3 * A:] @ sd['fc2.weight'].numpy()[:, 512:].T], 1)
        rows = slice(r + H, r + H + T)
        for k, got, want in (('aux', aux_g[rows, :128], a), ('melp', melp_g[rows], want_melp), ('auxp', auxp_g[rows], want_auxp)):
            err[k] = max(err[k], float(np.abs(got - want).max() / max(1.0, np.abs(want).max())))
        assert not melp_g[r:r + H].any() and not melp_g[r + H + T:r + 2 * H + T].any()
        r += T + 2 * H
    print(f'conditioning {precision}: relative max errors {err}')
    assert max(err.values()) < GATES[precision]['cond'], err


def _replay_check(mode, precision, bits=9, lengths=(21, 22, 47), seed=0, batched=True, target=TGT, overlap=OVL):
    sd, g = _gen(mode, precision, seed=seed, bits=bits)
    mels = wo.make_mels(list(lengths), seed=seed + 10)
    seeds = [5 + c for c in range(len(mels))]
    rows, L = wr.fold_rows([m.shape[1] for m in mels], g.hop, batched, target, overlap)
    cap_steps = min(L, 64)
    wav, cap, samples = g._generate(_fm(mels), seeds, batched, target, overlap, capture_steps=cap_steps, keep_samples=True)
    wav, cap, samples = wav.cpu().numpy(), cap.cpu().numpy(), samples.cpu().numpy()
    net = wo.build(sd, device='cuda')
    rep = wo.replay(net, mels, samples, seeds, batched, target, overlap, capture_steps=cap_steps)
    lerr = float(np.abs(cap - rep['logits']).max() / max(1.0, np.abs(rep['logits']).max()))
    if (mode, precision) == ('RAW', 'bf16'):
        n = 2 ** bits
        dk = np.abs(np.rint((samples + 1) * (n - 1) / 2) - np.rint((rep['draws'] + 1) * (n - 1) / 2))
        cls = dict(differ=float((dk > 0).mean()), p99=float(np.percentile(dk, 99)), max=float(dk.max()))
        keep = np.ones_like(dk, dtype=bool)
        print(f'replay RAW bf16 class distance: {cls}')
        assert all(cls[k] <= RAW_BF16_CLASS[k] for k in cls), cls
    else:
        keep = rep['margins'] >= MARGIN[mode, precision]
    excluded = float(1.0 - keep.mean())
    serr = float(np.abs(samples - rep['draws'])[keep].max())
    # the crossfade, crop and fade-out of the GPU's own samples
    y = samples.astype(np.float64)
    if mode == 'RAW':
        y = wo.decode_mu_law(y, 2 ** bits, False)
    off, werr = 0, 0.0
    for c, m in enumerate(mels):
        mine = [i for i, rw in enumerate(rows) if rw[0] == c]
        want = wo.xfade_and_unfold(y[mine].copy(), target, overlap) if batched else y[mine[0]]
        wl = (m.shape[1] - 1) * g.hop
        want = want[:wl].copy()
        want[-20 * g.hop:] *= np.linspace(1, 0, 20 * g.hop)
        werr = max(werr, float(np.abs(wav[off:off + wl] - want).max()))
        off += wl
    print(f'replay {mode} {precision}: {len(rows)} folds x {L} steps, logits rel err {lerr:.3e}, sample err {serr:.3e}, '
          f'excluded {excluded:.4f}, unfold err {werr:.3e}')
    gt = GATES[precision]
    assert lerr < gt['logits'], lerr
    if (mode, precision) != ('RAW', 'bf16'):
        assert excluded < MAX_EXCLUDED[mode, precision], excluded
        assert serr < (gt['sample'] if mode == 'MOL' else 1e-6), serr
    assert werr < 1e-6, werr
    return g, mels, seeds


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('mode', ['MOL', 'RAW'])
def test_replay(mode, precision):
    _replay_check(mode, precision)


@pytest.mark.parametrize('overlap', [1, 2, 3])
def test_replay_small_overlap(overlap):
    """Overlaps whose fades are one or two points long (np.linspace(-1, 1, 1) is [-1])."""
    _replay_check('MOL', 'bf16x3', lengths=(21,), overlap=overlap)


def test_replay_raw_10_bits():
    _replay_check('RAW', 'bf16x3', bits=10, lengths=(23,))


def test_unbatched_is_one_fold():
    g, mels, seeds = _replay_check('MOL', 'bf16x3', lengths=(21, 24), batched=False)
    rows, L = wr.fold_rows([21, 24], g.hop, False, TGT, OVL)
    assert len(rows) == 2 and L == 24 * 275


def test_default_fold_size():
    """One ~3 s clip at target 11000 / overlap 550: 241 frames -> 66275 samples -> 6 folds of 12100 steps."""
    sd, g = _gen('MOL', 'bf16x3', seed=4)
    assert wr.fold_count(241 * 275, 11000, 550) == 6
    mels = wo.make_mels([241], seed=5)
    wav, cap, samples = g._generate(_fm(mels), [0], True, 11000, 550, capture_steps=16, keep_samples=True)
    assert samples.shape == (6, 12100) and wav.shape == (240 * 275,)
    net = wo.build(sd, device='cuda')
    # teacher-forced replay of the first 600 steps of every fold
    rep = wo.replay(net, mels, samples.cpu().numpy()[:, :600].copy(), [0], True, 11000, 550, capture_steps=16, steps=600)
    lerr = float(np.abs(cap.cpu().numpy() - rep['logits']).max() / max(1.0, np.abs(rep['logits']).max()))
    keep = rep['margins'] >= MARGIN['MOL', 'bf16x3']
    serr = float(np.abs(samples.cpu().numpy()[:, :600] - rep['draws'])[keep].max())
    print(f'default folds: logits rel err {lerr:.3e}, sample err {serr:.3e}, excluded {1 - keep.mean():.4f}')
    assert lerr < GATES['bf16x3']['logits'] and serr < GATES['bf16x3']['sample'] and 1 - keep.mean() < MAX_EXCLUDED['MOL', 'bf16x3']
    # the equal-power crossfade of two folds reaches sqrt(2) of a fold's full scale
    assert np.isfinite(wav.cpu().numpy()).all() and np.abs(wav.cpu().numpy()).max() <= np.sqrt(2.0) + 1e-6


def test_per_clip_determinism():
    _, g = _gen('MOL', 'bf16x3', seed=6)
    mels = wo.make_mels([21, 30, 22, 45, 26], seed=7)
    kw = dict(target=TGT, overlap=OVL)
    alone = [g.vocode_batch([m], seeds=[100 + c], **kw)[0] for c, m in enumerate(mels)]
    batch = g.vocode_batch(mels, seeds=[100 + c for c in range(5)], **kw)
    for c in range(5):
        assert np.array_equal(batch[c], alone[c]), c
    for shift in range(1, 5):   # every position
        order = [(c + shift) % 5 for c in range(5)]
        out = g.vocode_batch([mels[c] for c in order], seeds=[100 + c for c in order], **kw)
        for j, c in enumerate(order):
            assert np.array_equal(out[j], alone[c]), (shift, c)
    for n in (1, 3, 64):
        out = g.vocode_batch([mels[0]] * n, seeds=[100] * n, **kw)
        assert all(np.array_equal(o, alone[0]) for o in out), n
    assert np.array_equal(g.vocode_batch([mels[1]], seeds=[101], **kw)[0], alone[1])          # run to run
    assert not np.array_equal(g.vocode_batch([mels[1]], seeds=[102], **kw)[0], alone[1])      # another seed


def _predict(tmp_path, lines, ckpt, name):
    (tmp_path / f'{name}.txt').write_text('\n'.join(lines) + '\n')
    return subprocess.run([sys.executable, str(ROOT / 'predict_tts.py'), '-p', str(tmp_path / 'model'), '-f', str(tmp_path / f'{name}.txt'),
                           '-o', str(tmp_path / 'out'), '-m', '-s', '--vocoder', 'wavernn', '--vocoder_checkpoint', str(ckpt)],
                          capture_output=True, text=True, timeout=900, cwd=str(ROOT))


def test_predict_tts_end_to_end(tmp_path):
    """predict_tts.py --vocoder wavernn with a seeded ForwardTransformer at the WaveRNN audio section: line i's file is
    (T_i - 1) 275 samples, the bytes save_wav writes for vocode_batch of its stored mel with seed i."""
    import predict_tts
    from oracle import forward_oracle as fo
    from transformertts_b200.data.audio import Audio
    from transformertts_b200.model.models import ForwardTransformer
    audio_cfg = dict(sampling_rate=22050, n_fft=2048, hop_length=275, win_length=1100, f_min=40, f_max=11025, normalizer='WaveRNN')
    cfg = dict(fo.CONFIGS['C1'], data_name='ljspeech', **audio_cfg)
    p = fo.init_params(cfg, seed=7)
    p['dur_pred.out.b'] = torch.tensor([6.0])
    model = ForwardTransformer(**cfg)
    model.set_weights(p)
    model.save_model(tmp_path / 'model', with_optimizer=False)
    sd = wo.init_state_dict(seed=8)
    ckpt = tmp_path / 'latest_weights.pyt'
    torch.save(sd, ckpt)
    lines = ['həloʊ wɜːld', 'ðɪs ɪz ɐ lɔŋɡɚ tɛst sɛntəns.', 'ɐbɐ ɐbɐ ɐbɐ']
    r = _predict(tmp_path, lines, ckpt, 'lines')
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    out = tmp_path / 'out' / 'outputs' / 'lines'
    stem = 'lines_ljspeech_unknown_0'
    g = wr.WaveRNNGenerator(precision='bf16x3').load_state_dict(sd)
    a = Audio(mel_channels=80, **audio_cfg)
    for i in range(len(lines)):
        mel = np.load(out / f'{stem}_{i}.mel.npy')
        assert mel.shape[0] >= wr.MIN_FRAMES, (i, mel.shape)
        a.save_wav(g.vocode_batch([mel.T], seeds=[i])[0], tmp_path / f'want_{i}.wav')
        _, want = scipy.io.wavfile.read(tmp_path / f'want_{i}.wav')
        sr, got = scipy.io.wavfile.read(out / f'{stem}_{i}.wav')
        assert sr == 22050 and got.dtype == np.int16 and got.shape == (275 * (mel.shape[0] - 1),), i
        assert np.array_equal(got, want), i
    # a line below 21 frames is refused by its index
    r = _predict(tmp_path, [lines[0], 'ɐ'], ckpt, 'short')
    assert r.returncode != 0 and 'line 1 gives a mel of' in r.stderr, (r.stdout[-2000:], r.stderr[-3000:])
    # a model at another hop, or with another normaliser, is refused
    m = ForwardTransformer(**dict(cfg, hop_length=256))
    with pytest.raises(SystemExit, match='hop_length 256'):
        predict_tts.load_vocoder('wavernn', str(ckpt), None, m)
    m = ForwardTransformer(**dict(cfg, normalizer='MelGAN'))
    with pytest.raises(SystemExit, match='normaliser'):
        predict_tts.load_vocoder('wavernn', str(ckpt), None, m)
