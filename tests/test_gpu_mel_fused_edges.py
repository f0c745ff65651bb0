"""The fused log-mel kernels (csrc/stft_mel.cu: ttsb_stft_mel_log, ttsb_stft_mel_log_batch) against float64 for every mel basis
and frame-pair edge.

Contract under test (include/ttsb.h).  For clip y (L > 512 fp32 samples) and basis rows b_m (fp32, non-zero only inside the
host band table), frame t of the output is
    MelGAN : log(max(S[t, m], 1e-5f)),   WaveRNN : clip((20 log10(max(S, 1e-5f)) + 100) / 100, 0, 1) * 8 - 4,
    S[t, m] = sum_k b_m[k] |rfft(hann * x_t)[k]|,  x_t = reflect_pad(y, 512)[256 t : 256 t + 1024],  t < 1 + L // 256.
The reference (_spectrum, _mel64) states exactly that in float64 on the float32 samples and basis the kernels receive.  The
kernels transform frames 2j and 2j + 1 as one complex FFT and separate the two spectra; a basis whose bands span at most
2048 weights runs the packed persistent kernel, a wider one the v1 kernel in the single-clip path and is refused by the batch.

Error model.  A radix-2^k fp32 FFT of 1024 points is off per bin by about u log2(1024) times the 2-norm of its input, here
the two windowed frames sharing one transform: e_t = C u 10 sqrt(|w_A|^2 + |w_B|^2), u = 2^-24 (the partner of an unpaired
last frame is zero).  A mel sum adds its fmaf chain and the magnitude rounding, (len_m + 4) u sum_k |b_mk| |X_k|, so
    E_tm = e_t sum_k |b_mk| + (len_m + 4) u sum_k |b_mk| |X_tk|,
    MelGAN |got - ref| <= E / max(S, 1e-5) + 8 u |ref| (logf),   WaveRNN: that times 20 / ln 10 * 8 / 100, + 128 u.
Where the WaveRNN value before the clip lies below 0 or above 1 by more than its bound, the output must be -4 or 4 exactly.
A bin read from the wrong frame, a band shifted by one bin or a stale filterbank is off by many bounds.
"""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from gpu_util import DEV
from transformertts_b200 import lib
from transformertts_b200.data.audio import Audio, mel_band, slaney_mel_basis

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
U = 2.0 ** -24
C_FFT = 4.0                                      # the one constant of the bound (largest err / bound printed at the end)
CLAMP = float(np.float32(1e-5))
HANN = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(1024) / 1024)
WAVERNN_SLOPE = 20.0 / np.log(10.0) * 8.0 / 100.0
RATIOS = {}                                      # case -> largest err / bound

# (sr, n_mels, f_min, f_max): the shipped basis first
BASES = [(22050, 80, 0, 8000), (22050, 128, 0, None), (16000, 80, 0, 8000), (24000, 100, 0, 12000), (44100, 128, 40, None),
         (48000, 128, 0, None), (22050, 1, 0, 8000), (22050, 20, 300, 3000)]
# every frame-pair and reflection edge: 3 frames (last pair single, both edges reflected) .. 10 s; odd and even frame counts
LENGTHS = [513, 767, 768, 1023, 1024, 1025] + [256 * k + d for k in (5, 6, 9, 10) for d in (-1, 0, 1)] + [220500]


def _clip(L: int, seed: int) -> np.ndarray:
    """float32 test clip: noise, a DC offset and a Nyquist tone (so bins 0 and 512 carry energy), two tones; clips of a second
    or more also get a loud 0.004-cycle (88 Hz at 22.05 kHz) segment and 8192 samples of digital silence."""
    rng = np.random.default_rng(seed)
    t = np.arange(L)
    y = (0.05 * rng.standard_normal(L) + 0.01 + 0.02 * (-1.0) ** t + 0.2 * np.sin(2 * np.pi * 0.031 * t)
         + 0.1 * np.sin(2 * np.pi * 0.27 * t + 1.0)) * (0.3 + 0.7 * np.abs(np.sin(2 * np.pi * t / 9000.0)))
    if L >= 20000:
        y[L // 8:L // 4] = 0.9 * np.sin(2 * np.pi * 0.004 * t[L // 8:L // 4])
        y[L // 2:L // 2 + 8192] = 0.0
    return y.astype(np.float32)


_SPEC = {}


def _spectrum(y: np.ndarray):
    """float64 (|X| (T, 513), e (T,)) of a float32 clip: reflect pad 512, exact periodic Hann, rfft; e is the per-bin FFT bound."""
    key = (len(y), hash(y.tobytes()))
    if key not in _SPEC:
        if len(_SPEC) > 400:
            _SPEC.clear()
        x = np.pad(y.astype(np.float64), 512, mode='reflect')
        T = 1 + len(y) // 256
        fr = x[np.arange(T)[:, None] * 256 + np.arange(1024)[None, :]] * HANN
        n2 = (fr * fr).sum(1)
        partner = np.zeros(T)
        even, odd = np.arange(0, T - 1, 2), np.arange(1, T, 2)
        partner[even], partner[odd] = n2[even + 1], n2[odd - 1]
        _SPEC[key] = (np.abs(np.fft.rfft(fr, axis=1)), C_FFT * U * 10.0 * np.sqrt(n2 + partner))
    return _SPEC[key]


def _mel64(y: np.ndarray, basis: np.ndarray):
    """float64 (S, E) (T, n_mels) of a clip for a float32 basis (n_mels, 513)."""
    mag, e = _spectrum(y)
    b = np.abs(basis.astype(np.float64))
    length = np.array([hi - lo for lo, hi in mel_band(basis)], dtype=np.float64)
    S = mag @ basis.astype(np.float64).T
    E = e[:, None] * b.sum(1)[None, :] + (length + 4.0)[None, :] * U * (mag @ b.T)
    return S, E


def _check(case: str, got, y: np.ndarray, basis: np.ndarray, normalizer: int):
    """got (T, n_mels) against the float64 reference under the bound; records the largest err / bound of the case."""
    got = got.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(got) else np.asarray(got, dtype=np.float64)
    S, E = _mel64(y, basis)
    assert got.shape == S.shape, (case, got.shape, S.shape)
    Sc = np.maximum(S, CLAMP)
    if normalizer == 0:
        ref = np.log(Sc)
        bound = E / Sc + 8 * U * np.maximum(np.abs(ref), 1.0)
    else:
        pre = (20.0 * np.log10(Sc) + 100.0) / 100.0
        ref = np.clip(pre, 0.0, 1.0) * 8.0 - 4.0
        bound = E / Sc * WAVERNN_SLOPE + 128 * U
        low, high = pre < -bound / 8.0, pre > 1.0 + bound / 8.0
        assert np.all(got[low] == -4.0) and np.all(got[high] == 4.0), case
    ratio = np.abs(got - ref) / bound
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert np.all(np.isfinite(got)) and ratio.max() <= 1.0, (
        f'{case}: frame {worst[0]} mel {worst[1]}: got {got[worst]!r} ref {ref[worst]!r} err/bound {ratio[worst]:.3g}')
    RATIOS[case] = max(RATIOS.get(case, 0.0), float(ratio.max()))
    return ratio


def _audio(sr, n_mels, f_min, f_max, normalizer='MelGAN') -> Audio:
    return Audio(sampling_rate=sr, n_fft=1024, mel_channels=n_mels, hop_length=256, win_length=1024, f_min=f_min, f_max=f_max,
                 normalizer=normalizer, device=DEV)


def _dev(y: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(y)).to(DEV)


def _fused(wav: torch.Tensor, basis: torch.Tensor, band, normalizer: int) -> torch.Tensor:
    """ttsb_stft_mel_log of (n_clips, L) clips -> (n_clips, T, n_mels); the output starts as NaN."""
    n, L = wav.shape
    out = torch.full((n, 1 + L // 256, basis.shape[0]), float('nan'), device=DEV)
    lib.stft_mel_log(wav, basis, band, normalizer, out)
    torch.cuda.synchronize()
    return out


def _fused_batch(clips, basis: torch.Tensor, band, normalizer: int):
    """ttsb_stft_mel_log_batch of a list of clips -> list of (T_c, n_mels) CPU tensors."""
    so = np.concatenate([[0], np.cumsum([len(y) for y in clips])])
    fo = np.concatenate([[0], np.cumsum([1 + len(y) // 256 for y in clips])])
    out = torch.full((int(fo[-1]), basis.shape[0]), float('nan'), device=DEV)
    lib.stft_mel_log_batch(_dev(np.concatenate(clips)), so, fo, basis, band, normalizer, out)
    out = out.cpu()
    return [out[fo[c]:fo[c + 1]] for c in range(len(clips))]


# ----------------------------------------------------------------------------------------------------------
# bases from Audio at the reference STFT, every length, both normalisers, single clip and batch
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sr,n_mels,f_min,f_max', BASES)
def test_audio_bases_every_length(sr, n_mels, f_min, f_max):
    clips = [_clip(L, seed=L) for L in LENGTHS]
    for norm_name, code in (('MelGAN', 0), ('WaveRNN', 1)):
        a = _audio(sr, n_mels, f_min, f_max, norm_name)
        basis = a._mel_basis().cpu().numpy()
        case = f'audio {sr} {n_mels} {f_min}-{f_max} {norm_name}'
        alone = []
        for y in clips:
            got = a.mel_spectrogram_device(_dev(y)[None])[0]
            _check(case, got, y, basis, code)
            alone.append(got.cpu())
        # the ragged batch: every clip bit-identical to the clip alone, in two orders
        order = np.random.default_rng(n_mels + code).permutation(len(clips))
        for perm in (np.arange(len(clips)), order):
            packed, so = a._pack([clips[i] for i in perm])
            mel, fo = a.mel_spectrogram_ragged_device(packed, so)
            mel = mel.cpu()
            for j, i in enumerate(perm):
                assert torch.equal(mel[fo[j]:fo[j + 1]], alone[i]), (case, LENGTHS[i])


def test_wavernn_clamps_both_ends():
    """The 10 s clip holds a loud 88 Hz segment (mel far above 1: WaveRNN 4) and digital silence (mel 0: WaveRNN -4)."""
    y = _clip(220500, seed=3)
    a = _audio(22050, 80, 0, 8000, 'WaveRNN')
    got = a.mel_spectrogram_device(_dev(y)[None])[0].cpu().numpy()
    _check('wavernn clamp', got, y, a._mel_basis().cpu().numpy(), 1)
    assert (got == 4.0).sum() > 100
    # frames wholly inside the silence: S = 0 exactly, the clamp value 1e-5f, whose WaveRNN value is -4 up to rounding
    silent = got[(220500 // 2 + 512) // 256 + 1:(220500 // 2 + 8192 - 512) // 256]
    assert silent.size and np.all(silent == silent.flat[0]) and abs(silent.flat[0] + 4.0) <= 128 * U


# ----------------------------------------------------------------------------------------------------------
# hand-made bases through the C ABI
# ----------------------------------------------------------------------------------------------------------
SINGLE_BINS = [0, 1, 2, 255, 256, 257, 510, 511, 512]


@pytest.mark.parametrize('normalizer', [0, 1])
def test_single_bin_rows_separate_dc_and_nyquist(normalizer):
    """Row i weighs bin SINGLE_BINS[i] by 1: each output is |X_k| of one bin of one frame of the pair."""
    basis = np.zeros((len(SINGLE_BINS), 513), dtype=np.float32)
    basis[np.arange(len(SINGLE_BINS)), SINGLE_BINS] = 1.0
    bd, band = _dev(basis), mel_band(basis)
    assert band.tolist() == [[k, k + 1] for k in SINGLE_BINS]
    clips = [_clip(L, seed=100 + L) for L in LENGTHS]
    for y in clips:
        _check(f'single bins n{normalizer}', _fused(_dev(y)[None], bd, band, normalizer)[0], y, basis, normalizer)
    for y, got in zip(clips, _fused_batch(clips, bd, band, normalizer)):
        assert torch.equal(got, _fused(_dev(y)[None], bd, band, normalizer)[0].cpu())


def _random_banded(bands, seed: int) -> np.ndarray:
    """float32 basis with uniform (0.25, 1) weights inside each [lo, hi) and exact zeros outside."""
    rng = np.random.default_rng(seed)
    basis = np.zeros((len(bands), 513), dtype=np.float32)
    for m, (lo, hi) in enumerate(bands):
        basis[m, lo:hi] = rng.uniform(0.25, 1.0, hi - lo)
    return basis


def test_zero_row_gives_the_clamp_value_in_both_kernels():
    """An all-zero row is 1e-5f after the clamp: the same float32 value in every frame, in the packed and the v1 kernel."""
    packed = _random_banded([(0, 0), (10, 40), (200, 260)], seed=1)
    wide = _random_banded([(0, 0), (0, 513), (0, 513), (0, 513), (0, 513)], seed=2)      # 2052 weights: v1
    y = _clip(5000, seed=5)
    for code, want in ((0, np.log(CLAMP)), (1, (20.0 * np.log10(CLAMP) + 100.0) / 100.0 * 8.0 - 4.0)):
        vals = []
        for basis in (packed, wide):
            got = _fused(_dev(y)[None], _dev(basis), mel_band(basis), code)[0]
            _check(f'zero row n{code}', got, y, basis, code)
            vals.append(got[:, 0].cpu())
        assert torch.equal(vals[0], vals[1]) and torch.all(vals[0] == vals[0][0])
        assert abs(float(vals[0][0]) - want) <= (8 * U * abs(want) if code == 0 else 128 * U)


# 4 rows: 1539 + 509 = 2048 weights (the most the packed table holds) and 1539 + 510 = 2049 (one more)
BANDS_2048 = [(0, 513), (0, 513), (0, 513), (2, 511)]
BANDS_2049 = [(0, 513), (0, 513), (0, 513), (2, 512)]


@pytest.mark.parametrize('normalizer', [0, 1])
def test_packed_table_boundary(normalizer):
    clips = [_clip(L, seed=200 + L) for L in (513, 1024, 1281, 220500)]
    b48, b49 = _random_banded(BANDS_2048, seed=3), _random_banded(BANDS_2049, seed=3)
    assert sum(hi - lo for lo, hi in mel_band(b48)) == 2048 and sum(hi - lo for lo, hi in mel_band(b49)) == 2049
    # 2048 weights: the packed kernel in both paths (its magnitudes differ from v1's in the last bits, so bit-identity of the
    # batch with the single clip says the single clip ran the packed kernel too)
    alone = [_fused(_dev(y)[None], _dev(b48), mel_band(b48), normalizer)[0] for y in clips]
    for y, got in zip(clips, alone):
        _check(f'2048 taps n{normalizer}', got, y, b48, normalizer)
    for got, one in zip(_fused_batch(clips, _dev(b48), mel_band(b48), normalizer), alone):
        assert torch.equal(got, one.cpu())
    # 2049 weights: v1 in the single-clip path, refused by the batch before any launch
    for y in clips:
        _check(f'2049 taps v1 n{normalizer}', _fused(_dev(y)[None], _dev(b49), mel_band(b49), normalizer)[0], y, b49, normalizer)
    lib.reset_launch_count()
    with pytest.raises(lib.TtsbError, match=r'failed \(-3\).*packed filterbank holds \(2048\)'):
        _fused_batch(clips, _dev(b49), mel_band(b49), normalizer)
    assert lib.launch_count() == 0


def test_dense_basis_through_v1():
    """128 dense positive rows (65664 weights): the v1 kernel, one clip and several clips per call."""
    basis = np.random.default_rng(4).uniform(0.0, 1.0, (128, 513)).astype(np.float32) / 64
    basis[:, ::7] += 0.01
    clips = np.stack([_clip(3000, seed=300 + c) for c in range(3)])
    for code in (0, 1):
        got = _fused(_dev(clips), _dev(basis), mel_band(basis), code)
        for c in range(3):
            _check(f'dense v1 n{code}', got[c], clips[c], basis, code)
        assert torch.equal(got[1], _fused(_dev(clips[1])[None], _dev(basis), mel_band(basis), code)[0])


def test_v1_switch_selects_v1_with_the_same_table(tmp_path):
    """TTSB_STFT_V1=1 runs the shipped basis through the v1 kernel: within the bound, and not bit-identical to the packed kernel
    (whose magnitudes are computed differently), so the switch did select v1."""
    code = ('import sys, numpy as np, torch; sys.path.insert(0, %r)\n'
            'from transformertts_b200.data.audio import Audio\n'
            'a = Audio(22050, 1024, 80, 256, 1024, 0, 8000, "MelGAN")\n'
            'y = np.load(%r)\n'
            'np.save(%r, a.mel_spectrogram_device(torch.from_numpy(y).cuda()[None])[0].cpu().numpy())\n')
    y = _clip(20000, seed=7)
    np.save(tmp_path / 'y.npy', y)
    env = dict(os.environ, TTSB_STFT_V1='1')
    flags = ['-s'] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, '-c', code % (str(ROOT), str(tmp_path / 'y.npy'), str(tmp_path / 'v1.npy'))],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    v1 = np.load(tmp_path / 'v1.npy')
    a = _audio(22050, 80, 0, 8000)
    basis = a._mel_basis().cpu().numpy()
    _check('v1 switch', v1, y, basis, 0)
    v2 = a.mel_spectrogram_device(_dev(y)[None])[0].cpu().numpy()
    assert not np.array_equal(v1, v2)


# ----------------------------------------------------------------------------------------------------------
# persistence: the grid-stride loop and the next-pair prefetch across clip boundaries
# ----------------------------------------------------------------------------------------------------------
def test_dense_many_clips_cross_clip_boundaries():
    a = _audio(22050, 80, 0, 8000)
    basis = a._mel_basis().cpu().numpy()
    clips = np.stack([_clip(220500, seed=400 + c) for c in range(40)])   # 40 x 431 pairs > 2 blocks x 132 SMs x 8 warps
    got = a.mel_spectrogram_device(_dev(clips)).cpu()
    for c in range(40):
        _check('40 clips x 10 s', got[c], clips[c], basis, 0)
    for c in (0, 17, 39):
        assert torch.equal(got[c], a.mel_spectrogram_device(_dev(clips[c])[None])[0].cpu())


@pytest.mark.parametrize('sr,n_mels,f_min,f_max,normalizer', [(22050, 80, 0, 8000, 'MelGAN'), (44100, 128, 40, None, 'WaveRNN')])
def test_ragged_batch_of_300_clips(sr, n_mels, f_min, f_max, normalizer):
    rng = np.random.default_rng(n_mels)
    lengths = [513 if i % 3 == 0 else int(rng.integers(514, 40000)) for i in range(300)]
    lengths[7], lengths[150] = 220500, 220500
    clips = [_clip(L, seed=1000 + i) for i, L in enumerate(lengths)]
    a = _audio(sr, n_mels, f_min, f_max, normalizer)
    code = a.normalizer.code
    basis = a._mel_basis().cpu().numpy()
    alone = [a.mel_spectrogram_device(_dev(y)[None])[0].cpu() for y in clips]
    for k, perm in enumerate([np.arange(300), rng.permutation(300), rng.permutation(300)]):
        packed, so = a._pack([clips[i] for i in perm])
        mel, fo = a.mel_spectrogram_ragged_device(packed, so)
        mel = mel.cpu()
        for j, i in enumerate(perm):
            row = mel[fo[j]:fo[j + 1]]
            if k == 0:
                _check(f'300 ragged {n_mels} {normalizer}', row, clips[i], basis, code)
            assert torch.equal(row, alone[i]), (k, i, lengths[i])


# ----------------------------------------------------------------------------------------------------------
# basis identity: the filterbank is the call's own, whatever address it has
# ----------------------------------------------------------------------------------------------------------
def test_basis_rewritten_in_place():
    """One device buffer holds basis A, then B (rewritten in place), then C with fewer rows through a view of the same
    storage: every call matches the reference for the buffer's current contents."""
    storage = torch.zeros(128 * 513, device=DEV)
    y = _clip(9000, seed=11)
    for sr, n_mels, f_min, f_max in [(22050, 80, 0, 8000), (16000, 80, 0, 8000), (22050, 20, 300, 3000), (22050, 80, 0, 8000)]:
        basis = slaney_mel_basis(sr, 1024, n_mels, f_min, f_max)
        view = storage[:n_mels * 513].view(n_mels, 513)
        view.copy_(torch.from_numpy(basis))
        for code in (0, 1):
            _check(f'in place {sr} {n_mels}', _fused(_dev(y)[None], view, mel_band(basis), code)[0], y, basis, code)
            _check(f'in place batch {sr} {n_mels}', _fused_batch([y], view, mel_band(basis), code)[0], y, basis, code)


def test_new_audio_at_a_freed_basis_address():
    """Audio A is used and freed; Audio B with other settings (the same basis size) is correct whether or not the caching
    allocator gives its basis A's address."""
    y = _clip(7000, seed=12)
    a = _audio(22050, 80, 0, 8000)
    a.mel_spectrogram_device(_dev(y)[None])
    ptr_a = a._mel_basis().data_ptr()
    del a
    b = _audio(16000, 80, 0, 8000)
    reused = b._mel_basis().data_ptr() == ptr_a
    print(f'basis address reused: {reused}')
    _check('freed address', b.mel_spectrogram_device(_dev(y)[None])[0], y, b._mel_basis().cpu().numpy(), 0)


def test_two_live_audios_alternate_and_two_streams():
    y = _clip(12000, seed=13)
    a, b = _audio(22050, 80, 0, 8000), _audio(24000, 100, 0, 12000)
    ba, bb = a._mel_basis().cpu().numpy(), b._mel_basis().cpu().numpy()
    first = {}
    for k, (name, au, basis) in enumerate([('A', a, ba), ('B', b, bb)] * 2):
        got = au.mel_spectrogram_device(_dev(y)[None])[0].cpu()
        _check(f'alternate {name}', got, y, basis, 0)
        if name in first:
            assert torch.equal(got, first[name])
        first.setdefault(name, got)
    # both on their own streams, back to back, nothing in between
    wav = _dev(np.stack([_clip(220500, seed=14 + c) for c in range(8)]))
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        out_a = a.mel_spectrogram_device(wav)
    with torch.cuda.stream(s2):
        out_b = b.mel_spectrogram_device(wav)
    torch.cuda.synchronize()
    assert torch.equal(out_a, a.mel_spectrogram_device(wav)) and torch.equal(out_b, b.mel_spectrogram_device(wav))
    _check('stream A', out_a[0], wav[0].cpu().numpy(), ba, 0)
    _check('stream B', out_b[0], wav[0].cpu().numpy(), bb, 0)


def test_single_clip_path_captures_in_a_cuda_graph():
    """The single-clip entry point never waits for the device: a call with a basis it has never seen is captured in a CUDA
    graph and replayed."""
    y = _clip(6000, seed=15)
    _audio(22050, 80, 0, 8000).mel_spectrogram_device(_dev(y)[None])      # the library's one-time set-up on this device
    a = _audio(24000, 100, 0, 12000, 'WaveRNN')
    a._mel_basis()
    wav = _dev(y)[None]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = a.mel_spectrogram_device(wav)
    out.fill_(float('nan'))
    g.replay()
    torch.cuda.synchronize()
    _check('graph replay', out[0], y, a._mel_basis().cpu().numpy(), 1)


# ----------------------------------------------------------------------------------------------------------
# refusals: TTSB_ERR_INVALID_ARGUMENT before any launch, naming the argument
# ----------------------------------------------------------------------------------------------------------
def test_refusals_name_the_argument_before_any_launch():
    cdll = lib.load()
    basis = torch.from_numpy(slaney_mel_basis(22050, 1024, 128, 0, None)).to(DEV)
    band = (C.c_int32 * 256)(*mel_band(basis.cpu().numpy()).reshape(-1).tolist())
    wav = torch.randn(2, 4096, device=DEV)
    out = torch.full((2 * 17 * 129,), float('nan'), device=DEV)
    p = lambda t: C.c_void_p(t.data_ptr())
    lib.reset_launch_count()
    for (L, n_mels, norm), what in (((512, 80, 0), b'n_samples'), ((4096, 0, 0), b'n_mels'), ((4096, 129, 0), b'n_mels'),
                                    ((4096, 80, 2), b'normalizer')):
        assert cdll.ttsb_stft_mel_log(p(wav), 1, L, p(basis), band, n_mels, norm, p(out), None) == -1
        assert what in cdll.ttsb_last_error(), what
    ws = torch.empty(4096, dtype=torch.uint8, device=DEV)
    i32 = lambda *v: (C.c_int32 * len(v))(*v)
    batch = lambda so, fo, n_mels=80, norm=0: cdll.ttsb_stft_mel_log_batch(p(wav), so, fo, 2, p(basis), band, n_mels, norm, p(ws),
                                                                           C.c_int64(4096), p(out), None)
    for args, what in (((i32(0, 512, 4096), i32(0, 3, 17)), b'clip 0 has 512 samples'),
                       ((i32(0, 1000, 4096), i32(0, 5, 18)), b'frame_offsets'),
                       ((i32(0, 1000, 4096), i32(0, 4, 18)), b'frame_offsets'),
                       ((i32(0, 1000, 4096), i32(0, 4, 17), 0), b'n_mels'),
                       ((i32(0, 1000, 4096), i32(0, 4, 17), 129), b'n_mels'),
                       ((i32(0, 1000, 4096), i32(0, 4, 17), 80, 2), b'normalizer')):
        assert batch(*args) == -1, what
        assert what in cdll.ttsb_last_error(), what
    assert lib.launch_count() == 0
    assert torch.isnan(out).all()


def test_zz_bound_is_sharp():
    """The largest err / bound over every case above: inside (0.01, 1), so the bound neither fails on rounding nor hides a
    wrong bin."""
    if not RATIOS:
        pytest.skip('no case ran')
    worst = max(RATIOS, key=RATIOS.get)
    print(f'largest err/bound {RATIOS[worst]:.3f} ({worst}); per case: '
          + ', '.join(f'{k} {v:.3f}' for k, v in sorted(RATIOS.items(), key=lambda kv: -kv[1])))
    assert 0.01 < RATIOS[worst] < 1.0
