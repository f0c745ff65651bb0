"""DIO + StoneMask on the GPU (ttsb_pitch_dio_stonemask, csrc/pitch.cu) against the numpy restatement of WORLD
(oracle/pitch_oracle.py) at every sampling rate the project prepares data at, at frame periods that give FixF0Contour's
voice_range_minimum (vrm) the values 3, 5, 7 and 11, at clip lengths around the frame, filter-tile and refusal edges, in
batches of up to 80 clips, on signals that reach each threshold of the algorithm, and at non-default parameters.

The gate is the one the corpus tests use: voicing identical and f0 within 1e-6 relative on voiced frames.  The oracle's
default filters are WORLD's circular FFT convolution; the kernels convolve directly.  A clip whose voicing differs from the
FFT formulation anywhere is compared in full with the oracle's direct formulation instead, and each frame where the two
formulations of the oracle disagree is counted and printed as excused.  A difference the direct formulation does not share
fails.  Every f0 output is NaN before the call, so a frame the kernels never write fails too."""
import math

import numpy as np
import pytest
import torch

from oracle import pitch_oracle as po

pytestmark = pytest.mark.gpu
REL_TOL = 1e-6
# sampling rate and its usual hop
RATES = [(8000, 80), (16000, 200), (22050, 256), (24000, 300), (44100, 512), (48000, 600), (96000, 1200)]
FS = 22050
# frame periods (ms) at 22050 Hz: hops 64, 128, 256, 275 and 5 ms, with vrm 11, 5, 3, 3 and 7 at f0_floor 71
FRAME_PERIODS = [(64 / FS * 1000, 11), (128 / FS * 1000, 5), (256 / FS * 1000, 3), (275 / FS * 1000, 3), (5.0, 7)]
TILE = 512                     # outputs per block of the low-cut and band filter kernels


def _lib():
    from transformertts_b200 import lib
    return lib


def _frame_offsets(clips, fs, fp):
    return np.concatenate([[0], np.cumsum([po.n_frames(len(x), fs, fp) for x in clips])]).astype(np.int64)


def _gpu(clips, fs, fp, fill=0x00, fo=None, f0_floor=71.0, f0_ceil=800.0, channels_in_octave=2.0, allowed_range=0.1):
    """ttsb_pitch_dio_stonemask on a packed batch, the workspace filled with the byte `fill` and f0 filled with NaN -> list of
    float64 f0 per clip."""
    lib = _lib()
    ws_clips = [np.asarray(x, dtype=np.float32) for x in clips]
    so = np.concatenate([[0], np.cumsum([len(x) for x in ws_clips])]).astype(np.int64)
    fo = _frame_offsets(clips, fs, fp) if fo is None else np.asarray(fo, dtype=np.int64)
    wav = torch.from_numpy(np.concatenate(ws_clips)).cuda()
    nb = lib.pitch_workspace_bytes(so, fs, fp, f0_floor, f0_ceil, channels_in_octave)
    ws = torch.full((nb,), fill, dtype=torch.uint8, device='cuda')
    out = torch.full((int(fo[-1]),), float('nan'), dtype=torch.float64, device='cuda')
    lib.pitch_dio_stonemask(wav, so, fs, fp, fo, out, ws, f0_floor=f0_floor, f0_ceil=f0_ceil, channels_in_octave=channels_in_octave,
                            allowed_range=allowed_range)
    out = out.cpu().numpy()
    return [out[a:b] for a, b in zip(fo[:-1], fo[1:])]


def _reference(x, fs, fp, direct=False, **params):
    """po.dio then po.stonemask -> (final f0, DIO's f0)."""
    x = np.asarray(x, dtype=np.float64)
    f0, t = po.dio(x, fs, fp, direct=direct, **params)
    return po.stonemask(x, f0, t, fs), f0


def _check(label, clips, got, fs, fp, **params):
    """Compare every clip with the oracle, print a MEASURED line, return (final f0, DIO f0) of the oracle per clip."""
    worst, voiced, excused, refs = 0.0, 0, 0, []
    for c, (x, f) in enumerate(zip(clips, got)):
        want, dio = _reference(x, fs, fp, **params)
        assert f.shape == want.shape == (po.n_frames(len(x), fs, fp),), (label, c)
        assert not np.isnan(f).any(), (label, c, np.nonzero(np.isnan(f))[0])
        differ = (f != 0) != (want != 0)
        if differ.any():
            want, dio = _reference(x, fs, fp, direct=True, **params)
            assert np.array_equal(f != 0, want != 0), (label, c, 'voicing differs from both formulations of the oracle',
                                                       np.nonzero((f != 0) != (want != 0))[0])
            excused += int(differ.sum())
            print(f'EXCUSED {label} clip {c}: frames {np.nonzero(differ)[0].tolist()}, where the FFT and the direct filters of the '
                  f'oracle disagree; the clip is compared with the direct formulation')
        v = want != 0
        voiced += int(v.sum())
        if v.any():
            worst = max(worst, float(np.max(np.abs(f[v] / want[v] - 1))))
        refs.append((want, dio))
    print(f'MEASURED {label}: {len(clips)} clips, {voiced} voiced frames, max |f0 / oracle - 1| = {worst:.3e}, '
          f'{excused} excused frames')
    assert worst < REL_TOL, (label, worst)
    return refs


def _bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def _n_fft(fs, f0):
    """StoneMask's DFT size at f0: 2^(2 + int(log2(2 half + 1))) with half = int(1.5 fs / f0 + 1)."""
    return 1 << (2 + int(math.log(2 * int(1.5 * fs / f0 + 1.0) + 1.0) / po.K_LOG2))


def _min_accepted_length(fs, fp, vrm):
    """Fewest samples whose WORLD frame count exceeds vrm."""
    L = max(1, int(vrm * fs * fp / 1000.0))
    while L > 1 and po.n_frames(L - 1, fs, fp) > vrm:
        L -= 1
    while po.n_frames(L, fs, fp) <= vrm:
        L += 1
    return L


def _tone(f0, L, fs, seed):
    return po.tone(f0, L / fs + 0.01, fs=float(fs), seed=seed)[:L]


def _audio(fs, hop):
    from transformertts_b200.data.audio import Audio
    n = min(4096, 1 << (4 * hop - 1).bit_length())
    return Audio(sampling_rate=fs, n_fft=n, mel_channels=80, hop_length=hop, win_length=n, f_min=0, f_max=None, normalizer='MelGAN')


# ---- 1 and 8: every rate, through the library and through Audio, and the frame-count table --------------------------------
@pytest.mark.parametrize('fs,hop', RATES)
def test_every_rate(fs, hop):
    from transformertts_b200.lib import TtsbError
    fp = hop / fs * 1000
    # speech-like clips and a low glide whose StoneMask windows need the largest DFTs of the rate (8192 points at 96 kHz)
    clips = po.make_corpus(3, seed=fs, min_s=1.0, max_s=3.0, fs=float(fs)) + [po.glide(75, 110, 2.5, fs=float(fs), seed=1)]
    got = _gpu(clips, fs, fp)
    refs = _check(f'rate {fs} hop {hop}', clips, got, fs, fp)
    big = 1024 if fs == 8000 else 8192 if fs == 96000 else 2048
    long_windows = sum(int(np.sum([_n_fft(fs, f) >= big for f in want[want != 0]])) for want, _ in refs)
    print(f'MEASURED rate {fs}: {long_windows} frames with StoneMask DFTs of {big}+ points')
    assert long_windows > 50
    # Audio's frame count and default parameters give the same bits
    audio = _audio(fs, hop)
    assert np.array_equal(audio._pitch_frames([len(x) for x in clips]), [po.n_frames(len(x), fs, fp) for x in clips])
    for a, b in zip(audio.extract_pitch_batch(clips), got):
        assert np.array_equal(_bits(a), _bits(b))
    # a frame table that gives a clip one frame too many or too few is refused
    fo = _frame_offsets(clips[:2], fs, fp)
    for d in (-1, 1):
        with pytest.raises(TtsbError, match="WORLD's frame count differs"):
            _gpu(clips[:2], fs, fp, fo=[0, fo[1] + d, fo[2]])


def test_sixty_seconds_at_48k():
    fs, hop = 48000, 600
    fp = hop / fs * 1000
    x = po.speech_like_clip(60.0, seed=60, fs=float(fs))
    refs = _check('60 s at 48000 Hz', [x], _gpu([x], fs, fp), fs, fp)
    assert np.count_nonzero(refs[0][0]) > 1000


# ---- 2 and 3: frame periods and clip lengths ---------------------------------------------------------------------------------
def _tile_edge_clips(fs, P, start, seed):
    """Clips whose padded slots (L + 1 + 2P each, packed from `start`) end one slot before, on and one slot after a 512-slot tile
    boundary of the filter kernels."""
    clips, at = [], start
    for i, d in enumerate((-1, 0, 1)):
        m = (at + int(0.4 * fs) + 1 + 2 * P) // TILE + 1
        L = TILE * m + d - at - 1 - 2 * P
        clips.append(_tone(140 + 20 * i, L, fs, seed + i))
        at += L + 1 + 2 * P
        assert at % TILE == (d % TILE)
    return clips


@pytest.mark.parametrize('fp,vrm', FRAME_PERIODS, ids=['hop64', 'hop128', 'hop256', 'hop275', '5ms'])
def test_frame_periods_and_clip_lengths(fp, vrm):
    from transformertts_b200.lib import TtsbError
    assert po.voice_range_minimum(fp, 71.0) == vrm
    P = po.matlab_round(FS / 50.0)
    hop = FS * fp / 1000.0
    L_min = _min_accepted_length(FS, fp, vrm)
    assert po.n_frames(L_min, FS, fp) == vrm + 1 and po.n_frames(L_min - 1, FS, fp) == vrm
    clips = po.make_corpus(2, seed=int(fp * 1000), min_s=1.0, max_s=2.5)
    clips += [_tone(150, L_min, FS, 1), _tone(150, L_min + 1, FS, 2)]
    for k in (2 * vrm + 2, 37):
        L0 = int(round(k * hop))
        clips += [_tone(120 + k, L, FS, 3 + L - L0) for L in (L0 - 1, L0, L0 + 1)]
    clips += _tile_edge_clips(FS, P, sum(len(x) + 1 + 2 * P for x in clips), seed=7)
    _check(f'frame period {fp:.4f} ms (vrm {vrm})', clips, _gpu(clips, FS, fp), FS, fp)
    # one sample shorter than the shortest clip is refused by the kernels and by the oracle
    short = _tone(150, L_min - 1, FS, 1)
    with pytest.raises(TtsbError, match='voice_range_minimum'):
        _gpu([clips[0], short], FS, fp)
    with pytest.raises(ValueError):
        _reference(short, FS, fp)


# ---- 4: a batch of many short clips -----------------------------------------------------------------------------------------
def test_eighty_short_clips_bit_identical_alone_and_reversed():
    fp = 256 / FS * 1000
    rng = np.random.default_rng(80)
    clips = []
    for c in range(80):
        L = int(rng.integers(800, 12000))
        clips.append(_tone(float(rng.uniform(80, 400)), L, FS, c) if c % 2 else po.speech_like_clip(L / FS + 0.01, seed=c)[:L])
    got = _gpu(clips, FS, fp)
    rev = _gpu(clips[::-1], FS, fp)[::-1]
    _check('80 short clips', clips, got, FS, fp)
    for c, x in enumerate(clips):
        alone = _gpu([x], FS, fp)[0]
        assert np.array_equal(_bits(got[c]), _bits(alone)), c
        assert np.array_equal(_bits(got[c]), _bits(rev[c])), c


# ---- 5: signal content -------------------------------------------------------------------------------------------------------
def _segments(parts, fs, seed):
    """Concatenated (f0 track or None for low noise, samples) parts, phase-continuous within each voiced part."""
    rng = np.random.default_rng(seed)
    out = []
    for f0, n in parts:
        out.append(1e-4 * rng.standard_normal(n) if f0 is None else po.harmonic_tone(np.full(n, float(f0)), fs))
    return np.concatenate(out).astype(np.float32)


def test_signal_content():
    fp = 256 / FS * 1000
    bounds = po.boundary_f0s()
    rng = np.random.default_rng(5)
    t = np.arange(FS)
    hf = 0.5 * np.sin(2 * np.pi * 0.45 * np.arange(15000) + 0.3)
    clips = {
        'silence': np.zeros(FS, np.float32),
        'dc': np.full(8000, 0.5, np.float32),
        # a quiet tone on a large offset: the frames near the clip edges depend on the mean over L + 1 samples
        'tone on dc 4000': (1e-3 / 0.3 * _tone(200, 4000, FS, 1) + 0.9).astype(np.float32),
        'tone on dc 8000': (1e-3 / 0.3 * _tone(120, 8000, FS, 2) + 0.9).astype(np.float32),
        'tone on dc 1 s': (_tone(150, FS, FS, 3) + 0.9).astype(np.float32),
        'clipped square': np.clip(3.0 * np.sign(np.sin(2 * np.pi * 150 * t / FS)), -1, 1).astype(np.float32),
        'white noise': (0.3 * rng.standard_normal(FS)).astype(np.float32),
        # 0.45 fs then a tone: the zero-crossing lists of the first part fill over half their capacity (L + 1) / 2 + 1
        'hf then tone': np.concatenate([hf, _tone(150, 7000, FS, 4)]).astype(np.float32),
        'tone 70 (below floor)': _tone(70, FS, FS, 5), 'tone 72': _tone(72, FS, FS, 6),
        'tone 795': _tone(795, FS, FS, 7), 'tone 805 (above ceil)': _tone(805, FS, FS, 8),
    }
    for b in (0, 2, 4):
        clips[f'tone at bound[{b}]'] = _tone(bounds[b], FS, FS, 10 + b)
        clips[f'tone at bound[{b}] / 2'] = _tone(bounds[b] / 2, FS, FS, 20 + b)
    # voiced sections 1 .. vrm + 1 frames apart, and f0 jumps just under and over allowed_range
    hop = 256
    gaps = []
    for g in range(1, 5):
        gaps += [(150 + 10 * g, int(0.3 * FS)), (None, g * hop)]
    clips['gaps of 1 .. 4 frames'] = _segments(gaps + [(150, int(0.3 * FS))], FS, 30)
    for r in (1.08, 1.095, 1.105, 1.12):
        clips[f'jump x{r}'] = _segments([(150, int(0.5 * FS)), (150 * r, int(0.5 * FS))], FS, 40)
    names, xs = list(clips), list(clips.values())
    got = _gpu(xs, FS, fp)
    refs = _check('signal content at 22050 Hz', xs, got, FS, fp)
    res = dict(zip(names, zip(got, refs)))
    for name in ('silence', 'dc', 'white noise', 'tone 70 (below floor)', 'tone 805 (above ceil)'):
        assert not res[name][0].any(), name
    for name in ('tone 72', 'tone 795', 'clipped square', 'hf then tone', 'tone on dc 4000', 'tone on dc 8000'):
        assert np.count_nonzero(res[name][0]) > 5, name
    # tones voiced from their first sample to their last: StoneMask's window is clamped at both ends
    assert res['tone 795'][0][1] != 0 and res['tone 795'][0][-1] != 0
    x = clips['hf then tone'].astype(np.float64)
    most = max(int(np.sum((s[:-1] > 0) & (s[1:] <= 0))) for f in po.filtered_bands_direct(x, FS, bounds)
               for s in (f, -f, f[1:] - f[:-1], f[:-1] - f[1:]))
    assert most > ((len(x) + 1) // 2 + 1) / 2
    # each gap of the gaps clip stays an unvoiced run after FixF0Contour, most of them no longer than vrm = 3 frames
    v = np.nonzero(res['gaps of 1 .. 4 frames'][0])[0]
    runs = np.diff(v) - 1
    runs = runs[runs > 0]
    assert len(runs) == 4 and np.sum(runs <= 3) >= 3, runs


def test_stonemask_upper_limit_at_8k():
    fs, hop = 8000, 80
    fp = hop / fs * 1000
    x = po.tone(700, 1.0, fs=float(fs), seed=1)
    refs = _check('700 Hz at 8000 Hz', [x], _gpu([x], fs, fp), fs, fp)
    want, dio = refs[0]
    # DIO voices the tone; StoneMask's limit fs / 12 = 666.7 Hz zeroes it
    assert np.count_nonzero(dio) > 50 and not want.any()


# ---- 6: non-default parameters ----------------------------------------------------------------------------------------------
def _lowest_floor(fs, channels_in_octave=2.0):
    """Lowest integer f0_floor whose first band's low-pass (4h taps, delay 2h) fits the low-cut margin P = round(fs / 50)."""
    P = po.matlab_round(fs / 50.0)
    f = 1
    while 2 * po.band_half_lengths(fs, [f * pow(2.0, 1.0 / channels_in_octave)])[0] > P:
        f += 1
    return f


PARAMS = [dict(f0_floor=36.0), dict(f0_floor=50.0), dict(f0_floor=100.0), dict(f0_ceil=400.0), dict(f0_ceil=1100.0),
          dict(channels_in_octave=1.0), dict(channels_in_octave=3.0), dict(channels_in_octave=4.5), dict(allowed_range=0.05),
          dict(allowed_range=0.2)]


@pytest.mark.parametrize('params', PARAMS, ids=lambda p: '-'.join(f'{k}{v}' for k, v in p.items()))
def test_parameters(params):
    fp = 256 / FS * 1000
    clips = po.make_corpus(2, seed=11, min_s=1.0, max_s=2.5)
    clips += [po.glide(60, 240, 2.0, seed=2), _tone(900, FS, FS, 3), _tone(45, 2 * FS, FS, 4)]
    clips += [_segments([(150, int(0.5 * FS)), (150 * r, int(0.5 * FS))], FS, 40) for r in (1.04, 1.06, 1.15, 1.25)]
    label = ' '.join(f'{k} {v}' for k, v in params.items())
    full = dict(po.DEFAULTS, **params)
    if 'channels_in_octave' in params:
        n_bands = len(po.boundary_f0s(full['f0_floor'], full['f0_ceil'], full['channels_in_octave']))
        label += f' ({n_bands} bands)'
    refs = _check(label, clips, _gpu(clips, FS, fp, **params), FS, fp, **params)
    assert sum(np.count_nonzero(w) for w, _ in refs) > 100


def test_band_count_and_low_cut_margin_refusals():
    from transformertts_b200.lib import TtsbError
    fp = 256 / FS * 1000
    x = po.speech_like_clip(1.5, seed=3)
    assert len(po.boundary_f0s(71.0, 800.0, 4.5)) == 16 and len(po.boundary_f0s(71.0, 800.0, 4.6)) == 17
    with pytest.raises(TtsbError, match='17 bands; at most 16'):
        _gpu([x], FS, fp, channels_in_octave=4.6)
    for fs, hop in ((FS, 256), (8000, 80), (48000, 600)):
        fp = hop / fs * 1000
        lo = _lowest_floor(fs)
        y = po.glide(lo + 5.0, 4 * lo, 1.5, fs=float(fs), seed=fs)
        _check(f'lowest f0_floor {lo} at {fs} Hz', [y], _gpu([y], fs, fp, f0_floor=float(lo)), fs, fp, f0_floor=float(lo))
        with pytest.raises(TtsbError, match='band 0 low-pass longer than the low-cut margin'):
            _gpu([y], fs, fp, f0_floor=float(lo - 1))


def test_stonemask_floor_below_dio_floor():
    fp = 256 / FS * 1000
    x = po.tone(38, 2.0, seed=2)
    refs = _check('38 Hz tone at f0_floor 36', [x], _gpu([x], FS, fp, f0_floor=36.0), FS, fp, f0_floor=36.0)
    want, dio = refs[0]
    # DIO voices 38 Hz; StoneMask's floor of 40 Hz zeroes every such frame
    assert np.count_nonzero((dio > 0) & (dio <= po.K_FLOOR_F0_STONEMASK)) > 50 and not want.any()
    # below 71 Hz the DFT grows to 16384 points at 96 kHz
    fs, hop = 96000, 1200
    fp = hop / fs * 1000
    y = po.glide(50, 90, 2.0, fs=float(fs), seed=5)
    refs = _check('50-90 Hz glide at 96000 Hz, f0_floor 45', [y], _gpu([y], fs, fp, f0_floor=45.0), fs, fp, f0_floor=45.0)
    assert sum(_n_fft(fs, f) == 16384 for f in refs[0][0][refs[0][0] != 0]) > 10


# ---- 7: workspace independence ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fs,hop', [(22050, 256), (96000, 1200)])
def test_workspace_contents_do_not_matter(fs, hop):
    fp = hop / fs * 1000
    clips = po.make_corpus(4, seed=77, min_s=0.5, max_s=2.0, fs=float(fs))
    a = _gpu(clips, fs, fp, fill=0x00)
    b = _gpu(clips, fs, fp, fill=0xFF)
    for x, y in zip(a, b):
        assert not np.isnan(x).any() and np.array_equal(_bits(x), _bits(y))
