"""CPU checks of oracle/pitch_oracle.py, the numpy restatement of WORLD's DIO + StoneMask as the reference calls them
(data/audio.py:146-151): the filters against a second formulation, hand cases of each step, and known answers."""
import numpy as np
import pytest

from oracle import pitch_oracle as po

FS, HOP = 22050, 256
FP = HOP / FS * 1000
# largest relative f0 error on interior frames measured with this oracle: 2.6e-5 after DIO, 2.4e-4 after StoneMask (tones),
# 3.8e-4 (glide); the thresholds leave a margin of about 4x
TONE_TOL, GLIDE_TOL = 1e-3, 1.5e-3


def test_lowcut_filter_is_symmetric_with_zero_dc_gain():
    h = po.lowcut_filter(FS)
    assert len(h) == 883 and np.allclose(h, h[::-1], rtol=0, atol=1e-17)
    assert abs(h.sum()) < 1e-15


@pytest.mark.parametrize('L', [3328 + 1, 5000, 22050 * 10])
def test_world_fft_filters_equal_direct_linear_convolution(L):
    x = po.speech_like_clip(L / FS, seed=L)[:L]
    bounds = po.boundary_f0s()
    for a, b in zip(po.filtered_bands_fft(x, FS, bounds), po.filtered_bands_direct(x, FS, bounds)):
        assert np.max(np.abs(a - b)) <= 1e-12 * np.max(np.abs(b))


def test_bands_and_filter_lengths():
    b = po.boundary_f0s()
    assert np.allclose(b, [100.4092, 142.0, 200.8183, 284.0, 401.6367, 568.0, 803.2733], atol=1e-3)
    assert po.band_half_lengths(FS, b) == [110, 78, 55, 39, 27, 19, 14]
    assert po.voice_range_minimum(FP, 71.0) == 3


def test_zero_crossing_engine_hand_case():
    s = np.array([1.0, -1.0, -1.0, 3.0, 1.0, -3.0, 2.0, 2.0, -2.0])
    loc, freq = po.zero_crossing_engine(s, 10.0)
    fe = np.array([1.5, 5.25, 8.5])                         # e - s[e-1] / (s[e] - s[e-1]) at edges 1, 5, 8
    assert np.allclose(freq, 10.0 / np.diff(fe)) and np.allclose(loc, (fe[:-1] + fe[1:]) / 2 / 10.0)
    assert len(po.zero_crossing_engine(np.array([1.0, -1.0, -1.0]), 10.0)[0]) == 0


def test_interp1_extrapolates_from_end_segments():
    x, y = np.array([1.0, 2.0, 4.0]), np.array([10.0, 20.0, 0.0])
    got = po.interp1(x, y, np.array([0.0, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0]))
    assert np.allclose(got, [0.0, 10.0, 15.0, 20.0, 10.0, 0.0, -20.0])


def test_fix_steps_hand_cases():
    best = np.array([0, 100, 101, 100, 102, 130, 101, 100, 0, 100, 100, 100.0])
    # frames < 3 and >= 9 are zeroed first; frame 3 jumps from 0, 5 and 6 jump by more than 10 %, frame 8 is 0
    assert np.array_equal(po.fix_step1(best, 3, 0.1), [0, 0, 0, 0, 102, 0, 0, 100, 0, 0, 0, 0])
    s2 = po.fix_step2(np.array([0, 0, 0, 100, 102, 103, 0, 100, 101, 102, 103, 0.0]), 3)
    assert np.array_equal(s2, [0, 0, 0, 0, 102, 0, 0, 0, 101, 102, 0, 0])
    pos, neg = po.voiced_sections(s2)
    assert pos == [4, 8] and neg == [4, 9]
    cands = np.array([[0, 0, 0, 0, 0, 104, 105, 0, 0, 0, 0, 0.0], [0, 0, 95, 99, 0, 0, 0, 0, 0, 0, 111, 0.0]])
    s3 = po.fix_step3(s2, cands, neg, 0.1)                  # 102 -> 104 -> 105 -> (nothing within 10 %) stop; 102 -> 111 -> stop
    assert np.array_equal(s3, [0, 0, 0, 0, 102, 104, 105, 0, 101, 102, 111, 0])
    s4 = po.fix_step4(s3, cands, pos, 0.1)                  # from 8: frame 7 has no candidate; from 4: 99, then 95, then stop
    assert np.array_equal(s4, [0, 0, 95, 99, 102, 104, 105, 0, 101, 102, 111, 0])
    assert po.select_best_f0(100.0, np.array([[95.0], [105.0]]), 0, 0.1) == 105.0   # equal error: the later band wins


def test_stonemask_harmonic_fix_hand_case():
    # n_fft 16, fs 16: f = 2 reads bins 2 and 4; IF_1 = 2 + 0, IF_2 = 4 + (pi/16)/1 * 16/(2 pi) = 4.5; amplitudes 2 and 1
    P, Q = np.zeros(16), np.zeros(16)
    P[2], P[4], Q[4] = 4.0, 1.0, np.pi / 16
    assert np.isclose(po.stonemask_fix_f0(P, Q, 16, 16.0, 2.0, 2), (2 * 2 + 1 * 4.5) / (2 * 1 + 1 * 2), rtol=1e-14)
    P[4] = 0.0                                              # an empty bin contributes no frequency and no weight
    assert np.isclose(po.stonemask_fix_f0(P, Q, 16, 16.0, 2.0, 2), 2 * 2 / 2, rtol=1e-14)


def test_stonemask_floor_and_refinement():
    x = po.tone(200, 0.5, seed=1).astype(np.float64)
    assert po.stonemask_frame(x, FS, 0.25, 39.0) == 0.0 and po.stonemask_frame(x, FS, 0.25, FS / 12 + 1) == 0.0
    assert abs(po.stonemask_frame(x, FS, 0.25, 190.0) / 200 - 1) < 1e-3
    # from 150 Hz the refinement lands near the 200 Hz tone, more than 20 % away: the input is returned unchanged
    assert po.stonemask_frame(x, FS, 0.25, 150.0) == 150.0


def test_frame_count_rule_and_pad():
    n = [L for L in range(256, 1280000, 256) if po.n_frames(L, FS, FP) != 1 + L // HOP]
    assert n[0] == 3328 and len(n) == 185
    assert all(po.n_frames(L + 1, FS, FP) == 1 + (L + 1) // HOP for L in n)
    assert len(po.pad_for_hop(np.zeros(3328, np.float32))) == 3329 and len(po.pad_for_hop(np.zeros(3329, np.float32))) == 3329


def test_silence_gives_zeros():
    assert not po.extract_pitch(np.zeros(22050, np.float32)).any()


@pytest.mark.parametrize('f', [90, 120, 180, 250, 350])
def test_tones(f):
    x = po.tone(f, 2.0, seed=f).astype(np.float64)
    f0, t = po.dio(x, FS, FP)
    sm = po.stonemask(x, f0, t, FS)
    assert (f0[3:-3] > 0).all() and (sm[3:-3] > 0).all()
    assert np.max(np.abs(sm[3:-3] / f - 1)) < TONE_TOL


def test_glide_vibrato_and_gaps():
    x = po.glide(110, 220, 2.0, seed=1)
    f0 = po.extract_pitch(x)
    n = len(x)
    track = 110 * 2.0 ** (np.arange(n) / n)
    t = np.minimum(np.arange(len(f0)) * HOP, n - 1)
    assert (f0[3:-3] > 0).all() and np.max(np.abs(f0[3:-3] / track[t][3:-3] - 1)) < GLIDE_TOL
    v = po.extract_pitch(po.vibrato(150, 0.03, 5.0, 2.0, seed=2))
    assert (v[3:-3] > 0).all() and np.max(np.abs(v[3:-3] / 150 - 1)) < 0.04
    gap = np.concatenate([1e-4 * np.random.default_rng(3).standard_normal(11025), po.tone(150, 1.0, seed=4),
                          1e-4 * np.random.default_rng(5).standard_normal(11025)]).astype(np.float32)
    g = po.extract_pitch(gap)
    voiced = np.nonzero(g)[0]
    assert 40 <= voiced[0] <= 48 and 124 <= voiced[-1] <= 132 and (g[voiced[0]:voiced[-1] + 1] > 0).all()
    assert not g[:38].any() and not g[135:].any()


# the other sampling rates the project prepares data at, each at its usual hop (vrm 3 at all of them)
RATES = [(8000, 80), (16000, 200), (44100, 512), (48000, 600), (96000, 1200)]


@pytest.mark.parametrize('fs,hop', RATES)
def test_world_fft_filters_equal_direct_linear_convolution_at_other_rates(fs, hop):
    x = po.speech_like_clip(1.3, seed=fs, fs=float(fs))
    bounds = po.boundary_f0s()
    for a, b in zip(po.filtered_bands_fft(x, fs, bounds), po.filtered_bands_direct(x, fs, bounds)):
        assert np.max(np.abs(a - b)) <= 1e-12 * np.max(np.abs(b))


@pytest.mark.parametrize('fs,hop', RATES)
def test_tones_glide_and_silence_at_other_rates(fs, hop):
    fp = hop / fs * 1000
    v = po.voice_range_minimum(fp, 71.0)
    assert v == 3
    for f in (90, 180, 350):
        x = po.tone(f, 2.0, fs=float(fs), seed=f).astype(np.float64)
        f0, t = po.dio(x, fs, fp)
        sm = po.stonemask(x, f0, t, fs)
        assert (f0[v:-v] > 0).all() and (sm[v:-v] > 0).all(), f
        assert np.max(np.abs(sm[v:-v] / f - 1)) < TONE_TOL, f
    x = po.glide(110, 220, 2.0, fs=float(fs), seed=1)
    g = po.extract_pitch(x, fs, hop)
    n = len(x)
    track = 110 * 2.0 ** (np.arange(n) / n)
    t = np.minimum(np.arange(len(g)) * hop, n - 1)
    assert (g[v:-v] > 0).all() and np.max(np.abs(g[v:-v] / track[t][v:-v] - 1)) < GLIDE_TOL
    assert not po.extract_pitch(np.zeros(fs, np.float32), fs, hop).any()


def test_stonemask_upper_limit_at_8k():
    # fs / 12 = 666.7 Hz is below f0_ceil at 8 kHz: DIO voices a 700 Hz tone and StoneMask zeroes it; at 16 kHz it is refined
    for fs, hop, kept in ((8000, 80, False), (16000, 200, True)):
        x = po.tone(700, 1.0, fs=float(fs), seed=1).astype(np.float64)
        f0, t = po.dio(x, fs, hop / fs * 1000)
        sm = po.stonemask(x, f0, t, fs)
        assert np.count_nonzero(f0 > 8000 / 12.0) > 50
        if kept:
            assert (sm[3:-3] > 0).all() and np.max(np.abs(sm[3:-3] / 700 - 1)) < TONE_TOL
        else:
            assert not sm.any()


@pytest.mark.parametrize('hop,vrm', [(64, 11), (128, 5), (256, 3), (275, 3), (FS * 5.0 / 1000, 7)])
def test_fix_f0_contour_needs_more_than_voice_range_minimum_frames(hop, vrm):
    fp = hop / FS * 1000
    assert po.voice_range_minimum(fp, 71.0) == vrm
    with pytest.raises(ValueError, match=f'more than {vrm}'):
        po.fix_f0_contour(np.full(vrm, 100.0), np.full((7, vrm), 100.0), fp, 71.0, 0.1)
    assert not po.fix_f0_contour(np.full(vrm + 1, 100.0), np.full((7, vrm + 1), 100.0), fp, 71.0, 0.1).any()


def test_pitch_statistics_and_normalisation():
    a, b = np.array([0.0, 100.0, 200.0]), np.array([300.0, 0.0])
    mean, std = po.pitch_stats([a, b])
    assert mean == 200.0 and np.isclose(std, np.std([100.0, 200.0, 300.0]))
    assert np.array_equal(po.normalize_pitch(a, mean, std), np.array([0.0, -100.0 / std, 0.0]))
