"""CPU tests of audio settings other than n_fft 1024 / hop 256 / win 1024: the supported set Audio accepts and the boundaries it
refuses by name, f_max None, the minimum clip rules, the mel / WORLD frame-count agreement, and the refusals of the general STFT
entry points (include/ttsb.h: ttsb_stft_mel_log_ragged ...) before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from oracle import audio_oracle as ao

WAVERNN = dict(sampling_rate=22050, n_fft=2048, mel_channels=80, hop_length=275, win_length=1100, f_min=40, f_max=None,
               normalizer='WaveRNN')


def _audio(**kw):
    from transformertts_b200.data.audio import Audio
    return Audio(**dict(WAVERNN, **kw))


@pytest.mark.parametrize('cfg', [dict(), dict(sampling_rate=24000, hop_length=300, win_length=1200, f_min=0, f_max=12000),
                                 dict(sampling_rate=16000, n_fft=1024, hop_length=200, win_length=800, f_max=8000),
                                 dict(sampling_rate=16000, n_fft=512, hop_length=128, win_length=512),
                                 dict(sampling_rate=48000, n_fft=4096, hop_length=1024, win_length=4096, mel_channels=128),
                                 dict(n_fft=256, hop_length=1, win_length=2, mel_channels=1),
                                 dict(sampling_rate=22050, n_fft=1024, hop_length=256, win_length=1024, f_max=8000)])
def test_supported_settings_are_accepted(cfg):
    a = _audio(**cfg)
    assert a.f_max == (a.sampling_rate / 2 if cfg.get('f_max', WAVERNN['f_max']) is None else cfg['f_max'])


@pytest.mark.parametrize('cfg, name', [(dict(n_fft=3000), 'n_fft'), (dict(n_fft=128, win_length=128, hop_length=64), 'n_fft'),
                                       (dict(n_fft=8192), 'n_fft'), (dict(win_length=2049), 'win_length'),
                                       (dict(win_length=0), 'win_length'), (dict(win_length=1, hop_length=1), 'win_length'), (dict(hop_length=1101), 'hop_length'),
                                       (dict(hop_length=0), 'hop_length'), (dict(f_max=11026), 'f_max'),
                                       (dict(f_min=-1), 'f_min'), (dict(f_min=8000, f_max=8000), 'f_min'),
                                       (dict(mel_channels=129), 'mel_channels'), (dict(mel_channels=0), 'mel_channels'),
                                       (dict(sampling_rate=0), 'sampling_rate'), (dict(sampling_rate=22050.5), 'sampling_rate')])
def test_settings_outside_the_supported_set_are_refused_by_name(cfg, name):
    with pytest.raises(ValueError, match=name):
        _audio(**cfg)


def test_f_max_none_is_the_nyquist_rate():
    from transformertts_b200.data.audio import slaney_mel_basis
    a = _audio()
    want = ao.mel_filterbank(22050, 2048, 80, 40, 22050 / 2)
    assert np.abs(slaney_mel_basis(22050, 2048, 80, 40, None) - want).max() < 1e-7
    assert a.f_max == 11025.0


@pytest.mark.parametrize('n_fft, hop, frames', [(1024, 256, 4), (2048, 275, 5), (1024, 200, 4), (512, 128, 4), (4096, 1024, 4),
                                                (2048, 300, 5), (256, 1, 130)])
def test_minimum_clip_rules(n_fft, hop, frames):
    a = _audio(n_fft=n_fft, hop_length=hop, win_length=max(hop, n_fft // 2))
    assert a.min_griffinlim_frames == frames == n_fft // 2 // hop + 2
    assert hop * (frames - 1) > n_fft // 2 >= hop * (frames - 2)
    assert a.min_mel_samples == n_fft // 2 + 1


def test_griffinlim_frame_check_uses_the_configuration():
    from transformertts_b200.data.audio import _clip_frame_counts
    assert list(_clip_frame_counts([0, 4, 9], 9)) == [4, 5]
    with pytest.raises(ValueError, match='at least 5 frames'):
        _clip_frame_counts([0, 4, 9], 9, _audio().min_griffinlim_frames)
    with pytest.raises(ValueError, match='T >= 5'):
        _audio().reconstruct_waveform_batch([np.zeros((80, 4), np.float32)])


def test_mel_and_world_frame_counts_agree_at_hop_275():
    """preprocess pads a clip with L % hop == 0 by one sample; every other L gives 1 + L // hop frames in both front ends."""
    a = _audio()
    L = np.array([n for n in range(1000, 5001) if n % 275 != 0])
    assert np.array_equal(a._frames_per_clip(L), a._pitch_frames(L))
    assert len(a.preprocess(np.zeros(275 * 8, np.float32))) % 275 != 0


def _i32(*v):
    return (C.c_int32 * len(v))(*v)


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def test_general_entry_points_refuse_bad_tables_and_configurations_without_gpu(cdll):
    dev = C.c_void_p(256)          # never dereferenced: every check below fails before any CUDA call
    big = C.c_int64(1 << 30)

    def err():
        return cdll.ttsb_last_error()

    def mel(so, fo, n, n_fft=2048, hop=275, win=1100, n_mels=80, norm=1, ws=big):
        return cdll.ttsb_stft_mel_log_ragged(dev, so, fo, n, n_fft, hop, win, dev, dev, n_mels, norm, dev, ws, dev, None)

    good_so, good_fo = _i32(0, 2000, 5000), _i32(0, 8, 19)            # 1 + 2000 // 275 = 8, 1 + 3000 // 275 = 11
    for n_fft, hop, win in [(3000, 275, 1100), (2048, 275, 2049), (2048, 1101, 1100), (2048, 0, 1100), (128, 64, 128), (8192, 275, 1100), (2048, 1, 1)]:
        assert mel(good_so, good_fo, 2, n_fft, hop, win) == -1 and b'unsupported STFT configuration' in err()
    assert mel(good_so, good_fo, 2, n_mels=129) == -1 and b'n_mels' in err()
    assert mel(good_so, good_fo, 2, norm=2) == -1 and b'normalizer' in err()
    assert mel(_i32(1, 2000, 5000), good_fo, 2) == -1 and b'start at 0' in err()
    assert mel(_i32(0, 1024, 5000), _i32(0, 4, 15), 2) == -1 and b'more than 1024' in err()
    assert mel(good_so, _i32(0, 8, 18), 2) == -1 and b'1 + L / hop' in err()
    need = cdll.ttsb_stft_mel_log_ragged_workspace_bytes(2, 2048)
    assert need > 0 and mel(good_so, good_fo, 2, ws=C.c_int64(need - 1)) == -1 and b'workspace' in err()
    assert cdll.ttsb_stft_mel_log_ragged(None, good_so, good_fo, 2, 2048, 275, 1100, dev, dev, 80, 1, dev, big, dev, None) == -1
    assert cdll.ttsb_stft_mel_log_ragged(dev, good_so, good_fo, 2, 2048, 275, 1100, dev, None, 80, 1, dev, big, dev, None) == -1
    assert b'NULL' in err()
    assert cdll.ttsb_stft_mel_log_ragged_workspace_bytes(0, 2048) == -1
    assert cdll.ttsb_stft_mel_log_ragged_workspace_bytes(1, 8192) == -1

    assert cdll.ttsb_stft_complex_ragged(dev, _i32(0, 1024), 1, 2048, 275, 1100, dev, big, dev, None) == -1 and b'more than 1024' in err()
    assert cdll.ttsb_stft_complex_ragged(dev, _i32(0, 5000), 1, 2048, 300, 200, dev, big, dev, None) == -1 and b'unsupported' in err()
    assert cdll.ttsb_stft_complex_ragged(dev, _i32(0, 5000), 1, 2048, 275, 1100, dev, C.c_int64(100), dev, None) == -1 and b'workspace' in err()

    def gl(fo, n, n_fft=2048, hop=275, win=1100, n_iter=32, momentum=0.99, ws=big):
        return cdll.ttsb_griffinlim_ragged(dev, dev, fo, n, n_fft, hop, win, n_iter, C.c_float(momentum), dev, ws, dev, None)

    assert gl(_i32(0, 5, 9), 2) == -1 and b'clip 1 has 4 frames; need at least 5' in err()
    assert gl(_i32(1, 6, 11), 2) == -1 and b'start at 0' in err()
    assert gl(_i32(0, 7, 5), 2) == -1
    assert gl(_i32(0, 5, 10), 2, n_iter=-1) == -1 and b'n_iter' in err()
    assert gl(_i32(0, 5, 10), 2, momentum=float('inf')) == -1 and b'momentum' in err()
    assert gl(_i32(0, 5, 10), 2, n_fft=2000) == -1 and b'unsupported' in err()
    need = cdll.ttsb_griffinlim_ragged_workspace_bytes(10, 2, 2048)
    assert need > 10 * 2048 * 4 + 2 * 10 * 1025 * 8 and gl(_i32(0, 5, 10), 2, ws=C.c_int64(need - 1)) == -1 and b'workspace' in err()
    assert cdll.ttsb_griffinlim_ragged_workspace_bytes(3, 2, 2048) == -1

    def istft(fo, n, ws=big):
        return cdll.ttsb_istft_ragged(dev, fo, n, 2048, 275, 1100, dev, ws, dev, None)

    assert istft(_i32(0, 1, 5), 2) == -1
    assert istft(_i32(0, 3, 4), 2) == -1 and b'clip 1 has 1 frames' in err()
    need = cdll.ttsb_istft_ragged_workspace_bytes(5, 2, 2048)
    assert istft(_i32(0, 2, 5), 2, ws=C.c_int64(need - 1)) == -1 and b'workspace' in err()

    def m2l(n_bins=1025, n_mels=80, step=1.0, n_iter=64):
        return cdll.ttsb_mel_to_linear_ex(dev, 10, n_mels, n_bins, dev, dev, dev, dev, C.c_float(step), n_iter, dev, None)

    assert m2l(n_bins=2050) == -1 and b'n_bins' in err()
    assert m2l(n_bins=128) == -1
    assert m2l(n_mels=129) == -1
    assert m2l(step=0.0) == -1 and b'step' in err()
    assert m2l(n_iter=-1) == -1


def test_wavernn_mels_map_back_to_natural_log_mels():
    """MCD is defined on ln(max(S, 1e-5)); WaveRNN's -100 dB floor is the same 1e-5, so the map is exact below 0 dB."""
    import torch
    from transformertts_b200.utils import evaluation as ev
    S = np.geomspace(1e-7, 1.0, 2000).reshape(25, 80)
    y = torch.from_numpy(ao.wavernn_normalize(S).astype(np.float32))
    ln = ev.natural_log_mels({'normalizer': 'WaveRNN'})(y).numpy()
    assert np.abs(ln - np.log(np.maximum(S, 1e-5))).max() < 2e-5
    m = torch.zeros(3, 80)
    assert ev.natural_log_mels({'normalizer': 'MelGAN'})(m) is m
    with pytest.raises(ValueError, match="normalizer is 'other'"):
        ev.natural_log_mels({'normalizer': 'other'}, 'config')
