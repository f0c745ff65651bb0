"""CPU tests of how create_training_data.py groups files into GPU batches: the budget counts each file's samples at the configured
rate, so a corpus at that rate is split exactly as by Audio.load_wav, and off-rate files count what they become after resampling."""
import numpy as np
import scipy.io.wavfile

FS = 22050


def _audio():
    from transformertts_b200.data.audio import Audio
    return Audio(sampling_rate=FS, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                 normalizer='MelGAN')


def _write(path, n, sr, seed):
    scipy.io.wavfile.write(path, sr, (np.random.default_rng(seed).standard_normal(n) * 3000).astype(np.int16))


def test_budget_counts_samples_of_files_at_the_configured_rate(tmp_path):
    import create_training_data as ctd
    audio = _audio()
    paths = []
    for i in range(200):
        paths.append(tmp_path / f'{i:03d}.wav')
        _write(paths[-1], 100000, FS, i)
    got = list(ctd.batches(paths, 400000, ctd.wav_loader(audio), ctd.loaded_samples(audio)))
    assert [len(b) for b in got] == [4] * 50
    # the grouping and the samples are those of the loader that reads every file with Audio.load_wav
    plain = list(ctd.batches(paths, 400000, lambda p: audio.load_wav(str(p))[0]))
    assert [[p for p, _ in b] for b in got] == [[p for p, _ in b] for b in plain]
    for b, c in zip(got, plain):
        for (_, (y, sr)), (_, z) in zip(b, c):
            assert sr is None and np.array_equal(y, z)


def test_budget_counts_off_rate_files_after_resampling(tmp_path):
    import create_training_data as ctd
    audio = _audio()
    paths = []
    for i in range(30):
        paths.append(tmp_path / f'{i:03d}.wav')
        _write(paths[-1], 96000, 48000, i)             # 44100 samples at 22050 Hz
    got = list(ctd.batches(paths, 4 * 44100, ctd.wav_loader(audio), ctd.loaded_samples(audio)))
    assert [len(b) for b in got] == [4] * 7 + [2]
    assert all(sr == 48000 and len(y) == 96000 for b in got for _, (y, sr) in b)
