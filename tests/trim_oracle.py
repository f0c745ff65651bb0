"""numpy restatement of the reference's silence trim, Audio.trim_audio_silence (data/audio.py:164-169):
librosa.effects.trim(y, top_db, frame_length=256, hop_length=64) of librosa 0.7.1, which is

    mse = feature.rms(y, frame_length, hop_length) ** 2             # reflect-padded by frame_length // 2, mean of squares
    non_silent = power_to_db(mse, ref=np.max, amin=1e-10, top_db=None) > -top_db
    [start, end) = [hop * first, min(len(y), hop * (last + 1))), or [0, 0) when no frame is non-silent.

`bounds64` computes it in float64, the squares added in sample order within each frame, as ttsb_trim_silence_bounds does.
`bounds32` writes librosa's own float32 expressions as they stand; the numpy installed here promotes scalars differently from
the numpy 1.x that librosa 0.7.1 ran on, so it approximates librosa's float32 result rather than reproducing it."""
import numpy as np

FRAME, HOP, AMIN = 256, 64, 1e-10


def frames(y: np.ndarray) -> np.ndarray:
    """(1 + L // 64, 256) view of the reflect-padded clip (librosa's util.frame of np.pad(y, 128, 'reflect'))."""
    x = np.pad(np.asarray(y), FRAME // 2, mode='reflect')
    n = 1 + (len(x) - FRAME) // HOP
    return np.lib.stride_tricks.as_strided(x, shape=(n, FRAME), strides=(HOP * x.itemsize, x.itemsize))


def powers64(y: np.ndarray) -> np.ndarray:
    """Frame powers in float64, each frame's 256 squares added in sample order -> (1 + L // 64,)."""
    fr = frames(np.asarray(y, dtype=np.float32)).astype(np.float64)
    acc = np.zeros(fr.shape[0])
    for k in range(FRAME):
        acc = acc + fr[:, k] * fr[:, k]
    return acc / FRAME


def db64(y: np.ndarray) -> np.ndarray:
    p = powers64(y)
    return 10.0 * np.log10(np.maximum(AMIN, p)) - 10.0 * np.log10(np.maximum(AMIN, p.max()))


def _bounds(non_silent: np.ndarray, n_samples: int) -> tuple:
    nz = np.flatnonzero(non_silent)
    if nz.size == 0:
        return 0, 0
    return int(nz[0] * HOP), int(min(n_samples, (nz[-1] + 1) * HOP))


def bounds64(y: np.ndarray, top_db: float) -> tuple:
    """[start, end) of the trimmed clip, float64 arithmetic."""
    return _bounds(db64(y) > -top_db, len(y))


def bounds32(y: np.ndarray, top_db: float) -> tuple:
    """[start, end) from librosa 0.7.1's float32 expressions, as this numpy evaluates them."""
    y = np.asarray(y, dtype=np.float32)
    x = frames(y).T                                                      # util.frame: (frame_length, n_frames)
    power = np.mean(np.abs(x) ** 2, axis=0, keepdims=True)               # feature.rms
    mse = np.sqrt(power) ** 2
    S = mse.squeeze()
    log_spec = 10.0 * np.log10(np.maximum(AMIN, S))                     # core.power_to_db(S, ref=np.max, top_db=None)
    log_spec -= 10.0 * np.log10(np.maximum(AMIN, np.max(S)))
    return _bounds(log_spec > -top_db, len(y))


def margin_db(y: np.ndarray, top_db: float) -> float:
    """Distance in dB of the frame closest to the threshold -top_db (float64)."""
    return float(np.min(np.abs(db64(y) + top_db)))


def trim(y: np.ndarray, top_db: float) -> np.ndarray:
    a, b = bounds64(y, top_db)
    return np.asarray(y)[a:b]


def padded_speech(n_clips: int, seed: int, fs: float = 22050.0, min_s: float = 1.0, max_s: float = 4.0) -> list:
    """Seeded speech-like clips (oracle/pitch_oracle.py speech_like_clip) with 0-2 s of leading and of trailing silence each, the
    silence digital zero or noise at a floor drawn from -100 to -50 dB re full scale -> list of float32 arrays."""
    from oracle import pitch_oracle as po
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_clips):
        x = po.speech_like_clip(float(rng.uniform(min_s, max_s)), seed * 1000 + i, fs=fs) * np.float32(rng.uniform(0.05, 0.9))
        parts = []
        for _ in range(2):
            n = int(rng.integers(0, int(2 * fs) + 1))
            floor = 0.0 if rng.random() < 0.25 else 10.0 ** (rng.uniform(-100.0, -50.0) / 20.0)
            parts.append((floor * rng.standard_normal(n)).astype(np.float32))
        out.append(np.concatenate([parts[0], x.astype(np.float32), parts[1]]))
    return out
