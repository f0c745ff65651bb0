"""numpy restatement of what librosa 0.7.1 ``load(path, sr=...)`` does to a mono clip at another rate (reference:
data/audio.py:126-130): ``resample(y, sr_native, sr, res_type='kaiser_best')``, i.e. resampy (>= 0.2.2) ``resample(...,
filter='kaiser_best')`` followed by ``fix_length`` to ceil(L ratio).  The test-side counterpart of ``ttsb_resample_batch``; the
product package never imports it.

The filter is built here from resampy's published parameters (64 zero crossings, 512 table entries per crossing, Kaiser beta
14.769656459379492, rolloff 0.9475937167399596).  resampy ships the table as a precomputed file; agreement with that file in the
last bits is not verified.

resample_f's loop is vectorised over output samples, one tap index at a time, with resampy's operation order: float64 throughout,
the float32 accumulator rounded after every tap, and the time register r_{t+1} = r_t + 1/ratio accumulated serially
(np.add.accumulate adds left to right)."""
import numpy as np

NUM_ZEROS, NUM_TABLE = 64, 512
BETA, ROLLOFF = 14.769656459379492, 0.9475937167399596


def half_window() -> np.ndarray:
    """The right half of the kaiser_best interpolation filter -> float64 (NUM_ZEROS * NUM_TABLE + 1,)."""
    from scipy.signal.windows import kaiser
    n = NUM_ZEROS * NUM_TABLE
    sinc_win = ROLLOFF * np.sinc(ROLLOFF * np.linspace(0, NUM_ZEROS, num=n + 1, endpoint=True))
    return kaiser(2 * n + 1, BETA)[n:] * sinc_win


_WINDOW = None


def _window():
    global _WINDOW
    if _WINDOW is None:
        _WINDOW = half_window()
    return _WINDOW


def tables(ratio: float):
    """(h', D', scale, step): the table scaled by ratio when downsampling, its forward differences (last one 0)."""
    win = _window()
    if ratio < 1:
        win = win * ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    scale = min(1.0, ratio)
    return win, delta, scale, int(scale * NUM_TABLE)


def time_register(n_out: int, ratio: float) -> np.ndarray:
    """r_0 = 0, r_{t+1} = fl(r_t + 1/ratio) -> float64 (n_out,)."""
    steps = np.full(n_out, 1.0 / ratio)
    steps[0] = 0.0
    return np.add.accumulate(steps)


def resample(x, sr_orig: int, sr_new: int) -> np.ndarray:
    """float32 mono clip at sr_orig -> float32 clip of ceil(L sr_new / sr_orig) samples at sr_new (unchanged when the rates
    agree).  Raises ValueError when int(L ratio) < 1, as resampy does."""
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    if sr_orig == sr_new:
        return x.copy()
    ratio = float(sr_new) / sr_orig
    n_out = int(len(x) * ratio)
    if n_out < 1:
        raise ValueError(f'input of {len(x)} samples is too short to resample from {sr_orig} to {sr_new} Hz')
    win, delta, scale, step = tables(ratio)
    nwin, L = len(win), len(x)
    r = time_register(n_out, ratio)
    m = r.astype(np.int64)
    frac = scale * (r - m)
    xd = x.astype(np.float64)
    y = np.zeros(n_out, np.float32)
    for side in (0, 1):
        f = frac if side == 0 else scale - frac
        idx = f * NUM_TABLE
        off = idx.astype(np.int64)
        eta = idx - off
        count = np.minimum(m + 1, (nwin - off) // step) if side == 0 else np.minimum(L - m - 1, (nwin - off) // step)
        for i in range(int(max(count.max(), 0))):
            sel = np.nonzero(i < count)[0]
            j = off[sel] + i * step
            w = win[j] + eta[sel] * delta[j]
            src = m[sel] - i if side == 0 else m[sel] + i + 1
            y[sel] = (y[sel].astype(np.float64) + w * xd[src]).astype(np.float32)
    n_total = int(np.ceil(L * ratio))
    return np.concatenate([y, np.zeros(max(0, n_total - n_out), np.float32)])[:n_total]


def tone(freq: float, sr: int, seconds: float, amp: float = 0.5) -> np.ndarray:
    t = np.arange(int(round(seconds * sr))) / sr
    return (amp * np.sin(2 * np.pi * freq * t)).astype(np.float32)


def noisy_tones(n: int, sr: int, seed: int) -> np.ndarray:
    """Seeded noise plus a few tones below the Nyquist rate of 8 kHz, about 0.3 rms -> float32 (n,)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    y = 0.1 * rng.standard_normal(n)
    for f in rng.uniform(80.0, 3900.0, size=3):
        y += 0.2 * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi))
    return y.astype(np.float32)
