"""Float64 numpy restatement of WORLD's CheapTrick (pyworld.cheaptrick with q1 = -0.15, f0_floor = 71) and of pysptk's sp2mc /
mcepalpha, written from the published algorithms (WORLD's cheaptrick.cpp and common.cpp, SPTK's freqt) as csrc/world_sp.cu
reads them, step by step and one frame at a time.  The safeguard noise is the counter-based draw world_sp.cu uses in place of
WORLD's sequential generator, restated bit for bit.  Test infrastructure only: the product package never imports it."""
import numpy as np

SAFE_GUARD = 1e-12                 # world::kMySafeGuardMinimum
EPS = 2.220446049250313e-16        # world::kEps
DEFAULT_F0 = 500.0                 # world::kDefaultF0
Q1 = -0.15
F0_FLOOR = 71.0


def matlab_round(x: float) -> int:
    return int(x + 0.5) if x > 0 else int(x - 0.5)


def n_frames(L: int, fs: int, frame_period: float) -> int:
    return int(1000.0 * L / fs / frame_period) + 1


def fft_size(fs: int, f0_floor: float = F0_FLOOR) -> int:
    """WORLD's GetFFTSizeForCheapTrick: 2^(1 + int(log2(3 fs / f0_floor + 1)))."""
    return int(2.0 ** (1 + int(np.log(3.0 * fs / f0_floor + 1) / np.log(2.0))))


# ---- the safeguard noise: WORLD's randn (12 uniforms of 28 bits, / 2^28 - 6) of splitmix64-hashed uniforms
def _mix(x):
    with np.errstate(over='ignore'):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def randn(frame: int, index, site: int) -> np.ndarray:
    """Draws keyed by (clip-local frame, index array, site 0: windowed samples / 1: spectrum bins)."""
    idx = np.asarray(index, dtype=np.uint64)
    z = _mix((np.uint64(frame) << np.uint64(32)) | (np.uint64(site) << np.uint64(16)) | idx)
    s = np.zeros(idx.shape, dtype=np.uint64)
    for r in range(6):
        h = _mix(z ^ np.uint64(r))
        s += (h >> np.uint64(36)) + ((h >> np.uint64(4)) & np.uint64(0xFFFFFFF))
    return s.astype(np.float64) / 268435456.0 - 6.0


def interp1q(x0: float, dx: float, y: np.ndarray, xi: np.ndarray) -> np.ndarray:
    """WORLD's interp1Q: y on the axis x0 + k dx, linear, the step past the last point taken as 0."""
    base = ((xi - x0) / dx).astype(np.int64)          # C's truncation toward zero
    frac = (xi - x0) / dx - base
    dy = np.append(np.diff(y), 0.0)
    return y[base] + dy[base] * frac


def cheaptrick_frame(x: np.ndarray, fs: int, frame: int, frame_period: float, f0: float, n: int, q1: float = Q1) -> np.ndarray:
    """The envelope (n / 2 + 1,) of clip x at clip-local frame `frame` (t = frame frame_period / 1000)."""
    x = np.asarray(x, dtype=np.float64)
    nh = n // 2
    if f0 <= 3.0 * fs / (n - 3.0):
        f0 = DEFAULT_F0
    if not f0 <= fs / 4.0:
        return np.full(nh + 1, np.nan)
    t = frame * frame_period / 1000.0
    # windowed waveform
    half = matlab_round(1.5 * fs / f0)
    k = np.arange(-half, half + 1)
    origin = matlab_round(t * fs + 0.001)
    idx = np.minimum(len(x) - 1, np.maximum(0, origin + k))
    w = 0.5 * np.cos(np.pi * (k / 1.5 / fs) * f0) + 0.5
    w = w / np.sqrt(np.sum(w * w))
    v = x[idx] * w + randn(frame, np.arange(2 * half + 1), 0) * SAFE_GUARD
    v = v - w * (np.sum(v) / np.sum(w))
    # power spectrum with the DC correction
    spec = np.fft.fft(np.concatenate([v, np.zeros(n - len(v))]))[:nh + 1]
    p = spec.real * spec.real + spec.imag * spec.imag
    ul = 2 + int(f0 * n / fs)
    axis = np.arange(ul - 1) * fs / n
    p[:ul - 1] = p[:ul - 1] + interp1q(f0, -fs / n, p[:ul + 1], axis)
    # linear smoothing
    width = f0 * 2.0 / 3.0
    bd = int(width * n / fs) + 1
    mirrored = np.concatenate([p[bd:0:-1], p[:nh], p[nh::-1][:bd + 1]])
    seg = np.cumsum(mirrored * fs / n)
    f_lo = np.arange(nh + 1) / n * fs - width / 2.0
    x0 = -(bd - 0.5) * fs / n
    lo = interp1q(x0, fs / n, seg, f_lo)
    hi = interp1q(x0, fs / n, seg, f_lo + width)
    p = (hi - lo) / width + np.abs(randn(frame, np.arange(nh + 1), 1)) * EPS
    # smoothing with recovery on the cepstrum
    logp = np.log(p)
    cep = np.fft.fft(np.concatenate([logp, logp[nh - 1:0:-1]])).real[:nh + 1]
    q = np.arange(1, nh + 1) / fs
    sl = np.concatenate([[1.0], np.sin(np.pi * f0 * q) / (np.pi * f0 * q)])
    cl = np.concatenate([[(1.0 - 2.0 * q1) + 2.0 * q1], (1.0 - 2.0 * q1) + 2.0 * q1 * np.cos(2.0 * np.pi * q * f0)])
    lift = cep * sl * cl / n
    return np.exp(np.fft.irfft(lift, n) * n)[:nh + 1]


def cheaptrick(x: np.ndarray, fs: int, f0: np.ndarray, frame_period: float, n: int = None, q1: float = Q1) -> np.ndarray:
    """(frames, n / 2 + 1) envelope of one clip at its F0 contour (one value per WORLD frame)."""
    n = fft_size(fs) if n is None else n
    return np.stack([cheaptrick_frame(x, fs, i, frame_period, float(f), n, q1) for i, f in enumerate(f0)])


# ---- SPTK
def freqt(c: np.ndarray, order: int, alpha: float) -> np.ndarray:
    """SPTK's freqt: the frequency-warped cepstrum (order + 1,) of c (all of its coefficients), the recursion as written; c may
    carry trailing axes (one recursion per column)."""
    c = np.asarray(c, dtype=np.float64)
    b = 1.0 - alpha * alpha
    g = np.zeros((order + 1,) + c.shape[1:])
    for i in range(len(c) - 1, -1, -1):
        d = g.copy()
        g[0] = c[i] + alpha * d[0]
        if order >= 1:
            g[1] = b * d[0] + alpha * d[1]
        for j in range(2, order + 1):
            g[j] = d[j - 1] + alpha * (d[j] - g[j - 1])
    return g


def sp2mc(sp: np.ndarray, order: int, alpha: float) -> np.ndarray:
    """pysptk.sp2mc of one envelope (n / 2 + 1,): irfft of log sp, c0 halved, freqt."""
    c = np.fft.irfft(np.log(sp))
    c[0] /= 2.0
    return freqt(c, order, alpha)


def mcepalpha(fs: int, start: float = 0.0, stop: float = 1.0, step: float = 0.001, num_points: int = 1000) -> float:
    """pysptk.util.mcepalpha: the alpha on a grid whose all-pass warping is closest (mean square) to the mel scale."""
    f = (fs / 2.0) / num_points * np.arange(num_points)
    mel = 1000.0 / np.log(2) * np.log(1 + f / 1000.0)
    mel = mel / mel[-1]
    omega = np.pi / num_points * np.arange(num_points)
    best, best_d = None, np.inf
    for a in np.arange(start, stop, step):
        with np.errstate(divide='ignore', invalid='ignore'):
            warp = np.arctan((1 - a * a) * np.sin(omega) / ((1 + a * a) * np.cos(omega) - 2 * a))
        warp[warp < 0] += np.pi
        warp = warp / warp[-1]
        d = np.sum(np.abs((mel - warp) ** 2)) / num_points
        if d < best_d:
            best, best_d = a, d
    return float(best)


def world_mcep(x: np.ndarray, fs: int, f0: np.ndarray, frame_period: float, order: int = 24, alpha: float = None) -> np.ndarray:
    """(frames, order + 1) mel-cepstra of one clip: CheapTrick at f0, then sp2mc at alpha (mcepalpha(fs) when None)."""
    alpha = mcepalpha(fs) if alpha is None else alpha
    sp = cheaptrick(x, fs, f0, frame_period)
    return np.stack([sp2mc(s, order, alpha) for s in sp])
