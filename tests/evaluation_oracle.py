"""Float64 restatement of MCD-DTW (include/ttsb.h: ttsb_mcd_dtw), in numpy, for the tests.

Every numpy elementwise operation rounds on its own, and the sums run in the order the definition gives (cepstra in increasing
mel bin, squared differences in increasing k), so ttsb_mcd_dtw must equal this bit for bit.  The DTW sweeps anti-diagonals
with the definition's tie rule: the diagonal predecessor unless another is strictly smaller, then (i - 1, j) before (i, j - 1)."""
import math

import numpy as np

KAPPA = 10.0 / math.log(10.0)


def dct_matrix(n_mels: int, n_ceps: int) -> np.ndarray:
    """Rows k = 1..n_ceps of the orthonormal DCT-II: sqrt(2 / M) cos(pi k (2m + 1) / (2M))."""
    m = np.arange(n_mels, dtype=np.float64)[None, :]
    k = np.arange(1, n_ceps + 1, dtype=np.float64)[:, None]
    return np.sqrt(2.0 / n_mels) * np.cos(np.pi * k * (2 * m + 1) / (2 * n_mels))


def cepstra(mel: np.ndarray, dct: np.ndarray) -> np.ndarray:
    """(T, M) float32 log-mels -> (T, K) float64: c_k[t] = sum_m dct[k][m] x[t][m], summed in increasing m from 0."""
    x = np.asarray(mel, dtype=np.float32).astype(np.float64)
    acc = np.zeros((x.shape[0], dct.shape[0]))
    for m in range(x.shape[1]):
        acc = acc + dct[:, m][None, :] * x[:, m][:, None]
    return acc


def frame_distances(ca: np.ndarray, cb: np.ndarray, kappa: float = KAPPA) -> np.ndarray:
    """(Ta, Tb): kappa sqrt(2 sum_k (ca_k - cb_k)^2), summed in increasing k from 0."""
    s = np.zeros((ca.shape[0], cb.shape[0]))
    for k in range(ca.shape[1]):
        t = ca[:, k][:, None] - cb[:, k][None, :]
        s = s + t * t
    return kappa * np.sqrt(2.0 * s)


def dtw(dist: np.ndarray) -> tuple:
    """-> (C[Tx-1][Ty-1], L[Tx-1][Ty-1]) over the cost matrix dist, by anti-diagonals."""
    Tx, Ty = dist.shape
    C = np.full((Tx, Ty), np.inf)
    L = np.zeros((Tx, Ty), dtype=np.int64)
    C[0, 0], L[0, 0] = dist[0, 0], 1
    for d in range(1, Tx + Ty - 1):
        i = np.arange(max(0, d - Ty + 1), min(d, Tx - 1) + 1)
        j = d - i
        best = np.full(i.shape, np.inf)
        ln = np.zeros(i.shape, dtype=np.int64)
        im, jm = np.maximum(i - 1, 0), np.maximum(j - 1, 0)
        diag = (i > 0) & (j > 0)
        best[diag], ln[diag] = C[im, jm][diag], L[im, jm][diag]
        for ok, ci, cj in ((i > 0, im, j), (j > 0, i, jm)):   # (i - 1, j), then (i, j - 1)
            sel = ok & (C[ci, cj] < best)
            best[sel], ln[sel] = C[ci, cj][sel], L[ci, cj][sel]
        C[i, j] = dist[i, j] + best
        L[i, j] = ln + 1
    return float(C[-1, -1]), int(L[-1, -1])


def mcd_dtw(mel_a: np.ndarray, mel_b: np.ndarray, n_ceps: int = 24) -> tuple:
    """-> (cost, path length, MCD = cost / length) of one pair of (T, n_mels) log-mels."""
    dct = dct_matrix(mel_a.shape[1], n_ceps)
    cost, length = dtw(frame_distances(cepstra(mel_a, dct), cepstra(mel_b, dct)))
    return cost, length, cost / length
