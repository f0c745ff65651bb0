"""Float64 restatement of the warping path of ttsb_mcd_dtw_path (include/ttsb.h), in numpy, for the tests.

The sweep is evaluation_oracle.dtw's (anti-diagonals, the same float64 sums and the same tie rule: the diagonal predecessor
unless another is strictly smaller, then (i - 1, j) before (i, j - 1)); it also records which predecessor each cell took and
walks back from (Tx - 1, Ty - 1) to (0, 0)."""
import numpy as np

DIAG, UP, LEFT = 0, 1, 2   # (i - 1, j - 1), (i - 1, j), (i, j - 1)
STEP = {DIAG: (1, 1), UP: (1, 0), LEFT: (0, 1)}


def dtw_path(dist: np.ndarray) -> tuple:
    """-> (C[Tx-1][Ty-1], L[Tx-1][Ty-1], path int32 (L, 2) of (i, j) from (0, 0) to (Tx - 1, Ty - 1))."""
    Tx, Ty = dist.shape
    C = np.full((Tx, Ty), np.inf)
    L = np.zeros((Tx, Ty), dtype=np.int64)
    choice = np.zeros((Tx, Ty), dtype=np.int8)
    C[0, 0], L[0, 0] = dist[0, 0], 1
    for d in range(1, Tx + Ty - 1):
        i = np.arange(max(0, d - Ty + 1), min(d, Tx - 1) + 1)
        j = d - i
        best = np.full(i.shape, np.inf)
        ln = np.zeros(i.shape, dtype=np.int64)
        ch = np.zeros(i.shape, dtype=np.int8)
        im, jm = np.maximum(i - 1, 0), np.maximum(j - 1, 0)
        diag = (i > 0) & (j > 0)
        best[diag], ln[diag] = C[im, jm][diag], L[im, jm][diag]
        for code, ok, ci, cj in ((UP, i > 0, im, j), (LEFT, j > 0, i, jm)):
            sel = ok & (C[ci, cj] < best)
            best[sel], ln[sel], ch[sel] = C[ci, cj][sel], L[ci, cj][sel], code
        C[i, j] = dist[i, j] + best
        L[i, j] = ln + 1
        choice[i, j] = ch
    return float(C[-1, -1]), int(L[-1, -1]), traceback(choice)


def traceback(choice: np.ndarray) -> np.ndarray:
    """The path that ends at the last cell of a (Tx, Ty) table of predecessor choices, from (0, 0)."""
    i, j = choice.shape[0] - 1, choice.shape[1] - 1
    path = [(i, j)]
    while (i, j) != (0, 0):
        di, dj = STEP[int(choice[i, j])]
        i, j = i - di, j - dj
        path.append((i, j))
    return np.array(path[::-1], dtype=np.int32)


def path_sum(dist: np.ndarray, path: np.ndarray) -> float:
    """d along the path summed as the recursion does: d_n + (d_{n-1} + (... + d_0))."""
    acc = float(dist[path[0][0], path[0][1]])
    for i, j in path[1:]:
        acc = float(dist[i, j]) + acc
    return acc
