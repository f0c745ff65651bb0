"""The duration-extraction kernels (csrc/alignment.cu) and the decode-step and length kernels around them (csrc/decode.cu,
csrc/rowops.cu) against float64 / numpy / scipy at their edge shapes.

alignment.cu turns every Aligner attention map into the integer durations the ForwardTransformer trains on, so an error
there is a wrong label, not a wrong number.  Each kernel is called through lib.py on inputs built here:

- ttsb_attention_scores against a float64 restatement of utils/metrics.py (``scores_reference``): jumpiness exact,
  peakiness and diagonality relative to the sum of |terms|, with argmax ties in the same lane's strided scan and across
  lanes, uniform and all-zero rows, lengths above / below / equal to the padded shape, 0 and 1.
- ttsb_durations_from_attention against the dynamic programme of oracle/alignment_oracle.py (bit-exact, vectorised here
  over anti-diagonals in ``dp_durations``) and against scipy's Dijkstra (what the reference calls) on tie-free maps, fed
  with its own scores and with hand-made ones (tied best heads, a +inf head, score weighting).
- ttsb_decode_commit / ttsb_decode_prologue against numpy restatements of model/models.py:271-292 and the decoder
  prologue; ttsb_mel_lengths / ttsb_phoneme_lengths / ttsb_expand_indices against oracle/audio_oracle.py and
  oracle/forward_oracle.py, bit-exact.

Outputs start as a fill the kernel never writes (NaN, 0x7f or 0xff bytes): a cell left unwritten fails.

The builders of the inputs and the references are plain numpy, so tests/test_aligner_oracle.py also runs them on the CPU
to show that these inputs tell a right oracle from three wrong ones.
"""
import math

import numpy as np
import pytest
import torch

from oracle import alignment_oracle as ao
from oracle import audio_oracle as audio_o
from oracle import forward_oracle as fo
from transformertts_b200 import lib

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
U = 2.0 ** -24   # unit roundoff of float32
FILL_I32 = 0x7F7F7F7F
# fp32 LayerNorm + PE of the decode prologue, max |err| on outputs of magnitude up to ~5.  Measured on an H100 80GB HBM3
# (SXM, 700 W power limit): 5.4e-7 at d = 512, 1.8e-7 at d = 4.
GATE_PROLOGUE = 4e-6


# ----------------------------------------------------------------------------------------------------------------------
# references (numpy, float64 where the kernel rounds)
# ----------------------------------------------------------------------------------------------------------------------
def first_argmax(x, axis=-1):
    return np.argmax(x, axis=axis)


def last_argmax(x, axis=-1):
    """A WRONG argmax (the last maximum), used to show that the inputs below tell it apart."""
    n = x.shape[axis]
    return n - 1 - np.argmax(np.flip(x, axis=axis), axis=axis)


def scores_reference(att, mel_len, phon_len, r, argmax=first_argmax):
    """utils/metrics.py:5-44 with products and sums in float64 of the float32 inputs (the diagonal mask is cast to float32
    first, as the reference does).  -> jump (B,H) float32 (exact: an integer count over mel_len - 1 in double), then
    peak, sum|peak terms|, diag, sum|diag terms| (B,H) float64.  Lengths are the kernel's (``mel_lengths - 1``)."""
    B, H, Tq, Tk = att.shape
    jump = np.empty((B, H), np.float32)
    peak, peak_abs, diag, diag_abs = (np.empty((B, H)) for _ in range(4))
    q = np.arange(Tq)
    for b in range(B):
        ml, pl = int(mel_len[b]), int(phon_len[b])
        a = att[b].astype(np.float64)
        idx = argmax(att[b], axis=-1)                                        # (H, Tq)
        diff = np.abs(np.diff(idx, axis=-1))
        cnt = ((diff <= r) & (q[1:] < ml)[None]).sum(-1)
        with np.errstate(divide='ignore', invalid='ignore'):
            jump[b] = (cnt.astype(np.float64) / np.float64(ml - 1)).astype(np.float32)
            dm = ao.diagonal_mask(ml, pl, (Tq, Tk)).astype(np.float64)
        mx = att[b].max(-1).astype(np.float64) * (q < ml)[None]
        peak[b], peak_abs[b] = mx.sum(-1) / Tq, np.abs(mx).sum(-1) / Tq
        diag[b], diag_abs[b] = (a * dm).sum((-2, -1)), (np.abs(a) * dm).sum((-2, -1))
    return jump, peak, peak_abs, diag, diag_abs


def scores_tolerance(Tq, Tk):
    """|err| / sum|terms| of peakiness and diagonality.  From the kernel's accumulation order: a per-lane strided sum
    (ceil(Tk/32) adds), a 5-level warp tree, a per-warp row loop (ceil(Tq/8) adds), 8 warps in sequence, the product, the
    final division and, for diagonality, inverting 3 / d back here.

    Measured on an H100 80GB HBM3 (SXM, 700 W power limit), the worst case of each shape stays far inside the bound:
    27 u against 1642 u at Tq = 13000, Tk = 32; 14 u against 1651 u at 13000 x 300; 3.4 u against 151 u at 1000 x 300;
    at most 2.4 u against 18-58 u below that.  A dropped or doubled row costs 1 / Tq of the sum, which the shapes up to
    Tq = 1000 resolve (the largest one is there for its shared-memory path)."""
    return (math.ceil(Tk / 32) + math.ceil(Tq / 8) + 16) * U


def dp_durations(a, order='lud'):
    """oracle/alignment_oracle.py:durations_by_dynamic_programming vectorised over anti-diagonals: the same comparisons in
    the same order (``order``: left, up, diagonal) on the same float64 sums, so its result is the loop's, bit for bit.
    ``order`` other than 'lud' is a WRONG tie order, used to show that the plateau maps below tell it apart."""
    a = np.asarray(a, np.float32)
    M, N = a.shape
    w = (np.max(a) - a).astype(np.float64)
    dist = np.full((M, N), np.inf)
    code = np.zeros((M, N), np.int8)
    dist[0, 0] = 0.0
    for d in range(1, M + N - 1):
        j = np.arange(max(0, d - M + 1), min(d, N - 1) + 1)
        i = d - j
        cand = {'l': (j > 0, dist[i, j - 1], 0), 'u': (i > 0, dist[i - 1, j], 1), 'd': ((i > 0) & (j > 0), dist[i - 1, j - 1], 2)}
        best, c = np.full(j.size, np.inf), np.zeros(j.size, np.int8)
        for k in order:
            ok, v, cc = cand[k]
            take = ok & (v < best)
            best, c = np.where(take, v, best), np.where(take, cc, c)
        dist[i, j] = best + w[i, j]
        code[i, j] = c
    dur = np.zeros(N, np.int32)
    i, j, last_row = M - 1, N - 1, -1
    while True:
        if i != last_row:          # walking back, the first visit of a row is its right-most column on the path
            dur[j] += 1
            last_row = i
        if i == 0 and j == 0:
            return dur
        c = code[i, j]
        i, j = (i, j - 1) if c == 0 else ((i - 1, j) if c == 1 else (i - 1, j - 1))


def reference_matrix(al, s, ml, pl, weighted, start=1, argmax=first_argmax):
    """utils/alignments.py:119-126 for one batch row: al (H,Tq,Tk), s (H,3) float32 scores.  ``start`` = 0 is a WRONG crop
    (from row / column 0), used to show that the inputs below tell it apart."""
    Tq, Tk = al.shape[1:]
    M, N = min(ml, Tq) - 1, min(pl, Tk) - 1
    unpad = al[:, start:start + M, start:start + N]
    tot = (s[:, 2] + s[:, 0]) + s[:, 1]                     # diag_measure + jumpiness + peakiness, float32
    if weighted:
        return np.sum(unpad * tot[:, None, None], axis=0)   # float32, heads added in order
    return unpad[int(argmax(tot))]


def durations_reference(att, mel_len, phon_len, scores, weighted, start=1, argmax=first_argmax, order='lud'):
    """(B,Tk) int32: the kernel's contract, row by row.  A row whose cropped matrix is empty is all zero."""
    B, H, Tq, Tk = att.shape
    out = np.zeros((B, Tk), np.int32)
    for b in range(B):
        ml, pl = int(mel_len[b]), int(phon_len[b])
        M, N = min(ml, Tq) - 1, min(pl, Tk) - 1
        if M <= 0 or N <= 0:
            continue
        out[b, :N] = dp_durations(reference_matrix(att[b], scores[b], ml, pl, weighted, start, argmax), order)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------------
def diagonal_maps(rng, B, H, Tq, Tk, sharp=(6.0,)):
    """Softmax rows with a noisy diagonal, float32 (B,H,Tq,Tk): what a trained Aligner's cross-attention looks like.  The
    slope is capped so that no cell underflows to an exact 0: these maps are tie-free, the plateau maps below are not."""
    q = np.arange(Tq, dtype=np.float32)[:, None] / Tq
    k = np.arange(Tk, dtype=np.float32)[None, :] / Tk
    out = np.empty((B, H, Tq, Tk), np.float32)
    for b in range(B):
        for h in range(H):
            s = min(sharp[h % len(sharp)] * Tk / 8, 60.0)
            lg = rng.standard_normal((Tq, Tk), dtype=np.float32) - np.float32(s) * np.abs(q - k)
            e = np.exp(lg - lg.max(-1, keepdims=True))
            out[b, h] = e / e.sum(-1, keepdims=True)
    return out


# Pairs of equal maxima (k1 < k2) the argmax must resolve to k1.  Element k is read by lane k % 32 at stride k // 32:
# (0, 32) and (0, 64) are the same lane's strided scan one and two strides apart; (5, 22) are different lanes with the first
# maximum in the lower lane; (31, 40) are different lanes with the first maximum in the HIGHER lane (lane 31 against lane 8),
# which only the index comparison of the warp tree gets right.
TIE_PAIRS = ((0, 32), (0, 64), (5, 22), (31, 40))


def argmax_edge_rows(Tk):
    """Rows whose argmax is an edge (uniform, all zero, two equal maxima), each between rows peaked at the index the argmax
    must return.  A wrong choice is at least 9 columns away (or Tk - 1 away for the uniform and zero rows), so for r <= 5
    it changes the jumpiness count whenever Tk > 6."""
    def peaked(k):
        row = np.full(Tk, 0.01 / Tk, np.float32)
        row[k] = 0.9
        return row
    rows = [peaked(0), np.full(Tk, 1.0 / Tk, np.float32), np.full(Tk, 1.0 / Tk, np.float32), peaked(0),
            np.zeros(Tk, np.float32), np.zeros(Tk, np.float32), peaked(0)]             # uniform rows, all-zero rows
    for k1, k2 in TIE_PAIRS:
        if k2 < Tk:
            tie = np.full(Tk, 0.01 / Tk, np.float32)
            tie[k1] = tie[k2] = 0.45
            rows += [peaked(k1), tie, peaked(k1)]
    return np.stack(rows)


def make_score_inputs(Tq, Tk, H, seed):
    """(att (B,H,Tq,Tk), mel_len (B,), phon_len (B,)) with one row per length edge: mel_len = Tq, < Tq, > Tq, 1 (jumpiness
    0/0: NaN), 0; phon_len = Tk, < Tk, 0.  The argmax edge rows sit at the start of every map, padded rows are zero."""
    rng = np.random.default_rng(seed)
    lens = [(Tq, Tk), (max(Tq * 2 // 3, 2), max(Tk - 3, 0)), (Tq + 7, Tk), (1, Tk // 2), (0, 0), (max(Tq - 1, 2), 0)]
    mel_len = np.array([m for m, _ in lens], np.int32)
    phon_len = np.array([p for _, p in lens], np.int32)
    att = diagonal_maps(rng, len(lens), H, Tq, Tk, sharp=(3.0, 6.0, 12.0, 24.0))
    edge = argmax_edge_rows(Tk)
    n = min(len(edge), Tq - 1)
    att[:, :, 1:1 + n] = edge[:n]
    for b, (ml, pl) in enumerate(lens):
        att[b, :, max(ml, 0):] = 0.0          # padded frames: all-zero rows (argmax 0)
        att[b, :, :, pl + 1:] = 0.0           # padded phonemes
    return att, mel_len, phon_len


# (Tq, Tk, H, r): every Tq edge {2, 255, 257, 1000, 13000} (13000 * 4 B > 48 KB: the dynamic shared-memory path), every Tk
# edge {1, 31, 32, 33, 300} (one lane, a lane short of a warp, one warp, a warp and one, a strided scan), H in {1, 4} and
# r in {1, 2, 5}, each at least once.
SCORE_SHAPES = [(2, 1, 1, 1), (2, 33, 4, 2), (255, 31, 4, 5), (255, 300, 1, 1), (257, 32, 4, 2), (257, 1, 1, 5),
                (1000, 33, 1, 5), (1000, 300, 4, 1), (13000, 32, 1, 2), (13000, 300, 1, 5)]


def plateau_maps():
    """Maps whose path costs tie exactly: only the DP's comparison order (left, up, diagonal) decides them."""
    maps = {}
    # saturated softmax: exact 0 / 1 cells on a monotone staircase (several rows on one phoneme, phonemes skipped)
    M, N = 40, 25
    a = np.zeros((M, N), np.float32)
    cols = np.minimum((np.arange(M) * 0.7).astype(int), N - 1)
    a[np.arange(M), cols] = 1.0
    maps['saturated'] = a
    # M < N saturated: one 1 per row, the path must move right inside rows and skip phonemes
    a = np.zeros((12, 50), np.float32)
    a[np.arange(12), (np.arange(12) * 4.2).astype(int)] = 1.0
    maps['saturated_wide'] = a
    maps['all_equal'] = np.full((30, 17), 0.25, np.float32)
    # equal regions: constant blocks along the diagonal, one constant background
    a = np.full((48, 20), 0.125, np.float32)
    for s in range(4):
        a[12 * s:12 * s + 12, 5 * s:5 * s + 5] = 0.5
    maps['equal_blocks'] = a
    return maps


# Duration cases: name -> (Tq, Tk, H, rows of (mel_len, phon_len)); cropped M x N = min(len, T) - 1.
DURATION_SHAPES = {
    'M<N': (41, 121, 2, [(41, 121)]),                      # 40 x 120: moves right inside rows, zero durations
    'M=1,N>1': (8, 50, 2, [(2, 50)]),
    'N=1,M>1': (60, 8, 2, [(60, 2)]),
    'M=N': (65, 65, 2, [(65, 65)]),
    'M=N=1': (6, 6, 2, [(2, 2)]),
    'N=255': (301, 256, 1, [(301, 256)]),                  # the j loop of 256 threads: just short of a wrap
    'N=256': (301, 257, 1, [(301, 257)]),                  # exactly one pass
    'N=257': (301, 258, 1, [(301, 258)]),                  # wraps by one
    'N=600': (701, 601, 1, [(701, 601)]),                  # wraps twice
    'Tk=2100': (40, 2100, 1, [(40, 2100)]),                # 3 * 2100 * 8 B > 48 KB: dynamic shared memory, M << N
    'lj_1000x200': (1001, 201, 4, [(1001, 201)]),          # the LJSpeech scale
    'mel_len>Tq': (50, 30, 2, [(80, 30)]),                 # cropped at Tq as numpy slices do
    'ragged': (400, 150, 4, [(400, 150), (2, 150), (400, 2), (37, 149), (150, 1), (1, 40), (0, 9), (90, 0), (200, 77)]),
}


def make_duration_case(name, seed=0):
    Tq, Tk, H, rows = DURATION_SHAPES[name]
    rng = np.random.default_rng(seed + sum(map(ord, name)))
    ml = np.array([m for m, _ in rows], np.int32)
    pl = np.array([p for _, p in rows], np.int32)
    att = diagonal_maps(rng, len(rows), H, Tq, Tk, sharp=(2.0, 5.0, 3.0, 8.0))
    return att, ml, pl


def hand_scored_cases():
    """Hand-made scores that isolate the head selection: name -> (att, mel_len, phon_len, scores, weighted)."""
    rng = np.random.default_rng(77)
    att = diagonal_maps(rng, 2, 4, 60, 24, sharp=(1.0, 2.0, 4.0, 8.0))
    ml, pl = np.array([60, 45], np.int32), np.array([24, 20], np.int32)
    cases = {}
    s = np.zeros((2, 4, 3), np.float32)
    s[:, 1] = s[:, 3] = (0.5, 0.25, 2.0)       # heads 1 and 3 tie exactly: the first (1) wins
    s[:, 0], s[:, 2] = (0.5, 0.25, 1.0), (0.1, 0.1, 0.1)
    cases['tied_heads'] = (att, ml, pl, s, False)
    s = np.full((2, 4, 3), 1e30, np.float32)
    s[:, 2, 2] = np.inf                        # 3 / diagonality = +inf (a map with no weight on the diagonal mask) wins
    cases['inf_head'] = (att, ml, pl, s, False)
    s = rng.uniform(0.1, 3.0, (2, 4, 3)).astype(np.float32)
    cases['weighted'] = (att, ml, pl, s, True)
    return cases


def plateau_cases():
    """The plateau maps as one-head batches (mel_len / phon_len one past the map, cropped from row / column 1)."""
    cases = {}
    for name, m in plateau_maps().items():
        M, N = m.shape
        att = np.zeros((1, 1, M + 1, N + 1), np.float32)
        att[0, 0, 1:, 1:] = m
        att[0, 0, 0, :] = att[0, 0, :, 0] = 0.75   # row / column 0 are cropped away: a different map if read
        cases[name] = (att, np.array([M + 1], np.int32), np.array([N + 1], np.int32), np.zeros((1, 1, 3), np.float32), False)
    return cases


# ----------------------------------------------------------------------------------------------------------------------
# kernel calls
# ----------------------------------------------------------------------------------------------------------------------
def _i32(x):
    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.int32)).to(DEV)


def gpu_scores(att_d, ml, pl, r):
    B, H = att_d.shape[:2]
    scores = torch.full((B, H, 3), 0.0, device=DEV)
    scores.view(torch.int32).fill_(FILL_I32)               # 0x7f bytes: a finite 3.4e38, not NaN (jumpiness may be NaN)
    lib.attention_scores(att_d, _i32(ml), _i32(pl), r, scores)
    return scores


def gpu_durations(att_d, ml, pl, scores_d, weighted):
    B, H, Tq, Tk = att_d.shape
    scratch = torch.full((B * Tq * Tk,), 0xFF, dtype=torch.uint8, device=DEV)
    dur = torch.full((B, Tk), FILL_I32, dtype=torch.int32, device=DEV)
    lib.durations_from_attention(att_d, _i32(ml), _i32(pl), scores_d, weighted, scratch, dur)
    return dur.cpu().numpy()


def check_duration_rows(got, att, ml, pl, want, what):
    """The contract of every row: durations equal ``want``; sum(durations[:N]) == M when M, N >= 1 (the host assertion
    of durations_to_host); columns N.. are 0; an empty cropped matrix gives a row of zeros, written (not the fill)."""
    Tq, Tk = att.shape[2:]
    for b in range(att.shape[0]):
        M, N = min(int(ml[b]), Tq) - 1, min(int(pl[b]), Tk) - 1
        assert np.array_equal(got[b], want[b]), f'{what} row {b} (M={M}, N={N}): {got[b][:12]}... != {want[b][:12]}...'
        if M >= 1 and N >= 1:
            assert int(got[b, :N].sum()) == M, (what, b)
            assert (got[b, :N] >= 0).all(), (what, b)
            assert not got[b, N:].any(), (what, b)
        else:
            assert not got[b].any(), (what, b)


# ----------------------------------------------------------------------------------------------------------------------
# 1a. ttsb_attention_scores
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('Tq,Tk,H,r', SCORE_SHAPES, ids=[f'Tq{a}-Tk{b}-H{c}-r{d}' for a, b, c, d in SCORE_SHAPES])
def test_attention_scores_vs_float64(Tq, Tk, H, r):
    att, ml, pl = make_score_inputs(Tq, Tk, H, seed=Tq * 7 + Tk)
    got = gpu_scores(torch.from_numpy(att).to(DEV), ml, pl, r).cpu().numpy()
    jump, peak, peak_abs, diag, diag_abs = scores_reference(att, ml, pl, r)
    # jumpiness: an integer count over mel_len - 1 in double -> exact (NaN for mel_len 1, -0 for mel_len 0)
    np.testing.assert_array_equal(got[..., 0], jump)
    assert np.isnan(got[ml == 1, :, 0]).all() and np.isfinite(got[ml != 1, :, 0]).all()
    tol = scores_tolerance(Tq, Tk)
    err_p = np.abs(got[..., 1].astype(np.float64) - peak)
    assert (err_p <= tol * peak_abs).all(), f'peakiness {err_p.max():.3e}'
    # diagonality: the kernel returns 3 / d; a map with no weight under the mask gives d = 0 -> +inf
    empty = diag_abs == 0
    assert (got[..., 2][empty] == np.inf).all()
    with np.errstate(divide='ignore'):
        d_gpu = 3.0 / got[..., 2].astype(np.float64)
    err_d = np.abs(d_gpu - diag)[~empty]
    assert (err_d <= tol * diag_abs[~empty]).all(), f'diagonality {err_d.max():.3e}'
    worst = max((err_p / np.where(peak_abs > 0, peak_abs, 1)).max(), (err_d / diag_abs[~empty]).max(initial=0.0))
    print(f'[scores] Tq={Tq} Tk={Tk} H={H} r={r}: worst |err| / sum|terms| = {worst / U:.2f} u (bound {tol / U:.0f} u)')


# ----------------------------------------------------------------------------------------------------------------------
# 1b. ttsb_durations_from_attention
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('weighted', [False, True], ids=['best_head', 'weighted'])
@pytest.mark.parametrize('name', list(DURATION_SHAPES))
def test_durations_with_kernel_scores_vs_dp_and_dijkstra(name, weighted):
    att, ml, pl = make_duration_case(name)
    att_d = torch.from_numpy(att).to(DEV)
    scores_d = gpu_scores(att_d, ml, pl, 1)
    got = gpu_durations(att_d, ml, pl, scores_d, weighted)
    scores = scores_d.cpu().numpy()
    want = durations_reference(att, ml, pl, scores, weighted)
    check_duration_rows(got, att, ml, pl, want, name)
    Tq, Tk = att.shape[2:]
    for b in range(att.shape[0]):
        M, N = min(int(ml[b]), Tq) - 1, min(int(pl[b]), Tk) - 1
        if M < 1 or N < 1:
            continue
        ref = reference_matrix(att[b], scores[b], int(ml[b]), int(pl[b]), weighted)
        if M == 1 and N == 1:
            # The reference's Dijkstra path walk raises here (the source node's predecessor is -9999); the kernel answers
            # [1], the only vector the sum assertion accepts.  A deliberate divergence from the reference.
            with pytest.raises(IndexError):
                ao.extract_durations_with_dijkstra(ref)
            assert got[b, :1].tolist() == [1]
        elif M * N <= 250_000:
            # random float maps: no two path costs tie, so scipy's Dijkstra (what the reference calls) agrees
            assert np.array_equal(got[b, :N], ao.extract_durations_with_dijkstra(ref)), (name, b)
    if att.shape[0] > 1:   # every row of a ragged batch is bit-identical to that row run alone
        for b in range(att.shape[0]):
            alone = gpu_durations(att_d[b:b + 1].contiguous(), ml[b:b + 1], pl[b:b + 1], scores_d[b:b + 1].contiguous(), weighted)
            assert np.array_equal(alone[0], got[b]), (name, b)


@pytest.mark.parametrize('name', ['tied_heads', 'inf_head', 'weighted', 'saturated', 'saturated_wide', 'all_equal', 'equal_blocks'])
def test_durations_with_hand_made_scores_and_plateaus(name):
    """The search alone: head selection on hand-made scores (exact ties -> the first head, +inf wins, weighting as numpy
    does it in float32), and plateau maps whose path costs tie exactly, where the DP's comparison order decides."""
    att, ml, pl, s, weighted = {**hand_scored_cases(), **plateau_cases()}[name]
    got = gpu_durations(torch.from_numpy(att).to(DEV), ml, pl, torch.from_numpy(s).to(DEV), weighted)
    want = durations_reference(att, ml, pl, s, weighted)
    check_duration_rows(got, att, ml, pl, want, name)
    if name == 'tied_heads':   # the first of the tied heads, not the second, decides the durations
        assert not np.array_equal(want, durations_reference(att, ml, pl, s, weighted, argmax=last_argmax))


def test_durations_refuse_and_zero_empty_rows():
    """M <= 0 or N <= 0 on every row: all zero, written over the fill; Tk beyond shared memory is refused."""
    rng = np.random.default_rng(5)
    att = diagonal_maps(rng, 5, 2, 10, 7)
    ml, pl = np.array([1, 0, 10, 10, 1], np.int32), np.array([7, 7, 1, 0, 1], np.int32)
    s = np.ones((5, 2, 3), np.float32)
    got = gpu_durations(torch.from_numpy(att).to(DEV), ml, pl, torch.from_numpy(s).to(DEV), False)
    assert not got.any()
    big = torch.zeros(1, 1, 2, 7000, device=DEV)
    with pytest.raises(lib.TtsbError, match='Tk too large'):
        gpu_durations(big, np.array([2]), np.array([7000]), torch.ones(1, 1, 3, device=DEV), False)


# ----------------------------------------------------------------------------------------------------------------------
# 1c. decode step: ttsb_decode_commit, ttsb_decode_prologue
# ----------------------------------------------------------------------------------------------------------------------
def bf16_split(v):
    """split_bf16 of csrc/ttsb_common.cuh: hi = bf16_rn(v), lo = bf16_rn(v - hi) -> int16 bit patterns."""
    t = torch.from_numpy(np.ascontiguousarray(v, np.float32))
    hi = t.to(torch.bfloat16)
    lo = (t - hi.float()).to(torch.bfloat16)
    return hi.view(torch.int16).numpy(), lo.view(torch.int16).numpy()


def commit_reference(post, B, r, mel, stop_col, stop_index, max_iters, mel_out, stop_out, next_hi, next_lo, pos, done, n):
    """model/models.py:271-292, one iteration for a batch (as ttsb_decode_commit states it in include/ttsb.h); updates the
    arrays in place and returns all_done."""
    for b in range(B):
        if done[b]:
            continue
        ps = int(pos[b])
        frames = post[b * r:(b + 1) * r]
        mel_out[b, ps * r:(ps + 1) * r] = frames[:, :mel]
        if stop_out is not None:
            stop_out[b, ps * r:(ps + 1) * r] = frames[:, stop_col:stop_col + 3]
        hi, lo = bf16_split(frames[r - 1, :mel])                          # models.py:280: the last frame is the next input
        next_hi[b, :mel] = hi
        if next_lo is not None:
            next_lo[b, :mel] = lo
        am = int(np.argmax(frames[r - 1, stop_col:stop_col + 3]))        # tf.argmax: the first maximum
        n[b] = ps + 1
        if am == stop_index or ps + 1 >= max_iters:
            done[b] = 1
        else:
            pos[b] = ps + 1
    return int(all(done))


@pytest.mark.parametrize('nulls', [False, True], ids=['all_outputs', 'no_stop_out_no_next_lo'])
@pytest.mark.parametrize('scenario', ['mixed', 'all_stop'])
@pytest.mark.parametrize('r', [1, 2, 10])
def test_decode_commit_vs_numpy(r, scenario, nulls):
    """B = 20 sentences on 8 warps (the warp loop wraps), stop logits in columns above mel with a wider post row, the next
    input in a wider row; sentences already done are left alone; stop-logit ties go to the first maximum; a row stops by
    reaching max_iters; all_done set ('all_stop') and not set ('mixed')."""
    B, mel, stop_col, max_iters, stop_index = 20, 80, 84, 7, 1
    ld_post, ld_next = stop_col + 3 + 5, 96
    rng = np.random.default_rng(r * 10 + (scenario == 'all_stop'))
    post = rng.standard_normal((B * r, ld_post)).astype(np.float32)
    pos = rng.integers(0, max_iters - 1, B).astype(np.int32)
    done = np.zeros(B, np.int32)
    done[[6, 13, 19]] = 1
    stop_logits = {0: (0.0, 3.0, 1.0),    # clear stop
                   1: (3.0, 0.0, 1.0),    # clear continue
                   2: (2.0, 2.0, 0.0),    # tie of index 0 and the stop index: the first (0) wins -> continues
                   3: (0.0, 2.0, 2.0),    # tie of the stop index and index 2: the first (the stop index) wins -> stops
                   4: (3.0, 0.0, 1.0)}    # would continue, but reaches max_iters
    for b in range(B):
        kind = b % 5
        if scenario == 'all_stop' and kind in (1, 2):
            kind = 3
        post[b * r + r - 1, stop_col:stop_col + 3] = stop_logits[kind]
        if kind == 4:
            pos[b] = max_iters - 1
    T = max_iters * r
    mel_out = np.full((B, T, mel), np.nan, np.float32)
    stop_out = None if nulls else np.full((B, T, 3), np.nan, np.float32)
    next_hi = np.full((B, ld_next), -1, np.int16)        # 0xffff: a bf16 NaN
    next_lo = None if nulls else np.full((B, ld_next), -1, np.int16)
    n = np.full(B, -5, np.int32)
    d = {k: (None if v is None else torch.from_numpy(v.copy()).to(DEV))
         for k, v in dict(mel_out=mel_out, stop_out=stop_out, next_hi=next_hi, next_lo=next_lo, pos=pos, done=done, n=n).items()}
    all_done = torch.full((1,), FILL_I32, dtype=torch.int32, device=DEV)
    lib.decode_commit(torch.from_numpy(post).to(DEV), B, r, mel, stop_col, stop_index, max_iters, d['mel_out'], d['stop_out'],
                      d['next_hi'].view(torch.bfloat16), None if nulls else d['next_lo'].view(torch.bfloat16), d['pos'], d['done'],
                      d['n'], all_done)
    want_all = commit_reference(post, B, r, mel, stop_col, stop_index, max_iters, mel_out, stop_out, next_hi, next_lo, pos, done, n)
    np.testing.assert_array_equal(d['mel_out'].cpu().numpy(), mel_out)      # NaN where nothing is written
    if not nulls:
        np.testing.assert_array_equal(d['stop_out'].cpu().numpy(), stop_out)
        np.testing.assert_array_equal(d['next_lo'].cpu().numpy(), next_lo)
    np.testing.assert_array_equal(d['next_hi'].cpu().numpy(), next_hi)
    np.testing.assert_array_equal(d['pos'].cpu().numpy(), pos)
    np.testing.assert_array_equal(d['done'].cpu().numpy(), done)
    np.testing.assert_array_equal(d['n'].cpu().numpy(), n)
    assert int(all_done) == want_all == (1 if scenario == 'all_stop' else 0)
    if not nulls:   # hi + lo is the last frame up to the rounding of lo: |v - hi - lo| <= 2^-8 |v - hi| <= 2^-16 |v|
        live = np.flatnonzero(np.isin(np.arange(B), [6, 13, 19], invert=True))
        v = post[live * r + r - 1, :mel].astype(np.float64)
        hi = d['next_hi'].view(torch.bfloat16).float().cpu().numpy()[live, :mel].astype(np.float64)
        lo = d['next_lo'].view(torch.bfloat16).float().cpu().numpy()[live, :mel].astype(np.float64)
        assert (np.abs(hi + lo - v) <= 2.0 ** -16 * np.abs(v)).all()


@pytest.mark.parametrize('d', [4, 132, 384, 512])
def test_decode_prologue_vs_float64(d):
    """out[b] = LayerNorm(x[b]) + scalar * pe[clamp(pos[b], 0, pe_rows - 1)] for B = 13 rows (not a multiple of the 8 rows
    of a CTA), with positions below 0 and at or above pe_rows; hi / lo are the split of the fp32 output, bit-exact."""
    B, pe_rows, eps = 13, 50, 1e-6
    g = torch.Generator().manual_seed(d)
    x = torch.randn(B, d, generator=g) * 2.0 + 0.5
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    pe = fo.positional_encoding(pe_rows, d)[0]
    scalar = torch.tensor([1.3])
    pos = torch.tensor([-3, 0, 1, 49, 50, 1000, -1, 25, 7, 48, 2, 51, 13], dtype=torch.int32)
    out = torch.full((B, d), float('nan'), device=DEV)
    hi = torch.full((B, d), -1, dtype=torch.int16, device=DEV)
    lo = torch.full((B, d), -1, dtype=torch.int16, device=DEV)
    lib.decode_prologue(x.to(DEV), pos.to(DEV), gamma.to(DEV), beta.to(DEV), pe.to(DEV), scalar.to(DEV), eps, out,
                        hi.view(torch.bfloat16), lo.view(torch.bfloat16))
    t = pos.clamp(0, pe_rows - 1).long()
    ref = fo.layer_norm(x.double(), gamma.double(), beta.double(), eps) + scalar.double() * pe.double()[t]
    got = out.cpu()
    err = float((got.double() - ref).abs().max())
    print(f'[prologue] d={d}: max |err| {err:.2e}')
    assert err < GATE_PROLOGUE
    h_ref, l_ref = bf16_split(got.numpy())
    assert np.array_equal(hi.cpu().numpy(), h_ref) and np.array_equal(lo.cpu().numpy(), l_ref)


# ----------------------------------------------------------------------------------------------------------------------
# 1c. length kernels: ttsb_mel_lengths, ttsb_phoneme_lengths, ttsb_expand_indices
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('pad', [0.5, -1.0])
@pytest.mark.parametrize('C', [31, 80])
@pytest.mark.parametrize('T', [63, 64, 65, 1000])
def test_mel_lengths_nonzero_padding(T, C, pad):
    """utils/spectrogram_ops.py counts a frame when its number of non-pad channels differs from C * pad.  So a negative pad
    counts every frame, and with pad = 0.5, C = 80 a frame with exactly 40 non-pad channels is NOT counted, while an
    all-pad frame is.  T in {63, 64, 65, 1000}: one 64-frame block, exactly one, one and a frame, sixteen."""
    rng = np.random.default_rng(T * C)
    B = 4
    mel = rng.standard_normal((B, T, C)).astype(np.float32)
    mel[0, T // 2:] = pad                                          # trailing padding
    mel[1, ::3] = pad                                              # interior all-pad frames
    half = np.arange(C) < C // 2
    mel[2, 1::2, :][:, half] = pad                                 # exactly C // 2 pad channels (40 of 80 non-pad)
    k = rng.integers(0, C + 1, T)
    mel[3] = np.where(np.arange(C)[None] < k[:, None], pad, mel[3])   # any count of pad channels
    out = torch.full((B,), FILL_I32, dtype=torch.int32, device=DEV)
    lib.mel_lengths(torch.from_numpy(mel).to(DEV), pad, out)
    got = out.cpu().numpy()
    nonpad = (mel != np.float32(pad)).sum(-1)
    want = (nonpad != C * pad).sum(-1)
    np.testing.assert_array_equal(got, audio_o.mel_lengths(mel, pad))
    np.testing.assert_array_equal(got, want)
    if pad < 0:
        assert (got == T).all()
    if C == 80 and pad == 0.5:
        assert got[2] == T - T // 2                                # the 40-channel frames are not counted


@pytest.mark.parametrize('T', [37, 300, 1000])
def test_phoneme_lengths_nonzero_padding(T):
    """A non-zero padding token with pads inside the sequence (counted out) and zeros (counted in)."""
    rng = np.random.default_rng(T)
    ph = rng.integers(0, 8, (5, T)).astype(np.int32)
    ph[1, T // 3:] = 3
    ph[2] = 3
    ph[3] = 0
    out = torch.full((5,), FILL_I32, dtype=torch.int32, device=DEV)
    lib.phoneme_lengths(torch.from_numpy(ph).to(DEV), 3, out)
    got = out.cpu().numpy()
    np.testing.assert_array_equal(got, audio_o.phoneme_lengths(ph, 3))
    assert got[2] == 0 and got[3] == T


def test_expand_indices_at_the_shared_memory_limit():
    """Tp = 12000 (48 000 B of scan, the largest accepted) is exact; 12001 is refused.  A row of zero durations maps every
    frame to -1; Tm above every row total pads with -1, Tm below a row total keeps that row's first Tm frames."""
    rng = np.random.default_rng(12000)
    B, Tp = 3, 12000
    dur = rng.integers(0, 3, (B, Tp)).astype(np.int32)
    dur[1] = 0
    dur[2, ::2] = 0
    dur_t = torch.from_numpy(dur)
    lens, idx_ref = fo.expand_indices(dur_t)
    tot = lens.numpy()
    for Tm in (int(tot.max()) + 5, int(tot[2]) - 100):
        want = np.full((B, Tm), -1, np.int32)
        w = idx_ref.numpy()[:, :Tm]
        want[:, :w.shape[1]] = w
        out = torch.full((B, Tm), FILL_I32, dtype=torch.int32, device=DEV)
        lib.expand_indices(dur_t.to(DEV), Tm, out)
        np.testing.assert_array_equal(out.cpu().numpy(), want)
        assert (out[1] == -1).all()
    with pytest.raises(lib.TtsbError, match='Tp too large for the shared-memory scan'):
        lib.expand_indices(torch.zeros(1, Tp + 1, dtype=torch.int32, device=DEV), 4, torch.zeros(1, 4, dtype=torch.int32, device=DEV))
