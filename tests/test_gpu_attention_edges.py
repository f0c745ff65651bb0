"""The attention kernels against float64 at their tile edges, with peaked logits and in every operand layout the model passes.

ttsb_mha_fwd streams 64-key tiles past 128-query tiles and keeps a lazy running maximum (the reference point moves only when
a row maximum grows by more than 2^8 in exp2 units, so P reaches 256 before normalisation; the O rescale is gated per warp).
ttsb_attn_probs_fwd / ttsb_attn_ds_bwd run 128x64 tiles through a ring of K boxes, ttsb_decode_attn splits the keys over
CTAs and combines the parts.  randn inputs give flat softmax rows that none of this matters for, so the logits here are
constructed (_peaked): coordinate s < 4 of each head of q selects schedule s, whose scaled logit per key the same coordinate
of k carries, and the other coordinates are small noise; schedule 'f' rows instead copy the +-beta code of one key, so that
row is near one-hot.  Every reference is float64 on the exact 16-bit operands the kernel reads (gpu_util.operand16), and
every tolerance is a bound derived from the kernel's arithmetic (_out_tol, _prob_tol), not fitted to an observed error.
Outputs start poisoned: every element a kernel owns must be written, every other one left alone, padding exactly +0.
"""
import math

import pytest
import torch

from gpu_util import DEV, _poison16, operand16, ref_mha_general, run_mha_general

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24   # fp32 unit roundoff
SCHEDULES = 'abcdf'
NSEL = 4           # selector coordinates per head: schedules a, b, c, d
MASKED_LOGIT = 40.0  # scaled logit of keys >= kv_len: far above every live key, so a key the kernel fails to mask shows


def _lib():
    from transformertts_b200 import lib
    lib.load()
    return lib


def _schedule(s: str, n: int, Tk: int, gen) -> torch.Tensor:
    """float64 (Tk,) scaled logits of schedule s for a row with n live keys, in natural-log units (the threshold of the
    lazy maximum, 8 in exp2 units, is 8 ln 2 = 5.545 here):
    a  the tile maximum grows by 1.75 per 64-key tile: 5.25 after three tiles (P = e^5.25 = 190 before normalisation), the
       reference moves at the fourth;
    b  it grows by 6.0 per tile, just over the threshold: O is rescaled at every tile;
    c  the maximum is in the first tile and every later tile is 300 lower: P flushes to 0 through ex2.approx.ftz;
    d  the maximum (+12) is the last live key n - 1, in the last, partial key tile.
    Within a tile the keys sit up to 2 below the schedule value (uniform)."""
    tile = (torch.arange(Tk) // 64).double()
    jit = -2.0 * torch.rand(Tk, generator=gen, dtype=torch.float64)
    if s == 'a':
        L = 1.75 * tile + jit
    elif s == 'b':
        L = 6.0 * tile + jit
    elif s == 'c':
        L = torch.where(tile == 0, jit, jit - 300.0)
    else:
        L = jit.clone()
        L[n - 1] = 12.0
    L[n:] = MASKED_LOGIT
    return L


def _peaked(B, T, Tk, H, dh, lens, rows, seed, causal=False):
    """fp32 CPU q (B,T,H*dh), k, v (B,Tk,H*dh).  rows: (B,T) schedule letter per query row ('f': near one-hot on a live,
    causally visible key).  The selector and code values are exact in bf16 and fp16 (their bf16x3 lo parts are zero), the
    noise is not."""
    g = torch.Generator().manual_seed(seed)
    beta = 2.0 if dh <= 128 else 4.0
    q = 0.01 * torch.randn(B, T, H, dh, generator=g)
    k = beta * (2.0 * torch.randint(0, 2, (B, Tk, H, dh), generator=g).float() - 1.0)
    v = torch.randn(B, Tk, H, dh, generator=g)
    for b in range(B):
        n = int(lens[b])
        for s in range(NSEL):
            col = (_schedule(SCHEDULES[s], n, Tk, g) * math.sqrt(dh)).float().bfloat16().float()
            k[b, :, :, s] = col[:, None]
    sel = torch.tensor([[SCHEDULES.index(c) for c in r] for r in rows])          # (B, T)
    q[..., :NSEL] = 0.0
    onehot = torch.nn.functional.one_hot(sel.clamp(max=NSEL - 1), NSEL).float()[:, :, None, :]
    q[..., :NSEL] = torch.where((sel < NSEL)[:, :, None, None], onehot, q[..., :NSEL])
    t = torch.arange(T)[None, :]
    visible = torch.as_tensor(lens)[:, None].clamp(max=Tk)
    if causal:
        visible = torch.minimum(visible, t + 1)
    tgt = (7 * t + 3) % visible                                                   # (B, T) live key of each 'f' row
    code = k[torch.arange(B)[:, None], tgt][..., NSEL:]                            # (B, T, H, dh - NSEL)
    f = (sel == NSEL)[:, :, None, None]
    q[..., NSEL:] = torch.where(f, code, q[..., NSEL:])
    d = H * dh
    return q.reshape(B, T, d), k.reshape(B, Tk, d), v.reshape(B, Tk, d)


def _rows(B, T, kind):
    if kind == 'mix':      # every schedule inside every warp's 16 rows
        return [[SCHEDULES[(t + 2 * b) % 5] for t in range(T)] for b in range(B)]
    if kind == 'e':        # (a) and (c) alternate: the warp-wide rescale multiplies rows whose alpha is 1
        return [['a' if t % 2 else 'c' for t in range(T)] for _ in range(B)]
    return [[kind] * T for _ in range(B)]


def _heads(t, H):
    B, n, d = t.shape
    return t.reshape(B, n, H, d // H).permute(0, 2, 1, 3)


def _logit_err(q, k, H, precision):
    """float64 (B,H,T,Tk): bound on the error of a kernel's scaled logit in natural-log units.  An fp32 dot product of dh
    terms accumulated with unit 2^-23 (truncating tensor-core adds included) errs by at most dh 2^-23 sum_i |q_i k_i|; the
    exp2 argument s*c - m*c and the running reference are rounded once more per key tile, 2^-23 |logit| each; bf16x3 drops
    the lo*lo product, at most sum_i |lo(q_i) lo(k_i)|."""
    qd, kd = operand16(q, precision), operand16(k, precision)
    dh = q.shape[-1] // H
    E = _heads(qd, H).abs() @ _heads(kd, H).abs().transpose(-1, -2) / math.sqrt(dh)
    n_tiles = (k.shape[1] + 63) // 64 + 1
    err = 2 * U24 * (dh + n_tiles) * E
    if precision == 'bf16x3':
        ql, kl = qd - operand16(q, 'bf16'), kd - operand16(k, 'bf16')
        err = err + _heads(ql, H).abs() @ _heads(kl, H).abs().transpose(-1, -2) / math.sqrt(dh)
    return err


# P as the A operand of O += P V, rounded to nearest: fp16 (11 significant bits), bf16 (8) or bf16 hi + lo (16)
P_ROUND = {'fp16': 2.0 ** -11, 'bf16': 2.0 ** -8, 'bf16x3': 2.0 ** -16}


def _out_tol(q, k, v, w, H, precision, impl, out_lo=True):
    """float64 (B,T,d) bound on |O_kernel - O_ref| per element.  With w the float64 softmax and e_k the logit error bound
    of key k (_logit_err), the kernel's O = sum_k P~_k V_k / sum_k P_k differs from sum_k w_k V_k by at most
      sum_k w_k (u_P + u_exp + u_acc + e_k) |V_k|          P rounded to the MMA operand type (u_P, SIMT: none), ex2.approx
                                                          (2^-22 per call, one more per rescale of O and l), fp32 sums of
                                                          P V and of l over Tk keys (Tk 2^-23)
      + (sum_k w_k e_k) sum_k w_k |V_k|                    the logit errors through the normalisation
      + u_out |O| + Tk 2^-25 max|V|                        the bf16 (hi + lo) output, fp16 subnormal P (spacing 2^-24, l >= 1)."""
    B, T, d = q.shape
    Tk = k.shape[1]
    n_tiles = (Tk + 63) // 64
    u_p = P_ROUND[precision] if impl == 'tcgen05' else 0.0
    u = u_p + (n_tiles + 2) * 2.0 ** -22 + (Tk + 64) * 2 * U24
    e = _logit_err(q, k, H, precision)
    va = _heads(operand16(v, precision), H).abs()
    A = w @ va
    tol = u * A + (w * e) @ va + (w * e).sum(-1, keepdim=True) * A
    tol = tol.permute(0, 2, 1, 3).reshape(B, T, d)
    u_out = 2.0 ** -16 if out_lo else 2.0 ** -8 + 2 * U24
    return tol, u_out, Tk * 2.0 ** -25 * float(va.max())


def _check_out(got, ref, tol, u_out, floor, what):
    got = got.detach().cpu().double()
    assert torch.isfinite(got).all(), f'{what}: unwritten or non-finite output'
    bound = tol + u_out * ref.abs() + floor
    err = (got - ref).abs()
    worst = float((err / bound).max())
    assert worst <= 1.0, f'{what}: error {worst:.3g} x its bound (max abs err {float(err.max()):.3g})'


def _check_weights(wts, wref, e, causal, lens, what):
    """Reference-exact fp32 weights (logits + mask * -1e9, softmax): |dw_k| <= w_k (e_k + sum_j w_j e_j + Tk 2^-23 + 2^-21)
    (fp32 logits, expf, the fp32 sum and the division) + 2^-126 (expf underflow); masked keys exactly 0."""
    got = wts.detach().cpu().double()
    Tk = got.shape[-1]
    assert torch.isfinite(got).all(), f'{what}: unwritten weights'
    bound = wref * (e + (wref * e).sum(-1, keepdim=True) + Tk * 2 * U24 + 2.0 ** -21) + 2.0 ** -126
    assert bool(((got - wref).abs() <= bound).all()), f'{what}: weights off by {float(((got - wref).abs() / bound).max()):.3g} x bound'
    T = got.shape[-2]
    key = torch.arange(Tk)
    masked = key[None, None, :] >= torch.as_tensor(lens)[:, None, None]                 # (B?, 1, Tk)
    if causal:
        masked = masked | (key[None, :] > torch.arange(T)[:, None])[None]
    masked = masked[:, None].expand(got.shape) if got.dim() == 4 else masked.expand(got.shape)
    assert bool((got[masked] == 0).all()), f'{what}: masked keys with non-zero weight'


def _edge_lens(T, B, shift):
    edges = [1, 63, 64, 65, 127, 128, 129, T]
    return [min(edges[(i + shift) % len(edges)], T) for i in range(B)]


# every supported (head size, precision) pairing of the tensor-core kernel: dh 192 and 256 run in single-pass precisions
INSTANTIATIONS = [(64, 'bf16x3'), (64, 'bf16'), (64, 'fp16'), (128, 'bf16x3'), (128, 'bf16'), (128, 'fp16'),
                  (192, 'bf16'), (192, 'fp16'), (256, 'bf16'), (256, 'fp16')]
SELF_T = [1, 63, 64, 65, 127, 128, 129, 257]
CAUSAL_T = [64, 65, 128, 129, 192, 257]
CROSS = [(1, 1), (130, 63), (1, 64), (130, 65), (1, 129), (130, 1), (130, 129), (1, 63), (130, 64), (1, 65)]
EXTRA_ROWS = 130   # rows past B*T in the output buffers: a 128-row query tile that overruns T must not reach them


def _run_case(dh, precision, impl, T, Tk, lens, *, causal=False, cross=False, full_queries=True, rows='mix', seed=0,
              weights=None, ld_qk=None, ld_kv=None, cols=None, ld_out=None, out_lo=True):
    H = max(1, 256 // dh)
    B, d = len(lens), H * dh
    q, k, v = _peaked(B, T, Tk, H, dh, lens, _rows(B, T, rows), seed, causal=causal)
    kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    lo_cols = ld_out or d
    hi_buf = _poison16((B * T + EXTRA_ROWS, lo_cols))
    lo_buf = _poison16((B * T + EXTRA_ROWS, lo_cols)) if out_lo else None
    out, wts = run_mha_general(q.to(DEV), k.to(DEV), v.to(DEV), kv_len, H, precision=precision, impl=impl, causal=causal,
                               cross=cross, full_queries=full_queries, weights_all=weights == 'all',
                               weights_b=weights if isinstance(weights, int) else None, ld_qk=ld_qk, ld_kv=ld_kv, cols=cols,
                               out=(hi_buf, lo_buf))
    what = f'dh={dh} {precision} {impl} T={T} Tk={Tk} lens={lens} causal={causal} cross={cross}'
    ref, w = ref_mha_general(q, k, v, kv_len, H, precision, causal=causal, full_queries=full_queries)
    tol, u_out, floor = _out_tol(q, k, v, w, H, precision, impl, out_lo=out_lo)
    _check_out(out, ref, tol, u_out, floor, what)
    # ownership: columns [0, d) of the B*T rows are written; other columns and the rows past B*T keep their poison
    for buf in (hi_buf, lo_buf):
        if buf is None:
            continue
        bits = buf.view(torch.int16).cpu()
        assert bool((bits[:B * T, d:] == -1).all()), f'{what}: wrote columns outside [0, H*dh)'
        assert bool((bits[B * T:] == -1).all()), f'{what}: wrote rows past B*T'
        if not full_queries:
            rows_bits = bits[:B * T, :d].reshape(B, T, d)
            for b, n in enumerate(lens):
                assert bool((rows_bits[b, n:] == 0).all()), f'{what}: padded query rows of batch row {b} are not +0'
    if weights is not None:
        e = _logit_err(q, k, H, precision)
        if weights == 'all':
            _check_weights(wts, w, e, causal, lens, what)
        else:
            _check_weights(wts[None], w[weights:weights + 1], e[weights:weights + 1], causal, lens[weights:weights + 1], what)


@pytest.mark.parametrize('impl', ['tcgen05', 'simt'])
@pytest.mark.parametrize('dh,precision', INSTANTIATIONS)
def test_mha_self_attention_tile_edges_padded_rows_zero(dh, precision, impl):
    """Self-attention at every query-tile edge T, ragged kv_len on the key-tile edges (eight rows, a short row next to a
    full one), full_queries = 0: valid rows against float64, padded rows exactly +0 in both planes."""
    for i, T in enumerate(SELF_T):
        _run_case(dh, precision, impl, T, T, _edge_lens(T, 8, i), full_queries=False, seed=i)


@pytest.mark.parametrize('impl', ['tcgen05', 'simt'])
@pytest.mark.parametrize('dh,precision', INSTANTIATIONS)
def test_mha_causal_tile_edges(dh, precision, impl):
    """Look-ahead mask at the edges where the key-tile clamp of a query tile changes; full_queries alternates."""
    for i, T in enumerate(CAUSAL_T):
        _run_case(dh, precision, impl, T, T, _edge_lens(T, 4, 2 * i), causal=True, full_queries=bool(i % 2), seed=10 + i,
                  weights='all' if i % 3 == 0 else None)


@pytest.mark.parametrize('dh,precision', INSTANTIATIONS)
def test_mha_cross_attention_tile_edges(dh, precision):
    """Cross-attention with Tk on the key-tile edges, one and 130 queries, with the weights of every batch row."""
    for i, (T, Tk) in enumerate(CROSS):
        _run_case(dh, precision, 'tcgen05', T, Tk, _edge_lens(Tk, 4, i), cross=True, seed=20 + i, weights='all')
    _run_case(dh, precision, 'simt', 130, 65, _edge_lens(65, 4, 1), cross=True, seed=30, weights=1)


@pytest.mark.parametrize('causal', [False, True])
@pytest.mark.parametrize('rows', ['a', 'b', 'c', 'd', 'e', 'f'])
@pytest.mark.parametrize('dh,precision', [(64, 'bf16x3'), (128, 'fp16'), (256, 'bf16')])
def test_mha_peaked_logits(dh, precision, rows, causal):
    """One logit schedule for every row (e: a and c alternate) over five key tiles, with the weights of one batch row."""
    T = 257
    lens = [257, 200, 129, 65]
    _run_case(dh, precision, 'tcgen05', T, T, lens, causal=causal, full_queries=not causal, rows=rows, seed=40, weights=1)
    if rows in 'ae':
        _run_case(dh, precision, 'simt', T, T, lens, causal=causal, full_queries=False, rows=rows, seed=41)


@pytest.mark.parametrize('impl', ['tcgen05', 'simt'])
@pytest.mark.parametrize('dh,precision', [(64, 'bf16x3'), (128, 'bf16'), (192, 'fp16'), (256, 'bf16')])
def test_mha_layouts(dh, precision, impl):
    """The layouts the model passes: ld_qk wider than 3d (pad columns NaN), V before K and Q not at column 0, ld_out wider
    than H*dh (columns outside [0, H*dh) untouched), no lo output plane, cross-attention with ld_kv > 2d."""
    d = (max(1, 256 // dh)) * dh
    T, lens = 129, [129, 64, 1, 128]
    _run_case(dh, precision, impl, T, T, lens, full_queries=False, ld_qk=3 * d + 64, cols=(d + 32, 2 * d + 48, 8),
              ld_out=d + 48, seed=50)
    if precision != 'bf16x3':
        _run_case(dh, precision, impl, T, T, lens, causal=True, ld_qk=3 * d + 16, cols=(16, 2 * d + 16, d + 16),
                  out_lo=False, seed=51)
    _run_case(dh, precision, impl, 130, 65, [65, 64, 1, 63], cross=True, ld_qk=d + 32, ld_kv=2 * d + 40,
              cols=(16, d + 32, 0), ld_out=d + 16, seed=52, weights='all')


# ----------------------------------------------------------------------------------------------------------------------
# training: ttsb_attn_probs_fwd and ttsb_attn_ds_bwd
# ----------------------------------------------------------------------------------------------------------------------
def _round_up(x, m):
    return (x + m - 1) // m * m


def _train_qkv(B, T, H, dh, lens, rows, seed, ld, cols):
    """bf16 (B,T,ld) activation tensor with peaked Q, K and random V at the column offsets cols = (q, k, v); NaN elsewhere."""
    q, k, v = _peaked(B, T, T, H, dh, lens, rows, seed)
    d = H * dh
    buf = torch.full((B, T, ld), float('nan'))
    for x, c0 in zip((q, k, v), cols):
        buf[..., c0:c0 + d] = x
    return buf.bfloat16()


def _prob_tol(w, e, T):
    """|P - w| <= w (2^-8 + e_k + sum_j w_j e_j + (T + 4) 2^-22) + 2^-126: the bf16 rounding of P, the logit errors through
    the exponential and the normalisation, ex2.approx, the fp32 row sum and 1/l; ex2.approx.ftz flushes below 2^-126."""
    return w * (2.0 ** -8 + e + (w * e).sum(-1, keepdim=True) + (T + 4) * 2.0 ** -22) + 2.0 ** -126


PROB_CASES = [  # (dh, T, lens, ld_p beyond round_up(T, 8), schedule)
    (64, 1, [1, 1, 1, 1], 0, 'mix'), (64, 63, [63, 1, 62, 32], 64, 'd'), (128, 64, [64, 1, 63, 64], 0, 'c'),
    (128, 65, [65, 64, 1, 65], 72, 'd'), (192, 128, [128, 64, 65, 127], 0, 'mix'), (192, 129, [129, 128, 64, 1], 64, 'c'),
    (64, 129, [129, 128, 65, 64], 128, 'b'), (128, 128, [128, 127, 1, 64], 64, 'd'), (192, 65, [65, 63, 64, 2], 0, 'd'),
]


@pytest.mark.parametrize('dh,T,lens,extra,rows', PROB_CASES)
def test_attn_probs_and_ds_edges(dh, T, lens, extra, rows):
    """P_pre (rate 0, P_drop == P_pre: one output) against the float64 softmax at the tile edges, with the row maximum in
    the last live tile (d) and row ranges beyond 126 in log2 (c), Q and K at non-zero columns of a wider buffer, ld_p the
    smallest legal one or >= T + 64 (tiles past the last live one written as zeros); then dS = scale P (dO V^T - D) on the
    same edges against float64."""
    lib = _lib()
    H = 1 if dh == 192 else 2
    B, d = len(lens), H * dh
    ld, cols = 3 * d + 64, (d + 40, 8, 2 * d + 56)
    rr = _rows(B, T, rows)
    x = _train_qkv(B, T, H, dh, lens, rr, 60 + dh + T, ld, cols)
    ldp = _round_up(T, 8) + extra
    Z = B * H
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    scale = 1.0 / math.sqrt(dh)
    P = torch.full((Z * T + 64, ldp), float('nan'), dtype=torch.bfloat16, device=DEV)   # 64 guard rows past the output
    assert lib.attn_probs_supported(dh, ldp)
    lib.attn_probs_fwd(x.to(DEV), ld, cols[0], cols[1], B, H, T, dh, lens_d, scale, 0.0, 5, 3, P, P, ldp)
    torch.cuda.synchronize()
    Pc = P.float().cpu()
    assert bool(torch.isnan(Pc[Z * T:]).all()), 'wrote past the (B*H, T, ld_p) output'
    p = Pc[:Z * T].double().reshape(Z, T, ldp)
    assert torch.isfinite(p).all()
    xd = x.double()
    q, k = (xd[..., c:c + d].reshape(B, T, H, dh).permute(0, 2, 1, 3) for c in cols[:2])
    logits = (q @ k.transpose(-1, -2)) * scale
    kmask = torch.arange(T)[None, :] >= torch.tensor(lens)[:, None]                          # (B, T) dead keys
    qlive = (torch.arange(T)[None, :] < torch.tensor(lens)[:, None])                        # (B, T) live query rows
    w = torch.softmax(logits.masked_fill(kmask[:, None, None, :], float('-inf')), -1) * qlive[:, None, :, None]
    E = q.abs() @ k.abs().transpose(-1, -2) * scale
    e = 2 * U24 * (dh + (T + 63) // 64 + 1) * E                                              # see _logit_err (bf16 operands)
    w, e = w.reshape(Z, T, T), e.reshape(Z, T, T)
    live = p[:, :, :T]
    assert bool((p[:, :, T:] == 0).all()), 'columns >= T not zero'
    dead = (kmask[:, None, :] | ~qlive[:, :, None]).repeat_interleave(H, 0)                  # (Z, T, T)
    assert bool((live[dead] == 0).all()), 'masked keys or padded rows not zero'
    tol = _prob_tol(w, e, T)
    assert bool(((live - w).abs() <= tol).all()), f'P off by {float(((live - w).abs() / tol).max()):.3g} x bound'
    rows_live = qlive.repeat_interleave(H, 0)
    rs = live.sum(-1)[rows_live]
    assert bool(((rs - 1).abs() <= tol.sum(-1)[rows_live]).all()), 'row sums off 1 beyond the bf16 rounding bound'

    # ---- dS at the same edges: dO random, V at a non-zero column of the wide buffer, D random
    g = torch.Generator().manual_seed(70 + T)
    dO = torch.full((B, T, d + 16), float('nan'))
    dO[..., 16:] = torch.randn(B, T, d, generator=g)
    dO = dO.bfloat16()
    D = torch.randn(Z * T, generator=g) * 0.1
    dS = torch.full((Z * T + 64, ldp), float('nan'), dtype=torch.bfloat16, device=DEV)
    lib.attn_ds_bwd(dO.to(DEV), d + 16, 16, x.to(DEV), ld, cols[2], B, H, T, dh, lens_d, P, D.to(DEV), scale, 0.0, 5, 3, dS, ldp)
    torch.cuda.synchronize()
    s = dS.float().cpu()
    assert bool(torch.isnan(s[Z * T:]).all()), 'dS written past the output'
    s = s[:Z * T].double().reshape(Z, T, ldp)
    assert torch.isfinite(s).all()
    assert bool((s[:, :, T:] == 0).all()) and bool((s[:, :, :T][dead] == 0).all()), 'dS not zero on masked keys / rows / columns'
    do = dO.double()[..., 16:].reshape(B, T, H, dh).permute(0, 2, 1, 3).reshape(Z, T, dh)
    vv = xd[..., cols[2]:cols[2] + d].reshape(B, T, H, dh).permute(0, 2, 1, 3).reshape(Z, T, dh)
    dP = do @ vv.transpose(-1, -2)
    Dz = D.double().reshape(Z, T, 1)
    Pp = p[:, :, :T]
    ref = scale * Pp * (dP - Dz) * ~dead
    # fp32 dP over dh products (dh 2^-23 sum |dO||V|), the products and the fma (2^-22 of each term), bf16 output (2^-8)
    a = scale * Pp * (dh * 2 * U24 * (do.abs() @ vv.abs().transpose(-1, -2)) + 2.0 ** -21 * (dP.abs() + Dz.abs()))
    bound = a + 2.0 ** -8 * (ref.abs() + a) + 2.0 ** -126
    err = (s[:, :, :T] - ref).abs()
    assert bool((err <= bound).all()), f'dS off by {float((err / bound).max()):.3g} x bound'


# ----------------------------------------------------------------------------------------------------------------------
# ttsb_decode_attn across key splits
# ----------------------------------------------------------------------------------------------------------------------
def _decode_split(B, H, Tk):
    """decode.cu decode_split: keys per CTA and CTAs per (b, h) on this device."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    want = min(max((2 * sms + B * H - 1) // (B * H), 1), 32)
    c = (Tk + want - 1) // want
    c = 64 if c < 64 else (c + 31) // 32 * 32
    if c * 32 < Tk:
        c = (Tk + 31) // 32
    return c, (Tk + c - 1) // c


def _decode_call(lib, q, kv, Tk, H, dh, pos, prec, *, kv_len=None, new=None, probs=None):
    B, d = pos.shape[0], H * dh
    out_hi, out_lo = _poison16((B, d)), _poison16((B, d))
    ws = torch.zeros((lib.decode_attn_workspace_bytes(B, H, dh),), dtype=torch.uint8, device=DEV)
    a = lib.DecodeAttnArgs()
    a.B, a.H, a.dh = B, H, dh
    a.q, a.ld_q, a.q_col0 = q.data_ptr(), q.shape[-1], 0
    a.kv, a.ld_kv, a.Tk, a.k_col0, a.v_col0 = kv.data_ptr(), kv.shape[-1], Tk, 0, d
    if new is not None:
        a.new_kv, a.ld_new, a.new_k_col0, a.new_v_col0 = new.data_ptr(), new.shape[-1], d, 2 * d
    else:
        a.kv_len = kv_len.data_ptr()
    a.pos = pos.data_ptr()
    a.out_hi, a.out_lo, a.ld_out = out_hi.data_ptr(), out_lo.data_ptr(), d
    a.probs, a.probs_T = probs.data_ptr(), probs.shape[2]
    a.precision = prec
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    lib.decode_attn(a)
    torch.cuda.synchronize()
    assert int(ws[:B * H * 4].view(torch.int32).count_nonzero()) == 0
    return out_hi.float() + out_lo.float()


def _decode_check(out, probs, pos, q, k, v, lens, H, prec, what):
    """float64 on the 16-bit operands: out within _out_tol (no P rounding, fp32 everywhere; the combine adds one expf and
    one product per split, inside the per-tile terms), the probability row within the weights bound and exactly 0 past
    the row's length; every other probability row keeps its sentinel."""
    B, Tk, d = k.shape
    q3 = q[:, None, :]
    kvl = torch.tensor(lens, dtype=torch.int32)
    ref, w = ref_mha_general(q3, k, v, kvl, H, prec)
    tol, u_out, floor = _out_tol(q3, k, v, w, H, prec, 'simt')
    _check_out(out[:, None].cpu(), ref, tol, u_out, floor, what)
    e = _logit_err(q3, k, H, prec)
    pr = probs.cpu().double()
    row = pr[torch.arange(B), :, pos.long().cpu()]                                 # (B, H, Tk)
    _check_weights(row[:, :, None], w, e, False, lens, what)
    others = pr.clone()
    others[torch.arange(B), :, pos.long().cpu()] = -1.0
    assert bool((others == -1.0).all()), f'{what}: wrote another probability row'


def _decode_inputs(Tk, H, dh, lens, logits, dt, seed):
    """q (B, d), k / v (B, Tk, d) fp32 whose scaled logits of batch row b are logits[b] (float64 (Tk,); keys past lens[b]
    at MASKED_LOGIT) up to 0.01-noise, on every head."""
    g = torch.Generator().manual_seed(seed)
    B, d = len(lens), H * dh
    q = torch.zeros(B, H, dh)
    q[..., 0] = 1.0
    q[..., 1:] = 0.01 * torch.randn(B, H, dh - 1, generator=g)
    k = 0.05 * torch.randn(B, Tk, H, dh, generator=g)
    for b in range(B):
        L = logits[b].clone()
        L[lens[b]:] = MASKED_LOGIT
        k[b, :, :, 0] = (L * math.sqrt(dh)).float().to(dt).float()[:, None]
    v = torch.randn(B, Tk, H, dh, generator=g)
    return q.reshape(B, d), k.reshape(B, Tk, d), v.reshape(B, Tk, d)


@pytest.mark.parametrize('dh,prec', [(64, 'fp16'), (128, 'bf16'), (256, 'fp16')])
def test_decode_attn_split_combine(dh, prec):
    """Cross mode over a key range split across CTAs: the argmax key in the last and in the first split, and splits whose
    maxima lie 150 apart (expf(m_i - mx) underflows to 0 in the combine).  Self mode with pos at chunk - 1, chunk and
    chunk + 1, where the number of live splits changes, the maximum on the new key or on key 0."""
    lib = _lib()
    pc = lib.PREC_FP16 if prec == 'fp16' else lib.PREC_BF16
    dt = torch.float16 if prec == 'fp16' else torch.bfloat16
    H, Tk = 2, 1000
    B = 4
    chunk, n_split = _decode_split(B, H, Tk)
    assert n_split > 2, 'the key range must be split across several CTAs'
    g = torch.Generator().manual_seed(dh)
    key = torch.arange(Tk)
    L = [-2.0 * torch.rand(Tk, generator=g, dtype=torch.float64) for _ in range(B)]
    L[0][Tk - 1] = 15.0                                  # argmax in the last split
    L[1][0] = 15.0                                       # argmax in the first split
    L[2] -= 150.0 * (key // chunk)                       # split maxima 150 apart: all but the first underflow in the combine
    L[3][chunk], L[3][chunk - 1] = 9.0, 8.5              # the two largest keys on both sides of a split boundary
    lens = [Tk, 777, 900, 2 * chunk - 1]
    q, k, v = _decode_inputs(Tk, H, dh, lens, L, dt, seed=dh)
    qd, kvd = q.to(dt).to(DEV), torch.cat([k, v], -1).to(dt).to(DEV)
    pos = torch.tensor([0, 3, 1, 4], dtype=torch.int32, device=DEV)
    probs = torch.full((B, H, 5, Tk), -1.0, device=DEV)
    out = _decode_call(lib, qd, kvd, Tk, H, dh, pos, pc, kv_len=torch.tensor(lens, dtype=torch.int32, device=DEV), probs=probs)
    _decode_check(out, probs, pos, q, k, v, lens, H, prec, f'cross dh={dh} {prec} chunk={chunk}')

    # self mode: the cache holds rows 0..pos-1, the new row (key pos) comes from the QKV buffer and is copied into the cache
    Tmax = Tk
    chunk, n_split = _decode_split(3, H, Tmax)
    assert n_split > 2
    P = [chunk - 1, chunk, chunk + 1]
    L = [-2.0 * torch.rand(Tmax, generator=g, dtype=torch.float64) for _ in range(3)]
    L[0][P[0]] = 12.0                                    # maximum on the new key
    L[1][0] = 12.0                                       # maximum on key 0, the new key opens the second split
    L[2][P[2]], L[2][0] = 14.0, 13.0                     # both
    q, k, v = _decode_inputs(Tmax, H, dh, [p + 1 for p in P], L, dt, seed=dh + 1)
    d = H * dh
    cache = torch.cat([k, v], -1).to(dt)
    new = torch.full((3, 3 * d), float('nan'), dtype=dt)
    new[:, :d] = q.to(dt)
    new[:, d:] = cache[torch.arange(3), torch.tensor(P)]
    cache_d = cache.clone()
    cache_d[torch.arange(3), torch.tensor(P)] = -cache_d[torch.arange(3), torch.tensor(P)]   # overwritten by the new row
    cache_d = cache_d.to(DEV)
    pos = torch.tensor(P, dtype=torch.int32, device=DEV)
    probs = torch.full((3, H, Tmax, Tmax), -1.0, device=DEV)
    new_d = new.to(DEV)
    out = _decode_call(lib, new_d, cache_d, Tmax, H, dh, pos, pc, new=new_d, probs=probs)
    assert torch.equal(cache_d.cpu(), cache), 'the new key / value rows did not land in the cache bit for bit'
    _decode_check(out, probs, pos, q, k, v, [p + 1 for p in P], H, prec, f'self dh={dh} {prec} chunk={chunk}')
