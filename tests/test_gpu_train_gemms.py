"""The batched GEMM, weight-gradient GEMM and softmax kernels of the training step (csrc/bgemm_tc.cu, csrc/train_ops.cu)
against float64, element by element.

Contract under test.  ttsb_bgemm computes out_z[m][n] = alpha * sum_{k < K} A_z[m][k] * B_z[n][k] for every (b, h) from
two bf16 tensors addressed through (dims, strides, per-head offsets, majorness); ttsb_wgrad adds sum_{b,t} X[b][t +
shift][c] * G[b][t][n] onto dW; ttsb_softmax_fwd / _bwd are the masked row softmax with attention dropout and its
gradient, and the `sm_*` epilogue of ttsb_bgemm is that gradient fused into the dP product.  Kernels are called through
lib.py and TrainEngine._bgemm / _wgrad with the argument tuples of model/training.py and model/aligner_training.py.  The
batched reference (gpu_util.ref_bgemm) evaluates the argument description literally, by indexing the host copy of the
buffers, so it does not share training.py's idea of which product a call is (tests/test_host_logic.py checks it against
einsum).

Poison.  Blocks of a q | k | v buffer that a product does not use hold gpu_util.WIDE_SOURCE_FILL and head h's data is
scaled by 2^h, so a read across a block or head boundary is far off.  What the kernels never read holds NaN: the columns
[Tk, ld) of P / dS as a GEMM operand, the columns past Cin / N of the weight gradient's X / G (all outside the tensor
maps, which fill with zeros), the columns [Tk, ld) of the softmax kernels' S / dP / P_pre inputs, columns past
round_up(C, 8) of a column sum.  Masked keys of S and dP hold large finite values.  The fused epilogue reads P_pre in
whole 16-column chunks, so there the padding is what ttsb_softmax_fwd wrote.  Outputs start as NaN (weight gradients and
column sums, which accumulate, as random values inside guard rows): every element the contract writes must be finite,
columns [N, out_cols), rows at or past row_len, masked keys and dead rows exact zeros, everything else untouched.

Error model.  bf16 operands are exact in float64 and their products exact in fp32, so a GEMM element differs from the
reference by the fp32 accumulation (order, and the tensor core's alignment of addends) -- bounded by a small multiple of
K * 2^-24 * sum_k |a_k b_k| -- plus, for a bf16 output, one rounding of at most 2^-8 |value| (bf16 keeps 8 significant
bits).  Every element is gated on (|err| - 2^-8 |ref| if bf16) / sum_k |a_k b_k|, never on a tensor norm.  A missing,
doubled or foreign term changes an element by about sum|terms| / K >= 1e-3 of the denominator at the K used here (K <=
1100), more than a thousand times the gates; an error confined to one element fails as surely as one that is everywhere.
The softmax adds __expf (ex2.approx after an fp32 multiply by log2 e: relative error about 2^-22 + |x| 2^-23, |x| <= 20
here) and fp32 row sums; its bf16 probabilities hide what is inside their own rounding.  Weight-gradient and column sums
are fp32 atomics in a run-dependent order: their gates are bounds and each call runs once.
"""
import math

import numpy as np
import pytest
import torch

from gpu_util import DEV, WIDE_SOURCE_FILL, _poison16, bgemm_out_index, dropout_keep, dropout_scale, ref_bgemm
from transformertts_b200 import lib
from transformertts_b200.model.models import _round_up
from transformertts_b200.model.training import TrainEngine

pytestmark = pytest.mark.gpu

SALT = 0xC2B2AE35   # high bit set: the XOR of the whole word into the seed is covered
SEED = 0x2545F491
BF16_U = 2.0 ** -8  # largest relative error of one rounding to bf16

# Measured on an H100 80GB HBM3 (SXM, 700 W power limit): in brackets the largest error of any case under each gate.  Where
# that is 0 every error was inside the bf16 rounding allowance and the gate is the bound of the error model.
GATE_ACC = 4e-7          # ttsb_bgemm element, (|err| - bf16 rounding) / sum |terms| (fp32 out 1.7e-7, bf16 out 4.6e-8)
GATE_EPILOGUE = 3e-8     # fused softmax backward, (|err| - bf16 rounding) / (scale P (ks sum |terms| + |D|)) (1.4e-8)
GATE_WGRAD = 3e-7        # ttsb_wgrad element, |err| / (|dw before| + sum |terms|); atomics, a bound (1.2e-7)
GATE_SOFTMAX = 4e-6      # P_pre / kept P_drop, (|err| - bf16 rounding) / ref; the __expf bound (0)
GATE_ROWSUM = 6e-3       # |sum_k P_pre - 1| of the bf16 probabilities of a live row (3.0e-3)
GATE_SOFTMAX_BWD = 2e-8  # dS, (|err| - bf16 rounding) / (scale P (|g| + sum |P g|)) (1.0e-8)
GATE_SUM = 2e-7          # rowdot_heads, colsum_bf16(_x3): |err| / sum |terms|; the column sums are atomics, a bound (5.9e-8)


@pytest.fixture(scope='module', autouse=True)
def dropout_salt():
    lib.load()
    lib.set_dropout_salt(torch.tensor([np.uint32(SALT).view(np.int32)], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    yield SALT
    lib.set_dropout_salt(torch.zeros(1, dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()


@pytest.fixture(scope='module')
def eng():
    e = TrainEngine.__new__(TrainEngine)
    e.dev = torch.device(DEV)
    return e


def _report(case, what, err, gate):
    print(f'[train-gemms] {case}: {what} err {err:.2e} (gate {gate:.1e})')
    assert err < gate, f'{case}: {what} error {err:.3e} >= gate {gate:.1e}'


def _elem_err(case, got, ref, denom, bf16):
    """max over elements of (|got - ref| - one bf16 rounding of ref) / denom; where denom == 0 got must equal ref."""
    assert np.isfinite(got).all(), f'{case}: non-finite values where the contract writes'
    assert np.isfinite(ref).all() and np.isfinite(denom).all(), f'{case}: the reference read a NaN (a region marked as never read is read)'
    err = np.abs(got - ref)
    if bf16:
        err = np.maximum(err - BF16_U * np.abs(ref), 0.0)
    empty = denom == 0
    assert np.array_equal(got[empty], ref[empty]), f'{case}: elements without any term differ from the reference'
    return float((err[~empty] / denom[~empty]).max()) if (~empty).any() else 0.0


def _host(t):
    return t.detach().double().cpu().numpy()


def _lens(Tk, extra=()):
    return torch.tensor([Tk, Tk // 2, 1, 0, Tk + 5, -3, *extra], dtype=torch.int32)


def _key_mask(lens, H, T, Tk, width, flags):
    """bool (B*H, T, width): key k of query row t of problem z takes part (ttsb_softmax_fwd's rules)."""
    ln = lens.long().clamp(0, Tk).repeat_interleave(H)[:, None].expand(-1, T)     # (Z, T)
    t = torch.arange(T)[None, :]
    live = (ln > 0) if flags & 2 else (t < ln)
    if flags & 1:
        ln = torch.minimum(ln, t + 1)
    return ((torch.arange(width)[None, None, :] < ln[..., None]) & live[..., None]).numpy()


def _keep(Z, T, ld, width, p, site):
    """bool (Z, T, width) keep decisions of a (Z, T, ld) tensor drawn at (z*T + t)*ld + k (all kept at p = 0)."""
    if p == 0:
        return np.ones((Z, T, width), dtype=bool)
    idx = (np.arange(Z * T, dtype=np.uint64)[:, None] * np.uint64(ld) + np.arange(width, dtype=np.uint64)[None, :])
    return dropout_keep(SEED, site, idx, p, SALT).reshape(Z, T, width)


# ----------------------------------------------------------------------------------------------------------
# ttsb_bgemm: the six attention products
# ----------------------------------------------------------------------------------------------------------
def _heads_scaled(g, B, T, H, dh):
    """bf16 (B, T, H*dh) with head h scaled by 2^h (exact): the next head's columns are not this head's size."""
    x = torch.randn(B, T, H, dh, generator=g) * (2.0 ** torch.arange(H, dtype=torch.float32))[:, None]
    return x.reshape(B, T, H * dh).bfloat16()


def _probs_like(g, Z, T, Tk, ldp):
    """bf16 (Z, T, ldp) operand standing for P / dS: random in [:Tk], NaN in the padding columns (outside the tensor map)."""
    x = _poison16((Z, T, ldp))
    x[..., :Tk] = torch.randn(Z, T, Tk, generator=g).bfloat16().to(DEV)
    return x


class _Attn:
    """The buffers of one attention call as _attn_fwd / _attn_bwd see them, and the argument tuple of each product."""

    def __init__(self, g, B, H, dh, T, Tk, cross, use):
        """use: which of 'q', 'k', 'v' hold data; the other blocks hold WIDE_SOURCE_FILL."""
        d = H * dh
        self.B, self.H, self.dh, self.T, self.Tk, self.d, self.Z, self.ldp = B, H, dh, T, Tk, d, B * H, _round_up(Tk, 16)
        blk = lambda rows, name: _heads_scaled(g, B, rows, H, dh) if name in use else torch.full((B, rows, d), WIDE_SOURCE_FILL).bfloat16()
        if cross:
            self.qb = blk(T, 'q').contiguous().to(DEV)
            self.kb = torch.cat([blk(Tk, 'k'), blk(Tk, 'v')], -1).contiguous().to(DEV)
            self.q_ld, self.q_col, self.k_ld, self.k_col, self.v_col = d, 0, 2 * d, 0, d
        else:
            assert T == Tk
            self.qb = self.kb = torch.cat([blk(T, 'q'), blk(T, 'k'), blk(T, 'v')], -1).contiguous().to(DEV)
            self.q_ld, self.q_col, self.k_ld, self.k_col, self.v_col = 3 * d, 0, 3 * d, d, 2 * d
        self.dout = _heads_scaled(g, B, T, H, dh).to(DEV)
        self.P = _probs_like(g, self.Z, T, Tk, self.ldp)

    def args(self, kind):
        B, H, dh, T, Tk, d, Z, ldp = self.B, self.H, self.dh, self.T, self.Tk, self.d, self.Z, self.ldp
        q = (self.qb, (d, T, B), (self.q_ld, self.q_ld * T))
        kv = (self.kb, (d, Tk, B), (self.k_ld, self.k_ld * Tk))
        do = (self.dout, (d, T, B), (d, d * T))
        p = (self.P, (Tk, T, Z), (ldp, T * ldp))
        return {
            'S': (B, H, T, Tk, dh, *q, (dh, 0, 0, self.q_col), *kv, (dh, 0, 0, self.k_col)),
            'dP': (B, H, T, Tk, dh, *do, (dh, 0, 0, 0), *kv, (dh, 0, 0, self.v_col)),
            'O': (B, H, T, dh, Tk, *p, (0, 0, 1, 0), *kv, (dh, 0, 0, self.v_col, 1)),
            'dQ': (B, H, T, dh, Tk, *p, (0, 0, 1, 0), *kv, (dh, 0, 0, self.k_col, 1)),
            'dK': (B, H, Tk, dh, T, *p, (0, 0, 1, 0, 1), *q, (dh, 0, 0, self.q_col, 1)),
            'dV': (B, H, Tk, dh, T, *p, (0, 0, 1, 0, 1), *do, (dh, 0, 0, 0, 1)),
        }[kind]

    def out(self, kind):
        """(elements of the output buffer, layout keywords of _bgemm) as _attn_fwd / _attn_bwd place the product."""
        B, dh, T, Tk, d, Z, ldp = self.B, self.dh, self.T, self.Tk, self.d, self.Z, self.ldp
        if kind in ('S', 'dP'):
            return Z * T * ldp, dict(ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp)
        by_b = dict(out_h_col=dh, out_by_b=1, out_cols=dh)
        if kind == 'O':
            return B * T * d, dict(ld_out=d, out_batch_stride=T * d, **by_b)
        if kind == 'dQ':   # into the q block of the d(q|k|v) buffer (self) or the dq buffer (cross)
            return B * T * self.q_ld, dict(ld_out=self.q_ld, out_batch_stride=T * self.q_ld, out_ptr_off=self.q_col, **by_b)
        col = self.k_col if kind == 'dK' else self.v_col
        return B * Tk * self.k_ld, dict(ld_out=self.k_ld, out_batch_stride=Tk * self.k_ld, out_ptr_off=col, **by_b)


def _check_bgemm(eng, case, args, numel, layout, *, alpha=1.0, f32=False, bf16=False, row_len=None, col_len=None):
    """One ttsb_bgemm call into NaN buffers, every element of the buffers against the literal reference."""
    B, H, M, N, K = args[:5]
    ref, terms = ref_bgemm(*args)
    alpha32 = float(np.float32(alpha))
    out_f = torch.full((numel,), float('nan'), device=DEV) if f32 else None
    out_b = _poison16((numel,)) if bf16 else None
    eng._bgemm(*args, alpha=alpha, out_f32=out_f, out_bf16=out_b, row_len=None if row_len is None else row_len.to(DEV),
               col_len=None if col_len is None else col_len.to(DEV), **layout)
    torch.cuda.synchronize()
    cols = layout['out_cols']
    idx = bgemm_out_index(B, H, M, cols, layout['ld_out'], layout['out_batch_stride'], layout.get('out_h_col', 0),
                          layout.get('out_by_b', 0), layout.get('out_ptr_off', 0))
    own = np.zeros(numel, dtype=bool)
    own[idx.ravel()] = True
    assert int(own.sum()) == idx.size, f'{case}: the case maps two output elements to one address'
    b_of_z = np.arange(B * H) // H
    rl = np.full(B, M) if row_len is None else row_len.numpy()
    cl = np.full(B, N) if col_len is None else col_len.numpy()
    n = np.arange(cols)[None, None, :]
    live = (n < N) & (n < cl[b_of_z][:, None, None]) & (np.arange(M)[None, :, None] < rl[b_of_z][:, None, None])
    want, denom = np.zeros(idx.shape), np.zeros(idx.shape)
    want[..., :N], denom[..., :N] = alpha32 * ref, abs(alpha32) * terms
    want[~live], denom[~live] = 0.0, 0.0
    for name, buf in (('fp32', out_f), ('bf16', out_b)):
        if buf is None:
            continue
        flat = _host(buf)
        assert np.isnan(flat[~own]).all(), f'{case}: {name} output written outside the call\'s own rows and columns'
        _report(case, f'{name} out', _elem_err(f'{case} {name}', flat[idx], want, denom, name == 'bf16'), GATE_ACC)


# (H, dh, T, Tk, cross): M and N inside a 128-row / block_n tile (130, 333, 200, 97, 65, 300), several N tiles (333, 1100),
# direct stores (block_n 144, 48, 32, 16) next to staged ones (64, 128, 192, 256), one head of 256, T = Tk = 1.
ATTN_SHAPES = [(2, 64, 130, 130, False), (2, 128, 333, 333, False), (2, 192, 200, 200, False), (2, 128, 1, 1, False),
               (1, 256, 97, 40, True), (4, 64, 65, 20, True), (2, 64, 300, 1100, True)]
# which q | k | v blocks each product reads
USES = {'S': 'qk', 'dP': 'v', 'O': 'v', 'dQ': 'k', 'dK': 'q', 'dV': ''}


@pytest.mark.parametrize('H,dh,T,Tk,cross', ATTN_SHAPES)
def test_bgemm_attention_products(eng, H, dh, T, Tk, cross):
    """S and dP (fp32, as the softmax kernels take them, alpha = 1/sqrt(dh) on S; and bf16 with alpha = -0.5, the staged
    store path when round_up(Tk, 16) is a multiple of 64), O, dQ, dK, dV (bf16 into the head's columns of the (B, T, d) /
    d(q|k|v) / d(k|v) buffers).  B = 3 so that b and z differ."""
    B = 3
    for kind in ('S', 'dP', 'O', 'dQ', 'dK', 'dV'):
        g = torch.Generator().manual_seed(1000 + 7 * T + dh + len(kind))
        at = _Attn(g, B, H, dh, T, Tk, cross, USES[kind])
        numel, layout = at.out(kind)
        case = f'{kind} H={H} dh={dh} T={T} Tk={Tk} {"cross" if cross else "self"}'
        if kind in ('S', 'dP'):
            _check_bgemm(eng, case, at.args(kind), numel, layout, alpha=1.0 / math.sqrt(dh) if kind == 'S' else 1.0, f32=True)
            _check_bgemm(eng, case + ' alpha=-0.5', at.args(kind), numel, layout, alpha=-0.5, bf16=True)
        else:
            _check_bgemm(eng, case, at.args(kind), numel, layout, bf16=True)


@pytest.mark.parametrize('T', [128, 130])
def test_bgemm_row_and_column_lengths(eng, T):
    """row_len / col_len of T, T/2, 1, 0 per batch row on S: rows and columns at or past them are exact zeros, in fp32 and
    bf16 together (direct stores) and in bf16 alone (T = 128: staged stores)."""
    B, H, dh = 4, 2, 64
    g = torch.Generator().manual_seed(1100 + T)
    at = _Attn(g, B, H, dh, T, T, False, 'qk')
    numel, layout = at.out('S')
    lens = torch.tensor([T, T // 2, 1, 0], dtype=torch.int32)
    case = f'S H={H} dh={dh} T={T} row/col_len'
    _check_bgemm(eng, case, at.args('S'), numel, layout, alpha=0.125, f32=True, bf16=True, row_len=lens, col_len=lens.flip(0))
    _check_bgemm(eng, case + ' bf16 only', at.args('S'), numel, layout, alpha=0.125, bf16=True, row_len=lens, col_len=lens.flip(0))
    _check_bgemm(eng, case + ' rows only', at.args('S'), numel, layout, bf16=True, row_len=lens)


@pytest.mark.parametrize('dh', [32, 96])
def test_bgemm_refuses_heads_whose_k_block_reaches_the_next_head(eng, dh):
    """Two heads of 32 or 96 columns: the 64-wide k block of head 0 would take in head 1's columns.  Refused at the entry
    point, before any launch: the output is untouched."""
    B, H, T = 2, 2, 40
    g = torch.Generator().manual_seed(1200 + dh)
    at = _Attn(g, B, H, dh, T, T, False, 'qkv')
    for kind, operand in (('S', 'A'), ('dP', 'A')):
        numel, layout = at.out(kind)
        out = torch.full((numel,), float('nan'), device=DEV)
        with pytest.raises(lib.TtsbError, match=rf'ttsb_bgemm failed \(-1\): ttsb_bgemm: K = {dh} is not a multiple of 64.*operand {operand}'):
            eng._bgemm(*at.args(kind), out_f32=out, **layout)
        torch.cuda.synchronize()
        assert torch.isnan(out).all()
    # only B at fault: A's extent ends at K, B carries a per-head column offset
    a = at.args('S')
    one_head_a = (B, H, T, T, dh, at.qb, (dh, T, B), a[7], (0, 0, 0, 0), *a[9:])
    with pytest.raises(lib.TtsbError, match=r'\(-1\).*operand B'):
        eng._bgemm(*one_head_a, out_f32=torch.full((at.out('S')[0],), float('nan'), device=DEV), **at.out('S')[1])
    # the products that contract over keys or queries keep working at this head size for every Tk (K = 40 here)
    for kind in ('O', 'dQ', 'dK', 'dV'):
        g = torch.Generator().manual_seed(1210 + dh + len(kind))
        at = _Attn(g, B, H, dh, T, T, False, USES[kind])
        numel, layout = at.out(kind)
        _check_bgemm(eng, f'{kind} H={H} dh={dh} T={T}', at.args(kind), numel, layout, bf16=True)


def test_bgemm_single_head_of_32_is_computed(eng):
    """H = 1, dh = 32: the tensor ends where the head ends, the tail of the k block is the map's zero fill (the neighbouring
    blocks of the q | k | v buffer hold WIDE_SOURCE_FILL)."""
    B, H, dh, T = 3, 1, 32, 70
    for kind in ('S', 'dP'):
        g = torch.Generator().manual_seed(1300 + len(kind))
        at = _Attn(g, B, H, dh, T, T, False, USES[kind])
        numel, layout = at.out(kind)
        _check_bgemm(eng, f'{kind} H=1 dh=32 T={T}', at.args(kind), numel, layout, f32=True)


# ----------------------------------------------------------------------------------------------------------
# ttsb_bgemm with the fused softmax backward
# ----------------------------------------------------------------------------------------------------------
def _softmax_inputs(g, Z, T, Tk, ld, mask):
    """fp32 (Z, T, ld) scores: random at the keys that take part, 1e30 at masked keys and dead rows, NaN in [Tk, ld)."""
    S = torch.full((Z, T, ld), float('nan'))
    S[..., :Tk] = torch.where(torch.from_numpy(mask[..., :Tk]), 2.0 * torch.randn(Z, T, Tk, generator=g), torch.tensor(1e30))
    return S


# (T, Tk): block_n 128 (staged), 144 (direct), 256 x 2 tiles (staged, the second ends at out_cols = 304)
@pytest.mark.parametrize('T,Tk', [(130, 128), (70, 130), (200, 300)])
def test_bgemm_fused_softmax_backward(eng, T, Tk):
    """dS = scale * P_pre * (keep * dP / (1-p) - D) out of the dP product's epilogue, for every flag combination, without
    dropout, with the mask re-drawn from the hash and with the mask read back from P_drop.  P_pre / P_drop come from
    ttsb_softmax_fwd under the same flags and lengths; D is arbitrary."""
    B, H, dh = 6, 2, 64
    Z, ldp = B * H, _round_up(Tk, 16)
    scale = float(np.float32(1.0 / math.sqrt(dh)))
    lens = _lens(Tk)
    lens_d = lens.to(DEV)
    for flags in range(4):
        g = torch.Generator().manual_seed(2000 + T + flags)
        at = _Attn(g, B, H, dh, T, Tk, True, 'v')
        mask = _key_mask(lens, H, T, Tk, ldp, flags)
        S = _softmax_inputs(g, Z, T, Tk, ldp, mask).to(DEV)
        D = torch.randn(Z * T, generator=g)
        dP, terms = ref_bgemm(*at.args('dP'))
        numel, layout = at.out('dP')
        for p, site, saved in ((0.0, 0, False), (0.25, 3 + flags, False), (0.25, 3 + flags, True)):
            case = f'dS epilogue T={T} Tk={Tk} flags={flags} p={p} mask from {"P_drop" if saved else "hash"}'
            P_pre = _poison16((Z, T, ldp))
            P_drop = _poison16((Z, T, ldp)) if p > 0 else P_pre
            lib.softmax_fwd(S, B, H, T, Tk, ldp, lens_d, p, SEED, site, P_pre, P_drop, flags=flags)
            dS = _poison16((numel,))
            eng._bgemm(*at.args('dP'), out_bf16=dS, **layout,
                       softmax_bwd=(P_pre, D.to(DEV), scale, p, SEED, site, flags, lens_d, P_drop if saved else None))
            torch.cuda.synchronize()
            Pp = _host(P_pre)
            assert np.isfinite(Pp).all() and (Pp[~mask] == 0).all()
            keep = _keep(Z, T, ldp, Tk, p, site)
            if p > 0:   # what the epilogue reads back is what the hash says
                decides = mask[..., :Tk] & (Pp[..., :Tk] != 0)
                assert np.array_equal((_host(P_drop)[..., :Tk] != 0)[decides], keep[decides]), f'{case}: P_drop mask differs from the hash'
            ks = dropout_scale(p) if p > 0 else 1.0
            sp = scale * Pp[..., :Tk] * mask[..., :Tk]
            Dz = D.double().numpy().reshape(Z, T, 1)
            want, denom = np.zeros((Z, T, ldp)), np.zeros((Z, T, ldp))
            want[..., :Tk] = sp * (keep * dP * ks - Dz)
            denom[..., :Tk] = sp * (keep * terms * ks + np.abs(Dz))
            got = _host(dS).reshape(Z, T, ldp)
            _report(case, 'dS', _elem_err(case, got, want, denom, True), GATE_EPILOGUE)
            if p > 0:   # the mask bit for bit: an element sits at its kept or at its dropped value, wherever the two are apart
                dropped = sp * -Dz
                kept = sp * (dP * ks - Dz)
                decides = np.abs(kept - dropped) > 2.0 ** -4 * np.maximum(np.abs(kept), np.abs(dropped))
                decides &= (sp != 0)
                assert int(decides.sum()) > 0
                got_kept = np.abs(got[..., :Tk] - kept) < np.abs(got[..., :Tk] - dropped)
                bad = int((got_kept != keep)[decides].sum())
                assert bad == 0, f'{case}: dropout mask differs from the restated hash at {bad} elements'


def test_bgemm_fused_softmax_backward_above_1024_keys(eng):
    """More than 1024 keys: P_pre / P_drop come from the scalar softmax kernel.  The epilogue that reads the mask back from
    that P_drop and the one that re-draws it from the hash give the same dS, bit for bit."""
    B, H, dh, T, Tk, flags, p, site = 2, 2, 64, 40, 1100, 2, 0.25, 11
    Z, ldp = B * H, _round_up(Tk, 16)
    scale = float(np.float32(1.0 / math.sqrt(dh)))
    g = torch.Generator().manual_seed(2100)
    lens = torch.tensor([Tk, 1029], dtype=torch.int32)
    lens_d = lens.to(DEV)
    at = _Attn(g, B, H, dh, T, Tk, True, 'v')
    mask = _key_mask(lens, H, T, Tk, ldp, flags)
    S = _softmax_inputs(g, Z, T, Tk, ldp, mask).to(DEV)
    D = torch.randn(Z * T, generator=g).to(DEV)
    P_pre, P_drop = _poison16((Z, T, ldp)), _poison16((Z, T, ldp))
    lib.softmax_fwd(S, B, H, T, Tk, ldp, lens_d, p, SEED, site, P_pre, P_drop, flags=flags)
    numel, layout = at.out('dP')
    outs = []
    for saved in (P_drop, None):
        dS = _poison16((numel,))
        eng._bgemm(*at.args('dP'), out_bf16=dS, **layout, softmax_bwd=(P_pre, D, scale, p, SEED, site, flags, lens_d, saved))
        outs.append(dS)
    torch.cuda.synchronize()
    assert torch.isfinite(outs[0].float()).all()
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), 'dS differs between the saved and the re-drawn mask'
    keep = _keep(Z, T, ldp, Tk, p, site)
    decides = mask[..., :Tk] & (_host(P_pre)[..., :Tk] != 0)
    assert int(decides.sum()) > 100000
    assert np.array_equal((_host(P_drop)[..., :Tk] != 0)[decides], keep[decides]), 'P_drop mask of the scalar kernel differs from the hash'


# ----------------------------------------------------------------------------------------------------------
# ttsb_wgrad
# ----------------------------------------------------------------------------------------------------------
def _split_case_batch():
    """A batch size the split count of Cin = N = 1536 (72 base tiles) does not divide: the last split is short."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    splits = -(-2 * sms // 72)
    for B in range(splits + 1, 3 * splits + 2):
        per = -(-B // splits)
        if per > 1 and B % per != 0:
            return B
    return splits + 1


# name: (B, T, Cin, ldx, N, ldg, g column offset, [(source, shift)])
WGRAD_CASES = {
    'mel 80 of 128': (3, 97, 80, 128, 80, 128, 0, [(0, 0)]),
    'stop token N=3 at column 80': (3, 97, 80, 128, 3, 128, 80, [(0, 0)]),
    'conv 3 taps N=226': (2, 333, 256, 256, 226, 256, 0, [(0, -1), (0, 0), (0, 1)]),
    'four segments two sources': (2, 150, 72, 72, 40, 40, 0, [(0, -2), (1, -1), (1, 1), (0, 2)]),
    'concat two sources': (5, 65, 128, 128, 128, 128, 0, [(0, 0), (1, 0)]),
    'tiles Cin=200 N=300': (3, 130, 200, 200, 300, 304, 0, [(0, 0)]),
    'T=1 shifts past T': (1, 1, 64, 64, 64, 64, 0, [(0, -1), (0, 0), (0, 1)]),
    'T=63': (1, 63, 48, 48, 24, 24, 0, [(0, -1), (0, 0), (0, 1)]),
    'T=64': (1, 64, 48, 48, 24, 24, 0, [(0, -1), (0, 0), (0, 1)]),
    'T=65': (2, 65, 48, 48, 24, 24, 0, [(0, -65), (0, 0), (0, 64)]),
    'short last split': (None, 40, 1536, 1536, 1536, 1536, 0, [(0, 0)]),
}


@pytest.mark.parametrize('name', list(WGRAD_CASES))
def test_wgrad(eng, name):
    """dW += X^T G per segment onto a non-zero dW framed by guard rows.  X's columns past Cin and G's past N are NaN (outside
    the tensor maps), G's columns before its pointer hold WIDE_SOURCE_FILL."""
    B, T, Cin, ldx, N, ldg, g_off, segs = WGRAD_CASES[name]
    if B is None:
        B = _split_case_batch()
    g = torch.Generator().manual_seed(3000 + T + Cin + N)
    n_src = 1 + max(s for s, _ in segs)
    xs = []
    for _ in range(n_src):
        x = torch.full((B, T, ldx), float('nan')).bfloat16()
        x[..., :Cin] = torch.randn(B, T, Cin, generator=g).bfloat16()
        xs.append(x)
    gy = torch.full((B, T, ldg), float('nan')).bfloat16()
    gy[..., :g_off] = WIDE_SOURCE_FILL
    gy[..., g_off:g_off + N] = torch.randn(B, T, N, generator=g).bfloat16()
    rows, guard = len(segs) * Cin, 4
    buf0 = torch.randn(rows + 2 * guard, N, generator=g)
    buf = buf0.to(DEV, copy=True)
    xs_d, gy_d = [x.to(DEV) for x in xs], gy.to(DEV)
    eng._wgrad([(x, ldx) for x in xs_d], gy_d[..., g_off:], ldg, B, T, Cin, N, segs, buf[guard:guard + rows])
    torch.cuda.synchronize()
    ref, terms = torch.zeros(len(segs), Cin, N, dtype=torch.float64), torch.zeros(len(segs), Cin, N, dtype=torch.float64)
    gd = gy[..., g_off:g_off + N].double()
    for s, (src, sh) in enumerate(segs):
        lo, hi = max(0, -sh), min(T, T - sh)
        if hi > lo:
            xd = xs[src][:, lo + sh:hi + sh, :Cin].double()
            ref[s] = torch.einsum('btc,btn->cn', xd, gd[:, lo:hi])
            terms[s] = torch.einsum('btc,btn->cn', xd.abs(), gd[:, lo:hi].abs())
    got = buf.cpu()
    assert torch.equal(got[:guard], buf0[:guard]) and torch.equal(got[guard + rows:], buf0[guard + rows:]), f'{name}: guard rows changed'
    dw0 = buf0[guard:guard + rows].double()
    want = dw0 + ref.reshape(rows, N)
    # a segment without any term (|shift| >= T) leaves its rows bit for bit as they were
    denom = np.where(terms.reshape(rows, N).numpy() > 0, dw0.abs().numpy() + terms.reshape(rows, N).numpy(), 0.0)
    case = f'wgrad {name} B={B}'
    _report(case, 'dw', _elem_err(case, _host(got[guard:guard + rows]), want.numpy(), denom, False), GATE_WGRAD)


# ----------------------------------------------------------------------------------------------------------
# ttsb_softmax_fwd / ttsb_softmax_bwd
# ----------------------------------------------------------------------------------------------------------
# ld 16 ... 1024: the four register kernels (<= 128, 256, 512, 1024) at and next to their boundaries; 1040, 1504: the scalar kernel
@pytest.mark.parametrize('ld,Tk', [(16, 13), (128, 128), (144, 141), (256, 250), (512, 509), (1024, 1021), (1040, 1037), (1504, 1500)])
def test_softmax_forward_and_backward(ld, Tk):
    """T = 37 query rows against Tk keys (T != Tk), key lengths Tk, Tk/2, 1, 0, Tk + 5, -3, 20, flags 0..3, rates 0 (P_drop is
    P_pre), 0.1 and 0.25.  Forward: P_pre against the float64 softmax, rows summing to one, exact zeros at masked keys, dead rows
    and padding, P_drop zero exactly where the hash drops.  Backward, on synthetic inputs with the same mask: dS against float64."""
    B, H, T = 7, 2, 37
    Z = B * H
    lens = _lens(Tk, extra=(min(20, Tk),))
    lens_d = lens.to(DEV)
    scale = float(np.float32(0.125))
    for flags in range(4):
        mask = _key_mask(lens, H, T, Tk, ld, flags)
        for p in (0.0, 0.1, 0.25):
            g = torch.Generator().manual_seed(4000 + ld + 10 * flags + int(100 * p))
            site = 5 + flags
            case = f'softmax ld={ld} Tk={Tk} flags={flags} p={p}'
            S = _softmax_inputs(g, Z, T, Tk, ld, mask)
            P_pre = _poison16((Z, T, ld))
            P_drop = _poison16((Z, T, ld)) if p > 0 else P_pre
            lib.softmax_fwd(S.to(DEV), B, H, T, Tk, ld, lens_d, p, SEED, site, P_pre, P_drop, flags=flags)
            torch.cuda.synchronize()
            logits = torch.where(torch.from_numpy(mask), S.double(), torch.tensor(float('-inf'), dtype=torch.float64))
            ref = torch.nan_to_num(torch.softmax(logits, -1), nan=0.0).numpy()      # rows without a key: zeros
            got = _host(P_pre)
            assert np.isfinite(got).all() and (got[~mask] == 0).all(), f'{case}: P_pre not an exact zero at masked keys, dead rows or padding'
            _report(case, 'P_pre', _elem_err(case, got, ref, ref, True), GATE_SOFTMAX)
            has_key = mask.any(-1)
            _report(case, 'row sum', float(np.abs(got.sum(-1) - 1.0)[has_key].max()) if has_key.any() else 0.0, GATE_ROWSUM)
            keep = _keep(Z, T, ld, ld, p, site)
            if p > 0:
                gd = _host(P_drop)
                assert np.isfinite(gd).all() and (gd[~mask] == 0).all(), f'{case}: P_drop not an exact zero at masked keys, dead rows or padding'
                decides = mask & (got != 0)
                assert np.array_equal((gd != 0)[decides], keep[decides]), f'{case}: P_drop mask differs from the restated hash'
                kept_ref = ref * keep * dropout_scale(p)
                _report(case, 'P_drop', _elem_err(case, gd, kept_ref, kept_ref, True), GATE_SOFTMAX)
            # backward on synthetic inputs: P_pre non-zero at masked keys too (the kernel masks by length, not by P == 0)
            Pb = _poison16((Z, T, ld))
            Pb[..., :Tk] = (torch.rand(Z, T, Tk, generator=g) * (2.0 / Tk)).bfloat16().to(DEV)
            dP = torch.full((Z, T, ld), float('nan'))
            dP[..., :Tk] = torch.where(torch.from_numpy(mask[..., :Tk]), torch.randn(Z, T, Tk, generator=g), torch.tensor(WIDE_SOURCE_FILL))
            dS = _poison16((Z, T, ld))
            lib.softmax_bwd(Pb, dP.to(DEV), B, H, T, Tk, ld, lens_d, scale, p, SEED, site, dS, flags=flags)
            torch.cuda.synchronize()
            ks = dropout_scale(p) if p > 0 else 1.0
            Pm = np.where(mask, np.nan_to_num(_host(Pb)), 0.0)
            gg = np.where(mask, np.nan_to_num(dP.double().numpy()), 0.0) * keep * ks
            dot, adot = (Pm * gg).sum(-1, keepdims=True), np.abs(Pm * gg).sum(-1, keepdims=True)
            want = scale * Pm * (gg - dot)
            denom = scale * Pm * (np.abs(gg) + adot)
            got = _host(dS)
            assert np.isfinite(got).all() and (got[~mask] == 0).all(), f'{case}: dS not an exact zero at masked keys, dead rows or padding'
            _report(case, 'dS', _elem_err(case, got, want, denom, True), GATE_SOFTMAX_BWD)


# ----------------------------------------------------------------------------------------------------------
# small reductions
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dh', [2, 64, 130, 256])
def test_rowdot_heads(dh):
    """D = sum_c x y per (row, head); 74 rows (not a multiple of the 8 rows of a block), NaN in the columns past H * dh."""
    B, T, H = 2, 37, 3
    ld = H * dh + 6
    g = torch.Generator().manual_seed(5000 + dh)
    x, y = torch.full((B, T, ld), float('nan')).bfloat16(), torch.full((B, T, ld), float('nan')).bfloat16()
    x[..., :H * dh] = _heads_scaled(g, B, T, H, dh)
    y[..., :H * dh] = _heads_scaled(g, B, T, H, dh)
    out = torch.full((B * H * T,), float('nan'), device=DEV)
    lib.rowdot_heads(x.to(DEV), y.to(DEV), H, dh, out)
    torch.cuda.synchronize()
    prod = (x[..., :H * dh].double() * y[..., :H * dh].double()).reshape(B, T, H, dh).permute(0, 2, 1, 3)
    case = f'rowdot_heads dh={dh}'
    _report(case, 'D', _elem_err(case, _host(out).reshape(B, H, T), prod.sum(-1).numpy(), prod.abs().sum(-1).numpy(), False), GATE_SUM)


def _colsum_input(g, rows, C, ld, col0=0):
    """bf16 (rows, ld): data in [col0, col0 + C), WIDE_SOURCE_FILL before it and up to the 8-column group the kernel reads,
    NaN past that."""
    x = torch.full((rows, ld), float('nan')).bfloat16()
    x[:, :col0 + _round_up(C, 8)] = WIDE_SOURCE_FILL
    x[:, col0:col0 + C] = torch.randn(rows, C, generator=g).bfloat16()
    return x


@pytest.mark.parametrize('rows', [1, 127, 128, 129, 1000])
@pytest.mark.parametrize('C,ld,col0', [(226, 232, 0), (226, 256, 0), (3, 8, 0), (3, 128, 80)])
def test_colsum_bf16(C, ld, col0, rows):
    """Column sums accumulated onto a non-zero out; (3, 128, 80) is the stop-token bias gradient, three columns at column 80
    of the 128-wide post-net gradient."""
    g = torch.Generator().manual_seed(6000 + C + ld + rows)
    x = _colsum_input(g, rows, C, ld, col0)
    out0 = torch.randn(C + 5, generator=g)
    out = out0.to(DEV, copy=True)
    lib.colsum_bf16(x.to(DEV)[:, col0:], rows, C, ld, out)
    torch.cuda.synchronize()
    xd = x[:, col0:col0 + C].double()
    got = out.cpu()
    assert torch.equal(got[C:], out0[C:]), 'elements past C changed'
    case = f'colsum_bf16 C={C} ld={ld} col0={col0} rows={rows}'
    denom = out0[:C].double().abs() + xd.abs().sum(0)
    _report(case, 'sum', _elem_err(case, _host(got[:C]), (out0[:C].double() + xd.sum(0)).numpy(), denom.numpy(), False), GATE_SUM)


@pytest.mark.parametrize('rows', [129, 1000])
@pytest.mark.parametrize('seg,ld', [(128, 384), (72, 224)])
def test_colsum_bf16_x3(seg, ld, rows):
    """The q | k | v bias gradients from one (rows, ld) buffer into three accumulated outputs."""
    g = torch.Generator().manual_seed(6500 + seg + rows)
    x = _colsum_input(g, rows, 3 * seg, ld)
    outs0 = [torch.randn(seg + 3, generator=g) for _ in range(3)]
    outs = [o.to(DEV, copy=True) for o in outs0]
    lib.colsum_bf16_x3(x.to(DEV), rows, seg, ld, *outs)
    torch.cuda.synchronize()
    for i in range(3):
        xd = x[:, i * seg:(i + 1) * seg].double()
        got = outs[i].cpu()
        assert torch.equal(got[seg:], outs0[i][seg:]), 'elements past the segment changed'
        case = f'colsum_bf16_x3 seg={seg} ld={ld} rows={rows} out{i}'
        denom = outs0[i][:seg].double().abs() + xd.abs().sum(0)
        _report(case, 'sum', _elem_err(case, _host(got[:seg]), (outs0[i][:seg].double() + xd.sum(0)).numpy(), denom.numpy(), False), GATE_SUM)
