"""The row, scatter and loss kernels of the training step (csrc/train_ops.cu, csrc/rowops.cu) against float64, one by one
and as the two stack prologues issue them.

Each kernel is called through lib.py exactly as model/training.py calls it, at the shapes where it can go wrong: block
scans that carry between passes, channel loops that wrap, rows that are not a multiple of a block, padded and masked
rows, clamped ids and lengths.  Outputs start as NaN (or a non-zero fill where the contract accumulates or must leave
elements alone): every element the contract writes must have lost its NaN, padding must be an exact zero and everything
else stays as it was.  Dropout masks are the numpy restatement of the hash (gpu_util.dropout_keep), under a non-zero
dropout salt with the high bit set.

Exact operations are compared for equality.  Sums in fp32 are gated relative to the sum of the absolute values of their
terms: a different summation order than float64 costs about n * 2^-24 of that in the worst case, and a wrong or missing
term costs the size of a term.
"""
import numpy as np
import pytest
import torch

from gpu_util import DEV, dropout_mask, dropout_scale
from transformertts_b200 import lib

pytestmark = pytest.mark.gpu

SALT = 0xC2B2AE35   # high bit set: the XOR of the whole word into the seed is covered
SEED = 0x2545F491
EPS = 1e-6

# Measured on an H100 80GB HBM3 (SXM, 700 W power limit), the largest error of any case under each gate.  The atomics
# of embedding_bwd, pe_scalar_bwd and the dw / db sums add in a different order on every run: their gates are bounds.
GATE_SUM = 4e-7        # fp32 sums (segment sums, scatter-adds, channel sums), |err| / sum |terms| (1.8e-7, embedding_bwd)
GATE_SCALAR = 1.5e-8   # pe_scalar_bwd: one fp32 number summing every element, |err| / sum |terms| (5.9e-9)
GATE_LOSS = 8e-8       # the diagonal loss, |err| / loss, all terms >= 0 (3.3e-8)
GATE_LN_FWD = 2e-5     # the prologue forward: max abs error of fp32 LayerNorm + PE, the gate of test_embed_ln_pe (1.0e-6)
GATE_BWD = 6e-7        # the prologue backward chains (LayerNorm bwd, then a scatter or a segment sum), max |err| / max |ref| (2.6e-7)


@pytest.fixture(scope='module', autouse=True)
def dropout_salt():
    lib.load()
    lib.set_dropout_salt(torch.tensor([np.uint32(SALT).view(np.int32)], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    yield SALT
    lib.set_dropout_salt(torch.zeros(1, dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()


def _report(case, what, err, gate):
    print(f'[train-rowops] {case}: {what} err {err:.2e} (gate {gate:.1e})')
    assert err < gate, f'{case}: {what} error {err:.3e} >= gate {gate:.1e}'


def _sum_err(got, ref, abs_terms):
    """max |got - ref| / sum|terms| over the elements that have terms; elements without any term must equal ref exactly."""
    got = got.detach().double().cpu()
    ref, abs_terms = ref.detach().double().cpu(), abs_terms.detach().double().cpu()
    assert torch.isfinite(got).all(), 'non-finite values in kernel output'
    empty = abs_terms == 0
    assert torch.equal(got[empty], ref[empty]), 'elements without any term differ from their initial value'
    if (~empty).any():
        return float(((got - ref).abs()[~empty] / abs_terms[~empty]).max())
    return 0.0


def _relerr(got, ref):
    got = got.detach().double().cpu()
    ref = ref.detach().double().cpu()
    assert torch.isfinite(got).all(), 'non-finite values in kernel output'
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _nan(*shape):
    return torch.full(shape, float('nan'), device=DEV)


def _check_mask(case, got_kept, keep, decidable):
    """Dropout mask bit for bit: an element is dropped iff its output is exactly zero (where the undropped value is not ~0)."""
    assert int(decidable.sum()) > 0, f'{case}: no element decides the mask'
    bad = int((got_kept != keep)[decidable].sum())
    assert bad == 0, f'{case}: dropout mask differs from the restated hash at {bad} elements'


def _keep(B, T, d, p, site):
    """(B,T,d) float64 keep * fp32(1/(1-p)) of a (B,T,d) tensor drawn at (b*T + t)*d + c (1 everywhere at p = 0)."""
    if p == 0:
        return torch.ones(B, T, d, dtype=torch.float64)
    return torch.from_numpy(dropout_mask(B, T, d, d, SEED, site, p, SALT)).double() * dropout_scale(p)


def _layer_norm(u, gamma, beta):
    mean = u.mean(-1, keepdim=True)
    var = ((u - mean) ** 2).mean(-1, keepdim=True)
    return (u - mean) * torch.rsqrt(var + EPS) * gamma + beta


# ----------------------------------------------------------------------------------------------------------
# length-regulator backward: segment sums of frame gradients per phoneme
# ----------------------------------------------------------------------------------------------------------
def _durations(g, Tp):
    """Rows: random with zeros and negatives (summing past Tm: clipped), a third of it (short of Tm: trailing frames
    belong to nobody), all zero, random again.  Tm is three frames short of row 0's total."""
    dur = torch.randint(-2, 8, (4, Tp), generator=g, dtype=torch.int32)
    dur[0, 0] = 7
    dur[1] = torch.div(dur[0], 3, rounding_mode='floor')
    dur[2] = 0
    tot = dur.clamp_min(0).sum(1)
    Tm = int(tot[0]) - 3
    assert 0 < tot[1] < Tm and tot[0] > Tm
    return dur, Tm


def _segment_sums(x, dur, Tm):
    """float64 sums of x[b, t] over t in [s_i, s_i + max(dur_i, 0)) clipped to [0, Tm), s_i the exclusive prefix sum."""
    B, Tp = dur.shape
    d = x.shape[-1]
    cs = torch.cat([torch.zeros(B, 1, d, dtype=torch.float64), x.double().cumsum(1)], 1)
    ends = dur.clamp_min(0).long().cumsum(1)
    starts = (ends - dur.clamp_min(0).long()).clamp(max=Tm)
    ends = ends.clamp(max=Tm)
    take = lambda idx: torch.gather(cs, 1, idx[..., None].expand(B, Tp, d))
    return take(ends) - take(starts)


@pytest.mark.parametrize('d', [4, 256, 516])
@pytest.mark.parametrize('Tp', [1, 257, 1500])
def test_expand_bwd(Tp, d):
    """Tp = 257 and 1500 run the 256-wide block scan over several passes with a carry; d = 516 makes lanes loop more than
    once over d/4 with a partial last pass; segments of odd length take the unroll-by-two tail."""
    g = torch.Generator().manual_seed(200 + Tp + d)
    dur, Tm = _durations(g, Tp)
    B = dur.shape[0]
    dm = torch.randn(B, Tm, d, generator=g)
    dx = _nan(B, Tp, d)
    lib.expand_bwd(dm.to(DEV), dur.to(DEV), dx)
    torch.cuda.synchronize()
    ref = _segment_sums(dm, dur, Tm)
    abs_terms = _segment_sums(dm.abs(), dur, Tm)
    if Tp > 1:
        assert (dur < 0).any() and (dur == 0).any() and (dur % 2 == 1).any()
    _report(f'expand_bwd Tp={Tp} d={d} Tm={Tm}', 'dx', _sum_err(dx, ref, abs_terms), GATE_SUM)


# ----------------------------------------------------------------------------------------------------------
# embedding backward: scatter-add into the table
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', [100, 384])
def test_embedding_bwd(d):
    """600 rows into 37 table rows (every row collides), ids < 0 and >= vocab clamped to the first and last row as in the
    forward, accumulated onto a non-zero table; rows no id reaches stay bit for bit as they were."""
    g = torch.Generator().manual_seed(300 + d)
    B, T, vocab = 4, 150, 37
    tok = torch.randint(1, vocab - 10, (B, T), generator=g, dtype=torch.int32)
    tok[0, :7] = torch.tensor([-1, -5, vocab, vocab + 3, 2 ** 30, -2 ** 31, 5], dtype=torch.int32)
    tok[1, :] = 3    # one table row receives a whole sentence
    dx = torch.randn(B, T, d, generator=g)
    demb0 = torch.randn(vocab, d, generator=g)
    demb = demb0.to(DEV, copy=True)
    lib.embedding_bwd(dx.to(DEV), tok.to(DEV), demb)
    torch.cuda.synchronize()
    rows = tok.long().clamp(0, vocab - 1).reshape(-1)
    ref = demb0.double().index_add(0, rows, dx.double().reshape(-1, d))
    abs_terms = demb0.double().abs().index_add(0, rows, dx.double().abs().reshape(-1, d))
    hit = torch.zeros(vocab, dtype=torch.bool)
    hit[rows] = True
    assert (~hit).any() and hit[0] and hit[vocab - 1]
    assert torch.equal(demb.cpu()[~hit], demb0[~hit]), 'table rows no id reaches changed'
    _report(f'embedding_bwd d={d}', 'demb', _sum_err(demb[hit], ref[hit], abs_terms[hit]), GATE_SUM)


# ----------------------------------------------------------------------------------------------------------
# gradient of the positional-encoding scalar
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('p', [0.0, 0.1])
@pytest.mark.parametrize('d', [256, 160, 130, 1600])
def test_pe_scalar_bwd(d, p):
    """d = 256 and 160 take the float4 kernel (160: 384 threads hold 9 rows of 40 vectors, the last 24 threads idle);
    130 and 1600 (wider than a block) the scalar kernel.  The mask is drawn at row*d + c; the result, one number, is
    accumulated onto a non-zero value."""
    g = torch.Generator().manual_seed(400 + d)
    B, T, site = 3, 200, 9
    grad = torch.randn(B, T, d, generator=g)
    pe = torch.randn(T, d, generator=g)
    out = torch.tensor([0.25], device=DEV)
    lib.pe_scalar_bwd(grad.to(DEV), pe.to(DEV), out, drop=(p, SEED, site))
    torch.cuda.synchronize()
    terms = grad.double() * _keep(B, T, d, p, site) * pe.double()
    ref = 0.25 + terms.sum()
    err = abs(float(out.item()) - float(ref)) / float(terms.abs().sum())
    _report(f'pe_scalar_bwd d={d} p={p}', 'dscalar', err, GATE_SCALAR)


# ----------------------------------------------------------------------------------------------------------
# pitch embedding Dense(1 -> d, ReLU): kernel and bias gradients
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', [226, 640])
def test_pitch_embed_bwd(d):
    """111 rows (not a multiple of the 64-row slab); 640 channels need more than the 512 threads of a block.  Rows with
    pitch 0, and channels whose bias makes p*w + b exactly 0 at pitch 2 or 0: there the ReLU passes no gradient.  The
    gate is decided on the exact p*w + b, whose sign float64 gets right for fp32 inputs, and so does the kernel's fmaf."""
    g = torch.Generator().manual_seed(500 + d)
    B, T = 3, 37
    grad = torch.randn(B, T, d, generator=g)
    pitch = torch.randn(B, T, generator=g)
    pitch[0, :5] = 0.0
    pitch[1, :6] = 2.0
    w = torch.randn(d, generator=g)
    b = 0.5 * torch.randn(d, generator=g)
    w[:8] = 0.5 * torch.arange(1, 9, dtype=torch.float32)
    b[:8] = -torch.arange(1, 9, dtype=torch.float32)    # p = 2: p*w + b == 0
    b[8:12] = 0.0                                        # p = 0: p*w + b == 0
    b[12:16] = 0.25                                      # p = 0: gradient reaches the bias, none the kernel
    dw0, db0 = torch.randn(d, generator=g), torch.randn(d, generator=g)
    dw, db = dw0.to(DEV, copy=True), db0.to(DEV, copy=True)
    lib.pitch_embed_bwd(grad.to(DEV), pitch.to(DEV), w.to(DEV), b.to(DEV), dw, db)
    torch.cuda.synchronize()
    pre = pitch.double()[..., None] * w.double() + b.double()
    assert (pre == 0).sum() >= 8 * 6 + 4 * 5
    on = (pre > 0).double()
    gp = grad.double() * on * pitch.double()[..., None]
    gb = grad.double() * on
    case = f'pitch_embed_bwd d={d}'
    _report(case, 'dw', _sum_err(dw, dw0.double() + gp.sum((0, 1)), dw0.double().abs() + gp.abs().sum((0, 1))), GATE_SUM)
    _report(case, 'db', _sum_err(db, db0.double() + gb.sum((0, 1)), db0.double().abs() + gb.abs().sum((0, 1))), GATE_SUM)


# ----------------------------------------------------------------------------------------------------------
# StatPredictor head backward
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('relu', [0, 1])
@pytest.mark.parametrize('C,ldh', [(226, 256), (256, 256)])
def test_statpred_head_bwd(C, ldh, relu):
    """out = act(h.w + b) * (t < row_len): rows past row_len (row_len 0 and T included) and, with the ReLU, outputs <= 0
    (0 and -0 included) pass no gradient.  dh = g * w is one fp32 product (bit-exact), its padding columns [C, ldh) are
    exact zeros; dw and db accumulate onto existing values."""
    g = torch.Generator().manual_seed(600 + C + relu)
    B, T = 4, 50
    h = torch.randn(B, T, ldh, generator=g)
    gout = torch.randn(B, T, generator=g)
    out = torch.randn(B, T, generator=g)
    out[0, :4] = torch.tensor([0.0, -0.0, 1e-30, -1e-30])
    w = torch.randn(C, generator=g)
    lens = torch.tensor([T, 0, 17, 33], dtype=torch.int32)
    dw0, db0 = torch.randn(C, generator=g), torch.randn(1, generator=g)
    dh = _nan(B, T, ldh)
    dw, db = dw0.to(DEV, copy=True), db0.to(DEV, copy=True)
    lib.statpred_head_bwd(gout.to(DEV), out.to(DEV), h.to(DEV), C, w.to(DEV), relu, lens.to(DEV), dh, dw, db)
    torch.cuda.synchronize()
    live = (torch.arange(T)[None, :] < lens[:, None]).double()
    gate = live * ((out > 0).double() if relu else 1.0)
    gg = gout.double() * gate
    case = f'statpred_head_bwd C={C} ldh={ldh} relu={relu}'
    want_dh = torch.zeros(B, T, ldh)
    want_dh[..., :C] = (gg[..., None] * w.double()).float()
    assert torch.equal(dh.cpu(), want_dh), f'{case}: dh differs from g * w (padding columns and gated rows must be 0)'
    tw = gg[..., None] * h.double()[..., :C]
    _report(case, 'dw', _sum_err(dw, dw0.double() + tw.sum((0, 1)), dw0.double().abs() + tw.abs().sum((0, 1))), GATE_SUM)
    _report(case, 'db', _sum_err(db, db0.double() + gg.sum(), db0.double().abs() + gg.abs().sum()), GATE_SUM)


# ----------------------------------------------------------------------------------------------------------
# diagonal loss of the Aligner on the bf16 probabilities, and its gradient added into dP
# ----------------------------------------------------------------------------------------------------------
def _grad_scale_power_of_two(BH, target=0.125):
    """A grad_scale whose fp32 product with the host's 1/(10*B*H) is exactly `target`: the kernel's per-element term
    grad_scale/(10*B*H) * m is then exact in fp32, and dP + term rounds the same with or without an FMA."""
    inv = np.float32(1.0) / (np.float32(10.0) * np.float32(BH))
    gs = np.float32(target) * np.float32(10 * BH)
    for _ in range(64):
        prod = gs * inv
        if prod == np.float32(target):
            return float(gs), float(inv)
        gs = np.nextafter(gs, np.float32(np.inf) if prod < target else np.float32(-np.inf))
    raise AssertionError('no grad_scale found')


def _diag_mask(B, Tq, Tk, q_len, k_len):
    """(B, Tq, Tk) float32 |k/k_len - q/q_len| over q < q_len, k < k_len (lengths clamped to [0, Tq] / [0, Tk]), divided
    in float64 and cast to float32 as the reference does; 0 outside, with the region as a bool mask."""
    m = np.zeros((B, Tq, Tk), dtype=np.float32)
    region = np.zeros((B, Tq, Tk), dtype=bool)
    for b in range(B):
        qn, kn = min(max(int(q_len[b]), 0), Tq), min(max(int(k_len[b]), 0), Tk)
        if qn == 0 or kn == 0:
            continue
        q = np.arange(qn, dtype=np.float64)[:, None] / qn
        k = np.arange(kn, dtype=np.float64)[None, :] / kn
        m[b, :qn, :kn] = np.abs(k - q).astype(np.float32)
        region[b, :qn, :kn] = True
    return torch.from_numpy(m), torch.from_numpy(region)


def test_diag_loss_train():
    """Rows: q_len = Tq with k_len > Tk (clamped), q_len = 0, lengths inside, q_len > Tq (clamped); Tq = 45 is not a
    multiple of the 32-query blocks.  dP gains exactly grad_scale/(10*B*H) * m inside the region and is unchanged outside
    it and in the padding columns [Tk, ld); the loss matches float64 on the bf16 maps and ttsb_diag_loss on the same maps
    widened to fp32; the loss-only call (dP = None) gives the same loss."""
    g = torch.Generator().manual_seed(700)
    B, H, Tq, Tk, ld = 4, 2, 45, 40, 48
    q_len = torch.tensor([Tq, 0, 30, Tq + 15], dtype=torch.int32)
    k_len = torch.tensor([Tk + 15, 20, 17, Tk], dtype=torch.int32)
    P = torch.rand(B * H, Tq, ld, generator=g).bfloat16()
    dP0 = torch.randn(B * H, Tq, ld, generator=g)
    gs, inv = _grad_scale_power_of_two(B * H)
    loss_scale = 1.0
    m, region = _diag_mask(B, Tq, Tk, q_len, k_len)
    m = m.repeat_interleave(H, 0)
    region = region.repeat_interleave(H, 0)
    region_ld = torch.zeros(B * H, Tq, ld, dtype=torch.bool)
    region_ld[..., :Tk] = region
    m_ld = torch.zeros(B * H, Tq, ld)
    m_ld[..., :Tk] = m

    loss = torch.tensor([0.5], device=DEV)
    dP = dP0.to(DEV, copy=True)
    P_d, ql, kl = P.to(DEV), q_len.to(DEV), k_len.to(DEV)
    lib.diag_loss_train(P_d, B, H, Tq, Tk, ld, ql, kl, loss_scale, loss, gs, dP)
    loss_only = torch.tensor([0.5], device=DEV)
    lib.diag_loss_train(P_d, B, H, Tq, Tk, ld, ql, kl, loss_scale, loss_only, gs, None)
    att = P.float()[..., :Tk].reshape(B, H, Tq, Tk).contiguous()
    loss_f32 = torch.zeros(1, device=DEV)
    lib.diag_loss(att.to(DEV), ql, kl, loss_f32)
    torch.cuda.synchronize()

    case = f'diag_loss_train B={B} H={H} Tq={Tq} Tk={Tk} ld={ld}'
    term = np.float32(gs) * np.float32(inv)
    assert term == np.float32(0.125)
    want = dP0.clone()
    want[region_ld] = dP0[region_ld] + float(term) * m_ld[region_ld]     # float32: the product is exact, one rounding in the sum
    got = dP.cpu()
    assert torch.equal(got[~region_ld], dP0[~region_ld]), f'{case}: dP changed outside q < q_len, k < k_len'
    assert torch.equal(got[region_ld], want[region_ld]), f'{case}: dP did not gain exactly grad_scale/(10*B*H) * m'
    terms = P.double() * m_ld.double()
    scale = float(np.float32(loss_scale) * np.float32(inv))
    ref = float(terms.sum()) * scale
    _report(case, 'loss', abs(float(loss.item()) - 0.5 - ref) / ref, GATE_LOSS)
    _report(case, 'loss (dP = None)', abs(float(loss_only.item()) - 0.5 - ref) / ref, GATE_LOSS)
    _report(case, 'loss vs ttsb_diag_loss on fp32 maps', abs(float(loss.item()) - 0.5 - float(loss_f32.item())) / ref, GATE_LOSS)


# ----------------------------------------------------------------------------------------------------------
# bf16 cast with zero padding, in-place ReLU mask
# ----------------------------------------------------------------------------------------------------------
def _specials():
    return torch.tensor([0.0, -0.0, float('nan'), float('inf'), -float('inf'), 1e-40, -1e-40, 1 + 2 ** -8, 1 + 3 * 2 ** -9,
                         3.3961776e38, 3.4028235e38, -1.0, 2 ** -133])


@pytest.mark.parametrize('C,ld', [(80, 128), (226, 256), (64, 64)])
def test_cast_bf16_pad(C, ld):
    """Round to nearest even, bit for bit with torch (NaN stays NaN); padding columns [C, ld), poisoned first, come out
    +0."""
    g = torch.Generator().manual_seed(800 + C)
    rows = 333
    x = torch.randn(rows, C, generator=g) * torch.exp2(torch.randint(-30, 30, (rows, C), generator=g).float())
    sp = _specials()
    x.view(-1)[:sp.numel()] = sp
    out = torch.empty(rows, ld, dtype=torch.bfloat16, device=DEV)
    out.view(torch.int16).fill_(-1)
    lib.cast_bf16_pad(x.to(DEV), rows, C, out, ld)
    torch.cuda.synchronize()
    got = out.cpu()
    want = x.bfloat16()
    nan = torch.isnan(x)
    assert torch.isnan(got[:, :C][nan]).all()
    assert torch.equal(got[:, :C].view(torch.int16)[~nan], want.view(torch.int16)[~nan]), 'bf16 cast is not round-to-nearest-even'
    assert (got[:, C:].view(torch.int16) == 0).all(), 'padding columns are not +0'


def test_relu_bwd():
    """dy *= (h > 0) in place: h in {0, -0, NaN, -inf, negative} drops the gradient (written as +0), h > 0 (a subnormal
    and +inf included) keeps its bits, NaN gradients included."""
    g = torch.Generator().manual_seed(900)
    n = 8 * 1001
    h = torch.randn(n, generator=g)
    sp = _specials()
    h[:sp.numel()] = sp
    h[sp.numel():2 * sp.numel()] = -sp
    h = h.bfloat16()
    dy = torch.randn(n, generator=g).bfloat16()
    dy[7::97] = float('nan')
    dy_d = dy.to(DEV)
    lib.relu_bwd(dy_d, h.to(DEV))
    torch.cuda.synchronize()
    want = torch.where(h.float() > 0, dy.view(torch.int16), torch.zeros((), dtype=torch.int16))
    assert torch.equal(dy_d.cpu().view(torch.int16), want)


# ----------------------------------------------------------------------------------------------------------
# the two train-mode prologues with dropout on
# ----------------------------------------------------------------------------------------------------------
def _check_prologue(case, out, hi, u64, gamma, beta, pe_rows, scalar, p, site):
    """out / hi: the kernel's fp32 and bf16 outputs (B,T,d); u64: float64 LayerNorm inputs; pe_rows (B,T,d) float64."""
    B, T, d = out.shape
    undropped = _layer_norm(u64, gamma.double(), beta.double()) + float(scalar) * pe_rows
    keep = torch.from_numpy(dropout_mask(B, T, d, d, SEED, site, p, SALT))
    ref = undropped * keep * dropout_scale(p)
    got = out.cpu()
    assert not torch.isnan(got).any() and not torch.isnan(hi.cpu().float()).any(), f'{case}: unwritten output elements'
    _check_mask(case, got != 0, keep, undropped.abs() > 1e-3 * undropped.abs().max())
    _report(case, 'f32 max abs err', float((got.double() - ref).abs().max()), GATE_LN_FWD)
    assert torch.equal(hi.cpu(), got.bfloat16()), f'{case}: bf16 output is not the rounded fp32 output'


@pytest.mark.parametrize('d', [100, 384])
def test_embed_ln_pe_fwd_dropout(d):
    """Embedding rows (ids < 0 and >= vocab clamped) -> LayerNorm + scalar * PE -> dropout at (b*T + t)*d + c."""
    g = torch.Generator().manual_seed(1000 + d)
    B, T, vocab, p, site = 3, 77, 53, 0.1, 13
    tok = torch.randint(0, vocab, (B, T), generator=g, dtype=torch.int32)
    tok[0, :3] = torch.tensor([-3, vocab, vocab + 9], dtype=torch.int32)
    emb = torch.randn(vocab, d, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    pe = torch.randn(T, d, generator=g)
    scalar = torch.tensor([0.8])
    out = _nan(B, T, d)
    hi = torch.full((B, T, d), float('nan'), device=DEV, dtype=torch.bfloat16)
    lib.embed_ln_pe_fwd(tok.to(DEV), emb.to(DEV), gamma.to(DEV), beta.to(DEV), pe.to(DEV), scalar.to(DEV), EPS, out, hi, None,
                        drop=(p, SEED, site))
    torch.cuda.synchronize()
    u64 = emb.double()[tok.long().clamp(0, vocab - 1)]
    _check_prologue(f'embed_ln_pe_fwd d={d} p={p}', out, hi, u64, gamma, beta, pe.double().expand(B, T, d), scalar, p, site)


@pytest.mark.parametrize('d', [100, 384])
def test_expand_ln_pe_fwd_dropout(d):
    """Frames gathered from phoneme rows by idx (-1: a zero row, normalised to beta) -> LayerNorm + scalar * PE of the
    frame index -> dropout at (b*Tm + t)*d + c."""
    g = torch.Generator().manual_seed(1100 + d)
    B, Tp, Tm, p, site = 3, 29, 90, 0.1, 14
    x = torch.randn(B, Tp, d, generator=g)
    idx = torch.randint(-1, Tp, (B, Tm), generator=g, dtype=torch.int32)
    idx[:, -7:] = -1
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    pe = torch.randn(Tm, d, generator=g)
    scalar = torch.tensor([1.1])
    out = _nan(B, Tm, d)
    hi = torch.full((B, Tm, d), float('nan'), device=DEV, dtype=torch.bfloat16)
    lib.expand_ln_pe_fwd(x.to(DEV), idx.to(DEV), gamma.to(DEV), beta.to(DEV), pe.to(DEV), scalar.to(DEV), EPS, out, hi, None,
                         drop=(p, SEED, site))
    torch.cuda.synchronize()
    src = idx.long().clamp_min(0)
    u64 = torch.gather(x.double(), 1, src[..., None].expand(B, Tm, d)) * (idx >= 0)[..., None]
    _check_prologue(f'expand_ln_pe_fwd d={d} p={p}', out, hi, u64, gamma, beta, pe.double().expand(B, Tm, d), scalar, p, site)


# ----------------------------------------------------------------------------------------------------------
# the prologues forward and backward, issued as model/training.py issues them, against float64 autograd
# ----------------------------------------------------------------------------------------------------------
P_DROP = 0.1


def _prologue_bwd(dz, u, gamma, pe, B, T, d, site, dscalar, dgamma, dbeta):
    """TrainEngine._prologue_bwd: the pos_scalar gradient and the LayerNorm backward with the prologue's dropout mask."""
    lib.pe_scalar_bwd(dz, pe, dscalar, drop=(P_DROP, SEED, site))
    du = _nan(B, T, d)
    lib.layernorm_bwd(dz, u.contiguous(), gamma, B, T, d, d, EPS, None, False, du, None, dgamma, dbeta,
                      post_drop=(P_DROP, site), seed=SEED)
    return du


def _params(g, d):
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    return gamma, beta, torch.tensor([0.9])


@pytest.mark.parametrize('d', [256, 192])
def test_encoder_prologue_forward_backward(d):
    """embed_ln_pe_fwd(dropout) -> pe_scalar_bwd + layernorm_bwd(post dropout) + embedding_bwd.  d = 256 takes the
    vectorised LayerNorm backward, 192 the generic one.  A forward and a backward that draw their masks at different
    indices agree with themselves but not with autograd through the restated mask."""
    g = torch.Generator().manual_seed(1200 + d)
    B, T, vocab, site = 4, 61, 45, 21
    tok = torch.randint(0, vocab, (B, T), generator=g, dtype=torch.int32)
    emb = 0.5 * torch.randn(vocab, d, generator=g)
    gamma, beta, scalar = _params(g, d)
    pe = torch.randn(T, d, generator=g)
    dz = torch.randn(B, T, d, generator=g)

    tok_d, emb_d, gamma_d, pe_d, dz_d = tok.to(DEV), emb.to(DEV), gamma.to(DEV), pe.to(DEV), dz.to(DEV)
    e_rows = emb_d[tok_d.long()].contiguous()           # the trainer keeps the gathered rows as the LayerNorm input
    h = _nan(B, T, d)
    lib.embed_ln_pe_fwd(tok_d, emb_d, gamma_d, beta.to(DEV), pe_d, scalar.to(DEV), EPS, h, None, None, drop=(P_DROP, SEED, site))
    dscalar, dgamma, dbeta = torch.zeros(1, device=DEV), torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
    du = _prologue_bwd(dz_d, e_rows, gamma_d, pe_d, B, T, d, site, dscalar, dgamma, dbeta)
    demb = torch.zeros(vocab, d, device=DEV)
    lib.embedding_bwd(du, tok_d, demb)
    torch.cuda.synchronize()

    keep = _keep(B, T, d, P_DROP, site)
    emb64, g64, b64, s64 = (t.double().requires_grad_() for t in (emb, gamma, beta, scalar))
    u64 = emb64[tok.long()]
    u64.retain_grad()
    y = (_layer_norm(u64, g64, b64) + s64 * pe.double()) * keep
    (y * dz.double()).sum().backward()
    case = f'encoder prologue d={d}'
    _report(case, 'forward (max abs err)', float((h.cpu().double() - y.detach()).abs().max()), GATE_LN_FWD)
    _report(case, 'd embedding rows', _relerr(du, u64.grad), GATE_BWD)
    _report(case, 'd embedding table', _relerr(demb, emb64.grad), GATE_BWD)
    _report(case, 'd gamma', _relerr(dgamma, g64.grad), GATE_BWD)
    _report(case, 'd beta', _relerr(dbeta, b64.grad), GATE_BWD)
    _report(case, 'd pos_scalar', abs(float(dscalar.item()) - float(s64.grad)) / float((dz.double() * keep * pe.double()).abs().sum()),
            GATE_SCALAR)


@pytest.mark.parametrize('d', [256, 192])
def test_decoder_prologue_forward_backward(d):
    """pitch_embed_add_fwd -> expand_indices / length_regulate_fwd / expand_ln_pe_fwd(dropout) -> pe_scalar_bwd +
    layernorm_bwd(post dropout) -> expand_bwd -> pitch_embed_bwd: the gradients of the encoder output, pitch_embed.w / .b,
    LN gamma / beta and pos_scalar against autograd.  Tm runs past every row's frames (idx = -1, gradients to nobody)."""
    g = torch.Generator().manual_seed(1300 + d)
    B, Tp, site = 3, 37, 22
    h_f = torch.randn(B, Tp, d, generator=g)
    pitch = torch.randn(B, Tp, generator=g)
    pw, pb = torch.randn(d, generator=g), 0.5 * torch.randn(d, generator=g)
    dur = torch.randint(0, 6, (B, Tp), generator=g, dtype=torch.int32)
    Tm = int(dur.sum(1).max()) + 5
    gamma, beta, scalar = _params(g, d)
    pe = torch.randn(Tm, d, generator=g)
    dz = torch.randn(B, Tm, d, generator=g)

    h_d, pitch_d, pw_d, pb_d, dur_d = h_f.to(DEV), pitch.to(DEV), pw.to(DEV), pb.to(DEV), dur.to(DEV)
    gamma_d, pe_d = gamma.to(DEV), pe.to(DEV)
    h_pe = _nan(B, Tp, d)
    lib.pitch_embed_add_fwd(h_d, pitch_d, pw_d, pb_d, h_pe)
    idx = torch.empty(B, Tm, dtype=torch.int32, device=DEV)
    lib.expand_indices(dur_d, Tm, idx)
    expanded = _nan(B, Tm, d)
    lib.length_regulate_fwd(h_pe, idx, expanded)
    m_f = _nan(B, Tm, d)
    lib.expand_ln_pe_fwd(h_pe, idx, gamma_d, beta.to(DEV), pe_d, scalar.to(DEV), EPS, m_f, None, None, drop=(P_DROP, SEED, site))
    dscalar, dgamma, dbeta = torch.zeros(1, device=DEV), torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
    d_exp = _prologue_bwd(dz.to(DEV), expanded, gamma_d, pe_d, B, Tm, d, site, dscalar, dgamma, dbeta)
    dh_pe = _nan(B, Tp, d)
    lib.expand_bwd(d_exp, dur_d, dh_pe)
    dpw, dpb = torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
    lib.pitch_embed_bwd(dh_pe, pitch_d, pw_d, pb_d, dpw, dpb)
    torch.cuda.synchronize()

    keep = _keep(B, Tm, d, P_DROP, site)
    h64, pw64, pb64, g64, b64, s64 = (t.double().requires_grad_() for t in (h_f, pw, pb, gamma, beta, scalar))
    hpe64 = h64 + torch.relu(pitch.double()[..., None] * pw64 + pb64)
    frames = torch.arange(Tm)[None, :] < dur.long().sum(1)[:, None]
    src = torch.repeat_interleave(torch.arange(Tp).expand(B, Tp), dur.long().reshape(-1)).reshape(-1)
    idx_ref = torch.full((B, Tm), -1, dtype=torch.long)
    idx_ref[frames] = src
    assert torch.equal(idx.cpu().long(), idx_ref)
    ex64 = torch.gather(hpe64, 1, idx_ref.clamp_min(0)[..., None].expand(B, Tm, d)) * frames[..., None]
    y = (_layer_norm(ex64, g64, b64) + s64 * pe.double()) * keep
    (y * dz.double()).sum().backward()
    case = f'decoder prologue d={d} Tm={Tm}'
    _report(case, 'forward (max abs err)', float((m_f.cpu().double() - y.detach()).abs().max()), GATE_LN_FWD)
    _report(case, 'd encoder output', _relerr(dh_pe, h64.grad), GATE_BWD)
    _report(case, 'd pitch_embed.w', _relerr(dpw, pw64.grad), GATE_BWD)
    _report(case, 'd pitch_embed.b', _relerr(dpb, pb64.grad), GATE_BWD)
    _report(case, 'd gamma', _relerr(dgamma, g64.grad), GATE_BWD)
    _report(case, 'd beta', _relerr(dbeta, b64.grad), GATE_BWD)
    _report(case, 'd pos_scalar', abs(float(dscalar.item()) - float(s64.grad)) / float((dz.double() * keep * pe.double()).abs().sum()),
            GATE_SCALAR)
