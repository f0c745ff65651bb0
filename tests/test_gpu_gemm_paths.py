"""Every code path of the tensor-core forward GEMM (ttsb_linear_fwd, csrc/gemm_tc.cu) against float64 at its edge shapes.

The host picks one of several kernels / epilogues per call: SIMT; single CTA with direct stores; single CTA with staged TMA
tile stores (16-bit outputs only); the LayerNorm epilogue on one CTA, on a CTA pair, or as full single-CTA waves followed
by a pair tail (two launches).  Each case below derives its shape from the SM count so that it lands on the path it
names, asserts that `_schedule` (a mirror of the host's choice) agrees, and checks the launch count.  Outputs start as
NaN: every element the contract says is written must have lost its NaN, padding columns and masked rows must be exact
zeros, and columns past the tiles must stay untouched.  Dropout masks are compared bit for bit with a numpy restatement
of the hash, under a non-zero dropout salt.
"""
import numpy as np
import pytest
import torch

from gpu_util import DEV, dropout_mask, dropout_scale, ref_gemm, run_gemm
from transformertts_b200 import lib

pytestmark = pytest.mark.gpu

SALT = 0x9E3779B9   # high bit set: the XOR of the whole word into the seed is covered
SEED = 0x1234ABCD

# max |err| / max |ref| over every row.  Measured on an H100 SXM (700 W), the largest error of any case under each gate:
GATE_X3 = 2e-5        # bf16x3, fp32 output, hi + lo or out_preln (8.3e-6)
GATE_X3_LN = 4e-5     # bf16x3 with the LayerNorm epilogue (6.8e-6)
GATE_BF16 = 2e-6      # one bf16 product, fp32 output or out_preln; the reference rounds the operands to bf16 (3.1e-7)
GATE_BF16_LN = 8e-6   # the same through the LayerNorm epilogue (2.4e-6)
GATE_BF16_OUT = 4e-3  # a bf16 output plane: round to nearest with 8 significant bits, error <= 2^-8 (2.9e-3)
GATE_FP16_OUT = 3e-3  # an fp16 output plane (4.0e-4)
GATE_BWD = 2e-6       # ttsb_layernorm_bwd: du, dgamma, dbeta in fp32


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _schedule(B, T, N, block_n, ln, sms):
    """Mirror of the schedule choice of ttsb_linear_fwd (csrc/gemm_tc.cu:735-749, in float32 as there): LayerNorm GEMMs
    whose row splits into equal halves of at most 192 columns (pair_ok) run single-CTA, as CTA pairs (cost 0.57 per round
    of sms/2 clusters) or as full single-CTA waves followed by a pair tail, whichever costs the fewest rounds."""
    pair_ok = ln and N == block_n and N % 32 == 0 and N // 2 <= 192 and N >= 64
    if not pair_ok:
        return 'single'
    f32 = np.float32
    single_ok = block_n <= 256
    t = B * (-(-T // 128))
    clusters = sms // 2
    k = f32(0.57)
    c_single = f32(-(-t // sms)) if single_ok else f32(1e30)
    c_pair = k * f32(-(-t // clusters))
    full = (t // sms) * sms
    rem = t - full
    c_hyb = f32(full // sms) + k * f32(-(-rem // clusters)) if (single_ok and full > 0 and rem > 0) else f32(1e30)
    if c_hyb < c_single and c_hyb < c_pair:
        return 'hybrid'
    return 'pair' if c_pair < c_single else 'single'


def _ln_shape(sched, sms):
    """(B, T) whose tile count t = B * ceil(T/128) puts an N=256 LayerNorm GEMM on the named schedule."""
    if sched == 'single':
        return 3 * sms // 4, 100            # t in (sms/2, sms]
    if sched == 'hybrid':
        return round(1.2 * sms / 8), 1000   # t ~ 1.2 sms: one full wave + a pair tail
    return 3, 300                           # t = 9


@pytest.fixture(scope='module', autouse=True)
def dropout_salt():
    lib.load()
    lib.set_dropout_salt(torch.tensor([np.uint32(SALT).view(np.int32)], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    yield SALT
    lib.set_dropout_salt(torch.zeros(1, dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()


def _report(case, what, err, gate):
    print(f'[gemm-paths] {case}: {what} max rel err {err:.2e} (gate {gate:.0e})')
    assert err < gate, f'{case}: {what} error {err:.3e} >= gate {gate:.1e}'


def _relerr(got, ref):
    got = got.double()
    assert torch.isfinite(got).all(), 'non-finite values in kernel output'
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _inputs(g, B, T, Cs, K, N, *, w_taps=None):
    xs = [torch.randn(B, T, C, generator=g).to(DEV) for C in Cs]
    shape = (K, N) if w_taps is None else (w_taps, K // w_taps, N)
    w = (torch.randn(*shape, generator=g) / K ** 0.5).to(DEV)
    b = (0.5 * torch.randn(N, generator=g)).to(DEV)
    return xs, w, b


def _row_len(g, B, T):
    lens = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = T
    if B > 2:
        lens[1] = 0
    return lens.to(DEV)


def _ln_params(g, N):
    return (1 + 0.1 * torch.randn(N, generator=g)).to(DEV), (0.1 * torch.randn(N, generator=g)).to(DEV)


def _check_layout(case, t, N, n_pad, T, row_len=None, masked=True):
    """t: float view (B,T,ld) of one output.  Everything the contract writes has lost its NaN, padding columns [N, n_pad)
    are zero, columns past the tiles are untouched, rows t >= row_len[b] are zero (masked outputs)."""
    assert not torch.isnan(t[..., :n_pad]).any(), f'{case}: unwritten output elements'
    if n_pad > N:
        assert torch.count_nonzero(t[..., N:n_pad]) == 0, f'{case}: padding columns not zero'
    if t.shape[-1] > n_pad:
        assert torch.isnan(t[..., n_pad:]).all(), f'{case}: wrote past the tile columns'
    if row_len is not None and masked:
        dead = torch.arange(T, device=DEV)[None, :] >= row_len[:, None]
        assert torch.count_nonzero(t[..., :n_pad][dead]) == 0, f'{case}: masked rows not zero'


def _check_mask(case, what, got_kept, keep, decidable, live=None):
    """Dropout mask bit for bit: an element is dropped iff its output is exactly zero (where the undropped value is not ~0)."""
    sel = decidable if live is None else decidable & live
    assert int(sel.sum()) > 0, f'{case}: no element decides the {what} mask'
    bad = int((got_kept != keep)[sel].sum())
    assert bad == 0, f'{case}: {what} dropout mask differs from the restated hash at {bad} elements'


def _live(row_len, B, T):
    return (torch.arange(T, device=DEV)[None, :] < row_len[:, None])[..., None].expand(B, T, 1)


# ----------------------------------------------------------------------------------------------------------
# plain epilogue: staged TMA tile stores (16-bit outputs only, block_n % 64 == 0) and direct stores
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('plane', ['fp16', 'bf16', 'bf16x3_hilo'])
def test_staged_many_tiles_per_cta(plane):
    """B=64, T=1000, K=256, N=768 in three 256-wide tiles: ~12 tiles per persistent CTA, so the staging boxes are reused
    across tiles (one plane alternates two boxes, two planes reuse both every slab)."""
    g = torch.Generator().manual_seed(100)
    B, T, K, N = 64, 1000, 256, 768
    xs, w, b = _inputs(g, B, T, [K], K, N)
    lens = _row_len(g, B, T)
    precision = 'bf16' if plane == 'bf16' else 'bf16x3'
    outputs = ('hi', 'lo') if plane == 'bf16x3_hilo' else ('hi',)
    ld_out = N + 64
    out = run_gemm(xs, w, b, [0], [0], [K], precision=precision, block_n=256, outputs=outputs, out_fp16=plane == 'fp16',
                   ld_out=ld_out, row_len=lens, relu=plane == 'bf16')
    assert _schedule(B, T, N, 256, False, _sms()) == 'single' and out['launches'] == 1
    ref = ref_gemm(xs, w, b, [0], [0], [K], precision=precision, row_len=lens, relu=plane == 'bf16', device=DEV)
    case = f'staged {plane} B={B} T={T} N={N}'
    if plane == 'fp16':
        got = out['hi'].view(torch.float16).float()
        _check_layout(case, got, N, N, T, lens)
        _report(case, 'fp16', _relerr(got[..., :N], ref), GATE_FP16_OUT)
    elif plane == 'bf16':
        got = out['hi'].float()
        _check_layout(case, got, N, N, T, lens)
        _report(case, 'bf16', _relerr(got[..., :N], ref), GATE_BF16_OUT)
    else:
        hi, lo = out['hi'].float(), out['lo'].float()
        _check_layout(case, hi, N, N, T, lens)
        _check_layout(case, lo, N, N, T, lens)
        _report(case, 'hi+lo', _relerr((hi + lo)[..., :N], ref), GATE_X3)


@pytest.mark.parametrize('B,T,shifts', [(1, 1, [0]), (1, 7, [0]), (1, 31, [0]), (1, 33, [0]), (40, 5, [-1, 0, 1])])
@pytest.mark.parametrize('plane', ['fp16', 'bf16x3_hilo'])
def test_staged_short_T(B, T, shifts, plane):
    """T < 32 (the Aligner's one-row decode GEMMs) and a 3-tap conv over 5-row sentences: rows outside [0, T) of a
    sentence read as zero, never as a neighbouring sentence's rows; rows >= T are never stored."""
    g = torch.Generator().manual_seed(101)
    C, N = 128, 256
    K = C * len(shifts)
    xs, w, b = _inputs(g, B, T, [C], K, N, w_taps=len(shifts) if len(shifts) > 1 else None)
    segs = ([0] * len(shifts), shifts, [C] * len(shifts))
    outputs = ('hi', 'lo') if plane == 'bf16x3_hilo' else ('hi',)
    out = run_gemm(xs, w, b, *segs, precision='bf16x3', block_n=256, outputs=outputs, out_fp16=plane == 'fp16')
    assert out['launches'] == 1
    ref = ref_gemm(xs, w, b, *segs, precision='bf16x3', device=DEV)
    case = f'staged short {plane} B={B} T={T} taps={len(shifts)}'
    if plane == 'fp16':
        got = out['hi'].view(torch.float16).float()
        _check_layout(case, got, N, N, T)
        _report(case, 'fp16', _relerr(got, ref), GATE_FP16_OUT)
    else:
        hi, lo = out['hi'].float(), out['lo'].float()
        _check_layout(case, hi, N, N, T)
        _check_layout(case, lo, N, N, T)
        _report(case, 'hi+lo', _relerr(hi + lo, ref), GATE_X3)


@pytest.mark.parametrize('impl', ['tcgen05', 'simt'])
@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('N', [80, 226])
def test_direct_odd_widths_residual(impl, precision, N):
    """Tile widths that are not a multiple of 64 (80; 226 -> 240) take the direct-store epilogue: fp32 + 16-bit outputs,
    fp32 residual, ReLU, row mask, outputs inside wider rows."""
    g = torch.Generator().manual_seed(102)
    B, T, K = 3, 333, 256
    xs, w, b = _inputs(g, B, T, [K], K, N)
    n_pad = -(-N // 16) * 16
    res = torch.randn(B, T, n_pad + 8, generator=g).to(DEV)
    lens = _row_len(g, B, T)
    ld_out = n_pad + 16
    out = run_gemm(xs, w, b, [0], [0], [K], precision=precision, impl=impl, residual=res, relu=True, row_len=lens,
                   ld_out=ld_out)
    assert out['n_pad'] == n_pad and out['launches'] == 1
    ref = ref_gemm(xs, w, b, [0], [0], [K], precision=precision, residual=res, relu=True, row_len=lens, device=DEV)
    case = f'direct {impl} {precision} N={N}'
    _check_layout(case, out['f32'], N, n_pad, T, lens)
    _check_layout(case, out['hi'].float(), N, n_pad, T, lens)
    gate = GATE_X3 if precision == 'bf16x3' else GATE_BF16
    _report(case, 'f32', _relerr(out['f32'][..., :N], ref), gate)
    if precision == 'bf16x3':
        _check_layout(case, out['lo'].float(), N, n_pad, T, lens)
        _report(case, 'hi+lo', _relerr((out['hi'].float() + out['lo'].float())[..., :N], ref), GATE_X3)
    else:
        _report(case, 'bf16', _relerr(out['hi'].float()[..., :N], ref), GATE_BF16_OUT)


# ----------------------------------------------------------------------------------------------------------
# LayerNorm epilogue: single CTA, CTA pair, hybrid
# ----------------------------------------------------------------------------------------------------------
LN_CASES = [('single', 256), ('pair', 256), ('pair', 384), ('pair', 96), ('pair', 160), ('pair', 224), ('hybrid', 256),
            ('single', 226)]


@pytest.mark.parametrize('precision,residual', [('bf16x3', 'pair'), ('bf16x3', 'f32'), ('bf16', 'f32')])
@pytest.mark.parametrize('sched,N', LN_CASES)
def test_layernorm_epilogue(sched, N, precision, residual):
    """Projection + residual + LayerNorm + row mask on each schedule.  The pair cases at 96 / 160 / 224 give each CTA an
    odd number of 16-column chunks; 384 always runs as a pair; 226 (not a multiple of 32) normalises over its logical
    columns on one CTA.  out_preln = acc + bias + residual, on every row (rows >= row_len included).  The bf16 hi/lo
    residual is the activation stream of bf16x3 inference."""
    sms = _sms()
    B, T = _ln_shape(sched, sms) if N == 256 else (3, 300)
    g = torch.Generator().manual_seed(103)
    K = 256
    xs, w, b = _inputs(g, B, T, [K], K, N)
    ln = _ln_params(g, N)
    lens = _row_len(g, B, T)
    n_pad = -(-N // 16) * 16
    kw = dict(ln=ln, row_len=lens)
    if residual == 'pair':
        hi, lo = lib.split_bf16(torch.randn(B, T, n_pad, generator=g).to(DEV), True)
        kw['residual_pair'] = (hi, lo)
    else:
        kw['residual'] = torch.randn(B, T, n_pad, generator=g).to(DEV)
    out = run_gemm(xs, w, b, [0], [0], [K], precision=precision, single_tile=True, out_preln=True, **kw)
    block_n = N if N % 32 == 0 else n_pad
    want_sched = _schedule(B, T, N, block_n, True, sms)
    if N == 256:
        assert want_sched == sched, (want_sched, sched, B, T, sms)
    assert out['launches'] == (2 if want_sched == 'hybrid' else 1), out['launches']
    ref, u_ref = ref_gemm(xs, w, b, [0], [0], [K], precision=precision, device=DEV, return_preln=True, **kw)
    case = f'LN {sched} N={N} {precision} residual={residual} B={B} T={T} launches={out["launches"]}'
    for name in ('f32', 'hi', 'lo'):
        if out[name] is not None:
            _check_layout(case, out[name].float(), N, n_pad, T, lens)
    _check_layout(case, out['preln'], N, n_pad, T, lens, masked=False)
    gate, gate_u = (GATE_X3_LN, GATE_X3) if precision == 'bf16x3' else (GATE_BF16_LN, GATE_BF16)
    _report(case, 'f32', _relerr(out['f32'][..., :N], ref), gate)
    _report(case, 'preln', _relerr(out['preln'][..., :N], u_ref), gate_u)
    if precision == 'bf16x3':
        _report(case, 'hi+lo', _relerr((out['hi'].float() + out['lo'].float())[..., :N], ref), GATE_X3_LN)
    if sched == 'single' and residual == 'f32':
        # the SIMT bring-up kernel, same contract (no pair residual)
        out_s = run_gemm(xs, w, b, [0], [0], [K], precision=precision, impl='simt', single_tile=True, out_preln=True, **kw)
        for name in ('f32', 'hi'):
            _check_layout(case + ' simt', out_s[name].float(), N, n_pad, T, lens)
        _report(case + ' simt', 'f32', _relerr(out_s['f32'][..., :N], ref), gate)
        _report(case + ' simt', 'preln', _relerr(out_s['preln'][..., :N], u_ref), gate_u)


# ----------------------------------------------------------------------------------------------------------
# sources inside wider buffers, three and four segments over two sources
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('path', ['direct', 'staged', 'ln_pair', 'simt'])
@pytest.mark.parametrize('nseg', [3, 4])
@pytest.mark.parametrize('a_col0', [8, 64])
def test_wide_sources_multi_segment(path, nseg, a_col0):
    """Each source sits at column a_col0 of a buffer with lda = C + 64 columns, the other columns hold 3e4: a wrong offset
    or stride is far off the reference.  Segments mix both sources and time shifts."""
    g = torch.Generator().manual_seed(104)
    B, T, C, N = 3, 200, 128, 256
    if nseg == 3:
        segs = ([0, 0, 1], [-1, 0, 1], [128, 128, 64])
    else:
        segs = ([0, 1, 0, 1], [-1, -1, 1, 0], [128, 64, 128, 128])
    K = sum(segs[2])
    xs, w, b = _inputs(g, B, T, [C, C], K, N)
    kw = dict(lda=[C + 64, C + 64], a_col0=[a_col0, 64 - a_col0])
    epi = {}
    if path == 'ln_pair':
        epi = dict(ln=_ln_params(g, N))
    lens = _row_len(g, B, T)
    epi['row_len'] = lens
    impl = 'simt' if path == 'simt' else 'tcgen05'
    outputs = ('hi', 'lo') if path == 'staged' else ('f32',)
    out = run_gemm(xs, w, b, *segs, precision='bf16x3', impl=impl, outputs=outputs, single_tile=path == 'ln_pair', **kw, **epi)
    ref = ref_gemm(xs, w, b, *segs, precision='bf16x3', device=DEV, **epi)
    case = f'wide sources {path} a_col0={a_col0} segments={nseg}'
    if path == 'ln_pair':
        assert _schedule(B, T, N, N, True, _sms()) == 'pair'
    if path == 'staged':
        got = out['hi'].float() + out['lo'].float()
    else:
        got = out['f32']
    _check_layout(case, got, N, N, T, lens)
    _report(case, 'out', _relerr(got, ref), GATE_X3_LN if path == 'ln_pair' else GATE_X3)


# ----------------------------------------------------------------------------------------------------------
# dropout
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('path', ['direct', 'staged'])
def test_dropout_plain(path):
    """drop_pre on the plain epilogue: the mask, drawn at (b*T + t)*ld_out + n with ld_out wider than the tiles, is the
    restated hash bit for bit; kept values are x / (1-p)."""
    g = torch.Generator().manual_seed(105)
    B, T, K, N, p, site = 8, 300, 256, 512, 0.3, 7
    xs, w, b = _inputs(g, B, T, [K], K, N)
    lens = _row_len(g, B, T)
    ld_out = N + 32
    precision = 'bf16' if path == 'staged' else 'bf16x3'
    outputs = ('hi',) if path == 'staged' else ('f32',)
    out = run_gemm(xs, w, b, [0], [0], [K], precision=precision, block_n=256, outputs=outputs, ld_out=ld_out, row_len=lens,
                   dropout=(p, site), seed=SEED)
    assert out['launches'] == 1
    ref = ref_gemm(xs, w, b, [0], [0], [K], precision=precision, row_len=lens, dropout=(p, site), seed=SEED, salt=SALT,
                   ld_out=ld_out, device=DEV)
    undropped = ref_gemm(xs, w, b, [0], [0], [K], precision=precision, device=DEV)
    got = out['hi'].float() if path == 'staged' else out['f32']
    case = f'dropout {path} p={p}'
    _check_layout(case, got, N, N, T, lens)
    keep = torch.from_numpy(dropout_mask(B, T, N, ld_out, SEED, site, p, SALT)).to(DEV)
    decidable = undropped.abs() > 1e-3 * undropped.abs().max()
    _check_mask(case, 'pre', got[..., :N] != 0, keep, decidable, _live(lens, B, T))
    _report(case, 'out', _relerr(got[..., :N], ref), GATE_BF16_OUT if path == 'staged' else GATE_X3)


@pytest.mark.parametrize('sched,N', [('single', 256), ('pair', 256), ('hybrid', 256), ('pair', 384), ('pair', 160)])
def test_dropout_layernorm_forward_backward(sched, N):
    """drop_pre + drop_post on the LayerNorm epilogue, then ttsb_layernorm_bwd from the saved pre-norm value with the same
    sites and seed: both kernels draw the masks the numpy restatement draws (the pair CTA of rank 1 at its column offset),
    and du, dgamma, dbeta and the bf16 GEMM gradient g match float64 autograd through the restated masks."""
    sms = _sms()
    B, T = _ln_shape(sched, sms) if N == 256 else (3, 300)
    g = torch.Generator().manual_seed(106)
    K, p_pre, p_post, s_pre, s_post = 256, 0.2, 0.1, 11, 12
    xs, w, b = _inputs(g, B, T, [K], K, N)
    gamma, beta = _ln_params(g, N)
    lens = _row_len(g, B, T)
    res = torch.randn(B, T, N, generator=g).to(DEV)
    kw = dict(ln=(gamma, beta), row_len=lens, residual=res, dropout=(p_pre, s_pre), dropout_post=(p_post, s_post), seed=SEED)
    out = run_gemm(xs, w, b, [0], [0], [K], precision='bf16x3', single_tile=True, out_preln=True, **kw)
    want_sched = _schedule(B, T, N, N, True, sms)
    assert want_sched == sched, (want_sched, sched)
    assert out['launches'] == (2 if sched == 'hybrid' else 1)
    ref, u_ref = ref_gemm(xs, w, b, [0], [0], [K], precision='bf16x3', salt=SALT, ld_out=N, device=DEV, return_preln=True, **kw)
    case = f'dropout LN {sched} N={N} B={B} T={T} launches={out["launches"]}'
    for name in ('f32', 'hi', 'lo'):
        _check_layout(case, out[name].float(), N, N, T, lens)
    _check_layout(case, out['preln'], N, N, T, lens, masked=False)
    live = _live(lens, B, T)
    keep_pre = torch.from_numpy(dropout_mask(B, T, N, N, SEED, s_pre, p_pre, SALT)).to(DEV)
    keep_post = torch.from_numpy(dropout_mask(B, T, N, N, SEED, s_post, p_post, SALT)).to(DEV)
    acc = ref_gemm(xs, w, b, [0], [0], [K], precision='bf16x3', device=DEV)
    _check_mask(case, 'pre', (out['preln'] - res) != 0, keep_pre, acc.abs() > 1e-3 * acc.abs().max())
    post_in = ref_gemm(xs, w, b, [0], [0], [K], precision='bf16x3', salt=SALT, ld_out=N, device=DEV,
                       **{k: v for k, v in kw.items() if k not in ('dropout_post', 'row_len')})
    _check_mask(case, 'post', out['f32'] != 0, keep_post, post_in.abs() > 1e-3 * post_in.abs().max(), live)
    _report(case, 'f32', _relerr(out['f32'], ref), GATE_X3_LN)
    _report(case, 'preln', _relerr(out['preln'], u_ref), GATE_X3)

    # backward from the kernel's own pre-norm value
    dz = torch.randn(B, T, N, generator=g).to(DEV)
    du = torch.full((B, T, N), float('nan'), device=DEV)
    gb = torch.full((B, T, N), float('nan'), device=DEV, dtype=torch.bfloat16)
    dgamma, dbeta = torch.zeros(N, device=DEV), torch.zeros(N, device=DEV)
    lib.layernorm_bwd(dz, out['preln'].contiguous(), gamma, B, T, N, N, 1e-6, lens, False, du, gb, dgamma, dbeta,
                      pre_drop=(p_pre, s_pre), post_drop=(p_post, s_post), seed=SEED)
    torch.cuda.synchronize()
    u = out['preln'].double().requires_grad_()
    g64, b64 = gamma.double().requires_grad_(), beta.double().requires_grad_()
    mean = u.mean(-1, keepdim=True)
    var = ((u - mean) ** 2).mean(-1, keepdim=True)
    z = ((u - mean) * torch.rsqrt(var + 1e-6) * g64 + b64) * keep_post * dropout_scale(p_post) * live
    (z * dz.double()).sum().backward()
    g_ref = u.grad * keep_pre * dropout_scale(p_pre)
    _report(case, 'bwd du', _relerr(du, u.grad), GATE_BWD)
    _report(case, 'bwd g bf16', _relerr(gb.float(), g_ref), GATE_BF16_OUT)
    _report(case, 'bwd dgamma', _relerr(dgamma, g64.grad), GATE_BWD)
    _report(case, 'bwd dbeta', _relerr(dbeta, b64.grad), GATE_BWD)
    # the bf16 gradient is zero exactly where the pre-LayerNorm dropout dropped
    _check_mask(case, 'bwd pre', gb.float() != 0, keep_pre, u.grad.abs() > 1e-3 * u.grad.abs().max(), live)


# ----------------------------------------------------------------------------------------------------------
# the stand-alone LayerNorm row kernel and the bf16 hi/lo split
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d,ld', [(384, 384), (512, 512), (100, 112)])
def test_layernorm_fwd_rows(d, ld):
    """ttsb_layernorm_fwd: rows whose mean (1e3) dwarfs their spread (1e-1) next to ordinary rows, row_len 0 included;
    fp32 and hi + lo against float64, masked rows exactly zero."""
    g = torch.Generator().manual_seed(107)
    B, T = 4, 50
    x = torch.randn(B, T, ld, generator=g)
    x[:, ::2] = 1e3 + 0.1 * torch.randn(B, (T + 1) // 2, ld, generator=g)
    x = x.to(DEV)
    gamma, beta = _ln_params(g, d)
    lens = torch.tensor([T, 0, 17, 1], dtype=torch.int32, device=DEV)
    out = torch.full((B, T, ld), float('nan'), device=DEV)
    hi = torch.full((B, T, ld), float('nan'), device=DEV, dtype=torch.bfloat16)
    lo = torch.full((B, T, ld), float('nan'), device=DEV, dtype=torch.bfloat16)
    lib.layernorm_fwd(x, gamma, beta, d, 1e-6, lens, out, hi, lo)
    torch.cuda.synchronize()
    xd = x[..., :d].double()
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    ref = ((xd - mean) * torch.rsqrt(var + 1e-6) * gamma.double() + beta.double()) * _live(lens, B, T)
    case = f'layernorm_fwd d={d} ld={ld}'
    for t in (out, hi.float(), lo.float()):
        _check_layout(case, t[..., :d], d, d, T, lens)
    # ordinary rows (odd t): fp32 arithmetic (measured 1.3e-7), hi + lo carries 16 significant bits (5.3e-6).  The kernel
    # holds the row mean in fp32: on the rows with mean 1e3 and spread 1e-1 (even t) its rounding alone, ulp(1e3)/2 = 3e-5,
    # is 3e-4 of the spread, so they get their own gate (measured 2.6e-4)
    odd, even = slice(1, None, 2), slice(0, None, 2)
    hilo = hi.float() + lo.float()
    _report(case, 'f32 ordinary rows', _relerr(out[:, odd, :d], ref[:, odd]), 1e-6)
    _report(case, 'hi+lo ordinary rows', _relerr(hilo[:, odd, :d], ref[:, odd]), GATE_X3_LN)
    _report(case, 'f32 mean 1e3, std 1e-1 rows', _relerr(out[:, even, :d], ref[:, even]), 1e-3)
    _report(case, 'hi+lo mean 1e3, std 1e-1 rows', _relerr(hilo[:, even, :d], ref[:, even]), 1e-3)


def test_split_bf16_bit_exact():
    """hi = round-to-nearest-even bf16 of x and lo = bf16(x - hi), bit for bit, on subnormals, signed zeros, values at the
    bf16 overflow edge and an odd element count."""
    g = torch.Generator().manual_seed(108)
    bf16_max = float(torch.finfo(torch.bfloat16).max)
    special = torch.tensor([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, 1.1754942e-38, 9.2e-41, 1.0, -1.0, 1 + 2 ** -8,
                            1 + 3 * 2 ** -9, bf16_max, -bf16_max, 3.3961e38, 3.3962e38, 3.4028235e38, -3.4028235e38,
                            np.nextafter(np.float32(3.3961776e38), np.float32(0)).item(), 65504.0, 2 ** -126, 2 ** -133],
                           dtype=torch.float32)
    rnd = torch.randn(100_001, generator=g) * torch.exp2(torch.randint(-140, 120, (100_001,), generator=g).float())
    x = torch.cat([special, rnd])
    assert x.numel() % 2 == 1
    hi, lo = lib.split_bf16(x.to(DEV), True)
    torch.cuda.synchronize()
    want_hi = x.bfloat16()
    want_lo = (x - want_hi.float()).bfloat16()
    assert torch.equal(hi.cpu().view(torch.int16), want_hi.view(torch.int16))
    assert torch.equal(lo.cpu().view(torch.int16), want_lo.view(torch.int16))
