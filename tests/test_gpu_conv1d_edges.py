"""The ragged Conv1D kernels (csrc/conv1d_tc.cu) against float64 at every tile width, tile edge, halo mode and epilogue.

Contract under test (include/ttsb.h).  ttsb_conv1d_ex_tc computes, for every clip row t,
    y[c, t, :] = bias + sum_s in_{src_s}[c, t + shift_s, :] @ W_s  (+ residual, then the multi-receptive-field sum step)
and writes column n of y[c, t] to output row t up + n // ld_out, channel n % ld_out, as bf16 hi (+ lo) planes of y and of
LeakyReLU_slope(y); it mirrors (REFLECT) or zeroes (ZERO) the output halo rows, or leaves them alone (NONE).
ttsb_conv1d_out_tanh_ex is the generators' N = 1 output layer.  The reference (_formula) states the header formula in float64
on the exact 16-bit planes the kernel reads, with a random (K_total, N) matrix rather than conv weights; the one CPU test
ties it to F.conv1d / F.conv_transpose1d through melgan.conv_taps / transposed_taps.

Poison.  Every input row is random, halo rows included, so a tap that reads the wrong row reads a different value.  bf16
calls pass NaN in_lo planes (never read) and poisoned out_lo / act_lo planes (never written).  The residual's and the sum's
halo rows are NaN, every output plane and the sum carry EXTRA poisoned rows past out_rows, and planes start as all-ones bit
patterns: what the contract does not write keeps those bits.

Error model.  bf16 operands are exact in float64 and their products exact in fp32.  The kernel accumulates one fp32 sum per
k16 wgmma step (three products per k step in bf16x3: hi hi + lo hi + hi lo, dropping lo lo), then adds bias, residual and sum
and scales by the slope or 1 / sum_div, each one fp32 rounding.  The reference sums exactly those products (so the dropped
lo lo term needs no allowance), and an element of y is off by at most one fp32 unit (2^-23 when a step truncates) per step,
relative to sum |terms|: steps = products K_total / 16 + 6.  It is gated on
    (|err| - output rounding) / (2^-24 steps sum |terms|) <= GATE_ACC,
with the output rounding 2^-8 |y| for hi alone and 2^-8 |lo| (at most 2^-16 |y|) for hi + lo.
A term read from a wrong row or column moves an element by about sum |terms| / K_total, at least 16 / (K_total^2 2^-24)
gate units: 16 at the largest K_total here (4096), thousands at the usual ones.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import DEV, _poison16
from transformertts_b200 import lib
from transformertts_b200.model import melgan as mg

gpu = pytest.mark.gpu

U24 = 2.0 ** -24   # fp32 unit roundoff
BF16_U = 2.0 ** -8   # largest relative error of one rounding to bf16
EXTRA = 5            # poisoned rows past out_rows in every output plane and the sum
NONE, REFLECT, ZERO = lib.HALO_NONE, lib.HALO_REFLECT, lib.HALO_ZERO

# Measured on an H100 80GB HBM3 (SXM, 700 W power limit): in brackets the largest error of any case under each gate.
GATE_ACC = 4.0   # conv1d_ex y, act and sum, in units of 2^-24 steps sum |terms|; the model's bound is 2 (bf16x3 y / act 0.32,
                 # sum 0.17; bf16 y / act 0.031, sum 0.11)
GATE_TANH = 1.0  # out_tanh, (|err| - 4 ulp of tanh) / (2^-24 7 channels (|bias| + sum |terms|)): an fmaf chain (0.026)


class Layout:
    """The packed ragged layout of include/ttsb.h: clip c has counts[c] rows, framed by `halo` rows on each side, in the
    input layout, and up counts[c] rows in the output layout."""

    def __init__(self, counts, halo, up=1):
        self.counts = [int(L) for L in counts]
        n = len(self.counts)
        self.n, self.H, self.up = n, halo, up
        self.off = np.concatenate([[0], np.cumsum(self.counts)]).astype(np.int64)
        self.rows_in = int(self.off[-1]) + 2 * halo * n
        self.rows_out = int(self.off[-1]) * up + 2 * halo * n
        self.in_start = self.off[:-1] + (2 * np.arange(n) + 1) * halo      # input row of clip row 0
        self.out_start = self.off[:-1] * up + (2 * np.arange(n) + 1) * halo
        self.in_rows = np.concatenate([s + np.arange(L) for s, L in zip(self.in_start, self.counts)])
        self.out_rows = np.concatenate([s + np.arange(L * up) for s, L in zip(self.out_start, self.counts)])

    def halo_rows(self, mode):
        """(every output halo row, the output row a REFLECT halo copies): row -k copies row k, row Lo - 1 + k row Lo - 1 - k."""
        rows, src = [], []
        for s, L in zip(self.out_start, self.counts):
            Lo = L * self.up
            i = np.concatenate([np.arange(-self.H, 0), np.arange(Lo, Lo + self.H)])
            rows.append(s + i)
            src.append(s + np.where(i < 0, -i, 2 * (Lo - 1) - i) if mode == REFLECT else np.full(len(i), -1))
        return np.concatenate(rows).astype(np.int64), np.concatenate(src).astype(np.int64)


def _formula(xs, taps, w, lay, ld_out, bias=None):
    """float64 y = bias + sum_s xs[src_s][t + shift_s] @ w[koff_s : koff_s + ld_in[src_s]] for every clip row t, as output
    rows (len(lay.out_rows), ld_out) in lay.out_rows order: column n of row t is channel n % ld_out of row t up + n // ld_out."""
    rows = torch.as_tensor(lay.in_rows, device=w.device)
    y = torch.zeros(len(rows), w.shape[1], dtype=torch.float64, device=w.device)
    koff = 0
    for src, sh in taps:
        ld = xs[src].shape[1]
        y += xs[src][rows + sh] @ w[koff:koff + ld]
        koff += ld
    assert koff == w.shape[0]
    if bias is not None:
        y += bias
    return y.reshape(-1, ld_out)


def test_reference_formula_matches_torch_convs():
    """The header formula over melgan.pack_clips' layout, with melgan.conv_taps / transposed_taps as W, is F.conv1d with
    reflect padding and F.conv_transpose1d (CPU, no GPU needed)."""
    g = torch.Generator().manual_seed(1)
    counts = [4, 11, 1, 30]
    for k, d in ((3, 3), (7, 1), (3, 9)):
        cin, cout, H = 20, 24, d * (k - 1) // 2
        w, b = torch.randn(cout, cin, k, generator=g, dtype=torch.float64), torch.randn(cout, generator=g, dtype=torch.float64)
        clips = [torch.randn(max(L, H + 1), cin, generator=g, dtype=torch.float64) for L in counts]
        lay = Layout([len(x) for x in clips], H)
        buf = torch.from_numpy(mg.pack_clips([x.numpy() for x in clips], 64, REFLECT, halo=H)).double()
        mat = torch.from_numpy(mg.conv_taps(w.numpy(), d, 64, 64))
        bias = torch.zeros(64, dtype=torch.float64)
        bias[:cout] = b
        y = _formula([buf], [(0, (s - (k - 1) // 2) * d) for s in range(k)], mat, lay, 64, bias)
        for c, x in enumerate(clips):
            x32 = x.float().double()        # pack_clips stores float32
            want = F.conv1d(F.pad(x32.T[None], (H, H), mode='reflect'), w, b, dilation=d)[0].T
            got = y[lay.off[c]:lay.off[c + 1], :cout]
            assert (got - want).abs().max().item() < 1e-12, (k, d, c)
    for u in (2, 4, 8):
        cin, cout, cc = 20, 12, 16
        w, b = torch.randn(cin, cout, 2 * u, generator=g, dtype=torch.float64), torch.randn(cout, generator=g, dtype=torch.float64)
        clips = [torch.randn(L, cin, generator=g, dtype=torch.float64) for L in counts]
        lay = Layout(counts, 1, up=u)
        buf = torch.from_numpy(mg.pack_clips([x.numpy() for x in clips], 64, ZERO, halo=1)).double()
        mat = torch.from_numpy(mg.transposed_taps(w.numpy(), u, 64, cc))
        bias = torch.zeros(u * cc, dtype=torch.float64)
        for r in range(u):
            bias[r * cc:r * cc + cout] = b
        y = _formula([buf], [(0, -1), (0, 0), (0, 1)], mat, lay, cc, bias)
        for c, x in enumerate(clips):
            want = F.conv_transpose1d(x.float().double().T[None], w, b, stride=u, padding=u // 2)[0].T
            got = y[lay.off[c] * u:lay.off[c + 1] * u, :cout]
            assert got.shape == want.shape and (got - want).abs().max().item() < 1e-12, (u, c)


# ---------------------------------------------------------------------------------------------------- helpers on the GPU
def _randn(shape, gen, scale=1.0):
    return (torch.randn(shape, generator=gen) * scale).to(DEV)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _poison32(shape):
    t = torch.empty(shape, device=DEV, dtype=torch.float32)
    t.view(torch.int32).fill_(-1)
    return t


def _val(hi, lo):
    return hi.double() + (lo.double() if lo is not None else 0.0)


class Conv:
    """One ttsb_conv1d_ex_tc problem: random sources over every row of the layout (halos included), a random (K_total, N)
    matrix and bias, a residual with NaN halo rows; the value and sum |terms| of each output row, from _formula."""

    def __init__(self, prec, lay, taps, ld_in, ld_out, *, seed, bias=True, res=True, xs=None):
        self.split = prec == 'bf16x3'
        self.lay, self.taps, self.ld_out, self.N = lay, taps, ld_out, lay.up * ld_out
        g = torch.Generator().manual_seed(seed)
        self.srcs = xs if xs is not None else [self.source(lay.rows_in, ld, g) for ld in ld_in]
        k_total = sum(self.srcs[s][0].shape[1] for s, _ in taps)
        w = _randn((k_total, self.N), g, k_total ** -0.5)
        self.w_hi, self.w_lo = lib.pack_weight(w, self.N, self.split)
        self.bias = _randn(self.N, g, 0.5) if bias else None
        b64 = self.bias.double() if bias else None
        self.res = None
        if res:
            r = _randn((lay.rows_out + EXTRA, ld_out), g)
            keep = torch.zeros(lay.rows_out + EXTRA, dtype=torch.bool, device=DEV)
            keep[torch.as_tensor(lay.out_rows, device=DEV)] = True
            r[~keep] = float('nan')         # only clip rows of the residual are read
            self.res = lib.split_bf16(r, self.split)
        # the products the kernel issues: hi hi in bf16; hi hi + lo hi + hi lo in bf16x3 (lo lo is dropped)
        his = [hi.double() for hi, _ in self.srcs]
        prods = [(his, self.w_hi.double().T)]
        if self.split:
            prods += [([lo.double() for _, lo in self.srcs], self.w_hi.double().T), (his, self.w_lo.double().T)]
        self.y = sum(_formula(x, taps, w, lay, ld_out, b64 if i == 0 else None) for i, (x, w) in enumerate(prods))
        self.den = sum(_formula([v.abs() for v in x], taps, w.abs(), lay, ld_out, b64.abs() if bias and i == 0 else None)
                       for i, (x, w) in enumerate(prods))
        if res:
            idx = torch.as_tensor(lay.out_rows, device=DEV)
            rv = _val(self.res[0][idx], self.res[1][idx] if self.split else None)
            self.y, self.den = self.y + rv, self.den + rv.abs()
        self.steps = (3 if self.split else 1) * k_total // 16 + 6

    def source(self, rows, ld, g):
        hi, lo = lib.split_bf16(_randn((rows, ld), g), self.split)
        return hi, (lo if self.split else _poison16((rows, ld)))   # bf16: a NaN lo plane the kernel must not read

    def planes(self):
        """Poisoned (hi, lo) output planes with EXTRA rows past out_rows; bf16 passes lo planes too (never written)."""
        return _poison16((self.lay.rows_out + EXTRA, self.ld_out)), _poison16((self.lay.rows_out + EXTRA, self.ld_out))

    def run(self, *, out=None, act=None, mode=NONE, slope=0.2, sum_plane=None, sum_mode=lib.SUM_NONE, sum_div=1.0):
        lay = self.lay
        a = lib.Conv1dExArgs()
        tab = (C.c_int32 * (lay.n + 1))(*lay.off.tolist())
        a.n_clips, a.clip_offsets, a.halo, a.num_taps = lay.n, C.cast(tab, C.c_void_p), lay.H, len(self.taps)
        for s, (src, sh) in enumerate(self.taps):
            a.tap_src[s], a.tap_shift[s] = src, sh
        for i, (hi, lo) in enumerate(self.srcs):
            a.in_hi[i], a.in_lo[i], a.ld_in[i] = hi.data_ptr(), lo.data_ptr(), hi.shape[1]
        a.w_hi, a.w_lo, a.bias = lib.ptr(self.w_hi), lib.ptr(self.w_lo), lib.ptr(self.bias)
        a.N, a.up, a.ld_out, a.out_rows = self.N, lay.up, self.ld_out, lay.rows_out
        if self.res is not None:
            a.res_hi, a.res_lo = lib.ptr(self.res[0]), lib.ptr(self.res[1])
        if out is not None:
            a.out_hi, a.out_lo = lib.ptr(out[0]), lib.ptr(out[1])
        if act is not None:
            a.act_hi, a.act_lo = lib.ptr(act[0]), lib.ptr(act[1])
        a.sum, a.sum_mode, a.sum_div = lib.ptr(sum_plane), sum_mode, sum_div
        a.slope, a.halo_mode = slope, mode
        a.precision = lib.PREC_BF16X3 if self.split else lib.PREC_BF16
        ws = torch.empty(lib.conv1d_workspace_bytes(lay.n), dtype=torch.uint8, device=DEV)
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        lib.conv1d_ex_tc(a)
        torch.cuda.synchronize()

    # ------------------------------------------------------------------------------------------------ checks
    def err(self, case, got, want, den, rounding):
        """max over the clip rows of (|got - want| - rounding) / (2^-24 steps den), in gate units."""
        assert torch.isfinite(got).all(), f'{case}: non-finite values in clip rows'
        e = ((got - want).abs() - rounding).clamp_min(0.0) / (U24 * self.steps * den)
        return float(e.max())

    def check_planes(self, case, name, planes, want, den, mode, lo_given=True):
        """One (hi, lo) output: clip rows against want, halos by mode, poison past out_rows, bf16's lo plane untouched."""
        lay, hi, lo = self.lay, planes[0], planes[1]
        written = [hi, lo] if self.split and lo_given else [hi]
        idx = torch.as_tensor(lay.out_rows, device=DEV)
        got = _val(hi[idx], lo[idx] if len(written) == 2 else None)
        # one rounding to bf16 of y, or of y - hi to lo: at most 2^-8 of the value rounded (2^-8 |lo| <= 2^-16 |y|)
        rounding = BF16_U * (lo[idx].double().abs() if len(written) == 2 else want.abs())
        e = self.err(f'{case} {name}', got, want, den, rounding)
        rows, src = (torch.as_tensor(v, device=DEV) for v in lay.halo_rows(mode))
        for p in written:
            b = _bits(p)
            assert (b[lay.rows_out:] == -1).all(), f'{case} {name}: a row past out_rows was written'
            if mode == NONE:
                assert (b[rows] == -1).all(), f'{case} {name}: a NONE halo row was written'
            elif mode == ZERO:
                assert (b[rows] == 0).all(), f'{case} {name}: a ZERO halo row is not +0'
            else:
                assert torch.equal(b[rows], b[src]), f'{case} {name}: a REFLECT halo row is not a bit copy of its source row'
        if lo is not None and len(written) == 1:
            assert (_bits(lo) == -1).all(), f'{case} {name}: a lo plane the call does not use was written'
        return e

    def check_sum(self, case, sum_plane, want, den):
        lay = self.lay
        idx = torch.as_tensor(lay.out_rows, device=DEV)
        e = self.err(f'{case} sum', sum_plane[idx].double(), want, den, 0.0)
        rows, _ = lay.halo_rows(NONE)
        b = _bits(sum_plane)
        assert (b[torch.as_tensor(rows, device=DEV)] == -1).all(), f'{case}: a halo row of the sum was written'
        assert (b[lay.rows_out:] == -1).all(), f'{case}: a sum row past out_rows was written'
        return e

    def sum_plane(self, init=True, seed=5):
        """fp32 sum plane, all-ones bits; clip rows random (what ADD / FINISH read) when init."""
        s = _poison32((self.lay.rows_out + EXTRA, self.ld_out))
        if init:
            g = torch.Generator().manual_seed(seed)
            s[torch.as_tensor(self.lay.out_rows, device=DEV)] = _randn((len(self.lay.out_rows), self.ld_out), g)
        return s


def _lrelu(y, slope):
    return torch.where(y > 0, y, slope * y)


def _report(case, what, err, gate=GATE_ACC):
    print(f'[conv1d-edges] {case}: {what} err {err:.3f} (gate {gate})')
    assert err <= gate, f'{case}: {what} error {err:.3f} > gate {gate}'


def _plain(prec, lay, taps, ld_in, ld_out, *, mode=NONE, seed=0, slope=0.2, bias=True, res=True, case=''):
    """Run one conv writing out and act, check every plane; returns the Conv and its planes."""
    cv = Conv(prec, lay, taps, ld_in, ld_out, seed=seed, bias=bias, res=res)
    out, act = cv.planes(), cv.planes()
    cv.run(out=out, act=act, mode=mode, slope=slope)
    case = f'{prec} {case}'
    _report(case, 'out', cv.check_planes(case, 'out', out, cv.y, cv.den, mode))
    _report(case, 'act', cv.check_planes(case, 'act', act, _lrelu(cv.y, slope), cv.den, mode))
    return cv, out, act


PRECS = ['bf16', 'bf16x3']


# ---------------------------------------------------------------------------------------------------- tile widths and phases
@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('up,ld_out,N', [(1, 64, 64), (1, 128, 128), (1, 192, 192), (1, 256, 256), (1, 512, 512),
                                         (2, 32, 64), (4, 16, 64), (4, 48, 192), (16, 16, 256), (3, 256, 768), (8, 256, 2048)])
def test_tile_widths_and_phases(prec, up, ld_out, N):
    """Every wgmma width (64 .. 256 and the n-tiled 512 .. 2048), output widths that change phase inside a 64-column tile,
    odd up; clips straddle the 128-row tiles, REFLECT halos."""
    assert N == up * ld_out
    lay = Layout([3, 5, 130, 61, 3, 200], 2, up)
    _plain(prec, lay, [(0, -2), (0, 0), (0, 1)], [128 if N <= 256 else 64], ld_out, mode=REFLECT, seed=N + up,
           case=f'up={up} ld_out={ld_out} N={N}')


# ---------------------------------------------------------------------------------------------------- taps and sources
TAP_CASES = {
    '16 taps over [-64, 64]': ([1, 70, 200, 5], 64, [(0, int(s)) for s in np.linspace(-64, 64, 16).round()], [64], 64, NONE),
    'halo 0, one tap': ([1, 1, 50, 300, 2], 0, [(0, 0)], [64], 128, NONE),
    'two sources 64 / 192, order 1 0 1 0': ([3, 100, 150], 2, [(1, -2), (0, 0), (1, 1), (0, 2)], [64, 192], 256, REFLECT),
    'K_total 16 x 256': ([9, 120, 130], 8, [(0, s) for s in range(-8, 8)], [256], 64, ZERO),
}


@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('name', list(TAP_CASES))
def test_taps_and_sources(prec, name):
    counts, H, taps, ld_in, N, mode = TAP_CASES[name]
    if name.startswith('16 taps'):
        assert len(taps) == 16 and taps[0][1] == -64 and taps[-1][1] == 64
    _plain(prec, Layout(counts, H), taps, ld_in, N, mode=mode, seed=len(name), case=name)


# ---------------------------------------------------------------------------------------------------- clip layouts
def _edge_layouts():
    """Clip starts and ends at rows 127, 128 and 129 of the packed input layout (halo 2)."""
    H, out = 2, {}
    for r in (127, 128, 129):
        out[f'clip 0 ends at row {r}'] = [r - H + 1, 4, 60]
        out[f'clip 1 starts at row {r}'] = [r - 3 * H, 4, 60]
    return out


def _many_tiles_counts():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    need = 3 * sms * 128 // 2 + 128          # n_tiles = 2: 3 SMs' worth of tiles and more
    g = np.random.default_rng(9)
    counts = []
    while sum(counts) + 6 * len(counts) < need:
        counts.append(int(g.integers(4, 400)))
    return counts


LAYOUT_CASES = ['single clip of length 1', 'edges at 127 / 128 / 129', '300 clips of length 1 at halo 0',
                'length-1 clips at halo 64', 'every CTA runs several tiles']


@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('name', LAYOUT_CASES)
def test_clip_layouts(prec, name):
    if name == 'single clip of length 1':
        _plain(prec, Layout([1], 1), [(0, -1), (0, 0), (0, 1)], [64], 64, case=name)
    elif name == 'edges at 127 / 128 / 129':
        for what, counts in _edge_layouts().items():
            lay = Layout(counts, 2)
            starts = lay.in_start.tolist() + (lay.in_start + np.asarray(counts) - 1).tolist()
            assert any(s in (127, 128, 129) for s in starts)
            _plain(prec, lay, [(0, -2), (0, 0), (0, 2)], [64], 128, mode=ZERO, seed=counts[0], case=f'{name}: {what}')
    elif name == '300 clips of length 1 at halo 0':
        _plain(prec, Layout([1] * 300, 0), [(0, 0)], [128], 64, case=name)       # a tile holds 128 clips
    elif name == 'length-1 clips at halo 64':
        _plain(prec, Layout([1] * 5, 64), [(0, -64), (0, 0), (0, 64)], [64], 64, case=name)   # tiles of halo rows only
    else:
        counts = _many_tiles_counts()
        lay = Layout(counts, 3)
        tiles = -(-lay.rows_in // 128) * 2
        assert tiles >= 3 * torch.cuda.get_device_properties(0).multi_processor_count
        _plain(prec, lay, [(0, -3), (0, 0), (0, 3)], [64], 512, mode=REFLECT, case=f'{name} ({tiles} tiles)')


# ---------------------------------------------------------------------------------------------------- halo modes
def _min_layout(mode, up):
    """Each mode's shortest legal clips: REFLECT up L = halo + 1, ZERO up L = halo, NONE L = 1 (halo 7 or 8)."""
    H = 8 if mode == ZERO else 7
    L = {NONE: 1, REFLECT: (H + 1) // up, ZERO: H // up}[mode]
    assert (mode == NONE) or up * L == (H + 1 if mode == REFLECT else H)
    return Layout([L, L, 37, L, 5 * L], H, up)


@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('up', [1, 4, 8])
@pytest.mark.parametrize('mode', [NONE, REFLECT, ZERO], ids=['none', 'reflect', 'zero'])
@pytest.mark.parametrize('halo', ['min length', 'halo 0'])
def test_halo_modes(prec, up, mode, halo):
    """Mirrored rows are bit copies in all four planes, ZERO rows +0, NONE halos keep their poison (check_planes)."""
    ld_out = {1: 64, 4: 16, 8: 32}[up]
    if halo == 'halo 0':
        lay, taps = Layout([1, 1, 37, 1, 5], 0, up), [(0, 0)]
    else:
        lay = _min_layout(mode, up)
        taps = [(0, -lay.H), (0, 0), (0, lay.H)]
    _plain(prec, lay, taps, [64], ld_out, mode=mode, seed=10 * up + mode, case=f'mode={mode} up={up} {halo} {lay.counts}')


# ---------------------------------------------------------------------------------------------------- epilogue
@gpu
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('slope', [0.0, 0.2, 1.0])
def test_slopes_and_no_bias(prec, slope):
    lay = Layout([4, 150, 9], 3, 2)
    _plain(prec, lay, [(0, -3), (0, 1)], [64], 64, mode=REFLECT, slope=slope, bias=slope != 0.2, res=slope != 1.0,
           case=f'slope {slope} bias={slope != 0.2} residual={slope != 1.0}')


@gpu
@pytest.mark.parametrize('prec', PRECS)
def test_sum_chain(prec):
    """WRITE -> ADD -> ADD -> FINISH (sum_div 4) over one sum plane: out NULL throughout, act only on FINISH, which leaves the
    sum alone; the sum's halo rows and rows past out_rows are never written.  Each step's reference starts from the sum
    the previous step stored."""
    lay = Layout([3, 40, 130, 7], 3, 2)
    taps = [(0, -3), (0, 0), (0, 2)]
    s = Conv(prec, lay, taps, [64], 64, seed=20).sum_plane(init=False)
    idx = torch.as_tensor(lay.out_rows, device=DEV)
    for step, mode in enumerate([lib.SUM_WRITE, lib.SUM_ADD, lib.SUM_ADD, lib.SUM_FINISH]):
        cv = Conv(prec, lay, taps, [64], 64, seed=21 + step)
        case = f'{prec} sum step {step}'
        old = s[idx].double() if step else torch.zeros_like(cv.y)
        before = s.clone()
        act = cv.planes() if mode == lib.SUM_FINISH else None
        cv.run(act=act, mode=REFLECT, sum_plane=s, sum_mode=mode, sum_div=4.0)
        if mode == lib.SUM_FINISH:
            assert torch.equal(_bits(s), _bits(before)), f'{case}: FINISH wrote the sum'
            want, den = (old + cv.y) / 4.0, (old.abs() + cv.den) / 4.0
            _report(case, 'act', cv.check_planes(case, 'act', act, _lrelu(want, 0.2), den, REFLECT))
        else:
            _report(case, 'sum', cv.check_sum(case, s, old + cv.y, old.abs() + cv.den))


@gpu
def test_bf16x3_without_lo_planes():
    """bf16x3 with out_lo = act_lo = NULL: the hi planes are RN(y), bit for bit what the call with lo planes writes."""
    lay = Layout([3, 140, 20], 2, 4)
    cv = Conv('bf16x3', lay, [(0, -2), (0, 0), (0, 2)], [64], 48, seed=30)
    out, act = cv.planes(), cv.planes()
    cv.run(out=out, act=act, mode=REFLECT)
    out1, act1 = (_poison16(out[0].shape), None), (_poison16(act[0].shape), None)
    cv.run(out=out1, act=act1, mode=REFLECT)
    assert torch.equal(_bits(out1[0]), _bits(out[0])) and torch.equal(_bits(act1[0]), _bits(act[0]))
    _report('bf16x3 no lo', 'out', cv.check_planes('bf16x3 no lo', 'out', out1, cv.y, cv.den, REFLECT, lo_given=False))


# ---------------------------------------------------------------------------------------------------- placement invariance
@gpu
@pytest.mark.parametrize('prec', PRECS)
def test_placement_invariance(prec):
    """One 203-row clip behind a prefix clip that puts its first row at residues 0, 1, 63, 64 and 127 of a 128-row tile:
    its out, act and sum (ADD) are bit-identical in every placement."""
    H, L, up, ld_out = 4, 203, 2, 64
    split = prec == 'bf16x3'
    g = torch.Generator().manual_seed(40)
    target = _randn((L + 2 * H, 64), g)          # the clip's input rows, halos included
    sum_target = _randn((L * up, ld_out), g)
    taps = [(0, -4), (0, 1), (0, 3)]
    first = None
    for r in (0, 1, 63, 64, 127):
        counts = [(r - 3 * H) % 128, L, 50]
        lay = Layout(counts, H, up)
        assert lay.in_start[1] % 128 == r
        x = _randn((lay.rows_in, 64), g)
        x[lay.in_start[1] - H:lay.in_start[1] + L + H] = target
        hi, lo = lib.split_bf16(x, split)
        cv = Conv(prec, lay, taps, None, ld_out, seed=41, res=False, xs=[(hi, lo if split else _poison16(hi.shape))])
        s = cv.sum_plane()
        o0 = lay.out_start[1]
        s[o0:o0 + L * up] = sum_target
        out, act = cv.planes(), cv.planes()
        cv.run(out=out, act=act, mode=REFLECT, sum_plane=s, sum_mode=lib.SUM_ADD)
        rows = slice(o0 - H, o0 + L * up + H)
        got = [_bits(t[rows]).clone() for t in (out[0], out[1], act[0], act[1], s)]
        if first is None:
            first = got
            case = f'{prec} placement'
            _report(case, 'out', cv.check_planes(case, 'out', out, cv.y, cv.den, REFLECT))
        else:
            for a, b, what in zip(first, got, ('out_hi', 'out_lo', 'act_hi', 'act_lo', 'sum')):
                assert torch.equal(a, b), f'{prec}: {what} of the clip differs when its first row is at residue {r}'


# ---------------------------------------------------------------------------------------------------- the output layer
def _tanh_case(halo, channels, ld_in, drop_tail, counts, with_lo, seed):
    lay = Layout(counts, halo)
    g = torch.Generator().manual_seed(seed)
    x = _randn((lay.rows_in, ld_in), g)
    hi, lo = lib.split_bf16(x, True)
    hi[:, channels:] = float('nan')                 # columns past `channels` are never read
    lo[:, channels:] = float('nan')
    w = _randn((7, channels), g, (7 * channels) ** -0.5)
    bias = 0.3
    n_out = sum(L - drop_tail for L in counts)
    wav = _poison32(n_out + 64)
    ws = torch.empty(lib.conv1d_workspace_bytes(lay.n), dtype=torch.uint8, device=DEV)
    lib.conv1d_out_tanh_ex(hi, lo if with_lo else None, channels, halo, lay.off.tolist(), drop_tail, w, bias, ws, wav)
    torch.cuda.synchronize()
    xv = _val(hi[:, :channels], lo[:, :channels] if with_lo else None)
    keep = np.concatenate([s + np.arange(L - drop_tail) for s, L in zip(lay.in_start, counts)])
    rows = torch.as_tensor(keep, device=DEV)
    acc = torch.full((len(keep),), bias, dtype=torch.float64, device=DEV)
    den = torch.full_like(acc, abs(bias))
    for k in range(7):
        acc += xv[rows + k - 3] @ w[k].double()
        den += xv[rows + k - 3].abs() @ w[k].double().abs()
    want = torch.tanh(acc)
    got = wav[:n_out].double()
    assert torch.isfinite(got).all(), 'non-finite samples'
    assert (_bits(wav[n_out:]) == -1).all(), 'a sample past the output was written'
    e = ((got - want).abs() - 2.0 ** -21 * want.abs()).clamp_min(0.0) / (U24 * 7 * channels * den)
    return float(e.max()), n_out


TANH_CASES = [  # halo, channels, ld_in, drop_tail, counts, in_lo given
    (3, 1, 8, 0, [1, 2, 5, 300], True),
    (64, 7, 64, 1, [2, 3, 64, 129], False),
    (3, 33, 40, 2560, [2561, 2562, 4000], True),
    (64, 256, 256, 0, [1, 17, 400], True),
    (9, 32, 64, 1, [2, 100, 3], False),
]


@gpu
@pytest.mark.parametrize('case', range(len(TANH_CASES)))
def test_out_tanh_edges(case):
    halo, channels, ld_in, drop_tail, counts, with_lo = TANH_CASES[case]
    e, _ = _tanh_case(halo, channels, ld_in, drop_tail, counts, with_lo, seed=50 + case)
    _report(f'out_tanh {TANH_CASES[case][:4]} lo={with_lo}', 'wav', e, GATE_TANH)


@gpu
def test_out_tanh_beyond_one_grid_pass():
    """More samples than one pass of the grid-stride loop (8 SMs 256 threads), MelGAN's drop_tail, clips of drop_tail + 1."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    counts = [2561, 2561 + 37] + [2561 + 31 * i for i in range(100)]
    e, n_out = _tanh_case(9, 32, 64, mg.HOP * mg.PAD_FRAMES, counts, True, seed=60)
    assert sum(counts) > 8 * sms * 256 and n_out > 0
    _report('out_tanh many samples', 'wav', e, GATE_TANH)
