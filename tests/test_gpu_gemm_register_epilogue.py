"""The register epilogue of the tensor-core forward GEMM (csrc/gemm_tc.cu, epilogue_regs) against its image epilogue.

A plain GEMM whose only outputs are 16-bit planes and whose tile width is a multiple of 64 runs its epilogue from the
wgmma accumulators and stores [16 x 32] boxes with TMA, while its producer already loads the next tile.  Asking the same
call for an fp32 output as well sends it through the image epilogue (the tile parked in shared memory, direct stores).
Both must write the same bits into the 16-bit planes: the same bias, ReLU, dropout mask and scale, padding columns,
row mask and rounding.  The whole buffers are compared, so columns past the tiles must stay untouched in both.
"""
import numpy as np
import pytest
import torch

from gpu_util import DEV, run_gemm
from transformertts_b200 import lib

pytestmark = pytest.mark.gpu

SALT = 0x9E3779B9
SEED = 0x1234ABCD


@pytest.fixture(scope='module', autouse=True)
def dropout_salt():
    lib.load()
    lib.set_dropout_salt(torch.tensor([np.uint32(SALT).view(np.int32)], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    yield SALT
    lib.set_dropout_salt(torch.zeros(1, dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()


def _inputs(g, B, T, Cs, K, N, taps=None):
    xs = [torch.randn(B, T, C, generator=g).to(DEV) for C in Cs]
    shape = (K, N) if taps is None else (taps, K // taps, N)
    w = (torch.randn(*shape, generator=g) / K ** 0.5).to(DEV)
    b = (0.5 * torch.randn(N, generator=g)).to(DEV)
    return xs, w, b


def _row_len(g, B, T):
    lens = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = T
    if B > 2:
        lens[1] = 0
    return lens.to(DEV)


def _same_bits(case, xs, w, b, segs, *, precision, out_fp16=False, **kw):
    planes = ('hi',) if out_fp16 or precision == 'bf16' else ('hi', 'lo')
    reg = run_gemm(xs, w, b, *segs, precision=precision, out_fp16=out_fp16, outputs=planes, **kw)
    img = run_gemm(xs, w, b, *segs, precision=precision, out_fp16=out_fp16, outputs=('f32',) + planes, **kw)
    assert reg['launches'] == 1 and img['launches'] == 1
    for name in planes:
        got, want = reg[name].view(torch.int16), img[name].view(torch.int16)
        assert not (want[..., :img['n_pad']] == -1).all(), f'{case}: {name} plane not written'
        bad = int((got != want).sum())
        assert bad == 0, f'{case}: {name} plane differs from the image epilogue at {bad} of {got.numel()} elements'


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('block_n', [64, 128, 192, 256])
def test_every_width_partial_tile(block_n, precision):
    """Every wgmma width; N = 2 * block_n - 32 leaves the last N tile 32 columns short, T = 300 ends the row tiles inside
    a 16-row box, row_len masks rows (one sentence entirely)."""
    g = torch.Generator().manual_seed(200 + block_n)
    B, T, K = 3, 300, 256
    N = 2 * block_n - 32
    xs, w, b = _inputs(g, B, T, [K], K, N)
    _same_bits(f'{precision} block_n={block_n}', xs, w, b, ([0], [0], [K]), precision=precision, block_n=block_n,
               relu=True, row_len=_row_len(g, B, T))


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('segments', ['three_taps', 'two_sources'])
def test_segments(segments, precision):
    """A 3-tap conv (rows shifted by -1, 0, +1) and a concat projection over two sources inside wider buffers."""
    g = torch.Generator().manual_seed(210)
    B, T, C, N = 4, 257, 128, 320
    if segments == 'three_taps':
        segs = ([0, 0, 0], [-1, 0, 1], [C, C, C])
        xs, w, b = _inputs(g, B, T, [C], 3 * C, N, taps=3)
        kw = {}
    else:
        segs = ([0, 1], [0, 0], [C, C])
        xs, w, b = _inputs(g, B, T, [C, C], 2 * C, N)
        kw = dict(lda=[C + 64, C + 64], a_col0=[64, 8])
    _same_bits(f'{segments} {precision}', xs, w, b, segs, precision=precision, block_n=128, relu=True,
               row_len=_row_len(g, B, T), **kw)


@pytest.mark.parametrize('precision', ['bf16x3', 'bf16'])
def test_dropout(precision):
    """drop_pre under a non-zero salt, with ld_out wider than the tiles: the mask is drawn at (b*T + t)*ld_out + n."""
    g = torch.Generator().manual_seed(220)
    B, T, K, N = 8, 300, 256, 512
    xs, w, b = _inputs(g, B, T, [K], K, N)
    _same_bits(f'dropout {precision}', xs, w, b, ([0], [0], [K]), precision=precision, block_n=256, ld_out=N + 32,
               relu=True, row_len=_row_len(g, B, T), dropout=(0.3, 7), seed=SEED)


@pytest.mark.parametrize('block_n', [128, 256])
def test_fp16_output(block_n):
    """One IEEE fp16 plane (the q|k|v operands of the fp16 attention): the two staging buffers alternate per half slab."""
    g = torch.Generator().manual_seed(230)
    B, T, K, N = 5, 333, 256, 768
    xs, w, b = _inputs(g, B, T, [K], K, N)
    _same_bits(f'fp16 block_n={block_n}', xs, w, b, ([0], [0], [K]), precision='bf16x3', out_fp16=True, block_n=block_n)


@pytest.mark.parametrize('plane', ['bf16x3_hilo', 'fp16', 'bf16_dropout'])
def test_many_tiles_per_cta(plane):
    """B=64, T=1000, N=768 in three 256-wide tiles (the decoder's q|k|v and conv shapes): about a dozen tiles per
    persistent CTA, so the producer runs into the next tile while the epilogue of the last one still stores."""
    g = torch.Generator().manual_seed(240)
    B, T, K, N = 64, 1000, 256, 768
    xs, w, b = _inputs(g, B, T, [K], K, N)
    kw = dict(block_n=256, row_len=_row_len(g, B, T))
    if plane == 'bf16x3_hilo':
        _same_bits(plane, xs, w, b, ([0], [0], [K]), precision='bf16x3', relu=True, **kw)
    elif plane == 'fp16':
        _same_bits(plane, xs, w, b, ([0], [0], [K]), precision='bf16x3', out_fp16=True, **kw)
    else:
        _same_bits(plane, xs, w, b, ([0], [0], [K]), precision='bf16', relu=True, dropout=(0.1, 3), seed=SEED, **kw)
