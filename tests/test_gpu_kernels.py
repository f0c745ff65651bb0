"""GPU parity tests, kernel by kernel, through the C ABI (libttsb.so) against the CPU oracle.

Integer / index outputs must be bit-exact; floating point outputs within the tolerance written in each test.
"""
import numpy as np
import pytest
import torch

from oracle import audio_oracle as ao
from oracle import forward_oracle as fo

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
IMPLS = ['simt', 'tcgen05']
PRECS = ['bf16x3', 'bf16']


def _lib():
    from transformertts_b200 import lib
    lib.load()
    return lib


def _relerr(got: torch.Tensor, ref: torch.Tensor) -> float:
    got = got.detach().cpu().double()
    assert torch.isfinite(got).all(), 'non-finite values in kernel output'
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


# ----------------------------------------------------------------------------------------------------------
# row kernels
# ----------------------------------------------------------------------------------------------------------
def test_embed_ln_pe():
    lib = _lib()
    g = torch.Generator().manual_seed(1)
    B, T, d, vocab = 3, 37, 256, 127
    tok = torch.randint(0, vocab, (B, T), generator=g, dtype=torch.int32)
    emb = torch.randn(vocab, d, generator=g) * 0.05
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    pe = fo.positional_encoding(2000, d)[0]
    scalar = torch.tensor([0.8])
    ref = fo.layer_norm(emb[tok.long()], gamma, beta) + scalar * pe[:T]
    out = torch.empty(B, T, d, device=DEV)
    hi = torch.empty(B, T, d, device=DEV, dtype=torch.bfloat16)
    lo = torch.empty_like(hi)
    lib.embed_ln_pe_fwd(tok.to(DEV), emb.to(DEV), gamma.to(DEV), beta.to(DEV), pe.to(DEV), scalar.to(DEV), 1e-6, out, hi, lo)
    torch.cuda.synchronize()
    assert (out.cpu() - ref).abs().max() < 2e-5
    assert (hi.float() + lo.float() - out).abs().max() < 1e-4


def test_durations_to_int_bit_exact():
    lib = _lib()
    g = torch.Generator().manual_seed(2)
    B, Tp = 5, 130
    dur = torch.rand(B, Tp, generator=g) * 12
    dur[0, :8] = torch.tensor([0.5, 1.5, 2.5, 3.5, 2.4999, 2.5001, 0.0, 7.5])
    for scalar in (1.0, float(np.float32(1 / 0.9)), float(np.float32(1 / 1.2))):
        mx = torch.full((B, Tp), float('inf'))
        mx[:, ::7] = 3.0
        mn = torch.zeros(B, Tp)
        mn[:, ::5] = 2.0
        use = torch.maximum(torch.minimum(dur * np.float32(scalar), mx), mn)
        want = fo.round_durations(use[..., None])
        out = torch.empty(B, Tp, dtype=torch.int32, device=DEV)
        lens = torch.empty(B, dtype=torch.int32, device=DEV)
        lib.durations_to_int(dur.to(DEV), scalar, mx.to(DEV), mn.to(DEV), out, lens)
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), want)
        assert torch.equal(lens.cpu(), want.sum(1).to(torch.int32))


@pytest.mark.parametrize('B,Tp,d', [(4, 50, 128), (64, 128, 256), (2, 1500, 384)])
def test_length_regulator_bit_exact(B, Tp, d):
    """Expand (model/layers.py:549-565): indices and gathered values are bit-exact."""
    lib = _lib()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, Tp, d, generator=g)
    dur = torch.randint(0, 16, (B, Tp), generator=g, dtype=torch.int32)
    dur[B - 1, Tp // 2:] = 0  # ragged
    want = fo.expand(x, dur[..., None].float())
    lens, idx_ref = fo.expand_indices(dur)
    Tm = want.shape[1]
    idx = torch.empty(B, Tm, dtype=torch.int32, device=DEV)
    lib.expand_indices(dur.to(DEV), Tm, idx)
    out = torch.full((B, Tm, d), float('nan'), device=DEV)
    lib.length_regulate_fwd(x.to(DEV), idx, out)
    torch.cuda.synchronize()
    assert torch.equal(idx.cpu(), idx_ref)
    assert torch.equal(out.cpu(), want)
    # mel padding mask derived from values == derived from lengths
    assert torch.equal(fo.create_mel_padding_mask(out.cpu())[:, 0, 0], (torch.arange(Tm)[None] >= lens[:, None]).float())


def test_expand_ln_pe_fused():
    lib = _lib()
    g = torch.Generator().manual_seed(4)
    B, Tp, d = 3, 40, 256
    x = torch.randn(B, Tp, d, generator=g)
    dur = torch.randint(0, 9, (B, Tp), generator=g, dtype=torch.int32)
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    pe = fo.positional_encoding(10000, d)[0]
    scalar = torch.tensor([1.1])
    ex = fo.expand(x, dur[..., None].float())
    Tm = ex.shape[1]
    ref = fo.layer_norm(ex, gamma, beta) + scalar * pe[:Tm]
    idx = torch.empty(B, Tm, dtype=torch.int32, device=DEV)
    lib.expand_indices(dur.to(DEV), Tm, idx)
    out = torch.empty(B, Tm, d, device=DEV)
    hi = torch.empty(B, Tm, d, device=DEV, dtype=torch.bfloat16)
    lo = torch.empty_like(hi)
    lib.expand_ln_pe_fwd(x.to(DEV), idx, gamma.to(DEV), beta.to(DEV), pe.to(DEV), scalar.to(DEV), 1e-6, out, hi, lo)
    torch.cuda.synchronize()
    assert (out.cpu() - ref).abs().max() < 5e-5


def test_predictor_head_pitch_embed_and_lengths():
    lib = _lib()
    g = torch.Generator().manual_seed(5)
    B, T, C = 4, 33, 226
    h = torch.randn(B, T, 240, generator=g)
    w, b = torch.randn(C, generator=g) * 0.1, torch.randn(1, generator=g)
    lens = torch.tensor([33, 10, 0, 20], dtype=torch.int32)
    keep = (torch.arange(T)[None] < lens[:, None]).float()
    for relu in (True, False):
        ref = h[..., :C] @ w + b
        ref = (torch.relu(ref) if relu else ref) * keep
        out = torch.empty(B, T, device=DEV)
        lib.statpred_head_fwd(h.to(DEV), C, w.to(DEV), b.to(DEV), relu, lens.to(DEV), out)
        torch.cuda.synchronize()
        assert (out.cpu() - ref).abs().max() < 1e-4
    d = 256
    x, pitch = torch.randn(B, T, d, generator=g), torch.randn(B, T, generator=g)
    pw, pb = torch.randn(d, generator=g), torch.randn(d, generator=g)
    out = torch.empty(B, T, d, device=DEV)
    lib.pitch_embed_add_fwd(x.to(DEV), pitch.to(DEV), pw.to(DEV), pb.to(DEV), out)
    ref = x + torch.relu(pitch[..., None] * pw + pb)
    torch.cuda.synchronize()
    assert (out.cpu() - ref).abs().max() < 1e-5
    # utils/spectrogram_ops.py: integer outputs, bit-exact
    mel = torch.randn(3, 50, 80, generator=g)
    mel[0, 30:] = 0
    mel[1, 45:] = 0
    mel[1, 10, :] = 0  # an all-zero frame inside counts as padding too (value-derived)
    o = torch.empty(3, dtype=torch.int32, device=DEV)
    lib.mel_lengths(mel.to(DEV), 0.0, o)
    torch.cuda.synchronize()
    assert o.cpu().tolist() == ao.mel_lengths(mel.numpy()).tolist() == [30, 44, 50]
    ph = torch.randint(1, 127, (3, 40), generator=g, dtype=torch.int32)
    ph[0, 25:] = 0
    ph[2, 39:] = 0
    o2 = torch.empty(3, dtype=torch.int32, device=DEV)
    lib.phoneme_lengths(ph.to(DEV), 0, o2)
    torch.cuda.synchronize()
    assert o2.cpu().tolist() == ao.phoneme_lengths(ph.numpy()).tolist()


# ----------------------------------------------------------------------------------------------------------
# tensor-core GEMM family
# ----------------------------------------------------------------------------------------------------------
def _tol(precision):
    return 2e-5 if precision == 'bf16x3' else 2e-3


@pytest.mark.parametrize('impl', IMPLS)
@pytest.mark.parametrize('precision', PRECS)
def test_gemm_qkv_projection(impl, precision):
    """Dense d -> 3d with bias into one (B,T,3d) buffer: bf16 hi/lo planes and the fp16 plane the fp16 attention reads."""
    from gpu_util import ref_gemm, run_gemm
    g = torch.Generator().manual_seed(10)
    B, T, d = 3, 200, 256
    x = torch.randn(B, T, d, generator=g).to(DEV)
    w = (torch.randn(d, 3 * d, generator=g) / 16).to(DEV)
    b = torch.randn(3 * d, generator=g).to(DEV)
    out = run_gemm([x], w, b, [0], [0], [d], precision=precision, impl=impl, block_n=d)
    ref = ref_gemm([x], w, b, [0], [0], [d], precision=precision)
    assert _relerr(out['f32'], ref) < _tol(precision)
    if precision == 'bf16x3':
        assert _relerr(out['hi'].float() + out['lo'].float(), ref) < 1e-4
    out16 = run_gemm([x], w, b, [0], [0], [d], precision=precision, impl=impl, block_n=d, out_fp16=True)
    h16 = out16['hi'].view(torch.float16).float()
    assert _relerr(h16, ref) < 3e-3


@pytest.mark.parametrize('impl', IMPLS)
@pytest.mark.parametrize('precision', PRECS)
def test_gemm_concat_projection_residual_layernorm_mask(impl, precision):
    """Dense on concat([x, attn]) (2d -> d) + residual + LayerNorm + row mask (layers.py:148-149, 211, 229)."""
    from gpu_util import ref_gemm, run_gemm
    g = torch.Generator().manual_seed(11)
    B, T, d = 3, 300, 256
    x = torch.randn(B, T, d, generator=g).to(DEV)
    a = torch.randn(B, T, d, generator=g).to(DEV)
    w = (torch.randn(2 * d, d, generator=g) / 22).to(DEV)
    b = torch.randn(d, generator=g).to(DEV)
    gamma, beta = (1 + 0.1 * torch.randn(d, generator=g)).to(DEV), (0.1 * torch.randn(d, generator=g)).to(DEV)
    lens = torch.tensor([300, 131, 7], dtype=torch.int32, device=DEV)
    kw = dict(residual=x, ln=(gamma, beta), row_len=lens)
    out = run_gemm([x, a], w, b, [0, 1], [0, 0], [d, d], precision=precision, impl=impl, single_tile=True, **kw)
    ref = ref_gemm([x, a], w, b, [0, 1], [0, 0], [d, d], precision=precision, **kw)
    assert _relerr(out['f32'], ref) < _tol(precision) * 2
    assert torch.count_nonzero(out['f32'][1, 131:]) == 0 and torch.count_nonzero(out['hi'][2, 7:]) == 0


@pytest.mark.parametrize('impl', IMPLS)
@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('T', [128, 333])
def test_gemm_conv3_relu_then_conv3_layernorm(impl, precision, T):
    """Conv1D(k=3,'same') d->F + relu, then Conv1D F->d + residual + LayerNorm + mask (CNNResNorm, layers.py:36-40)."""
    from gpu_util import ref_gemm, run_gemm
    g = torch.Generator().manual_seed(12)
    B, d, F = 2, 128, 512
    x = torch.randn(B, T, d, generator=g).to(DEV)
    w1 = (torch.randn(3, d, F, generator=g) / 20).to(DEV)
    b1 = torch.randn(F, generator=g).to(DEV)
    out1 = run_gemm([x], w1, b1, [0, 0, 0], [-1, 0, 1], [d, d, d], precision=precision, impl=impl, relu=True)
    ref1 = ref_gemm([x], w1, b1, [0, 0, 0], [-1, 0, 1], [d, d, d], precision=precision, relu=True)
    assert _relerr(out1['f32'], ref1) < _tol(precision)
    # cross-check the reference against the oracle's literal conv
    lit = torch.relu(fo.conv1d_same(x.cpu(), w1.cpu(), b1.cpu()))
    if precision == 'bf16x3':
        assert (lit.double() - ref1).abs().max() < 1e-4
    h = out1['f32'].contiguous()
    w2 = (torch.randn(3, F, d, generator=g) / 40).to(DEV)
    b2 = torch.randn(d, generator=g).to(DEV)
    gamma, beta = (1 + 0.1 * torch.randn(d, generator=g)).to(DEV), (0.1 * torch.randn(d, generator=g)).to(DEV)
    lens = torch.tensor([T, T // 3], dtype=torch.int32, device=DEV)
    kw = dict(residual=x, ln=(gamma, beta), row_len=lens)
    out2 = run_gemm([h], w2, b2, [0, 0, 0], [-1, 0, 1], [F, F, F], precision=precision, impl=impl, single_tile=True, **kw)
    ref2 = ref_gemm([h], w2, b2, [0, 0, 0], [-1, 0, 1], [F, F, F], precision=precision, **kw)
    assert _relerr(out2['f32'], ref2) < _tol(precision) * 2


@pytest.mark.parametrize('impl', IMPLS)
def test_gemm_predictor_226_columns_and_mel_80(impl):
    """N=226 (padded to 240 columns, LayerNorm statistics over 226 only) and the final Dense(80)."""
    from gpu_util import ref_gemm, run_gemm
    g = torch.Generator().manual_seed(13)
    B, T, d = 2, 150, 256
    x = torch.randn(B, T, d, generator=g).to(DEV)
    w = (torch.randn(3, d, 226, generator=g) / 28).to(DEV)
    b = torch.randn(226, generator=g).to(DEV)
    gamma, beta = (1 + 0.1 * torch.randn(226, generator=g)).to(DEV), (0.1 * torch.randn(226, generator=g)).to(DEV)
    out = run_gemm([x], w, b, [0, 0, 0], [-1, 0, 1], [d, d, d], impl=impl, relu=True, ln=(gamma, beta), single_tile=True)
    ref = ref_gemm([x], w, b, [0, 0, 0], [-1, 0, 1], [d, d, d], precision='bf16x3', relu=True, ln=(gamma, beta))
    assert out['n_pad'] == 240
    assert _relerr(out['f32'][..., :226], ref) < 5e-5
    assert torch.count_nonzero(out['f32'][..., 226:]) == 0
    wm = (torch.randn(d, 80, generator=g) / 16).to(DEV)
    bm = torch.randn(80, generator=g).to(DEV)
    out = run_gemm([x], wm, bm, [0], [0], [d], impl=impl)
    assert out['n_pad'] == 80
    assert _relerr(out['f32'], ref_gemm([x], wm, bm, [0], [0], [d], precision='bf16x3')) < 2e-5


@pytest.mark.parametrize('precision', PRECS)
def test_gemm_persistent_many_tiles(precision):
    """More tiles than SMs: exercises the persistent loop, the accumulator image over the drained ring and the smem ring wrap."""
    from gpu_util import ref_gemm, run_gemm
    g = torch.Generator().manual_seed(14)
    B, T, d, F = 40, 1000, 256, 1024
    x = torch.randn(B, T, d, generator=g).to(DEV)
    w = (torch.randn(3, d, F, generator=g) / 28).to(DEV)
    b = torch.randn(F, generator=g).to(DEV)
    out = run_gemm([x], w, b, [0, 0, 0], [-1, 0, 1], [d, d, d], precision=precision, relu=True)
    sel = [0, 17, 39]
    ref = ref_gemm([x[sel]], w, b, [0, 0, 0], [-1, 0, 1], [d, d, d], precision=precision, relu=True)
    assert _relerr(out['f32'][sel], ref) < _tol(precision)
    assert torch.isfinite(out['f32']).all()


# ----------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('impl', IMPLS)
@pytest.mark.parametrize('precision', PRECS + ['fp16'])
@pytest.mark.parametrize('H,d,T', [(2, 256, 200), (2, 128, 333), (2, 256, 64), (2, 384, 200)])
def test_mha_varlen(impl, precision, H, d, T):
    from gpu_util import ref_mha, run_mha
    if d == 384 and precision == 'bf16x3' and impl == 'tcgen05':
        pytest.skip('head_dim 192 runs in the single-pass modes (fp16 is the default attention precision)')
    g = torch.Generator().manual_seed(20)
    B = 3
    q = torch.randn(B, T, d, generator=g).to(DEV)
    k = torch.randn(B, T, d, generator=g).to(DEV)
    v = torch.randn(B, T, d, generator=g).to(DEV)
    lens = torch.tensor([T, max(1, T // 3), min(T, 65)], dtype=torch.int32, device=DEV)
    out, wts = run_mha(q, k, v, lens, H, precision=precision, impl=impl, weights_b=1)
    ref, wref = ref_mha(q, k, v, lens, H, precision)
    tol = {'bf16x3': 5e-5, 'bf16': 8e-3, 'fp16': 1e-3}[precision]
    for b in range(B):
        n = int(lens[b])  # padded query rows are zeroed by the caller's row mask; only valid rows are compared
        assert _relerr(out[b, :n], ref[b, :n]) < tol
    # reference-exact softmax weights of one batch row (all query rows, incl. padded ones)
    assert (wts.cpu().double() - wref[1]).abs().max() < (1e-5 if precision == 'bf16x3' else 5e-3)
    assert torch.isfinite(out).all()


@pytest.mark.parametrize('impl', ['tcgen05', 'simt'])
@pytest.mark.parametrize('precision,H,d,T,Tk,causal,cross', [
    ('fp16', 4, 256, 300, 300, True, False),     # Aligner decoder self-attention: look-ahead + padding (models.py:136-138)
    ('fp16', 1, 256, 200, 200, True, False),     # last decoder block: one head of 256
    ('fp16', 4, 256, 333, 77, False, True),      # cross-attention onto the encoder output
    ('fp16', 1, 256, 130, 45, False, True),
    ('bf16x3', 4, 256, 140, 70, False, True),
    ('bf16x3', 2, 256, 260, 260, True, False),
    ('bf16', 4, 256, 129, 129, True, False),
])
def test_mha_causal_and_cross(impl, precision, H, d, T, Tk, causal, cross):
    from gpu_util import ref_mha_general, run_mha_general
    g = torch.Generator().manual_seed(21)
    B = 3
    q = torch.randn(B, T, d, generator=g).to(DEV)
    k = torch.randn(B, Tk, d, generator=g).to(DEV)
    v = torch.randn(B, Tk, d, generator=g).to(DEV)
    lens = torch.tensor([Tk, max(1, Tk // 3), min(Tk, 65)], dtype=torch.int32, device=DEV)
    out, wts = run_mha_general(q, k, v, lens, H, precision=precision, impl=impl, causal=causal, cross=cross,
                               full_queries=True, weights_all=True)
    ref, wref = ref_mha_general(q, k, v, lens, H, precision, causal=causal)
    tol = {'bf16x3': 5e-5, 'bf16': 8e-3, 'fp16': 1e-3}[precision]
    assert torch.isfinite(out).all()
    assert _relerr(out, ref) < tol                      # every query row, padded ones included (full_queries)
    assert (wts.cpu().double() - wref).abs().max() < (1e-5 if precision == 'bf16x3' else 5e-3)


# ----------------------------------------------------------------------------------------------------------
# STFT -> mel -> log
# ----------------------------------------------------------------------------------------------------------
def test_stft_mel_golden_and_oracle():
    from transformertts_b200.data.audio import Audio
    g = np.load('tests/golden/audio_mel.npz')
    clips = ao.make_clips(2, int(g['n_samples']), seed=int(g['clips_seed']))
    audio = Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
                  normalizer='MelGAN')
    got = audio.mel_spectrogram_batch(clips)
    assert got.shape == g['mel'].shape
    assert np.abs(got - g['mel']).max() < 1e-3  # log-mel, absolute
    one = audio.mel_spectrogram(clips[0])
    assert one.shape == (44, 80) and np.abs(one - g['mel'][0]).max() < 1e-3
    w = Audio(sampling_rate=22050, n_fft=1024, mel_channels=80, hop_length=256, win_length=1024, f_min=0, f_max=8000,
              normalizer='WaveRNN').mel_spectrogram(clips[0])
    assert np.abs(w - g['mel_wavernn']).max() < 1e-3
    # odd frame count, short clip, edge reflection on both sides
    y = ao.make_clips(1, 1500, seed=9)[0]
    assert np.abs(audio.mel_spectrogram(y) - ao.mel_spectrogram(y)).max() < 1e-3
