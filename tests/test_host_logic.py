"""CPU tests of the host-side logic (no GPU): tile selection, parameter inventory, config handling, tables."""
import numpy as np
import pytest
import torch

from oracle import forward_oracle as fo


def test_block_n_selection():
    from transformertts_b200.model.models import _pick_block_n
    assert _pick_block_n(768, False) == 256
    assert _pick_block_n(1024, False) == 256
    assert _pick_block_n(1536, False) == 256
    assert _pick_block_n(226, True) == 240
    assert _pick_block_n(80, False) == 80
    assert _pick_block_n(128, True) == 128
    assert _pick_block_n(384, True) == 384    # d=384 LayerNorm GEMM: one logical tile, run as a CTA pair of 192 columns each
    assert _pick_block_n(400, True) == 80     # not pairable: several N tiles + separate LayerNorm row kernel
    assert _pick_block_n(1152, False) == 192


def test_positional_encoding_matches_oracle_bitwise():
    from transformertts_b200.model.transformer_utils import positional_encoding
    for n, d in ((2000, 256), (300, 128)):
        assert torch.equal(positional_encoding(n, d), fo.positional_encoding(n, d))


def test_masks_mirror_reference_semantics():
    from transformertts_b200.model import transformer_utils as tu
    seq = torch.tensor([[3, 4, 0, 0], [1, 2, 3, 4]])
    assert torch.equal(tu.create_encoder_padding_mask(seq), fo.create_encoder_padding_mask(seq))
    mel = torch.zeros(2, 5, 3)
    mel[0, :2] = 1
    mel[1, :5] = -1
    assert torch.equal(tu.create_mel_padding_mask(mel), fo.create_mel_padding_mask(mel))
    assert torch.equal(tu.mask_from_lengths(torch.tensor([2, 5]), 5), fo.create_mel_padding_mask(mel))
    assert tu.create_look_ahead_mask(3).tolist() == [[0, 1, 1], [0, 0, 1], [0, 0, 0]]


def test_scheduling_and_losses_mirror_reference():
    from transformertts_b200.utils.scheduling import piecewise_linear_schedule, reduction_schedule
    sched = [[0, 1.0e-4], [100, 5.0e-5], [200, 1.0e-5]]
    assert piecewise_linear_schedule(0, sched) == pytest.approx(1e-4)
    assert piecewise_linear_schedule(50, sched) == pytest.approx(7.5e-5)
    assert piecewise_linear_schedule(1000, sched) == pytest.approx(1e-5)
    assert reduction_schedule(90000, [[0, 10], [80000, 5], [100000, 2]]) == 5


def test_aligner_host_mirror_parameters_and_persistence(tmp_path):
    """Constructor / parameter dictionary / save-load of the Aligner mirror (no kernels involved: device='cpu')."""
    import torch
    from oracle import aligner_oracle as alo
    from transformertts_b200 import lib
    from transformertts_b200.model.aligner import Aligner
    cfg = alo.ALIGNER_CONFIGS['A5']
    m = Aligner.from_config(dict(cfg, device='cpu'), max_r=cfg['max_r'])
    want = alo.init_aligner_params(cfg, seed=7)
    shapes = m._param_shapes()
    assert set(shapes) == set(want)
    assert all(tuple(want[k].shape) == tuple(shapes[k]) for k in want)
    m.set_weights(want)
    m.save_model(tmp_path / 'aligner')
    m2 = Aligner.load_model(tmp_path / 'aligner', device='cpu')
    assert m2.max_r == cfg['max_r'] and m2.r == cfg['max_r']
    assert all(torch.equal(m2.weights[k].cpu(), want[k]) for k in want)
    m2.set_constants(reduction_factor=2, force_decoder_diagonal=True)
    assert m2.r == 2 and m2.force_decoder_diagonal and not m2.force_encoder_diagonal
    import pytest
    with pytest.raises(NotImplementedError):
        m2.predict('text')          # encode=True needs the external phonemizer (no text_pipeline attached)


def test_duration_to_alignment_matrix():
    import numpy as np
    from transformertts_b200.utils.alignments import duration_to_alignment_matrix
    m = duration_to_alignment_matrix([2, 0, 3, 1])
    assert m.shape == (4, 6)
    assert np.array_equal(m, np.array([[1, 1, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0], [0, 0, 1, 1, 1, 0], [0, 0, 0, 0, 0, 1]], dtype=float))
    assert np.array_equal(m.sum(1), [2, 0, 3, 1]) and np.array_equal(m.sum(0), np.ones(6))


# ----------------------------------------------------------------------------------------------------------
# the literal ttsb_bgemm reference of the GPU tests (gpu_util.ref_bgemm) against einsum, and the head sizes that train
# ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cross', [False, True])
def test_ref_bgemm_matches_einsum_for_the_six_attention_products(cross):
    """The argument tuples of TrainEngine._attn_fwd / _attn_bwd, evaluated literally, are S = Q K^T, O = P V, dP = dO V^T,
    dQ = dS K, dK = dS^T Q, dV = P^T dO per (b, h); T and Tk are not multiples of anything, the probabilities have NaN in
    their padding columns [Tk, ldp), which lie outside the operand's extent."""
    from gpu_util import ref_bgemm
    g = torch.Generator().manual_seed(11)
    B, H, dh, T = 2, 3, 8, 5
    Tk = 7 if cross else T
    d, Z, ldp = H * dh, B * H, 16
    if cross:
        qb, kb = torch.randn(B, T, d, generator=g), torch.randn(B, Tk, 2 * d, generator=g)
        q_ld, q_col, k_ld, k_col, v_col = d, 0, 2 * d, 0, d
    else:
        qb = kb = torch.randn(B, T, 3 * d, generator=g)
        q_ld, q_col, k_ld, k_col, v_col = 3 * d, 0, 3 * d, d, 2 * d
    dO = torch.randn(B, T, d, generator=g)
    P = torch.full((Z, T, ldp), float('nan'))
    P[..., :Tk] = torch.randn(Z, T, Tk, generator=g)
    heads = lambda x, col: x[..., col:col + d].reshape(B, -1, H, dh).permute(0, 2, 1, 3).reshape(Z, -1, dh).double()
    q, k, v, do, p = heads(qb, q_col), heads(kb, k_col), heads(kb, v_col), heads(dO, 0), P[..., :Tk].double()
    p_op, qa, ka, da = (P, (Tk, T, Z), (ldp, T * ldp)), (qb, (d, T, B), (q_ld, q_ld * T)), (kb, (d, Tk, B), (k_ld, k_ld * Tk)), \
        (dO, (d, T, B), (d, d * T))
    cases = {
        'S': ((T, Tk, dh), qa, (dh, 0, 0, q_col), ka, (dh, 0, 0, k_col), torch.einsum('zmk,znk->zmn', q, k)),
        'O': ((T, dh, Tk), p_op, (0, 0, 1, 0), ka, (dh, 0, 0, v_col, 1), torch.einsum('zmk,zkn->zmn', p, v)),
        'dP': ((T, Tk, dh), da, (dh, 0, 0, 0), ka, (dh, 0, 0, v_col), torch.einsum('zmk,znk->zmn', do, v)),
        'dQ': ((T, dh, Tk), p_op, (0, 0, 1, 0), ka, (dh, 0, 0, k_col, 1), torch.einsum('zmk,zkn->zmn', p, k)),
        'dK': ((Tk, dh, T), p_op, (0, 0, 1, 0, 1), qa, (dh, 0, 0, q_col, 1), torch.einsum('zkm,zkn->zmn', p, q)),
        'dV': ((Tk, dh, T), p_op, (0, 0, 1, 0, 1), da, (dh, 0, 0, 0, 1), torch.einsum('zkm,zkn->zmn', p, do)),
    }
    for name, ((M, N, K), a, a_off, b, b_off, want) in cases.items():
        ref, terms = ref_bgemm(B, H, M, N, K, *a, a_off, *b, b_off)
        assert ref.shape == (Z, M, N) and np.isfinite(ref).all(), name
        assert np.abs(ref - want.numpy()).max() < 1e-12, name
        assert (terms >= np.abs(ref) - 1e-12).all(), name


def test_ref_bgemm_reads_the_next_head_past_a_short_head_block():
    """What the reference is for: with K taken past the head size it sums the next head's columns too (the defect
    ttsb_bgemm refuses), and zero past the extent of the tensor."""
    from gpu_util import ref_bgemm
    x = torch.arange(2 * 3 * 8, dtype=torch.float32).reshape(2, 3, 8)     # (B, T, d), two heads of 4
    one = torch.ones(2, 3, 8)
    args = lambda K: (2, 2, 3, 3, K, x, (8, 3, 2), (8, 24), (4, 0, 0, 0), one, (8, 3, 2), (8, 24), (4, 0, 0, 0))
    own, _ = ref_bgemm(*args(4))
    over, _ = ref_bgemm(*args(8))
    rows = x.reshape(2, 3, 2, 4).permute(0, 2, 1, 3).reshape(4, 3, 4).sum(-1).numpy()
    assert np.array_equal(own, np.repeat(rows[..., None], 3, -1))
    assert np.array_equal(over[0::2], own[0::2] + own[1::2]) and np.array_equal(over[1::2], own[1::2])


def test_training_refuses_head_sizes_the_batched_gemm_reads_across():
    from transformertts_b200.model.training import check_head_sizes
    stack = lambda d, heads: {'encoder': dict(d=d, heads=heads), 'decoder': dict(d=256, heads=[4, 4, 1])}
    for d, heads in ((128, [2, 2]), (256, [4, 2, 1]), (384, [2, 6]), (192, [1, 3]), (32, [1]), (48, [1])):
        check_head_sizes(stack(d, heads))
    for d, heads, dh in ((128, [4, 2], 32), (384, [2, 8], 48), (192, [2, 1], 96), (40, [1], 40)):
        with pytest.raises(ValueError, match=f'head size of {dh}.*multiples of 64'):
            check_head_sizes(stack(d, heads))
