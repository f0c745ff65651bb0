"""GPU parity of the training step: gradient kernels one by one, then loss / gradients / Adam of the whole
ForwardTransformer against torch autograd on the CPU oracle (dropout off; the forward runs in single-pass bf16, so
gradients are compared per tensor with a relative tolerance)."""
import math

import numpy as np
import pytest
import torch

from oracle import forward_oracle as fo

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _lib():
    from transformertts_b200 import lib
    lib.load()
    return lib


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_wgrad_conv_and_concat():
    """dW of Conv1D(k=3,'same') and of the concat projection against x^T g on the CPU (operands read MN-major)."""
    lib = _lib()
    g = torch.Generator().manual_seed(1)
    B, T, Cin, N = 5, 333, 256, 226
    x = torch.randn(B, T, Cin, generator=g).bfloat16()
    gy = torch.zeros(B, T, 256).bfloat16()
    gy[..., :N] = torch.randn(B, T, N, generator=g).bfloat16()
    x_d, g_d = x.to(DEV), gy.to(DEV)
    dw = torch.zeros(3 * Cin, N, device=DEV)
    a = lib.WgradArgs()
    a.B, a.T, a.Cin, a.N, a.num_segments = B, T, Cin, N, 3
    for s_, sh in enumerate((-1, 0, 1)):
        a.seg_src[s_], a.seg_shift[s_] = 0, sh
    a.x[0], a.ldx[0] = x_d.data_ptr(), Cin
    a.g, a.ldg, a.dw = g_d.data_ptr(), 256, dw.data_ptr()
    lib.wgrad(a)
    torch.cuda.synchronize()
    xd, gd = x.double(), gy[..., :N].double()
    ref = torch.zeros(3, Cin, N, dtype=torch.float64)
    for tap, sh in enumerate((-1, 0, 1)):
        lo, hi = max(0, -sh), min(T, T - sh)
        ref[tap] = torch.einsum('btc,btn->cn', xd[:, lo + sh:hi + sh], gd[:, lo:hi])
    assert _rel(dw.view(3, Cin, N), ref) < 1e-4
    # two sources (concat projection), accumulate on top of existing values
    x2 = torch.randn(B, T, Cin, generator=g).bfloat16()
    x2_d = x2.to(DEV)
    dw2 = torch.ones(2 * Cin, N, device=DEV)
    a2 = lib.WgradArgs()
    a2.B, a2.T, a2.Cin, a2.N, a2.num_segments = B, T, Cin, N, 2
    a2.seg_src[0], a2.seg_src[1] = 0, 1
    a2.x[0], a2.x[1], a2.ldx[0], a2.ldx[1] = x_d.data_ptr(), x2_d.data_ptr(), Cin, Cin
    a2.g, a2.ldg, a2.dw = g_d.data_ptr(), 256, dw2.data_ptr()
    lib.wgrad(a2)
    torch.cuda.synchronize()
    ref2 = 1 + torch.cat([torch.einsum('btc,btn->cn', xd, gd), torch.einsum('btc,btn->cn', x2.double(), gd)])
    assert _rel(dw2, ref2) < 1e-4


@pytest.mark.parametrize('H,dh,T', [(2, 128, 200), (2, 64, 333)])
def test_attention_train_path_forward_and_backward(H, dh, T):
    """S = QK^T, softmax, O = PV and the five gradient GEMMs, through TrainEngine helpers on a standalone block."""
    lib = _lib()
    from transformertts_b200.model.training import TrainEngine
    from transformertts_b200.model.models import _round_up
    g = torch.Generator().manual_seed(2)
    B, d = 3, H * dh
    qkv = torch.randn(B, T, 3 * d, generator=g).bfloat16()
    dO = torch.randn(B, T, d, generator=g).bfloat16()
    lens = torch.tensor([T, T // 2, 70], dtype=torch.int32)
    eng = TrainEngine.__new__(TrainEngine)
    eng.dev = torch.device(DEV)
    qkv_d, dO_d, lens_d = qkv.to(DEV), dO.to(DEV), lens.to(DEV)
    Z, ldp = B * H, _round_up(T, 16)
    S = torch.empty(Z, T, ldp, device=DEV)
    eng._bgemm(B, H, T, T, dh, qkv_d, (3 * d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 0), qkv_d, (2 * d, T, B), (3 * d, 3 * d * T),
               (dh, 0, 0, d), alpha=1.0 / math.sqrt(dh), out_f32=S, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp)
    P = torch.empty(Z, T, ldp, dtype=torch.bfloat16, device=DEV)
    lib.softmax_fwd(S, B, H, T, T, ldp, lens_d, 0.0, 0, 0, P, P)
    attn = torch.empty(B, T, d, dtype=torch.bfloat16, device=DEV)
    eng._bgemm(B, H, T, dh, T, P, (T, T, Z), (ldp, T * ldp), (0, 0, 1, 0), qkv_d, (d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 2 * d, 1),
               out_bf16=attn, ld_out=d, out_batch_stride=T * d, out_h_col=dh, out_by_b=1, out_cols=dh)
    torch.cuda.synchronize()
    # reference with autograd (fp64) on the bf16 inputs
    x = qkv.double().requires_grad_(True)
    q, k, v = [t.reshape(B, T, H, dh).permute(0, 2, 1, 3) for t in x.split(d, dim=-1)]
    logits = q @ k.transpose(-1, -2) / math.sqrt(dh)
    mask = torch.arange(T)[None, :] >= lens[:, None]
    logits = logits.masked_fill(mask[:, None, None, :], float('-inf'))
    w = torch.softmax(logits, -1)
    o = (w @ v).permute(0, 2, 1, 3).reshape(B, T, d)
    keep = (~mask)[..., None].double()
    (o * keep * dO.double()).sum().backward()
    for b in range(B):
        n = int(lens[b])
        assert _rel(attn[b, :n], o[b, :n]) < 1e-2
        assert _rel(P.view(B, H, T, ldp)[b, :, :n, :T].float(), w[b, :, :n]) < 1e-2
    # backward
    dO_m = (dO.double() * keep).bfloat16().to(DEV)  # rows of padded queries carry zero gradient (row mask upstream)
    dP = torch.empty(Z, T, ldp, device=DEV)
    eng._bgemm(B, H, T, T, dh, dO_m, (d, T, B), (d, d * T), (dh, 0, 0, 0), qkv_d, (d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 2 * d),
               out_f32=dP, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp)
    dS = torch.empty(Z, T, ldp, dtype=torch.bfloat16, device=DEV)
    lib.softmax_bwd(P, dP, B, H, T, T, ldp, lens_d, 1.0 / math.sqrt(dh), 0.0, 0, 0, dS)
    dqkv = torch.full((B, T, 3 * d), float('nan'), dtype=torch.bfloat16, device=DEV)
    common = dict(out_bf16=dqkv, ld_out=3 * d, out_batch_stride=T * 3 * d, out_h_col=dh, out_by_b=1, out_cols=dh)
    qd, qs = (d, T, B), (3 * d, 3 * d * T)
    eng._bgemm(B, H, T, dh, T, dS, (T, T, Z), (ldp, T * ldp), (0, 0, 1, 0), qkv_d, qd, qs, (dh, 0, 0, d, 1), out_ptr_off=0, **common)
    eng._bgemm(B, H, T, dh, T, dS, (T, T, Z), (ldp, T * ldp), (0, 0, 1, 0, 1), qkv_d, qd, qs, (dh, 0, 0, 0, 1), out_ptr_off=d, **common)
    eng._bgemm(B, H, T, dh, T, P, (T, T, Z), (ldp, T * ldp), (0, 0, 1, 0, 1), dO_m, (d, T, B), (d, d * T), (dh, 0, 0, 0, 1), out_ptr_off=2 * d, **common)
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all()
    assert _rel(dqkv.float(), x.grad) < 3e-2
    # the fused form: dS straight from the dP product's epilogue with D = dO . O (no fp32 dP round trip) -- without and
    # with attention dropout (same hash => same masks as the stand-alone kernels)
    for rate in (0.0, 0.25):
        Pp = torch.empty(Z, T, ldp, dtype=torch.bfloat16, device=DEV)
        Pd = torch.empty(Z, T, ldp, dtype=torch.bfloat16, device=DEV) if rate > 0 else Pp
        lib.softmax_fwd(S, B, H, T, T, ldp, lens_d, rate, 77, 5, Pp, Pd)
        O2 = torch.empty(B, T, d, dtype=torch.bfloat16, device=DEV)
        eng._bgemm(B, H, T, dh, T, Pd, (T, T, Z), (ldp, T * ldp), (0, 0, 1, 0), qkv_d, (d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 2 * d, 1),
                   out_bf16=O2, ld_out=d, out_batch_stride=T * d, out_h_col=dh, out_by_b=1, out_cols=dh)
        eng._bgemm(B, H, T, T, dh, dO_m, (d, T, B), (d, d * T), (dh, 0, 0, 0), qkv_d, (d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 2 * d),
                   out_f32=dP, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp)
        dS_ref = torch.empty(Z, T, ldp, dtype=torch.bfloat16, device=DEV)
        lib.softmax_bwd(Pp, dP, B, H, T, T, ldp, lens_d, 1.0 / math.sqrt(dh), rate, 77, 5, dS_ref)
        D = torch.empty(Z * T, device=DEV)
        lib.rowdot_heads(dO_m, O2, H, dh, D)
        dS_f = torch.full((Z, T, ldp), float('nan'), dtype=torch.bfloat16, device=DEV)
        eng._bgemm(B, H, T, T, dh, dO_m, (d, T, B), (d, d * T), (dh, 0, 0, 0), qkv_d, (d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 2 * d),
                   out_bf16=dS_f, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp,
                   softmax_bwd=(Pp, D, 1.0 / math.sqrt(dh), rate, 77, 5, 0, lens_d))
        torch.cuda.synchronize()
        assert torch.isfinite(dS_f.float()).all()
        # D comes from the bf16-rounded O instead of the fp32 dP: equal up to bf16 rounding of O
        assert _rel(dS_f.float(), dS_ref.float()) < 2e-2, rate
        if rate > 0:  # dropout decision read back from the saved P_drop instead of the hash: identical result
            dS_g = torch.full((Z, T, ldp), float('nan'), dtype=torch.bfloat16, device=DEV)
            eng._bgemm(B, H, T, T, dh, dO_m, (d, T, B), (d, d * T), (dh, 0, 0, 0), qkv_d, (d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 2 * d),
                       out_bf16=dS_g, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp,
                       softmax_bwd=(Pp, D, 1.0 / math.sqrt(dh), rate, 77, 5, 0, lens_d, Pd))
            torch.cuda.synchronize()
            assert torch.equal(dS_g, dS_f)


def test_layernorm_bwd_and_small_ops():
    lib = _lib()
    g = torch.Generator().manual_seed(3)
    B, T, C, ld = 4, 77, 226, 256
    u = torch.zeros(B, T, ld)
    u[..., :C] = torch.relu(torch.randn(B, T, C, generator=g))
    dz = torch.zeros(B, T, ld)
    dz[..., :C] = torch.randn(B, T, C, generator=g)
    gamma = torch.zeros(ld)
    gamma[:C] = 1 + 0.1 * torch.randn(C, generator=g)
    lens = torch.tensor([77, 30, 0, 50], dtype=torch.int32)
    uu = u[..., :C].double().requires_grad_(True)
    gg = gamma[:C].double().requires_grad_(True)
    bb = torch.zeros(C, dtype=torch.float64, requires_grad=True)
    keep = (torch.arange(T)[None] < lens[:, None])[..., None].double()
    y = fo.layer_norm(uu, gg, bb) * keep
    (y * dz[..., :C].double()).sum().backward()
    du = torch.full((B, T, ld), float('nan'), device=DEV)
    gb = torch.full((B, T, ld), float('nan'), dtype=torch.bfloat16, device=DEV)
    dg, db, dbias = torch.zeros(ld, device=DEV), torch.zeros(ld, device=DEV), torch.zeros(ld, device=DEV)
    lib.layernorm_bwd(dz.to(DEV), u.to(DEV), gamma.to(DEV), B, T, C, ld, 1e-6, lens.to(DEV), True, du, gb, dg, db, dbias=dbias)
    torch.cuda.synchronize()
    assert _rel(du[..., :C], uu.grad) < 1e-4 and torch.count_nonzero(du[..., C:]) == 0
    assert _rel(dg[:C], gg.grad) < 1e-4 and _rel(db[:C], bb.grad) < 1e-4
    assert _rel(gb[..., :C].float(), uu.grad * (u[..., :C] > 0)) < 1e-2
    assert _rel(dbias[:C], (uu.grad * (u[..., :C] > 0)).sum((0, 1))) < 1e-4
    cs = torch.zeros(C, device=DEV)
    lib.colsum_bf16(gb, B * T, C, ld, cs)
    torch.cuda.synchronize()
    assert _rel(cs, gb[..., :C].float().sum((0, 1))) < 1e-5
    # MAE loss + gradient (unmasked mean over all elements, int targets)
    pred = torch.randn(3, 20, 1, generator=g)
    tgt = torch.randint(0, 5, (3, 20), generator=g, dtype=torch.int32)
    loss = torch.zeros(1, device=DEV)
    grad = torch.empty(3, 20, device=DEV)
    lib.mae_loss(pred.to(DEV), 3, 20, 20, 1, tgt.to(DEV), 3.0, loss, grad)
    torch.cuda.synchronize()
    ref = fo.masked_mean_absolute_error(tgt[..., None], pred)
    assert abs(loss.item() - ref.item()) < 1e-5
    assert _rel(grad, 3.0 * torch.sign(pred[..., 0] - tgt) / 60) < 1e-6
    # Adam (Keras form)
    p, gr = torch.randn(1000, generator=g), torch.randn(1000, generator=g) * 1e-3
    m0, v0 = torch.zeros(1000), torch.zeros(1000)
    pd, md, vd = p.to(DEV), m0.to(DEV), v0.to(DEV)
    pr = p.clone()
    for step in (1, 2, 3):
        lr_t = 1e-4 * math.sqrt(1 - 0.98 ** step) / (1 - 0.9 ** step)
        lib.adam_tf_step(pd, gr.to(DEV), md, vd, lr_t, 0.9, 0.98, 1e-9)
        fo.adam_tf_step(pr, gr, m0, v0, step, 1e-4)
    torch.cuda.synchronize()
    assert (pd.cpu() - pr).abs().max() < 1e-7


def _grad_report(eng, ref_g, zero_names, gscale):
    rows = []
    for name, gref in ref_g.items():
        got = eng.g[name].detach().double().cpu()
        if name in zero_names:
            assert float(got.norm()) < 2e-3 * gscale, name        # analytically zero (key bias: softmax shift invariance)
            continue
        gr = gref.double()
        if gr.dim() == 0:
            rows.append((abs(float(got) - float(gr)) / abs(float(gr)), 1.0 if float(got) * float(gr) > 0 else -1.0, name))
        else:
            rows.append((_rel(got, gr), float((got * gr).sum() / (got.norm() * gr.norm())), name))
    rows.sort(reverse=True)
    return rows


@pytest.mark.parametrize('cfg_name,B,Tp,Tm,tol_emu,cos_emu,tol_f32,cos_f32', [
    ('C1', 16, 48, 400, 0.06, 0.998, 0.15, 0.99),          # shallow model, larger batch: bf16 noise averages out
    ('LJ256', 8, 48, 400, 0.16, 0.99, 0.25, 0.975),        # 6+6 blocks: rounding differences decorrelate through the depth
    ('REF384', 2, 24, 200, 0.30, 0.95, 0.30, 0.95)])
def test_train_step_loss_grads_and_adam(cfg_name, B, Tp, Tm, tol_emu, cos_emu, tol_f32, cos_f32):
    """One deterministic training step (dropout off): loss, every parameter gradient and the Adam update against torch
    autograd on the restated graph -- once with the oracle's matrix products fed bf16-rounded operands like the tensor-core
    path (forward_oracle.EMULATE_BF16: what remains is summation order and the decorrelation of individual roundings), once
    against the plain fp32 oracle.  Gates come from tools/grad_noise.py measurements of the step's gradient noise with ~1.5x
    margin; the pos_encoding_scalar gradients (one number each, heavy cancellation) are gated on sign and a factor of two."""
    torch.set_num_threads(8)
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.model.training import Adam
    cfg = fo.CONFIGS[cfg_name]
    p = fo.init_params(cfg, seed=7)
    tok, dur, pit = fo.make_inputs('ragged', B, Tp, Tm, seed=301)
    mel_tgt = fo.make_mel_targets(dur, 80, seed=302)
    ref_out, ref_g = fo.loss_and_grads(p, cfg, tok, mel_tgt, dur, pit)
    emu_out, emu_g = fo.loss_and_grads(p, cfg, tok, mel_tgt, dur, pit, emulate_bf16=True)
    model = ForwardTransformer(**cfg, train_dropout=False)
    model.set_weights(p)
    model._compile(Adam(1e-4))
    eng = model._get_engine()
    out = eng.forward_backward(tok, mel_tgt, dur, pit, training=True)
    torch.cuda.synchronize()
    assert abs(out['loss'].item() - float(ref_out['loss'])) < 2e-3 * abs(float(ref_out['loss']))
    assert abs(out['loss'].item() - float(emu_out['loss'])) < 5e-4 * abs(float(emu_out['loss']))
    for k in ('mel', 'duration', 'pitch'):
        assert abs(out['losses'][k].item() - float(emu_out['losses'][k])) < 2e-3 * abs(float(emu_out['losses'][k])) + 1e-4
    gscale = max(float(g.norm()) for g in ref_g.values())
    zero = {n for n, g in ref_g.items() if float(g.norm()) < 1e-6 * gscale}
    for tag, oracle_g, tol, cmin in (('bf16-emulating oracle', emu_g, tol_emu, cos_emu), ('fp32 oracle', ref_g, tol_f32, cos_f32)):
        rows = _grad_report(eng, oracle_g, zero, gscale)
        print(f'{cfg_name} vs {tag}: worst', [(n, round(r, 4), round(c, 5)) for r, c, n in rows[:5]])
        for r, c, n in rows:
            if n.endswith('pos_scalar'):
                assert c > 0 and r < 1.0, (tag, n, r)
            else:
                assert r < tol and c > cmin, (tag, n, r, c)
    # Adam: the update applied to the flat buffer equals the oracle formula on the same gradients
    w0 = eng.flat_w.clone()
    g0 = eng.flat_g.clone()
    eng.apply_adam(model.optimizer)
    torch.cuda.synchronize()
    m_ref, v_ref, w_ref = torch.zeros_like(w0).cpu(), torch.zeros_like(w0).cpu(), w0.cpu().clone()
    fo.adam_tf_step(w_ref, g0.cpu(), m_ref, v_ref, 1, 1e-4)
    assert (eng.flat_w.cpu() - w_ref).abs().max() < 3e-7
    assert model.step == 1
    # a second full step runs (weights were re-packed) and lowers nothing to NaN
    out2 = model.train_step(tok, mel_tgt, dur, pit)
    assert math.isfinite(out2['loss'].item())


def test_train_step_full_size_c3_against_oracle():
    """BASELINE config C3 at its full size (LJ256, 32 rows, 128 tokens, 1000 frames, ragged) through the path bench.py times
    (train_graphs=True: two CUDA graphs + eager Adam): loss and every parameter gradient against torch autograd on the
    bf16-operand-emulating oracle.  At this size the rounding noise averages out: measured worst tensor 2.7 % / cosine 0.99963
    (embedding), so the per-tensor gate is 5 % / 0.999 (a wrong small term, e.g. a sign error in a bias-sized gradient, fails
    it); the positional-encoding scalars, single numbers with heavy cancellation (measured 16 %), on sign and a factor 2."""
    torch.set_num_threads(16)
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.model.training import Adam
    cfg = fo.CONFIGS['LJ256']
    p = fo.init_params(cfg, seed=7)
    tok, dur, pit = fo.make_inputs('ragged', 32, 128, 1000, seed=401)
    mel_tgt = fo.make_mel_targets(dur, 80, seed=402)
    emu_out, emu_g = fo.loss_and_grads(p, cfg, tok, mel_tgt, dur, pit, emulate_bf16=True)
    model = ForwardTransformer(**cfg, train_dropout=False, train_graphs=True)
    model.set_weights(p)
    model._compile(Adam(1e-4))
    out = model.train_step(tok, mel_tgt, dur, pit)
    torch.cuda.synchronize()
    eng = model._get_engine()
    assert abs(float(out['loss']) - float(emu_out['loss'])) < 5e-4 * abs(float(emu_out['loss']))
    for k in ('mel', 'duration', 'pitch'):
        assert abs(float(out['losses'][k]) - float(emu_out['losses'][k])) < 2e-3 * abs(float(emu_out['losses'][k])) + 1e-4
    gscale = max(float(g.norm()) for g in emu_g.values())
    zero = {n for n, g in emu_g.items() if float(g.norm()) < 1e-6 * gscale}
    rows = _grad_report(eng, emu_g, zero, gscale)
    print('C3 full size vs bf16-emulating oracle: worst', [(n, round(r, 4), round(c, 5)) for r, c, n in rows[:5]])
    for r, c, n in rows:
        if n.endswith('pos_scalar'):
            assert c > 0 and r < 1.0, (n, r)
        else:
            assert r < 0.05 and c > 0.999, (n, r, c)


def test_train_step_gradients_against_reference_code_golden():
    """tests/golden/ref_train_c1.npz: loss and (sampled) gradients of one _train_step of the UNMODIFIED reference model
    (run on tests/tf_shim by tests/golden/make_golden_ref.py) -- the CUDA step against numbers the reference's code produced."""
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent / 'golden'))
    from make_golden_ref import grad_sample_index
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.model.training import Adam
    g = np.load(Path(__file__).resolve().parent / 'golden' / 'ref_train_c1.npz')
    cfg = dict(fo.CONFIGS['C1'], dropout_rate=0.0, predictors_dropout=0.0)
    p = fo.init_params(cfg, seed=7)
    tok, dur, pit = fo.make_inputs('ragged', int(g['B']), int(g['Tp']), int(g['Tm']), seed=int(g['seed']))
    mel_tgt = fo.make_mel_targets(dur, 80, seed=int(g['mel_seed']))
    model = ForwardTransformer(**cfg, train_dropout=False)
    model.set_weights(p)
    model._compile(Adam(1e-4))
    eng = model._get_engine()
    out = eng.forward_backward(tok, mel_tgt, dur, pit, training=True)
    torch.cuda.synchronize()
    assert abs(out['loss'].item() - float(g['loss'])) < 2e-3 * float(g['loss'])
    for k, key in (('mel', 'mel_loss'), ('duration', 'duration_loss'), ('pitch', 'pitch_loss')):
        assert abs(out['losses'][k].item() - float(g[key])) < 5e-3 * float(g[key]) + 1e-4
    gscale = max(float(g['n:' + n]) for n in eng.names)
    worst = []
    for n in eng.names:
        want = torch.from_numpy(g['g:' + n]).double()
        got = eng.g[n].detach().reshape(-1).cpu()[torch.from_numpy(grad_sample_index(n, eng.g[n].numel()))].double()
        if float(g['n:' + n]) < 1e-6 * gscale:
            assert float(got.norm()) < 2e-3 * gscale, n
            continue
        if want.numel() == 1:
            assert float(got) * float(want) > 0 and abs(float(got) - float(want)) < abs(float(want)), n
            continue
        worst.append((_rel(got, want), n))
    worst.sort(reverse=True)
    print('vs reference-code gradients: worst', worst[:5])
    assert worst[0][0] < 0.2, worst[:5]          # single-pass bf16 on a 3-row batch: ~0.11 measured (tools/grad_noise.py)


def _directional_check(train_dropout, eps):
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.model.training import Adam
    cfg = dict(fo.CONFIGS['C1'])
    p = fo.init_params(cfg, seed=7)
    tok, dur, pit = fo.make_inputs('ragged', 4, 24, 150, seed=311)
    mel_tgt = fo.make_mel_targets(dur, 80, seed=312)
    model = ForwardTransformer(**cfg, train_dropout=train_dropout)
    model.set_weights(p)
    model._compile(Adam(1e-4))
    eng = model._get_engine()
    out = eng.forward_backward(tok, mel_tgt, dur, pit, training=True)
    l0 = out['loss'].item()
    out_b = eng.forward_backward(tok, mel_tgt, dur, pit, training=True)
    assert abs(out_b['loss'].item() - l0) < 1e-5 * abs(l0)  # same step counter -> same masks (loss sum order may differ)
    l_eval = eng.forward_backward(tok, mel_tgt, dur, pit, training=False)['loss'].item()
    g = eng.flat_g.clone()
    v = g / g.norm()
    w0 = eng.flat_w.clone()
    vals = []
    for sgn in (1.0, -1.0):
        eng.flat_w.copy_(w0 + sgn * eps * v)
        vals.append(eng.forward_backward(tok, mel_tgt, dur, pit, training=True)['loss'].item())
    eng.flat_w.copy_(w0)
    return (vals[0] - vals[1]) / (2 * eps), g.norm().item(), l0, l_eval


def test_dropout_training_step_is_consistent():
    """Dropout on (rate 0.1 everywhere): masks are regenerated identically in the backward pass.  Checked through the
    directional derivative along the gradient with frozen masks, (L(w + e v) - L(w - e v)) / 2e ~= |g|, against the
    same check without dropout (the L1 loss is only piecewise linear, so the control calibrates the tolerance)."""
    fd0, g0, l0, le0 = _directional_check(False, 0.01)
    fd1, g1, l1, le1 = _directional_check(True, 0.01)
    print('no dropout: fd %.3f |g| %.3f ; dropout: fd %.3f |g| %.3f' % (fd0, g0, fd1, g1))
    assert abs(le0 - l0) < 1e-4 * abs(l0)       # without dropout train == eval forward
    assert abs(le1 - l1) > 1e-4                  # dropout really was active
    assert abs(fd0 / g0 - 1) < 0.1
    assert abs(fd1 / g1 - 1) < 0.1


def _run_train_tts(args, cwd, nproc=1, timeout=900):
    import subprocess
    import sys
    cmd = [sys.executable]
    if nproc > 1:
        cmd += ['-m', 'torch.distributed.run', '--nnodes=1', f'--nproc-per-node={nproc}', '--master-addr', '127.0.0.1',
                '--master-port', '29531']
    r = subprocess.run(cmd + [str(cwd / 'train_tts.py')] + args, capture_output=True, text=True, timeout=timeout, cwd=str(cwd))
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout


def _losses(stdout):
    import re
    return {int(m.group(1)): float(m.group(2)) for m in re.finditer(r'step (\d+)  loss ([0-9.]+)', stdout)}


def test_train_tts_driver_saves_and_resumes(tmp_path):
    """train_tts.py (loop contract of the reference's script) on synthetic batches: a checkpoint directory in the reference's
    layout (config.yaml + model_weights.hdf5, plus optimizer.pt) is written and loads back; a run that is stopped and
    restarted continues with the SAME loss curve as an uninterrupted run (weights, Adam moments, step counter, learning-rate
    schedule position, dropout seeds and the batch stream are all restored) -- reference train_tts.py:119-129."""
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    base = ['--config', str(root / 'config' / 'training_config.yaml'), '--synthetic', '--batch_size', '2', '--checkpoint_frequency', '1']
    full = _losses(_run_train_tts(base + ['--max_steps', '12', '--weights_dir', str(tmp_path / 'a')], root))
    assert set(full) >= {1, 10} and all(math.isfinite(v) for v in full.values())
    out1 = _run_train_tts(base + ['--max_steps', '5', '--weights_dir', str(tmp_path / 'b')], root)
    assert 'starting training from scratch' in out1
    out2 = _run_train_tts(base + ['--max_steps', '12', '--weights_dir', str(tmp_path / 'b')], root)
    assert 'resuming training from step 5' in out2 and 'Done.' in out2
    resumed = _losses(out2)
    # weight-gradient sums use fp32 atomics (order varies run to run): equal to rounding noise, not bit-identical
    assert abs(resumed[10] - full[10]) < 2e-3 * abs(full[10]), (resumed, full)
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.utils import hdf5_lite
    m = ForwardTransformer.load_model(str(tmp_path / 'b' / 'step_12'))
    assert m.config['encoder_model_dimension'] == 256 and m.step == 12 and m.optimizer.m is not None
    tree = hdf5_lite.read_hdf5(tmp_path / 'b' / 'step_12' / 'model_weights.hdf5')      # the Keras-format weight file
    assert [n.decode() for n in tree.attrs['layer_names']][:2] == ['Embedding', 'Encoder']
    (tmp_path / 'b' / 'step_12' / 'model_weights.pt').unlink()                          # load from the HDF5 file alone
    m2 = ForwardTransformer.load_model(str(tmp_path / 'b' / 'step_12'))
    for k, v in m.weights.items():
        assert torch.equal(v, m2.weights[k]), k


def _write_training_data(cm, n_train=40, n_valid=8, seed=1):
    """The on-disk layout of the reference's create_training_data.py / extract_durations.py, filled with random utterances."""
    from transformertts_b200.data.text import ALL_PHONEMES
    rng = np.random.default_rng(seed)
    for d in (cm.data_dir, cm.mel_dir, cm.duration_dir, cm.pitch_per_char):
        d.mkdir(parents=True, exist_ok=True)
    letters = [c for c in ALL_PHONEMES if c.isalpha()][:30] + [' ']
    for meta, n, tag in ((cm.train_metadata_path, n_train, 't'), (cm.valid_metadata_path, n_valid, 'v')):
        lines = []
        for i in range(n):
            n_tok = int(rng.integers(8, 30))
            dur = rng.integers(1, 7, n_tok).astype(np.int32)
            name = f'{tag}{i:03d}'
            np.save(cm.mel_dir / f'{name}.npy', np.clip(rng.normal(-5, 2, (int(dur.sum()), 80)), -11.5, 2).astype(np.float32))
            np.save(cm.duration_dir / f'{name}.npy', dur)
            np.save(cm.pitch_per_char / f'{name}.npy', rng.normal(0, 1, n_tok).astype(np.float32))
            lines.append(f'{name}|' + ''.join(rng.choice(letters, n_tok)) + ('?' if i % 7 == 0 else '') * 0 + '\n')
        meta.write_text(''.join(lines), encoding='utf-8')


def _data_config(tmp_path):
    import yaml
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    raw = yaml.safe_load((root / 'config' / 'training_config.yaml').read_text())
    raw.setdefault('paths', {}).update(log_directory=str(tmp_path / 'logs'), train_data_directory=str(tmp_path / 'data'))
    raw['training_data_settings'].update(bucket_boundaries=[60, 100], bucket_batch_sizes=[8, 6, 4], val_bucket_batch_size=[4, 4, 2])
    raw['tts_settings'].update(validation_frequency=3, weights_save_frequency=1000, max_steps=4)
    cfg_path = tmp_path / 'cfg.yaml'
    cfg_path.write_text(yaml.safe_dump(raw))
    return cfg_path


def test_train_tts_from_disk_dataset(tmp_path):
    """SURVEY 8(f) row 3 wired in: train_tts.py reads per-utterance .npy files + metadata through data/datasets.py (bucketing,
    pinned batches, side-stream prefetch), trains and validates."""
    from pathlib import Path
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    root = Path(__file__).resolve().parent.parent
    cfg_path = _data_config(tmp_path)
    _write_training_data(TrainingConfigManager(str(cfg_path)))
    out = _run_train_tts(['--config', str(cfg_path), '--max_steps', '4'], root)
    losses = _losses(out)
    assert 1 in losses and math.isfinite(losses[1]) and 'validation loss at step 3' in out and 'Done.' in out


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_train_tts_from_disk_dataset_data_parallel(tmp_path):
    """The same under torchrun with 2 ranks: each rank takes its row slice of every global batch, NCCL all-reduce of the
    gradient buckets, identical weights on both ranks afterwards (checked through the printed loss being finite and the run
    completing; weight equality across ranks is asserted in tests/test_gpu_dp.py)."""
    from pathlib import Path
    from transformertts_b200.utils.training_config_manager import TrainingConfigManager
    root = Path(__file__).resolve().parent.parent
    cfg_path = _data_config(tmp_path)
    _write_training_data(TrainingConfigManager(str(cfg_path)))
    out = _run_train_tts(['--config', str(cfg_path), '--max_steps', '4'], root, nproc=2)
    assert 'validation loss at step 3' in out and 'Done.' in out


def test_prefetch_loader_feeds_training_steps(tmp_path):
    """Row f-3 end to end: per-utterance .npy files -> bucketed, padded, pinned batches -> side-stream H2D -> train_step."""
    from transformertts_b200.data import datasets as ds
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.model.training import Adam
    rng = np.random.default_rng(1)
    for d in ('mels', 'durations', 'pitch_char'):
        (tmp_path / d).mkdir()
    lines = []
    for i in range(24):
        n_tok = int(rng.integers(8, 24))
        dur = rng.integers(1, 6, n_tok).astype(np.int32)
        np.save(tmp_path / 'mels' / f'u{i}.npy', rng.normal(-5, 2, (int(dur.sum()), 80)).astype(np.float32))
        np.save(tmp_path / 'durations' / f'u{i}.npy', dur)
        np.save(tmp_path / 'pitch_char' / f'u{i}.npy', rng.normal(0, 1, n_tok).astype(np.float32))
        lines.append(f'u{i}|' + ''.join(chr(97 + int(c)) for c in rng.integers(0, 26, n_tok)) + '\n')
    (tmp_path / 'train.txt').write_text(''.join(lines))
    reader = ds.DataReader(tmp_path / 'train.txt', training=True, is_processed=True)
    data = ds.TTSDataset(reader, ds.TTSPreprocessor(80, lambda t: [1 + (ord(c) % 100) for c in t]), tmp_path / 'mels',
                         tmp_path / 'durations', tmp_path / 'pitch_char')
    loader = ds.PrefetchLoader(data.get_dataset(bucket_batch_sizes=[4, 4], bucket_boundaries=[60], drop_remainder=True), prefetch=2,
                               device=DEV)
    model = ForwardTransformer(**fo.CONFIGS['C1'])
    model._compile(Adam(1e-4))
    try:
        for _ in range(3):
            b = loader.next()
            assert b['mel'].is_cuda and b['tokens'].dtype == torch.int32
            out = model.train_step(b['tokens'], b['mel'], b['durations'], b['pitch'])
            assert math.isfinite(out['loss'].item())
    finally:
        loader.close()
    assert model.step == 3


def test_graphed_training_step_equals_eager_step():
    """train_graphs=True replays the step as two CUDA graphs.  Without dropout the graphed step must reproduce the eager step
    (same kernels, same arguments; weight-gradient sums use fp32 atomics, so equality is to rounding noise); with dropout the
    per-step salt must change the masks from step to step and keep forward and backward masks consistent."""
    from transformertts_b200.model.models import ForwardTransformer
    from transformertts_b200.model.training import Adam
    cfg = fo.CONFIGS['C1']
    p = fo.init_params(cfg, seed=7)
    tok, dur, pit = fo.make_inputs('ragged', 4, 24, 150, seed=321)
    mel_tgt = fo.make_mel_targets(dur, 80, seed=322)
    models = []
    for graphs in (False, True):
        m = ForwardTransformer(**cfg, train_dropout=False, train_graphs=graphs)
        m.set_weights(p)
        m._compile(Adam(1e-4))
        losses = [float(m.train_step(tok, mel_tgt, dur, pit)['loss']) for _ in range(4)]
        models.append((m, losses))
    (me, le), (mg, lg) = models
    # The first steps agree to fp32 rounding (measured 1e-7).  Later ones drift: the order of the fp32 atomics in the weight
    # gradients changes the last bit of an Adam update, a bf16 rounding of a re-packed weight flips, and with the loss falling
    # 12 % per step that is visible (measured up to 2.3e-4 at step 4, different from run to run).
    assert all(abs(a - b) < 2e-5 * abs(a) for a, b in zip(le[:2], lg[:2])), (le, lg)
    assert all(abs(a - b) < 2e-3 * abs(a) for a, b in zip(le, lg)), (le, lg)
    assert le[3] < le[0]                                                       # the steps do train
    we, wg = me._get_engine().flat_w, mg._get_engine().flat_w
    # 4 Adam steps of lr 1e-4: a parameter whose gradient is rounding noise around zero (key biases) moves by +-lr per step with
    # a sign set by the order of fp32 atomics, so two runs may drift apart by up to 2*lr per step there; everything else agrees
    assert float((we - wg).abs().max()) < 8.5e-4
    assert float((we - wg).abs().mean()) < 2e-6
    assert mg.step == 4 and len(mg._get_engine()._graphs) == 1
    # another shape gets its own graphs; the first one still replays
    tok2, dur2, pit2 = fo.make_inputs('ragged', 3, 24, 120, seed=323)
    mg.train_step(tok2, fo.make_mel_targets(dur2, 80, seed=324), dur2, pit2)
    assert len(mg._get_engine()._graphs) == 2 and math.isfinite(float(mg.train_step(tok, mel_tgt, dur, pit)['loss']))
    # dropout on: the loss on the same batch changes from step to step (new masks), and the directional derivative along the
    # gradient matches |g| (forward and backward of one step use the same masks)
    md = ForwardTransformer(**cfg, train_dropout=True, train_graphs=True)
    md.set_weights(p)
    md._compile(Adam(0.0))                                                     # lr 0: weights stay put
    l = [float(md.train_step(tok, mel_tgt, dur, pit)['loss']) for _ in range(3)]
    assert abs(l[0] - l[1]) > 1e-4 and abs(l[1] - l[2]) > 1e-4
    # eager evaluation afterwards is unaffected by the salt left in the library (no dropout in val_step)
    mv = ForwardTransformer(**cfg, train_dropout=False)
    mv.set_weights(p)
    mv._compile(Adam(0.0))
    v1, v2 = float(md.val_step(tok, mel_tgt, dur, pit)['loss']), float(mv.val_step(tok, mel_tgt, dur, pit)['loss'])
    assert abs(v1 - v2) < 1e-6 * abs(v2)


@pytest.mark.parametrize('C', [128, 256, 384])
def test_layernorm_bwd_vectorised_and_fused_column_sums(C):
    """The vectorised persistent LayerNorm-backward kernel (C == ld, C % 128 == 0) against fp64 autograd, and the fused
    ReLU-mask + bias-gradient pass / the three-output column sum against their two-step definitions."""
    lib = _lib()
    g = torch.Generator().manual_seed(5)
    B, T = 5, 333
    u = torch.randn(B, T, C, generator=g)
    dz = torch.randn(B, T, C, generator=g)
    gamma = 1 + 0.1 * torch.randn(C, generator=g)
    lens = torch.tensor([333, 100, 0, 250, 333], dtype=torch.int32)
    uu = u.double().requires_grad_(True)
    gg = gamma.double().requires_grad_(True)
    bb = torch.zeros(C, dtype=torch.float64, requires_grad=True)
    keep = (torch.arange(T)[None] < lens[:, None])[..., None].double()
    (fo.layer_norm(uu, gg, bb) * keep * dz.double()).sum().backward()
    du = torch.full((B, T, C), float('nan'), device=DEV)
    gb = torch.full((B, T, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    dg, db, dbias = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    lib.layernorm_bwd(dz.to(DEV), u.to(DEV), gamma.to(DEV), B, T, C, C, 1e-6, lens.to(DEV), False, du, gb, dg, db, dbias=dbias)
    torch.cuda.synchronize()
    assert _rel(du, uu.grad) < 1e-5
    assert _rel(dg, gg.grad) < 1e-5 and _rel(db, bb.grad) < 1e-5
    assert _rel(gb.float(), uu.grad) < 5e-3 and _rel(dbias, uu.grad.sum((0, 1))) < 1e-4
    # relu mask + bias gradient in one pass
    h = torch.randn(B, T, C, generator=g).bfloat16().to(DEV)
    dy = torch.randn(B, T, C, generator=g).bfloat16().to(DEV)
    want = dy.float() * (h.float() > 0)
    cs = torch.zeros(C, device=DEV)
    lib.relu_bwd_colsum(dy, h, cs)
    torch.cuda.synchronize()
    assert torch.equal(dy.float(), want) and _rel(cs, want.sum((0, 1))) < 1e-5
    # q | k | v column sums of one (rows, 3C) buffer into three outputs
    x = torch.randn(B * T, 3 * C, generator=g).bfloat16().to(DEV)
    o = [torch.zeros(C, device=DEV) for _ in range(3)]
    lib.colsum_bf16_x3(x, B * T, C, 3 * C, *o)
    torch.cuda.synchronize()
    for k in range(3):
        assert _rel(o[k], x[:, k * C:(k + 1) * C].float().sum(0)) < 1e-5


@pytest.mark.parametrize('H,dh,T,rate', [(2, 128, 1000, 0.1), (2, 64, 333, 0.1), (2, 192, 200, 0.0), (1, 128, 130, 0.25)])
def test_fused_attention_probabilities_match_two_kernel_path(H, dh, T, rate):
    """ttsb_attn_probs_fwd (logits in registers, two passes) against the materialised path (ttsb_bgemm fp32 logits +
    ttsb_softmax_fwd) and an fp64 softmax: same probabilities to bf16 rounding, identical dropout decisions, exact zeros on
    masked keys and padded query rows, poisoned outputs fully overwritten."""
    lib = _lib()
    from transformertts_b200.model.training import TrainEngine
    from transformertts_b200.model.models import _round_up
    g = torch.Generator().manual_seed(5)
    B, d = 4, H * dh
    qkv = (torch.randn(B, T, 3 * d, generator=g) * 1.5).bfloat16()
    lens = torch.tensor([T, max(T // 2, 1), min(70, T), 1], dtype=torch.int32)
    qkv_d, lens_d = qkv.to(DEV), lens.to(DEV)
    Z, ldp = B * H, _round_up(T, 16)
    eng = TrainEngine.__new__(TrainEngine)
    eng.dev = torch.device(DEV)
    S = torch.empty(Z, T, ldp, device=DEV)
    eng._bgemm(B, H, T, T, dh, qkv_d, (3 * d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 0), qkv_d, (2 * d, T, B), (3 * d, 3 * d * T),
               (dh, 0, 0, d), alpha=1.0 / math.sqrt(dh), out_f32=S, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp)
    seed, site = 77, 5
    P0 = torch.full((Z, T, ldp), float('nan'), dtype=torch.bfloat16, device=DEV)
    D0 = torch.full((Z, T, ldp), float('nan'), dtype=torch.bfloat16, device=DEV) if rate > 0 else P0
    lib.softmax_fwd(S, B, H, T, T, ldp, lens_d, rate, seed, site, P0, D0)
    P1 = torch.full((Z, T, ldp), float('nan'), dtype=torch.bfloat16, device=DEV)
    D1 = torch.full((Z, T, ldp), float('nan'), dtype=torch.bfloat16, device=DEV) if rate > 0 else P1
    assert lib.attn_probs_supported(dh, ldp)
    lib.attn_probs_fwd(qkv_d, 3 * d, 0, d, B, H, T, dh, lens_d, 1.0 / math.sqrt(dh), rate, seed, site, P1, D1, ldp)
    torch.cuda.synchronize()
    assert torch.isfinite(P1.float()).all() and torch.isfinite(D1.float()).all()
    p0, p1, d0, d1 = P0.float().cpu(), P1.float().cpu(), D0.float().cpu(), D1.float().cpu()
    # fp64 reference on the bf16 inputs
    x = qkv.double()
    q, k = [t.reshape(B, T, H, dh).permute(0, 2, 1, 3) for t in x.split(d, dim=-1)[:2]]
    logits = q @ k.transpose(-1, -2) / math.sqrt(dh)
    kmask = torch.arange(T)[None, :] >= lens[:, None]
    w = torch.softmax(logits.masked_fill(kmask[:, None, None, :], float('-inf')), -1)
    w = w * (torch.arange(T)[None, :] < lens[:, None])[:, None, :, None]           # padded query rows are written as zeros
    w = w.reshape(Z, T, T)
    assert (p1[:, :, T:] == 0).all() and (d1[:, :, T:] == 0).all()
    assert (p1[:, :, :T][w == 0] == 0).all()
    err = (p1[:, :, :T].double() - w).abs()
    assert float((err / (w + 1e-6)).max()) < 6e-3                                  # bf16 rounding (2^-9) + ex2.approx
    assert float((p1 - p0).abs().max()) <= float(p0.abs().max()) * 2 ** -7         # the two CUDA paths agree to one bf16 ulp
    if rate > 0:
        big = p1 > 1e-30
        assert ((d1 != 0) == (d0 != 0))[big & (p0 > 1e-30)].all()                  # identical keep decisions
        kept = (d1 != 0)
        assert abs(float(kept[big].float().mean()) - (1 - rate)) < 0.01
        ratio = d1[kept] / p1[kept]
        assert float((ratio - 1 / (1 - rate)).abs().max()) < 0.01 / (1 - rate)
        assert (d1[~big] == 0).all()


@pytest.mark.parametrize('H,dh,T,rate', [(2, 128, 1000, 0.1), (2, 64, 333, 0.1), (2, 192, 200, 0.0), (1, 128, 130, 0.25)])
def test_fused_attention_ds_matches_bgemm_epilogue_and_fp64(H, dh, T, rate):
    """ttsb_attn_ds_bwd against the fused dS epilogue of ttsb_bgemm (same formula, same dropout hash) and against an fp64
    evaluation of scale * P * (mask * dP / (1-p) - D) on the same bf16 inputs and the same mask."""
    lib = _lib()
    from transformertts_b200.model.training import TrainEngine
    from transformertts_b200.model.models import _round_up
    g = torch.Generator().manual_seed(9)
    B, d = 4, H * dh
    qkv = torch.randn(B, T, 3 * d, generator=g).bfloat16()
    dO = torch.randn(B, T, d, generator=g).bfloat16()
    lens = torch.tensor([T, max(T // 2, 1), min(70, T), 1], dtype=torch.int32)
    Z, ldp = B * H, _round_up(T, 16)
    Pm = torch.rand(Z, T, ldp, generator=g)
    kmask = (torch.arange(ldp)[None, :] < lens[:, None]).repeat_interleave(H, 0)[:, None, :]
    qmask = (torch.arange(T)[None, :] < lens[:, None]).repeat_interleave(H, 0)[:, :, None]
    Pm = (Pm * kmask * qmask / Pm.sum(-1, keepdim=True).clamp_min(1e-3)).bfloat16()
    D = torch.randn(Z * T, generator=g) * 0.1
    qkv_d, dO_d, lens_d, P_d, D_d = qkv.to(DEV), dO.to(DEV), lens.to(DEV), Pm.to(DEV), D.to(DEV)
    eng = TrainEngine.__new__(TrainEngine)
    eng.dev = torch.device(DEV)
    seed, site, scale = 31, 4, 1.0 / math.sqrt(dh)
    dS0 = torch.full((Z, T, ldp), float('nan'), dtype=torch.bfloat16, device=DEV)
    eng._bgemm(B, H, T, T, dh, dO_d, (d, T, B), (d, d * T), (dh, 0, 0, 0), qkv_d, (d, T, B), (3 * d, 3 * d * T), (dh, 0, 0, 2 * d),
               out_bf16=dS0, ld_out=ldp, out_batch_stride=T * ldp, out_cols=ldp,
               softmax_bwd=(P_d, D_d, scale, rate, seed, site, 0, lens_d, None))
    dS1 = torch.full((Z, T, ldp), float('nan'), dtype=torch.bfloat16, device=DEV)
    assert lib.attn_probs_supported(dh, ldp)
    lib.attn_ds_bwd(dO_d, d, 0, qkv_d, 3 * d, 2 * d, B, H, T, dh, lens_d, P_d, D_d, scale, rate, seed, site, dS1, ldp)
    torch.cuda.synchronize()
    a, b = dS0.float().cpu(), dS1.float().cpu()
    assert torch.isfinite(b).all()
    assert float((a - b).abs().max()) <= 2 ** -7 * float(a.abs().max()) + 1e-6       # same arithmetic up to fma contraction
    assert ((b == 0) | (kmask & qmask).expand_as(b)).all()                            # zeros on masked keys / padded rows
    # fp64 with the mask read back from the forward kernel's P_drop (same hash, same element index)
    if rate > 0:
        Pd = torch.empty(Z, T, ldp, dtype=torch.bfloat16, device=DEV)
        S = torch.zeros(Z, T, ldp, device=DEV)
        lib.softmax_fwd(S, B, H, T, T, ldp, lens_d, rate, seed, site, torch.empty_like(Pd), Pd)   # uniform rows: P > 0 on live keys
        keep = (Pd.float().cpu() != 0).double()
    else:
        keep = torch.ones(Z, T, ldp, dtype=torch.float64)
    v = qkv.double()[..., 2 * d:].reshape(B, T, H, dh).permute(0, 2, 1, 3).reshape(Z, T, dh)
    do = dO.double().reshape(B, T, H, dh).permute(0, 2, 1, 3).reshape(Z, T, dh)
    dP = torch.zeros(Z, T, ldp, dtype=torch.float64)
    dP[:, :, :T] = do @ v.transpose(-1, -2)
    ref = scale * Pm.double() * (keep * dP / (1 - rate) - D.double().reshape(Z, T, 1)) * (kmask & qmask)
    err = (b.double() - ref).abs()
    assert float(err.max()) < 8e-3 * float(ref.abs().max()) + 1e-6, float(err.max())
