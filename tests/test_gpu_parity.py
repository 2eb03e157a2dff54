"""-m gpu parity tests: the CUDA path (through the C ABI, via the host-side mirror) against
  (a) the committed golden fixtures produced by the live reference, and
  (b) the CPU oracle on seeded inputs,
for every kernel family and for the whole forward + loss + backward.  Tolerance: 1e-3 relative (fp32), bit-exact
argmax ids on real decoder positions.  Dropout is 0 in parity runs (SURVEY.md §8d)."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import asr_oracle as O
from tests.helpers import GOLDEN_CASES, assert_grads_close, grads_rel_err, load_golden, rel_err, vgg_pools_well_separated

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def b200_mod():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr


@pytest.fixture(params=["fp32", "default"])
def b200(request, b200_mod):
    """Every test runs twice: on the exact-fp32 CUDA-core kernels and on the package default (tensor-core GEMM/conv).
    `b200.k` scales the per-kernel tolerances (set for exact fp32) for the tensor-core mode; the end-to-end 1e-3 bar is
    the same in both."""
    import importlib
    ops = importlib.import_module(b200_mod.__name__ + ".ops")
    saved = (ops.config.linear, ops.config.conv, ops.config.conv_wgrad, ops.config.attn, ops.config.attn_bwd)
    if request.param == "fp32":
        ops.config.set(linear="fp32", conv="fp32", conv_wgrad="fp32", attn="fp32", attn_bwd="fp32")
        b200_mod.k = 1.0
    else:
        b200_mod.k = 20.0
    yield b200_mod
    ops.config.linear, ops.config.conv, ops.config.conv_wgrad, ops.config.attn, ops.config.attn_bwd = saved


def _ops(b200):
    import importlib
    return importlib.import_module(b200.__name__ + ".ops")


def _cases(*rows):
    """Parametrize rows whose last value is emb_trg_sharing (the decoder's output projection tied to its embedding, one
    parameter with a sunk GEMM gradient plus the embedding's returned one); untied rows keep their plain ids."""
    return [pytest.param(*r, id="-".join(str(v) for v in r[:-1]) + ("-tied" if r[-1] else "")) for r in rows]


def _untie(grads_o, grads):
    """The oracle's gradient dict lists a tied weight under both names; the model's named_parameters() under one."""
    return {k: v for k, v in grads_o.items() if k in grads}


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_golden_forward_loss_backward(b200, case):
    from tests.gpu_util import TOL, cuda_model, cuda_step
    cfg, P, G, io, smoothing = load_golden(case)
    model = cuda_model(cfg, P)
    pred, gold, hyp, loss, stats, grads = cuda_step(model, io["in.src"], io["in.lengths"], io["in.tgt"], smoothing)
    assert torch.equal(gold, io["out.gold"])
    assert rel_err(pred, io["out.pred"]) < TOL
    real = gold.ne(O.PAD)
    assert torch.equal(hyp[real], io["out.hyp"][real])               # bit-exact argmax token ids
    assert abs(loss.item() - io["out.loss"].item()) < TOL * abs(io["out.loss"].item())
    assert int(stats[2].item()) == int(io["out.num_correct"])
    assert int(stats[1].item()) == int(real.sum())
    assert_grads_close(grads, G, TOL, exact_kernels=b200.k == 1.0)


@pytest.mark.parametrize("feat,L,H,d,dk,dv,di,B,T,Tt,V,freq,tied", _cases(
    ("vgg_cnn", 2, 4, 128, 32, 32, 256, 2, 20, 9, 77, 41, False),
    ("", 2, 2, 64, 16, 32, 128, 4, 70, 13, 33, 161, False),
    ("emb_cnn", 1, 2, 64, 32, 32, 64, 2, 36, 6, 20, 161, False),
    ("vgg_cnn", 1, 8, 512, 64, 64, 2048, 2, 16, 12, 4364, 41, False),        # cfg2 architecture, 1 layer, small spectrogram
    ("vgg_cnn", 2, 4, 128, 32, 32, 256, 2, 20, 9, 77, 41, True),
    ("", 2, 2, 64, 16, 32, 128, 4, 70, 13, 33, 161, True),
))
def test_oracle_forward_loss_backward(b200, feat, L, H, d, dk, dv, di, B, T, Tt, V, freq, tied):
    from tests.gpu_util import TOL, cuda_model, cuda_step
    cfg = O.OracleConfig(num_layers=L, num_heads=H, dim_model=d, dim_key=dk, dim_value=dv, dim_inner=di, vocab=V,
                         feat_extractor=feat, tgt_max_len=Tt, freq=freq, emb_trg_sharing=tied)
    P = O.init_params(cfg, seed=3)
    g = torch.Generator().manual_seed(17)
    for k in sorted(P):             # move norm scales / biases off (1, 0)
        if P[k].dim() == 1:
            P[k] = P[k] + 0.1 * torch.randn(P[k].shape, generator=g)
    for seed in range(1, 200):      # max-pool routing is discontinuous: use an input without near-tied pooling windows
        src, lens, tgt = O.synthetic_batch(cfg, B, T, seed=seed, ragged=True)
        if feat != "vgg_cnn" or vgg_pools_well_separated(P, src):
            break
    # reference = the oracle evaluated in float64 ("truth"): separates our error from the fp32 oracle's own rounding,
    # which on its own flips ReLU / max-pool decisions in small models (SURVEY.md §8c)
    pred_o, gold_o, hyp_o, loss_o, n_word, grads_o = O.forward_backward({k: v.double() for k, v in P.items()}, cfg, src.double(),
                                                                        lens, tgt, 0.1)
    pred_o, loss_o = pred_o.float(), loss_o.float()
    grads_o = {k: v.float() for k, v in grads_o.items()}
    model = cuda_model(cfg, P)
    pred, gold, hyp, loss, stats, grads = cuda_step(model, src, lens, tgt, 0.1)
    assert torch.equal(gold, gold_o)
    assert rel_err(pred, pred_o) < TOL
    real = gold.ne(O.PAD)
    # argmax: identical ids wherever the oracle's top-2 margin exceeds the tolerance band (near-ties excluded)
    top2 = pred_o.topk(2, dim=2).values
    clear = real & ((top2[..., 0] - top2[..., 1]) > 2 * TOL * pred_o.abs().max())
    assert torch.equal(hyp[clear], hyp_o[clear])
    assert abs(loss.item() - loss_o.item()) < TOL * abs(loss_o.item())
    assert int(stats[1].item()) == n_word
    assert_grads_close(grads, _untie(grads_o, grads), TOL, exact_kernels=b200.k == 1.0)


# ------------------------------------------------------------------------------------------------ kernel families
@pytest.mark.parametrize("M,N,K", [(77, 50, 161), (300, 512, 512), (130, 4364, 128), (513, 128, 2048), (1, 8, 4)])
def test_linear_fwd_bwd(b200, M, N, K):
    ops = _ops(b200)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(M, K, generator=g, requires_grad=True)
    w = torch.randn(N, K, generator=g, requires_grad=True) * 0.1
    w = w.detach().requires_grad_(True)
    b = torch.randn(N, generator=g, requires_grad=True)
    y = F.linear(x, w, b)
    dy = torch.randn(M, N, generator=g)
    y.backward(dy)
    xc, wc, bc = (t.detach().cuda().requires_grad_(True) for t in (x, w, b))
    yc = ops.LinearFn.apply(xc, wc, bc)
    yc.backward(dy.cuda())
    assert rel_err(yc, y) < 1e-5 * b200.k
    assert rel_err(xc.grad, x.grad) < 1e-5 * b200.k
    assert rel_err(wc.grad, w.grad) < 1e-5 * b200.k
    assert rel_err(bc.grad, b.grad) < 1e-5 * b200.k


def test_ffn_fwd_bwd(b200):
    ops = _ops(b200)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(3, 41, 64, generator=g, requires_grad=True)
    w1 = (torch.randn(96, 64, 1, generator=g) * 0.2).requires_grad_(True)
    b1 = torch.randn(96, generator=g, requires_grad=True)
    w2 = (torch.randn(64, 96, 1, generator=g) * 0.2).requires_grad_(True)
    b2 = torch.randn(64, generator=g, requires_grad=True)
    y = F.linear(F.relu(F.linear(x, w1.squeeze(-1), b1)), w2.squeeze(-1), b2)
    dy = torch.randn_like(y)
    y.backward(dy)
    cs = [t.detach().cuda().requires_grad_(True) for t in (x, w1, b1, w2, b2)]
    yc = ops.FFNFn.apply(*cs)
    yc.backward(dy.cuda())
    assert rel_err(yc, y) < 1e-5 * b200.k
    for c, r in zip(cs, (x, w1, b1, w2, b2)):
        assert rel_err(c.grad, r.grad) < 1e-5 * b200.k


@pytest.mark.parametrize("rows,T,d,with_res,with_pe,with_scale", [(37, 37, 64, True, False, True), (120, 40, 512, False, True, False),
                                                                  (9, 3, 768, True, True, True), (5, 5, 128, True, False, False)])
def test_add_layernorm_fwd_bwd(b200, rows, T, d, with_res, with_pe, with_scale):
    ops = _ops(b200)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(rows, d, generator=g, requires_grad=True)
    res = torch.randn(rows, d, generator=g, requires_grad=True) if with_res else None
    gamma = (1 + 0.1 * torch.randn(d, generator=g)).requires_grad_(True)
    beta = (0.1 * torch.randn(d, generator=g)).requires_grad_(True)
    pe = torch.randn(T, d, generator=g) if with_pe else None
    rs = (torch.rand(rows, generator=g) > 0.3).float() if with_scale else None
    z = x + res if with_res else x
    y = F.layer_norm(z, (d,), gamma, beta)
    if with_pe:
        y = y + pe.repeat(rows // T, 1)
    if with_scale:
        y = y * rs.unsqueeze(1)
    dy = torch.randn(rows, d, generator=g)
    y.backward(dy)
    cu = lambda t: None if t is None else t.detach().cuda().requires_grad_(t.requires_grad)
    xc, rc, gc, bc = cu(x), cu(res), cu(gamma), cu(beta)
    yc = ops.AddLNFn.apply(xc, rc, gc, bc, cu(pe), cu(rs), 1e-5, 0.0)
    yc.backward(dy.cuda())
    assert rel_err(yc, y) < 1e-5
    assert rel_err(xc.grad, x.grad) < 1e-4
    if with_res:
        assert rel_err(rc.grad, res.grad) < 1e-4
    assert rel_err(gc.grad, gamma.grad) < 1e-4
    assert rel_err(bc.grad, beta.grad) < 1e-4


@pytest.mark.parametrize("feat,L,H,d,dk,dv,di,B,T,Tt,V,freq,tied", _cases(
    ("vgg_cnn", 2, 4, 128, 32, 32, 256, 2, 20, 9, 77, 41, False),
    ("", 2, 2, 64, 32, 64, 128, 3, 50, 11, 33, 161, False),           # dk != dv: the stacked Q|K|V rows differ in width
    ("vgg_cnn", 2, 4, 128, 32, 32, 256, 2, 20, 9, 77, 41, True),
    ("", 2, 2, 64, 32, 64, 128, 3, 50, 11, 33, 161, True),
))
def test_flat_params_stack_qkv_projections(b200, feat, L, H, d, dk, dv, di, B, T, Tt, V, freq, tied):
    """optim.FlatParams lays W_q|W_k|W_v (and biases, and their gradients) back to back, which makes ops.AttnProjFn run
    the projections as one stacked GEMM with the weight / bias gradients accumulated straight into the flat buffer
    (self-attention: Q|K|V, encoder-decoder attention: K|V).  Same oracle, same tolerance as the separate-GEMM path."""
    from tests.gpu_util import TOL, cuda_model, cuda_step
    ops = _ops(b200)
    cfg = O.OracleConfig(num_layers=L, num_heads=H, dim_model=d, dim_key=dk, dim_value=dv, dim_inner=di, vocab=V,
                         feat_extractor=feat, tgt_max_len=Tt, freq=freq, emb_trg_sharing=tied)
    P = O.init_params(cfg, seed=5)
    for seed in range(1, 200):
        src, lens, tgt = O.synthetic_batch(cfg, B, T, seed=seed, ragged=True)
        if feat != "vgg_cnn" or vgg_pools_well_separated(P, src):
            break
    pred_o, gold_o, hyp_o, loss_o, n_word, grads_o = O.forward_backward({k: v.double() for k, v in P.items()}, cfg, src.double(),
                                                                        lens, tgt, 0.1)
    model = cuda_model(cfg, P)
    flat = b200.FlatParams(model)
    att = model.encoder.layers[0].self_attn
    ws = [att.query_linear.weight, att.key_linear.weight, att.value_linear.weight]
    assert ops._adjacent(*ws) and ops._adjacent(*[w.grad for w in ws])          # the layout the fused path keys on
    cross = model.decoder.layers[0].encoder_attn
    assert ops._adjacent(cross.key_linear.weight, cross.value_linear.weight)
    flat.zero_grad()
    pred, gold, hyp, _ = model(src.cuda(), lens, tgt.cuda())
    loss, stats = b200.loss_and_stats(pred, gold, 0.1)
    loss.backward()
    flat.ensure_grad_views()
    grads = {n: p.grad.detach().cpu() for n, p in model.named_parameters()}
    assert rel_err(pred.cpu(), pred_o.float()) < TOL
    assert abs(loss.item() - loss_o.item()) < TOL * abs(loss_o.item())
    assert_grads_close(grads, {k: v.float() for k, v in _untie(grads_o, grads).items()}, TOL, exact_kernels=b200.k == 1.0)


def _attention_case(ops, B, H, Tq, Tk, dk, dv, mode, seed=0):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Tq, H * dk, generator=g, requires_grad=True)
    k = torch.randn(B, Tk, H * dk, generator=g, requires_grad=True)
    v = torch.randn(B, Tk, H * dv, generator=g, requires_grad=True)
    key_pad = dense = None
    causal = False
    mask = torch.zeros(B, Tq, Tk, dtype=torch.bool)
    if mode in ("keypad", "causal+keypad"):
        lens = torch.randint(max(1, Tk // 2), Tk + 1, (B,), generator=g)
        key_pad = (torch.arange(Tk)[None, :] >= lens[:, None])
        if mode == "causal+keypad":
            key_pad[:, 0] = False
        mask |= key_pad[:, None, :]
    if mode in ("causal", "causal+keypad"):
        causal = True
        mask |= torch.triu(torch.ones(Tq, Tk, dtype=torch.bool), diagonal=1)[None]
    if mode == "dense":
        dense = torch.rand(B, Tq, Tk, generator=g) < 0.3
        dense[:, :, 0] = False
        mask |= dense
    # oracle in the reference's head-major layout
    qh = q.view(B, Tq, H, dk).permute(2, 0, 1, 3).reshape(H * B, Tq, dk)
    kh = k.view(B, Tk, H, dk).permute(2, 0, 1, 3).reshape(H * B, Tk, dk)
    vh = v.view(B, Tk, H, dv).permute(2, 0, 1, 3).reshape(H * B, Tk, dv)
    o, _ = O.scaled_dot_attention(qh, kh, vh, mask.repeat(H, 1, 1), float(dk) ** 0.5)
    o = o.view(H, B, Tq, dv).permute(1, 2, 0, 3).reshape(B, Tq, H * dv)
    do = torch.randn(B, Tq, H * dv, generator=g)
    o.backward(do)
    qc, kc, vc = (t.detach().cuda().requires_grad_(True) for t in (q, k, v))
    u8 = lambda t: None if t is None else t.to(torch.uint8).cuda().contiguous()
    oc = ops.SdpaFn.apply(qc.view(B, Tq, H, dk).permute(0, 2, 1, 3), kc.view(B, Tk, H, dk).permute(0, 2, 1, 3),
                          vc.view(B, Tk, H, dv).permute(0, 2, 1, 3), u8(key_pad), u8(dense), causal, 1.0 / math.sqrt(dk), 0.0)
    oc = oc.permute(0, 2, 1, 3).reshape(B, Tq, H * dv)
    oc.backward(do.cuda())
    return (oc, o), (qc.grad, q.grad), (kc.grad, k.grad), (vc.grad, v.grad)


@pytest.mark.parametrize("B,H,Tq,Tk,dk,dv,mode", [
    (2, 2, 50, 50, 64, 64, "keypad"), (3, 4, 13, 13, 32, 32, "causal+keypad"), (2, 8, 100, 200, 64, 64, "keypad"),
    (2, 3, 70, 70, 16, 32, "dense"), (1, 2, 129, 65, 128, 128, "none"), (2, 2, 64, 64, 64, 64, "causal"),
    (1, 1, 200, 200, 64, 64, "keypad"),
])
def test_attention_fwd_bwd(b200, B, H, Tq, Tk, dk, dv, mode):
    pairs = _attention_case(_ops(b200), B, H, Tq, Tk, dk, dv, mode)
    for got, ref in pairs:
        assert rel_err(got, ref) < 2e-5


def test_attention_fully_masked_row_is_nan_like_reference(b200):
    ops = _ops(b200)
    q = torch.randn(1, 1, 4, 16).cuda(); k = torch.randn(1, 1, 6, 16).cuda(); v = torch.randn(1, 1, 6, 16).cuda()
    key_pad = torch.ones(1, 6, dtype=torch.uint8).cuda()
    o = ops.SdpaFn.apply(q, k, v, key_pad, None, False, 0.25, 0.0)
    assert torch.isnan(o).all()


@pytest.mark.parametrize("B,F_,T", [(2, 41, 24), (1, 161, 12), (3, 23, 10)])
def test_vgg_frontend_fwd_bwd(b200, B, F_, T):
    ops = _ops(b200)
    cfg = O.OracleConfig(num_layers=1, feat_extractor="vgg_cnn", freq=F_)
    P = {k: v.requires_grad_(True) for k, v in O.init_params(cfg, seed=5).items() if k.startswith("conv.")}
    for seed in range(4, 200):                                # first input without max-pool near-ties
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(B, 1, F_, T, generator=g)
        if vgg_pools_well_separated(P, x):
            break
    y = O.vgg_frontend(x, P)                                  # (B,128,F/4,T/4)
    dy = torch.randn(y.shape, generator=g)
    y.backward(dy)
    names = ["conv.0.weight", "conv.0.bias", "conv.2.weight", "conv.2.bias", "conv.5.weight", "conv.5.bias", "conv.7.weight", "conv.7.bias"]
    cs = [P[n].detach().cuda().requires_grad_(True) for n in names]
    yc = ops.VggFrontendFn.apply(x.cuda(), *cs)               # [B,T/4,F/4,128]
    yc.backward(dy.permute(0, 3, 2, 1).contiguous().cuda())
    assert rel_err(yc.permute(0, 3, 2, 1), y) < 1e-5 * b200.k
    # The tensor-core mode differs from fp32 by ~1e-5, enough to flip max-pool / ReLU decisions on near-tied windows
    # (a discontinuity of the model, not of the kernels).  If the input is free of such windows at that noise level the
    # max-norm bound applies; otherwise the few moved gradient entries are bounded in the L2 norm.
    strict = b200.k == 1.0 or vgg_pools_well_separated(P, x, rel_gap=1e-4)
    for c, n in zip(cs, names):
        if strict:
            assert rel_err(c.grad, P[n].grad) < 1e-4 * b200.k, n
        else:
            g, r = c.grad.detach().cpu().double(), P[n].grad.double()
            assert float((g - r).norm() / r.norm()) < 2e-2, n


def test_emb_frontend_fwd_bwd(b200):
    ops = _ops(b200)
    cfg = O.OracleConfig(num_layers=1, feat_extractor="emb_cnn")
    P = {k: v for k, v in O.init_params(cfg, seed=6).items() if k.startswith("conv.")}
    g = torch.Generator().manual_seed(5)
    for k in ("conv.1.weight", "conv.1.bias", "conv.4.weight", "conv.4.bias"):
        P[k] = P[k] + 0.2 * torch.randn(P[k].shape, generator=g)
    P = {k: v.requires_grad_(True) for k, v in P.items()}
    x = torch.randn(3, 1, 161, 38, generator=g)
    y = O.flatten_features(O.emb_frontend(x, P))
    dy = torch.randn(y.shape, generator=g)
    y.backward(dy)
    names = ["conv.0.weight", "conv.0.bias", "conv.1.weight", "conv.1.bias", "conv.3.weight", "conv.3.bias", "conv.4.weight", "conv.4.bias"]
    cs = [P[n].detach().cuda().requires_grad_(True) for n in names]
    yc = ops.EmbFrontendFn.apply(x.cuda(), *cs, 1e-5)
    yc.backward(dy.cuda())
    assert rel_err(yc, y) < 1e-4
    errs = grads_rel_err({n: c.grad for n, c in zip(names, cs)}, {n: P[n].grad for n in names})
    assert max(errs.values()) < 1e-3, errs


def test_emb_frontend_rejects_other_weight_shapes(b200_mod):
    """At the default (tensor-core) precision the front end's kernels are given the reference's geometry, so any other
    weight shape is refused before a kernel is launched: it would be read out of bounds."""
    ops = _ops(b200_mod)
    assert ops.config.conv != b200_mod._lib.PREC_FP32
    lib = b200_mod._lib.load()
    r = lambda *s: torch.randn(s, device="cuda")
    x, w0, w3 = r(2, 1, 161, 38), r(32, 1, 41, 11), r(32, 32, 21, 11)
    for a, b in ((r(32, 1, 21, 11), w3), (w0, r(32, 32, 11, 11)), (r(16, 1, 41, 11), r(16, 16, 21, 11))):
        v = [r(a.shape[0]) for _ in range(6)]
        n0 = lib.b200asr_launch_count()
        with pytest.raises(RuntimeError, match=r"\(32, 1, 41, 11\) and \(32, 32, 21, 11\)"):
            ops.EmbFrontendFn.apply(x, a, v[0], v[1], v[2], b, v[3], v[4], v[5], 1e-5)
        assert lib.b200asr_launch_count() == n0


def test_emb_frontend_batchnorm_state_and_eval_mode(b200):
    """nn.BatchNorm2d state of the emb_cnn front end (models/asr/transformer.py:34,38): three training steps update
    running_mean / running_var / num_batches_tracked exactly as torch does, and model.eval() normalises with them."""
    from tests.gpu_util import TOL, cuda_model
    cfg = O.OracleConfig(num_layers=1, num_heads=2, dim_model=64, dim_key=32, dim_value=32, dim_inner=64, vocab=30,
                         feat_extractor="emb_cnn", tgt_max_len=8)
    P = O.init_params(cfg, seed=3)
    g = torch.Generator().manual_seed(9)
    for k in ("conv.1.weight", "conv.1.bias", "conv.4.weight", "conv.4.bias"):
        P[k] = P[k] + 0.2 * torch.randn(P[k].shape, generator=g)
    state = O.bn_initial_state()
    model = cuda_model(cfg, P)
    model.train()
    with torch.no_grad():
        for step in range(3):
            src, lens, tgt = O.synthetic_batch(cfg, 3, 44, seed=20 + step, ragged=False)
            O.transformer_forward(P, cfg, src, lens, tgt, training=True, bn_state=state)
            model(src.cuda(), lens, tgt.cuda())
    sd = model.state_dict()
    for i in (1, 4):
        assert int(sd[f"conv.{i}.num_batches_tracked"]) == 3 == int(state[f"conv.{i}.num_batches_tracked"])
        assert rel_err(sd[f"conv.{i}.running_mean"], state[f"conv.{i}.running_mean"]) < 1e-4
        assert rel_err(sd[f"conv.{i}.running_var"], state[f"conv.{i}.running_var"]) < 1e-4
    src, lens, tgt = O.synthetic_batch(cfg, 2, 44, seed=40, ragged=False)
    pred_o, _, _ = O.transformer_forward(P, cfg, src, lens, tgt, training=False, bn_state=state)
    model.eval()
    with torch.no_grad():
        pred, *_ = model(src.cuda(), lens, tgt.cuda())
    assert rel_err(pred, pred_o) < TOL
    assert int(model.state_dict()["conv.1.num_batches_tracked"]) == 3          # eval does not touch the state
    pred_t, _, _ = O.transformer_forward(P, cfg, src, lens, tgt, training=True, bn_state=None)
    assert rel_err(pred_t, pred_o) > 10 * TOL                                  # ... and differs from batch statistics


def test_preprocess_embedding_and_masks(b200):
    ops = _ops(b200)
    tgt = torch.tensor([[5, 6, 7, 0, 0], [9, 0, 4, 0, 0], [3, 3, 3, 3, 3]])
    s_in, s_out, key_pad, non_pad = ops.preprocess_targets(tgt.cuda(), 6)
    o_in, o_out = O.preprocess_targets(tgt, 6)
    assert torch.equal(s_in.cpu(), o_in) and torch.equal(s_out.cpu(), o_out)
    assert torch.equal(key_pad.cpu().bool(), o_in.eq(O.EOS)) and torch.equal(non_pad.cpu(), o_in.ne(O.EOS).float())
    with pytest.raises(RuntimeError):
        ops.preprocess_targets(tgt.cuda(), 5)                 # [SOS]+5 tokens does not fit 5 positions
    kp, npad = ops.length_masks(torch.tensor([7, 3, 12], dtype=torch.int32), 3, 8, "cuda")
    assert torch.equal(npad.cpu(), O.length_non_pad(3, 8, [7, 3, 12]))
    assert torch.equal(kp.cpu().bool(), O.length_non_pad(3, 8, [7, 3, 12]).lt(1))
    table = torch.randn(11, 32, requires_grad=True)
    pe = O.sinusoid_table(6, 32)
    e = F.embedding(o_in, table, padding_idx=0) * 0.5 + pe.unsqueeze(0)
    de = torch.randn_like(e)
    e.backward(de)
    tc = table.detach().cuda().requires_grad_(True)
    ec = ops.EmbedFn.apply(s_in, tc, pe.cuda(), 0.5, 0.0, 0)
    ec.backward(de.cuda())
    assert rel_err(ec, e) < 1e-6 and rel_err(tc.grad, table.grad) < 1e-5


@pytest.mark.parametrize("smoothing", [0.0, 0.1])
def test_cross_entropy_argmax(b200, smoothing):
    ops = _ops(b200)
    g = torch.Generator().manual_seed(7)
    pred = (torch.randn(4, 9, 4364, generator=g) * 2).requires_grad_(True)
    gold = torch.randint(1, 4364, (4, 9), generator=g)
    gold[1, 5:] = 0; gold[3, 2:] = 0
    loss, n_word = O.cross_entropy_loss(pred, gold, smoothing)
    loss.backward()
    pc = pred.detach().cuda().requires_grad_(True)
    lc, stats = ops.CrossEntropyFn.apply(pc, gold.cuda(), smoothing, "mean")
    lc.backward()
    assert abs(lc.item() - loss.item()) < 1e-5 * abs(loss.item())
    assert int(stats[1].item()) == n_word and int(stats[2].item()) == O.num_correct(pred, gold)
    assert rel_err(pc.grad, pred.grad) < 1e-5
    assert torch.equal(ops.argmax_rows(pc).cpu(), pred.argmax(dim=2))
    ls, st2 = ops.CrossEntropyFn.apply(pc, gold.cuda(), smoothing, "sum")
    assert abs(ls.item() - loss.item() * n_word) < 1e-5 * abs(ls.item())


def test_dropout_statistics_and_backward_consistency(b200):
    """Dropout is statistically (not bitwise) equivalent to torch's: check the keep rate, the 1/(1-p) scale and that
    backward regenerates the forward mask."""
    ops = _ops(b200)
    b200.manual_seed(1234)
    x = torch.ones(512, 512, device="cuda", requires_grad=True)
    res = torch.zeros(512, 512, device="cuda")
    gamma = torch.ones(512, device="cuda"); beta = torch.zeros(512, device="cuda")
    # z = dropout(x) + 0: recover the mask from the LN input saved for backward via dz -> dx relation
    y = ops.AddLNFn.apply(x, res, gamma, beta, None, None, 1e-5, 0.25)
    dy = torch.randn_like(y)
    y.backward(dy)
    kept = (x.grad != 0).float().mean().item()
    assert abs(kept - 0.75) < 0.01
    tok = torch.randint(3, 50, (8, 64), device="cuda")
    table = torch.ones(50, 256, device="cuda", requires_grad=True)
    e = ops.EmbedFn.apply(tok, table, torch.zeros(64, 256, device="cuda"), 1.0, 0.1, 0)
    keep = (e != 0)
    assert abs(keep.float().mean().item() - 0.9) < 0.01
    assert abs(e[keep].mean().item() - 1.0 / 0.9) < 1e-3
    e.backward(torch.ones_like(e))
    assert abs(table.grad.sum().item() - e.sum().item()) < 1e-2 * e.sum().item()
    # attention dropout: rows still average to ~1 in expectation and backward matches finite differences of the same mask
    q = torch.randn(2, 2, 40, 32, device="cuda", requires_grad=True)
    k = torch.randn(2, 2, 40, 32, device="cuda"); v = torch.ones(2, 2, 40, 32, device="cuda")
    state = (ops.rng.seed, ops.rng.offset)
    o1 = ops.SdpaFn.apply(q, k, v, None, None, False, 0.2, 0.3)
    assert abs(o1.mean().item() - 1.0) < 0.05
    ops.rng.seed, ops.rng.offset = state
    o2 = ops.SdpaFn.apply(q, k, v, None, None, False, 0.2, 0.3)
    assert torch.equal(o1, o2)                                     # same (seed, offset) -> same mask


def test_fused_adam_matches_torch(b200):
    torch.manual_seed(0)
    lin = torch.nn.Linear(33, 17).cuda()
    ref = torch.nn.Linear(33, 17).cuda()
    ref.load_state_dict(lin.state_dict())
    flat = b200.FlatParams(lin)
    opt = b200.NoamOpt(512, 1.0, 10, b200.FusedAdam(flat), min_lr=1e-6)
    ropt = b200.NoamOpt(512, 1.0, 10, torch.optim.Adam(ref.parameters(), betas=(0.9, 0.98), eps=1e-9), min_lr=1e-6)
    for _ in range(5):
        x = torch.randn(8, 33, device="cuda")
        opt.zero_grad(); ropt.optimizer.zero_grad()
        lin(x).pow(2).sum().backward(); ref(x).pow(2).sum().backward()
        flat.ensure_grad_views()
        opt.step(); ropt.step()
    for a, b in zip(lin.parameters(), ref.parameters()):
        assert rel_err(a, b) < 1e-5


def test_greedy_decode_token_ids_match_oracle(b200):
    _greedy_decode_matches_oracle(b200, tied=False)


def test_greedy_decode_token_ids_match_oracle_tied(b200):
    """The same with emb_trg_sharing: the logits come from the embedding table itself."""
    _greedy_decode_matches_oracle(b200, tied=True)


def _greedy_decode_matches_oracle(b200, tied):
    """SURVEY.md §8 A18: greedy decode (full-prefix re-decode, argmax per step) gives the oracle's token ids bit-exactly.
    Decoding is compared up to the first step whose oracle top-2 logit margin is inside the rounding band (a near-tie may
    legitimately resolve either way and then changes the rest of the sequence)."""
    from tests.gpu_util import cuda_model
    cfg = O.OracleConfig(num_layers=2, num_heads=4, dim_model=128, dim_key=32, dim_value=32, dim_inner=256, vocab=60,
                         feat_extractor="", tgt_max_len=40, freq=161, emb_trg_sharing=tied)
    P = O.init_params(cfg, seed=21)
    g = torch.Generator().manual_seed(3)
    for k in P:
        if P[k].dim() == 1:
            P[k] = P[k] + 0.1 * torch.randn(P[k].shape, generator=g)
    P["decoder.output_linear.weight"] = P["decoder.output_linear.weight"] * 4.0       # spread the logits
    if tied:
        P["decoder.trg_embedding.weight"] = P["decoder.output_linear.weight"]
    src, lens, _ = O.synthetic_batch(cfg, 3, 30, seed=5, ragged=False)
    enc = O.encoder_forward(O.flatten_features(src), lens, P, cfg)
    ids_o, margins = O.greedy_decode(P, cfg, enc, steps=16)
    model = cuda_model(cfg, P, train=False)
    ids = model.decoder.greedy_decode_ids(enc.cuda(), steps=16).cpu()
    ids_cached = model.decoder.greedy_decode_cached(enc.cuda(), steps=16).cpu()
    assert torch.equal(ids_cached, ids)          # KV-cached incremental decode == full-prefix re-decode, bit for bit
    band = 1e-3 * float(enc.abs().max())
    for b in range(ids.shape[0]):
        safe = int((margins[b] > band).long().cumprod(0).sum())      # steps before the first near-tie
        assert safe >= 4, "test input degenerate: near-tie too early"
        assert torch.equal(ids[b, :safe], ids_o[b, :safe]), (b, ids[b].tolist(), ids_o[b].tolist())


def test_greedy_decode_matches_reference_greedy_search_fixture(b200):
    """A18 / f3 pinned by the reference itself: tests/golden/greedy.npz holds the token ids of the reference's
    Decoder.greedy_search (300 steps, cut at EOS).  Full-prefix decode, KV-cached decode and the KV-cached decode with the
    on-device EOS stop must reproduce them id for id (up to the first step whose top-2 logit margin is inside the rounding
    band: a near-tie may resolve either way and then changes the rest of the sequence)."""
    from tests.gpu_util import cuda_model
    from tests.helpers import cut_at_eos, load_greedy_golden
    cfg, P, enc, ref_ids, ref_len = load_greedy_golden()
    _, margins = O.greedy_decode(P, cfg, enc, steps=300)
    full = dict(O.init_params(cfg, seed=1))              # encoder / front-end entries are unused by the decode
    full.update(P)
    model = cuda_model(cfg, full, train=False)
    dec = model.decoder
    ids_cached = dec.greedy_decode_cached(enc.cuda(), steps=300).cpu()
    ids_stop = dec.greedy_decode_cached(enc.cuda(), steps=300, stop_at_eos=True).cpu()
    ids_full = dec.greedy_decode_ids(enc.cuda(), steps=64).cpu()
    band = 1e-4 * float(margins.abs().max())             # ~7e-4 on logits of magnitude ~15: a few times the fp32-grade error
    for b in range(enc.shape[0]):
        n = int(ref_len[b])
        safe = int((margins[b] > band).long().cumprod(0).sum())          # steps before the first near-tie
        m = min(n, safe)
        assert m >= 32, "fixture degenerate: near-tie too early"
        ref = ref_ids[b, :n].tolist()
        assert cut_at_eos(ids_cached[b])[:m] == ref[:m], b
        assert cut_at_eos(ids_full[b])[:min(m, 64)] == ref[:min(m, 64)], b
        got = ids_stop[b]
        k = int((got >= 0).sum())
        assert got[:k].tolist()[:m] == ref[:m] and (got[k:] == -1).all(), b      # ids, then -1 from the first EOS on
        if safe >= n:
            assert k == n and cut_at_eos(ids_cached[b]) == ref, b                # whole utterance incl. the cut position
    # early exit: with every utterance finished the loop stops (utterances 1..3 of the fixture end before step 200)
    sub = enc[1:].cuda()
    ids_sub = dec.greedy_decode_cached(sub, steps=300, stop_at_eos=True, check_every=4)
    assert ids_sub.shape == (3, 300) and int((ids_sub >= 0).sum(1).max()) < 300


@pytest.mark.gpu
def test_host_batch_prefetcher_hands_over_each_batch_intact():
    """HostBatchPrefetcher: pinned host batches copied on a side stream one step ahead; the consumer's stream waits for exactly
    that copy (the kernels launched right after take() must see the data), batch after batch."""
    import b200asr
    dev = torch.device("cuda")
    pf = b200asr.HostBatchPrefetcher(dev)
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randn(4, 1, 161, 300, generator=g).pin_memory(), torch.randint(0, 100, (4, 20), generator=g).pin_memory()) for _ in range(4)]
    busy = torch.randn(4096, 4096, device=dev)
    pf.submit(*batches[0])
    sums = []
    for i in range(len(batches)):
        src, tgt = pf.take()
        if i + 1 < len(batches):
            pf.submit(*batches[i + 1])
        busy = busy @ busy * 1e-4                      # keep the compute stream busy while the next copy runs
        sums.append((src.double().sum(), tgt.sum(), src, tgt))
    torch.cuda.synchronize()
    for (s_sum, t_sum, src, tgt), (hs, ht) in zip(sums, batches):
        assert torch.equal(src.cpu(), hs) and torch.equal(tgt.cpu(), ht)
        assert float(s_sum) == pytest.approx(float(hs.double().sum()), rel=1e-9) and int(t_sum) == int(ht.sum())
    with pytest.raises(RuntimeError):
        pf.take()
