"""Attention maps on the device: b200asr_sdpa_probs against float64 and against the forwards that wrote the log-sum-exp, its
write extent and determinism, and b200asr.attention_maps on the model forwards (the reference installed against the
reference eager; training mode unchanged by the switch)."""
import importlib

import pytest
import torch

import b200asr
from oracle import ref_shim

pytestmark = pytest.mark.gpu

# b200asr_sdpa_probs's write extent is guarded here (test_writes_only_its_extent_and_repeats_bit_for_bit): register it with the
# ABI-wide sweep of tests/test_gpu_write_extent.py, which requires every pointer entry point to be covered or exempted
from tests import test_gpu_write_extent as _write_extent  # noqa: E402

_write_extent.EXEMPT.setdefault("b200asr_sdpa_probs", "tests/test_gpu_attention_maps.py: NaN-poisoned output with guard bands "
                                "around a padded strided extent, at every precision")

ops = importlib.import_module(b200asr.__name__ + ".ops")
L = b200asr._lib
FP32, TF32, BF16X3 = L.PREC_FP32, L.PREC_TF32, L.PREC_BF16X3
# per grade: |P - P64|, row sums, P V against the forward's out
TOL = {FP32: (2e-5, 2e-5, 5e-5), TF32: (4e-3, 4e-3, 1e-2), BF16X3: (1e-4, 1e-4, 3e-4)}
LIMIT_TK = {FP32: 2050, TF32: 447, BF16X3: 447}        # fp32: past the materialised path's 2048; tensor cores: Tk <= 448


def _lib():
    return L.load()


def _qkv(B, H, Tq, Tk, dk, dv, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = 0.6 * torch.randn(B, Tq, H, dk, device="cuda", generator=g)
    k = 0.6 * torch.randn(B, Tk, H, dk, device="cuda", generator=g)
    v = torch.randn(B, Tk, H, dv, device="cuda", generator=g)
    return q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3)      # (B,H,T,d) views of token-major memory


def _masks(kind, B, Tq, Tk, seed):
    """(key_pad [B,Tk] or None, dense [B,Tq,Tk] or None, causal) of a mask kind; each kind has fully masked rows somewhere
    when the shape allows (an utterance of length 0, or all-masked dense rows)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "dense":
        dense = (torch.rand(B, Tq, Tk, generator=g) < 0.3).to(torch.uint8)
        dense[0, Tq // 2] = 1
        return None, dense.cuda(), False
    lens = torch.randint(1, Tk + 1, (B,), generator=g)
    lens[0] = Tk
    if kind == "enc" and B > 2:
        lens[2] = 0
    key_pad = (torch.arange(Tk)[None, :] >= lens[:, None]).to(torch.uint8).cuda()
    return key_pad, None, kind == "dec"


def _forward(prec, q, k, v, key_pad, dense, causal, scale, p, seed=11, off=3):
    B, H, Tq, dk = q.shape
    Tk, dv = k.shape[2], v.shape[3]
    out = torch.empty(B, Tq, H, dv, device="cuda").permute(0, 2, 1, 3)
    lse = torch.empty(B, H, Tq, device="cuda")
    st = [L.ptr(q), L.ptr(k), L.ptr(v), *q.stride()[:3], *k.stride()[:3], *v.stride()[:3], L.ptr(key_pad), L.ptr(dense),
          int(causal), L.ptr(out), *out.stride()[:3], L.ptr(lse)]
    stream = torch.cuda.current_stream().cuda_stream
    if prec == BF16X3:
        ws = torch.empty(_lib().b200asr_sdpa_fused_ws_bytes(B, H, Tq, Tk), device="cuda", dtype=torch.uint8)
        L.check(_lib().b200asr_sdpa_fused_fwd(*st, L.ptr(ws), B, H, Tq, Tk, dk, dv, scale, p, seed, off, stream), "fused_fwd")
    else:
        L.check(_lib().b200asr_sdpa_fwd(*st, B, H, Tq, Tk, dk, dv, scale, p, seed, off, prec, stream), "sdpa_fwd")
    return out, lse


def _probs_call(prec, q, k, key_pad, dense, causal, lse, buf, strides, scale, p, seed=11, off=3, dk=None):
    B, H, Tq, dkq = q.shape
    Tk = k.shape[2]
    return _lib().b200asr_sdpa_probs(L.ptr(q), L.ptr(k), *q.stride()[:3], *k.stride()[:3], L.ptr(key_pad), L.ptr(dense),
                                     int(causal), L.ptr(lse), L.ptr(buf), *strides, B, H, Tq, Tk, dk or dkq, scale, p, seed,
                                     off, prec, torch.cuda.current_stream().cuda_stream)


def _probs(prec, q, k, key_pad, dense, causal, lse, scale, p, seed=11, off=3):
    B, H, Tq, _ = q.shape
    Tk = k.shape[2]
    shape, strides = ops.maps_layout(B, H, Tq, Tk)
    P = torch.full(shape, float("nan"), device="cuda")
    L.check(_probs_call(prec, q, k, key_pad, dense, causal, lse, P, strides, scale, p, seed, off), "sdpa_probs")
    return P


def _masked(key_pad, dense, causal, B, H, Tq, Tk):
    """[H*B, Tq, Tk] bool, True = masked, in the maps' order."""
    m = torch.zeros(B, Tq, Tk, dtype=torch.bool, device="cuda")
    if key_pad is not None:
        m |= key_pad.bool()[:, None, :]
    if dense is not None:
        m |= dense.bool()
    if causal:
        m |= torch.ones(Tq, Tk, dtype=torch.bool, device="cuda").triu(1)[None]
    return m.repeat(H, 1, 1)


def _heads_first(t):           # (B,H,...) -> (H*B, ...)
    return t.transpose(0, 1).reshape(-1, *t.shape[2:])


def _check_eval(prec, B, H, Tq, Tk, dk, dv, kind, seed):
    q, k, v = _qkv(B, H, Tq, Tk, dk, dv, seed)
    key_pad, dense, causal = _masks(kind, B, Tq, Tk, seed)
    scale = dk ** -0.5
    out, lse = _forward(prec, q, k, v, key_pad, dense, causal, scale, 0.0)
    P = _probs(prec, q, k, key_pad, dense, causal, lse, scale, 0.0)
    masked = _masked(key_pad, dense, causal, B, H, Tq, Tk)
    dead = masked.all(-1)
    s64 = torch.matmul(_heads_first(q).double(), _heads_first(k).double().transpose(1, 2)) * scale
    P64 = torch.softmax(s64.masked_fill(masked, float("-inf")), dim=-1)
    tp, ts, to = TOL[prec]
    assert torch.isnan(P[dead]).all() and not torch.isnan(P[~dead]).any()
    live = ~dead
    assert (P[live][masked[live]] == 0).all()
    assert (P[live].double().sum(-1) - 1).abs().max().item() <= ts
    assert (P[live].double() - P64[live]).abs().max().item() <= tp
    o = torch.matmul(P.double(), _heads_first(v).double())
    ref = _heads_first(out).double()
    assert torch.isnan(ref[dead]).all()
    assert (o[live] - ref[live]).abs().max().item() <= to


def _pairs(limit):
    return [(1, 1), (2, 63), (63, 65), (64, 200), (65, 2), (200, 64), (2, 1), (65, limit), (limit, 63)]


CASES = []
for _prec, _dks in ((FP32, (32, 64, 16)), (TF32, (32, 64)), (BF16X3, (64,))):
    for _dk in _dks:
        for _Tq, _Tk in _pairs(LIMIT_TK[_prec]):
            for _kind in ("enc", "dec", "cross", "dense"):
                CASES.append((_prec, _dk, _Tk if _kind in ("enc", "dec") else _Tq, _Tk, _kind))    # enc / dec: self-attention


@pytest.mark.parametrize("prec,dk,Tq,Tk,kind", CASES)
def test_probs_match_float64_and_the_forward(prec, dk, Tq, Tk, kind):
    B, H = (3, 2) if Tq * Tk < 100000 else (1, 2)
    dv = 64 if prec == BF16X3 else (128 if dk == 16 else dk)
    _check_eval(prec, B, H, Tq, Tk, dk, dv, kind, seed=Tq * 1000 + Tk + dk)


@pytest.mark.parametrize("prec,dk", [(FP32, 64), (TF32, 32), (BF16X3, 64)])
@pytest.mark.parametrize("kind", ["enc", "dec", "cross"])
def test_dropout_is_the_forwards_mask(prec, dk, kind):
    B, H, Tq, Tk, p = 2, 3, 70, 131 if kind == "cross" else 70, 0.1
    if kind != "cross":
        Tk = Tq
    q, k, v = _qkv(B, H, Tq, Tk, dk, dk, 5)
    key_pad, dense, causal = _masks(kind, B, Tq, Tk, 5)
    scale = dk ** -0.5
    out, lse = _forward(prec, q, k, v, key_pad, dense, causal, scale, p, seed=77, off=9)
    P = _probs(prec, q, k, key_pad, dense, causal, lse, scale, p, seed=77, off=9)
    Pe = _probs(prec, q, k, key_pad, dense, causal, lse, scale, 0.0)
    masked = _masked(key_pad, dense, causal, B, H, Tq, Tk)
    o = torch.matmul(P.double(), _heads_first(v).double())
    assert (o - _heads_first(out).double()).abs().max().item() <= TOL[prec][2]
    kept = P != 0
    dropped = (~masked) & (~kept)
    frac = dropped.sum().item() / (~masked).sum().item()
    assert 0.07 < frac < 0.13, frac
    inv_keep = P[kept] / Pe[kept]
    assert (inv_keep - 1 / (1 - p)).abs().max().item() < 1e-4
    assert (P[masked] == 0).all()


@pytest.mark.parametrize("prec,dk", [(FP32, 32), (TF32, 64), (BF16X3, 64)])
def test_writes_only_its_extent_and_repeats_bit_for_bit(prec, dk):
    B, H, Tq, Tk, G, pad = 2, 3, 67, 45, 64, 3
    q, k, v = _qkv(B, H, Tq, Tk, dk, dk, 9)
    key_pad, dense, causal = _masks("dec", B, Tq, Tk, 9)
    key_pad = None
    scale = dk ** -0.5
    _, lse = _forward(prec, q, k, v, key_pad, dense, causal, scale, 0.1)
    rs, bs = Tk + pad, (Tk + pad) * Tq + pad
    hs = bs * B + pad
    n = hs * H
    outs = []
    for _ in range(2):
        buf = torch.full((G + n + G,), float("nan"), device="cuda")
        view = buf[G:G + n]
        L.check(_probs_call(prec, q, k, key_pad, dense, causal, lse, view, (bs, hs, rs), scale, 0.1), "sdpa_probs")
        torch.cuda.synchronize()
        inside = torch.zeros(n, dtype=torch.bool, device="cuda")
        idx = (torch.arange(B)[:, None, None, None] * bs + torch.arange(H)[None, :, None, None] * hs +
               torch.arange(Tq)[None, None, :, None] * rs + torch.arange(Tk)[None, None, None, :]).reshape(-1).cuda()
        inside[idx] = True
        assert not torch.isnan(view[inside]).any()
        assert torch.isnan(view[~inside]).all() and torch.isnan(buf[:G]).all() and torch.isnan(buf[G + n:]).all()
        outs.append(view[inside].clone())
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))


def test_rejected_calls_write_and_launch_nothing():
    B, H, T = 2, 2, 40
    q, k, v = _qkv(B, H, T, T, 64, 64, 3)
    _, lse = _forward(FP32, q, k, v, None, None, False, 0.125, 0.0)
    shape, strides = ops.maps_layout(B, H, T, T)
    buf = torch.full(shape, float("nan"), device="cuda")
    q16, k16, _ = _qkv(B, H, T, T, 16, 16, 3)
    q48 = torch.randn(B, H, T, 48, device="cuda")
    k48 = torch.randn(B, H, T, 48, device="cuda")
    qlong, klong, _ = _qkv(1, 1, 4, 449, 64, 64, 3)
    lse_long = torch.zeros(1, 1, 4, device="cuda")
    bad = [(L.PREC_TF32X3, q, k, lse, None), (L.PREC_BF16, q, k, lse, None), (7, q, k, lse, None),
           (TF32, q16, k16, lse, None), (BF16X3, q16, k16, lse, None), (FP32, q48, k48, lse, None),
           (BF16X3, q[..., :32], k[..., :32], lse, 32), (TF32, qlong, klong, lse_long, None), (BF16X3, qlong, klong, lse_long, None)]
    torch.cuda.synchronize()
    n0 = _lib().b200asr_launch_count()
    for prec, qq, kk, ll, dk in bad:
        rc = _probs_call(prec, qq, kk, None, None, False, ll, buf, strides, 0.125, 0.0, dk=dk)
        assert rc == -1, (prec, qq.shape, kk.shape, rc)            # B200ASR_BAD_SHAPE
    torch.cuda.synchronize()
    assert _lib().b200asr_launch_count() == n0
    assert torch.isnan(buf).all()


# ------------------------------------------------------------------------------------------ model forwards
MODES = ["default", "bf16x3", "tf32", "fp32"]


@pytest.fixture
def attn_mode():
    saved = ops.config.attn

    def set_mode(mode):
        ops.config.attn = saved if mode == "default" else ops._PREC_NAMES[mode]
    yield set_mode
    ops.config.attn = saved


def _mirror_model(feat="vgg_cnn", dropout=0.1):
    cfg = b200asr.ASRConfig(num_layers=2, num_heads=2, dim_model=128, dim_key=64, dim_value=64, dim_inner=256, vocab=40,
                            feat_extractor=feat, tgt_max_len=20, dropout=dropout)
    torch.manual_seed(3)
    return b200asr.build_model(cfg).cuda(), cfg


def _train_batch(B=3, freq=161, T=64, V=40, Lt=12, seed=4):
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(B, 1, freq, T, generator=g).cuda()
    lens = torch.tensor([T, T - 9, T - 23], dtype=torch.int32).cuda()
    tgt = torch.randint(3, V, (B, Lt), generator=g)
    tgt[1, 8:] = 0
    tgt[2, 5:] = 0
    return src, lens, tgt.cuda()


def _count_launches(fn):
    ops.profiler.start()
    try:
        fn()
    finally:
        ops.profiler.stop()
    rec = ops.profiler.report()
    return {name: len(v) for name, v in rec.items()}


@pytest.mark.parametrize("mode", MODES)
def test_training_step_identical_with_maps_on(mode, attn_mode):
    attn_mode(mode)
    model, cfg = _mirror_model()
    model.train()
    src, lens, tgt = _train_batch()
    results = []
    for on in (False, True):
        with b200asr.attention_maps(on):
            b200asr.manual_seed(21)
            model.zero_grad(set_to_none=True)
            pred, gold, _, _ = model(src, lens, tgt)
            loss, _ = b200asr.loss_and_stats(pred, gold, 0.1)
            loss.backward()
            results.append((pred.detach().clone(), loss.detach().clone(),
                            {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}))
            counts = _count_launches(lambda: model(src, lens, tgt))
            results[-1] = results[-1] + (counts,)
    (p0, l0, g0, c0), (p1, l1, g1, c1) = results
    assert torch.equal(p0.view(torch.int32), p1.view(torch.int32))
    assert torch.equal(l0.view(torch.int32), l1.view(torch.int32))
    assert g0.keys() == g1.keys()
    for n in g0:
        assert torch.equal(g0[n].view(torch.int32), g1[n].view(torch.int32)), n
    assert c0 == c1 and "sdpa_probs" not in c1


@pytest.mark.parametrize("mode", MODES)
def test_training_maps_are_detached_and_dropped(mode, attn_mode):
    """Encoder / Decoder forwards in training mode return the maps the kernels multiplied into V (dropout applied)."""
    attn_mode(mode)
    model, _ = _mirror_model(dropout=0.1)
    model.train()
    src, lens, tgt = _train_batch()
    feats = torch.randn(3, 40, model.encoder.dim_input, device="cuda")
    with b200asr.attention_maps(True):
        enc, enc_maps = model.encoder(feats, lens.clamp(max=40))
        pred, gold, self_maps, cross_maps = model.decoder(tgt, enc, lens.clamp(max=40))
        (pred.sum() + enc.sum()).backward()
    for m in enc_maps + self_maps + cross_maps:
        assert m is not None and not m.requires_grad and m.grad_fn is None and m.dtype == torch.float32
        live = ~torch.isnan(m).any(-1)
        sums = m[live].sum(-1)
        assert (sums - 1).abs().max() > 1e-3          # dropout rescales the kept entries, so rows no longer sum to 1
    assert enc_maps[0].shape == (2 * 3, 40, 40) and cross_maps[0].shape == (2 * 3, self_maps[0].shape[1], 40)


def test_switch_off_returns_none_and_launches_nothing_extra():
    model, _ = _mirror_model()
    model.eval()
    src, lens, tgt = _train_batch()
    feats = torch.randn(3, 40, model.encoder.dim_input, device="cuda")
    lens = lens.clamp(max=40)
    with torch.no_grad():
        enc, enc_maps = model.encoder(feats, lens)
        out = model.decoder(tgt, enc, lens)
        assert enc_maps == [None, None] and out[2] == [None, None] and out[3] == [None, None]
        x = torch.randn(3, 40, 128, device="cuda")
        assert model.encoder.layers[0].self_attn(x, x, x)[1] is None
        c_off = _count_launches(lambda: (model.decoder(tgt, model.encoder(feats, lens)[0], lens)))
        with b200asr.attention_maps(True):
            c_on = _count_launches(lambda: (model.decoder(tgt, model.encoder(feats, lens)[0], lens)))
    assert "sdpa_probs" not in c_off
    extra = {n: c_on.get(n, 0) - c_off.get(n, 0) for n in set(c_on) | set(c_off)}
    assert {n: d for n, d in extra.items() if d} in ({"sdpa_probs": 6}, {})     # the materialised path copies instead
    ref = b200asr._lib.load().b200asr_launch_count
    torch.cuda.synchronize()
    n0 = ref()
    with torch.no_grad():
        model.decoder(tgt, model.encoder(feats, lens)[0], lens)
    n1 = ref()
    with torch.no_grad():
        model.decoder(tgt, model.encoder(feats, lens)[0], lens)
    assert ref() - n1 == n1 - n0


# ------------------------------------------------------------------------------------------ the unmodified reference
REF_FLAGS = ["--num-layers", "2", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "64", "--dim-value", "64",
             "--dim-inner", "128", "--tgt-max-len", "301", "--dropout", "0.1", "--cuda"]


def _reference_model(feat):
    ns = ref_shim.load(REF_FLAGS + ["--feat_extractor", feat], q12_shim=True)
    l2i, i2l = ref_shim.labels(40)
    torch.manual_seed(123456)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
        if feat == "emb_cnn":
            for bn in (model.conv[1], model.conv[4]):
                bn.running_mean.copy_(0.2 * torch.randn(bn.running_mean.shape, generator=g))
                bn.running_var.copy_(0.5 + torch.rand(bn.running_var.shape, generator=g))
    return ns, model.cuda().eval(), g


def _all_maps(model, src, lens, tgt, g_seed):
    """Every map the reference API returns: SDPA.forward, MHA.forward, Encoder.forward, Decoder.forward, evaluate's first value."""
    g = torch.Generator().manual_seed(g_seed)
    mha = model.encoder.layers[0].self_attn
    B, T, D, H, dk = 2, 37, 64, 2, 64
    x = torch.randn(B, T, D, generator=g).cuda()
    mlen = torch.tensor([T, 25])
    mask = (torch.arange(T)[None, None, :] >= mlen[:, None, None]).expand(B, T, T).cuda()
    qh = torch.randn(H * B, T, dk, generator=g).cuda()
    kh = torch.randn(H * B, T + 5, dk, generator=g).cuda()
    vh = torch.randn(H * B, T + 5, dk, generator=g).cuda()
    smask = (torch.rand(B, T, T + 5, generator=g) < 0.2).cuda().repeat(H, 1, 1)
    feats = torch.randn(B, 30, model.encoder.dim_input, generator=g).cuda()
    flens = torch.tensor([30, 21], dtype=torch.int32).cuda()
    out = {}
    with torch.no_grad():
        out["sdpa"] = [mha.attention(qh, kh, vh, mask=smask)[1]]
        out["mha"] = [mha(x, x, x, mask=mask)[1]]
        enc, out["encoder"] = model.encoder(feats, flens)
        _, _, out["dec_self"], out["dec_cross"] = model.decoder(tgt, enc, flens)
        first, hyps, gold = model.evaluate(src, lens, tgt)
        out["eval_self"], out["eval_cross"] = first
    return out, hyps, gold


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
@pytest.mark.parametrize("feat", ["", "vgg_cnn", "emb_cnn"])
def test_installed_maps_match_the_reference(feat, attn_mode):
    ns, model, g = _reference_model(feat)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    T = 48
    src = torch.randn(2, 1, 161, T, generator=g).cuda()
    lens = torch.tensor([T, 35], dtype=torch.int32).cuda()
    tgt = torch.randint(3, 40, (2, 6), generator=g)
    tgt[1, 4:] = 0
    tgt = tgt.cuda()
    ref, hyps_ref, gold_ref = _all_maps(model, src, lens, tgt, 5)
    try:
        b200asr.install()
        for mode in MODES:
            attn_mode(mode)
            with b200asr.attention_maps(True):
                ours, hyps, gold = _all_maps(model, src, lens, tgt, 5)
            assert (hyps, gold) == (hyps_ref, gold_ref)
            for name, maps in ref.items():
                assert len(ours[name]) == len(maps), name
                for a, b in zip(ours[name], maps):
                    assert a.shape == b.shape and a.dtype == torch.float32 and not a.requires_grad, (name, mode)
                    assert torch.equal(torch.isnan(a), torch.isnan(b)), (name, mode)
                    fin = ~torch.isnan(b)
                    err = (a[fin] - b[fin]).abs().max().item()
                    assert err <= 1e-3, (feat, mode, name, err)
                    assert (a[fin][b[fin] == 0] == 0).all(), (name, mode)
            with b200asr.attention_maps(False):
                first, hyps_off, _ = model.evaluate(src, lens, tgt)
            assert first == [[None, None], [None, None]] and hyps_off == hyps_ref
    finally:
        b200asr.uninstall()
