"""Gradient routing of the autograd Functions of ops.py against float64, in every memory arrangement and autograd state that
routes differently, and PyTorch's autograd semantics for all of them.

Where a gradient goes depends on more than the math:
  * _grad_sink: a parameter re-homed by optim.FlatParams gets its weight gradient added straight into .grad by the kernel,
    which then returns None to autograd -- only when the parameter requires grad and the engine will run its AccumulateGrad
    node (not under autograd.grad, not for a parameter backward(inputs=...) leaves out, not with tensor hooks);
  * AttnProjFn runs Q|K|V, K|V or three GEMMs depending on which weights, biases and .grad views lie back to back, and cuts
    the packed outputs and gradients at the offsets n_q and n_q + n_k;
  * ResidualLink hands AddLNFn's residual gradient to the data-gradient epilogue of the next node instead of autograd's add.

The kernels' accuracy is tested elsewhere; the bars here only show that each route computes the right function (a wrong
slice, a dropped or doubled accumulation is an O(1) error).  Where two arrangements launch the same kernels on the same
shapes the bits must agree: a sunk gradient vs. the same gradient returned into a zeroed or pre-filled .grad (the kernel's
accumulate epilogue computes old + acc, one rounding, as AccumulateGrad's in-place add does), and a linked residual vs.
autograd's sum of the two branches (a + b in either order).

SWEEP runs every Function through backward(retain_graph=True), backward() (identical bits: the second pass reads nothing the
first consumed), a third backward (PyTorch's "second time" error wherever the node saves tensors) and create_graph=True
(refused).  tests/test_autograd_routing_host.py keeps SWEEP complete.

The model-level tests use a small configuration with FlatParams and the float64 oracle (oracle/asr_oracle.py): two
backwards without zero_grad, autograd.grad, backward(inputs=...), parameters frozen after FlatParams, tensor hooks, and
tied embedding / output weights (emb_trg_sharing)."""
import importlib
import itertools

import pytest
import torch
import torch.nn.functional as F

import b200asr
from oracle import asr_oracle as O
from tests.helpers import assert_grads_close, rel_err, vgg_pools_well_separated

pytestmark = pytest.mark.gpu
ops = importlib.import_module(b200asr.__name__ + ".ops")
DEV = "cuda"
LIN_BAR = 1e-4          # linear grades: bf16x3 6e-5 at worst (test_gpu_default_precision.LIN_BARS), tf32x3 2.5e-5, fp32 exact
LN_BAR = 1e-4           # add_ln (test_gpu_row_kernels.LN_BARS)
ATTN_BARS = {"tf32x3": 1e-3, "fp32": 1e-3, "bf16x3": 5e-3, "tf32": 3e-2}     # projections + attention + their gradients
LN_EPS = 1e-5


@pytest.fixture(scope="module", autouse=True)
def _lib():
    b200asr._lib.load(check_device=True)
    saved_cfg = (ops.config.linear, ops.config.conv, ops.config.conv_wgrad, ops.config.attn, ops.config.attn_bwd)
    saved_cache = ops.weight_cache
    yield
    ops.config.linear, ops.config.conv, ops.config.conv_wgrad, ops.config.attn, ops.config.attn_bwd = saved_cfg
    ops.weight_cache = saved_cache


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


# ================================================================================================ parameter arrangements
def flat_layout(values, gaps, grad="R", flat=True, seed=0):
    """Leaf parameters with the given values laid out as optim.FlatParams lays them: each a view of one data buffer and its
    .grad a view of one gradient buffer, `gaps[i]` floats before parameter i (0: back to back with its predecessor), and
    `_b200_flat_grad` set.  `gaps` may be a pair (data gaps, grad gaps).  grad: None (no .grad), "zero", or "R" (random
    values the backward must add to).  flat=False gives the same .grad values without the flag: autograd accumulates."""
    dgaps, ggaps = gaps if isinstance(gaps, tuple) else (gaps, gaps)
    g = _gen(1000 + seed)

    def place(gp):
        offs, o = [], 0
        for v, gap in zip(values, gp):
            o += gap
            offs.append(o)
            o += v.numel()
        return offs, o

    doffs, dn = place(dgaps)
    goffs, gn = place(ggaps)
    data = torch.zeros(dn, device=DEV)
    gbuf = torch.randn(gn, generator=g).to(DEV) if grad == "R" else torch.zeros(gn, device=DEV)
    ps = []
    for v, do, go in zip(values, doffs, goffs):
        n = v.numel()
        data[do:do + n].copy_(v.reshape(-1))
        p = data[do:do + n].view(v.shape).detach().requires_grad_(True)
        if grad is not None:
            p.grad = gbuf[go:go + n].view(v.shape)
            if flat:
                p._b200_flat_grad = True
        ps.append(p)
    return ps


def grads_before(ps):
    return [None if p.grad is None else p.grad.clone() for p in ps]


def check_param_grads(ps, before, refs, bar, what):
    """Every parameter that requires grad ends with before + ref (float64 ref), every frozen one with its .grad untouched."""
    for i, (p, b, r) in enumerate(zip(ps, before, refs)):
        if p is None:
            continue
        if not p.requires_grad:
            assert (p.grad is None and b is None) or torch.equal(p.grad, b), (what, i, "frozen parameter's .grad written")
            continue
        want = r.cpu() + (b.double().cpu() if b is not None else 0)
        assert p.grad is not None, (what, i)
        assert rel_err(p.grad, want) < bar, (what, i, rel_err(p.grad, want))


# ================================================================================================ LinearFn
def linear_ref(x, w, b, dy):
    x64, w64, dy64 = x.double().cpu(), w.double().cpu(), dy.double().cpu()
    x2, dy2 = x64.reshape(-1, w64.shape[1]), dy64.reshape(-1, w64.shape[0])
    y = x2 @ w64.T + (b.double().cpu() if b is not None else 0)
    return y.view(*x.shape[:-1], -1), (dy2 @ w64).view(x.shape), dy2.T @ x2, dy2.sum(0)


@pytest.mark.parametrize("N,K,route", [(48, 64, "bf16x3"), (50, 64, "fp32: N % 4 != 0"), (48, 68, "tf32x3: K % 8 != 0")])
@pytest.mark.parametrize("xdim", [2, 3])
@pytest.mark.parametrize("bias", [True, False])
def test_linear_routes(N, K, route, xdim, bias):
    g = _gen(N + K + xdim)
    xshape = (37, K) if xdim == 2 else (3, 13, K)
    x0, w0, b0 = _randn(g, *xshape), _randn(g, N, K, scale=K ** -0.5), _randn(g, N)
    dy = _randn(g, *xshape[:-1], N)
    y64, dx64, dw64, db64 = linear_ref(x0, w0, b0 if bias else None, dy)
    for need in itertools.product([False, True], repeat=3):
        if not any(need) or (not bias and not any(need[:2])):
            continue
        for grad in (None, "zero", "R"):
            runs = {}
            for flat in ((False, True) if grad else (False,)):
                w, b = flat_layout([w0, b0], [0, 0], grad=grad, flat=flat, seed=7)
                x = x0.clone().requires_grad_(need[0])
                w.requires_grad_(need[1])
                b.requires_grad_(need[2])
                b_arg = b if bias else None
                before = grads_before([w, b])
                y = ops.LinearFn.apply(x, w, b_arg)
                assert rel_err(y, y64) < LIN_BAR
                y.backward(dy)
                what = (route, need, grad, flat)
                if need[0]:
                    assert rel_err(x.grad, dx64) < LIN_BAR, what
                check_param_grads([w, b if bias else None], before, [dw64, db64], LIN_BAR, what)
                runs[flat] = (x.grad, w.grad, b.grad)
            if grad:           # sunk into .grad vs. returned to autograd and added there: the same bits
                for a, c in zip(runs[False], runs[True]):
                    assert (a is None and c is None) or torch.equal(a, c), (route, need, grad)


# ================================================================================================ FFNFn (+ AddLNFn, link)
def ffn_ln_ref(x, w1, b1, w2, b2, gamma, beta, dy, residual=True):
    ts = [t.double().cpu().requires_grad_(True) for t in (x, w1, b1, w2, b2, gamma, beta)]
    x64, w164, b164, w264, b264, g64, be64 = ts
    h = F.relu(F.linear(x64, w164.squeeze(-1), b164))
    z = F.linear(h, w264.squeeze(-1), b264) + (x64 if residual else 0)
    y = F.layer_norm(z, (z.shape[-1],), g64, be64, LN_EPS)
    y.backward(dy.double().cpu())
    return y.detach(), [t.grad for t in ts]


def test_ffn_routes():
    """Every subset of (x, w1, b1, w2, b2) needing grad, with and without the residual link to the AddLNFn that follows;
    the FFN parameters sunk into a pre-filled flat .grad vs. returned into the same values, and link vs. no link, bit for
    bit."""
    g = _gen(5)
    d, di = 64, 96
    x0 = _randn(g, 2, 11, d)
    p0 = [_randn(g, di, d, 1, scale=0.2), _randn(g, di, scale=0.3), _randn(g, d, di, 1, scale=0.2), _randn(g, d, scale=0.3),
          1 + _randn(g, d, scale=0.1), _randn(g, d, scale=0.1)]
    dy = _randn(g, 2, 11, d)
    y64, refs = ffn_ln_ref(x0, *p0, dy)
    for need in itertools.product([False, True], repeat=5):
        runs = {}
        for flat, linked in ((False, False), (True, False), (True, True), (False, True)):
            ps = flat_layout(p0, [0, 4, 0, 4, 0, 0], grad="R", flat=flat, seed=3)
            for p, n in zip(ps, need[1:]):
                p.requires_grad_(n)
            x = x0.clone().requires_grad_(need[0])
            before = grads_before(ps)
            link = ops.ResidualLink() if linked else None
            z = ops.FFNFn.apply(x, *ps[:4], link)
            y = ops.AddLNFn.apply(z, x, ps[4], ps[5], None, None, LN_EPS, 0.0, link)
            assert rel_err(y, y64) < LIN_BAR
            if linked:
                assert link.armed == need[0] and (y.grad_fn.link is not None) == need[0]
            y.backward(dy)
            what = (need, flat, linked)
            if need[0]:
                assert rel_err(x.grad, refs[0]) < LIN_BAR, what
            check_param_grads(ps, before, refs[1:], LIN_BAR, what)
            runs[(flat, linked)] = [x.grad] + [p.grad for p in ps]
        for key in ((True, False), (True, True), (False, True)):
            for i, (a, c) in enumerate(zip(runs[(False, False)], runs[key])):
                assert (a is None and c is None) or torch.equal(a, c), (need, key, i)


# ================================================================================================ AddLNFn
def _inv_keep(p):
    from tests.test_gpu_row_kernels import _inv_keep as ik
    return ik(p)


@pytest.mark.parametrize("residual", [True, False])
@pytest.mark.parametrize("post,scale", [(False, False), (True, True)])
@pytest.mark.parametrize("p_drop", [0.0, 0.2])
def test_add_ln_routes(residual, post, scale, p_drop):
    """gamma / beta sunk together, returned, or mixed (one frozen, one sinkable); x and the residual with and without grad.
    Dropout: the keep mask is read back from the saved z (z == residual exactly where a unit was dropped, as in
    test_gpu_row_kernels) and applied in the float64 restatement."""
    g = _gen(int(residual) + 2 * int(post) + int(10 * p_drop))
    rows_b, T, d = 3, 10, 128
    x0, res0 = _randn(g, rows_b, T, d), _randn(g, rows_b, T, d)
    gamma0, beta0 = 1 + _randn(g, d, scale=0.1), _randn(g, d, scale=0.1)
    pe = _randn(g, T, d) if post else None
    rs = (torch.rand(rows_b * T, generator=g) > 0.3).float().to(DEV) if scale else None
    dy = _randn(g, rows_b, T, d)
    runs = {}
    for need_g, need_b, flat in [(True, True, True), (True, True, False), (False, True, True), (True, False, True),
                                 (False, False, True)]:
        for need_x in (True, False):
            gamma, beta = flat_layout([gamma0, beta0], [0, 0], grad="R", flat=flat, seed=11)
            gamma.requires_grad_(need_g)
            beta.requires_grad_(need_b)
            x = x0.clone().requires_grad_(need_x)
            r = res0.clone().requires_grad_(True) if residual else None
            before = grads_before([gamma, beta])
            ops.manual_seed(77)                   # the same dropout mask in every arrangement
            y = ops.AddLNFn.apply(x, r, gamma, beta, pe, rs, LN_EPS, p_drop)
            if not y.requires_grad:
                continue
            z = y.grad_fn.saved_tensors[0].view(x0.shape)
            keep = ((z != r) if residual else (z != 0)).detach().double().cpu() if p_drop > 0 else 1.0
            ts = [t.double().cpu().requires_grad_(True) for t in (x0, res0, gamma0, beta0)]
            z64 = ts[0] * keep * (_inv_keep(p_drop) if p_drop > 0 else 1.0) + (ts[1] if residual else 0)
            y64 = F.layer_norm(z64, (d,), ts[2], ts[3], LN_EPS)
            if post:
                y64 = y64 + pe.double().cpu()
            if scale:
                y64 = y64 * rs.double().cpu().view(rows_b, T, 1)
            y64.backward(dy.double().cpu())
            assert rel_err(y, y64) < LN_BAR
            y.backward(dy)
            what = (need_g, need_b, flat, need_x)
            if need_x:
                assert rel_err(x.grad, ts[0].grad) < LN_BAR, what
            if residual:
                assert rel_err(r.grad, ts[1].grad) < LN_BAR, what
            check_param_grads([gamma, beta], before, [ts[2].grad, ts[3].grad], LN_BAR, what)
            runs[(need_g, need_b, flat, need_x)] = (gamma.grad, beta.grad)
    for need_x in (True, False):
        a, c = runs[(True, True, True, need_x)], runs[(True, True, False, need_x)]
        assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1]), need_x


# ================================================================================================ attention
def attn_ref(xq, xkv, w, b, H, dk, dv, key_pad, dense, causal, scale):
    """Float64 projections + masked softmax attention; returns (out [B, Tq, H*dv], probs [B, H, Tq, Tk]) on the CPU."""
    wq, wk, wv = w
    bq, bk, bv = b if b is not None else (0, 0, 0)
    B, Tq, _ = xq.shape
    Tk = xkv.shape[1]
    q = (xq @ wq.T + bq).view(B, Tq, H, dk).transpose(1, 2)
    k = (xkv @ wk.T + bk).view(B, Tk, H, dk).transpose(1, 2)
    v = (xkv @ wv.T + bv).view(B, Tk, H, dv).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) * scale
    mask = torch.zeros(B, 1, Tq, Tk, dtype=torch.bool)
    if key_pad is not None:
        mask |= key_pad.bool().cpu()[:, None, None, :]
    if dense is not None:
        mask |= dense.bool().cpu()[:, None]
    if causal:
        mask |= torch.triu(torch.ones(Tq, Tk, dtype=torch.bool), diagonal=1)
    p = torch.softmax(s.masked_fill(mask, float("-inf")), -1)
    return (p @ v).transpose(1, 2).reshape(B, Tq, H * dv), p


# route name -> (self-attention?, data gaps of (wq, wk, wv, bq, bk, bv), grad gaps, expected (fuse3, fuse2))
ARRANGEMENTS = {
    "fuse3 self": (True, [0, 0, 0, 4, 0, 0], [0, 0, 0, 4, 0, 0], (True, False)),
    "fuse2 cross": (False, [0, 0, 0, 4, 0, 0], [0, 0, 0, 4, 0, 0], (False, True)),
    "fuse2 self, Q apart": (True, [0, 4, 0, 4, 4, 0], [0, 4, 0, 4, 4, 0], (False, True)),
    "separate": (True, [0, 4, 4, 4, 4, 4], [0, 4, 4, 4, 4, 4], (False, False)),
    "weights adjacent, biases not": (True, [0, 0, 0, 4, 4, 4], [0, 0, 0, 4, 4, 4], (False, False)),
    "grads not adjacent": (True, [0, 0, 0, 4, 0, 0], [0, 4, 4, 4, 4, 4], (True, False)),
}


def _masks(g, B, Tq, Tk, kind):
    key_pad = dense = None
    causal = kind == "causal"
    if kind in ("keypad", "causal"):
        lens = torch.randint(max(1, Tk // 2), Tk + 1, (B,), generator=g)
        lens[0] = Tk
        key_pad = (torch.arange(Tk)[None, :] >= lens[:, None]).to(torch.uint8).to(DEV)
    if kind == "dense":
        dn = torch.rand(B, Tq, Tk, generator=g) < 0.3
        dn[:, :, 0] = False
        dense = dn.to(torch.uint8).to(DEV)
    return key_pad, dense, causal


def _attn_case(arr, mask, bias, grade, dk, dv, need_w=(True,) * 6, linked=False, flat=True, grad="R", seed=0):
    self_attn, dgaps, ggaps, route = ARRANGEMENTS[arr]
    g = _gen(seed)
    B, H, D = 2, 2, 64
    Tq = 9
    Tk = Tq if self_attn else 13
    xq0 = _randn(g, B, Tq, D)
    xkv0 = xq0 if self_attn else _randn(g, B, Tk, D)
    w0 = [_randn(g, H * dk, D, scale=D ** -0.5), _randn(g, H * dk, D, scale=D ** -0.5), _randn(g, H * dv, D, scale=D ** -0.5)]
    b0 = [_randn(g, H * dk, scale=0.1), _randn(g, H * dk, scale=0.1), _randn(g, H * dv, scale=0.1)]
    gamma0, beta0 = 1 + _randn(g, H * dv, scale=0.1), _randn(g, H * dv, scale=0.1)
    key_pad, dense, causal = _masks(g, B, Tq, Tk, mask if self_attn or mask != "causal" else "keypad")
    dout = _randn(g, B, Tq, H * dv)
    scale = dk ** -0.5
    # float64 reference (with the AddLN that the link runs through when linked)
    xs64 = [t.double().cpu().requires_grad_(True) for t in ([xq0] if self_attn else [xq0, xkv0])]
    w64 = [t.double().cpu().requires_grad_(True) for t in w0]
    b64 = [t.double().cpu().requires_grad_(True) for t in b0]
    o64, p64 = attn_ref(xs64[0], xs64[-1], w64, b64 if bias else None, H, dk, dv, key_pad, dense, causal, scale)
    if linked:         # y = LN(attn(x) + x): needs dv * H == D
        o64 = F.layer_norm(o64 + xs64[0], (H * dv,), gamma0.double().cpu(), beta0.double().cpu(), LN_EPS)
    o64.backward(dout.double().cpu())
    # the kernel path
    ops.config.set(attn=grade)
    ps = flat_layout(w0 + b0, (dgaps, ggaps), grad=grad, flat=flat, seed=seed)
    for p, n in zip(ps, need_w):
        p.requires_grad_(n)
    xq = xq0.clone().requires_grad_(True)
    xkv = xq if self_attn else xkv0.clone().requires_grad_(True)
    before = grads_before(ps)
    link = ops.ResidualLink() if linked else None
    maps = []
    wq, wk, wv, bq, bk, bv = ps
    out = ops.AttnProjFn.apply(xq, xkv, wq, bq if bias else None, wk, bk if bias else None, wv, bv if bias else None, H, dk, dv,
                               key_pad, dense, causal, scale, 0.0, link, maps)
    if not bias and arr == "weights adjacent, biases not":
        route = (True, False)                       # without biases only the weights' adjacency counts
    assert tuple(out.grad_fn.shapes[3:5]) == route, (arr, out.grad_fn.shapes[3:5])
    y = ops.AddLNFn.apply(out, xq, gamma0, beta0, None, None, LN_EPS, 0.0, link) if linked else out
    y.backward(dout)
    bar = ATTN_BARS[grade]
    what = (arr, mask, bias, grade, need_w, linked)
    assert rel_err(y, o64) < bar, what
    assert len(maps) == 1 and rel_err(maps[0].view(H, B, Tq, Tk).transpose(0, 1), p64) < bar, what
    assert rel_err(xq.grad, xs64[0].grad) < bar, what
    if not self_attn:
        assert rel_err(xkv.grad, xs64[1].grad) < bar, what
    check_param_grads(ps if bias else ps[:3], before, [t.grad for t in w64 + b64], bar, what)
    return [xq.grad] + [p.grad for p in ps]


@pytest.mark.parametrize("arr", list(ARRANGEMENTS))
@pytest.mark.parametrize("mask", ["keypad", "causal", "dense"])
@pytest.mark.parametrize("bias", [True, False])
def test_attention_projection_routes(arr, mask, bias):
    """dk = 32, dv = 64 (a swapped n_k / n_v offset shows), Tq != Tk for cross-attention; the sunk route and the returned
    route give the same bits."""
    sunk = _attn_case(arr, mask, bias, "tf32x3", 32, 64, seed=3)
    returned = _attn_case(arr, mask, bias, "tf32x3", 32, 64, flat=False, seed=3)
    for i, (a, c) in enumerate(zip(sunk, returned)):
        assert (a is None and c is None) or torch.equal(a, c), (arr, mask, bias, i)


@pytest.mark.parametrize("arr", ["fuse3 self", "fuse2 self, Q apart", "fuse2 cross"])
def test_attention_projection_frozen_members_and_link(arr):
    """Each single member of the stacked group frozen (the group falls back from the stacked sink, the frozen .grad stays
    untouched), everything frozen (no weight-gradient GEMM), and the residual link against float64."""
    for frozen in range(7):
        need = tuple(i != frozen for i in range(6)) if frozen < 6 else (False,) * 6
        _attn_case(arr, "keypad", True, "tf32x3", 32, 64, need_w=need, seed=4)
    if ARRANGEMENTS[arr][0]:           # self-attention under y = LN(attn(x) + x): the link carries dz into dxq
        _attn_case(arr, "keypad", True, "tf32x3", 32, 32, linked=True, seed=5)


def test_attention_link_matches_autograd_sum_bitwise():
    """AttnProjFn + AddLNFn with the ResidualLink (dxq starts from AddLN's dz, the data-gradient GEMM adds into it) vs. the
    same graph with autograd summing the two gradients of x."""
    g = _gen(21)
    B, T, H, dk, dv = 2, 9, 2, 32, 32
    D = H * dv
    x0 = _randn(g, B, T, D)
    ps0 = [_randn(g, H * d, D, scale=D ** -0.5) for d in (dk, dk, dv)] + [_randn(g, H * d, scale=0.1) for d in (dk, dk, dv)]
    gamma, beta = 1 + _randn(g, D, scale=0.1), _randn(g, D, scale=0.1)
    dy = _randn(g, B, T, D)
    res = []
    for linked in (False, True):
        ps = flat_layout(ps0, [0] * 6, grad="zero", seed=1)
        x = x0.clone().requires_grad_(True)
        link = ops.ResidualLink() if linked else None
        wq, wk, wv, bq, bk, bv = ps
        out = ops.AttnProjFn.apply(x, x, wq, bq, wk, bk, wv, bv, H, dk, dv, None, None, False, dk ** -0.5, 0.0, link)
        y = ops.AddLNFn.apply(out, x, gamma, beta, None, None, LN_EPS, 0.0, link)
        assert (y.grad_fn.link is not None) == linked
        y.backward(dy)
        res.append([x.grad] + [p.grad for p in ps])
    for i, (a, c) in enumerate(zip(*res)):
        assert torch.equal(a, c), i


@pytest.mark.parametrize("grade,dk,dv", [("tf32x3", 32, 64), ("bf16x3", 64, 64), ("tf32", 32, 64), ("fp32", 32, 64)])
@pytest.mark.parametrize("arr", ["fuse3 self", "fuse2 cross"])
def test_attention_projection_grades(grade, dk, dv, arr):
    """One case per config.attn grade that selects a different kernel path: materialised 3xTF32, fused bf16x3 (64-wide
    heads), TF32 flash, fp32 CUDA cores."""
    _attn_case(arr, "keypad", True, grade, dk, dv, seed=6)


@pytest.mark.parametrize("head_major", [False, True])
def test_sdpa_head_major_and_foreign_dout_strides(head_major):
    """SdpaFn with the head-major output and a dout whose strides differ from the output's (copied before the kernels)."""
    g = _gen(8)
    B, H, Tq, Tk, dk, dv = 2, 3, 10, 14, 32, 64
    q0, k0, v0 = _randn(g, B, H, Tq, dk), _randn(g, B, H, Tk, dk), _randn(g, B, H, Tk, dv)
    key_pad, _, _ = _masks(g, B, Tq, Tk, "keypad")
    q, k, v = (t.clone().requires_grad_(True) for t in (q0, k0, v0))
    out = ops.SdpaFn.apply(q, k, v, key_pad, None, False, dk ** -0.5, 0.0, head_major)
    dout = _randn(g, B, H, Tq, dv)           # contiguous (B,H,Tq,dv): neither output layout has these strides
    assert dout.stride() != out.stride()
    out.backward(dout)
    t64 = [t.double().cpu().requires_grad_(True) for t in (q0, k0, v0)]
    s = (t64[0] @ t64[1].transpose(-1, -2)) * dk ** -0.5
    p = torch.softmax(s.masked_fill(key_pad.bool().cpu()[:, None, None, :], float("-inf")), -1)
    o64 = p @ t64[2]
    o64.backward(dout.double().cpu())
    bar = ATTN_BARS["tf32x3"]
    assert rel_err(out, o64) < bar
    for a, r in zip((q, k, v), t64):
        assert rel_err(a.grad, r.grad) < bar


# ================================================================================================ semantics sweep
def _sweep_linear(g):
    x, w, b = _randn(g, 3, 7, 64), _randn(g, 48, 64, scale=0.125), _randn(g, 48)
    leaves = [t.requires_grad_(True) for t in (x, w, b)]
    return leaves, lambda: (ops.LinearFn.apply(*leaves),)


def _sweep_ffn(g):
    leaves = [_randn(g, 2, 9, 64), _randn(g, 96, 64, 1, scale=0.2), _randn(g, 96), _randn(g, 64, 96, 1, scale=0.2), _randn(g, 64)]
    leaves = [t.requires_grad_(True) for t in leaves]
    return leaves, lambda: (ops.FFNFn.apply(*leaves),)


def _sweep_add_ln(g):
    leaves = [t.requires_grad_(True) for t in (_randn(g, 4, 9, 64), _randn(g, 4, 9, 64), 1 + _randn(g, 64, scale=0.1),
                                                _randn(g, 64, scale=0.1))]
    return leaves, lambda: (ops.AddLNFn.apply(*leaves, None, None, LN_EPS, 0.2),)          # dropout: the seed is reused


def _sweep_sdpa(g):
    leaves = [t.requires_grad_(True) for t in (_randn(g, 2, 2, 9, 32), _randn(g, 2, 2, 11, 32), _randn(g, 2, 2, 11, 32))]
    return leaves, lambda: (ops.SdpaFn.apply(*leaves, None, None, False, 32 ** -0.5, 0.1),)


def _sweep_attn_proj(g):
    D, H, dk, dv = 64, 2, 32, 64
    x = _randn(g, 2, 9, D).requires_grad_(True)
    ps = flat_layout([_randn(g, H * dk, D, scale=0.125), _randn(g, H * dk, D, scale=0.125), _randn(g, H * dv, D, scale=0.125),
                      _randn(g, H * dk), _randn(g, H * dk), _randn(g, H * dv)], [0] * 6, grad=None)
    wq, wk, wv, bq, bk, bv = ps
    return [x] + ps, lambda: (ops.AttnProjFn.apply(x, x, wq, bq, wk, bk, wv, bv, H, dk, dv, None, None, True, dk ** -0.5, 0.1),)


def _sweep_vgg(g):
    cfg = O.OracleConfig(num_layers=1, feat_extractor="vgg_cnn", freq=41)
    P = O.init_params(cfg, seed=5)
    ws = [P[f"conv.{i}.{k}"].to(DEV).requires_grad_(True) for i in (0, 2, 5, 7) for k in ("weight", "bias")]
    x = _randn(g, 2, 1, 41, 24)
    return ws, lambda: (ops.VggFrontendFn.apply(x, *ws),)


def _sweep_permute_cols(g):
    w = _randn(g, 40, 3 * 7).requires_grad_(True)
    return [w], lambda: (ops.PermuteColsFn.apply(w, 3, 7),)


def _sweep_emb_frontend(g):
    cfg = O.OracleConfig(num_layers=1, feat_extractor="emb_cnn")
    P = O.init_params(cfg, seed=6)
    names = ["conv.0.weight", "conv.0.bias", "conv.1.weight", "conv.1.bias", "conv.3.weight", "conv.3.bias", "conv.4.weight",
             "conv.4.bias"]
    ws = [P[n].to(DEV).requires_grad_(True) for n in names]
    x = _randn(g, 2, 1, 161, 30)
    return ws, lambda: (ops.EmbFrontendFn.apply(x, *ws, 1e-5),)


def _sweep_flatten(g):
    x = _randn(g, 2, 1, 17, 9).requires_grad_(True)
    return [x], lambda: (ops.FlattenFn.apply(x),)


def _sweep_embed(g):
    table = _randn(g, 30, 64).requires_grad_(True)
    tokens = torch.randint(0, 30, (3, 8), generator=g).to(DEV)
    pe = _randn(g, 8, 64)
    return [table], lambda: (ops.EmbedFn.apply(tokens, table, pe, 0.5, 0.1, 0),)


def _sweep_lstm(g):
    M = importlib.import_module(b200asr.__name__ + ".modules")
    torch.manual_seed(2)
    model = M.RNNModel("LSTM", 40, 24, 24, 2, dropout=0.0).to(DEV)
    inp = torch.randint(0, 40, (6, 3), generator=g).to(DEV)
    h0 = _randn(g, 2, 3, 24).requires_grad_(True)
    c0 = _randn(g, 2, 3, 24).requires_grad_(True)
    leaves = [h0, c0] + list(model.parameters())

    def run():
        out, (hn, cn) = ops.lstm_stack(model, inp, (h0, c0), p_emb=0.1, p_mid=0.1, p_out=0.1)
        return out, hn, cn
    return leaves, run


def _sweep_cross_entropy(g):
    pred = _randn(g, 3, 7, 50).requires_grad_(True)
    gold = torch.randint(1, 50, (3, 7), generator=g).to(DEV)
    gold[1, 4:] = 0
    return [pred], lambda: ops.CrossEntropyFn.apply(pred, gold, 0.1, "mean")[:1]


def _sweep_xent(g):
    logits = _randn(g, 21, 37).requires_grad_(True)
    tg = torch.randint(0, 37, (21,), generator=g).to(DEV)
    return [logits], lambda: (ops.XentFn.apply(logits, tg),)


def _sweep_ctc(g):
    pred = _randn(g, 3, 20, 12).requires_grad_(True)
    tg = torch.randint(1, 12, (3, 6), generator=g).to(DEV)
    il, tl = torch.tensor([20, 17, 12]), torch.tensor([6, 4, 5])
    return [pred], lambda: (ops.CtcLossFn.apply(pred, tg, il, tl),)


# Function name -> (builder(generator) -> (leaves, run() -> outputs), whether the node saves tensors for its backward).
# FlattenFn and PermuteColsFn save none: like torch's own views they may be backpropagated any number of times.
SWEEP = {
    "LinearFn": (_sweep_linear, True),
    "FFNFn": (_sweep_ffn, True),
    "AddLNFn": (_sweep_add_ln, True),
    "SdpaFn": (_sweep_sdpa, True),
    "AttnProjFn": (_sweep_attn_proj, True),
    "VggFrontendFn": (_sweep_vgg, True),
    "PermuteColsFn": (_sweep_permute_cols, False),
    "EmbFrontendFn": (_sweep_emb_frontend, True),
    "FlattenFn": (_sweep_flatten, False),
    "EmbedFn": (_sweep_embed, True),
    "LstmStackFn": (_sweep_lstm, True),
    "CrossEntropyFn": (_sweep_cross_entropy, True),
    "XentFn": (_sweep_xent, True),
    "CtcLossFn": (_sweep_ctc, True),
}


@pytest.mark.parametrize("name", list(SWEEP))
def test_retained_graph_third_backward_and_create_graph(name):
    build, saves = SWEEP[name]
    leaves, run = build(_gen(31))
    outs = run()
    g = _gen(32)
    douts = [torch.randn(o.shape, generator=g).to(DEV) for o in outs]

    def backward(**kw):
        for t in leaves:
            t.grad = None
        torch.autograd.backward(outs, douts, **kw)
        return [t.grad for t in leaves]

    first = backward(retain_graph=True)
    assert any(t is not None for t in first)
    second = backward()
    for i, (a, c) in enumerate(zip(first, second)):
        assert (a is None and c is None) or torch.equal(a, c), (name, i)
    if saves:
        with pytest.raises(RuntimeError, match="backward through the graph a second time"):
            backward()
    else:
        third = backward()
        assert all((a is None and c is None) or torch.equal(a, c) for a, c in zip(first, third))
    outs = run()
    with pytest.raises(RuntimeError, match="create_graph=True is not supported"):
        torch.autograd.grad(outs, [t for t in leaves if t.requires_grad], douts, create_graph=True, allow_unused=True)


# ================================================================================================ model level
MODEL_CFG = dict(num_layers=1, num_heads=2, dim_model=64, dim_key=32, dim_value=32, dim_inner=128, vocab=33, tgt_max_len=9)


def _model_case(feat="", tied=False, seed=3):
    from tests.gpu_util import cuda_model
    cfg = O.OracleConfig(**MODEL_CFG, feat_extractor=feat, freq=161 if feat == "" else 41, emb_trg_sharing=tied)
    P = O.init_params(cfg, seed=seed)
    g = _gen(17)
    for k in sorted(P):
        if P[k].dim() == 1:
            P[k] = P[k] + 0.1 * torch.randn(P[k].shape, generator=g)
    if tied:
        P["decoder.output_linear.weight"] = P["decoder.trg_embedding.weight"]
    for s in range(5, 200):          # max-pool routing is discontinuous: an input without near-tied pooling windows
        src, lens, tgt = O.synthetic_batch(cfg, 3, 40, seed=s, ragged=True)
        if feat != "vgg_cnn" or vgg_pools_well_separated(P, src, rel_gap=1e-4):
            break
    _, _, _, _, _, grads_o = O.forward_backward({k: v.double() for k, v in P.items()}, cfg, src.double(), lens, tgt, 0.1)
    model = cuda_model(cfg, P)
    flat = b200asr.FlatParams(model)
    named = dict(model.named_parameters())
    grads_o = {k: v for k, v in grads_o.items() if k in named}

    def loss_fn():
        pred, gold, _, _ = model(src.cuda(), lens, tgt.cuda())
        return b200asr.loss_and_stats(pred, gold, 0.1)[0]
    return model, flat, named, grads_o, loss_fn


def _grads(named):
    return {n: p.grad.detach().clone() for n, p in named.items()}


def _assert_model_grads(got, ref, scale=1.0, names=None):
    from tests.gpu_util import TOL
    from tests.helpers import grads_rel_err
    names = names if names is not None else list(ref)
    errs = grads_rel_err({n: got[n] for n in names}, {n: scale * ref[n].float() for n in names})
    worst = max(errs, key=errs.get)
    assert errs[worst] < TOL, (worst, errs[worst])


def test_model_two_backwards_without_zero_grad():
    model, flat, named, grads_o, loss_fn = _model_case()
    flat.zero_grad()
    loss = loss_fn()
    loss.backward(retain_graph=True)
    g1 = flat.flat_grad.clone()
    _assert_model_grads(_grads(named), grads_o)
    loss.backward()
    assert torch.equal(flat.flat_grad, 2 * g1)
    _assert_model_grads(_grads(named), grads_o, scale=2.0)


def test_model_autograd_grad_returns_backward_grads_and_leaves_flat_buffer():
    model, flat, named, grads_o, loss_fn = _model_case()
    names = list(named)
    flat.zero_grad()
    loss_fn().backward()
    via_backward = _grads(named)
    flat.flat_grad.copy_(torch.randn(flat.flat_grad.shape, generator=_gen(4)).to(DEV))
    snap = flat.flat_grad.clone()
    got = torch.autograd.grad(loss_fn(), [named[n] for n in names])
    assert torch.equal(flat.flat_grad, snap)
    for n, g in zip(names, got):
        assert torch.equal(g, via_backward[n]), n
    _assert_model_grads(dict(zip(names, got)), grads_o)


def test_model_backward_inputs_writes_only_that_subset():
    model, flat, named, grads_o, loss_fn = _model_case()
    subset = ["encoder.layers.0.self_attn.key_linear.weight", "encoder.layers.0.pos_ffn.conv_2.bias",
              "decoder.layers.0.encoder_attn.layer_norm.weight", "decoder.layers.0.self_attn.query_linear.bias"]
    R = torch.randn(flat.flat_grad.shape, generator=_gen(6)).to(DEV)
    flat.flat_grad.copy_(R)
    loss_fn().backward()
    full = _grads(named)
    flat.flat_grad.copy_(R)
    before = _grads(named)
    loss_fn().backward(inputs=[named[n] for n in subset])
    after = _grads(named)
    for n in named:
        want = full[n] if n in subset else before[n]
        assert torch.equal(after[n], want), n


def test_model_frozen_after_flat_params():
    model, flat, named, grads_o, loss_fn = _model_case()
    frozen = ["encoder.layers.0.self_attn.key_linear.weight", "decoder.layers.0.encoder_attn.value_linear.bias",
              "encoder.layers.0.pos_ffn.conv_2.bias", "decoder.layers.0.pos_ffn.layer_norm.weight"]
    for n in frozen:
        named[n].requires_grad_(False)
    R = 1e-4 * torch.randn(flat.flat_grad.shape, generator=_gen(7)).to(DEV)       # small: (R + g) - R stays close to g
    flat.flat_grad.copy_(R)
    before = _grads(named)
    loss_fn().backward()
    after = _grads(named)
    for n in frozen:
        assert torch.equal(after[n], before[n]), n
    rest = [n for n in named if n not in frozen]
    _assert_model_grads({n: after[n] - before[n] for n in rest}, grads_o, names=rest)


def test_model_tensor_hooks():
    model, flat, named, grads_o, loss_fn = _model_case()
    hooked = "encoder.layers.0.self_attn.value_linear.weight"
    post = "decoder.layers.0.pos_ffn.conv_1.weight"
    named[hooked].register_hook(lambda g: 2 * g)
    fired = []
    named[post].register_post_accumulate_grad_hook(lambda p: fired.append(p.grad.clone()))
    flat.zero_grad()
    loss_fn().backward()
    got = _grads(named)
    assert len(fired) == 1 and torch.equal(fired[0], got[post])
    _assert_model_grads(got, grads_o, names=[n for n in named if n != hooked])
    _assert_model_grads(got, grads_o, scale=2.0, names=[hooked])
    # the hooked gradient was added into the flat .grad view by AccumulateGrad, not stored in a new tensor
    slot = next(o for p, o in zip(flat.params, flat.offsets) if p is named[hooked])
    assert named[hooked].grad.data_ptr() == flat.flat_grad[slot:].data_ptr()


@pytest.mark.parametrize("feat", ["", "vgg_cnn"])
def test_model_tied_embedding_and_output_weights(feat):
    """emb_trg_sharing: one parameter gets LinearFn's sunk weight gradient and EmbedFn's returned one."""
    model, flat, named, grads_o, loss_fn = _model_case(feat=feat, tied=True)
    assert model.decoder.output_linear.weight is model.decoder.trg_embedding.weight
    flat.zero_grad()
    loss_fn().backward()
    if feat == "vgg_cnn":           # the parity tests' criterion at the tensor-core default (a pooling decision may move)
        from tests.gpu_util import TOL
        assert_grads_close(_grads(named), {k: v.float() for k, v in grads_o.items()}, TOL, exact_kernels=False)
    else:
        _assert_model_grads(_grads(named), grads_o)
