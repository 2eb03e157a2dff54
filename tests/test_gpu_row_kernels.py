"""The memory-bound row kernels of the training step, through the raw C ABI, against float64 references, at every template
instantiation and at the edges where row kernels go wrong (partial warps, partial float4 blocks, empty splits, grid-stride
tails, padding columns), plus the reproducibility of their reductions:

  1. residual + LayerNorm (norm.cu): every NV instantiation, the backward's grid-stride loop, constant rows, dropout with the
     keep mask read back from the saved input, dz == dx aliasing, accumulation into dgamma / dbeta;
  2. materialised attention and its masked-softmax rows (attention_mat.cu) with NaN-poisoned probability and dP buffers:
     every NV instantiation, padding columns, key-pad / causal / dense masks, a fully masked row, dropout;
  3. label-smoothed cross-entropy, argmax and the greedy decoding step (embed_loss.cu), including shifted logits and ties;
  4. the embedding forward / backward (embed_loss.cu) with heavy token repetition and PAD rows;
  5. the step tail: Adam, the gradient sum of squares past its grid cap, the clip coefficient of grad_scale;
  6. BatchNorm + Hardtanh (emb_frontend.cu): empty splits, row pitches, a large-mean channel, values exactly at the clamp
     bounds, running statistics, eval mode;
  7. CPU pins (no GPU): the float64 references used here equal the golden-pinned oracle;
  8. one emb_cnn training step run twice from the same state: identical bits;
  9. the spectrogram front end's per-utterance statistics: identical bits from two calls.

Outputs and workspaces are filled with NaN before each call, so an element a kernel fails to write, or reads without
writing, shows up.  Bars are max-norm relative errors (tests.helpers.rel_err); each states the error measured on one
H100 80GB HBM3 (400 W limit) and sits about 3x above it."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import asr_oracle as O
from tests.helpers import rel_err

NAN = float("nan")
BAD_SHAPE = -1
gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape):
    return torch.full(shape, NAN, device="cuda")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _thresh16(p):
    """common.cuh dropout_thresh16, in float32 as the host computes it."""
    t = np.float32(p) * np.float32(65536.0) + np.float32(0.5)
    return int(min(max(t, np.float32(0.0)), np.float32(65535.0)))


def _inv_keep(p):
    """common.cuh dropout_inv_keep: 1 / (1 - threshold / 65536) in float32."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(_thresh16(p)) / np.float32(65536.0)))


def _same_nan(a, b):
    return torch.equal(torch.isnan(a.cpu()), torch.isnan(b.cpu()))


def _finite_err(a, b):
    """rel_err over the elements where the reference is finite (the NaN pattern is asserted separately)."""
    m = torch.isfinite(b).cpu()
    return rel_err(a.cpu()[m], b.cpu()[m])


# ================================================================================================ float64 references
def ln_ref(z64, g64, b64, post64, rs64, eps, dy64):
    """torch's own F.layer_norm in float64 (what the oracle calls), + post_add[row % period], * row_scale; and its gradients."""
    rows, d = z64.shape
    z = z64.clone().requires_grad_(True)
    g = g64.clone().requires_grad_(True)
    b = b64.clone().requires_grad_(True)
    y = F.layer_norm(z, (d,), g, b, eps)
    if post64 is not None:
        y = y + post64[torch.arange(rows, device=z64.device) % post64.shape[0]]
    if rs64 is not None:
        y = y * rs64[:, None]
    y.backward(dy64)
    mean = z64.mean(1)
    rstd = 1.0 / torch.sqrt(z64.var(1, unbiased=False) + eps)
    return y.detach(), z.grad, g.grad, b.grad, mean, rstd


def attn_mask(B, Tq, Tk, key_pad=None, dense=None, causal=False, device="cpu"):
    """Boolean [B, Tq, Tk], True = masked: the union the kernels apply (key padding, causal k > q, the dense mask)."""
    m = torch.zeros(B, Tq, Tk, dtype=torch.bool, device=device)
    if key_pad is not None:
        m |= key_pad.bool()[:, None, :]
    if causal:
        m |= (torch.arange(Tk, device=device)[None, :] > torch.arange(Tq, device=device)[:, None])[None]
    if dense is not None:
        m |= dense.bool()
    return m


def attn_ref(q, k, v, mask, scale, keep=None, inv_keep=1.0):
    """float64 materialised attention on [B, H, T, d]: S = scale q k^T, masked_fill(-inf), softmax, dropout with the given
    keep mask, P V.  Returns (out, P) -- models/common_layers.py:215-223 with the heads as a batch dimension."""
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    s = s.masked_fill(mask[:, None], float("-inf"))
    p = torch.softmax(s, dim=-1)
    pd = p * keep * inv_keep if keep is not None else p
    return torch.matmul(pd, v), p


def ce_rows_ref(x64, gold, eps):
    """float64 restatement of calculate_loss (utils/metrics.py:115-132) per row: weights eps/V off target and 1 - eps on it
    (eps = 0: the plain negative log-likelihood), PAD rows 0.  Returns (row losses, row log-sum-exp)."""
    V = x64.shape[1]
    lse = torch.logsumexp(x64, dim=1)
    logp = x64 - lse[:, None]
    if eps > 0.0:
        w = torch.full_like(x64, eps / V)
        w.scatter_(1, gold.view(-1, 1), 1.0 - eps)
        loss = -(w * logp).sum(1)
    else:
        loss = -logp.gather(1, gold.view(-1, 1)).squeeze(1)
    return torch.where(gold != O.PAD, loss, torch.zeros_like(loss)), lse


def adam_ref(p, g, m, v, step, lr, b1, b2, eps):
    """torch.optim.Adam's update (no weight decay): bias corrections in double, denom = sqrt(v) / sqrt(bc2) + eps."""
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    denom = v.sqrt() / bc2 ** 0.5 + eps
    return p - (lr / bc1) * m / denom, m, v


# ================================================================================================ 1. LayerNorm
LN_D = [4, 64, 200, 512, 640, 768, 1024]          # NV = 1, 1, 2, 4, 6 (5 float4 per lane), 6, 8
LN_ROWS = [1, 37, 10000]                          # 10000 > 4 x 2368: the backward's grid-stride loop runs
LN_EPS = 1e-5
# measured maxima: y 1.1e-6, mean 1.6e-7, rstd 1.6e-7, dz 2.9e-7, dgamma / dbeta 1.1e-6 (1.1e-6 accumulating).  At d = 4 the
# rows offset by 30 are ill-conditioned -- four values may lie within 0.1 of each other, and the fp32 mean's rounding (~2e-6)
# is then 2e-5 of their spread --: y 1.2e-5, dz 4.0e-6, dgamma / dbeta 4.1e-6, hence LN_D4 times the bars there.
LN_BARS = dict(y=4e-6, mean=5e-7, rstd=5e-7, dz=1.2e-6, dgb=4e-6)
LN_D4 = 10.0


def _ln_fwd(L, x, res, gamma, beta, post, rs, rows, d, p=0.0, want_z=True):
    lib = L.load()
    y, mean, rstd = _nan(rows, d), _nan(rows), _nan(rows)
    z = _nan(rows, d) if want_z else None
    L.check(lib.b200asr_add_ln_fwd(L.ptr(x), L.ptr(res), L.ptr(gamma), L.ptr(beta), L.ptr(post),
                                   post.shape[0] if post is not None else 0, L.ptr(rs), L.ptr(y), L.ptr(z), L.ptr(mean),
                                   L.ptr(rstd), rows, d, LN_EPS, p, 11, 3, _stream()), "add_ln_fwd")
    return y, z, mean, rstd


def _ln_bwd(L, dy, z, gamma, mean, rstd, rs, dz, dx, dgamma, dbeta, rows, d, p=0.0, accumulate=0):
    lib = L.load()
    ws = torch.empty(lib.b200asr_add_ln_bwd_ws_bytes(rows, d) // 4, device="cuda").fill_(NAN)
    L.check(lib.b200asr_add_ln_bwd(L.ptr(dy), L.ptr(z), L.ptr(gamma), L.ptr(mean), L.ptr(rstd), L.ptr(rs), L.ptr(dz),
                                   L.ptr(dx), L.ptr(dgamma), L.ptr(dbeta), L.ptr(ws), rows, d, p, 11, 3, accumulate,
                                   _stream()), "add_ln_bwd")


@gpu
@pytest.mark.parametrize("flags", ["plain", "residual+pe+row_scale"])
@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("d", LN_D)
def test_add_layernorm_against_float64(L, d, rows, flags):
    """b200asr_add_ln_fwd / _bwd against F.layer_norm in float64.  Every third row carries an offset of 30 (a variance
    computed as E[x^2] - mean^2 loses its digits there); one row is constant (variance 0: the output must be beta exactly);
    'plain' passes no residual and no saved z (the backward reads x), the other variant adds a residual, the positional
    encoding with period 7 and a row scale with zero rows.  The backward runs with separate dz and dx, then with dx == dz
    (the aliasing branch), then accumulating into random dgamma / dbeta; two calls give identical bits.
    Measured maxima and bars: see LN_BARS."""
    full = flags != "plain"
    bars = {k: v * (LN_D4 if d == 4 and k in ("y", "dz", "dgb") else 1.0) for k, v in LN_BARS.items()}
    g = _gen(d * 7 + rows)
    x = torch.randn(rows, d, generator=g)
    x[::3] += 30.0
    res = torch.randn(rows, d, generator=g) if full else None
    const = rows // 2 if rows > 1 else None
    if const is not None:
        x[const] = 0.75
        if full:
            res[const] = 0.5
    gamma = 1.0 + 0.5 * torch.randn(d, generator=g)
    beta = torch.randn(d, generator=g)
    post = torch.randn(7, d, generator=g) if full else None
    rs = (torch.arange(rows) % 5 != 4).float() if full else None
    if rs is not None and const is not None:
        rs[const] = 1.0
    dy = torch.randn(rows, d, generator=g)
    cu = lambda t: None if t is None else t.cuda()
    xc, resc, gc, bc, pc, rsc, dyc = map(cu, (x, res, gamma, beta, post, rs, dy))

    y, z, mean, rstd = _ln_fwd(L, xc, resc, gc, bc, pc, rsc, rows, d, want_z=full)
    z64 = (x + res).double() if full else x.double()
    if full:
        assert torch.equal(z.cpu(), x + res)
    d64 = lambda t: None if t is None else t.double().cuda()
    y_ref, dz_ref, dg_ref, db_ref, m_ref, r_ref = ln_ref(z64.cuda(), d64(gamma), d64(beta), d64(post), d64(rs), LN_EPS,
                                                         d64(dy))
    reg = torch.ones(rows, dtype=torch.bool)
    if const is not None:
        reg[const] = False
        if not full:
            assert torch.equal(y[const].cpu(), beta)
        assert rel_err(y[const], y_ref[const]) < bars["y"]
    assert rel_err(y.cpu()[reg], y_ref.cpu()[reg]) < bars["y"]
    assert rel_err(mean, m_ref) < bars["mean"]
    assert rel_err(rstd.cpu()[reg], r_ref.cpu()[reg]) < bars["rstd"]

    zin = z if full else xc
    dz, dx = _nan(rows, d), _nan(rows, d)
    dgam, dbet = _nan(d), _nan(d)
    _ln_bwd(L, dyc, zin, gc, mean, rstd, rsc, dz, dx, dgam, dbet, rows, d)
    assert torch.equal(dz, dx)
    assert rel_err(dz.cpu()[reg], dz_ref.cpu()[reg]) < bars["dz"]
    if const is not None:
        assert rel_err(dz[const], dz_ref[const]) < bars["dz"]
    assert rel_err(dgam, dg_ref) < bars["dgb"] and rel_err(dbet, db_ref) < bars["dgb"]

    alias, dgam2, dbet2 = _nan(rows, d), _nan(d), _nan(d)
    _ln_bwd(L, dyc, zin, gc, mean, rstd, rsc, alias, alias, dgam2, dbet2, rows, d)
    assert torch.equal(alias, dz) and torch.equal(dgam2, dgam) and torch.equal(dbet2, dbet)

    gbase, bbase = torch.randn(d, generator=g), torch.randn(d, generator=g)
    dgam3, dbet3 = gbase.cuda(), bbase.cuda()
    _ln_bwd(L, dyc, zin, gc, mean, rstd, rsc, _nan(rows, d), None, dgam3, dbet3, rows, d, accumulate=1)
    assert rel_err(dgam3, gbase.double().cuda() + dg_ref) < bars["dgb"]
    assert rel_err(dbet3, bbase.double().cuda() + db_ref) < bars["dgb"]


@gpu
@pytest.mark.parametrize("rows,d", [(300, 64), (301, 200), (40, 1024), (10000, 512)])
def test_add_layernorm_dropout_against_float64(L, rows, d):
    """Dropout on the LayerNorm input (residual NULL, nonzero x): the keep mask is read back from the saved z -- kept
    elements equal x * 1/(1-p) bit for bit, dropped ones are 0 --, the float64 reference normalises that z, and the backward
    must apply the same mask: dx = dz * keep / (1-p), bit for bit from dz and against float64; with dx == dz the buffer ends
    up holding dx.  Measured maxima: y 1.4e-7, dz 2.6e-7, dx 3.0e-7, dgamma / dbeta 2.0e-7 (LN_BARS)."""
    p = 0.1
    g = _gen(rows + d)
    x = torch.randn(rows, d, generator=g) + 0.5
    x[x == 0] = 1.0
    gamma = 1.0 + 0.5 * torch.randn(d, generator=g)
    beta = torch.randn(d, generator=g)
    dy = torch.randn(rows, d, generator=g)
    xc, gc, bc, dyc = x.cuda(), gamma.cuda(), beta.cuda(), dy.cuda()
    y, z, mean, rstd = _ln_fwd(L, xc, None, gc, bc, None, None, rows, d, p=p)
    keep = z != 0
    ik = _inv_keep(p)
    assert torch.equal(z[keep], (xc * ik)[keep])
    assert 0.85 < float(keep.float().mean()) < 0.95
    y_ref, dz_ref, dg_ref, db_ref, _, _ = ln_ref(z.double(), gamma.double().cuda(), beta.double().cuda(), None, None,
                                                 LN_EPS, dy.double().cuda())
    assert rel_err(y, y_ref) < LN_BARS["y"]
    dz, dx, dgam, dbet = _nan(rows, d), _nan(rows, d), _nan(d), _nan(d)
    _ln_bwd(L, dyc, z, gc, mean, rstd, None, dz, dx, dgam, dbet, rows, d, p=p)
    assert rel_err(dz, dz_ref) < LN_BARS["dz"]
    assert torch.equal(dx, torch.where(keep, dz * ik, torch.zeros_like(dz)))
    assert rel_err(dx, dz_ref * keep * ik) < LN_BARS["dz"]
    assert rel_err(dgam, dg_ref) < LN_BARS["dgb"] and rel_err(dbet, db_ref) < LN_BARS["dgb"]
    alias = _nan(rows, d)
    _ln_bwd(L, dyc, z, gc, mean, rstd, None, alias, alias, _nan(d), _nan(d), rows, d, p=p)
    assert torch.equal(alias, dx)


@gpu
def test_add_layernorm_rejects_wide_rows(L):
    """d = 1028 is past the NV = 8 instantiation (d <= 1024): both directions return B200ASR_BAD_SHAPE without launching."""
    lib = L.load()
    rows, d = 4, 1028
    t = torch.zeros(rows, d, device="cuda")
    v = torch.zeros(d, device="cuda")
    s = torch.zeros(rows, device="cuda")
    assert lib.b200asr_add_ln_fwd(L.ptr(t), None, L.ptr(v), L.ptr(v), None, 0, None, L.ptr(t), L.ptr(t), L.ptr(s), L.ptr(s),
                                  rows, d, LN_EPS, 0.0, 0, 0, _stream()) == BAD_SHAPE
    ws = torch.zeros(1 << 16, device="cuda")
    assert lib.b200asr_add_ln_bwd(L.ptr(t), L.ptr(t), L.ptr(v), L.ptr(s), L.ptr(s), None, L.ptr(t), L.ptr(t), L.ptr(v), L.ptr(v),
                                  L.ptr(ws), rows, d, 0.0, 0, 0, 0, _stream()) == BAD_SHAPE


# ================================================================================================ 2. attention
ATT_TK = [1, 3, 128, 129, 300, 515, 1025, 2048]    # row pitch 4..2048: NV = 1, 1, 1, 2, 4, 8, 16, 16
ATT_MODES = ["key_pad", "causal_long_q", "causal_short_q", "dense", "dead_row"]
# measured maxima: 3xTF32 P 2.4e-6, O 2.2e-5, gradients 2.2e-5 (with dropout 1.4e-5); TF32 P 6.6e-4, O 7.2e-4, gradients 1.1e-3
ATT_BARS = {3: dict(p=1e-5, o=7e-5, grad=7e-5), 1: dict(p=2e-3, o=2.5e-3, grad=3e-3)}
ATT_B, ATT_H, ATT_DK, ATT_DV = 2, 2, 64, 32


def _attn_case(Tq, Tk, mode, seed):
    """q token-major [B, Tq, H, dk] (the projections' layout), k / v head-major [B, H, Tk, d]; masks for `mode`."""
    B, H = ATT_B, ATT_H
    g = _gen(seed)
    q = torch.randn(B, Tq, H, ATT_DK, generator=g)
    k = torch.randn(B, H, Tk, ATT_DK, generator=g)
    v = torch.randn(B, H, Tk, ATT_DV, generator=g)
    dout = torch.randn(B, Tq, H, ATT_DV, generator=g)
    key_pad = dense = None
    causal = mode.startswith("causal")
    if mode in ("key_pad", "dead_row"):
        lens = torch.tensor([Tk, max(1, Tk - Tk // 3)])
        key_pad = (torch.arange(Tk)[None, :] >= lens[:, None]).to(torch.uint8)
    if mode == "dense":
        dense = (torch.rand(B, Tq, Tk, generator=g) < 0.3).to(torch.uint8)
        dense[:, torch.arange(Tq), torch.arange(Tq) % Tk] = 0          # every row keeps a key
    if mode == "dead_row":
        dense = torch.zeros(B, Tq, Tk, dtype=torch.uint8)
        dense[1, Tq // 2] = 1                                          # one fully masked query row in batch 1 (every head)
    return q, k, v, dout, key_pad, dense, causal


def _bhtd(t):
    """element (b, h, t, c) strides of a [B, T, H, d] (token-major) or [B, H, T, d] tensor, as (bs, hs, rs)."""
    return t.stride(0), t.stride(1), t.stride(2)


def _mat_call(L, q, k, v, dout, key_pad, dense, causal, Tq, Tk, prec, p_drop=0.0):
    """Runs b200asr_sdpa_mat_fwd / _bwd with every output and workspace NaN-poisoned.  q / dout / out / dq are token-major
    [B, Tq, H, d], passed through their (b, h, t) strides."""
    lib = L.load()
    B, H = ATT_B, ATT_H
    st = _stream()
    qc, kc, vc, doc = q.cuda(), k.cuda(), v.cuda(), dout.cuda()
    qv = qc.permute(0, 2, 1, 3)                        # (b, h, t, c) views
    dov = doc.permute(0, 2, 1, 3)
    kp = None if key_pad is None else key_pad.cuda()
    dn = None if dense is None else dense.cuda()
    n = lib.b200asr_sdpa_mat_ws_bytes(B, H, Tq, Tk) // 4
    ldp = (Tk + 3) // 4 * 4
    assert n == B * H * Tq * ldp
    probs, dp = _nan(n), _nan(n)
    probs_drop = _nan(n) if p_drop > 0 else None
    out = _nan(B, Tq, H, ATT_DV)
    ov = out.permute(0, 2, 1, 3)
    scale = ATT_DK ** -0.5
    L.check(lib.b200asr_sdpa_mat_fwd(L.ptr(qc), L.ptr(kc), L.ptr(vc), *_bhtd(qv), *_bhtd(kc), *_bhtd(vc), L.ptr(kp), L.ptr(dn),
                                     int(causal), L.ptr(out), *_bhtd(ov), L.ptr(probs), L.ptr(probs_drop), B, H, Tq, Tk,
                                     ATT_DK, ATT_DV, scale, p_drop, 77, 5, prec, st), "sdpa_mat_fwd")
    dq, dk, dv = _nan(B, Tq, H, ATT_DK), _nan(B, H, Tk, ATT_DK), _nan(B, H, Tk, ATT_DV)
    L.check(lib.b200asr_sdpa_mat_bwd(L.ptr(doc), L.ptr(qc), L.ptr(kc), L.ptr(vc), *_bhtd(qv), *_bhtd(kc), *_bhtd(vc),
                                     *_bhtd(dov), L.ptr(probs), L.ptr(probs_drop), L.ptr(dq), L.ptr(dk), L.ptr(dv), L.ptr(dp),
                                     B, H, Tq, Tk, ATT_DK, ATT_DV, scale, p_drop, 77, 5, prec, st), "sdpa_mat_bwd")
    shape = (B, H, Tq, ldp)
    pd = None if probs_drop is None else probs_drop.view(shape)
    return probs.view(shape), pd, ov, dq.permute(0, 2, 1, 3), dk, dv


def _attn_ref_grads(q, k, v, dout, mask, keep=None, inv_keep=1.0):
    """float64 forward and autograd backward on the GPU; q / dout token-major as given to the kernels."""
    q64 = q.permute(0, 2, 1, 3).double().cuda().requires_grad_(True)
    k64 = k.double().cuda().requires_grad_(True)
    v64 = v.double().cuda().requires_grad_(True)
    o, p = attn_ref(q64, k64, v64, mask.cuda(), ATT_DK ** -0.5, None if keep is None else keep.double(), inv_keep)
    o.backward(dout.permute(0, 2, 1, 3).double().cuda())
    return p.detach(), o.detach(), q64.grad, k64.grad, v64.grad


@gpu
@pytest.mark.parametrize("prec", [3, 1])
@pytest.mark.parametrize("mode", ATT_MODES)
@pytest.mark.parametrize("Tk", ATT_TK)
def test_materialised_attention_against_float64(L, Tk, mode, prec):
    """b200asr_sdpa_mat_fwd / _bwd at 3xTF32 and TF32 with probs and the dP workspace poisoned with NaN: P against a
    float64 masked softmax; P's padding columns Tk..ldp-1 exactly 0 (the QK^T and dO V^T GEMMs must write them: the softmax
    backward's rowsum(P * dP) reads them); O, dQ, dK, dV against float64.  Masks: key padding, causal with Tq > Tk and
    Tq < Tk, a dense mask, and one fully masked query row (in every head of one utterance: the masks are per utterance).
    NaN must appear exactly where the float64 reference has it: in that row of P (padding columns included) and O, and,
    through P, in all of dV of those heads; masked_fill's backward gives the masked scores a zero gradient, so that row of
    dQ is 0 and dK stays finite.  Measured maxima and bars: ATT_BARS."""
    Tq = {"causal_long_q": Tk + 9, "causal_short_q": max(1, Tk // 3)}.get(mode, 37)
    q, k, v, dout, key_pad, dense, causal = _attn_case(Tq, Tk, mode, seed=Tk * 5 + len(mode) + prec)
    P, _, out, dq, dk, dv = _mat_call(L, q, k, v, dout, key_pad, dense, causal, Tq, Tk, prec)
    mask = attn_mask(ATT_B, Tq, Tk, key_pad, dense, causal)
    p_ref, o_ref, dq_ref, dk_ref, dv_ref = _attn_ref_grads(q, k, v, dout, mask)
    bars = ATT_BARS[prec]
    dead = torch.isnan(p_ref).any(-1)                                  # [B, H, Tq]
    assert bool(dead.any()) == (mode == "dead_row")
    for got, ref in ((P[..., :Tk], p_ref), (out, o_ref), (dq, dq_ref), (dk, dk_ref), (dv, dv_ref)):
        assert _same_nan(got, ref)
    pad = P[..., Tk:]
    assert torch.equal(torch.isnan(pad).any(-1).cpu(), dead.cpu() & (pad.shape[-1] > 0))
    assert not pad[~dead].any()
    assert _finite_err(P[..., :Tk], p_ref) < bars["p"]
    assert _finite_err(out, o_ref) < bars["o"]
    for got, ref in ((dq, dq_ref), (dk, dk_ref), (dv, dv_ref)):
        assert _finite_err(got, ref) < bars["grad"]


@gpu
@pytest.mark.parametrize("Tk", [3, 129, 515, 2048])
def test_materialised_attention_dropout_against_float64(L, Tk):
    """With dropout (p = 0.2, key padding, 3xTF32): probs_drop equals P * 1/(1-p) bit for bit wherever it is nonzero, and is 0
    in the padding columns; the keep mask read back from it, handed to the float64 reference, reproduces O and the
    backward's dQ / dK / dV -- so the backward regenerates the forward's mask."""
    p = 0.2
    Tq = 37
    q, k, v, dout, key_pad, dense, causal = _attn_case(Tq, Tk, "key_pad", seed=Tk)
    P, Pd, out, dq, dk, dv = _mat_call(L, q, k, v, dout, key_pad, dense, causal, Tq, Tk, 3, p_drop=p)
    ik = _inv_keep(p)
    nz = Pd != 0
    assert torch.equal(Pd[nz], (P * ik)[nz])
    assert not Pd[..., Tk:].any()
    live = P[..., :Tk] != 0
    keep = nz[..., :Tk]
    frac = float(keep[live].float().mean())
    assert 0.7 < frac < 0.9 or Tk == 3
    mask = attn_mask(ATT_B, Tq, Tk, key_pad, dense, causal)
    _, o_ref, dq_ref, dk_ref, dv_ref = _attn_ref_grads(q, k, v, dout, mask, keep=keep, inv_keep=ik)
    bars = ATT_BARS[3]
    assert rel_err(out, o_ref) < bars["o"]
    for got, ref in ((dq, dq_ref), (dk, dk_ref), (dv, dv_ref)):
        assert rel_err(got, ref) < bars["grad"]


@gpu
def test_materialised_attention_rejects_long_keys(L):
    """Tk = 2049 is past the NV = 16 softmax instantiation: B200ASR_BAD_SHAPE naming precision 0 as the path that takes it.
    The check runs on the host after the QK^T GEMM has been enqueued, so the buffers are sized by b200asr_sdpa_mat_ws_bytes."""
    lib = L.load()
    B, H, Tq, Tk, d = 1, 1, 8, 2049, 32
    q = torch.randn(B, H, Tq, d, device="cuda")
    k = torch.randn(B, H, Tk, d, device="cuda")
    out = torch.empty(B, H, Tq, d, device="cuda")
    probs = torch.empty(lib.b200asr_sdpa_mat_ws_bytes(B, H, Tq, Tk) // 4, device="cuda")
    rc = lib.b200asr_sdpa_mat_fwd(L.ptr(q), L.ptr(k), L.ptr(k), *_bhtd(q), *_bhtd(k), *_bhtd(k), None, None, 0, L.ptr(out),
                                  *_bhtd(out), L.ptr(probs), None, B, H, Tq, Tk, d, d, 0.125, 0.0, 0, 0, 3, _stream())
    torch.cuda.synchronize()
    assert rc == BAD_SHAPE and "precision 0" in L.last_error()


# ================================================================================================ 3. loss, argmax, greedy
CE_V = [2, 33, 255, 256, 257, 4364]
CE_ROWS = 41
CE_PAD_ROWS = (3, 17, 40)
# measured maxima: row_lse 8.9e-8, loss sum 1.4e-7, mean 1.7e-7, single row losses 2.5e-7, gradient 7.9e-6 (exp(x - lse) with
# x - lse down to -200 at x30: the argument's rounding).  Logits shifted by +200 measure the same; before the loss was
# computed relative to the row maximum they measured 2.8e-6 on the sum and 7.6e-5 on single rows.
CE_BARS = dict(lse=3e-7, loss=5e-7, row_loss=8e-7, grad=2.5e-5)


def _ce_case(V, scale, shift, seed):
    """Logits with PAD rows, rows whose maximum is tied between two indices (gold = the first one: correct; the second:
    incorrect), and rows whose gold is the argmax."""
    g = _gen(seed)
    x = torch.randn(CE_ROWS, V, generator=g) * scale + shift
    gold = torch.randint(1, max(V, 2), (CE_ROWS,), generator=g)
    ties = [(5, 0, V - 1, "first"), (6, V // 2 - 1, V // 2, "second"), (7, 1 % V, V - 1, "second")]
    for r, a, b, who in ties:
        if a == b:
            continue
        top = x[r].max() + scale
        x[r, a] = x[r, b] = top
        gold[r] = a if who == "first" else b
    for r in range(8, 13):
        gold[r] = int(x[r].argmax())
    gold[gold == 0] = 1 if V > 1 else 0
    for r in CE_PAD_ROWS:
        gold[r] = O.PAD
    return x, gold


@gpu
@pytest.mark.parametrize("scale,shift", [(1.0, 0.0), (30.0, 0.0), (1.0, 200.0)])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("V", CE_V)
def test_cross_entropy_against_float64(L, V, eps, scale, shift):
    """b200asr_ce_fwd / _finalize / _bwd against the float64 restatement of calculate_loss: row_lse against logsumexp, the loss
    sum (and, from one-row calls, single row losses), exact counts of non-PAD rows and of correct argmaxes (ties: the first
    index wins), mean and reciprocal count; the gradient scaled by gscale * gscale_dev * gscale_dev2 against float64 autograd,
    PAD rows exactly 0.  V from 2 (a partial warp) to 4364, V % 32 != 0, V around one 256-thread block; logits x1, x30 and
    shifted by +200.  Measured maxima and bars: CE_BARS."""
    lib = L.load()
    st = _stream()
    x, gold = _ce_case(V, scale, shift, seed=V * 3 + int(eps * 10) + int(scale) + int(shift))
    xc, gc = x.cuda(), gold.cuda()
    x64 = x.double().cuda().requires_grad_(True)
    loss_ref, lse_ref = ce_rows_ref(x64, gc, eps)
    loss_ref.sum().backward()
    valid = gold != O.PAD
    n = int(valid.sum())
    hyp = np.argmax(x.numpy(), axis=1)
    correct = int(((torch.from_numpy(hyp) == gold) & valid).sum())

    lse, stats, loss_out = _nan(CE_ROWS), _nan(5), _nan(1)
    L.check(lib.b200asr_ce_fwd(L.ptr(xc), L.ptr(gc), L.ptr(lse), L.ptr(stats), CE_ROWS, V, eps, st), "ce_fwd")
    L.check(lib.b200asr_ce_finalize(L.ptr(stats), L.ptr(loss_out), 1, st), "ce_finalize")
    s = stats.cpu()
    assert rel_err(lse, lse_ref) < CE_BARS["lse"]
    assert rel_err(s[0:1], loss_ref.sum().view(1)) < CE_BARS["loss"]
    assert s[1].item() == n and s[2].item() == correct
    assert rel_err(s[3:4], (loss_ref.sum() / n).view(1)) < CE_BARS["loss"]
    assert s[4].item() == float(np.float32(1.0) / np.float32(n)) and loss_out.item() == s[3].item()
    for r in (0, 5, 6, 20):                                            # losses well away from 0
        one_lse, one = _nan(1), _nan(5)
        L.check(lib.b200asr_ce_fwd(L.ptr(xc[r:r + 1]), L.ptr(gc[r:r + 1]), L.ptr(one_lse), L.ptr(one), 1, V, eps, st), "ce_fwd")
        assert rel_err(one[0:1], loss_ref[r:r + 1]) < CE_BARS["row_loss"], r

    gs_dev, gs_dev2 = torch.tensor([0.25], device="cuda"), torch.tensor([3.0], device="cuda")
    dl = _nan(CE_ROWS, V)
    L.check(lib.b200asr_ce_bwd(L.ptr(xc), L.ptr(gc), L.ptr(lse), L.ptr(dl), CE_ROWS, V, eps, 0.5, L.ptr(gs_dev), L.ptr(gs_dev2),
                               st), "ce_bwd")
    assert not dl[~valid.cuda()].any()
    assert rel_err(dl, x64.grad * 0.375) < CE_BARS["grad"]


@gpu
@pytest.mark.parametrize("V", [1, 5, 17, 31, 32, 33, 4364])
def test_argmax_rows_ties_and_infinite_rows(L, V):
    """b200asr_argmax_rows: the first index of the maximum (torch.max / numpy), with ties inside a lane, across lanes and at
    both ends of the row, rows that are entirely -inf (index 0), and V below one warp."""
    lib = L.load()
    g = _gen(V)
    rows = 12
    x = torch.randn(rows, V, generator=g)
    x[0] = float("-inf")
    x[1, :] = 2.0                                              # every element ties
    if V > 1:
        x[2, V - 1] = x[2, 0] = 9.0
        x[3, V // 2] = x[3, V - 1] = 9.0
    if V > 33:
        x[4, 1] = x[4, 33] = 9.0                               # the same lane, two strides apart
    x[5, :] = float("-inf")
    x[5, V - 1] = -1e30
    out = torch.full((rows,), -7, dtype=torch.int64, device="cuda")
    L.check(lib.b200asr_argmax_rows(L.ptr(x.cuda()), L.ptr(out), rows, V, _stream()), "argmax_rows")
    assert out.cpu().tolist() == np.argmax(x.numpy(), axis=1).tolist()


@gpu
def test_greedy_step_eos_bookkeeping(L):
    """b200asr_greedy_step over several steps: utterance b emits EOS at step b (and again two steps later), one utterance
    never does, one step has a tie.  next_tok is the first argmax; ys holds the token, or -1 from the first EOS on;
    finished marks each utterance once and n_finished counts each once."""
    lib = L.load()
    st = _stream()
    B, V, steps = 6, 37, 7
    g = _gen(4)
    logits = torch.randn(steps, B, V, generator=g)
    logits[:, :, 2] = -50.0
    for b in range(5):
        logits[b, b, 2] = 50.0
        if b + 2 < steps:
            logits[b + 2, b, 2] = 50.0
    logits[3, 5, 4] = logits[3, 5, 30] = 60.0
    ys = torch.full((B, steps), -9, dtype=torch.int64, device="cuda")
    nxt = torch.full((B,), -9, dtype=torch.int64, device="cuda")
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    nfin = torch.zeros(1, dtype=torch.int32, device="cuda")
    done = [False] * B
    want_ys = torch.empty(B, steps, dtype=torch.int64)
    for t in range(steps):
        L.check(lib.b200asr_greedy_step(L.ptr(logits[t].cuda()), L.ptr(nxt), L.ptr(ys), L.ptr(fin), L.ptr(nfin), B, V, t, steps,
                                        st), "greedy_step")
        tok = np.argmax(logits[t].numpy(), axis=1)
        assert nxt.cpu().tolist() == tok.tolist()
        for b in range(B):
            want_ys[b, t] = -1 if done[b] or tok[b] == 2 else int(tok[b])
            done[b] = done[b] or tok[b] == 2
        assert fin.cpu().tolist() == [int(d) for d in done]
        assert nfin.item() == sum(done)
    assert torch.equal(ys.cpu(), want_ys) and nfin.item() == 5


# ================================================================================================ 4. embedding
EMB_BARS = dict(fwd=3e-7, bwd=1e-6)           # measured maxima 8.0e-8, 2.9e-7


@gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("d", [200, 512])
def test_embedding_against_float64(L, d, p):
    """b200asr_embed_fwd / _bwd (pad_idx 0) against float64 with heavy repetition: tokens drawn from 12 ids, one id in every
    utterance, one only in the last row, PAD tails.  Forward: table[tok] * scale + pe[row % T], dropout mask read back from
    the output.  Backward: dtable starts nonzero and must end as that base plus the scattered gradient of the non-PAD rows
    (the same mask); untouched table rows (the PAD row included) keep their bits; two calls give identical bits."""
    lib = L.load()
    st = _stream()
    B, T, V, scale = 8, 75, 60, 0.7
    rows = B * T
    g = _gen(d + int(p * 10))
    tok = torch.randint(1, 13, (B, T), generator=g)
    tok[torch.arange(B), (torch.arange(B) * 7) % 11] = 20               # in every utterance
    tok[tok == V - 1] = 1
    tok[B - 1, T - 1] = V - 1                                           # only in the last row
    tok[2, 50:] = 0
    tok[5, 11:] = 0
    tok = tok.view(-1)
    table = torch.randn(V, d, generator=g)
    pe = torch.randn(T, d, generator=g)
    dout = torch.randn(rows, d, generator=g)
    base = torch.randn(V, d, generator=g)
    tc, tabc, pec, doc = tok.cuda(), table.cuda(), pe.cuda(), dout.cuda()
    out = _nan(rows, d)
    L.check(lib.b200asr_embed_fwd(L.ptr(tc), L.ptr(tabc), L.ptr(pec), L.ptr(out), rows, T, d, V, scale, p, 13, 2, st),
            "embed_fwd")
    ref = table.double()[tok] * scale + pe.double()[torch.arange(rows) % T]
    ik = _inv_keep(p) if p > 0 else 1.0
    keep = (out != 0).cpu()
    if p == 0:
        assert bool(keep.all())
    else:
        assert 0.85 < float(keep.float().mean()) < 0.95
    assert rel_err(out, ref * keep * ik) < EMB_BARS["fwd"]

    outs = []
    for _ in range(2):
        dt = base.cuda()
        L.check(lib.b200asr_embed_bwd(L.ptr(tc), L.ptr(doc), L.ptr(dt), rows, d, V, scale, p, 13, 2, 0, st), "embed_bwd")
        outs.append(dt)
    assert torch.equal(outs[0], outs[1])
    contrib = dout.double() * keep * (scale * ik)
    live = tok != 0
    want = base.double().index_add(0, tok[live], contrib[live])
    assert rel_err(outs[0], want) < EMB_BARS["bwd"]
    untouched = torch.ones(V, dtype=torch.bool)
    untouched[tok[live]] = False
    assert untouched[0] and torch.equal(outs[0].cpu()[untouched], base[untouched])



# ================================================================================================ 5. step tail
ADAM = dict(lr=2e-3, b1=0.9, b2=0.98, eps=1e-9)
ADAM_BARS = dict(p=3e-6, m=5e-7, v=3e-6)     # measured maxima 8.1e-7, 1.6e-7, 1.0e-6


@gpu
@pytest.mark.parametrize("dev", [False, True])
@pytest.mark.parametrize("step", [1, 2, 10, 1000, 100000])
def test_adam_step_against_float64(L, step, dev):
    """b200asr_adam_step from a given (m, v) at step counts up to 100000 (the host's float bias corrections against torch's
    double ones), with the gradient scaled by gscale and optionally *gscale_dev.  The parameters are small next to one
    step's update, so p measures the update itself.  Measured maxima and bars: ADAM_BARS."""
    lib = L.load()
    n = 10007
    g = _gen(step + dev)
    p = torch.randn(n, generator=g) * 1e-3
    gr = torch.randn(n, generator=g) * 0.1
    m = torch.randn(n, generator=g) * 1e-2
    v = torch.rand(n, generator=g) * 1e-4
    pc, gc, mc, vc = p.cuda(), gr.cuda(), m.cuda(), v.cuda()
    gdev = torch.tensor([0.3], device="cuda") if dev else None
    L.check(lib.b200asr_adam_step(L.ptr(pc), L.ptr(gc), L.ptr(mc), L.ptr(vc), n, ADAM["lr"], ADAM["b1"], ADAM["b2"], ADAM["eps"],
                                  step, 0.5, L.ptr(gdev), _stream()), "adam_step")
    gscaled = gr.double() * 0.5 * (float(np.float32(0.3)) if dev else 1.0)
    p_ref, m_ref, v_ref = adam_ref(p.double(), gscaled, m.double(), v.double(), step, **ADAM)
    assert rel_err(pc, p_ref) < ADAM_BARS["p"]
    assert rel_err(mc, m_ref) < ADAM_BARS["m"]
    assert rel_err(vc, v_ref) < ADAM_BARS["v"]


SUMSQ_BAR = 4e-7                               # measured maximum 1.1e-7
GRAD_SCALE_BAR = 1e-7                           # measured maximum 2.4e-8


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@gpu
@pytest.mark.parametrize("which", ["1", "4099", "cap+5", "5e7"])
def test_sumsq_against_float64(L, which):
    """b200asr_sumsq adds sum(g^2) to out[0]: n = 1, 4099, and two sizes past the grid cap of 8 blocks per SM of 2048
    elements each, where the blocks stride over the tail.  Against float64; two calls give identical bits."""
    lib = L.load()
    n = {"1": 1, "4099": 4099, "cap+5": 8 * _sms() * 2048 + 5, "5e7": 50_000_000}[which]
    gen = torch.Generator(device="cuda").manual_seed(n % 1000)
    x = torch.randn(n, generator=gen, device="cuda")
    outs = []
    for _ in range(2):
        out = torch.tensor([1.5], device="cuda")
        L.check(lib.b200asr_sumsq(L.ptr(x), n, L.ptr(out), _stream()), "sumsq")
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    want = 1.5 + (x.double() ** 2).sum()
    assert rel_err(outs[0], want.view(1)) < SUMSQ_BAR



@gpu
@pytest.mark.parametrize("clip", ["active", "inactive", "off"])
def test_grad_scale_against_clip_grad_norm(L, clip):
    """b200asr_grad_scale on 3e6 elements (past the sum of squares' grid cap): out[0] = (1 / n_tokens) * clip coefficient and
    out[1] = the norm of the token-normalised gradient, against torch.nn.utils.clip_grad_norm_ in float64 on g / n_tokens;
    without clipping (max_norm 0) out = (1 / n_tokens, 0).  Two calls give identical bits."""
    lib = L.load()
    n = 3_000_000
    gen = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(n, generator=gen, device="cuda")
    ntok = torch.tensor([37.0], device="cuda")
    norm = float((x.double() ** 2).sum().sqrt()) / 37.0
    max_norm = {"active": 0.1 * norm, "inactive": 10.0 * norm, "off": 0.0}[clip]
    outs = []
    for _ in range(2):
        out, scratch = _nan(2), _nan(1)
        L.check(lib.b200asr_grad_scale(L.ptr(x), n, L.ptr(ntok), max_norm, L.ptr(scratch), L.ptr(out), _stream()), "grad_scale")
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    got = outs[0].cpu()
    if clip == "off":
        assert got[0].item() == float(np.float32(1.0) / np.float32(37.0)) and got[1].item() == 0.0
        return
    g64 = x.double() / 37.0
    prm = torch.nn.Parameter(torch.zeros(n, dtype=torch.float64, device="cuda"))
    prm.grad = g64.clone()
    total = float(torch.nn.utils.clip_grad_norm_([prm], float(np.float32(max_norm))))
    coef = float(prm.grad.norm() / g64.norm())
    assert (coef < 1.0) == (clip == "active")
    assert rel_err(got[0:1], torch.tensor([coef / 37.0], dtype=torch.float64)) < GRAD_SCALE_BAR
    assert rel_err(got[1:2], torch.tensor([total], dtype=torch.float64)) < GRAD_SCALE_BAR



# ================================================================================================ 6. BatchNorm + Hardtanh
BN_EPS, BN_MOM, BN_LO, BN_HI = 1e-5, 0.1, 0.0, 20.0
# measured maxima: y 5.3e-8, dx 1.7e-7, dgamma 3.8e-7, dbeta 2.5e-7, mean 1.1e-7, invstd 4.3e-6, running statistics 1.1e-7.
# The channel with mean 1e3 has its own bars: there x itself carries 3e-5 of its std in rounding and the fp32 batch mean about
# 1e-4, which every normalised value inherits -- measured y 1.3e-5, dx 5.9e-6, and 1.2e-4 on dgamma / dbeta over all channels.
BN_BARS = dict(y=2e-7, dx=5e-7, dgb=1.2e-6, stats=4e-7, invstd=1.5e-5, running=4e-7)
BN_BARS_MEAN1E3 = dict(y=4e-5, dx=2e-5, dgb=4e-4)


def _bn_input(B, C, H, W, seed):
    """[B, C, H, W] with C = 6 channels: 0 -- mean 1e3, std 1; 1 and 2 -- every (b, h) row is a set of multiples of 1/8, their
    negations and zeros, so every partial sum and the batch mean are exactly 0 and the zeros normalise to beta exactly
    (beta 0 and 20: the clamp bounds); 3 -- a mean that moves with h (the per-split means differ); 4, 5 -- normal."""
    g = _gen(seed)
    x = torch.randn(B, C, H, W, generator=g)
    x[:, 0] += 1000.0
    for c in (1, 2):
        k = (W - 1) // 2
        for b in range(B):
            for h in range(H):
                half = torch.randint(1, 33, (k,), generator=g).float() / 8.0
                half *= torch.where(torch.rand(k, generator=g) < 0.5, -1.0, 1.0)
                row = torch.cat([half, -half, torch.zeros(W - 2 * k)])
                x[b, c, h] = row[torch.randperm(W, generator=g)]
    x[:, 3] += 0.5 * torch.arange(H).float()[None, :, None]
    gamma = torch.tensor([1.0, 1.5, 2.0, 0.8, 1.2, -0.7])
    beta = torch.tensor([5.0, 0.0, 20.0, 1.0, 3.0, 4.0])
    dy = torch.randn(B, C, H, W, generator=g)
    return x, gamma, beta, dy


def _pitched(t, pitch):
    """t [B, C, H, W] copied into a NaN-filled [B, C, H, pitch] buffer; returns (buffer, view)."""
    buf = _nan(*t.shape[:3], pitch)
    view = buf[..., :t.shape[3]]
    view.copy_(t)
    return buf, view


@gpu
@pytest.mark.parametrize("training", [1, 0])
@pytest.mark.parametrize("B,H,W", [(1, 7, 13), (3, 11, 37), (2, 40, 50)])
def test_batchnorm_hardtanh_against_float64(L, B, H, W, training):
    """b200asr_bn_clamp_fwd / _bwd against F.batch_norm + hardtanh(0, 20) + autograd in float64.  B*H = 7 (25 of the 32 row
    splits empty), 33 (not a multiple of 32) and 80; row pitches W+3 (x), W+1 (y), W+5 (dy) and W+2 (dx), whose padding
    (NaN) must be neither read nor written; a channel with mean 1e3 and std 1; values exactly at both clamp bounds after
    normalisation, whose gradient must be 0 (ATen's strict inequalities).  Training: batch statistics, the running-state
    update with momentum and num_batches_tracked + 1; eval: the running statistics and no statistics term in the backward.
    Two calls give identical bits.  Measured maxima and bars: BN_BARS."""
    lib = L.load()
    st = _stream()
    C = 6
    x, gamma, beta, dy = _bn_input(B, C, H, W, seed=B * 100 + H + W)
    g = _gen(W)
    x64 = x.double()
    bmean, bvar = x64.mean((0, 2, 3)), x64.var((0, 2, 3), unbiased=False)
    rm = (bmean + 0.1 * torch.randn(C, generator=g).double()).float()
    rv = (bvar * (1.0 + 0.2 * torch.rand(C, generator=g).double())).float()
    rm[1] = rm[2] = 0.0
    xb, xv = _pitched(x.cuda(), W + 3)
    dyb, dyv = _pitched(dy.cuda(), W + 5)
    gc, bc = gamma.cuda(), beta.cuda()
    ws = _nan(lib.b200asr_bn_ws_bytes(C) // 4)
    runs = []
    for _ in range(2):
        yb = _nan(B, C, H, W + 1)
        dxb = _nan(B, C, H, W + 2)
        mean, invstd = _nan(C), _nan(C)
        rmc, rvc = rm.cuda(), rv.cuda()
        nbt = torch.tensor([5], dtype=torch.int64, device="cuda")
        dgam, dbet = _nan(C), _nan(C)
        L.check(lib.b200asr_bn_clamp_fwd(L.ptr(xv), L.ptr(gc), L.ptr(bc), L.ptr(yb), L.ptr(mean), L.ptr(invstd), L.ptr(rmc),
                                         L.ptr(rvc), L.ptr(nbt), L.ptr(ws), B, C, H, W, W + 3, W + 1, BN_EPS, BN_MOM, training,
                                         BN_LO, BN_HI, st), "bn_clamp_fwd")
        L.check(lib.b200asr_bn_clamp_bwd(L.ptr(dyv), L.ptr(xv), L.ptr(yb), L.ptr(gc), L.ptr(mean), L.ptr(invstd), L.ptr(dxb),
                                         L.ptr(dgam), L.ptr(dbet), L.ptr(ws), B, C, H, W, W + 5, W + 3, W + 1, W + 2, training,
                                         BN_LO, BN_HI, st), "bn_clamp_bwd")
        runs.append((yb, dxb, mean, invstd, rmc, rvc, nbt, dgam, dbet))
    for a, b in zip(*runs):
        assert torch.equal(a.cpu().view(torch.int32) if a.dtype == torch.float32 else a.cpu(),
                           b.cpu().view(torch.int32) if b.dtype == torch.float32 else b.cpu())
    yb, dxb, mean, invstd, rmc, rvc, nbt, dgam, dbet = runs[0]
    assert torch.isnan(yb[..., W:]).all() and torch.isnan(dxb[..., W:]).all()
    y, dx = yb[..., :W], dxb[..., :W]

    xr = x64.clone().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rm64, rv64 = rm.double(), rv.double()
    y_ref = F.hardtanh(F.batch_norm(xr, rm64, rv64, gr, br, training=bool(training), momentum=BN_MOM, eps=BN_EPS), BN_LO, BN_HI)
    y_ref.backward(dy.double())
    at_bound = (y_ref.detach() == BN_LO) | (y_ref.detach() == BN_HI)
    exact = y_ref.detach()[:, 1:3]
    assert bool(((exact == BN_LO) | (exact == BN_HI)).any())            # the exact-bound values occur
    zero_x = x[:, 1:3] == 0
    assert torch.equal(y[:, 1:3].cpu()[zero_x], y_ref.detach()[:, 1:3][zero_x].float())
    if not training:                                                    # no statistics term: clamped elements get 0
        assert not dx.cpu()[at_bound].any()
    assert rel_err(y[:, :1], y_ref[:, :1]) < BN_BARS_MEAN1E3["y"]
    assert rel_err(dx[:, :1], xr.grad[:, :1]) < BN_BARS_MEAN1E3["dx"]
    assert rel_err(y[:, 1:], y_ref[:, 1:]) < BN_BARS["y"]
    assert rel_err(dx[:, 1:], xr.grad[:, 1:]) < BN_BARS["dx"]
    assert rel_err(dgam, gr.grad) < BN_BARS_MEAN1E3["dgb"] and rel_err(dbet, br.grad) < BN_BARS_MEAN1E3["dgb"]
    assert rel_err(dgam[1:], gr.grad[1:]) < BN_BARS["dgb"]
    assert rel_err(dbet[1:], br.grad[1:]) < BN_BARS["dgb"]
    if training:
        assert rel_err(mean, bmean) < BN_BARS["stats"]
        assert rel_err(invstd, 1.0 / torch.sqrt(bvar + BN_EPS)) < BN_BARS["invstd"]
        assert rel_err(rmc, rm64) < BN_BARS["running"] and rel_err(rvc, rv64) < BN_BARS["running"]
        assert nbt.item() == 6
    else:
        assert torch.equal(mean.cpu(), rm) and torch.equal(rmc.cpu(), rm) and torch.equal(rvc.cpu(), rv) and nbt.item() == 5
        assert rel_err(invstd, 1.0 / torch.sqrt(rv.double() + BN_EPS)) < BN_BARS["invstd"]


# ================================================================================================ 7. CPU pins of the references
@pytest.mark.parametrize("shift", [0.0, 200.0])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_cross_entropy_reference_matches_oracle(eps, shift):
    """ce_rows_ref, summed over the non-PAD rows and divided by their count, is the oracle's cross_entropy_loss (golden
    pinned) in float64."""
    g = _gen(5)
    x = torch.randn(30, 257, generator=g, dtype=torch.float64) * 3 + shift
    gold = torch.randint(1, 257, (30,), generator=g)
    gold[[2, 11, 29]] = O.PAD
    loss, _ = ce_rows_ref(x, gold, eps)
    want, n_word = O.cross_entropy_loss(x, gold, eps)
    got = loss.sum() / n_word
    assert abs(float(got) - float(want)) <= 1e-12 * abs(float(want))


def test_attention_reference_matches_oracle():
    """attn_ref with the masks of attn_mask is the oracle's scaled_dot_attention (golden pinned) in float64: heads as
    a batch dimension, key padding + causal + dense masks, a temperature of 1 / scale."""
    g = _gen(6)
    B, H, Tq, Tk, dk = 2, 3, 9, 13, 64
    q = torch.randn(B, H, Tq, dk, generator=g, dtype=torch.float64)
    k = torch.randn(B, H, Tk, dk, generator=g, dtype=torch.float64)
    v = torch.randn(B, H, Tk, 32, generator=g, dtype=torch.float64)
    key_pad = (torch.arange(Tk)[None, :] >= torch.tensor([Tk, 8])[:, None]).to(torch.uint8)
    dense = (torch.rand(B, Tq, Tk, generator=g) < 0.2).to(torch.uint8)
    dense[:, :, 0] = 0
    for causal in (False, True):
        mask = attn_mask(B, Tq, Tk, key_pad, dense, causal)
        o, p = attn_ref(q, k, v, mask, dk ** -0.5)
        flat = lambda t: t.reshape(B * H, *t.shape[2:])
        o_or, p_or = O.scaled_dot_attention(flat(q), flat(k), flat(v), flat(mask[:, None].expand(B, H, Tq, Tk)), dk ** 0.5)
        assert rel_err(flat(o), o_or) < 1e-12 and rel_err(flat(p), p_or) < 1e-12


@pytest.mark.parametrize("step", [1, 10, 100000])
def test_adam_reference_matches_oracle(step):
    """adam_ref (torch.optim.Adam's arrangement of the bias corrections) is the oracle's adam_reference in float64."""
    g = _gen(step)
    p, gr, m = (torch.randn(1000, generator=g, dtype=torch.float64) for _ in range(3))
    v = torch.rand(1000, generator=g, dtype=torch.float64)
    got = adam_ref(p, gr, m, v, step, **ADAM)
    want = O.adam_reference(p, gr, m, v, step, ADAM["lr"], ADAM["b1"], ADAM["b2"], ADAM["eps"])
    assert rel_err(got[0] - p, want[0] - p) < 1e-12
    assert rel_err(got[1], want[1]) < 1e-12 and rel_err(got[2], want[2]) < 1e-12


# ================================================================================================ 8. emb_cnn step reproducibility
@gpu
def test_emb_cnn_training_step_is_bit_reproducible(L):
    """Two identical training steps of a 1-layer model with the cfg3 architecture (emb_cnn front end: implicit-GEMM
    convolutions with split weight gradients, BatchNorm partial statistics, bias sums; d 512, 8 heads of 32) with dropout 0.1,
    from the same parameters, optimizer state, BatchNorm buffers and dropout seed: identical loss statistics, flat
    gradients, updated parameters and BatchNorm running buffers."""
    import dataclasses
    import importlib
    import b200asr
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    prev = ops.weight_cache
    try:
        cfg = dataclasses.replace(b200asr.BASELINE_CONFIGS["cfg3"]["cfg"], num_layers=1, dropout=0.1)
        assert cfg.feat_extractor == "emb_cnn"
        torch.manual_seed(31)
        model = b200asr.build_model(cfg).cuda().train()
        B, T = 8, 300
        g = _gen(7)
        src = torch.randn(B, 1, cfg.freq, T, generator=g)
        lens = torch.randint(T // 2, T + 1, (B,), generator=g).sort(descending=True).values.to(torch.int32)
        lens[0] = T
        for i in range(B):
            src[i, :, :, int(lens[i]):] = 0
        tgt = torch.randint(3, cfg.vocab, (B, 30), generator=g)
        for i in range(B):
            tgt[i, 10 + 2 * i:] = 0
        src, tgt = src.cuda(), tgt.cuda()
        dp = b200asr.DataParallelStep(model, model_size=cfg.dim_model, warmup=100, smoothing=cfg.label_smoothing)
        p0 = dp.flat.flat.clone()
        bufs = {k: b for k, b in model.named_buffers() if "running" in k or "num_batches" in k}
        assert len(bufs) == 6
        b0 = {k: b.clone() for k, b in bufs.items()}

        def step():
            dp.flat.flat.copy_(p0)
            for k, b in bufs.items():
                b.copy_(b0[k])
            dp.adam.m.zero_(); dp.adam.v.zero_(); dp.adam.t = 0; dp.opt._step = 0
            ops.manual_seed(77)
            dp.step(src, lens, tgt)
            torch.cuda.synchronize()
            return (dp.flat.extras.clone(), dp.flat.flat_grad[:dp.flat.numel].clone(), dp.flat.flat.clone(),
                    torch.cat([b.double().view(-1) for b in bufs.values()]))

        first, second = step(), step()
        assert torch.isfinite(first[0]).all() and float(first[0][1]) > 0
        assert float(first[1].abs().max()) > 0 and not torch.equal(first[2], p0)
        assert not torch.equal(first[3], torch.cat([b.double().view(-1) for b in b0.values()]))
        for name, a, b in zip(("loss statistics", "gradients", "parameters", "BatchNorm buffers"), first, second):
            assert torch.equal(a, b), name
    finally:
        ops.weight_cache = prev


# ================================================================================================ 9. spectrogram statistics
@gpu
def test_spectrogram_batch_is_bit_reproducible(L):
    """b200asr_stft_features sums each utterance's normalisation statistics from per-tile partials in a fixed order: two
    calls on the same batch (utterances spanning many 32 x 32 tiles) return identical bits."""
    import b200asr
    gen = torch.Generator(device="cuda").manual_seed(2)
    waves = [0.1 * torch.randn(n, generator=gen, device="cuda") for n in (160000, 123457, 48000, 700)]
    a, _, _ = b200asr.spectrogram_batch(waves)
    b, _, _ = b200asr.spectrogram_batch(waves)
    assert torch.isfinite(a).all() and torch.equal(a.view(torch.int32), b.view(torch.int32))
