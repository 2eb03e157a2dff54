"""-m gpu tests of the edges the tile engine's schedule has (tc_engine.cuh: the k-loop builds k-block kb + 1's A fragments while
kb's MMAs run, in two fragment buffers, and releases each stage one k-block late; the producer and consumer warpgroups split
the registers with setmaxnreg), for the default bf16x3 instantiations, the linear layer's TF32 (NSPLIT 1) and 3xTF32
(NSPLIT 3) instantiations, whose fragments are built differently, and the halo convolution that shares the k-loop:

  * one and two k-blocks (the pipeline's prologue and drain), an odd number of k-blocks (the loop runs two per trip), and
    contractions that end in a partial k-block, in every direction of the linear layer (forward: K, data gradient: N, weight
    gradient: M);
  * M off the 64 / 128-row grid, and 1, 2, 131, 132, 133 and 265 output tiles (fewer CTAs than SMs, one round, a second
    round on one CTA, several rounds);
  * split-K weight gradients whose splits hold an odd number of k-blocks;
  * the halo kernel with T and F off the 16 x 8 tile, one, two, three and four 32-channel slices, with the fused pool and
    the ReLU mask;
  * the 3xTF32 batched GEMMs of the materialised attention (BGemmPolicy: K-major / K-major, K-major / MN-major and
    MN-major / MN-major operands, B converted in place by the consumers) with 1, 2, 3 and partial k-blocks, rows and columns
    off the tile, and 1, 2, 131, 132, 133 and 265 tiles;
  * the LSTM cell policy (one engine launch per time step);
  * schedule independence: the same rows computed in one launch and in two launches (other CTAs) are bit-identical.

Every output is NaN-poisoned first.  The bf16x3 bars are those of tests/test_gpu_default_precision.py (about 3x the error
measured on one H100 80GB HBM3 at a 700 W limit); the schedule changes no arithmetic, so the errors are the same.  The TF32
and 3xTF32 bars are about 3x the error measured here on the same card and limit (stated at BARS)."""
import math

import numpy as np
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

BF16X3 = 6
# TF32 / 3xTF32 measured over EDGE_SHAPES + TILE_SHAPES: forward 3.7e-4 / 1.0e-6 (K <= 96), data gradient 4.3e-4 / 3.5e-5
# (over N = 4364), weight gradient 3.7e-4 / 1.5e-5
BARS = {BF16X3: dict(fwd=3e-5, dgrad=6e-5, wgrad=4e-5), 1: dict(fwd=1.2e-3, dgrad=1.3e-3, wgrad=1.2e-3),
        3: dict(fwd=3e-6, dgrad=1e-4, wgrad=5e-5)}


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _split(L, w, prec=BF16X3):
    """The weight operands of the bf16x3 forward and data gradient; TF32 and 3xTF32 split inside the kernel."""
    if prec != BF16X3:
        return None, None
    N, K = w.shape
    fwd = torch.empty(2, N, K, device="cuda", dtype=torch.bfloat16)
    bwd = torch.empty(2, K, (N + 7) // 8 * 8, device="cuda", dtype=torch.bfloat16)
    L.check(L.load().b200asr_split_bf16(L.ptr(w), L.ptr(fwd), L.ptr(bwd), N, K, 2, _stream()), "split_bf16")
    return fwd, bwd


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


# (M, N, K): 1 / 2 / 3 k-blocks and partial k-blocks in each direction; M off the 64- and 128-row grids
EDGE_SHAPES = [(32, 32, 32), (64, 64, 64), (96, 96, 96), (100, 40, 72), (200, 136, 96), (130, 64, 32), (64, 4364, 64)]
# forward / data-gradient tile counts (M = 128 t, N = 128): t = 1, 2, 131, 132, 133, 265
TILE_SHAPES = [(128 * t, 128, 96) for t in (1, 2, 131, 132, 133, 265)]


def _with_precisions(rows):
    """Each row at bf16x3 (its id unchanged), then at TF32 and 3xTF32 (ids suffixed "tf32" / "tf32x3")."""
    return [pytest.param(*row, prec, id="-".join(map(str, row)) + suffix)
            for prec, suffix in ((BF16X3, ""), (1, "-tf32"), (3, "-tf32x3")) for row in rows]


@pytest.mark.parametrize("M,N,K,prec", _with_precisions(EDGE_SHAPES + TILE_SHAPES))
def test_linear_bf16x3_schedule_edges(L, M, N, K, prec):
    """b200asr_linear_fwd (bias), _bwd_data (ReLU mask) and _bwd_weight (bias gradient) at bf16x3, TF32 and 3xTF32 against
    float64."""
    lib = L.load()
    st = _stream()
    g = torch.Generator().manual_seed(M + 5 * N + 11 * K)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) * K ** -0.5
    b = torch.randn(N, generator=g)
    dy = torch.randn(M, N, generator=g)
    h = torch.randn(M, K, generator=g)
    x64, w64, dy64 = x.double(), w.double(), dy.double()
    xc, wc, bc, dyc, hc = x.cuda(), w.cuda(), b.cuda(), dy.cuda(), h.cuda()
    fwd, bwd = _split(L, wc, prec)
    bars = BARS[prec]
    y = _nan(M, N)
    L.check(lib.b200asr_linear_fwd(L.ptr(xc), L.ptr(wc), L.ptr(bc), L.ptr(y), M, N, K, 0, prec, L.ptr(fwd), st), "fwd")
    assert rel_err(y, x64 @ w64.t() + b.double()) < bars["fwd"]
    dx = _nan(M, K)
    L.check(lib.b200asr_linear_bwd_data(L.ptr(dyc), L.ptr(wc), L.ptr(hc), L.ptr(dx), M, N, K, 0, prec, L.ptr(bwd), st), "dgrad")
    assert rel_err(dx, (dy64 @ w64) * (h > 0)) < bars["dgrad"]
    dw, db = _nan(N, K), _nan(N)
    L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw), L.ptr(db), M, N, K, 0, prec, st), "wgrad")
    assert rel_err(dw, dy64.t() @ x64) < bars["wgrad"]
    assert rel_err(db, dy64.sum(0)) < 1e-6


# weight-gradient GEMM (rows N, columns K, contraction M): 1, 2, 131, 132, 133 and 265 tiles; then split-K shapes whose
# splits hold an odd number of k-blocks (2080 rows, 2 tiles: 8 splits of 9 k-blocks, the last of 2) and a partial one
WGRAD_SHAPES = [(64, 128, 128), (64, 256, 128), (64, 128, 131 * 128), (96, 11 * 128, 12 * 128), (96, 7 * 128, 19 * 128),
                (64, 5 * 128, 53 * 128), (2080, 128, 256), (3300, 64, 136)]


@pytest.mark.parametrize("M,N,K", WGRAD_SHAPES)
def test_linear_bf16x3_weight_gradient_tiles_and_splits(L, M, N, K):
    """b200asr_linear_bwd_weight at bf16x3 against float64, overwriting and accumulating; two calls give identical bits."""
    lib = L.load()
    st = _stream()
    g = torch.Generator().manual_seed(M + 7 * N + 3 * K)
    dy = torch.randn(M, N, generator=g)
    x = torch.randn(M, K, generator=g)
    dyc, xc = dy.cuda(), x.cuda()
    ref, bref = dy.double().t() @ x.double(), dy.double().sum(0)
    outs = []
    for _ in range(2):
        dw, db = _nan(N, K), _nan(N)
        L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw), L.ptr(db), M, N, K, 0, BF16X3, st), "wgrad")
        outs.append((dw, db))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert rel_err(outs[0][0], ref) < BARS[BF16X3]["wgrad"]
    assert rel_err(outs[0][1], bref) < 1e-6
    wbase, bbase = torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    dw, db = wbase.cuda(), bbase.cuda()
    L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw), L.ptr(db), M, N, K, 1, BF16X3, st), "wgrad acc")
    assert rel_err(dw, wbase.double() + ref) < BARS[BF16X3]["wgrad"]
    assert rel_err(db, bbase.double() + bref) < 1e-6


@pytest.mark.parametrize("M,split,prec", _with_precisions([(128 * 133, 128 * 67), (128 * 265 + 40, 128 * 132)]))
def test_linear_bf16x3_rows_independent_of_launch(L, M, split, prec):
    """The forward and the data gradient of rows [0, M) in one launch equal, bit for bit, the same rows computed as [0, split)
    and [split, M) in two launches: each tile runs on another CTA, so nothing may depend on which CTA or warpgroup took it."""
    lib = L.load()
    st = _stream()
    N, K = 512, 512
    g = torch.Generator().manual_seed(M)
    xc = torch.randn(M, K, generator=g).cuda()
    wc = (torch.randn(N, K, generator=g) * K ** -0.5).cuda()
    bc = torch.randn(N, generator=g).cuda()
    dyc = torch.randn(M, N, generator=g).cuda()
    fwd, bwd = _split(L, wc, prec)

    def run(rows):
        y, dx = _nan(M, N), _nan(M, K)
        for r0, r1 in rows:
            L.check(lib.b200asr_linear_fwd(L.ptr(xc[r0:r1]), L.ptr(wc), L.ptr(bc), L.ptr(y[r0:r1]), r1 - r0, N, K, 1, prec,
                                           L.ptr(fwd), st), "fwd")
            L.check(lib.b200asr_linear_bwd_data(L.ptr(dyc[r0:r1]), L.ptr(wc), None, L.ptr(dx[r0:r1]), r1 - r0, N, K, 0, prec,
                                                L.ptr(bwd), st), "dgrad")
        return y, dx

    y1, dx1 = run([(0, M)])
    y2, dx2 = run([(0, split), (split, M)])
    assert not y1.isnan().any() and not dx1.isnan().any()
    assert torch.equal(y1, y2) and torch.equal(dx1, dx2)


# T and F off the 16 x 8 tile; 1, 2, 3 and 4 input-channel slices (9, 18, 27 and 36 k-blocks)
HALO_SHAPES = [(1, 5, 3, 32, 64), (2, 19, 13, 64, 64), (1, 17, 9, 96, 128), (2, 33, 41, 128, 128), (1, 18, 170, 64, 128)]


@pytest.mark.parametrize("B,T,F_,Ci,Co", HALO_SHAPES)
def test_halo_conv_bf16x3_schedule_edges(L, B, T, F_, Ci, Co):
    """The halo kernel at bf16x3: forward with the fused 2 x 2 pool (pooled = b200asr_maxpool2x2_fwd of y, bit for bit) and the
    data gradient through a ReLU mask, against float64."""
    from tests.test_gpu_tensorcore import _conv_case
    lib = L.load()
    st = _stream()
    x, w, b, y_ref, dy, dx_ref = _conv_case(L, B, T, F_, Ci, Co, seed=T * F_ + Ci)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    y, pooled = _nan(B, T, F_, Co), _nan(B, T // 2, F_ // 2, Co)
    L.check(lib.b200asr_conv3x3_fwd_pool(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(pooled), None, L.ptr(ws), B, T, F_, Ci, Co,
                                         1, BF16X3, st), "conv+pool")
    assert rel_err(y, y_ref.relu()) < 2e-5
    if T >= 2 and F_ >= 2:
        p_ref = torch.full_like(pooled, float("nan"))
        L.check(lib.b200asr_maxpool2x2_fwd(L.ptr(y), L.ptr(p_ref), B, T, F_, Co, st), "pool")
        assert torch.equal(pooled, p_ref)
    if Ci in (64, 128):                     # the data gradient's output channels are the halo kernel's Cout
        mask = torch.randn(B, T, F_, Ci, device="cuda")
        dx = _nan(B, T, F_, Ci)
        L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(mask), L.ptr(dx), None, L.ptr(ws), B, T, F_, Ci, Co,
                                             BF16X3, st), "dgrad")
        assert rel_err(dx, dx_ref * (mask > 0).double().cpu()) < 2e-5


@pytest.mark.parametrize("nhid,nseq", [(64, 1), (200, 133), (512, 265)])
def test_lstm_cell_policy_matches_float64(nhid, nseq):
    """The LSTM recurrence (one LstmCellPolicy engine launch per step, the cell in the epilogue) against float64 nn.LSTM:
    ragged lengths, so the launches shrink from nseq rows down to one."""
    import importlib

    import b200asr
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    M = importlib.import_module(b200asr.__name__ + ".modules")
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(nhid + nseq)
    ntoken, ninp = 53, 48
    lens = rng.integers(1, 12, nseq)
    torch.manual_seed(nseq)
    model = M.RNNModel("LSTM", ntoken, ninp, nhid, 1, dropout=0.0, tie_weights=False)
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(2.0 / math.sqrt(nhid) * torch.randn(p.shape))
    model = model.to(dev)
    op = ops.lstm_lm_operands(model, dev)
    order = np.argsort(-lens, kind="stable")
    Mt = np.array([(lens > t).sum() for t in range(int(lens.max()))])
    off = np.concatenate([[0], np.cumsum(Mt)[:-1]])
    seqs = [rng.integers(0, ntoken, int(n)) for n in lens]
    inp = np.empty(int(Mt.sum()), dtype=np.int64)
    for j, s in enumerate(order):
        inp[off[:lens[s]] + j] = seqs[s]
    out = ops.lstm_lm_layers(op, torch.from_numpy(inp).to(dev), Mt)[-1].cpu()
    assert not out.isnan().any()
    ref = torch.nn.LSTM(ninp, nhid, 1).double()
    ref.load_state_dict({k[4:]: v.double().cpu() for k, v in model.state_dict().items() if k.startswith("rnn.")})
    emb = model.encoder.weight.detach().double().cpu()
    worst = 0.0
    with torch.no_grad():
        for j, s in enumerate(order):
            y, _ = ref(emb[torch.from_numpy(seqs[s])].unsqueeze(1))
            worst = max(worst, float((out[off[:lens[s]] + j, :nhid].double() - y[:, 0]).abs().max()))
    assert worst < 2e-5, worst


# (B, H, Tq, Tk, causal).  Contractions: QK^T over dk = 64 (2 k-blocks), dO V^T over dv = 32 (1), PV and dQ over Tk, dV and
# dK over Tq.  QK^T tiles = B * H * ceil(Tq / 128) * ceil(Tk / BN) with BN = 64 for Tk <= 64: 1, 2, 131, 132, 133, 265.
ATTN_SHAPES = [(1, 1, 32, 32, False), (1, 2, 64, 64, True), (1, 1, 96, 100, False), (2, 3, 130, 33, False),
               (1, 131, 40, 64, False), (1, 132, 33, 96, False), (1, 133, 100, 32, True), (1, 265, 32, 32, False),
               (2, 2, 300, 129, False)]


@pytest.mark.parametrize("B,H,Tq,Tk,causal", ATTN_SHAPES)
def test_attention_bgemm_3xtf32_schedule_edges(L, B, H, Tq, Tk, causal):
    """b200asr_sdpa_mat_fwd / _bwd at 3xTF32 (the default attention path: six BGemmPolicy products per layer) with every
    output and workspace NaN-poisoned: P, O, dQ, dK and dV against float64, with the bars of the materialised-attention test
    (P 1e-5, O and gradients 7e-5)."""
    from tests.test_gpu_row_kernels import attn_mask, attn_ref
    lib = L.load()
    st = _stream()
    dk_, dv_ = 64, 32
    g = torch.Generator().manual_seed(B * 1000 + H * 7 + Tq + Tk)
    q = torch.randn(B, Tq, H, dk_, generator=g)                 # token-major, as the projections write it
    k = torch.randn(B, H, Tk, dk_, generator=g)
    v = torch.randn(B, H, Tk, dv_, generator=g)
    dout = torch.randn(B, Tq, H, dv_, generator=g)
    qc, kc, vc, doc = q.cuda(), k.cuda(), v.cuda(), dout.cuda()
    qv, dov = qc.permute(0, 2, 1, 3), doc.permute(0, 2, 1, 3)
    bhtd = lambda t: (t.stride(0), t.stride(1), t.stride(2))
    n = lib.b200asr_sdpa_mat_ws_bytes(B, H, Tq, Tk) // 4
    ldp = (Tk + 3) // 4 * 4
    probs, dp = _nan(n), _nan(n)
    out = _nan(B, Tq, H, dv_)
    ov = out.permute(0, 2, 1, 3)
    scale = dk_ ** -0.5
    L.check(lib.b200asr_sdpa_mat_fwd(L.ptr(qc), L.ptr(kc), L.ptr(vc), *bhtd(qv), *bhtd(kc), *bhtd(vc), None, None, int(causal),
                                     L.ptr(out), *bhtd(ov), L.ptr(probs), None, B, H, Tq, Tk, dk_, dv_, scale, 0.0, 77, 5, 3, st),
            "sdpa_mat_fwd")
    dq, dk, dv = _nan(B, Tq, H, dk_), _nan(B, H, Tk, dk_), _nan(B, H, Tk, dv_)
    L.check(lib.b200asr_sdpa_mat_bwd(L.ptr(doc), L.ptr(qc), L.ptr(kc), L.ptr(vc), *bhtd(qv), *bhtd(kc), *bhtd(vc), *bhtd(dov),
                                     L.ptr(probs), None, L.ptr(dq), L.ptr(dk), L.ptr(dv), L.ptr(dp), B, H, Tq, Tk, dk_, dv_,
                                     scale, 0.0, 77, 5, 3, st), "sdpa_mat_bwd")
    q64 = q.permute(0, 2, 1, 3).double().cuda().requires_grad_(True)
    k64, v64 = k.double().cuda().requires_grad_(True), v.double().cuda().requires_grad_(True)
    o_ref, p_ref = attn_ref(q64, k64, v64, attn_mask(B, Tq, Tk, causal=causal).cuda(), scale)
    o_ref.backward(dout.permute(0, 2, 1, 3).double().cuda())
    P = probs.view(B, H, Tq, ldp)
    assert not P[..., Tk:].any()                                    # padding columns written as 0
    assert rel_err(P[..., :Tk], p_ref.detach()) < 1e-5
    for got, ref in ((ov, o_ref.detach()), (dq.permute(0, 2, 1, 3), q64.grad), (dk, k64.grad), (dv, v64.grad)):
        assert rel_err(got, ref) < 7e-5
