"""-m gpu tests of the tensor-core kernels against the exact-fp32 CUDA-core kernels and the CPU oracle.

precision 1 (TF32, one pass) is checked at TF32 tolerance; precision 3 (3xTF32 split) must meet fp32-grade error."""
import ctypes

import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


SHAPES = [(128, 128, 32), (128, 128, 128), (256, 384, 512), (300, 512, 512), (77, 52, 164), (6400 // 8, 512, 5120 // 4),
          (130, 4364, 128), (513, 128, 2048), (1, 8, 4), (200, 64, 96)]


@pytest.mark.parametrize("prec,tol", [(1, 2e-3), (3, 2e-5)])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_linear_forward_tensor_core(L, M, N, K, prec, tol):
    lib = L.load()
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).cuda()
    w = torch.randn(N, K, generator=g).cuda()
    b = torch.randn(N, generator=g).cuda()
    ref = (x.double() @ w.double().t() + b.double()).relu()
    y = torch.full((M, N), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), M, N, K, 1, prec, None, _stream()), "linear_fwd")
    torch.cuda.synchronize()
    assert rel_err(y, ref) < tol


@pytest.mark.parametrize("prec,tol", [(1, 2e-3), (3, 1e-4)])   # 3xTF32: operands exact to ~2^-22; the residual is the
@pytest.mark.parametrize("M,N,K", SHAPES)                      # tensor core's own fp32 accumulation over long K
def test_linear_backward_tensor_core(L, M, N, K, prec, tol):
    """bwd_data exercises an MN-major B operand, bwd_weight MN-major A and B (plus split-K atomics)."""
    lib = L.load()
    g = torch.Generator().manual_seed(M * 3 + N + K)
    x = torch.randn(M, K, generator=g).cuda()
    w = torch.randn(N, K, generator=g).cuda()
    dy = torch.randn(M, N, generator=g).cuda()
    h = torch.randn(M, K, generator=g).cuda()
    dx = torch.full((M, K), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(h), L.ptr(dx), M, N, K, 0, prec, None, _stream()), "bwd_data")
    ref_dx = (dy.double() @ w.double()) * (h > 0)
    assert rel_err(dx, ref_dx) < tol
    dw = torch.full((N, K), float("nan"), device="cuda")
    db = torch.full((N,), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw), L.ptr(db), M, N, K, 0, prec, _stream()), "bwd_weight")
    assert rel_err(dw, dy.double().t() @ x.double()) < tol
    assert rel_err(db, dy.double().sum(0)) < 1e-5
    # accumulate path
    base = torch.randn(N, K, generator=g).cuda()
    dw2 = base.clone()
    L.check(lib.b200asr_linear_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw2), None, M, N, K, 1, prec, _stream()), "bwd_weight acc")
    assert rel_err(dw2, base.double() + dy.double().t() @ x.double()) < tol


def test_unaligned_shapes_are_rejected_not_rerouted(L):
    lib = L.load()
    x = torch.randn(8, 161).cuda(); w = torch.randn(16, 161).cuda(); y = torch.empty(8, 16).cuda()
    rc = lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), None, L.ptr(y), 8, 16, 161, 0, 3, None, _stream())
    assert rc == -1 and "multiples of 4" in L.last_error()


# ------------------------------------------------------------------------------------------------ convolution
def _conv_case(L, B, T, F_, Ci, Co, seed=0):
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Ci, F_, T, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) * 0.1
    b = torch.randn(Co, generator=g)
    y = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    dy = torch.randn(B, Co, F_, T, generator=g)
    dx = torch.nn.grad.conv2d_input(x.shape, w.double(), dy.double(), padding=1)
    nhwc = lambda t: t.permute(0, 3, 2, 1).contiguous()
    return nhwc(x).cuda(), w.cuda(), b.cuda(), nhwc(y), nhwc(dy).cuda(), nhwc(dx)


@pytest.mark.parametrize("prec,tol", [(1, 2e-3), (3, 2e-5)])
@pytest.mark.parametrize("B,T,F_,Ci,Co", [(2, 16, 32, 64, 64), (1, 9, 21, 64, 128), (3, 24, 41, 128, 128), (2, 10, 23, 64, 64),
                                          (1, 40, 161, 64, 64)])
def test_conv3x3_forward_and_dgrad_tensor_core(L, B, T, F_, Ci, Co, prec, tol):
    lib = L.load()
    x, w, b, y_ref, dy, dx_ref = _conv_case(L, B, T, F_, Ci, Co, seed=B + T)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    y = torch.full((B, T, F_, Co), float("nan"), device="cuda")
    L.check(lib.b200asr_conv3x3_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F_, Ci, Co, 0, prec, _stream()), "conv fwd")
    assert rel_err(y, y_ref) < tol
    y2 = torch.empty_like(y)
    L.check(lib.b200asr_conv3x3_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y2), L.ptr(ws), B, T, F_, Ci, Co, 1, prec, _stream()), "conv fwd relu")
    assert rel_err(y2, y_ref.relu()) < tol
    dx = torch.full((B, T, F_, Ci), float("nan"), device="cuda")
    mask = torch.randn(B, T, F_, Ci, device="cuda")
    L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(mask), L.ptr(dx), None, L.ptr(ws), B, T, F_, Ci, Co, prec, _stream()), "conv dgrad")
    assert rel_err(dx, dx_ref.cuda() * (mask > 0)) < tol


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("B,H,Tq,Tk,dk,dv,mode", [
    (2, 2, 50, 50, 64, 64, "keypad"), (3, 4, 13, 13, 32, 32, "causal+keypad"), (2, 8, 100, 200, 64, 64, "keypad"),
    (2, 3, 70, 70, 64, 32, "dense"), (1, 2, 129, 65, 32, 64, "none"), (2, 2, 100, 100, 64, 64, "causal"),
    (1, 1, 200, 200, 64, 64, "keypad"), (1, 2, 300, 448, 64, 64, "keypad"), (2, 2, 257, 400, 64, 64, "none"),
])
@pytest.mark.parametrize("bwd", ["fp32", "tf32"])
def test_attention_tensor_core(L, B, H, Tq, Tk, dk, dv, mode, bwd):
    """TF32 tensor-core forward with either the fp32 CUDA-core backward or the TF32 backward (dK/dV kernel + dQ kernel)."""
    import importlib
    import b200asr
    from tests.test_gpu_parity import _attention_case
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    old = (ops.config.attn, ops.config.attn_bwd)
    ops.config.set(attn="tf32", attn_bwd=bwd)
    try:
        pairs = _attention_case(ops, B, H, Tq, Tk, dk, dv, mode)
    finally:
        ops.config.attn, ops.config.attn_bwd = old
    (got, ref) = pairs[0]
    assert rel_err(got, ref) < 2e-3
    for got, ref in pairs[1:]:
        assert rel_err(got, ref) < 3e-3


@pytest.mark.parametrize("B,H,Tq,Tk,dk,dv,mode", [
    (2, 2, 50, 50, 64, 64, "keypad"), (3, 4, 13, 13, 32, 32, "causal+keypad"), (2, 8, 100, 200, 64, 64, "keypad"),
    (2, 3, 70, 70, 64, 32, "dense"), (1, 2, 129, 65, 128, 128, "none"), (2, 2, 100, 100, 64, 64, "causal"),
    (1, 1, 200, 200, 64, 64, "keypad"), (1, 2, 300, 450, 64, 64, "keypad"), (2, 2, 257, 401, 32, 64, "none"),
    (1, 2, 40, 1030, 64, 64, "keypad"),
])
def test_attention_materialised_3xtf32(L, B, H, Tq, Tk, dk, dv, mode):
    """bmm -> masked softmax -> bmm on batched 3xTF32 GEMMs (attention_mat.cu): fp32-grade against the fp64-free oracle
    at the same tolerance as the exact-fp32 CUDA-core kernel (ragged Tk incl. Tk % 4 != 0 -> padded row pitch)."""
    import importlib
    import b200asr
    from tests.test_gpu_parity import _attention_case
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    old = ops.config.attn
    ops.config.set(attn="tf32x3")
    try:
        pairs = _attention_case(ops, B, H, Tq, Tk, dk, dv, mode)
    finally:
        ops.config.attn = old
    for got, ref in pairs:
        assert rel_err(got, ref) < 2e-5


@pytest.mark.parametrize("B,H,Tq,Tk,mode", [
    (2, 2, 50, 50, "keypad"), (3, 4, 13, 13, "causal+keypad"), (2, 8, 100, 200, "keypad"), (2, 3, 70, 70, "dense"),
    (2, 2, 100, 100, "causal"), (1, 1, 200, 200, "keypad"), (1, 2, 300, 448, "keypad"), (2, 2, 257, 400, "none"), (1, 2, 129, 65, "none"),
])
def test_attention_fused_bf16x3(L, B, H, Tq, Tk, mode):
    """The fused bf16x3 attention (tc_flash.cu: one forward kernel, two backward kernels, scores / probabilities
    only ever in registers): fp32-grade against the oracle -- 3e-5 (the 2-term bf16 split carries 16 significant bits)."""
    import importlib
    import b200asr
    from tests.test_gpu_parity import _attention_case
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    old = ops.config.attn
    ops.config.set(attn="bf16x3")
    try:
        pairs = _attention_case(ops, B, H, Tq, Tk, 64, 64, mode)
    finally:
        ops.config.attn = old
    for got, ref in pairs:
        assert rel_err(got, ref) < 3e-5


def test_attention_fused_bf16x3_dropout_matches_cuda_core_kernel(L):
    """Same counter-based dropout stream as the other attention paths (forward and both recomputing backward kernels)."""
    import importlib
    import b200asr
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    B, H, d, Tq, Tk = 2, 3, 64, 70, 132
    g = torch.Generator().manual_seed(9)
    base = [torch.randn(B, H, t, d, generator=g).cuda() for t in (Tq, Tk, Tk)]
    do = torch.randn(B, H, Tq, d, generator=g).cuda()
    key_pad = (torch.arange(Tk)[None, :] >= torch.tensor([Tk, Tk - 7])[:, None]).to(torch.uint8).cuda()
    outs = {}
    old = ops.config.attn
    try:
        for mode in ("fp32", "bf16x3"):
            ops.config.set(attn=mode)
            ops.rng.seed, ops.rng.offset = 77, 5
            q, k, v = (t.clone().requires_grad_(True) for t in base)
            o = ops.SdpaFn.apply(q, k, v, key_pad, None, False, 0.125, 0.3)
            o.backward(do)
            outs[mode] = (o.detach(), q.grad, k.grad, v.grad)
    finally:
        ops.config.attn = old
    for a, b in zip(outs["bf16x3"], outs["fp32"]):
        assert rel_err(a, b) < 3e-5


@pytest.mark.parametrize("Tq,Tk,causal", [(40, 40, True), (33, 70, False), (64, 101, False)])
def test_attention_materialised_dropout_matches_cuda_core_kernel(L, Tq, Tk, causal):
    """Both attention paths index the same counter-based dropout stream: with the same (seed, offset) the materialised
    3xTF32 path and the fp32 flash kernel drop the same probabilities, so outputs and all three gradients agree."""
    import importlib
    import b200asr
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    B, H, d = 2, 3, 64
    g = torch.Generator().manual_seed(Tq + Tk)
    base = [torch.randn(B, H, t, d, generator=g).cuda() for t in (Tq, Tk, Tk)]
    do = torch.randn(B, H, Tq, d, generator=g).cuda()
    key_pad = (torch.arange(Tk)[None, :] >= torch.tensor([Tk, Tk - 5])[:, None]).to(torch.uint8).cuda()
    outs = {}
    old = ops.config.attn
    try:
        for mode in ("fp32", "tf32x3"):
            ops.config.set(attn=mode)
            ops.rng.seed, ops.rng.offset = 77, 5
            q, k, v = (t.clone().requires_grad_(True) for t in base)
            o = ops.SdpaFn.apply(q, k, v, key_pad, None, causal, 0.125, 0.3)
            o.backward(do)
            outs[mode] = (o.detach(), q.grad, k.grad, v.grad)
    finally:
        ops.config.attn = old
    assert float((outs["fp32"][0] == 0).float().mean()) < 0.05        # only the first causal rows can lose every key
    for a, b in zip(outs["tf32x3"], outs["fp32"]):
        assert rel_err(a, b) < 2e-5


def test_attention_materialised_fully_masked_row_is_nan(L):
    import importlib
    import b200asr
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    q = torch.randn(1, 1, 4, 32).cuda(); k = torch.randn(1, 1, 6, 32).cuda(); v = torch.randn(1, 1, 6, 32).cuda()
    old = ops.config.attn
    ops.config.set(attn="tf32x3")
    try:
        o = ops.SdpaFn.apply(q, k, v, torch.ones(1, 6, dtype=torch.uint8).cuda(), None, False, 0.25, 0.0)
    finally:
        ops.config.attn = old
    assert torch.isnan(o).all()


def test_attention_tensor_core_rejects_long_keys(L):
    lib = L.load()
    q = torch.randn(1, 1, 64, 64, device="cuda"); k = torch.randn(1, 1, 500, 64, device="cuda"); v = torch.randn(1, 1, 500, 64, device="cuda")
    o = torch.empty(1, 1, 64, 64, device="cuda"); lse = torch.empty(1, 1, 64, device="cuda")
    rc = lib.b200asr_sdpa_fwd(L.ptr(q), L.ptr(k), L.ptr(v), 4096, 4096, 64, 32000, 32000, 64, 32000, 32000, 64, None, None, 0,
                              L.ptr(o), 4096, 4096, 64, L.ptr(lse), 1, 1, 64, 500, 64, 64, 0.125, 0.0, 0, 0, 1, _stream())
    assert rc == -1 and "precision 0" in L.last_error()


@pytest.mark.parametrize("prec,tol", [(1, 2e-3), (3, 1e-4)])
@pytest.mark.parametrize("B,T,F_,Ci,Co", [(2, 16, 32, 64, 64), (1, 9, 21, 64, 128), (3, 24, 41, 128, 128), (2, 10, 23, 128, 64),
                                          (1, 40, 161, 64, 64)])
def test_conv3x3_weight_gradient_tensor_core(L, B, T, F_, Ci, Co, prec, tol):
    lib = L.load()
    g = torch.Generator().manual_seed(B * 7 + T)
    x = torch.randn(B, Ci, F_, T, generator=g)
    dy = torch.randn(B, Co, F_, T, generator=g)
    dw_ref = torch.nn.grad.conv2d_weight(x.double(), (Co, Ci, 3, 3), dy.double(), padding=1)
    nhwc = lambda t: t.permute(0, 3, 2, 1).contiguous().cuda()
    xc, dyc = nhwc(x), nhwc(dy)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    dw = torch.full((Co, Ci, 3, 3), float("nan"), device="cuda")
    db = torch.full((Co,), float("nan"), device="cuda")
    L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(dyc), None, L.ptr(xc), L.ptr(dw), L.ptr(db), L.ptr(ws), B, T, F_, Ci, Co, prec, _stream()), "conv wgrad")
    assert rel_err(dw, dw_ref) < tol
    assert rel_err(db, dy.double().sum((0, 2, 3))) < 1e-5


@pytest.mark.parametrize("prec,tol", [(6, 1e-4), (2, 1e-2)])
@pytest.mark.parametrize("B,T,F_,Ci,Co", [(2, 16, 32, 64, 64), (1, 9, 21, 64, 128), (3, 24, 41, 128, 128), (2, 10, 23, 128, 64), (1, 40, 161, 64, 64)])
def test_conv3x3_weight_gradient_bf16_modes_and_pairs(L, B, T, F_, Ci, Co, prec, tol):
    """bf16 weight gradient: (a) dy converted inside the kernel, (b) dy arriving as the bf16 hi | lo pairs its producers
    write (max-pool backward with the ReLU mask, incl. the odd-F tail) -- B tiles by TMA, bias gradient from the bf16 tiles."""
    lib = L.load()
    g = torch.Generator().manual_seed(B * 11 + T)
    x = torch.randn(B, Ci, F_, T, generator=g)
    nhwc = lambda t: t.permute(0, 3, 2, 1).contiguous().cuda()
    # dy = max-pool backward of a random upstream gradient through a random post-ReLU activation (as in the VGG front end)
    act = torch.randn(B, Co, F_, T, generator=g).relu()
    up = torch.randn(B, Co, F_ // 2, T // 2, generator=g)
    a64 = act.double().requires_grad_(True)
    torch.nn.functional.max_pool2d(a64, 2, 2).backward(up.double())
    dy = (a64.grad * (act.double() > 0)).float()
    dyc = torch.full((B, T, F_, Co), float("nan"), device="cuda")
    dy16 = torch.full((2, B, T, F_, Co), float("nan"), device="cuda", dtype=torch.bfloat16)
    upc, actc = nhwc(up), nhwc(act)                      # keep the device tensors alive across the call
    L.check(lib.b200asr_maxpool2x2_bwd(L.ptr(upc), L.ptr(actc), L.ptr(dyc), L.ptr(dy16), B, T, F_, Co, 1, _stream()), "pool bwd")
    assert rel_err(dyc, nhwc(dy)) < 1e-6
    assert rel_err(dy16[0].float() + dy16[1].float(), nhwc(dy)) < 2e-5          # hi + lo carries 16 significant bits
    dw_ref = torch.nn.grad.conv2d_weight(x.double(), (Co, Ci, 3, 3), dy.double(), padding=1)
    xc = nhwc(x)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    for pairs in (None, dy16):
        dw = torch.full((Co, Ci, 3, 3), float("nan"), device="cuda")
        db = torch.full((Co,), float("nan"), device="cuda")
        L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(dyc), L.ptr(pairs), L.ptr(xc), L.ptr(dw), L.ptr(db), L.ptr(ws), B, T, F_, Ci, Co, prec,
                                               _stream()), "conv wgrad")
        assert rel_err(dw, dw_ref) < tol, ("dw", pairs is not None)
        # from the pairs the bias gradient is the column sum of the bf16 tiles: hi + lo (16 bits) at bf16x3, hi alone at bf16
        db_tol = 1e-5 if pairs is None else (2e-5 if prec == 6 else 1e-2)
        assert rel_err(db, dy.double().sum((0, 2, 3))) < db_tol, ("db", pairs is not None)


@pytest.mark.parametrize("M,N,K", [(300, 512, 512), (130, 4364, 128), (77, 52, 164), (800, 512, 1280)])
def test_linear_with_presplit_weights(L, M, N, K):
    """3xTF32 GEMM with the weight pre-split once by b200asr_split_tf32 (forward K-major B, data-gradient MN-major B)."""
    lib = L.load()
    g = torch.Generator().manual_seed(5 * M + N)
    x = torch.randn(M, K, generator=g).cuda(); w = torch.randn(N, K, generator=g).cuda(); b = torch.randn(N, generator=g).cuda()
    dy = torch.randn(M, N, generator=g).cuda()
    ws = torch.empty(2, N, K, device="cuda")
    L.check(lib.b200asr_split_tf32(L.ptr(w), L.ptr(ws), N * K, _stream()), "split")
    assert torch.equal(ws[0] + ws[1], w) and float((ws[1].abs() / w.abs().clamp_min(1e-30)).max()) < 2.0 ** -11
    y = torch.full((M, N), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), M, N, K, 0, 3, L.ptr(ws), _stream()), "fwd")
    assert rel_err(y, x.double() @ w.double().t() + b.double()) < 2e-5
    dx = torch.full((M, K), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_bwd_data(L.ptr(dy), L.ptr(w), None, L.ptr(dx), M, N, K, 0, 3, L.ptr(ws), _stream()), "dgrad")
    assert rel_err(dx, dy.double() @ w.double()) < 1e-4


# ------------------------------------------------------------------------------------------------ emb_cnn implicit GEMM
@pytest.mark.parametrize("B,H,W,KH,KW,SH", [(2, 61, 45, 21, 11, 2), (1, 30, 205, 21, 11, 2), (3, 25, 140, 5, 3, 1), (2, 23, 131, 21, 11, 2)])
@pytest.mark.parametrize("prec,tol", [(3, 1e-4), (6, 3e-5), (2, 1e-2)])
def test_conv2d_implicit_gemm_32ch(L, B, H, W, KH, KW, SH, prec, tol):
    """tc_emb.cu through the raw C ABI: forward, data gradient and weight gradient of Conv2d(32, 32, (KH, KW), stride (SH, 1))
    on row-pitched NCHW tensors against float64 (W and OW deliberately not multiples of 4 / 32 / 128)."""
    import torch.nn.functional as F
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator().manual_seed(B * 1000 + W)
    OH, OW = (H - KH) // SH + 1, W - KW + 1
    xp, yp = (W + 3) // 4 * 4, (OW + 3) // 4 * 4
    x = torch.randn(B, 32, H, W, generator=g).cuda()
    w = (torch.randn(32, 32, KH, KW, generator=g) * (32 * KH * KW) ** -0.5).cuda()
    b = torch.randn(32, generator=g).cuda()
    dy = torch.randn(B, 32, OH, OW, generator=g).cuda()
    x64 = x.double().requires_grad_(True)
    w64 = w.double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, b.double(), stride=(SH, 1))
    y64.backward(dy.double())
    # pitched copies, pad columns poisoned with NaN: nothing may read them
    xpad = torch.full((B, 32, H, xp), float("nan"), device="cuda"); xpad[..., :W] = x
    dypad = torch.full((B, 32, OH, yp), float("nan"), device="cuda"); dypad[..., :OW] = dy
    ypad = torch.full((B, 32, OH, yp), float("nan"), device="cuda")
    dxpad = torch.full((B, 32, H, xp), float("nan"), device="cuda")
    ws = torch.empty(lib.b200asr_conv2d_tc_ws_bytes(B, H, W, KH, KW) // 4, device="cuda")
    L.check(lib.b200asr_conv2d_tc_fwd(L.ptr(xpad), L.ptr(w), L.ptr(b), L.ptr(ypad), L.ptr(ws), B, 32, H, W, 32, KH, KW, SH, xp, yp, prec, st), "fwd")
    assert rel_err(ypad[..., :OW], y64) < tol
    L.check(lib.b200asr_conv2d_tc_bwd_data(L.ptr(dypad), L.ptr(w), L.ptr(dxpad), L.ptr(ws), B, 32, H, W, 32, KH, KW, SH, xp, yp, prec, st), "dgrad")
    assert rel_err(dxpad[..., :W], x64.grad) < tol
    if prec == 3:
        dw = torch.empty_like(w)
        db = torch.empty(32, device="cuda")
        L.check(lib.b200asr_conv2d_tc_bwd_weight(L.ptr(dypad), L.ptr(xpad), L.ptr(dw), L.ptr(db), L.ptr(ws), B, 32, H, W, 32, KH, KW, SH, xp, yp, st), "wgrad")
        assert rel_err(dw, w64.grad) < tol
        assert rel_err(db, dy.double().sum((0, 2, 3))) < 1e-5


@pytest.mark.parametrize("B,H,W", [(2, 161, 400), (1, 75, 133), (3, 41, 50)])
@pytest.mark.parametrize("prec,tol", [(3, 3e-5), (6, 3e-5), (2, 1e-2)])
def test_conv2d_first_layer_implicit_gemm(L, B, H, W, prec, tol):
    """tc_emb.cu, Conv2d(1, 32, (41, 11), stride (2, 2), padding (0, 10)) through the raw C ABI: forward and weight gradient
    against float64 -- the taps along H as the contraction "channels" of an overlapping tensor-map view, the stride along W
    through de-interleaved copies (odd and even W, tiles with out-of-range columns on both sides)."""
    import torch.nn.functional as F
    lib = L.load()
    g = torch.Generator().manual_seed(7 * B + W)
    KH, KW, PW = 41, 11, 10
    OH, OW = (H - KH) // 2 + 1, (W + 2 * PW - KW) // 2 + 1
    yp = (OW + 3) // 4 * 4
    x = torch.randn(B, 1, H, W, generator=g).cuda()
    w = (torch.randn(32, 1, KH, KW, generator=g) * (KH * KW) ** -0.5).cuda()
    b = torch.randn(32, generator=g).cuda()
    dy = torch.randn(B, 32, OH, OW, generator=g).cuda()
    x64, w64 = x.double(), w.double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, b.double(), stride=(2, 2), padding=(0, PW))
    y64.backward(dy.double())
    st = _stream()
    ws = torch.empty(lib.b200asr_conv2d_c1_tc_ws_bytes(B, H, W, KH, KW) // 4, device="cuda")
    y = torch.full((B, 32, OH, yp), float("nan"), device="cuda")
    L.check(lib.b200asr_conv2d_c1_tc_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, H, W, 32, KH, KW, PW, yp, prec, st), "fwd")
    assert rel_err(y[..., :OW], y64.detach()) < tol
    if prec == 3:
        dypad = torch.zeros(B, 32, OH, yp, device="cuda"); dypad[..., :OW] = dy
        dw = torch.full_like(w, float("nan")); db = torch.full((32,), float("nan"), device="cuda")
        L.check(lib.b200asr_conv2d_c1_tc_bwd_weight(L.ptr(dypad), L.ptr(x), L.ptr(dw), L.ptr(db), L.ptr(ws), B, H, W, 32, KH, KW, PW, yp, st), "wgrad")
        assert rel_err(dw, w64.grad) < 3e-5
        assert rel_err(db, dy.double().sum((0, 2, 3))) < 1e-5


@pytest.mark.parametrize("prec", [6, 2, 3, 0])
@pytest.mark.parametrize("B,T,F_,Ci,Co", [(2, 32, 16, 64, 64), (1, 37, 21, 64, 128), (2, 18, 161, 128, 128)])
def test_conv3x3_with_fused_max_pool(L, B, T, F_, Ci, Co, prec):
    """b200asr_conv3x3_fwd_pool == b200asr_conv3x3_fwd followed by b200asr_maxpool2x2_fwd, bit for bit (the bf16 modes take
    the 2x2 maximum in the convolution's epilogue; odd T / F exercise the floor-mode edges and partial tiles)."""
    lib = L.load()
    g = torch.Generator().manual_seed(B + T)
    x = torch.randn(B, T, F_, Ci, generator=g).cuda()
    w = (torch.randn(Co, Ci, 3, 3, generator=g) * (9 * Ci) ** -0.5).cuda()
    b = torch.randn(Co, generator=g).cuda()
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    st = _stream()
    y0 = torch.full((B, T, F_, Co), float("nan"), device="cuda")
    p0 = torch.full((B, T // 2, F_ // 2, Co), float("nan"), device="cuda")
    L.check(lib.b200asr_conv3x3_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y0), L.ptr(ws), B, T, F_, Ci, Co, 1, prec, st), "conv")
    L.check(lib.b200asr_maxpool2x2_fwd(L.ptr(y0), L.ptr(p0), B, T, F_, Co, st), "pool")
    y1, p1 = torch.full_like(y0, float("nan")), torch.full_like(p0, float("nan"))
    i1 = torch.full(p0.shape, 255, device="cuda", dtype=torch.uint8)
    L.check(lib.b200asr_conv3x3_fwd_pool(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y1), L.ptr(p1), L.ptr(i1), L.ptr(ws), B, T, F_, Ci, Co, 1, prec, st), "conv+pool")
    assert torch.equal(y0, y1) and torch.equal(p0, p1)
    # the index bytes: the stand-alone pooling kernel writes the same ones, and the backward that reads them routes every
    # gradient exactly as the backward that re-reads the activation (post-ReLU zeros make exact ties: first maximum wins)
    i0 = torch.full_like(i1, 255)
    p0b = torch.full_like(p0, float("nan"))
    L.check(lib.b200asr_maxpool2x2_fwd_idx(L.ptr(y0), L.ptr(p0b), L.ptr(i0), B, T, F_, Co, st), "pool idx")
    assert torch.equal(p0b, p0) and torch.equal(i0, i1) and int(i1.max()) <= 7
    g = torch.randn(p0.shape, device="cuda")
    dx0, dx1 = torch.full_like(y0, float("nan")), torch.full_like(y0, float("nan"))
    pr0 = torch.full((2,) + tuple(y0.shape), float("nan"), device="cuda", dtype=torch.bfloat16)
    pr1 = torch.full_like(pr0, float("nan"))
    L.check(lib.b200asr_maxpool2x2_bwd(L.ptr(g), L.ptr(y0), L.ptr(dx0), L.ptr(pr0), B, T, F_, Co, 1, st), "pool bwd")
    L.check(lib.b200asr_maxpool2x2_bwd_idx(L.ptr(g), L.ptr(i1), L.ptr(dx1), L.ptr(pr1), B, T, F_, Co, 1, st), "pool bwd idx")
    assert torch.equal(dx0, dx1) and torch.equal(pr0.view(torch.int16), pr1.view(torch.int16))
