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


# short time axes (T = 17 is one past a 16-row halo tile) and the cfg2 layer shapes (F = 161: 64 -> 64; F = 80: 64 -> 128, 128 -> 128)
CONV_EDGE_SHAPES = [(2, 1, 41, 64, 64), (2, 2, 23, 64, 128), (1, 3, 80, 128, 128), (2, 17, 21, 64, 64), (2, 33, 161, 64, 64),
                    (2, 25, 80, 64, 128), (2, 25, 80, 128, 128)]


@pytest.mark.parametrize("prec,tol", [(1, 2e-3), (3, 2e-5), (6, 2e-5), (2, 1e-2)])
@pytest.mark.parametrize("B,T,F_,Ci,Co", [(2, 16, 32, 64, 64), (1, 9, 21, 64, 128), (3, 24, 41, 128, 128), (2, 10, 23, 64, 64),
                                          (1, 40, 161, 64, 64)] + CONV_EDGE_SHAPES)
def test_conv3x3_forward_and_dgrad_tensor_core(L, B, T, F_, Ci, Co, prec, tol):
    """Forward (with and without ReLU) and data gradient (through a ReLU mask) against float64.  In the bf16 modes (the halo
    kernel: bf16x3 is the default, bf16 is cfg5's) the data gradient also writes the bf16 pairs the layer below's weight
    gradient reads: they must be the round-to-nearest-even split of the returned dx, bit for bit.  Measured on one H100 80GB
    HBM3: bf16x3 <= 6.7e-6 (bar 2e-5), bf16 <= 2.7e-3 (bar 1e-2)."""
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
    dx16 = torch.full((2, B, T, F_, Ci), float("nan"), device="cuda", dtype=torch.bfloat16) if prec in (2, 6) else None
    L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(mask), L.ptr(dx), L.ptr(dx16), L.ptr(ws), B, T, F_, Ci, Co, prec,
                                         _stream()), "conv dgrad")
    assert rel_err(dx, dx_ref.cuda() * (mask > 0)) < tol
    if dx16 is not None:
        hi = dx.to(torch.bfloat16)
        lo = (dx - hi.float()).to(torch.bfloat16)
        assert torch.equal(dx16[0].view(torch.int16), hi.view(torch.int16))
        assert torch.equal(dx16[1].view(torch.int16), lo.view(torch.int16))


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
                                          (1, 40, 161, 64, 64)] + CONV_EDGE_SHAPES)
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


@pytest.mark.parametrize("prec", [6, 2, 3, 0])
@pytest.mark.parametrize("B,T,F_,Ci,Co", [(2, 32, 16, 64, 64), (1, 37, 21, 64, 128), (2, 18, 161, 128, 128)])
def test_conv3x3_with_fused_max_pool(L, B, T, F_, Ci, Co, prec):
    """b200asr_conv3x3_fwd_pool with the pooling index bytes == b200asr_conv3x3_fwd followed by b200asr_maxpool2x2_fwd, bit
    for bit, in every precision: asking for the index bytes routes the call to the convolution followed by the stand-alone
    pooling kernel (odd T / F exercise the floor-mode edges).  The bf16 modes' epilogue pooling, taken when no index bytes are
    asked for, is tested by test_gpu_default_precision.py::test_conv3x3_pool_in_epilogue."""
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
