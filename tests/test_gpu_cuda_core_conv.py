"""The CUDA-core convolution and pooling kernels (conv_simt.cu, the direct convolutions of emb_frontend.cu) and the layout
permutations of the front ends, through the raw C ABI, against float64 references, at every instantiation and at the
edges where these kernels go wrong:

  1. the first VGG convolution (C_in = 1), conv3x3_c1_fwd / _bwd_weight -- it runs on CUDA cores in every precision:
     every accepted Co (every channel-quad / pixel-slot split), ReLU and bias on and off, the edges of the 32 (time) x 8
     (freq) tile with tiles crossing utterances, the weight gradient's grid-stride loop on both sides of 4 x SM-count
     tiles and at the cfg2 layer, the empty problem, identical bits from two weight-gradient calls, rejections;
  2. max pooling, maxpool2x2_fwd / _fwd_idx / _bwd / _bwd_idx, bit-exact against ATen's max_pool2d and its autograd in
     float64 on inputs dense with exact ties (post-ReLU zeros, small integers, all-zero and all-negative windows): the
     first maximum in ATen's scan order, the index bytes, relu_mask 0 and 1, the odd-T / odd-F tail and T or F = 1,
     the bf16 hi | lo pairs against a host restatement of pair_of, the cfg2 pool-1 shape;
  3. the precision-0 3x3 convolution (the exact-fp32 cross-check): the implicit GEMM forward and data gradient at both
     column-tile widths with one and several column tiles, 1 and 3 channel chunks per tap, pixel counts off the 128-pixel
     tile, T or F in {1, 2}, the ReLU mask's exact zeros; the weight gradient at all four <BMC, BNC> instantiations, one
     chunk, a short last chunk, the cfg2 layer, and past 2^20 pixels (the bias column sum's long-slice branch);
  4. the emb_cnn direct convolutions conv2d_fwd / _bwd_data / _bwd_weight (+ bias gradient) at the reference's two
     geometries and at generic ones (KW = 16, stride larger than the kernel, padding larger than the kernel, OH = 1,
     OW > 128), their rejections, and flatten_bcft / permute_cols_cf bit-exact against the torch permutations;
  5. misaligned pointers (a view offset by 4 bytes, or by 1 byte for the index bytes) are rejected with BAD_ALIGN and
     nothing is written.

Outputs and the workspaces the caller owns are filled with NaN before each call, so an element a kernel fails to write
shows up.  Inputs are finite.  Bars are max-norm relative errors (tests.helpers.rel_err); each states the error measured
on one H100 80GB HBM3 (700 W limit) and sits about 3x above it.  Small references run in float64 on the CPU, those with
B*T*F of 1e5 pixels and more in float64 on the GPU (a reference, not the path under test)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

NAN = float("nan")
OK, BAD_SHAPE, BAD_ALIGN, BAD_ARG = 0, -1, -2, -5
PREC_FP32 = 0


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


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _off(n):
    """n NaN floats starting 4 bytes into a fresh allocation: a view no float4 access may use."""
    return torch.full((n + 4,), NAN, device="cuda")[1:n + 1]


def _all_nan(t):
    return bool(torch.isnan(t).all())


def _nchw(t):
    """channels-last [B, T, F, C] -> torch's (B, C, F, T)"""
    return t.permute(0, 3, 2, 1)


# ================================================================================================ float64 references
def c1_ref(x, w, b, relu):
    """x [B, F, T] -> [B, T, F, Co]: F.conv2d on the (B, 1, F, T) input, padding 1 (+ ReLU)."""
    y = F.conv2d(x.double()[:, None], w.double(), None if b is None else b.double(), padding=1)
    return _nchw(y.relu() if relu else y)


def conv3x3_ref(x, w, b, relu):
    """x [B, T, F, Ci] -> [B, T, F, Co]"""
    y = F.conv2d(_nchw(x.double()), w.double(), None if b is None else b.double(), padding=1)
    return _nchw(y.relu() if relu else y)


def conv3x3_dgrad_ref(dy, w, mask):
    """dy [B, T, F, Co] -> dx [B, T, F, Ci] .* (mask > 0)"""
    B, T, F_, _ = dy.shape
    dx = _nchw(torch.nn.grad.conv2d_input((B, w.shape[1], F_, T), w.double(), _nchw(dy.double()), padding=1))
    return dx if mask is None else dx * (mask.double() > 0)


def conv3x3_wgrad_ref(x_nchw, dy, Ci):
    """x (B, Ci, F, T), dy [B, T, F, Co] -> dw [Co, Ci, 3, 3], dbias [Co]"""
    Co = dy.shape[3]
    dw = torch.nn.grad.conv2d_weight(x_nchw.double(), (Co, Ci, 3, 3), _nchw(dy.double()), padding=1)
    return dw, dy.double().sum((0, 1, 2))


def pool_ref(x):
    """ATen's max_pool2d on the (B, C, F, T) view of x [B, T, F, C], in float64 on the CPU.  Returns the graph's input and
    output (for the backward) and, channels-last, the pooled values and the index bytes: 2 * df + dt of ATen's argmax
    (its first maximum in freq-major scan order), | 4 when the maximum is not positive.  None when no window exists."""
    B, T, F_, C = x.shape
    if T // 2 == 0 or F_ // 2 == 0:
        return None
    xn = _nchw(x.double().cpu()).contiguous().requires_grad_(True)
    y, i = F.max_pool2d(xn, 2, return_indices=True)
    df = i // T - 2 * torch.arange(F_ // 2)[:, None]
    dt = i % T - 2 * torch.arange(T // 2)[None, :]
    assert bool(((df >= 0) & (df <= 1) & (dt >= 0) & (dt <= 1)).all())
    code = (2 * df + dt + 4 * (y <= 0)).to(torch.uint8)
    return xn, y, _nchw(y.detach()), _nchw(code)


def pool_bwd_ref(ref, dy, shape, relu_mask):
    """max_pool2d's autograd in float64: dy routed to the argmax; relu_mask: a window whose maximum is not positive passes
    nothing (a ReLU in front of the pooling).  Rows and columns no window covers get 0."""
    if ref is None:
        return torch.zeros(shape, dtype=torch.float64)
    xn, y, _, _ = ref
    g = _nchw(dy.double().cpu())
    if relu_mask:
        g = g * (y.detach() > 0)
    dx, = torch.autograd.grad(y, xn, g, retain_graph=True)
    return _nchw(dx) + 0.0                   # + 0.0: a -0.0 (negative dy times a zero mask) is stored as +0.0


def pairs_ref(v):
    """conv_simt.cu pair_of on the host: hi = the top half of bits(x) + 0x8000, lo the same of x - hi (in float32).
    Returns int16 [2, *v.shape] -- the layout of the dx16 output."""
    a = v.float().contiguous().cpu().numpy()
    r = a.view(np.uint32) + np.uint32(0x8000)
    hi = (r >> np.uint32(16)).astype(np.uint16)
    lo = a - (r & np.uint32(0xFFFF0000)).view(np.float32)
    lb = (lo.view(np.uint32) + np.uint32(0x8000)) >> np.uint32(16)
    return torch.from_numpy(np.stack([hi, lb.astype(np.uint16)]).view(np.int16))


# ================================================================================================ 1. first VGG convolution
C1_CO = [4, 8, 16, 32, 64, 128, 256, 512, 1024]      # every Co with Co % 4 == 0, 256 % (Co / 4) == 0, Co <= 1024
# measured maxima: forward 2.0e-7 (nine products and a bias); weight gradient 7.4e-7, bias gradient 7.3e-7 (both at Co = 4)
C1_FWD_BAR = 6e-7
C1_WGRAD_BAR = 2.5e-6


def _c1_fwd(L, x, w, b, y, B, F_, T, Co, relu):
    return L.load().b200asr_conv3x3_c1_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), B, F_, T, Co, relu, _stream())


def _c1_wgrad(L, x, dy, dw, db, B, F_, T, Co):
    return L.load().b200asr_conv3x3_c1_bwd_weight(L.ptr(x), L.ptr(dy), L.ptr(dw), L.ptr(db), B, F_, T, Co, _stream())


def _c1_case(B, F_, T, Co, seed, device="cpu"):
    g = _gen(seed)
    x = torch.randn(B, F_, T, generator=g)
    w = torch.randn(Co, 1, 3, 3, generator=g) / 3
    b = torch.randn(Co, generator=g)
    dy = torch.randn(B, T, F_, Co, generator=g)
    return x.to(device), w.to(device), b.to(device), dy.to(device)


def _check_c1(L, B, F_, T, Co, seed, relus=(0, 1), biases=(True, False), fwd_bar=C1_FWD_BAR, wgrad_bar=C1_WGRAD_BAR,
              ref_device="cpu"):
    x, w, b, dy = _c1_case(B, F_, T, Co, seed, ref_device)
    xc, wc, bc, dyc = x.cuda(), w.cuda(), b.cuda(), dy.cuda()
    for relu in relus:
        for has_bias in biases:
            y = _nan(B, T, F_, Co)
            L.check(_c1_fwd(L, xc, wc, bc if has_bias else None, y, B, F_, T, Co, relu), "conv3x3_c1_fwd")
            assert rel_err(y, c1_ref(x, w, b if has_bias else None, relu)) < fwd_bar, (relu, has_bias)
    dw, db = _nan(Co, 1, 3, 3), _nan(Co)
    L.check(_c1_wgrad(L, xc, dyc, dw, db, B, F_, T, Co), "conv3x3_c1_bwd_weight")
    dw_ref = torch.nn.grad.conv2d_weight(x.double()[:, None], (Co, 1, 3, 3), _nchw(dy.double()), padding=1)
    assert rel_err(dw, dw_ref) < wgrad_bar
    assert rel_err(db, dy.double().sum((0, 1, 2))) < wgrad_bar
    return xc, dyc, dw, db


@pytest.mark.parametrize("Co", C1_CO)
def test_conv3x3_c1_every_channel_count(L, Co):
    """Every accepted Co -- from 256 pixel slots of one channel quad (Co = 4) down to one slot of 256 quads (Co = 1024) --
    forward with ReLU on and off and with bias NULL, and the weight and bias gradients."""
    _check_c1(L, 2, 13, 37, Co, seed=Co)


@pytest.mark.parametrize("F_", [1, 7, 8, 9, 161])
@pytest.mark.parametrize("T", [1, 31, 32, 33])
def test_conv3x3_c1_tile_edges(L, T, F_):
    """Both sides of the 32 (time) x 8 (freq) tile; B = 3, so the weight gradient's tiles cross utterances."""
    _check_c1(L, 3, F_, T, 64, seed=T * 1000 + F_, relus=(1,), biases=(True,))


# measured maxima over 1.3e5 - 5.2e5 pixels: weight gradient 2.8e-7, bias gradient 4.0e-7 (both at cfg2)
C1_LARGE_WGRAD_BAR = 1.2e-6


@pytest.mark.parametrize("case", ["4sms-1_tiles", "4sms+1_tiles", "cfg2"])
def test_conv3x3_c1_weight_gradient_grid_stride(L, case):
    """The weight gradient launches 4 x SM-count blocks that stride over the tiles: one tile fewer than blocks (one block
    idle), one tile more (one block takes two), and the cfg2 layer at B = 4 (about four tiles per block).  float64
    references on the GPU.  Two calls give identical bits (partials summed in a fixed order)."""
    if case == "cfg2":
        B, F_, T = 4, 161, 800
    else:
        B, F_ = 1, 8
        T = 32 * (4 * _sms() + (1 if case == "4sms+1_tiles" else -1))
    xc, dyc, dw, db = _check_c1(L, B, F_, T, 64, seed=len(case), relus=(1,), biases=(True,),
                                wgrad_bar=C1_LARGE_WGRAD_BAR, ref_device="cuda")
    dw2, db2 = _nan(64, 1, 3, 3), _nan(64)
    L.check(_c1_wgrad(L, xc, dyc, dw2, db2, B, F_, T, 64), "conv3x3_c1_bwd_weight")
    assert torch.equal(dw, dw2) and torch.equal(db, db2)


def test_conv3x3_c1_empty_problem(L):
    """T = 0: the forward writes nothing, the weight gradient writes zeros.  x and dy are one-element buffers (an empty
    tensor's data_ptr() is NULL, which is rejected)."""
    Co = 64
    x, dy = torch.zeros(1, device="cuda"), torch.zeros(Co, device="cuda")
    w, b = torch.randn(Co, 1, 3, 3, device="cuda"), torch.randn(Co, device="cuda")
    y = _nan(Co)
    assert _c1_fwd(L, x, w, b, y, 1, 8, 0, Co, 1) == OK
    dw, db = _nan(Co, 1, 3, 3), _nan(Co)
    assert _c1_wgrad(L, x, dy, dw, db, 1, 8, 0, Co) == OK
    torch.cuda.synchronize()
    assert _all_nan(y)
    assert bool((dw == 0).all()) and bool((db == 0).all())


def test_conv3x3_c1_rejections(L):
    """Unsupported Co -> BAD_SHAPE, a NULL pointer -> BAD_ARG, y or dy 4 bytes off a 16-byte boundary -> BAD_ALIGN; the
    poisoned outputs stay untouched."""
    B, F_, T = 1, 8, 32
    x = torch.randn(B, F_, T, device="cuda")
    for Co in (12, 2048):
        w, b = torch.randn(Co, 1, 3, 3, device="cuda"), torch.randn(Co, device="cuda")
        dy = torch.randn(B, T, F_, Co, device="cuda")
        y, dw, db = _nan(B, T, F_, Co), _nan(Co, 1, 3, 3), _nan(Co)
        assert _c1_fwd(L, x, w, b, y, B, F_, T, Co, 1) == BAD_SHAPE
        assert _c1_wgrad(L, x, dy, dw, db, B, F_, T, Co) == BAD_SHAPE
        torch.cuda.synchronize()
        assert _all_nan(y) and _all_nan(dw) and _all_nan(db)
    Co = 64
    w, b = torch.randn(Co, 1, 3, 3, device="cuda"), torch.randn(Co, device="cuda")
    dy = torch.randn(B, T, F_, Co, device="cuda")
    y, dw, db = _nan(B, T, F_, Co), _nan(Co, 1, 3, 3), _nan(Co)
    assert _c1_fwd(L, None, w, b, y, B, F_, T, Co, 1) == BAD_ARG
    assert _c1_wgrad(L, x, dy, dw, None, B, F_, T, Co) == BAD_ARG
    y_off = _off(B * T * F_ * Co)
    assert _c1_fwd(L, x, w, b, y_off, B, F_, T, Co, 1) == BAD_ALIGN
    dy_off = _off(B * T * F_ * Co)
    dy_off.copy_(dy.flatten())
    assert _c1_wgrad(L, x, dy_off, dw, db, B, F_, T, Co) == BAD_ALIGN
    assert "align" in L.last_error()
    torch.cuda.synchronize()
    assert _all_nan(y) and _all_nan(y_off) and _all_nan(dw) and _all_nan(db)


# ================================================================================================ 2. max pooling
POOL_TF = [(1, 1), (1, 7), (2, 1), (2, 2), (3, 5), (33, 161)]
POOL_C = [4, 8, 64, 128]


def pool_input(kind, B, T, F_, C, seed):
    """'relu': relu(randn), half of it exact zeros.  'ints': values in {-2, ..., 2}, and a sixth of the windows all zero
    and another sixth all negative (values in {-3, -2, -1}, still tied)."""
    g = _gen(seed)
    if kind == "relu":
        return torch.randn(B, T, F_, C, generator=g).relu()
    x = torch.randint(-2, 3, (B, T, F_, C), generator=g).float()
    T2, F2 = T // 2, F_ // 2
    if T2 and F2:
        sel = torch.randint(0, 6, (B, T2, F2, C), generator=g)
        win = lambda m: m.repeat_interleave(2, 1).repeat_interleave(2, 2)
        xs = x[:, :2 * T2, :2 * F2]
        xs[win(sel == 0)] = 0.0
        neg = win(sel == 1)
        xs[neg] = -xs[neg].abs() - 1.0
    return x


def _pool_buf(shape, fill, dtype=torch.float32):
    """(buffer, view): max(numel, 1) elements -- never NULL, unlike the data_ptr() of an empty tensor -- and the first
    numel of them viewed as `shape`.  The kernels get the buffer's pointer."""
    n = int(np.prod(shape))
    buf = torch.full((max(n, 1),), fill, device="cuda", dtype=dtype)
    return buf, buf[:n].view(shape)


def _check_pool(L, B, T, F_, C, kind, seed):
    lib, st = L.load(), _stream()
    x = pool_input(kind, B, T, F_, C, seed)
    ref = pool_ref(x)
    ps = (B, T // 2, F_ // 2, C)
    xc = x.cuda()
    (yb, y), (y2b, y2) = _pool_buf(ps, NAN), _pool_buf(ps, NAN)
    idxb, idx = _pool_buf(ps, 255, torch.uint8)
    L.check(lib.b200asr_maxpool2x2_fwd(L.ptr(xc), L.ptr(yb), B, T, F_, C, st), "maxpool2x2_fwd")
    L.check(lib.b200asr_maxpool2x2_fwd_idx(L.ptr(xc), L.ptr(y2b), L.ptr(idxb), B, T, F_, C, st), "maxpool2x2_fwd_idx")
    if ref is not None:
        assert torch.equal(y.cpu(), ref[2].float()) and torch.equal(y2.cpu(), ref[2].float())
        assert torch.equal(idx.cpu(), ref[3])
    else:                                    # no window: nothing written
        assert _all_nan(yb) and _all_nan(y2b) and int(idxb[0]) == 255
    dy = torch.randn(ps, generator=_gen(seed + 1))
    dyc_b, dyc = _pool_buf(ps, NAN)
    dyc.copy_(dy)
    for relu_mask in (0, 1):
        dx_ref = pool_bwd_ref(ref, dy, x.shape, relu_mask).float()
        pr_ref = pairs_ref(dx_ref)
        for via_idx in (False, True):
            dx = _nan(B, T, F_, C)
            dx16 = torch.full((2, B, T, F_, C), NAN, device="cuda", dtype=torch.bfloat16)
            if via_idx:
                rc = lib.b200asr_maxpool2x2_bwd_idx(L.ptr(dyc_b), L.ptr(idxb), L.ptr(dx), L.ptr(dx16), B, T, F_, C, relu_mask, st)
            else:
                rc = lib.b200asr_maxpool2x2_bwd(L.ptr(dyc_b), L.ptr(xc), L.ptr(dx), L.ptr(dx16), B, T, F_, C, relu_mask, st)
            L.check(rc, "maxpool2x2_bwd")
            assert torch.equal(dx.cpu(), dx_ref), (relu_mask, via_idx)
            assert torch.equal(dx16.view(torch.int16).cpu(), pr_ref), (relu_mask, via_idx)
            # and without the pairs: the same gradient
            dx_b = _nan(B, T, F_, C)
            if via_idx:
                rc = lib.b200asr_maxpool2x2_bwd_idx(L.ptr(dyc_b), L.ptr(idxb), L.ptr(dx_b), None, B, T, F_, C, relu_mask, st)
            else:
                rc = lib.b200asr_maxpool2x2_bwd(L.ptr(dyc_b), L.ptr(xc), L.ptr(dx_b), None, B, T, F_, C, relu_mask, st)
            L.check(rc, "maxpool2x2_bwd")
            assert torch.equal(dx_b, dx)


@pytest.mark.parametrize("kind", ["relu", "ints"])
@pytest.mark.parametrize("C", POOL_C)
@pytest.mark.parametrize("T,F_", POOL_TF)
def test_maxpool2x2_against_aten(L, T, F_, C, kind):
    """Forward values and index bytes, and both backwards (from the activation and from the index bytes) with relu_mask
    0 and 1, with and without the bf16 pairs, bit-exact: every dx position -- routed, not routed, the odd-T rows and
    odd-F columns no window covers, the whole tensor when T or F is 1 -- is written."""
    _check_pool(L, 2, T, F_, C, kind, seed=T * 10000 + F_ * 10 + C)


def test_maxpool2x2_cfg2_pool1(L):
    """The cfg2 pool-1 layer at B = 4: 800 x 161 x 64 (odd F)."""
    _check_pool(L, 4, 800, 161, 64, "relu", seed=5)


def test_maxpool2x2_misaligned_pointers_are_rejected(L):
    """A float tensor 4 bytes off a 16-byte boundary, the index bytes 1 byte off a 4-byte one, the pairs 4 bytes off an
    8-byte one: BAD_ALIGN, nothing written."""
    lib, st = L.load(), _stream()
    B, T, F_, C = 1, 4, 6, 8
    n, m = B * T * F_ * C, B * (T // 2) * (F_ // 2) * C
    x, dy = torch.randn(n, device="cuda"), torch.randn(m, device="cuda")
    y, dx = _nan(m), _nan(n)
    idx = torch.zeros(m, device="cuda", dtype=torch.uint8)
    idx_off = torch.zeros(m + 4, device="cuda", dtype=torch.uint8)[1:m + 1]
    dx16 = torch.full((2 * n,), NAN, device="cuda", dtype=torch.bfloat16)
    dx16_off = torch.full((2 * n + 4,), NAN, device="cuda", dtype=torch.bfloat16)[2:2 * n + 2]
    x_off, y_off, dy_off, dx_off = _off(n), _off(m), _off(m), _off(n)
    x_off.copy_(x)
    dy_off.copy_(dy)
    calls = [
        lambda: lib.b200asr_maxpool2x2_fwd(L.ptr(x_off), L.ptr(y), B, T, F_, C, st),
        lambda: lib.b200asr_maxpool2x2_fwd(L.ptr(x), L.ptr(y_off), B, T, F_, C, st),
        lambda: lib.b200asr_maxpool2x2_fwd_idx(L.ptr(x), L.ptr(y), L.ptr(idx_off), B, T, F_, C, st),
        lambda: lib.b200asr_maxpool2x2_bwd(L.ptr(dy_off), L.ptr(x), L.ptr(dx), None, B, T, F_, C, 1, st),
        lambda: lib.b200asr_maxpool2x2_bwd(L.ptr(dy), L.ptr(x_off), L.ptr(dx), None, B, T, F_, C, 1, st),
        lambda: lib.b200asr_maxpool2x2_bwd(L.ptr(dy), L.ptr(x), L.ptr(dx_off), None, B, T, F_, C, 1, st),
        lambda: lib.b200asr_maxpool2x2_bwd(L.ptr(dy), L.ptr(x), L.ptr(dx), L.ptr(dx16_off), B, T, F_, C, 1, st),
        lambda: lib.b200asr_maxpool2x2_bwd_idx(L.ptr(dy), L.ptr(idx_off), L.ptr(dx), None, B, T, F_, C, 1, st),
        lambda: lib.b200asr_maxpool2x2_bwd_idx(L.ptr(dy_off), L.ptr(idx), L.ptr(dx), None, B, T, F_, C, 1, st),
        lambda: lib.b200asr_maxpool2x2_bwd_idx(L.ptr(dy), L.ptr(idx), L.ptr(dx_off), None, B, T, F_, C, 1, st),
        lambda: lib.b200asr_maxpool2x2_bwd_idx(L.ptr(dy), L.ptr(idx), L.ptr(dx), L.ptr(dx16_off), B, T, F_, C, 1, st),
    ]
    for i, call in enumerate(calls):
        assert call() == BAD_ALIGN, i
    torch.cuda.synchronize()
    assert _all_nan(y) and _all_nan(y_off) and _all_nan(dx) and _all_nan(dx_off)
    assert bool((idx_off == 0).all()) and _all_nan(dx16_off.float())
    # the same calls on aligned pointers run
    L.check(lib.b200asr_maxpool2x2_fwd_idx(L.ptr(x), L.ptr(y), L.ptr(idx), B, T, F_, C, st), "maxpool2x2_fwd_idx")
    L.check(lib.b200asr_maxpool2x2_bwd_idx(L.ptr(dy), L.ptr(idx), L.ptr(dx), L.ptr(dx16), B, T, F_, C, 1, st), "bwd_idx")
    torch.cuda.synchronize()
    assert not bool(torch.isnan(dx).any())


# ================================================================================================ 3. precision-0 3x3 convolution
# measured maxima: forward 1.4e-6, data gradient 1.1e-6 (contractions of 9 * Ci <= 2304 terms, one fp32 accumulator each)
CONV_FWD_BAR = 4e-6
CONV_DGRAD_BAR = 4e-6
# measured maxima: weight gradient 1.4e-6 (P <= 1029), 2.4e-6 (1.16e6 pixels); bias gradient 1.7e-7, 4.3e-7
CONV_WGRAD_BAR = 4e-6
CONV_WGRAD_LARGE_BAR = 7e-6


def _conv_ws(L, Ci, Co):
    return torch.full((L.load().b200asr_conv3x3_ws_bytes(Ci, Co) // 4,), NAN, device="cuda")


def _conv_fwd(L, x, w, b, y, ws, B, T, F_, Ci, Co, relu):
    return L.load().b200asr_conv3x3_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F_, Ci, Co, relu,
                                        PREC_FP32, _stream())


def _conv_dgrad(L, dy, w, mask, dx, ws, B, T, F_, Ci, Co):
    return L.load().b200asr_conv3x3_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(mask), L.ptr(dx), None, L.ptr(ws), B, T, F_, Ci,
                                             Co, PREC_FP32, _stream())


def _conv_wgrad(L, dy, x, dw, db, ws, B, T, F_, Ci, Co):
    return L.load().b200asr_conv3x3_bwd_weight(L.ptr(dy), None, L.ptr(x), L.ptr(dw), L.ptr(db), L.ptr(ws), B, T, F_, Ci,
                                               Co, PREC_FP32, _stream())


# (B, T, F, Ci, Co): Ci = 16 / 48 give one / three 16-channel chunks per tap; Co = 64 and 192 run BN = 64 (one and three
# column tiles), Co = 128 and 256 BN = 128 (one and two); no P = B*T*F is a multiple of the 128-pixel tile
CONV_FWD = [(2, 13, 11, 16, 64), (1, 1, 37, 48, 192), (3, 17, 2, 64, 256), (2, 2, 29, 128, 128), (1, 40, 1, 48, 64),
            (2, 9, 21, 128, 192), (1, 33, 7, 16, 256)]


@pytest.mark.parametrize("B,T,F_,Ci,Co", CONV_FWD)
def test_conv3x3_precision0_forward(L, B, T, F_, Ci, Co):
    """conv3x3_fwd at precision 0 with ReLU on and off and with bias NULL."""
    g = _gen(B * T * F_ + Ci + Co)
    x = torch.randn(B, T, F_, Ci, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) * (9 * Ci) ** -0.5
    b = torch.randn(Co, generator=g)
    xc, wc, bc = x.cuda(), w.cuda(), b.cuda()
    for relu in (0, 1):
        for has_bias in (True, False):
            y, ws = _nan(B, T, F_, Co), _conv_ws(L, Ci, Co)
            L.check(_conv_fwd(L, xc, wc, bc if has_bias else None, y, ws, B, T, F_, Ci, Co, relu), "conv3x3_fwd")
            assert rel_err(y, conv3x3_ref(x, w, b if has_bias else None, relu)) < CONV_FWD_BAR, (relu, has_bias)


# (B, T, F, Ci, Co): Ci (the data gradient's output channels) 64 / 128 / 192, contraction over Co
CONV_DGRAD = [(2, 13, 11, 64, 64), (1, 1, 37, 192, 128), (3, 17, 2, 64, 256), (2, 9, 21, 128, 64), (1, 40, 1, 192, 64),
              (1, 33, 5, 128, 48)]


@pytest.mark.parametrize("B,T,F_,Ci,Co", CONV_DGRAD)
def test_conv3x3_precision0_data_gradient(L, B, T, F_, Ci, Co):
    """conv3x3_bwd_data at precision 0, without a mask and with a relu_out mask a third of which is exactly 0 (and the rest
    of either sign): the mask passes a gradient where it is > 0 only."""
    g = _gen(B * T * F_ + 3 * Ci + Co)
    dy = torch.randn(B, T, F_, Co, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) * (9 * Co) ** -0.5
    mask = torch.randn(B, T, F_, Ci, generator=g)
    mask[torch.rand(mask.shape, generator=g) < 1 / 3] = 0.0
    dyc, wc = dy.cuda(), w.cuda()
    for m in (None, mask):
        dx, ws = _nan(B, T, F_, Ci), _conv_ws(L, Ci, Co)
        L.check(_conv_dgrad(L, dyc, wc, None if m is None else m.cuda(), dx, ws, B, T, F_, Ci, Co), "conv3x3_bwd_data")
        ref = conv3x3_dgrad_ref(dy, w, m)
        assert rel_err(dx, ref) < CONV_DGRAD_BAR
        if m is not None:
            assert bool((dx.cpu()[m <= 0] == 0).all())


def _check_conv_wgrad(L, B, T, F_, Ci, Co, seed, bar, ref_device="cpu", with_bias=True):
    g = _gen(seed)
    x = torch.randn(B, T, F_, Ci, generator=g).to(ref_device)
    dy = torch.randn(B, T, F_, Co, generator=g).to(ref_device)
    xc, dyc = x.cuda(), dy.cuda()
    dw, db, ws = _nan(Co, Ci, 3, 3), _nan(Co), _conv_ws(L, Ci, Co)
    L.check(_conv_wgrad(L, dyc, xc, dw, db if with_bias else None, ws, B, T, F_, Ci, Co), "conv3x3_bwd_weight")
    dw_ref, db_ref = conv3x3_wgrad_ref(_nchw(x), dy, Ci)
    assert rel_err(dw, dw_ref) < bar
    if with_bias:
        assert rel_err(db, db_ref) < bar
    else:
        assert _all_nan(db)


@pytest.mark.parametrize("Co", [64, 128, 192])
@pytest.mark.parametrize("Ci", [64, 128, 192])
@pytest.mark.parametrize("P", ["one_chunk", "1024+5"])
def test_conv3x3_precision0_weight_gradient(L, P, Ci, Co):
    """conv3x3_bwd_weight at precision 0 at all four <BMC, BNC> instantiations (128 where the channel count is a
    multiple of 128, 64 otherwise): P = 143 pixels (one chunk, not a multiple of 16) and P = 1029 = 1024 + 5 (the chunk is
    1024 pixels there, so the last one holds 5).  The pixel axis is split over CTAs that add with atomics: tolerance
    only."""
    B, T, F_ = (1, 13, 11) if P == "one_chunk" else (1, 49, 21)
    _check_conv_wgrad(L, B, T, F_, Ci, Co, seed=Ci * 7 + Co + T, bar=CONV_WGRAD_BAR, with_bias=(Ci != Co))


@pytest.mark.parametrize("B", [4, 9])
def test_conv3x3_precision0_weight_gradient_large(L, B):
    """cfg2's conv2 (64 -> 64, 800 x 161) at B = 4, where the chunk comes from the SM-count formula, and at B = 9:
    1.16e6 >= 2^20 pixels, where the bias gradient's column sum takes its 2048-row slices.  float64 references on the
    GPU."""
    _check_conv_wgrad(L, B, 800, 161, 64, 64, seed=B, bar=CONV_WGRAD_LARGE_BAR, ref_device="cuda")


def test_conv3x3_precision0_misaligned_pointers_are_rejected(L):
    """Precision 0: x, y, dy, relu_out, dx and ws 4 bytes off a 16-byte boundary -> BAD_ALIGN, nothing written."""
    B, T, F_, Ci, Co = 1, 4, 4, 64, 64
    n = B * T * F_ * Ci
    x, w, b = torch.randn(n, device="cuda"), torch.randn(Co, Ci, 3, 3, device="cuda"), torch.randn(Co, device="cuda")
    dy, mask = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    x_off, dy_off, mask_off = _off(n), _off(n), _off(n)
    x_off.copy_(x)
    dy_off.copy_(dy)
    mask_off.copy_(mask)
    y, y_off, ws = _nan(n), _off(n), _conv_ws(L, Ci, Co)
    ws_off = _off(ws.numel())
    dw, db = _nan(Co, Ci, 3, 3), _nan(Co)
    fwd = lambda x_, y_, ws_: _conv_fwd(L, x_, w, b, y_, ws_, B, T, F_, Ci, Co, 1)
    dgrad = lambda dy_, m_, dx_, ws_: _conv_dgrad(L, dy_, w, m_, dx_, ws_, B, T, F_, Ci, Co)
    wgrad = lambda dy_, x_: _conv_wgrad(L, dy_, x_, dw, db, ws, B, T, F_, Ci, Co)
    assert fwd(x_off, y, ws) == BAD_ALIGN
    assert fwd(x, y_off, ws) == BAD_ALIGN
    assert fwd(x, y, ws_off) == BAD_ALIGN
    assert dgrad(dy_off, mask, y, ws) == BAD_ALIGN
    assert dgrad(dy, mask_off, y, ws) == BAD_ALIGN
    assert dgrad(dy, mask, y_off, ws) == BAD_ALIGN
    assert dgrad(dy, mask, y, ws_off) == BAD_ALIGN
    assert wgrad(dy_off, x) == BAD_ALIGN
    assert wgrad(dy, x_off) == BAD_ALIGN
    torch.cuda.synchronize()
    assert _all_nan(y) and _all_nan(y_off) and _all_nan(ws) and _all_nan(ws_off) and _all_nan(dw) and _all_nan(db)


# ================================================================================================ 4. emb_cnn direct convolutions
# (B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW)
EMB_GEOMS = {
    "ref_conv1": (2, 1, 161, 51, 32, 41, 11, 2, 2, 0, 10),       # models/asr/transformer.py:34, odd W
    "ref_conv2": (2, 32, 161, 25, 32, 21, 11, 2, 1, 0, 0),       # :37
    "kw16": (2, 3, 20, 40, 5, 3, 16, 1, 1, 1, 7),                # the weight gradient's widest kernel
    "stride_gt_kernel": (2, 4, 17, 23, 6, 2, 1, 3, 2, 0, 0),     # rows and columns no window reads: dx exactly 0
    "pad_ge_kernel": (2, 3, 6, 7, 4, 3, 3, 1, 1, 4, 3),          # outputs whose window is all padding: y == bias
    "oh1": (3, 2, 5, 9, 3, 5, 3, 1, 2, 0, 1),                    # OH = 1
    "ow1": (2, 2, 9, 4, 3, 3, 4, 2, 1, 1, 0),                    # OW = 1
    "ow_gt_128": (2, 2, 7, 300, 3, 3, 5, 1, 1, 1, 2),            # OW = 300: each weight-gradient thread takes 3 columns
}
# measured maxima: forward 3.4e-7, data gradient 5.8e-7, weight gradient 2.9e-7, bias gradient 2.0e-7
EMB_BAR = 2e-6
# The forward and data gradient of the reference's geometries: measured 4.7e-6 and 2.9e-6 (ref_conv2).  The direct kernels
# sum each output in one sequential fp32 chain -- 32 x 21 x 11 = 7392 products for conv2's forward -- and the rounding
# of such a chain grows with the square root of its length, so these two sit above the exact-fp32 1e-5 mark.
EMB_LONG_BAR = 1.5e-5


@pytest.mark.parametrize("name", list(EMB_GEOMS))
def test_conv2d_direct_against_float64(L, name):
    """conv2d_fwd / _bwd_data / _bwd_weight (+ bias gradient) against F.conv2d and its autograd in float64; the weight
    gradient once more with dbias NULL."""
    lib, st = L.load(), _stream()
    B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW = EMB_GEOMS[name]
    OH, OW = (H + 2 * PH - KH) // SH + 1, (W + 2 * PW - KW) // SW + 1
    g = _gen(len(name) * 31 + H)
    x = torch.randn(B, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, KH, KW, generator=g) * (Ci * KH * KW) ** -0.5
    b = torch.randn(Co, generator=g)
    dy = torch.randn(B, Co, OH, OW, generator=g)
    x64, w64, b64 = (t.double().requires_grad_(True) for t in (x, w, b))
    y64 = F.conv2d(x64, w64, b64, stride=(SH, SW), padding=(PH, PW))
    assert y64.shape == (B, Co, OH, OW)
    y64.backward(dy.double())
    xc, wc, bc, dyc = x.cuda(), w.cuda(), b.cuda(), dy.cuda()
    args = EMB_GEOMS[name]

    y = _nan(B, Co, OH, OW)
    L.check(lib.b200asr_conv2d_fwd(L.ptr(xc), L.ptr(wc), L.ptr(bc), L.ptr(y), *args, st), "conv2d_fwd")
    bar = EMB_LONG_BAR if name.startswith("ref_") else EMB_BAR
    assert rel_err(y, y64.detach()) < bar
    # windows that read only padding: exactly the bias
    seen = F.conv2d(torch.ones(1, 1, H, W, dtype=torch.float64), torch.ones(1, 1, KH, KW, dtype=torch.float64),
                    stride=(SH, SW), padding=(PH, PW))[0, 0] > 0
    if name == "pad_ge_kernel":
        assert not bool(seen.all())
    yb = y.cpu()
    assert torch.equal(yb[:, :, ~seen], b[None, :, None].expand(B, Co, int((~seen).sum())))

    dx = _nan(B, Ci, H, W)
    L.check(lib.b200asr_conv2d_bwd_data(L.ptr(dyc), L.ptr(wc), L.ptr(dx), *args, st), "conv2d_bwd_data")
    assert rel_err(dx, x64.grad) < bar
    # input positions no window reads: exactly 0
    read = torch.nn.grad.conv2d_input((1, 1, H, W), torch.ones(1, 1, KH, KW, dtype=torch.float64),
                                      torch.ones(1, 1, OH, OW, dtype=torch.float64), stride=(SH, SW), padding=(PH, PW))[0, 0] > 0
    if name == "stride_gt_kernel":
        assert not bool(read.all())
    assert bool((dx.cpu()[:, :, ~read] == 0).all())

    dw, db = _nan(Co, Ci, KH, KW), _nan(Co)
    L.check(lib.b200asr_conv2d_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw), L.ptr(db), *args, st), "conv2d_bwd_weight")
    assert rel_err(dw, w64.grad) < EMB_BAR
    assert rel_err(db, b64.grad) < EMB_BAR
    dw2, db2 = _nan(Co, Ci, KH, KW), _nan(Co)
    L.check(lib.b200asr_conv2d_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw2), None, *args, st), "conv2d_bwd_weight")
    torch.cuda.synchronize()
    assert torch.equal(dw2, dw) and _all_nan(db2)


def test_conv2d_direct_rejections(L):
    """KW = 17 in the weight gradient, an empty output and a zero stride -> BAD_SHAPE; nothing written."""
    lib, st = L.load(), _stream()
    x, w, b, dy = (torch.randn(4096, device="cuda") for _ in range(4))
    out, dw, db = _nan(4096), _nan(4096), _nan(64)
    kw17 = (1, 1, 8, 40, 1, 1, 17, 1, 1, 0, 0)
    assert lib.b200asr_conv2d_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw), L.ptr(db), *kw17, st) == BAD_SHAPE
    for geom in [(1, 2, 5, 9, 3, 7, 3, 1, 1, 0, 0),        # KH = 7 > H = 5, no padding: OH = 0
                 (1, 2, 5, 9, 3, 3, 3, 0, 1, 1, 1),        # SH = 0
                 (1, 2, 5, 9, 3, 3, 3, 1, 0, 1, 1)]:       # SW = 0
        assert lib.b200asr_conv2d_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(out), *geom, st) == BAD_SHAPE
        assert lib.b200asr_conv2d_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(out), *geom, st) == BAD_SHAPE
        assert lib.b200asr_conv2d_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw), L.ptr(db), *geom, st) == BAD_SHAPE
    torch.cuda.synchronize()
    assert _all_nan(out) and _all_nan(dw) and _all_nan(db)


@pytest.mark.parametrize("B,C,F_,T", [(2, 3, 13, 45), (1, 32, 5, 33), (3, 7, 1, 70), (1, 1, 41, 1)])
def test_flatten_bcft_bit_exact(L, B, C, F_, T):
    """flatten_bcft_fwd: y[b][t][c*F + f] = x[b][c][f][t]; _bwd its inverse; sizes off the 32 x 32 transpose tile."""
    lib, st = L.load(), _stream()
    x = torch.randn(B, C, F_, T, generator=_gen(B * C * F_ * T)).cuda()
    y = _nan(B, T, C * F_)
    L.check(lib.b200asr_flatten_bcft_fwd(L.ptr(x), L.ptr(y), B, C, F_, T, st), "flatten_bcft_fwd")
    assert torch.equal(y, x.permute(0, 3, 1, 2).reshape(B, T, C * F_))
    dy = torch.randn(B, T, C * F_, device="cuda")
    dx = _nan(B, C, F_, T)
    L.check(lib.b200asr_flatten_bcft_bwd(L.ptr(dy), L.ptr(dx), B, C, F_, T, st), "flatten_bcft_bwd")
    assert torch.equal(dx, dy.view(B, T, C, F_).permute(0, 2, 3, 1))
    back = _nan(B, C, F_, T)
    L.check(lib.b200asr_flatten_bcft_bwd(L.ptr(y), L.ptr(back), B, C, F_, T, st), "flatten_bcft_bwd")
    assert torch.equal(back, x)


@pytest.mark.parametrize("rows,C,F_", [(37, 3, 13), (5, 64, 41), (1, 128, 40), (70, 1, 33), (3, 31, 1)])
def test_permute_cols_cf_bit_exact(L, rows, C, F_):
    """permute_cols_cf: dst[r, f*C + c] = src[r, c*F + f]; inverse != 0 the inverse permutation; a round trip."""
    lib, st = L.load(), _stream()
    src = torch.randn(rows, C * F_, generator=_gen(rows + C + F_)).cuda()
    dst, back = _nan(rows, C * F_), _nan(rows, C * F_)
    L.check(lib.b200asr_permute_cols_cf(L.ptr(src), L.ptr(dst), rows, C, F_, 0, st), "permute_cols_cf")
    assert torch.equal(dst, src.view(rows, C, F_).transpose(1, 2).reshape(rows, F_ * C))
    inv = _nan(rows, C * F_)
    L.check(lib.b200asr_permute_cols_cf(L.ptr(src), L.ptr(inv), rows, C, F_, 1, st), "permute_cols_cf inverse")
    assert torch.equal(inv, src.view(rows, F_, C).transpose(1, 2).reshape(rows, C * F_))
    L.check(lib.b200asr_permute_cols_cf(L.ptr(dst), L.ptr(back), rows, C, F_, 1, st), "permute_cols_cf round trip")
    assert torch.equal(back, src)
