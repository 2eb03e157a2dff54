"""The VGG front end's ReLU decisions as packed bits (include/b200asr.h: conv3x3_c1_fwd_bits, conv3x3_fwd_bits,
conv3x3_bwd_data_bits), through the raw C ABI, BIT-EXACT against the entry points they derive from:

  1. the bits of conv3x3_c1_fwd_bits and of conv3x3_fwd_bits at every precision (the halo epilogue in modes 6, 2 and 3, the
     TF32 engine's epilogue, the precision-0 ballot pass) equal (y > 0) packed, and y itself equals the plain forward's;
  1b. the pooling codes of conv3x3_fwd_pool_codes (the halo epilogue in the bf16 modes, the stand-alone pooling kernel
     otherwise) equal the first-maximum positions of y in ATen's scan order, pooled and y equal conv3x3_fwd_pool's, y = NULL
     gives the same pooled output and codes, and maxpool2x2_bwd_codes equals maxpool2x2_bwd(dy, y) incl. dx16;
  2. the data gradient from the bits equals the one from relu_out, dx and the bf16 pairs dx16, at every precision, with
     relu_out holding exact zeros, -0.0 and NaN (none of which sets a bit, as none passes `relu_out > 0`);
  3. a whole VggFrontendFn forward and backward gives the same bits as the call sequence that reads the fp32 activations;
  4. the new entry points reject a NULL or misaligned bit pointer and an unsupported Co before launching anything, and launch
     as many kernels as the calls they derive from (one more at precision 0's forward: the ballot pass).

Shapes: odd T and F, T and F off the halo kernel's 16 x 8 tile, C = 64 and 128, cfg2's layer shapes at B = 2, and halo tile
counts just below, at and above 132 (the H100 SXM's SM count).  Outputs are filled with NaN before each call."""
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
OK, BAD_SHAPE, BAD_ALIGN, BAD_ARG = 0, -1, -2, -5
PRECS = [6, 2, 3, 1, 0]          # bf16x3, bf16 (halo), 3xTF32 (halo), TF32 (engine), fp32 (CUDA cores)


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _st():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def pack_bits(v):
    """[..., C] -> int32 [..., C / 32]: bit c % 32 of word c / 32 = (v > 0)."""
    b = (v > 0).to(torch.int64).reshape(*v.shape[:-1], v.shape[-1] // 32, 32)
    w = (b << torch.arange(32, device=v.device)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def _bits_nan(*shape):
    """int32 words filled with the bit pattern of a NaN, so an unwritten word cannot pass for a decision."""
    return torch.full(shape[:-1] + (shape[-1] // 32,), 0x7FC00000, dtype=torch.int32, device="cuda")


def _intish(shape, seed, lo=-3, hi=4):
    """small integers: exact ties, exact zeros after the bias, all-non-positive regions"""
    return torch.randint(lo, hi, shape, generator=_gen(seed)).float().cuda()


def _eq(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ================================================================================================ 1. forward bits
C1_SHAPES = [(2, 17, 9, 64), (1, 161, 33, 32), (2, 8, 31, 128), (1, 5, 3, 256), (2, 161, 800, 64)]   # (B, F, T, Co); last: cfg2 conv1


@pytest.mark.parametrize("B,F_,T,Co", C1_SHAPES)
@pytest.mark.parametrize("relu", [1, 0])
def test_c1_fwd_bits(L, B, F_, T, Co, relu):
    lib = L.load()
    x = _intish((B, F_, T), 1)
    w = _intish((Co, 1, 3, 3), 2, -2, 3)
    b = _intish((Co,), 3, -2, 2)
    x[0, 0, :3] = -0.0
    y0, y1 = torch.full((B, T, F_, Co), NAN, device="cuda"), torch.full((B, T, F_, Co), NAN, device="cuda")
    bits = _bits_nan(B, T, F_, Co)
    L.check(lib.b200asr_conv3x3_c1_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y0), B, F_, T, Co, relu, _st()), "c1_fwd")
    L.check(lib.b200asr_conv3x3_c1_fwd_bits(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y1), B, F_, T, Co, relu, L.ptr(bits), _st()), "c1_bits")
    assert _eq(y0, y1)
    assert torch.equal(bits, pack_bits(y0))
    assert bool((y0 == 0).any()) and bool((y0 > 0).any())


# (B, T, F, Ci, Co); halo tiles = B * ceil(T / 16) * ceil(F / 8)
FWD_SHAPES = [(2, 17, 9, 64, 64), (1, 16, 8, 64, 128), (2, 33, 15, 128, 128), (2, 1, 41, 64, 64),
              (1, 2096, 8, 64, 64), (1, 176, 96, 64, 128), (1, 304, 56, 128, 64),      # 131, 132, 133 tiles
              (2, 400, 80, 64, 128)]                                                    # cfg2 conv3


@pytest.mark.parametrize("B,T,F_,Ci,Co", FWD_SHAPES)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("relu", [1, 0])
def test_conv3x3_fwd_bits(L, B, T, F_, Ci, Co, prec, relu):
    lib = L.load()
    x = _intish((B, T, F_, Ci), 4, -1, 3)
    w = (_intish((Co, Ci, 3, 3), 5, -2, 3) / 64)
    b = _intish((Co,), 6, -2, 2)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    y0, y1 = torch.full((B, T, F_, Co), NAN, device="cuda"), torch.full((B, T, F_, Co), NAN, device="cuda")
    bits = _bits_nan(B, T, F_, Co)
    args = lambda y: (L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F_, Ci, Co, relu, prec)
    L.check(lib.b200asr_conv3x3_fwd(*args(y0), _st()), "fwd")
    L.check(lib.b200asr_conv3x3_fwd_bits(*args(y1), L.ptr(bits), _st()), "fwd_bits")
    assert _eq(y0, y1)
    assert torch.equal(bits, pack_bits(y0))


# ================================================================================================ 1b. pooling codes
def pool_codes_ref(x):
    """x [B, T, F, C] (the pool input) -> int32 [B, T/2, F/2, C/8]: nibble c % 8 of word c / 8 = the first maximum's position
    in ATen's scan order (f, t), (f, t+1), (f+1, t), (f+1, t+1) | 4 when that maximum is not positive."""
    B, T, F_, C = x.shape
    T2, F2 = T // 2, F_ // 2
    v = x[:, :2 * T2, :2 * F2].reshape(B, T2, 2, F2, 2, C)
    a = [v[:, :, 0, :, 0], v[:, :, 1, :, 0], v[:, :, 0, :, 1], v[:, :, 1, :, 1]]
    best, m = torch.zeros_like(a[0], dtype=torch.int64), a[0]
    for k in (1, 2, 3):
        gt = a[k] > m
        best, m = torch.where(gt, k, best), torch.where(gt, a[k], m)
    code = (best | torch.where(m > 0, 0, 4)).reshape(B, T2, F2, C // 8, 8)
    w = (code << (4 * torch.arange(8, device=x.device))).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def _codes_nan(B, T, F_, C):
    return torch.full((B, T // 2, F_ // 2, C // 8), 0x7FC00000, dtype=torch.int32, device="cuda")


# (B, T, F, Ci, Co): odd T / F, off the 16 x 8 tile, 131-133 halo tiles, cfg2 conv2 / conv4 at B = 2
POOL_SHAPES = [(2, 17, 9, 64, 64), (1, 16, 8, 64, 128), (2, 33, 15, 128, 128), (1, 3, 21, 64, 128),
               (1, 2096, 8, 64, 64), (1, 176, 96, 64, 128), (1, 304, 56, 128, 64),
               (2, 800, 161, 64, 64), (2, 400, 80, 128, 128)]


@pytest.mark.parametrize("B,T,F_,Ci,Co", POOL_SHAPES)
@pytest.mark.parametrize("prec", PRECS)
def test_conv3x3_fwd_pool_codes(L, B, T, F_, Ci, Co, prec):
    """pooled and y bit-identical to b200asr_conv3x3_fwd_pool, the codes equal to those of y (integer data: exact ties,
    all-non-positive windows, exact zeros); in the bf16 modes the same pooled output and codes with y = NULL."""
    lib = L.load()
    x = _intish((B, T, F_, Ci), 9, -1, 3)
    w = (_intish((Co, Ci, 3, 3), 10, -2, 3) / 64)
    b = _intish((Co,), 11, -3, 2)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    full = lambda *s_: torch.full(s_, NAN, device="cuda")
    y0, y1 = full(B, T, F_, Co), full(B, T, F_, Co)
    p0, p1, p2 = (full(B, T // 2, F_ // 2, Co) for _ in range(3))
    c1, c2 = _codes_nan(B, T, F_, Co), _codes_nan(B, T, F_, Co)
    head = lambda y: (L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y))
    tail = (L.ptr(ws), B, T, F_, Ci, Co, 1, prec, _st())
    L.check(lib.b200asr_conv3x3_fwd_pool(*head(y0), L.ptr(p0), None, *tail), "fwd_pool")
    L.check(lib.b200asr_conv3x3_fwd_pool_codes(*head(y1), L.ptr(p1), L.ptr(c1), *tail), "fwd_pool_codes")
    assert _eq(y0, y1) and _eq(p0, p1)
    ref = pool_codes_ref(y0)
    assert torch.equal(c1, ref)
    assert bool(((ref & 4) != 0).any())
    if prec in (2, 6):
        L.check(lib.b200asr_conv3x3_fwd_pool_codes(*head(None), L.ptr(p2), L.ptr(c2), *tail), "fwd_pool_codes y=NULL")
        assert _eq(p0, p2) and torch.equal(c2, ref)
    else:
        rc, n = _launches(lib, lambda: lib.b200asr_conv3x3_fwd_pool_codes(*head(None), L.ptr(p2), L.ptr(c2), *tail))
        assert (rc, n) == (BAD_ARG, 0)


def _pool_input(shape, seed):
    """post-ReLU small integers: exact ties, all-zero windows, -0.0"""
    x = _intish(shape, seed, -2, 3).relu()
    x[..., 0, 0, :] = -0.0
    return x


@pytest.mark.parametrize("B,T,F_,C", [(2, 8, 6, 64), (1, 17, 9, 128), (2, 3, 5, 64), (1, 31, 3, 64), (2, 800, 161, 64),
                                      (2, 400, 80, 128)])
@pytest.mark.parametrize("relu_mask", [1, 0])
@pytest.mark.parametrize("pairs", [False, True])
def test_maxpool2x2_bwd_codes(L, B, T, F_, C, relu_mask, pairs):
    """maxpool2x2_bwd_codes == maxpool2x2_bwd(dy, x) bit for bit, dx and the bf16 pairs, incl. the odd-T / odd-F tail."""
    lib = L.load()
    x = _pool_input((B, T, F_, C), 12)
    codes = pool_codes_ref(x)
    dy = torch.randn(B, T // 2, F_ // 2, C, generator=_gen(13)).cuda()
    dx0, dx1 = torch.full((B, T, F_, C), NAN, device="cuda"), torch.full((B, T, F_, C), NAN, device="cuda")
    q0 = torch.full((2, B, T, F_, C), -1, dtype=torch.int16, device="cuda") if pairs else None
    q1 = torch.full((2, B, T, F_, C), -1, dtype=torch.int16, device="cuda") if pairs else None
    L.check(lib.b200asr_maxpool2x2_bwd(L.ptr(dy), L.ptr(x), L.ptr(dx0), L.ptr(q0), B, T, F_, C, relu_mask, _st()), "bwd")
    L.check(lib.b200asr_maxpool2x2_bwd_codes(L.ptr(dy), L.ptr(codes), L.ptr(dx1), L.ptr(q1), B, T, F_, C, relu_mask, _st()), "bwd_codes")
    assert _eq(dx0, dx1) and not bool(torch.isnan(dx1).any())
    if pairs:
        assert torch.equal(q0, q1)


# ================================================================================================ 2. data gradient from bits
# (B, T, F, Ci = dx channels, Co = dy channels)
DGRAD_SHAPES = [(2, 17, 9, 64, 64), (1, 16, 8, 128, 64), (2, 33, 15, 128, 128), (1, 3, 21, 64, 128),
                (1, 2096, 8, 64, 64), (1, 176, 96, 128, 64), (1, 304, 56, 64, 128),
                (2, 800, 161, 64, 64), (2, 400, 80, 128, 128)]                       # cfg2 conv2, conv4


def _relu_out(shape, seed):
    """post-ReLU-like values with exact zeros, plus -0.0, NaN and negatives (none of which passes `> 0`)"""
    g = _gen(seed)
    v = torch.randn(shape, generator=g).relu()
    r = torch.rand(shape, generator=g)
    v[r < 0.05] = -0.0
    v[(r >= 0.05) & (r < 0.07)] = NAN
    v[(r >= 0.07) & (r < 0.1)] = -1.0
    return v.cuda()


@pytest.mark.parametrize("B,T,F_,Ci,Co", DGRAD_SHAPES)
@pytest.mark.parametrize("prec", PRECS)
def test_conv3x3_bwd_data_bits(L, B, T, F_, Ci, Co, prec):
    lib = L.load()
    g = _gen(7)
    dy = torch.randn(B, T, F_, Co, generator=g).cuda()
    w = (torch.randn(Co, Ci, 3, 3, generator=g) * (9 * Co) ** -0.5).cuda()
    relu_out = _relu_out((B, T, F_, Ci), 8)
    bits = pack_bits(relu_out)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    pairs = prec in (2, 6)
    dx0, dx1 = torch.full((B, T, F_, Ci), NAN, device="cuda"), torch.full((B, T, F_, Ci), NAN, device="cuda")
    p0 = torch.full((2, B, T, F_, Ci), -1, dtype=torch.int16, device="cuda") if pairs else None
    p1 = torch.full((2, B, T, F_, Ci), -1, dtype=torch.int16, device="cuda") if pairs else None
    L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(relu_out), L.ptr(dx0), L.ptr(p0), L.ptr(ws), B, T, F_, Ci, Co,
                                         prec, _st()), "dgrad")
    L.check(lib.b200asr_conv3x3_bwd_data_bits(L.ptr(dy), L.ptr(w), L.ptr(bits), L.ptr(dx1), L.ptr(p1), L.ptr(ws), B, T, F_, Ci, Co,
                                              prec, _st()), "dgrad_bits")
    assert _eq(dx0, dx1)
    assert not bool(torch.isnan(dx1).any())
    if pairs:
        assert torch.equal(p0, p1)


# ================================================================================================ 3. the whole front end
def _frontend_by_activations(lib, L, x, ws_, dp2, prec, prec_w):
    """VggFrontendFn's forward and backward as the sequence of calls that masks the data gradients with the fp32 activations
    y1 / y3 (what the front end ran before it kept the decisions as bits)."""
    w0, b0, w2, b2, w5, b5, w7, b7 = ws_
    B, _, F_, T = x.shape
    C1, C2 = w0.shape[0], w5.shape[0]
    T2, F2, T4, F4 = T // 2, F_ // 2, T // 4, F_ // 4
    new = lambda *s: torch.empty(s, device="cuda")
    st = _st()
    ws = new(lib.b200asr_conv3x3_ws_bytes(C2, C2) // 4)
    y1, y2, p1 = new(B, T, F_, C1), new(B, T, F_, C1), new(B, T2, F2, C1)
    y3, y4, p2 = new(B, T2, F2, C2), new(B, T2, F2, C2), new(B, T4, F4, C2)
    L.check(lib.b200asr_conv3x3_c1_fwd(L.ptr(x), L.ptr(w0), L.ptr(b0), L.ptr(y1), B, F_, T, C1, 1, st))
    L.check(lib.b200asr_conv3x3_fwd_pool(L.ptr(y1), L.ptr(w2), L.ptr(b2), L.ptr(y2), L.ptr(p1), None, L.ptr(ws), B, T, F_, C1, C1, 1,
                                         prec, st))
    L.check(lib.b200asr_conv3x3_fwd(L.ptr(p1), L.ptr(w5), L.ptr(b5), L.ptr(y3), L.ptr(ws), B, T2, F2, C1, C2, 1, prec, st))
    L.check(lib.b200asr_conv3x3_fwd_pool(L.ptr(y3), L.ptr(w7), L.ptr(b7), L.ptr(y4), L.ptr(p2), None, L.ptr(ws), B, T2, F2, C2, C2, 1,
                                         prec, st))
    pairs = prec in (2, 6) and prec_w in (2, 6)
    new16 = lambda *s: torch.empty((2,) + s, device="cuda", dtype=torch.bfloat16) if pairs else None
    d4, d4p = new(B, T2, F2, C2), new16(B, T2, F2, C2)
    L.check(lib.b200asr_maxpool2x2_bwd(L.ptr(dp2), L.ptr(y4), L.ptr(d4), L.ptr(d4p), B, T2, F2, C2, 1, st))
    dw7, db7 = torch.empty_like(w7), new(C2)
    L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(d4), L.ptr(d4p), L.ptr(y3), L.ptr(dw7), L.ptr(db7), L.ptr(ws), B, T2, F2, C2, C2, prec_w, st))
    d3, d3p = new(B, T2, F2, C2), new16(B, T2, F2, C2)
    L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(d4), L.ptr(w7), L.ptr(y3), L.ptr(d3), L.ptr(d3p), L.ptr(ws), B, T2, F2, C2, C2, prec, st))
    dw5, db5 = torch.empty_like(w5), new(C2)
    L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(d3), L.ptr(d3p), L.ptr(p1), L.ptr(dw5), L.ptr(db5), L.ptr(ws), B, T2, F2, C1, C2, prec_w, st))
    dp1 = new(B, T2, F2, C1)
    L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(d3), L.ptr(w5), None, L.ptr(dp1), None, L.ptr(ws), B, T2, F2, C1, C2, prec, st))
    d2, d2p = new(B, T, F_, C1), new16(B, T, F_, C1)
    L.check(lib.b200asr_maxpool2x2_bwd(L.ptr(dp1), L.ptr(y2), L.ptr(d2), L.ptr(d2p), B, T, F_, C1, 1, st))
    dw2, db2 = torch.empty_like(w2), new(C1)
    L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(d2), L.ptr(d2p), L.ptr(y1), L.ptr(dw2), L.ptr(db2), L.ptr(ws), B, T, F_, C1, C1, prec_w, st))
    d1 = new(B, T, F_, C1)
    L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(d2), L.ptr(w2), L.ptr(y1), L.ptr(d1), None, L.ptr(ws), B, T, F_, C1, C1, prec, st))
    dw0, db0 = torch.empty_like(w0), new(C1)
    L.check(lib.b200asr_conv3x3_c1_bwd_weight(L.ptr(x), L.ptr(d1), L.ptr(dw0), L.ptr(db0), B, F_, T, C1, st))
    return p2, [dw0, db0, dw2, db2, dw5, db5, dw7, db7]


@pytest.mark.parametrize("B,F_,T", [(2, 41, 24), (1, 161, 37), (2, 161, 800)])
@pytest.mark.parametrize("prec", PRECS)
def test_vgg_frontend_same_bits_as_activation_masks(L, B, F_, T, prec):
    """The weight gradients run at 3xTF32 (the default), whose split sums are reproducible bit for bit."""
    prec_w = 3
    import b200asr
    ops = b200asr.ops
    lib = L.load()
    g = _gen(11)
    shapes = [(64, 1, 3, 3), (64,), (64, 64, 3, 3), (64,), (128, 64, 3, 3), (128,), (128, 128, 3, 3), (128,)]
    ws_ = [(torch.randn(s, generator=g) * (0.3 if len(s) == 1 else (s[1] * 9) ** -0.5)).cuda() for s in shapes]
    x = torch.randn(B, 1, F_, T, generator=g).cuda()
    dp2 = torch.randn(B, T // 4, F_ // 4, 128, generator=g).cuda()
    old = (ops.config.conv, ops.config.conv_wgrad)
    ops.config.set(conv=prec, conv_wgrad=prec_w)
    try:
        ps = [w.clone().requires_grad_(True) for w in ws_]
        p2 = ops.VggFrontendFn.apply(x, *ps)
        p2.backward(dp2)
    finally:
        ops.config.set(conv=old[0], conv_wgrad=old[1])
    p2_ref, grads_ref = _frontend_by_activations(lib, L, x, ws_, dp2, prec, prec_w)
    torch.cuda.synchronize()
    assert _eq(p2.detach(), p2_ref)
    for i, (p, r) in enumerate(zip(ps, grads_ref)):
        assert _eq(p.grad, r), i


# ================================================================================================ 4. rejections, launches
def _launches(lib, f):
    n0 = lib.b200asr_launch_count()
    rc = f()
    torch.cuda.synchronize()
    return rc, lib.b200asr_launch_count() - n0


def test_rejections_launch_nothing(L):
    lib = L.load()
    B, T, F_, C = 1, 16, 8, 64
    x1 = torch.randn(B, F_, T, device="cuda")
    x = torch.randn(B, T, F_, C, device="cuda")
    w1, w = torch.randn(C, 1, 3, 3, device="cuda"), torch.randn(C, C, 3, 3, device="cuda")
    b = torch.randn(C, device="cuda")
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(C, C) // 4, device="cuda")
    y = torch.full((B, T, F_, C), NAN, device="cuda")
    raw = torch.zeros(B * T * F_ * C // 32 * 4 + 4, dtype=torch.uint8, device="cuda")
    off = raw[1:].data_ptr()          # 1 byte into an allocation: no uint32 access may use it
    cases = [
        (BAD_ARG, lambda: lib.b200asr_conv3x3_c1_fwd_bits(L.ptr(x1), L.ptr(w1), L.ptr(b), L.ptr(y), B, F_, T, C, 1, None, _st())),
        (BAD_ALIGN, lambda: lib.b200asr_conv3x3_c1_fwd_bits(L.ptr(x1), L.ptr(w1), L.ptr(b), L.ptr(y), B, F_, T, C, 1, off, _st())),
        (BAD_SHAPE, lambda: lib.b200asr_conv3x3_c1_fwd_bits(L.ptr(x1), L.ptr(w1[:16]), L.ptr(b), L.ptr(y), B, F_, T, 16, 1,
                                                            L.ptr(raw), _st())),
    ]
    for prec in PRECS:
        cases += [
            (BAD_ARG, lambda p=prec: lib.b200asr_conv3x3_fwd_bits(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F_, C, C, 1, p,
                                                                  None, _st())),
            (BAD_ALIGN, lambda p=prec: lib.b200asr_conv3x3_fwd_bits(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F_, C, C, 1,
                                                                    p, off, _st())),
            (BAD_ARG, lambda p=prec: lib.b200asr_conv3x3_bwd_data_bits(L.ptr(x), L.ptr(w), None, L.ptr(y), None, L.ptr(ws), B, T, F_, C,
                                                                       C, p, _st())),
            (BAD_ALIGN, lambda p=prec: lib.b200asr_conv3x3_bwd_data_bits(L.ptr(x), L.ptr(w), off, L.ptr(y), None, L.ptr(ws), B, T, F_,
                                                                         C, C, p, _st())),
        ]
    for want, f in cases:
        rc, n = _launches(lib, f)
        assert (rc, n) == (want, 0)
    assert bool(torch.isnan(y).all())


@pytest.mark.parametrize("prec", PRECS)
def test_launch_counts(L, prec):
    """The bit variants launch what the calls they derive from launch; the precision-0 forward adds its ballot pass."""
    lib = L.load()
    B, T, F_, C = 1, 16, 8, 64
    x1 = torch.randn(B, F_, T, device="cuda")
    x = torch.randn(B, T, F_, C, device="cuda")
    w1, w = torch.randn(C, 1, 3, 3, device="cuda"), torch.randn(C, C, 3, 3, device="cuda")
    b = torch.randn(C, device="cuda")
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(C, C) // 4, device="cuda")
    y = torch.empty(B, T, F_, C, device="cuda")
    bits = torch.empty(B, T, F_, C // 32, dtype=torch.int32, device="cuda")
    c1 = _launches(lib, lambda: lib.b200asr_conv3x3_c1_fwd(L.ptr(x1), L.ptr(w1), L.ptr(b), L.ptr(y), B, F_, T, C, 1, _st()))
    c1b = _launches(lib, lambda: lib.b200asr_conv3x3_c1_fwd_bits(L.ptr(x1), L.ptr(w1), L.ptr(b), L.ptr(y), B, F_, T, C, 1, L.ptr(bits),
                                                                 _st()))
    assert c1 == c1b == (OK, 1)
    f = _launches(lib, lambda: lib.b200asr_conv3x3_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F_, C, C, 1, prec, _st()))
    fb = _launches(lib, lambda: lib.b200asr_conv3x3_fwd_bits(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F_, C, C, 1, prec,
                                                             L.ptr(bits), _st()))
    assert f == (OK, 2) and fb == (OK, 3 if prec == 0 else 2)
    d = _launches(lib, lambda: lib.b200asr_conv3x3_bwd_data(L.ptr(x), L.ptr(w), L.ptr(y), L.ptr(y), None, L.ptr(ws), B, T, F_, C, C, prec,
                                                            _st()))
    db = _launches(lib, lambda: lib.b200asr_conv3x3_bwd_data_bits(L.ptr(x), L.ptr(w), L.ptr(bits), L.ptr(y), None, L.ptr(ws), B, T, F_,
                                                                  C, C, prec, _st()))
    assert d == db == (OK, 2)


def test_pool_codes_rejections_and_launches(L):
    lib = L.load()
    B, T, F_, C = 1, 17, 9, 64
    x = torch.randn(B, T, F_, C, device="cuda")
    w, b = torch.randn(C, C, 3, 3, device="cuda"), torch.randn(C, device="cuda")
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(C, C) // 4, device="cuda")
    y, p = torch.empty(B, T, F_, C, device="cuda"), torch.full((B, T // 2, F_ // 2, C), NAN, device="cuda")
    dy, dx = torch.randn(B, T // 2, F_ // 2, C, device="cuda"), torch.full((B, T, F_, C), NAN, device="cuda")
    codes = torch.zeros(B * (T // 2) * (F_ // 2) * C // 8 + 1, dtype=torch.int32, device="cuda")
    off = codes.data_ptr() + 2
    fp = lambda cp, prec=6, co=C: lib.b200asr_conv3x3_fwd_pool_codes(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(p), cp, L.ptr(ws),
                                                                    B, T, F_, C, co, 1, prec, _st())
    bw = lambda cp, c=C: lib.b200asr_maxpool2x2_bwd_codes(L.ptr(dy), cp, L.ptr(dx), None, B, T, F_, c, 1, _st())
    for want, f in [(BAD_ARG, lambda: fp(None)), (BAD_ALIGN, lambda: fp(off)), (BAD_ARG, lambda: bw(None)),
                    (BAD_ALIGN, lambda: bw(off)), (BAD_ARG, lambda: bw(codes.data_ptr(), 4))]:
        assert _launches(lib, f) == (want, 0)
    assert bool(torch.isnan(p).all()) and bool(torch.isnan(dx).all())
    # bf16 modes: weight repack + the convolution with the pooling in its epilogue; otherwise + the stand-alone pooling
    for prec in PRECS:
        assert _launches(lib, lambda: fp(codes.data_ptr(), prec)) == (OK, 2 if prec in (2, 6) else 3)
    assert _launches(lib, lambda: bw(codes.data_ptr())) == (OK, 2)          # + the odd-T / odd-F tail
