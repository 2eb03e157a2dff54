"""-m gpu tests of the default arithmetic (ops._Config: bf16x3 = precision 6) and of cfg5's bf16 (precision 2) at kernel level,
against float64 references, plus the code paths every default training step runs that no other test reaches:

  * the bf16 weight-operand conversion (b200asr_split_bf16 / _batched), bit for bit against a host restatement;
  * the linear forward / data gradient / weight gradient in the bf16 modes with every epilogue variant the ops use;
  * split-K weight gradients (partial tiles summed by gemm_splitk_reduce_kernel, fused bias row sums by reduce_parts) at
    every tensor-core precision, guarded by the launch count so that a shape that stops splitting cannot pass unnoticed;
  * the max-pool epilogue of the halo convolution (b200asr_conv3x3_fwd_pool without index bytes);
  * one whole default training step, run twice from the same state: bit-identical loss, gradients and parameters.

Bars are max-norm relative errors (tests.helpers.rel_err); each states the error measured on one H100 80GB HBM3 (700 W limit)."""
import functools

import numpy as np
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

BF16X3, BF16 = 6, 2


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ops():
    import importlib
    import b200asr
    return importlib.import_module(b200asr.__name__ + ".ops")


# ------------------------------------------------------------------------------------------------ A. weight operands
def _split_bf16_host(w: torch.Tensor, terms: int) -> np.ndarray:
    """The kernels' rounding (linear.cu, split_bf16_kernel): add 0x8000 to the bit pattern and keep the top 16 bits (round half
    away from zero); hi of w, lo of w - float(hi).  Returns uint16 [terms][N][K]."""
    x = w.detach().cpu().numpy().astype(np.float32)
    r = x.view(np.uint32) + np.uint32(0x8000)
    hi = (r >> np.uint32(16)).astype(np.uint16)
    lo_f = x - (r & np.uint32(0xFFFF0000)).view(np.float32)
    lo = ((lo_f.view(np.uint32) + np.uint32(0x8000)) >> np.uint32(16)).astype(np.uint16)
    return np.stack([hi, lo][:terms])


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


_SENTINEL = -12345          # an int16 pattern no conversion of these inputs produces where the test looks for it


def _weights_with_ties(N, K, seed):
    """Normal weights in which every third element has its low 16 bits exactly 0x8000 (a rounding tie for hi)."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g)
    u = w.view(torch.int32)
    tie = (torch.arange(N * K).view(N, K) % 3) == 0
    u[tie] = (u[tie] & ~0xFFFF) | 0x8000
    return w


@pytest.mark.parametrize("terms", [1, 2])
@pytest.mark.parametrize("N,K", [(4364, 512), (52, 168), (512, 512), (512, 168), (12, 20)])
def test_split_bf16_layouts_bit_exact(L, N, K, terms):
    """b200asr_split_bf16: dst [terms][N][K] and the transposed dst_t [terms][K][N8] equal the host restatement of the rounding
    bit for bit; the padding columns N..N8-1 of dst_t are written as zeros (pre-filled with a sentinel); each orientation alone
    (the other NULL) gives the same bits.  N % 8 in {0, 4}, K not a multiple of 32, and a matrix smaller than one 32x32 tile."""
    lib = L.load()
    w = _weights_with_ties(N, K, seed=N + K)
    ref = _split_bf16_host(w, terms)
    n8 = (N + 7) // 8 * 8
    wc = w.cuda()
    dst = torch.full((terms, N, K), _SENTINEL, device="cuda", dtype=torch.int16).view(torch.bfloat16)
    dst_t = torch.full((terms, K, n8), _SENTINEL, device="cuda", dtype=torch.int16).view(torch.bfloat16)
    L.check(lib.b200asr_split_bf16(L.ptr(wc), L.ptr(dst), L.ptr(dst_t), N, K, terms, _stream()), "split_bf16")
    got, got_t = _bits(dst), _bits(dst_t)
    assert np.array_equal(got, ref)
    assert np.array_equal(got_t[:, :, :N], ref.transpose(0, 2, 1))
    assert not got_t[:, :, N:].any()
    only = torch.empty_like(dst).view(torch.int16).fill_(_SENTINEL).view(torch.bfloat16)
    only_t = torch.empty_like(dst_t).view(torch.int16).fill_(_SENTINEL).view(torch.bfloat16)
    L.check(lib.b200asr_split_bf16(L.ptr(wc), L.ptr(only), None, N, K, terms, _stream()), "split_bf16 dst")
    L.check(lib.b200asr_split_bf16(L.ptr(wc), None, L.ptr(only_t), N, K, terms, _stream()), "split_bf16 dst_t")
    assert np.array_equal(_bits(only), got) and np.array_equal(_bits(only_t), got_t)


def test_split_bf16_batched_matches_per_matrix_conversion(L):
    """ops.WeightOperandCache on a real FlatParams model: after refresh() (b200asr_split_bf16_batched, one launch over the
    descriptor table and tile prefix) every registered matrix's fwd / bwd operands -- as get() hands them to the GEMMs -- equal
    what b200asr_split_bf16 makes of that matrix, bit for bit, in both term counts; the alignment gaps between the entries
    (pre-filled with a sentinel) are untouched.  The matrices include K = 9 (conv.0 as [64, 9]), N = 52 (vocab) and K = 576."""
    import b200asr
    ops = _ops()
    lib = L.load()
    prev = ops.weight_cache
    try:
        torch.manual_seed(3)
        cfg = b200asr.ASRConfig(num_layers=1, num_heads=2, dim_model=72, dim_key=32, dim_value=32, dim_inner=136, vocab=52,
                                feat_extractor="vgg_cnn", freq=41)
        model = b200asr.build_model(cfg).cuda()
        flat = b200asr.FlatParams(model)
        cache = ops.weight_cache
        assert cache is not None and cache.flat is flat
        mats = [p.detach().view(p.shape[0], -1) for p in flat.params if p.dim() >= 2]
        assert len(mats) >= 10
        for w2 in mats:
            for prec in (BF16X3, BF16):
                ops.split_weight(w2, prec)                    # registers the matrix (served by the per-matrix kernel)
        cache.refresh()                                       # allocates the operand buffer
        assert len(cache.entries) == 2 * len(mats)
        cache.buf.view(torch.int16).fill_(_SENTINEL)
        cache.refresh()
        torch.cuda.synchronize()
        covered = torch.zeros(cache.buf.numel(), dtype=torch.bool)
        for w2 in mats:
            N, K = w2.shape
            n8 = (N + 7) // 8 * 8
            for prec in (BF16X3, BF16):
                terms = 2 if prec == BF16X3 else 1
                _, _, _, _, do, dto = cache.entries[(w2.data_ptr(), N, K, terms)]
                covered[do:do + terms * N * K] = True
                covered[dto:dto + terms * K * n8] = True
                ws = cache.get(w2, prec)
                fwd = torch.empty(terms, N, K, device="cuda", dtype=torch.bfloat16)
                bwd = torch.empty(terms, K, n8, device="cuda", dtype=torch.bfloat16)
                L.check(lib.b200asr_split_bf16(L.ptr(w2), L.ptr(fwd), L.ptr(bwd), N, K, terms, _stream()), "split_bf16")
                assert np.array_equal(_bits(ws.fwd), _bits(fwd)), (N, K, terms)
                assert np.array_equal(_bits(ws.bwd), _bits(bwd)), (N, K, terms)
                assert np.array_equal(_bits(fwd), _split_bf16_host(w2, terms))
        gaps = _bits(cache.buf)[~covered.numpy()]
        assert gaps.size > 0 and (gaps.view(np.int16) == _SENTINEL).all()
    finally:
        ops.weight_cache = prev


# ------------------------------------------------------------------------------------------------ B. linear, bf16 modes
# K % 8 == 0 (the bf16 weight operand's rule); vocab (N8 padding), N % 8 == 4 with K % 32 != 0, M = 1
LIN_SHAPES = [(128, 128, 32), (128, 128, 128), (256, 384, 512), (300, 512, 512), (800, 512, 1280), (130, 4364, 128),
              (513, 128, 2048), (200, 64, 96), (130, 4364, 512), (77, 52, 168), (1, 64, 136), (1, 4364, 512)]
# bars about 3x the maxima measured over these cases on one H100 80GB HBM3 (docstring below)
LIN_BARS = {BF16X3: dict(fwd=3e-5, dgrad=6e-5, wgrad=4e-5), BF16: dict(fwd=1e-2, dgrad=1e-2, wgrad=1e-2)}


def _split(L, w, prec):
    lib = L.load()
    N, K = w.shape
    terms = 2 if prec == BF16X3 else 1
    fwd = torch.empty(terms, N, K, device="cuda", dtype=torch.bfloat16)
    bwd = torch.empty(terms, K, (N + 7) // 8 * 8, device="cuda", dtype=torch.bfloat16)
    L.check(lib.b200asr_split_bf16(L.ptr(w), L.ptr(fwd), L.ptr(bwd), N, K, terms, _stream()), "split_bf16")
    return fwd, bwd


@pytest.mark.parametrize("prec", [BF16X3, BF16])
@pytest.mark.parametrize("M,N,K,relu_x", [s + (False,) for s in LIN_SHAPES] + [(300, 512, 2048, True)])
def test_linear_bf16_modes_against_float64(L, M, N, K, relu_x, prec):
    """b200asr_linear_fwd / _bwd_data / _bwd_weight at precisions 6 and 2 with the weight converted by b200asr_split_bf16, every
    epilogue the ops use: forward with bias and with NULL bias + ReLU; data gradient with the ReLU mask, and accumulating into
    an existing gradient (the residual link); weight gradient overwriting, and accumulating dw AND dbias into a base (the flat
    gradient buffer).  relu_x: post-ReLU activations (about half zeros), as the second FFN GEMM sees.  Measured maxima and
    bars: bf16x3 forward 8.4e-6 (bar 3e-5), data gradient 2.1e-5 (bar 6e-5: the error is the tensor core's fp32 accumulation,
    which grows with the contraction, here up to N = 4364 -- 3xTF32 shows 3.3e-5 there), weight gradient 1.3e-5 (bar 4e-5);
    bf16 3.9e-3 (bar 1e-2); the bias gradient, summed from the fp32 tiles the kernel stages, 3.1e-7 (bar 1e-6)."""
    lib = L.load()
    bars = LIN_BARS[prec]
    g = torch.Generator().manual_seed(M * 7 + N + K + prec)
    x = torch.randn(M, K, generator=g)
    if relu_x:
        x = x.relu()
    w = torch.randn(N, K, generator=g) * K ** -0.5
    b = torch.randn(N, generator=g)
    dy = torch.randn(M, N, generator=g)
    h = torch.randn(M, K, generator=g)
    x64, w64, dy64 = x.double(), w.double(), dy.double()
    xc, wc, bc, dyc, hc = x.cuda(), w.cuda(), b.cuda(), dy.cuda(), h.cuda()
    fwd, bwd = _split(L, wc, prec)
    st = _stream()
    xw = x64 @ w64.t()
    y = torch.full((M, N), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_fwd(L.ptr(xc), L.ptr(wc), L.ptr(bc), L.ptr(y), M, N, K, 0, prec, L.ptr(fwd), st), "fwd")
    assert rel_err(y, xw + b.double()) < bars["fwd"]
    y = torch.full((M, N), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_fwd(L.ptr(xc), L.ptr(wc), None, L.ptr(y), M, N, K, 1, prec, L.ptr(fwd), st), "fwd relu")
    assert rel_err(y, xw.relu()) < bars["fwd"]

    dyw = dy64 @ w64
    dx = torch.full((M, K), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_bwd_data(L.ptr(dyc), L.ptr(wc), L.ptr(hc), L.ptr(dx), M, N, K, 0, prec, L.ptr(bwd), st), "dgrad")
    assert rel_err(dx, dyw * (h > 0)) < bars["dgrad"]
    base = torch.randn(M, K, generator=g)
    dx = base.cuda()
    L.check(lib.b200asr_linear_bwd_data(L.ptr(dyc), L.ptr(wc), None, L.ptr(dx), M, N, K, 1, prec, L.ptr(bwd), st), "dgrad acc")
    assert rel_err(dx, base.double() + dyw) < bars["dgrad"]

    dw_ref, db_ref = dy64.t() @ x64, dy64.sum(0)
    dw = torch.full((N, K), float("nan"), device="cuda")
    db = torch.full((N,), float("nan"), device="cuda")
    L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw), L.ptr(db), M, N, K, 0, prec, st), "wgrad")
    assert rel_err(dw, dw_ref) < bars["wgrad"]
    assert rel_err(db, db_ref) < 1e-6
    wbase, bbase = torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    dw, db = wbase.cuda(), bbase.cuda()
    L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw), L.ptr(db), M, N, K, 1, prec, st), "wgrad acc")
    assert rel_err(dw, wbase.double() + dw_ref) < bars["wgrad"]
    assert rel_err(db, bbase.double() + db_ref) < 1e-6


# ------------------------------------------------------------------------------------------------ C. split-K weight gradients
def _expected_splits(M, N, K, sms):
    """gemm_tc's split rule for dw[N, K] = dy[M, N]^T x[M, K] (tc_gemm.cu): GEMM rows N, columns K, contraction M."""
    tiles = -(-N // 128) * -(-K // 128)
    if M < 1024 or tiles * 2 > sms:
        return 1
    s = min(sms // tiles, M // 256, 16)
    if s <= 1:
        return 1
    klen = -(-(-(-M // s)) // 32) * 32
    return -(-M // klen)


@functools.lru_cache(maxsize=None)
def _wgrad_case(M, N, K):
    g = torch.Generator().manual_seed(M + 3 * N + 5 * K)
    dy = torch.randn(M, N, generator=g)
    x = torch.randn(M, K, generator=g)
    wbase, bbase = torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    return dy, x, wbase, bbase, dy.double().t() @ x.double(), dy.double().sum(0)


# 8 splits on 132 SMs (7 on 114); 12 splits with a last split of 33 rows (a partial k-block); the split count rounds down to 15
# of the 16 requested with a short last split; the cfg2 FFN shape, which splits only where 2 * 64 tiles fit the SMs
SPLIT_SHAPES = [(6400, 512, 512), (3201, 256, 256), (4100, 52, 164), (6400, 2048, 512)]


@pytest.mark.parametrize("prec,tol", [(1, 1e-3), (3, 1e-4), (6, 5e-5), (2, 1e-2)])
@pytest.mark.parametrize("M,N,K", SPLIT_SHAPES)
def test_linear_weight_gradient_split_k(L, M, N, K, prec, tol):
    """b200asr_linear_bwd_weight with a contraction >= 1024 and few output tiles: each split writes its partial tile to the
    stream scratch, gemm_splitk_reduce_kernel sums them in split order (adding to dw when accumulating), and the fused bias
    row sums go through reduce_parts(accumulate=1) (TF32 takes the column-sum kernel instead).  dw and dbias against float64,
    overwriting and accumulating into a random base; two calls return identical bits; and the launch count shows that the
    split path ran: the split kernels add launches over the same call with a 512-row contraction, exactly where the split rule
    for this GPU's SM count says they should.  Measured maxima (132 SMs) and bars: TF32 3.3e-4 (1e-3), 3xTF32 2.5e-5 (1e-4),
    bf16x3 1.3e-5 (5e-5), bf16 2.5e-3 (1e-2), bias 3.6e-7 (1e-6).  The largest errors are the FFN shape's, whose 2 splits
    accumulate 3200 rows each; on a 114-SM part it runs unsplit, twice as long, hence the extra margin at 3xTF32 / bf16x3."""
    lib = L.load()
    st = _stream()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dy, x, wbase, bbase, dw_ref, db_ref = _wgrad_case(M, N, K)
    dyc, xc = dy.cuda(), x.cuda()

    def call(rows, dw, db, acc):
        L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw), L.ptr(db), rows, N, K, acc, prec, st), "wgrad")

    outs = []
    for _ in range(2):
        dw = torch.full((N, K), float("nan"), device="cuda")
        db = torch.full((N,), float("nan"), device="cuda")
        n0 = lib.b200asr_launch_count()
        call(M, dw, db, 0)
        n_split = lib.b200asr_launch_count() - n0
        outs.append((dw, db))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert rel_err(outs[0][0], dw_ref) < tol
    assert rel_err(outs[0][1], db_ref) < 1e-6

    small_dw, small_db = torch.empty(N, K, device="cuda"), torch.empty(N, device="cuda")
    n0 = lib.b200asr_launch_count()
    call(512, small_dw, small_db, 0)
    n_plain = lib.b200asr_launch_count() - n0
    assert _expected_splits(512, N, K, sms) == 1
    splits = _expected_splits(M, N, K, sms)
    assert splits > 1 or (M, N, K) == (6400, 2048, 512)          # only the FFN shape's split depends on the SM count
    if splits > 1:
        assert n_split > n_plain, (n_split, n_plain)
    else:
        assert n_split == n_plain, (n_split, n_plain)

    dw, db = wbase.cuda(), bbase.cuda()
    call(M, dw, db, 1)
    assert rel_err(dw, wbase.double() + dw_ref) < tol
    assert rel_err(db, bbase.double() + db_ref) < 1e-6


# ------------------------------------------------------------------------------------------------ D. fused conv + max-pool
@pytest.mark.parametrize("prec,tol", [(BF16X3, 2e-5), (BF16, 1e-2)])
@pytest.mark.parametrize("B,T,F_,Ci,Co", [(2, 2, 23, 64, 64), (1, 3, 21, 64, 128), (2, 17, 41, 128, 128), (2, 33, 161, 64, 64),
                                          (1, 25, 80, 64, 128), (2, 16, 32, 128, 64)])
def test_conv3x3_pool_in_epilogue(L, B, T, F_, Ci, Co, prec, tol):
    """b200asr_conv3x3_fwd_pool without index bytes in the bf16 modes: the 2x2 maximum is taken in the halo kernel's epilogue by
    lane shuffles over {l, l^1, l^8, l^9} (tc_conv_halo.cu).  `pooled` must equal b200asr_maxpool2x2_fwd of the returned y,
    bit for bit, and y must match float64 (measured <= 6.5e-6 at bf16x3, bar 2e-5; 2.7e-3 at bf16, bar 1e-2).
    With and without the ReLU; odd T / F (floor mode, windows cut by the tile edges) and T = 2, 3 (one pooled row)."""
    from tests.test_gpu_tensorcore import _conv_case
    lib = L.load()
    x, w, b, y_ref, _, _ = _conv_case(L, B, T, F_, Ci, Co, seed=3 * B + T)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    st = _stream()
    for relu in (1, 0):
        y = torch.full((B, T, F_, Co), float("nan"), device="cuda")
        pooled = torch.full((B, T // 2, F_ // 2, Co), float("nan"), device="cuda")
        L.check(lib.b200asr_conv3x3_fwd_pool(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(pooled), None, L.ptr(ws), B, T, F_, Ci, Co,
                                             relu, prec, st), "conv+pool")
        assert rel_err(y, y_ref.relu() if relu else y_ref) < tol, relu
        p_ref = torch.full_like(pooled, float("nan"))
        L.check(lib.b200asr_maxpool2x2_fwd(L.ptr(y), L.ptr(p_ref), B, T, F_, Co, st), "pool")
        assert torch.equal(pooled, p_ref), relu


# ------------------------------------------------------------------------------------------------ E. whole-step reproducibility
def test_default_training_step_is_bit_reproducible(L):
    """Two identical default-precision training steps (forward, label-smoothed loss, backward, Adam through DataParallelStep)
    from the same parameters, optimizer state and dropout seed give identical bits: loss statistics, the flat gradient buffer
    and the updated parameters.  A 1-layer model at cfg2 width (d 512, 8 heads, inner 2048, vocab 4364, VGG front end) with
    dropout 0.1 and B = 8, T = 600: 1200 encoder rows, so the encoder's weight gradients take the split-K path.  The state is
    restored by writing the flat parameter buffer, which the bf16 weight operands must follow (ops.WeightOperandCache)."""
    import dataclasses
    import b200asr
    ops = _ops()
    prev = ops.weight_cache
    try:
        cfg = dataclasses.replace(b200asr.ASRConfig(), num_layers=1, dropout=0.1)
        torch.manual_seed(21)
        model = b200asr.build_model(cfg).cuda().train()
        B, T = 8, 600
        g = torch.Generator().manual_seed(5)
        src = torch.randn(B, 1, cfg.freq, T, generator=g)
        lens = torch.randint(T // 2, T + 1, (B,), generator=g).sort(descending=True).values.to(torch.int32)
        lens[0] = T
        for i in range(B):
            src[i, :, :, int(lens[i]):] = 0
        tgt = torch.randint(3, cfg.vocab, (B, 40), generator=g)
        for i in range(B):
            tgt[i, 12 + 3 * i:] = 0
        src, tgt = src.cuda(), tgt.cuda()
        dp = b200asr.DataParallelStep(model, model_size=cfg.dim_model, warmup=100, smoothing=cfg.label_smoothing)
        p0 = dp.flat.flat.clone()
        rows = cfg.t_enc(T) * B
        assert rows >= 1024 and _expected_splits(rows, 512, 512, torch.cuda.get_device_properties(0).multi_processor_count) > 1

        def step():
            dp.flat.flat.copy_(p0)
            dp.adam.m.zero_(); dp.adam.v.zero_(); dp.adam.t = 0; dp.opt._step = 0
            ops.manual_seed(77)
            dp.step(src, lens, tgt)
            torch.cuda.synchronize()
            return dp.flat.extras.clone(), dp.flat.flat_grad[:dp.flat.numel].clone(), dp.flat.flat.clone()

        first, second = step(), step()
        assert torch.isfinite(first[0]).all() and float(first[0][1]) > 0
        assert float(first[1].abs().max()) > 0 and not torch.equal(first[2], p0)
        for name, a, b in zip(("loss statistics", "gradients", "parameters"), first, second):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), name
    finally:
        ops.weight_cache = prev
