"""The dense-layer GEMMs at precisions 0, 1 and 3, and the spectrogram GEMM, through the raw C ABI against float64:

  A. precision 0 (gemm_simt.cu, fp32 on CUDA cores) against a rigorous elementwise bound instead of a measured bar:
     sequential fp32 FMA over `terms` terms gives |y_hat - y| <= (terms + 4) 2^-24 env, env = the float64 sum of absolute
     values (|x| |w|^T + |b|, + |C| when accumulating), terms = contraction + split count; db: (M + 16) 2^-24 sum |dy|.
     Every instantiation the ABI reaches -- (T, T) forward, (T, F) data gradient, (F, F) weight gradient -- with vector
     and scalar loads (operands one float off the 16-byte grid force scalar loads); M and N at 1, 127, 128, 129, 257, K at
     1, 15, 16, 17 and 4k + {0, 1, 2, 3}; every epilogue (bias or NULL, ReLU, the mask, accumulate); the atomic split-K of
     the weight gradient on both sides of its rule (contraction 1023 / 1024, SMs - 1 / SMs tiles, a partial last split,
     accumulating onto a base); the column sum's two row-slice sizes on integer data, where fp32 sums are exact;
  B. precisions 1 (TF32) and 3 (3xTF32) on the tile engine (tc_gemm.cu): the forward and data-gradient split-K (the bias is
     added by gemm_splitk_reduce_kernel) on both sides of its rule with exact launch counts; the scalar epilogue (N % 4 != 0,
     and bias, relu_out or the output one float off the 16-byte grid); b200asr_split_tf32 bit for bit against a host
     restatement, and pre-split weights giving the same bits as the split inside the kernel;
  C. all five precisions: M = 0, rejections that launch and write nothing, and the launch count of every entry point;
  D. b200asr_stft_features (the only caller whose A rows overlap: row stride hop < K = n_fft) at precisions 0, 1 and 3
     against oracle/features_oracle.collate, which tests/test_features.py pins to torch.stft.

Outputs and caller-owned workspaces are filled with NaN before each call and sit between two bands of a sentinel value
that must come back unchanged.  Inputs are finite.  The float64 references run on the GPU (a reference, not the path
under test).  Bars of precisions 1 and 3 and of the spectrogram are max-norm relative errors (tests.helpers.rel_err) about
3x the largest error measured over this file's cases on one H100 80GB HBM3 at a 700 W power limit; each bar states that
value.  The tests taken over from test_gpu_tensorcore.py keep their bars."""
import math

import numpy as np
import pytest
import torch

from oracle import features_oracle as FO
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

NAN = float("nan")
OK, BAD_SHAPE, BAD_ALIGN, BAD_ARG = 0, -1, -2, -5
FP32, TF32, TF32X3, BF16, BF16X3 = 0, 1, 3, 2, 6
PRECS = [FP32, TF32, TF32X3, BF16, BF16X3]
U = 2.0 ** -24
BAND = 64                       # sentinel floats on each side of an output
SENTINEL = -7.75e33             # no kernel here writes this value


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launches(L):
    return L.load().b200asr_launch_count()


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _cdiv(a, b):
    return -(-a // b)


def _nan(*shape):
    return torch.full(shape, NAN, device="cuda")


class Banded:
    """An output of `shape` inside one allocation, BAND sentinel floats before and after it; `shift` more floats in front
    move it off the 16-byte grid.  Filled with NaN, or with `init`."""

    def __init__(self, shape, init=None, shift=0):
        self.n = math.prod(shape)
        self.lo = BAND + shift
        self.buf = torch.full((self.lo + self.n + BAND,), SENTINEL, device="cuda")
        self.t = self.buf[self.lo:self.lo + self.n].view(shape)
        if init is None:
            self.t.fill_(NAN)
        else:
            self.t.copy_(init)

    def bands_intact(self):
        return bool((self.buf[:self.lo] == SENTINEL).all() and (self.buf[self.lo + self.n:] == SENTINEL).all())


def _placed(t, shift):
    """A device copy of t starting `shift` floats after a 16-byte boundary."""
    buf = torch.empty(t.numel() + 4, device="cuda")
    v = buf[shift:shift + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _check(got, ref, bar, what):
    err = rel_err(got, ref)
    assert err < bar, (what, err)


def _within_bound(got, ref, env, terms, what):
    """|got - ref| <= (terms + 4) 2^-24 env elementwise, and got finite."""
    got = got.detach().double().to(ref.device)
    err = (got - ref).abs()
    bound = (terms + 4) * U * env
    assert bool(torch.isfinite(got).all()), (what, "not finite")
    worst = float((err - bound).max())
    assert worst <= 0.0, (what, worst, float((err / bound.clamp_min(1e-300)).max()))


def _simt_split(M, N, K, sms):
    """gemm_simt's split-K rule (gemm_simt.cu) for C[M, N] over a contraction K, where the caller allows it (the weight
    gradient only) and there is no ReLU or mask: the split count."""
    tiles = _cdiv(M, 128) * _cdiv(N, 128)
    splits = 1
    if K >= 1024 and tiles < sms:
        splits = max(min(_cdiv(2 * sms, tiles), K // 256, 32), 1)
    if splits > 1:
        klen = _cdiv(_cdiv(K, splits), 16) * 16
        splits = _cdiv(K, klen)
    return splits


def _tc_split(M, N, K, sms, relu=False, mask=False):
    """gemm_tc's split-K rule (tc_gemm.cu) for C[M, N] over a contraction K: the split count."""
    tiles = _cdiv(M, 128) * _cdiv(N, 128)
    if relu or mask or K < 1024 or tiles * 2 > sms:
        return 1
    s = min(sms // tiles, K // 256, 16)
    if s <= 1:
        return 1
    klen = _cdiv(_cdiv(K, s), 32) * 32
    return _cdiv(K, klen)


# ================================================================================================ A. precision 0
# (M, N, K): M, N in {1, 127, 128, 129, 257}; K in {1, 15, 16, 17} and 4k + {0, 1, 2, 3}; N or K in {1, 2, 3, 5, 161}
FWD0_SHAPES = [(1, 1, 1), (127, 128, 15), (128, 129, 16), (129, 127, 17), (257, 257, 33), (128, 1, 161), (1, 257, 34),
               (129, 128, 35), (257, 129, 64), (127, 5, 2), (33, 3, 3), (300, 161, 161), (64, 2, 5), (2, 128, 1024)]


@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("M,N,K", FWD0_SHAPES)
def test_fp32_forward_within_bound(L, M, N, K, shift):
    """b200asr_linear_fwd at precision 0 (the (T, T) instantiation; vector loads iff shift = 0 and K % 4 == 0): bias or NULL,
    with and without ReLU, one launch, inside the bound; two calls give identical bits."""
    lib, st = L.load(), _stream()
    g = _gen(M * 7 + N * 3 + K)
    x, w, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * K ** -0.5, torch.randn(N, generator=g)
    xc, wc, bc = _placed(x, shift), _placed(w, shift), _placed(b, shift)
    x64, w64, b64 = xc.double(), wc.double(), bc.double()
    xw, env = x64 @ w64.t(), x64.abs() @ w64.abs().t()
    for bias in (bc, None):
        for relu in (0, 1):
            ys = []
            for _ in range(2):
                y = Banded((M, N), shift=shift)
                n0 = _launches(L)
                L.check(lib.b200asr_linear_fwd(L.ptr(xc), L.ptr(wc), L.ptr(bias), L.ptr(y.t), M, N, K, relu, FP32, None, st), "fwd")
                assert _launches(L) - n0 == 1
                ys.append(y)
            ref = xw + b64 if bias is not None else xw
            _within_bound(ys[0].t, ref.relu() if relu else ref, env + b64.abs() if bias is not None else env, K + 1,
                          ("fwd", bias is not None, relu))
            assert ys[0].bands_intact() and torch.equal(ys[0].t, ys[1].t)


# (M, N, K): dx[M, K] = dy[M, N] w[N, K], contraction N
DGRAD0_SHAPES = [(1, 1, 1), (127, 15, 128), (128, 16, 129), (129, 17, 127), (257, 64, 257), (128, 161, 1), (1, 34, 257),
                 (129, 35, 128), (257, 128, 129), (127, 2, 5), (33, 3, 3), (300, 161, 161), (64, 5, 2), (2, 1024, 128)]


@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("M,N,K", DGRAD0_SHAPES)
def test_fp32_data_gradient_within_bound(L, M, N, K, shift):
    """b200asr_linear_bwd_data at precision 0 (the (T, F) instantiation; vector loads iff shift = 0 and N, K % 4 == 0): with
    the ReLU mask and without it, overwriting and accumulating (the residual link), one launch, inside the bound."""
    lib, st = L.load(), _stream()
    g = _gen(M * 5 + N * 11 + K)
    dy, w = torch.randn(M, N, generator=g), torch.randn(N, K, generator=g) * N ** -0.5
    h, base = torch.randn(M, K, generator=g), torch.randn(M, K, generator=g)
    dyc, wc, hc = _placed(dy, shift), _placed(w, shift), _placed(h, shift)
    dy64, w64, base64 = dyc.double(), wc.double(), base.cuda().double()
    dyw, env = dy64 @ w64, dy64.abs() @ w64.abs()
    for mask in (hc, None):
        for acc in (0, 1):
            dx = Banded((M, K), init=base if acc else None, shift=shift)
            n0 = _launches(L)
            L.check(lib.b200asr_linear_bwd_data(L.ptr(dyc), L.ptr(wc), L.ptr(mask), L.ptr(dx.t), M, N, K, acc, FP32, None, st),
                    "dgrad")
            assert _launches(L) - n0 == 1
            ref = dyw * (hc > 0) if mask is not None else dyw
            _within_bound(dx.t, ref + base64 if acc else ref, env + base64.abs() if acc else env, N + 1,
                          ("dgrad", mask is not None, acc))
            assert dx.bands_intact()


# Dimensions that depend on the GPU's SM count, resolved when the test runs (collection needs no GPU)
SM_DIMS = {"128 (SMs - 1)": lambda s: 128 * (s - 1), "128 SMs": lambda s: 128 * s,
           "128 SMs/2": lambda s: 128 * (s // 2), "128 (SMs/2 + 1)": lambda s: 128 * (s // 2 + 1)}


def _dims(*dims):
    return [SM_DIMS[d](_sms()) if isinstance(d, str) else d for d in dims]


# (M, N, K): dw[N, K] = dy[M, N]^T x[M, K], contraction M (the split rule's K)
WGRAD0_SHAPES = [(1, 1, 1), (127, 128, 129), (128, 257, 127), (129, 1, 257), (257, 129, 128), (5, 161, 161), (300, 3, 2),
                 (1023, 64, 160),               # one short of the contraction the split needs; M % 4 != 0: scalar loads
                 (1024, 64, 160),               # 4 splits of 256
                 (1100, 64, 160),               # 4 splits of 288, the last 236
                 (1025, 5, 3),                  # scalar loads, 4 splits, the last 209
                 (4096, 128, 128),              # 16 splits of 256
                 (1024, 128, "128 (SMs - 1)"),  # SMs - 1 tiles: 3 splits
                 (1024, 128, "128 SMs")]        # SMs tiles: unsplit


@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("M,N,K", WGRAD0_SHAPES)
def test_fp32_weight_gradient_within_bound(L, M, N, K, shift):
    """b200asr_linear_bwd_weight at precision 0 (the (F, F) instantiation; vector loads iff shift = 0, N, K % 4 == 0 and the
    split length % 4 == 0): dw and db overwriting and accumulating onto a base (the flat-gradient sink: the atomic
    split-K adds onto existing values), three launches with db (GEMM, column sums, their reduction), one without; inside the
    bound with terms = M + splits.  Unsplit shapes give identical bits from two calls."""
    lib, st = L.load(), _stream()
    M, N, K = _dims(M, N, K)
    splits = _simt_split(N, K, M, _sms())
    g = _gen(M + 13 * N + 7 * K)
    dy, x = torch.randn(M, N, generator=g), torch.randn(M, K, generator=g)
    wbase, bbase = torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    dyc, xc = _placed(dy, shift), _placed(x, shift)
    dy64, x64, wb64, bb64 = dyc.double(), xc.double(), wbase.cuda().double(), bbase.cuda().double()
    ref, env = dy64.t() @ x64, dy64.abs().t() @ x64.abs()
    dbref, dbenv = dy64.sum(0), dy64.abs().sum(0)
    outs = []
    for acc in (0, 1, 0):
        dw = Banded((N, K), init=wbase if acc else None, shift=shift)
        db = Banded((N,), init=bbase if acc else None, shift=shift)
        n0 = _launches(L)
        L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw.t), L.ptr(db.t), M, N, K, acc, FP32, st), "wgrad")
        assert _launches(L) - n0 == 3
        _within_bound(dw.t, ref + wb64 if acc else ref, env + wb64.abs() if acc else env, M + splits, ("dw", acc, splits))
        _within_bound(db.t, dbref + bb64 if acc else dbref, dbenv + bb64.abs() if acc else dbenv, M + 12, ("db", acc))
        assert dw.bands_intact() and db.bands_intact()
        outs.append((dw.t, db.t))
    assert torch.equal(outs[0][1], outs[2][1])                       # the column sums are ordered
    if splits == 1:
        assert torch.equal(outs[0][0], outs[2][0])
    dw = Banded((N, K), shift=shift)
    n0 = _launches(L)
    L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw.t), None, M, N, K, 0, FP32, st), "wgrad no db")
    assert _launches(L) - n0 == 1
    _within_bound(dw.t, ref, env, M + splits, "dw without db")
    assert dw.bands_intact()


@pytest.mark.parametrize("M", [(1 << 20) - 1, (1 << 20) + 3])
def test_fp32_weight_gradient_long_batch_is_exact(L, M):
    """Both row-slice sizes of the column sum (128 rows below M = 2^20, 2048 from there) and 32 atomic splits, on integer
    data in [-2, 2]: every partial sum is an integer below 2^24, so fp32 is exact in any order and dw, db must equal the
    float64 result exactly, overwriting and accumulating onto an integer base.  A dropped or repeated row shows."""
    lib, st = L.load(), _stream()
    N, K = 8, 4
    assert _simt_split(N, K, M, _sms()) == 32
    g = _gen(M)
    dy = torch.randint(-2, 3, (M, N), generator=g).float().cuda()
    x = torch.randint(-2, 3, (M, K), generator=g).float().cuda()
    wbase = torch.randint(-100, 100, (N, K), generator=g).float()
    bbase = torch.randint(-100, 100, (N,), generator=g).float()
    ref, dbref = dy.double().t() @ x.double(), dy.double().sum(0)
    for acc in (0, 1):
        dw = Banded((N, K), init=wbase if acc else None)
        db = Banded((N,), init=bbase if acc else None)
        L.check(lib.b200asr_linear_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw.t), L.ptr(db.t), M, N, K, acc, FP32, st), "wgrad")
        want_w = ref + wbase.double().cuda() if acc else ref
        want_b = dbref + bbase.double().cuda() if acc else dbref
        assert torch.equal(dw.t.double(), want_w), ("dw", acc)
        assert torch.equal(db.t.double(), want_b), ("db", acc)
        assert dw.bands_intact() and db.bands_intact()


# ================================================================================================ B. precisions 1 and 3
SHAPES = [(128, 128, 32), (128, 128, 128), (256, 384, 512), (300, 512, 512), (77, 52, 164), (6400 // 8, 512, 5120 // 4),
          (130, 4364, 128), (513, 128, 2048), (1, 8, 4), (200, 64, 96)]
# the forward accepts any N at precisions 1 and 3: N % 4 != 0 takes the scalar epilogue
SCALAR_N_SHAPES = [(300, 1, 96), (77, 3, 164), (130, 50, 256), (513, 130, 64)]


@pytest.mark.parametrize("prec,tol", [(1, 2e-3), (3, 2e-5)])
@pytest.mark.parametrize("M,N,K", SHAPES + SCALAR_N_SHAPES)
def test_linear_forward_tensor_core(L, M, N, K, prec, tol):
    """Forward with bias and ReLU (never split) against float64, one launch, sentinel bands intact.  Measured: TF32
    3.7e-4, 3xTF32 1.7e-5 (at K = 1280 with unit-variance weights)."""
    lib = L.load()
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).cuda()
    w = torch.randn(N, K, generator=g).cuda()
    b = torch.randn(N, generator=g).cuda()
    ref = (x.double() @ w.double().t() + b.double()).relu()
    y = Banded((M, N))
    n0 = _launches(L)
    L.check(lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y.t), M, N, K, 1, prec, None, _stream()), "linear_fwd")
    assert _launches(L) - n0 == 1
    _check(y.t, ref, tol, "fwd")
    assert y.bands_intact()


@pytest.mark.parametrize("prec,tol", [(1, 2e-3), (3, 1e-4)])   # 3xTF32: operands exact to ~2^-22; the residual is the
@pytest.mark.parametrize("M,N,K", SHAPES)                      # tensor core's own fp32 accumulation over long K
def test_linear_backward_tensor_core(L, M, N, K, prec, tol):
    """bwd_data exercises an MN-major B operand, bwd_weight MN-major A and B.  Every contraction here is below 1024 rows, so
    the weight gradients run unsplit; the split-K path is tested in test_gpu_default_precision.py.  Measured: TF32 4.0e-4,
    3xTF32 3.3e-5 (the data gradient over N = 4364)."""
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


# bars of the split-K forward / data gradient.  Measured: TF32 2.4e-4 / 3.3e-4, 3xTF32 6.6e-6 / 7.6e-6
SPLIT_BARS = {1: (1e-3, 1e-3), 3: (2e-5, 2.5e-5)}


# (M, N, K): both sides of K >= 1024 (1020 / 1024) and of 2 tiles <= SMs (SMs/2 and SMs/2 + 1 tiles), a partial last split
TC_SPLIT_SHAPES = [(256, 512, 2048), (300, 50, 2048), (300, 52, 1020), (300, 52, 1024), (200, 44, 1100),
                   ("128 SMs/2", 128, 1024), ("128 (SMs/2 + 1)", 128, 1024)]


@pytest.mark.parametrize("prec", [1, 3])
@pytest.mark.parametrize("M,N,K", TC_SPLIT_SHAPES)
def test_linear_tensor_core_split_k(L, M, N, K, prec):
    """Forward without ReLU, with a bias (which gemm_splitk_reduce_kernel adds) and the partial tiles of N = 44 / 50 / 52 on
    the scalar stores; data gradient without mask, overwriting and accumulating (the residual link), contraction N = K
    here (only where N % 4 == 0: N is the row pitch of w).  Launches: 1 unsplit, 2 split, exactly where the host
    restatement of the split rule says."""
    lib, st, sms = L.load(), _stream(), _sms()
    M, N, K = _dims(M, N, K)
    fbar, dbar = SPLIT_BARS[prec]
    g = _gen(M + 3 * N + 5 * K)
    x, w, b = torch.randn(M, K, generator=g).cuda(), (torch.randn(N, K, generator=g) * K ** -0.5).cuda(), torch.randn(N, generator=g).cuda()
    y = Banded((M, N))
    n0 = _launches(L)
    L.check(lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y.t), M, N, K, 0, prec, None, st), "fwd")
    assert _launches(L) - n0 == (2 if _tc_split(M, N, K, sms) > 1 else 1)
    _check(y.t, x.double() @ w.double().t() + b.double(), fbar, "split fwd")
    assert y.bands_intact()
    if N % 4:
        return
    # data gradient with contraction C = K: dy [M, C], w2 [C, N]
    C = K
    dy, w2 = torch.randn(M, C, generator=g).cuda(), (torch.randn(C, N, generator=g) * C ** -0.5).cuda()
    base = torch.randn(M, N, generator=g)
    expect = 2 if _tc_split(M, N, C, sms) > 1 else 1
    for acc in (0, 1):
        dx = Banded((M, N), init=base if acc else None)
        n0 = _launches(L)
        L.check(lib.b200asr_linear_bwd_data(L.ptr(dy), L.ptr(w2), None, L.ptr(dx.t), M, C, N, acc, prec, None, st), "dgrad")
        assert _launches(L) - n0 == expect
        ref = dy.double() @ w2.double()
        _check(dx.t, ref + base.double().cuda() if acc else ref, dbar, ("split dgrad", acc))
        assert dx.bands_intact()


@pytest.mark.parametrize("prec", [1, 3])
@pytest.mark.parametrize("what", ["bias", "y", "relu_out", "dx"])
def test_linear_tensor_core_misaligned_epilogue_operands(L, prec, what):
    """bias, the forward's output, the data gradient's relu_out or its output one float off the 16-byte grid: the GEMM
    operands stay TMA-aligned, the epilogue takes its scalar path, and the result is still right (forward with bias and
    ReLU; data gradient with the mask, overwriting and accumulating).  Measured: TF32 3.3e-4, 3xTF32 1.1e-6."""
    lib, st = L.load(), _stream()
    M, N, K = 200, 136, 96
    bar = 1e-3 if prec == 1 else 4e-6
    g = _gen(17)
    x, w = torch.randn(M, K, generator=g).cuda(), torch.randn(N, K, generator=g).cuda()
    b, dy = torch.randn(N, generator=g), torch.randn(M, N, generator=g).cuda()
    h, base = torch.randn(M, K, generator=g), torch.randn(M, K, generator=g)
    if what in ("bias", "y"):
        bc = _placed(b, 1 if what == "bias" else 0)
        y = Banded((M, N), shift=1 if what == "y" else 0)
        L.check(lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(bc), L.ptr(y.t), M, N, K, 1, prec, None, st), "fwd")
        _check(y.t, (x.double() @ w.double().t() + b.double().cuda()).relu(), bar, what)
        assert y.bands_intact()
        return
    hc = _placed(h, 1 if what == "relu_out" else 0)
    for acc in (0, 1):
        dx = Banded((M, K), init=base if acc else None, shift=1 if what == "dx" else 0)
        L.check(lib.b200asr_linear_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(hc), L.ptr(dx.t), M, N, K, acc, prec, None, st), "dgrad")
        ref = (dy.double() @ w.double()) * (hc > 0)
        _check(dx.t, ref + base.double().cuda() if acc else ref, bar, (what, acc))
        assert dx.bands_intact()


def _tf32_split_host(a):
    """b200asr_split_tf32 restated: hi = (bits + 0x1000) & 0xFFFFE000 (nearest, ties away from zero), lo = x - hi."""
    bits = a.view(np.uint32).astype(np.uint64)
    hi = ((bits + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)
    return hi, (a - hi).astype(np.float32)


@pytest.mark.parametrize("n", [0, 1, 257, 4099])
def test_split_tf32_matches_host_restatement(L, n):
    """Ties (low 13 bits exactly 0x1000, either sign), one below and above them, negatives, subnormals, both zeros, the
    largest values that still round to a finite hi, then random values: hi and lo bit for bit; n = 0 launches nothing."""
    lib = L.load()
    special = [0x00001000, 0x80001000, 0x3F801000, 0xBF801000, 0x3F803000, 0x3F800FFF, 0x3F801001, 0xC1234FFF,
               0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00401000, 0x00000000, 0x80000000, 0x7F7FEFFF, 0xFF7FEFFF,
               0x00800000, 0x3F7FF000]
    rng = np.random.default_rng(n)
    vals = np.concatenate([np.array(special, dtype=np.uint32).view(np.float32),
                           (rng.standard_normal(max(n, 1)) * 10.0 ** rng.integers(-30, 30, max(n, 1))).astype(np.float32)])[:n]
    src = torch.zeros(n + 4, device="cuda")
    src[:n] = torch.from_numpy(vals.copy())
    dst = Banded((2, n))
    n0 = _launches(L)
    # raw addresses: a tensor with no elements has a NULL data_ptr(), and n = 0 still passes valid pointers
    L.check(lib.b200asr_split_tf32(src.data_ptr(), dst.buf.data_ptr() + 4 * dst.lo, n, _stream()), "split_tf32")
    assert _launches(L) - n0 == (1 if n else 0)
    hi, lo = _tf32_split_host(vals)
    got = dst.t.cpu().numpy()
    assert np.array_equal(got[0].view(np.uint32), hi.view(np.uint32))
    assert np.array_equal(got[1].view(np.uint32), lo.view(np.uint32))
    assert dst.bands_intact()


@pytest.mark.parametrize("M,N,K", [(300, 512, 512), (130, 4364, 128), (77, 52, 164), (800, 512, 1280), (257, 132, 96)])
def test_linear_with_presplit_weights(L, M, N, K):
    """3xTF32 GEMM with the weight pre-split once by b200asr_split_tf32 (forward K-major B, data-gradient MN-major B): the
    same bits as the split inside the kernel, which rounds with the same tf32_rn.  N % 128 != 0, and data-gradient
    contractions N % 32 != 0, whose hi half's last k-block reads lo rows against zero-filled A columns; (800, 512, 1280)
    splits K in the forward."""
    lib = L.load()
    g = torch.Generator().manual_seed(5 * M + N)
    x = torch.randn(M, K, generator=g).cuda(); w = torch.randn(N, K, generator=g).cuda(); b = torch.randn(N, generator=g).cuda()
    dy = torch.randn(M, N, generator=g).cuda()
    ws = torch.empty(2, N, K, device="cuda")
    L.check(lib.b200asr_split_tf32(L.ptr(w), L.ptr(ws), N * K, _stream()), "split")
    assert torch.equal(ws[0] + ws[1], w) and float((ws[1].abs() / w.abs().clamp_min(1e-30)).max()) < 2.0 ** -11
    ys, dxs = [], []
    for wsplit in (ws, None):
        y = torch.full((M, N), float("nan"), device="cuda")
        L.check(lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), M, N, K, 0, 3, L.ptr(wsplit), _stream()), "fwd")
        dx = torch.full((M, K), float("nan"), device="cuda")
        L.check(lib.b200asr_linear_bwd_data(L.ptr(dy), L.ptr(w), None, L.ptr(dx), M, N, K, 0, 3, L.ptr(wsplit), _stream()), "dgrad")
        ys.append(y)
        dxs.append(dx)
    assert rel_err(ys[0], x.double() @ w.double().t() + b.double()) < 2e-5
    assert rel_err(dxs[0], dy.double() @ w.double()) < 1e-4
    assert torch.equal(ys[0], ys[1]) and torch.equal(dxs[0], dxs[1])


# ================================================================================================ C. every precision
def _bf16_split(L, w, prec):
    N, K = w.shape
    terms = 2 if prec == BF16X3 else 1
    fwd = torch.empty(terms, N, K, device="cuda", dtype=torch.bfloat16)
    bwd = torch.empty(terms, K, (N + 7) // 8 * 8, device="cuda", dtype=torch.bfloat16)
    L.check(L.load().b200asr_split_bf16(L.ptr(w), L.ptr(fwd), L.ptr(bwd), N, K, terms, _stream()), "split_bf16")
    return fwd, bwd


def _weight_operands(L, w, prec):
    """w_split for the forward and the data gradient at `prec` (NULL where the precision takes none)."""
    if prec in (BF16, BF16X3):
        return _bf16_split(L, w, prec)
    return None, None


def test_empty_batch_at_every_precision(L):
    """M = 0 with valid pointers: the forward and the data gradient return OK and write nothing; the weight gradient sets
    dw and db to 0, or leaves both unchanged when accumulating.  Nothing is launched, at every precision."""
    lib, st = L.load(), _stream()
    N, K = 64, 96
    g = _gen(3)
    x, dy, h = torch.randn(8, K, generator=g).cuda(), torch.randn(8, N, generator=g).cuda(), torch.randn(8, K, generator=g).cuda()
    w, b = torch.randn(N, K, generator=g).cuda(), torch.randn(N, generator=g).cuda()
    wbase, bbase = torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    for prec in PRECS:
        fsplit, bsplit = _weight_operands(L, w, prec)
        y, dx = Banded((4, N)), Banded((4, K))
        n0 = _launches(L)
        assert lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y.t), 0, N, K, 1, prec, L.ptr(fsplit), st) == OK, prec
        for acc in (0, 1):
            assert lib.b200asr_linear_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(h), L.ptr(dx.t), 0, N, K, acc, prec, L.ptr(bsplit),
                                               st) == OK, (prec, acc)
        dw, db = Banded((N, K)), Banded((N,))
        assert lib.b200asr_linear_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw.t), L.ptr(db.t), 0, N, K, 0, prec, st) == OK, prec
        dwa, dba = Banded((N, K), init=wbase), Banded((N,), init=bbase)
        assert lib.b200asr_linear_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dwa.t), L.ptr(dba.t), 0, N, K, 1, prec, st) == OK, prec
        assert _launches(L) == n0, prec
        torch.cuda.synchronize()
        assert bool(y.t.isnan().all() and dx.t.isnan().all()), prec
        assert not dw.t.any() and not db.t.any(), prec
        assert torch.equal(dwa.t.cpu(), wbase) and torch.equal(dba.t.cpu(), bbase), prec
        assert all(o.bands_intact() for o in (y, dx, dw, db, dwa, dba)), prec


def test_rejections_launch_nothing_and_write_nothing(L):
    """Unknown precision, N or K = 0, M < 0 or a NULL pointer -> BAD_ARG; at the tensor-core precisions a K, N or row pitch
    that is not a multiple of 4, or a GEMM operand (or the pre-split weight) one float off the 16-byte grid -> BAD_SHAPE;
    bf16 without w_split, or its forward with K % 8 != 0 -> BAD_SHAPE.  No launch, and every output -- dbias of the fused
    3xTF32 / bf16 bias gradient included -- keeps its NaN and its sentinel bands."""
    lib, st = L.load(), _stream()
    M, N, K = 64, 64, 96
    n = 1 << 16
    x, dy, h, w = (torch.randn(n, device="cuda") for _ in range(4))
    b = torch.randn(4096, device="cuda")
    x_off, dy_off, w_off = _placed(x, 1), _placed(dy, 1), _placed(w, 1)
    wsplit = torch.randn(2 * n, device="cuda")
    wsplit_off = _placed(wsplit, 1)
    y, dx, dw, db = Banded((n,)), Banded((n,)), Banded((n,)), Banded((4096,))
    fwd = lambda X, W, m, nn, k, p, s=None: lib.b200asr_linear_fwd(L.ptr(X), L.ptr(W), L.ptr(b), L.ptr(y.t), m, nn, k, 0, p,
                                                                  L.ptr(s), st)
    dgrad = lambda D, W, m, nn, k, p, s=None: lib.b200asr_linear_bwd_data(L.ptr(D), L.ptr(W), L.ptr(h), L.ptr(dx.t), m, nn, k, 0, p,
                                                                          L.ptr(s), st)
    wgrad = lambda D, X, m, nn, k, p: lib.b200asr_linear_bwd_weight(L.ptr(D), L.ptr(X), L.ptr(dw.t), L.ptr(db.t), m, nn, k, 0, p, st)
    cases = []
    for p in (4, 5, 7, -1):
        cases += [(("fwd prec", p), lambda p=p: fwd(x, w, M, N, K, p), BAD_ARG),
                  (("dgrad prec", p), lambda p=p: dgrad(dy, w, M, N, K, p), BAD_ARG),
                  (("wgrad prec", p), lambda p=p: wgrad(dy, x, M, N, K, p), BAD_ARG)]
    for p in PRECS:
        s = wsplit if p in (BF16, BF16X3) else None
        for what, (m, nn, k) in {"N = 0": (M, 0, K), "K = 0": (M, N, 0), "M < 0": (-1, N, K)}.items():
            cases += [(("fwd", what, p), lambda p=p, m=m, nn=nn, k=k, s=s: fwd(x, w, m, nn, k, p, s), BAD_ARG),
                      (("dgrad", what, p), lambda p=p, m=m, nn=nn, k=k, s=s: dgrad(dy, w, m, nn, k, p, s), BAD_ARG),
                      (("wgrad", what, p), lambda p=p, m=m, nn=nn, k=k: wgrad(dy, x, m, nn, k, p), BAD_ARG)]
        cases += [(("fwd x NULL", p), lambda p=p, s=s: fwd(None, w, M, N, K, p, s), BAD_ARG),
                  (("fwd w NULL", p), lambda p=p, s=s: fwd(x, None, M, N, K, p, s), BAD_ARG),
                  (("dgrad dy NULL", p), lambda p=p, s=s: dgrad(None, w, M, N, K, p, s), BAD_ARG),
                  (("dgrad w NULL", p), lambda p=p, s=s: dgrad(dy, None, M, N, K, p, s), BAD_ARG),
                  (("wgrad dy NULL", p), lambda p=p: wgrad(None, x, M, N, K, p), BAD_ARG),
                  (("wgrad x NULL", p), lambda p=p: wgrad(dy, None, M, N, K, p), BAD_ARG)]
    for p in (TF32, TF32X3):
        cases += [(("fwd K % 4", p), lambda p=p: fwd(x, w, M, N, 97, p), BAD_SHAPE),
                  (("fwd x off", p), lambda p=p: fwd(x_off, w, M, N, K, p), BAD_SHAPE),
                  (("fwd w off", p), lambda p=p: fwd(x, w_off, M, N, K, p), BAD_SHAPE),
                  (("dgrad N % 4", p), lambda p=p: dgrad(dy, w, M, 97, K, p), BAD_SHAPE),
                  (("dgrad K % 4", p), lambda p=p: dgrad(dy, w, M, N, 97, p), BAD_SHAPE),
                  (("dgrad dy off", p), lambda p=p: dgrad(dy_off, w, M, N, K, p), BAD_SHAPE),
                  (("dgrad w off", p), lambda p=p: dgrad(dy, w_off, M, N, K, p), BAD_SHAPE)]
    cases += [("fwd w_split off", lambda: fwd(x, w, M, N, K, TF32X3, wsplit_off), BAD_SHAPE),
              ("dgrad w_split off", lambda: dgrad(dy, w, M, N, K, TF32X3, wsplit_off), BAD_SHAPE)]
    for p in (TF32, TF32X3, BF16, BF16X3):
        cases += [(("wgrad N % 4", p), lambda p=p: wgrad(dy, x, M, 97, K, p), BAD_SHAPE),
                  (("wgrad K % 4", p), lambda p=p: wgrad(dy, x, M, N, 97, p), BAD_SHAPE),
                  (("wgrad dy off", p), lambda p=p: wgrad(dy_off, x, M, N, K, p), BAD_SHAPE),
                  (("wgrad x off", p), lambda p=p: wgrad(dy, x_off, M, N, K, p), BAD_SHAPE)]
    for p in (BF16, BF16X3):
        cases += [(("fwd no w_split", p), lambda p=p: fwd(x, w, M, N, K, p), BAD_SHAPE),
                  (("dgrad no w_split", p), lambda p=p: dgrad(dy, w, M, N, K, p), BAD_SHAPE),
                  (("fwd K % 8", p), lambda p=p: fwd(x, w, M, N, 100, p, wsplit), BAD_SHAPE),
                  (("dgrad N % 4", p), lambda p=p: dgrad(dy, w, M, 98, K, p, wsplit), BAD_SHAPE)]
    for what, call, code in cases:
        n0 = _launches(L)
        assert call() == code, what
        assert _launches(L) == n0, what
    torch.cuda.synchronize()
    for o in (y, dx, dw, db):
        assert bool(o.t.isnan().all()) and o.bands_intact()


def test_launch_counts(L):
    """b200asr_launch_count grows by the kernels each call enqueues, as include/b200asr.h states: forward and data gradient
    1, or 2 when precisions 1 and 3 split the contraction; weight gradient at precision 0: 1 (+ 2 with dbias: column sums
    and their reduction), precision 1: 1 unsplit / 2 split (+ 2 with dbias), precisions 3, 2, 6: 1 / 2, + 1 with dbias when
    split (its partial row sums are reduced).  Both shapes' splits are checked against the host restatements."""
    lib, st, sms = L.load(), _stream(), _sms()
    g = _gen(5)
    # (M, N, K) of the forward / data gradient and of the weight gradient; the second pair splits every contraction
    shapes = {False: ((128, 128, 96), (128, 128, 96)), True: ((256, 1024, 1024), (2048, 128, 256))}
    assert _tc_split(256, 1024, 1024, sms) > 1 and _tc_split(128, 256, 2048, sms) > 1 and _simt_split(128, 256, 2048, sms) > 1
    assert _tc_split(128, 128, 96, sms) == 1 and _simt_split(128, 96, 128, sms) == 1
    for split, ((M, N, K), (Mw, Nw, Kw)) in shapes.items():
        x, w, b = torch.randn(M, K, generator=g).cuda(), (torch.randn(N, K, generator=g) * K ** -0.5).cuda(), torch.randn(N, generator=g).cuda()
        dy = torch.randn(M, N, generator=g).cuda()
        dyw, xw = torch.randn(Mw, Nw, generator=g).cuda(), torch.randn(Mw, Kw, generator=g).cuda()
        for prec in PRECS:
            fsplit, bsplit = _weight_operands(L, w, prec)
            tc = prec in (TF32, TF32X3)
            y, dx, dw, db = _nan(M, N), _nan(M, K), _nan(Nw, Kw), _nan(Nw)
            wg = 2 if split and prec != FP32 else 1
            wg_db = {FP32: 3, TF32: wg + 2}.get(prec, 3 if split else 1)
            calls = [("fwd", lambda: lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), M, N, K, 0, prec, L.ptr(fsplit), st),
                      2 if split and tc else 1),
                     ("dgrad", lambda: lib.b200asr_linear_bwd_data(L.ptr(dy), L.ptr(w), None, L.ptr(dx), M, N, K, 0, prec,
                                                                   L.ptr(bsplit), st), 2 if split and tc else 1),
                     ("wgrad", lambda: lib.b200asr_linear_bwd_weight(L.ptr(dyw), L.ptr(xw), L.ptr(dw), None, Mw, Nw, Kw, 0, prec, st),
                      wg),
                     ("wgrad db", lambda: lib.b200asr_linear_bwd_weight(L.ptr(dyw), L.ptr(xw), L.ptr(dw), L.ptr(db), Mw, Nw, Kw, 0, prec,
                                                                       st), wg_db)]
            for what, call, launches in calls:
                n0 = _launches(L)
                L.check(call(), what)
                assert _launches(L) - n0 == launches, (what, prec, split)
            torch.cuda.synchronize()
            assert all(bool(torch.isfinite(t).all()) for t in (y, dx, dw, db)), prec


# ================================================================================================ D. spectrogram GEMM
GEOMS = [(160, 80), (320, 160), (320, 80), (960, 480), (320, 320)]     # (n_fft, hop): 8 kHz, 16 kHz, hop n_fft/4, 48 kHz, no overlap
# against the oracle, measured over this file's cases: fp32 2.1e-6, TF32 7.9e-4 (the 30 s utterance), 3xTF32 5.6e-6
STFT_BARS = {0: 6e-6, 1: 2.5e-3, 3: 2e-5}
GUARD = 1024


def _waves(lengths, seed):
    g = np.random.default_rng(seed)
    out = []
    for n in lengths:
        t = np.arange(n) / 16000.0
        y = 0.3 * np.sin(2 * np.pi * (200 + 50 * g.random()) * t) + 0.1 * g.standard_normal(n) * (1 + np.sin(2 * np.pi * 3 * t))
        out.append(y.astype(np.float32))
    return out


def _stft_lengths(n_fft, hop):
    """1-3 samples (reflect padding wraps more than once), hop - 1 .. hop + 1, n_fft/2 - 1 .. n_fft/2 + 1, and 31, 32, 33 and
    65 frames (the 32-frame tiles of feat_mag)."""
    half = n_fft // 2
    frames = [hop * 30, hop * 32 - 1, hop * 32, hop * 64 + hop - 1]
    return sorted({1, 2, 3, hop - 1, hop, hop + 1, half - 1, half, half + 1, *frames})


def _stft(L, waves, n_fft, hop, reflect, normalize, prec, Lmax=None, Tmax=None):
    """b200asr_stft_features on a [B, Lmax] batch whose samples past each length are NaN (they must not be read), with a
    NaN workspace of exactly stft_ws_bytes followed by a NaN guard and an output between sentinel bands.  Returns the
    output and the oracle's batch zero padded to Tmax frames."""
    lib = L.load()
    B, lens = len(waves), [len(w) for w in waves]
    Lmax = Lmax or max(lens)
    Tmax = Tmax or 1 + max(lens) // hop
    nb = n_fft // 2 + 1
    wave = torch.full((B, Lmax), NAN)
    for i, w in enumerate(waves):
        wave[i, :len(w)] = torch.from_numpy(w)
    wave, lens_t = wave.cuda(), torch.tensor(lens, dtype=torch.int32, device="cuda")
    nws = lib.b200asr_stft_ws_bytes(B, Lmax, n_fft, hop) // 4
    buf = _nan(nws + GUARD)
    ws, guard = buf[:nws], buf[nws:]
    out = Banded((B, 1, nb, Tmax))
    frames = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    n0 = _launches(L)
    L.check(lib.b200asr_stft_features(L.ptr(wave), L.ptr(lens_t), L.ptr(out.t), L.ptr(frames), L.ptr(ws), B, Lmax, Tmax, n_fft,
                                      hop, reflect, normalize, 0, prec, _stream()), "stft_features")
    assert _launches(L) - n0 == (6 if normalize else 4)          # pad, basis, GEMM, magnitudes (+ statistics, normalisation)
    torch.cuda.synchronize()
    assert bool(guard.isnan().all()) and out.bands_intact()
    assert frames.cpu().tolist() == [1 + n // hop for n in lens]
    want, sizes, _ = FO.collate(waves, n_fft, hop, reflect=bool(reflect), normalize=bool(normalize))
    full = np.zeros((B, 1, nb, Tmax), dtype=np.float32)
    full[..., :want.shape[3]] = want
    return out.t, torch.from_numpy(full)


@pytest.mark.parametrize("prec", [0, 1, 3])
@pytest.mark.parametrize("n_fft,hop", GEOMS)
def test_stft_lengths_and_geometries(L, n_fft, hop, prec):
    """Every edge length in one batch, reflect-padded and normalised, then zero-padded and not normalised."""
    waves = _waves(_stft_lengths(n_fft, hop), seed=n_fft + hop)
    for reflect, normalize in ((1, 1), (0, 0)):
        got, want = _stft(L, waves, n_fft, hop, reflect, normalize, prec)
        _check(got, want, STFT_BARS[prec], ("stft", reflect, normalize))


@pytest.mark.parametrize("prec", [0, 1, 3])
def test_stft_thirty_second_utterance(L, prec):
    """480 000 samples at 320 / 160: 3001 frames, the statistics summed over 94 x 6 = 564 tiles, next to a short one."""
    waves = _waves([480000, 1234], seed=30)
    got, want = _stft(L, waves, 320, 160, 1, 1, prec)
    _check(got, want, STFT_BARS[prec], "stft 30 s")


@pytest.mark.parametrize("prec", [0, 1, 3])
@pytest.mark.parametrize("reflect,normalize", [(1, 0), (0, 1)])
def test_stft_padded_batch(L, prec, reflect, normalize):
    """B = 37 utterances of 4 to 4000 samples in a [37, Lmax] batch with Lmax 777 samples above the longest, and Tmax =
    1 + Lmax/hop, more frames than any utterance has: the columns past each utterance's frames come back 0."""
    lens = np.random.default_rng(37).integers(4, 4001, 37).tolist()
    waves = _waves(lens, seed=37)
    Lmax = max(lens) + 777
    got, want = _stft(L, waves, 320, 160, reflect, normalize, prec, Lmax=Lmax, Tmax=1 + Lmax // 160)
    _check(got, want, STFT_BARS[prec], "stft padded")


def test_stft_rejections(L):
    """n_fft % 32 != 0 (22.05 kHz: n_fft = 441), hop % 4 != 0, hop > n_fft and Tmax > 1 + Lmax/hop -> BAD_SHAPE; ws or out
    one float off the 16-byte grid -> BAD_ALIGN; precision 2, 6 or 4, or a NULL wave -> BAD_ARG.  No launch, nothing
    written.  Tmax = 1 + Lmax/hop, the limit itself, runs."""
    lib, st = L.load(), _stream()
    B, Lmax = 2, 4000
    waves = _waves([4000, 2500], seed=1)
    wave = torch.from_numpy(np.stack([np.pad(w, (0, Lmax - len(w))) for w in waves])).cuda()
    lens = torch.tensor([4000, 2500], dtype=torch.int32, device="cuda")
    ws = _nan(1 << 21)
    ws_off = _placed(ws, 1)
    out, out_off = Banded((B * 161 * 64,)), Banded((B * 161 * 64,), shift=1)

    def call(n_fft=320, hop=160, Tmax=26, prec=3, o=out, w=ws, x=wave):
        return lib.b200asr_stft_features(L.ptr(x), L.ptr(lens), L.ptr(o.t), None, L.ptr(w), B, Lmax, Tmax, n_fft, hop, 1, 1, 0,
                                         prec, st)

    cases = [("n_fft 441", lambda: call(n_fft=441, hop=220), BAD_SHAPE), ("hop % 4", lambda: call(hop=162), BAD_SHAPE),
             ("hop > n_fft", lambda: call(hop=352, Tmax=12), BAD_SHAPE), ("Tmax", lambda: call(Tmax=27), BAD_SHAPE),
             ("ws off", lambda: call(w=ws_off), BAD_ALIGN), ("out off", lambda: call(o=out_off), BAD_ALIGN),
             ("prec 2", lambda: call(prec=2), BAD_ARG), ("prec 6", lambda: call(prec=6), BAD_ARG),
             ("prec 4", lambda: call(prec=4), BAD_ARG), ("wave NULL", lambda: call(x=None), BAD_ARG)]
    for what, fn, code in cases:
        n0 = _launches(L)
        assert fn() == code, what
        assert _launches(L) == n0, what
    torch.cuda.synchronize()
    assert bool(out.t.isnan().all() and out_off.t.isnan().all() and ws.isnan().all() and ws_off.isnan().all())
    assert out.bands_intact() and out_off.bands_intact()
    got, want = _stft(L, waves, 320, 160, 1, 1, 3, Lmax=Lmax, Tmax=1 + Lmax // 160)
    _check(got, want, STFT_BARS[3], "stft at the Tmax limit")
