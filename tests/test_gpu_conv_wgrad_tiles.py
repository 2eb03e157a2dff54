"""-m gpu: the halo convolution weight gradient (64-input x 64-output-channel tiles) against float64, at every channel
combination and at the edges of its pixel-block splits.

Outputs and the library's scratch are filled with NaN first, so an unwritten or stale partial shows up.  Each case runs twice
and must give identical bits (fixed-order split reduction, no atomics)."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

TOL = {3: 1e-4, 1: 2e-3}

# (B, T, F, Ci, Co); pixel blocks are 4 (time) x 8 (freq), splits hold at least 32 blocks
CASES = [(1, 13, 21, Ci, Co) for Ci in (64, 128) for Co in (64, 128)] + [
    (2, 9, 19, 64, 64),          # T not a multiple of 4, F not a multiple of 8, 3 x 3 x 2 = 18 blocks: a single split
    (1, 4, 8, 64, 128),          # one pixel block: fewer blocks than stages
    (1, 8, 16, 128, 64),         # four pixel blocks
    (1, 33, 65, 64, 64),         # 9 x 9 = 81 blocks: three splits, the last one 17 blocks
    (3, 37, 80, 128, 128),       # 3 x 10 x 10 = 300 blocks: ten splits of 32, the last one 12 blocks
    (4, 102, 161, 64, 64),       # cfg2 conv2 at B = 4
    (4, 50, 80, 64, 128),        # cfg2 conv3 at B = 4
    (4, 50, 80, 128, 128),       # cfg2 conv4 at B = 4
]


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _run(L, x, dy, Ci, Co, prec, with_bias):
    lib = L.load()
    B, T, F_ = x.shape[:3]
    st = torch.cuda.current_stream().cuda_stream
    ws = torch.full((lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4,), float("nan"), device="cuda")
    dw = torch.full((Co, Ci, 3, 3), float("nan"), device="cuda")
    db = torch.full((Co,), float("nan"), device="cuda") if with_bias else None
    L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(dy), None, L.ptr(x), L.ptr(dw), L.ptr(db) if with_bias else None, L.ptr(ws),
                                           B, T, F_, Ci, Co, prec, st), "conv wgrad")
    torch.cuda.synchronize()
    return dw, db


@pytest.mark.parametrize("with_bias", [True, False])
@pytest.mark.parametrize("prec", [3, 1])
@pytest.mark.parametrize("B,T,F_,Ci,Co", CASES)
def test_conv3x3_weight_gradient_tiles(L, B, T, F_, Ci, Co, prec, with_bias):
    g = torch.Generator().manual_seed(B * 1000 + T * 10 + F_ + Ci + Co)
    x = torch.randn(B, T, F_, Ci, generator=g).cuda()
    dy = torch.randn(B, T, F_, Co, generator=g).cuda()
    dw, db = _run(L, x, dy, Ci, Co, prec, with_bias)
    dw2, db2 = _run(L, x, dy, Ci, Co, prec, with_bias)
    assert torch.equal(dw, dw2)
    nchw = lambda t: t.permute(0, 3, 2, 1).double().cpu()          # [B, T, F, C] -> [B, C, F, T]
    dw_ref = torch.nn.grad.conv2d_weight(nchw(x), (Co, Ci, 3, 3), nchw(dy), padding=1)
    assert not torch.isnan(dw).any()
    assert rel_err(dw, dw_ref) < TOL[prec]
    if with_bias:
        assert torch.equal(db, db2)
        assert rel_err(db, dy.double().sum((0, 1, 2)).cpu()) < 1e-5
