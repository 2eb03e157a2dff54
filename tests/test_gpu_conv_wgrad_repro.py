"""-m gpu: the 3xTF32 convolution weight gradient is reproducible bit for bit.

Each CTA reduces its own range of pixel blocks (a split) into a private slot and the slots are summed in a fixed order, so
two calls on the same inputs must return identical weight and bias gradients.  The shapes give many splits and a last split
shorter than the others."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


@pytest.mark.parametrize("B,T,F_,Ci,Co", [(4, 102, 161, 64, 64), (4, 102, 161, 128, 128), (3, 37, 80, 64, 128)])
def test_conv3x3_weight_gradient_is_reproducible(L, B, T, F_, Ci, Co):
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator().manual_seed(B * 1000 + T + Ci)
    x = torch.randn(B, T, F_, Ci, generator=g).cuda()
    dy = torch.randn(B, T, F_, Co, generator=g).cuda()
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    outs = []
    for _ in range(2):
        dw = torch.full((Co, Ci, 3, 3), float("nan"), device="cuda")
        db = torch.full((Co,), float("nan"), device="cuda")
        L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(dy), None, L.ptr(x), L.ptr(dw), L.ptr(db), L.ptr(ws), B, T, F_, Ci, Co, 3, st),
                "conv wgrad")
        outs.append((dw, db))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1])
    nchw = lambda t: t.permute(0, 3, 2, 1).double().cpu()          # [B, T, F, C] -> [B, C, F, T]
    dw_ref = torch.nn.grad.conv2d_weight(nchw(x), (Co, Ci, 3, 3), nchw(dy), padding=1)
    assert rel_err(outs[0][0], dw_ref) < 1e-4
    assert rel_err(outs[0][1], dy.double().sum((0, 1, 2)).cpu()) < 1e-5
