"""-m gpu tests of the halo convolution's schedule (tc_conv_halo.cu): the two consumer warpgroups take a CTA's tiles in turn and
hand the mainloop to each other, and in the bf16 modes warps 1-3 split each input patch once into a converted ring.

  * tile counts of 1, 2, 3 and around the SM count (SMs - 1, SMs, SMs + 1, 2 SMs +- 1), so that CTAs end with one tile, an
    odd number of tiles, or warpgroups with unequal numbers of tiles;
  * contraction widths of 32 to 128 channels (one to four patch slices per tile) with T and F off the 16 x 8 tile grid;
  * an utterance's outputs do not depend on which CTA or warpgroup computed them: a B = 1 call equals its rows of a B = 37 call.

Every call runs the fused paths the training step uses: forward with ReLU and the 2 x 2 max-pool epilogue, data gradient with
the ReLU mask and (bf16 modes) the bf16 pairs.  Outputs and scratch are NaN-filled before each call.  Bars as in
test_gpu_tensorcore: 2e-5 for bf16x3 and 3xTF32, 1e-2 for bf16."""
import functools

import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

MODES = [(6, 2e-5), (2, 1e-2), (3, 2e-5)]


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


@functools.lru_cache(maxsize=8)
def _case(B, T, F_, Ci, Co, seed):
    from tests.test_gpu_tensorcore import _conv_case
    import b200asr
    x, w, b, y_ref, dy, dx_ref = _conv_case(b200asr._lib, B, T, F_, Ci, Co, seed=seed)
    mask = torch.randn(B, T, F_, Ci, generator=torch.Generator().manual_seed(seed + 1)).cuda()
    return x, w, b, y_ref, dy, dx_ref, mask


def _run(L, prec, x, w, b, dy, mask, B, T, F_, Ci, Co, fwd=True, dgrad=True):
    """conv3x3_fwd_pool (ReLU) and conv3x3_bwd_data (mask, pairs in the bf16 modes) into NaN-filled buffers."""
    lib = L.load()
    st = _stream()
    y = pooled = dx = dx16 = None
    if fwd:
        ws = _nan(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4)
        y, pooled = _nan(B, T, F_, Co), _nan(B, T // 2, F_ // 2, Co)
        L.check(lib.b200asr_conv3x3_fwd_pool(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(pooled), None, L.ptr(ws), B, T, F_, Ci,
                                             Co, 1, prec, st), "conv+pool")
    if dgrad:
        ws = _nan(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4)
        dx = _nan(B, T, F_, Ci)
        dx16 = _nan(2, B, T, F_, Ci, dtype=torch.bfloat16) if prec in (2, 6) else None
        L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(mask), L.ptr(dx), L.ptr(dx16), L.ptr(ws), B, T, F_, Ci, Co,
                                             prec, st), "conv dgrad")
    torch.cuda.synchronize()
    return y, pooled, dx, dx16


def _check(L, prec, tol, B, T, F_, Ci, Co, seed, fwd=True, dgrad=True):
    x, w, b, y_ref, dy, dx_ref, mask = _case(B, T, F_, Ci, Co, seed)
    y, pooled, dx, dx16 = _run(L, prec, x, w, b, dy, mask, B, T, F_, Ci, Co, fwd, dgrad)
    if fwd:
        assert rel_err(y, y_ref.relu()) < tol
        p_ref = _nan(*pooled.shape)
        L.check(L.load().b200asr_maxpool2x2_fwd(L.ptr(y), L.ptr(p_ref), B, T, F_, Co, _stream()), "pool")
        assert torch.equal(pooled, p_ref)
    if dgrad:
        assert rel_err(dx, dx_ref.cuda() * (mask > 0)) < tol
    if dx16 is not None:
        hi = dx.to(torch.bfloat16)
        assert torch.equal(dx16[0].view(torch.int16), hi.view(torch.int16))
        assert torch.equal(dx16[1].view(torch.int16), (dx - hi.float()).to(torch.bfloat16).view(torch.int16))


@pytest.mark.parametrize("prec,tol", MODES)
@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("sms_times,plus", [(0, 1), (0, 2), (0, 3), (1, -1), (1, 0), (1, 1), (2, -1), (2, 1)])
def test_tile_counts(L, prec, tol, C, sms_times, plus):
    """One 16 x 8 tile per utterance (T = 13, F = 7: both off the grid), B = the tile count = sms_times * SMs + plus: the grid
    is min(tiles, SMs) CTAs, so the counts around the SM count leave some CTAs with one tile and some with two or three."""
    B = sms_times * torch.cuda.get_device_properties(0).multi_processor_count + plus
    _check(L, prec, tol, B, 13, 7, C, C, seed=B)


@pytest.mark.parametrize("prec,tol", MODES)
@pytest.mark.parametrize("Ci,Co", [(32, 64), (96, 128), (64, 32), (128, 96), (64, 128), (128, 64)])
def test_contraction_widths_off_grid(L, prec, tol, Ci, Co):
    """The forward contracts over Ci (output channels Co), the data gradient over Co (output channels Ci): 1 to 4 patch
    slices per tile; each runs where its output width is 64 or 128.  T = 37, F = 21 are off the tile grid in both directions,
    B = 3 gives 27 tiles."""
    _check(L, prec, tol, 3, 37, 21, Ci, Co, seed=Ci + Co, fwd=Co in (64, 128), dgrad=Ci in (64, 128))


@pytest.mark.parametrize("prec,tol", MODES)
@pytest.mark.parametrize("C", [64, 128])
def test_outputs_do_not_depend_on_the_schedule(L, prec, tol, C):
    """B = 37 at T = 40, F = 23 (9 tiles per utterance, 333 in all: every CTA has two or three tiles, on both warpgroups)
    against B = 1 calls of single utterances (9 tiles: one per CTA, all on warpgroup 0): bit-identical rows."""
    B, T, F_ = 37, 40, 23
    x, w, b, _, dy, _, mask = _case(B, T, F_, C, C, seed=5)
    full = _run(L, prec, x, w, b, dy, mask, B, T, F_, C, C)
    for u in (0, 18, 36):
        one = _run(L, prec, x[u:u + 1].contiguous(), w, b, dy[u:u + 1].contiguous(), mask[u:u + 1].contiguous(), 1, T, F_, C, C)
        for name, a, c in zip(("y", "pooled", "dx"), full[:3], one[:3]):
            assert torch.equal(a[u:u + 1].view(torch.int32), c.view(torch.int32)), (name, u)
        if full[3] is not None:
            assert torch.equal(full[3][:, u:u + 1].view(torch.int16), one[3].view(torch.int16)), ("dx16", u)
