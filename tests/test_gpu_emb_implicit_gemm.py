"""The emb_cnn implicit-GEMM convolutions (tc_emb.cu) through the raw C ABI, against float64 references, at every
instantiation and at the edges of their index arithmetic:

  1. the 32 -> 32 layer, conv2d_tc_fwd / _bwd_data (EmbConvPolicy<false / true> at precisions 3, 6 and 2) and
     conv2d_tc_bwd_weight (EmbWgradPolicy, 3xTF32, + the bias gradient): the reference geometry (21 x 11, stride (2, 1),
     H = 61); OW in {1, 31, 32, 127, 128, 129, 257} with every residue of W mod 4 (the four shifted copies); KW in
     {1, 3, 4, 5, 8, 11, 12, 13} (0-3 padded taps in the last weight-gradient tile, read at channel coordinate 32);
     KH = 1; SH in {1, 2, 3} with SH > KH and (H - KH) % SH != 0, where data-gradient rows no tap reaches are tiles with
     zero k-blocks and come back exactly 0; row pitches round4(width) and round4(width) + 60 with NaN pad columns that
     stay NaN; the forward with bias NULL;
  2. the 1 -> 32 layer, conv2d_c1_tc_fwd (Emb1ConvPolicy, precisions 3, 6, 2) and conv2d_c1_tc_bwd_weight
     (Emb1WgradPolicy): KH in {1, 31, 32, 33, 41, 64} (one or two 32-deep kh blocks of the overlapping view, exact fill at
     32 and 64, padded taps at kh coordinate 64), KW in {1, 4, 11, 12}, PW in {0, 1, 10, 15} (PW > KW: whole windows in
     the padding give exactly the bias), odd and even W (the parity copies), OW in {1, 18, 25, 30, 34, 35, 72, 128, 129,
     205}; the forward at y_pitch = OW (what ops.EmbFrontendFn passes) and at OW + 5, the weight gradient at round4(OW)
     and round4(OW) + 60;
  3. the persistent schedule: forward and data-gradient tile counts of 1, SMs, SMs + 1 and 2 SMs + 1; a batch of SMs + 1
     images bit-identical to each image computed alone; weight gradients over B*OH in {1, 7, 8, 9, 257} rows (one row
     split, the 8-row minimum, two splits, the bias gradient's second 256-row sweep) and OW % 32 in {0, 1, 31}, with and
     without dbias, two calls giving identical bits;
  4. the production batch: the exact argument lists of ops.EmbFrontendFn at cfg3 (B = 64, x [64, 1, 161, 400]), all five
     entry points, at the package's default precision and at 3xTF32, against float64 on the GPU;
  5. the workspace: forward, data gradient and weight gradient on one buffer of exactly *_ws_bytes followed by a NaN
     guard that stays untouched;
  6. rejections (BAD_SHAPE, BAD_ARG, BAD_ALIGN) launch nothing and write nothing; every entry point's launch count.

Outputs and the workspaces the caller owns are filled with NaN before each call, so an element a kernel fails to write
shows up.  Inputs are finite.  Bars are max-norm relative errors (tests.helpers.rel_err); each states the largest error
measured over this file's cases on one H100 80GB HBM3 (400 W power limit).  Small references run in float64 on the CPU, large
ones in float64 on the GPU (a reference, not the path under test)."""
import functools

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

NAN = float("nan")
OK, BAD_SHAPE, BAD_ALIGN, BAD_ARG = 0, -1, -2, -5
PRECS = [3, 6, 2]                  # 3xTF32, bf16x3, bf16
EC = 32

# The bars of the tests this file took over, kept.  Measured maxima over every case here, B = 64 included:
#   32 -> 32 forward / data gradient: 3xTF32 5.4e-5 / 2.9e-5, bf16x3 2.5e-5 / 1.6e-5 (both at the reference geometry, whose
#   contraction is 32 x 21 x 11 = 7392 terms), bf16 2.9e-3 / 3.6e-3;
#   first-layer forward: 3xTF32 4.0e-6, bf16x3 8.0e-6, bf16 3.1e-3
FWD_BAR = {3: 1e-4, 6: 3e-5, 2: 1e-2}
C1_FWD_BAR = {3: 3e-5, 6: 3e-5, 2: 1e-2}
# weight gradients (3xTF32, partials summed in split order) up to B = 3: measured 1.2e-5 (32 -> 32, H = 61), 1.3e-5 (first
# layer, H = 161, W = 400); the bias gradients (fp32 sums in a fixed order), B = 64 included: 2.4e-7
WGRAD_BAR = 1e-4
C1_WGRAD_BAR = 3e-5
BIAS_BAR = 1e-5
# The weight gradients at cfg3's B = 64.  Their error grows linearly with the output pixels one row split accumulates
# (on 132 SMs): 32 -> 32, 1792 pixels per split at B = 1 (1.2e-5), 50176 at B = 64: measured 3.2e-4; first layer, 1792
# at B = 2 (1.3e-5), 13440 at B = 64: measured 9.6e-5.  Bars about 3x above.
PROD_WGRAD_BAR = 1e-3
PROD_C1_WGRAD_BAR = 3e-4


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
    """n NaN floats starting 4 bytes into a fresh allocation: a view no TMA box may start from."""
    return torch.full((n + 4,), NAN, device="cuda")[1:n + 1]


def _all_nan(t):
    return bool(torch.isnan(t).all())


def _r4(v):
    return (v + 3) // 4 * 4


def _pitched(t, pitch):
    """t [..., w] -> a [..., pitch] tensor on the GPU holding t in its first w columns and NaN in the rest."""
    out = torch.full((*t.shape[:-1], pitch), NAN, device="cuda")
    out[..., :t.shape[-1]] = t.to("cuda")
    return out


def _launches(L):
    return L.load().b200asr_launch_count()


def _check(got, ref, bar, what):
    err = rel_err(got, ref)
    assert err < bar, (what, err)


# 32 -> 32 layer: geom = (B, Ci, H, W, Co, KH, KW, SH, x_pitch, y_pitch)
def _fwd(L, x, w, b, y, ws, geom, prec):
    return L.load().b200asr_conv2d_tc_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), *geom, prec, _stream())


def _dgrad(L, dy, w, dx, ws, geom, prec):
    return L.load().b200asr_conv2d_tc_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(dx), L.ptr(ws), *geom, prec, _stream())


def _wgrad(L, dy, x, dw, db, ws, geom):
    return L.load().b200asr_conv2d_tc_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw), L.ptr(db), L.ptr(ws), *geom, _stream())


def _ws(L, B, H, W, KH, KW):
    return _nan(L.load().b200asr_conv2d_tc_ws_bytes(B, H, W, KH, KW) // 4)


# first layer: geom = (B, H, W, Co, KH, KW, PW, y_pitch)
def _c1_fwd(L, x, w, b, y, ws, geom, prec):
    return L.load().b200asr_conv2d_c1_tc_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), *geom, prec, _stream())


def _c1_wgrad(L, dy, x, dw, db, ws, geom):
    return L.load().b200asr_conv2d_c1_tc_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw), L.ptr(db), L.ptr(ws), *geom, _stream())


def _c1_ws(L, B, H, W, KH, KW):
    return _nan(L.load().b200asr_conv2d_c1_tc_ws_bytes(B, H, W, KH, KW) // 4)


# ================================================================================================ float64 references
def _ref_device(macs):
    return "cuda" if macs > 5e7 else "cpu"


def emb2_ref(B, H, W, KH, KW, SH, seed):
    """Inputs and float64 results of Conv2d(32, 32, (KH, KW), stride (SH, 1)): x, w, b, dy and y (without bias), dx, dw,
    db, all on the CPU; `reach` [H]: the rows of x some tap reads."""
    OH, OW = (H - KH) // SH + 1, W - KW + 1
    g = _gen(seed)
    x = torch.randn(B, EC, H, W, generator=g)
    w = torch.randn(EC, EC, KH, KW, generator=g) * (EC * KH * KW) ** -0.5
    b = torch.randn(EC, generator=g)
    dy = torch.randn(B, EC, OH, OW, generator=g)
    dev = _ref_device(B * OH * OW * EC * EC * KH * KW)
    x64, w64 = (t.to(dev).double().requires_grad_(True) for t in (x, w))
    y64 = F.conv2d(x64, w64, stride=(SH, 1))
    y64.backward(dy.to(dev).double())
    reach = torch.zeros(H, dtype=torch.bool)
    for oh in range(OH):
        reach[SH * oh:SH * oh + KH] = True
    return dict(x=x, w=w, b=b, dy=dy, y=y64.detach().cpu(), dx=x64.grad.cpu(), dw=w64.grad.cpu(),
                db=dy.double().sum((0, 2, 3)), reach=reach)


def emb1_ref(B, H, W, KH, KW, PW, seed):
    """The same for Conv2d(1, 32, (KH, KW), stride 2, padding (0, PW)); `seen` [OH, OW]: outputs whose window reads at
    least one input element (the others are exactly the bias)."""
    OH, OW = (H - KH) // 2 + 1, (W + 2 * PW - KW) // 2 + 1
    g = _gen(seed)
    x = torch.randn(B, 1, H, W, generator=g)
    w = torch.randn(EC, 1, KH, KW, generator=g) * (KH * KW) ** -0.5
    b = torch.randn(EC, generator=g)
    dy = torch.randn(B, EC, OH, OW, generator=g)
    dev = _ref_device(B * OH * OW * EC * KH * KW)
    w64 = w.to(dev).double().requires_grad_(True)
    y64 = F.conv2d(x.to(dev).double(), w64, stride=2, padding=(0, PW))
    y64.backward(dy.to(dev).double())
    seen = F.conv2d(torch.ones(1, 1, H, W, dtype=torch.float64), torch.ones(1, 1, KH, KW, dtype=torch.float64), stride=2,
                    padding=(0, PW))[0, 0] > 0
    return dict(x=x, w=w, b=b, dy=dy, y=y64.detach().cpu(), dw=w64.grad.cpu(), db=dy.double().sum((0, 2, 3)), seen=seen)


# ================================================================================================ 1. the 32 -> 32 layer
# (B, H, W, KH, KW, SH, pad): pitches round4(W) + pad and round4(OW) + pad.  OW = W - KW + 1, OH = (H - KH) // SH + 1.
EMB2 = {
    "ref_h61": (1, 61, 205, 21, 11, 2, 0),            # cfg3's layer at H1 = 61, W1 = 205: OH = 21, OW = 195
    "ref_w45": (2, 61, 45, 21, 11, 2, 60),
    "ref_h30": (1, 30, 205, 21, 11, 2, 0),            # OH = 5
    "kh5_sh1_kw3": (3, 25, 140, 5, 3, 1, 0),
    "ref_w131": (2, 23, 131, 21, 11, 2, 60),          # OH = 2
    "ow1_kw4": (2, 9, 4, 3, 4, 1, 60),                # W % 4 = 0
    "ow1_kw13_kh1_sh3": (2, 5, 13, 1, 13, 3, 0),      # W % 4 = 1; SH > KH: rows 1, 2 and the trailing row 4 get no tap
    "ow31_kw8_kh2_sh3": (2, 12, 38, 2, 8, 3, 0),      # W % 4 = 2; SH > KH, (H - KH) % SH = 1
    "ow31_kw1_kh1_sh3": (1, 9, 31, 1, 1, 3, 60),      # W % 4 = 3; KW = 1: three padded taps; (H - KH) % SH = 2
    "ow32_kw5_sh2": (3, 24, 36, 21, 5, 2, 60),        # (H - KH) % SH = 1: trailing row 23
    "ow127_kw1_kh1": (2, 3, 127, 1, 1, 1, 0),
    "ow127_kw4_sh3": (2, 15, 130, 5, 4, 3, 0),        # W % 4 = 2; (H - KH) % SH = 1
    "ow128_kw8_sh3": (2, 10, 135, 4, 8, 3, 60),
    "ow129_kw12_sh3": (1, 14, 140, 5, 12, 3, 0),
    "ow257_kw13": (1, 7, 269, 3, 13, 2, 60),          # three 128-wide tiles per row, the last with one column
}


@functools.lru_cache(maxsize=None)
def _emb2_case(name):
    B, H, W, KH, KW, SH, _ = EMB2[name]
    return emb2_ref(B, H, W, KH, KW, SH, seed=list(EMB2).index(name) + 1)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", list(EMB2))
def test_conv2d_implicit_gemm_32ch(L, name, prec):
    """Forward (with bias and with bias NULL) and data gradient at every precision, weight and bias gradient at 3xTF32,
    on row-pitched tensors whose pad columns are NaN: the outputs' pads stay NaN, nothing reads the inputs' pads, and
    data-gradient rows no tap reaches are exactly 0."""
    B, H, W, KH, KW, SH, pad = EMB2[name]
    c = _emb2_case(name)
    OH, OW = c["y"].shape[2:]
    xp, yp = _r4(W) + pad, _r4(OW) + pad
    geom = (B, EC, H, W, EC, KH, KW, SH, xp, yp)
    x, dy, w, b = _pitched(c["x"], xp), _pitched(c["dy"], yp), c["w"].cuda(), c["b"].cuda()
    ws = _ws(L, B, H, W, KH, KW)
    for bias in (b, None):
        y = _nan(B, EC, OH, yp)
        L.check(_fwd(L, x, w, bias, y, ws, geom, prec), "conv2d_tc_fwd")
        ref = c["y"] + (0.0 if bias is None else c["b"].double()[:, None, None])
        _check(y[..., :OW], ref, FWD_BAR[prec], ("fwd", bias is None))
        assert _all_nan(y[..., OW:])
    dx = _nan(B, EC, H, xp)
    L.check(_dgrad(L, dy, w, dx, ws, geom, prec), "conv2d_tc_bwd_data")
    _check(dx[..., :W], c["dx"], FWD_BAR[prec], "dgrad")
    assert _all_nan(dx[..., W:])
    assert bool((dx[..., :W].cpu()[:, :, ~c["reach"]] == 0).all())
    if prec == 3:
        dw, db = _nan(EC, EC, KH, KW), _nan(EC)
        L.check(_wgrad(L, dy, x, dw, db, ws, geom), "conv2d_tc_bwd_weight")
        _check(dw, c["dw"], WGRAD_BAR, "dw")
        _check(db, c["db"], BIAS_BAR, "db")


# ================================================================================================ 2. the first layer
# (B, H, W, KH, KW, PW): OH = (H - KH) // 2 + 1, OW = (W + 2 PW - KW) // 2 + 1
EMB1 = {
    "ref_w400": (2, 161, 400, 41, 11, 10),            # cfg3's layer: OH = 61, OW = 205
    "ref_w133": (1, 75, 133, 41, 11, 10),             # OW = 72
    "ref_w50": (3, 41, 50, 41, 11, 10),               # OH = 1, OW = 30
    "kh1_kw4_pw1": (2, 9, 37, 1, 4, 1),               # OW = 18
    "kh31": (2, 40, 60, 31, 11, 10),                  # OW = 35
    "kh32_ow128": (1, 35, 266, 32, 12, 0),            # one exactly full kh block
    "kh33_ow129": (2, 33, 255, 33, 1, 1),             # a second kh block with one tap; KW = 1: three padded taps
    "kh64_pw15": (1, 70, 41, 64, 4, 15),              # two full kh blocks; PW > KW; OW = 34
    "ow1_kw12": (2, 45, 12, 41, 12, 0),
    "kw1_pw15": (2, 50, 20, 32, 1, 15),               # OW = 25, outputs 0-7 and 18-24 read only padding
    "ow128_odd_w": (1, 45, 245, 41, 11, 10),
    "ow129_even_w": (1, 43, 258, 41, 4, 1),
}


@functools.lru_cache(maxsize=None)
def _emb1_case(name):
    return emb1_ref(*EMB1[name], seed=100 + list(EMB1).index(name))


@pytest.mark.parametrize("pitch", ["ops", "padded"])
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", list(EMB1))
def test_conv2d_first_layer_implicit_gemm(L, name, prec, pitch):
    """Forward with bias and with bias NULL at every precision, at y_pitch = OW ("ops": what ops.EmbFrontendFn passes, not
    a multiple of 4) or OW + 5 with a NaN pad that stays NaN ("padded"); outputs whose window lies in the padding are
    exactly the bias.  The weight and bias gradient (3xTF32) at y_pitch = round4(OW) or round4(OW) + 60, dy's pad NaN."""
    B, H, W, KH, KW, PW = EMB1[name]
    c = _emb1_case(name)
    OH, OW = c["y"].shape[2:]
    x, w, b = c["x"].cuda(), c["w"].cuda(), c["b"].cuda()
    ws = _c1_ws(L, B, H, W, KH, KW)
    yp = OW if pitch == "ops" else OW + 5
    for bias in (b, None):
        y = _nan(B, EC, OH, yp)
        L.check(_c1_fwd(L, x, w, bias, y, ws, (B, H, W, EC, KH, KW, PW, yp), prec), "conv2d_c1_tc_fwd")
        ref = c["y"] + (0.0 if bias is None else c["b"].double()[:, None, None])
        _check(y[..., :OW], ref, C1_FWD_BAR[prec], ("fwd", bias is None))
        assert _all_nan(y[..., OW:])
        unseen = y[..., :OW].cpu()[:, :, ~c["seen"]]
        expect = torch.zeros(EC) if bias is None else c["b"]
        assert torch.equal(unseen, expect[None, :, None].expand_as(unseen))
    if prec == 3:
        yp = _r4(OW) + (0 if pitch == "ops" else 60)
        dy, dw, db = _pitched(c["dy"], yp), _nan(EC, 1, KH, KW), _nan(EC)
        L.check(_c1_wgrad(L, dy, x, dw, db, ws, (B, H, W, EC, KH, KW, PW, yp)), "conv2d_c1_tc_bwd_weight")
        _check(dw, c["dw"], C1_WGRAD_BAR, "dw")
        _check(db, c["db"], BIAS_BAR, "db")


# ================================================================================================ 3. the persistent schedule
def _tile_count(case):
    s = _sms()
    return {"1": 1, "sms": s, "sms+1": s + 1, "2sms+1": 2 * s + 1}[case]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("tiles", ["1", "sms", "sms+1", "2sms+1"])
def test_tile_counts_around_the_sm_count(L, tiles, prec):
    """The engine launches min(tiles, SMs) CTAs that stride over the tiles: one round, one round on every SM, a second
    round with one tile, a third round with one tile.  With OH = 1 (H = KH) and OW <= 128 each image is one forward tile,
    and with H = 1 one data-gradient tile, so B sets the tile count exactly."""
    B = _tile_count(tiles)
    c = emb2_ref(B, 1, 40, 1, 5, 1, seed=B)                   # OW = 36
    geom = (B, EC, 1, 40, EC, 1, 5, 1, 40, 36)
    x, dy, w, b = c["x"].cuda(), c["dy"].cuda(), c["w"].cuda(), c["b"].cuda()
    ws = _ws(L, B, 1, 40, 1, 5)
    y, dx = _nan(B, EC, 1, 36), _nan(B, EC, 1, 40)
    L.check(_fwd(L, x, w, b, y, ws, geom, prec), "conv2d_tc_fwd")
    _check(y, c["y"] + c["b"].double()[:, None, None], FWD_BAR[prec], "fwd")
    L.check(_dgrad(L, dy, w, dx, ws, geom, prec), "conv2d_tc_bwd_data")
    _check(dx, c["dx"], FWD_BAR[prec], "dgrad")

    c = emb1_ref(B, 41, 50, 41, 11, 10, seed=B)               # OH = 1, OW = 30
    y = _nan(B, EC, 1, 30)
    L.check(_c1_fwd(L, c["x"].cuda(), c["w"].cuda(), c["b"].cuda(), y, _c1_ws(L, B, 41, 50, 41, 11),
                    (B, 41, 50, EC, 41, 11, 10, 30), prec), "conv2d_c1_tc_fwd")
    _check(y, c["y"] + c["b"].double()[:, None, None], C1_FWD_BAR[prec], "c1 fwd")


@pytest.mark.parametrize("prec", PRECS)
def test_batch_equals_each_image_alone(L, prec):
    """A batch of SMs + 1 images -- 22 forward and 50 data-gradient tiles per image of the 32 -> 32 layer, 3 forward tiles
    per image of the first layer -- gives the same bits as each image computed alone, where its tiles run on other CTAs
    and in another round."""
    B = _sms() + 1
    g = _gen(prec)
    H, W, KH, KW, SH = 25, 140, 5, 3, 2                       # OH = 11, OW = 138: two 128-wide tiles per row
    OH, OW, xp, yp = 11, 138, 140, 140
    x = torch.randn(B, EC, H, xp, generator=g).cuda()
    dy = torch.randn(B, EC, OH, yp, generator=g).cuda()
    w = (torch.randn(EC, EC, KH, KW, generator=g) * (EC * KH * KW) ** -0.5).cuda()
    b = torch.randn(EC, generator=g).cuda()
    y, dx = _nan(B, EC, OH, yp), _nan(B, EC, H, xp)
    L.check(_fwd(L, x, w, b, y, _ws(L, B, H, W, KH, KW), (B, EC, H, W, EC, KH, KW, SH, xp, yp), prec), "conv2d_tc_fwd")
    L.check(_dgrad(L, dy, w, dx, _ws(L, B, H, W, KH, KW), (B, EC, H, W, EC, KH, KW, SH, xp, yp), prec), "conv2d_tc_bwd_data")
    H1, W1, KH1, KW1, PW = 45, 50, 41, 11, 10                 # OH = 3, OW = 30
    x1 = torch.randn(B, 1, H1, W1, generator=g).cuda()
    w1 = (torch.randn(EC, 1, KH1, KW1, generator=g) * (KH1 * KW1) ** -0.5).cuda()
    y1 = _nan(B, EC, 3, 30)
    L.check(_c1_fwd(L, x1, w1, b, y1, _c1_ws(L, B, H1, W1, KH1, KW1), (B, H1, W1, EC, KH1, KW1, PW, 30), prec), "c1_fwd")
    ws, ws1 = _ws(L, 1, H, W, KH, KW), _c1_ws(L, 1, H1, W1, KH1, KW1)
    one, one1 = (1, EC, H, W, EC, KH, KW, SH, xp, yp), (1, H1, W1, EC, KH1, KW1, PW, 30)
    for i in range(B):
        yi, dxi, y1i = _nan(1, EC, OH, yp), _nan(1, EC, H, xp), _nan(1, EC, 3, 30)
        L.check(_fwd(L, x[i:i + 1], w, b, yi, ws, one, prec), "conv2d_tc_fwd")
        L.check(_dgrad(L, dy[i:i + 1], w, dxi, ws, one, prec), "conv2d_tc_bwd_data")
        L.check(_c1_fwd(L, x1[i:i + 1], w1, b, y1i, ws1, one1, prec), "conv2d_c1_tc_fwd")
        assert torch.equal(yi[..., :OW], y[i:i + 1, ..., :OW]), i
        assert torch.equal(dxi[..., :W], dx[i:i + 1, ..., :W]), i
        assert torch.equal(y1i, y1[i:i + 1]), i


# (B, OH): B * OH = 1, 7 (one split shorter than the 8-row minimum), 8, 9 (two splits, the second with one row), 257 (the
# bias gradient's 32 x 8 warps take 256 rows per sweep)
WG_ROWS = [(1, 1), (7, 1), (2, 4), (3, 3), (257, 1)]
WG_OW = [32, 33, 63]                                          # OW % 32 = 0, 1, 31


def _repeatable_wgrad(L, call, dw_shape):
    """call(dw, db) with dbias, once more without (dw identical, db untouched), once more with (identical bits)."""
    dw, db = _nan(*dw_shape), _nan(EC)
    L.check(call(dw, db), "bwd_weight")
    dw2, db2 = _nan(*dw_shape), _nan(EC)
    L.check(call(dw2, None), "bwd_weight without dbias")
    dw3, db3 = _nan(*dw_shape), _nan(EC)
    L.check(call(dw3, db3), "bwd_weight again")
    torch.cuda.synchronize()
    assert torch.equal(dw2, dw) and _all_nan(db2)
    assert torch.equal(dw3, dw) and torch.equal(db3, db)
    return dw, db


@pytest.mark.parametrize("OW", WG_OW)
@pytest.mark.parametrize("B,OH", WG_ROWS)
def test_weight_gradient_row_splits(L, B, OH, OW):
    """Both weight gradients over B * OH output rows split into chunks of at least 8 rows, against float64; with and
    without dbias; repeated calls give identical bits.  32 -> 32: KH = 3, KW = 5, SH = 2; first layer: KH = 33 (two kh
    blocks), KW = 5, PW = 1."""
    KH, KW, SH = 3, 5, 2
    H, W = SH * (OH - 1) + KH, OW + KW - 1
    c = emb2_ref(B, H, W, KH, KW, SH, seed=B * 100 + OW)
    geom = (B, EC, H, W, EC, KH, KW, SH, _r4(W), _r4(OW))
    x, dy = _pitched(c["x"], _r4(W)), _pitched(c["dy"], _r4(OW))
    ws = _ws(L, B, H, W, KH, KW)
    dw, db = _repeatable_wgrad(L, lambda dw, db: _wgrad(L, dy, x, dw, db, ws, geom), (EC, EC, KH, KW))
    _check(dw, c["dw"], WGRAD_BAR, "dw")
    _check(db, c["db"], BIAS_BAR, "db")

    KH, KW, PW = 33, 5, 1
    H, W = 2 * (OH - 1) + KH, 2 * OW + 1
    c = emb1_ref(B, H, W, KH, KW, PW, seed=B * 100 + OW + 1)
    assert tuple(c["y"].shape[2:]) == (OH, OW)
    geom = (B, H, W, EC, KH, KW, PW, _r4(OW))
    x, dy = c["x"].cuda(), _pitched(c["dy"], _r4(OW))
    ws = _c1_ws(L, B, H, W, KH, KW)
    dw, db = _repeatable_wgrad(L, lambda dw, db: _c1_wgrad(L, dy, x, dw, db, ws, geom), (EC, 1, KH, KW))
    _check(dw, c["dw"], C1_WGRAD_BAR, "c1 dw")
    _check(db, c["db"], BIAS_BAR, "c1 db")


# ================================================================================================ 4. the production batch
@pytest.mark.parametrize("precision", ["default", "tf32x3"])
def test_cfg3_production_batch(L, precision):
    """ops.EmbFrontendFn's five calls at cfg3 (B = 64, x [64, 1, 161, 400]; H1 = 61, W1 = 205, OH = 21, OW = 195; pitches
    P1 = 208, P2 = 196), with its argument lists: the first layer's forward at y_pitch = W1, the 32 -> 32 layer at
    (P1, P2), its weight and data gradient on one workspace, the first layer's weight gradient at P1.  The package's
    default precision (ops.config.conv) and 3xTF32, against float64 on the GPU."""
    import b200asr.ops as ops
    prec = 3
    if precision == "default":
        prec = ops.config.conv if ops.config.conv in PRECS else 3      # ops.EmbFrontendFn's prec2
    B, H, W = 64, 161, 400
    H1, W1 = (H - 41) // 2 + 1, (W + 20 - 11) // 2 + 1
    H2, W2 = (H1 - 21) // 2 + 1, W1 - 11 + 1
    P1, P2 = (W1 + 3) // 4 * 4, (W2 + 3) // 4 * 4
    assert (H1, W1, H2, W2, P1, P2) == (61, 205, 21, 195, 208, 196)
    g = _gen(64)
    x = torch.randn(B, 1, H, W, generator=g).cuda()
    w0 = (torch.randn(EC, 1, 41, 11, generator=g) * 451 ** -0.5).cuda()
    b0 = torch.randn(EC, generator=g).cuda()
    w3 = (torch.randn(EC, EC, 21, 11, generator=g) * 7392 ** -0.5).cuda()
    b3 = torch.randn(EC, generator=g).cuda()
    a1 = torch.randn(B, EC, H1, W1, generator=g)
    dc2 = torch.randn(B, EC, H2, W2, generator=g)
    dc1 = torch.randn(B, EC, H1, W1, generator=g)

    # float64 on the GPU
    x64 = x.double()
    w0_64, w3_64 = w0.double().requires_grad_(True), w3.double().requires_grad_(True)
    a1_64 = a1.cuda().double().requires_grad_(True)
    c1_ref = F.conv2d(x64, w0_64, b0.double(), stride=2, padding=(0, 10))
    c1_ref.backward(dc1.cuda().double())
    c2_ref = F.conv2d(a1_64, w3_64, b3.double(), stride=(2, 1))
    c2_ref.backward(dc2.cuda().double())

    c1 = _nan(B, EC, H1, W1)
    ws1 = _c1_ws(L, B, H, W, 41, 11)
    L.check(_c1_fwd(L, x, w0, b0, c1, ws1, (B, H, W, EC, 41, 11, 10, W1), prec), "emb_conv1_tc")
    _check(c1, c1_ref.detach(), C1_FWD_BAR[prec], "c1 fwd")
    del c1, c1_ref

    a1p, dc2p = _pitched(a1, P1), _pitched(dc2, P2)
    c2 = _nan(B, EC, H2, P2)
    ws = _ws(L, B, H1, W1, 21, 11)
    geom = (B, EC, H1, W1, EC, 21, 11, 2, P1, P2)
    L.check(_fwd(L, a1p, w3, b3, c2, ws, geom, prec), "emb_conv2_tc")
    _check(c2[..., :W2], c2_ref.detach(), FWD_BAR[prec], "fwd")
    del c2, c2_ref
    dw3, db3 = _nan(EC, EC, 21, 11), _nan(EC)
    L.check(_wgrad(L, dc2p, a1p, dw3, db3, ws, geom), "emb_conv2_tc_wgrad")
    _check(dw3, w3_64.grad, PROD_WGRAD_BAR, "dw")
    _check(db3, dc2.double().sum((0, 2, 3)), BIAS_BAR, "db")
    da1 = _nan(B, EC, H1, P1)
    L.check(_dgrad(L, dc2p, w3, da1, ws, geom, prec), "emb_conv2_tc_dgrad")
    _check(da1[..., :W1], a1_64.grad, FWD_BAR[prec], "dgrad")
    del da1, a1_64, a1p, ws

    dc1p = _pitched(dc1, P1)
    dw0, db0 = _nan(EC, 1, 41, 11), _nan(EC)
    ws1 = _c1_ws(L, B, H, W, 41, 11)
    L.check(_c1_wgrad(L, dc1p, x, dw0, db0, ws1, (B, H, W, EC, 41, 11, 10, P1)), "emb_conv1_tc_wgrad")
    _check(dw0, w0_64.grad, PROD_C1_WGRAD_BAR, "c1 dw")
    _check(db0, dc1.double().sum((0, 2, 3)), BIAS_BAR, "c1 db")


# ================================================================================================ 5. workspace size
GUARD = 1024                                                   # 4 KiB


def _guarded(n):
    buf = _nan(n + GUARD)
    return buf[:n], buf[n:]


@pytest.mark.parametrize("name", ["ref_h61", "ow1_kw13_kh1_sh3", "ow31_kw1_kh1_sh3", "ow257_kw13"])
def test_conv2d_implicit_gemm_32ch_workspace_size(L, name):
    """Forward, data gradient and weight gradient at 3xTF32 (the largest weight slices) on one workspace of exactly
    conv2d_tc_ws_bytes: the NaN guard after it stays NaN after every call."""
    B, H, W, KH, KW, SH, pad = EMB2[name]
    c = _emb2_case(name)
    OH, OW = c["y"].shape[2:]
    xp, yp = _r4(W) + pad, _r4(OW) + pad
    geom = (B, EC, H, W, EC, KH, KW, SH, xp, yp)
    x, dy, w, b = _pitched(c["x"], xp), _pitched(c["dy"], yp), c["w"].cuda(), c["b"].cuda()
    ws, guard = _guarded(L.load().b200asr_conv2d_tc_ws_bytes(B, H, W, KH, KW) // 4)
    y, dx, dw, db = _nan(B, EC, OH, yp), _nan(B, EC, H, xp), _nan(EC, EC, KH, KW), _nan(EC)
    for what, call in [("fwd", lambda: _fwd(L, x, w, b, y, ws, geom, 3)),
                       ("dgrad", lambda: _dgrad(L, dy, w, dx, ws, geom, 3)),
                       ("wgrad", lambda: _wgrad(L, dy, x, dw, db, ws, geom))]:
        L.check(call(), what)
        torch.cuda.synchronize()
        assert _all_nan(guard), what
    _check(y[..., :OW], c["y"] + c["b"].double()[:, None, None], FWD_BAR[3], "fwd")
    _check(dx[..., :W], c["dx"], FWD_BAR[3], "dgrad")
    _check(dw, c["dw"], WGRAD_BAR, "dw")


@pytest.mark.parametrize("name", ["ref_w50", "kh1_kw4_pw1", "kh64_pw15", "ow129_even_w"])
def test_conv2d_first_layer_workspace_size(L, name):
    """Forward and weight gradient at 3xTF32 on one workspace of exactly conv2d_c1_tc_ws_bytes + a NaN guard."""
    B, H, W, KH, KW, PW = EMB1[name]
    c = _emb1_case(name)
    OH, OW = c["y"].shape[2:]
    x, w, b, dy = c["x"].cuda(), c["w"].cuda(), c["b"].cuda(), _pitched(c["dy"], _r4(OW))
    ws, guard = _guarded(L.load().b200asr_conv2d_c1_tc_ws_bytes(B, H, W, KH, KW) // 4)
    y, dw, db = _nan(B, EC, OH, OW), _nan(EC, 1, KH, KW), _nan(EC)
    L.check(_c1_fwd(L, x, w, b, y, ws, (B, H, W, EC, KH, KW, PW, OW), 3), "conv2d_c1_tc_fwd")
    torch.cuda.synchronize()
    assert _all_nan(guard), "fwd"
    L.check(_c1_wgrad(L, dy, x, dw, db, ws, (B, H, W, EC, KH, KW, PW, _r4(OW))), "conv2d_c1_tc_bwd_weight")
    torch.cuda.synchronize()
    assert _all_nan(guard), "wgrad"
    _check(y, c["y"] + c["b"].double()[:, None, None], C1_FWD_BAR[3], "fwd")
    _check(dw, c["dw"], C1_WGRAD_BAR, "dw")


# ================================================================================================ 6. rejections, launch counts
def _rejected(L, call, code, what):
    n0 = _launches(L)
    assert call() == code, what
    assert _launches(L) == n0, what


def test_conv2d_implicit_gemm_32ch_rejections(L):
    """Ci or Co != 32, a pitch that is not a multiple of 4 or does not cover its row, H < KH, W < KW -> BAD_SHAPE;
    precision 0 or 1 -> BAD_ARG; x, dy or ws 4 bytes off a 16-byte boundary -> BAD_ALIGN.  No launch, nothing written."""
    B, H, W, KH, KW, SH = 1, 8, 40, 3, 5, 1                   # OH = 6, OW = 36
    n = 1 << 16
    x, dy, w = (torch.randn(n, device="cuda") for _ in range(3))
    b = torch.randn(EC, device="cuda")
    ws = _nan(L.load().b200asr_conv2d_tc_ws_bytes(B, H, W, KH, KW) // 4)
    y, dx, dw, db = _nan(n), _nan(n), _nan(n), _nan(EC)
    good = (B, EC, H, W, EC, KH, KW, SH, 40, 36)
    bad_shapes = {
        "Ci = 16": (B, 16, H, W, EC, KH, KW, SH, 40, 36),
        "Co = 64": (B, EC, H, W, 64, KH, KW, SH, 40, 36),
        "x_pitch % 4": (B, EC, H, W, EC, KH, KW, SH, 42, 36),
        "x_pitch < W": (B, EC, H, W, EC, KH, KW, SH, 36, 36),
        "y_pitch % 4": (B, EC, H, W, EC, KH, KW, SH, 40, 38),
        "y_pitch < OW": (B, EC, H, W, EC, KH, KW, SH, 40, 32),
        "H < KH": (B, EC, 2, W, EC, KH, KW, SH, 40, 36),
        "W < KW": (B, EC, H, 4, EC, KH, KW, SH, 4, 4),
    }
    for what, geom in bad_shapes.items():
        _rejected(L, lambda: _fwd(L, x, w, b, y, ws, geom, 3), BAD_SHAPE, ("fwd", what))
        _rejected(L, lambda: _dgrad(L, dy, w, dx, ws, geom, 3), BAD_SHAPE, ("dgrad", what))
        _rejected(L, lambda: _wgrad(L, dy, x, dw, db, ws, geom), BAD_SHAPE, ("wgrad", what))
    for prec in (0, 1):
        _rejected(L, lambda: _fwd(L, x, w, b, y, ws, good, prec), BAD_ARG, ("fwd", prec))
        _rejected(L, lambda: _dgrad(L, dy, w, dx, ws, good, prec), BAD_ARG, ("dgrad", prec))
    x_off, dy_off, ws_off = _off(n), _off(n), _off(ws.numel())
    x_off.copy_(x)
    dy_off.copy_(dy)
    for what, call in [("fwd x", lambda: _fwd(L, x_off, w, b, y, ws, good, 3)),
                       ("fwd ws", lambda: _fwd(L, x, w, b, y, ws_off, good, 3)),
                       ("dgrad dy", lambda: _dgrad(L, dy_off, w, dx, ws, good, 3)),
                       ("dgrad ws", lambda: _dgrad(L, dy, w, dx, ws_off, good, 3)),
                       ("wgrad dy", lambda: _wgrad(L, dy_off, x, dw, db, ws, good)),
                       ("wgrad x", lambda: _wgrad(L, dy, x_off, dw, db, ws, good)),
                       ("wgrad ws", lambda: _wgrad(L, dy, x, dw, db, ws_off, good))]:
        _rejected(L, call, BAD_ALIGN, what)
    torch.cuda.synchronize()
    assert _all_nan(y) and _all_nan(dx) and _all_nan(dw) and _all_nan(db) and _all_nan(ws) and _all_nan(ws_off)


def test_conv2d_first_layer_rejections(L):
    """Co != 32, KH > 64, H < KH, W + 2 PW < KW, y_pitch < OW, a weight-gradient y_pitch that is not a multiple of 4 ->
    BAD_SHAPE; precision 0 or 1 -> BAD_ARG; ws, or the weight gradient's dy, 4 bytes off a 16-byte boundary -> BAD_ALIGN.
    No launch, nothing written."""
    B, H, W, KH, KW, PW = 1, 45, 40, 41, 11, 10               # OH = 3, OW = 25
    n = 1 << 16
    x, dy = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    w, b = torch.randn(EC * 65 * KW, device="cuda"), torch.randn(EC, device="cuda")
    ws = _nan(L.load().b200asr_conv2d_c1_tc_ws_bytes(B, 70, W, 65, KW) // 4)
    y, dw, db = _nan(n), _nan(n), _nan(EC)
    bad_shapes = {
        "Co = 16": ((B, H, W, 16, KH, KW, PW, 25), (B, H, W, 16, KH, KW, PW, 28)),
        "KH = 65": ((B, 70, W, EC, 65, KW, PW, 25), (B, 70, W, EC, 65, KW, PW, 28)),
        "H < KH": ((B, 40, W, EC, KH, KW, PW, 25), (B, 40, W, EC, KH, KW, PW, 28)),
        "W + 2 PW < KW": ((B, H, 3, EC, KH, KW, 0, 4), (B, H, 3, EC, KH, KW, 0, 4)),
        "y_pitch < OW": ((B, H, W, EC, KH, KW, PW, 24), (B, H, W, EC, KH, KW, PW, 24)),
        "y_pitch % 4": (None, (B, H, W, EC, KH, KW, PW, 26)),
    }
    for what, (gf, gw) in bad_shapes.items():
        if gf is not None:
            _rejected(L, lambda: _c1_fwd(L, x, w, b, y, ws, gf, 3), BAD_SHAPE, ("fwd", what))
        _rejected(L, lambda: _c1_wgrad(L, dy, x, dw, db, ws, gw), BAD_SHAPE, ("wgrad", what))
    good_f, good_w = (B, H, W, EC, KH, KW, PW, 25), (B, H, W, EC, KH, KW, PW, 28)
    for prec in (0, 1):
        _rejected(L, lambda: _c1_fwd(L, x, w, b, y, ws, good_f, prec), BAD_ARG, ("fwd", prec))
    dy_off, ws_off = _off(n), _off(ws.numel())
    dy_off.copy_(dy)
    _rejected(L, lambda: _c1_fwd(L, x, w, b, y, ws_off, good_f, 3), BAD_ALIGN, "fwd ws")
    _rejected(L, lambda: _c1_wgrad(L, dy_off, x, dw, db, ws, good_w), BAD_ALIGN, "wgrad dy")
    _rejected(L, lambda: _c1_wgrad(L, dy, x, dw, db, ws_off, good_w), BAD_ALIGN, "wgrad ws")
    torch.cuda.synchronize()
    assert _all_nan(y) and _all_nan(dw) and _all_nan(db) and _all_nan(ws) and _all_nan(ws_off)


def test_launch_counts(L):
    """b200asr_launch_count grows by the kernels each entry point enqueues: forward and data gradient 3 (weight repack,
    shifted or de-interleaved copies, engine), weight gradients 3 (copies, engine, split reduction) and 5 with dbias (+
    bias partials, their reduction)."""
    B, H, W, KH, KW, SH = 2, 9, 40, 3, 5, 2                   # OH = 4, OW = 36
    c = emb2_ref(B, H, W, KH, KW, SH, seed=3)
    geom = (B, EC, H, W, EC, KH, KW, SH, 40, 36)
    x, dy, w, b = c["x"].cuda(), c["dy"].cuda(), c["w"].cuda(), c["b"].cuda()
    ws = _ws(L, B, H, W, KH, KW)
    y, dx, dw, db = _nan(B, EC, 4, 36), _nan(B, EC, H, W), _nan(EC, EC, KH, KW), _nan(EC)
    c1 = emb1_ref(2, 45, 40, 41, 11, 10, seed=4)              # OH = 3, OW = 25
    geom1 = (2, 45, 40, EC, 41, 11, 10, 28)
    x1, w1, dy1 = c1["x"].cuda(), c1["w"].cuda(), _pitched(c1["dy"], 28)
    ws1 = _c1_ws(L, 2, 45, 40, 41, 11)
    y1, dw1 = _nan(2, EC, 3, 28), _nan(EC, 1, 41, 11)
    calls = []
    for prec in PRECS:
        calls += [(f"conv2d_tc_fwd {prec}", lambda p=prec: _fwd(L, x, w, b, y, ws, geom, p), 3),
                  (f"conv2d_tc_bwd_data {prec}", lambda p=prec: _dgrad(L, dy, w, dx, ws, geom, p), 3),
                  (f"conv2d_c1_tc_fwd {prec}", lambda p=prec: _c1_fwd(L, x1, w1, b, y1, ws1, geom1, p), 3)]
    calls += [("conv2d_tc_bwd_weight", lambda: _wgrad(L, dy, x, dw, db, ws, geom), 5),
              ("conv2d_tc_bwd_weight no dbias", lambda: _wgrad(L, dy, x, dw, None, ws, geom), 3),
              ("conv2d_c1_tc_bwd_weight", lambda: _c1_wgrad(L, dy1, x1, dw1, db, ws1, geom1), 5),
              ("conv2d_c1_tc_bwd_weight no dbias", lambda: _c1_wgrad(L, dy1, x1, dw1, None, ws1, geom1), 3)]
    for what, call, launches in calls:
        n0 = _launches(L)
        L.check(call(), what)
        assert _launches(L) - n0 == launches, what
    torch.cuda.synchronize()
    assert bool(torch.isfinite(y).all() and torch.isfinite(dx).all() and torch.isfinite(dw).all())
    assert bool(torch.isfinite(y1[..., :25]).all() and torch.isfinite(dw1).all())
