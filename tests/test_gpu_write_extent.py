"""Write extent of every kernel entry point: each output and workspace sits inside one larger allocation between two guard
bands of a fixed byte pattern, every input comes back bit for bit, and strided outputs keep the gap columns between their rows.

The value tests of the other kernel files allocate each output with exactly its size, so a store that lands past the end of
an output -- a partial last tile stored whole, a pooled row written for an odd T, a bit word one pixel too far, a workspace
used beyond its *_ws_bytes -- falls into the caching allocator's rounding slack there and goes unnoticed, while in training it
lands in whatever tensor the allocator placed next (a neighbouring weight of the flat parameter buffer, another activation,
the Adam state).  Here:

  * `Guarded` lays a buffer out as [front guard | region | back guard]; the guards (and, for a row pitch wider than the row,
    the gap columns) are 0xA5 bytes compared through a uint8 view, so the check is the same for fp32, bf16, int32, bit words
    and outputs that legitimately hold NaN.  A guard is at least 64 KiB -- one 128 x 128 fp32 output tile -- and a multiple
    of 256 bytes, so the region keeps the allocator's alignment (TMA) unless a case shifts it by 16 bytes on purpose (the
    entry points that only require 16-byte alignment run both placements).
  * `Arena.call` launches one entry point through the C ABI, synchronises, and checks every buffer of the arena: inputs
    bit-identical (guards included), outputs / workspaces with untouched guards and gaps.  Outputs start NaN (or a sentinel
    for integers), and every call also compares its result with the float64 reference of its family at that family's bar,
    so a guarded call is known to have done the real computation at its edge shape.
  * The shapes are the partial last tiles of each kernel's tiling (halo 16 x 8, weight-gradient 4 x 8 pixel blocks, the
    engine's 128-row tiles, BN_SPLITS = 32), odd T and F under pooling, bit words and codes at C = 32, 64, 96, decode keys
    around the split-key threshold, one-row / one-utterance calls.  The optional store paths run too: dropout (probs_drop
    of the materialised attention, the dropout masks of the flash paths and of add_ln with its separate dx), add_ln_bwd
    accumulating into dgamma / dbeta, the head-major attention output, packed LSTM sequences of decreasing length.

Two CPU tests keep the sweep complete: every entry point of b200asr._lib.SIGNATURES that takes a pointer is either covered
here (COVERAGE, whose test must name it) or exempted with the test that already guards it (EXEMPT); and the guard check
itself detects a byte written just before, just after or between the rows of a region, and nothing else."""
import inspect
import math
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import asr_oracle as O
from tests.ctc_util import ctc_float64
from tests.helpers import rel_err

PAT = 0xA5                 # guard byte: as fp32 0xA5A5A5A5 is -2.9e-16, as int32 a large negative id -- nothing a kernel writes
MIN_GUARD = 64 * 1024      # one 128 x 128 fp32 tile
NAN = float("nan")
SENT32 = -0x3A3A3A3B       # int32 / int64 poison
gpu = pytest.mark.gpu


# ================================================================================================ the guarded allocator
def _round_up(n, m):
    return (n + m - 1) // m * m


class Guarded:
    """A tensor of `shape` / `dtype` inside [front guard | region | back guard] of one uint8 allocation.

    pitch: elements per row of the last dimension (>= shape[-1]); the columns past shape[-1] are gap bytes that keep the
    guard pattern.  shift: bytes between the end of the front guard and the region (16: a 16-byte but not 256-byte aligned
    placement).  role: "in" (every byte, guards included, must come back unchanged), "out" / "inout" / "ws" (guards and
    gaps untouched).  fill: a tensor copied in, a scalar, or None (the region keeps the guard pattern)."""

    def __init__(self, shape, dtype=torch.float32, fill=None, *, role="out", pitch=None, shift=0, guard=MIN_GUARD,
                 device="cuda", name="buf"):
        self.shape = tuple(int(s) for s in shape)
        self.dtype, self.role, self.name = dtype, role, name
        self.isz = torch.empty(0, dtype=dtype).element_size()
        self.width = self.shape[-1] if self.shape else 1
        self.rows = math.prod(self.shape[:-1]) if self.shape else 1
        self.pitch = self.width if pitch is None else int(pitch)
        assert self.pitch >= self.width and shift % 16 == 0
        self.nbytes = self.rows * self.pitch * self.isz
        self.guard = _round_up(max(guard, MIN_GUARD), 256)
        self.off = self.guard + shift
        self.raw = torch.full((self.off + self.nbytes + self.guard,), PAT, dtype=torch.uint8, device=device)
        self.t = self._logical(self.raw)
        if isinstance(fill, torch.Tensor):
            self.t.copy_(fill.reshape(self.shape).to(dtype))
        elif fill is not None:
            self.t.fill_(fill)
        self.snap = None
        if role == "in":
            self.freeze()

    def _logical(self, buf):
        region = buf[self.off:self.off + self.nbytes].view(self.dtype)
        return region.view(self.rows, self.pitch)[:, :self.width].view(self.shape)

    def _logical_bytes(self, buf):
        region = buf[self.off:self.off + self.nbytes]
        return region.view(self.rows, self.pitch * self.isz)[:, :self.width * self.isz]

    def freeze(self):
        """From now on the buffer is an input: every byte must stay as it is now."""
        self.role = "in"
        self.snap = self.raw.clone()

    @property
    def ptr(self):
        return self.raw.data_ptr() + self.off

    def damage(self):
        """(number of bytes that must not have changed but did, their first few offsets relative to the region start)."""
        if self.role == "in":
            bad = self.raw != self.snap
        else:
            c = self.raw.clone()
            self._logical_bytes(c).fill_(PAT)
            bad = c != PAT
        idx = bad.nonzero().flatten()
        return int(idx.numel()), [int(i) - self.off for i in idx[:6].cpu()]


class Arena:
    """The guarded buffers of one case.  `call` runs an entry point and checks every buffer afterwards."""

    def __init__(self, lib=None, shift=0, device="cuda"):
        self.lib, self.shift, self.device = lib, shift, device
        self.bufs = []

    def _new(self, name, shape, dtype, fill, role, pitch=None):
        g = Guarded(shape, dtype, fill, role=role, pitch=pitch, shift=self.shift, device=self.device, name=name)
        self.bufs.append(g)
        return g

    def inp(self, name, t, pitch=None):
        return self._new(name, t.shape, t.dtype, t, "in", pitch)

    def out(self, name, shape, dtype=torch.float32, fill=None, pitch=None):
        if fill is None:
            fill = NAN if dtype.is_floating_point else SENT32 if dtype in (torch.int32, torch.int64) else 0x5A
        return self._new(name, shape, dtype, fill, "out", pitch)

    def inout(self, name, t, pitch=None):
        return self._new(name, t.shape, t.dtype, t, "inout", pitch)

    def ws(self, name, nbytes):
        """Exactly nbytes of workspace (0: a guard-only buffer whose pointer is still passed), filled with NaN bytes."""
        return self._new(name, (int(nbytes),), torch.uint8, 0xFF, "ws")

    def verify(self, what):
        for g in self.bufs:
            n, where = g.damage()
            kind = "input bytes changed" if g.role == "in" else "guard / gap bytes written"
            assert n == 0, f"{what}: {g.name} ({g.role}, shape {g.shape}, pitch {g.pitch}): {n} {kind}, " \
                           f"at region offsets {where} (region is {g.nbytes} bytes)"

    def call(self, name, *args):
        fn = getattr(self.lib, "b200asr_" + name)
        rc = fn(*[a.ptr if isinstance(a, Guarded) else a for a in args], torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert rc == 0, f"b200asr_{name} returned {rc}: {self.lib.b200asr_last_error().decode()}"
        self.verify(name)


@pytest.fixture(scope="module")
def lib():
    import b200asr
    return b200asr._lib.load(check_device=True)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(*shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=_gen(seed)) * scale).cuda()


# ================================================================================================ CPU: the harness
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.int32, torch.uint8])
@pytest.mark.parametrize("shift", [0, 16])
def test_guard_detects_planted_overruns(dtype, shift):
    """A byte written just before the region, just after it, or into a gap column is reported; writes anywhere inside the
    logical region -- NaN included -- are not."""
    def fresh():
        return Guarded((3, 5, 7), dtype, 0, pitch=9, shift=shift, device="cpu")

    g = fresh()
    assert g.off % 256 == shift
    assert g.damage()[0] == 0
    if dtype.is_floating_point:
        g.t.fill_(NAN)
    else:
        g.t.fill_(7)
    g.t[0, 0, 0] = 7
    g.t[-1, -1, -1] = 3
    assert g.damage()[0] == 0
    isz = g.isz
    for pos in (g.off - 1, g.off + g.nbytes, g.off + g.nbytes + g.guard - 1, 0,      # before, after, both outer ends
                g.off + 7 * isz,                                                    # first gap column of row 0
                g.off + g.nbytes - 1):                                              # last gap byte of the last row
        g = fresh()
        g.raw[pos] = 0
        n, where = g.damage()
        assert n == 1 and where == [pos - g.off], (pos, n, where)

    i = Guarded((4, 4), dtype, 1, role="in", device="cpu")
    assert i.damage()[0] == 0
    i.t[2, 3] = 0                                         # an input may not change anywhere
    assert 0 < i.damage()[0] <= i.isz
    i = Guarded((4, 4), dtype, 1, role="in", device="cpu")
    i.raw[0] = 0
    assert i.damage() == (1, [-i.off])


def test_arena_reports_the_damaged_buffer():
    a = Arena(device="cpu")
    x = a.inp("x", torch.arange(6.0))
    y = a.out("y", (6,))
    ws = a.ws("ws", 0)
    a.verify("ok")
    y.raw[y.off + y.nbytes + 3] = 1
    with pytest.raises(AssertionError, match="y .*1 guard"):
        a.verify("overrun")
    y.raw[y.off + y.nbytes + 3] = PAT
    ws.raw[ws.off] = 0                                    # a zero-byte workspace: any write is an overrun
    with pytest.raises(AssertionError, match="ws"):
        a.verify("ws")
    ws.raw[ws.off] = PAT
    x.t[0] = 5.0
    with pytest.raises(AssertionError, match="input bytes changed"):
        a.verify("input")


# ================================================================================================ CPU: coverage of the ABI
_LINEAR = "tests/test_gpu_linear_precisions.py: BAND sentinel floats on both sides of every output, shifted placements"
_EMB = "tests/test_gpu_emb_implicit_gemm.py: guarded workspaces (GUARD) and NaN-poisoned outputs at every instantiation"
_STFT = "tests/test_gpu_feature_augment.py / tests/test_gpu_loader.py: guarded STFT workspace (GUARD)"
_OPT = "tests/test_gpu_optimizer_step.py: the tensors are views into one shared storage, compared bit for bit"
EXEMPT = {
    "b200asr_linear_fwd": _LINEAR, "b200asr_linear_bwd_data": _LINEAR, "b200asr_linear_bwd_weight": _LINEAR,
    "b200asr_split_bf16": "tests/test_gpu_default_precision.py: _SENTINEL fill of dst / dst_t and of the unwritten layout",
    "b200asr_stft_features": _STFT, "b200asr_stft_features_ex": _STFT, "b200asr_stft_features_packed": _STFT,
    "b200asr_conv2d_tc_fwd": _EMB, "b200asr_conv2d_tc_bwd_data": _EMB, "b200asr_conv2d_tc_bwd_weight": _EMB,
    "b200asr_conv2d_c1_tc_fwd": _EMB, "b200asr_conv2d_c1_tc_bwd_weight": _EMB,
    "b200asr_edit_counts": "tests/test_gpu_edit_counts.py: guarded workspace and sentinel-filled per_utt / totals",
    "b200asr_adam_multi": _OPT, "b200asr_norm_multi": _OPT, "b200asr_clip_coef": _OPT, "b200asr_scale_multi": _OPT,
}

# entry point -> the test of this file that guards it (its source names the entry point)
COVERAGE = {
    "b200asr_conv3x3_fwd": "test_conv3x3_forward", "b200asr_conv3x3_fwd_bits": "test_conv3x3_forward",
    "b200asr_conv3x3_fwd_pool": "test_conv3x3_forward", "b200asr_conv3x3_fwd_pool_codes": "test_conv3x3_forward",
    "b200asr_conv3x3_bwd_data": "test_conv3x3_data_gradient", "b200asr_conv3x3_bwd_data_bits": "test_conv3x3_data_gradient",
    "b200asr_conv3x3_bwd_weight": "test_conv3x3_weight_gradient",
    "b200asr_conv3x3_c1_fwd": "test_conv3x3_c1", "b200asr_conv3x3_c1_fwd_bits": "test_conv3x3_c1",
    "b200asr_conv3x3_c1_bwd_weight": "test_conv3x3_c1",
    "b200asr_maxpool2x2_fwd": "test_maxpool", "b200asr_maxpool2x2_fwd_idx": "test_maxpool",
    "b200asr_maxpool2x2_bwd": "test_maxpool", "b200asr_maxpool2x2_bwd_idx": "test_maxpool",
    "b200asr_maxpool2x2_bwd_codes": "test_maxpool",
    "b200asr_conv2d_fwd": "test_conv2d_cuda_core", "b200asr_conv2d_bwd_data": "test_conv2d_cuda_core",
    "b200asr_conv2d_bwd_weight": "test_conv2d_cuda_core",
    "b200asr_flatten_bcft_fwd": "test_flatten_and_permute", "b200asr_flatten_bcft_bwd": "test_flatten_and_permute",
    "b200asr_permute_cols_cf": "test_flatten_and_permute",
    "b200asr_bn_clamp_fwd": "test_bn_clamp", "b200asr_bn_clamp_bwd": "test_bn_clamp",
    "b200asr_add_ln_fwd": "test_add_ln", "b200asr_add_ln_bwd": "test_add_ln",
    "b200asr_sdpa_fwd": "test_sdpa_flash", "b200asr_sdpa_bwd": "test_sdpa_flash",
    "b200asr_sdpa_fused_fwd": "test_sdpa_flash", "b200asr_sdpa_fused_bwd": "test_sdpa_flash",
    "b200asr_sdpa_mat_fwd": "test_sdpa_materialised", "b200asr_sdpa_mat_bwd": "test_sdpa_materialised",
    "b200asr_decode_attn": "test_decode_attn", "b200asr_beam_self_attn": "test_beam_self_attn",
    "b200asr_beam_step": "test_beam_step", "b200asr_beam_step_log": "test_beam_step",
    "b200asr_beam_backtrack": "test_beam_backtrack", "b200asr_beam_backtrack_packed": "test_beam_backtrack",
    "b200asr_argmax_rows": "test_argmax_and_greedy_step", "b200asr_greedy_step": "test_argmax_and_greedy_step",
    "b200asr_ce_fwd": "test_cross_entropy", "b200asr_ce_finalize": "test_cross_entropy", "b200asr_ce_bwd": "test_cross_entropy",
    "b200asr_embed_fwd": "test_embedding", "b200asr_embed_bwd": "test_embedding",
    "b200asr_length_masks": "test_target_preprocessing_and_masks",
    "b200asr_preprocess_targets": "test_target_preprocessing_and_masks",
    "b200asr_ctc_fwd": "test_ctc", "b200asr_ctc_bwd": "test_ctc",
    "b200asr_lstm_prepare": "test_lstm_prepare_and_unprepare", "b200asr_lstm_grad_unprepare": "test_lstm_prepare_and_unprepare",
    "b200asr_lstm_layer_fwd": "test_lstm_layers", "b200asr_lstm_layer_train_fwd": "test_lstm_layers",
    "b200asr_lstm_layer_train_bwd": "test_lstm_layers", "b200asr_lstm_dropout": "test_lstm_dropout",
    "b200asr_lm_nll": "test_lm_nll_and_seq_sum", "b200asr_lm_seq_sum": "test_lm_nll_and_seq_sum",
    "b200asr_sumsq": "test_step_tail", "b200asr_grad_scale": "test_step_tail", "b200asr_adam_step": "test_step_tail",
    "b200asr_split_tf32": "test_split_tf32", "b200asr_split_bf16_batched": "test_split_bf16_batched",
}


def _pointer_entry_points():
    import ctypes
    from b200asr import _lib as Lb
    return sorted(n for n, (_, args) in Lb.SIGNATURES.items() if ctypes.c_void_p in args or ctypes.c_char_p in args)


def test_every_pointer_entry_point_is_guarded_or_exempt():
    """A kernel added to the ABI without guard coverage fails here, on any machine."""
    names = _pointer_entry_points()
    missing = [n for n in names if n not in COVERAGE and n not in EXEMPT]
    assert not missing, f"entry points with no write-extent test and no exemption: {missing}"
    assert not set(COVERAGE) & set(EXEMPT)
    assert set(COVERAGE) | set(EXEMPT) <= set(names), sorted((set(COVERAGE) | set(EXEMPT)) - set(names))
    mod = sys.modules[__name__]
    for name, test in COVERAGE.items():
        fn = getattr(mod, test, None)
        assert fn is not None and getattr(fn, "pytestmark", None), (name, test)
        assert any(m.name == "gpu" for m in fn.pytestmark), test
        assert f'"{name[len("b200asr_"):]}"' in inspect.getsource(fn), f"{test} does not call {name}"
    for name, why in EXEMPT.items():
        assert why.startswith("tests/test_") and ":" in why, name


# ================================================================================================ references
def _nchw(t):
    return t.permute(0, 3, 2, 1)


def conv3x3_ref(x, w, b, relu):
    y = F.conv2d(_nchw(x.double()), w.double(), None if b is None else b.double(), padding=1)
    return _nchw(y.relu() if relu else y)


def pack_bits(y):
    """[..., C] -> int32 [..., C/32]: bit c % 32 of word c / 32 = (y > 0)."""
    b = (y > 0).to(torch.int64).reshape(*y.shape[:-1], y.shape[-1] // 32, 32)
    w = (b << torch.arange(32, device=y.device)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def pool_positions(x):
    """x [B, T, F, C] -> (pooled [B, T/2, F/2, C], position of the first maximum in ATen's scan order (f, t), (f, t+1),
    (f+1, t), (f+1, t+1) | 4 when it is not positive)."""
    B, T, F_, C = x.shape
    T2, F2 = T // 2, F_ // 2
    v = x[:, :2 * T2, :2 * F2].reshape(B, T2, 2, F2, 2, C)
    a = [v[:, :, 0, :, 0], v[:, :, 1, :, 0], v[:, :, 0, :, 1], v[:, :, 1, :, 1]]
    best, m = torch.zeros_like(a[0], dtype=torch.int64), a[0]
    for k in (1, 2, 3):
        gt = a[k] > m
        best, m = torch.where(gt, k, best), torch.where(gt, a[k], m)
    return m, best | torch.where(m > 0, 0, 4)


def pool_codes(x):
    _, code = pool_positions(x)
    B, T2, F2, C = code.shape
    w = (code.reshape(B, T2, F2, C // 8, 8) << (4 * torch.arange(8, device=x.device))).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def pool_bwd_ref(x, dy, relu_mask):
    """dy routed to each window's first maximum (x.* (max > 0) with relu_mask); uncovered rows / columns 0."""
    B, T, F_, C = x.shape
    m, pos = pool_positions(x)
    dx = torch.zeros(B, T, F_, C, dtype=torch.float64, device=x.device)
    T2, F2 = T // 2, F_ // 2
    g = dy.double() * ((m > 0) if relu_mask else 1)
    p = pos & 3
    v = dx[:, :2 * T2, :2 * F2].reshape(B, T2, 2, F2, 2, C)
    for k, (dt, df) in enumerate([(0, 0), (1, 0), (0, 1), (1, 1)]):
        v[:, :, dt, :, df] += torch.where(p == k, g, 0.0)
    return dx


def pairs_rne(v):
    """The convolution epilogue's bf16 pairs (cvt.rn.bf16x2, round to nearest even): [2, *shape] int16 hi = bf16(v),
    lo = bf16(v - hi)."""
    hi = v.float().bfloat16()
    lo = (v.float() - hi.float()).bfloat16()
    return torch.stack([hi, lo]).view(torch.int16)


def pairs_ref(v):
    """The pooling backward's and the operand split's bf16 pairs [2, *shape] as int16: hi = top half of bits(v) + 0x8000
    (round half away from zero), lo the same of v - hi."""
    a = v.float().contiguous().cpu().numpy()
    r = a.view(np.uint32) + np.uint32(0x8000)
    hi = (r >> np.uint32(16)).astype(np.uint16)
    lo = a - (r & np.uint32(0xFFFF0000)).view(np.float32)
    lb = (lo.view(np.uint32) + np.uint32(0x8000)) >> np.uint32(16)
    return torch.from_numpy(np.stack([hi, lb.astype(np.uint16)]).view(np.int16))


def _inv_keep(p):
    """common.cuh dropout_inv_keep: 1 / (1 - threshold / 65536) in float32."""
    t = int(min(max(np.float32(p) * np.float32(65536.0) + np.float32(0.5), np.float32(0.0)), np.float32(65535.0)))
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(t) / np.float32(65536.0)))


SEED, OFFSET = 7, 3


def _eq(a, b):
    return torch.equal(a.cpu(), b.cpu())


# ================================================================================================ 3x3 convolutions
PRECS = [0, 1, 3, 6, 2]
CONV_BARS = {0: 4e-6, 1: 3e-3, 3: 3e-5, 6: 3e-5, 2: 1e-2}
WGRAD_BARS = {0: 4e-6, 1: 2e-3, 3: 1e-4, 6: 4e-5, 2: 1e-2}
# (B, T, F, Ci, Co): T, F off the halo kernel's 16 x 8 tile and odd (pooled floor), B*T*F off the engine's 128 rows; one pixel
CONV_FWD_SHAPES = [(1, 19, 13, 32, 64), (2, 17, 9, 64, 128), (1, 1, 1, 32, 64)]
CONV_DGRAD_SHAPES = [(1, 19, 13, 64, 32), (2, 17, 9, 128, 64), (1, 1, 1, 64, 32)]
# weight gradient: T, F off its 4 x 8 pixel blocks, Co off and on its 64-wide tiles
CONV_WGRAD_SHAPES = [(1, 7, 13, 64, 64), (2, 9, 11, 64, 128), (1, 1, 1, 64, 64)]


def _shifts(prec):
    return [0, 16]                                 # every precision requires 16-byte alignment only (TMA included)


@gpu
@pytest.mark.parametrize("shape", CONV_FWD_SHAPES, ids=str)
@pytest.mark.parametrize("prec", PRECS)
def test_conv3x3_forward(lib, prec, shape):
    """conv3x3_fwd, _fwd_bits, _fwd_pool (with and without index bytes) and _fwd_pool_codes (in the bf16 modes also with
    y = NULL: the halo epilogue's pool, pool_codes and out_bits stores): y against float64, the bits, pooled values, index
    bytes and codes against the kernel's own y, exactly."""
    B, T, F_, Ci, Co = shape
    x, w, b = _randn(B, T, F_, Ci, seed=1), _randn(Co, Ci, 3, 3, seed=2, scale=0.1), _randn(Co, seed=3)
    y_ref = conv3x3_ref(x, w, b, 1)
    ws_bytes = lib.b200asr_conv3x3_ws_bytes(Ci, Co)
    T2, F2 = T // 2, F_ // 2
    bf16 = prec in (2, 6)
    for shift in _shifts(prec):
        A = Arena(lib, shift)
        xg, wg, bg = A.inp("x", x), A.inp("w", w), A.inp("b", b)
        ws = A.ws("ws", ws_bytes)
        head = lambda y: (xg, wg, bg, y)
        dims = (B, T, F_, Ci, Co, 1, prec)

        y = A.out("y", (B, T, F_, Co))
        A.call("conv3x3_fwd", *head(y), ws, *dims)
        assert rel_err(y.t, y_ref) < CONV_BARS[prec]
        y.freeze()

        y1, bits = A.out("y1", (B, T, F_, Co)), A.out("bits", (B, T, F_, Co // 32), torch.int32)
        A.call("conv3x3_fwd_bits", *head(y1), ws, *dims, bits)
        assert _eq(y1.t, y.t) and _eq(bits.t, pack_bits(y.t))

        for with_idx in (False, True):
            y2, p2 = A.out("y2", (B, T, F_, Co)), A.out("pooled", (B, T2, F2, Co))
            idx = A.out("idx", (B, T2, F2, Co), torch.uint8) if with_idx else None
            A.call("conv3x3_fwd_pool", *head(y2), p2, idx, ws, *dims)
            assert rel_err(y2.t, y_ref) < CONV_BARS[prec]
            assert _eq(p2.t, pool_positions(y2.t)[0])
            if with_idx:
                assert _eq(idx.t, pool_positions(y2.t)[1].to(torch.uint8))

        y3, p3 = A.out("y3", (B, T, F_, Co)), A.out("pooled3", (B, T2, F2, Co))
        c3 = A.out("codes", (B, T2, F2, Co // 8), torch.int32)
        A.call("conv3x3_fwd_pool_codes", *head(y3), p3, c3, ws, *dims)
        assert rel_err(y3.t, y_ref) < CONV_BARS[prec]
        assert _eq(p3.t, pool_positions(y3.t)[0]) and _eq(c3.t, pool_codes(y3.t))
        if bf16:                                             # the epilogue alone: y is not written at all
            p4, c4 = A.out("pooled4", (B, T2, F2, Co)), A.out("codes4", (B, T2, F2, Co // 8), torch.int32)
            A.call("conv3x3_fwd_pool_codes", xg, wg, bg, None, p4, c4, ws, *dims)
            assert _eq(p4.t, p3.t) and _eq(c4.t, c3.t)


@gpu
@pytest.mark.parametrize("shape", CONV_DGRAD_SHAPES, ids=str)
@pytest.mark.parametrize("prec", PRECS)
def test_conv3x3_data_gradient(lib, prec, shape):
    """conv3x3_bwd_data with relu_out and _bwd_data_bits with packed bits, and in the bf16 modes the bf16 pair output dx16
    (hi at 0, lo at + B*T*F*Ci): dx against float64, the two masks bit-identical, dx16 the (round-to-nearest-even) pairs of
    dx exactly."""
    B, T, F_, Ci, Co = shape
    dy, w, mask = _randn(B, T, F_, Co, seed=4), _randn(Co, Ci, 3, 3, seed=5, scale=0.1), _randn(B, T, F_, Ci, seed=6)
    dx_ref = _nchw(torch.nn.grad.conv2d_input((B, Ci, F_, T), w.double(), _nchw(dy.double()), padding=1)) * (mask > 0)
    bf16 = prec in (2, 6)
    for shift in _shifts(prec):
        A = Arena(lib, shift)
        dyg, wg, mg, bits = A.inp("dy", dy), A.inp("w", w), A.inp("relu_out", mask), A.inp("relu_bits", pack_bits(mask))
        ws = A.ws("ws", lib.b200asr_conv3x3_ws_bytes(Ci, Co))
        dims = (B, T, F_, Ci, Co, prec)
        dx = A.out("dx", (B, T, F_, Ci))
        dx16 = A.out("dx16", (2, B, T, F_, Ci), torch.int16) if bf16 else None
        A.call("conv3x3_bwd_data", dyg, wg, mg, dx, dx16, ws, *dims)
        assert rel_err(dx.t, dx_ref) < CONV_BARS[prec]
        if bf16:
            assert _eq(dx16.t, pairs_rne(dx.t))
        dx2 = A.out("dx_bits", (B, T, F_, Ci))
        dx216 = A.out("dx16_bits", (2, B, T, F_, Ci), torch.int16) if bf16 else None
        A.call("conv3x3_bwd_data_bits", dyg, wg, bits, dx2, dx216, ws, *dims)
        assert _eq(dx2.t, dx.t) and (not bf16 or _eq(dx216.t, dx16.t))


@gpu
@pytest.mark.parametrize("shape", CONV_WGRAD_SHAPES, ids=str)
@pytest.mark.parametrize("prec", PRECS)
def test_conv3x3_weight_gradient(lib, prec, shape):
    """conv3x3_bwd_weight into dw / dbias (the weight-gradient reductions and the unpack), with and without dbias, and in
    the bf16 modes from the dy16 pairs as well: against float64, and the workspace used within conv3x3_ws_bytes."""
    B, T, F_, Ci, Co = shape
    x, dy = _randn(B, T, F_, Ci, seed=7), _randn(B, T, F_, Co, seed=8)
    dw_ref = torch.nn.grad.conv2d_weight(_nchw(x.double()), (Co, Ci, 3, 3), _nchw(dy.double()), padding=1)
    db_ref = dy.double().sum((0, 1, 2))
    pair_options = [None, pairs_ref(dy).cuda()] if prec in (2, 6) else [None]
    for shift in _shifts(prec):
        for pairs in pair_options:
            for with_bias in (True, False):
                A = Arena(lib, shift)
                dyg, xg = A.inp("dy", dy), A.inp("x", x)
                dy16 = A.inp("dy16", pairs) if pairs is not None else None
                dw, db = A.out("dw", (Co, Ci, 3, 3)), (A.out("dbias", (Co,)) if with_bias else None)
                ws = A.ws("ws", lib.b200asr_conv3x3_ws_bytes(Ci, Co))
                A.call("conv3x3_bwd_weight", dyg, dy16, xg, dw, db, ws, B, T, F_, Ci, Co, prec)
                assert rel_err(dw.t, dw_ref) < WGRAD_BARS[prec]
                if with_bias:
                    assert rel_err(db.t, db_ref) < (1e-5 if pairs is None else 2e-5 if prec == 6 else 1e-2)


@gpu
@pytest.mark.parametrize("B,F_,T,Co", [(1, 13, 19, 32), (2, 9, 7, 64), (1, 1, 1, 4), (3, 5, 3, 128)])
def test_conv3x3_c1(lib, B, F_, T, Co):
    """The first VGG convolution: conv3x3_c1_fwd, _fwd_bits (Co % 32 == 0) and conv3x3_c1_bwd_weight (dw and dbias), both
    placements."""
    x, w, b = _randn(B, F_, T, seed=9), _randn(Co, 1, 3, 3, seed=10), _randn(Co, seed=11)
    y_ref = _nchw(F.conv2d(x.double()[:, None], w.double(), b.double(), padding=1).relu())
    dy = _randn(B, T, F_, Co, seed=12)
    dw_ref = torch.nn.grad.conv2d_weight(x.double()[:, None], (Co, 1, 3, 3), _nchw(dy.double()), padding=1)
    for shift in (0, 16):
        A = Arena(lib, shift)
        xg, wg, bg = A.inp("x", x), A.inp("w", w), A.inp("b", b)
        y = A.out("y", (B, T, F_, Co))
        A.call("conv3x3_c1_fwd", xg, wg, bg, y, B, F_, T, Co, 1)
        assert rel_err(y.t, y_ref) < 6e-7
        if Co % 32 == 0:
            y1, bits = A.out("y1", (B, T, F_, Co)), A.out("bits", (B, T, F_, Co // 32), torch.int32)
            A.call("conv3x3_c1_fwd_bits", xg, wg, bg, y1, B, F_, T, Co, 1, bits)
            assert _eq(y1.t, y.t) and _eq(bits.t, pack_bits(y.t))
        dyg = A.inp("dy", dy)
        dw, db = A.out("dw", (Co, 1, 3, 3)), A.out("dbias", (Co,))
        A.call("conv3x3_c1_bwd_weight", xg, dyg, dw, db, B, F_, T, Co)
        assert rel_err(dw.t, dw_ref) < 2.5e-6 and rel_err(db.t, dy.double().sum((0, 1, 2))) < 2.5e-6


@gpu
@pytest.mark.parametrize("C", [32, 64, 96])
@pytest.mark.parametrize("B,T,F_", [(1, 7, 5), (2, 6, 9), (1, 1, 3), (1, 2, 2)])
def test_maxpool(lib, B, T, F_, C):
    """maxpool2x2_fwd / _fwd_idx, and the three backwards (from the activation, the index bytes and the codes) with the
    bf16 pairs dx16, at odd T / F (rows and columns no window covers) and one-window / no-window shapes: exact."""
    x, dy = _randn(B, T, F_, C, seed=13), _randn(B, T // 2, F_ // 2, C, seed=14)
    pooled_ref, pos = pool_positions(x)
    dx_ref = pool_bwd_ref(x, dy, True)
    for shift in (0, 16):
        A = Arena(lib, shift)
        xg, dyg = A.inp("x", x), A.inp("dy", dy)
        y = A.out("y", (B, T // 2, F_ // 2, C))
        A.call("maxpool2x2_fwd", xg, y, B, T, F_, C)
        assert _eq(y.t, pooled_ref)
        y2, idx = A.out("y2", y.shape), A.out("idx", y.shape, torch.uint8)
        A.call("maxpool2x2_fwd_idx", xg, y2, idx, B, T, F_, C)
        assert _eq(y2.t, pooled_ref) and _eq(idx.t, pos.to(torch.uint8))
        idx.freeze()
        codes = A.inp("codes", pool_codes(x))
        for name, src in (("maxpool2x2_bwd", xg), ("maxpool2x2_bwd_idx", idx), ("maxpool2x2_bwd_codes", codes)):
            dx, dx16 = A.out("dx_" + name, (B, T, F_, C)), A.out("dx16_" + name, (2, B, T, F_, C), torch.int16)
            A.call(name, dyg, src, dx, dx16, B, T, F_, C, 1)
            assert _eq(dx.t.double() + 0.0, dx_ref + 0.0), name
            assert _eq(dx16.t, pairs_ref(dx.t)), name


# ================================================================================================ emb_cnn front end
# (B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW): output rows off every tile of the CUDA-core kernels, B = 1, a 1x1 output
CONV2D_GEOMS = [(2, 1, 41, 27, 32, 11, 5, 2, 2, 0, 2), (1, 32, 21, 9, 32, 5, 3, 2, 1, 1, 0), (1, 3, 4, 3, 5, 4, 3, 1, 1, 0, 0)]


@gpu
@pytest.mark.parametrize("geom", CONV2D_GEOMS, ids=str)
def test_conv2d_cuda_core(lib, geom):
    """conv2d_fwd / _bwd_data / _bwd_weight (with and without dbias) against float64 autograd."""
    B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW = geom
    x, w, b = _randn(B, Ci, H, W, seed=15), _randn(Co, Ci, KH, KW, seed=16, scale=0.2), _randn(Co, seed=17)
    x64, w64, b64 = (t.double().requires_grad_(True) for t in (x, w, b))
    y64 = F.conv2d(x64, w64, b64, stride=(SH, SW), padding=(PH, PW))
    dy = _randn(*y64.shape, seed=18)
    y64.backward(dy.double())
    args = (B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW)
    A = Arena(lib)
    xg, wg, bg, dyg = A.inp("x", x), A.inp("w", w), A.inp("b", b), A.inp("dy", dy)
    y = A.out("y", y64.shape)
    A.call("conv2d_fwd", xg, wg, bg, y, *args)
    assert rel_err(y.t, y64) < 2e-6
    dx = A.out("dx", x.shape)
    A.call("conv2d_bwd_data", dyg, wg, dx, *args)
    assert rel_err(dx.t, x64.grad) < 2e-6
    for with_bias in (True, False):
        dw, db = A.out("dw", w.shape), (A.out("dbias", (Co,)) if with_bias else None)
        A.call("conv2d_bwd_weight", dyg, xg, dw, db, *args)
        assert rel_err(dw.t, w64.grad) < 2e-6
        if with_bias:
            assert rel_err(db.t, b64.grad) < 2e-6


@gpu
@pytest.mark.parametrize("B,C,F_,T", [(1, 1, 1, 1), (2, 32, 5, 7), (3, 3, 17, 33)])
def test_flatten_and_permute(lib, B, C, F_, T):
    """flatten_bcft_fwd / _bwd and permute_cols_cf (both directions): exact permutations."""
    x = _randn(B, C, F_, T, seed=19)
    for shift in (0, 16):
        A = Arena(lib, shift)
        xg = A.inp("x", x)
        y = A.out("y", (B, T, C * F_))
        A.call("flatten_bcft_fwd", xg, y, B, C, F_, T)
        want = x.permute(0, 3, 1, 2).reshape(B, T, C * F_)
        assert _eq(y.t, want)
        y.freeze()
        dx = A.out("dx", x.shape)
        A.call("flatten_bcft_bwd", y, dx, B, C, F_, T)
        assert _eq(dx.t, x)
        rows = B * T
        src = A.inp("src", want.reshape(rows, C * F_))
        for inverse in (0, 1):
            dst = A.out(f"dst{inverse}", (rows, C * F_))
            A.call("permute_cols_cf", src, dst, rows, C, F_, inverse)
            s = want.reshape(rows, C, F_)
            expect = (s.reshape(rows, F_, C) if inverse else s).transpose(1, 2).reshape(rows, -1)
            assert _eq(dst.t, expect), inverse


# (B, C, H, W, x_pitch, y_pitch): rows = B*H below, off and above the 32 row splits; pitches wider than W
BN_SHAPES = [(1, 32, 5, 7, 7, 9), (3, 32, 23, 11, 12, 16), (1, 1, 1, 5, 8, 6), (2, 3, 40, 5, 8, 5)]


@gpu
@pytest.mark.parametrize("shape", BN_SHAPES, ids=str)
@pytest.mark.parametrize("shift", [0, 16])
def test_bn_clamp(lib, shape, shift):
    """bn_clamp_fwd (training, running statistics) and bn_clamp_bwd with their bn_ws_bytes partials: y / dx in rows with
    gap columns, the statistics, the running state and the gradients against float64."""
    B, C, H, W, xp, yp = shape
    lo, hi, eps, mom = -1.5, 1.5, 1e-5, 0.1
    x, gamma, beta = _randn(B, C, H, W, seed=20, scale=2.0) + 0.5, _randn(C, seed=21), _randn(C, seed=22)
    rm, rv = _randn(C, seed=23), _randn(C, seed=24).abs() + 0.5
    dy = _randn(B, C, H, W, seed=25)
    x64, g64, b64 = (t.double().requires_grad_(True) for t in (x, gamma, beta))
    y64 = F.hardtanh(F.batch_norm(x64, None, None, g64, b64, True, 0.0, eps), lo, hi)
    y64.backward(dy.double())
    mean = x.double().mean((0, 2, 3))
    var = x.double().var((0, 2, 3), unbiased=False)
    n = B * H * W
    A = Arena(lib, shift)
    xg = A.inp("x", x, pitch=xp)
    gg, bg = A.inp("gamma", gamma), A.inp("beta", beta)
    y, mg, ig = A.out("y", x.shape, pitch=yp), A.out("mean", (C,)), A.out("invstd", (C,))
    rmg, rvg = A.inout("running_mean", rm), A.inout("running_var", rv)
    nbt = A.inout("num_batches_tracked", torch.tensor([5], dtype=torch.int64, device="cuda"))
    ws = A.ws("ws", lib.b200asr_bn_ws_bytes(C))
    A.call("bn_clamp_fwd", xg, gg, bg, y, mg, ig, rmg, rvg, nbt, ws, B, C, H, W, xp, yp, eps, mom, 1, lo, hi)
    assert rel_err(y.t, y64) < 2e-6
    assert rel_err(mg.t, mean) < 1e-6 and rel_err(ig.t, 1 / (var + eps).sqrt()) < 1e-6
    unb = var * n / max(n - 1, 1)
    assert rel_err(rmg.t, 0.9 * rm.double() + 0.1 * mean) < 1e-6
    if n > 1:
        assert rel_err(rvg.t, 0.9 * rv.double() + 0.1 * unb) < 1e-5
    assert int(nbt.t.item()) == 6
    for g in (y, mg, ig):
        g.freeze()
    dyg = A.inp("dy", dy, pitch=xp)
    dx, dg, db = A.out("dx", x.shape, pitch=yp), A.out("dgamma", (C,)), A.out("dbeta", (C,))
    A.call("bn_clamp_bwd", dyg, xg, y, gg, mg, ig, dx, dg, db, ws, B, C, H, W, xp, xp, yp, yp, 1, lo, hi)
    assert rel_err(dx.t, x64.grad) < 2e-5
    assert rel_err(dg.t, g64.grad) < 2e-5 and rel_err(db.t, b64.grad) < 2e-5


@gpu
@pytest.mark.parametrize("shift", [0, 16])
@pytest.mark.parametrize("mode", ["plain", "dropout", "accumulate"])
@pytest.mark.parametrize("rows,d", [(1, 4), (37, 200), (130, 1024), (3, 64)])
def test_add_ln(lib, rows, d, mode, shift):
    """add_ln_fwd (residual, post_add, row_scale, z, mean, rstd) and add_ln_bwd (dgamma, dbeta, the add_ln_bwd_ws_bytes
    partials) against float64.  plain: dx == dz, one buffer.  dropout: no residual, p = 0.2 -- the keep mask read back
    from the saved z (z = x / (1-p) bit for bit where kept), dx a separate guarded output equal to dz * keep / (1-p).
    accumulate: dgamma / dbeta added into existing values, as into the parameters' views of the flat gradient buffer."""
    p = 0.2 if mode == "dropout" else 0.0
    x, res = _randn(rows, d, seed=26), (None if p else _randn(rows, d, seed=27))
    gamma, beta, post = _randn(d, seed=28), _randn(d, seed=29), _randn(3, d, seed=30)
    rs = (torch.rand(rows, generator=_gen(31)) > 0.2).float().cuda()
    dy = _randn(rows, d, seed=32)
    g0, b0 = _randn(d, seed=33), _randn(d, seed=34)
    A = Arena(lib, shift)
    xg, gg, bg, pg, sg = (A.inp(n, t) for n, t in (("x", x), ("gamma", gamma), ("beta", beta), ("post_add", post),
                                                    ("row_scale", rs)))
    rg = None if res is None else A.inp("residual", res)
    y, z, mean, rstd = A.out("y", (rows, d)), A.out("z", (rows, d)), A.out("mean", (rows,)), A.out("rstd", (rows,))
    A.call("add_ln_fwd", xg, rg, gg, bg, pg, 3, sg, y, z, mean, rstd, rows, d, 1e-5, p, SEED, OFFSET)
    if p:
        ik = _inv_keep(p)
        keep = z.t != 0
        assert torch.equal(z.t[keep], (x * ik)[keep]) and not z.t[~keep].any()
        if rows * d > 1000:
            assert 0.7 < float(keep.float().mean()) < 0.9
        z_ref = x.double() * keep * ik
    else:
        z_ref = (x + res).double()
    z64 = z_ref.clone().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    y64 = (F.layer_norm(z64, (d,), g64, b64, 1e-5) + post.double()[torch.arange(rows) % 3]) * rs.double()[:, None]
    y64.backward(dy.double())
    assert rel_err(y.t, y64) < 4e-6 and rel_err(z.t, z_ref) < 1e-7
    assert rel_err(mean.t, z_ref.mean(1)) < 5e-7
    assert rel_err(rstd.t, 1 / (z_ref.var(1, unbiased=False) + 1e-5).sqrt()) < 5e-7
    for g in (z, mean, rstd):
        g.freeze()
    dyg = A.inp("dy", dy)
    dz = A.out("dz", (rows, d))
    dx = A.out("dx", (rows, d)) if p else dz
    acc = int(mode == "accumulate")
    dg, db = (A.inout("dgamma", g0), A.inout("dbeta", b0)) if acc else (A.out("dgamma", (d,)), A.out("dbeta", (d,)))
    ws = A.ws("ws", lib.b200asr_add_ln_bwd_ws_bytes(rows, d))
    A.call("add_ln_bwd", dyg, z, gg, mean, rstd, sg, dz, dx, dg, db, ws, rows, d, p, SEED, OFFSET, acc)
    assert rel_err(dz.t, z64.grad) < 1.2e-6
    if p:
        assert torch.equal(dx.t, torch.where(keep, dz.t * ik, torch.zeros_like(dz.t)))
        assert rel_err(dx.t, z64.grad * keep * ik) < 1.2e-6
    base_g, base_b = (g0.double(), b0.double()) if acc else (0.0, 0.0)
    assert rel_err(dg.t, base_g + g64.grad) < 4e-6 and rel_err(db.t, base_b + b64.grad) < 4e-6


# ================================================================================================ attention
def _attn_inputs(B, H, Tq, Tk, dk, dv, mode, seed):
    """q, k, v, dout token-major [B, T, H*d] and the union of the masks of `mode` as a bool [B, Tq, Tk] (True = masked),
    plus the (key_pad, dense, causal) arguments that express it: key padding with the second utterance shorter, causal,
    or a dense mask that leaves every row a key."""
    q, k, v = _randn(B, Tq, H * dk, seed=seed), _randn(B, Tk, H * dk, seed=seed + 1), _randn(B, Tk, H * dv, seed=seed + 2)
    dout = _randn(B, Tq, H * dv, seed=seed + 3)
    key_pad = dense = None
    mask = torch.zeros(B, Tq, Tk, dtype=torch.bool, device="cuda")
    if mode == "key_pad":
        lens = [Tk] + [max(1, Tk - 5)] * (B - 1)
        key_pad = (torch.arange(Tk)[None, :] >= torch.tensor(lens)[:, None]).to(torch.uint8).cuda()
        mask |= key_pad.bool()[:, None, :]
    if mode == "causal":
        mask |= (torch.arange(Tk)[None, :] > torch.arange(Tq)[:, None]).cuda()[None]
    if mode == "dense":
        dense = (torch.rand(B, Tq, Tk, generator=_gen(seed + 4)) < 0.3).to(torch.uint8)
        dense[:, torch.arange(Tq), torch.arange(Tq) % Tk] = 0
        dense = dense.cuda()
        mask |= dense.bool()
    return q, k, v, dout, mask, (key_pad, dense, int(mode == "causal"))


def _heads(t, H):
    B, T, HD = t.shape
    return t.reshape(B, T, H, HD // H).permute(0, 2, 1, 3)


def _attn_ref(q, k, v, dout_bhtd, mask, H, scale, keep=None, inv_keep=1.0):
    """float64 masked softmax attention with an optional dropout keep mask [B, H, Tq, Tk]: (out [B, H, Tq, dv], lse, P,
    dq / dk / dv token-major [B, T, H*d])."""
    q64, k64, v64 = (_heads(t.double(), H).requires_grad_(True) for t in (q, k, v))
    s = torch.matmul(q64, k64.transpose(-1, -2)) * scale
    s = s.masked_fill(mask[:, None], float("-inf"))
    p = torch.softmax(s, -1)
    pd = p * keep.double() * inv_keep if keep is not None else p
    o = torch.matmul(pd, v64)
    o.backward(dout_bhtd.double())
    back = lambda t: t.permute(0, 2, 1, 3).reshape(t.shape[0], t.shape[2], -1)
    return o.detach(), torch.logsumexp(s.detach(), -1), p.detach(), back(q64.grad), back(k64.grad), back(v64.grad)


def _tm(g, H, d):
    """(batch, head, row) strides of a token-major [B, T, H*d] guarded tensor (row pitch g.pitch)."""
    s = g.t.stride()
    return s[0], d, s[1]


class _AttnOut:
    """An attention output (or dout) in one of the two layouts the library serves: token-major [B, Tq, H*dv] in rows of
    H*dv + 12 floats, or head-major [H, B, Tq, dv] (the reference's (H*B) x Tq x dv memory, ops.py head_major_out) in
    rows of dv + 4 floats; the gap columns are guarded."""

    def __init__(self, A, name, layout, B, H, Tq, dv, fill=None):
        self.layout, self.H = layout, H
        if layout == "token":
            shape, pitch = (B, Tq, H * dv), H * dv + 12
        else:
            shape, pitch = (H, B, Tq, dv), dv + 4
        if fill is not None:
            self.g = A.inp(name, fill.permute(0, 2, 1, 3).reshape(shape) if layout == "token" else fill.permute(1, 0, 2, 3),
                           pitch=pitch)
        else:
            self.g = A.out(name, shape, pitch=pitch)
        s = self.g.t.stride()
        self.strides = (s[0], dv, s[1]) if layout == "token" else (s[1], s[0], s[2])

    def bhtd(self):
        t = self.g.t
        return _heads(t, self.H) if self.layout == "token" else t.permute(1, 0, 2, 3)


def _mat_keep(lib, q, k, v, H, d, masks, scale, p):
    """The dropout keep mask [B, H, Tq, Tk] of the counter stream at (SEED, OFFSET), read back from the probs_drop of a plain
    sdpa_mat_fwd call -- every attention path draws the same mask.  Exact where P != 0 (elsewhere it does not matter)."""
    B, Tq, Tk = q.shape[0], q.shape[1], k.shape[1]
    Tk4 = _round_up(Tk, 4)
    probs, pd = (torch.full((B, H, Tq, Tk4), NAN, device="cuda") for _ in range(2))
    out = torch.empty(B, Tq, H * d, device="cuda")
    key_pad, dense, causal = masks
    st = (Tq * H * d, d, H * d)
    ks = (Tk * H * d, d, H * d)
    rc = lib.b200asr_sdpa_mat_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), *st, *ks, *ks,
                                  None if key_pad is None else key_pad.data_ptr(), None if dense is None else dense.data_ptr(),
                                  causal, out.data_ptr(), *st, probs.data_ptr(), pd.data_ptr(), B, H, Tq, Tk, d, d, scale, p,
                                  SEED, OFFSET, 3, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0
    return pd[..., :Tk] != 0


FLASH_BARS = {0: dict(o=3.5e-6, lse=6e-7, grad=3e-6), 1: dict(o=2.5e-3, lse=3e-3, grad=4e-3),
              "fused": dict(o=4.5e-5, lse=4e-5, grad=6e-5)}
# (B, H, Tq, Tk): one query / one key; Tq, Tk off every 64- and 128-row block; mask, dropout and out layout per case
ATTN_CASES = [((1, 1, 1, 1), "key_pad", 0.0, "token"), ((2, 2, 129, 77), "key_pad", 0.2, "head"),
              ((1, 2, 37, 130), "causal", 0.0, "head"), ((2, 1, 65, 33), "dense", 0.2, "token")]
# head dims per path: fp32 every one, the TF32 flash kernels 32 / 64, the fused bf16x3 kernels 64
FLASH_CASES = [(path, (*bhtt, d), mode, p if d % 32 == 0 else 0.0, layout)
               for path, ds in ((0, (64, 16, 128)), (1, (64, 32)), ("fused", (64,)))
               for d in ds for bhtt, mode, p, layout in ATTN_CASES]


@gpu
@pytest.mark.parametrize("shift", [0, 16])
@pytest.mark.parametrize("path,shape,mode,p_drop,layout", FLASH_CASES, ids=str)
def test_sdpa_flash(lib, path, shape, mode, p_drop, layout, shift):
    """sdpa_fwd / _bwd (fp32, tf32) and sdpa_fused_fwd / _bwd (bf16x3, both workspaces): q, k, v and their gradients
    token-major in rows wider than H*d, out / dout token- or head-major, with guard bytes in every gap column; key-padding,
    causal and dense masks; dropout (its keep mask read back from the materialised path's probs_drop, the same counter
    stream) in the forward and regenerated by the backward."""
    B, H, Tq, Tk, d = shape
    scale = 1.0 / math.sqrt(d)
    q, k, v, dout, mask, masks = _attn_inputs(B, H, Tq, Tk, d, d, mode, seed=40)
    keep = _mat_keep(lib, q, k, v, H, d, masks, scale, p_drop) if p_drop > 0 else None
    ik = _inv_keep(p_drop) if p_drop > 0 else 1.0
    o_ref, lse_ref, _, dq_ref, dk_ref, dv_ref = _attn_ref(q, k, v, _heads(dout, H), mask, H, scale, keep, ik)
    pitch = H * d + 8
    A = Arena(lib, shift)
    qg, kg, vg = (A.inp(n, t, pitch=pitch) for n, t in (("q", q), ("k", k), ("v", v)))
    mg = [None if m is None else A.inp(n, m) for n, m in (("key_pad", masks[0]), ("dense_mask", masks[1]))]
    out, lse = _AttnOut(A, "out", layout, B, H, Tq, d), A.out("lse", (B, H, Tq))
    strides = (*_tm(qg, H, d), *_tm(kg, H, d), *_tm(vg, H, d))
    dims = (B, H, Tq, Tk, d, d, scale, p_drop, SEED, OFFSET)
    bars = FLASH_BARS[path]
    if path == "fused":
        ws16 = A.ws("ws16", lib.b200asr_sdpa_fused_ws_bytes(B, H, Tq, Tk))
        A.call("sdpa_fused_fwd", qg, kg, vg, *strides, *mg, masks[2], out.g, *out.strides, lse, ws16, *dims)
    else:
        A.call("sdpa_fwd", qg, kg, vg, *strides, *mg, masks[2], out.g, *out.strides, lse, *dims, path)
    assert rel_err(out.bhtd(), o_ref) < bars["o"] and rel_err(lse.t, lse_ref) < bars["lse"]
    out.g.freeze()
    lse.freeze()
    dog = _AttnOut(A, "dout", layout, B, H, Tq, d, fill=_heads(dout, H))
    dq, dk, dv = (A.out(n, t.shape, pitch=pitch) for n, t in (("dq", q), ("dk", k), ("dv", v)))
    head = (dog.g, qg, kg, vg, out.g, lse, *strides, *out.strides, *mg, masks[2], dq, dk, dv)
    if path == "fused":
        ws16.freeze()
        wsb = A.ws("ws_bwd", lib.b200asr_sdpa_fused_bwd_ws_bytes(B, H, Tq))
        A.call("sdpa_fused_bwd", *head, ws16, wsb, *dims)
    else:
        delta = A.out("delta_ws", (B, H, Tq))
        A.call("sdpa_bwd", *head, delta, *dims, path)
    for got, ref in ((dq, dq_ref), (dk, dk_ref), (dv, dv_ref)):
        assert rel_err(got.t, ref) < bars["grad"], got.name


MAT_BARS = {3: dict(p=1e-5, o=7e-5, grad=7e-5), 1: dict(p=2e-3, o=2.5e-3, grad=3e-3)}
MAT_CASES = [((1, 1, 1, 1, 32), "key_pad", 0.0, "token"), ((2, 2, 129, 77, 64), "key_pad", 0.2, "head"),
             ((1, 3, 5, 130, 32), "causal", 0.2, "token"), ((2, 1, 37, 33, 96), "dense", 0.0, "head"),
             ((1, 1, 1, 1, 32), "key_pad", 0.2, "token")]


@gpu
@pytest.mark.parametrize("shift", [0, 16])
@pytest.mark.parametrize("shape,mode,p_drop,layout", MAT_CASES, ids=str)
@pytest.mark.parametrize("prec", [1, 3])
def test_sdpa_materialised(lib, prec, shape, mode, p_drop, layout, shift):
    """sdpa_mat_fwd / _bwd with probs, probs_drop (p_drop > 0) and dP of sdpa_mat_ws_bytes each (the padding columns
    Tk .. round_up(Tk, 4) - 1 belong to them), strided q, k, v, gradients and token- or head-major out / dout.  probs_drop
    equals probs * 1/(1-p) bit for bit wherever it is nonzero and is 0 in the padding columns; the keep mask read back from
    it reproduces out and the gradients of the float64 reference, so the backward applies the forward's mask."""
    B, H, Tq, Tk, d = shape
    scale = 1.0 / math.sqrt(d)
    q, k, v, dout, mask, masks = _attn_inputs(B, H, Tq, Tk, d, d, mode, seed=50)
    pitch, Tk4 = H * d + 8, _round_up(Tk, 4)
    nws = lib.b200asr_sdpa_mat_ws_bytes(B, H, Tq, Tk)
    assert nws == 4 * B * H * Tq * Tk4
    A = Arena(lib, shift)
    qg, kg, vg = (A.inp(n, t, pitch=pitch) for n, t in (("q", q), ("k", k), ("v", v)))
    mg = [None if m is None else A.inp(n, m) for n, m in (("key_pad", masks[0]), ("dense_mask", masks[1]))]
    out, probs = _AttnOut(A, "out", layout, B, H, Tq, d), A.out("probs", (B, H, Tq, Tk4))
    pdrop = A.out("probs_drop", (B, H, Tq, Tk4)) if p_drop > 0 else None
    strides = (*_tm(qg, H, d), *_tm(kg, H, d), *_tm(vg, H, d))
    dims = (B, H, Tq, Tk, d, d, scale, p_drop, SEED, OFFSET, prec)
    A.call("sdpa_mat_fwd", qg, kg, vg, *strides, *mg, masks[2], out.g, *out.strides, probs, pdrop, *dims)
    keep, ik = None, 1.0
    if p_drop > 0:
        ik = _inv_keep(p_drop)
        P, Pd = probs.t, pdrop.t
        nz = Pd != 0
        assert torch.equal(Pd[nz], (P * ik)[nz]) and not Pd[..., Tk:].any()
        keep = nz[..., :Tk]
        if P.numel() > 1000:
            assert 0.7 < float(keep[P[..., :Tk] != 0].float().mean()) < 0.9
    o_ref, _, p_ref, dq_ref, dk_ref, dv_ref = _attn_ref(q, k, v, _heads(dout, H), mask, H, scale, keep, ik)
    bars = MAT_BARS[prec]
    assert rel_err(out.bhtd(), o_ref) < bars["o"] and rel_err(probs.t[..., :Tk], p_ref) < bars["p"]
    probs.freeze()
    out.g.freeze()
    if pdrop is not None:
        pdrop.freeze()
    dog = _AttnOut(A, "dout", layout, B, H, Tq, d, fill=_heads(dout, H))
    dq, dk, dv = (A.out(n, t.shape, pitch=pitch) for n, t in (("dq", q), ("dk", k), ("dv", v)))
    dp = A.ws("dp_ws", nws)
    A.call("sdpa_mat_bwd", dog.g, qg, kg, vg, *strides, *dog.strides, probs, pdrop, dq, dk, dv, dp, *dims)
    for got, ref in ((dq, dq_ref), (dk, dk_ref), (dv, dv_ref)):
        assert rel_err(got.t, ref) < bars["grad"], got.name


@gpu
@pytest.mark.parametrize("Tk", [1, 129, 2048, 2049])
@pytest.mark.parametrize("R,H,d", [(1, 1, 64), (3, 2, 32), (2, 4, 128)])
@pytest.mark.parametrize("shift", [0, 16])
def test_decode_attn(lib, R, H, d, Tk, shift):
    """decode_attn with its chunk partials in exactly decode_attn_ws_bytes (a guard-only buffer when that is 0), K / V
    token-major in rows wider than H*d (gap columns guarded): against float64."""
    scale = 1.0 / math.sqrt(d)
    q = _randn(R, H * d, seed=60)
    k, v = _randn(R, Tk, H * d, seed=61), _randn(R, Tk, H * d, seed=62)
    s = torch.einsum("rhd,rjhd->rhj", q.double().view(R, H, d), k.double().view(R, Tk, H, d)) * scale
    ref = torch.einsum("rhj,rjhd->rhd", torch.softmax(s, -1), v.double().view(R, Tk, H, d)).reshape(R, H * d)
    pitch = H * d + 12
    A = Arena(lib, shift)
    qg, kg, vg = A.inp("q", q), A.inp("k", k, pitch=pitch), A.inp("v", v, pitch=pitch)
    out = A.out("out", (R, H * d))
    ws = A.ws("ws", lib.b200asr_decode_attn_ws_bytes(R, H, Tk, d))
    A.call("decode_attn", qg, kg, vg, out, ws, R, H, d, d, Tk, Tk * pitch, pitch, Tk * pitch, pitch, scale)
    assert rel_err(out.t, ref) < 6e-6


@gpu
@pytest.mark.parametrize("t", [0, 6])
@pytest.mark.parametrize("B,W,H,dk,dv", [(1, 1, 1, 16, 16), (2, 3, 2, 64, 32), (1, 5, 4, 128, 64)])
@pytest.mark.parametrize("shift", [0, 16])
def test_beam_self_attn(lib, B, W, H, dk, dv, t, shift):
    """beam_self_attn over the K/V cache slabs through the per-row index table: against float64."""
    R, stride, steps = B * W, t + 3, t + 2
    q = _randn(R, H * dk, seed=70)
    kc, vc = _randn(steps, R, H * dk, seed=71), _randn(steps, R, H * dv, seed=72)
    idx = torch.randint(0, W, (R, stride), generator=_gen(73), dtype=torch.int32).cuda()
    scale = 1.0 / math.sqrt(dk)
    rows = (torch.arange(R)[:, None] // W * W).cuda() + idx[:, :t + 1].long()              # [R, t+1] cache rows
    pos = torch.arange(t + 1).cuda()[None, :].expand(R, -1)
    K = kc.double()[pos, rows].view(R, t + 1, H, dk)
    V = vc.double()[pos, rows].view(R, t + 1, H, dv)
    s = torch.einsum("rhd,rjhd->rhj", q.double().view(R, H, dk), K) * scale
    ref = torch.einsum("rhj,rjhd->rhd", torch.softmax(s, -1), V).reshape(R, H * dv)
    A = Arena(lib, shift)
    qg, kg, vg, ig = A.inp("q", q), A.inp("k_cache", kc), A.inp("v_cache", vc), A.inp("idx", idx)
    out = A.out("out", (R, H * dv))
    A.call("beam_self_attn", qg, kg, vg, ig, out, R, H, W, dk, dv, t, stride, scale)
    assert rel_err(out.t, ref) < 6e-6


# ================================================================================================ beam search
def _word_tab(V, seed):
    return torch.randint(0, 32, (V,), generator=_gen(seed), dtype=torch.int32)


def ref_beam_step(logits, recs, W, t, t_eos, nbest, c_weight, score, state, idx_cur, pool):
    """float64 restatement of one b200asr_beam_step (the host restatement of tests/test_gpu_beam_search.py), plus the end
    log of every ended hypothesis (b200asr_beam_step_log)."""
    B = logits.shape[0] // W
    lg = logits.double().cpu()
    exp = dict(score=score.clone(), state=state.clone(), tok={}, idx={}, hist={}, pool=[list(p) for p in pool], died=0,
               ends=[[] for _ in range(B)])
    for b in range(B):
        live = [j for j in range(W) if state[b * W + j, 0]]
        cands = []
        for j in live:
            x = lg[b * W + j]
            lp = (x - torch.logsumexp(x, 0)).tolist()
            order = sorted(range(len(lp)), key=lambda v: (-lp[v], v))[:W]
            cands += [(float(score[b * W + j]) + lp[v], j * W + r, v, j) for r, v in enumerate(order)]
        kept = sorted(cands, key=lambda c: (-c[0], c[1]))[:W]
        n = 0
        for k, (s, _, v, j) in enumerate(kept):
            words, tail = int(state[b * W + j, 1]), int(state[b * W + j, 2])
            r = int(recs[v])
            words += (r >> 3) - (tail & ((r >> 2) & 1))
            if not r & 1:
                tail = (r >> 1) & 1
            exp["hist"][(b, k)] = (v, int(state[b * W + j, 3]))
            if t == t_eos or v == O.EOS:
                fs = s + math.sqrt(words) * c_weight
                p = exp["pool"][b]
                pos = 0
                while pos < len(p) and not fs > p[pos][0]:
                    pos += 1
                ref = ((t * W + k) << 1) | (t == t_eos)
                p.insert(pos, (fs, s, ref))
                del p[nbest:]
                exp["ends"][b].append((ref, s))
            else:
                exp["score"][b * W + n] = s
                exp["state"][b * W + n] = torch.tensor([1, words, tail, k])
                exp["tok"][b * W + n] = v
                exp["idx"][b * W + n] = idx_cur[b * W + j, :t + 1].tolist() + [n]
                n += 1
        for s_ in range(n, W):
            exp["score"][b * W + s_] = float("-inf")
            exp["state"][b * W + s_] = torch.tensor([0, 0, 0, -1])
            exp["tok"][b * W + s_] = 0
            exp["idx"][b * W + s_] = [s_] * (t + 2)
        exp["died"] += int(len(kept) > 0 and n == 0)
    return exp


@gpu
@pytest.mark.parametrize("t,t_eos", [(0, 9), (3, 9), (4, 4)])
@pytest.mark.parametrize("B,W,V,nbest", [(1, 1, 5, 1), (2, 4, 33, 3), (3, 32, 65, 32)])
def test_beam_step(lib, B, W, V, nbest, t, t_eos):
    """beam_step and beam_step_log with every BeamBuffers / EndLog tensor guarded: scores, states, next tokens, index rows,
    history rows, pools and the end log against the float64 restatement.  EOS-topped rows and the forced EOS at t_eos
    fill the pools."""
    R, steps, c_weight = B * W, 10, 0.3
    stride = steps + 1
    g = _gen(B * 100 + W + t)
    logits = torch.randn(R, V, generator=g) * 3.0
    logits[::3, O.EOS] = logits[::3].max(1).values + 1.0
    tab = _word_tab(V, W)
    state = torch.zeros(R, 4, dtype=torch.int32)
    score = torch.full((R,), float("-inf"))
    for b in range(B):
        n = 1 if t == 0 else max(1, W - b)
        for j in range(n):
            state[b * W + j] = torch.tensor([1, int(torch.randint(0, 4, (1,), generator=g)), j % 2, j if t else -1])
            score[b * W + j] = -float(j) - float(torch.rand(1, generator=g))
        for j in range(n, W):
            state[b * W + j] = torch.tensor([0, 0, 0, -1])
    idx_cur = torch.full((R, stride), -1, dtype=torch.int32)
    idx_cur[:, :t + 1] = torch.randint(0, W, (R, t + 1), generator=g, dtype=torch.int32)
    pool = [[(-5.0 - i, -5.5 - i, 2 * i) for i in range(min(nbest - 1, 2))] for _ in range(B)]
    exp = ref_beam_step(logits, tab, W, t, t_eos, nbest, c_weight, score, state, idx_cur, pool)
    end_cap = W * steps
    for log in (False, True):
        A = Arena(lib)
        lg, tg, icur = A.inp("logits", logits.cuda()), A.inp("word_tab", tab.cuda()), A.inp("idx_cur", idx_cur.cuda())
        sc, stt = A.inout("score", score.cuda()), A.inout("state", state.cuda())
        tok = A.out("next_tok", (R,), torch.int64)
        inxt = A.out("idx_nxt", (R, stride), torch.int32, fill=-1)
        ht, hp = A.out("hist_tok", (steps, R), torch.int32, fill=-1), A.out("hist_par", (steps, R), torch.int32, fill=-1)
        ps, pf = torch.full((B, nbest), NAN), torch.full((B, nbest), NAN)
        pr, pn = torch.full((B, nbest), -1, dtype=torch.int32), torch.zeros(B, dtype=torch.int32)
        for b, p in enumerate(pool):
            for i, (fs, s, ref) in enumerate(p):
                pf[b, i], ps[b, i], pr[b, i] = fs, s, ref
            pn[b] = len(p)
        psg, pfg, prg, png = (A.inout(n, x.cuda()) for n, x in (("pool_score", ps), ("pool_final", pf), ("pool_ref", pr),
                                                               ("pool_n", pn)))
        nl = A.inout("n_live", torch.tensor([B], dtype=torch.int32, device="cuda"))
        args = (lg, tg, B, W, V, t, t_eos, steps, nbest, c_weight, sc, stt, tok, icur, inxt, stride, ht, hp, psg, pfg, prg, png, nl)
        if log:
            er = A.out("end_ref", (B, end_cap), torch.int32, fill=-1)
            es = A.out("end_score", (B, end_cap))
            en = A.inout("end_n", torch.zeros(B, dtype=torch.int32, device="cuda"))
            A.call("beam_step_log", *args, er, es, en, end_cap)
            for b in range(B):
                ends = exp["ends"][b]
                assert int(en.t[b]) == len(ends)
                assert er.t[b, :len(ends)].tolist() == [e[0] for e in ends] and bool((er.t[b, len(ends):] == -1).all())
                for i, (_, s) in enumerate(ends):
                    assert abs(float(es.t[b, i]) - s) <= 2e-6 * max(1.0, abs(s))
        else:
            A.call("beam_step", *args)
        st_, sc_ = stt.t.cpu(), sc.t.cpu()
        assert torch.equal(st_, exp["state"])
        live = exp["state"][:, 0] == 1
        if live.any():
            err = ((sc_[live].double() - exp["score"][live].double()).abs() / exp["score"][live].double().abs().clamp_min(1)).max()
            assert float(err) < 2e-6
        assert bool(torch.isinf(sc_[~live]).all())
        for r in range(R):
            assert int(tok.t[r]) == exp["tok"][r] and inxt.t[r, :t + 2].tolist() == exp["idx"][r], r
        for (b, k), (v, par) in exp["hist"].items():
            assert int(ht.t[t, b * W + k]) == v and int(hp.t[t, b * W + k]) == par
        for b in range(B):
            p = exp["pool"][b]
            assert int(png.t[b]) == len(p) and prg.t[b, :len(p)].tolist() == [e[2] for e in p]
            for i, (fs, s, _) in enumerate(p):
                assert abs(float(pfg.t[b, i]) - fs) <= 2e-6 * max(1.0, abs(fs))
                assert abs(float(psg.t[b, i]) - s) <= 2e-6 * max(1.0, abs(s))
        assert int(nl.t.item()) == B - exp["died"]


@gpu
@pytest.mark.parametrize("B,W,nbest,steps", [(1, 1, 1, 1), (2, 4, 3, 7), (3, 32, 32, 5)])
def test_beam_backtrack(lib, B, W, nbest, steps):
    """beam_backtrack (ids [B][nbest][steps + 2], lengths) and beam_backtrack_packed (ids sized exactly by the entries'
    refs) against a host walk along the back-pointers; forced and unforced ends, empty pool slots."""
    g = _gen(B * W + steps)
    R = B * W
    hist_tok = torch.randint(3, 50, (steps, R), generator=g, dtype=torch.int32)
    hist_par = torch.randint(0, W, (steps, R), generator=g, dtype=torch.int32)
    refs = torch.full((B, nbest), -1, dtype=torch.int32)
    counts = torch.zeros(B, dtype=torch.int32)
    for b in range(B):
        n = min(nbest, b + 1)
        counts[b] = n
        for i in range(n):
            tt, k = int(torch.randint(0, steps, (1,), generator=g)), int(torch.randint(0, W, (1,), generator=g))
            refs[b, i] = ((tt * W + k) << 1) | (i % 2)

    def walk(b, ref):
        forced, tt = ref & 1, (ref >> 1) // W
        k = (ref >> 1) - tt * W
        toks = []
        for s in range(tt, -1, -1):
            toks.append(int(hist_tok[s, b * W + k]))
            k = int(hist_par[s, b * W + k])
        return [O.SOS] + toks[::-1] + ([O.EOS] if forced else [])

    A = Arena(lib)
    htg, hpg, rg, cg = (A.inp(n, x.cuda()) for n, x in (("hist_tok", hist_tok), ("hist_par", hist_par), ("pool_ref", refs),
                                                         ("pool_n", counts)))
    ids, lens = A.out("ids", (B, nbest, steps + 2), torch.int64), A.out("lengths", (B, nbest), torch.int64)
    A.call("beam_backtrack", htg, hpg, rg, cg, ids, lens, B, W, nbest, steps)
    want = []
    for b in range(B):
        for i in range(nbest):
            seq = walk(b, int(refs[b, i])) if i < counts[b] else []
            assert int(lens.t[b, i]) == len(seq)
            assert ids.t[b, i].tolist() == seq + [-1] * (steps + 2 - len(seq)), (b, i)
            if seq:
                want.append((b * nbest + i, seq))
    want = want[::-1]                                          # any order
    entries = torch.tensor([e for e, _ in want], dtype=torch.int64)
    sizes = [len(s) for _, s in want]
    offsets = torch.tensor([0] + list(np.cumsum(sizes)[:-1]), dtype=torch.int64)
    eg, og = A.inp("entries", entries.cuda()), A.inp("offsets", offsets.cuda())
    packed = A.out("packed_ids", (sum(sizes),), torch.int64)
    A.call("beam_backtrack_packed", htg, hpg, rg, cg, nbest, eg, og, len(want), packed, B, W, steps)
    assert packed.t.tolist() == [x for _, s in want for x in s]


@gpu
@pytest.mark.parametrize("rows,V", [(1, 1), (1, 1025), (37, 33), (5, 4097)])
def test_argmax_and_greedy_step(lib, rows, V):
    """argmax_rows and greedy_step (next token, the ys column of step t, finished flags): first index of the maximum."""
    x = _randn(rows, V, seed=80)
    am = x.cpu().numpy().argmax(1)
    A = Arena(lib)
    xg = A.inp("logits", x)
    out = A.out("out", (rows,), torch.int64)
    A.call("argmax_rows", xg, out, rows, V)
    assert out.t.cpu().tolist() == am.tolist()
    steps, t = 4, 2
    nxt = A.out("next_tok", (rows,), torch.int64)
    ys = A.inout("ys", torch.full((rows, steps), 9, dtype=torch.int64, device="cuda"))
    fin = A.inout("finished", torch.zeros(rows, dtype=torch.int32, device="cuda"))
    nfin = A.inout("n_finished", torch.zeros(1, dtype=torch.int32, device="cuda"))
    A.call("greedy_step", xg, nxt, ys, fin, nfin, rows, V, t, steps)
    assert nxt.t.cpu().tolist() == am.tolist()
    exp_ys = torch.full((rows, steps), 9, dtype=torch.int64)
    exp_ys[:, t] = torch.from_numpy(np.where(am == O.EOS, -1, am))
    assert _eq(ys.t, exp_ys)
    eos = torch.from_numpy(am == O.EOS)
    assert _eq(fin.t.bool(), eos) and int(nfin.t.item()) == int(eos.sum())


@gpu
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("rows,V", [(1, 2), (37, 1025), (3, 4097)])
def test_cross_entropy(lib, rows, V, eps):
    """ce_fwd (row_lse, stats[0..2]), ce_finalize (stats[3..4], loss) and ce_bwd against float64; V one past a power of
    two, rows = 1, PAD rows."""
    x = _randn(rows, V, seed=81)
    gold = torch.randint(1, V, (rows,), generator=_gen(82))
    gold[1::4] = O.PAD
    x64 = x.double().requires_grad_(True)
    lse_ref = torch.logsumexp(x64, 1)
    logp = x64 - lse_ref[:, None]
    if eps > 0:
        wts = torch.full_like(x64, eps / V).scatter_(1, gold.cuda().view(-1, 1), 1.0 - eps)
        loss = -(wts * logp).sum(1)
    else:
        loss = -logp.gather(1, gold.cuda().view(-1, 1)).squeeze(1)
    valid = (gold != O.PAD).cuda()
    loss = torch.where(valid, loss, 0.0)
    loss.sum().backward()
    n = int(valid.sum())
    correct = int(((x.argmax(1) == gold.cuda()) & valid).sum())
    A = Arena(lib)
    xg, gg = A.inp("logits", x), A.inp("gold", gold.cuda())
    lse, stats, lo = A.out("row_lse", (rows,)), A.out("stats", (5,)), A.out("loss_out", (1,))
    A.call("ce_fwd", xg, gg, lse, stats, rows, V, eps)
    assert rel_err(lse.t, lse_ref.detach()) < 3e-7
    s = stats.t.cpu()
    assert rel_err(s[0:1], loss.detach().sum().view(1)) < 5e-7 and s[1] == n and s[2] == correct
    A.call("ce_finalize", stats, lo, 1)
    if n:
        assert rel_err(stats.t[3:4], (loss.detach().sum() / n).view(1)) < 5e-7 and lo.t.item() == stats.t[3].item()
    lse.freeze()
    gdev = A.inp("gscale_dev", torch.tensor([0.25], device="cuda"))
    gdev2 = A.inp("gscale_dev2", torch.tensor([3.0], device="cuda"))
    dl = A.out("dlogits", (rows, V))
    A.call("ce_bwd", xg, gg, lse, dl, rows, V, eps, 0.5, gdev, gdev2)
    assert rel_err(dl.t, x64.grad * 0.375) < 2.5e-5


@gpu
@pytest.mark.parametrize("rows,T,d,V", [(1, 1, 4, 2), (37, 5, 200, 1025), (4, 4, 512, 33)])
@pytest.mark.parametrize("shift", [0, 16])
def test_embedding(lib, rows, T, d, V, shift):
    """embed_fwd (table * scale + pe) and embed_bwd (scatter into dtable, PAD rows skipped) against float64."""
    tok = torch.randint(0, V, (rows,), generator=_gen(83)).cuda()
    table, pe, dout = _randn(V, d, seed=84), _randn(T, d, seed=85), _randn(rows, d, seed=86)
    scale = math.sqrt(d)
    A = Arena(lib, shift)
    tg, tab, peg, dog = A.inp("tokens", tok), A.inp("table", table), A.inp("pe", pe), A.inp("dout", dout)
    out = A.out("out", (rows, d))
    A.call("embed_fwd", tg, tab, peg, out, rows, T, d, V, scale, 0.0, 13, 2)
    ref = table.double()[tok] * scale + pe.double()[torch.arange(rows).cuda() % T]
    assert rel_err(out.t, ref) < 3e-7
    dt = A.inout("dtable", torch.zeros(V, d, device="cuda"))
    A.call("embed_bwd", tg, dog, dt, rows, d, V, scale, 0.0, 13, 2, O.PAD)
    want = torch.zeros(V, d, dtype=torch.float64, device="cuda")
    keep = tok != O.PAD
    want.index_add_(0, tok[keep], dout.double()[keep] * scale)
    assert rel_err(dt.t, want) < 1e-6


@gpu
@pytest.mark.parametrize("B,L,Tt", [(1, 1, 2), (3, 7, 9), (5, 12, 13)])
def test_target_preprocessing_and_masks(lib, B, L, Tt):
    """preprocess_targets (seq_in, seq_out, key_pad, non_pad, status) and length_masks: exact."""
    g = _gen(B + L)
    lens = [L] + [int(torch.randint(0, L + 1, (1,), generator=g)) for _ in range(B - 1)]
    tgt = torch.zeros(B, L, dtype=torch.int64)
    for b, n in enumerate(lens):
        tgt[b, :n] = torch.randint(3, 30, (n,), generator=g)
    seq_in = torch.full((B, Tt), O.EOS, dtype=torch.int64)
    seq_out = torch.full((B, Tt), O.PAD, dtype=torch.int64)
    for b, n in enumerate(lens):
        seq_in[b, 0], seq_in[b, 1:n + 1] = O.SOS, tgt[b, :n]
        seq_out[b, :n], seq_out[b, n] = tgt[b, :n], O.EOS
    A = Arena(lib)
    tg = A.inp("padded_target", tgt.cuda())
    si, so = A.out("seq_in", (B, Tt), torch.int64), A.out("seq_out", (B, Tt), torch.int64)
    kp, npd = A.out("key_pad", (B, Tt), torch.uint8), A.out("non_pad", (B, Tt))
    stt = A.inout("status", torch.zeros(1, dtype=torch.int32, device="cuda"))
    A.call("preprocess_targets", tg, L, si, so, kp, npd, stt, B, Tt)
    assert _eq(si.t, seq_in) and _eq(so.t, seq_out) and int(stt.t.item()) == 0
    assert _eq(kp.t, (seq_in == O.EOS).to(torch.uint8)) and _eq(npd.t, (seq_in != O.EOS).float())
    T = Tt + 3
    lg = A.inp("lengths", torch.tensor(lens, dtype=torch.int32, device="cuda"))
    kp2, np2 = A.out("key_pad2", (B, T), torch.uint8), A.out("non_pad2", (B, T))
    A.call("length_masks", lg, kp2, np2, B, T)
    pad = torch.arange(T)[None, :] >= torch.tensor(lens)[:, None]
    assert _eq(kp2.t, pad.to(torch.uint8)) and _eq(np2.t, (~pad).float())


@gpu
@pytest.mark.parametrize("B,T,V,lmax", [(1, 1, 5, 1), (3, 37, 33, 12), (2, 40, 129, 17)])
def test_ctc(lib, B, T, V, lmax):
    """ctc_fwd / ctc_bwd with exactly ctc_ws_bytes of workspace, T = 1 and targets at the maximum length: nll, loss and the
    gradient against the float64 recursion of tests/ctc_util.py."""
    g = _gen(T + V)
    x = torch.randn(B, T, V, generator=g)
    S = lmax + 2
    il = [T] + [max(1, T - 2 * b) for b in range(1, B)]
    tl = [min(max(0, lmax - 3 * b), (i - 1) // 2) for b, i in enumerate(il)]      # alignable even with repeated labels
    gold = torch.randint(1, V, (B, S), generator=g)
    nll_ref, loss_ref, grad_ref = ctc_float64(x, gold, il, tl)
    A = Arena(lib)
    xg, gg = A.inp("logits", x.cuda()), A.inp("targets", gold.cuda())
    ilg = A.inp("input_lengths", torch.tensor(il, dtype=torch.int32).cuda())
    tlg = A.inp("target_lengths", torch.tensor(tl, dtype=torch.int32).cuda())
    nll, loss = A.out("nll", (B,)), A.out("loss", (1,))
    ws = A.ws("ws", lib.b200asr_ctc_ws_bytes(B, T, lmax))
    A.call("ctc_fwd", xg, gg, ilg, tlg, nll, loss, ws, B, T, V, S, lmax)
    assert rel_err(nll.t, torch.as_tensor(nll_ref)) < 1e-5 and rel_err(loss.t, torch.as_tensor(loss_ref).view(1)) < 1e-5
    nll.freeze()
    ws.role = "inout"                       # written by the forward, read by the backward
    dloss = A.inp("dloss", torch.tensor([1.5], device="cuda"))
    dz = A.out("dlogits", (B, T, V))
    A.call("ctc_bwd", xg, gg, ilg, tlg, nll, dloss, dz, ws, B, T, V, S, lmax)
    assert rel_err(dz.t, torch.as_tensor(grad_ref) * 1.5) < 1e-5


# ================================================================================================ LSTM language model
def _interleave(m, nhid, H):
    """[4*nhid, K] in nn.LSTM's gate blocks -> [4H, K] with row 4u + g = gate g of unit u, zero rows for u >= nhid."""
    out = torch.zeros(4 * H, *m.shape[1:], dtype=m.dtype, device=m.device)
    for gte in range(4):
        out[gte:4 * nhid:4] = m[gte * nhid:(gte + 1) * nhid]
    return out


@gpu
@pytest.mark.parametrize("ninp,nhid", [(1, 1), (13, 13), (20, 64), (7, 30)])
def test_lstm_prepare_and_unprepare(lib, ninp, nhid):
    """lstm_prepare (interleaved, zero-padded w_ih_p / w_hh_p / bias_p for nhid, ninp not multiples of 8) and
    lstm_grad_unprepare (its inverse, every output guarded): exact."""
    H, I = _round_up(nhid, 8), _round_up(ninp, 8)
    wih, whh = _randn(4 * nhid, ninp, seed=90), _randn(4 * nhid, nhid, seed=91)
    bih, bhh = _randn(4 * nhid, seed=92), _randn(4 * nhid, seed=93)
    A = Arena(lib)
    a, b_, c, d = A.inp("w_ih", wih), A.inp("w_hh", whh), A.inp("b_ih", bih), A.inp("b_hh", bhh)
    wp, hp, bp = A.out("w_ih_p", (4 * H, I)), A.out("w_hh_p", (4 * H, H)), A.out("bias_p", (4 * H,))
    A.call("lstm_prepare", a, b_, c, d, ninp, nhid, wp, hp, bp)
    pad = lambda m, K: F.pad(m, (0, K - m.shape[1]))
    assert _eq(wp.t, _interleave(pad(wih, I), nhid, H)) and _eq(hp.t, _interleave(pad(whh, H), nhid, H))
    assert _eq(bp.t, _interleave((bih + bhh)[:, None], nhid, H)[:, 0])
    for g in (wp, hp, bp):
        g.freeze()
    outs = [A.out("dw_ih", (4 * nhid, ninp)), A.out("dw_hh", (4 * nhid, nhid)), A.out("db_ih", (4 * nhid,)),
            A.out("db_hh", (4 * nhid,))]
    A.call("lstm_grad_unprepare", wp, hp, bp, ninp, nhid, *outs)
    assert _eq(outs[0].t, wih) and _eq(outs[1].t, whh) and _eq(outs[2].t, bih + bhh) and _eq(outs[3].t, bih + bhh)


def _cell_ref(xproj, whh, h0, c0, T, B, H):
    """float64 LSTM recurrence on interleaved gates: (h [T*B, H], c [T*B, H], activated gates [T*B, 4H]) as graph nodes."""
    hs, cs, gs = [], [], []
    h, c = h0, c0
    for t in range(T):
        z = xproj[t * B:(t + 1) * B] + h @ whh.T
        i, f, gg, o = (z[:, k::4] for k in range(4))
        i, f, gg, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(gg), torch.sigmoid(o)
        c = f * c + i * gg
        h = o * torch.tanh(c)
        hs.append(h)
        cs.append(c)
        gs.append(torch.stack([i, f, gg, o], -1).reshape(B, 4 * H))
    return torch.cat(hs), torch.cat(cs), torch.cat(gs)


def _packed_ref(xproj, whh, batch_sizes, H):
    """float64 zero-state recurrence over packed sequences (t-major, longest first): h [sum(batch_sizes), H]."""
    h = torch.zeros(batch_sizes[0], H, dtype=torch.float64, device=xproj.device)
    c = torch.zeros_like(h)
    out, off = [], 0
    for M in batch_sizes:
        z = xproj[off:off + M] + h[:M] @ whh.T
        i, f, g, o = torch.sigmoid(z[:, 0::4]), torch.sigmoid(z[:, 1::4]), torch.tanh(z[:, 2::4]), torch.sigmoid(z[:, 3::4])
        c = torch.cat([f * c[:M] + i * g, c[M:]])
        h = torch.cat([o * torch.tanh(c[:M]), h[M:]])
        out.append(h[:M])
        off += M
    return torch.cat(out)


@gpu
@pytest.mark.parametrize("shift", [0, 16])
@pytest.mark.parametrize("T,B,H,batch_sizes", [(1, 1, 8, [1]), (5, 3, 16, [3, 3, 2, 1, 1]), (4, 130, 24, [130, 100, 37, 1])])
def test_lstm_layers(lib, T, B, H, batch_sizes, shift):
    """lstm_layer_fwd (packed sequences of decreasing lengths, host batch_sizes, the c workspace of batch_sizes[0] rows),
    lstm_layer_train_fwd (h with its h0 slot, c, gates) and lstm_layer_train_bwd (dgates, dc0, the dc workspace) against
    the float64 recurrence; B past the engine's 128 rows."""
    xproj = _randn(T * B, 4 * H, seed=94, scale=0.5)
    whh = _randn(4 * H, H, seed=95, scale=1.0 / math.sqrt(H))
    h0, c0 = _randn(B, H, seed=96, scale=0.5), _randn(B, H, seed=97, scale=0.5)
    dh_out, dh_n, dc_n = _randn(T * B, H, seed=98), _randn(B, H, seed=99), _randn(B, H, seed=100)
    A = Arena(lib, shift)
    wg = A.inp("w_hh_p", whh)
    w16 = A.out("w_hh_split", (2, 4 * H, H), torch.int16)
    w16t = A.out("w_hh_split_t", (2, H, 4 * H), torch.int16)
    rc = lib.b200asr_split_bf16(wg.ptr, w16.ptr, w16t.ptr, 4 * H, H, 2, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    w16.freeze()
    w16t.freeze()
    xg, c0g = A.inp("xproj", xproj), A.inp("c0", c0)

    # zero-state inference over packed sequences of decreasing lengths
    bs = np.array(batch_sizes, dtype=np.int32)
    P = int(bs.sum())
    xpg = A.inp("xproj_packed", xproj[:P])
    h, c = A.out("h", (P, H)), A.out("c_ws", (B, H))
    A.call("lstm_layer_fwd", xpg, w16, bs.ctypes.data, T, H, c, h)
    assert (h.t.double() - _packed_ref(xproj[:P].double(), whh.double(), batch_sizes, H)).abs().max() < 1.2e-4

    # training forward with a state, then its backward
    hbuf = torch.full(((T + 1) * B, H), NAN, device="cuda")
    hbuf[:B] = h0
    ht = A.inout("h_train", hbuf)
    ct, gt = A.out("c", (T * B, H)), A.out("gates", (T * B, 4 * H))
    A.call("lstm_layer_train_fwd", xg, w16, T, B, H, 1, c0g, ht, ct, gt)
    x64 = xproj.double().requires_grad_(True)
    h064, c064 = h0.double().requires_grad_(True), c0.double().requires_grad_(True)
    hr, cr, gr = _cell_ref(x64, whh.double(), h064, c064, T, B, H)
    assert (ht.t[B:].double() - hr).abs().max() < 1.2e-4 and (ct.t.double() - cr).abs().max() < 1.2e-4
    assert (gt.t.double() - gr).abs().max() < 1.2e-4 and _eq(ht.t[:B], h0)
    ct.freeze()
    gt.freeze()
    dhg, dhn, dcn = A.inp("dh_out", dh_out), A.inp("dh_n", dh_n), A.inp("dc_n", dc_n)
    dc, dgates, dc0 = A.out("dc_ws", (B, H)), A.out("dgates", (T * B, 4 * H)), A.out("dc0", (B, H))
    A.call("lstm_layer_train_bwd", gt, ct, c0g, dhg, dhn, dcn, w16t, T, B, H, dc, dgates, dc0)
    hT, cT = hr[-B:], cr[-B:]
    torch.autograd.backward([hr, hT, cT], [dh_out.double(), dh_n.double(), dc_n.double()])
    assert rel_err(dgates.t, x64.grad) < 5e-4 and rel_err(dc0.t, c064.grad) < 5e-4


@gpu
@pytest.mark.parametrize("n", [4, 1028, 99996])
@pytest.mark.parametrize("shift", [0, 16])
def test_lstm_dropout(lib, n, shift):
    """lstm_dropout: every element either x / (1 - p16) or 0, about p of them dropped, the same mask for the same key."""
    x = _randn(n, seed=101).abs() + 0.1
    A = Arena(lib, shift)
    xg = A.inp("x", x)
    y, y2 = A.out("y", (n,)), A.out("y2", (n,))
    A.call("lstm_dropout", xg, y, n, 0.25, 5, 9)
    A.call("lstm_dropout", xg, y2, n, 0.25, 5, 9)
    t16 = int(min(max(np.float32(0.25) * np.float32(65536.0) + np.float32(0.5), 0), 65535))
    inv = float(np.float32(1.0) / (np.float32(1.0) - np.float32(t16) / np.float32(65536.0)))
    kept = y.t != 0
    assert rel_err(y.t[kept], x.double()[kept] * inv) < 1e-7 and _eq(y.t, y2.t)
    if n > 1000:
        assert abs(float((~kept).float().mean()) - 0.25) < 0.05


@gpu
@pytest.mark.parametrize("rows,V,ld", [(1, 2, 4), (37, 1025, 1032), (5, 33, 33)])
def test_lm_nll_and_seq_sum(lib, rows, V, ld):
    """lm_nll over logits with a row pitch wider than V (gap columns guarded) and lm_seq_sum over t-major packed rows."""
    x = _randn(rows, V, seed=102)
    tgt = torch.randint(0, V, (rows,), generator=_gen(103)).cuda()
    A = Arena(lib)
    xg, tg = A.inp("logits", x, pitch=ld), A.inp("targets", tgt)
    nll = A.out("nll", (rows,))
    A.call("lm_nll", xg, ld, tg, nll, rows, V)
    ref = torch.logsumexp(x.double(), 1) - x.double().gather(1, tgt[:, None])[:, 0]
    assert rel_err(nll.t, ref) < 1e-6
    nll.freeze()
    lens = [rows] if rows < 3 else [rows // 2, rows // 2 - 1, 1]
    nseq = len(lens)
    offsets = [0]
    for t in range(max(lens) - 1):
        offsets.append(offsets[-1] + sum(1 for n in lens if n > t))
    og, lg = A.inp("offsets", torch.tensor(offsets, device="cuda")), A.inp("lengths", torch.tensor(lens, device="cuda"))
    sums = A.out("sums", (nseq,))
    A.call("lm_seq_sum", nll, og, lg, nseq, sums)
    want = [sum(float(nll.t[offsets[t] + s]) for t in range(lens[s])) for s in range(nseq)]
    assert rel_err(sums.t, torch.tensor(want, dtype=torch.float64)) < 1e-6


# ================================================================================================ step tail and operands
@gpu
@pytest.mark.parametrize("n", [1, 4, 1027, 300001])
def test_step_tail(lib, n):
    """sumsq (adds into out[0]), grad_scale (out[0..1], one float of scratch) and adam_step (p, m, v in place)."""
    g = _randn(n, seed=104)
    A = Arena(lib)
    gg = A.inp("g", g)
    out = A.inout("sumsq_out", torch.zeros(1, device="cuda"))
    A.call("sumsq", gg, n, out)
    total = float(g.double().pow(2).sum())
    assert rel_err(out.t, torch.tensor([total], dtype=torch.float64)) < 4e-7
    ntok = A.inp("n_tokens", torch.tensor([37.0], device="cuda"))
    scratch, gs = A.ws("scratch", 4), A.out("scale_out", (2,))
    A.call("grad_scale", gg, n, ntok, 1.0, scratch, gs)
    norm = math.sqrt(total) / 37.0
    coef = min(1.0, 1.0 / (norm + 1e-6))
    assert rel_err(gs.t[0:1], torch.tensor([coef / 37.0], dtype=torch.float64)) < 1e-6
    assert rel_err(gs.t[1:2], torch.tensor([norm], dtype=torch.float64)) < 1e-6
    p, m, v = _randn(n, seed=105), _randn(n, seed=106) * 0.1, _randn(n, seed=107).abs() * 0.01
    pg, mg, vg = A.inout("p", p), A.inout("m", m), A.inout("v", v)
    gsd = A.inp("gscale_dev", torch.tensor([0.5], device="cuda"))
    lr, b1, b2, eps, step = 1e-3, 0.9, 0.98, 1e-9, 3
    A.call("adam_step", pg, gg, mg, vg, n, lr, b1, b2, eps, step, 2.0, gsd)
    gd = g.double()
    m2 = b1 * m.double() + (1 - b1) * gd
    v2 = b2 * v.double() + (1 - b2) * gd * gd
    p2 = p.double() - (lr / (1 - b1 ** step)) * m2 / (v2.sqrt() / (1 - b2 ** step) ** 0.5 + eps)
    # relative to the terms' magnitude: with a handful of elements m's two terms may cancel
    assert rel_err(pg.t, p2) < 3e-6 and rel_err(vg.t, v2) < 3e-6
    assert float((mg.t.double() - m2).abs().max()) < 5e-7 * float(torch.maximum(b1 * m.double().abs(), (1 - b1) * gd.abs()).max())


@gpu
@pytest.mark.parametrize("n", [1, 3, 4, 1027, 65537])
def test_split_tf32(lib, n):
    """split_tf32: dst [2][n] = hi (a TF32 value) and lo = src - hi, exactly; both placements."""
    src = _randn(n, seed=108)
    for shift in (0, 16):
        A = Arena(lib, shift)
        sg = A.inp("src", src)
        dst = A.out("dst", (2, n))
        A.call("split_tf32", sg, dst, n)
        hi, lo = dst.t[0], dst.t[1]
        assert bool((hi.view(torch.int32) & 0x1FFF == 0).all())
        assert _eq(hi + lo, src) and bool(((src - hi).abs() <= src.abs() * 2.0 ** -10).all())


@gpu
def test_split_bf16_batched(lib):
    """split_bf16_batched over matrices of one flat buffer into one output buffer: both orientations of every matrix
    (the transposed one with zero padding columns to N8) exactly, and nothing written outside the described ranges."""
    mats = [(5, 40, 2), (64, 8, 1), (1, 8, 2), (33, 72, 2)]           # (N, K, terms)
    base_parts, desc, tiles, src_off, dst_off = [], [], [], 0, 0
    expect = []
    for i, (N, K, terms) in enumerate(mats):
        w = _randn(N, K, seed=110 + i).cpu()
        N8 = _round_up(N, 8)
        pr = pairs_ref(w)[:terms]                                     # [terms, N, K] int16
        pt = torch.zeros(terms, K, N8, dtype=torch.int16)
        pt[:, :, :N] = pr.transpose(1, 2)
        d_off, dt_off = dst_off, dst_off + terms * N * K
        desc.append([src_off, N, K, terms, d_off, dt_off])
        tiles.append(sum(math.ceil(K2 / 32) * math.ceil(_round_up(N2, 8) / 32) for N2, K2, _ in mats[:i]))
        expect.append((d_off, pr.flatten()))
        expect.append((dt_off, pt.flatten()))
        base_parts.append(w.flatten())
        src_off += N * K
        dst_off = dt_off + terms * K * N8
    total = sum(math.ceil(K / 32) * math.ceil(_round_up(N, 8) / 32) for N, K, _ in mats)
    want = torch.zeros(dst_off, dtype=torch.int16)
    for off, vals in expect:
        want[off:off + vals.numel()] = vals
    A = Arena(lib)
    bg = A.inp("base", torch.cat(base_parts).cuda())
    dg = A.inp("desc", torch.tensor(desc, dtype=torch.int64).cuda())
    tg = A.inp("tile_prefix", torch.tensor(tiles, dtype=torch.int32).cuda())
    out = A.out("out", (dst_off,), torch.int16, fill=0)
    A.call("split_bf16_batched", bg, out, dg, tg, len(mats), total)
    assert _eq(out.t, want)
