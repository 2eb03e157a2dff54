"""torch.autograd.Function wrappers over the C ABI (one per kernel group of SURVEY.md §2.3).

PyTorch is used here for device memory, streams and the autograd graph only: every FLOP on the path is a
kernel of libb200asr.so.  All functions require CUDA tensors; there is no CPU implementation.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch

from . import _lib as L

# ----------------------------------------------------------------------------------------------- configuration
_PREC_NAMES = {"fp32": L.PREC_FP32, "tf32": L.PREC_TF32, "tf32x3": L.PREC_TF32X3, "bf16": L.PREC_BF16, "bf16x3": L.PREC_BF16X3}
_BF16_PRECS = (L.PREC_BF16, L.PREC_BF16X3)


class _Config:
    """Arithmetic mode per kernel family (include/b200asr.h `precision`).

    Default = the fp32-grade mix, everything on the tensor cores with a 2-term operand split and three MMAs per product:
    "bf16x3" (x ~ bf16 hi + bf16 lo, twice the tf32 MMA rate) for the linear and convolution forward / data gradient,
    "tf32x3" for the weight gradients and the attention contractions; tests/test_gpu_fullsize_parity.py holds it to the fp64
    oracle at the TRUE cfg2 dims (every gradient tensor in the max norm at the path's own ReLU / pooling decisions).
    Attention: the default "tf32x3" is the materialised path (batched 3xTF32 GEMMs around exact fp32 softmax kernels; at
    these shapes -- T <= 250, 256 heads -- the 41 MB score tensor fits the 50 MB L2); "bf16x3" selects the fused kernels
    (tc_flash.cu: QK^T / PV with masks, softmax and dropout on the score fragments in registers, the backward
    recomputing the probabilities), opt-in: its flash-style delta = rowsum(dO o O) injects a row-constant error into dS that
    the near-uniform attention of this model amplifies in the Q/K projection gradients.
    Alternatives per family: "fp32" = CUDA-core kernels (exact fp32; attention = the flash-style kernel, which is also
    what shapes outside the tensor-core shape rules run on), "tf32" = single-pass TF32 (attention = the flash forward /
    backward kernels) -- neither meets the 1e-3 gradient bar, so they are opt-in only."""

    def __init__(self):
        self.linear = _PREC_NAMES[os.environ.get("B200ASR_LINEAR", "bf16x3")]
        self.conv = _PREC_NAMES[os.environ.get("B200ASR_CONV", "bf16x3")]
        self.conv_wgrad = _PREC_NAMES[os.environ.get("B200ASR_CONV_WGRAD", "tf32x3")]
        self.attn = _PREC_NAMES[os.environ.get("B200ASR_ATTN", "tf32x3")]          # "bf16x3" = the fused single-kernel path (opt-in)
        self.attn_bwd = _PREC_NAMES[os.environ.get("B200ASR_ATTN_BWD", "fp32")]

    def set(self, linear=None, conv=None, attn=None, conv_wgrad=None, attn_bwd=None):
        if attn_bwd is not None:
            self.attn_bwd = _PREC_NAMES[attn_bwd] if isinstance(attn_bwd, str) else int(attn_bwd)
        if conv_wgrad is not None:
            self.conv_wgrad = _PREC_NAMES[conv_wgrad] if isinstance(conv_wgrad, str) else int(conv_wgrad)
        if linear is not None:
            self.linear = _PREC_NAMES[linear] if isinstance(linear, str) else int(linear)
        if conv is not None:
            self.conv = _PREC_NAMES[conv] if isinstance(conv, str) else int(conv)
        if attn is not None:
            self.attn = _PREC_NAMES[attn] if isinstance(attn, str) else int(attn)


config = _Config()


class _Rng:
    """Seed + per-call offset for the counter-based dropout generator of the kernels."""

    def __init__(self):
        self.seed = 0x5EED
        self.offset = 0

    def manual_seed(self, seed: int):
        self.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self.offset = 0

    def next(self):
        self.offset += 1
        return self.seed, self.offset


rng = _Rng()


def manual_seed(seed: int):
    rng.manual_seed(seed)


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _Profiler:
    """Optional CUDA-event timing of every C-ABI call (bench.py uses it for per-kernel-group durations).
    Events are recorded on the launching stream around the call; nothing synchronises until report()."""

    def __init__(self):
        self.enabled = False
        self.records = []

    def start(self):
        self.records, self.enabled = [], True

    def stop(self):
        self.enabled = False

    def report(self):
        torch.cuda.synchronize()
        out = {}
        for name, args, e0, e1 in self.records:
            out.setdefault(name, []).append((args, e0.elapsed_time(e1)))
        return out        # name -> [(raw C-ABI args, milliseconds)]


profiler = _Profiler()

# Test hook: when set to a list, the forwards append (kind, activation) for every discontinuous unit of the path -- post-ReLU
# FFN / conv outputs, max-pool inputs, post-Hardtanh outputs -- in call order.  The parity tests derive the path's discrete
# decisions (active units, pooling winners) from them and evaluate the fp64 oracle AT those decisions (oracle.Decisions).
decision_capture = None

# Called (if set) at the START of the CNN front end's backward -- the first node of the graph, hence the last to run: every
# gradient except the front end's own is complete at that point.  parallel.DataParallelStep launches the all-reduce of that
# part of the flat gradient buffer from here, so it overlaps the convolution backward (~40% of the backward at cfg2).
frontend_backward_hook = None


class _ProfiledLib:
    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("b200asr_") or name.endswith("_bytes"):
            return fn

        def call(*args):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*args)
            e1.record()
            profiler.records.append((name[len("b200asr_"):], args, e0, e1))
            return rc

        return call


def _lib():
    lib = L.load()
    return _ProfiledLib(lib) if profiler.enabled else lib


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("b200asr ops run on CUDA tensors only (no CPU path exists); got a CPU tensor")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise RuntimeError(f"b200asr: expected float32, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


# ----------------------------------------------------------------------------------------------- dense layers
class WSplit:
    """Tensor-core operand copies of one weight matrix, made once per step and shared by forward and backward:
    `fwd` feeds y = x w^T, `bwd` feeds dx = dy w.  3xTF32: one fp32 [2,N,K] = (rn_tf32(w), w - hi) for both.  bf16 modes:
    bf16 [terms,N,K] and the transposed [terms,K,N8] (so that both GEMMs see a K-major B operand)."""
    __slots__ = ("fwd", "bwd")

    def __init__(self, fwd, bwd):
        self.fwd, self.bwd = fwd, bwd


class WeightOperandCache:
    """bf16 tensor-core operands of every weight matrix that lives in a FlatParams buffer, refreshed by ONE kernel launch per
    optimizer step (b200asr_split_bf16_batched) instead of one conversion launch per weight and step.

    A matrix is registered the first time split_weight() is asked for it (that request is served by the per-weight kernel);
    from the next refresh on its operands are views of one bf16 buffer.  Freshness: the Adam kernel writes through raw
    pointers, so FusedAdam.step() calls refresh() itself; any other in-place change of a weight (torch optimizers,
    load_state_dict, manual edits) moves that tensor's autograd version counter away from the one recorded at the last
    conversion, and get() then converts again (once: a refresh records the versions of all registered weights).  A write
    through the flat buffer itself (flat.flat.copy_(snapshot), a broadcast into it) moves only the BUFFER's version counter --
    the parameters were re-homed with `p.data = view`, which keeps their own counters -- so that one is tracked as well."""

    def __init__(self, flat):
        self.flat = flat                      # optim.FlatParams
        self.entries, self.pending = {}, {}   # key -> (src_off, N, K, terms, dst_off, dstT_off); key -> the weight tensor
        self.buf = self.desc = self.prefix = None
        self.tiles = 0
        self.tensors = {}                     # key -> the weight (a view of the flat buffer) as last seen
        self.converted_at = {}                # key -> its version counter when its operands were last converted
        self.flat_converted_at = None         # the flat buffer's version counter at the last conversion

    def owns(self, w2):
        f = self.flat.flat
        return w2.is_contiguous() and f.data_ptr() <= w2.data_ptr() and w2.data_ptr() + w2.numel() * 4 <= f.data_ptr() + f.numel() * 4

    def refresh(self):
        if self.pending:
            off = 0 if self.buf is None else self.buf.numel()
            for key, w2 in self.pending.items():
                ptr, N, K, terms = key
                n8 = (N + 7) // 8 * 8
                self.entries[key] = ((ptr - self.flat.flat.data_ptr()) // 4, N, K, terms, off, off + terms * N * K)
                off += (terms * N * K + terms * K * n8 + 63) // 64 * 64
                self.tensors[key] = w2
            self.pending = {}
            dev = self.flat.flat.device
            self.buf = torch.empty(off, device=dev, dtype=torch.bfloat16)
            rows, prefix, tiles = [], [], 0
            for (so, N, K, terms, do, dto) in self.entries.values():
                rows.append([so, N, K, terms, do, dto])
                prefix.append(tiles)
                tiles += ((K + 31) // 32) * (((N + 7) // 8 * 8 + 31) // 32)
            self.desc = torch.tensor(rows, dtype=torch.int64, device=dev)
            self.prefix = torch.tensor(prefix, dtype=torch.int32, device=dev)
            self.tiles = tiles
        if self.entries:
            L.check(_lib().b200asr_split_bf16_batched(L.ptr(self.flat.flat), L.ptr(self.buf), L.ptr(self.desc), L.ptr(self.prefix),
                                                      len(self.entries), self.tiles, _stream()), "split_bf16_batched")
            for key, w2 in self.tensors.items():
                self.converted_at[key] = w2._version
            self.flat_converted_at = self.flat.flat._version

    def after_optimizer_step(self):
        if self.entries or self.pending:
            self.refresh()

    def get(self, w2, prec):
        N, K = w2.shape
        terms = 2 if prec == L.PREC_BF16X3 else 1
        key = (w2.data_ptr(), N, K, terms)
        e = self.entries.get(key)
        if e is None:
            self.pending.setdefault(key, w2)
            return None
        self.tensors[key] = w2
        if self.converted_at.get(key) != w2._version or self.flat.flat._version != self.flat_converted_at:
            self.refresh()                                  # changed in place since the last conversion (not by our optimizer)
        _, _, _, _, do, dto = e
        n8 = (N + 7) // 8 * 8
        return WSplit(self.buf[do:do + terms * N * K].view(terms, N, K), self.buf[dto:dto + terms * K * n8].view(terms, K, n8))


weight_cache = None       # set by optim.FlatParams


def split_weight(w2, prec, need_bwd=True):
    if prec in _BF16_PRECS and weight_cache is not None and weight_cache.owns(w2):
        ws = weight_cache.get(w2, prec)
        if ws is not None:
            return ws
    if prec == L.PREC_TF32X3:
        ws = torch.empty((2,) + tuple(w2.shape), device=w2.device, dtype=torch.float32)
        L.check(_lib().b200asr_split_tf32(L.ptr(w2), L.ptr(ws), w2.numel(), _stream()), "split_tf32")
        return WSplit(ws, ws)
    if prec in _BF16_PRECS:
        N, K = w2.shape
        terms = 2 if prec == L.PREC_BF16X3 else 1
        fwd = torch.empty((terms, N, K), device=w2.device, dtype=torch.bfloat16)
        bwd = torch.empty((terms, K, (N + 7) // 8 * 8), device=w2.device, dtype=torch.bfloat16) if need_bwd else None
        L.check(_lib().b200asr_split_bf16(L.ptr(w2), L.ptr(fwd), L.ptr(bwd), N, K, terms, _stream()), "split_bf16")
        return WSplit(fwd, bwd)
    return None


def linear_fwd(x2, w, b, relu, prec, w_split=None, out=None):
    M, K = x2.shape
    N = w.shape[0]
    y = torch.empty((M, N), device=x2.device, dtype=torch.float32) if out is None else out
    L.check(_lib().b200asr_linear_fwd(L.ptr(x2), L.ptr(w), L.ptr(b), L.ptr(y), M, N, K, int(relu), prec,
                                      L.ptr(w_split.fwd if w_split is not None else None), _stream()), "linear_fwd")
    return y


def linear_bwd_data(dy2, w, relu_out, prec, w_split=None, accumulate_into=None):
    """dx = dy W (masked by relu_out > 0 if given); accumulate_into: a contiguous fp32 [M, K] tensor the product is ADDED to in
    the GEMM epilogue (and which is returned) -- how residual-branch gradients are summed without an extra pass."""
    M, N = dy2.shape
    K = w.shape[1]
    acc = accumulate_into is not None
    if acc and not (accumulate_into.is_contiguous() and accumulate_into.dtype == torch.float32 and accumulate_into.numel() == M * K):
        raise RuntimeError("linear_bwd_data: accumulate_into must be a contiguous fp32 tensor of M * K elements")
    dx = accumulate_into.view(M, K) if acc else torch.empty((M, K), device=dy2.device, dtype=torch.float32)
    L.check(_lib().b200asr_linear_bwd_data(L.ptr(dy2), L.ptr(w), L.ptr(relu_out), L.ptr(dx), M, N, K, int(acc), prec,
                                           L.ptr(w_split.bwd if w_split is not None else None), _stream()), "linear_bwd_data")
    return dx


class ResidualLink:
    """One per sub-layer y = LN(dropout(f(x)) + x): carries the residual-branch gradient from AddLNFn.backward to the backward
    of the node that consumes x (FFNFn / AttnProjFn), whose data-gradient GEMM adds its product into it (accumulate epilogue).
    Without it autograd sums the two gradients of x with a separate elementwise kernel per sub-layer.  `armed` is set in the
    consumer's forward (x needs a gradient and the consumer will compute one); AddLNFn then hands dz over instead of
    returning it."""
    __slots__ = ("armed", "dz")

    def __init__(self):
        self.armed, self.dz = False, None

    def take(self):
        dz, self.dz = self.dz, None
        return dz


def _grad_sink(param):
    """The parameter's existing .grad if a kernel can accumulate straight into it (the flat gradient buffer of
    optim.FlatParams), else None.  Writing there removes autograd's AccumulateGrad add kernel and a temporary per weight."""
    if param is None or not param.is_leaf or not getattr(param, "_b200_flat_grad", False):
        return None          # opt-in: only parameters re-homed by optim.FlatParams (it owns their .grad views)
    if getattr(param, "_backward_hooks", None) or getattr(param, "_post_accumulate_grad_hooks", None):
        return None          # tensor hooks (DDP, clipping hooks ...) must see the gradient: let autograd deliver it
    g = param.grad
    if g is None or not g.is_cuda or g.dtype != torch.float32 or not g.is_contiguous() or g.shape != param.shape:
        return None
    return g


def linear_bwd_weight(dy2, x2, want_bias, prec, w_sink=None, b_sink=None):
    """dW = dy^T x (+ column sums).  With sinks the kernels ACCUMULATE into the given .grad tensors and (None, None) is
    returned for them, so autograd has nothing left to add."""
    M, N = dy2.shape
    K = x2.shape[1]
    direct = w_sink is not None and (not want_bias or b_sink is not None)
    if direct:
        L.check(_lib().b200asr_linear_bwd_weight(L.ptr(dy2), L.ptr(x2), L.ptr(w_sink), L.ptr(b_sink) if want_bias else None, M, N, K,
                                                 1, prec, _stream()), "linear_bwd_weight")
        return None, None
    dw = torch.empty((N, K), device=dy2.device, dtype=torch.float32)
    db = torch.empty((N,), device=dy2.device, dtype=torch.float32) if want_bias else None
    L.check(_lib().b200asr_linear_bwd_weight(L.ptr(dy2), L.ptr(x2), L.ptr(dw), L.ptr(db), M, N, K, 0, prec,
                                             _stream()), "linear_bwd_weight")
    return dw, db


def _linear_prec(N, K):
    """Shape rule (documented in DESIGN.md, not a fallback): TMA needs 16-byte row pitches, i.e. N % 4 == 0 and
    K % 4 == 0 for fp32 operands (other shapes, e.g. dim_input = 161 with feat_extractor='', run on the fp32 CUDA-core
    GEMM) and additionally K % 8 == 0 for the bf16 weight operand of the bf16 modes (else the matching tf32 grade)."""
    if not (N % 4 == 0 and K % 4 == 0):
        return L.PREC_FP32
    prec = config.linear
    if prec in _BF16_PRECS and K % 8 != 0:
        prec = L.PREC_TF32X3 if prec == L.PREC_BF16X3 else L.PREC_TF32
    return prec


def linear_into(x, w, b, out):
    """y = x W^T + b written by the GEMM straight into `out`, a contiguous fp32 tensor of x.rows x N elements (one step of a
    K/V cache); no autograd."""
    _need_cuda(x, w, b, out)
    w2 = _f32c(w.reshape(w.shape[0], -1))
    x2 = _f32c(x).reshape(-1, w2.shape[1])
    if not (out.is_contiguous() and out.dtype == torch.float32 and out.numel() == x2.shape[0] * w2.shape[0]):
        raise RuntimeError("linear_into: out must be a contiguous fp32 tensor of rows x N elements")
    prec = _linear_prec(w2.shape[0], w2.shape[1])
    linear_fwd(x2, w2, b, False, prec, split_weight(w2, prec, need_bwd=False), out=out)
    return out


class LinearFn(torch.autograd.Function):
    """y = x W^T + b   (nn.Linear / Conv1d(k=1) call sites, include/b200asr.h)."""

    @staticmethod
    def forward(ctx, x, w, b):
        _need_cuda(x, w, b)
        w2 = _f32c(w.reshape(w.shape[0], -1))
        x2 = _f32c(x).reshape(-1, w2.shape[1])
        ctx.prec = _linear_prec(w2.shape[0], w2.shape[1])
        ws = split_weight(w2, ctx.prec, need_bwd=ctx.needs_input_grad[0])
        y = linear_fwd(x2, w2, b, False, ctx.prec, ws)
        ctx.save_for_backward(x2, w2)
        ctx.ws = ws
        ctx.xshape, ctx.wshape, ctx.has_bias = x.shape, w.shape, b is not None
        ctx.params = (w, b)
        return y.view(*x.shape[:-1], w2.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w2 = ctx.saved_tensors
        ws, ctx.ws = ctx.ws, None
        dy2 = _f32c(dy).reshape(-1, w2.shape[0])
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = linear_bwd_data(dy2, w2, None, ctx.prec, ws).view(ctx.xshape)
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            w, b = ctx.params
            dw, db = linear_bwd_weight(dy2, x2, ctx.has_bias, ctx.prec, _grad_sink(w), _grad_sink(b))
            dw = dw.view(ctx.wshape) if dw is not None else None
        return dx, dw, db


class FFNFn(torch.autograd.Function):
    """y = relu(x W1^T + b1) W2^T + b2   (models/common_layers.py:137-139; dropout/residual/LN follow in AddLNFn)."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, link=None):
        _need_cuda(x, w1, w2)
        ctx.link = link
        if link is not None:
            link.armed = bool(ctx.needs_input_grad[0])
        w1m = _f32c(w1.reshape(w1.shape[0], -1))
        w2m = _f32c(w2.reshape(w2.shape[0], -1))
        x2 = _f32c(x).reshape(-1, w1m.shape[1])
        ctx.prec = _linear_prec(w1m.shape[0], w1m.shape[1])
        ws1, ws2 = split_weight(w1m, ctx.prec), split_weight(w2m, ctx.prec)
        h = linear_fwd(x2, w1m, b1, True, ctx.prec, ws1)
        if decision_capture is not None:
            decision_capture.append(("relu", h.view(*x.shape[:-1], w1m.shape[0])))
        y = linear_fwd(h, w2m, b2, False, ctx.prec, ws2)
        ctx.save_for_backward(x2, h, w1m, w2m)
        ctx.ws = (ws1, ws2)
        ctx.shapes = (x.shape, w1.shape, w2.shape)
        ctx.params = (w1, b1, w2, b2)
        return y.view(*x.shape[:-1], w2m.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, h, w1m, w2m = ctx.saved_tensors
        (ws1, ws2), ctx.ws = ctx.ws, None
        xs, w1s, w2s = ctx.shapes
        dy2 = _f32c(dy).reshape(-1, w2m.shape[0])
        w1, b1, w2, b2 = ctx.params
        need = ctx.needs_input_grad                          # (x, w1, b1, w2, b2): frozen weights get no wgrad GEMM
        dw1 = db1 = dw2 = db2 = None
        if need[3] or need[4]:
            dw2, db2 = linear_bwd_weight(dy2, h, True, ctx.prec, _grad_sink(w2), _grad_sink(b2))
        dh = linear_bwd_data(dy2, w2m, h, ctx.prec, ws2) if (need[0] or need[1] or need[2]) else None     # masked by relu'(h)
        if need[1] or need[2]:
            dw1, db1 = linear_bwd_weight(dh, x2, True, ctx.prec, _grad_sink(w1), _grad_sink(b1))
        res = ctx.link.take() if ctx.link is not None else None          # residual-branch gradient of x, if AddLNFn handed it over
        dx = linear_bwd_data(dh, w1m, None, ctx.prec, ws1, accumulate_into=res) if need[0] else None
        return ((dx.view(xs) if dx is not None else None), (dw1.view(w1s) if dw1 is not None else None), db1,
                (dw2.view(w2s) if dw2 is not None else None), db2, None)


# ----------------------------------------------------------------------------------------------- residual + LN
class AddLNFn(torch.autograd.Function):
    """y = (LN(dropout(x) + residual) * gamma + beta + post_add[row % period]) * row_scale[row]."""

    @staticmethod
    def forward(ctx, x, residual, gamma, beta, post_add, row_scale, eps, p_drop, link=None):
        _need_cuda(x, gamma, beta)
        ctx.link = link if (link is not None and link.armed and residual is not None and ctx.needs_input_grad[1]) else None
        d = x.shape[-1]
        x2 = _f32c(x).reshape(-1, d)
        rows = x2.shape[0]
        res2 = _f32c(residual).reshape(-1, d) if residual is not None else None
        rs = _f32c(row_scale).reshape(-1) if row_scale is not None else None
        if rs is not None and rs.numel() != rows:
            raise RuntimeError("AddLN: row_scale must have one entry per row")
        period = post_add.shape[0] if post_add is not None else 0
        y = torch.empty_like(x2)
        need_z = res2 is not None or p_drop > 0.0
        z = torch.empty_like(x2) if need_z else None
        mean = torch.empty(rows, device=x.device, dtype=torch.float32)
        rstd = torch.empty(rows, device=x.device, dtype=torch.float32)
        seed, off = rng.next() if p_drop > 0.0 else (0, 0)
        L.check(_lib().b200asr_add_ln_fwd(L.ptr(x2), L.ptr(res2), L.ptr(gamma), L.ptr(beta), L.ptr(post_add), period,
                                          L.ptr(rs), L.ptr(y), L.ptr(z), L.ptr(mean), L.ptr(rstd), rows, d, float(eps),
                                          float(p_drop), seed, off, _stream()), "add_ln_fwd")
        ctx.save_for_backward(z if need_z else x2, gamma, mean, rstd, rs)
        ctx.meta = (x.shape, residual is not None, float(p_drop), seed, off, rows, d)
        ctx.params = (gamma, beta)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        z, gamma, mean, rstd, rs = ctx.saved_tensors
        xshape, has_res, p_drop, seed, off, rows, d = ctx.meta
        dy2 = _f32c(dy).reshape(-1, d)
        lib = _lib()
        dz = torch.empty_like(dy2)
        # with a link, dz is later added to in place by the consumer of the residual: keep it distinct from dx
        dx = torch.empty_like(dy2) if (p_drop > 0.0 or ctx.link is not None) else dz
        # gamma / beta gradients go straight into the parameters' .grad (flat gradient buffer) when that exists: no
        # zero-fill, no AccumulateGrad add -- four tiny launches less per LayerNorm
        g_sink, b_sink = _grad_sink(ctx.params[0]), _grad_sink(ctx.params[1])
        direct = g_sink is not None and b_sink is not None
        dgamma = g_sink if direct else torch.empty(d, device=dy.device, dtype=torch.float32)
        dbeta = b_sink if direct else torch.empty(d, device=dy.device, dtype=torch.float32)
        ws = torch.empty(lib.b200asr_add_ln_bwd_ws_bytes(rows, d) // 4, device=dy.device, dtype=torch.float32)
        L.check(lib.b200asr_add_ln_bwd(L.ptr(dy2), L.ptr(z), L.ptr(gamma), L.ptr(mean), L.ptr(rstd), L.ptr(rs), L.ptr(dz),
                                       L.ptr(dx), L.ptr(dgamma), L.ptr(dbeta), L.ptr(ws), rows, d, p_drop, seed, off,
                                       int(direct), _stream()), "add_ln_bwd")
        if ctx.link is not None:
            ctx.link.dz = dz                       # summed into the data gradient of the node that consumes the residual
            has_res = False
        return (dx.view(xshape), (dz.view(xshape) if has_res else None), None if direct else dgamma, None if direct else dbeta,
                None, None, None, None, None)


# ----------------------------------------------------------------------------------------------- attention
_maps_enabled = False


class attention_maps:
    """Whether the attention forwards return their probability maps, as ScaledDotProductAttention.forward and everything
    above it do in the reference (models/common_layers.py:211-225).  Off by default: the forwards then return None in their
    place and launch or allocate nothing for them.  Like torch.set_grad_enabled, calling it sets the state and using it as a
    `with` block restores the previous state on exit (exceptions and nesting included).

    A map is an fp32 (H*B) x Tq x Tk tensor in the reference's order (maps_layout): the matrix the kernel multiplied into V,
    i.e. softmax(scale * Q K^T, masks) with the forward's own dropout mask and 1 / (1 - p) applied in training.  Masked keys
    are 0, a fully masked row is NaN.  Maps are detached (requires_grad=False): no gradient flows through them."""

    def __init__(self, enabled: bool):
        global _maps_enabled
        self.prev = _maps_enabled
        _maps_enabled = bool(enabled)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        global _maps_enabled
        _maps_enabled = self.prev
        return False


def attention_maps_enabled() -> bool:
    return _maps_enabled


def maps_layout(B, H, Tq, Tk):
    """(shape, (bs, hs, rs)) of an attention map: (H*B) x Tq x Tk with row block h*B + b -- the order of the reference's
    mask.repeat(H, 1, 1) (models/common_layers.py:189) -- so probability (b, h, t, j) lives at b*bs + h*hs + t*rs + j."""
    return (H * B, Tq, Tk), (Tq * Tk, B * Tq * Tk, Tk)


def attention_probs(state):
    """The attention map of the forward that produced `state` (_sdpa_forward_impl), in maps_layout.  The materialised
    path copies the probabilities it kept for the backward (after dropout when p > 0, without the pad columns); the flash
    paths rebuild them with b200asr_sdpa_probs from Q, K and the forward's log-sum-exp at the forward's precision, with the
    forward's (seed, offset), so nothing is drawn from `rng`."""
    q, k = state["tensors"][:2]
    B, H, Tq, dk = q.shape
    Tk = k.shape[2]
    causal, scale, p_drop, seed, off, _ = state["meta"]
    shape, (bs, hs, rs) = maps_layout(B, H, Tq, Tk)
    maps = torch.empty(shape, device=q.device, dtype=torch.float32)
    if state["mat"]:
        probs, probs_drop = state["tensors"][4:6]
        src = (probs_drop if p_drop > 0.0 else probs).view(B, H, Tq, -1)[..., :Tk]
        maps.view(H, B, Tq, Tk).copy_(src.permute(1, 0, 2, 3))
        return maps
    lse, key_pad, dense_mask = state["tensors"][4:7]
    L.check(_lib().b200asr_sdpa_probs(L.ptr(q), L.ptr(k), *_bhtd_strides(q), *_bhtd_strides(k), L.ptr(key_pad), L.ptr(dense_mask),
                                      causal, L.ptr(lse), L.ptr(maps), bs, hs, rs, B, H, Tq, Tk, dk, scale, p_drop, seed, off,
                                      state["fwd_prec"], _stream()), "sdpa_probs")
    return maps


def _bhtd_strides(t):
    """(batch, head, row) element strides of a 4-D (B,H,T,d) view whose last dim is contiguous."""
    if t.dim() != 4 or t.stride(3) != 1:
        raise RuntimeError("sdpa: expected a (B,H,T,d) view with unit stride on d")
    return t.stride(0), t.stride(1), t.stride(2)


def _sdpa_forward_impl(q, k, v, key_pad, dense_mask, causal, scale, p_drop, head_major_out=False):
    """Attention forward over (B,H,T,d) views (any batch/head/row strides).  Returns (out, state); `state` is what
    _sdpa_backward_impl needs.  Output memory is token-major [B,Tq,H,dv] (returned as the (B,H,Tq,dv) view), so the head
    merge of models/common_layers.py:194-195 is free."""
    _need_cuda(q, k, v)
    B, H, Tq, dk = q.shape
    Tk, dv = k.shape[2], v.shape[3]
    if head_major_out:      # (H,B,Tq,dv) memory: the reference's (H*B) x Tq x dv layout (common_layers.py:185)
        out = torch.empty((H, B, Tq, dv), device=q.device, dtype=torch.float32).permute(1, 0, 2, 3)
    else:                   # token-major memory [B,Tq,H,dv]: the head merge of common_layers.py:194-195 is a view
        out = torch.empty((B, Tq, H, dv), device=q.device, dtype=torch.float32).permute(0, 2, 1, 3)
    seed, off = rng.next() if p_drop > 0.0 else (0, 0)
    qs, ks, vs, os_ = _bhtd_strides(q), _bhtd_strides(k), _bhtd_strides(v), _bhtd_strides(out)
    # shape rules (not fallbacks; DESIGN.md section 4): the materialised 3xTF32 path needs head dims that are whole
    # 32-float k-blocks and rows of at most 2048 keys; the TF32 flash kernels take Tk <= 448 and d in {32,64};
    # everything else runs on the fp32 CUDA-core kernel
    prec = config.attn
    if prec == L.PREC_BF16X3 and not (dk == 64 and dv == 64 and Tk <= 448 and not head_major_out):
        prec = L.PREC_TF32X3     # the fused bf16x3 kernels take Tk <= 448 and 64-wide heads
    if prec == L.PREC_BF16:
        prec = L.PREC_TF32       # "bf16" (cfg5) attention = the single-pass TF32 flash kernels
    if prec == L.PREC_BF16X3:
        lib = _lib()
        ws16 = torch.empty(lib.b200asr_sdpa_fused_ws_bytes(B, H, Tq, Tk) // 2, device=q.device, dtype=torch.bfloat16)
        lse = torch.empty((B, H, Tq), device=q.device, dtype=torch.float32)
        L.check(lib.b200asr_sdpa_fused_fwd(L.ptr(q), L.ptr(k), L.ptr(v), *qs, *ks, *vs, L.ptr(key_pad), L.ptr(dense_mask), int(causal),
                                           L.ptr(out), *os_, L.ptr(lse), L.ptr(ws16), B, H, Tq, Tk, dk, dv, float(scale), float(p_drop),
                                           seed, off, _stream()), "sdpa_fused_fwd")
        return out, dict(mat=False, fused=True, tensors=(q, k, v, out, lse, key_pad, dense_mask, ws16),
                         meta=(int(causal), float(scale), float(p_drop), seed, off, prec), fwd_prec=prec)
    if prec == L.PREC_TF32X3 and not (dk % 32 == 0 and dv % 32 == 0 and dk <= 256 and dv <= 256 and Tk <= 2048):
        prec = L.PREC_FP32
    if prec == L.PREC_TF32 and not (Tk <= 448 and dk in (32, 64) and dv in (32, 64)):
        prec = L.PREC_FP32
    if prec == L.PREC_FP32 and not (dk in (16, 32, 64, 128) and dv in (16, 32, 64, 128)):
        raise RuntimeError(f"b200asr attention: head dims (dk={dk}, dv={dv}) are supported for multiples of 32 up to 256 with "
                           f"Tk <= 2048 (tensor-core path) or for 16/32/64/128 (fp32 path); no kernel covers this shape")
    if prec == L.PREC_TF32X3:
        n = _lib().b200asr_sdpa_mat_ws_bytes(B, H, Tq, Tk) // 4
        probs = torch.empty(n, device=q.device, dtype=torch.float32)
        probs_drop = torch.empty(n, device=q.device, dtype=torch.float32) if p_drop > 0.0 else None
        L.check(_lib().b200asr_sdpa_mat_fwd(L.ptr(q), L.ptr(k), L.ptr(v), *qs, *ks, *vs, L.ptr(key_pad), L.ptr(dense_mask),
                                            int(causal), L.ptr(out), *os_, L.ptr(probs), L.ptr(probs_drop), B, H, Tq, Tk,
                                            dk, dv, float(scale), float(p_drop), seed, off, prec, _stream()), "sdpa_mat_fwd")
        return out, dict(mat=True, tensors=(q, k, v, out, probs, probs_drop),
                         meta=(int(causal), float(scale), float(p_drop), seed, off, prec))
    lse = torch.empty((B, H, Tq), device=q.device, dtype=torch.float32)
    L.check(_lib().b200asr_sdpa_fwd(L.ptr(q), L.ptr(k), L.ptr(v), *qs, *ks, *vs, L.ptr(key_pad), L.ptr(dense_mask),
                                    int(causal), L.ptr(out), *os_, L.ptr(lse), B, H, Tq, Tk, dk, dv, float(scale),
                                    float(p_drop), seed, off, prec, _stream()), "sdpa_fwd")
    bwd_prec = config.attn_bwd if (dk in (32, 64) and dv in (32, 64)) else L.PREC_FP32
    if bwd_prec == L.PREC_TF32X3:
        bwd_prec = L.PREC_FP32       # the flash-style backward exists as fp32 (CUDA cores) and TF32 (tensor cores) only
    return out, dict(mat=False, tensors=(q, k, v, out, lse, key_pad, dense_mask),
                     meta=(int(causal), float(scale), float(p_drop), seed, off, bwd_prec), fwd_prec=prec)


def _sdpa_backward_impl(state, dout, dq=None, dkk=None, dvv=None):
    """Attention backward.  dq/dk/dv may be given as preallocated (B,H,T,d) views (they must have the strides of q/k/v;
    the fused projection path passes column slices of one [tokens, 3*H*d] buffer); otherwise they are allocated."""
    causal, scale, p_drop, seed, off, prec = state["meta"]
    q, k, v, out = state["tensors"][:4]
    B, H, Tq, dk = q.shape
    Tk, dv = k.shape[2], v.shape[3]
    if dout.stride() != out.stride():
        dout = torch.empty_strided(out.shape, out.stride(), device=out.device, dtype=out.dtype).copy_(dout)
    if dq is None:
        dq = torch.empty_strided(q.shape, q.stride(), device=q.device, dtype=torch.float32) if _dense_like(q) else None
        dkk = torch.empty_strided(k.shape, k.stride(), device=q.device, dtype=torch.float32) if _dense_like(k) else None
        dvv = torch.empty_strided(v.shape, v.stride(), device=q.device, dtype=torch.float32) if _dense_like(v) else None
        if dq is None or dkk is None or dvv is None:
            raise RuntimeError("sdpa backward: q/k/v views must be dense permutations of a contiguous tensor")
    elif dq.stride() != q.stride() or dkk.stride() != k.stride() or dvv.stride() != v.stride():
        raise RuntimeError("sdpa backward: preallocated gradients must have the strides of q/k/v")
    qs, ks, vs, os_ = _bhtd_strides(q), _bhtd_strides(k), _bhtd_strides(v), _bhtd_strides(out)
    if state["mat"]:
        probs, probs_drop = state["tensors"][4:6]
        dp = torch.empty_like(probs)
        L.check(_lib().b200asr_sdpa_mat_bwd(L.ptr(dout), L.ptr(q), L.ptr(k), L.ptr(v), *qs, *ks, *vs, *os_, L.ptr(probs),
                                            L.ptr(probs_drop), L.ptr(dq), L.ptr(dkk), L.ptr(dvv), L.ptr(dp), B, H, Tq, Tk,
                                            dk, dv, scale, p_drop, seed, off, prec, _stream()), "sdpa_mat_bwd")
        return dq, dkk, dvv
    lse, key_pad, dense_mask = state["tensors"][4:7]
    if state.get("fused"):
        lib = _lib()
        ws16 = state["tensors"][7]
        wsb = torch.empty(lib.b200asr_sdpa_fused_bwd_ws_bytes(B, H, Tq) // 4, device=q.device, dtype=torch.float32)
        L.check(lib.b200asr_sdpa_fused_bwd(L.ptr(dout), L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(out), L.ptr(lse), *qs, *ks, *vs, *os_,
                                           L.ptr(key_pad), L.ptr(dense_mask), causal, L.ptr(dq), L.ptr(dkk), L.ptr(dvv), L.ptr(ws16),
                                           L.ptr(wsb), B, H, Tq, Tk, dk, dv, scale, p_drop, seed, off, _stream()), "sdpa_fused_bwd")
        return dq, dkk, dvv
    delta = torch.empty((B, H, Tq), device=q.device, dtype=torch.float32)
    L.check(_lib().b200asr_sdpa_bwd(L.ptr(dout), L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(out), L.ptr(lse), *qs, *ks, *vs, *os_,
                                    L.ptr(key_pad), L.ptr(dense_mask), causal, L.ptr(dq), L.ptr(dkk), L.ptr(dvv),
                                    L.ptr(delta), B, H, Tq, Tk, dk, dv, scale, p_drop, seed, off, prec, _stream()),
            "sdpa_bwd")
    return dq, dkk, dvv


class SdpaFn(torch.autograd.Function):
    """Fused softmax(q k^T * scale, masks) v over (B,H,T,d) *views* (any batch/head/row strides).  When `maps` is a list,
    the forward appends its attention map (attention_probs) to it."""

    @staticmethod
    def forward(ctx, q, k, v, key_pad, dense_mask, causal, scale, p_drop, head_major_out=False, maps=None):
        out, state = _sdpa_forward_impl(q, k, v, key_pad, dense_mask, causal, scale, p_drop, head_major_out)
        if maps is not None:
            maps.append(attention_probs(state))
        ctx.state = state        # tensors are kept alive by the dict (no in-place ops touch them afterwards)
        return out

    @staticmethod
    def backward(ctx, dout):
        dq, dkk, dvv = _sdpa_backward_impl(ctx.state, dout)
        ctx.state = None
        return dq, dkk, dvv, None, None, None, None, None, None, None


def _adjacent(*ts):
    """True if the tensors are contiguous, same-width row blocks lying back to back in memory (FlatParams lays the
    q/k/v projection weights -- and their gradients -- out like that), i.e. they can be used as ONE stacked matrix."""
    for a, b in zip(ts[:-1], ts[1:]):
        if a is None or b is None or not (a.is_contiguous() and b.is_contiguous()):
            return False
        if a.shape[1:] != b.shape[1:] or a.data_ptr() + a.numel() * 4 != b.data_ptr():
            return False
        if a.untyped_storage().data_ptr() != b.untyped_storage().data_ptr():
            return False        # neighbours by accident of the allocator: a view cannot span two storages
    return True


def _stacked(*ts):
    """The tensors of _adjacent() as one view [sum rows, ...]."""
    rows = sum(t.shape[0] for t in ts)
    shape = (rows,) + tuple(ts[0].shape[1:])
    stride = ts[0].stride() if ts[0].dim() > 1 else (1,)
    return ts[0].as_strided(shape, stride, ts[0].storage_offset())


class AttnProjFn(torch.autograd.Function):
    """Q/K/V projections + attention as ONE autograd node (MultiHeadAttention.forward up to the head merge,
    models/common_layers.py:176-195).

    When the three projection weights (and biases, and their .grad) lie back to back in memory -- optim.FlatParams
    arranges that -- the projections of a common input run as one GEMM with N = 3*H*d (self-attention) or N = 2*H*d (K and
    V of encoder-decoder attention): 200-tile problems on 132 SMs become 600-tile ones, the three data gradients become one
    GEMM with K = 3*H*d (no gradient-accumulation adds), the three weight gradients one split-K GEMM.  The attention kernels
    read Q/K/V as column slices of the packed projection output and write dQ/dK/dV into column slices of one packed
    buffer, all through strides.  Any other memory arrangement runs the same arithmetic as three GEMMs.  When `maps` is a
    list, the forward appends the attention map (attention_probs) to it."""

    @staticmethod
    def forward(ctx, xq, xkv, wq, bq, wk, bk, wv, bv, H, dk, dv, key_pad, dense_mask, causal, scale, p_drop, link=None, maps=None):
        _need_cuda(xq, xkv, wq, wk, wv)
        ctx.link = link
        if link is not None:
            link.armed = bool(ctx.needs_input_grad[0])
        same = xq is xkv
        B, Tq, D = xq.shape
        Tk = xkv.shape[1]
        xq2 = _f32c(xq).reshape(-1, D)
        xkv2 = xq2 if same else _f32c(xkv).reshape(-1, xkv.shape[2])
        ws_list = [_f32c(w.reshape(w.shape[0], -1)) for w in (wq, wk, wv)]
        has_bias = bq is not None and bk is not None and bv is not None
        n_q, n_k, n_v = (w.shape[0] for w in ws_list)
        fuse3 = same and _adjacent(*ws_list) and (not has_bias or _adjacent(bq, bk, bv))
        fuse2 = (not fuse3) and _adjacent(ws_list[1], ws_list[2]) and (not has_bias or _adjacent(bk, bv))
        if fuse3:
            groups = [((0, 1, 2), xq2)]
        elif fuse2:
            groups = [((0,), xq2), ((1, 2), xkv2)]
        else:
            groups = [((0,), xq2), ((1,), xkv2), ((2,), xkv2)]
        bs_list = [bq, bk, bv]
        packed, saved = [], []
        for idx, x2 in groups:
            W = _stacked(*[ws_list[i] for i in idx])
            b = _stacked(*[bs_list[i] for i in idx]) if has_bias else None
            prec = _linear_prec(W.shape[0], W.shape[1])       # shape rule per stacked group (N = H*dk, H*dv or their sums)
            wsplit = split_weight(W, prec)
            y = linear_fwd(x2, W, b, False, prec, wsplit)
            packed.append(y)
            saved.append((idx, x2, W, wsplit, prec))
        # column slices of the packed outputs as (B,H,T,d) views
        def head_view(y, col0, T, d):
            return y.view(B, T, y.shape[1])[:, :, col0:col0 + H * d].unflatten(2, (H, d)).permute(0, 2, 1, 3)
        if fuse3:
            q = head_view(packed[0], 0, Tq, dk); k = head_view(packed[0], n_q, Tk, dk); v = head_view(packed[0], n_q + n_k, Tk, dv)
        elif fuse2:
            q = head_view(packed[0], 0, Tq, dk); k = head_view(packed[1], 0, Tk, dk); v = head_view(packed[1], n_k, Tk, dv)
        else:
            q = head_view(packed[0], 0, Tq, dk); k = head_view(packed[1], 0, Tk, dk); v = head_view(packed[2], 0, Tk, dv)
        out, state = _sdpa_forward_impl(q, k, v, key_pad, dense_mask, causal, scale, p_drop)
        if maps is not None:
            maps.append(attention_probs(state))
        ctx.state, ctx.saved, ctx.has_bias = state, saved, has_bias
        ctx.params = (wq, bq, wk, bk, wv, bv)
        ctx.shapes = (xq.shape, xkv.shape, same, fuse3, fuse2, (n_q, n_k, n_v), H, dk, dv)
        return out.permute(0, 2, 1, 3).reshape(B, Tq, H * dv)          # free: memory is token-major

    @staticmethod
    def backward(ctx, dout):
        xq_shape, xkv_shape, same, fuse3, fuse2, (n_q, n_k, n_v), H, dk, dv = ctx.shapes
        q, k, v = ctx.state["tensors"][:3]
        B, Tq, Tk = q.shape[0], q.shape[2], k.shape[2]
        dev = q.device
        new = lambda m, n: torch.empty((m, n), device=dev, dtype=torch.float32)
        def head_view(y, col0, T, d):
            return y.view(B, T, y.shape[1])[:, :, col0:col0 + H * d].unflatten(2, (H, d)).permute(0, 2, 1, 3)
        if fuse3:
            dys = [new(B * Tq, n_q + n_k + n_v)]
            dq, dkk, dvv = head_view(dys[0], 0, Tq, dk), head_view(dys[0], n_q, Tk, dk), head_view(dys[0], n_q + n_k, Tk, dv)
        elif fuse2:
            dys = [new(B * Tq, n_q), new(B * Tk, n_k + n_v)]
            dq, dkk, dvv = head_view(dys[0], 0, Tq, dk), head_view(dys[1], 0, Tk, dk), head_view(dys[1], n_k, Tk, dv)
        else:
            dys = [new(B * Tq, n_q), new(B * Tk, n_k), new(B * Tk, n_v)]
            dq, dkk, dvv = head_view(dys[0], 0, Tq, dk), head_view(dys[1], 0, Tk, dk), head_view(dys[2], 0, Tk, dv)
        dout4 = dout.reshape(B, Tq, H, dv).permute(0, 2, 1, 3)
        _sdpa_backward_impl(ctx.state, dout4, dq, dkk, dvv)
        ctx.state = None
        params = ctx.params
        grads_w, grads_b = [None] * 3, [None] * 3
        dxkv = None
        need_xq, need_xkv = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        # running sums: every further contribution is added in its GEMM's epilogue; dxq starts from the residual-branch
        # gradient of the query input when AddLNFn handed it over (ResidualLink)
        dxq = ctx.link.take() if ctx.link is not None else None
        if dxq is not None and not need_xq:
            dxq = None
        for (idx, x2, W, wsplit, prec), dy in zip(ctx.saved, dys):
            feeds_q = 0 in idx
            if (feeds_q and need_xq) or (not feeds_q and (need_xkv or (same and need_xq))):
                if feeds_q or same:
                    dxq = linear_bwd_data(dy, W, None, prec, wsplit, accumulate_into=dxq)
                else:
                    dxkv = linear_bwd_data(dy, W, None, prec, wsplit, accumulate_into=dxkv)
            ws_ = [params[2 * i] for i in idx]
            bs_ = [params[2 * i + 1] for i in idx]
            sinks_w = [_grad_sink(w) for w in ws_]
            sinks_b = [_grad_sink(b) for b in bs_] if ctx.has_bias else []
            w_sink = b_sink = None
            if all(g is not None for g in sinks_w) and _adjacent(*[g.reshape(g.shape[0], -1) for g in sinks_w]):
                w_sink = _stacked(*[g.reshape(g.shape[0], -1) for g in sinks_w])
            if ctx.has_bias and all(g is not None for g in sinks_b) and _adjacent(*sinks_b):
                b_sink = _stacked(*sinks_b)
            dw, db = linear_bwd_weight(dy, x2, ctx.has_bias, prec, w_sink, b_sink)
            if dw is not None:          # no direct accumulation: hand the slices to autograd
                r0 = 0
                for i in idx:
                    n_i = (n_q, n_k, n_v)[i]
                    grads_w[i] = dw[r0:r0 + n_i].view(params[2 * i].shape)
                    grads_b[i] = db[r0:r0 + n_i] if db is not None else None
                    r0 += n_i
        dxq = dxq.view(xq_shape) if dxq is not None else None
        dxkv = dxkv.view(xkv_shape) if dxkv is not None else None
        return (dxq, dxkv, grads_w[0], grads_b[0], grads_w[1], grads_b[1], grads_w[2], grads_b[2],
                None, None, None, None, None, None, None, None, None, None)


def _dense_like(t):
    """True if the view covers a dense block (so empty_strided with the same strides is a plain allocation)."""
    n = 1
    for s, st in sorted(zip(t.shape, t.stride()), key=lambda x: x[1]):
        if s == 1:
            continue
        if st != n:
            return False
        n *= s
    return True


# ----------------------------------------------------------------------------------------------- VGG front end
class VggFrontendFn(torch.autograd.Function):
    """models/asr/transformer.py:42-53 on channels-last [B,T,F,C] activations.
    Input (B,1,F,T); output [B, T//4, (F//2//2), 128] whose flat view [B, T', F'*128] feeds input_linear."""

    @staticmethod
    def forward(ctx, x, w0, b0, w2, b2, w5, b5, w7, b7):
        _need_cuda(x, w0)
        lib, st, prec = _lib(), _stream(), config.conv
        x = _f32c(x)
        B, _, F, T = x.shape
        dev = x.device
        C1, C2 = w0.shape[0], w5.shape[0]
        new = lambda *s: torch.empty(s, device=dev, dtype=torch.float32)
        ws = new(lib.b200asr_conv3x3_ws_bytes(C2, C2) // 4)
        # the ReLU decisions of y1 and y3 also as packed bits [B,T,F,C/32], and the pooling decisions of y2 and y4 as packed
        # codes [B,T/2,F/2,C/8] (1/32 of the bytes each): the backward takes its masks and routes from these instead of reading
        # fp32 activations back.  In the bf16 modes y2 / y4 are not written at all (the pooling is the convolution's epilogue);
        # the other precisions pool in a kernel of their own, which reads them, and drop them after the forward.
        bits = lambda *s: torch.empty(s[:-1] + (s[-1] // 32,), device=dev, dtype=torch.int32)
        codes = lambda *s: torch.empty(s[:-1] + (s[-1] // 8,), device=dev, dtype=torch.int32)
        keep_y = decision_capture is not None or prec not in _BF16_PRECS
        y1 = new(B, T, F, C1)
        y1b = bits(B, T, F, C1)
        L.check(lib.b200asr_conv3x3_c1_fwd_bits(L.ptr(x), L.ptr(_f32c(w0)), L.ptr(b0), L.ptr(y1), B, F, T, C1, 1, L.ptr(y1b), st),
                "conv1")
        y2 = new(B, T, F, C1) if keep_y else None
        T2, F2 = T // 2, F // 2
        p1 = new(B, T2, F2, C1)
        c1 = codes(B, T2, F2, C1)
        # (pool_idx = None: asking for the arg-max bytes of b200asr_maxpool2x2_bwd_idx runs the stand-alone pooling kernel)
        # conv + ReLU + MaxPool2d(2, 2): in the bf16 modes the pooling is the convolution's epilogue
        L.check(lib.b200asr_conv3x3_fwd_pool_codes(L.ptr(y1), L.ptr(_f32c(w2)), L.ptr(b2), L.ptr(y2), L.ptr(p1), L.ptr(c1), L.ptr(ws),
                                                   B, T, F, C1, C1, 1, prec, st), "conv2+pool1")
        y3 = new(B, T2, F2, C2)
        y3b = bits(B, T2, F2, C2)
        L.check(lib.b200asr_conv3x3_fwd_bits(L.ptr(p1), L.ptr(_f32c(w5)), L.ptr(b5), L.ptr(y3), L.ptr(ws), B, T2, F2, C1, C2, 1,
                                             prec, L.ptr(y3b), st), "conv3")
        y4 = new(B, T2, F2, C2) if keep_y else None
        T4, F4 = T2 // 2, F2 // 2
        p2 = new(B, T4, F4, C2)
        c2 = codes(B, T4, F4, C2)
        L.check(lib.b200asr_conv3x3_fwd_pool_codes(L.ptr(y3), L.ptr(_f32c(w7)), L.ptr(b7), L.ptr(y4), L.ptr(p2), L.ptr(c2), L.ptr(ws),
                                                   B, T2, F2, C2, C2, 1, prec, st), "conv4+pool2")
        ctx.save_for_backward(x, y1, p1, y3, y1b, y3b, c1, c2, w0, w2, w5, w7)
        if decision_capture is not None:      # channels-last [B,T,F,C] -> the reference's (B,C,F,T)
            nchw = lambda t: t.permute(0, 3, 2, 1)
            decision_capture.extend([("relu", nchw(y1)), ("relu", nchw(y2)), ("pool", nchw(y2)), ("relu", nchw(y3)), ("relu", nchw(y4)),
                                     ("pool", nchw(y4))])
        ctx.prec, ctx.prec_w = prec, config.conv_wgrad
        return p2

    @staticmethod
    def backward(ctx, dp2):
        if frontend_backward_hook is not None:
            frontend_backward_hook()
        x, y1, p1, y3, y1b, y3b, c1, c2, w0, w2, w5, w7 = ctx.saved_tensors
        lib, st, prec, prec_w = _lib(), _stream(), ctx.prec, ctx.prec_w
        B, _, F, T = x.shape
        C1, C2 = w0.shape[0], w5.shape[0]
        T2, F2 = T // 2, F // 2
        dev = x.device
        new = lambda *s: torch.empty(s, device=dev, dtype=torch.float32)
        ws = new(lib.b200asr_conv3x3_ws_bytes(C2, C2) // 4)
        dp2 = _f32c(dp2)
        # bf16 weight gradient: the producers of the three dy tensors (both max-pool backward passes, conv4's data gradient)
        # also write them as bf16 hi | lo pairs, which the weight-gradient kernel takes as its B operand by TMA
        pairs = prec_w in _BF16_PRECS and prec in _BF16_PRECS
        new16 = lambda *s_: torch.empty((2,) + s_, device=dev, dtype=torch.bfloat16) if pairs else None
        d4, d4p = new(B, T2, F2, C2), new16(B, T2, F2, C2)
        L.check(lib.b200asr_maxpool2x2_bwd_codes(L.ptr(dp2), L.ptr(c2), L.ptr(d4), L.ptr(d4p), B, T2, F2, C2, 1, st), "pool2_bwd")
        dw7, db7 = torch.empty_like(w7), new(C2)
        L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(d4), L.ptr(d4p), L.ptr(y3), L.ptr(dw7), L.ptr(db7), L.ptr(ws), B, T2, F2, C2, C2,
                                               prec_w, st), "conv4_wgrad")
        d3, d3p = new(B, T2, F2, C2), new16(B, T2, F2, C2)
        L.check(lib.b200asr_conv3x3_bwd_data_bits(L.ptr(d4), L.ptr(_f32c(w7)), L.ptr(y3b), L.ptr(d3), L.ptr(d3p), L.ptr(ws), B, T2, F2,
                                                  C2, C2, prec, st), "conv4_dgrad")
        del d4, d4p
        dw5, db5 = torch.empty_like(w5), new(C2)
        L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(d3), L.ptr(d3p), L.ptr(p1), L.ptr(dw5), L.ptr(db5), L.ptr(ws), B, T2, F2, C1, C2,
                                               prec_w, st), "conv3_wgrad")
        dp1 = new(B, T2, F2, C1)
        L.check(lib.b200asr_conv3x3_bwd_data(L.ptr(d3), L.ptr(_f32c(w5)), None, L.ptr(dp1), None, L.ptr(ws), B, T2, F2, C1, C2,
                                             prec, st), "conv3_dgrad")
        del d3, d3p
        d2, d2p = new(B, T, F, C1), new16(B, T, F, C1)
        L.check(lib.b200asr_maxpool2x2_bwd_codes(L.ptr(dp1), L.ptr(c1), L.ptr(d2), L.ptr(d2p), B, T, F, C1, 1, st), "pool1_bwd")
        dw2, db2 = torch.empty_like(w2), new(C1)
        L.check(lib.b200asr_conv3x3_bwd_weight(L.ptr(d2), L.ptr(d2p), L.ptr(y1), L.ptr(dw2), L.ptr(db2), L.ptr(ws), B, T, F, C1, C1,
                                               prec_w, st), "conv2_wgrad")
        d1 = new(B, T, F, C1)
        L.check(lib.b200asr_conv3x3_bwd_data_bits(L.ptr(d2), L.ptr(_f32c(w2)), L.ptr(y1b), L.ptr(d1), None, L.ptr(ws), B, T, F, C1, C1,
                                                  prec, st), "conv2_dgrad")
        del d2, d2p
        dw0, db0 = torch.empty_like(w0), new(C1)
        L.check(lib.b200asr_conv3x3_c1_bwd_weight(L.ptr(x), L.ptr(d1), L.ptr(dw0), L.ptr(db0), B, F, T, C1, st), "conv1_wgrad")
        return None, dw0, db0, dw2, db2, dw5, db5, dw7, db7


class PermuteColsFn(torch.autograd.Function):
    """w' [rows, F*C] with w'[:, f*C+c] = w[:, c*F+f]: input_linear's columns re-ordered to the channels-last
    feature order of VggFrontendFn (replaces the activation transpose of models/asr/transformer.py:74-76)."""

    @staticmethod
    def forward(ctx, w, C, F):
        _need_cuda(w)
        w = _f32c(w)
        out = torch.empty_like(w)
        L.check(_lib().b200asr_permute_cols_cf(L.ptr(w), L.ptr(out), w.shape[0], C, F, 0, _stream()), "permute_cols")
        ctx.cf = (C, F)
        return out

    @staticmethod
    def backward(ctx, dw):
        C, F = ctx.cf
        dw = _f32c(dw)
        out = torch.empty_like(dw)
        L.check(_lib().b200asr_permute_cols_cf(L.ptr(dw), L.ptr(out), dw.shape[0], C, F, 1, _stream()), "permute_cols_inv")
        return out, None, None


# ----------------------------------------------------------------------------------------------- emb_cnn front end
class EmbFrontendFn(torch.autograd.Function):
    """models/asr/transformer.py:33-40 (+ flatten :74-76): conv(41x11,s2x2,p0x10)+BN+clamp, conv(21x11,s2x1)+BN+clamp.
    BatchNorm2d semantics of torch: `training` -> batch statistics, and the module's running_mean / running_var /
    num_batches_tracked buffers (bn1, bn2 = (running_mean, running_var, num_batches_tracked, momentum) or None) are
    updated in the kernel; eval -> the running statistics normalise (the reference validates with model.eval(),
    trainer.py:123, and Transformer.evaluate reads the same buffers through the stock nn.BatchNorm2d).
    Tensor-core modes: both convolutions run as IMPLICIT GEMMs (tc_emb.cu) for forward and weight gradient, the second
    (32 -> 32 channels, 21 x 11 taps, 88% of the front end's FLOPs) also for its data gradient, on row-pitched NCHW tensors
    -- no column matrix.  These kernels take the reference's two weight shapes only; any other shape is an error.
    Precision "fp32": direct CUDA-core kernels."""

    W0, W3 = (32, 1, 41, 11), (32, 32, 21, 11)

    @staticmethod
    def forward(ctx, x, w0, b0, g1, be1, w3, b3, g4, be4, eps, training=True, bn1=None, bn2=None):
        _need_cuda(x, w0)
        if not training and (bn1 is None or bn2 is None):
            raise RuntimeError("emb_cnn front end in eval mode needs the BatchNorm running statistics")
        tc = config.conv != L.PREC_FP32
        if tc and (tuple(w0.shape) != EmbFrontendFn.W0 or tuple(w3.shape) != EmbFrontendFn.W3):
            # the kernels are given the reference's geometry: another weight shape would be read out of bounds
            raise RuntimeError(f"emb_cnn front end: the tensor-core kernels support conv weights {EmbFrontendFn.W0} and "
                               f"{EmbFrontendFn.W3} only, got {tuple(w0.shape)} and {tuple(w3.shape)}")

        def bn_args(bn):
            if bn is None:
                return None, None, None, 0.1
            rm, rv, nbt, mom = bn
            if mom is None:
                raise RuntimeError("BatchNorm2d(momentum=None) (cumulative average) is not used by the reference and not implemented")
            return rm, rv, nbt, float(mom)
        lib, st = _lib(), _stream()
        x = _f32c(x)
        B, _, H, W = x.shape
        dev = x.device
        new = lambda *s: torch.empty(s, device=dev, dtype=torch.float32)
        C = w0.shape[0]
        H1, W1 = (H - 41) // 2 + 1, (W + 20 - 11) // 2 + 1
        H2, W2 = (H1 - 21) // 2 + 1, (W1 - 11) // 1 + 1
        P1, P2 = ((W1 + 3) // 4 * 4, (W2 + 3) // 4 * 4) if tc else (W1, W2)      # TMA: 16-byte row pitches
        prec2 = config.conv if config.conv in (L.PREC_TF32X3, L.PREC_BF16X3, L.PREC_BF16) else L.PREC_TF32X3
        c1 = new(B, C, H1, W1)
        if tc:
            ws1 = torch.empty(lib.b200asr_conv2d_c1_tc_ws_bytes(B, H, W, 41, 11) // 4, device=dev, dtype=torch.float32)
            L.check(lib.b200asr_conv2d_c1_tc_fwd(L.ptr(x), L.ptr(_f32c(w0)), L.ptr(b0), L.ptr(c1), L.ptr(ws1), B, H, W, C, 41, 11, 10, W1, prec2, st),
                    "emb_conv1_tc")
        else:
            L.check(lib.b200asr_conv2d_fwd(L.ptr(x), L.ptr(_f32c(w0)), L.ptr(b0), L.ptr(c1), B, 1, H, W, C, 41, 11, 2, 2, 0, 10, st), "emb_conv1")
        a1, m1, s1 = new(B, C, H1, P1), new(C), new(C)
        bws = new(lib.b200asr_bn_ws_bytes(C) // 4)
        rm, rv, nbt, mom = bn_args(bn1)
        L.check(lib.b200asr_bn_clamp_fwd(L.ptr(c1), L.ptr(g1), L.ptr(be1), L.ptr(a1), L.ptr(m1), L.ptr(s1), L.ptr(rm), L.ptr(rv),
                                         L.ptr(nbt), L.ptr(bws), B, C, H1, W1, W1, P1, eps, mom, int(training), 0.0, 20.0, st), "emb_bn1")
        c2 = new(B, C, H2, P2)
        if tc:
            ws = torch.empty(lib.b200asr_conv2d_tc_ws_bytes(B, H1, W1, 21, 11) // 4, device=dev, dtype=torch.float32)
            L.check(lib.b200asr_conv2d_tc_fwd(L.ptr(a1), L.ptr(_f32c(w3)), L.ptr(b3), L.ptr(c2), L.ptr(ws), B, C, H1, W1, C, 21, 11, 2,
                                              P1, P2, prec2, st), "emb_conv2_tc")
        else:
            L.check(lib.b200asr_conv2d_fwd(L.ptr(a1), L.ptr(_f32c(w3)), L.ptr(b3), L.ptr(c2), B, C, H1, W1, C, 21, 11, 2, 1, 0, 0, st), "emb_conv2")
        a2, m2, s2 = new(B, C, H2, W2), new(C), new(C)
        rm, rv, nbt, mom = bn_args(bn2)
        L.check(lib.b200asr_bn_clamp_fwd(L.ptr(c2), L.ptr(g4), L.ptr(be4), L.ptr(a2), L.ptr(m2), L.ptr(s2), L.ptr(rm), L.ptr(rv),
                                         L.ptr(nbt), L.ptr(bws), B, C, H2, W2, P2, W2, eps, mom, int(training), 0.0, 20.0, st), "emb_bn2")
        out = new(B, W2, C * H2)
        L.check(lib.b200asr_flatten_bcft_fwd(L.ptr(a2), L.ptr(out), B, C, H2, W2, st), "emb_flatten")
        ctx.save_for_backward(x, c1, a1, m1, s1, c2, a2, m2, s2, w0, g1, w3, g4)
        if decision_capture is not None:
            decision_capture.extend([("hardtanh", a1[..., :W1]), ("hardtanh", a2)])
        ctx.prec2 = prec2 if tc else None          # None: the direct fp32 kernels
        ctx.geom = (H1, W1, P1, H2, W2, P2)
        ctx.training = bool(training)
        return out

    @staticmethod
    def backward(ctx, dout):
        if frontend_backward_hook is not None:
            frontend_backward_hook()
        x, c1, a1, m1, s1, c2, a2, m2, s2, w0, g1, w3, g4 = ctx.saved_tensors
        prec2 = ctx.prec2
        H1, W1, P1, H2, W2, P2 = ctx.geom
        lib, st = _lib(), _stream()
        B, _, H, W = x.shape
        C = w0.shape[0]
        dev = x.device
        new = lambda *s: torch.empty(s, device=dev, dtype=torch.float32)
        dout = _f32c(dout)
        tr = int(ctx.training)
        bws = new(lib.b200asr_bn_ws_bytes(C) // 4)
        da2 = new(B, C, H2, W2)
        L.check(lib.b200asr_flatten_bcft_bwd(L.ptr(dout), L.ptr(da2), B, C, H2, W2, st), "emb_flatten_bwd")
        dc2, dg4, dbe4 = new(B, C, H2, P2), new(C), new(C)
        L.check(lib.b200asr_bn_clamp_bwd(L.ptr(da2), L.ptr(c2), L.ptr(a2), L.ptr(g4), L.ptr(m2), L.ptr(s2), L.ptr(dc2), L.ptr(dg4), L.ptr(dbe4),
                                         L.ptr(bws), B, C, H2, W2, W2, P2, W2, P2, tr, 0.0, 20.0, st), "emb_bn2_bwd")
        da1 = new(B, C, H1, P1)
        dw3, db3 = torch.empty_like(w3), new(C)
        if prec2 is not None:
            ws = torch.empty(lib.b200asr_conv2d_tc_ws_bytes(B, H1, W1, 21, 11) // 4, device=dev, dtype=torch.float32)
            L.check(lib.b200asr_conv2d_tc_bwd_weight(L.ptr(dc2), L.ptr(a1), L.ptr(dw3), L.ptr(db3), L.ptr(ws), B, C, H1, W1, C, 21, 11, 2, P1, P2, st),
                    "emb_conv2_tc_wgrad")
            L.check(lib.b200asr_conv2d_tc_bwd_data(L.ptr(dc2), L.ptr(_f32c(w3)), L.ptr(da1), L.ptr(ws), B, C, H1, W1, C, 21, 11, 2, P1, P2,
                                                   prec2, st), "emb_conv2_tc_dgrad")
        else:
            L.check(lib.b200asr_conv2d_bwd_weight(L.ptr(dc2), L.ptr(a1), L.ptr(dw3), L.ptr(db3), B, C, H1, W1, C, 21, 11, 2, 1, 0, 0, st), "emb_conv2_wgrad")
            L.check(lib.b200asr_conv2d_bwd_data(L.ptr(dc2), L.ptr(_f32c(w3)), L.ptr(da1), B, C, H1, W1, C, 21, 11, 2, 1, 0, 0, st), "emb_conv2_dgrad")
        dc1, dg1, dbe1 = new(B, C, H1, P1), new(C), new(C)          # P1 = W1 unless the implicit-GEMM weight gradient reads it by TMA
        L.check(lib.b200asr_bn_clamp_bwd(L.ptr(da1), L.ptr(c1), L.ptr(a1), L.ptr(g1), L.ptr(m1), L.ptr(s1), L.ptr(dc1), L.ptr(dg1), L.ptr(dbe1),
                                         L.ptr(bws), B, C, H1, W1, P1, W1, P1, P1, tr, 0.0, 20.0, st), "emb_bn1_bwd")
        dw0, db0 = torch.empty_like(w0), new(C)
        if prec2 is not None:
            ws1 = torch.empty(lib.b200asr_conv2d_c1_tc_ws_bytes(B, H, W, 41, 11) // 4, device=dev, dtype=torch.float32)
            L.check(lib.b200asr_conv2d_c1_tc_bwd_weight(L.ptr(dc1), L.ptr(x), L.ptr(dw0), L.ptr(db0), L.ptr(ws1), B, H, W, C, 41, 11, 10, P1, st),
                    "emb_conv1_tc_wgrad")
        else:
            L.check(lib.b200asr_conv2d_bwd_weight(L.ptr(dc1), L.ptr(x), L.ptr(dw0), L.ptr(db0), B, 1, H, W, C, 41, 11, 2, 2, 0, 10, st), "emb_conv1_wgrad")
        return None, dw0, db0, dg1, dbe1, dw3, db3, dg4, dbe4, None, None, None, None


class FlattenFn(torch.autograd.Function):
    """(B,C,F,T) -> (B,T,C*F) for feat_extractor='' (C=1) -- models/asr/transformer.py:74-76."""

    @staticmethod
    def forward(ctx, x):
        _need_cuda(x)
        x = _f32c(x)
        B, C, F, T = x.shape
        out = torch.empty((B, T, C * F), device=x.device, dtype=torch.float32)
        L.check(_lib().b200asr_flatten_bcft_fwd(L.ptr(x), L.ptr(out), B, C, F, T, _stream()), "flatten")
        ctx.shape = (B, C, F, T)
        return out

    @staticmethod
    def backward(ctx, dout):
        B, C, F, T = ctx.shape
        dout = _f32c(dout)
        dx = torch.empty((B, C, F, T), device=dout.device, dtype=torch.float32)
        L.check(_lib().b200asr_flatten_bcft_bwd(L.ptr(dout), L.ptr(dx), B, C, F, T, _stream()), "flatten_bwd")
        return dx


# ----------------------------------------------------------------------------------------------- decoder input side
def preprocess_targets(padded_target: torch.Tensor, tgt_max_len: int):
    """Device-side Decoder.preprocess: returns seq_in, seq_out (int64 [B,Tt]), key_pad (uint8), non_pad (float)."""
    _need_cuda(padded_target)
    tgt = padded_target.to(torch.long).contiguous()
    B, Lt = tgt.shape
    dev = tgt.device
    seq_in = torch.empty((B, tgt_max_len), device=dev, dtype=torch.long)
    seq_out = torch.empty((B, tgt_max_len), device=dev, dtype=torch.long)
    key_pad = torch.empty((B, tgt_max_len), device=dev, dtype=torch.uint8)
    non_pad = torch.empty((B, tgt_max_len), device=dev, dtype=torch.float32)
    status = None
    if Lt + 1 > tgt_max_len:          # only then can an utterance overflow; otherwise no host sync is needed
        status = torch.zeros(1, device=dev, dtype=torch.int32)
    L.check(_lib().b200asr_preprocess_targets(L.ptr(tgt), Lt, L.ptr(seq_in), L.ptr(seq_out), L.ptr(key_pad), L.ptr(non_pad),
                                              L.ptr(status), B, tgt_max_len, _stream()), "preprocess_targets")
    if status is not None and int(status.item()) != 0:
        raise RuntimeError("target longer than tgt_max_len (the reference fails in pad_list, common_layers.py:21)")
    return seq_in, seq_out, key_pad, non_pad


class _PinnedStage:
    """Small host tensors -> device without stalling the launch queue.  The reference's loader hands `input_lengths` over as a
    pageable CPU tensor (utils/data_loader.py:213, trainer.py:63-68); a cudaMemcpyAsync from pageable memory synchronises the
    stream before it starts, i.e. the host stops running ahead of the GPU twice per step (measured: 16.8 -> 19.8 ms per step at
    cfg2).  Here the values go through a small ring of pinned buffers (an event per slot guards reuse) and an async copy."""

    def __init__(self, slots=8):
        self.bufs, self.events, self.i = [None] * slots, [None] * slots, 0

    def to_device(self, t, device):
        t = t.detach().to(torch.int32).contiguous().view(-1)
        n, i = t.numel(), self.i
        self.i = (i + 1) % len(self.bufs)
        if self.bufs[i] is None or self.bufs[i].numel() < n:
            self.bufs[i], self.events[i] = torch.empty(max(n, 256), dtype=torch.int32).pin_memory(), None
        if self.events[i] is not None:
            self.events[i].synchronize()          # the copy that used this slot last has run (it is several steps old)
        buf = self.bufs[i][:n]
        buf.copy_(t)
        with torch.cuda.device(device):
            out = buf.to(device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
        self.events[i] = ev
        return out


_pinned_stage = _PinnedStage()


def length_masks(lengths: torch.Tensor, B: int, T: int, device):
    """key_pad (uint8 [B,T], 1 = frame >= length) and non_pad (float [B,T]) from raw lengths (quirk Q1 preserved)."""
    if lengths.device.type == "cpu":
        lens = _pinned_stage.to_device(lengths, device)
    else:
        lens = lengths.to(device=device, dtype=torch.int32).contiguous()
    key_pad = torch.empty((B, T), device=device, dtype=torch.uint8)
    non_pad = torch.empty((B, T), device=device, dtype=torch.float32)
    L.check(_lib().b200asr_length_masks(L.ptr(lens), L.ptr(key_pad), L.ptr(non_pad), B, T, _stream()), "length_masks")
    return key_pad, non_pad


class EmbedFn(torch.autograd.Function):
    """dropout(Embedding(tokens) * scale + PE[:T])  (models/asr/transformer.py:292-293)."""

    @staticmethod
    def forward(ctx, tokens, table, pe, scale, p_drop, pad_idx):
        _need_cuda(tokens, table, pe)
        B, T = tokens.shape
        V, d = table.shape
        out = torch.empty((B, T, d), device=table.device, dtype=torch.float32)
        seed, off = rng.next() if p_drop > 0.0 else (0, 0)
        L.check(_lib().b200asr_embed_fwd(L.ptr(tokens), L.ptr(_f32c(table)), L.ptr(pe), L.ptr(out), B * T, T, d, V, float(scale),
                                         float(p_drop), seed, off, _stream()), "embed_fwd")
        ctx.save_for_backward(tokens)
        ctx.meta = (V, d, float(scale), float(p_drop), seed, off, int(pad_idx))
        return out

    @staticmethod
    def backward(ctx, dout):
        (tokens,) = ctx.saved_tensors
        V, d, scale, p_drop, seed, off, pad_idx = ctx.meta
        dout = _f32c(dout)
        dtable = torch.zeros((V, d), device=dout.device, dtype=torch.float32)
        L.check(_lib().b200asr_embed_bwd(L.ptr(tokens), L.ptr(dout), L.ptr(dtable), tokens.numel(), d, V, scale, p_drop, seed,
                                         off, pad_idx, _stream()), "embed_bwd")
        return None, dtable, None, None, None, None


# ----------------------------------------------------------------------------------------------- output side
def argmax_rows(logits: torch.Tensor) -> torch.Tensor:
    _need_cuda(logits)
    V = logits.shape[-1]
    x = _f32c(logits.detach()).reshape(-1, V)
    out = torch.empty(x.shape[0], device=x.device, dtype=torch.long)
    L.check(_lib().b200asr_argmax_rows(L.ptr(x), L.ptr(out), x.shape[0], V, _stream()), "argmax_rows")
    return out.view(logits.shape[:-1])


def greedy_step(logits: torch.Tensor, ys: torch.Tensor, finished: torch.Tensor, t: int) -> torch.Tensor:
    """One step of greedy decoding on the device (include/b200asr.h b200asr_greedy_step): returns the next input tokens
    [B,1]; writes ys[:, t] (-1 from the first EOS on) and updates finished[:B] / the finished-utterance counter finished[B]."""
    _need_cuda(logits, ys, finished)
    B, V = logits.shape
    x = _f32c(logits.detach())
    tok = torch.empty((B, 1), device=x.device, dtype=torch.long)
    L.check(_lib().b200asr_greedy_step(L.ptr(x), L.ptr(tok), L.ptr(ys), L.ptr(finished), finished.data_ptr() + 4 * B, B, V, int(t),
                                       ys.shape[1], _stream()), "greedy_step")
    return tok


class BeamBuffers:
    """Device state of one batched beam search over B utterances of W slots (include/b200asr.h b200asr_beam_step): slot 0 of
    every utterance starts live with score 0 and the SOS token, the others dead; the n-best pools start empty."""

    def __init__(self, B, W, nbest, steps, device):
        R = B * W
        self.B, self.W, self.nbest, self.steps = B, W, nbest, steps
        first = torch.arange(R, device=device) % W == 0
        self.score = torch.where(first, 0.0, float("-inf")).to(torch.float32)
        self.state = torch.zeros((R, 4), device=device, dtype=torch.int32)      # live, words, tail, kept index
        self.state[:, 0] = first.to(torch.int32)
        self.state[:, 3] = -1
        self.next_tok = torch.where(first, 1, 0).to(torch.long).view(R, 1)       # SOS; PAD in dead slots
        self.idx = [torch.empty((R, steps + 1), device=device, dtype=torch.int32) for _ in range(2)]
        self.idx[0][:, 0] = (torch.arange(R, device=device) % W).to(torch.int32)
        self.hist_tok = torch.empty((steps, R), device=device, dtype=torch.int32)
        self.hist_par = torch.empty((steps, R), device=device, dtype=torch.int32)
        self.pool_score = torch.full((B, nbest), float("nan"), device=device, dtype=torch.float32)     # NaN: no entry
        self.pool_final = torch.full((B, nbest), float("nan"), device=device, dtype=torch.float32)
        self.pool_ref = torch.full((B, nbest), -1, device=device, dtype=torch.int32)
        self.pool_n = torch.zeros(B, device=device, dtype=torch.int32)
        self.n_live = torch.full((1,), B, device=device, dtype=torch.int32)


def beam_step(buf: BeamBuffers, logits: torch.Tensor, word_tab: torch.Tensor, t: int, t_eos: int, c_weight: float):
    """Step t of the beam search on the device: selection, EOS, word counts, n-best pools, compaction and the index table of
    step t + 1 (written into buf.idx[(t + 1) % 2] from buf.idx[t % 2])."""
    _need_cuda(logits, word_tab)
    x = _f32c(logits.detach())
    V = x.shape[1]
    L.check(_lib().b200asr_beam_step(L.ptr(x), L.ptr(word_tab), buf.B, buf.W, V, int(t), int(t_eos), buf.steps, buf.nbest,
                                     float(c_weight), L.ptr(buf.score), L.ptr(buf.state), L.ptr(buf.next_tok),
                                     L.ptr(buf.idx[t % 2]), L.ptr(buf.idx[(t + 1) % 2]), buf.steps + 1, L.ptr(buf.hist_tok),
                                     L.ptr(buf.hist_par), L.ptr(buf.pool_score), L.ptr(buf.pool_final), L.ptr(buf.pool_ref),
                                     L.ptr(buf.pool_n), L.ptr(buf.n_live), _stream()), "beam_step")


def beam_self_attn(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, idx: torch.Tensor, W: int, H: int, t: int,
                   scale: float) -> torch.Tensor:
    """Single-query attention of every beam row over its history 0..t: q [R, H*dk]; caches [steps, R, H*d]; idx [R, stride]."""
    _need_cuda(q, k_cache, v_cache, idx)
    R = q.shape[0]
    dk, dv = k_cache.shape[2] // H, v_cache.shape[2] // H
    q = _f32c(q)
    if not (k_cache.is_contiguous() and v_cache.is_contiguous() and idx.is_contiguous() and idx.dtype == torch.int32):
        raise RuntimeError("beam_self_attn: caches and the index table must be contiguous (index table int32)")
    out = torch.empty((R, H * dv), device=q.device, dtype=torch.float32)
    L.check(_lib().b200asr_beam_self_attn(L.ptr(q), L.ptr(k_cache), L.ptr(v_cache), L.ptr(idx), L.ptr(out), R, H, W, dk, dv,
                                          int(t), idx.shape[1], float(scale), _stream()), "beam_self_attn")
    return out


def decode_attn(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, H: int, Tk: int, k_strides, v_strides, dv: int,
                scale: float) -> torch.Tensor:
    """Single-query attention of a decode step (include/b200asr.h b200asr_decode_attn): q [R, H*dk] -> out [R, H*dv].  Key j of
    row r starts at element r * k_strides[0] + j * k_strides[1] of `k` (from its first element), V likewise; (H*d, B*H*d) reads
    a slab-major cache [steps, B, H*d], (T*H*d, H*d) a token-major projection [B, T, H*d]."""
    _need_cuda(q, k, v)
    q = _f32c(q)
    R = q.shape[0]
    dk = q.shape[1] // H
    for t, (rs, ks), d in ((k, k_strides, dk), (v, v_strides, dv)):
        if t.dtype != torch.float32:
            raise RuntimeError(f"decode_attn: expected float32 K/V, got {t.dtype}")
        last = t.storage_offset() + (R - 1) * rs + (Tk - 1) * ks + H * d
        if last > t.untyped_storage().nbytes() // 4:
            raise RuntimeError(f"decode_attn: R={R}, Tk={Tk} with strides ({rs}, {ks}) reach past the end of the K/V storage")
    out = torch.empty((R, H * dv), device=q.device, dtype=torch.float32)
    nws = _lib().b200asr_decode_attn_ws_bytes(R, H, int(Tk), dv) // 4
    ws = torch.empty(nws, device=q.device, dtype=torch.float32) if nws else None
    L.check(_lib().b200asr_decode_attn(L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(out), L.ptr(ws), R, H, dk, dv, int(Tk),
                                       int(k_strides[0]), int(k_strides[1]), int(v_strides[0]), int(v_strides[1]), float(scale),
                                       _stream()), "decode_attn")
    return out


def beam_backtrack(buf: BeamBuffers):
    """(ids [B, nbest, steps + 2] int64, lengths [B, nbest] int64) of the pooled hypotheses; see b200asr_beam_backtrack."""
    ids = torch.empty((buf.B, buf.nbest, buf.steps + 2), device=buf.score.device, dtype=torch.long)
    lengths = torch.empty((buf.B, buf.nbest), device=buf.score.device, dtype=torch.long)
    L.check(_lib().b200asr_beam_backtrack(L.ptr(buf.hist_tok), L.ptr(buf.hist_par), L.ptr(buf.pool_ref), L.ptr(buf.pool_n),
                                          L.ptr(ids), L.ptr(lengths), buf.B, buf.W, buf.nbest, buf.steps, _stream()),
            "beam_backtrack")
    return ids, lengths


class EndLog:
    """Every ended hypothesis of a beam search, per utterance in insertion order (include/b200asr.h b200asr_beam_step_log):
    one int32 buffer [B counts | B * cap refs | B * cap fp32 scores], so that the host reads the whole log in one copy."""

    def __init__(self, B, W, steps, device):
        self.B, self.cap = B, W * steps
        self.buf = torch.zeros(B * (1 + 2 * self.cap), device=device, dtype=torch.int32)
        self.n = self.buf[:B]
        self.ref = self.buf[B:B + B * self.cap]
        self.score = self.buf[B + B * self.cap:].view(torch.float32)


def beam_step_log(buf: BeamBuffers, log: EndLog, logits: torch.Tensor, word_tab: torch.Tensor, t: int, t_eos: int, c_weight: float):
    """beam_step that also appends every hypothesis ending at step t to `log`."""
    _need_cuda(logits, word_tab)
    x = _f32c(logits.detach())
    V = x.shape[1]
    L.check(_lib().b200asr_beam_step_log(L.ptr(x), L.ptr(word_tab), buf.B, buf.W, V, int(t), int(t_eos), buf.steps, buf.nbest,
                                         float(c_weight), L.ptr(buf.score), L.ptr(buf.state), L.ptr(buf.next_tok),
                                         L.ptr(buf.idx[t % 2]), L.ptr(buf.idx[(t + 1) % 2]), buf.steps + 1, L.ptr(buf.hist_tok),
                                         L.ptr(buf.hist_par), L.ptr(buf.pool_score), L.ptr(buf.pool_final), L.ptr(buf.pool_ref),
                                         L.ptr(buf.pool_n), L.ptr(buf.n_live), L.ptr(log.ref), L.ptr(log.score), L.ptr(log.n),
                                         log.cap, _stream()), "beam_step_log")


def beam_backtrack_packed(buf: BeamBuffers, log: EndLog, entries, offsets, total: int) -> torch.Tensor:
    """yseqs of the end-log entries `entries` (host int64, b * cap + e), packed from `offsets` (host int64): one copy up, the
    ids stay on the device (int64 [total])."""
    n = len(entries)
    dev = buf.score.device
    ids = torch.empty(max(total, 1), device=dev, dtype=torch.long)
    if n:
        up = torch.from_numpy(np.concatenate([entries, offsets]).astype(np.int64)).to(dev)
        L.check(_lib().b200asr_beam_backtrack_packed(L.ptr(buf.hist_tok), L.ptr(buf.hist_par), L.ptr(log.ref), L.ptr(log.n), log.cap,
                                                     L.ptr(up), up.data_ptr() + 8 * n, n, L.ptr(ids), buf.B, buf.W, buf.steps,
                                                     _stream()), "beam_backtrack_packed")
    return ids[:total]


# ----------------------------------------------------------------------------------------------- LSTM language model
LM_LOGIT_SCRATCH_BYTES = 256 << 20      # logits of at most this many bytes exist at once (chunks of packed positions)


def _pad8(n):
    return (n + 7) // 8 * 8


class LstmLmOperands:
    """Device operands of an LSTM LM (RNNModel("LSTM"): encoder nn.Embedding, rnn nn.LSTM, decoder nn.Linear), built on the
    GPU by b200asr_lstm_prepare / b200asr_split_bf16: the embedding and decoder weights zero-padded to I / H columns, per layer
    the gate-interleaved bf16x3 W_ih and W_hh operands and the folded bias.  `train` (LstmStackFn) also keeps, per layer,
    W_hh_p and the transposed bf16x3 operands of both matrices for the data gradients (`grad_layers`), and builds no decoder
    operands (the decoder runs through LinearFn).  `fresh()` is False once any parameter's version counter (or storage)
    moved since the operands were built."""

    def __init__(self, model, device, train=False):
        rnn = model.rnn
        self.ntoken, self.ninp = model.encoder.weight.shape
        self.nhid, self.nlayers = rnn.hidden_size, rnn.num_layers
        self.I, self.H = _pad8(self.ninp), _pad8(self.nhid)
        self.device = device
        self.params = list(model.parameters())
        self.stamp = self._stamp()
        f32 = dict(device=device, dtype=torch.float32)
        with torch.no_grad():
            dv = lambda t: None if t is None else t.detach().to(**f32).contiguous()
            self.emb = torch.zeros((self.ntoken, self.I), **f32)
            self.emb[:, :self.ninp] = dv(model.encoder.weight)
            self.dec = self.dec_b = self.dec_split = None
            if not train:
                dec = torch.zeros((self.ntoken, self.H), **f32)
                dec[:, :self.nhid] = dv(model.decoder.weight)
                self.dec_b = dv(model.decoder.bias) if model.decoder.bias is not None else torch.zeros(self.ntoken, **f32)
                self.dec_split = self._split(dec)
                self.dec = dec
            self.zero_pe = torch.zeros((1, self.I), **f32)
            self.layers, self.grad_layers = [], []
            for l in range(self.nlayers):
                K = self.I if l == 0 else self.H
                kin = self.ninp if l == 0 else self.nhid
                w_ih_p = torch.empty((4 * self.H, K), **f32)
                w_hh_p = torch.empty((4 * self.H, self.H), **f32)
                bias_p = torch.empty(4 * self.H, **f32)
                g = lambda n: dv(getattr(rnn, f"{n}_l{l}", None))
                w_ih, w_hh, b_ih, b_hh = g("weight_ih"), g("weight_hh"), g("bias_ih"), g("bias_hh")
                L.check(_lib().b200asr_lstm_prepare(L.ptr(w_ih), L.ptr(w_hh), L.ptr(b_ih), L.ptr(b_hh), kin, self.nhid, L.ptr(w_ih_p),
                                                    L.ptr(w_hh_p), L.ptr(bias_p), _stream()), "lstm_prepare")
                ih, ih_t = self._split(w_ih_p, train)
                hh, hh_t = self._split(w_hh_p, train)
                self.layers.append((w_ih_p, ih, hh, bias_p))
                if train:
                    self.grad_layers.append((w_hh_p, ih_t, hh_t))

    def _stamp(self):
        return [(p.data_ptr(), p._version) for p in self.params]

    def fresh(self):
        return self._stamp() == self.stamp

    @staticmethod
    def _split(w, transposed=None):
        """bf16x3 operand [2][N][K] of w [N, K]; with `transposed` given (False / True), the pair (that, the transposed
        operand [2][K][N] or None)."""
        N, K = w.shape
        out = torch.empty((2, N, K), device=w.device, dtype=torch.bfloat16)
        out_t = torch.empty((2, K, N), device=w.device, dtype=torch.bfloat16) if transposed else None
        L.check(_lib().b200asr_split_bf16(L.ptr(w), L.ptr(out), L.ptr(out_t), N, K, 2, _stream()), "split_bf16")
        return out if transposed is None else (out, out_t)


def lstm_lm_operands(model, device) -> LstmLmOperands:
    """The LM's prepared rescoring operands, cached on the module and rebuilt when a parameter changed in place."""
    device = torch.device(device)
    if device.index is None:
        device = torch.device(device.type, torch.cuda.current_device())
    ops_ = model.__dict__.get("_b200_lm_operands")
    if ops_ is None or ops_.device != device or not ops_.fresh():
        ops_ = LstmLmOperands(model, device)
        model.__dict__["_b200_lm_operands"] = ops_
    return ops_


def lstm_layer_fwd(xproj, w_hh_split, batch_sizes, H):
    """One LSTM layer over packed sequences (b200asr_lstm_layer_fwd): xproj [P, 4H] -> h [P, H]; batch_sizes host int32 [T]."""
    bs = np.ascontiguousarray(batch_sizes, dtype=np.int32)
    P = xproj.shape[0]
    h = torch.empty((P, H), device=xproj.device, dtype=torch.float32)
    c = torch.empty((int(bs[0]), H), device=xproj.device, dtype=torch.float32)
    L.check(_lib().b200asr_lstm_layer_fwd(L.ptr(xproj), L.ptr(w_hh_split), bs.ctypes.data, len(bs), H, L.ptr(c), L.ptr(h),
                                          _stream()), "lstm_layer_fwd")
    return h


def lstm_lm_layers(op: LstmLmOperands, inp, batch_sizes):
    """Outputs [P, H] of every LSTM layer over packed word ids `inp` (device int64 [P], t-major, M_t = batch_sizes[t] live
    sequences at step t): layer 0 reads the embedding rows (b200asr_embed_fwd: scale 1, a zero one-row positional table, no
    dropout), each layer's input projection is one linear GEMM over all packed positions, then the recurrence."""
    P = inp.shape[0]
    x = torch.empty((P, op.I), device=inp.device, dtype=torch.float32)
    L.check(_lib().b200asr_embed_fwd(L.ptr(inp), L.ptr(op.emb), L.ptr(op.zero_pe), L.ptr(x), P, 1, op.I, op.ntoken, 1.0, 0.0, 0, 0,
                                     _stream()), "embed_fwd")
    outs = []
    for w_ih_p, ih_split, hh_split, bias_p in op.layers:
        xproj = linear_fwd(x, w_ih_p, bias_p, False, L.PREC_BF16X3, WSplit(ih_split, None))
        x = lstm_layer_fwd(xproj, hh_split, np.asarray(batch_sizes, dtype=np.int32), op.H)
        outs.append(x)
    return outs


def lm_nll(logits, targets, out=None):
    """Exact-fp32 logsumexp(row) - row[target] of every row of logits [rows, V] (row pitch logits.stride(0))."""
    rows, V = logits.shape
    out = torch.empty(rows, device=logits.device, dtype=torch.float32) if out is None else out
    L.check(_lib().b200asr_lm_nll(L.ptr(logits), logits.stride(0), L.ptr(targets), L.ptr(out), rows, V, _stream()), "lm_nll")
    return out


def lstm_lm_nll_sums(model, seqs, device):
    """Summed token NLL of every word-id sequence in `seqs` under the LSTM LM (LM.evaluate, utils/lstm_utils.py:105-127): the
    LSTM runs from a zero state over ids[0 .. n-2] and scores targets ids[1 .. n-1].  Each sequence has n >= 2 ids.  Sequences
    are packed t-major, longest first (stable); the ids go up in one copy.  Returns the fp32 sums in `seqs` order (host)."""
    op = lstm_lm_operands(model, device)
    n = len(seqs)
    if n == 0:
        return np.zeros(0, dtype=np.float32)
    lens = np.array([len(s) - 1 for s in seqs], dtype=np.int64)
    order = np.argsort(-lens, kind="stable")
    T = int(lens[order[0]])
    M = np.array([(lens > t).sum() for t in range(T)], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(M)[:-1]]).astype(np.int64)
    P = int(M.sum())
    inp, tgt = np.empty(P, dtype=np.int64), np.empty(P, dtype=np.int64)
    for j, s in enumerate(order):
        ids = seqs[s]
        pos = off[:lens[s]] + j
        inp[pos] = ids[:-1]
        tgt[pos] = ids[1:]
    up = torch.from_numpy(np.concatenate([inp, tgt, off, lens[order]])).to(device)
    inp_d, tgt_d, off_d, len_d = up[:P], up[P:2 * P], up[2 * P:2 * P + T], up[2 * P + T:]
    x = lstm_lm_layers(op, inp_d, M)[-1]
    nll = torch.empty(P, device=device, dtype=torch.float32)
    chunk = max(1, min(P, LM_LOGIT_SCRATCH_BYTES // (4 * op.ntoken)))
    scratch = torch.empty((chunk, op.ntoken), device=device, dtype=torch.float32)
    for r0 in range(0, P, chunk):
        r1 = min(P, r0 + chunk)
        lg = scratch[:r1 - r0]
        linear_fwd(x[r0:r1], op.dec, op.dec_b, False, L.PREC_BF16X3, WSplit(op.dec_split, None), out=lg)
        lm_nll(lg, tgt_d[r0:r1], out=nll[r0:r1])
    sums = torch.empty(n, device=device, dtype=torch.float32)
    L.check(_lib().b200asr_lm_seq_sum(L.ptr(nll), L.ptr(off_d), L.ptr(len_d), n, L.ptr(sums), _stream()), "lm_seq_sum")
    out = np.empty(n, dtype=np.float32)
    out[order] = sums.cpu().numpy()
    return out


def _lstm_check(model, input, hidden):
    """The argument checks of lstm_stack (ValueError), made before anything is launched."""
    if not torch.is_tensor(input) or input.dtype != torch.int64 or input.dim() != 2 or min(input.shape) < 1:
        raise ValueError("RNNModel.forward: input must be an int64 tensor [T, B] with T, B >= 1, got "
                         f"{getattr(input, 'dtype', type(input))} {tuple(getattr(input, 'shape', ()))}")
    dev = model.encoder.weight.device
    if not input.is_cuda or input.device != dev:
        raise ValueError(f"RNNModel.forward: input is on {input.device}, the model on {dev} (a CUDA device is required)")
    if hidden is None:
        return
    if not isinstance(hidden, (tuple, list)) or len(hidden) != 2:
        raise ValueError("RNNModel.forward: hidden must be the pair (h0, c0)")
    want = (model.rnn.num_layers, input.shape[1], model.rnn.hidden_size)
    for name, t in zip(("h0", "c0"), hidden):
        if not torch.is_tensor(t) or t.dtype != torch.float32 or tuple(t.shape) != want or t.device != dev:
            raise ValueError(f"RNNModel.forward: {name} must be float32 {list(want)} on {dev}, got "
                             f"{getattr(t, 'dtype', type(t))} {list(getattr(t, 'shape', ()))} on {getattr(t, 'device', None)}")


def _pad_rows(x, H):
    """x [..., n] -> contiguous fp32 [rows, H] with zero columns n .. H-1."""
    x2 = x.reshape(-1, x.shape[-1])
    if x2.shape[1] == H:
        return x2.contiguous()
    out = torch.zeros((x2.shape[0], H), device=x.device, dtype=torch.float32)
    out[:, :x2.shape[1]] = x2
    return out


class LstmStackFn(torch.autograd.Function):
    """drop(nn.LSTM(drop(encoder(input)), (h0, c0))) of RNNModel("LSTM").forward (utils/lstm_utils.py:185-190) and its
    backward through time, in the prepared layout of LstmLmOperands(train=True).

    Per layer: the input projection (one bf16x3 GEMM over all T * B rows), b200asr_lstm_layer_train_fwd (gates and cell
    states saved), the dropout of the layer output (between layers: nn.LSTM's, after the last: the model's).  Backward, per
    layer from the top: the output's mask applied again, b200asr_lstm_layer_train_bwd, the weight and bias gradients as
    fixed-order split-K bf16x3 GEMMs, b200asr_lstm_grad_unprepare back to nn.LSTM's layout, dh0 and the input gradient as
    data-gradient GEMMs; the embedding gradient through b200asr_embed_bwd.  Returns (output [T, B, nhid], h_n, c_n)."""

    @staticmethod
    def forward(ctx, op, input, h0, c0, p_emb, p_mid, p_out, enc_w, *rnn_params):
        T, B = input.shape
        H, I, nl = op.H, op.I, op.nlayers
        lib, st = _lib(), _stream()
        dev = input.device
        f32 = dict(device=dev, dtype=torch.float32)
        inp = input.contiguous().view(-1)
        x = torch.empty((T * B, I), **f32)
        emb_key = rng.next() if p_emb > 0.0 else (0, 0)
        L.check(lib.b200asr_embed_fwd(L.ptr(inp), L.ptr(op.emb), L.ptr(op.zero_pe), L.ptr(x), T * B, 1, I, op.ntoken, 1.0,
                                      float(p_emb), emb_key[0], emb_key[1], st), "embed_fwd")
        has_state = h0 is not None
        h0p = _pad_rows(h0, H).view(nl, B, H) if has_state else None
        c0p = _pad_rows(c0, H).view(nl, B, H) if has_state else None
        saved, keys = [], []
        for l, (w_ih_p, ih_split, hh_split, bias_p) in enumerate(op.layers):
            xproj = linear_fwd(x, w_ih_p, bias_p, False, L.PREC_BF16X3, WSplit(ih_split, None))
            h = torch.empty(((T + 1) * B, H), **f32)
            c = torch.empty((T * B, H), **f32)
            gates = torch.empty((T * B, 4 * H), **f32)
            if has_state:
                h[:B] = h0p[l]
            L.check(lib.b200asr_lstm_layer_train_fwd(L.ptr(xproj), L.ptr(hh_split), T, B, H, int(has_state),
                                                     L.ptr(c0p[l]) if has_state else None, L.ptr(h), L.ptr(c), L.ptr(gates), st),
                    "lstm_layer_train_fwd")
            saved += [x, h, c, gates]
            y = h[B:]
            p = float(p_mid if l < nl - 1 else p_out)
            key = rng.next() if p > 0.0 else None
            if key is not None:
                yd = torch.empty_like(y)
                L.check(lib.b200asr_lstm_dropout(L.ptr(y), L.ptr(yd), y.numel(), p, key[0], key[1], st), "lstm_dropout")
                y = yd
            keys.append((p, key))
            x = y
        n = op.nhid
        out = x.view(T, B, H)[:, :, :n]
        h_n = torch.stack([saved[4 * l + 1][T * B:, :n] for l in range(nl)])
        c_n = torch.stack([saved[4 * l + 2][(T - 1) * B:, :n] for l in range(nl)])
        ctx.save_for_backward(inp, c0p, *saved)
        ctx.op, ctx.keys, ctx.emb_key, ctx.p_emb, ctx.TB = op, keys, emb_key, float(p_emb), (T, B)
        if n != H or keys[-1][1] is None:        # (otherwise out views a saved buffer)
            out = out.clone(memory_format=torch.contiguous_format)
        return out, h_n, c_n

    @staticmethod
    def backward(ctx, d_out, d_hn, d_cn):
        inp, c0p, *saved = ctx.saved_tensors
        op, (T, B) = ctx.op, ctx.TB
        H, I, nl, n = op.H, op.I, op.nlayers, op.nhid
        lib, st = _lib(), _stream()
        f32 = dict(device=inp.device, dtype=torch.float32)
        need = ctx.needs_input_grad
        grads = [None] * (4 * nl)
        dh0 = torch.zeros((nl, B, n), **f32) if need[2] else None
        dc0 = torch.zeros((nl, B, n), **f32) if need[3] else None
        dy = _pad_rows(d_out, H) if d_out is not None else torch.zeros((T * B, H), **f32)
        need_emb = need[7]
        for l in range(nl - 1, -1, -1):
            x, h, c, gates = saved[4 * l:4 * l + 4]
            w_ih_p, _, _, _ = op.layers[l]
            w_hh_p, ih_t, hh_t = op.grad_layers[l]
            p, key = ctx.keys[l]
            if key is not None:
                dym = torch.empty_like(dy)
                L.check(lib.b200asr_lstm_dropout(L.ptr(dy), L.ptr(dym), dy.numel(), p, key[0], key[1], st), "lstm_dropout")
                dy = dym
            dh_n = _pad_rows(d_hn[l], H) if d_hn is not None else None
            dc_n = _pad_rows(d_cn[l], H) if d_cn is not None else None
            dgates = torch.empty((T * B, 4 * H), **f32)
            dc = torch.empty((B, H), **f32)
            dc0p = torch.empty((B, H), **f32) if dc0 is not None else None
            L.check(lib.b200asr_lstm_layer_train_bwd(L.ptr(gates), L.ptr(c), L.ptr(c0p[l]) if c0p is not None else None, L.ptr(dy),
                                                     L.ptr(dh_n), L.ptr(dc_n), L.ptr(hh_t), T, B, H, L.ptr(dc), L.ptr(dgates),
                                                     L.ptr(dc0p), st), "lstm_layer_train_bwd")
            if dc0 is not None:
                dc0[l] = dc0p[:, :n]
            if dh0 is not None:
                dh0[l] = linear_bwd_data(dgates[:B], w_hh_p, None, L.PREC_BF16X3, WSplit(None, hh_t))[:, :n]
            pw = [need[8 + 4 * l + j] for j in range(4)]
            if any(pw):
                kin = op.ninp if l == 0 else n
                dw_ih_p, db_p = linear_bwd_weight(dgates, x, True, L.PREC_BF16X3)
                dw_hh_p, _ = linear_bwd_weight(dgates, h[:T * B], False, L.PREC_BF16X3)
                g = [torch.empty((4 * n, kin), **f32) if pw[0] else None, torch.empty((4 * n, n), **f32) if pw[1] else None,
                     torch.empty(4 * n, **f32) if pw[2] else None, torch.empty(4 * n, **f32) if pw[3] else None]
                L.check(lib.b200asr_lstm_grad_unprepare(L.ptr(dw_ih_p), L.ptr(dw_hh_p), L.ptr(db_p), kin, n, *[L.ptr(t) for t in g], st),
                        "lstm_grad_unprepare")
                grads[4 * l:4 * l + 4] = g
            if l > 0 or need_emb:
                dy = linear_bwd_data(dgates, w_ih_p, None, L.PREC_BF16X3, WSplit(None, ih_t))
        d_enc = None
        if need_emb:
            dtable = torch.zeros((op.ntoken, I), **f32)
            L.check(lib.b200asr_embed_bwd(L.ptr(inp), L.ptr(dy), L.ptr(dtable), T * B, I, op.ntoken, 1.0, ctx.p_emb, ctx.emb_key[0],
                                          ctx.emb_key[1], -1, st), "embed_bwd")
            d_enc = dtable[:, :op.ninp] if I != op.ninp else dtable
        return (None, None, dh0, dc0, None, None, None, d_enc, *grads)


def lstm_stack(model, input, hidden, p_emb=0.0, p_mid=0.0, p_out=0.0):
    """The embedding, the LSTM and the output dropout of RNNModel("LSTM").forward on the device (LstmStackFn): input int64
    [T, B], hidden (h0, c0) fp32 [nlayers, B, nhid] or None (zero state); p_emb / p_mid / p_out are the dropout
    probabilities of the embedding, between layers and of the last layer's output.  Returns (output, (h_n, c_n))."""
    _lstm_check(model, input, hidden)
    rnn = model.rnn
    # prepared on every call, not cached by version stamp: the word-language-model loop updates the weights through
    # `p.data`, which leaves the parameters' version counters unchanged (and in training they change every step anyway)
    op = LstmLmOperands(model, input.device, train=True)
    params = [getattr(rnn, f"{nm}_l{l}", None) for l in range(rnn.num_layers) for nm in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    h0, c0 = hidden if hidden is not None else (None, None)
    out, h_n, c_n = LstmStackFn.apply(op, input, h0, c0, float(p_emb), float(p_mid), float(p_out), model.encoder.weight, *params)
    return out, (h_n, c_n)


class CrossEntropyFn(torch.autograd.Function):
    """Label-smoothed CE / CE of utils/metrics.py:115-132 plus num_correct (:88-94), one pass over the logits.

    Returns (loss, stats): loss is a 0-dim tensor -- the mean over non-PAD tokens (reduction='mean', the
    reference's value) or the plain sum (reduction='sum', used by the data-parallel step which divides by the
    all-reduced global token count).  stats = [sum, n_tokens, n_correct, mean, 1/n_tokens] (not differentiable)."""

    @staticmethod
    def forward(ctx, pred, gold, smoothing, reduction):
        _need_cuda(pred, gold)
        V = pred.shape[-1]
        x = _f32c(pred).reshape(-1, V)
        g = gold.to(torch.long).contiguous().reshape(-1)
        rows = x.shape[0]
        lse = torch.empty(rows, device=x.device, dtype=torch.float32)
        stats = torch.empty(5, device=x.device, dtype=torch.float32)
        loss = torch.empty((), device=x.device, dtype=torch.float32)
        mean = reduction == "mean"
        lib, st = _lib(), _stream()
        L.check(lib.b200asr_ce_fwd(L.ptr(x), L.ptr(g), L.ptr(lse), L.ptr(stats), rows, V, float(smoothing), st), "ce_fwd")
        L.check(lib.b200asr_ce_finalize(L.ptr(stats), L.ptr(loss), int(mean), st), "ce_finalize")
        ctx.save_for_backward(x, g, lse, stats)
        ctx.meta = (pred.shape, float(smoothing), mean)
        ctx.mark_non_differentiable(stats)
        return loss, stats

    @staticmethod
    def backward(ctx, dloss, _dstats):
        x, g, lse, stats = ctx.saved_tensors
        shape, smoothing, mean = ctx.meta
        rows, V = x.shape
        gs = _f32c(dloss)                               # device scalar: no host sync
        inv_n = stats[4:5] if mean else None            # device scalar 1/num_word
        dx = torch.empty_like(x)
        L.check(_lib().b200asr_ce_bwd(L.ptr(x), L.ptr(g), L.ptr(lse), L.ptr(dx), rows, V, smoothing, 1.0, L.ptr(gs),
                                      L.ptr(inv_n), _stream()), "ce_bwd")
        return dx.view(shape), None, None, None


def _ctc_host_lengths(lengths, B, limit, what):
    """The lengths of one ctc_loss argument as host ints, checked as torch's ctc_loss checks them: B values in [0, limit].
    CPU tensors (the reference's `sizes` and loader `tgt_lengths`) need no device sync; device tensors are read back."""
    if not torch.is_tensor(lengths):
        lengths = torch.as_tensor(lengths)
    vals = lengths.detach().reshape(-1).cpu().tolist()
    if len(vals) != B:
        raise RuntimeError(f"ctc_loss: expected {what} to have {B} entries, got {len(vals)}")
    for v in vals:
        if v < 0:
            raise RuntimeError(f"ctc_loss: {what} must be non-negative, got {v}")
        if v > limit:
            raise RuntimeError(f"ctc_loss: expected {what} to have value at most {limit}, but got value {v}")
    return vals


class CtcLossFn(torch.autograd.Function):
    """CTC loss of utils/metrics.py:133-154 -- F.ctc_loss(log_softmax(pred.transpose(0, 1), 2), gold, input_lengths,
    target_lengths, blank=0, reduction="mean") -- from the [B, T, V] logits in place (b200asr_ctc_fwd / _bwd).

    pred: CUDA fp32 [B, T, V]; targets: [B, S] (padded, row b read up to target_lengths[b]); the lengths: [B] integer
    tensors, validated on the host (0 <= input_lengths <= T, 0 <= target_lengths <= S) and staged through pinned memory,
    so with CPU lengths neither direction synchronises the host.  Returns the 0-dim mean loss (+inf if some utterance has
    no alignment; its gradient rows are then NaN, as torch's)."""

    @staticmethod
    def forward(ctx, pred, targets, input_lengths, target_lengths):
        _need_cuda(pred, targets)
        if pred.dim() != 3 or targets.dim() != 2 or targets.shape[0] != pred.shape[0]:
            raise RuntimeError(f"ctc_loss: expected pred [B, T, V] and targets [B, S], got {tuple(pred.shape)} and "
                               f"{tuple(targets.shape)}")
        B, T, V = pred.shape
        S = targets.shape[1]
        il = _ctc_host_lengths(input_lengths, B, T, "input_lengths")
        tl = _ctc_host_lengths(target_lengths, B, S, "target_lengths")
        lmax = max(tl)
        dev = pred.device
        x = _f32c(pred)
        tg = targets.to(torch.long).contiguous()
        lens = _pinned_stage.to_device(torch.tensor(il + tl, dtype=torch.int32), dev)
        lib, st = _lib(), _stream()
        ws = torch.empty(lib.b200asr_ctc_ws_bytes(B, T, lmax), device=dev, dtype=torch.uint8)
        nll = torch.empty(B, device=dev, dtype=torch.float32)
        loss = torch.empty((), device=dev, dtype=torch.float32)
        L.check(lib.b200asr_ctc_fwd(L.ptr(x), L.ptr(tg), L.ptr(lens), L.ptr(lens[B:]), L.ptr(nll), L.ptr(loss), L.ptr(ws), B, T,
                                    V, S, lmax, st), "ctc_fwd")
        ctx.save_for_backward(x, tg, lens, nll, ws)
        ctx.meta = (pred.shape, lmax)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        x, tg, lens, nll, ws = ctx.saved_tensors
        (B, T, V), lmax = ctx.meta
        dx = torch.empty_like(x)
        L.check(_lib().b200asr_ctc_bwd(L.ptr(x), L.ptr(tg), L.ptr(lens), L.ptr(lens[B:]), L.ptr(nll), L.ptr(_f32c(dloss)),
                                       L.ptr(dx), L.ptr(ws), B, T, V, tg.shape[1], lmax, _stream()), "ctc_bwd")
        return dx, None, None, None
