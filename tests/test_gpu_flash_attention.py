"""The flash-style attention kernels through the raw C ABI against float64 references, at every template instantiation and at
the edges where tiled attention goes wrong:

  - fp32 (attention_simt.cu, b200asr_sdpa_fwd / _bwd precision 0): every (dk, dv) pair of the forward and the backward;
  - TF32 (tc_flash.cu, precision 1): (dk, dv) in {32, 64}^2;
  - bf16x3 (tc_flash.cu, b200asr_sdpa_fused_fwd / _bwd): dk = dv = 64.

Both kernel families use 64-row query and key tiles; the tensor-core kernels split them into 16-row warps and 8-key MMA
steps.  Covered: Tq and Tk on both sides of every tile and warp boundary (Tq = 1 is cached greedy decoding), Tk above the
materialised path's cap for fp32, no mask, ragged key padding with an utterance of one live key, causal with Tq > Tk and
Tq < Tk (the kernels skip whole tiles there), a dense mask, a fully masked query row (alone and under causal), the layouts
the library passes (token-major q / out, q / k / v / dq / dk / dv as column slices of one packed projection buffer, the
head-major output of the reference signature), dropout against float64 with the keep mask restated on the host, the
log-sum-exp both backward kernels read, reproducibility of the tensor-core backward, the shape rejections, and the shape
rules of ops.SdpaFn.

Outputs and workspaces (out, lse, dq, dk, dv, delta, ws16, ws_bwd) are filled with NaN before each call, so an element a
kernel fails to write, or reads without writing, shows up.  A fully masked row follows the reference's masked_fill ->
softmax: that row of O is NaN, its lse is NaN (the value pinned for all three paths), its dQ row is exactly 0, dK stays
finite, and all of dV of that (utterance, head) is NaN, because the row of P is NaN and dV = P^T dO.  Bars are max-norm
relative errors (tests.helpers.rel_err); each states the error measured on one H100 80GB HBM3 (700 W limit) and sits about 3x above it."""
import numpy as np
import pytest
import torch

from tests.helpers import rel_err
from tests.test_gpu_row_kernels import _finite_err, _gen, _inv_keep, _nan, _same_nan, _stream, _thresh16, attn_mask, attn_ref

NAN = float("nan")
BAD_SHAPE = -1
gpu = pytest.mark.gpu
PATHS = ["fp32", "tf32", "bf16x3"]
PREC = {"fp32": 0, "tf32": 1}
SEED, OFFSET = 0x5EED1234, 9

# measured maxima over every case of this file (see compare() for grad / grad_1key):
#   fp32   o 1.2e-6 (Tk = 2500), lse 1.8e-7, grad 9.3e-7, grad_1key 2.1e-5 (Tk = 2049)
#   tf32   o 8.5e-4, lse 9.3e-4 (Tq = 1), grad 1.3e-3, grad_1key 1.2e-2 (Tq = 129, Tk = 448)
#   bf16x3 o 1.5e-5, lse 1.3e-5 (Tq = 1), grad 2.1e-5, grad_1key 2.8e-4 (Tq = 129, Tk = 448)
BARS = {
    "fp32": dict(o=3.5e-6, lse=6e-7, grad=3e-6, grad_1key=6e-5),
    "tf32": dict(o=2.5e-3, lse=3e-3, grad=4e-3, grad_1key=3.5e-2),
    "bf16x3": dict(o=4.5e-5, lse=4e-5, grad=6e-5, grad_1key=9e-4),
}


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _s(t):
    """(batch, head, row) element strides of a (B, H, T, d) view."""
    assert t.stride(3) == 1
    return t.stride(0), t.stride(1), t.stride(2)


def _nan_like(t):
    return torch.empty_strided(t.shape, t.stride(), device="cuda").fill_(NAN)


def _token_major(B, T, H, d):
    """A NaN-filled [B, T, H, d] buffer as its (B, H, T, d) view."""
    return _nan(B, T, H, d).permute(0, 2, 1, 3)


def _check_errs(errs, bars):
    for key, err in errs.items():
        assert err < bars[key], f"{key}: {err:.3e} >= {bars[key]:.1e}"


# ================================================================================================ host restatements
_U64 = (1 << 64) - 1


def _splitmix64(z):
    """common.cuh splitmix64 on a numpy uint64 array (wrapping arithmetic)."""
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _dropout_key(seed, offset):
    """common.cuh dropout_key(seed, stream = offset)."""
    mixed = (seed ^ ((offset * 0xD1342543DE82EF95 + 0x2545F4914F6CDD1D) & _U64)) & _U64
    return int(_splitmix64(np.array([mixed], dtype=np.uint64))[0])


def keep_mask(B, H, Tq, Tk, p, seed=SEED, offset=OFFSET):
    """common.cuh dropout_keep for every (b, h, q, key) of an attention call: element index (((b H + h) Tq + q) Tk + key),
    16-bit lane idx & 3 of splitmix64(key + (idx >> 2) * golden); kept iff the lane >= the 16-bit threshold.  [B, H, Tq, Tk]
    bool."""
    with np.errstate(over="ignore"):
        idx = np.arange(B * H * Tq * Tk, dtype=np.uint64)
        r = _splitmix64(np.uint64(_dropout_key(seed, offset)) + (idx >> np.uint64(2)) * np.uint64(0x9E3779B97F4A7C15))
        bits = (r >> (np.uint64(16) * (idx & np.uint64(3)))) & np.uint64(0xFFFF)
    return torch.from_numpy(bits >= np.uint64(_thresh16(p))).view(B, H, Tq, Tk)


# ================================================================================================ problems and calls
class Problem:
    """q / k / v / dout as (B, H, T, d) views plus the masks of one attention call."""

    def __init__(self, q, k, v, dout, key_pad=None, dense=None, causal=False, p_drop=0.0):
        self.q, self.k, self.v, self.dout = q, k, v, dout
        self.key_pad = None if key_pad is None else key_pad.cuda()
        self.dense = None if dense is None else dense.cuda()
        self.causal, self.p_drop = causal, p_drop
        self.B, self.H, self.Tq, self.dk = q.shape
        self.Tk, self.dv = k.shape[2], v.shape[3]
        self.scale = self.dk ** -0.5

    def dims(self):
        return self.B, self.H, self.Tq, self.Tk, self.dk, self.dv


MASKS = ["none", "key_pad", "causal", "dense", "dead_row", "dead_row_causal"]


def make_problem(B, H, Tq, Tk, dk, dv, mode, seed, p_drop=0.0):
    """q token-major [B, Tq, H, dk] (the projections' layout), k / v head-major [B, H, Tk, d]; masks for `mode`: key padding
    with the second utterance down to one live key, causal, a dense mask that leaves every row a key, and one fully masked
    query row in every head of the last utterance (dense), alone or under causal."""
    g = _gen(seed)
    q = torch.randn(B, Tq, H, dk, generator=g).cuda().permute(0, 2, 1, 3)
    k = torch.randn(B, H, Tk, dk, generator=g).cuda()
    v = torch.randn(B, H, Tk, dv, generator=g).cuda()
    dout = torch.randn(B, Tq, H, dv, generator=g).cuda().permute(0, 2, 1, 3)
    key_pad = dense = None
    if mode == "key_pad":
        lens = torch.tensor([Tk] + [max(1, Tk - 7 * i) for i in range(1, B - 1)] + [1])[:B]
        key_pad = (torch.arange(Tk)[None, :] >= lens[:, None]).to(torch.uint8)
    if mode == "dense":
        dense = (torch.rand(B, Tq, Tk, generator=g) < 0.3).to(torch.uint8)
        dense[:, torch.arange(Tq), torch.arange(Tq) % Tk] = 0
    if mode.startswith("dead_row"):
        dense = torch.zeros(B, Tq, Tk, dtype=torch.uint8)
        dense[B - 1, Tq // 2] = 1
    return Problem(q, k, v, dout, key_pad, dense, mode in ("causal", "dead_row_causal"), p_drop)


def call_fwd(L, path, pb, out, lse, ws16=None):
    """b200asr_sdpa_fwd (fp32 / tf32) or b200asr_sdpa_fused_fwd (bf16x3); returns the status code."""
    lib = L.load()
    args = (L.ptr(pb.q), L.ptr(pb.k), L.ptr(pb.v), *_s(pb.q), *_s(pb.k), *_s(pb.v), L.ptr(pb.key_pad), L.ptr(pb.dense),
            int(pb.causal), L.ptr(out), *_s(out), L.ptr(lse))
    tail = (*pb.dims(), pb.scale, pb.p_drop, SEED, OFFSET)
    if path == "bf16x3":
        if ws16 is None:
            ws16 = torch.full((lib.b200asr_sdpa_fused_ws_bytes(pb.B, pb.H, pb.Tq, pb.Tk) // 2,), NAN, dtype=torch.bfloat16,
                              device="cuda")
        return lib.b200asr_sdpa_fused_fwd(*args, L.ptr(ws16), *tail, _stream())
    return lib.b200asr_sdpa_fwd(*args, *tail, PREC[path], _stream())


def call_bwd(L, path, pb, dout, out, lse, dq, dk, dv, ws=None):
    """b200asr_sdpa_bwd (fp32 / tf32; ws = delta) or b200asr_sdpa_fused_bwd (bf16x3; ws = ws_bwd, ws16 NaN-filled);
    returns the status code."""
    lib = L.load()
    args = (L.ptr(dout), L.ptr(pb.q), L.ptr(pb.k), L.ptr(pb.v), L.ptr(out), L.ptr(lse), *_s(pb.q), *_s(pb.k), *_s(pb.v),
            *_s(out), L.ptr(pb.key_pad), L.ptr(pb.dense), int(pb.causal), L.ptr(dq), L.ptr(dk), L.ptr(dv))
    tail = (*pb.dims(), pb.scale, pb.p_drop, SEED, OFFSET)
    if path == "bf16x3":
        ws16 = torch.full((lib.b200asr_sdpa_fused_ws_bytes(pb.B, pb.H, pb.Tq, pb.Tk) // 2,), NAN, dtype=torch.bfloat16,
                          device="cuda")
        if ws is None:
            ws = _nan(lib.b200asr_sdpa_fused_bwd_ws_bytes(pb.B, pb.H, pb.Tq) // 4)
        return lib.b200asr_sdpa_fused_bwd(*args, L.ptr(ws16), L.ptr(ws), *tail, _stream())
    if ws is None:
        ws = _nan(pb.B, pb.H, pb.Tq)
    return lib.b200asr_sdpa_bwd(*args, L.ptr(ws), *tail, PREC[path], _stream())


def run(L, path, pb, out=None, grads=None):
    """Forward then backward with every output and workspace NaN-poisoned.  out: a (B, H, Tq, dv) view (default
    token-major); grads: (dq, dk, dv) views with the strides of q / k / v (default: NaN buffers of those strides).
    Returns (out, lse, dq, dk, dv)."""
    if out is None:
        out = _token_major(pb.B, pb.Tq, pb.H, pb.dv)
    lse = _nan(pb.B, pb.H, pb.Tq)
    L.check(call_fwd(L, path, pb, out, lse), f"{path} fwd")
    dout = torch.empty_strided(out.shape, out.stride(), device="cuda").copy_(pb.dout)
    dq, dk, dv = grads if grads is not None else (_nan_like(pb.q), _nan_like(pb.k), _nan_like(pb.v))
    L.check(call_bwd(L, path, pb, dout, out, lse, dq, dk, dv), f"{path} bwd")
    return out, lse, dq, dk, dv


def reference(pb, keep=None):
    """float64 masked_fill -> softmax -> (dropout with the given keep mask) -> matmul and its autograd backward, on the GPU;
    plus the log-sum-exp of the masked scaled scores (-inf on a fully masked row)."""
    mask = attn_mask(pb.B, pb.Tq, pb.Tk, pb.key_pad, pb.dense, pb.causal, device="cuda")
    q64, k64, v64 = (t.detach().double().requires_grad_(True) for t in (pb.q, pb.k, pb.v))
    kd = None if keep is None else keep.cuda().double()
    o, _ = attn_ref(q64, k64, v64, mask, pb.scale, kd, _inv_keep(pb.p_drop) if keep is not None else 1.0)
    o.backward(pb.dout.double())
    with torch.no_grad():
        s = torch.matmul(q64, k64.transpose(-1, -2)) * pb.scale
        lse = torch.logsumexp(s.masked_fill(mask[:, None], float("-inf")), dim=-1)
    return o.detach(), lse, q64.grad, k64.grad, v64.grad


def compare(got, ref, pb):
    """NaN exactly where float64 has it (out, dq, dk, dv), lse NaN exactly on the fully masked rows and their dQ rows exactly
    0; returns the max-norm relative errors on the rest: o, lse, and the gradients as `grad` over the utterances where some
    query row sees two keys or more, and as `grad_1key` over whole tensors when an utterance's rows each see at most one
    key.  There P is 1 or 0, dQ and dK are exactly 0 in float64, and the kernels return the rounding of dP - delta with the
    flash-style delta = rowsum(dO o O): error measured against the rest of the tensor (absolute where all of it is 0)."""
    out, lse, dq, dk, dv = got
    o_ref, lse_ref, dq_ref, dk_ref, dv_ref = ref
    dead = torch.isinf(lse_ref).cpu()
    for name, a, b in (("out", out, o_ref), ("dq", dq, dq_ref), ("dk", dk, dk_ref), ("dv", dv, dv_ref)):
        assert _same_nan(a, b), f"{name}: NaN pattern differs from float64"
    assert torch.equal(torch.isnan(lse).cpu(), dead), "lse: NaN pattern differs from the fully masked rows"
    assert not dq.cpu()[dead].any(), "dq of a fully masked row is not 0"
    lc = lse.cpu()
    errs = dict(o=_finite_err(out, o_ref), lse=rel_err(lc[~dead], lse_ref.cpu()[~dead]) if bool((~dead).any()) else 0.0)
    mask = attn_mask(pb.B, pb.Tq, pb.Tk, pb.key_pad, pb.dense, pb.causal, device="cuda")
    single = ((~mask).sum(-1) <= 1).all(-1).cpu()                       # [B]
    pairs = ((dq, dq_ref), (dk, dk_ref), (dv, dv_ref))
    if not bool(single.all()):
        errs["grad"] = max(_finite_err(a.cpu()[~single], b.cpu()[~single]) for a, b in pairs)
    if bool(single.any()):
        errs["grad_1key"] = max(_finite_err(a, b) for a, b in pairs)
    return errs


# ================================================================================================ tile edges and masks
TQ_EDGE = [1, 15, 16, 17, 63, 64, 65, 129]
TK_EDGE = [1, 7, 63, 64, 65, 128, 129, 447, 448]
EDGE_SHAPES = list(dict.fromkeys([(tq, 65) for tq in TQ_EDGE] + [(17, tk) for tk in TK_EDGE] + [(129, 448), (65, 129)]))
EDGE_CASES = [(path, tq, tk) for path in PATHS for tq, tk in EDGE_SHAPES] + [("fp32", 17, 2049), ("fp32", 70, 2500)]


@gpu
@pytest.mark.parametrize("mode", MASKS)
@pytest.mark.parametrize("path,Tq,Tk", EDGE_CASES)
def test_flash_attention_edges_against_float64(L, path, Tq, Tk, mode):
    """dk = dv = 64, B = 2, H = 2: out, lse, dQ, dK, dV against float64 at Tq on both sides of the 16-row warp and 64-row tile
    boundaries and Tk on both sides of the 8-key MMA step and the 64-key block up to the tensor-core cap of 448 (fp32: also
    2049 and 2500, past the materialised path's cap), for every mask; causal covers Tq > Tk and Tq < Tk.  The fully masked
    row follows the reference (see the module docstring), also under causal, where the dK / dV kernel skips the query tiles
    before its key block.  Measured maxima and bars: BARS."""
    pb = make_problem(2, 2, Tq, Tk, 64, 64, mode, seed=Tq * 1000 + Tk + len(mode))
    errs = compare(run(L, path, pb), reference(pb), pb)
    _check_errs(errs, BARS[path])


# ================================================================================================ every instantiation
INSTANCES = ([("fp32", dk, dv) for dk in (16, 32, 64, 128) for dv in (16, 32, 64, 128)] +
             [("tf32", dk, dv) for dk in (32, 64) for dv in (32, 64)] + [("bf16x3", 64, 64)])


@gpu
@pytest.mark.parametrize("mode", ["key_pad", "dead_row_causal"])
@pytest.mark.parametrize("path,dk,dv", INSTANCES)
def test_flash_attention_instantiations_against_float64(L, path, dk, dv, mode):
    """Every (dk, dv) instantiation of each path -- for fp32 all 16 pairs of the forward (templated on dv, dk a runtime
    loop bound) and of the backward --, Tq = 70 and Tk = 131 (partial last tiles), with ragged key padding and with a
    fully masked row under causal.  Measured maxima and bars: BARS."""
    pb = make_problem(2, 3, 70, 131, dk, dv, mode, seed=dk * 10 + dv + len(mode))
    errs = compare(run(L, path, pb), reference(pb), pb)
    _check_errs(errs, BARS[path])


# ================================================================================================ layouts
LAYOUT_DIMS = {"fp32": (64, 32), "tf32": (32, 64), "bf16x3": (64, 64)}


@gpu
@pytest.mark.parametrize("layout", ["packed", "head_major_out"])
@pytest.mark.parametrize("path", PATHS)
def test_flash_attention_layouts_against_float64(L, path, layout):
    """The layouts ops passes.  packed: q, k and v are column slices of one [B*T, 3*H*d + 16] buffer and dq, dk, dv are
    written into the matching slices of a second one (AttnProjFn's stacked projections), with 4 NaN columns before, between
    and after the slices that must stay NaN in both buffers; out token-major.  head_major_out: out in (H, B, Tq, dv) memory
    (the reference signature's (H*B) x Tq x dv), q token-major.  Key padding and causal (a decoder self-attention).
    Measured maxima and bars: BARS."""
    dk, dv = LAYOUT_DIMS[path]
    B, H, T = 3, 2, 100
    seed = len(path) * 10 + len(layout)
    if layout == "packed":
        cols = [4, 4 + H * dk + 4, 4 + 2 * H * dk + 8]                 # q, k, v column offsets (16-byte aligned)
        W = cols[2] + H * dv + 4
        buf, gbuf = _nan(B * T, W), _nan(B * T, W)
        view = lambda t, c0, d: t.view(B, T, W)[:, :, c0:c0 + H * d].unflatten(2, (H, d)).permute(0, 2, 1, 3)
        g = _gen(seed)
        q, k, v = view(buf, cols[0], dk), view(buf, cols[1], dk), view(buf, cols[2], dv)
        for t in (q, k, v):
            t.copy_(torch.randn(t.shape, generator=g))
        dout = torch.randn(B, T, H, dv, generator=g).cuda().permute(0, 2, 1, 3)
        lens = torch.tensor([T, T - 37, 1])
        key_pad = (torch.arange(T)[None, :] >= lens[:, None]).to(torch.uint8)
        pb = Problem(q, k, v, dout, key_pad, None, True)
        grads = (view(gbuf, cols[0], dk), view(gbuf, cols[1], dk), view(gbuf, cols[2], dv))
        got = run(L, path, pb, grads=grads)
        gaps = torch.ones(W, dtype=torch.bool)
        for c0, d in zip(cols, (dk, dk, dv)):
            gaps[c0:c0 + H * d] = False
        assert torch.isnan(buf[:, gaps.cuda()]).all() and torch.isnan(gbuf[:, gaps.cuda()]).all()
    else:
        pb = make_problem(B, H, T, T + 29, dk, dv, "key_pad", seed=seed)
        pb.causal = True
        out = _nan(H, B, T, dv).permute(1, 0, 2, 3)
        got = run(L, path, pb, out=out)
    errs = compare(got, reference(pb), pb)
    _check_errs(errs, BARS[path])


# ================================================================================================ dropout
@gpu
@pytest.mark.parametrize("Tk", [64, 131])
def test_dropout_restatement_matches_materialised_keep_mask(L, Tk):
    """keep_mask (the host restatement of splitmix64 / dropout_key / dropout_keep) equals, bit for bit, the keep mask the
    materialised path exposes (probs_drop != 0 where P != 0).  Tk = 64 draws four columns per 64-bit number in one go, Tk =
    131 one element at a time."""
    lib = L.load()
    B, H, Tq, d, p = 2, 2, 37, 32, 0.3
    g = _gen(Tk)
    q, k, v = (torch.randn(B, H, t, d, generator=g).cuda() for t in (Tq, Tk, Tk))
    n = lib.b200asr_sdpa_mat_ws_bytes(B, H, Tq, Tk) // 4
    ldp = n // (B * H * Tq)
    probs, probs_drop, out = _nan(n), _nan(n), _nan(B, H, Tq, d)
    L.check(lib.b200asr_sdpa_mat_fwd(L.ptr(q), L.ptr(k), L.ptr(v), *_s(q), *_s(k), *_s(v), None, None, 0, L.ptr(out), *_s(out),
                                     L.ptr(probs), L.ptr(probs_drop), B, H, Tq, Tk, d, d, d ** -0.5, p, SEED, OFFSET, 3,
                                     _stream()), "sdpa_mat_fwd")
    P = probs.view(B, H, Tq, ldp)[..., :Tk].cpu()
    kept = (probs_drop.view(B, H, Tq, ldp)[..., :Tk] != 0).cpu()
    live = P != 0
    assert bool(live.all())
    host = keep_mask(B, H, Tq, Tk, p)
    assert torch.equal(host, kept)
    assert 0.6 < float(host.float().mean()) < 0.8


@gpu
@pytest.mark.parametrize("mode", ["key_pad", "causal"])
@pytest.mark.parametrize("p", [0.1, 0.3])
@pytest.mark.parametrize("path", PATHS)
def test_flash_attention_dropout_against_float64(L, path, p, mode):
    """Dropout in the forward and both backward kernels against float64 with the host keep mask and the 1/(1-p) scale of
    the 16-bit threshold: out, lse (unaffected by dropout), dQ, dK, dV.  Tq = 70, Tk = 131.  Measured maxima and bars:
    BARS."""
    B, H, Tq, Tk = 2, 2, 70, 131
    pb = make_problem(B, H, Tq, Tk, 64, 64, mode, seed=int(p * 10) + len(mode), p_drop=p)
    keep = keep_mask(B, H, Tq, Tk, p)
    errs = compare(run(L, path, pb), reference(pb, keep), pb)
    _check_errs(errs, BARS[path])


# ================================================================================================ reproducibility
@gpu
@pytest.mark.parametrize("path", ["tf32", "bf16x3"])
def test_tensor_core_flash_backward_is_bit_reproducible(L, path):
    """The tensor-core forward and backward use no atomics: two calls return identical out, lse, dQ, dK and dV bits (at
    B = 4, H = 4, Tq = 200, Tk = 300 with key padding and dropout: 80 dK / dV and 64 dQ CTAs).  The fp32 backward still
    accumulates dQ with atomicAdd and is exempt."""
    pb = make_problem(4, 4, 200, 300, 64, 64, "key_pad", seed=3, p_drop=0.1)
    a, b = run(L, path, pb), run(L, path, pb)
    for name, x, y in zip(("out", "lse", "dq", "dk", "dv"), a, b):
        assert torch.equal(x.cpu().view(torch.int32), y.cpu().view(torch.int32)), name


# ================================================================================================ rejections
REJECTIONS = [
    ("tf32", 64, 64, 449, "exceeds 448"), ("bf16x3", 64, 64, 449, "exceeds 448"), ("bf16x3", 32, 32, 65, "dk = dv = 64"),
    ("tf32", 16, 64, 65, "(dk=16, dv=64) unsupported"), ("tf32", 64, 16, 65, "(dk=64, dv=16) unsupported"),
    ("tf32", 128, 64, 65, "(dk=128, dv=64) unsupported"), ("tf32", 64, 128, 65, "(dk=64, dv=128) unsupported"),
]


@gpu
@pytest.mark.parametrize("path,dk,dv,Tk,msg", REJECTIONS)
def test_flash_attention_rejections(L, path, dk, dv, Tk, msg):
    """Shapes outside a tensor-core path's rules return B200ASR_BAD_SHAPE with a message, launch nothing, and leave the
    NaN-filled outputs untouched: Tk = 449 in the forward; bf16x3 with d = 32 and TF32 with a head dim of 16 or 128 in the
    forward and the backward."""
    pb = make_problem(1, 2, 20, Tk, dk, dv, "none", seed=1)
    out, lse = _token_major(1, 20, 2, dv), _nan(1, 2, 20)
    assert call_fwd(L, path, pb, out, lse) == BAD_SHAPE
    assert msg in L.last_error()
    if Tk <= 448:
        dq, dkk, dvv, ws = _nan_like(pb.q), _nan_like(pb.k), _nan_like(pb.v), _nan(1 << 16)
        assert call_bwd(L, path, pb, out.clone(), out, lse, dq, dkk, dvv, ws) == BAD_SHAPE
        assert msg in L.last_error()
        for t in (dq, dkk, dvv, ws):
            assert torch.isnan(t).all()
    torch.cuda.synchronize()
    assert torch.isnan(out).all() and torch.isnan(lse).all()


# ================================================================================================ ops shape rules
MODES = ["fp32", "tf32", "tf32x3", "bf16", "bf16x3"]
HEAD_DIMS = [16, 32, 64, 128]
# measured maxima o 2.8e-4, gradients 7.4e-3 (the TF32 forward with the fp32 backward; whole tensors, with an utterance of
# one live key -- see compare())
SHAPE_RULE_BARS = dict(o=1e-3, grad=2.5e-2)


@gpu
@pytest.mark.parametrize("attn_bwd", ["fp32", "tf32"])
@pytest.mark.parametrize("attn", MODES)
@pytest.mark.parametrize("dv", HEAD_DIMS)
@pytest.mark.parametrize("dk", HEAD_DIMS)
def test_sdpa_shape_rules_never_fail_in_backward(L, dk, dv, attn, attn_bwd):
    """ops.SdpaFn with every (dk, dv) in {16, 32, 64, 128}^2 under every attention mode: the forward's shape rules pick a
    path whose backward exists, so forward + backward either matches float64 or raises in the forward; it never fails in
    the backward.  Every pair has a kernel, so here it must match, to bars that admit every path and every mix of forward
    and backward precision the rules may pick (each kernel's own accuracy is pinned above).  Key padding with one live key
    in the second utterance.  Measured maxima and bars: SHAPE_RULE_BARS."""
    import importlib
    import b200asr
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    pb = make_problem(2, 2, 45, 70, dk, dv, "key_pad", seed=dk + dv)
    q, k, v = (t.detach().contiguous().requires_grad_(True) for t in (pb.q, pb.k, pb.v))
    old = (ops.config.attn, ops.config.attn_bwd)
    ops.config.set(attn=attn, attn_bwd=attn_bwd)
    try:
        out = ops.SdpaFn.apply(q, k, v, pb.key_pad, None, False, pb.scale, 0.0)
        out.backward(pb.dout)
    finally:
        ops.config.attn, ops.config.attn_bwd = old
    o_ref, _, dq_ref, dk_ref, dv_ref = reference(pb)
    _check_errs(dict(o=rel_err(out, o_ref), grad=max(rel_err(q.grad, dq_ref), rel_err(k.grad, dk_ref), rel_err(v.grad, dv_ref))),
                SHAPE_RULE_BARS)


# ================================================================================================ CPU pin
def test_keep_mask_restatement_spot_values():
    """keep_mask's 64-bit arithmetic: splitmix64 of 0 is the published first output of the generator seeded with 0
    (0xE220A8397B1DCDAF), and every threshold keeps the expected share."""
    assert int(_splitmix64(np.array([0], dtype=np.uint64))[0]) == 0xE220A8397B1DCDAF
    for p in (0.1, 0.3):
        frac = float(keep_mask(2, 3, 50, 70, p).float().mean())
        assert abs(frac - (1 - p)) < 0.02
