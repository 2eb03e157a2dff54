"""CTC loss kernels (csrc/ctc.cu) at every recursion width, on trained-model logits and at their edges, against float64.

ctc_rec_kernel<K, BACK> keeps K states per thread, K = 1, 2, 4, 8, 16, 32 for target lengths up to 127, 255, 511, 1023,
2047, 4095; one call runs the K of its longest target.  Every call here goes through the raw C ABI on `Arena` buffers
(tests/test_gpu_write_extent.py): exactly b200asr_ctc_ws_bytes of workspace, NaN-filled outputs, guard bands that must stay
untouched, inputs that must come back bit for bit.  The references are tests/ctc_util.py's `ctc_float64_fb` (float64
forward-backward) and `ctc_unique_path` (closed form when one alignment exists).

  * Widths: max target length 1 .. 4095 on both sides of every width boundary, each batch with an utterance at the maximum,
    one at the previous width's limit, L = 1, an empty target, T_b = 0 and T_b < T; targets with adjacent repeats and the
    label 0, padded to S > Lmax with out-of-range ids; V in {5, 32} (4364 up to 256 labels); logits also shifted by +200.
  * Trained-model logits: N(0, sigma^2) with sigma in {2, 10, 30}, and "aligned" logits (+M on a forced alignment, M in {10,
    30, 80}, a few frames tied between two symbols) at T in {100, 1000, 8200} and K in {1, 4, 32}.
  * The feasibility boundary: T_b = L_b + r_b frames (r_b adjacent repeats) has one alignment (`ctc_unique_path`),
    T_b = L_b + r_b - 1 has none (+inf, NaN rows t < T_b, zero rows after).  A skip allowed between equal labels would
    make the second finite.
  * Degenerate batches: all targets empty at T in {1, 17}; V = 1; an empty target beside 4095 labels.
  * Independence: one call at B = 257 against B = 1 calls on each row -- nll and, with dloss = B, dz identical bit for
    bit -- and two calls at K = 32 identical bit for bit.
  * ops.CtcLossFn / metrics.calculate_loss with (c * loss).backward(), c != 1, at K = 8; a target above 4095 labels is
    rejected before any launch.

tools/ctc_kernel_names.py lists, with torch.profiler, the ctc_rec_kernel instantiations these widths launch (all 12); it
runs outside the suite because a profiler session here would share the process with the suite's own kernel counts.
  * Broken lengths on the device (input length T + 1 or -1, target length Lmax + 1): that utterance's nll and every row of
    its gradient are NaN, the others keep their float64 values, and nothing is written outside the outputs.

Errors: nll and the mean loss relative to max(1, |nll64|); the gradient per row in units of g_b = dloss / (B max(L_b, 1)),
the largest |dz| a row can have -- dz = g_b (softmax - occupation) is a difference of two numbers near 1 on peaky logits,
so its error is measured against g_b, not against max |dz64| (which, over a batch holding a short target, hides the error
of the long ones by the ratio of their lengths).  Bars (per regime, below) are 3x the largest error measured on an H100 80GB
HBM3 at a 700 W power limit.
"""
import importlib

import numpy as np
import pytest
import torch

import b200asr
from b200asr import _lib as L
from tests.ctc_util import ctc_float64_fb, ctc_unique_path, repeats
from tests.test_gpu_write_extent import Arena

pytestmark = pytest.mark.gpu
metrics = importlib.import_module(b200asr.__name__ + ".metrics")

# Bars: (nll and loss, gradient in units of g_b), 3x the largest error of each regime measured on an H100 80GB HBM3 at a 700 W
# power limit (in brackets, with its case).  The gradient of diffuse logits loses accuracy with T: the alpha / beta of the
# states that carry the occupation can sit hundreds below the step's maximum, where one fp32 ulp is 1e-5 or more, so gamma
# carries ~1e-3 relative error at T = 8200; trained-model (peaky) logits keep it at 3e-7.
BARS = {
    "widths": (1.2e-5, 4.5e-3),      # [3.6e-6 Lmax=4095 V=5; 1.4e-3 Lmax=4095 V=32 T=4612]
    "sigma": (1.5e-6, 6e-3),         # [4.1e-7 T=8200 K=4 sigma=2; 1.8e-3 T=8200 K=4 sigma=30]
    "aligned": (2e-5, 1e-6),         # [6.4e-6 T=1000 M=10, nll64 = 0.37; 3.4e-7 T=8200 K=32 M=10]
    "boundary": (1.2e-6, 6e-7),      # [3.8e-7 Lmax=1000; 2.0e-7 Lmax=3000]
    "edge": (3e-6, 1.4e-3),          # [9.4e-7; 4.6e-4 L=0 beside L=4095, T=4400]
}
LIMITS = [127, 255, 511, 1023, 2047, 4095]          # the longest target of K = 1, 2, 4, 8, 16, 32


def _k(lmax):
    k = 1
    while k * 256 < 2 * lmax + 1:
        k *= 2
    return k


@pytest.fixture(scope="module")
def lib():
    return L.load(check_device=True)


def _target(rng, n, V, zero=True):
    """n labels in [1, V): neighbours differ except a planted repeat every 16 positions; one label 0 if `zero`."""
    y = []
    for i in range(n):
        v = int(rng.integers(1, V))
        if y and v == y[-1]:
            v = v % (V - 1) + 1
        y.append(v)
    for i in range(2, n, 16):
        y[i] = y[i - 1]
    if zero and n >= 3:
        y[n // 3] = 0
    return y


def _pack(ys, V, pad=2):
    S = max([len(y) for y in ys] + [0]) + pad
    gold = torch.full((len(ys), S), V + 7, dtype=torch.int64)           # out of range: reading one past L_b gives NaN
    for b, y in enumerate(ys):
        if y:
            gold[b, :len(y)] = torch.tensor(y, dtype=torch.int64)
    return gold


def _call(lib, x, gold, il, tl, lmax=None, dloss=1.0):
    """ctc_fwd + ctc_bwd on guarded buffers -> (nll, loss, dz) on the CPU; every buffer's guards and inputs checked."""
    B, T, V = x.shape
    S = gold.shape[1]
    il, tl = torch.as_tensor(il, dtype=torch.int32), torch.as_tensor(tl, dtype=torch.int32)
    lmax = int(tl.clamp(min=0).max()) if lmax is None else lmax
    A = Arena(lib)
    xg, gg = A.inp("logits", x.float().cuda()), A.inp("targets", gold.cuda())
    ilg, tlg = A.inp("input_lengths", il.cuda()), A.inp("target_lengths", tl.cuda())
    nll, loss = A.out("nll", (B,)), A.out("loss", (1,))
    ws = A.ws("ws", lib.b200asr_ctc_ws_bytes(B, T, lmax))
    A.call("ctc_fwd", xg, gg, ilg, tlg, nll, loss, ws, B, T, V, S, lmax)
    nll.freeze()
    ws.role = "inout"                       # written by the forward, read by the backward
    dl = A.inp("dloss", torch.tensor([dloss], device="cuda"))
    dz = A.out("dlogits", (B, T, V))
    A.call("ctc_bwd", xg, gg, ilg, tlg, nll, dl, dz, ws, B, T, V, S, lmax)
    out = nll.t.cpu(), loss.t.cpu()[0], dz.t.cpu()
    del A, xg, gg, ilg, tlg, nll, loss, ws, dl, dz
    torch.cuda.empty_cache()                # the workspace reaches gigabytes at 4095 labels
    return out


def _errors(got, ref, il, tl, dloss, rows=None):
    """(nll error, loss error, gradient error in units of g_b) after the exact checks: +inf where the reference is +inf,
    NaN exactly on the rows t < T_b of infeasible utterances, 0 on the rows t >= T_b.  rows: the utterances to compare
    (ref holds those only); a None in got or ref leaves that quantity out."""
    nll, loss, dz = got
    nll64, loss64, dz64 = ref
    B = dz.shape[0]
    rows = range(B) if rows is None else rows
    e_nll = e_grad = e_loss = 0.0
    for j, b in enumerate(rows):
        Tb, Lb = int(il[b]), int(tl[b])
        n64 = float(nll64[j])
        if np.isinf(n64):
            assert nll is None or float(nll[b]) == n64, (b, float(nll[b]))
            assert torch.isnan(dz[b, :Tb]).all() and (dz[b, Tb:] == 0).all(), b
            continue
        if nll is not None:
            e_nll = max(e_nll, abs(float(nll[b]) - n64) / max(1.0, abs(n64)))
        assert (dz[b, Tb:] == 0).all(), b
        g = dloss / (B * max(Lb, 1))
        d = (dz[b, :Tb].double() - dz64[j, :Tb]).abs()
        assert not torch.isnan(d).any(), b
        e_grad = max(e_grad, float(d.max()) / abs(g) if Tb else 0.0)
    if loss64 is not None and np.isfinite(float(loss64)):
        e_loss = abs(float(loss) - float(loss64)) / max(1.0, abs(float(loss64)))
    elif loss64 is not None:
        assert float(loss) == float(loss64), (float(loss), float(loss64))
    return e_nll, e_loss, e_grad


def _check(what, regime, got, ref, il, tl, dloss=1.0, rows=None):
    e_nll, e_loss, e_grad = _errors(got, ref, il, tl, dloss, rows)
    nb, gb = BARS[regime]
    print(f"{regime:8s} {what}: nll {e_nll:.2e} loss {e_loss:.2e} grad/g {e_grad:.2e}")
    assert e_nll <= nb and e_loss <= nb and e_grad <= gb, (what, e_nll, e_loss, e_grad)


# ================================================================================================ every width
def _width_batch(lmax, V, seed):
    rng = np.random.default_rng(seed)
    prev = max([l for l in LIMITS if l < lmax], default=lmax // 2)
    y0 = _target(rng, lmax, V)
    T = lmax + repeats(y0) + max(2, lmax // 16)
    mid = _target(rng, lmax // 3, V)
    if _k(lmax) >= 16:                      # 4 utterances: the workspace is 12 B T (2 Lmax + 1) bytes
        ys = [y0, _target(rng, prev, V), [1], []]
        il = [T, T - 1, T - T // 3, 0]
    else:
        ys = [y0, _target(rng, prev, V), [1], [], [], mid]
        il = [T, T - 1, T, T // 2 + 1, 0, max(len(mid) + repeats(mid), (2 * T) // 3)]
    tl = [len(y) for y in ys]
    assert all(t >= l + repeats(y) for t, l, y in zip(il, tl, ys) if l)
    x = torch.randn(len(ys), T, V, generator=torch.Generator().manual_seed(seed)) * 2.0
    return x, _pack(ys, V), il, tl


WIDTH_CASES = [(lm, V) for lm in [1, 127, 128, 255, 256, 511, 512, 1023, 1024, 2047, 2048, 4095] for V in (5, 32)] + \
              [(lm, 4364) for lm in [1, 127, 128, 255, 256]]


@pytest.mark.parametrize("lmax,V", WIDTH_CASES)
def test_every_width_matches_float64(lib, lmax, V):
    x, gold, il, tl = _width_batch(lmax, V, seed=lmax * 13 + V)
    assert max(tl) == lmax
    for shift in (0.0, 200.0):
        xs = (x + shift).float()
        got = _call(lib, xs, gold, il, tl)
        # the float64 reference sees the same fp32 logits (xs - 200 is exact; log_softmax drops the shift)
        ref = ctc_float64_fb(xs.double() - shift, gold, il, tl)
        _check(f"Lmax={lmax} K={_k(lmax)} V={V} T={x.shape[1]} shift={shift:g}", "widths", got, ref, il, tl)


# ================================================================================================ trained-model logits
def _alignment(rng, y, Tb):
    """A random path of Tb frames that emits y: the shortest path (blanks only between equal labels) with the spare
    frames spread over label repetitions and blank runs."""
    tokens = []
    for i, v in enumerate(y):
        if i and v == y[i - 1]:
            tokens.append(0)
        tokens.append(v)
    extra = Tb - len(tokens)
    assert extra >= 0
    bins = rng.multinomial(extra, np.full(2 * len(tokens) + 1, 1.0 / (2 * len(tokens) + 1)))
    path = [0] * int(bins[0])
    for j, v in enumerate(tokens):
        path += [v] * (1 + int(bins[2 * j + 1])) + [0] * int(bins[2 * j + 2])
    assert len(path) == Tb
    return path


TRAINED_SIZES = [(100, 1), (1000, 1), (1000, 4), (8200, 1), (8200, 4), (8200, 32)]
TRAINED_L = {(100, 1): 40, (1000, 1): 127, (1000, 4): 450, (8200, 1): 127, (8200, 4): 511, (8200, 32): 3000}


@pytest.mark.parametrize("kind,scale", [("sigma", 2.0), ("sigma", 10.0), ("sigma", 30.0), ("aligned", 10.0),
                                        ("aligned", 30.0), ("aligned", 80.0)])
@pytest.mark.parametrize("T,K", TRAINED_SIZES)
def test_trained_model_logits_match_float64(lib, T, K, kind, scale):
    V = 32
    seed = T + 7 * K + int(scale)
    rng = np.random.default_rng(seed)
    lm = TRAINED_L[(T, K)]
    ys = [_target(rng, lm, V), _target(rng, lm // 2, V)] + ([] if K == 32 else [[int(rng.integers(1, V))]])
    il = [T, T - T // 5] + ([] if K == 32 else [T // 2])
    tl = [len(y) for y in ys]
    assert _k(max(tl)) == K
    g = torch.Generator().manual_seed(seed)
    if kind == "sigma":
        x = torch.randn(len(ys), T, V, generator=g) * scale
    else:
        x = torch.randn(len(ys), T, V, generator=g)
        for b, (y, Tb) in enumerate(zip(ys, il)):
            path = _alignment(rng, y, Tb)
            x[b, torch.arange(Tb), torch.tensor(path)] += scale
            tied = rng.choice(Tb - 1, size=max(1, Tb // 30), replace=False)   # the boundary can move by a frame
            x[b, torch.as_tensor(tied), torch.tensor([path[t + 1] for t in tied])] = x[b, torch.as_tensor(tied),
                                                                                         torch.tensor([path[t] for t in tied])]
    x = x.float()
    got = _call(lib, x, _pack(ys, V), il, tl)
    ref = ctc_float64_fb(x.double(), _pack(ys, V), il, tl)
    if kind == "sigma" and T == 8200:
        assert float(ref[0][0]) > 5000.0                 # unscaled log alphas run to many thousands here
    _check(f"T={T} K={K} {kind}={scale:g} nll64={float(ref[0][0]):.4g}", kind, got, ref, il, tl)


# ================================================================================================ feasibility boundary
def _no_zero_target(rng, n, V):
    y = _target(rng, n, V, zero=False)
    for i in range(1, n, 5):
        y[i] = y[i - 1]
    return y


@pytest.mark.parametrize("lmax", [100, 1000, 3000])
def test_feasibility_boundary(lib, lmax):
    """T_b = L_b + r_b: the one alignment, against the closed form; T_b = L_b + r_b - 1: no alignment at all."""
    V = 32
    rng = np.random.default_rng(lmax)
    y0, y2 = _no_zero_target(rng, lmax, V), _no_zero_target(rng, lmax // 3 + 1, V)
    n0, n2 = lmax + repeats(y0), len(y2) + repeats(y2)
    ys, il = [y0, y0, y2], [n0, n0 - 1, n2]
    tl = [len(y) for y in ys]
    gold = _pack(ys, V)
    x = torch.randn(3, n0, V, generator=torch.Generator().manual_seed(lmax)) * 2.0
    got = _call(lib, x, gold, il, tl)
    sub = [0, 2]
    # the closed form of utterances 0 and 2 as a batch of 2: dloss 2/3 gives them the g_b of the batch of 3
    ref = ctc_unique_path(x[sub].double(), gold[sub], [il[b] for b in sub], [tl[b] for b in sub], dloss=2.0 / 3.0)
    assert float(got[0][1]) == float("inf") and float(got[1]) == float("inf")
    assert torch.isnan(got[2][1, :il[1]]).all() and (got[2][1, il[1]:] == 0).all()
    ref_all = (ref[0], torch.tensor(float("inf"), dtype=torch.float64), ref[2])
    _check(f"Lmax={lmax} K={_k(lmax)} T_b = L + r = {n0}", "boundary", got, ref_all, il, tl, rows=sub)
    _check(f"Lmax={lmax} K={_k(lmax)} forward-backward", "boundary", got, ctc_float64_fb(x.double(), gold, il, tl), il, tl)


# ================================================================================================ degenerate batches
@pytest.mark.parametrize("T", [1, 17])
def test_all_targets_empty(lib, T):
    il, tl = [T, T // 2, 0], [0, 0, 0]
    gold = torch.full((3, 2), 9, dtype=torch.int64)
    x = torch.randn(3, T, 5, generator=torch.Generator().manual_seed(T)) * 2.0
    got = _call(lib, x, gold, il, tl)
    _check(f"all empty T={T}", "edge", got, ctc_float64_fb(x.double(), gold, il, tl), il, tl)


def test_the_blank_is_the_whole_vocabulary(lib):
    """V = 1: empty targets only, then targets of the label 0 (every lp' is 0, nll = -log #alignments, dz = 0)."""
    x = torch.randn(3, 9, 1, generator=torch.Generator().manual_seed(1))
    gold = torch.full((3, 2), 4, dtype=torch.int64)
    got = _call(lib, x, gold, [9, 5, 0], [0, 0, 0])
    _check("V=1 empty", "edge", got, ctc_float64_fb(x.double(), gold, [9, 5, 0], [0, 0, 0]), [9, 5, 0], [0, 0, 0])
    assert (got[0] == 0).all() and (got[2] == 0).all()
    gold = torch.tensor([[0, 0, 4], [0, 4, 4], [4, 4, 4]])
    il, tl = [9, 5, 7], [2, 1, 0]
    got = _call(lib, x, gold, il, tl)
    _check("V=1 label 0", "edge", got, ctc_float64_fb(x.double(), gold, il, tl), il, tl)


def test_empty_target_beside_4095_labels_and_repeatable_at_k32(lib):
    rng = np.random.default_rng(4095)
    y = _target(rng, 4095, 32)
    T = 4095 + repeats(y) + 40
    ys, il = [y, []], [T, T]
    gold = _pack(ys, 32)
    x = torch.randn(2, T, 32, generator=torch.Generator().manual_seed(5)) * 2.0
    a = _call(lib, x, gold, il, [4095, 0])
    _check(f"L=0 beside L=4095 T={T}", "edge", a, ctc_float64_fb(x.double(), gold, il, [4095, 0]), il, [4095, 0])
    b = _call(lib, x, gold, il, [4095, 0])
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.int32), v.view(torch.int32))


# ================================================================================================ independence
def test_utterances_are_independent(lib):
    """B = 257 rows of lengths from the ranges of K = 1, 2 and 4 in one call (K = 4) against one B = 1 call per row (each
    at the K of its own length): nll bit for bit, and with dloss = B (so g_b is the same float) dz bit for bit."""
    B, T, V = 257, 340, 32
    rng = np.random.default_rng(257)
    lens = [0, 1, 127, 128, 255, 256, 300] + [int(v) for v in rng.integers(0, 301, B - 7)]
    ys = [_target(rng, n, V) for n in lens]
    il = [int(rng.integers(n + repeats(y), T + 1)) if n else int(rng.integers(0, T + 1)) for n, y in zip(lens, ys)]
    il[0], il[1] = 0, T
    tl = [len(y) for y in ys]
    gold = _pack(ys, V)
    x = torch.randn(B, T, V, generator=torch.Generator().manual_seed(257)) * 2.0
    nll, loss, dz = _call(lib, x, gold, il, tl, dloss=float(B))
    ref = ctc_float64_fb(x.double(), gold, il, tl, dloss=float(B))
    _check("B=257 against float64", "widths", (nll, loss, dz), ref, il, tl, dloss=float(B))
    for b in range(B):
        n1, _, d1 = _call(lib, x[b:b + 1], gold[b:b + 1], il[b:b + 1], tl[b:b + 1])
        assert torch.equal(n1.view(torch.int32), nll[b:b + 1].view(torch.int32)), (b, float(n1), float(nll[b]))
        assert torch.equal(d1.view(torch.int32), dz[b:b + 1].view(torch.int32)), b


# ================================================================================================ through ops
def test_ops_scales_by_dloss_at_k8():
    B, T, V, c = 3, 800, 32, -0.37
    rng = np.random.default_rng(8)
    ys = [_target(rng, 700, V), _target(rng, 300, V), []]
    il, tl = [T, 650, 400], [700, 300, 0]
    gold = _pack(ys, V)
    x = (torch.randn(B, T, V, generator=torch.Generator().manual_seed(8)) * 2.0).cuda().requires_grad_(True)
    loss = metrics.calculate_loss(x, gold.cuda(), torch.tensor(il), torch.tensor(tl), loss_type="ctc")
    (c * loss).backward()
    ref = ctc_float64_fb(x.detach().cpu().double(), gold, il, tl, dloss=c)
    _check(f"ops K=8 c={c}", "edge", (None, loss.detach().cpu(), x.grad.cpu()), ref, il, tl, dloss=c)


def test_ops_rejects_targets_above_4095_before_any_launch():
    lib = L.load()
    x = torch.randn(1, 10, 5, device="cuda")
    gold = torch.ones(1, 4100, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    n0 = lib.b200asr_launch_count()
    with pytest.raises(RuntimeError, match="4095"):
        metrics.calculate_loss(x, gold, torch.tensor([10]), torch.tensor([4096]), loss_type="ctc")
    assert lib.b200asr_launch_count() == n0


# ================================================================================================ device-side lengths
@pytest.mark.parametrize("lmax", [60, 700])
def test_broken_device_lengths_give_nan_only_there(lib, lmax):
    """ctc_lengths_ok fails on utterances 1 (T + 1 frames, Lmax + 1 labels), 3 (-1 frames) and 4 (Lmax + 1 labels): the
    three kernels return before forming any address from those lengths; nll and every dz row of those utterances are NaN,
    the mean loss NaN, utterances 0 and 2 keep their float64 values, and the guards stay intact."""
    V = 32
    rng = np.random.default_rng(lmax)
    y0, y2 = _target(rng, lmax, V), _target(rng, lmax // 2, V)
    T = lmax + repeats(y0) + 10
    ys = [y0, y0[:3], y2, [5], [7, 8]]
    il, tl = [T, T + 1, T - 5, -1, T], [lmax, lmax + 1, len(y2), 1, lmax + 1]
    gold = _pack(ys, V, pad=lmax + 2)
    x = torch.randn(5, T, V, generator=torch.Generator().manual_seed(lmax)) * 2.0
    got = _call(lib, x, gold, il, tl, lmax=lmax)
    nll, loss, dz = got
    for b in (1, 3, 4):
        assert torch.isnan(nll[b]) and torch.isnan(dz[b]).all(), b
    assert torch.isnan(loss)
    sub = [0, 2]
    # utterances 0 and 2 as a batch of 2: dloss 2/5 gives them the g_b of the batch of 5
    ref = ctc_float64_fb(x[sub].double(), gold[sub], [il[b] for b in sub], [tl[b] for b in sub], dloss=2.0 / 5.0)
    _check(f"broken lengths K={_k(lmax)}", "edge", got, (ref[0], None, ref[2]), il, tl, rows=sub)
