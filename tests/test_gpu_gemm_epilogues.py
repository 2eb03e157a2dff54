"""The two epilogues of the linear layers' tile-engine GEMM (tc_gemm.cu: GemmPolicy), through the raw C ABI:

  * the coalesced one (tc_engine.cuh: epilogue_vec4 -> GemmPolicy::load4 / store4): 64-column chunks, 16 lanes per row,
    16 rows per pass, two rows' loads in flight; a launch takes it when N % 4 == 0 and either the contraction is split or
    C, bias and relu_mask are 16-byte aligned with ldc % 4 == 0 (GemmPolicy::vec4_ok);
  * the 32-column row pieces (epilogue_rows -> GemmPolicy::store): every other launch, and every launch of the B_T32
    instantiations (TF32 / 3xTF32 with an MN-major B).

Which one runs depends only on where the caller's buffers sit, so both must compute the same bits: + bias, ReLU, mask
`> 0`, + old C, in that order.

  A. The instantiation map: every tc_engine_kernel<GemmPolicy<A_MN, B_MN, PRESPLIT>, NSPLIT> that tc_gemm.cu compiles, the
     calls that launch it (read with torch.profiler) and whether it can take the coalesced epilogue.  Two are compiled but
     reached by no call: gemm_tc's callers are b200asr_linear_fwd (A and B K-major), _bwd_data (A K-major, B MN-major),
     _bwd_weight (both MN-major) and b200asr_stft_features (both K-major), so nothing pairs an MN-major A with a K-major B.
  B. Both epilogues, same bits: every reachable instantiation at precisions 1, 3 (split in the kernel and pre-split), 6
     and 2, each call made once with every epilogue operand on the 16-byte grid and once with exactly one of them (the
     output, the bias or relu_out) one float off it; every epilogue variant; shapes at the edges of the coalesced
     epilogue's geometry and tile counts that make CTAs run several tiles back to back.
  C. Column independence: the forward with N % 4 != 0 (row pieces; never run before in the bf16 modes) equals columns
     [:N] of the same call at N rounded up to a multiple of 4 (coalesced), bit for bit, also where the contraction is split
     and the partial tiles go through `store` in one call and `store4` in the other.

Outputs are NaN-filled between sentinel bands that must come back unchanged.  The float64 references run on the GPU.  Bars
are those of tests/test_gpu_linear_precisions.py (precisions 1 and 3, SPLIT_BARS) and tests/test_gpu_default_precision.py
(LIN_BARS, the split-K weight gradient); where two apply, the tighter one.  Measured values are on one H100 80GB HBM3 at a
700 W power limit."""
import json
import os
import re
import subprocess
import sys

import pytest
import torch

from tests.helpers import rel_err
from tests.test_gpu_default_precision import LIN_BARS
from tests.test_gpu_linear_precisions import SPLIT_BARS, Banded, _bf16_split, _gen, _launches, _placed, _sms, _stream, _tc_split

pytestmark = pytest.mark.gpu

TF32, TF32X3, BF16, BF16X3 = 1, 3, 2, 6

# (A_MN, B_MN, PRESPLIT, NSPLIT) of tc_engine_kernel<GemmPolicy<A_MN, B_MN, PRESPLIT>, NSPLIT>:
#   (takes the coalesced epilogue when the launch allows it, [calls that launch it])
# A call is (entry point, precision, pre-split weight operand): at precision 3 w_split = b200asr_split_tf32(w); the bf16
# modes always take one (b200asr_split_bf16: dst for the forward, dst_t for the data gradient); "stft" is
# b200asr_stft_features.  Only B_T32 (NSPLIT 1 / 3 with an MN-major B) keeps the row pieces everywhere.
GEMM_INSTANTIATIONS = {
    (False, False, False, 1): (True, [("fwd", 1, False), ("stft", 1, False)]),
    (False, False, False, 3): (True, [("fwd", 3, False), ("stft", 3, False)]),
    (False, False, True, 3): (True, [("fwd", 3, True)]),
    (False, False, True, 6): (True, [("fwd", 6, True), ("dgrad", 6, True)]),
    (False, False, True, 2): (True, [("fwd", 2, True), ("dgrad", 2, True)]),
    (False, True, False, 1): (False, [("dgrad", 1, False)]),
    (False, True, False, 3): (False, [("dgrad", 3, False)]),
    (False, True, True, 3): (False, [("dgrad", 3, True)]),
    (True, True, False, 1): (False, [("wgrad", 1, False)]),
    (True, True, False, 3): (False, [("wgrad", 3, False)]),
    (True, True, False, 6): (True, [("wgrad", 6, False)]),
    (True, True, False, 2): (True, [("wgrad", 2, False)]),
    (True, False, False, 1): (True, []),          # compiled, reached by no call
    (True, False, False, 3): (True, []),          # compiled, reached by no call
}
CALLS = {c: inst for inst, (_, calls) in GEMM_INSTANTIATIONS.items() for c in calls}
LINEAR_CALLS = [c for c in CALLS if c[0] != "stft"]


def _call_id(c):
    return f"{c[0]}-p{c[1]}" + ("-presplit" if c[2] and c[1] == TF32X3 else "")


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _operands(L, w, prec, presplit):
    """(forward w_split, data-gradient w_split) of a call: NULL, the 3xTF32 hi | lo pair, or the bf16 dst / dst_t."""
    if prec in (BF16, BF16X3):
        return _bf16_split(L, w, prec)
    if presplit:
        ws = torch.empty(2, *w.shape, device="cuda")
        L.check(L.load().b200asr_split_tf32(L.ptr(w), L.ptr(ws), w.numel(), _stream()), "split_tf32")
        return ws, ws
    return None, None


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ================================================================================================ A. instantiation map
_GEMM_KERNEL = re.compile(r"tc_engine_kernel<b200asr::tc::GemmPolicy<([^<>]*)>, (?:\(int\))?(\d+)>")


def _flag(s):
    s = s.strip().replace("(bool)", "")
    return {"true": True, "1": True, "false": False, "0": False}[s]


def _gemm_kernels_launched(fn):
    """The GemmPolicy instantiations torch.profiler sees the device run for fn(), and every kernel name it saw.  Tracing is
    switched on for one warm-up step whose events are discarded, then fn() runs again in the recorded step; both steps run
    the same call, so an event that strays across the step boundary names the same kernels.  fn() launches at least one
    kernel, so a recorded step without any CUDA event means the tracer recorded nothing (seen now and then on an H100, for
    a whole session): that session is taken again, at most twice more."""
    for _ in range(3):
        seen = []

        def ready(prof):
            seen.append({e.name() for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA})

        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA], on_trace_ready=ready,
                                    schedule=torch.profiler.schedule(wait=0, warmup=1, active=1, repeat=1)) as prof:
            for _ in range(2):
                fn()
                torch.cuda.synchronize()
                prof.step()
        assert len(seen) == 1, len(seen)
        if seen[0]:
            break
    out = set()
    for n in seen[0]:
        m = _GEMM_KERNEL.search(n)
        if m:
            out.add(tuple(_flag(f) for f in m.group(1).split(",")) + (int(m.group(2)),))
    return out, sorted(seen[0])


def _one_call(L, call):
    """A small unsplit call of `call`, as a closure."""
    entry, prec, presplit = call
    lib, st = L.load(), _stream()
    g = _gen(11)
    M, N, K = 40, 72, 64
    x, w, b = torch.randn(M, K, generator=g).cuda(), torch.randn(N, K, generator=g).cuda(), torch.randn(N, generator=g).cuda()
    dy, h = torch.randn(M, N, generator=g).cuda(), torch.randn(M, K, generator=g).cuda()
    fsplit, bsplit = _operands(L, w, prec, presplit)
    y, dx, dw, db = torch.empty(M, N, device="cuda"), torch.empty(M, K, device="cuda"), torch.empty(N, K, device="cuda"), torch.empty(N, device="cuda")
    if entry == "fwd":
        return lambda: L.check(lib.b200asr_linear_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), M, N, K, 1, prec, L.ptr(fsplit), st))
    if entry == "dgrad":
        return lambda: L.check(lib.b200asr_linear_bwd_data(L.ptr(dy), L.ptr(w), L.ptr(h), L.ptr(dx), M, N, K, 0, prec, L.ptr(bsplit), st))
    if entry == "wgrad":
        return lambda: L.check(lib.b200asr_linear_bwd_weight(L.ptr(dy), L.ptr(x), L.ptr(dw), L.ptr(db), M, N, K, 0, prec, st))
    B, Lmax, n_fft, hop = 2, 1600, 320, 160
    wave = torch.randn(B, Lmax, generator=g).cuda()
    lens = torch.tensor([Lmax, 1000], dtype=torch.int32, device="cuda")
    Tmax = 1 + Lmax // hop
    ws = torch.empty(lib.b200asr_stft_ws_bytes(B, Lmax, n_fft, hop) // 4, device="cuda")
    out = torch.empty(B, 1, n_fft // 2 + 1, Tmax, device="cuda")
    return lambda: L.check(lib.b200asr_stft_features(L.ptr(wave), L.ptr(lens), L.ptr(out), None, L.ptr(ws), B, Lmax, Tmax, n_fft, hop,
                                                     1, 0, 0, prec, st))


def _launch_map():
    """Run in a process of its own by the test below: prints, as JSON, the instantiations and the kernel names that each
    call of the table launches."""
    import b200asr
    b200asr._lib.load(check_device=True)
    out = {}
    for call in CALLS:
        got, names = _gemm_kernels_launched(_one_call(b200asr._lib, call))
        out[_call_id(call)] = {"got": sorted(got), "names": names}
    print(json.dumps(out))


def test_every_gemm_instantiation_has_its_callers():
    """Each call of the table launches exactly its GemmPolicy instantiation, so together they launch every instantiation
    the table marks reachable and none it marks unreachable.  The coalesced-epilogue column follows the engine's rule:
    every B mode but B_T32.  The profiler sessions run in a child process: CUPTI, once started, stays in the process and
    can drop the first kernels of a later session there (tests/test_gpu_optimizer_step.py counts kernels by profiler)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    r = subprocess.run(py + ["-c", "from tests.test_gpu_gemm_epilogues import _launch_map; _launch_map()"], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    launched = json.loads(r.stdout.strip().splitlines()[-1])
    seen = set()
    for call, inst in CALLS.items():
        got = {tuple(i) for i in launched[_call_id(call)]["got"]}
        assert got == {inst}, (call, launched[_call_id(call)]["names"])
        seen |= got
    reachable = {inst for inst, (_, calls) in GEMM_INSTANTIATIONS.items() if calls}
    assert seen == reachable
    assert set(GEMM_INSTANTIATIONS) - reachable == {(True, False, False, 1), (True, False, False, 3)}
    for (a_mn, b_mn, presplit, nsplit), (vec4, _) in GEMM_INSTANTIATIONS.items():
        assert vec4 == (not (b_mn and nsplit in (TF32, TF32X3))), (a_mn, b_mn, presplit, nsplit)


# ================================================================================================ B. both epilogues
# bars: precisions 1 / 3 from test_gpu_linear_precisions.py (forward 2e-3 / 2e-5, backward 2e-3 / 1e-4, SPLIT_BARS for the
# split forward and data gradient); precisions 6 / 2: LIN_BARS; the split weight gradient: the tighter of those and
# test_linear_weight_gradient_split_k's (1e-3, 1e-4, 5e-5, 1e-2)
BARS = {TF32: dict(fwd=2e-3, dgrad=2e-3, wgrad=2e-3), TF32X3: dict(fwd=2e-5, dgrad=1e-4, wgrad=1e-4),
        BF16X3: LIN_BARS[BF16X3], BF16: LIN_BARS[BF16]}
SPLIT_WGRAD_BARS = {TF32: 1e-3, TF32X3: 1e-4, BF16X3: 5e-5, BF16: 1e-2}
DB_BAR = 1e-6


def _bar(prec, entry, split):
    bar = BARS[prec][entry]
    if split and entry == "wgrad":
        return min(bar, SPLIT_WGRAD_BARS[prec])
    if split:
        return min(bar, SPLIT_BARS[prec][0 if entry == "fwd" else 1])
    return bar


# (R, C, D, data): the GEMM's output rows and columns and its contraction -- forward y[M, N] with (M, N, K) = (R, C, D),
# data gradient dx[M, K] with (M, K, N) = (R, C, D), weight gradient dw[N, K] with (N, K, M) = (R rounded up to a multiple of
# 4, C, D); data "int": integers in [-2, 2] (many pre-ReLU sums exactly 0; every sum exact, so the result must equal float64)
EPI_SHAPES = [
    (1, 4, 32, "int"),            # one row, one 4-column group
    (15, 60, 40, "normal"),       # less than one 16-row pass; 15 of a chunk's 16 lanes; a partial k-block
    (16, 64, 32, "int"),          # exactly one pass and one 64-column chunk
    (17, 68, 64, "normal"),       # one row into the second pass (its batched partner row out of range); a 1-group chunk
    (127, 124, 96, "normal"),     # a row short of the tile, a group short of two chunks
    (128, 128, 32, "int"),        # one whole tile
    (129, 132, 32, "normal"),     # a second row tile of one row, a second column tile of one group
    (300, 192, 48, "int"),        # three row tiles (44 rows in the last); a second column tile of one chunk
    (300, 196, 32, "normal"),     # a second column tile of one chunk and one group
    (129, 260, 24, "normal"),     # three column tiles, the last one group; contraction shorter than one k-block
    (130, 4364, 32, "normal"),    # the vocabulary projection: 34 column tiles and 12 columns
    (127, 16708, 32, "normal"),   # 131 tiles (1 x 131)
    (500, 4200, 32, "int"),       # 132 tiles (4 x 33)
    (896, 2420, 32, "normal"),    # 133 tiles (7 x 19): on 132 SMs one CTA runs two tiles back to back
    (600, 6660, 16, "normal"),    # 265 tiles (5 x 53): CTAs run 2 or 3 tiles, reusing the staging buffer
    (300, 196, 2048, "normal"),   # split contraction (8 splits of 6 tiles at precisions 1 and 3 without ReLU / mask,
    (264, 132, 1024, "int"),      #   and in every weight gradient); 4 splits
]

_SPECIALS = [0.0, -0.0, float("nan"), float("inf"), float("-inf"), 2.0 ** -140, 2.0 ** -149, 2.0 ** -126, -(2.0 ** -149),
             1e-30]


def _data(shape, kind, g, scale=1.0):
    if kind == "int":
        return torch.randint(-2, 3, shape, generator=g).float()
    return torch.randn(shape, generator=g) * scale


def _relu_out(shape, kind, g):
    """relu_out with exact zeros of both signs, NaN, both infinities, denormals (the smallest), the smallest normal and tiny
    positives spread over rows and columns, the rest random."""
    h = _data(shape, kind, g)
    flat = h.view(-1)
    idx = torch.arange(flat.numel())
    pick = (idx * 7 + idx // max(shape[-1], 1)) % 16
    for i, v in enumerate(_SPECIALS):
        flat[pick == i] = v
    return h


def _expect(got, ref, kind, bar, what):
    """got against the float64 ref: exactly for integer data, else within bar.  Returns the error."""
    if kind == "int":
        assert torch.equal(got.double(), ref), what
        return 0.0
    err = rel_err(got, ref)
    assert err < bar, (what, err)
    return err


def _run_moves(make, moves, what):
    """make(moved) -> (Banded outputs...) for moved = None (every epilogue operand on the 16-byte grid) and each name in
    moves (that operand one float off it): identical bits and intact sentinel bands.  Returns the aligned call's outputs."""
    first = make(None)
    for moved in moves:
        other = make(moved)
        for a, b in zip(first, other):
            assert _same_bits(a.t, b.t), (what, moved)
            assert b.bands_intact(), (what, moved)
    for a in first:
        assert a.bands_intact(), what
    return first


def _fwd_case(L, prec, presplit, M, N, K, kind, g):
    lib, st, sms = L.load(), _stream(), _sms()
    x, w, b = _data((M, K), kind, g), _data((N, K), kind, g, K ** -0.5), _data((N,), kind, g)
    xc, wc = x.cuda(), w.cuda()
    fsplit, _ = _operands(L, wc, prec, presplit)
    xw = xc.double() @ wc.double().t()
    worst = 0.0
    for bias in (None, b):
        for relu in (0, 1):
            split = prec in (TF32, TF32X3) and _tc_split(M, N, K, sms, relu=bool(relu)) > 1

            def make(moved):
                bc = _placed(bias, 1 if moved == "bias" else 0) if bias is not None else None
                y = Banded((M, N), shift=1 if moved == "y" else 0)
                n0 = _launches(L)
                L.check(lib.b200asr_linear_fwd(L.ptr(xc), L.ptr(wc), L.ptr(bc), L.ptr(y.t), M, N, K, relu, prec, L.ptr(fsplit), st),
                        "fwd")
                assert _launches(L) - n0 == (2 if split else 1)
                return (y,)

            what = ("fwd", bias is not None, relu)
            (y,) = _run_moves(make, ["y"] + (["bias"] if bias is not None else []), what)
            ref = xw + b.double().cuda() if bias is not None else xw
            worst = max(worst, _expect(y.t, ref.relu() if relu else ref, kind, _bar(prec, "fwd", split), what))
    return worst


def _dgrad_case(L, prec, presplit, M, N, K, kind, g):
    lib, st, sms = L.load(), _stream(), _sms()
    dy, w = _data((M, N), kind, g), _data((N, K), kind, g, N ** -0.5)
    h, base = _relu_out((M, K), kind, g), _data((M, K), kind, g)
    dyc, wc = dy.cuda(), w.cuda()
    _, bsplit = _operands(L, wc, prec, presplit)
    dyw = dyc.double() @ wc.double()
    keep = (h > 0).cuda()                        # the kernel's test, on the fp32 values
    worst = 0.0
    for mask in (None, h):
        for acc in (0, 1):
            split = prec in (TF32, TF32X3) and _tc_split(M, K, N, sms, mask=mask is not None) > 1

            def make(moved):
                hc = _placed(mask, 1 if moved == "relu_out" else 0) if mask is not None else None
                dx = Banded((M, K), init=base if acc else None, shift=1 if moved == "dx" else 0)
                n0 = _launches(L)
                L.check(lib.b200asr_linear_bwd_data(L.ptr(dyc), L.ptr(wc), L.ptr(hc), L.ptr(dx.t), M, N, K, acc, prec, L.ptr(bsplit),
                                                    st), "dgrad")
                assert _launches(L) - n0 == (2 if split else 1)
                return (dx,)

            what = ("dgrad", mask is not None, acc)
            (dx,) = _run_moves(make, ["dx"] + (["relu_out"] if mask is not None else []), what)
            ref = dyw * keep if mask is not None else dyw
            ref = ref + base.double().cuda() if acc else ref
            worst = max(worst, _expect(dx.t, ref, kind, _bar(prec, "dgrad", split), what))
    return worst


def _wgrad_case(L, prec, M, N, K, kind, g):
    lib, st, sms = L.load(), _stream(), _sms()
    dy, x = _data((M, N), kind, g), _data((M, K), kind, g)
    wbase, bbase = _data((N, K), kind, g), _data((N,), kind, g)
    dyc, xc = dy.cuda(), x.cuda()
    dw_ref, db_ref = dyc.double().t() @ xc.double(), dyc.double().sum(0)
    split = _tc_split(N, K, M, sms) > 1
    worst = db_worst = 0.0
    for with_db in (False, True):
        for acc in (0, 1):
            launches = (2 if split else 1) + (0 if not with_db else 2 if prec == TF32 else 1 if split else 0)

            def make(moved):
                dw = Banded((N, K), init=wbase if acc else None, shift=1 if moved == "dw" else 0)
                db = Banded((N,), init=bbase if acc else None)
                n0 = _launches(L)
                L.check(lib.b200asr_linear_bwd_weight(L.ptr(dyc), L.ptr(xc), L.ptr(dw.t), L.ptr(db.t) if with_db else None, M, N, K,
                                                      acc, prec, st), "wgrad")
                assert _launches(L) - n0 == launches
                return (dw, db) if with_db else (dw,)

            what = ("wgrad", with_db, acc)
            outs = _run_moves(make, ["dw"], what)
            ref = dw_ref + wbase.double().cuda() if acc else dw_ref
            worst = max(worst, _expect(outs[0].t, ref, kind, _bar(prec, "wgrad", split), what))
            if with_db:
                db_worst = max(db_worst, _expect(outs[1].t, db_ref + bbase.double().cuda() if acc else db_ref, kind, DB_BAR, what + ("db",)))
    print(f"[epilogues] dbias p{prec} {N}x{K}x{M}: float64 rel err {db_worst:.2e}")
    return worst


@pytest.mark.parametrize("R,C,D,kind", EPI_SHAPES)
@pytest.mark.parametrize("call", LINEAR_CALLS, ids=_call_id)
def test_both_epilogues_give_the_same_bits(L, call, R, C, D, kind):
    """Each reachable instantiation with every epilogue operand on the 16-byte grid (the coalesced epilogue where the
    instantiation has it) and with one of them one float off (the row pieces), identical bits, the accumulated base
    included; then against float64 at the file's bars.  Forward: bias NULL / given x ReLU 0 / 1; data gradient: relu_out NULL
    / given (zeros of both signs, NaN, infinities, denormals) x accumulate 0 / 1; weight gradient: dbias NULL / given x
    accumulate 0 / 1, split and unsplit.  Integer data must equal float64 exactly.  Measured float64 errors (largest over
    the shapes), forward / data gradient / weight gradient: TF32 4.0e-4 / 4.9e-4 / 3.7e-4, 3xTF32 (both ways of splitting
    give the same bits) 1.3e-5 / 1.9e-5 / 2.0e-6, bf16x3 8.6e-6 / 8.3e-6 / 8.0e-6, bf16 3.2e-3 / 5.1e-3 / 3.5e-3.
    With the accumulation moved before the mask, the mask tested with >= 0, or the bias added after the ReLU in store4,
    this test fails at 16 or all 17 shapes of every call that the change reaches (the bf16 data gradients; the forwards)."""
    entry, prec, presplit = call
    g = _gen(R * 31 + C * 7 + D + prec)
    if entry == "fwd":
        err = _fwd_case(L, prec, presplit, R, C, D, kind, g)
    elif entry == "dgrad":
        err = _dgrad_case(L, prec, presplit, R, D, C, kind, g)
    else:
        err = _wgrad_case(L, prec, D, -(-R // 4) * 4, C, kind, g)
    print(f"[epilogues] {_call_id(call)} {R}x{C}x{D} {kind}: float64 rel err {err:.2e}")


# ================================================================================================ C. column independence
# (M, K, k): N = 4k + r against N' = 4k + 4
COL_SHAPES = [
    (17, 32, 0),          # N = 1, 2, 3 against 4
    (129, 64, 15),        # 61 .. 63 against one full chunk
    (300, 96, 31),        # 125 .. 127 against one full tile
    (300, 96, 32),        # 129 .. 131: a second column tile of 1 .. 3 columns against one group
    (16, 40, 48),         # 193 .. 195
    (130, 32, 1090),      # 4361 .. 4363 against the vocabulary's 4364
    (300, 2048, 32),      # 129 .. 131 with the contraction split (precisions 1 and 3, no ReLU): partial tiles by `store`
]                         #   against `store4`
COL_CALLS = [(BF16X3, True), (BF16, True), (TF32, False), (TF32X3, False), (TF32X3, True)]


@pytest.mark.parametrize("r", [1, 2, 3])
@pytest.mark.parametrize("M,K,k", COL_SHAPES)
def test_forward_columns_are_independent_of_n(L, M, K, k, r):
    """b200asr_linear_fwd at N = 4k + r (row pieces, scalar stores) equals columns [:N] of the call at N' = 4k + 4 (w and the
    bias padded with further rows; coalesced), bit for bit, at precisions 6, 2, 1, 3 and pre-split 3, with bias alone (split
    where the rule splits), bias and ReLU, and ReLU alone; both calls make the same number of launches, as the split rule
    says for either width; the N call is within the forward bars of float64.  Measured float64 errors (largest over the shapes): bf16x3 9.9e-6, bf16 3.4e-3, TF32 4.3e-4, 3xTF32 1.7e-5
    (the split contraction; 9.4e-7 unsplit)."""
    lib, st, sms = L.load(), _stream(), _sms()
    N, Np = 4 * k + r, 4 * k + 4
    g = _gen(M + 13 * N + K)
    wp, bp = torch.randn(Np, K, generator=g) * K ** -0.5, torch.randn(Np, generator=g)
    x = torch.randn(M, K, generator=g).cuda()
    w, b = wp[:N].clone().cuda(), bp[:N].clone().cuda()
    wp, bp = wp.cuda(), bp.cuda()
    xw = x.double() @ w.double().t()
    worst = {}
    for prec, presplit in COL_CALLS:
        fs, _ = _operands(L, w, prec, presplit)
        fsp, _ = _operands(L, wp, prec, presplit)
        for bias, biasp, relu in ((b, bp, 0), (b, bp, 1), (None, None, 1)):
            outs = []
            for n, ww, wsplit, bb in ((N, w, fs, bias), (Np, wp, fsp, biasp)):
                splits = _tc_split(M, n, K, sms, relu=bool(relu)) if prec in (TF32, TF32X3) else 1
                y = Banded((M, n))
                n0 = _launches(L)
                L.check(lib.b200asr_linear_fwd(L.ptr(x), L.ptr(ww), L.ptr(bb), L.ptr(y.t), M, n, K, relu, prec, L.ptr(wsplit), st), "fwd")
                assert _launches(L) - n0 == (2 if splits > 1 else 1), (prec, n)
                assert y.bands_intact()
                outs.append((y.t, splits))
            (y, s), (yp, sp) = outs
            what = (prec, presplit, bias is not None, relu)
            assert s == sp, what
            assert _same_bits(y, yp[:, :N]), what
            ref = xw + b.double() if bias is not None else xw
            err = rel_err(y, ref.relu() if relu else ref)
            assert err < _bar(prec, "fwd", s > 1), (what, err)
            worst[prec] = max(worst.get(prec, 0.0), err)
    print(f"[columns] {M}x{N}x{K}: float64 rel err " + " ".join(f"p{p} {e:.2e}" for p, e in worst.items()))
