"""CTC loss on the device (csrc/ctc.cu, ops.CtcLossFn, metrics.calculate_loss(loss_type="ctc")).

  * b200asr_ctc_fwd / _bwd against float64 F.ctc_loss on the CPU (tests/ctc_util.py): per-utterance nll, the mean loss and
    the logit gradient in the max norm at T in {1, 2, 17, 100, 1000} x V in {5, 32, 4364}, on batches that hold repeated
    labels, a target label 0, an empty target, an utterance without frames and input lengths below T; logits also shifted
    by +200; outputs and workspace NaN-poisoned, so every element checked was written.  Infeasible utterances: inf nll, NaN
    gradient rows t < T_b and zero rows t >= T_b.  Target entries past target_lengths[b] are out of range: reading one
    would make the result NaN.
  * Two calls give identical bits.
  * tests/golden/ctc.npz (the reference's calculate_metrics(..., loss_type="ctc")) through metrics.calculate_metrics; on the
    rows where torch's CPU backward is not the derivative (ctc_util.cpu_backward_differs) against torch's CUDA ctc_loss.
  * calculate_loss + backward with CPU int32 lengths under torch.cuda.set_sync_debug_mode("error").
  * Rejections: lengths > T, target lengths > S, negative lengths, CPU logits.
  * The reference's Trainer.train with --loss ctc for one epoch, eager and installed, with an infeasible training batch.

tests/test_gpu_ctc_widths.py covers the rest of the kernels, on guarded buffers against the float64 forward-backward of
tests/ctc_util.py: every recursion width K = 1 .. 32 (targets up to 4095 labels, the shared-memory opt-in at K = 32) on both
sides of each boundary, trained-model logits (sigma up to 30, forced alignments +80 over the rest) at T up to 8200, the
feasibility boundary T_b = L_b + r_b against the closed-form single alignment, all-empty batches and V = 1, bitwise
independence of the utterances at B = 257, dloss != 1 through ops, the 4095-label limit, and NaN results for lengths that
break the contract on the device.
"""
import copy
import importlib
import os
import tempfile

import numpy as np
import pytest
import torch

import b200asr
from b200asr import _lib as L
from oracle import ref_shim
from tests.ctc_util import cpu_backward_differs, ctc_float64, load_ctc_golden

pytestmark = pytest.mark.gpu
ops = importlib.import_module(b200asr.__name__ + ".ops")
metrics = importlib.import_module(b200asr.__name__ + ".metrics")

# Bounds from the float64 comparison on an H100 (largest over every case below, logits shifted or not: nll / loss 1.1e-7,
# gradient 1.9e-7 -- the per-step rescaling keeps the lattices near 0, so T = 1000 is no worse than T = 2):
NLL_RTOL = 1e-6          # |nll - nll64| / max(1, |nll64|), also for the mean loss
GRAD_RTOL = 2e-6         # max |dz - dz64| / max |dz64| over the finite entries of a batch


def _batch(T, V, seed, infeasible=False):
    """B = 6 utterances covering the edges; targets padded with V + 7 (out of range) past each target length."""
    rng = np.random.default_rng(seed)
    Tb = [T, max(1, (2 * T) // 3), T, T // 2, 0, max(1, T - 1 - T // 5)]
    tl = []
    ys = []
    for b in range(6):
        if b in (3, 4):
            y = []
        else:
            cap = (Tb[b] + 1) // 2                                           # L + repeats <= 2L - 1 <= T_b
            L_ = int(rng.integers(max(1, cap // 2), cap + 1)) if cap >= 1 else 0
            y = list(rng.integers(1, V, L_))
            if b == 1 and L_ >= 2:
                y[1] = y[0]                                                  # a repeated label
            if b == 2 and L_ >= 1:
                y[L_ // 2] = 0                                               # the blank as a label
        ys.append(y)
        tl.append(len(y))
    if infeasible:
        Tb[5] = max(1, Tb[5])
        ys[5] = [1] * (Tb[5] + 1)                                            # more labels than frames
        tl[5] = len(ys[5])
    S = max(tl) + 2
    gold = torch.full((6, S), V + 7, dtype=torch.int64)
    for b, y in enumerate(ys):
        if y:
            gold[b, :len(y)] = torch.tensor(y, dtype=torch.int64)
    pred = torch.randn(6, T, V, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * 2.0
    return pred, gold, torch.tensor(Tb, dtype=torch.int32), torch.tensor(tl, dtype=torch.int32)


def _run(x, gold, il, tl, poison=True):
    """(nll, loss, dz) from the C ABI with NaN-poisoned outputs and workspace."""
    B, T, V = x.shape
    S = gold.shape[1]
    lmax = int(tl.max())
    lib = L.load()
    dev = x.device
    g, ild, tld = gold.to(dev), il.to(dev), tl.to(dev)
    ws = torch.empty(lib.b200asr_ctc_ws_bytes(B, T, lmax), device=dev, dtype=torch.uint8)
    nll = torch.empty(B, device=dev)
    loss = torch.empty((), device=dev)
    dz = torch.empty_like(x)
    if poison:
        for t in (ws.view(torch.float32)[:ws.numel() // 4], nll, loss, dz):
            t.fill_(float("nan"))
    dloss = torch.ones((), device=dev)
    st = torch.cuda.current_stream().cuda_stream
    L.check(lib.b200asr_ctc_fwd(L.ptr(x), L.ptr(g), L.ptr(ild), L.ptr(tld), L.ptr(nll), L.ptr(loss), L.ptr(ws), B, T, V, S, lmax,
                                st), "ctc_fwd")
    L.check(lib.b200asr_ctc_bwd(L.ptr(x), L.ptr(g), L.ptr(ild), L.ptr(tld), L.ptr(nll), L.ptr(dloss), L.ptr(dz), L.ptr(ws), B, T,
                                V, S, lmax, st), "ctc_bwd")
    torch.cuda.synchronize()
    return nll.cpu(), loss.cpu(), dz.cpu()


def _compare(nll, loss, dz, ref, il, what):
    nll64, loss64, dz64 = ref
    fin = torch.isfinite(nll64)
    assert torch.equal(torch.isfinite(nll), fin), (what, nll, nll64)
    assert (nll[~fin] == nll64[~fin]).all(), what                            # +inf
    e_nll = float(((nll.double() - nll64).abs() / nll64.abs().clamp_min(1.0))[fin].max()) if fin.any() else 0.0
    if torch.isfinite(loss64):
        e_loss = abs(float(loss) - float(loss64)) / max(1.0, abs(float(loss64)))
    else:
        assert float(loss) == float(loss64), what
        e_loss = 0.0
    nan = torch.isnan(dz64)
    assert torch.equal(torch.isnan(dz), nan), what
    for b, Tb in enumerate(il.tolist()):                                     # NaN exactly on the infeasible rows t < T_b
        assert (dz[b, Tb:] == 0).all(), what
        assert bool(nan[b, :Tb].all()) if not fin[b] else not bool(nan[b].any()), what
    scale = float(dz64[~nan].abs().max()) if (~nan).any() else 1.0
    e_grad = float((dz.double() - dz64)[~nan].abs().max()) / scale if (~nan).any() else 0.0
    print(f"{what}: nll {e_nll:.2e} loss {e_loss:.2e} grad {e_grad:.2e}")
    assert e_nll <= NLL_RTOL and e_loss <= NLL_RTOL and e_grad <= GRAD_RTOL, (what, e_nll, e_loss, e_grad)


@pytest.mark.parametrize("V", [5, 32, 4364])
@pytest.mark.parametrize("T", [1, 2, 17, 100, 1000])
def test_kernels_match_float64(T, V):
    pred, gold, il, tl = _batch(T, V, seed=T * 7 + V)
    for shift in (0.0, 200.0):
        x = (pred + shift).float().cuda()
        nll, loss, dz = _run(x, gold, il, tl)
        # the float64 reference sees the same fp32 logits (x - 200 is exact; log_softmax drops the shift)
        _compare(nll, loss, dz, ctc_float64(x.cpu() - shift, gold, il, tl), il, f"T={T} V={V} shift={shift}")


@pytest.mark.parametrize("T,V", [(2, 5), (17, 32), (100, 4364)])
def test_infeasible_utterance_gives_inf_and_nan_rows(T, V):
    pred, gold, il, tl = _batch(T, V, seed=5 + T, infeasible=True)
    x = pred.float().cuda()
    nll, loss, dz = _run(x, gold, il, tl)
    assert torch.isinf(nll[5]) and torch.isinf(loss)
    _compare(nll, loss, dz, ctc_float64(x.cpu(), gold, il, tl), il, f"infeasible T={T} V={V}")


def test_two_calls_give_identical_bits():
    pred, gold, il, tl = _batch(100, 4364, seed=3)
    x = pred.float().cuda()
    a, b = _run(x, gold, il, tl), _run(x, gold, il, tl, poison=False)
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.int32), v.view(torch.int32))


@pytest.fixture(scope="module")
def golden():
    return load_ctc_golden()


@pytest.mark.parametrize("case", ["feasible", "repeats", "blank_label", "empty_target", "no_frames", "infeasible", "short_inputs"])
def test_calculate_metrics_matches_reference_fixture(golden, case):
    c = golden[case]
    pred = c["pred"].float().cuda().requires_grad_(True)
    loss, num_correct = metrics.calculate_metrics(pred, c["gold"].cuda(), input_lengths=c["sizes"],
                                                  target_lengths=c["target_lengths"], smoothing=0.1, loss_type="ctc")
    assert num_correct is None
    loss.backward()
    want, gwant = c["loss"], c["grad"]
    got, grad = loss.detach().cpu().double(), pred.grad.cpu().double()
    if torch.isinf(want):
        assert torch.isinf(got)
    else:
        # the fixture's logits rounded to fp32 move the loss by ~1e-7 relative
        assert abs(float(got) - float(want)) <= 1e-5 * max(1.0, abs(float(want))), (float(got), float(want))
    nan = torch.isnan(gwant)
    assert torch.equal(torch.isnan(grad), nan)
    keep = ~nan
    rows = cpu_backward_differs(c["gold"], c["sizes"], c["target_lengths"])
    for b, t in rows:
        keep[b, t] = False
    if keep.any():
        assert float((grad - gwant)[keep].abs().max()) <= 1e-5 * float(gwant[keep].abs().max())
    if rows:                                        # there: torch's CUDA kernel, which adds both blank terms, in float64
        x = c["pred"].cuda().requires_grad_(True)
        F = torch.nn.functional
        F.ctc_loss(F.log_softmax(x.transpose(0, 1), 2), c["gold"].cuda(), c["sizes"], c["target_lengths"]).backward()
        gc = x.grad.cpu()
        for b, t in rows:
            assert float((grad[b, t] - gc[b, t]).abs().max()) <= 1e-5 * float(gc[b, t].abs().max()), (b, t)


def test_loss_and_backward_do_not_sync_the_host():
    pred, gold, il, tl = _batch(100, 4364, seed=11)
    x = pred.float().cuda().requires_grad_(True)
    g = gold.clamp_max(4363).cuda()
    for _ in range(10):                                                      # pinned staging ring warmed up
        metrics.calculate_loss(x, g, il, tl, loss_type="ctc").backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = metrics.calculate_loss(x, g, il, tl, loss_type="ctc")
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(loss).item()


def test_rejections():
    pred, gold, il, tl = _batch(17, 32, seed=1)
    x, g = pred.float().cuda(), gold.cuda()
    T, S = x.shape[1], g.shape[1]
    bad = il.clone(); bad[0] = T + 1
    with pytest.raises(RuntimeError, match="input_lengths to have value at most"):
        ops.CtcLossFn.apply(x, g, bad, tl)
    bad = tl.clone(); bad[0] = S + 1
    with pytest.raises(RuntimeError, match="target_lengths to have value at most"):
        ops.CtcLossFn.apply(x, g, il, bad)
    for which in (0, 1):
        bad = (il if which == 0 else tl).clone(); bad[1] = -1
        with pytest.raises(RuntimeError, match="non-negative"):
            ops.CtcLossFn.apply(x, g, *((bad, tl) if which == 0 else (il, bad)))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        metrics.calculate_loss(x.cpu(), g, il, tl, loss_type="ctc")
    with pytest.raises(NotImplementedError):
        metrics.calculate_loss(x, g, il, tl, loss_type="l1")
    lib = L.load()
    P = L.ptr
    d = torch.zeros(64, device="cuda")
    # max_target_len above S or above 4095: a shape error before any launch
    assert lib.b200asr_ctc_fwd(P(d), P(d), P(d), P(d), P(d), P(d), P(d), 1, 4, 5, 2, 3, None) == -1
    assert lib.b200asr_ctc_fwd(P(d), P(d), P(d), P(d), P(d), P(d), P(d), 1, 4, 5, 5000, 4096, None) == -1
    assert lib.b200asr_ctc_bwd(P(d), P(d), P(d), P(d), P(d), None, P(d), P(d), 1, 4, 5, 2, 1, None) == -5


# ---------------------------------------------------------------------------------------------- the reference's trainer
def _trainer_batches(ns, freq, T, vocab, Lt, B):
    """_collate_fn-shaped batches (utils/data_loader.py:213) whose CTC alignments all fit, plus one training batch with an
    utterance that has more labels than frames: the decoder's T is max(target length) + 1 and the trainer gives utterance b
    int(percentage_b * T) frames."""
    def one(seed, infeasible=False):
        g = torch.Generator().manual_seed(seed)
        src = torch.randn(B, 1, freq, T, generator=g)
        lens = (T * (0.5 + 0.5 * torch.rand(B, generator=g))).long().clamp(1, T)
        lens[0] = T
        lens = torch.sort(lens, descending=True).values
        for i in range(B):
            src[i, :, :, int(lens[i]):] = 0
        pct = lens.float() / float(T)
        frames = pct.clone().mul_(Lt + 1).int()
        tl = torch.tensor([Lt] + [max(1, min(Lt, int(frames[i]))) for i in range(1, B)], dtype=torch.int32)
        if infeasible:
            tl[B - 1] = int(frames[B - 1]) + 1
            assert tl[B - 1] <= Lt
        tgt = torch.zeros(B, Lt, dtype=torch.int64)
        for i in range(B):                                                   # no two equal neighbours: L frames suffice
            prev = -1
            for j in range(int(tl[i])):
                v = prev
                while v == prev:
                    v = int(torch.randint(3, vocab, (1,), generator=g))
                tgt[i, j] = prev = v
        return (src, tgt, pct, lens.to(torch.int32), tl)
    train = [one(0), one(1, infeasible=True), one(2), one(3)]
    return train, [[one(100)]]


def _run_ctc_trainer(ns, model, l2i, i2l, train, valid, installed, tmp):
    ns.constant.args.save_folder, ns.constant.args.name = tmp, "b200" if installed else "eager"
    opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
    opt.lr, opt.lr_anneal = 0.0, 0.0          # read by the reference's save_model under --loss ctc; NoamOpt has neither
    losses = []
    if installed:
        b200asr.install()
    cur = ns.trainer.calculate_metrics

    def recording(*a, **k):
        out = cur(*a, **k)
        losses.append(float(out[0].item()))
        return out

    ns.trainer.calculate_metrics = recording
    try:
        tr = copy.deepcopy(train), copy.deepcopy(valid)
        ns.trainer.Trainer().train(model, tr[0], None, tr[1], opt, "ctc", 0, 1, l2i, i2l)
    finally:
        ns.trainer.calculate_metrics = cur
        if installed:
            b200asr.uninstall()
    assert os.path.exists(os.path.join(tmp, ns.constant.args.name, "best_model.th"))
    return losses, opt._step, {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items()}


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_reference_trainer_ctc_loop_runs_on_installed_kernels():
    from tests.test_gpu_reference import SMALL_VGG, TOL, _build, _fp32_flags
    vocab, freq, B, T = 40, 41, 4, 32
    _fp32_flags()
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        for installed in (False, True):
            ns, model, l2i, i2l = _build(SMALL_VGG, vocab, extra=["--cuda", "--warmup", "4", "--k-lr", "0.02", "--min-lr", "1e-6",
                                                                  "--clip", "--max-norm", "400", "--loss", "ctc"])
            init = {k: v.detach().float().clone() for k, v in model.state_dict().items()}
            model = model.cuda()
            train, valid = _trainer_batches(ns, freq, T, vocab, ns.constant.args.tgt_max_len - 1, B)
            results[installed] = _run_ctc_trainer(ns, model, l2i, i2l, train, valid, installed, tmp)
    (l_e, n_e, sd_e), (l_b, n_b, sd_b) = results[False], results[True]
    print(f"losses eager {l_e}\nlosses b200  {l_b}")
    assert len(l_e) == len(l_b) == 5                                         # 4 train iterations + 1 validation batch
    assert l_e[1] == l_b[1] == float("inf")                                  # skipped by the trainer's inf check
    assert n_e == n_b == 3                                                   # so the optimizer stepped 3 times
    for a, b in zip(l_e[:1] + l_e[2:], l_b[:1] + l_b[2:]):
        assert abs(a - b) < TOL * abs(a), (l_e, l_b)
    for k in sd_e:
        if k.endswith("positional_encoding.pe") or "num_batches_tracked" in k:
            continue
        d_e, d_b = sd_e[k] - init[k], sd_b[k] - init[k]
        if d_e.numel() < 256:
            continue
        assert float((d_e - d_b).norm() / d_e.norm().clamp_min(1e-30)) < (0.05 if d_e.numel() >= 16384 else 0.15), k
