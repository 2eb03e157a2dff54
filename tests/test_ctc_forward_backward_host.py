"""CPU check of the two float64 CTC references that scale to the kernels' 4095 labels (tests/ctc_util.py), which the GPU
width tests compare against:

  * `ctc_float64_fb`, the vectorised forward-backward, against `ctc_float64` (autograd through the alpha recursion) and
    against torch's float64 CPU F.ctc_loss: on tests/golden/ctc.npz, on random batches with adjacent repeats, the label 0,
    empty targets, utterances without frames, input lengths below T and infeasible utterances, on peaky logits (one symbol
    per frame +10, +30 or +80 over the rest), and with dloss != 1.  torch's gradient is left out on the rows of
    `cpu_backward_differs`.
  * `ctc_unique_path`, the closed form for T_b = L_b + r_b frames, against both.
  * At 4095 labels (the kernels' largest lattice) `ctc_float64_fb` agrees with the closed form, and over 8200 frames its
    gradient rows sum to 0; the time per utterance is printed (seconds).
"""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.ctc_util import (cpu_backward_differs, ctc_float64, ctc_float64_fb, ctc_unique_path, load_ctc_golden,
                            repeats)


def _torch_ctc(pred, gold, il, tl, dloss=1.0):
    """float64 F.ctc_loss on the CPU, reduction="mean" as utils/metrics.py uses it: (loss, d loss / d pred)."""
    x = pred.detach().double().clone().requires_grad_(True)
    loss = F.ctc_loss(F.log_softmax(x.transpose(0, 1), 2), gold, torch.as_tensor(il), torch.as_tensor(tl), blank=0,
                      reduction="mean", zero_infinity=False)
    (loss * dloss).backward()
    return loss.detach(), x.grad


def _amax(t):
    return float(t.abs().max()) if t.numel() else 0.0


def _check(pred, gold, il, tl, dloss=1.0, unique=False):
    nll, loss, grad = ctc_float64_fb(pred, gold, il, tl, dloss)
    nll_a, loss_a, grad_a = ctc_float64(pred, gold, il, tl)
    grad_a = grad_a * dloss
    fin = torch.isfinite(nll_a)
    assert torch.equal(torch.isfinite(nll), fin) and (nll[~fin] == nll_a[~fin]).all()
    assert _amax((nll - nll_a)[fin]) <= 1e-11 * max(1.0, _amax(nll_a[fin]))
    assert torch.equal(torch.isnan(grad), torch.isnan(grad_a))
    ok = ~torch.isnan(grad_a)
    assert _amax((grad - grad_a)[ok]) <= 1e-12
    for b, Tb in enumerate(torch.as_tensor(il).tolist()):
        assert (grad[b, Tb:] == 0).all()
    if torch.isfinite(loss_a):
        assert abs(float(loss) - float(loss_a)) <= 1e-12 * max(1.0, abs(float(loss_a)))
        lt, gt = _torch_ctc(pred, gold, il, tl, dloss)
        assert abs(float(loss) - float(lt)) <= 1e-12 * max(1.0, abs(float(lt)))
        keep = torch.ones_like(grad, dtype=torch.bool)
        for b, t in cpu_backward_differs(gold, il, tl):
            keep[b, t] = False
        assert float((grad - gt)[keep].abs().max()) <= 1e-12
    else:
        assert torch.isinf(loss) and loss > 0
    if unique:
        nll_u, loss_u, grad_u = ctc_unique_path(pred, gold, il, tl, dloss)
        assert float((nll_u - nll).abs().max()) <= 1e-11 * max(1.0, float(nll.abs().max()))
        assert float((grad_u - grad).abs().max()) <= 1e-12
        assert abs(float(loss_u) - float(loss)) <= 1e-11 * max(1.0, abs(float(loss)))


def _random_batch(seed, T, V, B=7, infeasible=False, peak=None):
    """Targets with adjacent repeats and the label 0, an empty target, an utterance without frames, input lengths below T;
    peak: logits N(0, 1) plus `peak` on one symbol per frame along a random alignment."""
    rng = np.random.default_rng(seed)
    il = [T, T - 1, T // 2, T, 0, max(1, T - 3), T][:B]
    ys = []
    for b in range(B):
        cap = (il[b] + 1) // 2
        L = 0 if b == 3 or cap == 0 else int(rng.integers(1, cap + 1))
        y = [int(v) for v in rng.integers(1, V, L)] if V > 1 else [0] * L
        if L >= 2 and b in (1, 5):
            y[1] = y[0]
        if L >= 1 and b == 2:
            y[L // 2] = 0
        ys.append(y)
    if infeasible:
        ys[6] = [1] * (il[6] + 1)
    tl = [len(y) for y in ys]
    S = max(tl) + 2
    gold = torch.full((B, S), V + 3, dtype=torch.int64)
    for b, y in enumerate(ys):
        gold[b, :len(y)] = torch.tensor(y, dtype=torch.int64)
    pred = torch.randn(B, T, V, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * 2.0
    if peak is not None:
        pred = pred / 2.0
        for b in range(B):
            pred[b, torch.arange(T), torch.as_tensor(rng.integers(0, V, T))] += peak
    return pred.float().double(), gold, torch.tensor(il, dtype=torch.int32), torch.tensor(tl, dtype=torch.int32)


@pytest.mark.parametrize("case", ["feasible", "repeats", "blank_label", "empty_target", "no_frames", "infeasible", "short_inputs"])
def test_fb_matches_autograd_and_torch_on_golden(case):
    c = load_ctc_golden()[case]
    _check(c["pred"], c["gold"], c["sizes"], c["target_lengths"])
    _, loss, grad = ctc_float64_fb(c["pred"], c["gold"], c["sizes"], c["target_lengths"])
    keep = ~torch.isnan(c["grad"])
    for b, t in cpu_backward_differs(c["gold"], c["sizes"], c["target_lengths"]):
        keep[b, t] = False
    assert float((grad - c["grad"])[keep].abs().max()) <= 1e-12
    assert float(loss) == pytest.approx(float(c["loss"]), rel=1e-12) if torch.isfinite(c["loss"]) else torch.isinf(loss)


@pytest.mark.parametrize("T,V,seed", [(1, 5, 0), (2, 5, 1), (17, 32, 2), (40, 5, 3), (60, 32, 4)])
def test_fb_matches_autograd_and_torch_on_random_batches(T, V, seed):
    _check(*_random_batch(seed, T, V))
    _check(*_random_batch(seed + 50, T, V, infeasible=True))


@pytest.mark.parametrize("peak", [10.0, 30.0, 80.0])
def test_fb_matches_autograd_and_torch_on_peaky_logits(peak):
    _check(*_random_batch(7, 40, 6, peak=peak))


def test_fb_scales_dloss():
    _check(*_random_batch(9, 30, 5), dloss=-2.75)


def test_fb_on_the_empty_vocabulary():
    """V = 1: the blank is every symbol; targets of label 0 only."""
    pred = torch.randn(3, 9, 1, dtype=torch.float64)
    gold = torch.tensor([[0, 0, 3], [0, 3, 3], [3, 3, 3]])
    _check(pred, gold, torch.tensor([9, 5, 7]), torch.tensor([2, 1, 0]))


def _unique_batch(seed, lens, V):
    """Targets without the label 0, with adjacent repeats, and T_b = L_b + r_b: exactly one alignment each."""
    rng = np.random.default_rng(seed)
    ys = []
    for L in lens:
        y = [int(v) for v in rng.integers(1, V, L)]
        for i in range(1, L, 5):
            y[i] = y[i - 1]
        ys.append(y)
    il = [len(y) + repeats(y) for y in ys]
    T = max(il) + 2
    S = max(lens) + 1
    gold = torch.full((len(lens), S), V + 1, dtype=torch.int64)
    for b, y in enumerate(ys):
        gold[b, :len(y)] = torch.tensor(y, dtype=torch.int64)
    pred = torch.randn(len(lens), T, V, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * 2.0
    return pred, gold, torch.tensor(il, dtype=torch.int32), torch.tensor(lens, dtype=torch.int32)


@pytest.mark.parametrize("V", [2, 5, 40])
def test_unique_path_matches_both_references(V):
    _check(*_unique_batch(V, [1, 3, 7, 12, 0], V), unique=True)
    _check(*_unique_batch(V + 1, [6, 11], V), dloss=0.5, unique=True)


def test_fb_at_4095_labels_and_8200_frames_is_fast_and_exact():
    """The largest lattice the kernels take: 4095 labels at T_b = L + r against the closed form, and the same target over
    8200 frames, where every gradient row sums to 0 (softmax and the occupations each sum to 1 per frame)."""
    pred, gold, il, tl = _unique_batch(3, [4095], 32)
    t0 = time.perf_counter()
    nll, _, grad = ctc_float64_fb(pred, gold, il, tl)
    dt = time.perf_counter() - t0
    nll_u, _, grad_u = ctc_unique_path(pred, gold, il, tl)
    assert abs(float(nll[0] - nll_u[0])) <= 1e-11 * float(nll_u[0].abs())
    assert float((grad - grad_u).abs().max()) <= 1e-12
    T = 8200
    x = torch.randn(1, T, 32, generator=torch.Generator().manual_seed(4), dtype=torch.float64) * 2.0
    t0 = time.perf_counter()
    nll2, _, grad2 = ctc_float64_fb(x, gold, torch.tensor([T]), tl)
    dt = max(dt, time.perf_counter() - t0)
    print(f"ctc_float64_fb at L = 4095: {dt:.1f} s per utterance")
    assert torch.isfinite(nll2).all()
    g = 1.0 / 4095
    assert float((grad2[0] / g).sum(dim=1).abs().max()) <= 1e-9               # softmax and gamma both sum to 1 per frame
