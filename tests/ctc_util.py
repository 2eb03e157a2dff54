"""The CTC loss of utils/metrics.py:133-154 restated in float64 on the CPU, and tests/golden/ctc.npz
(tests/golden/make_ctc_golden.py: the reference's calculate_metrics(..., loss_type="ctc"))."""
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ctc.npz")


def ctc_float64(pred, gold, input_lengths, target_lengths):
    """(nll [B], mean loss, d loss / d pred [B, T, V]) in float64 on the CPU, restated from the definition: the alpha
    recursion over the extended labels (blank, l_1, blank, ..., blank; the skip where l'(s) != l'(s - 2)) on
    log_softmax(pred), nll_b = -log P, loss = mean_b(nll_b / max(L_b, 1)), and the gradient by autograd through the
    recursion -- the exact derivative.  An utterance with no alignment gets nll = +inf and NaN gradient rows t < T_b; rows
    t >= T_b get 0.  torch's CPU ctc_loss agrees with this everywhere except `cpu_backward_differs` below."""
    x = pred.detach().cpu().double().requires_grad_(True)
    il = [int(v) for v in torch.as_tensor(input_lengths).reshape(-1)]
    tl = [int(v) for v in torch.as_tensor(target_lengths).reshape(-1)]
    B = x.shape[0]
    neg = -1e300                                       # a finite -inf: autograd through logsumexp stays NaN-free
    nlls, total = [], x.new_zeros(())
    for b in range(B):
        Tb, Lb = il[b], tl[b]
        if Tb == 0:
            nlls.append(x.new_zeros(()) if Lb == 0 else x.new_full((), float("inf")))
            continue
        lab = [0] * (2 * Lb + 1)
        for i in range(Lb):
            lab[2 * i + 1] = int(gold[b, i])
        Sb = len(lab)
        lp = torch.log_softmax(x[b, :Tb], dim=1)[:, lab]                    # [Tb, Sb]
        skip = torch.tensor([s % 2 == 1 and s >= 3 and lab[s] != lab[s - 2] for s in range(Sb)])
        a = torch.cat([lp[0, :min(2, Sb)], x.new_full((Sb - min(2, Sb),), neg)])
        for t in range(1, Tb):
            a1 = torch.cat([x.new_full((1,), neg), a[:-1]])
            a2 = torch.where(skip, torch.cat([x.new_full((2,), neg), a[:-2]])[:Sb], x.new_full((Sb,), neg))
            a = torch.logsumexp(torch.stack([a, a1, a2]), 0) + lp[t]
        nll = -torch.logsumexp(a[-2:] if Sb >= 2 else a, 0)
        if nll.item() > 1e200:                                               # no alignment fits
            nll = x.new_full((), float("inf"))
        else:
            total = total + nll / max(Lb, 1)
        nlls.append(nll)
    nll = torch.stack([n.detach() for n in nlls])
    loss = (nll / torch.tensor(tl, dtype=torch.float64).clamp_min(1)).mean()
    total = total / B
    grad = torch.autograd.grad(total, x, allow_unused=True)[0] if total.requires_grad else None
    grad = torch.zeros_like(x) if grad is None else grad.clone()
    for b in range(B):
        if torch.isinf(nll[b]):
            grad[b, :il[b]] = float("nan")
    return nll, loss, grad


def _log_softmax64(x):
    x = np.asarray(x, dtype=np.float64)
    m = x.max(axis=-1, keepdims=True)
    return (x - m) - np.log(np.exp(x - m).sum(axis=-1, keepdims=True))


def _shift(a, k):
    """a[s - k] (k > 0) or a[s + |k|] (k < 0), -inf where that index is outside a."""
    out = np.full_like(a, -np.inf)
    if k > 0:
        out[k:] = a[:-k]
    else:
        out[:k] = a[-k:]
    return out


def ctc_float64_fb(pred, gold, input_lengths, target_lengths, dloss=1.0):
    """(nll [B], mean loss, d loss / d pred [B, T, V]) in float64, the same quantities and conventions as `ctc_float64`
    (infeasible: nll +inf and NaN rows t < T_b; rows t >= T_b are 0), from the forward-backward recursions in log space,
    vectorised over the states of each step: alpha and beta over the extended labels l', gamma_t(s) = exp(alpha_t(s) +
    beta_t(s) - lp'_t(s) + nll_b), and dz_t = g_b (softmax_t - sum over s with l'(s) = v of gamma_t(s)) with g_b = dloss /
    (B max(L_b, 1)).  Memory is one [T_b, 2 L_b + 1] float64 array per utterance, so 4095 labels over 8200 frames take
    about 0.5 GB and a few seconds."""
    x = pred.detach().cpu().double().numpy() if torch.is_tensor(pred) else np.asarray(pred, dtype=np.float64)
    gold = np.asarray(gold.cpu() if torch.is_tensor(gold) else gold)
    il = [int(v) for v in np.asarray(input_lengths).reshape(-1)]
    tl = [int(v) for v in np.asarray(target_lengths).reshape(-1)]
    B, T, V = x.shape
    nll = np.zeros(B)
    grad = np.zeros((B, T, V))
    for b in range(B):
        Tb, Lb = il[b], tl[b]
        if Tb == 0:
            nll[b] = 0.0 if Lb == 0 else np.inf
            continue
        lab = np.zeros(2 * Lb + 1, dtype=np.int64)
        lab[1::2] = gold[b, :Lb]
        Sb = lab.size
        ls = _log_softmax64(x[b, :Tb])                                        # [Tb, V]
        rep = np.zeros(Sb, dtype=bool)                                        # l'(s) == l'(s - 2) for odd s >= 3
        rep[3::2] = lab[3::2] == lab[1:-2:2]
        skip_a = np.zeros(Sb, dtype=bool)
        skip_a[3::2] = ~rep[3::2]                                             # the skip into s
        skip_b = np.zeros(Sb, dtype=bool)
        skip_b[1:-2:2] = ~rep[3::2]                                           # the skip out of s
        alpha = np.empty((Tb, Sb))
        a = np.full(Sb, -np.inf)
        a[:2] = ls[0, lab[:2]]
        alpha[0] = a
        for t in range(1, Tb):
            a = np.logaddexp(np.logaddexp(a, _shift(a, 1)), np.where(skip_a, _shift(a, 2), -np.inf)) + ls[t, lab]
            alpha[t] = a
        lp_end = np.logaddexp(a[-1], a[-2]) if Sb >= 2 else a[-1]
        if not np.isfinite(lp_end):
            nll[b] = np.inf
            grad[b, :Tb] = np.nan
            continue
        nll[b] = -lp_end
        # beta from the last frame down; alpha[t] becomes log gamma_t in place (beta_t is not kept)
        bt = np.full(Sb, -np.inf)
        bt[-2:] = ls[Tb - 1, lab[-2:]] if Sb >= 2 else ls[Tb - 1, lab]
        alpha[Tb - 1] += bt - ls[Tb - 1, lab] + nll[b]
        for t in range(Tb - 2, -1, -1):
            lpt = ls[t, lab]
            bt = np.logaddexp(np.logaddexp(bt, _shift(bt, -1)), np.where(skip_b, _shift(bt, -2), -np.inf)) + lpt
            alpha[t] += bt - lpt + nll[b]
        g = dloss / (B * max(Lb, 1))
        onehot = np.zeros((Sb, V))                                            # state -> symbol
        onehot[np.arange(Sb), lab] = 1.0
        for c0 in range(0, Tb, 1024):                                         # gamma summed per symbol, 1024 rows at a time
            c1 = min(Tb, c0 + 1024)
            grad[b, c0:c1] = g * (np.exp(ls[c0:c1]) - np.exp(alpha[c0:c1]) @ onehot)
    loss = float(np.mean(nll / np.maximum(np.asarray(tl, dtype=np.float64), 1.0)))
    return torch.from_numpy(nll), torch.tensor(loss, dtype=torch.float64), torch.from_numpy(grad)


def repeats(y):
    """r: the number of adjacent equal labels of target y, so that L + r is the fewest frames that align y."""
    return sum(int(y[i]) == int(y[i + 1]) for i in range(len(y) - 1))


def ctc_unique_path(pred, gold, input_lengths, target_lengths, dloss=1.0):
    """(nll [B], mean loss, d loss / d pred [B, T, V]) in float64 for batches where every utterance has exactly one
    alignment: a target without the label 0 and T_b = L_b + r_b frames (r_b = repeats(target)).  The alignment emits
    each label once and a blank between equal neighbours, so nll_b = -sum_t log softmax_t(pi_t) and dz_t = g_b (softmax_t -
    onehot(pi_t)) -- no recursion at all."""
    x = pred.detach().cpu().double().numpy() if torch.is_tensor(pred) else np.asarray(pred, dtype=np.float64)
    il = [int(v) for v in np.asarray(input_lengths).reshape(-1)]
    tl = [int(v) for v in np.asarray(target_lengths).reshape(-1)]
    B, T, V = x.shape
    nll = np.zeros(B)
    grad = np.zeros((B, T, V))
    for b in range(B):
        y = [int(v) for v in gold[b, :tl[b]]]
        assert 0 not in y and il[b] == len(y) + repeats(y), "not a single-alignment utterance"
        path = []
        for i, v in enumerate(y):
            if i and v == y[i - 1]:
                path.append(0)
            path.append(v)
        Tb = il[b]
        if Tb == 0:
            continue
        ls = _log_softmax64(x[b, :Tb])
        nll[b] = -ls[np.arange(Tb), path].sum()
        d = np.exp(ls)
        d[np.arange(Tb), path] -= 1.0
        grad[b, :Tb] = dloss / (B * max(tl[b], 1)) * d
    loss = float(np.mean(nll / np.maximum(np.asarray(tl, dtype=np.float64), 1.0)))
    return torch.from_numpy(nll), torch.tensor(loss, dtype=torch.float64), torch.from_numpy(grad)


def cpu_backward_differs(gold, input_lengths, target_lengths):
    """[(b, t)]: the rows where torch's CPU ctc_loss backward is not the derivative.  When an utterance's last label is the
    blank 0, at its last frame t = T_b - 1 torch's CPU kernel assigns the blank's occupation from state 2 L_b - 1 over the
    one from state 2 L_b instead of adding the two (aten/src/ATen/native/LossCTC.cpp initialises the last frame assuming the
    last label differs from the blank), so that row of its gradient misses one term.  torch's CUDA kernel adds them."""
    il = torch.as_tensor(input_lengths).reshape(-1).tolist()
    tl = torch.as_tensor(target_lengths).reshape(-1).tolist()
    return [(b, il[b] - 1) for b in range(len(il)) if tl[b] > 0 and il[b] > 0 and int(gold[b, tl[b] - 1]) == 0]


def load_ctc_golden():
    """{case name: dict(pred, gold, percentages, sizes, target_lengths, loss, grad)} as tensors."""
    z = np.load(GOLDEN)
    out = {}
    for name in z["meta.cases"]:
        name = str(name)
        out[name] = {k: torch.from_numpy(np.array(z[f"{name}.{k}"]))
                     for k in ("pred", "gold", "percentages", "sizes", "target_lengths", "loss", "grad")}
    return out
