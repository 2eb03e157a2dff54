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
