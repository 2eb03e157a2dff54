"""Mirror of utils/metrics.py:78-154 (calculate_metrics / calculate_loss, CE and CTC branches) on the fused CE kernel and the
CTC kernels."""
from __future__ import annotations

import torch

from . import ops


def loss_and_stats(pred, gold, smoothing=0.0, reduction="mean"):
    """(loss, stats) without any host synchronisation.  stats = [sum, n_tokens, n_correct, mean, 1/n_tokens]."""
    return ops.CrossEntropyFn.apply(pred, gold, float(smoothing), reduction)


def calculate_loss(pred, gold, input_lengths=None, target_lengths=None, smoothing=0.0, loss_type="ce"):
    """utils/metrics.py:102-154.  "ce": label-smoothed CE / CE over the non-PAD tokens.  "ctc": F.ctc_loss of
    log_softmax(pred) with blank 0 and the mean reduction, `smoothing` ignored, as the reference (ops.CtcLossFn)."""
    if loss_type == "ce":
        loss, _ = loss_and_stats(pred, gold, smoothing)
        return loss
    if loss_type == "ctc":
        return ops.CtcLossFn.apply(pred, gold, input_lengths, target_lengths)
    raise NotImplementedError(f"b200asr implements the 'ce' and 'ctc' losses only, not {loss_type!r}")


def calculate_metrics(pred, gold, input_lengths=None, target_lengths=None, smoothing=0.0, loss_type="ce"):
    """utils/metrics.py:78-99 -> (loss, num_correct).  For "ce", num_correct is a Python int as in the reference (one D2H
    sync, the reference has the same at :94); use loss_and_stats() to stay asynchronous.  For "ctc" it is None (:96-97)."""
    if loss_type == "ctc":
        return calculate_loss(pred, gold, input_lengths, target_lengths, smoothing, loss_type), None
    if loss_type != "ce":
        raise NotImplementedError(f"b200asr implements the 'ce' and 'ctc' losses only, not {loss_type!r}")
    loss, stats = loss_and_stats(pred, gold, smoothing)
    return loss, int(stats[2].item())
