#!/usr/bin/env python
"""Generate tests/golden/ctc.npz from the UNMODIFIED reference's calculate_metrics(..., loss_type="ctc")
(utils/metrics.py:78-154) in float64 on the CPU.

Needs the reference checkout (found by oracle/ref_shim.py):

    python tests/golden/make_ctc_golden.py

The other fixtures are not touched.  Each case is one batch whose input lengths come from the trainer's own expression
`src_percentages.mul_(int(seq_length)).int()` (trainer/asr/trainer.py:81-82) and covers one edge of torch's CTC loss:
feasible targets without and with repeated labels, a target label equal to the blank 0, an empty target, an utterance with
no frames (and an empty target), an infeasible utterance (too few frames for its labels and repeats: the loss is inf), and
input lengths below T.  Stored per case: pred [B, T, V] float64, gold [B, S] int64, the percentages, the sizes,
target_lengths (int32), the loss and d loss / d pred.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
T, V, S = 12, 7, 6
# name -> (percentages, targets (unpadded))
CASES = {
    "feasible": ([1.0, 0.9, 0.75], [[3, 4, 5, 6], [1, 2, 3], [6, 5, 4, 3, 2]]),
    "repeats": ([1.0, 1.0, 0.9], [[3, 3, 4, 4, 4], [2, 5, 5, 2], [6, 6]]),
    "blank_label": ([1.0, 0.8, 0.95], [[3, 0, 4], [0, 0, 2], [0]]),
    "empty_target": ([1.0, 0.6, 0.5], [[4, 5], [], [1]]),
    "no_frames": ([1.0, 0.0, 0.7], [[2, 3, 2], [], [5, 5]]),
    "infeasible": ([1.0, 0.45, 0.8], [[3, 4], [3, 3, 3, 3], [2, 6, 2]]),
    "short_inputs": ([0.5, 0.34, 0.8], [[1, 6], [4], [3, 5, 5, 3]]),
}


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import ref_shim
    ns = ref_shim.load([])
    import torch
    g = torch.Generator().manual_seed(2024)
    out = {"meta.cases": np.array(list(CASES))}
    for name, (pct, tgts) in CASES.items():
        B = len(pct)
        pred = (2.0 * torch.randn(B, T, V, generator=g, dtype=torch.float64)).requires_grad_(True)
        gold = torch.zeros(B, S, dtype=torch.int64)
        for b, y in enumerate(tgts):
            gold[b, :len(y)] = torch.tensor(y, dtype=torch.int64)
        tgt_lengths = torch.tensor([len(y) for y in tgts], dtype=torch.int32)
        src_percentages = torch.tensor(pct, dtype=torch.float32)             # _collate_fn's FloatTensor
        sizes = src_percentages.clone().mul_(int(pred.size(1))).int()         # trainer.py:81-82
        loss, num_correct = ns.metrics.calculate_metrics(pred, gold, input_lengths=sizes, target_lengths=tgt_lengths,
                                                         smoothing=0.1, loss_type="ctc")
        assert num_correct is None
        loss.backward()
        grad = pred.grad.detach().numpy().copy()
        print(f"{name}: sizes {sizes.tolist()} target lengths {tgt_lengths.tolist()} loss {float(loss.detach()):.6f} "
              f"NaN grad rows {int(np.isnan(grad).any(axis=2).sum())}")
        for k, v in (("pred", pred.detach().numpy()), ("gold", gold.numpy()), ("percentages", src_percentages.numpy()),
                     ("sizes", sizes.numpy()), ("target_lengths", tgt_lengths.numpy()),
                     ("loss", np.array(float(loss.detach()), dtype=np.float64)), ("grad", grad)):
            out[f"{name}.{k}"] = v
    assert np.isinf(out["infeasible.loss"]) and np.isfinite(out["no_frames.loss"])
    path = os.path.join(HERE, "ctc.npz")
    np.savez_compressed(path, **out)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
