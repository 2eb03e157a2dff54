#!/usr/bin/env python
"""Forward + backward time of the CTC loss: b200asr (metrics.calculate_loss(loss_type="ctc") -> csrc/ctc.cu) against the
reference's own expression F.ctc_loss(F.log_softmax(pred.transpose(0, 1), 2), gold, sizes, target_lengths) on the same GPU.

    python tools/ctc_time.py [--iters 50] [--warmup 10]

Shapes: cfg2's decoder output (B = 32, T = 100, V = 4364) and the reference's default --tgt-max-len (T = 1000), target
lengths 40 .. 99 without equal neighbours (every alignment fits), CPU int32 lengths as the trainer passes them.  Each leg is
timed with CUDA events around `iters` forward + backward calls after `warmup` untimed ones; the two legs alternate over
three rounds and the median round is reported.  Also printed: the card, its power limit and max SM clock (read in the same
run), and the largest loss and gradient differences between the two (relative to the largest gradient entry).
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200asr  # noqa: E402

metrics = importlib.import_module(b200asr.__name__ + ".metrics")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def batch(B, T, V, seed):
    g = torch.Generator().manual_seed(seed)
    tl = torch.randint(40, 100, (B,), generator=g, dtype=torch.int32)
    il = torch.full((B,), T, dtype=torch.int32) if T <= 100 else torch.randint(T // 2, T + 1, (B,), generator=g, dtype=torch.int32)
    S = int(tl.max())
    gold = torch.zeros(B, S, dtype=torch.int64)
    for b in range(B):
        prev = -1
        for j in range(int(tl[b])):
            v = prev
            while v == prev:
                v = int(torch.randint(1, V, (1,), generator=g))
            gold[b, j] = prev = v
    pred = torch.randn(B, T, V, generator=g) * 2.0
    return pred.cuda().requires_grad_(True), gold.cuda(), il, tl


def ours(pred, gold, il, tl):
    loss = metrics.calculate_loss(pred, gold, il, tl, loss_type="ctc")
    return loss, torch.autograd.grad(loss, pred)[0]


def reference(pred, gold, il, tl):
    loss = F.ctc_loss(F.log_softmax(pred.transpose(0, 1), dim=2), gold, il, tl, reduction="mean")
    return loss, torch.autograd.grad(loss, pred)[0]


def time_leg(fn, args, iters, warmup):
    for _ in range(warmup):
        fn(*args)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn(*args)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ctc_time.py measures on the GPU; no CUDA device found")
    b200asr._lib.load(check_device=True)
    print("gpu:", gpu_info(), flush=True)
    for name, (B, T, V) in (("cfg2", (32, 100, 4364)), ("T1000", (32, 1000, 4364))):
        data = batch(B, T, V, seed=T)
        l_o, g_o = ours(*data)
        l_r, g_r = reference(*data)
        d_loss = abs(float(l_o.detach()) - float(l_r.detach())) / abs(float(l_r.detach()))
        d_grad = float((g_o - g_r).abs().max()) / float(g_r.abs().max())
        rounds = {"ours": [], "reference": []}
        for _ in range(3):
            rounds["ours"].append(time_leg(ours, data, args.iters, args.warmup))
            rounds["reference"].append(time_leg(reference, data, args.iters, args.warmup))
        med = {k: sorted(v)[1] for k, v in rounds.items()}
        out = dict(shape=name, B=B, T=T, V=V, S=int(data[1].shape[1]), ours_ms=round(med["ours"], 4),
                   reference_ms=round(med["reference"], 4), speedup=round(med["reference"] / med["ours"], 2),
                   rounds_ms={k: [round(x, 4) for x in v] for k, v in rounds.items()}, loss_ours=float(l_o.detach()),
                   loss_rel_diff=d_loss, grad_max_diff_rel=d_grad)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
